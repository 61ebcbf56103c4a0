// touchnet_b200 :: host-side helpers (error string, TMA descriptor encoding, device queries).
#include "host.h"

#include <stdarg.h>
#include <stdio.h>
#include <string.h>

#include <mutex>

#include "../../include/touchnet_b200.h"

namespace tn {

static thread_local char g_err[1024] = {0};

int fail(int code, const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
  return code;
}
void clear_error() { g_err[0] = 0; }

typedef CUresult (*PFN_encodeTiled)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                    const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                    CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static PFN_encodeTiled get_encode() {
  static PFN_encodeTiled fn = nullptr;
  static std::once_flag once;
  std::call_once(once, [] {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult qres;
    cudaError_t e = cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &qres);
    if (e == cudaSuccess && qres == cudaDriverEntryPointSuccess) fn = reinterpret_cast<PFN_encodeTiled>(p);
  });
  return fn;
}

static int encode_nd(CUtensorMap* out, const void* ptr, int elem_bytes, int rank, const uint64_t* dims,
                     const uint64_t* strides_bytes, const uint32_t* box, bool swizzle128) {
  PFN_encodeTiled enc = get_encode();
  if (!enc) return fail(TN_ERR_CUDA, "cuTensorMapEncodeTiled entry point unavailable (no CUDA driver?)");
  if ((reinterpret_cast<uintptr_t>(ptr) & 15u) != 0) return fail(TN_ERR_ARG, "TMA base pointer %p not 16B aligned", ptr);
  cuuint64_t gdim[5];
  cuuint64_t gstr[5];
  cuuint32_t gbox[5];
  cuuint32_t estr[5];
  for (int i = 0; i < rank; ++i) {
    gdim[i] = dims[i];
    gbox[i] = box[i];
    estr[i] = 1;
    if (box[i] == 0 || box[i] > 256) return fail(TN_ERR_ARG, "TMA box dim %d = %u out of range", i, box[i]);
  }
  for (int i = 0; i + 1 < rank; ++i) {
    gstr[i] = strides_bytes[i];
    if (strides_bytes[i] % 16 != 0)
      return fail(TN_ERR_ARG, "TMA stride %d = %llu bytes is not a multiple of 16", i,
                  (unsigned long long)strides_bytes[i]);
  }
  CUtensorMapDataType dt = elem_bytes == 1   ? CU_TENSOR_MAP_DATA_TYPE_UINT8
                           : elem_bytes == 2 ? CU_TENSOR_MAP_DATA_TYPE_BFLOAT16
                                             : CU_TENSOR_MAP_DATA_TYPE_FLOAT32;
  CUresult r = enc(out, dt, rank, const_cast<void*>(ptr), gdim, gstr, gbox, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                   swizzle128 ? CU_TENSOR_MAP_SWIZZLE_128B : CU_TENSOR_MAP_SWIZZLE_NONE,
                   CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS)
    return fail(TN_ERR_CUDA, "cuTensorMapEncodeTiled failed with CUresult %d (rank %d dims %llu,%llu box %u,%u)", (int)r,
                rank, (unsigned long long)dims[0], (unsigned long long)dims[1], box[0], box[1]);
  return TN_OK;
}

int encode_tmap_2d(CUtensorMap* out, const void* ptr, int elem_bytes, uint64_t dim0, uint64_t dim1,
                   uint64_t stride1_bytes, uint32_t box0, uint32_t box1, bool swizzle128) {
  uint64_t dims[2] = {dim0, dim1};
  uint64_t strides[1] = {stride1_bytes};
  uint32_t box[2] = {box0, box1};
  return encode_nd(out, ptr, elem_bytes, 2, dims, strides, box, swizzle128);
}

int encode_tmap_3d(CUtensorMap* out, const void* ptr, int elem_bytes, uint64_t dim0, uint64_t dim1, uint64_t dim2,
                   uint64_t stride1_bytes, uint64_t stride2_bytes, uint32_t box0, uint32_t box1, uint32_t box2,
                   bool swizzle128) {
  uint64_t dims[3] = {dim0, dim1, dim2};
  uint64_t strides[2] = {stride1_bytes, stride2_bytes};
  uint32_t box[3] = {box0, box1, box2};
  return encode_nd(out, ptr, elem_bytes, 3, dims, strides, box, swizzle128);
}

static int g_sm_margin = 0;
static int g_gemm_group = 8;

int gemm_group() { return g_gemm_group; }
void set_gemm_l2_hints(int on);
static int g_gemm_l2_hints = 0;   // opt-in: A strips evict-last, B strips evict-first
int gemm_l2_hints() { return g_gemm_l2_hints; }
void set_gemm_l2_hints(int on) { g_gemm_l2_hints = on ? 1 : 0; }

int sm_count() {
  static int n = 0;
  if (n == 0) {
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess) return 132;
    if (cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess) n = 132;
  }
  const int m = n - g_sm_margin;
  return m < 2 ? 2 : m;
}

}  // namespace tn

extern "C" {

const char* tn_last_error(void) { return tn::g_err; }

int tn_version(void) { return TOUCHNET_B200_VERSION; }

int tn_set_sm_margin(int sms) {
  if (sms < 0 || sms > 120) return tn::fail(tn::TN_ERR_ARG, "tn_set_sm_margin: %d out of range [0,120]", sms);
  tn::g_sm_margin = sms;
  return tn::TN_OK;
}

int tn_set_gemm_group(int m_blocks) {
  if (m_blocks < 1 || m_blocks > 64) return tn::fail(tn::TN_ERR_ARG, "tn_set_gemm_group: %d out of range [1,64]", m_blocks);
  tn::g_gemm_group = m_blocks;
  return tn::TN_OK;
}

int tn_set_gemm_split_tail(int on) {   // accepted for API compatibility: the GEMM has no half-tile tail mode
  (void)on;
  return tn::TN_OK;
}

int tn_set_gemm_l2_hints(int on) {
  tn::set_gemm_l2_hints(on);
  return tn::TN_OK;
}

int tn_device_check(void) {
  int dev = 0;
  cudaError_t e = cudaGetDevice(&dev);
  if (e != cudaSuccess) return tn::fail(tn::TN_ERR_CUDA, "cudaGetDevice: %s", cudaGetErrorString(e));
  int major = 0, minor = 0;
  cudaDeviceGetAttribute(&major, cudaDevAttrComputeCapabilityMajor, dev);
  cudaDeviceGetAttribute(&minor, cudaDevAttrComputeCapabilityMinor, dev);
  if (major != 9 || minor != 0)
    return tn::fail(tn::TN_ERR_UNSUPPORTED, "device is sm_%d%d; this library is built for sm_90a (H100) only", major, minor);
  return tn::TN_OK;
}

}  // extern "C"
