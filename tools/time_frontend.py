"""Time the GPU fbank kernel, the MFCC epilogue (80 mel / 40 ceps) and whisper log-mel (80 and 128 mel) on the same
bench-sized batch (CUDA events) and report achieved algorithmic GB/s (waveform read once, features written once), with
the GPU's name, power limit and SM clocks.  Log-mel is a 400-point table DFT, so it is also reported as fp32 FLOP/s:
2 FMAs (re, im) per sample and bin, 2 * 2 * 400 * 201 FLOP per frame, against the 67 TFLOP/s fp32 data-sheet figure of
the H100 SXM."""
import os, subprocess, sys, torch
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from touchnet_b200 import frontend
g = torch.Generator().manual_seed(0)
lens = [int(16000 * (1 + 29 * float(torch.rand((), generator=g)))) for _ in range(64)]      # ~16 min of audio
wav = (0.3 * (2 * torch.rand(sum(lens), generator=g) - 1)).cuda()
smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                     capture_output=True, text=True).stdout.strip()
print(f"GPU: {smi}")
e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")


def timed(fn):
    for _ in range(3): out, frames = fn()
    ts = []
    for _ in range(10):
        flush.zero_()                       # flush L2 between timed iterations
        e0.record(); out, frames = fn(); e1.record(); torch.cuda.synchronize()
        ts.append(e0.elapsed_time(e1))
    return sorted(ts)[len(ts) // 2], out, frames


ms, out, frames = timed(lambda: frontend.fbank_batch(wav, lens))
alg = wav.numel() * 4 + out.numel() * 4
print(f"fbank {'DFT' if os.environ.get('TN_FBANK_DFT') else 'FFT'}: {sum(frames)} frames, {ms*1e3:.1f} us, algorithmic {alg/1e6:.1f} MB -> {alg/ms/1e6:.1f} GB/s, {sum(frames)/ms/1e3:.1f} Mframes/s")
ms_m, out, frames = timed(lambda: frontend.mfcc_batch(wav, lens, num_mel_bins=80, num_ceps=40))
alg = wav.numel() * 4 + out.numel() * 4
print(f"mfcc_batch 80 mel / 40 ceps: {sum(frames)} frames, {ms_m*1e3:.1f} us ({ms_m/ms:.2f}x fbank), algorithmic {alg/1e6:.1f} MB -> {alg/ms_m/1e6:.1f} GB/s, {sum(frames)/ms_m/1e3:.1f} Mframes/s")
for n_mels in (80, 128):
    ms_l, out, frames = timed(lambda: frontend.log_mel_batch(wav, lens, num_mel_bins=n_mels))
    alg = wav.numel() * 4 + out.numel() * 4
    flop = 4 * 400 * 201 * sum(frames)
    print(f"log_mel_batch {n_mels} mel: {sum(frames)} frames, {ms_l*1e3:.1f} us ({ms_l/ms:.2f}x fbank), algorithmic {alg/1e6:.1f} MB -> {alg/ms_l/1e6:.1f} GB/s, {sum(frames)/ms_l/1e3:.1f} Mframes/s, DFT {flop/ms_l/1e9:.1f} TFLOP/s = {100*flop/ms_l/1e9/67:.1f} % of 67 TFLOP/s fp32")
