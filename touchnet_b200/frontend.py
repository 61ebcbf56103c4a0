"""GPU audio frontend behind the reference's data-stage interface.

The reference composes per-sample generator stages `f(data: Iterator[dict], config: DataConfig) -> Iterator[dict]`
(ref: touchnet/data/datapipe.py:183-205).  The feature stages are mirrored here with the same names, argument meaning
and dict keys:

    audio_compute_fbank                 ref: touchnet/data/functions.py:117-134
    audio_compute_mfcc                  ref: touchnet/data/functions.py:137-156
    audio_compute_log_mel_spectrogram   ref: touchnet/data/functions.py:159-190
    audiofeat_stack                     ref: touchnet/data/functions.py:258-286

and the recipe's augmentation stages (draws as the reference makes them, application on the GPU, csrc/augment.cu):

    audio_resample                      ref: touchnet/data/functions.py:83-96
    audio_speed_perturb                 ref: touchnet/data/functions.py:99-114
    audiofeat_spec_aug / _sub / _trim   ref: touchnet/data/functions.py:193-255

plus batch-level entry points (`fbank_batch`, `mfcc_batch`, `log_mel_batch`, `stack_batch`, `fbank_stack_batch`,
`resample_batch`, `speed_perturb_batch`, `spec_augment_batch`, `augmented_fbank_stack_batch`,
`augmented_mfcc_stack_batch`, `augmented_log_mel_stack_batch`) that process a whole packed batch of
utterances in one launch each - the form used after the H2D copy in the train step (SURVEY 8(b) "data-frontend
boundary", option (i)); for augmentation, the records come from augment.draw_stage in the DataLoader worker.  All
arithmetic happens in libtouchnet_b200.so (csrc/frontend.cu, csrc/augment.cu); windows, mel filter banks, the MFCC
DCT table and resampling banks are small constants built once on the host exactly as the reference's third-party code builds them and cached per
device.
"""
from __future__ import annotations

import math
import random
from functools import lru_cache
from typing import Iterable, Iterator, Sequence

import numpy as np
import torch

from . import _lib, augment

MILLISECONDS_TO_SECONDS = 0.001
MAX_MEL_BINS = 128        # mel bins the frontend kernels hold on chip (csrc/frontend.cu FE_MAX_MELS)


# ---------------------------------------------------------------------------------------------------------------
# constants (host-side, cached)
# ---------------------------------------------------------------------------------------------------------------
@lru_cache(maxsize=None)
def _povey_window(n: int, device: str) -> torch.Tensor:
    """ta: compliance/kaldi.py:99-101."""
    return torch.hann_window(n, periodic=False, dtype=torch.float32).pow(0.85).to(device)


@lru_cache(maxsize=None)
def _hann_window(n: int, device: str) -> torch.Tensor:
    """torch.hann_window(n) (periodic), ref: functions.py:171."""
    return torch.hann_window(n, dtype=torch.float32).to(device)


@lru_cache(maxsize=None)
def _kaldi_mel_banks(num_bins: int, n_fft: int, sample_freq: float, low_freq: float, high_freq: float, device: str):
    """ta: compliance/kaldi.py:436-511 get_mel_banks (no VTLN) + zero column of :622; same fp32 op order."""
    num_fft_bins = n_fft / 2
    nyquist = 0.5 * sample_freq
    if high_freq <= 0.0:
        high_freq += nyquist
    fft_bin_width = sample_freq / n_fft
    mel_low = 1127.0 * math.log(1.0 + low_freq / 700.0)
    mel_high = 1127.0 * math.log(1.0 + high_freq / 700.0)
    mel_delta = (mel_high - mel_low) / (num_bins + 1)
    b = torch.arange(num_bins).unsqueeze(1)
    left = mel_low + b * mel_delta
    center = mel_low + (b + 1.0) * mel_delta
    right = mel_low + (b + 2.0) * mel_delta
    mel = (1127.0 * (1.0 + (fft_bin_width * torch.arange(num_fft_bins)) / 700.0).log()).unsqueeze(0)
    up = (mel - left) / (center - left)
    down = (right - mel) / (right - center)
    bins = torch.max(torch.zeros(1), torch.min(up, down))
    return torch.nn.functional.pad(bins, (0, 1)).to(torch.float32).contiguous().to(device)


@lru_cache(maxsize=None)
def _kaldi_mfcc_table(n_mels: int, n_ceps: int, lifter: float = 22.0, device: str = "cpu") -> torch.Tensor:
    """[n_mels, n_ceps] fp32 table A with mfcc = log-mel row @ A.  ta: compliance/kaldi.py _get_dct_matrix
    (functional.create_dct(n_mels, n_mels, "ortho"), column 0 set to sqrt(1/n_mels), first n_ceps columns) and
    _get_lifter_coeffs, both with torchaudio's fp32 op sequence; the lifter is folded in as an fp64 product rounded
    once to fp32."""
    n = torch.arange(float(n_mels))
    k = torch.arange(float(n_mels)).unsqueeze(1)
    dct = torch.cos(math.pi / float(n_mels) * (n + 0.5) * k)
    dct[0] *= 1.0 / math.sqrt(2.0)
    dct *= math.sqrt(2.0 / float(n_mels))
    dct = dct.t()
    dct[:, 0] = math.sqrt(1 / float(n_mels))
    dct = dct[:, :n_ceps]
    lift = 1.0 + 0.5 * lifter * torch.sin(math.pi * torch.arange(n_ceps) / lifter)
    return (dct.double() * lift.double()).to(torch.float32).contiguous().to(device)


@lru_cache(maxsize=None)
def _slaney_mel_filters(sr: int, n_fft: int, n_mels: int, device: str) -> torch.Tensor:
    """librosa.filters.mel(sr=sr, n_fft=n_fft, n_mels=n_mels) defaults (Slaney scale + Slaney norm), ref: functions.py:180-183."""
    f_sp, min_log_hz = 200.0 / 3, 1000.0
    min_log_mel, logstep = min_log_hz / f_sp, np.log(6.4) / 27.0

    def hz_to_mel(f):
        f = np.asarray(f, dtype=np.float64)
        return np.where(f >= min_log_hz, min_log_mel + np.log(np.maximum(f, 1e-10) / min_log_hz) / logstep, f / f_sp)

    def mel_to_hz(m):
        m = np.asarray(m, dtype=np.float64)
        return np.where(m >= min_log_mel, min_log_hz * np.exp(logstep * (m - min_log_mel)), f_sp * m)

    fftfreqs = np.fft.rfftfreq(n=n_fft, d=1.0 / sr)
    mel_f = mel_to_hz(np.linspace(hz_to_mel(0.0), hz_to_mel(sr / 2.0), n_mels + 2))
    fdiff = np.diff(mel_f)
    ramps = np.subtract.outer(mel_f, fftfreqs)
    w = np.zeros((n_mels, 1 + n_fft // 2))
    for i in range(n_mels):
        w[i] = np.maximum(0, np.minimum(-ramps[i] / fdiff[i], ramps[i + 2] / fdiff[i + 1]))
    w *= (2.0 / (mel_f[2: n_mels + 2] - mel_f[:n_mels]))[:, None]
    return torch.from_numpy(w.astype(np.float32)).contiguous().to(device)


def _st() -> int:
    return torch.cuda.current_stream().cuda_stream


def _pack(waveforms: Sequence[torch.Tensor], device) -> tuple[torch.Tensor, list[int]]:
    lens = [int(w.numel()) for w in waveforms]
    flat = torch.cat([w.reshape(-1) for w in waveforms]) if len(waveforms) > 1 else waveforms[0].reshape(-1)
    return flat.to(device, non_blocking=True).contiguous(), lens


def _offsets(lens: Sequence[int], device) -> torch.Tensor:
    off = np.zeros(len(lens) + 1, dtype=np.int64)
    np.cumsum(np.asarray(lens, dtype=np.int64), out=off[1:])
    return torch.from_numpy(off).to(device, non_blocking=True)


# ---------------------------------------------------------------------------------------------------------------
# batch-level ops
# ---------------------------------------------------------------------------------------------------------------
def fbank_frames(n_samples: int, sample_rate: int, frame_length: float, frame_shift: float) -> int:
    win = int(sample_rate * frame_length * MILLISECONDS_TO_SECONDS)
    shift = int(sample_rate * frame_shift * MILLISECONDS_TO_SECONDS)
    return 0 if n_samples < win else 1 + (n_samples - win) // shift


def _kaldi_batch(name, wav, lens, sample_rate, num_mel_bins, frame_length, frame_shift, low_freq, high_freq,
                 preemphasis, num_ceps=None):
    """Framing, window and mel bank shared by fbank_batch (num_ceps None) and mfcc_batch."""
    if not wav.is_cuda:
        raise _lib.TouchNetB200Error(f"{name} needs the packed waveform on the GPU (no CPU path)")
    assert wav.dtype in (torch.float32, torch.int16) and wav.dim() == 1
    dev = str(wav.device)
    win = int(sample_rate * frame_length * MILLISECONDS_TO_SECONDS)
    shift = int(sample_rate * frame_shift * MILLISECONDS_TO_SECONDS)
    n_fft = 1 << (win - 1).bit_length()
    frames = [0 if n < win else 1 + (n - win) // shift for n in lens]
    total = int(sum(frames))
    out = torch.empty((total, num_mel_bins if num_ceps is None else num_ceps), dtype=torch.float32, device=wav.device)
    if total == 0:
        return out, frames
    utt_off, frm_off = _offsets(lens, wav.device), _offsets(frames, wav.device)
    window = _povey_window(win, dev)
    banks = _kaldi_mel_banks(num_mel_bins, n_fft, float(sample_rate), float(low_freq), float(high_freq), dev)
    args = (wav.data_ptr(), int(wav.dtype == torch.int16), utt_off.data_ptr(), frm_off.data_ptr(), len(lens), total, win,
            shift, n_fft, window.data_ptr(), banks.data_ptr(), num_mel_bins, float(preemphasis))
    if num_ceps is None:
        _lib.call("tn_fbank_f32", *args, out.data_ptr(), _st())
    else:
        table = _kaldi_mfcc_table(num_mel_bins, num_ceps, 22.0, dev)
        _lib.call("tn_mfcc_f32", *args, table.data_ptr(), num_ceps, out.data_ptr(), _st())
    return out, frames


def fbank_batch(wav: torch.Tensor, lens: Sequence[int], sample_rate: int = 16000, num_mel_bins: int = 80,
                frame_length: float = 25.0, frame_shift: float = 10.0, low_freq: float = 20.0, high_freq: float = 0.0,
                preemphasis: float = 0.97):
    """wav: packed utterances back to back on the GPU, fp32 in [-1,1] or int16 PCM.  Returns (feats [sum m_i, mel]
    fp32, frame_counts).  Semantics of kaldi.fbank(waveform * 2**15, dither=0, energy_floor=0) per utterance."""
    return _kaldi_batch("fbank_batch", wav, lens, sample_rate, num_mel_bins, frame_length, frame_shift, low_freq,
                        high_freq, preemphasis)


def mfcc_batch(wav: torch.Tensor, lens: Sequence[int], sample_rate: int = 16000, num_mel_bins: int = 80,
               num_ceps: int = 40, frame_length: float = 25.0, frame_shift: float = 10.0, low_freq: float = 20.0,
               high_freq: float = 0.0):
    """MFCC per utterance of a packed batch (fp32 in [-1,1] or int16 PCM, on the GPU), one launch.  Returns
    (feats [sum m_i, num_ceps] fp32, frame_counts); frames as fbank_batch.  Semantics of
    kaldi.mfcc(waveform * 2**15, dither=0, num_ceps, low_freq, high_freq) with torchaudio's other defaults (no energy,
    lifter 22), ref: functions.py:137-156: fbank's log-mel row times the lifted DCT table, fused into the fbank kernel."""
    if not 1 <= int(num_ceps) <= int(num_mel_bins):
        raise _lib.TouchNetB200Error(f"mfcc needs 1 <= num_ceps <= num_mel_bins, got num_ceps={num_ceps}, "
                                     f"num_mel_bins={num_mel_bins}")
    if int(num_mel_bins) > MAX_MEL_BINS:
        raise _lib.TouchNetB200Error(f"mfcc takes at most {MAX_MEL_BINS} mel bins, got {num_mel_bins}")
    return _kaldi_batch("mfcc_batch", wav, lens, sample_rate, num_mel_bins, frame_length, frame_shift, low_freq,
                        high_freq, 0.97, int(num_ceps))


def log_mel_batch(wav: torch.Tensor, lens: Sequence[int], sample_rate: int = 16000, n_fft: int = 400,
                  hop_length: int = 160, num_mel_bins: int = 80, padding: int = 0):
    """Whisper-style log-mel per utterance (ref: functions.py:159-190) of a packed batch on the GPU: fp32 in [-1,1] or
    int16 PCM (read as pcm / 32768, bit-identical to the fp32 input).  Every utterance is right-padded with `padding`
    zero samples (audiofeat_padding, functions.py:169-170) inside the kernel, without a copy.  Returns
    (feats [sum (N_i + padding)//hop, mel], counts)."""
    if wav.dtype not in (torch.float32, torch.int16) or wav.dim() != 1:
        raise _lib.TouchNetB200Error(f"log_mel_batch takes a 1-D packed fp32 or int16 waveform, got {wav.dtype} "
                                     f"of rank {wav.dim()}")
    if int(padding) < 0:
        raise _lib.TouchNetB200Error(f"log_mel_batch: padding must be >= 0, got {padding}")
    if not wav.is_cuda:
        raise _lib.TouchNetB200Error("log_mel_batch needs the packed waveform on the GPU (no CPU path)")
    dev = str(wav.device)
    padding = int(padding)
    frames = [(n + padding) // hop_length for n in lens]   # 1 + (N+pad)//hop stft frames, last one dropped (:176)
    total = int(sum(frames))
    out = torch.empty((total, num_mel_bins), dtype=torch.float32, device=wav.device)
    if total == 0:
        return out, frames
    utt_off, frm_off = _offsets(lens, wav.device), _offsets(frames, wav.device)
    utt_max = torch.empty(len(lens), dtype=torch.float32, device=wav.device)
    window = _hann_window(n_fft, dev)
    filters = _slaney_mel_filters(sample_rate, n_fft, num_mel_bins, dev)
    _lib.call("tn_logmel_power_f32", wav.data_ptr(), int(wav.dtype == torch.int16), utt_off.data_ptr(),
              frm_off.data_ptr(), len(lens), total, n_fft, hop_length, padding, window.data_ptr(), filters.data_ptr(),
              num_mel_bins, out.data_ptr(), utt_max.data_ptr(), _st())
    _lib.call("tn_logmel_finish_f32", out.data_ptr(), frm_off.data_ptr(), utt_max.data_ptr(), len(lens), total,
              num_mel_bins, _st())
    return out, frames


def stack_batch(feats: torch.Tensor, frames: Sequence[int], stack_length: int, stride_length: int,
                normalize: bool = True, into: torch.Tensor | None = None, dst_rows: Sequence[int] | None = None):
    """Low-frame-rate stacking per utterance (ref: functions.py:258-286).  Returns (out [sum ceil(T_i/stride), mel*stack], counts).
    With `into` ([rows, F] fp32 batch buffer) and `dst_rows` (first destination row per utterance) the stacked rows are
    written straight into the packed-batch `input_features` buffer (layout of processing_touch_audio.py:200)."""
    assert feats.is_cuda and feats.dtype == torch.float32 and feats.dim() == 2
    n_mels = feats.shape[1]
    rows = [int(math.ceil(t / stride_length)) if t > 0 else 0 for t in frames]
    total = int(sum(rows))
    if into is None:
        out = torch.empty((total, n_mels * stack_length), dtype=torch.float32, device=feats.device)
        dst, ld = None, 0
    else:
        assert into.is_cuda and into.dtype == torch.float32 and into.dim() == 2 and into.stride(1) == 1
        assert into.shape[1] == n_mels * stack_length and dst_rows is not None and len(dst_rows) == len(frames)
        out, ld = into, into.stride(0)
        dst = torch.tensor(list(dst_rows), dtype=torch.int64).to(feats.device, non_blocking=True)
    if total == 0:
        return out, rows
    frm_off, out_off = _offsets(frames, feats.device), _offsets(rows, feats.device)
    _lib.call("tn_feat_stack_f32", feats.data_ptr(), frm_off.data_ptr(), out_off.data_ptr(), len(frames), total, n_mels,
              stack_length, stride_length, int(bool(normalize)), out.data_ptr(), None if dst is None else dst.data_ptr(),
              ld, _st())
    return out, rows


def fbank_stack_batch(wav: torch.Tensor, lens: Sequence[int], *, sample_rate=16000, num_mel_bins=80, frame_length=25.0,
                      frame_shift=10.0, stack_length=5, stride_length=4, normalize=True):
    feats, frames = fbank_batch(wav, lens, sample_rate, num_mel_bins, frame_length, frame_shift)
    return stack_batch(feats, frames, stack_length, stride_length, normalize)


# ---------------------------------------------------------------------------------------------------------------
# augmentation (draws: augment.py; application: csrc/augment.cu)
# ---------------------------------------------------------------------------------------------------------------
RESAMPLE_TILE = 1024      # output samples per CTA of tn_resample_f32


def _resample_pairs(wav: torch.Tensor, lens: Sequence[int], pairs: Sequence[tuple[int, int] | None]):
    """Resample utterance i from pairs[i] = (orig, new) (None: exact copy) in one launch.  Returns (fp32 out, lens)."""
    if not wav.is_cuda:
        raise _lib.TouchNetB200Error("resampling needs the packed waveform on the GPU (no CPU path)")
    if wav.dtype not in (torch.float32, torch.int16) or wav.dim() != 1:
        raise _lib.TouchNetB200Error("resampling takes a 1-D packed fp32 or int16 waveform")
    if len(pairs) != len(lens):
        raise _lib.TouchNetB200Error(f"{len(lens)} utterances but {len(pairs)} rate pairs")
    dev = str(wav.device)
    keys, table, banks, utt_bank, bank_off = {}, [], [], [], 0
    out_lens = []
    for n, pr in zip(lens, pairs):
        key = (1, 1) if pr is None or int(pr[0]) == int(pr[1]) else augment.reduced_ratio(*pr)
        if pr is not None and (int(pr[0]) <= 0 or int(pr[1]) <= 0):
            raise _lib.TouchNetB200Error(f"resampling rates must be positive, got {pr}")
        if key not in keys:
            keys[key] = len(table)
            if key == (1, 1):
                table.append((1, 1, 0, 1, 0))
            else:
                bank, width = augment.sinc_resample_bank(key[0], key[1], dev)
                table.append((key[0], key[1], width, bank.shape[1], bank_off))
                banks.append(bank.reshape(-1))
                bank_off += bank.numel()
        utt_bank.append(keys[key])
        out_lens.append(int(n) if key == (1, 1) else augment.resampled_length(int(n), key[0], key[1]))
    if len(table) > 16:
        raise _lib.TouchNetB200Error(f"one resampling launch takes at most 16 distinct rate ratios, got {len(table)}")
    out = torch.empty(int(sum(out_lens)), dtype=torch.float32, device=wav.device)
    tiles = [(m + RESAMPLE_TILE - 1) // RESAMPLE_TILE for m in out_lens]
    n_tiles = int(sum(tiles))
    if n_tiles == 0:
        return out, out_lens
    meta = np.zeros((3, len(lens) + 1), dtype=np.int64)
    for r, v in enumerate((lens, out_lens, tiles)):
        np.cumsum(np.asarray(v, dtype=np.int64), out=meta[r, 1:])
    meta_d = torch.from_numpy(meta).to(wav.device, non_blocking=True)
    utt_bank_d = torch.tensor(utt_bank, dtype=torch.int32).to(wav.device, non_blocking=True)
    table_h = np.ascontiguousarray(np.asarray(table, dtype=np.int32))
    banks_d = torch.cat(banks) if banks else torch.zeros(1, dtype=torch.float32, device=wav.device)
    _lib.call("tn_resample_f32", wav.data_ptr(), int(wav.dtype == torch.int16), meta_d[0].data_ptr(),
              meta_d[1].data_ptr(), meta_d[2].data_ptr(), utt_bank_d.data_ptr(), len(lens), n_tiles, RESAMPLE_TILE,
              table_h.ctypes.data, len(table), banks_d.data_ptr(), out.data_ptr(), _st())
    return out, out_lens


def resample_batch(wav: torch.Tensor, lens: Sequence[int], orig_freqs, new_freq: int):
    """torchaudio.transforms.Resample(orig, new_freq) per utterance (ref: functions.py:83-96), one launch for the packed
    batch.  orig_freqs: one rate or one per utterance; an utterance already at new_freq is copied exactly.
    Returns (fp32 out, out_lens)."""
    origs = [int(orig_freqs)] * len(lens) if np.isscalar(orig_freqs) else [int(o) for o in orig_freqs]
    return _resample_pairs(wav, lens, [(o, int(new_freq)) for o in origs])


def speed_perturb_batch(wav: torch.Tensor, lens: Sequence[int], speeds: Sequence[float], sample_rate: int):
    """Speed perturbation per utterance (ref: functions.py:99-114): sox `speed s` + `rate sr` is resampling from sr*s to
    sr, here with torchaudio's sinc filter (not sox's).  Speed 1.0 copies.  Returns (fp32 out, out_lens)."""
    pairs = [None if float(s) == 1.0 else (augment.speed_source_rate(int(sample_rate), s), int(sample_rate))
             for s in speeds]
    return _resample_pairs(wav, lens, pairs)


def spec_augment_batch(feats: torch.Tensor, frames: Sequence[int], records: Sequence[dict]):
    """SpecAugment time/frequency masks, SpecSub and SpecTrim of augment.draw_record records (ref: functions.py:193-255),
    out of place, one launch.  Returns (out [sum(frames_i - trim_i), F], out_frames).  Bit-exact (copies and zeros)."""
    if not (feats.is_cuda and feats.dtype == torch.float32 and feats.dim() == 2 and feats.is_contiguous()):
        raise _lib.TouchNetB200Error("spec_augment_batch takes contiguous [frames, F] fp32 features on the GPU")
    if len(records) != len(frames):
        raise _lib.TouchNetB200Error(f"{len(frames)} utterances but {len(records)} records")
    out_frames = []
    for t, r in zip(frames, records):
        if r["trim"] < 0 or r["trim"] > t:
            raise _lib.TouchNetB200Error(f"trim {r['trim']} out of range for {t} frames")
        out_frames.append(int(t) - int(r["trim"]))
    total = int(sum(out_frames))
    out = torch.empty((total, feats.shape[1]), dtype=torch.float32, device=feats.device)
    if total == 0:
        return out, out_frames

    def table(key, width):
        n = max(len(r[key]) for r in records)
        tab = np.zeros((len(records), max(n, 1), width), dtype=np.int32)   # empty entries: start == end == 0
        for i, r in enumerate(records):
            if r[key]:
                tab[i, :len(r[key])] = np.asarray(r[key], dtype=np.int32).reshape(-1, width)
        return torch.from_numpy(tab).to(feats.device, non_blocking=True), n

    tm, n_t = table("t_masks", 2)
    fm, n_f = table("f_masks", 2)
    sb, n_s = table("subs", 3)
    in_off, out_off = _offsets(frames, feats.device), _offsets(out_frames, feats.device)
    _lib.call("tn_spec_augment_f32", feats.data_ptr(), in_off.data_ptr(), out_off.data_ptr(), len(frames), total,
              feats.shape[1], tm.data_ptr(), n_t, fm.data_ptr(), n_f, sb.data_ptr(), n_s, out.data_ptr(), _st())
    return out, out_frames


def _augmented_stack(wav, lens, records, sample_rate, features, stack_length, stride_length, normalize, into, dst_rows):
    """resample -> speed perturb -> features(wav, lens) -> SpecAugment / SpecSub / SpecTrim -> stack, skipping the stages
    no utterance needs."""
    if len(records) != len(lens):
        raise _lib.TouchNetB200Error(f"{len(lens)} utterances but {len(records)} records")
    for r in records:
        if r["resample"] is not None and int(r["resample"][1]) != int(sample_rate):
            raise _lib.TouchNetB200Error(f"record resamples to {r['resample'][1]} Hz but features run at {sample_rate}")
    if any(r["resample"] is not None for r in records):
        wav, lens = _resample_pairs(wav, lens, [r["resample"] for r in records])
    if any(float(r["speed"]) != 1.0 for r in records):
        wav, lens = speed_perturb_batch(wav, lens, [r["speed"] for r in records], sample_rate)
    feats, frames = features(wav, lens)
    if any(augment.record_has_feature_ops(r) for r in records):
        feats, frames = spec_augment_batch(feats, frames, records)
    return stack_batch(feats, frames, stack_length, stride_length, normalize, into=into, dst_rows=dst_rows)


def augmented_fbank_stack_batch(wav: torch.Tensor, lens: Sequence[int], records: Sequence[dict], *, sample_rate=16000,
                                num_mel_bins=80, frame_length=25.0, frame_shift=10.0, stack_length=5, stride_length=4,
                                normalize=True, into: torch.Tensor | None = None, dst_rows: Sequence[int] | None = None):
    """The recipe's chain resample -> speed perturb -> fbank -> SpecAugment -> SpecSub -> SpecTrim -> stack on a packed
    batch of raw waveforms (fp32 or int16), applying the host-drawn records of augment.draw_record / draw_stage.
    sample_rate is the rate features are computed at (the records' resampling target).  Stages no utterance needs are
    skipped, so with every augmentation off this is exactly fbank_batch + stack_batch.  Returns stack_batch's result."""
    return _augmented_stack(wav, lens, records, sample_rate,
                            lambda w, n: fbank_batch(w, n, sample_rate, num_mel_bins, frame_length, frame_shift),
                            stack_length, stride_length, normalize, into, dst_rows)


def augmented_mfcc_stack_batch(wav: torch.Tensor, lens: Sequence[int], records: Sequence[dict], *, sample_rate=16000,
                               num_mel_bins=80, num_ceps=40, frame_length=25.0, frame_shift=10.0, low_freq=20.0,
                               high_freq=0.0, stack_length=5, stride_length=4, normalize=True,
                               into: torch.Tensor | None = None, dst_rows: Sequence[int] | None = None):
    """augmented_fbank_stack_batch with MFCC features: resample -> speed perturb -> MFCC -> SpecAugment -> SpecSub ->
    SpecTrim -> stack, for records drawn with audio_feat_type="mfcc" (frequency masks over the num_ceps columns).
    With every augmentation off this is exactly mfcc_batch + stack_batch.  Returns stack_batch's result."""
    return _augmented_stack(wav, lens, records, sample_rate,
                            lambda w, n: mfcc_batch(w, n, sample_rate, num_mel_bins, num_ceps, frame_length,
                                                    frame_shift, low_freq, high_freq),
                            stack_length, stride_length, normalize, into, dst_rows)


def augmented_log_mel_stack_batch(wav: torch.Tensor, lens: Sequence[int], records: Sequence[dict], *,
                                  sample_rate=16000, num_mel_bins=80, n_fft=400, hop_length=160, padding=0,
                                  stack_length=5, stride_length=4, normalize=True, into: torch.Tensor | None = None,
                                  dst_rows: Sequence[int] | None = None):
    """augmented_fbank_stack_batch with whisper log-mel features: resample -> speed perturb -> log-mel (audiofeat_padding
    zeros appended, the per-utterance max-8 clamp and (x+4)/4 included, so masked cells are 0 as in the reference) ->
    SpecAugment -> SpecSub -> SpecTrim -> stack, for records drawn with audio_feat_type="log_mel_spectrogram".  An
    utterance whose length after augmentation plus padding is at most n_fft // 2 raises, as the reference's reflect
    padding does.  With every augmentation off this is exactly log_mel_batch + stack_batch.  Returns stack_batch's
    result."""
    if int(padding) < 0:
        raise _lib.TouchNetB200Error(f"log-mel padding must be >= 0, got {padding}")

    def features(w, n):
        for i, m in enumerate(n):
            if int(m) + int(padding) <= n_fft // 2:
                raise _lib.TouchNetB200Error(
                    f"utterance {i} has {m} samples (+{padding} padding) at {sample_rate} Hz: log-mel's reflect padding "
                    f"needs more than n_fft // 2 = {n_fft // 2}")
        return log_mel_batch(w, n, sample_rate, n_fft, hop_length, num_mel_bins, padding)

    return _augmented_stack(wav, lens, records, sample_rate, features, stack_length, stride_length, normalize, into,
                            dst_rows)


# ---------------------------------------------------------------------------------------------------------------
# per-sample generator stages (the reference's operator interface)
# ---------------------------------------------------------------------------------------------------------------
def _device(config) -> torch.device:
    return torch.device(getattr(config, "frontend_device", "cuda"))


def audio_compute_fbank(data: Iterable[dict], config) -> Iterator[dict]:
    """Extract fbank.  Same contract as ref: touchnet/data/functions.py:117-134."""
    for sample in data:
        assert "sample_rate" in sample
        assert "waveform" in sample
        wav, lens = _pack([sample["waveform"]], _device(config))
        mat, _ = fbank_batch(wav.float() if wav.dtype not in (torch.float32, torch.int16) else wav, lens,
                             sample_rate=sample["sample_rate"], num_mel_bins=config.audiofeat_num_mel_bins,
                             frame_length=config.audiofeat_frame_length, frame_shift=config.audiofeat_frame_shift)
        if getattr(config, "audiofeat_dither", 0.0) != 0.0:
            raise _lib.TouchNetB200Error("dither != 0 is not supported (all reference recipes use 0.0)")
        sample["audiofeat"] = mat
        yield sample


def audio_compute_mfcc(data: Iterable[dict], config) -> Iterator[dict]:
    """Extract MFCC.  Same contract as ref: touchnet/data/functions.py:137-156."""
    for sample in data:
        assert "sample_rate" in sample
        assert "waveform" in sample
        if getattr(config, "audiofeat_dither", 0.0) != 0.0:
            raise _lib.TouchNetB200Error("dither != 0 is not supported (all reference recipes use 0.0)")
        wav, lens = _pack([sample["waveform"]], _device(config))
        mat, _ = mfcc_batch(wav.float() if wav.dtype not in (torch.float32, torch.int16) else wav, lens,
                            sample_rate=sample["sample_rate"], num_mel_bins=config.audiofeat_num_mel_bins,
                            num_ceps=config.audiofeat_num_ceps, frame_length=config.audiofeat_frame_length,
                            frame_shift=config.audiofeat_frame_shift, low_freq=config.audiofeat_low_freq,
                            high_freq=config.audiofeat_high_freq)
        sample["audiofeat"] = mat
        yield sample


def audio_compute_log_mel_spectrogram(data: Iterable[dict], config) -> Iterator[dict]:
    """Extract whisper-style log mel spectrogram.  Same contract as ref: touchnet/data/functions.py:159-190; an int16
    waveform is read as pcm / 32768 and audiofeat_padding is applied inside the kernel."""
    for sample in data:
        assert "sample_rate" in sample
        assert "waveform" in sample
        waveform = sample["waveform"].squeeze(0)
        pad = getattr(config, "audiofeat_padding", 0)
        wav, lens = _pack([waveform], _device(config))
        mat, _ = log_mel_batch(wav if wav.dtype in (torch.float32, torch.int16) else wav.float(), lens,
                               sample_rate=sample["sample_rate"], n_fft=config.audiofeat_n_fft,
                               hop_length=config.audiofeat_hop_length, num_mel_bins=config.audiofeat_num_mel_bins,
                               padding=pad if pad > 0 else 0)
        sample["audiofeat"] = mat
        yield sample


def audiofeat_stack(data: Iterable[dict], config) -> Iterator[dict]:
    """Stack audio features (low frame rate).  Same contract as ref: touchnet/data/functions.py:258-286."""
    for sample in data:
        assert "audiofeat" in sample
        x = sample["audiofeat"]
        if not x.is_cuda:
            x = x.to(_device(config))
        out, _ = stack_batch(x.float().contiguous(), [x.shape[0]], config.audiofeat_stack_length,
                             config.audiofeat_stride_length, config.audiofeat_normalize)
        sample["audiofeat"] = out
        yield sample


def _one_utt_record(**ops) -> dict:
    rec = {"resample": None, "speed": 1.0, "t_masks": [], "f_masks": [], "subs": [], "trim": 0}
    rec.update(ops)
    return rec


def _apply_feature_ops(sample: dict, config, **ops) -> dict:
    x = sample["audiofeat"]
    if not x.is_cuda:
        x = x.to(_device(config))
    out, _ = spec_augment_batch(x.float().contiguous(), [x.shape[0]], [_one_utt_record(**ops)])
    sample["audiofeat"] = out
    return sample


def audio_resample(data: Iterable[dict], config) -> Iterator[dict]:
    """Resample to config.audio_resample_rate.  Same contract as ref: touchnet/data/functions.py:83-96 (torchaudio's
    sinc_interp_hann filter); the waveform comes back [1, T] fp32 on the frontend device."""
    for sample in data:
        assert "sample_rate" in sample
        assert "waveform" in sample
        sample_rate = sample["sample_rate"]
        if sample_rate != config.audio_resample_rate:
            wav, lens = _pack([sample["waveform"]], _device(config))
            out, _ = resample_batch(wav if wav.dtype in (torch.float32, torch.int16) else wav.float(), lens,
                                    sample_rate, config.audio_resample_rate)
            sample["sample_rate"] = config.audio_resample_rate
            sample["waveform"] = out[None]
        yield sample


def audio_speed_perturb(data: Iterable[dict], config) -> Iterator[dict]:
    """Speed perturbation.  Same contract and draw as ref: touchnet/data/functions.py:99-114; sox's `speed` + `rate` is
    done as torchaudio-style sinc resampling from sample_rate*speed to sample_rate (not sox's filter)."""
    for sample in data:
        assert "sample_rate" in sample
        assert "waveform" in sample
        sample_rate = sample["sample_rate"]
        speed = random.choice(config.audio_speed_perturb_speeds)
        if speed != 1.0:
            wav, lens = _pack([sample["waveform"]], _device(config))
            out, _ = speed_perturb_batch(wav if wav.dtype in (torch.float32, torch.int16) else wav.float(), lens,
                                         [speed], sample_rate)
            sample["waveform"] = out[None]
        yield sample


def audiofeat_spec_aug(data: Iterable[dict], config) -> Iterator[dict]:
    """SpecAugment time and frequency masks.  Same contract and draws as ref: touchnet/data/functions.py:193-217."""
    for sample in data:
        assert "audiofeat" in sample
        x = sample["audiofeat"]
        t_masks, f_masks = augment.draw_time_freq_masks(x.size(0), x.size(1), config)
        yield _apply_feature_ops(sample, config, t_masks=t_masks, f_masks=f_masks)


def audiofeat_spec_sub(data: Iterable[dict], config) -> Iterator[dict]:
    """SpecSub.  Same contract and draws as ref: touchnet/data/functions.py:220-239 (every sub reads the input)."""
    for sample in data:
        assert "audiofeat" in sample
        subs = augment.draw_subs(sample["audiofeat"].size(0), config)
        yield _apply_feature_ops(sample, config, subs=subs)


def audiofeat_spec_trim(data: Iterable[dict], config) -> Iterator[dict]:
    """SpecTrim (tail frames).  Same contract and draw as ref: touchnet/data/functions.py:242-255."""
    for sample in data:
        assert "audiofeat" in sample
        trim = augment.draw_trim(sample["audiofeat"].size(0), config)
        yield _apply_feature_ops(sample, config, trim=trim) if trim else sample
