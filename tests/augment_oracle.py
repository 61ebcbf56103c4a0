"""ORACLE for the data augmentation (test infrastructure, never on the product path): numpy restatements of
  resample()       ref: touchnet/data/functions.py:83-96 audio_resample -> torchaudio.transforms.Resample (sinc_interp_hann,
                   lowpass_filter_width 6, rolloff 0.99); speed perturbation (functions.py:99-114) is resampling from
                   sr*speed to sr with the same filter
  apply_record()   ref: touchnet/data/functions.py:193-255 audiofeat_spec_aug / spec_sub / spec_trim with given draws
Pinned against tests/golden/augment.npz (made by tests/golden/make_golden_augment.py from the reference functions)."""
from __future__ import annotations

import math

import numpy as np

U32 = 2.0 ** -24     # unit roundoff of fp32


def sinc_resample_bank(orig: int, new: int, lowpass_filter_width: int = 6, rolloff: float = 0.99):
    """The filter bank of ta: functional/functional.py _get_sinc_resample_kernel (float64 but for the fp32 phase
    offsets, as torchaudio computes it), as [new', 2*width + orig'] (gcd-reduced rates), and width."""
    g = math.gcd(orig, new)
    o, n = orig // g, new // g
    base = min(o, n) * rolloff
    width = math.ceil(lowpass_filter_width * o / base)
    idx = np.arange(-width, width + o, dtype=np.float64)[None, :] / o
    phase = (np.arange(0, -n, -1)[:, None] / n).astype(np.float32)      # torchaudio divides these in the default fp32
    t = (phase.astype(np.float64) + idx) * base
    t = np.clip(t, -lowpass_filter_width, lowpass_filter_width)
    window = np.cos(t * np.pi / lowpass_filter_width / 2) ** 2
    t = t * np.pi
    with np.errstate(invalid="ignore", divide="ignore"):
        sinc = np.where(t == 0, 1.0, np.sin(t) / t)
    return sinc * window * (base / o), width


def _polyphase(x: np.ndarray, orig: int, new: int, w: np.ndarray, width: int) -> np.ndarray:
    """y[i*new' + j] = sum_k w[j, k] x[i*orig' - width + k] (x = 0 outside), length ceil(new' N / orig') through fp32."""
    g = math.gcd(orig, new)
    o, n = orig // g, new // g
    N = x.shape[0]
    out_len = int(math.ceil(float(np.float32(n * N / o))))
    blocks = (out_len + n - 1) // n
    taps = w.shape[1]
    xp = np.concatenate([np.zeros(width), x, np.zeros(blocks * o + taps)])
    frames = xp[np.arange(blocks)[:, None] * o + np.arange(taps)[None, :]]      # [blocks, taps]
    return (frames @ w.T).reshape(-1)[:out_len]                                   # row-major [blocks, new']


def resample(x: np.ndarray, orig: int, new: int) -> np.ndarray:
    """torchaudio.transforms.Resample(orig, new)(x): the bank rounded to float32 as torchaudio stores it, the sums in
    float64.  Returns float32."""
    x = np.asarray(x, dtype=np.float64)
    if orig == new:
        return x.astype(np.float32)
    w, width = sinc_resample_bank(orig, new)
    return _polyphase(x, orig, new, w.astype(np.float32).astype(np.float64), width).astype(np.float32)


def resample_tolerance(x: np.ndarray, orig: int, new: int, y_ref: np.ndarray) -> np.ndarray:
    """Per-output bound on |y - y_ref| for two fp32 evaluations of the same resampling in any summation order:
    2 * gamma_taps * sum_k |w_k||x_k| + 2u|y_ref|, gamma_n = n u / (1 - n u) (the standard dot-product bound), plus the
    fp32 rounding of both results."""
    if orig == new:
        return np.zeros(np.asarray(x).shape[0])
    w, width = sinc_resample_bank(orig, new)
    taps = w.shape[1]
    gamma = taps * U32 / (1 - taps * U32)
    mag = _polyphase(np.abs(np.asarray(x, dtype=np.float64)), orig, new,
                     np.abs(w.astype(np.float32).astype(np.float64)), width)
    return 2 * gamma * mag + 2 * U32 * np.abs(np.asarray(y_ref, dtype=np.float64))


def apply_record(feats: np.ndarray, rec: dict) -> np.ndarray:
    """SpecAugment masks, SpecSub and SpecTrim of one record, literally in the reference's order: masks on a copy, every
    sub reads the masked features (not the subs before it), the trim cuts the tail last."""
    y = np.array(feats, dtype=np.float32, copy=True)
    for s, e in rec["t_masks"]:
        y[s:e, :] = 0
    for s, e in rec["f_masks"]:
        y[:, s:e] = 0
    x = y.copy()
    for s, e, pos in rec["subs"]:
        y[s:e, :] = x[s - pos:e - pos, :]
    if rec["trim"]:
        y = y[:y.shape[0] - rec["trim"]]
    return y
