"""ORACLE (test infrastructure): numpy restatement of kaldi MFCC as the reference computes it (touchnet/data/
functions.py:137-156 -> torchaudio.compliance.kaldi.mfcc with use_energy off, cepstral_lifter 22, no htk_compat, no mean
subtraction), and the tolerance the GPU tests derive from the reference's log-mel row.

  fbank()       oracle.frontend_oracle.fbank with the low / high frequency of the mel bank exposed (its bank builder
                kaldi_mel_banks already takes them)
  mfcc_table()  A = DCT-II (orthonormal, column 0 = sqrt(1/n_mels), first n_ceps columns) * lifter, in fp64, rounded
                once to fp32
  mfcc()        fbank() @ A
Pinned against the reference's own outputs in tests/golden/mfcc.npz (tests/golden/make_golden_mfcc.py).
"""
from __future__ import annotations

import numpy as np

from oracle import frontend_oracle as fo

U32 = 2.0 ** -24       # fp32 unit roundoff


def fbank(waveform: np.ndarray, sample_rate: int = 16000, num_mel_bins: int = 80, frame_length_ms: float = 25.0,
          frame_shift_ms: float = 10.0, low_freq: float = 20.0, high_freq: float = 0.0,
          preemph: float = 0.97) -> np.ndarray:
    """Same framing and arithmetic as frontend_oracle.fbank (see there); only the mel bank's edges differ."""
    x = (waveform.astype(np.float32) * np.float32(32768.0)).astype(np.float32)
    shift = int(sample_rate * frame_shift_ms * 0.001)
    win = int(sample_rate * frame_length_ms * 0.001)
    n_fft = 1 << (win - 1).bit_length()
    n = x.shape[0]
    if n < win:
        return np.zeros((0, num_mel_bins), np.float32)
    m = 1 + (n - win) // shift
    frames = x[np.arange(m)[:, None] * shift + np.arange(win)[None, :]]
    frames = frames - frames.mean(axis=1, keepdims=True, dtype=np.float32)
    prev = np.concatenate([frames[:, :1], frames[:, :-1]], axis=1)
    frames = frames - np.float32(preemph) * prev
    frames = frames * fo.povey_window(win)[None, :]
    frames = np.pad(frames, ((0, 0), (0, n_fft - win))).astype(np.float32)
    spec = np.abs(np.fft.rfft(frames, axis=1).astype(np.complex64)).astype(np.float32) ** np.float32(2.0)
    mel = spec @ fo.kaldi_mel_banks(num_mel_bins, n_fft, float(sample_rate), low_freq, high_freq).T
    return np.log(np.maximum(mel, fo.EPS_F32)).astype(np.float32)


def mfcc_table(n_mels: int, n_ceps: int, lifter: float = 22.0) -> np.ndarray:
    """[n_mels, n_ceps] fp32: kaldi's DCT (ta: compliance/kaldi.py _get_dct_matrix) times the lifter
    1 + (L/2) sin(pi i / L) (_get_lifter_coeffs), both in fp64."""
    n = np.arange(n_mels, dtype=np.float64)[:, None]
    k = np.arange(n_ceps, dtype=np.float64)[None, :]
    d = np.cos(np.pi / n_mels * (n + 0.5) * k) * np.sqrt(2.0 / n_mels)
    d[:, 0] = np.sqrt(1.0 / n_mels)
    lift = 1.0 + 0.5 * lifter * np.sin(np.pi * np.arange(n_ceps, dtype=np.float64) / lifter)
    return (d * lift[None, :]).astype(np.float32)


def mfcc(waveform: np.ndarray, sample_rate: int = 16000, num_mel_bins: int = 80, num_ceps: int = 40,
         frame_length_ms: float = 25.0, frame_shift_ms: float = 10.0, low_freq: float = 20.0,
         high_freq: float = 0.0) -> np.ndarray:
    y = fbank(waveform, sample_rate, num_mel_bins, frame_length_ms, frame_shift_ms, low_freq, high_freq)
    return (y.astype(np.float64) @ mfcc_table(num_mel_bins, num_ceps).astype(np.float64)).astype(np.float32)


def reference_logmel(g, fbank_golden, tag: str, name: str) -> np.ndarray:
    """The reference's kaldi.fbank rows behind mfcc.npz's `mfcc/<tag>/<name>`: `fbank/<tag>/<name>`, except for the
    16 kHz 80-bin configuration "80_40", whose rows are frontend_fbank.npz's `fbank/<name>` (the generator checks that
    they are the same bits, so the fixture does not store them twice)."""
    key = f"fbank/{tag}/{name}"
    return g[key] if key in g.files else fbank_golden["fbank/" + name]


def mfcc_tolerance(ref_logmel: np.ndarray, table: np.ndarray) -> np.ndarray:
    """Per-coefficient bound [frames, n_ceps] on |mfcc - mfcc_ref| for any implementation whose mel powers meet the
    fbank tolerance |p - p_ref| <= 1e-4 p_ref + 1e-6 max_frame(p_ref) (tests/test_oracle_golden.power_close).
    Through the log that is delta_m = log1p(1e-4 + 1e-6 P_max / P_m) per mel bin, carried through the linear map:
    sum_m |A[m, i]| delta_m.  Plus fp32 rounding of the two DCT products (the reference rounds y @ D and the lifter
    product, an implementation rounds its own sum): 2 (n_mels + 2) u sum_m |y_m| |A[m, i]|."""
    y = ref_logmel.astype(np.float64)
    p = np.exp(y)
    delta = np.log1p(1e-4 + 1e-6 * p.max(axis=1, keepdims=True) / p)
    a = np.abs(table.astype(np.float64))
    return delta @ a + 2 * (y.shape[1] + 2) * U32 * (np.abs(y) @ a)


def epilogue_tolerance(logmel: np.ndarray, table: np.ndarray) -> np.ndarray:
    """Bound on |fp32 sum_m y_m A[m, i] - exact| for a sequential fp32 sum over n_mels terms: gamma_n sum |y_m A|."""
    n = logmel.shape[1]
    gamma = n * U32 / (1 - n * U32)
    return gamma * (np.abs(logmel.astype(np.float64)) @ np.abs(table.astype(np.float64)))
