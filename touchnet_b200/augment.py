"""Host side of the ASR recipe's data augmentation: the random draws, the length arithmetic and the resampling banks.

The reference chains its augmentation stages lazily, one sample at a time (ref: touchnet/data/datapipe.py:183-201;
order of touchnet/models/touch_audio/processing_touch_audio.py:453-476):

    audio_resample        ref: touchnet/data/functions.py:83-96     (torchaudio.transforms.Resample, no draw)
    audio_speed_perturb   ref: touchnet/data/functions.py:99-114    random.choice(speeds)
    audiofeat_spec_aug    ref: touchnet/data/functions.py:193-217   per time mask, then per freq mask: randint start, length
    audiofeat_spec_sub    ref: touchnet/data/functions.py:220-239   per sub: randint start, length, pos
    audiofeat_spec_trim   ref: touchnet/data/functions.py:242-255   randint length

How many draws a sample consumes, and their ranges, depend only on its length.  So `draw_record` makes them here, in the
DataLoader worker and in exactly the reference's order, from the waveform length alone; the result is a small record
that the GPU applies after the H2D copy (`frontend.augmented_fbank_stack_batch`; `augmented_mfcc_stack_batch` for
audio_feat_type "mfcc", whose frames are fbank's and whose frequency masks span the audiofeat_num_ceps columns;
`augmented_log_mel_stack_batch` for "log_mel_spectrogram", whose frames are (n + audiofeat_padding) // hop and whose
frequency masks span the audiofeat_num_mel_bins columns).  No tensor is touched on the host.
"""
from __future__ import annotations

import math
import random
from functools import lru_cache
from typing import Iterable, Iterator

import numpy as np
import torch

from ._lib import TouchNetB200Error

LOWPASS_FILTER_WIDTH = 6      # torchaudio.transforms.Resample defaults (the reference passes only the two rates)
ROLLOFF = 0.99


# ---------------------------------------------------------------------------------------------------------------
# resampling: lengths and the sinc filter bank of torchaudio.transforms.Resample
# ---------------------------------------------------------------------------------------------------------------
def reduced_ratio(orig: int, new: int) -> tuple[int, int]:
    g = math.gcd(int(orig), int(new))
    return int(orig) // g, int(new) // g


def resampled_length(n: int, orig: int, new: int) -> int:
    """Output length of torchaudio's resampling: ceil(new*n/orig) after the gcd reduction, rounded through fp32 as
    torch.ceil(torch.as_tensor(...)) rounds it (ta: functional/functional.py _apply_sinc_resample_kernel)."""
    if orig == new:
        return int(n)
    o, w = reduced_ratio(orig, new)
    return int(math.ceil(float(np.float32(w * int(n) / o))))


def speed_source_rate(sample_rate: int, speed: float) -> int:
    """sox `speed s` then `rate sr` is resampling from sr*s to sr; sr*s must be an integer rate."""
    r = sample_rate * float(speed)
    ri = int(round(r))
    if ri <= 0 or abs(r - ri) > 1e-6 * max(1.0, abs(r)):
        raise TouchNetB200Error(f"speed perturbation needs sample_rate*speed to be an integer rate, got "
                                f"{sample_rate}*{speed} = {r}")
    return ri


@lru_cache(maxsize=None)
def sinc_resample_bank(orig: int, new: int, device: str = "cpu") -> tuple[torch.Tensor, int]:
    """The bank torchaudio.transforms.Resample(orig, new) caches (sinc_interp_hann, lowpass_filter_width 6, rolloff 0.99,
    computed in float64 and stored as float32), as [new', 2*width + orig'] with (orig', new') the gcd-reduced rates.
    Output sample i*new' + j is sum_k bank[j, k] * x[i*orig' - width + k].  Same op sequence as
    ta: functional/functional.py _get_sinc_resample_kernel, so the bank is bit-identical to it."""
    o, n = reduced_ratio(orig, new)
    base = min(o, n) * ROLLOFF
    width = math.ceil(LOWPASS_FILTER_WIDTH * o / base)
    idx = torch.arange(-width, width + o, dtype=torch.float64)[None, None] / o
    # the phase offsets are an integer arange divided in the default float dtype, then promoted by the float64 idx
    t = torch.arange(0, -n, -1)[:, None, None] / n + idx
    t *= base
    t = t.clamp_(-LOWPASS_FILTER_WIDTH, LOWPASS_FILTER_WIDTH)
    window = torch.cos(t * math.pi / LOWPASS_FILTER_WIDTH / 2) ** 2
    t *= math.pi
    scale = base / o
    bank = torch.where(t == 0, torch.tensor(1.0).to(t), t.sin() / t)
    bank *= window * scale
    return bank.to(torch.float32).reshape(n, 2 * width + o).contiguous().to(device), width


# ---------------------------------------------------------------------------------------------------------------
# feature lengths
# ---------------------------------------------------------------------------------------------------------------
def _kaldi_frames(n_samples: int, sample_rate: int, config) -> int:
    """snip_edges framing of kaldi fbank, which kaldi mfcc shares."""
    win = int(sample_rate * config.audiofeat_frame_length * 0.001)
    shift = int(sample_rate * config.audiofeat_frame_shift * 0.001)
    return 0 if n_samples < win else 1 + (n_samples - win) // shift


def feature_frames(n_samples: int, sample_rate: int, config) -> int:
    """Frames the configured feature extractor produces for n_samples (fbank: snip_edges framing; whisper log-mel:
    (n + padding) // hop, ref: functions.py:159-190)."""
    kind = getattr(config, "audio_feat_type", "fbank")
    if kind == "fbank":
        return _kaldi_frames(n_samples, sample_rate, config)
    if kind == "log_mel_spectrogram":
        return (n_samples + getattr(config, "audiofeat_padding", 0)) // config.audiofeat_hop_length
    raise TouchNetB200Error(f"augmentation records support audio_feat_type fbank / log_mel_spectrogram, not {kind!r}")


def stacked_rows(frames: int, stride: int) -> int:
    return int(math.ceil(frames / stride)) if frames > 0 else 0


# ---------------------------------------------------------------------------------------------------------------
# the draws
# ---------------------------------------------------------------------------------------------------------------
def draw_time_freq_masks(max_frames: int, max_freq: int, config, rng=random):
    """ref: functions.py:204-215 - per time mask, then per freq mask: start, length; end = min(max, start + length)."""
    t_masks, f_masks = [], []
    for _ in range(config.audiofeat_spec_aug_num_t_mask):
        start = rng.randint(0, max_frames - 1)
        length = rng.randint(1, config.audiofeat_spec_aug_max_t)
        t_masks.append((start, min(max_frames, start + length)))
    for _ in range(config.audiofeat_spec_aug_num_f_mask):
        start = rng.randint(0, max_freq - 1)
        length = rng.randint(1, config.audiofeat_spec_aug_max_f)
        f_masks.append((start, min(max_freq, start + length)))
    return t_masks, f_masks


def draw_subs(max_frames: int, config, rng=random):
    """ref: functions.py:231-237 - per sub: start, length, pos; frames [start, end) take frames [start-pos, end-pos)."""
    subs = []
    for _ in range(config.audiofeat_spec_sub_num_t_sub):
        start = rng.randint(0, max_frames - 1)
        length = rng.randint(1, config.audiofeat_spec_sub_max_t)
        end = min(max_frames, start + length)
        pos = rng.randint(0, start)
        subs.append((start, end, pos))
    return subs


def draw_trim(max_frames: int, config, rng=random) -> int:
    """ref: functions.py:250-254 - frames cut from the tail (0 when the draw is not below half the length)."""
    length = rng.randint(1, config.audiofeat_spec_trim_max_t)
    return length if length < max_frames / 2 else 0


def draw_record(n_samples: int, sample_rate: int, config, rng=random) -> dict:
    """All draws of one sample, in the reference's order, plus the lengths they imply.

    Returns {resample: (orig, new) | None, speed, t_masks [(start, end)], f_masks [(start, end)],
    subs [(start, end, pos)], trim, sample_rate (the rate the features are computed at), num_samples (after resampling
    and speed perturbation), num_frames (feature frames before trim), num_feat_frames (stacked rows)}."""
    if getattr(config, "audiofeat_dither", 0.0) != 0.0:
        raise TouchNetB200Error("dither != 0 is not supported (all reference recipes use 0.0)")
    n, sr = int(n_samples), int(sample_rate)
    rec = {"resample": None, "speed": 1.0, "t_masks": [], "f_masks": [], "subs": [], "trim": 0}
    target = getattr(config, "audio_resample_rate", None)
    if target is not None and sr != int(target):
        rec["resample"] = (sr, int(target))
        n, sr = resampled_length(n, sr, int(target)), int(target)
    if getattr(config, "audio_speed_perturb", False):
        speed = rng.choice(config.audio_speed_perturb_speeds)
        rec["speed"] = float(speed)
        if speed != 1.0:
            n = resampled_length(n, speed_source_rate(sr, speed), sr)
    mfcc = getattr(config, "audio_feat_type", "fbank") == "mfcc"
    frames = _kaldi_frames(n, sr, config) if mfcc else feature_frames(n, sr, config)
    if getattr(config, "audiofeat_spec_aug", False):
        # frequency masks span the feature's columns (y.size(1) of ref: functions.py:203)
        n_freq = config.audiofeat_num_ceps if mfcc else config.audiofeat_num_mel_bins
        rec["t_masks"], rec["f_masks"] = draw_time_freq_masks(frames, n_freq, config, rng)
    if getattr(config, "audiofeat_spec_sub", False):
        rec["subs"] = draw_subs(frames, config, rng)
    if getattr(config, "audiofeat_spec_trim", False):
        rec["trim"] = draw_trim(frames, config, rng)
    rec.update(sample_rate=sr, num_samples=n, num_frames=frames,
               num_feat_frames=stacked_rows(frames - rec["trim"], config.audiofeat_stride_length))
    return rec


def record_has_feature_ops(rec: dict) -> bool:
    return bool(rec["t_masks"] or rec["f_masks"] or rec["subs"] or rec["trim"])


def draw_stage(data: Iterable[dict], config) -> Iterator[dict]:
    """DataLoader-worker stage: attaches `augment` (the record of `draw_record`) and `num_feat_frames` to each sample and
    leaves the waveform as it is, so the raw (e.g. int16) waveform is shipped and the GPU applies the record after the
    H2D copy.  Stands in for audio_resample .. audiofeat_spec_trim of the reference chain; batching.plan_documents reads
    `num_feat_frames`, so placement follows the augmented lengths."""
    for sample in data:
        assert "sample_rate" in sample
        assert "waveform" in sample
        rec = draw_record(sample["waveform"].shape[-1], sample["sample_rate"], config)
        sample["augment"] = rec
        sample["num_feat_frames"] = rec["num_feat_frames"]
        yield sample
