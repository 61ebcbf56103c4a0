"""Generates tests/golden/logmel_chain.npz FROM THE REFERENCE'S log-mel stage (touchnet/data/functions.py:159-190).

    TOUCHNET_REF=/path/to/TouchNet python tests/golden/make_golden_logmel.py

What is executed
  logmel/<pad>/<name>/<n_mels>   the reference's audio_compute_log_mel_spectrogram (torch.stft as installed) on the
                                 waveforms of frontend_logmel.npz (`wav/<name>`) with audiofeat_padding = PADDING (not a
                                 multiple of the hop), at 80 and 128 mel bins.  At padding 0 the same call reproduces
                                 frontend_logmel.npz's `logmel/<name>/<n_mels>` bit for bit; the generator checks that
                                 instead of storing those arrays twice.
  chain/*                        a seeded run of the reference's lazily chained stages audio_speed_perturb ->
                                 audio_compute_log_mel_spectrogram -> audiofeat_spec_aug -> audiofeat_spec_sub ->
                                 audiofeat_spec_trim -> audiofeat_stack on a few 16 kHz int16 utterances, with
                                 audiofeat_padding = PADDING; every intermediate is stored, with the log of every draw the
                                 stages made (`chain/draws`: kind 0 = choice, 1 = randint; a, b, result) and the
                                 `random.random()` drawn after the chain.
librosa.filters.mel (absent here) is supplied by transformers.audio_utils.mel_filter_bank(norm="slaney",
mel_scale="slaney"), the independent implementation frontend_logmel.npz uses.  Speed perturbation's sox call is stubbed
by torchaudio's resampler as in make_golden_augment.py.  The archive is written with fixed entry timestamps and one
torch thread, so running this again reproduces it bit for bit.
"""
import json
import os
import random
import sys
import types

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from make_golden_augment import DrawLog, import_reference, pcm, sox_stub  # noqa: E402  (needs TOUCHNET_REF)
from make_golden import HERE  # noqa: E402
from make_golden_mfcc import save_npz  # noqa: E402

PADDING = 250
BASE = dict(audiofeat_n_fft=400, audiofeat_hop_length=160)
SEED = 20261033
CHAIN = dict(BASE, audio_speed_perturb=True, audio_speed_perturb_speeds=[0.9, 1.0, 1.1],
             audio_feat_type="log_mel_spectrogram", audiofeat_num_mel_bins=80, audiofeat_padding=PADDING,
             audiofeat_spec_aug=True, audiofeat_spec_aug_num_t_mask=2, audiofeat_spec_aug_num_f_mask=2,
             audiofeat_spec_aug_max_t=50, audiofeat_spec_aug_max_f=10, audiofeat_spec_sub=True,
             audiofeat_spec_sub_num_t_sub=3, audiofeat_spec_sub_max_t=30, audiofeat_spec_trim=True,
             audiofeat_spec_trim_max_t=20, audiofeat_stack_length=5, audiofeat_stride_length=4,
             audiofeat_normalize=True)
CHAIN_SECONDS = (0.3, 0.52, 0.27)     # the first and last are shorter than one 50-frame time mask


def slaney_mel(sr, n_fft, n_mels):
    from transformers.audio_utils import mel_filter_bank
    return mel_filter_bank(num_frequency_bins=1 + n_fft // 2, num_mel_filters=n_mels, min_frequency=0.0,
                           max_frequency=sr / 2.0, sampling_rate=sr, norm="slaney",
                           mel_scale="slaney").T.astype(np.float32)


def main():
    functions = import_reference()
    import torchaudio
    torchaudio.sox_effects = types.SimpleNamespace(apply_effects_tensor=sox_stub)
    functions.librosa = types.SimpleNamespace(filters=types.SimpleNamespace(mel=slaney_mel))
    torch.set_num_threads(1)
    lm = np.load(os.path.join(HERE, "frontend_logmel.npz"))
    names = sorted(k[4:] for k in lm.files if k.startswith("wav/"))
    out = {"padding": np.array(PADDING)}
    for name in names:
        for n_mels in (80, 128):
            for pad in (0, PADDING):
                cfg = types.SimpleNamespace(**BASE, audiofeat_num_mel_bins=n_mels, audiofeat_padding=pad)
                s = next(functions.audio_compute_log_mel_spectrogram(
                    iter([{"waveform": torch.from_numpy(lm["wav/" + name])[None], "sample_rate": 16000}]), cfg))
                y = s["audiofeat"].contiguous().numpy().astype(np.float32)
                if pad == 0:
                    assert np.array_equal(y, lm[f"logmel/{name}/{n_mels}"]), (name, n_mels)
                else:
                    out[f"logmel/{pad}/{name}/{n_mels}"] = y

    g = torch.Generator().manual_seed(13)
    pcms = [pcm(int(d * 16000), 16000, g) for d in CHAIN_SECONDS]
    samples = [{"waveform": torch.from_numpy(x.astype(np.float32) / 32768.0)[None], "sample_rate": 16000} for x in pcms]
    taps = {k: [] for k in ("speed_wav", "logmel", "spec_aug", "spec_sub", "spec_trim", "stack")}

    def tap(gen, key, name):
        for s in gen:
            taps[name].append(s[key].clone())
            yield s

    cfg = types.SimpleNamespace(**CHAIN)
    log = DrawLog()
    functions.random = log
    random.seed(SEED)
    d = tap(functions.audio_speed_perturb(iter(samples), cfg), "waveform", "speed_wav")
    d = tap(functions.audio_compute_log_mel_spectrogram(d, cfg), "audiofeat", "logmel")
    d = tap(functions.audiofeat_spec_aug(d, cfg), "audiofeat", "spec_aug")
    d = tap(functions.audiofeat_spec_sub(d, cfg), "audiofeat", "spec_sub")
    d = tap(functions.audiofeat_spec_trim(d, cfg), "audiofeat", "spec_trim")
    d = tap(functions.audiofeat_stack(d, cfg), "audiofeat", "stack")
    assert len(list(d)) == len(samples)
    out["chain/post_random"] = np.array(random.random())
    out["chain/seed"] = np.array(SEED)
    out["chain/config_json"] = np.frombuffer(json.dumps(CHAIN).encode(), dtype=np.uint8)
    out["chain/draws"] = np.array(log.log, dtype=np.float64)
    for i, x in enumerate(pcms):
        out[f"chain/pcm/{i}"] = x
        for name, vals in taps.items():
            v = vals[i][0] if name == "speed_wav" else vals[i]
            out[f"chain/{name}/{i}"] = v.contiguous().numpy().astype(np.float32)
    path = os.path.join(HERE, "logmel_chain.npz")
    save_npz(path, out)
    print(path, os.path.getsize(path), "bytes;", len(log.log), "draws;",
          "speeds", [r[3] for r in log.log if r[0] == 0])


if __name__ == "__main__":
    main()
