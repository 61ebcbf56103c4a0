"""Generates tests/golden/augment.npz FROM THE REFERENCE'S augmentation functions (touchnet/data/functions.py:83-255).

    TOUCHNET_REF=/path/to/TouchNet python tests/golden/make_golden_augment.py

What is executed
  resample/<sr>/*   the reference's audio_resample stage (torchaudio.transforms.Resample as installed) on short seeded
                    int16 utterances at 8 / 22.05 / 44.1 / 48 kHz -> 16 kHz.
  chain/*           a seeded run of the reference's lazily chained stages audio_speed_perturb -> audio_compute_fbank ->
                    audiofeat_spec_aug -> audiofeat_spec_sub -> audiofeat_spec_trim -> audiofeat_stack on a few 16 kHz
                    int16 utterances (spec_trim on, which the ASR recipe leaves off), with the reference's module-level
                    `random` seeded.  Every intermediate output is stored, with a log of every draw the stages made
                    (`chain/draws`: kind 0 = choice, 1 = randint; a, b, result) and the `random.random()` drawn after the
                    chain, which pins how many draws were consumed.
The reference's speed perturbation calls torchaudio.sox_effects.apply_effects_tensor, which current torchaudio no longer
has.  Here it is STUBBED: `speed s` + `rate sr` is done as torchaudio.transforms.Resample(sr*s, sr), the restatement
the project implements (not sox's filter, whose output cannot be checked without sox).
"""
import json
import os
import random
import sys
import types

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from make_golden import HERE, import_reference  # noqa: E402  (exits with a message when TOUCHNET_REF is unset)

SEED = 20261015
CONFIG = dict(audio_resample_rate=16000, audio_speed_perturb=True, audio_speed_perturb_speeds=[0.9, 1.0, 1.1],
              audio_feat_type="fbank", audiofeat_num_mel_bins=80, audiofeat_frame_length=25, audiofeat_frame_shift=10,
              audiofeat_dither=0.0, audiofeat_spec_aug=True, audiofeat_spec_aug_num_t_mask=2,
              audiofeat_spec_aug_num_f_mask=2, audiofeat_spec_aug_max_t=50, audiofeat_spec_aug_max_f=10,
              audiofeat_spec_sub=True, audiofeat_spec_sub_num_t_sub=3, audiofeat_spec_sub_max_t=30,
              audiofeat_spec_trim=True, audiofeat_spec_trim_max_t=20, audiofeat_stack_length=5,
              audiofeat_stride_length=4, audiofeat_normalize=True)
CHAIN_SECONDS = (0.3, 0.62, 0.41, 0.55, 0.35, 0.48)     # the first is shorter than one 50-frame time mask


def pcm(n, sr, g):
    t = np.arange(n, dtype=np.float64) / sr
    x = 0.4 * np.sin(2 * np.pi * (150.0 + 0.2 * sr * t) * t) + 0.1 * (2 * torch.rand(n, generator=g).double().numpy() - 1)
    return np.round(x * 32767).astype(np.int16)


class DrawLog:
    """Stands in for the `random` module inside the reference's functions and logs every draw."""

    def __init__(self):
        self.log = []

    def choice(self, seq):
        r = random.choice(seq)
        self.log.append((0, 0, len(seq), float(r)))
        return r

    def randint(self, a, b):
        r = random.randint(a, b)
        self.log.append((1, a, b, r))
        return r


def sox_stub(waveform, sample_rate, effects):
    import torchaudio
    assert [e[0] for e in effects] == ["speed", "rate"]
    src = int(round(sample_rate * float(effects[0][1])))
    rate = int(effects[1][1])
    return torchaudio.transforms.Resample(src, rate)(waveform), rate


def main():
    functions = import_reference()
    import torchaudio
    torchaudio.sox_effects = types.SimpleNamespace(apply_effects_tensor=sox_stub)
    cfg = types.SimpleNamespace(**CONFIG)
    g = torch.Generator().manual_seed(7)
    out = {}
    for sr in (8000, 22050, 44100, 48000):
        x = pcm(int(0.25 * sr), sr, g)
        s = next(functions.audio_resample(iter([{"waveform": torch.from_numpy(x.astype(np.float32) / 32768.0)[None],
                                                  "sample_rate": sr}]), cfg))
        assert s["sample_rate"] == 16000
        out[f"resample/{sr}/pcm"] = x
        out[f"resample/{sr}/out"] = s["waveform"][0].numpy().astype(np.float32)

    pcms = [pcm(int(d * 16000), 16000, g) for d in CHAIN_SECONDS]
    samples = [{"waveform": torch.from_numpy(x.astype(np.float32) / 32768.0)[None], "sample_rate": 16000} for x in pcms]
    taps = {k: [] for k in ("speed_wav", "fbank", "spec_aug", "spec_sub", "spec_trim", "stack")}

    def tap(gen, key, name):
        for s in gen:
            taps[name].append(s[key].clone())
            yield s

    log = DrawLog()
    functions.random = log
    random.seed(SEED)
    d = tap(functions.audio_speed_perturb(iter(samples), cfg), "waveform", "speed_wav")
    d = tap(functions.audio_compute_fbank(d, cfg), "audiofeat", "fbank")
    d = tap(functions.audiofeat_spec_aug(d, cfg), "audiofeat", "spec_aug")
    d = tap(functions.audiofeat_spec_sub(d, cfg), "audiofeat", "spec_sub")
    d = tap(functions.audiofeat_spec_trim(d, cfg), "audiofeat", "spec_trim")
    d = tap(functions.audiofeat_stack(d, cfg), "audiofeat", "stack")
    assert len(list(d)) == len(samples)
    out["chain/post_random"] = np.array(random.random())
    out["chain/seed"] = np.array(SEED)
    out["chain/config_json"] = np.frombuffer(json.dumps(CONFIG).encode(), dtype=np.uint8)
    out["chain/draws"] = np.array(log.log, dtype=np.float64)
    for i, x in enumerate(pcms):
        out[f"chain/pcm/{i}"] = x
        for name, vals in taps.items():
            v = vals[i][0] if name == "speed_wav" else vals[i]
            out[f"chain/{name}/{i}"] = v.numpy().astype(np.float32)
    path = os.path.join(HERE, "augment.npz")
    np.savez_compressed(path, **out)
    print(path, os.path.getsize(path), "bytes;", len(log.log), "draws;",
          "speeds", [r[3] for r in log.log if r[0] == 0])


if __name__ == "__main__":
    main()
