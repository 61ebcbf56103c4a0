"""Generates tests/golden/mfcc.npz FROM THE REFERENCE'S MFCC stage (touchnet/data/functions.py:137-156).

    TOUCHNET_REF=/path/to/TouchNet python tests/golden/make_golden_mfcc.py

What is executed
  mfcc/<cfg>/<name>    the reference's audio_compute_mfcc (torchaudio.compliance.kaldi.mfcc as installed) on the
                       waveforms of frontend_fbank.npz (`wav/<name>`) - all of them for the configurations the recipes
                       use, a few for the edge configurations - for every configuration of CONFIGS; the 8 kHz one reads
                       the same samples as 8 kHz audio (n_fft 256, the table-DFT path of the GPU frontend).
  fbank/<cfg>/<name>   kaldi.fbank with the same mel bins / low / high frequency: the log-mel row MFCC is computed from,
                       from which the tests derive their tolerance.  Not stored for "80_40": those rows are
                       frontend_fbank.npz's `fbank/<name>` (checked here to be the same bits), see
                       tests/mfcc_oracle.reference_logmel.
  config/<cfg>         the configuration as JSON.
  chain/*              a seeded run of the reference's lazily chained stages audio_compute_mfcc -> audiofeat_spec_aug ->
                       audiofeat_spec_sub -> audiofeat_spec_trim -> audiofeat_stack on a few 16 kHz int16 utterances,
                       every intermediate stored, with `chain/fbank/<i>` as above, the log of every draw the stages made
                       (`chain/draws`: kind 1 = randint; a, b, result) and the `random.random()` drawn after the chain.
The archive is written with fixed entry timestamps and one torch thread, so running this again reproduces it bit for bit.
"""
import json
import os
import random
import sys
import types
import zipfile

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from make_golden import HERE, import_reference  # noqa: E402  (exits with a message when TOUCHNET_REF is unset)
from make_golden_augment import DrawLog, pcm  # noqa: E402

BASE = dict(audiofeat_frame_length=25, audiofeat_frame_shift=10, audiofeat_dither=0.0, audiofeat_low_freq=20.0,
            audiofeat_high_freq=0.0)
EDGE_WAVES = ("short", "noise_odd")      # the edge configurations run on these (keeps the fixture small)
CONFIGS = {   # tag -> (sample rate, config, waveforms; None = every waveform of frontend_fbank.npz)
    "80_40": (16000, dict(BASE, audiofeat_num_mel_bins=80, audiofeat_num_ceps=40), None),
    "23_13": (16000, dict(BASE, audiofeat_num_mel_bins=23, audiofeat_num_ceps=13), None),
    "40_40_hf-400": (16000, dict(BASE, audiofeat_num_mel_bins=40, audiofeat_num_ceps=40, audiofeat_high_freq=-400.0),
                     EDGE_WAVES),
    "8k_80_40": (8000, dict(BASE, audiofeat_num_mel_bins=80, audiofeat_num_ceps=40), EDGE_WAVES),
}
SEED = 20261016
CHAIN = dict(BASE, audio_feat_type="mfcc", audiofeat_num_mel_bins=80, audiofeat_num_ceps=40, audiofeat_spec_aug=True,
             audiofeat_spec_aug_num_t_mask=2, audiofeat_spec_aug_num_f_mask=2, audiofeat_spec_aug_max_t=50,
             audiofeat_spec_aug_max_f=10, audiofeat_spec_sub=True, audiofeat_spec_sub_num_t_sub=3,
             audiofeat_spec_sub_max_t=30, audiofeat_spec_trim=True, audiofeat_spec_trim_max_t=20,
             audiofeat_stack_length=5, audiofeat_stride_length=4, audiofeat_normalize=True)
CHAIN_SECONDS = (0.3, 0.62, 0.41)     # the first is shorter than one 50-frame time mask


def kaldi_fbank(wav, sr, cfg):
    import torchaudio
    return torchaudio.compliance.kaldi.fbank(
        torch.from_numpy(wav)[None] * (1 << 15), num_mel_bins=cfg["audiofeat_num_mel_bins"],
        frame_length=cfg["audiofeat_frame_length"], frame_shift=cfg["audiofeat_frame_shift"], dither=0.0,
        energy_floor=0.0, low_freq=cfg["audiofeat_low_freq"], high_freq=cfg["audiofeat_high_freq"],
        sample_frequency=sr).numpy()


def save_npz(path, arrays):
    """np.savez_compressed with fixed entry timestamps (numpy stamps the current time)."""
    with zipfile.ZipFile(path, "w", zipfile.ZIP_DEFLATED) as z:
        for k in sorted(arrays):
            info = zipfile.ZipInfo(k + ".npy", date_time=(1980, 1, 1, 0, 0, 0))
            info.compress_type = zipfile.ZIP_DEFLATED
            with z.open(info, "w", force_zip64=True) as f:
                np.lib.format.write_array(f, np.asanyarray(arrays[k]), allow_pickle=False)


def main():
    functions = import_reference()
    torch.set_num_threads(1)
    fb = np.load(os.path.join(HERE, "frontend_fbank.npz"))
    names = sorted(k[4:] for k in fb.files if k.startswith("wav/"))
    out = {}
    for tag, (sr, cfg, subset) in CONFIGS.items():
        out[f"config/{tag}"] = np.frombuffer(json.dumps(dict(cfg, sample_rate=sr)).encode(), dtype=np.uint8)
        for name in names if subset is None else subset:
            wav = fb["wav/" + name]
            s = next(functions.audio_compute_mfcc(iter([{"waveform": torch.from_numpy(wav)[None], "sample_rate": sr}]),
                                                  types.SimpleNamespace(**cfg)))
            out[f"mfcc/{tag}/{name}"] = s["audiofeat"].numpy().astype(np.float32)
            logmel = kaldi_fbank(wav, sr, cfg).astype(np.float32)
            if tag == "80_40":
                assert np.array_equal(logmel, fb["fbank/" + name]), name
            else:
                out[f"fbank/{tag}/{name}"] = logmel

    g = torch.Generator().manual_seed(11)
    pcms = [pcm(int(d * 16000), 16000, g) for d in CHAIN_SECONDS]
    samples = [{"waveform": torch.from_numpy(x.astype(np.float32) / 32768.0)[None], "sample_rate": 16000} for x in pcms]
    taps = {k: [] for k in ("mfcc", "spec_aug", "spec_sub", "spec_trim", "stack")}

    def tap(gen, name):
        for s in gen:
            taps[name].append(s["audiofeat"].clone())
            yield s

    cfg = types.SimpleNamespace(**CHAIN)
    log = DrawLog()
    functions.random = log
    random.seed(SEED)
    d = tap(functions.audio_compute_mfcc(iter(samples), cfg), "mfcc")
    d = tap(functions.audiofeat_spec_aug(d, cfg), "spec_aug")
    d = tap(functions.audiofeat_spec_sub(d, cfg), "spec_sub")
    d = tap(functions.audiofeat_spec_trim(d, cfg), "spec_trim")
    d = tap(functions.audiofeat_stack(d, cfg), "stack")
    assert len(list(d)) == len(samples)
    out["chain/post_random"] = np.array(random.random())
    out["chain/seed"] = np.array(SEED)
    out["chain/config_json"] = np.frombuffer(json.dumps(CHAIN).encode(), dtype=np.uint8)
    out["chain/draws"] = np.array(log.log, dtype=np.float64)
    for i, x in enumerate(pcms):
        out[f"chain/pcm/{i}"] = x
        out[f"chain/fbank/{i}"] = kaldi_fbank(x.astype(np.float32) / 32768.0, 16000, CHAIN).astype(np.float32)
        for name, vals in taps.items():
            out[f"chain/{name}/{i}"] = vals[i].numpy().astype(np.float32)
    path = os.path.join(HERE, "mfcc.npz")
    save_npz(path, out)
    print(path, os.path.getsize(path), "bytes;", len(log.log), "draws")


if __name__ == "__main__":
    main()
