"""CPU: the host half of MFCC - the numpy oracle and the DCT table against tests/golden/mfcc.npz (the reference's own
audio_compute_mfcc outputs, tests/golden/make_golden_mfcc.py), the augmentation draws of an MFCC recipe against the
reference chain's draw log, and argument errors (the C ABI validates before touching the device)."""
import json
import os
import random
from types import SimpleNamespace as NS

import numpy as np
import pytest
import torch

from tests import mfcc_oracle as mo
from tests.test_augment_cpu import DrawLog
from tests.test_oracle_golden import power_close
from touchnet_b200 import _lib, augment, frontend

TAGS = ("80_40", "23_13", "40_40_hf-400", "8k_80_40")


@pytest.fixture(scope="module")
def golden(golden_dir):
    return np.load(os.path.join(golden_dir, "mfcc.npz"))


@pytest.fixture(scope="module")
def fbank_golden(golden_dir):
    return np.load(os.path.join(golden_dir, "frontend_fbank.npz"))


@pytest.fixture(scope="module")
def waves(fbank_golden):
    return {k[4:]: fbank_golden[k] for k in fbank_golden.files if k.startswith("wav/")}


def config(g, tag):
    return json.loads(bytes(g[f"config/{tag}"]).decode())


@pytest.mark.parametrize("tag", TAGS)
def test_oracle_matches_the_reference(golden, fbank_golden, waves, tag):
    """The oracle's log-mel row meets the fbank power tolerance and its MFCC the derived bound of test_gpu_mfcc.py."""
    c = config(golden, tag)
    n_mels, n_ceps = c["audiofeat_num_mel_bins"], c["audiofeat_num_ceps"]
    a = mo.mfcc_table(n_mels, n_ceps)
    names = [k.split("/")[-1] for k in golden.files if k.startswith(f"mfcc/{tag}/")]
    assert names and set(names) <= set(waves)
    if tag == "80_40":                                         # the recipes' configuration covers every waveform
        assert len(names) == len(waves)
    for n in names:
        args = (waves[n], c["sample_rate"], n_mels)
        edges = dict(low_freq=c["audiofeat_low_freq"], high_freq=c["audiofeat_high_freq"])
        fb_ref, ref = mo.reference_logmel(golden, fbank_golden, tag, n), golden[f"mfcc/{tag}/{n}"]
        assert power_close(fb_ref, mo.fbank(*args, **edges)) < 1.0, n
        y = mo.mfcc(*args, num_ceps=n_ceps, **edges)
        assert y.shape == ref.shape, n
        assert np.all(np.abs(y.astype(np.float64) - ref) <= mo.mfcc_tolerance(fb_ref, a)), n


def test_default_oracle_fbank_is_the_existing_one(waves):
    from oracle import frontend_oracle as fo
    for w in waves.values():
        assert np.array_equal(mo.fbank(w), fo.fbank(w))


@pytest.mark.parametrize("n_mels,n_ceps", [(80, 40), (23, 13), (40, 40), (128, 128), (80, 1)])
def test_host_table_is_torchaudios_dct_times_lifter(n_mels, n_ceps):
    """The table equals torchaudio's _get_dct_matrix * _get_lifter_coeffs folded in fp64 and rounded once (so within
    an ulp of their fp32 product, what kaldi.mfcc multiplies by).  Against the fp64 oracle table the difference is
    torchaudio's fp32 cosine argument pi/n (m + 1/2) k <= pi k, rounded three times: 3 u pi k, times the column's
    scale sqrt(2/n) * lifter; its fp32 lifter 1 + 11 sin(pi k / 22), whose argument carries 3 u pi k / 22, times
    |D| <= sqrt(2/n); plus the final roundings."""
    K = pytest.importorskip("torchaudio.compliance.kaldi")
    a = frontend._kaldi_mfcc_table(n_mels, n_ceps)
    d, lift = K._get_dct_matrix(n_ceps, n_mels), K._get_lifter_coeffs(n_ceps, 22.0)
    assert tuple(a.shape) == (n_mels, n_ceps) and a.dtype == torch.float32
    assert torch.equal(a, (d.double() * lift.double()).float())
    ulp = np.spacing(np.abs(a.numpy()))
    assert np.all(np.abs(a.numpy() - (d * lift).numpy()) <= ulp)
    k = np.arange(n_ceps, dtype=np.float64)
    bound = np.sqrt(2.0 / n_mels) * (np.abs(lift.double().numpy()) * (3 * mo.U32 * np.pi * k + 4 * mo.U32)
                                     + 11.0 * (3 * mo.U32 * np.pi * k / 22.0 + 2 * mo.U32)) + 2 * ulp
    assert np.all(np.abs(a.numpy().astype(np.float64) - mo.mfcc_table(n_mels, n_ceps)) <= bound)


def chain_records(g, rng):
    cfg = NS(**json.loads(bytes(g["chain/config_json"]).decode()))
    n = len([k for k in g.files if k.startswith("chain/pcm/")])
    random.seed(int(g["chain/seed"]))
    recs = [augment.draw_record(g[f"chain/pcm/{i}"].shape[0], 16000, cfg, rng=rng) for i in range(n)]
    return cfg, recs, random.random()


def test_mfcc_draws_reproduce_the_reference_chain(golden):
    """Same draws, in the same order and count, as the reference's MFCC chain; frames are fbank's and frequency masks
    stay inside the num_ceps columns (the reference draws them over y.size(1))."""
    log = DrawLog()
    cfg, recs, post = chain_records(golden, log)
    assert np.array_equal(np.array(log.log, dtype=np.float64), golden["chain/draws"])
    assert post == float(golden["chain/post_random"])
    f_bounds = [(a, b) for kind, a, b, _ in log.log if kind == 1 and b == cfg.audiofeat_num_ceps - 1]
    assert len(f_bounds) == 2 * len(recs)                     # every freq-mask start drawn over the 40 columns
    for i, r in enumerate(recs):
        assert r["num_frames"] == golden[f"chain/mfcc/{i}"].shape[0]
        assert r["num_frames"] - r["trim"] == golden[f"chain/spec_trim/{i}"].shape[0]
        assert r["num_feat_frames"] == golden[f"chain/stack/{i}"].shape[0]
        assert r["f_masks"] and all(0 <= s < e <= cfg.audiofeat_num_ceps for s, e in r["f_masks"])
    fb = dict(vars(cfg), audio_feat_type="fbank")
    fb_recs = [augment.draw_record(golden[f"chain/pcm/{i}"].shape[0], 16000, NS(**fb), rng=random.Random(0))
               for i in range(len(recs))]
    assert [r["num_frames"] for r in fb_recs] == [r["num_frames"] for r in recs]


def test_draw_stage_accepts_mfcc():
    cfg = NS(audio_feat_type="mfcc", audiofeat_num_mel_bins=80, audiofeat_num_ceps=13, audiofeat_frame_length=25,
             audiofeat_frame_shift=10, audiofeat_spec_aug=True, audiofeat_spec_aug_num_t_mask=1,
             audiofeat_spec_aug_num_f_mask=30, audiofeat_spec_aug_max_t=5, audiofeat_spec_aug_max_f=30,
             audiofeat_stride_length=4)
    s = next(augment.draw_stage(iter([{"waveform": torch.zeros(1, 16000), "sample_rate": 16000}]), cfg))
    rec = s["augment"]
    assert rec["num_frames"] == 98 and s["num_feat_frames"] == 25
    assert len(rec["f_masks"]) == 30 and all(0 <= a < b <= 13 for a, b in rec["f_masks"])


def test_argument_errors():
    wav = torch.zeros(16000)
    with pytest.raises(_lib.TouchNetB200Error, match="num_ceps"):
        frontend.mfcc_batch(wav, [16000], num_mel_bins=23, num_ceps=40)     # DataConfig's defaults, as the reference
    with pytest.raises(_lib.TouchNetB200Error, match="num_ceps"):
        frontend.mfcc_batch(wav, [16000], num_ceps=0)
    with pytest.raises(_lib.TouchNetB200Error, match="128"):
        frontend.mfcc_batch(wav, [16000], num_mel_bins=160, num_ceps=40)
    with pytest.raises(_lib.TouchNetB200Error, match="GPU"):
        frontend.mfcc_batch(wav, [16000])
    with pytest.raises(_lib.TouchNetB200Error, match="GPU"):
        frontend.augmented_mfcc_stack_batch(wav, [16000], [{"resample": None, "speed": 1.0, "t_masks": [],
                                                            "f_masks": [], "subs": [], "trim": 0}])
    cfg = NS(audiofeat_num_mel_bins=80, audiofeat_num_ceps=40, audiofeat_frame_length=25, audiofeat_frame_shift=10,
             audiofeat_low_freq=20.0, audiofeat_high_freq=0.0, audiofeat_dither=1.0)
    with pytest.raises(_lib.TouchNetB200Error, match="dither"):
        next(frontend.audio_compute_mfcc(iter([{"waveform": wav[None], "sample_rate": 16000}]), cfg))


def test_c_abi_argument_errors():
    #            wav i16 utt frm n  T  win shift nfft window mel n_mels pre  dct  n_ceps out stream
    ok = dict(wav=8, i16=0, utt=8, frm=8, n=1, T=1, win=400, shift=160, nfft=512, window=8, mel=8, n_mels=80,
              pre=0.97, dct=8, n_ceps=40, out=8, stream=None)
    bad = [(dict(dct=None), "null DCT"), (dict(n_ceps=0), "n_ceps"), (dict(n_ceps=81), "n_ceps"),
           (dict(n_mels=129, n_ceps=40), "n_mels"), (dict(nfft=1024), "geometry"), (dict(wav=None), "null pointer")]
    for change, needle in bad:
        args = dict(ok, **change)
        with pytest.raises(_lib.TouchNetB200Error, match=needle):
            _lib.call("tn_mfcc_f32", *args.values())
