"""CPU: the host half of the data augmentation (touchnet_b200/augment.py) against tests/golden/augment.npz, made from the
reference's own stages: the draws in the reference's order, the lengths they imply, the sinc banks, and the oracle's
application of the records; plus argument errors (the C ABI validates before touching the device)."""
import ctypes
import json
import math
import os
import random
from types import SimpleNamespace as NS

import numpy as np
import pytest
import torch

from tests import augment_oracle as ao
from touchnet_b200 import _lib, augment, frontend


@pytest.fixture(scope="module")
def golden(golden_dir):
    return np.load(os.path.join(golden_dir, "augment.npz"))


def chain_config(g):
    return NS(**json.loads(bytes(g["chain/config_json"]).decode()))


def n_chain(g):
    return len([k for k in g.files if k.startswith("chain/pcm/")])


class DrawLog:
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


def chain_records(g):
    cfg = chain_config(g)
    log = DrawLog()
    random.seed(int(g["chain/seed"]))
    recs = [augment.draw_record(g[f"chain/pcm/{i}"].shape[0], 16000, cfg, rng=log) for i in range(n_chain(g))]
    return recs, log.log, random.random()


def test_host_draws_reproduce_the_reference_chain(golden):
    recs, log, post = chain_records(golden)
    assert np.array_equal(np.array(log, dtype=np.float64), golden["chain/draws"])
    assert post == float(golden["chain/post_random"])       # same number of draws consumed
    speeds = [r[3] for r in log if r[0] == 0]
    assert [r["speed"] for r in recs] == speeds
    assert any(r["trim"] for r in recs) and not all(r["trim"] for r in recs)


def test_lengths_match_the_reference_chain(golden):
    recs, _, _ = chain_records(golden)
    for i, r in enumerate(recs):
        assert r["resample"] is None
        assert r["num_samples"] == golden[f"chain/speed_wav/{i}"].shape[0]
        assert r["num_frames"] == golden[f"chain/fbank/{i}"].shape[0]
        assert r["num_frames"] - r["trim"] == golden[f"chain/spec_trim/{i}"].shape[0]
        assert r["num_feat_frames"] == golden[f"chain/stack/{i}"].shape[0]
    for sr in (8000, 22050, 44100, 48000):
        n = golden[f"resample/{sr}/pcm"].shape[0]
        assert augment.resampled_length(n, sr, 16000) == golden[f"resample/{sr}/out"].shape[0]
        rec = augment.draw_record(n, sr, NS(audio_resample_rate=16000, audiofeat_frame_length=25,
                                            audiofeat_frame_shift=10, audiofeat_stride_length=4))
        assert rec["resample"] == (sr, 16000) and rec["num_samples"] == golden[f"resample/{sr}/out"].shape[0]


def test_oracle_application_of_the_records_is_bit_exact(golden):
    recs, _, _ = chain_records(golden)
    for i, r in enumerate(recs):
        fb = golden[f"chain/fbank/{i}"]
        masks_only = dict(r, subs=[], trim=0)
        no_trim = dict(r, trim=0)
        assert np.array_equal(ao.apply_record(fb, masks_only), golden[f"chain/spec_aug/{i}"])
        assert np.array_equal(ao.apply_record(fb, no_trim), golden[f"chain/spec_sub/{i}"])
        assert np.array_equal(ao.apply_record(fb, r), golden[f"chain/spec_trim/{i}"])


def test_oracle_resample_matches_the_reference(golden):
    for sr in (8000, 22050, 44100, 48000):
        x = golden[f"resample/{sr}/pcm"].astype(np.float32) / 32768.0
        ref = golden[f"resample/{sr}/out"]
        y = ao.resample(x, sr, 16000)
        assert y.shape == ref.shape
        assert np.all(np.abs(y.astype(np.float64) - ref) <= ao.resample_tolerance(x, sr, 16000, ref)), sr
    recs, _, _ = chain_records(golden)
    for i, r in enumerate(recs):
        x = golden[f"chain/pcm/{i}"].astype(np.float32) / 32768.0
        ref = golden[f"chain/speed_wav/{i}"]
        if r["speed"] == 1.0:
            assert np.array_equal(x, ref)
            continue
        src = augment.speed_source_rate(16000, r["speed"])
        y = ao.resample(x, src, 16000)
        assert np.all(np.abs(y.astype(np.float64) - ref) <= ao.resample_tolerance(x, src, 16000, ref)), i


@pytest.mark.parametrize("orig,new,shape", [(17600, 16000, (10, 25)), (14400, 16000, (10, 23)),
                                            (48000, 16000, (1, 41)), (44100, 16000, (160, 475)),
                                            (22050, 16000, (320, 459)), (8000, 16000, (2, 15))])
def test_sinc_bank_equals_torchaudio(orig, new, shape):
    F = pytest.importorskip("torchaudio.functional.functional")
    bank, width = augment.sinc_resample_bank(orig, new)
    ref, ref_width = F._get_sinc_resample_kernel(orig, new, math.gcd(orig, new))
    assert tuple(bank.shape) == shape and width == ref_width
    assert torch.equal(bank, ref.reshape(shape))
    # the oracle's numpy restatement rounds to the same fp32 bank up to libm differences in sin / cos
    assert np.abs(ao.sinc_resample_bank(orig, new)[0].astype(np.float32) - bank.numpy()).max() <= 2 ** -24


def test_draws_only_for_enabled_stages_and_choice_even_at_speed_one():
    cfg = NS(audio_resample_rate=16000, audio_speed_perturb=True, audio_speed_perturb_speeds=[1.0],
             audiofeat_frame_length=25, audiofeat_frame_shift=10, audiofeat_stride_length=4)
    log = DrawLog()
    rec = augment.draw_record(16000, 16000, cfg, rng=log)
    assert [e[0] for e in log.log] == [0] and rec["speed"] == 1.0 and rec["num_samples"] == 16000
    assert rec["num_frames"] == 98 and rec["num_feat_frames"] == 25
    assert not augment.record_has_feature_ops(rec)


def test_draw_stage_attaches_records_without_touching_the_waveform():
    cfg = NS(audio_resample_rate=16000, audio_speed_perturb=True, audio_speed_perturb_speeds=[0.9, 1.0, 1.1],
             audiofeat_num_mel_bins=80, audiofeat_frame_length=25, audiofeat_frame_shift=10,
             audiofeat_spec_aug=True, audiofeat_spec_aug_num_t_mask=2, audiofeat_spec_aug_num_f_mask=2,
             audiofeat_spec_aug_max_t=50, audiofeat_spec_aug_max_f=10, audiofeat_spec_sub=True,
             audiofeat_spec_sub_num_t_sub=3, audiofeat_spec_sub_max_t=30, audiofeat_stride_length=4)
    wav = torch.zeros(1, 24000, dtype=torch.int16)
    s = next(augment.draw_stage(iter([{"waveform": wav, "sample_rate": 44100, "input_ids": [5]}]), cfg))
    assert s["waveform"] is wav
    assert s["augment"]["resample"] == (44100, 16000) and s["num_feat_frames"] == s["augment"]["num_feat_frames"]
    assert len(s["augment"]["t_masks"]) == 2 and len(s["augment"]["subs"]) == 3


def test_argument_errors():
    with pytest.raises(_lib.TouchNetB200Error, match="integer rate"):
        augment.speed_source_rate(16000, 1.00001)
    assert augment.speed_source_rate(16000, 1.1) == 17600
    with pytest.raises(_lib.TouchNetB200Error, match="dither"):
        augment.draw_record(16000, 16000, NS(audiofeat_dither=0.1))
    with pytest.raises(_lib.TouchNetB200Error, match="audio_feat_type"):
        augment.feature_frames(16000, 16000, NS(audio_feat_type="mfcc"))
    cfg = NS(audiofeat_num_mel_bins=80, audiofeat_frame_length=25, audiofeat_frame_shift=10, audiofeat_spec_aug=True,
             audiofeat_spec_aug_num_t_mask=1, audiofeat_spec_aug_num_f_mask=0, audiofeat_spec_aug_max_t=5,
             audiofeat_spec_aug_max_f=5, audiofeat_stride_length=4)
    with pytest.raises(ValueError):                          # randint(0, -1) on a zero-frame utterance, as the reference
        augment.draw_record(300, 16000, cfg)
    wav = torch.zeros(100)
    with pytest.raises(_lib.TouchNetB200Error, match="GPU"):
        frontend.resample_batch(wav, [100], 8000, 16000)
    with pytest.raises(_lib.TouchNetB200Error, match="GPU"):
        frontend.spec_augment_batch(torch.zeros(4, 80), [4], [{"trim": 0}])
    with pytest.raises(_lib.TouchNetB200Error, match="records"):
        frontend.augmented_fbank_stack_batch(wav, [50, 50], [])


def test_c_abi_argument_errors():
    table = (ctypes.c_int32 * 5)(11, 10, 7, 24, 0)            # taps != 2*width + orig
    ok_table = (ctypes.c_int32 * 5)(11, 10, 7, 25, 0)
    bad_calls = [
        ("tn_resample_f32", (None, 0, 8, 8, 8, 8, 1, 1, 1024, ok_table, 1, 8, 8, None), "null"),
        ("tn_resample_f32", (8, 0, 8, 8, 8, 8, 1, 1, 1024, ok_table, 0, 8, 8, None), "n_banks"),
        ("tn_resample_f32", (8, 0, 8, 8, 8, 8, 1, 1, 1000, ok_table, 1, 8, 8, None), "tile"),
        ("tn_resample_f32", (8, 0, 8, 8, 8, 8, 1, 1, 1024, table, 1, 8, 8, None), "taps"),
        ("tn_spec_augment_f32", (None, 8, 8, 1, 1, 80, None, 0, None, 0, None, 0, 8, None), "null"),
        ("tn_spec_augment_f32", (8, 8, 8, 1, 1, 80, None, 2, None, 0, None, 0, 8, None), "null mask"),
    ]
    for name, args, needle in bad_calls:
        with pytest.raises(_lib.TouchNetB200Error, match=needle):
            _lib.call(name, *args)
