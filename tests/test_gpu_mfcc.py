"""GPU: MFCC in the audio frontend (csrc/frontend.cu, the MFCC epilogue of the fbank kernels) through
touchnet_b200.frontend against tests/golden/mfcc.npz, which holds the reference's own audio_compute_mfcc outputs and a
seeded run of its MFCC augmentation chain (tests/golden/make_golden_mfcc.py).

Tolerances (tests/mfcc_oracle.py):
  against the reference  coefficient i of a frame within sum_m |A[m, i]| log1p(1e-4 + 1e-6 P_max / P_m) + fp32 DCT
                         rounding, A the folded table and P the reference's mel powers: the fbank power-domain tolerance
                         carried through the log and the linear map; plus relative L2 < 1e-4 per real recording.
  the epilogue alone     mfcc_batch against the fp64 product of fbank_batch (same parameters) and A: gamma_n sum |y A|,
                         the error of one sequential fp32 sum over n_mels terms.
  everything else        bit-identical (batch vs per-sample, int16 vs float, run to run, the chain's masks / subs / trim).
"""
import json
import os
import random
from types import SimpleNamespace as NS

import numpy as np
import pytest
import torch

from tests import mfcc_oracle as mo
from tests.gpu_util import require_cuda
from touchnet_b200 import augment, frontend as fe

pytestmark = pytest.mark.gpu

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


def kwargs(c):
    return dict(sample_rate=c["sample_rate"], num_mel_bins=c["audiofeat_num_mel_bins"], num_ceps=c["audiofeat_num_ceps"],
                low_freq=c["audiofeat_low_freq"], high_freq=c["audiofeat_high_freq"])


def table(c):
    return fe._kaldi_mfcc_table(c["audiofeat_num_mel_bins"], c["audiofeat_num_ceps"]).numpy()


def packed(arrays, dev):
    return fe._pack([torch.from_numpy(np.ascontiguousarray(a)) for a in arrays], dev)


def split(t, lens):
    return [y.numpy() for y in torch.split(t.cpu(), list(lens))]


@pytest.mark.parametrize("tag", TAGS)
def test_mfcc_matches_the_reference(golden, fbank_golden, waves, tag):
    """Every waveform of the fixture in one packed launch, within the derived per-coefficient bound; relative L2 error
    below 1e-4 on the real recordings.  8 kHz runs the table-DFT kernel, 16 kHz the FFT kernel."""
    dev = require_cuda()
    c = config(golden, tag)
    names = sorted(k.split("/")[-1] for k in golden.files if k.startswith(f"mfcc/{tag}/"))
    if tag == "80_40":
        assert sum(n.startswith("real_") for n in names) == 2
    wav, lens = packed([waves[n] for n in names], dev)
    out, frames = fe.mfcc_batch(wav, lens, **kwargs(c))
    a = table(c)
    for n, y in zip(names, split(out, frames)):
        ref = golden[f"mfcc/{tag}/{n}"]
        assert y.shape == ref.shape, n
        err = np.abs(y.astype(np.float64) - ref)
        tol = mo.mfcc_tolerance(mo.reference_logmel(golden, fbank_golden, tag, n), a)
        assert np.all(err <= tol), (n, float((err / tol).max()))
        if n.startswith("real_"):
            rel = np.linalg.norm(y.astype(np.float64) - ref) / np.linalg.norm(ref)
            assert rel < 1e-4, (n, rel)


@pytest.mark.parametrize("tag", TAGS)
def test_epilogue_is_the_log_mel_row_times_the_table(waves, golden, tag):
    """mfcc_batch == fp64(fbank_batch @ A) up to one fp32 sum over n_mels terms: catches scale, order or table errors
    the reference bound is too loose to see."""
    dev = require_cuda()
    c = config(golden, tag)
    wav, lens = packed(list(waves.values()), dev)
    kw = kwargs(c)
    out, frames = fe.mfcc_batch(wav, lens, **kw)
    fb, frames_fb = fe.fbank_batch(wav, lens, kw["sample_rate"], kw["num_mel_bins"], low_freq=kw["low_freq"],
                                   high_freq=kw["high_freq"])
    assert frames == frames_fb
    y = fb.cpu().numpy()
    a = table(c)
    want = y.astype(np.float64) @ a.astype(np.float64)
    err = np.abs(out.cpu().numpy().astype(np.float64) - want)
    assert np.all(err <= mo.epilogue_tolerance(y, a)), float(err.max())


def test_bit_identity_batch_stage_int16_and_run_to_run(waves):
    dev = require_cuda()
    names = sorted(waves)
    wavs = [waves[n] for n in names]
    pcms = [np.round(w * 32768.0).astype(np.int16) for w in wavs]
    wav16, lens = packed(pcms, dev)
    wavf, _ = packed([p.astype(np.float32) / 32768.0 for p in pcms], dev)
    a, frames = fe.mfcc_batch(wav16, lens)
    b, _ = fe.mfcc_batch(wavf, lens)
    assert torch.equal(a, b)                                        # int16 -> float is exact
    again, _ = fe.mfcc_batch(wav16, lens)
    assert torch.equal(a, again)                                    # run to run
    cfg = NS(audiofeat_num_mel_bins=80, audiofeat_num_ceps=40, audiofeat_frame_length=25, audiofeat_frame_shift=10,
             audiofeat_low_freq=20.0, audiofeat_high_freq=0.0, audiofeat_dither=0.0, frontend_device=str(dev))
    samples = [{"waveform": torch.from_numpy(p.astype(np.float32) / 32768.0)[None], "sample_rate": 16000} for p in pcms]
    for s, y in zip(fe.audio_compute_mfcc(iter(samples), cfg), torch.split(a, frames)):
        assert torch.equal(s["audiofeat"], y)                       # per-sample stage == packed batch


def test_edge_cases(waves):
    """Zero-frame utterances anywhere in the batch, an all-empty batch, and n_ceps == n_mels at the 128-bin limit."""
    dev = require_cuda()
    w = waves["noise_1s"]
    wav, lens = packed([w[:100], w, w[:399], w[:400]], dev)
    out, frames = fe.mfcc_batch(wav, lens)
    assert frames == [0, 98, 0, 1] and out.shape == (99, 40)
    ref, _ = fe.mfcc_batch(*packed([w], dev))
    assert torch.equal(out[:98], ref)
    empty, f0 = fe.mfcc_batch(*packed([w[:10]], dev))
    assert f0 == [0] and empty.shape == (0, 40)
    for n in (13, 128):
        out, frames = fe.mfcc_batch(*packed([w], dev), num_mel_bins=n, num_ceps=n)
        fb, _ = fe.fbank_batch(*packed([w], dev), num_mel_bins=n)
        y, a = fb.cpu().numpy(), fe._kaldi_mfcc_table(n, n).numpy()
        err = np.abs(out.cpu().numpy().astype(np.float64) - y.astype(np.float64) @ a.astype(np.float64))
        assert out.shape == (98, n) and np.all(err <= mo.epilogue_tolerance(y, a)), n


def chain(g):
    cfg = NS(**json.loads(bytes(g["chain/config_json"]).decode()))
    n = len([k for k in g.files if k.startswith("chain/pcm/")])
    random.seed(int(g["chain/seed"]))
    recs = [augment.draw_record(g[f"chain/pcm/{i}"].shape[0], 16000, cfg) for i in range(n)]
    return cfg, [g[f"chain/pcm/{i}"] for i in range(n)], recs


def test_augmented_chain_against_the_reference(golden):
    """resample -> speed perturb -> MFCC -> SpecAugment / SpecSub / SpecTrim -> stack: the stages' positions are exact
    (the GPU's augmentation applied to the reference's MFCC reproduces its spec_trim output bit for bit), the MFCC values
    are within the reference bound, and the stacked rows match the reference's stack of the same draws."""
    dev = require_cuda()
    cfg, pcms, recs = chain(golden)
    wav, lens = packed(pcms, dev)
    a = fe._kaldi_mfcc_table(80, 40).numpy()
    mf, frames = fe.mfcc_batch(wav, lens)
    for i, y in enumerate(split(mf, frames)):
        tol = mo.mfcc_tolerance(golden[f"chain/fbank/{i}"], a)
        assert np.all(np.abs(y.astype(np.float64) - golden[f"chain/mfcc/{i}"]) <= tol), i
    ref_mf = torch.from_numpy(np.concatenate([golden[f"chain/mfcc/{i}"] for i in range(len(recs))])).to(dev)
    aug, aframes = fe.spec_augment_batch(ref_mf, frames, recs)
    for i, y in enumerate(split(aug, aframes)):
        assert np.array_equal(y, golden[f"chain/spec_trim/{i}"]), i
    full, rows = fe.augmented_mfcc_stack_batch(wav, lens, recs)
    assert rows == [r["num_feat_frames"] for r in recs]
    for i, y in enumerate(split(full, rows)):
        np.testing.assert_allclose(y, golden[f"chain/stack/{i}"], rtol=5e-3, atol=5e-3, err_msg=str(i))
    ours, oframes = fe.spec_augment_batch(mf, frames, recs)
    st, _ = fe.stack_batch(ours, oframes, 5, 4, True)
    assert torch.equal(full, st)                                     # the chain launches exactly these stages
    again, _ = fe.augmented_mfcc_stack_batch(wav, lens, recs)
    assert torch.equal(full, again)
    wavf, _ = packed([p.astype(np.float32) / 32768.0 for p in pcms], dev)
    assert torch.equal(fe.augmented_mfcc_stack_batch(wavf, lens, recs)[0], full)
    dst = [5 + sum(rows[:i]) + 3 * i for i in range(len(rows))]
    buf = torch.full((dst[-1] + rows[-1] + 7, 200), -777.0, device=dev)
    fe.augmented_mfcc_stack_batch(wav, lens, recs, into=buf, dst_rows=dst)
    placed = torch.zeros(buf.shape[0], dtype=torch.bool)
    for d, r, y in zip(dst, rows, torch.split(full.cpu(), rows)):
        placed[d:d + r] = True
        assert torch.equal(buf[d:d + r].cpu(), y)
    assert torch.all(buf.cpu()[~placed] == -777.0)


def test_batch_chain_equals_per_sample_stages(golden):
    """Worker-drawn records + one batched MFCC chain == the per-sample GPU stages under the same seed, bit for bit,
    with speed perturbation and a resampled 44.1 kHz utterance in the batch."""
    dev = require_cuda()
    cfg, pcms, _ = chain(golden)
    cfg.frontend_device = str(dev)
    cfg.audio_resample_rate = 16000
    cfg.audio_speed_perturb = True
    cfg.audio_speed_perturb_speeds = [0.9, 1.0, 1.1]
    g = torch.Generator().manual_seed(3)
    x44 = np.round(0.2 * (2 * torch.rand(int(0.5 * 44100), generator=g).numpy() - 1) * 32767).astype(np.int16)
    utts = [(p, 16000) for p in pcms] + [(x44, 44100)]
    random.seed(7)
    recs = [augment.draw_record(p.shape[0], sr, cfg) for p, sr in utts]
    post = random.random()
    assert recs[-1]["resample"] == (44100, 16000)
    wav, lens = packed([p for p, _ in utts], dev)
    batch, rows = fe.augmented_mfcc_stack_batch(wav, lens, recs)
    random.seed(7)
    d = iter([{"waveform": torch.from_numpy(p.astype(np.float32) / 32768.0)[None], "sample_rate": sr} for p, sr in utts])
    for stage in (fe.audio_resample, fe.audio_speed_perturb, fe.audio_compute_mfcc, fe.audiofeat_spec_aug,
                  fe.audiofeat_spec_sub, fe.audiofeat_spec_trim, fe.audiofeat_stack):
        d = stage(d, cfg)
    per_sample = [s["audiofeat"] for s in d]
    assert random.random() == post
    for y, s in zip(torch.split(batch.cpu(), rows), per_sample):
        assert torch.equal(y, s.cpu())


def test_one_training_step_on_mfcc_features(golden):
    """A tiny B200TouchAudioForCausalLM (projector input num_ceps * stack = 200) trains one step on a packed batch
    featurised by augmented_mfcc_stack_batch."""
    from touchnet_b200 import batching, modeling
    dev = require_cuda()
    cfg, pcms, _ = chain(golden)
    torch.manual_seed(0)
    random.seed(5)
    samples = [{"waveform": torch.from_numpy(p), "sample_rate": 16000, "input_ids": list(range(3, 3 + 6 + i))}
               for i, p in enumerate(pcms)]
    samples = list(augment.draw_stage(iter(samples), cfg))
    B, T, F = 1, 256, 40 * 5
    plan = batching.plan_documents(iter(samples), B, T, with_audio=True)
    n = plan["num_sentence"]
    assert n == len(samples)
    buf = batching.assemble_on_device(plan, dev)
    feats = torch.zeros(B * T, F, device=dev)
    dst = [int(plan["doc_row"][i]) * T + int(plan["doc_off"][i]) for i in range(n)]
    wav, lens = packed([s["waveform"].numpy() for s in samples], dev)
    _, rows = fe.augmented_mfcc_stack_batch(wav, lens, [s["augment"] for s in samples], into=feats, dst_rows=dst)
    assert rows == [int(a) for a in plan["doc_audio"]]
    text = NS(hidden_size=256, intermediate_size=512, num_hidden_layers=2, num_attention_heads=2, num_key_value_heads=1,
              head_dim=128, vocab_size=320, rms_norm_eps=1e-5, rope_theta=500000.0, rope_scaling=None,
              attention_bias=False, tie_word_embeddings=False, initializer_range=0.02, model_type="llama",
              pad_token_id=0)
    model = modeling.B200TouchAudioForCausalLM(NS(audio_config=NS(input_size=F), text_config=text,
                                                  pad_token_id=0)).to(dev)
    model.post_init()
    out = model(input_ids=buf["input_ids"], input_features=feats.view(B, T, F), attention_mask=buf["attention_mask"],
                position_ids=buf["position_ids"])
    labels = buf["labels"].reshape(-1)
    keep = labels >= 0
    loss = torch.nn.functional.cross_entropy(out.logits.float().reshape(B * T, -1)[keep], labels[keep])
    loss.backward()
    assert torch.isfinite(loss)
    grads = [p.grad for p in model.parameters() if p.grad is not None]
    assert grads and all(torch.isfinite(g_).all() for g_ in grads)
    assert any(float(g_.abs().max()) > 0 for g_ in grads)
