"""GPU: the data augmentation kernels (csrc/augment.cu) through touchnet_b200.frontend against tests/golden/augment.npz,
which holds the reference's own stage outputs (see tests/golden/make_golden_augment.py), and against the numpy oracle.
Resampling is checked with a per-sample bound derived from fp32 summation over the taps (tests/augment_oracle.py);
SpecAugment / SpecSub / SpecTrim are copies and zeros and must be bit-exact."""
import json
import os
import random
from types import SimpleNamespace as NS

import numpy as np
import pytest
import torch

from tests import augment_oracle as ao
from tests.gpu_util import require_cuda
from tests.test_oracle_golden import power_close
from touchnet_b200 import augment, frontend as fe

pytestmark = pytest.mark.gpu

RATES = (8000, 22050, 44100, 48000)


@pytest.fixture(scope="module")
def golden(golden_dir):
    return np.load(os.path.join(golden_dir, "augment.npz"))


def chain(g):
    cfg = NS(**json.loads(bytes(g["chain/config_json"]).decode()))
    n = len([k for k in g.files if k.startswith("chain/pcm/")])
    random.seed(int(g["chain/seed"]))
    recs = [augment.draw_record(g[f"chain/pcm/{i}"].shape[0], 16000, cfg) for i in range(n)]
    return cfg, [g[f"chain/pcm/{i}"] for i in range(n)], recs


def packed(arrays, dev):
    return fe._pack([torch.from_numpy(np.ascontiguousarray(a)) for a in arrays], dev)


def split(t, lens):
    return list(torch.split(t.cpu(), list(lens)))


def test_resample_matches_the_reference_and_int16_equals_float(golden):
    dev = require_cuda()
    pcms = [golden[f"resample/{sr}/pcm"] for sr in RATES]
    wav16, lens = packed(pcms, dev)
    out, out_lens = fe.resample_batch(wav16, lens, list(RATES), 16000)      # four ratios in one launch
    for sr, x, y in zip(RATES, pcms, split(out, out_lens)):
        ref = golden[f"resample/{sr}/out"]
        assert y.shape[0] == ref.shape[0], sr
        xf = x.astype(np.float32) / 32768.0
        err = np.abs(y.numpy().astype(np.float64) - ref)
        assert np.all(err <= ao.resample_tolerance(xf, sr, 16000, ref)), (sr, float(err.max()))
    wavf, _ = packed([p.astype(np.float32) / 32768.0 for p in pcms], dev)
    out_f, _ = fe.resample_batch(wavf, lens, list(RATES), 16000)
    assert torch.equal(out, out_f)
    # one utterance at a time gives the same bits as the packed launch; a 1:1 ratio is an exact copy
    y0, _ = fe.resample_batch(wav16[:lens[0]].contiguous(), lens[:1], RATES[0], 16000)
    assert torch.equal(y0, out[:out_lens[0]])
    same, _ = fe.resample_batch(wavf, lens, 16000, 16000)
    assert torch.equal(same, wavf)


def test_speed_perturb_matches_the_reference_chain(golden):
    dev = require_cuda()
    _, pcms, recs = chain(golden)
    wav, lens = packed(pcms, dev)
    out, out_lens = fe.speed_perturb_batch(wav, lens, [r["speed"] for r in recs], 16000)
    assert out_lens == [r["num_samples"] for r in recs]
    for i, (x, y, r) in enumerate(zip(pcms, split(out, out_lens), recs)):
        ref = golden[f"chain/speed_wav/{i}"]
        if r["speed"] == 1.0:
            assert np.array_equal(y.numpy(), ref)
            continue
        src = augment.speed_source_rate(16000, r["speed"])
        err = np.abs(y.numpy().astype(np.float64) - ref)
        assert np.all(err <= ao.resample_tolerance(x.astype(np.float32) / 32768.0, src, 16000, ref)), i


def test_spec_augment_bit_exact_against_the_reference(golden):
    dev = require_cuda()
    _, _, recs = chain(golden)
    fbs = [golden[f"chain/fbank/{i}"] for i in range(len(recs))]
    feats = torch.from_numpy(np.concatenate(fbs)).to(dev)
    out, frames = fe.spec_augment_batch(feats, [f.shape[0] for f in fbs], recs)
    for i, y in enumerate(split(out, frames)):
        assert np.array_equal(y.numpy(), golden[f"chain/spec_trim/{i}"]), i


def test_spec_augment_edge_cases_against_the_oracle():
    dev = require_cuda()
    g = torch.Generator().manual_seed(3)
    T = [40, 12, 30, 9, 64]
    feats = [torch.randn(t, 80, generator=g).numpy() for t in T]
    rec = lambda **kw: dict({"t_masks": [], "f_masks": [], "subs": [], "trim": 0}, **kw)
    recs = [
        rec(t_masks=[(3, 20), (10, 25)], f_masks=[(70, 80), (75, 80)], subs=[(5, 30, 5), (20, 35, 20)], trim=19),
        rec(t_masks=[(4, 12)], f_masks=[(0, 10)], subs=[(11, 12, 11)], trim=5),   # shorter than a 50-frame mask
        rec(subs=[(0, 10, 0), (8, 30, 8), (9, 12, 3)], trim=14),                  # subs read the masked input, last wins
        rec(t_masks=[(0, 9)], trim=4),                                              # all masked, trim just below T/2
        rec(),                                                                      # untouched utterance in the batch
    ]
    x = torch.from_numpy(np.concatenate(feats)).to(dev)
    out, frames = fe.spec_augment_batch(x, T, recs)
    assert frames == [t - r["trim"] for t, r in zip(T, recs)]
    for f, r, y in zip(feats, recs, split(out, frames)):
        assert np.array_equal(y.numpy(), ao.apply_record(f, r))


def test_full_chain_against_the_reference(golden):
    dev = require_cuda()
    cfg, pcms, recs = chain(golden)
    wav, lens = packed(pcms, dev)
    sped, sl = fe.speed_perturb_batch(wav, lens, [r["speed"] for r in recs], 16000)
    fb, frames = fe.fbank_batch(sped, sl)
    for i, y in enumerate(split(fb, frames)):
        assert power_close(golden[f"chain/fbank/{i}"], y.numpy()) < 1.0, i
    aug, aframes = fe.spec_augment_batch(fb, frames, recs)
    for r, y in zip(recs, split(aug, aframes)):
        for s, e in r["t_masks"]:
            ok_rows = [f for f in range(y.shape[0]) if all(not (a <= f < b) for a, b, _ in r["subs"]) and s <= f < e]
            assert torch.all(y[ok_rows] == 0)
        for s, e in r["f_masks"]:
            assert torch.all(y[:, s:e] == 0)
    st, st_rows = fe.stack_batch(aug, aframes, 5, 4, True)
    for i, y in enumerate(split(st, st_rows)):
        np.testing.assert_allclose(y.numpy(), golden[f"chain/stack/{i}"], rtol=5e-3, atol=5e-3, err_msg=str(i))
    full, rows = fe.augmented_fbank_stack_batch(wav, lens, recs)
    assert rows == [r["num_feat_frames"] for r in recs] and torch.equal(full, st)
    again, _ = fe.augmented_fbank_stack_batch(wav, lens, recs)
    assert torch.equal(full, again)                                              # run to run
    wavf, _ = packed([p.astype(np.float32) / 32768.0 for p in pcms], dev)
    assert torch.equal(fe.augmented_fbank_stack_batch(wavf, lens, recs)[0], full)   # int16 == float input


def test_all_augmentation_off_is_todays_frontend(golden):
    dev = require_cuda()
    _, pcms, _ = chain(golden)
    wav, lens = packed(pcms, dev)
    off = [{"resample": None, "speed": 1.0, "t_masks": [], "f_masks": [], "subs": [], "trim": 0} for _ in lens]
    a, rows = fe.augmented_fbank_stack_batch(wav, lens, off)
    b, rows_b = fe.fbank_stack_batch(wav, lens)
    assert rows == rows_b and torch.equal(a, b)
    fb, frames = fe.fbank_batch(wav, lens)
    dst = [3 + sum(rows[:i]) + 2 * i for i in range(len(rows))]
    buf_a = torch.full((sum(rows) + 20, 400), -777.0, device=dev)
    buf_b = buf_a.clone()
    fe.augmented_fbank_stack_batch(wav, lens, off, into=buf_a, dst_rows=dst)
    fe.stack_batch(fb, frames, 5, 4, True, into=buf_b, dst_rows=dst)
    assert torch.equal(buf_a, buf_b)


def test_into_leaves_other_rows_untouched(golden):
    dev = require_cuda()
    _, pcms, recs = chain(golden)
    wav, lens = packed(pcms, dev)
    ref, rows = fe.augmented_fbank_stack_batch(wav, lens, recs)
    dst = [5 + sum(rows[:i]) + 3 * i for i in range(len(rows))]
    buf = torch.full((dst[-1] + rows[-1] + 7, 400), -777.0, device=dev)
    fe.augmented_fbank_stack_batch(wav, lens, recs, into=buf, dst_rows=dst)
    placed = torch.zeros(buf.shape[0], dtype=torch.bool)
    for d, r, y in zip(dst, rows, split(ref, rows)):
        placed[d:d + r] = True
        assert torch.equal(buf[d:d + r].cpu(), y)
    assert torch.all(buf.cpu()[~placed] == -777.0)


def test_batch_form_equals_per_sample_stages(golden):
    """Records drawn in the worker + one batched application == the reference-shaped per-sample GPU stages, bit for bit
    (same seed, same draws), including a resampled 44.1 kHz and 22.05 kHz utterance."""
    dev = require_cuda()
    cfg, pcms, _ = chain(golden)
    cfg.frontend_device = str(dev)
    utts = [(p, 16000) for p in pcms] + [(golden[f"resample/{sr}/pcm"], sr) for sr in (44100, 22050)]
    seed = 99
    random.seed(seed)
    recs = [augment.draw_record(p.shape[0], sr, cfg) for p, sr in utts]
    post = random.random()
    assert recs[-1]["resample"] == (22050, 16000)
    wav, lens = packed([p for p, _ in utts], dev)
    batch, rows = fe.augmented_fbank_stack_batch(wav, lens, recs)
    random.seed(seed)
    d = iter([{"waveform": torch.from_numpy(p.astype(np.float32) / 32768.0)[None], "sample_rate": sr} for p, sr in utts])
    for stage in (fe.audio_resample, fe.audio_speed_perturb, fe.audio_compute_fbank, fe.audiofeat_spec_aug,
                  fe.audiofeat_spec_sub, fe.audiofeat_spec_trim, fe.audiofeat_stack):
        d = stage(d, cfg)
    per_sample = [s["audiofeat"] for s in d]
    assert random.random() == post
    for y, s in zip(split(batch, rows), per_sample):
        assert torch.equal(y, s.cpu())


def test_one_training_step_on_augmented_features(golden):
    """A tiny B200TouchAudioForCausalLM trains one step on a packed batch featurised by augmented_fbank_stack_batch."""
    from touchnet_b200 import batching, modeling
    dev = require_cuda()
    cfg, pcms, _ = chain(golden)
    torch.manual_seed(0)
    random.seed(5)
    samples = [{"waveform": torch.from_numpy(p), "sample_rate": 16000, "input_ids": list(range(3, 3 + 6 + i))}
               for i, p in enumerate(pcms)]
    samples = list(augment.draw_stage(iter(samples), cfg))
    B, T = 1, 256
    plan = batching.plan_documents(iter(samples), B, T, with_audio=True)
    n = plan["num_sentence"]
    assert n == len(samples)
    buf = batching.assemble_on_device(plan, dev)
    feats = torch.zeros(B * T, 400, device=dev)
    dst = [int(plan["doc_row"][i]) * T + int(plan["doc_off"][i]) for i in range(n)]
    wav, lens = packed([s["waveform"].numpy() for s in samples], dev)
    _, rows = fe.augmented_fbank_stack_batch(wav, lens, [s["augment"] for s in samples], into=feats, dst_rows=dst)
    assert rows == [int(a) for a in plan["doc_audio"]]
    text = NS(hidden_size=256, intermediate_size=512, num_hidden_layers=2, num_attention_heads=2, num_key_value_heads=1,
              head_dim=128, vocab_size=320, rms_norm_eps=1e-5, rope_theta=500000.0, rope_scaling=None,
              attention_bias=False, tie_word_embeddings=False, initializer_range=0.02, model_type="llama",
              pad_token_id=0)
    model = modeling.B200TouchAudioForCausalLM(NS(audio_config=NS(input_size=400), text_config=text,
                                                  pad_token_id=0)).to(dev)
    model.post_init()
    out = model(input_ids=buf["input_ids"], input_features=feats.view(B, T, 400), attention_mask=buf["attention_mask"],
                position_ids=buf["position_ids"])
    labels = buf["labels"].reshape(-1)
    keep = labels >= 0
    loss = torch.nn.functional.cross_entropy(out.logits.float().reshape(B * T, -1)[keep], labels[keep])
    loss.backward()
    assert torch.isfinite(loss)
    assert all(torch.isfinite(p.grad).all() for p in model.parameters() if p.grad is not None)
