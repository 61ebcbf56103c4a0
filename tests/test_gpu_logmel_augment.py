"""GPU: whisper log-mel with int16 input, audiofeat_padding and the recipe's augmentation chain (csrc/frontend.cu MODE 1,
touchnet_b200.frontend.log_mel_batch / augmented_log_mel_stack_batch) against tests/golden/logmel_chain.npz, which holds
the reference's own audio_compute_log_mel_spectrogram outputs with padding and a seeded run of its log-mel chain
(tests/golden/make_golden_logmel.py).  At padding 0 the reference's outputs are frontend_logmel.npz's (the generator
checks the bits).

Tolerances: log-mel values atol 2e-4 (as test_logmel_matches_torch_stft_golden); stacked rows rtol / atol 5e-3 (as the
fbank chain); everything else bit-identical (int16 vs float, virtual vs explicit padding, batch vs per-sample, run to
run, the chain's masks / subs / trim)."""
import json
import os
import random
from types import SimpleNamespace as NS

import numpy as np
import pytest
import torch

from tests.gpu_util import require_cuda
from touchnet_b200 import _lib, augment, frontend as fe

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def golden(golden_dir):
    return np.load(os.path.join(golden_dir, "logmel_chain.npz"))


@pytest.fixture(scope="module")
def logmel_golden(golden_dir):
    return np.load(os.path.join(golden_dir, "frontend_logmel.npz"))


@pytest.fixture(scope="module")
def waves(logmel_golden):
    return {k[4:]: logmel_golden[k] for k in sorted(logmel_golden.files) if k.startswith("wav/")}


def packed(arrays, dev):
    return fe._pack([torch.from_numpy(np.ascontiguousarray(a)) for a in arrays], dev)


def split(t, lens):
    return [y.numpy() for y in torch.split(t.cpu(), list(lens))]


def int16_pcm(w):
    return np.clip(np.round(w.astype(np.float64) * 32768.0), -32768, 32767).astype(np.int16)


@pytest.mark.parametrize("n_mels", [80, 128])
@pytest.mark.parametrize("padded", [False, True])
def test_log_mel_matches_the_reference(golden, logmel_golden, waves, padded, n_mels):
    """Every waveform of frontend_logmel.npz in one packed launch, at padding 0 and at the fixture's padding."""
    dev = require_cuda()
    pad = int(golden["padding"]) if padded else 0
    names = list(waves)
    wav, lens = packed([waves[n] for n in names], dev)
    out, frames = fe.log_mel_batch(wav, lens, num_mel_bins=n_mels, padding=pad)
    assert frames == [(n + pad) // 160 for n in lens]
    for n, y in zip(names, split(out, frames)):
        ref = golden[f"logmel/{pad}/{n}/{n_mels}"] if pad else logmel_golden[f"logmel/{n}/{n_mels}"]
        assert y.shape == ref.shape, n
        np.testing.assert_allclose(y, ref, atol=2e-4, rtol=0, err_msg=f"{n} pad {pad}")


def test_int16_padding_batch_and_run_to_run_bit_identity(golden, waves):
    dev = require_cuda()
    pad = int(golden["padding"])
    pcms = [int16_pcm(w) for w in waves.values()]
    floats = [p.astype(np.float32) / np.float32(32768.0) for p in pcms]
    wav16, lens = packed(pcms, dev)
    wavf, _ = packed(floats, dev)
    for p in (0, pad):
        a, frames = fe.log_mel_batch(wav16, lens, padding=p)
        assert torch.equal(a, fe.log_mel_batch(wavf, lens, padding=p)[0])          # int16 * 2^-15 is exact
        assert torch.equal(a, fe.log_mel_batch(wav16, lens, padding=p)[0])         # run to run
        for y, x in zip(torch.split(a, frames), floats):                             # packed == one at a time
            assert torch.equal(y, fe.log_mel_batch(*packed([x], dev), padding=p)[0])
    # the padding is virtual: same bits as an explicitly zero-padded fp32 waveform
    explicit, elens = packed([np.concatenate([x, np.zeros(pad, np.float32)]) for x in floats], dev)
    assert torch.equal(fe.log_mel_batch(wavf, lens, padding=pad)[0], fe.log_mel_batch(explicit, elens)[0])


def test_per_sample_stage(golden, waves):
    """audio_compute_log_mel_spectrogram: fp32 input gives the bits of F.pad + log_mel_batch (what the stage did before
    padding moved into the kernel); int16 input gives the bits of pcm / 32768."""
    dev = require_cuda()
    pad = int(golden["padding"])
    for p in (0, pad):
        cfg = NS(audiofeat_n_fft=400, audiofeat_hop_length=160, audiofeat_num_mel_bins=80, audiofeat_padding=p,
                 frontend_device=str(dev))
        for w in waves.values():
            x = torch.from_numpy(w)
            s = next(fe.audio_compute_log_mel_spectrogram(iter([{"waveform": x[None], "sample_rate": 16000}]), cfg))
            want, _ = fe.log_mel_batch(torch.nn.functional.pad(x, (0, p)).to(dev), [x.numel() + p])
            assert torch.equal(s["audiofeat"], want)
            pcm = torch.from_numpy(int16_pcm(w))
            s16 = next(fe.audio_compute_log_mel_spectrogram(iter([{"waveform": pcm[None], "sample_rate": 16000}]),
                                                            cfg))
            sf = next(fe.audio_compute_log_mel_spectrogram(
                iter([{"waveform": (pcm.float() / 32768.0)[None], "sample_rate": 16000}]), cfg))
            assert torch.equal(s16["audiofeat"], sf["audiofeat"])


def chain(g):
    cfg = NS(**json.loads(bytes(g["chain/config_json"]).decode()))
    n = len([k for k in g.files if k.startswith("chain/pcm/")])
    random.seed(int(g["chain/seed"]))
    recs = [augment.draw_record(g[f"chain/pcm/{i}"].shape[0], 16000, cfg) for i in range(n)]
    return cfg, [g[f"chain/pcm/{i}"] for i in range(n)], recs


def test_augmented_chain_against_the_reference(golden):
    """speed perturb -> log-mel -> SpecAugment / SpecSub / SpecTrim -> stack: log-mel of the reference's speed-perturbed
    waveforms within atol 2e-4, the GPU's augmentation of the reference's log-mel bit-exact against its spec_trim
    output, the whole chain within 5e-3 of the reference's stacked rows and exactly the stages it is made of."""
    dev = require_cuda()
    cfg, pcms, recs = chain(golden)
    pad = cfg.audiofeat_padding
    sw, slens = packed([golden[f"chain/speed_wav/{i}"] for i in range(len(recs))], dev)
    lm, frames = fe.log_mel_batch(sw, slens, padding=pad)
    assert frames == [r["num_frames"] for r in recs]
    for i, y in enumerate(split(lm, frames)):
        np.testing.assert_allclose(y, golden[f"chain/logmel/{i}"], atol=2e-4, rtol=0, err_msg=str(i))
    ref_lm = torch.from_numpy(np.concatenate([golden[f"chain/logmel/{i}"] for i in range(len(recs))])).to(dev)
    aug, aframes = fe.spec_augment_batch(ref_lm, frames, recs)
    for i, y in enumerate(split(aug, aframes)):
        assert np.array_equal(y, golden[f"chain/spec_trim/{i}"]), i
    wav, lens = packed(pcms, dev)
    full, rows = fe.augmented_log_mel_stack_batch(wav, lens, recs, padding=pad)
    assert rows == [r["num_feat_frames"] for r in recs]
    for i, y in enumerate(split(full, rows)):
        np.testing.assert_allclose(y, golden[f"chain/stack/{i}"], rtol=5e-3, atol=5e-3, err_msg=str(i))
    sp, splens = fe.speed_perturb_batch(wav, lens, [r["speed"] for r in recs], 16000)
    ours, oframes = fe.spec_augment_batch(*fe.log_mel_batch(sp, splens, padding=pad), recs)
    assert torch.equal(full, fe.stack_batch(ours, oframes, 5, 4, True)[0])
    assert torch.equal(full, fe.augmented_log_mel_stack_batch(wav, lens, recs, padding=pad)[0])
    wavf, _ = packed([p.astype(np.float32) / 32768.0 for p in pcms], dev)
    assert torch.equal(fe.augmented_log_mel_stack_batch(wavf, lens, recs, padding=pad)[0], full)
    dst = [5 + sum(rows[:i]) + 3 * i for i in range(len(rows))]
    buf = torch.full((dst[-1] + rows[-1] + 7, 400), -777.0, device=dev)
    fe.augmented_log_mel_stack_batch(wav, lens, recs, padding=pad, into=buf, dst_rows=dst)
    placed = torch.zeros(buf.shape[0], dtype=torch.bool)
    for d, r, y in zip(dst, rows, torch.split(full.cpu(), rows)):
        placed[d:d + r] = True
        assert torch.equal(buf[d:d + r].cpu(), y)
    assert torch.all(buf.cpu()[~placed] == -777.0)


def test_without_augmentation_the_chain_is_log_mel_plus_stack(golden):
    dev = require_cuda()
    _, pcms, recs = chain(golden)
    wav, lens = packed(pcms, dev)
    off = [{"resample": None, "speed": 1.0, "t_masks": [], "f_masks": [], "subs": [], "trim": 0} for _ in recs]
    n0 = _lib.launch_count
    full, rows = fe.augmented_log_mel_stack_batch(wav, lens, off, num_mel_bins=128, padding=250, stack_length=7,
                                                  stride_length=6)
    n1 = _lib.launch_count
    lm, frames = fe.log_mel_batch(wav, lens, num_mel_bins=128, padding=250)
    st, rows2 = fe.stack_batch(lm, frames, 7, 6, True)
    assert _lib.launch_count - n1 == n1 - n0
    assert rows == rows2 and torch.equal(full, st)


def test_too_short_utterance_after_speed_perturbation_raises(golden):
    """n_fft // 2 = 200 samples: 210 at speed 1.1 leaves 191, which the reference's reflect padding rejects."""
    dev = require_cuda()
    wav, lens = packed([golden["chain/pcm/0"], golden["chain/pcm/1"][:210]], dev)
    recs = [{"resample": None, "speed": s, "t_masks": [], "f_masks": [], "subs": [], "trim": 0} for s in (1.0, 1.1)]
    with pytest.raises(_lib.TouchNetB200Error, match="utterance 1 has 191 samples"):
        fe.augmented_log_mel_stack_batch(wav, lens, recs)
    fe.augmented_log_mel_stack_batch(wav, lens, recs, padding=10)              # 191 + 10 > 200


def test_batch_chain_equals_per_sample_stages(golden):
    """Worker-drawn records + one batched log-mel chain == the per-sample GPU stages under the same seed, bit for bit,
    with speed perturbation, padding and a resampled 44.1 kHz utterance in the batch."""
    dev = require_cuda()
    cfg, pcms, _ = chain(golden)
    cfg.frontend_device = str(dev)
    cfg.audio_resample_rate = 16000
    g = torch.Generator().manual_seed(3)
    x44 = np.round(0.2 * (2 * torch.rand(int(0.5 * 44100), generator=g).numpy() - 1) * 32767).astype(np.int16)
    utts = [(p, 16000) for p in pcms] + [(x44, 44100)]
    random.seed(7)
    recs = [augment.draw_record(p.shape[0], sr, cfg) for p, sr in utts]
    post = random.random()
    assert recs[-1]["resample"] == (44100, 16000)
    wav, lens = packed([p for p, _ in utts], dev)
    batch, rows = fe.augmented_log_mel_stack_batch(wav, lens, recs, padding=cfg.audiofeat_padding)
    random.seed(7)
    d = iter([{"waveform": torch.from_numpy(p.astype(np.float32) / 32768.0)[None], "sample_rate": sr} for p, sr in utts])
    for stage in (fe.audio_resample, fe.audio_speed_perturb, fe.audio_compute_log_mel_spectrogram,
                  fe.audiofeat_spec_aug, fe.audiofeat_spec_sub, fe.audiofeat_spec_trim, fe.audiofeat_stack):
        d = stage(d, cfg)
    per_sample = [s["audiofeat"] for s in d]
    assert random.random() == post
    for y, s in zip(torch.split(batch.cpu(), rows), per_sample):
        assert torch.equal(y, s.cpu())


def test_one_training_step_on_log_mel_features(golden):
    """A tiny B200TouchAudioForCausalLM (projector input num_mel_bins * stack = 400) trains one step on a packed batch
    featurised by augmented_log_mel_stack_batch."""
    from touchnet_b200 import batching, modeling
    dev = require_cuda()
    cfg, pcms, _ = chain(golden)
    torch.manual_seed(0)
    random.seed(5)
    samples = [{"waveform": torch.from_numpy(p), "sample_rate": 16000, "input_ids": list(range(3, 3 + 6 + i))}
               for i, p in enumerate(pcms)]
    samples = list(augment.draw_stage(iter(samples), cfg))
    B, T, F = 1, 256, 80 * 5
    plan = batching.plan_documents(iter(samples), B, T, with_audio=True)
    n = plan["num_sentence"]
    assert n == len(samples)
    buf = batching.assemble_on_device(plan, dev)
    feats = torch.zeros(B * T, F, device=dev)
    dst = [int(plan["doc_row"][i]) * T + int(plan["doc_off"][i]) for i in range(n)]
    wav, lens = packed([s["waveform"].numpy() for s in samples], dev)
    _, rows = fe.augmented_log_mel_stack_batch(wav, lens, [s["augment"] for s in samples],
                                               padding=cfg.audiofeat_padding, into=feats, dst_rows=dst)
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
