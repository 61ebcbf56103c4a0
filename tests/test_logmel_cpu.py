"""CPU: the host half of the whisper log-mel chain against tests/golden/logmel_chain.npz (the reference's own
audio_compute_log_mel_spectrogram outputs with audiofeat_padding, and a seeded run of its log-mel augmentation chain,
tests/golden/make_golden_logmel.py): the oracle with padding, the draws of a log-mel recipe, and argument errors (the
host and the C ABI validate before touching the device)."""
import json
import os
import random
from types import SimpleNamespace as NS

import numpy as np
import pytest
import torch

from oracle import frontend_oracle as fo
from tests.test_augment_cpu import DrawLog
from touchnet_b200 import _lib, augment, frontend


@pytest.fixture(scope="module")
def golden(golden_dir):
    return np.load(os.path.join(golden_dir, "logmel_chain.npz"))


@pytest.fixture(scope="module")
def logmel_golden(golden_dir):
    return np.load(os.path.join(golden_dir, "frontend_logmel.npz"))


def chain_config(g):
    return NS(**json.loads(bytes(g["chain/config_json"]).decode()))


def n_chain(g):
    return len([k for k in g.files if k.startswith("chain/pcm/")])


def test_oracle_matches_the_reference_with_padding(golden, logmel_golden):
    """oracle.frontend_oracle.log_mel(padding=p) against the reference's padded outputs, at the log-mel atol of
    test_logmel_oracle_matches_torch_stft_path; the padding is not a multiple of the hop."""
    pad = int(golden["padding"])
    assert pad % 160 != 0
    keys = [k for k in golden.files if k.startswith(f"logmel/{pad}/")]
    assert len(keys) == 6                                     # 3 waveforms x (80, 128) mels
    for k in keys:
        _, _, name, nm = k.split("/")
        wav = logmel_golden["wav/" + name]
        out = fo.log_mel(wav, n_mels=int(nm), padding=pad)
        assert out.shape == golden[k].shape == ((wav.shape[0] + pad) // 160, int(nm)), k
        np.testing.assert_allclose(out, golden[k], atol=2e-4, rtol=0, err_msg=k)


def test_log_mel_draws_reproduce_the_reference_chain(golden):
    """Same draws, in the same order and count, as the reference's log-mel chain; frames are (n + padding) // hop of
    the speed-perturbed length and frequency masks stay inside the num_mel_bins columns."""
    cfg = chain_config(golden)
    log = DrawLog()
    random.seed(int(golden["chain/seed"]))
    recs = [augment.draw_record(golden[f"chain/pcm/{i}"].shape[0], 16000, cfg, rng=log) for i in range(n_chain(golden))]
    assert np.array_equal(np.array(log.log, dtype=np.float64), golden["chain/draws"])
    assert random.random() == float(golden["chain/post_random"])
    assert sorted(r["speed"] for r in recs) == [0.9, 1.0, 1.1]
    for i, r in enumerate(recs):
        n = golden[f"chain/speed_wav/{i}"].shape[0]
        assert r["num_samples"] == n
        assert r["num_frames"] == golden[f"chain/logmel/{i}"].shape[0] == (n + cfg.audiofeat_padding) // 160
        assert r["trim"] > 0 and r["num_frames"] - r["trim"] == golden[f"chain/spec_trim/{i}"].shape[0]
        assert r["num_feat_frames"] == golden[f"chain/stack/{i}"].shape[0]
        assert r["f_masks"] and all(0 <= s < e <= cfg.audiofeat_num_mel_bins for s, e in r["f_masks"])


def test_draw_stage_counts_padded_log_mel_frames():
    cfg = NS(audio_feat_type="log_mel_spectrogram", audiofeat_num_mel_bins=128, audiofeat_hop_length=160,
             audiofeat_padding=250, audiofeat_spec_aug=True, audiofeat_spec_aug_num_t_mask=1,
             audiofeat_spec_aug_num_f_mask=30, audiofeat_spec_aug_max_t=5, audiofeat_spec_aug_max_f=30,
             audiofeat_stride_length=4)
    s = next(augment.draw_stage(iter([{"waveform": torch.zeros(1, 16000), "sample_rate": 16000}]), cfg))
    rec = s["augment"]
    assert rec["num_frames"] == 101 and s["num_feat_frames"] == 26
    assert len(rec["f_masks"]) == 30 and all(0 <= a < b <= 128 for a, b in rec["f_masks"])


def identity(n):
    return [{"resample": None, "speed": 1.0, "t_masks": [], "f_masks": [], "subs": [], "trim": 0}] * n


def test_argument_errors():
    wav = torch.zeros(16000)
    with pytest.raises(_lib.TouchNetB200Error, match="padding"):
        frontend.log_mel_batch(wav, [16000], padding=-1)
    with pytest.raises(_lib.TouchNetB200Error, match="padding"):
        frontend.augmented_log_mel_stack_batch(wav, [16000], identity(1), padding=-1)
    for bad in (torch.zeros(16000, dtype=torch.float64), torch.zeros(1, 16000)):
        with pytest.raises(_lib.TouchNetB200Error, match="fp32 or int16"):
            frontend.log_mel_batch(bad, [16000])
    with pytest.raises(_lib.TouchNetB200Error, match="GPU"):
        frontend.log_mel_batch(wav, [16000])
    with pytest.raises(_lib.TouchNetB200Error, match="GPU"):
        frontend.log_mel_batch(wav.to(torch.int16), [16000], padding=250)
    with pytest.raises(_lib.TouchNetB200Error, match="records"):
        frontend.augmented_log_mel_stack_batch(wav, [8000, 8000], identity(1))
    # the reference's reflect padding rejects N + padding <= n_fft // 2; the utterance is named
    with pytest.raises(_lib.TouchNetB200Error, match="utterance 1 has 150 samples"):
        frontend.augmented_log_mel_stack_batch(wav, [15850, 150], identity(2), padding=50)
    with pytest.raises(_lib.TouchNetB200Error, match="GPU"):          # 150 + 51 > 200: valid, then needs the GPU
        frontend.augmented_log_mel_stack_batch(wav, [15850, 150], identity(2), padding=51)


def test_c_abi_argument_errors():
    #            wav i16 utt frm n  T  nfft hop pad window mel n_mels out max stream
    ok = dict(wav=8, i16=0, utt=8, frm=8, n=1, T=1, nfft=400, hop=160, pad=0, window=8, mel=8, n_mels=80, out=8,
              utt_max=8, stream=None)
    bad = [(dict(pad=-1), "negative padding"), (dict(nfft=1024), "n_fft"), (dict(hop=0), "n_fft"),
           (dict(n_mels=129), "n_mels"), (dict(wav=None), "null pointer"), (dict(utt_max=None), "null pointer")]
    for change, needle in bad:
        args = dict(ok, **change)
        with pytest.raises(_lib.TouchNetB200Error, match=needle):
            _lib.call("tn_logmel_power_f32", *args.values())
