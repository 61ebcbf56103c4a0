"""Time the augmented GPU frontend against the plain one on one bench-size packed row of audio, and the CPU chain it
replaces.

GPU (CUDA events, L2 flushed before every timed call, median of --iters):
  plain      fbank_batch + stack_batch(into=...)                         (what bench.py runs)
  augmented  augmented_fbank_stack_batch(into=...) with the recipe's draws: speed {0.9, 1.0, 1.1}, 2 time masks <= 50,
             2 freq masks <= 10, 3 subs <= 30 (examples/audio/sft/asr/wenetspeech/run.sh:258-270), trim off
  --feat-type mfcc times mfcc_batch / augmented_mfcc_stack_batch instead (80 mel bins, 40 cepstra, frequency masks drawn
  over the 40 columns) and kaldi.mfcc in the CPU chain; --feat-type log_mel_spectrogram times log_mel_batch /
  augmented_log_mel_stack_batch (whisper log-mel, n_fft 400, hop 160, 80 mel bins, audiofeat_padding 0) and the
  reference's torch.stft path in the CPU chain.
  and the two augmentation kernels on their own, with achieved algorithmic bytes against the 3.35 TB/s data-sheet HBM3
  bandwidth of the H100 SXM: resample reads each input sample once (2 B int16) and writes each output once (4 B);
  spec augment reads each output frame's source row unless it is zeroed and writes each output frame (4 B * F each).
CPU: the same chain with the same stand-in for sox (torchaudio.transforms.Resample from sr*speed to sr), then
  torchaudio.compliance.kaldi.fbank (or the feature type's features), the masks / subs as slice copies on a cloned
  tensor, and the oracle's stack - one process with one thread, and os.cpu_count() single-thread processes.
Prints the GPU name, power limit and SM clocks it ran at, then one JSON line."""
import argparse
import json
import os
import random
import subprocess
import sys
import time
from multiprocessing import Pool
from types import SimpleNamespace as NS

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from touchnet_b200 import augment, batching, frontend  # noqa: E402

HBM_TBS = 3.35
CFG = NS(audio_resample_rate=16000, audio_speed_perturb=True, audio_speed_perturb_speeds=[0.9, 1.0, 1.1],
         audio_feat_type="fbank", audiofeat_num_mel_bins=80, audiofeat_frame_length=25, audiofeat_frame_shift=10,
         audiofeat_dither=0.0, audiofeat_spec_aug=True, audiofeat_spec_aug_num_t_mask=2,
         audiofeat_spec_aug_num_f_mask=2, audiofeat_spec_aug_max_t=50, audiofeat_spec_aug_max_f=10,
         audiofeat_spec_sub=True, audiofeat_spec_sub_num_t_sub=3, audiofeat_spec_sub_max_t=30, audiofeat_spec_trim=False,
         audiofeat_stack_length=5, audiofeat_stride_length=4, audiofeat_normalize=True)


def one_row(seed, T):
    """The utterances of one packed row of T positions (placement of batching.plan_documents on the augmented lengths)."""
    seen = []

    def gen():
        for s in augment.draw_stage(batching.synthetic_utterances(seed, 128256, stride=4, max_s=30.0, int16=True), CFG):
            seen.append(s)
            yield s
    random.seed(seed)
    plan = batching.plan_documents(gen(), 1, T, True)
    placed = seen[:plan["num_sentence"]]
    assert [s["num_feat_frames"] for s in placed] == plan["doc_audio"].tolist()
    return placed, plan


def timed(fn, iters, flush):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    for _ in range(3):
        fn()
    ts = []
    for _ in range(iters):
        flush.zero_()
        e0.record(); fn(); e1.record()
        torch.cuda.synchronize()
        ts.append(e0.elapsed_time(e1))
    return sorted(ts)[len(ts) // 2]


def cpu_chain(items, feat_type="fbank"):
    import torchaudio
    from oracle import frontend_oracle as fo
    torch.set_num_threads(1)
    for pcm, rec in items:
        w = torch.from_numpy(pcm.astype(np.float32) / 32768.0)[None]
        if rec["speed"] != 1.0:
            w = torchaudio.transforms.Resample(augment.speed_source_rate(16000, rec["speed"]), 16000)(w)
        if feat_type == "log_mel_spectrogram":      # ref: functions.py:168-189 (padding 0)
            stft = torch.stft(w[0], 400, 160, window=torch.hann_window(400), return_complex=True)
            mel = frontend._slaney_mel_filters(16000, 400, 80, "cpu") @ (stft[..., :-1].abs() ** 2)
            x = torch.clamp(mel, min=1e-10).log10()
            x = ((torch.maximum(x, x.max() - 8.0) + 4.0) / 4.0).transpose(0, 1)
        elif feat_type == "mfcc":
            x = torchaudio.compliance.kaldi.mfcc(w * 32768, num_mel_bins=80, frame_length=25, frame_shift=10,
                                                 dither=0.0, num_ceps=40, high_freq=0.0, low_freq=20.0,
                                                 sample_frequency=16000)
        else:
            x = torchaudio.compliance.kaldi.fbank(w * 32768, num_mel_bins=80, frame_length=25, frame_shift=10,
                                                  dither=0.0, energy_floor=0.0, sample_frequency=16000)
        y = x.clone()
        for s, e in rec["t_masks"]:
            y[s:e, :] = 0
        for s, e in rec["f_masks"]:
            y[:, s:e] = 0
        x, y = y, y.clone()
        for s, e, pos in rec["subs"]:
            y[s:e, :] = x[s - pos:e - pos, :]
        fo.stack(y.numpy(), 5, 4, True)
    return len(items)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--seq-len", type=int, default=8192)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--seed", type=int, default=0)
    ap.add_argument("--no-cpu", action="store_true")
    ap.add_argument("--feat-type", choices=("fbank", "mfcc", "log_mel_spectrogram"), default="fbank")
    args = ap.parse_args()
    mfcc = args.feat_type == "mfcc"
    CFG.audio_feat_type = args.feat_type
    if mfcc:
        CFG.audiofeat_num_ceps = 40
    if args.feat_type == "log_mel_spectrogram":
        CFG.audiofeat_n_fft, CFG.audiofeat_hop_length, CFG.audiofeat_padding = 400, 160, 0
    n_feat = 40 if mfcc else 80
    features = {"fbank": lambda w, n: frontend.fbank_batch(w, n),
                "mfcc": lambda w, n: frontend.mfcc_batch(w, n, num_mel_bins=80, num_ceps=40),
                "log_mel_spectrogram": lambda w, n: frontend.log_mel_batch(w, n)}[args.feat_type]
    augmented_stack = {"fbank": frontend.augmented_fbank_stack_batch, "mfcc": frontend.augmented_mfcc_stack_batch,
                       "log_mel_spectrogram": frontend.augmented_log_mel_stack_batch}[args.feat_type]
    assert torch.cuda.is_available(), "time_augment.py measures on the GPU; there is no CPU fallback"
    dev = torch.device("cuda:0")
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    placed, plan = one_row(args.seed, args.seq_len)
    recs = [s["augment"] for s in placed]
    pcms = [s["waveform"] for s in placed]
    wav, lens = frontend._pack(pcms, dev)
    rows = plan["doc_audio"].tolist()
    dst = plan["doc_off"].tolist()
    feats = torch.zeros(args.seq_len, 5 * n_feat, device=dev)
    flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)
    plain_rows = [augment.stacked_rows(f, 4) for f in features(wav, lens)[1]]
    plain_dst = [sum(plain_rows[:i]) for i in range(len(plain_rows))]
    plain_buf = torch.zeros(sum(plain_rows), 5 * n_feat, device=dev)

    def plain():
        fb, fr = features(wav, lens)
        frontend.stack_batch(fb, fr, 5, 4, True, into=plain_buf, dst_rows=plain_dst)

    def augmented():
        augmented_stack(wav, lens, recs, into=feats, dst_rows=dst)

    sped, slens = frontend.speed_perturb_batch(wav, lens, [r["speed"] for r in recs], 16000)
    fb, frames = features(sped, slens)
    out_frames = [f - r["trim"] for f, r in zip(frames, recs)]
    t_plain = timed(plain, args.iters, flush)
    t_aug = timed(augmented, args.iters, flush)
    t_rs = timed(lambda: frontend.speed_perturb_batch(wav, lens, [r["speed"] for r in recs], 16000), args.iters, flush)
    t_sa = timed(lambda: frontend.spec_augment_batch(fb, frames, recs), args.iters, flush)
    sa_out, _ = frontend.spec_augment_batch(fb, frames, recs)
    rs_bytes = 2 * sum(lens) + 4 * sum(slens)
    zero_rows = int((sa_out == 0).all(dim=1).sum())
    sa_bytes = 4 * n_feat * (2 * sum(out_frames) - zero_rows)
    # kernel-only times from the profiler (the event windows above also hold the host-side table building and copies)
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(args.iters):
            flush.zero_()
            augmented()
        torch.cuda.synchronize()
    dur = {"resample_kernel": [], "spec_augment_kernel": []}
    for e in prof.events():
        for k in dur:
            if k in e.name and e.device_type == torch.autograd.DeviceType.CUDA:
                dur[k].append(e.device_time_total / 1e3)
    k_rs, k_sa = (sorted(v)[len(v) // 2] for v in dur.values())
    res = {"gpu": smi, "feat_type": args.feat_type, "utterances": len(lens), "audio_s": sum(lens) / 16000.0, "rows": sum(rows),
           "plain_call_ms": t_plain, "augmented_call_ms": t_aug, "resample_call_ms": t_rs, "spec_augment_call_ms": t_sa,
           "resample_kernel_ms": k_rs, "spec_augment_kernel_ms": k_sa,
           "resample_GBps": rs_bytes / k_rs / 1e6, "resample_pct_hbm": 100 * rs_bytes / k_rs / 1e9 / HBM_TBS,
           "spec_augment_GBps": sa_bytes / k_sa / 1e6, "spec_augment_pct_hbm": 100 * sa_bytes / k_sa / 1e9 / HBM_TBS}
    print(f"GPU: {smi}")
    print(f"one packed row of {args.seq_len}: {len(lens)} utterances, {res['audio_s']:.1f} s of 16 kHz int16 audio")
    print(f"features: {args.feat_type}")
    print(f"call times (events): plain frontend {t_plain * 1e3:.1f} us, augmented {t_aug * 1e3:.1f} us, "
          f"speed_perturb_batch {t_rs * 1e3:.1f} us, spec_augment_batch {t_sa * 1e3:.1f} us")
    print(f"kernels (profiler): resample {k_rs * 1e3:.1f} us, {res['resample_GBps']:.0f} GB/s = "
          f"{res['resample_pct_hbm']:.1f} % of {HBM_TBS} TB/s; spec augment {k_sa * 1e3:.1f} us, "
          f"{res['spec_augment_GBps']:.0f} GB/s = {res['spec_augment_pct_hbm']:.1f} %")
    if not args.no_cpu:
        items = [(p.numpy(), r) for p, r in zip(pcms, recs)]
        t0 = time.perf_counter(); cpu_chain(items, args.feat_type); t1 = time.perf_counter()
        n = os.cpu_count() or 1
        chunks = [(items[i::n], args.feat_type) for i in range(n)]
        with Pool(n) as pool:
            pool.starmap(cpu_chain, [(items[:1], args.feat_type)] * n)   # warm the workers (imports)
            t2 = time.perf_counter(); pool.starmap(cpu_chain, chunks); t3 = time.perf_counter()
        res.update(cpu_1thread_ms=(t1 - t0) * 1e3, cpu_procs=n, cpu_procs_ms=(t3 - t2) * 1e3)
        print(f"CPU chain (torchaudio stand-in): 1 thread {res['cpu_1thread_ms']:.0f} ms, "
              f"{n} processes {res['cpu_procs_ms']:.0f} ms")
    print(json.dumps(res))


if __name__ == "__main__":
    main()
