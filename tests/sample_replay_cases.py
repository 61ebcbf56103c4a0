"""The inputs of the replay tests of the sampling kernels (tests/test_gpu_sample_replay.py), built on the CPU so that
the CPU tests can measure, on the very same inputs, how many draws a defective kernel would get wrong.

Each select case is one launch of tn_sample_select_slots_bf16: a few base rows (random rows of two widths and rows
built for the edges: a tie group across the top-k boundary, the top-p boundary inside a tie, all the mass on the last
token of one draw_index_order warp chunk and the first of the next, weights near 2^-41, a NaN, +inf and all -inf),
each repeated over many slots with their own stream keys and lengths.  Each spec case is one launch of
tn_spec_sample_verify_bf16 over slots of chosen kinds (q near p, q = p, q disjoint from p, a degenerate draft row, a
draft token outside q's kept set or banned by the ngram over the extended history, eos and the limit mid-block,
finished slots)."""
import functools

import numpy as np
import torch

from tests.sample_replay import PLAIN, Dist, draw_bits, processed, spec_position

BF16 = torch.bfloat16
SELECT_V = (1, 2, 33, 1000, 1025, 32 * 1024 + 1, 128256, 156032)
# (temperature, top_k, top_p, repetition_penalty, no_repeat_ngram_size); top_k "V-1" / "V" are relative to V
SELECT_KNOBS = ((1.0, 0, 1.0, 1.0, 0), (0.7, 50, 0.9, 1.5, 2), (1.3, "V-1", 1 - 2.0 ** -20, 1.0, 0),
                (0.7, 2, 0.5, 1.3, 3), (1.0, "V", 0.0, 1.0, 1), (1.3, 1, 0.9, 1.5, 0), (0.7, 0, 0.5, 1.0, 0))
SEEDS = (987654321, -42, 2 ** 40 + 7, -(2 ** 62) + 3, 5, 2 ** 63 - 1, -1)
SPEC_V = (64, 1000, 128256)
SPEC_K = (1, 3, 8)
SPEC_KNOBS = ((1.0, 0, 1.0, 1.0, 0), (0.7, 50, 0.9, 1.5, 2), (1.3, 20, 0.5, 1.0, 3))
HIST_IDS = 40                                 # history ids lie in [0, HIST_IDS): the edge tokens lie above


def chunk_of(V):
    """draw_index_order's per-warp index range."""
    return ((V + 31) // 32 + 31) // 32 * 32


def _top_k(V, k):
    return V - 1 if k == "V-1" else V if k == "V" else k


def _bf16(x):
    return torch.as_tensor(x, dtype=torch.float32).to(BF16).float()


def _base_rows(V, t, top_k, top_p, g):
    rows = [torch.randn(V, generator=g) * 2, torch.randn(V, generator=g) * 4]
    if 2 <= top_k < V - 2:                                            # a tie group across the top-k boundary
        x = torch.randn(V, generator=g) * 3
        idx = torch.argsort(x, descending=True)
        lo = max(0, top_k - 3)
        x[idx[lo:top_k + 2]] = float(x[idx[top_k - 1]])
        rows.append(x)
    if 0 < top_p < 1 and V > 8:                                       # the top-p boundary inside a tie group
        x = _bf16(torch.randn(V, generator=g) * 3)
        idx = torch.argsort(x, descending=True)
        cum = torch.softmax(x.double() / t, 0)[idx].cumsum(0)
        b = int((cum < top_p).sum())
        lo, hi = max(1, b - 2), min(V, b + 3)
        x[idx[lo:hi]] = float(x[idx[b]])
        rows.append(x)
    c = chunk_of(V)
    if V > c:                                                         # the mass at the end of one chunk, the start of the next
        x = torch.full((V,), -60.0)
        x[c - 1] = x[c] = 1.0
        rows.append(x)
    if V > 4:                                                         # weights near 2^-41 (0 or 1 in fixed point)
        x = -28.5 + 0.125 * torch.randint(-2, 3, (V,), generator=g).float()
        x[int(torch.randint(0, V, (), generator=g))] = 0.0
        rows.append(x)
    nan = torch.randn(V, generator=g)
    nan[int(torch.randint(0, V, (), generator=g))] = float("nan")
    inf = torch.randn(V, generator=g)
    inf[int(torch.randint(0, V, (), generator=g))] = float("inf")
    rows += [nan, inf, torch.full((V,), float("-inf"))]
    return torch.stack(rows).to(BF16)


@functools.lru_cache(maxsize=None)
def select_cases():
    """[(name, case dict)] for every V and knob set; a case's tensors are CPU tensors (built once: read only)."""
    out = []
    for vi, V in enumerate(SELECT_V):
        for ci, (t, k, p, pen, ng) in enumerate(SELECT_KNOBS):
            g = torch.Generator().manual_seed(1000 * vi + ci)
            top_k = _top_k(V, k)
            base = _base_rows(V, t, top_k, p, g)
            nb = base.shape[0]
            mapped = ci % 2 == 1
            n_rows = 252 if mapped else (192 if V > 40000 else 504)
            n_rows -= n_rows % nb
            reps = n_rows // nb
            row_base = torch.arange(nb).repeat_interleave(reps)
            B = n_rows + 8 if mapped else n_rows
            S = 80
            hist = torch.randint(0, min(V, HIST_IDS), (S,), generator=g)
            hist[44:46] = hist[20:22]                                  # a repeated bigram: the ngram bans something
            length = 40 + torch.randint(0, 8, (B,), generator=g).to(torch.int32)
            limit = torch.full((B,), S, dtype=torch.int32)
            limit[::7] = length[::7] + 1                               # the last budgeted token: the slot finishes
            finished = torch.zeros(B, dtype=torch.int32)
            finished[3::11] = 1
            key = torch.randint(-2 ** 62, 2 ** 62, (B,), generator=g)
            key[::5] = torch.arange(0, B, 5)                           # small keys, as generate_many's prompt indices
            key[1::5] += 2 ** 32
            case = dict(V=V, knobs=(pen, ng, t, top_k, p), seed=SEEDS[(vi + ci) % len(SEEDS)],
                        eos=int(torch.randint(0, V, (), generator=g)), pad=0,
                        logits=base[row_base], row_base=row_base, base=base, history=hist[None].repeat(B, 1),
                        length=length, positions=torch.arange(B, dtype=torch.int64) * 3,
                        next_ids=torch.full((B,), -5, dtype=torch.int64), finished=finished, limit=limit,
                        stream_key=key, row_slot=None, row_key=None)
            if mapped:
                perm = torch.randperm(B, generator=g)[:n_rows]
                case["row_slot"] = perm.tolist()
                case["row_key"] = torch.randint(-2 ** 63, 2 ** 63 - 1, (n_rows,), generator=g).tolist()
                case["row_key"][:4] = [0, 1, 2 ** 32, -(2 ** 32)]
            out.append((f"V{V}-knobs{ci}", case))
    return out


@functools.lru_cache(maxsize=None)
def spec_cases():
    """[(name, case dict)] for every V, k and knob set; CPU tensors (built once: read only)."""
    kinds = ("near", "near", "near", "same", "disjoint", "qdegenerate", "outside_q", "ngram_banned", "eos", "limit",
             "finished", "near")
    out = []
    for vi, V in enumerate(SPEC_V):
        for k in SPEC_K:
            for ci, (t, tk, tp, pen, ng) in enumerate(SPEC_KNOBS):
                g = torch.Generator().manual_seed(7000 + 100 * vi + 10 * k + ci)
                reps = 1 if V > 40000 else 3 if V > 100 else 6
                kind = [kk for kk in kinds for _ in range(reps)]
                B, S = len(kind), 80
                hist = torch.randint(0, HIST_IDS, (B, S), generator=g)
                p = (torch.randn(B * (k + 1), V, generator=g) * 3).to(BF16)
                q = (p.view(B, k + 1, V)[:, :k].float() + torch.randn(B, k, V, generator=g) * 1.5).to(BF16)
                draft = torch.empty((B, k), dtype=torch.int64)
                for j in range(k):                                     # proposals drawn from q (temperature 1)
                    draft[:, j] = torch.multinomial(torch.softmax(q[:, j].float(), -1), 1, generator=g)[:, 0]
                length = 40 + torch.randint(0, 3, (B,), generator=g).to(torch.int32)
                limit = torch.full((B,), S, dtype=torch.int32)
                finished = torch.zeros(B, dtype=torch.int32)
                eos = V - 1
                for b, kd in enumerate(kind):
                    pr = p.view(B, k + 1, V)[b]
                    if kd == "same":
                        q[b] = pr[:k]
                    elif kd == "disjoint":                             # q's mass where p has none (after top-k)
                        lowest = torch.argsort(pr[:k].float(), dim=-1)[:, :60]
                        q[b] = torch.full((k, V), -40.0).to(BF16)
                        q[b].scatter_(1, lowest, 5.0)
                        draft[b] = lowest[:, 0]
                    elif kd == "qdegenerate":
                        q[b, 0, V // 2] = float("nan")
                    elif kd == "outside_q":
                        draft[b] = torch.argsort(q[b].float(), dim=-1)[:, 0]
                    elif kd == "ngram_banned":                         # draft[0] completes a bigram of the history
                        hist[b, int(length[b]) - 1] = hist[b, 10]
                        draft[b, 0] = hist[b, 11]
                    elif kd == "eos":
                        q[b] = pr[:k]
                        draft[b, k // 2] = eos
                        pr[k // 2, eos] = pr[k // 2].float().max().to(BF16)
                        q[b, k // 2] = pr[k // 2]
                    elif kd == "limit":
                        limit[b] = int(length[b]) + 2
                    elif kd == "finished":
                        finished[b] = 1
                key = torch.randint(-2 ** 63, 2 ** 63 - 1, (B,), generator=g)
                key[:2] = torch.tensor([0, 2 ** 32])
                out.append((f"V{V}-k{k}-knobs{ci}", dict(
                    V=V, k=k, knobs=(pen, ng, t, tk, tp), seed=SEEDS[(vi + k + ci) % len(SEEDS)], eos=eos, pad=0,
                    kind=kind, logits=p, dlogits=q.reshape(B * k, V).contiguous(), draft=draft, history=hist,
                    length=length, positions=torch.arange(B, dtype=torch.int64) + 100,
                    next_ids=torch.full((B,), -5, dtype=torch.int64), finished=finished, limit=limit,
                    stream_key=key)))
    return out


def replay_select(case, mut=()):
    """Per logits row, the set of tokens the replay allows (None for a row whose slot is finished)."""
    pen, ng, t, top_k, top_p = case["knobs"]
    slots = case["row_slot"] if case["row_slot"] is not None else list(range(case["logits"].shape[0]))
    keys = case["row_key"] if case["row_key"] is not None else [int(case["stream_key"][b]) for b in slots]
    lengths = [int(case["length"][b]) for b in slots]
    bits = draw_bits(case["seed"], np.array(lengths), PLAIN, np.array(keys, dtype=np.int64), mut)
    base = case["base"].float().numpy()
    hist = case["history"].numpy()
    shared = bool((hist == hist[:1]).all())
    dists, out = {}, []
    for r, b in enumerate(slots):
        if case["finished"][b]:
            out.append(None)
            continue
        i, L = int(case["row_base"][r]), lengths[r]
        ck = (i, L if pen != 1.0 or ng > 0 else None) if shared else (r,)
        if ck not in dists:
            dists[ck] = Dist(processed(base[i], hist[b, :L], pen, ng, t), top_k, top_p, mut)
        out.append(dists[ck].draw(bits[r]))
    return out


def replay_spec(case, mut=()):
    """Per slot, None (finished) or the list of k + 1 sets of possible picks (x accepted, ~t emitted)."""
    k, V = case["k"], case["V"]
    p = case["logits"].float().numpy().reshape(-1, k + 1, V)
    q = case["dlogits"].float().numpy().reshape(-1, k, V)
    out = []
    for b in range(p.shape[0]):
        if case["finished"][b]:
            out.append(None)
            continue
        L = int(case["length"][b])
        h = np.concatenate([case["history"][b, :L].numpy(), case["draft"][b].numpy()])
        key = int(case["stream_key"][b])
        out.append([spec_position(p[b, j], q[b, min(j, k - 1)], h[:L + j], int(case["draft"][b, j]) if j < k else None,
                                  case["seed"], L + j, key, case["knobs"], mut) for j in range(k + 1)])
    return out

