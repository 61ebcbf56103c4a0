"""fp64 restatement of the sampling distribution of tn_sample_select_slots_bf16 (DESIGN §3.4), shared by the CPU and GPU
sampling tests: the kept set under top-k (ties included) and the value-group top-p rule, and its probabilities."""
import torch


def processed(seq, logits, penalty, ngram, temperature):
    """HF's processors and temperature on fp32 logits [1, V] for the history seq [1, n] -> fp32 scores [V]."""
    from transformers.generation.logits_process import (NoRepeatNGramLogitsProcessor, RepetitionPenaltyLogitsProcessor,
                                                        TemperatureLogitsWarper)
    s = logits.float().clone()
    if penalty != 1.0:
        s = RepetitionPenaltyLogitsProcessor(penalty)(seq, s)
    if ngram > 0:
        s = NoRepeatNGramLogitsProcessor(ngram)(seq, s)
    if temperature != 1.0:
        s = TemperatureLogitsWarper(temperature)(seq, s)
    return s[0]


def distribution(x, top_k, top_p, eps=1e-5):
    """x: processed fp32 scores [V] without NaN, finite maximum.  Returns (probabilities fp64 [V], band [V] bool): band
    marks the value groups whose mass above lies within eps * Z of top_p * Z, where rounding may move the boundary."""
    x = x.double().cpu()
    V = x.numel()
    m = x.max()
    kept = torch.ones(V, dtype=torch.bool)
    if 0 < top_k < V:
        kept = x >= x.topk(top_k).values[-1]
    w = torch.where(kept, torch.exp(x - m), torch.zeros_like(x))
    band = torch.zeros(V, dtype=torch.bool)
    if top_p < 1.0:
        Z = w.sum()
        u, inv = torch.unique(x, return_inverse=True)                 # ascending distinct values
        gw = torch.zeros(u.numel(), dtype=torch.float64).index_add_(0, inv, w)
        above = gw.flip(0).cumsum(0).flip(0) - gw                     # kept mass strictly above each value
        keep_u = (above < top_p * Z) | (u == m)
        band = kept & ((above - top_p * Z).abs() <= eps * Z)[inv] & (u != m)[inv]
        kept = kept & keep_u[inv]
        w = torch.where(kept, w, torch.zeros_like(w))
    return w / w.sum(), band


def hf_kept(x, top_k, top_p):
    """The tokens HF's TopKLogitsWarper / TopPLogitsWarper keep (min_tokens_to_keep = 1) on scores x [V]."""
    from transformers.generation.logits_process import TopKLogitsWarper, TopPLogitsWarper
    s = x.float()[None].clone()
    ids = torch.zeros((1, 1), dtype=torch.int64)
    if top_k > 0:
        s = TopKLogitsWarper(top_k)(ids, s)
    if top_p < 1.0:
        s = TopPLogitsWarper(top_p)(ids, s)
    return s[0] > -float("inf")
