"""fp64 restatement of speculative sampling (Leviathan et al. 2023, Algorithm 1; transformers' `_speculative_sampling`)
for one position, shared by the CPU and GPU tests of tn_spec_sample_verify_bf16: the acceptance probability of a
proposal drawn from q, the residual distribution a rejection draws from, and the resulting distribution of the emitted
token, which is p."""
import torch


def acceptance(p, q):
    """P(accept) for x ~ q, accepted with probability min(1, p(x) / q(x)): sum_v min(p(v), q(v))."""
    return float(torch.minimum(p.double(), q.double()).sum())


def residual(p, q):
    """The distribution a rejection draws from: max(0, p - q), normalised (p itself when q == p nowhere exceeds it)."""
    r = (p.double() - q.double()).clamp(min=0)
    return r / r.sum() if float(r.sum()) > 0 else p.double()


def emitted(p, q):
    """Distribution of the token emitted at the position: q(v) min(1, p(v)/q(v)) + (1 - acceptance) residual(v)."""
    p, q = p.double(), q.double()
    ratio = torch.where(q > 0, torch.clamp(p / torch.where(q > 0, q, torch.ones_like(q)), max=1.0),
                        torch.zeros_like(q))
    return q * ratio + (1 - acceptance(p, q)) * residual(p, q)
