"""FP8 training (config key `float8_training`) under FSDP2 against the same FP8 model on one GPU without FSDP.
    torchrun --nproc-per-node N tools/check_fsdp_fp8.py [--recipe tensorwise|rowwise]   (N = 1: a one-rank mesh)
Each rank trains on its own packed row.  The single-GPU reference runs that row with fp32 master weights (the block casts
them to bf16 itself); under FSDP2 the block receives the bf16 all-gathered parameters.  Both hand the FP8 block the same
bf16 weights and the same row, so each rank's loss must be bitwise equal.  The reduced gradients are compared with the
sum of the reference gradients over the ranks: FSDP2 computes bf16 weight gradients and reduces them in fp32, the
reference computes fp32 ones, so they agree to bf16 rounding."""
import argparse
import os
import sys

import torch
import torch.distributed as dist
from torch.distributed.device_mesh import init_device_mesh
from torch.distributed.fsdp import MixedPrecisionPolicy, fully_shard

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from tests.gpu_util import packed_doc_ids, rel_err  # noqa: E402
from tests.test_gpu_model import small_cfg  # noqa: E402
from touchnet_b200 import modeling  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("--recipe", default="tensorwise", help="float8_recipe_name: tensorwise or rowwise")
args = ap.parse_args()
rank, world = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"])
dev = torch.device("cuda", int(os.environ.get("LOCAL_RANK", rank)))
torch.cuda.set_device(dev)
dist.init_process_group("nccl", device_id=dev)
cfg = small_cfg(L=2, d=512, H=4, KV=2, ffn=1024, V=512)
torch.manual_seed(1)
model = modeling.B200LlamaForCausalLM(cfg).to(dev)
model.post_init()
with torch.no_grad():
    for p in model.parameters():
        if p.dim() == 2:
            p.normal_(0, 0.05)
for p in model.parameters():
    dist.broadcast(p.data, 0)
model.float8_training = True
model.float8_recipe_name = args.recipe
T = 1024
lens = [[300, 500, 100], [1024], [512, 512], [1000]][:world]
doc, pos = packed_doc_ids(world, T, lens, dev)
g = torch.Generator(device="cpu").manual_seed(3)
ids = torch.randint(0, cfg.vocab_size, (world, T), generator=g).to(dev)
labels = torch.randint(0, cfg.vocab_size, (world, T), generator=g).to(dev)
labels[doc == 0] = -100
sl = slice(rank, rank + 1)


def step(m):
    lg = m(input_ids=ids[sl], attention_mask=doc[sl], position_ids=pos[sl]).logits
    return torch.nn.functional.cross_entropy(lg.float().view(-1, cfg.vocab_size), labels[sl].reshape(-1),
                                             ignore_index=-100)


# ---- single GPU, this rank's row, fp32 masters ----
ref_loss = step(model)
ref_loss.backward()
ref_grads = {}
for n, p in model.named_parameters():
    gsum = p.grad.detach().clone()
    dist.all_reduce(gsum)                    # the gradient of the sum of the rank losses
    ref_grads[n] = gsum
model.zero_grad()
# ---- FSDP2, bf16 all-gather ----
mesh = init_device_mesh("cuda", (world,), mesh_dim_names=("dp_shard",))
mp = MixedPrecisionPolicy(param_dtype=torch.bfloat16, reduce_dtype=torch.float32)
for layer in model.model.layers:
    fully_shard(layer, mesh=mesh, mp_policy=mp)
fully_shard(model, mesh=mesh, mp_policy=mp)
assert model.float8_training
loss = step(model)
loss.backward()
same = torch.equal(loss.detach(), ref_loss.detach())
worst = 0.0
for n, p in model.named_parameters():
    gfull = p.grad.full_tensor() * world     # FSDP averages over the ranks
    e = rel_err(gfull.float(), ref_grads[n].float())
    if rank == 0 and e > 1e-2:
        print(f"  {n}: rel err {e:.4g}")
    worst = max(worst, e)
flags = torch.tensor([0 if same else 1], device=dev)
dist.all_reduce(flags)
if rank == 0:
    print(f"FSDP{world} FP8 ({args.recipe}): loss {loss.item():.6f} vs {ref_loss.item():.6f} (bitwise on every rank: {int(flags) == 0}); "
          f"worst grad rel err {worst:.4g}")
    assert int(flags) == 0 and worst < 1e-2
    print("FSDP FP8 OK")
dist.destroy_process_group()
