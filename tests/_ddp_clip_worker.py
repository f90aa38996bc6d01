"""2-rank worker of tests/test_clip_ddp_gpu.py (launched with torch.distributed.run, one rank per GPU, NCCL): clipped
FusedAdamW steps after the gradient all-reduce. Each rank writes rank-specific gradients, averages them over the world, then
steps with max_grad_norm; the ranks must hold bitwise-equal norms and parameters, and a NaN written on one rank only must make
every rank skip the step (the all-reduce spreads it, and each rank decides on its own device)."""
import json
import os
import sys

import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import adamw_oracle as AO           # noqa: E402
from oracle import vilbert_oracle as O          # noqa: E402
from vilbert_b200.config import BertConfig     # noqa: E402
from vilbert_b200.ddp import FlatGradAllReducer  # noqa: E402
from vilbert_b200.engine import Engine         # noqa: E402
from vilbert_b200.optim import FusedAdamW       # noqa: E402


def equal_on_all_ranks(t):
    ref = t.clone()
    dist.broadcast(ref, 0)
    ok = torch.tensor([1 if torch.equal(ref, t) else 0], device=t.device)
    dist.all_reduce(ok, op=dist.ReduceOp.MIN)
    return bool(ok.item())


def main():
    out_path = sys.argv[1]
    rank, local = int(os.environ["RANK"]), int(os.environ["LOCAL_RANK"])
    torch.cuda.set_device(local)
    dev = torch.device("cuda", local)
    dist.init_process_group("nccl", device_id=dev)
    cfgj = json.load(open(os.path.join(ROOT, "tests", "golden", "tiny_b4.json")))["config"]
    P = O.synth_params(O.make_config(cfgj), seed=0, device=dev)
    eng = Engine(BertConfig.from_dict(cfgj), dev)
    for k in eng.ps.entries:
        eng.ps.p(k).copy_(P[k])
    eng.refresh_weights()
    named = [(name, torch.nn.Parameter(eng.ps.p(name))) for name in eng.ps.entries]
    opt = FusedAdamW(AO.reference_param_groups(named, base_lr=1e-3), lr=1e-3, correct_bias=False, engine=eng, max_grad_norm=0.5)
    red = FlatGradAllReducer(eng.ps.grad, n_buckets=4)
    gen = torch.Generator(device=dev)
    res = {"norm_equal": [], "params_equal": [], "norms": []}

    def step(t, poison=False):
        gen.manual_seed(1000 * t + rank)                       # different gradients on every rank
        eng.ps.grad.copy_(torch.randn(eng.ps.numel, device=dev, generator=gen) * 1e-2)
        if poison and rank == 1:
            off = eng.ps.entries["bert.encoder.layer.0.attention.self.query.weight"][0]
            eng.ps.grad[off + 3] = float("nan")
        red.allreduce()
        opt.step()
        torch.cuda.synchronize()

    for t in (1, 2, 3):
        step(t)
        res["norm_equal"].append(equal_on_all_ranks(opt.grad_norm.reshape(1)))
        res["params_equal"].append(equal_on_all_ranks(eng.ps.flat))
        res["norms"].append(opt.grad_norm.item())
    before = eng.ps.flat.clone()
    step(4, poison=True)
    res["skipped"] = int(opt.skipped_steps.item())
    res["unchanged_after_skip"] = bool(torch.equal(before, eng.ps.flat))
    res["step_after_skip"] = int(opt._step_dev.item())
    step(5)
    res["params_equal_after"] = equal_on_all_ranks(eng.ps.flat)
    skipped = torch.tensor([res["skipped"]], device=dev)
    dist.all_reduce(skipped, op=dist.ReduceOp.MIN)
    res["skipped_on_every_rank"] = int(skipped.item())
    if rank == 0:
        json.dump(res, open(out_path, "w"))
    dist.barrier()
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
