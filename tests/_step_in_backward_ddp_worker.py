"""2-rank worker of tests/test_step_in_backward_gpu.py (torch.distributed.run, one rank per GPU, NCCL): two models from the same
parameters under DistributedDataParallel(delay_allreduce=False) run the same train-mode ForwardModelsTrain steps, one with
backward + FusedAdamW.step(), the other with the step in the backward (each bucket stepped after its collective). Under
torch.use_deterministic_algorithms(True) their parameters must be bitwise equal after every step, and equal across the ranks."""
import json
import os
import sys
from datetime import timedelta

import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import _task_oracle as T                          # noqa: E402
from oracle import vilbert_oracle as O           # noqa: E402

Bl, NV, NT = 4, 101, 23


def main():
    import vilbert_b200
    from vilbert_b200.ddp import DistributedDataParallel as DDP
    from vilbert_b200.optim import FusedAdamW
    from vilbert_b200.tasks import ForwardModelsTrain, LoadLosses
    out_path = sys.argv[1]
    rank, world, local = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ["LOCAL_RANK"])
    torch.cuda.set_device(local)
    dev = torch.device("cuda", local)
    dist.init_process_group("nccl", device_id=dev, timeout=timedelta(minutes=5))
    torch.use_deterministic_algorithms(True)
    cfgj = dict(json.load(open(os.path.join(ROOT, "tests", "golden", "tiny_b4.json")))["config"], task_specific_tokens=True,
                max_position_embeddings=300)
    params = O.synth_params(O.make_config(cfgj), seed=3, device=dev)
    losses = LoadLosses(None, T.TASK_CFG, ["1"])
    runs = []
    for in_backward in (False, True):
        m = vilbert_b200.VILBertForVLTasks(vilbert_b200.BertConfig.from_dict(cfgj))
        m.load_state_dict(params, strict=False)
        m.train()
        d = DDP(m, delay_allreduce=False)
        opt = FusedAdamW(list(m.parameters()), lr=1e-3, model=m)
        snaps = []
        for s in range(6):
            b = T.make_batch(cfgj, "TASK1", Bl * world, NV, NT, seed=s)
            batch = tuple(t[rank * Bl:(rank + 1) * Bl] for t in b)
            m.engine.set_dropout_step(100 + s)
            loss, _ = ForwardModelsTrain(None, T.TASK_CFG, dev, "TASK1", {"TASK1": 0}, {}, {"TASK1": [batch]}, d, losses)
            if in_backward:
                with opt.step_in_backward():
                    loss.backward()
            else:
                loss.backward()
                opt.step()
            snaps.append(m.engine.ps.flat.clone())
        torch.cuda.synchronize()
        runs.append(snaps)
    params_equal = all(torch.equal(a, b) for a, b in zip(*runs))
    flat = runs[1][-1].clone()
    dist.broadcast(flat, 0)
    res = dict(rank=rank, params_equal=params_equal, ranks_equal=bool(torch.equal(flat, runs[1][-1])))
    gathered = [None] * world
    dist.all_gather_object(gathered, res)
    if rank == 0:
        json.dump(gathered, open(out_path, "w"))
    dist.barrier()
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
