"""Per-rank cost of the fused optimizer step with sharded state (shard_state=True) against the unsharded step, under torchrun:

    torchrun --nproc-per-node=N tools/shard_probe.py [--steps 10] [--warmup 3] [--out DIR]

Workloads on bert_base_6layer_6conect (random weights, synthetic batches already on the GPU, train mode): the VQA task step at
config-2 shape (B = 64 per rank, 101 regions x 36 tokens) and three 12-in-1 task shapes of config 5 at 8 ranks (VQA B = 16,
GuessWhatPointing B = 8 with 100 candidate regions after the first 101, retrieval B = 8 x 4 options). Per workload and arm (FusedAdamW unsharded / sharded, one after the other,
each on a fresh model): the optimizer step alone (opt.step() after the backward, CUDA events), the whole step (forward + backward
+ step) and the peak allocated memory, median over `steps` steps after `warmup`. The two step_ms do not time the same work: the
unsharded gradient all-reduce runs inside the backward, while the sharded step() includes the fp32 weight all-gather (the other
half of that exchange; its reduce-scatter runs inside the backward). Only total_ms compares like with like. One process (N = 1) measures the unsharded arm
only and reports the sharded one as not measured (shard_state needs more than one rank). Rank 0 prints one JSON line (also
DIR/shard_probe.json) with the card name and power limit read in the same run. Needs a GPU."""
import argparse
import json
import os
import statistics
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "tools"))
CONFIG = os.path.join(ROOT, "vilbert-multi-task_b200", "configs", "bert_base_6layer_6conect.json")

# name -> (task id, per-rank batch, regions, tokens)
WORKLOADS = {"config2_vqa_b64": ("TASK1", 64, 101, 36), "config5_vqa_b16": ("TASK1", 16, 101, 23),
             "config5_guesswhat_pointing_b8": ("TASK17", 8, 201, 23), "config5_retrieval_b8": ("TASK8", 8, 101, 36)}


def arm(name, shard, steps, warmup, world):
    import torch
    import _task_oracle as T
    import vilbert_b200
    from vilbert_b200.ddp import DistributedDataParallel as DDP
    from vilbert_b200.optim import FusedAdamW
    from vilbert_b200.tasks import ForwardModelsTrain, LoadLosses
    task, B, nv, nt = WORKLOADS[name]
    cfgj = dict(json.load(open(CONFIG)), task_specific_tokens=True)
    dev = torch.device("cuda", torch.cuda.current_device())
    torch.cuda.empty_cache()
    torch.cuda.reset_peak_memory_stats()
    model = vilbert_b200.VILBertForVLTasks(vilbert_b200.BertConfig.from_dict(cfgj))
    model.train()
    wrapped = DDP(model, delay_allreduce=True) if world > 1 else model
    opt = FusedAdamW(list(model.parameters()), lr=4e-5, correct_bias=False, model=wrapped if shard else model, shard_state=shard)
    batch = tuple(x.to(dev) for x in T.make_batch(cfgj, task, B, nv, nt, seed=0))
    losses = LoadLosses(None, T.TASK_CFG, [task[4:]])
    t_opt, t_all = [], []
    for i in range(warmup + steps):
        e0, e1, e2 = (torch.cuda.Event(enable_timing=True) for _ in range(3))
        e0.record()
        loss, _ = ForwardModelsTrain(None, T.TASK_CFG, dev, task, {task: 0}, {}, {task: [batch]}, wrapped, losses)
        loss.backward()
        e1.record()
        opt.step()
        e2.record()
        torch.cuda.synchronize()
        if i >= warmup:
            t_opt.append(e1.elapsed_time(e2))
            t_all.append(e0.elapsed_time(e2))
    res = dict(step_ms=statistics.median(t_opt), total_ms=statistics.median(t_all),
               peak_gib=torch.cuda.max_memory_allocated() / 2 ** 30, moments_gib=2 * opt.exp_avg.numel() * 4 / 2 ** 30)
    del model, wrapped, opt
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import torch
    import torch.distributed as dist
    from step_in_backward_probe import card
    world = int(os.environ.get("WORLD_SIZE", "1"))
    if world > 1:
        local = int(os.environ["LOCAL_RANK"])
        torch.cuda.set_device(local)
        dist.init_process_group("nccl", device_id=torch.device("cuda", local))
    out = dict(gpu=card(), world=world, steps=a.steps, warmup=a.warmup, workloads={})
    for name in WORKLOADS:
        row = dict(unsharded=arm(name, False, a.steps, a.warmup, world))
        row["sharded"] = arm(name, True, a.steps, a.warmup, world) if world > 1 else "not measured: one GPU (shard_state needs > 1 rank)"
        out["workloads"][name] = row
    if world == 1 or dist.get_rank() == 0:
        line = json.dumps(out)
        print(line)
        if a.out:
            os.makedirs(a.out, exist_ok=True)
            open(os.path.join(a.out, "shard_probe.json"), "w").write(line + "\n")
    if world > 1:
        dist.destroy_process_group()


if __name__ == "__main__":
    main()
