"""Times retrieval evaluation sharded over the GPUs of one node, evaluate_retrieval_both(group=dist.group.WORLD), at the settings of
tools/retrieval_probe.py: bert_base_6layer_6conect with task tokens, fp16 operands, random weights (rank 0's, broadcast), 1,000
random-feature images of 101 region rows, 30 + 1 token captions, with that probe's synthetic ragged masks (1 + U{10..100} valid
regions, caption lengths U{15..30} + the task token), chunk=500. Arms, one after the other, each with a warm-up evaluation of the
same captions (plans, graph capture) and then --rounds timed ones:

  padded   RetrievalEvaluator with neither packing nor recycling (one plan per chunk size);
  packed   pack=True on recycled plans (engine.recycle_forward_only), as the packed arm of tools/retrieval_probe.py.

    torchrun --nproc-per-node W tools/retrieval_ddp_probe.py [--captions 200] [--rounds 2] [--arms padded,packed] [--out f.json]

With W = 1 the group has one rank and the evaluation takes the single-GPU path. Per arm and round it reports the wall time of the
whole evaluate_retrieval_both (dataset read, scoring, gather and both rankings, between two barriers) and ms per caption of it, and
per rank: the scoring time of its caption block and ms per caption of it, the time of the chunk loads and image prefixes inside
it, the agreement check (checksums included), the wait for the slowest rank before the gather and the all-gather itself. Each
rank reads its card's name and power limit in the same run."""
import argparse
import json
import os
import subprocess
import sys
import time
from datetime import timedelta

import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card(index):
    q = subprocess.run(["nvidia-smi", f"--id={index}", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm",
                        "--format=csv,noheader"], capture_output=True, text=True, timeout=30)
    if q.returncode != 0:
        return dict(name=torch.cuda.get_device_name(index), error=q.stderr.strip())
    name, power, sm, sm_max = [x.strip() for x in q.stdout.strip().splitlines()[0].split(",")]
    return dict(name=name, power_limit=power, sm_clock=sm, sm_clock_max=sm_max)


class Gallery:
    """The reference's retrieval item protocol (item 2c + h: caption c against gallery half h) over host tensors."""

    def __init__(self, feats, locs, imask, caps, amask, target):
        self.feats, self.locs, self.imask, self.caps, self.amask, self.target = feats, locs, imask, caps, amask, target
        self.H = feats.shape[0] // 2

    def __len__(self):
        return 2 * len(self.caps)

    def __getitem__(self, i):
        c, h = i // 2, i % 2
        sl = slice(h * self.H, (h + 1) * self.H)
        t = torch.zeros(self.H)
        if h * self.H <= self.target[c] < (h + 1) * self.H:
            t[self.target[c] - h * self.H] = 1
        return (self.feats[sl], self.locs[sl], self.imask[sl], self.caps[c], self.amask[c], torch.zeros_like(self.caps[c]), t, c, h)


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--captions", type=int, default=200)
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--images", type=int, default=1000)
    ap.add_argument("--arms", default="padded,packed")
    ap.add_argument("--chunk", type=int, default=500)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if "RANK" not in os.environ:
        raise SystemExit("retrieval_ddp_probe: run under torchrun (--nproc-per-node 1 for the single-GPU path)")
    arms = a.arms.split(",")
    bad = [x for x in arms if x not in ("padded", "packed")]
    if bad:
        raise SystemExit(f"retrieval_ddp_probe: unknown arm(s) {bad}")
    rank, world, local = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ["LOCAL_RANK"])
    dev = torch.device("cuda", local)
    torch.cuda.set_device(dev)
    dist.init_process_group("nccl", device_id=dev, timeout=timedelta(minutes=30))
    group = dist.group.WORLD
    import vilbert_b200
    from vilbert_b200 import retrieval as RT

    cfgj = dict(json.load(open(os.path.join(ROOT, "vilbert-multi-task_b200", "configs", "bert_base_6layer_6conect.json"))),
                task_specific_tokens=True)
    torch.manual_seed(0)
    model = vilbert_b200.VILBertForVLTasks(vilbert_b200.BertConfig.from_dict(cfgj))
    model.eval()
    eng = model.engine
    dist.broadcast(eng.ps.flat, 0, group=group)
    eng.shadow_clean = False
    eng.max_plans = 64      # every capacity group of every chunk stays built across the rounds
    G, Nv, Nt, C = a.images, 101, 30, a.captions
    feats = torch.relu(torch.randn(G, Nv, 2048))
    locs = torch.rand(G, Nv, 5)
    caps = torch.randint(1000, 30000, (C, Nt))
    imask = (torch.arange(Nv) < 1 + torch.randint(10, Nv, (G, 1))).long()
    feats.mul_(imask.unsqueeze(-1))
    locs.mul_(imask.unsqueeze(-1))
    amask = (torch.arange(Nt) < torch.randint((Nt + 1) // 2, Nt + 1, (C, 1))).long()
    ds = Gallery(feats.pin_memory(), locs.pin_memory(), imask.pin_memory(), caps, amask, (torch.arange(C) % G).tolist())

    # per-rank timers around the pieces of a sharded evaluation (each piece synchronises the device before and after)
    t = {}

    def timed(key, fn, before=None):
        def run(*args, **kw):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            if before:
                before()
                torch.cuda.synchronize()
                t[key + "_wait"] = t.get(key + "_wait", 0.0) + time.perf_counter() - t0
                t0 = time.perf_counter()
            r = fn(*args, **kw)
            torch.cuda.synchronize()
            t[key] = t.get(key, 0.0) + time.perf_counter() - t0
            if key == "score":
                t["captions"] = t.get("captions", 0) + int(args[1].shape[0])
            return r
        return run
    RT.RetrievalEvaluator._score_rows = timed("score", RT.RetrievalEvaluator._score_rows)
    RT.RetrievalEvaluator._load_chunk = timed("prefix", RT.RetrievalEvaluator._load_chunk)
    RT.check_agreement = timed("agreement", RT.check_agreement)
    RT.gather_rows = timed("gather", RT.gather_rows, before=lambda: dist.barrier(group=group, device_ids=[local]))

    res = dict(world=world, config="bert_base_6layer_6conect + task tokens", precision=eng.precision, images=G, regions=Nv,
               tokens=Nt + 1, captions=C, chunk=a.chunk, rounds=a.rounds, valid_regions=float(imask.float().mean()) * Nv,
               valid_tokens=float(amask.float().mean()) * Nt + 1, arms={})
    cards = [None] * world
    dist.all_gather_object(cards, card(local), group=group)
    res["cards"] = cards
    for arm in arms:
        eng.release_plans()
        torch.cuda.empty_cache()
        torch.cuda.reset_peak_memory_stats()
        eng.recycle_forward_only = arm == "packed"
        rounds, out = [], None
        for r in range(a.rounds + 1):           # round 0: the warm-up
            t.clear()
            dist.barrier(group=group, device_ids=[local])
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            out = RT.evaluate_retrieval_both(model, ds, task_id=8, chunk=a.chunk, k=20, pack=arm == "packed", group=group)
            torch.cuda.synchronize()
            dist.barrier(group=group, device_ids=[local])
            wall = time.perf_counter() - t0
            per_rank = [None] * world
            mine = dict(score_s=t.get("score", 0.0), captions=t.get("captions", 0), prefix_s=t.get("prefix", 0.0),
                        agreement_s=t.get("agreement"), wait_before_gather_s=t.get("gather_wait"), gather_s=t.get("gather"),
                        max_memory_allocated_gb=torch.cuda.max_memory_allocated() / 1e9)
            mine["score_ms_per_caption"] = 1e3 * mine["score_s"] / mine["captions"] if mine["captions"] else None
            dist.all_gather_object(per_rank, mine, group=group)
            if r > 0:
                rounds.append(dict(wall_s=wall, wall_ms_per_caption=1e3 * wall / C, ranks=per_rank))
        res["arms"][arm] = dict(rounds=rounds, fallbacks=dict(eng.pack_fallbacks), t2i_r1=out["t2i"][0], i2t_r1=out["i2t"][0],
                                rsum=out["rsum"])
    if rank == 0:
        text = json.dumps(res, indent=1)
        print(text)
        if a.out:
            os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
            with open(a.out, "w") as f:
                f.write(text + "\n")
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
