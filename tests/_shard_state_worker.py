"""2-rank worker of tests/test_shard_state_gpu.py (torch.distributed.run): per case, a model with an unsharded fused optimizer and a
model with shard_state=True run the same five VQA task steps (task tokens, the reference's per-tensor param groups with their own
lr and weight decay, lr halved from step 3 on) from the same parameters. After every step it records whether the sharded run's
fp32 weights and 16-bit copies equal the unsharded run's (bitwise under torch.use_deterministic_algorithms(True), else their
relative L2 distance, one step apart from the same state: see _run_lockstep), and whether they equal rank 0's. At the end it compares the gathered state_dict() and the moment buffers'
size. argv: output path, backend ("nccl": one GPU per rank; "gloo": both ranks on cuda:0)."""
import copy
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

Bl, NV, NT, STEPS = 4, 37, 23, 5
TEXT = ("bert.embeddings.", "bert.encoder.layer.")

# name -> options: opt (AdamW / RAdam), correct_bias, clip (max_grad_norm), nan_step (rank 1's features hold a NaN there), sib
# (step_in_backward), delay (delay_allreduce), accum (two micro-batches, the first under no_sync), freeze_at, packed, precision,
# det (deterministic algorithms), exact (bitwise expected: not when clipping, whose global norm the sharded step sums in another
# order), reload (state dict round trip into a fresh optimizer after step 2)
CASES = {
    "adamw_bias": dict(correct_bias=True),
    "adamw_nobias": dict(correct_bias=False),
    "radam": dict(opt="RAdam"),
    "clip_skip": dict(clip=1e6, nan_step=3),
    "clip_small": dict(clip=0.05, exact=False),
    "radam_clip_skip": dict(opt="RAdam", clip=1e6, nan_step=2),
    "sib_overlap": dict(sib=True, delay=False),
    "sib_delay": dict(sib=True, delay=True),
    "overlap_step": dict(delay=False),
    "accum": dict(accum=True),
    "freeze": dict(freeze_at=2),
    "packed": dict(packed=True),
    "fp32": dict(precision="fp32"),
    "nondet": dict(det=False),
    "reload": dict(reload=True),
}


def _copies(eng):
    ps = eng.ps
    return [t for t in (ps.flat, ps.shadow, ps.shadow_lo, ps.shadow_b) if t is not None]


def _groups(m):
    """The reference's grouping (train_tasks.py:401-421): one group per tensor, its own lr, no decay on biases and LayerNorms."""
    out = []
    for i, (name, p) in enumerate(m.named_parameters()):
        wd = 0.0 if ("bias" in name or "LayerNorm" in name) else 0.01
        out.append(dict(params=[p], lr=1e-3 if i % 3 else 4e-4, weight_decay=wd))
    return out


class _Run:
    """One model, its data-parallel wrapper and its optimizer (sharded or not) stepping through the case's batches."""

    def __init__(self, case, cfgj, params, rank, world, dev, shard):
        import vilbert_b200
        from vilbert_b200.ddp import DistributedDataParallel as DDP
        from vilbert_b200.tasks import LoadLosses
        self.o, self.cfgj, self.rank, self.world, self.dev, self.shard = CASES[case], cfgj, rank, world, dev, shard
        o = self.o
        self.m = m = vilbert_b200.VILBertForVLTasks(vilbert_b200.BertConfig.from_dict(cfgj), precision=o.get("precision", "fp16"))
        m.load_state_dict(params, strict=False)
        m.train()
        if o.get("packed"):
            m.engine.pack_padding = True
        self.d = DDP(m, delay_allreduce=o.get("delay", True))
        self.opt = self.make_opt()
        self.losses = LoadLosses(None, T.TASK_CFG, ["1"])

    def make_opt(self):
        from vilbert_b200.optim import FusedAdamW, FusedRAdam
        o, m = self.o, self.m
        kw = dict(model=self.d if self.shard else m, shard_state=self.shard, max_grad_norm=o.get("clip"))
        if o.get("opt") == "RAdam":
            return FusedRAdam(_groups(m), lr=1e-3, **kw)
        return FusedAdamW(_groups(m), lr=1e-3, correct_bias=o.get("correct_bias", False), **kw)

    def step(self, s):
        """Step s of the case; -> snapshot of the fp32 weights and 16-bit copies."""
        from vilbert_b200.tasks import ForwardModelsTrain
        o, m, d, opt, rank, world = self.o, self.m, self.d, self.opt, self.rank, self.world
        if s == 3:
            for g in opt.param_groups:
                g["lr"] *= 0.5
        if o.get("freeze_at") == s:
            for name, p in m.named_parameters():
                if name.startswith(TEXT):
                    p.requires_grad_(False)
        micro = 2 if o.get("accum") else 1
        for u in range(micro):
            b = T.make_batch(self.cfgj, "TASK1", Bl * world, NV, NT, seed=10 * s + u)
            batch = [t[rank * Bl:(rank + 1) * Bl].clone() for t in b]
            if o.get("nan_step") == s and rank == 1:
                batch[0][0, 1, 0] = float("nan")
            m.engine.set_dropout_step(100 + 10 * s + u)
            last = u == micro - 1
            ctx = d.no_sync() if not last else _null()
            with ctx:
                loss, _ = ForwardModelsTrain(None, T.TASK_CFG, self.dev, "TASK1", {"TASK1": 0}, {}, {"TASK1": [tuple(batch)]}, d,
                                             self.losses)
                if last and o.get("sib"):
                    with opt.step_in_backward():
                        loss.backward()
                else:
                    loss.backward()
        if not o.get("sib"):
            opt.step()
        m.zero_grad()
        return [t.clone() for t in _copies(m.engine)]


def _run(case, cfgj, params, rank, world, dev, shard, sd_in=None, sd_at=None):
    """The five steps of `case`; -> (snapshots per step, final state dict, the optimizer, the state dict after step 2 when sd_at).
    sd_in: after step 2 the optimizer is replaced by a fresh one (zero moments, counter 0) that loads sd_in."""
    run = _Run(case, cfgj, params, rank, world, dev, shard)
    snaps, sd_mid = [], None
    for s in range(STEPS):
        snaps.append(run.step(s))
        if s == 1 and sd_at is not None:
            sd_mid = copy.deepcopy(run.opt.state_dict())      # state_dict() holds references to the live moments
        if s == 1 and sd_in is not None:
            # only a correct load lets the fresh optimizer continue bitwise as the run it replaces
            run.opt = run.make_opt()
            run.opt.load_state_dict(sd_in)
    torch.cuda.synchronize()
    return snaps, run.opt.state_dict(), run.opt, sd_mid


def _run_lockstep(case, cfgj, params, rank, world, dev):
    """Default mode (no deterministic algorithms): the backward's float atomics make two runs drift apart step after step, sharded or
    not, so each step of the sharded run starts from the unsharded run's weights and optimizer state (loaded through its
    state_dict()) and the two are compared one step apart. -> (unsharded snapshots, sharded snapshots, their final state dicts,
    the sharded optimizer)."""
    a = _Run(case, cfgj, params, rank, world, dev, False)
    b = _Run(case, cfgj, params, rank, world, dev, True)
    base, shard = [], []
    for s in range(STEPS):
        with torch.no_grad():
            b.m.engine.ps.flat.copy_(a.m.engine.ps.flat)
        b.m.engine.shadow_clean = False
        b.opt.load_state_dict(copy.deepcopy(a.opt.state_dict()))
        base.append(a.step(s))
        shard.append(b.step(s))
    torch.cuda.synchronize()
    return base, shard, a.opt.state_dict(), b.opt.state_dict(), b.opt


class _null:
    def __enter__(self):
        return self

    def __exit__(self, *a):
        return False


def _rel(a, b):
    a, b = a.double(), b.double()
    return float((a - b).norm() / b.norm().clamp_min(1e-30))


def _same_state(a, b):
    if set(a["state"]) != set(b["state"]):
        return False
    return all(int(a["state"][k]["step"]) == int(b["state"][k]["step"]) and
               all(torch.equal(a["state"][k][n], b["state"][k][n]) and a["state"][k][n].shape == b["state"][k][n].shape
                   for n in ("exp_avg", "exp_avg_sq")) for k in a["state"])


def main():
    out_path, backend = sys.argv[1], sys.argv[2]
    rank, world, local = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ["LOCAL_RANK"])
    dev = torch.device("cuda", local if backend == "nccl" else 0)
    torch.cuda.set_device(dev)
    if backend == "nccl":
        dist.init_process_group("nccl", device_id=dev, timeout=timedelta(minutes=5))
    else:
        dist.init_process_group("gloo", timeout=timedelta(minutes=5))
    cfgj = dict(json.load(open(os.path.join(ROOT, "tests", "golden", "tiny_b4.json")))["config"], task_specific_tokens=True,
                max_position_embeddings=300)
    params = O.synth_params(O.make_config(cfgj), seed=3, device=dev)
    only = os.environ.get("SHARD_CASES")
    res = {}
    for case in CASES if not only else only.split(","):
        o = CASES[case]
        torch.use_deterministic_algorithms(o.get("det", True))
        if o.get("reload"):
            # the unsharded run saves after step 2; a sharded run replaces its optimizer by a fresh one at the same point and loads
            # that state dict into it (and the reverse): both must continue bitwise as the run they left
            base, sd_base, _, sd_mid_u = _run(case, cfgj, params, rank, world, dev, False, sd_at=True)
            shard, sd_shard, _, sd_mid_s = _run(case, cfgj, params, rank, world, dev, True, sd_in=sd_mid_u, sd_at=True)
            back, sd_back, _, _ = _run(case, cfgj, params, rank, world, dev, False, sd_in=sd_mid_s)
            eq = [all(torch.equal(x, y) for x, y in zip(a, b)) and all(torch.equal(x, y) for x, y in zip(a, c))
                  for a, b, c in zip(base, shard, back)]
            res[case] = dict(step_equal=eq, state_equal=_same_state(sd_shard, sd_base) and _same_state(sd_back, sd_base),
                             mid_equal=_same_state(sd_mid_s, sd_mid_u))
            continue
        if o.get("det", True):
            base, sd_base, _, _ = _run(case, cfgj, params, rank, world, dev, False)
            shard, sd_shard, opt, _ = _run(case, cfgj, params, rank, world, dev, True)
        else:
            base, shard, sd_base, sd_shard, opt = _run_lockstep(case, cfgj, params, rank, world, dev)
        step_equal = [all(torch.equal(x, y) for x, y in zip(a, b)) for a, b in zip(base, shard)]
        rel = max(_rel(x, y) for a, b in zip(shard, base) for x, y in zip(a[:1], b[:1]))
        ranks_equal = []
        for snap in shard:
            ok = True
            for t in snap:
                r0 = t.clone()
                dist.broadcast(r0, 0)
                ok &= bool(torch.equal(r0, t))
            ranks_equal.append(ok)
        n = sum(k for _, _, k, _ in opt._tracked)
        state_ok = _same_state(sd_shard, sd_base)
        state_rel = max((_rel(sd_shard["state"][k][nm], sd_base["state"][k][nm]) for k in sd_base["state"]
                         for nm in ("exp_avg", "exp_avg_sq")), default=0.0)
        res[case] = dict(step_equal=step_equal, rel=rel, ranks_equal=ranks_equal, state_equal=state_ok, state_rel=state_rel,
                         moments=int(opt.exp_avg.numel()), bound=int(-(-opt.engine.ps.numel // world) + 4 * len(opt._shard.table)),
                         trainable=n, det=o.get("det", True), exact=o.get("exact", True),
                         skipped=None if opt.max_grad_norm is None else int(opt.skipped_steps.item()))
    gathered = [None] * world
    dist.all_gather_object(gathered, res)
    if rank == 0:
        json.dump(gathered, open(out_path, "w"))
    dist.barrier()
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
