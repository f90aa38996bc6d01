"""Times caption-to-image retrieval at the reference's real shapes: bert_base_6layer_6conect with task tokens, 101 regions, 30 + 1
tokens, a gallery of 1,000 random-feature images, random weights. The arms of --arms alternate in one process after a warm-up:

  plain     RetrievalEvaluator(chunk=--chunk): each chunk loaded and embedded once, one graph replay per caption and chunk;
  recycled  the same with recycle=True at chunk=--recycled-chunk (default --chunk): the plans' buffers placed by lifetime;
  packed    the same with pack=True and recycle=True at chunk=--chunk: each (caption, chunk) pair on a plan that holds the chunk's
            valid regions and the caption's valid tokens only (DESIGN.md §4g). With this arm every arm runs on ragged masks: 1 +
            U{10..100} regions per image (the features of the other rows zero) and caption lengths U{15..30} + the task token
            (SURVEY.md §8d), as no real gallery is available here;
  module    the reference loop (eval_retrieval.py:264-313) restated on the module surface: model(...) per caption and gallery half
            with config.fast_mode set, the half's features copied from pinned host memory on every call, the scores read back
            with .cpu().

    python tools/retrieval_probe.py [--captions 200] [--rounds 3] [--arms plain,module] [--chunk 500] [--recycled-chunk N]
                                    [--out retrieval_probe.json]            (--arms plain,packed: the packed measurement)

Reports per arm ms per caption (median and min-max over the rounds), model TFLOP/s from the FLOPs of the plans' GEMMs and attentions,
and for the evaluator arms the bytes their plans hold (Plan.held_bytes); the card's name, power limit and SM clock; and how far
each arm's scores and ranks are from the first arm's; for the evaluator arms also the plans built and the time spent building them.
A packed arm's FLOPs are summed over the plans each caption ran on; attention is counted at the padded lengths in every arm."""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def plan_flops(plan):
    """Forward FLOPs of one run of a plan: 2 M N K per GEMM, 4 B H Nq Nk D per attention."""
    total = 0
    for fn, args, _ in plan.fwd:
        if fn is None:
            continue
        if fn.__name__ == "vb_gemm_bf16":
            g = args[0]._obj
            total += 2 * g.M * g.N * g.K
        elif fn.__name__ == "vb_attention_fwd":
            a = args[0]._obj
            total += 4 * a.B * a.H * a.Nq * a.Nk * a.D
    return total


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power, sm, sm_max = [x.strip() for x in q.split(",")]
        return dict(name=name, power_limit=power, sm_clock=sm, sm_clock_max=sm_max)
    except Exception as ex:         # the probe still reports what torch knows
        return dict(name=torch.cuda.get_device_name(), error=str(ex))


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--captions", type=int, default=200)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--images", type=int, default=1000)
    ap.add_argument("--arms", default="plain,module")
    ap.add_argument("--chunk", type=int, default=500)
    ap.add_argument("--recycled-chunk", type=int, default=0)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import vilbert_b200
    from vilbert_b200.retrieval import RetrievalEvaluator
    cfgj = dict(json.load(open(os.path.join(ROOT, "vilbert-multi-task_b200", "configs", "bert_base_6layer_6conect.json"))),
                task_specific_tokens=True)
    torch.manual_seed(0)
    model = vilbert_b200.VILBertForVLTasks(vilbert_b200.BertConfig.from_dict(cfgj))
    model.eval()
    G, Nv, Nt, C, half = a.images, 101, 30, a.captions, 500
    feats = torch.relu(torch.randn(G, Nv, 2048)).pin_memory()
    locs = torch.rand(G, Nv, 5).pin_memory()
    imask = torch.ones(G, Nv, dtype=torch.long).pin_memory()
    caps = torch.randint(1000, 30000, (C, Nt))
    amask = torch.ones(C, Nt, dtype=torch.long)
    amask[:, 20:] = torch.randint(0, 2, (C, Nt - 20)).sort(dim=1, descending=True)[0]
    ragged = "packed" in a.arms.split(",")
    if ragged:          # SURVEY.md §8d: 1 + U{10..100} regions (padded rows zero), caption lengths U{ceil(Nt / 2)..Nt}
        imask = (torch.arange(Nv) < 1 + torch.randint(10, Nv, (G, 1))).long()
        feats.mul_(imask.unsqueeze(-1))
        locs.mul_(imask.unsqueeze(-1))
        imask = imask.pin_memory()
        amask = (torch.arange(Nt) < torch.randint((Nt + 1) // 2, Nt + 1, (C, 1))).long()
    seg = torch.zeros(C, Nt, dtype=torch.long)
    target = torch.arange(C) % G

    arms = a.arms.split(",")
    bad = [x for x in arms if x not in ("plain", "recycled", "packed", "module")]
    if bad:
        raise SystemExit(f"retrieval_probe: unknown arm(s) {bad}")
    evs = {"plain": RetrievalEvaluator(model, feats, locs, imask, chunk=a.chunk, recycle=False),
           "recycled": RetrievalEvaluator(model, feats, locs, imask, chunk=a.recycled_chunk or a.chunk, recycle=True),
           "packed": RetrievalEvaluator(model, feats, locs, imask, chunk=a.chunk, recycle=True, pack=True)}
    eng = model.engine
    eng.max_plans = 64      # every capacity group of every chunk stays built across the rounds
    builds = {name: [0, 0.0] for name in evs}       # plans built, seconds spent building them

    def counting(name, ev):
        plan = ev._plan

        def wrapped(*args, **kw):
            n0, t0 = len(eng.plans), time.perf_counter()
            p = plan(*args, **kw)
            if len(eng.plans) > n0:
                torch.cuda.synchronize()
                builds[name][0] += 1
                builds[name][1] += time.perf_counter() - t0
            return p
        ev._plan = wrapped
    for name, ev in evs.items():
        counting(name, ev)

    def evaluator(name):
        return lambda n: evs[name].score(caps[:n], amask[:n], seg[:n], task_id=8)

    def module_loop(n):
        model.config.fast_mode = True
        out = np.zeros((n, G), dtype=np.float32)
        task = torch.full((1, 1), 8, dtype=torch.long, device="cuda")
        with torch.no_grad():
            for c in range(n):
                cap, m, s = caps[c:c + 1].cuda(), amask[c:c + 1].cuda(), seg[c:c + 1].cuda()
                for h in range(0, G, half):
                    sl = slice(h, h + half)
                    logit = model(cap, feats[sl].cuda(non_blocking=True), locs[sl].cuda(non_blocking=True), s, m,
                                  imask[sl].cuda(non_blocking=True), task_ids=task)[2]
                    out[c, sl] = logit.view(-1).cpu().numpy()
        model.config.fast_mode = False
        return torch.from_numpy(out).cuda()
    fns = {name: module_loop if name == "module" else evaluator(name) for name in arms}

    def timed(f, n):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        r = f(n)
        torch.cuda.synchronize()
        return (time.perf_counter() - t0) * 1e3 / n, r

    for f in fns.values():
        timed(f, 4)        # warm-up: plans, graph capture, kernels loaded
    times, scores = {k: [] for k in fns}, {}
    for _ in range(a.rounds):
        for name, f in fns.items():
            t, scores[name] = timed(f, C)
            times[name].append(t)
    res = dict(card=card(), config="bert_base_6layer_6conect + task tokens", images=G, regions=Nv, tokens=Nt + 1, captions=C,
               rounds=a.rounds, precision=eng.precision, ragged_masks=ragged,
               valid_regions=float(imask.float().mean()) * Nv, valid_tokens=float(amask.float().mean()) * Nt + 1, arms={})
    ranks0, _ = RetrievalEvaluator.rank(scores[arms[0]], target, k=20)
    for name in arms:
        med = statistics.median(times[name])
        if name == "module":
            pb = [p for p in eng.plans.values() if not p.image_prefix and p.B == half]
            flops, held = (plan_flops(pb[0]) * (G // half) if pb else 0), None
        elif name == "packed":
            ev = evs[name]
            plans = [(ev._plan(n, Nt, None if rt is None else (rt, rv)), len(group)) for _, n, rv, groups in ev._chunks(amask, True)
                     for rt, group in groups.items()]
            flops = sum(plan_flops(p) * k for p, k in plans) / C
            held = {str(p.packed): p.held_bytes for p, _ in plans}
        else:
            ps = [p for p in eng.plans.values() if p.image_prefix and p.recycle == (name == "recycled") and not p.packed]
            flops = sum(plan_flops(p) for p in ps for _ in range(G // p.B if p.B == evs[name].chunk else 1))
            held = {p.B: p.held_bytes for p in ps}
        ranks, _ = RetrievalEvaluator.rank(scores[name], target, k=20)
        res["arms"][name] = dict(chunk=None if name == "module" else evs[name].chunk,
                                 ms_per_caption=dict(median=med, min=min(times[name]), max=max(times[name])),
                                 tflops=flops / (med * 1e-3) / 1e12, flops_per_caption=flops, plan_held_bytes=held,
                                 max_abs_score_diff_vs_first=float((scores[name] - scores[arms[0]]).abs().max()),
                                 ranks_differing_vs_first=int((ranks != ranks0).sum()),
                                 plan_builds=builds.get(name, [None])[0], plan_build_s=builds.get(name, [None, None])[1])
    text = json.dumps(res, indent=1)
    print(text)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(text + "\n")


if __name__ == "__main__":
    main()
