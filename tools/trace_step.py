"""Kernel-level timeline of one captured training step (development tool).

Replays the step graph under torch.profiler (CUPTI activity records: per-kernel start/end/stream, also for graph nodes) and
prints: busy time per stream, time with k kernels running concurrently, per-kernel-name totals of GPU time, and the idle
gaps of the whole device. Tells whether the step is bound by the sum of kernel times or by dependencies / launch gaps.
Writes the raw records to profiles/trace_step.json.
"""
import json, os, sys, collections
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch
from torch.profiler import profile, ProfilerActivity
from vilbert_b200 import BertConfig
from vilbert_b200.engine import Engine

dev = torch.device("cuda", 0)
cfgj = json.load(open(os.path.join(ROOT, "vilbert-multi-task_b200", "configs", "bert_base_6layer_6conect.json")))
B, Nt, Nv = 64, 36, 100
eng = Engine(BertConfig.from_dict(cfgj), dev)
g = torch.Generator(device=dev).manual_seed(0)
eng.ps.flat.normal_(0.0, 0.02, generator=g)
for name in eng.ps.entries:
    if "LayerNorm" in name or ".logit_fc.2." in name:
        eng.ps.p(name).fill_(1.0 if name.endswith("weight") else 0.0)
    elif name.endswith(".bias"):
        eng.ps.p(name).zero_()
plan = eng.plan(B, Nt, Nv, grad_outputs=("vil_prediction",), vqa_loss=True, train=True)
plan.enable_training_prologue()
gc = torch.Generator().manual_seed(1234)
inp = (torch.randint(1, 30522, (B, Nt), generator=gc), torch.randn(B, Nv, 2048, generator=gc), torch.rand(B, Nv, 5, generator=gc),
       torch.zeros(B, Nt, dtype=torch.long), torch.ones(B, Nt, dtype=torch.long), torch.ones(B, Nv, dtype=torch.long))
plan.load_inputs(*inp)
plan.vqa_target.copy_(torch.rand(B, 3129, generator=gc))
plan.capture()
for _ in range(5): plan.run_step()
torch.cuda.synchronize()

with profile(activities=[ProfilerActivity.CUDA, ProfilerActivity.CPU]) as prof:
    for _ in range(3): plan.run_step()
    torch.cuda.synchronize()
ev = []
os.makedirs(os.path.join(ROOT, "profiles"), exist_ok=True)
prof.export_chrome_trace(os.path.join(ROOT, "profiles", "trace_step_chrome.json"))
tr = json.load(open(os.path.join(ROOT, "profiles", "trace_step_chrome.json")))
for x in tr["traceEvents"]:
    if x.get("cat") == "kernel":
        ev.append((x["ts"], x["ts"] + x["dur"], x["name"], x.get("args", {}).get("stream")))
os.remove(os.path.join(ROOT, "profiles", "trace_step_chrome.json"))
ev.sort()
print(f"{len(ev)} kernel records over 3 steps")
# keep the middle step: split at the two largest gaps between "step_bump"-like starts -> simpler: take the middle third by count
n = len(ev) // 3
mid = ev[n:2 * n]
t0, t1 = mid[0][0], max(e[1] for e in mid)
print(f"middle step: {n} kernels, span {(t1 - t0) / 1e3:.3f} ms")
by_stream = collections.defaultdict(float); by_name = collections.defaultdict(lambda: [0, 0.0])
for s, e, nm, st in mid:
    by_stream[st] += e - s
    short = nm.split("<")[0].split("(")[0][-60:]
    if "gemm_wgmma" in nm:
        short = "gemm " + nm[nm.find("<"):nm.find(">") + 1]
    by_name[short][0] += 1; by_name[short][1] += e - s
print("busy time per stream (ms):", {k: round(v / 1e3, 3) for k, v in by_stream.items()})
print("sum of kernel durations: %.3f ms" % (sum(e - s for s, e, _, _ in mid) / 1e3))
# concurrency histogram
pts = []
for s, e, _, _ in mid: pts += [(s, 1), (e, -1)]
pts.sort()
lvl, last, hist = 0, pts[0][0], collections.defaultdict(float)
for t, d in pts:
    hist[lvl] += t - last; last = t; lvl += d
print("time with k kernels in flight (ms):", {k: round(v / 1e3, 3) for k, v in sorted(hist.items())})
print("kernel classes by GPU time:")
for nm, (c, tt) in sorted(by_name.items(), key=lambda kv: -kv[1][1])[:28]:
    print(f"  {nm:70s} n={c:4d} {tt / 1e3:8.3f} ms  avg {tt / c:7.1f} us")
json.dump([(s - t0, e - t0, nm[:120], st) for s, e, nm, st in mid], open(os.path.join(ROOT, "profiles", "trace_step.json"), "w"))
