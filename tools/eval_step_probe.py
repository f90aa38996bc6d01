"""Times one evaluation batch (eval_tasks.py:290, EvaluatingModel) per task type on one GPU in three ways, alternating them in the
same process:

  fused      vilbert_b200.tasks.EvaluatingModel: a forward-only plan with only the type's head, objective, score and
             vb_task_results; one device-to-host copy
  recycled   the same with engine.recycle_forward_only: the plan's buffers placed by lifetime (Plan(recycle=True))
  module     the module surface (VILBertForVLTasks.forward, all nine heads cloned) + the reference's step restated in
             tests/_eval_oracle.py (torch loss / score / softmax and one .item() per value)

    python tools/eval_step_probe.py [--iters K] [--warmup W] [--batches 30,256] [--arena-gb G] [--out DIR]

Model: bert_base_6layer_6conect with task tokens, random weights, eval mode. Shapes: the regions and tokens of the 12-in-1 tasks of
each evaluation type (bench.py's config 5) at eval_tasks.py's default --batch_size 30 and at 256. Batches are synthetic CPU tensors
(the arms move them to the GPU as the reference does). The arms' plans share one activation arena; an arm whose plan does not fit
is reported as not measured. Prints one JSON line (also written to DIR/eval_step_probe.json): per (type, batch) the median ms per
call of each arm and the bytes each arm's plan holds (Plan.held_bytes), with the card name and power limit. Needs a GPU."""
import argparse
import gc
import json
import os
import statistics
import subprocess
import sys
import types

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

# (type, task, regions, tokens, options) at the 12-in-1 shapes (bench.py config 5; VisDial: 100 options per round is eval_tasks.py's)
SHAPES = [("VL-classifier", "TASK1", 101, 23, 0), ("VL-classifier-GQA", "TASK15", 101, 26, 0), ("VL-logit", "TASK7", 101, 30, 4),
          ("V-logit", "TASK9", 101, 20, 0), ("V-logit-mc", "TASK4", 200, 20, 0), ("VL-binary-classifier", "TASK12", 101, 40, 0),
          ("VL-tri-classifier", "TASK13", 101, 56, 0)]


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--iters", type=int, default=7)
    ap.add_argument("--warmup", type=int, default=3)   # plans capture their CUDA graphs on the 3rd run
    ap.add_argument("--batches", default="30,256")
    ap.add_argument("--arena-gb", type=float, default=40.0)
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles"))
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("eval_step_probe: needs a GPU (there is nothing to time on the CPU)")
    import _eval_oracle as E
    import _task_oracle as T
    import vilbert_b200
    from vilbert_b200 import _lib as L
    from vilbert_b200.tasks import EvaluatingModel, LoadLosses
    cfgj = dict(json.load(open(os.path.join(ROOT, "vilbert-multi-task_b200", "configs", "bert_base_6layer_6conect.json"))), task_specific_tokens=True)
    model = vilbert_b200.VILBertForVLTasks(vilbert_b200.BertConfig.from_dict(cfgj))
    model.engine.enable_activation_arena(int(a.arena_gb * 2 ** 30))
    model.eval()
    dev = torch.device("cuda")
    rows = []
    for typ, task, Nv, Nt, opts in SHAPES:
        for B in (int(b) for b in a.batches.split(",")):
            cfg = {task: T.TASK_CFG[task]}
            batch = T.make_batch(cfgj, task, B, Nv, Nt, options=opts or 3, seed=B)
            label2ans = [f"answer {i}" for i in range(3129)]
            loader = {task: types.SimpleNamespace(dataset=types.SimpleNamespace(label2ans=label2ans))}
            losses = LoadLosses(None, cfg, [task[4:]])
            plans = {}

            def fused():
                EvaluatingModel(None, cfg, dev, task, batch, model, loader, losses, [], [])
                plans["fused"] = model._last_plan

            def recycled():
                model.engine.recycle_forward_only = True
                try:
                    EvaluatingModel(None, cfg, dev, task, batch, model, loader, losses, [], [])
                finally:
                    model.engine.recycle_forward_only = False
                plans["recycled"] = model._last_plan

            def module():
                E.evaluating_step(cfg, task, tuple(t.to(dev, non_blocking=True) for t in batch), model, label2ans, [], [])
                plans["module"] = model._last_plan
            arms = {"fused": fused, "recycled": recycled, "module": module}
            times = {k: [] for k in arms}
            row = {"type": typ, "task": task, "B": B, "regions": Nv, "tokens": Nt + 1, "options": opts or None}
            for i in range(a.warmup + a.iters):
                for name, fn in list(arms.items()):
                    torch.cuda.synchronize()
                    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    e0.record()
                    try:
                        fn()
                    except (L.VBError, torch.OutOfMemoryError) as ex:
                        row[f"not_measured_{name}"] = str(ex).splitlines()[0][:200]
                        del arms[name], times[name]
                        gc.collect()
                        torch.cuda.empty_cache()
                        continue
                    e1.record()
                    torch.cuda.synchronize()
                    if i >= a.warmup:
                        times[name].append(e0.elapsed_time(e1))
            row.update({f"ms_{k}_median": statistics.median(v) for k, v in times.items()})
            row.update({f"plan_bytes_{k}": p.held_bytes for k, p in plans.items() if k in arms})
            print(json.dumps(row), flush=True)
            rows.append(row)
            model.engine.release_plans()
            torch.cuda.empty_cache()
    res = {"what": "one EvaluatingModel call per task type, bert_base_6layer_6conect with task tokens, eval mode", "card": card(),
           "iters": a.iters, "warmup": a.warmup, "rows": rows}
    os.makedirs(a.out, exist_ok=True)
    with open(os.path.join(a.out, "eval_step_probe.json"), "w") as f:
        json.dump(res, f)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
