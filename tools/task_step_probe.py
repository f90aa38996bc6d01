"""Times one 12-in-1 training iteration (train_tasks.py:520-551) on one GPU in two ways, alternating them in the same process:

  fused      vilbert_b200.tasks.ForwardModelsTrain + (loss * loss_scale).backward() per task, then one FusedAdamW step
  module     the module surface (VILBertForVLTasks.forward) + the task's torch objective and score as the reference forms them
             (tests/_task_oracle.py) + float(score) per task (the reference's host read-back), then the same FusedAdamW step

    python tools/task_step_probe.py [--iters K] [--warmup W] [--batch-div D] [--arena-gb G] [--out DIR]

Model: bert_base_6layer_6conect with task tokens, random weights. Shapes: the 12 tasks of bench.py's config 5 (the same regions and
tokens) with their batches divided by D (default 4: at the full batches the module path's all-heads outputs of the largest
task do not fit next to the activation arena on one 80 GB card), each with its own objective of the task table. Batches are synthetic and already on the
GPU (no data loading). Prints one JSON line (also written to DIR/task_step_probe.json) with the median ms per iteration of each path,
the card name, power limit and SM clocks. Needs a GPU."""
import argparse
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

# (task, batch, regions, tokens) of bench.py's config 5; TASK17 carries 204 multiple-choice ids
SHAPES = [("TASK1", 128, 101, 23), ("TASK2", 128, 101, 26), ("TASK4", 256, 200, 20), ("TASK7", 128, 101, 30), ("TASK8", 128, 101, 30),
          ("TASK9", 256, 101, 20), ("TASK10", 256, 101, 20), ("TASK11", 256, 101, 20), ("TASK12", 64, 101, 40), ("TASK13", 256, 101, 56),
          ("TASK15", 128, 101, 26), ("TASK17", 64, 306, 256)]
LOSS_SCALE = {"TASK1": 2.0, "TASK2": 2.0, "TASK15": 2.0}      # task lr / min task lr in the 12-in-1 mix (train_tasks.py:247-251)


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--iters", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=3)   # the module surface captures its CUDA graphs on the 3rd run of a plan
    ap.add_argument("--batch-div", type=int, default=4)
    ap.add_argument("--arena-gb", type=float, default=40.0)
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles"))
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("task_step_probe: needs a GPU (there is nothing to time on the CPU)")
    import _task_oracle as T
    import vilbert_b200
    from vilbert_b200.optim import FusedAdamW
    from vilbert_b200.tasks import ForwardModelsTrain, LoadLosses
    cfgj = dict(json.load(open(os.path.join(ROOT, "vilbert-multi-task_b200", "configs", "bert_base_6layer_6conect.json"))), task_specific_tokens=True)
    model = vilbert_b200.VILBertForVLTasks(vilbert_b200.BertConfig.from_dict(cfgj))
    model.engine.enable_activation_arena(int(a.arena_gb * 2 ** 30))
    model.engine.max_plans = 2 * len(SHAPES) + 4      # both paths keep their plans of every shape
    model.train()
    opt = FusedAdamW(list(model.parameters()), lr=4e-5, correct_bias=False, model=model)
    tasks = [t for t, *_ in SHAPES]
    losses = LoadLosses(None, T.TASK_CFG, [t[4:] for t in tasks])
    dev = torch.device("cuda")
    shapes = [(t, max(2, B // a.batch_div // 2 * 2), Nv, Nt) for t, B, Nv, Nt in SHAPES]
    batches = {t: tuple(x.to(dev) for x in T.make_batch(cfgj, t, B, Nv, Nt, options=4, C=204 if t == "TASK17" else 4, seed=i))
               for i, (t, B, Nv, Nt) in enumerate(shapes)}

    def fused():
        for t in tasks:
            loss, score = ForwardModelsTrain(None, T.TASK_CFG, dev, t, {t: 1}, {t: iter([batches[t]])}, {t: [batches[t], None]}, model, losses)
            (loss * LOSS_SCALE.get(t, 1.0)).backward()
        opt.step()
        model.zero_grad()

    def module():
        for t in tasks:
            loss, score, bs = T.reference_step(T.kind_of(t), T.TASK_CFG[t]["process"], t, batches[t], model)
            float(score)
            (loss * LOSS_SCALE.get(t, 1.0)).backward()
        opt.step()
        model.zero_grad()

    paths = {"fused": fused, "module": module}
    times = {k: [] for k in paths}
    for i in range(a.warmup + a.iters):
        for name, fn in paths.items():
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            fn()
            e1.record()
            torch.cuda.synchronize()
            if i >= a.warmup:
                times[name].append(e0.elapsed_time(e1))
    res = {"what": "one 12-in-1 iteration (12 tasks fwd+bwd + FusedAdamW), bert_base_6layer_6conect, task tokens",
           "shapes": shapes,
           "card": card(), "iters": a.iters, "warmup": a.warmup,
           "ms_fused_median": statistics.median(times["fused"]), "ms_module_median": statistics.median(times["module"]),
           "ms_fused": times["fused"], "ms_module": times["module"]}
    os.makedirs(a.out, exist_ok=True)
    with open(os.path.join(a.out, "task_step_probe.json"), "w") as f:
        json.dump(res, f)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
