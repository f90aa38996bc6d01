"""Backward time of the engine with input gradients (Plan(input_grads=...)), at the config-2 shape of bench.py
(bert_base_6layer_6conect, B=64, 100 regions x 36 tokens), for three plans:

  train                 train mode, every parameter trainable, VQA BCE objective
  train_input_grads     the same, also differentiating the region features and boxes
  saliency              eval mode, every parameter frozen, d(vil_prediction) into the features and boxes only

Each plan's forward and backward are captured as separate CUDA graphs; the forward is replayed once and the backward graph --steps
times per CUDA-event window, the plans alternating within each of --reps repetitions. Prints the median backward time, the
backward launch count, and the card, its power limit and SM clock read in the same run.

    python tools/input_grad_probe.py [--steps 20] [--reps 7] [--out DIR]
"""
import argparse
import json
import os
import statistics
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--batch", type=int, default=64)
    ap.add_argument("--out", default=None, help="also write the results as JSON under this directory")
    a = ap.parse_args()
    import torch
    from freeze_probe import card
    from oracle import vilbert_oracle as O
    from vilbert_b200.config import BertConfig
    from vilbert_b200.engine import INPUT_GRAD_NAMES, LOSS_HEADS, Engine
    if not torch.cuda.is_available():
        raise SystemExit("input_grad_probe: needs a CUDA device")
    cfgj = json.load(open(os.path.join(ROOT, "vilbert-multi-task_b200", "configs", "bert_base_6layer_6conect.json")))
    B, Nv, Nt = a.batch, 100, 36
    eng = Engine(BertConfig.from_dict(cfgj), "cuda")
    eng.refresh_weights()
    cfg = O.make_config(cfgj)
    inp = O.synth_inputs(cfg, B, Nv, Nt, seed=0, device="cuda")
    both = frozenset(INPUT_GRAD_NAMES)
    train = dict(grad_outputs=LOSS_HEADS["vqa"], vqa_loss=True, train=True)
    kinds = {"train": train, "train_input_grads": dict(train, input_grads=both),
             "saliency": dict(grad_outputs=("vil_prediction",), frozen=frozenset(eng.ps.entries), input_grads=both)}
    plans, res = {}, {}
    for name, kw in kinds.items():
        plan = eng.plan(B, Nt, Nv, **kw)
        plan.load_inputs(inp["input_txt"], inp["input_imgs"], inp["image_loc"], inp["token_type_ids"], inp["attention_mask"],
                         inp["image_attention_mask"], inp["task_ids"])
        if plan.loss_kind == "vqa":
            plan.vqa_target.copy_(O.synth_vqa_target(B, 3129, device="cuda"))
        else:
            plan.gout["vil_prediction"].normal_()
        plan.capture(separate=True)
        plans[name] = plan
        res[name] = dict(bwd_launches=plan.n_kernels_bwd, ms=[])
    for plan in plans.values():            # warm-up of every graph
        for _ in range(3):
            plan.run_forward()
            plan.run_backward()
    torch.cuda.synchronize()
    for _ in range(a.reps):
        for name, plan in plans.items():
            plan.run_forward()
            e0, e1 = torch.cuda.Event(True), torch.cuda.Event(True)
            e0.record()
            for _ in range(a.steps):
                plan.graph_bwd.replay()
            e1.record()
            torch.cuda.synchronize()
            res[name]["ms"].append(e0.elapsed_time(e1) / a.steps)
    info = card()
    print(f"card: {info}")
    print(f"config 2 shape: bert_base_6layer_6conect B={B} Nv={Nv} Nt={Nt}; backward graph replays, median of {a.reps} x {a.steps}")
    print(f"{'plan':20s} {'median ms':>10s} {'min':>8s} {'max':>8s} {'bwd launches':>13s}")
    for name, r in res.items():
        r["median_ms"] = statistics.median(r["ms"])
        print(f"{name:20s} {r['median_ms']:10.3f} {min(r['ms']):8.3f} {max(r['ms']):8.3f} {r['bwd_launches']:13d}")
    t, ti, s = (res[k]["median_ms"] for k in ("train", "train_input_grads", "saliency"))
    print(f"input gradients add {ti - t:.3f} ms ({100 * (ti - t) / t:.2f} %) to the training backward; "
          f"the saliency backward takes {100 * s / t:.1f} % of it")
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "input_grad_probe.json"), "w") as f:
            json.dump(dict(card=info, batch=B, steps=a.steps, reps=a.reps, results=res), f, indent=1)


if __name__ == "__main__":
    main()
