"""Forward + backward time of the engine with frozen parameters (Plan(frozen=...)), at the config-2 shape of bench.py
(bert_base_6layer_6conect, B=64, 100 regions x 36 tokens, all heads + the VQA BCE objective), for four patterns:

  all_trainable                 nothing frozen
  text_below_first_connection   text embeddings + the text layers before the first connection layer
  vision_stream                 image embeddings + image layers + the image-side projections (query1 / key1 / value1) of the
                                connection layers
  heads_only                    every bert.* parameter

For each it prints the median step time over --reps CUDA-event windows of --steps captured steps (patterns alternate within
each repetition), the backward launch count and the bytes of the flat gradient buffer a data-parallel step all-reduces. The
card, its power limit and SM clock are read in the same run.

    python tools/freeze_probe.py [--steps 20] [--reps 5] [--out DIR]
"""
import argparse
import json
import os
import re
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def patterns(cfg, names):
    first_t = cfg.t_biattention_id[0]
    text = [n for n in names if n.startswith("bert.embeddings.") or any(n.startswith(f"bert.encoder.layer.{i}.") for i in range(first_t))]
    image = [n for n in names if n.startswith(("bert.v_embeddings.", "bert.encoder.v_layer.")) or
             re.match(r"bert\.encoder\.c_layer\.\d+\.biattention\.(query1|key1|value1)\.", n)]
    return {"all_trainable": frozenset(), "text_below_first_connection": frozenset(text), "vision_stream": frozenset(image),
            "heads_only": frozenset(n for n in names if n.startswith("bert."))}


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm,clocks.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError) as ex:
        return f"nvidia-smi unavailable: {ex}"


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--batch", type=int, default=64)
    ap.add_argument("--out", default=None, help="also write the results as JSON under this directory")
    a = ap.parse_args()
    import torch
    from oracle import vilbert_oracle as O
    from vilbert_b200.config import BertConfig
    from vilbert_b200.ddp import trainable_ranges
    from vilbert_b200.engine import LOSS_HEADS, Engine
    if not torch.cuda.is_available():
        raise SystemExit("freeze_probe: needs a CUDA device")
    cfgj = json.load(open(os.path.join(ROOT, "vilbert-multi-task_b200", "configs", "bert_base_6layer_6conect.json")))
    B, Nv, Nt = a.batch, 100, 36
    eng = Engine(BertConfig.from_dict(cfgj), "cuda")
    cfg = O.make_config(cfgj)
    inp = O.synth_inputs(cfg, B, Nv, Nt, seed=0, device="cuda")
    pats = patterns(eng.cfg, list(eng.ps.entries))
    plans, res = {}, {}
    for name, frozen in pats.items():
        plan = eng.plan(B, Nt, Nv, grad_outputs=LOSS_HEADS["vqa"], vqa_loss=True, train=True, frozen=frozen)
        plan.load_inputs(inp["input_txt"], inp["input_imgs"], inp["image_loc"], inp["token_type_ids"], inp["attention_mask"],
                         inp["image_attention_mask"], inp["task_ids"])
        plan.vqa_target.copy_(O.synth_vqa_target(B, 3129, device="cuda"))
        plan.enable_training_prologue()
        plan.capture()
        plans[name] = plan
        reduced = sum(hi - lo for lo, hi in trainable_ranges(eng.ps, frozen))
        res[name] = dict(frozen_params=len(frozen), bwd_launches=plan.n_kernels_bwd, fwd_launches=plan.n_kernels_fwd,
                         allreduce_bytes=4 * reduced, ms=[])
    for plan in plans.values():            # warm-up of every graph
        for _ in range(3):
            plan.run_step()
    torch.cuda.synchronize()
    for _ in range(a.reps):
        for name, plan in plans.items():
            e0, e1 = torch.cuda.Event(True), torch.cuda.Event(True)
            e0.record()
            for _ in range(a.steps):
                plan.run_step()
            e1.record()
            torch.cuda.synchronize()
            res[name]["ms"].append(e0.elapsed_time(e1) / a.steps)
    info = card()
    print(f"card: {info}")
    print(f"config 2 shape: bert_base_6layer_6conect B={B} Nv={Nv} Nt={Nt}, train mode, VQA BCE, forward + backward as one graph per step")
    print(f"{'pattern':32s} {'median ms':>10s} {'min':>8s} {'max':>8s} {'bwd launches':>13s} {'all-reduce MB':>14s}")
    for name, r in res.items():
        r["median_ms"] = statistics.median(r["ms"])
        print(f"{name:32s} {r['median_ms']:10.2f} {min(r['ms']):8.2f} {max(r['ms']):8.2f} {r['bwd_launches']:13d} {r['allreduce_bytes'] / 2**20:14.1f}")
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "freeze_probe.json"), "w") as f:
            json.dump(dict(card=info, batch=B, steps=a.steps, reps=a.reps, results=res), f, indent=1)


if __name__ == "__main__":
    main()
