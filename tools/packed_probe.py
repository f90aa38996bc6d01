"""Padded vs packed task steps (engine.pack_padding) at config 2 (bert_base_6layer_6conect) with the benchmark's synthetic mask
distribution: text lengths U{ceil(Nt/2)..Nt}, region counts U{10..Nv}. Per shape: ms per ForwardModelsTrain + backward in train mode
(every dropout active; the packed plan draws the padded plan's masks; the plans' passes replay as CUDA graphs after two eager runs),
plan builds, fallbacks and peak memory, with the card, its power limit and clocks read in the same run. GPU only:
python tools/packed_probe.py [--steps 20]."""
import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]
import vilbert_b200  # noqa: E402
from vilbert_b200.tasks import ForwardModelsTrain, LoadLosses  # noqa: E402

TASK_CFG = {"TASK1": dict(type="VL-classifier", loss="BCEWithLogitLoss", process="normal"),
            "TASK9": dict(type="V-logit", loss="BCEWithLogitLoss", process="normal"),
            "TASK4": dict(type="V-logit-mc", loss="BCEWithLogitLoss", process="normal"),
            "TASK17": dict(type="V-logit-mc", loss="BCEWithLogitLoss", process="normal")}
# (task, batch, regions, tokens): config 2's VQA shape, then VQA, refcoco, Visual7w and GuessWhatPointing shapes of the 12-in-1 table
SHAPES = [("TASK1", 64, 101, 36), ("TASK1", 128, 101, 23), ("TASK9", 128, 101, 20), ("TASK4", 64, 200, 20), ("TASK17", 16, 306, 256)]


def batch(task_id, B, Nv, Nt, Fv, V, seed):
    g = torch.Generator().manual_seed(seed)
    feats = torch.rand(B, Nv, Fv, generator=g)
    loc = torch.rand(B, Nv, 5, generator=g)
    nv = torch.randint(10, Nv + 1, (B,), generator=g)
    imask = (torch.arange(Nv) < nv.unsqueeze(1)).long()
    nt = torch.randint((Nt + 1) // 2, Nt + 1, (B,), generator=g)
    tmask = (torch.arange(Nt) < nt.unsqueeze(1)).long()
    q = torch.randint(0, V, (B, Nt), generator=g)
    seg = torch.zeros_like(q)
    co = torch.zeros(B, Nv, Nt)
    qid = torch.arange(B)
    if task_id == "TASK1":
        t = torch.zeros(B, 3129); t[:, 5] = 1.0
        return (feats, loc, imask, q, t, tmask, seg, co, qid)
    if task_id == "TASK9":
        return (feats, loc, imask, q, (torch.rand(B, Nv, 1, generator=g) * imask.unsqueeze(-1)).round(), tmask, seg, co, qid)
    C = 4 if task_id == "TASK4" else 204           # choices on the first regions after 101, always valid here
    mc = torch.arange(C).repeat(B, 1) % 9
    imask[:, :110] = 1
    return (feats, loc, imask, q, torch.zeros(B, C, 1), tmask, seg, mc, co, qid)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    a = ap.parse_args()
    cfgj = json.load(open(os.path.join(ROOT, "vilbert-multi-task_b200", "configs", "bert_base_6layer_6conect.json")))
    cfgj.update(task_specific_tokens=True)
    model = vilbert_b200.VILBertForVLTasks(vilbert_b200.BertConfig.from_dict(cfgj))
    model.train()
    eng = model.engine
    eng.enable_activation_arena(24 << 30)      # the plans of every shape and capacity overlay one arena, as in 12-in-1 training
    dev = torch.device("cuda")
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip()
    print(json.dumps({"gpu": torch.cuda.get_device_name(), "nvidia_smi name, power limit, sm clock, max sm clock": card}), flush=True)
    for task_id, B, Nv, Nt in SHAPES:
        losses = LoadLosses(None, TASK_CFG, [task_id[4:]])
        bs = [batch(task_id, B, Nv, Nt, cfgj["v_feature_size"], cfgj["vocab_size"], s) for s in range(4)]
        row = dict(task=task_id, B=B, Nv=Nv, Nt=Nt)
        for pack in (False, True, False, True):      # alternated: the second pair is the one reported
            eng.pack_padding = pack
            model._last_plan = None
            eng.release_plans(); eng.plan_builds.clear(); eng.pack_fallbacks.clear()
            torch.cuda.synchronize(); torch.cuda.reset_peak_memory_stats()

            def step(i):
                loss, _ = ForwardModelsTrain(None, TASK_CFG, dev, task_id, {task_id: 0}, {}, {task_id: [bs[i % 4]]}, model, losses)
                loss.backward()
            for i in range(6):
                step(i)
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for i in range(a.steps):
                step(i)
            e1.record(); torch.cuda.synchronize()
            key = "packed" if pack else "padded"
            row[key] = dict(ms_per_step=e0.elapsed_time(e1) / a.steps, plan_builds=sum(eng.plan_builds.values()),
                            fallbacks=dict(eng.pack_fallbacks), peak_gb=torch.cuda.max_memory_allocated() / 2**30)
        row["speedup"] = row["padded"]["ms_per_step"] / row["packed"]["ms_per_step"]
        print(json.dumps(row), flush=True)


if __name__ == "__main__":
    main()
