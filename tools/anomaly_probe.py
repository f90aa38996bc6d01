"""Cost of anomaly checks (torch.autograd.set_detect_anomaly(True), Plan(anomaly=True), DESIGN.md §4i) on the GPU.

    python tools/anomaly_probe.py [--steps 20] [--rounds 5] [--out FILE]

builds bench config 2 (bert_base_6layer_6conect, B=64, 100 regions x 36 tokens, train mode, VQA BCE objective) twice on one
engine, without and with the checks, captures each plan's forward + loss and backward as CUDA graphs, and times them alternately:
`rounds` rounds of `steps` steps per arm, a step being the forward graph, the backward graph and, in the checked arm, the
anomaly_report() read that the module surface makes after every backward (one host synchronisation). CUDA events around each
round. Prints one JSON line: median ms/step and range per arm, the overhead, the checks' launches and the bytes they read per step
(from the plan's region table), and the card's name and power limit read in the same run."""
import argparse
import json
import os
import statistics
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))


def checked_bytes(plan):
    """Bytes the vb_nan_check launches of one step read: every region's logical extent."""
    from vilbert_b200 import _lib as L
    es = {L.VB_NAN_F32: 4, L.VB_NAN_F16: 2, L.VB_NAN_BF16: 2}
    return sum(rows * cols * es[dt] for _, rows, cols, _, dt, _ in plan.nan_regions)


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--out")
    a = ap.parse_args()
    import torch
    import deterministic_probe as P
    from vilbert_b200.engine import LOSS_HEADS
    if not torch.cuda.is_available():
        raise SystemExit("anomaly_probe: no GPU")
    eng, plain = P.build("vqa", deterministic=False)
    checked = eng.plan(64, 36, 100, grad_outputs=LOSS_HEADS["vqa"], loss="vqa", train=True, anomaly=True)
    P.load(checked, "vqa", 0, P.bench_config())
    arms = {"off": plain, "on": checked}
    for plan in arms.values():
        plan.capture(separate=True)
    times = {k: [] for k in arms}
    for _ in range(a.rounds):
        for name, plan in arms.items():
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(a.steps):
                plan.run_forward()
                plan.run_backward()
                if plan.anomaly:
                    assert plan.anomaly_report() is None
            e1.record()
            torch.cuda.synchronize()
            times[name].append(e0.elapsed_time(e1) / a.steps)
    med = {k: statistics.median(v) for k, v in times.items()}
    gpu, power = P.card()
    n_checks = sum(1 for ops in (checked.fwd, checked.bwd) for fn, args, _ in ops if fn is not None and fn.__name__ == "vb_nan_check")
    res = dict(workload="config2 train fwd+loss+bwd graphs (B=64, 100x36)", gpu=gpu, power_limit=power, steps=a.steps, rounds=a.rounds,
               ms_off=round(med["off"], 3), ms_on=round(med["on"], 3), range_off=[round(min(times["off"]), 3), round(max(times["off"]), 3)],
               range_on=[round(min(times["on"]), 3), round(max(times["on"]), 3)],
               overhead_ms=round(med["on"] - med["off"], 3), overhead_pct=round(100 * (med["on"] / med["off"] - 1), 2),
               check_launches=n_checks, regions=len(checked.nan_records), bytes_checked=checked_bytes(checked))
    line = json.dumps(res)
    print(line)
    if a.out:
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
