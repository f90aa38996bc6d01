"""Times the fused optimizer step inside the backward (optimizer.step_in_backward) against the step after it, on one GPU, module
surface on CUDA graphs, train mode with every dropout active, the arms alternating in one process:

  a  loss.backward(); opt.step()
  b  with opt.step_in_backward(): loss.backward()
  c  loss.backward() alone (the floor: no step at all)

    python tools/step_in_backward_probe.py [--windows 5] [--steps 10] [--warmup 3] [--sweep] [--out DIR]

Workloads on bert_base_6layer_6conect with random weights and synthetic batches already on the GPU: VQA ForwardModelsTrain at
config-2 shape (B = 64, 101 regions x 36 tokens, task tokens) with FusedAdamW, the fused pre-training step at config-3 shape
(B = 64, 37 regions x 36 tokens) with FusedAdamW, and the VQA step with FusedRAdam. Each arm runs `windows` windows of `steps`
steps (each window timed with CUDA events around it, ending in a synchronize); the median and range over the windows are reported
in ms per step. --sweep first times the VQA FusedAdamW workload over the single-process bucket count (optim.STEP_BUCKETS), the CTA
cap of the step launches (optim.STEP_MAX_CTAS), a higher-priority side stream, and backward GEMMs that leave SMs free
(engine.bwd_gemm_max_ctas). Prints one JSON line (also written to DIR/step_in_backward_probe.json) with the card name, power
limit and SM clocks read in the same run. Needs a GPU."""
import argparse
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
CONFIG = os.path.join(ROOT, "vilbert-multi-task_b200", "configs", "bert_base_6layer_6conect.json")


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def vqa(opt_name):
    import torch
    import _task_oracle as T
    import vilbert_b200
    from vilbert_b200.optim import FusedAdamW, FusedRAdam
    from vilbert_b200.tasks import ForwardModelsTrain, LoadLosses
    cfgj = dict(json.load(open(CONFIG)), task_specific_tokens=True)
    model = vilbert_b200.VILBertForVLTasks(vilbert_b200.BertConfig.from_dict(cfgj))
    model.train()
    opt = (FusedAdamW(list(model.parameters()), lr=4e-5, correct_bias=False, model=model) if opt_name == "adamw" else
           FusedRAdam(list(model.parameters()), lr=4e-5, model=model))
    dev = torch.device("cuda")
    batch = tuple(x.to(dev) for x in T.make_batch(cfgj, "TASK1", 64, 101, 36, seed=0))
    losses = LoadLosses(None, T.TASK_CFG, ["1"])

    def loss():
        return ForwardModelsTrain(None, T.TASK_CFG, dev, "TASK1", {"TASK1": 0}, {}, {"TASK1": [batch]}, model, losses)[0]
    return model, opt, loss


def pretraining():
    import torch
    import vilbert_b200
    from oracle import vilbert_oracle as O
    from vilbert_b200.optim import FusedAdamW
    cfgj = json.load(open(CONFIG))
    model = vilbert_b200.BertForMultiModalPreTraining(vilbert_b200.BertConfig.from_dict(cfgj), fused_objective=True)
    model.train()
    opt = FusedAdamW(list(model.parameters()), lr=1e-4, correct_bias=False, model=model)
    cfg = O.make_config(cfgj)
    B, NV, NT = 64, 37, 36
    inp = O.synth_inputs(cfg, B, NV, NT, seed=0, device="cuda")
    g = torch.Generator().manual_seed(0)
    lm = torch.full((B, NT), -1, dtype=torch.long)
    sel = torch.rand(B, NT, generator=g) < 0.15
    lm[sel] = torch.randint(0, cfg["vocab_size"], (int(sel.sum()),), generator=g)
    il = torch.full((B, NV - 1), -1, dtype=torch.long)
    il[torch.rand(B, NV - 1, generator=g) < 0.15] = 1
    it = torch.softmax(torch.randn(B, NV - 1, cfg["v_target_size"], generator=g), -1)
    ns = torch.randint(0, 2, (B,), generator=g)
    args = [inp[k] for k in ("input_txt", "input_imgs", "image_loc", "token_type_ids", "attention_mask", "image_attention_mask")]
    args += [x.cuda() for x in (lm, il, it, ns)]

    def loss():
        return sum(model(*args)).sum()
    return model, opt, loss


def time_arms(model, opt, loss, windows, steps, warmup):
    """-> {arm: [ms per step of each window]}, the arms alternating window by window."""
    import torch

    def a():
        loss().backward()
        opt.step()

    def b():
        with opt.step_in_backward():
            loss().backward()
        assert opt._stepped, "the step did not run in the backward"

    def c():
        loss().backward()
    arms = {"a_step_after": a, "b_step_in_backward": b, "c_backward_only": c}
    for fn in arms.values():
        for _ in range(warmup):          # the module surface captures its graphs on the 3rd run of a plan and of its pieces
            fn()
    times = {k: [] for k in arms}
    for _ in range(windows):
        for name, fn in arms.items():
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(steps):
                fn()
            e1.record()
            torch.cuda.synchronize()
            times[name].append(e0.elapsed_time(e1) / steps)
    model.zero_grad()
    return times


def summary(times):
    out = {k: {"ms_median": round(statistics.median(v), 3), "ms_min": round(min(v), 3), "ms_max": round(max(v), 3)} for k, v in times.items()}
    a, b, c = (out[k]["ms_median"] for k in ("a_step_after", "b_step_in_backward", "c_backward_only"))
    out["step_exposed_ms"] = {"a": round(a - c, 3), "b": round(b - c, 3)}
    out["hidden_fraction"] = round((a - b) / (a - c), 3) if a > c else None
    return out


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--windows", type=int, default=5)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--sweep", action="store_true")
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles"))
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("step_in_backward_probe: needs a GPU (there is nothing to time on the CPU)")
    from vilbert_b200 import optim
    res = {"card_before": card(), "windows": a.windows, "steps_per_window": a.steps, "warmup": a.warmup,
           "defaults": {"STEP_BUCKETS": optim.STEP_BUCKETS, "STEP_MAX_CTAS": optim.STEP_MAX_CTAS}}
    run = lambda m, o, l: summary(time_arms(m, o, l, a.windows, a.steps, a.warmup))   # noqa: E731
    if a.sweep:
        model, opt, loss = vqa("adamw")
        sweep = []
        base = (optim.STEP_BUCKETS, optim.STEP_MAX_CTAS)
        settings = [(nb, cap, 0, 0) for nb in (4, 8, 16) for cap in (0, 264, 132)] + [(8, 0, -1, 0), (8, 0, 0, 116), (8, 132, 0, 116)]
        for nb, cap, prio, gemm in settings:
            optim.STEP_BUCKETS, optim.STEP_MAX_CTAS = nb, cap
            opt._single_tables.clear()
            opt._side = torch.cuda.Stream(priority=prio)
            model.engine.bwd_gemm_max_ctas = gemm
            r = run(model, opt, loss)
            sweep.append(dict(buckets=nb, max_ctas=cap, side_priority=prio, bwd_gemm_max_ctas=gemm, **r))
            print(json.dumps(sweep[-1]), flush=True)
        optim.STEP_BUCKETS, optim.STEP_MAX_CTAS = base
        model.engine.bwd_gemm_max_ctas = 0
        res["sweep_vqa_adamw"] = sweep
        del model, opt, loss
        torch.cuda.empty_cache()
    for name, make in (("vqa_config2_adamw", lambda: vqa("adamw")), ("pretraining_config3_adamw", pretraining),
                       ("vqa_config2_radam", lambda: vqa("radam"))):
        model, opt, loss = make()
        res[name] = run(model, opt, loss)
        print(json.dumps({name: res[name]}), flush=True)
        del model, opt, loss
        torch.cuda.empty_cache()
    res["card_after"] = card()
    os.makedirs(a.out, exist_ok=True)
    with open(os.path.join(a.out, "step_in_backward_probe.json"), "w") as f:
        json.dump(res, f)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
