"""GPU probe: one optimizer step over base-6-6's parameters with the reference's grouping (one group per tensor, lr 1e-4 for
vil_* heads, no decay on bias / LayerNorm; train_tasks.py:400-420), three ways:

  fused_radam   FusedRAdam.launch(advance_step=True): the step counter bump + one radam_kernel launch
  fused_adamw   FusedAdamW.launch(): one adamw_kernel launch
  fused_adamw_clip        FusedAdamW(max_grad_norm=1.0).launch(): the gradient norm (grad_sq_partials_kernel + the one-CTA
                          finalize) + the clipped adamw_kernel launch
  torch_clip_fused_adamw  torch.nn.utils.clip_grad_norm_(1.0) over the 558 gradient views, then FusedAdamW.launch()
  grad_norm               the gradient norm alone (vb_grad_norm), for its bandwidth at 4 B per parameter (one fp32 read)
  per_tensor    what `--optim RAdam` costs without FusedRAdam: the reference's RAdam algorithm stepping every CUDA tensor
                with torch ops (tests/_radam_oracle.py, fp32), then the 16-bit weight re-cast the model's _sync_weights
                performs before the next train-mode forward

Times come from CUDA events around `--iters` calls after `--warmup` calls; the optimizers alternate for `--rounds` rounds and
the median round is reported. Achieved bandwidth counts the fused kernels' traffic, 36 B per trainable parameter (p, g, m, v
read; p, m, v, fp16 and bf16 copies, zeroed g written), over the time, against the H100 SXM data-sheet 3.35 TB/s. The card
name and power limit are read in the same run. The gradient norm's bandwidth counts 4 B per trainable parameter.
Writes <out>/optim_probe.json.

    python tools/optim_probe.py --out profiles
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

HBM_TBPS = 3.35          # H100 SXM data sheet
BYTES_PER_PARAM = 36
NORM_BYTES_PER_PARAM = 4


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader,nounits", "-i", "0"],
                             capture_output=True, text=True, timeout=60).stdout.strip().split(", ")
        return {"gpu": out[0], "power_limit_w": float(out[1]), "sm_max_mhz": float(out[2])}
    except Exception as e:  # noqa: BLE001 - the measurement stands without it, but say why it is missing
        return {"gpu": None, "power_limit_w": None, "error": str(e)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--config", default=os.path.join(ROOT, "vilbert-multi-task_b200", "configs", "bert_base_6layer_6conect.json"))
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--per-tensor-iters", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles"), help="directory for optim_probe.json (profiles/ is kept out of git)")
    a = ap.parse_args()

    import torch
    if not torch.cuda.is_available():
        raise SystemExit("optim_probe needs a CUDA device")
    from vilbert_b200.config import BertConfig
    from vilbert_b200.engine import Engine
    from vilbert_b200.optim import FusedAdamW, FusedRAdam
    from oracle.adamw_oracle import reference_param_groups
    import _radam_oracle as RO

    eng = Engine(BertConfig.from_dict(json.load(open(a.config))), "cuda")
    g = torch.Generator(device="cuda").manual_seed(0)
    eng.ps.flat.normal_(0.0, 0.02, generator=g)
    eng.refresh_weights()
    named = [(name, torch.nn.Parameter(eng.ps.p(name))) for name in eng.ps.entries]
    n_params = sum(p.numel() for _, p in named)
    radam = FusedRAdam(reference_param_groups(named, base_lr=4e-5), lr=4e-5, engine=eng)
    adamw = FusedAdamW(reference_param_groups(named, base_lr=4e-5), lr=4e-5, correct_bias=False, engine=eng)
    adamw_clip = FusedAdamW(reference_param_groups(named, base_lr=4e-5), lr=4e-5, correct_bias=False, engine=eng, max_grad_norm=1.0)
    radam._step_dev.fill_(10)     # past the unrectified steps: the timed launches take the sqrt / divide path
    for name, p in named:
        p.grad = eng.ps.g(name)
    per_tensor = RO.RAdamOracle(reference_param_groups(named, base_lr=4e-5), lr=4e-5)
    grad_fill = lambda: eng.ps.grad.normal_(0.0, 1e-2, generator=g)   # noqa: E731

    def per_tensor_step():
        with torch.no_grad():
            per_tensor.step()
        eng.refresh_weights()

    def torch_clip_step():
        torch.nn.utils.clip_grad_norm_(views, 1.0)
        adamw.launch()

    views = [p for _, p in named]
    norm_fn, norm_args = adamw_clip.ops()[0]
    legs = {"fused_radam": (lambda: radam.launch(advance_step=True), a.iters),
            "fused_adamw": (adamw.launch, a.iters),
            "per_tensor": (per_tensor_step, a.per_tensor_iters),
            "fused_adamw_clip": (adamw_clip.launch, a.iters),
            "torch_clip_fused_adamw": (torch_clip_step, a.iters),
            "grad_norm": (lambda: adamw_clip._run([(norm_fn, norm_args)], None), a.iters)}
    grad_fill()
    for fn, _ in legs.values():
        for _ in range(a.warmup):
            fn()
    torch.cuda.synchronize()
    times = {k: [] for k in legs}
    for _ in range(a.rounds):
        for k, (fn, n) in legs.items():
            grad_fill()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(n):
                fn()
            e1.record()
            torch.cuda.synchronize()
            times[k].append(e0.elapsed_time(e1) / n)
    res = {"what": "one optimizer step over every parameter of bert_base_6layer_6conect, reference grouping (one group per tensor)",
           "n_params": n_params, "n_tensors": len(named), "bytes_per_param": BYTES_PER_PARAM, "hbm_datasheet_tbps": HBM_TBPS,
           "card": card(), "iters": a.iters, "per_tensor_iters": a.per_tensor_iters, "rounds": a.rounds, "legs": {}}
    for k, ts in times.items():
        ms = statistics.median(ts)
        nbytes = NORM_BYTES_PER_PARAM if k == "grad_norm" else BYTES_PER_PARAM
        gbs = nbytes * n_params / (ms * 1e-3) / 1e9
        res["legs"][k] = {"ms_per_step": ms, "ms_rounds": ts, f"gb_per_s_at_{nbytes}B_per_param": gbs,
                          "fraction_of_datasheet_hbm": gbs / (HBM_TBPS * 1e3)}
    res["per_tensor_over_fused_radam"] = res["legs"]["per_tensor"]["ms_per_step"] / res["legs"]["fused_radam"]["ms_per_step"]
    res["fused_radam_over_fused_adamw"] = res["legs"]["fused_radam"]["ms_per_step"] / res["legs"]["fused_adamw"]["ms_per_step"]
    res["clip_cost_ms"] = res["legs"]["fused_adamw_clip"]["ms_per_step"] - res["legs"]["fused_adamw"]["ms_per_step"]
    res["torch_clip_cost_ms"] = res["legs"]["torch_clip_fused_adamw"]["ms_per_step"] - res["legs"]["fused_adamw"]["ms_per_step"]
    res["skipped_steps_clip"] = int(adamw_clip.skipped_steps.item())      # 0: the timed clipped steps did their full work
    os.makedirs(a.out, exist_ok=True)
    with open(os.path.join(a.out, "optim_probe.json"), "w") as f:
        json.dump(res, f, indent=1)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
