"""Train-mode forward + backward of the single-stream baseline (BaseBertForVLTasks) against the two-stream VILBertForVLTasks on
bert_base_6layer_6conect at bench config 2's shape (B=64, 100 regions, 36 tokens: a 136-row stream for the baseline), on the same
card in the same process. Prints one JSON line: ms/step, (region, token) pairs/s, and the share of the step spent in the attention
backward (its launches replayed alone), with the card name and power limit.

    python tools/baseline_probe.py [--steps 20] [--warmup 5] [--out FILE]
"""
import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card():
    name = torch.cuda.get_device_name(0)
    try:
        pl = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True,
                            timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        pl = "unknown"
    return name, pl


def timed(fn, steps):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(steps):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / steps


def measure(eng, B, Nt, Nv, names, steps, warmup):
    from vilbert_b200.engine import BASE_FEATURE_SIZE
    g = torch.Generator(device="cuda").manual_seed(0)
    Fv = BASE_FEATURE_SIZE if eng.ps.base else eng.cfg.v_feature_size
    inp = dict(input_txt=torch.randint(1, eng.cfg.vocab_size, (B, Nt), device="cuda", generator=g),
               input_imgs=torch.randn(B, Nv, Fv, device="cuda", generator=g), image_loc=torch.rand(B, Nv, 5, device="cuda", generator=g),
               token_type_ids=torch.zeros(B, Nt, dtype=torch.int64, device="cuda"),
               attention_mask=torch.ones(B, Nt, dtype=torch.int64, device="cuda"),
               image_attention_mask=torch.ones(B, Nv, dtype=torch.int64, device="cuda"))
    eng.refresh_weights()
    plan = eng.plan(B, Nt, Nv, grad_outputs=names, train=True)
    plan.load_inputs(**inp)
    for n in names:
        plan.gout[n].copy_(torch.randn(plan.gout[n].shape, device="cuda", generator=g) * 1e-3)
    plan.capture(separate=True)

    def step():
        plan.run_forward()
        plan.run_backward()
    timed(step, warmup)
    ms = timed(step, steps)
    attn = [op for op in plan.bwd if op[0] is not None and op[0].__name__ == "vb_attention_bwd"]
    stream = torch.cuda.current_stream().cuda_stream
    ms_attn = timed(lambda: [op[0](*op[1], stream) for op in attn], steps)
    return dict(ms_per_step=round(ms, 3), pairs_per_s=round(B * Nv * Nt / (ms * 1e-3), 1), attn_bwd_ms=round(ms_attn, 3),
                attn_bwd_share=round(ms_attn / ms, 3), kernels_fwd=plan.n_kernels_fwd, kernels_bwd=plan.n_kernels_bwd)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("baseline_probe: needs a CUDA device (there is no CPU measurement)")
    from vilbert_b200.config import BertConfig
    from vilbert_b200.engine import BASE_HEAD_NAMES, HEAD_NAMES, Engine
    cfgj = json.load(open(os.path.join(ROOT, "vilbert-multi-task_b200", "configs", "bert_base_6layer_6conect.json")))
    B, Nv, Nt = 64, 100, 36
    res = dict(config="bert_base_6layer_6conect", B=B, Nv=Nv, Nt=Nt, stream_rows=Nv + Nt)
    base = Engine(BertConfig.from_dict(cfgj), "cuda", heads="base", num_labels=3129)
    res["basebert"] = measure(base, B, Nt, Nv, BASE_HEAD_NAMES, a.steps, a.warmup)
    del base
    torch.cuda.empty_cache()
    vil = Engine(BertConfig.from_dict(cfgj), "cuda")
    res["vilbert"] = measure(vil, B, Nt, Nv, HEAD_NAMES, a.steps, a.warmup)
    res["card"], res["power_limit"] = card()
    line = json.dumps(res)
    print(line)
    if a.out:
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
