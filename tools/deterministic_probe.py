"""Cost of deterministic plans (torch.use_deterministic_algorithms(True), DESIGN.md §4h) on the GPU, and the shared set-up of their
tests (tests/test_deterministic_gpu.py).

    python tools/deterministic_probe.py [--steps 20] [--rounds 5] [--out FILE]

builds the default and the deterministic plan of bench config 2 (bert_base_6layer_6conect, B=64, 100 regions x 36 tokens, train
mode, VQA BCE objective, forward + loss + backward + FusedAdamW step) and of the config-3 fused pre-training step (three losses in
the forward, B=64, 37 regions x 36 tokens, visual_target 0) in one process, and times them alternately: `rounds` rounds of `steps`
CUDA-graph steps per arm, CUDA events around each round. Also times the text-embedding backward alone, default and deterministic
(embed_kernel_times). Prints one JSON line: median ms/step and range per arm, the card's name and power limit read in the same run,
and the workspace bytes each deterministic plan allocated.

    python tools/deterministic_probe.py --hash FILE

runs the config-2 step and two optimizer steps of a deterministic plan from a fixed seed and writes the SHA-256 of the losses, the
gradient buffer and the parameters to FILE (the cross-process check of the tests)."""
import argparse
import hashlib
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

MODEL = "bert_base_6layer_6conect"
INPUT_KEYS = ("input_txt", "input_imgs", "image_loc", "token_type_ids", "attention_mask", "image_attention_mask")


def bench_config():
    import bench
    return bench.load_config_json(MODEL)


def build(kind="vqa", deterministic=True, B=64, Nv=100, Nt=36, precision="fp16", seed=0, **over):
    """-> (engine, plan) of one seeded training step: random weights (bench.py's init), synthetic inputs and objective targets.
    kind "vqa": bench config 2; "pretraining": the fused pre-training objective with its losses in the forward (config 3 shapes
    with Nv=37). `over`: config overrides (visual_target=...)."""
    import torch
    from vilbert_b200.config import BertConfig
    from vilbert_b200.engine import LOSS_HEADS, Engine
    cfgj = dict(bench_config(), **over)
    heads = "pretraining" if kind == "pretraining" else "vl"
    eng = Engine(BertConfig.from_dict(cfgj), torch.device("cuda"), heads=heads, precision=precision)
    g = torch.Generator(device="cuda").manual_seed(seed)
    eng.ps.flat.normal_(0.0, 0.02, generator=g)
    for name in eng.ps.entries:
        if "LayerNorm" in name:
            eng.ps.p(name).fill_(1.0 if name.endswith("weight") else 0.0)
        elif name.endswith(".bias"):
            eng.ps.p(name).zero_()
    eng.refresh_weights()
    extra = dict(loss_in_forward=True) if kind == "pretraining" else {}
    plan = eng.plan(B, Nt, Nv, grad_outputs=LOSS_HEADS[kind], loss=kind, train=True, deterministic=deterministic, **extra)
    load(plan, kind, seed, cfgj)
    return eng, plan


def load(plan, kind, seed, cfgj):
    """Loads seeded synthetic inputs and objective targets into `plan`."""
    import torch
    import bench
    from oracle import vilbert_oracle as O
    inp = O.synth_inputs(O.make_config(cfgj), plan.Bin, plan.Nv, plan.Nt_in, seed=1234 + seed)
    plan.load_inputs(*(inp[k] for k in INPUT_KEYS))
    g = torch.Generator().manual_seed(99 + seed)
    for k, v in bench.synth_loss_inputs(plan, kind, 99 + seed, torch).items():
        dst = plan.vqa_target if k == "vqa_target" else plan.loss_inputs[k]
        if v.numel() != dst.numel():       # a target whose width follows visual_target: softmax rows of the plan's shape
            v = torch.softmax(torch.randn(dst.shape, generator=g), -1)
        dst.copy_(v.reshape(dst.shape))
    torch.cuda.synchronize()


def optimizer(eng, max_grad_norm=1.0):
    import torch
    from vilbert_b200.optim import FusedAdamW
    params = [{"params": [torch.nn.Parameter(eng.ps.p(n))], "weight_decay": 0.0 if "bias" in n or "LayerNorm" in n else 0.01}
              for n in eng.ps.entries]
    return FusedAdamW(params, lr=4e-5, correct_bias=False, engine=eng, max_grad_norm=max_grad_norm)


def results(eng, plan):
    """Device copies of what one step yields: the loss scalar(s), the flat gradient buffer and the input gradients."""
    out = {"grad": eng.ps.grad.clone()}
    for name in ("loss", "objective_out", "score"):
        t = getattr(plan, name, None)
        if t is not None and hasattr(t, "clone"):
            out[name] = t.clone()
    for name, t in plan.input_grad.items():
        out["input_grad." + name] = t.clone()
    return out


def step(eng, plan):
    eng.zero_grad(force=True)
    plan.run_forward()
    plan.run_backward()
    import torch
    torch.cuda.synchronize()
    return results(eng, plan)


def digest(tensors):
    h = hashlib.sha256()
    for k in sorted(tensors):
        h.update(k.encode())
        h.update(tensors[k].detach().contiguous().cpu().numpy().tobytes())
    return h.hexdigest()


def hash_run(n_opt=2):
    """The config-2 step and n_opt optimizer steps of a deterministic plan from seed 0 -> SHA-256 of losses, gradients, parameters."""
    import torch
    eng, plan = build("vqa", deterministic=True)
    r = step(eng, plan)
    plan.enable_optimizer(optimizer(eng))
    for _ in range(n_opt):
        plan.run_step()
    torch.cuda.synchronize()
    r.update(params=eng.ps.flat.clone(), last_loss=plan.loss.clone())
    return digest(r)


def time_arms(arms, steps, rounds):
    """Alternates the arms (name -> (captured plan, its optimizer)) round by round, a step being the plan's graph and the optimizer
    launch after it, as bench.py runs them -> name -> list of ms/step."""
    import torch
    times = {name: [] for name in arms}
    for _ in range(rounds):
        for name, (plan, opt) in arms.items():
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(steps):
                plan.run_step()
                opt.launch()
            e1.record()
            torch.cuda.synchronize()
            times[name].append(e0.elapsed_time(e1) / steps)
    return times


def embed_kernel_times(B=64, Nt=36, H=768, vocab=30522, iters=50):
    """ms per launch of the text-embedding backward, default (scatter atomics) and deterministic (one owning warp per table row), at
    config 2's text shape with every token type 0, as in real batches: the token-type row's warp then sums all B * Nt rows alone."""
    import ctypes as C
    import torch
    from vilbert_b200 import _lib as L
    lib, dev = L.lib(), torch.device("cuda")
    g = torch.Generator(device=dev).manual_seed(0)
    ids = torch.randint(1, vocab, (B, Nt), device=dev, generator=g)
    ids[:, 0], ids[:, -1] = 101, 102
    tt = torch.zeros(B, Nt, dtype=torch.long, device=dev)
    dout = torch.randn(B * Nt, H, device=dev, generator=g)
    tabs = [torch.zeros(n, H, device=dev) for n in (vocab, 512, 2)]
    st = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    out = {}
    for name, fn in (("default", lib.vb_embed_text_bwd), ("deterministic", lib.vb_embed_text_bwd_det)):
        args = (dout.data_ptr(), ids.data_ptr(), tt.data_ptr(), None, *(t.data_ptr() for t in tabs), None, B, Nt, H, st)
        L.check(fn(*args))
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(iters):
            fn(*args)
        e1.record()
        torch.cuda.synchronize()
        out[name + "_ms"] = e0.elapsed_time(e1) / iters
    return out


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True,
                           timeout=30).stdout.strip().splitlines()[0]
        name, power = [s.strip() for s in q.split(",")]
        return name, power
    except Exception as ex:   # noqa: BLE001
        import torch
        return torch.cuda.get_device_name(), f"not read ({ex})"


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--hash", help="write the SHA-256 of a deterministic config-2 run to this file and exit")
    ap.add_argument("--out", help="also write the JSON line to this file")
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit("deterministic_probe: needs a CUDA device (no CPU timing)")
    if a.hash:
        with open(a.hash, "w") as f:
            f.write(hash_run() + "\n")
        return
    res = {}
    for label, kind in (("config2", "vqa"), ("config3_fused", "pretraining")):
        shape = {} if kind == "vqa" else dict(Nv=37)
        arms, ws = {}, {}
        for det in (False, True):
            eng, plan = build(kind, deterministic=det, **shape)
            plan.prologue = [(plan.lib.vb_step_counter_bump, (eng.drop_step.data_ptr(),), 0)]
            opt = optimizer(eng, max_grad_norm=None)
            plan.capture()
            arms["deterministic" if det else "default"] = (plan, opt)
            ws["deterministic" if det else "default"] = plan.det_ws_bytes
        times = time_arms(arms, a.steps, a.rounds)
        res[label] = {name: dict(median_ms=sorted(t)[len(t) // 2], min_ms=min(t), max_ms=max(t)) for name, t in times.items()}
        res[label]["workspace_bytes"] = ws["deterministic"]
        res[label]["cost"] = res[label]["deterministic"]["median_ms"] / res[label]["default"]["median_ms"] - 1.0
        del arms
        torch.cuda.empty_cache()
    res["embed_text_bwd"] = embed_kernel_times()
    name, power = card()
    res.update(gpu=name, power_limit=power, steps=a.steps, rounds=a.rounds)
    line = json.dumps(res)
    print(line)
    if a.out:
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
