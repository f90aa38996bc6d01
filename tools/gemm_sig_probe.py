"""Per-signature GEMM probe: every distinct vb_gemm_bf16 launch of a bench.py training step, timed on its own.

    python tools/gemm_sig_probe.py [--configs 2 3] [--iters 200] [--out DIR]     # on an H100 (DIR: also write JSON)
    python tools/gemm_sig_probe.py --list [--configs 2 3]                         # signatures only, no GPU needed

The step's plan is built on the CPU (Engine(..., "cpu", _build_only=True), tiles resolved for 132 SMs) and its GEMM launches
are grouped by signature: shape, operand majors and formats, epilogue (act, bias, residual, aux, dropout, column sums, outputs),
atomic / split-K / partials form and leading dimensions. Each signature then runs on fresh, device-resident random operands with
those exact flags (pointer alignment modulo 256 bytes included): >= `iters` queued launches between CUDA events give the time
per launch, and one launch with the kernel's per-CTA clock64 timeline gives the median cycles to the first full stage, the
k-loop cycles per 64-deep k-block and the epilogue cycles of the first tile. The floor of a launch is max(FLOP / 989 TFLOP/s,
bytes / 3.35 TB/s), the H100 SXM data-sheet rates (dense BF16 / FP16, HBM3); bytes count each operand and output once (atomic
outputs twice). The card's name, power limit and SM clock are read in the same run and stored with the numbers.
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402
from vilbert_b200 import _lib as L  # noqa: E402

PEAK_TFLOPS, PEAK_TBS = 989.0, 3.35
PTR_FIELDS = ("A", "B", "bias", "residual", "aux", "out_f32", "out_bf16", "out_pre", "out_colsum", "A_lo", "B_lo", "out_lo", "out_b16")
SCALAR_FIELDS = ("M", "N", "K", "lda", "a_mn_major", "ldb", "b_mn_major", "alpha", "ld_res", "ld_aux", "act", "ld_out_f32", "ld_out_bf16",
                 "ld_out_pre", "atomic_out", "split_k", "block_n", "max_ctas", "a_fp16", "b_fp16", "out_fp16")


def signature(g):
    """Hashable description of one launch: its scalar arguments, which pointers are set (and their alignment mod 256), dropout."""
    ptrs = tuple((f, (getattr(g, f) or 0) % 256) for f in PTR_FIELDS if getattr(g, f))
    drop = (g.dropout.site, round(g.dropout.p, 6)) if (g.dropout.step and g.dropout.p > 0) else None
    return tuple(getattr(g, f) for f in SCALAR_FIELDS) + (ptrs, drop)


def describe(sig):
    s = dict(zip(SCALAR_FIELDS, sig[:len(SCALAR_FIELDS)]))
    ptrs = dict(sig[len(SCALAR_FIELDS)])
    s["set"] = sorted(ptrs)
    s["dropout"] = sig[-1]
    return s


def short(s):
    out = [f for f in ("out_f32", "out_bf16", "out_pre", "out_lo", "out_b16", "out_colsum") if f in s["set"]]
    ep = {0: "", 1: "gelu", 2: "relu", 3: "dgelu"}[s["act"]]
    tag = "+".join(x for x in ([ep] if ep else []) + (["bias"] if "bias" in s["set"] else []) + (["res"] if "residual" in s["set"] else [])
                   + (["drop"] if s["dropout"] else []) + ([{1: "atomic", L.VB_GEMM_PARTIALS: "partials"}.get(s["atomic_out"], "")] if s["atomic_out"] else []))
    return (f"{s['M']}x{s['N']}x{s['K']} {'A^T' if s['a_mn_major'] else 'A'}{'B^T' if s['b_mn_major'] else 'B'} "
            f"{'f16' if s['a_fp16'] else 'bf16'}{'x3' if 'A_lo' in s['set'] else ''} {tag or 'plain'} -> {','.join(o[4:] for o in out)}")


def plan_gemm_signatures(config, kind="train", sm_count=132):
    """{signature: launches per step} of bench.py config `config`'s plans, in first-launch order. kind: "train" (the training step,
    forward + backward), "eval" (the forward-only evaluation plan), "capped" (the training step with the backward GEMMs capped at
    sm_count - 16 persistent CTAs, as data-parallel runs leave SMs to NCCL) or "det" (the deterministic training step)."""
    import bench
    from vilbert_b200.config import BertConfig
    from vilbert_b200.engine import Engine, LOSS_HEADS
    cf = bench.CONFIGS[config]
    cfgj = bench.load_config_json(cf["model"])
    if cf["task_tokens"]:
        cfgj = dict(cfgj, task_specific_tokens=True)
    eng = Engine(BertConfig.from_dict(cfgj), "cpu", heads=cf.get("heads", "vl"), _build_only=True)
    if kind == "capped":
        eng.bwd_gemm_max_ctas = sm_count - 16
    sigs = {}
    for (_name, gb, Nv, Nt, loss) in cf["tasks"]:
        B = gb if cf["per_gpu"] else gb // 8
        if kind == "eval":
            plan = eng.plan(B, Nt, Nv)
        else:
            plan = eng.plan(B, Nt, Nv, grad_outputs=LOSS_HEADS[loss], loss=loss, train=True, deterministic=(kind == "det"))
        for fn, args, _sid in plan.prologue + plan.fwd + plan.bwd:
            if fn is None or fn.__name__ != "vb_gemm_bf16":
                continue
            g = args[0]._obj
            k = signature(g)
            sigs[k] = sigs.get(k, 0) + 1
    return sigs


def plan_signature_union(kinds=None):
    """One signature per GEMM form the engine's plans launch: the union over `kinds` ((config, kind) pairs; default: every bench
    config's training step and config 2's evaluation, capped-backward and deterministic plans) with the row count M left out of
    the key and base addresses taken modulo 16 (the epilogue's vector-access conditions), each form represented by its launch of
    the fewest rows. {signature: [(config, kind), ...] it comes from}."""
    if kinds is None:
        import bench
        kinds = [(c, "train") for c in sorted(bench.CONFIGS)] + [(2, "eval"), (2, "capped"), (2, "det")]
    forms = {}
    for c, kind in kinds:
        for k in plan_gemm_signatures(c, kind):
            s = dict(zip(SCALAR_FIELDS, k[:len(SCALAR_FIELDS)]))
            s.pop("M")
            if s["a_mn_major"]:
                s.pop("lda")      # MN-major A: its pitch is M rounded up
            key = (tuple(s.items()), tuple((f, o % 16) for f, o in k[len(SCALAR_FIELDS)]), k[-1])
            rep, src = forms.get(key, (None, []))
            if rep is None or k[0] < rep[0]:
                rep = k
            forms[key] = (rep, src + [(c, kind)] if (c, kind) not in src else src)
    return {rep: src for rep, src in forms.values()}


def resolved_tiles(s):
    g = L.GemmArgs()
    for f in SCALAR_FIELDS:
        setattr(g, f, s[f])
    for f in s["set"]:
        setattr(g, f, 256)   # non-null placeholder: vb_gemm_plan reads only which pointers are set
    bn, sp = C.c_int32(), C.c_int32()
    L.check(L.lib().vb_gemm_plan(C.byref(g), 132, C.byref(bn), C.byref(sp)), "vb_gemm_plan")
    return bn.value, sp.value


class Launch:
    """One signature on fresh device buffers: random 16-bit operands, random fp32 bias / residual, bf16 aux."""

    def __init__(self, sig, seed=0):
        s = describe(sig)
        self.s = s
        offs = dict(sig[len(SCALAR_FIELDS)])
        M, N, K = s["M"], s["N"], s["K"]
        dev = torch.device("cuda")
        gen = torch.Generator(device=dev).manual_seed(seed)
        f16 = lambda fmt: torch.float16 if fmt else torch.bfloat16
        _, sp = resolved_tiles(s)
        rows = {"A": K if s["a_mn_major"] else M, "B": K if s["b_mn_major"] else N, "bias": 1, "residual": M, "aux": M,
                "out_f32": M * (sp if s["atomic_out"] == L.VB_GEMM_PARTIALS else 1), "out_bf16": M, "out_pre": M, "out_colsum": 1,
                "A_lo": K if s["a_mn_major"] else M, "B_lo": K if s["b_mn_major"] else N, "out_lo": M, "out_b16": M}
        cols = {"A": s["lda"], "B": s["ldb"], "bias": N, "residual": s["ld_res"], "aux": s["ld_aux"], "out_f32": s["ld_out_f32"],
                "out_bf16": s["ld_out_bf16"], "out_pre": s["ld_out_pre"], "out_colsum": N, "A_lo": s["lda"], "B_lo": s["ldb"],
                "out_lo": s["ld_out_bf16"], "out_b16": s["ld_out_bf16"]}
        dtype = {"A": f16(s["a_fp16"]), "B": f16(s["b_fp16"]), "A_lo": f16(s["a_fp16"]), "B_lo": f16(s["b_fp16"]), "aux": torch.bfloat16,
                 "out_bf16": f16(s["out_fp16"]), "out_lo": f16(s["out_fp16"]), "out_pre": torch.bfloat16, "out_b16": torch.bfloat16}
        self.g = g = L.GemmArgs()
        for f in SCALAR_FIELDS:
            setattr(g, f, s[f])
        self.bufs, self.views = {}, {}
        for f in s["set"]:
            dt = dtype.get(f, torch.float32)
            n = rows[f] * cols[f]
            el = torch.empty((), dtype=dt).element_size()
            raw = torch.empty(n + 512 // el, device=dev, dtype=dt)
            o = ((offs[f] - raw.data_ptr()) % 256) // el          # same address modulo 256 as in the plan
            v = raw[o:o + n]
            if f in ("A", "B", "A_lo", "B_lo", "aux", "bias", "residual"):
                v.copy_((torch.randn(n, device=dev, generator=gen) * (0.01 if f.endswith("_lo") else 0.5)).to(dt))
            else:
                v.zero_()
            self.bufs[f] = raw
            self.views[f] = v.view(rows[f], cols[f])
            setattr(g, f, v.data_ptr())
        if s["dropout"]:
            self.ctr = torch.ones(1, device=dev, dtype=torch.int32)
            g.dropout.step, g.dropout.site, g.dropout.p = self.ctr.data_ptr(), s["dropout"][0], s["dropout"][1]

    def __call__(self, stream):
        L.check(L.lib().vb_gemm_bf16(C.byref(self.g), stream), "vb_gemm_bf16")

    def flops(self):
        s = self.s
        return 2.0 * s["M"] * s["N"] * s["K"] * (1 + ("A_lo" in s["set"]) + ("B_lo" in s["set"]))

    def bytes(self):
        s = self.s
        M, N, K = s["M"], s["N"], s["K"]
        b = (M + N) * K * 2 * (1 + ("A_lo" in s["set"]))
        per = {"bias": 0, "residual": 4 * M * N, "aux": 2 * M * N, "out_bf16": 2 * M * N, "out_pre": 2 * M * N, "out_lo": 2 * M * N,
               "out_b16": 2 * M * N, "out_colsum": 0, "out_f32": 4 * M * N * (2 if s["atomic_out"] == 1 else 1)}
        return b + sum(per.get(f, 0) for f in s["set"] if f not in ("A", "B", "A_lo", "B_lo"))


def gpu_info():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader,nounits", "-i", "0"],
                           capture_output=True, text=True, timeout=30).stdout.strip().split(",")
        return dict(gpu=q[0].strip(), power_limit_w=float(q[1]), sm_mhz=int(q[2]), sm_max_mhz=int(q[3]))
    except Exception as e:   # noqa: BLE001
        return dict(gpu=torch.cuda.get_device_name(0), error=repr(e)[:200])


def probe(sig, iters, stream):
    ln = Launch(sig)
    for _ in range(3):
        ln(stream)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(True), torch.cuda.Event(True)
    torch.cuda._sleep(int(20e6))     # launches queued behind a busy GPU: the events bracket kernel time, not launch rate
    e0.record()
    for _ in range(iters):
        ln(stream)
    e1.record()
    torch.cuda.synchronize()
    us = e0.elapsed_time(e1) * 1e3 / iters
    # one timeline launch: [grid][10] = 8 x clock64 (slots 0 entry, 1 set-up, 2 first TMA, 3 first full stage, 5 first tile's
    # k-loop retired, 6 its epilogue done, 7 exit) + 2 x globaltimer
    nsm = torch.cuda.get_device_properties(0).multi_processor_count
    dbg = torch.zeros(2 * nsm * 10, dtype=torch.int64, device="cuda")
    ln.g.dbg_timeline = dbg.data_ptr()
    ln(stream)
    torch.cuda.synchronize()
    ln.g.dbg_timeline = None
    t = dbg.view(-1, 10).cpu()
    t = t[t[:, 0] != 0][:, :8].double()
    bn, sp = resolved_tiles(ln.s)
    s = ln.s
    kbs = -(-s["K"] // 64) * (1 + ("A_lo" in s["set"]) + ("B_lo" in s["set"]))
    kps = -(-kbs // sp)
    med = lambda x: float(x.median()) if len(x) else float("nan")
    fl, by = ln.flops(), ln.bytes()
    return dict(sig=short(s), args=s, block_n=bn, split_k=sp, us=us, tflops=fl / us / 1e6,
                floor_us=max(fl / PEAK_TFLOPS / 1e6, by / PEAK_TBS / 1e6), bytes=by, flops=fl,
                cyc_first_full=med(t[:, 3] - t[:, 0]), cyc_per_kblock=med((t[:, 5] - t[:, 3]) / kps), cyc_epilogue=med(t[:, 6] - t[:, 5]))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--configs", type=int, nargs="+", default=[2, 3])
    ap.add_argument("--iters", type=int, default=200)
    ap.add_argument("--out", default=None, help="also write the results as gemm_sig_probe.json under this directory")
    ap.add_argument("--list", action="store_true", help="print the signatures and their launches per step, no GPU")
    a = ap.parse_args()
    result = {}
    if not a.list:
        torch.cuda.set_device(0)
        result["device"] = gpu_info()
        print(json.dumps(result["device"]), flush=True)
        stream = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    for cfg in a.configs:
        sigs = plan_gemm_signatures(cfg)
        n, fl = sum(sigs.values()), sum(2.0 * describe(k)["M"] * describe(k)["N"] * describe(k)["K"] * c for k, c in sigs.items())
        print(f"=== config {cfg}: {len(sigs)} signatures, {n} launches, {fl / 1e12:.2f} TFLOP per step", flush=True)
        rows = []
        for k, cnt in sigs.items():
            s = describe(k)
            if a.list:
                bn, sp = resolved_tiles(s)
                print(f"  {short(s):64s} x{cnt:3d}  bn{bn} sk{sp}")
                continue
            r = probe(k, a.iters, stream)
            r["per_step"] = cnt
            r["us_per_step"] = cnt * r["us"]
            rows.append(r)
        if a.list:
            continue
        rows.sort(key=lambda r: -r["us_per_step"])
        print(f"  {'signature':64s} {'bn/sk':>7s} {'n':>3s} {'us':>8s} {'TFLOP/s':>8s} {'floor':>7s} {'us/step':>8s} "
              f"{'cyc->full':>9s} {'cyc/kblk':>8s} {'cyc epi':>8s}")
        for r in rows:
            print(f"  {r['sig']:64s} {r['block_n']:4d}/{r['split_k']:<2d} {r['per_step']:3d} {r['us']:8.1f} {r['tflops']:8.1f} "
                  f"{r['floor_us']:7.1f} {r['us_per_step']:8.1f} {r['cyc_first_full']:9.0f} {r['cyc_per_kblock']:8.0f} {r['cyc_epilogue']:8.0f}")
        tot = sum(r["us_per_step"] for r in rows)
        print(f"  total {tot / 1e3:.3f} ms of GEMM per step (serial), floor {sum(r['floor_us'] * r['per_step'] for r in rows) / 1e3:.3f} ms", flush=True)
        result[f"config{cfg}"] = rows
    if not a.list:
        result["device_after"] = gpu_info()
        print(json.dumps(result["device_after"]), flush=True)
    if not a.list and a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "gemm_sig_probe.json"), "w") as f:
            json.dump(result, f, indent=1)


if __name__ == "__main__":
    main()
