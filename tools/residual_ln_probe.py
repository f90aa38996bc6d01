"""Where the residual add of the residual stream costs time: kernel times of the fp32-output GEMMs of config 2 with and without
the fp32 residual (and with and without the fused dropout), and of the LayerNorm that follows them, plain (vb_layernorm_fwd) and
with the residual add and dropout fused into it (vb_add_layernorm_fwd, when the library has it). CUDA events over many queued
launches. Development tool: python tools/residual_ln_probe.py [--out FILE.json]"""
import argparse, ctypes as C, json, os, subprocess, sys, time
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from vilbert_b200 import _lib as L

BF, F16 = torch.bfloat16, torch.float16
ITERS = 200


def stream():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def timed(fn, iters=ITERS):
    for _ in range(5):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(True), torch.cuda.Event(True)
    torch.cuda._sleep(int(4e6))          # launches below are queued behind this: kernel time, not launch rate
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters * 1e3   # us


def gemm_us(M, N, K, dgrad, res, drop, step):
    """EPI_F32 GEMM out[M, N] = A[M, K] B^T (+ bias) (dropout) (+ residual): the forward dense of LN(dropout(dense(a)) + r)
    (fp16 operands, bias) or the dgrad into the residual-path gradient (bf16 operands, B stored n-major, no bias)."""
    dev = torch.device("cuda")
    dt = BF if dgrad else F16
    A = (torch.randn(M, K, device=dev) * 0.5).to(dt)
    B = (torch.randn(K, N, device=dev) * 0.5).to(dt) if dgrad else (torch.randn(N, K, device=dev) * 0.5).to(dt)
    bias = None if dgrad else torch.randn(N, device=dev)
    r = torch.randn(M, N, device=dev)
    out = torch.empty(M, N, device=dev)
    g = L.GemmArgs()
    g.M, g.N, g.K = M, N, K
    g.A, g.lda = A.data_ptr(), K
    g.B, g.ldb, g.b_mn_major = B.data_ptr(), (N if dgrad else K), int(dgrad)
    g.alpha = 1.0
    g.bias = bias.data_ptr() if bias is not None else None
    g.residual, g.ld_res = (r.data_ptr(), N) if res else (None, 0)
    g.out_f32, g.ld_out_f32 = out.data_ptr(), N
    g.a_fp16 = g.b_fp16 = g.out_fp16 = int(not dgrad)
    if drop:
        g.dropout.step, g.dropout.site, g.dropout.p = step.data_ptr(), 7, 0.1
    lib = L.lib()
    return timed(lambda: L.check(lib.vb_gemm_bf16(C.byref(g), stream()), "vb_gemm_bf16"))


def ln_us(M, H, add, drop, step):
    """LayerNorm of the residual stream as the engine runs it (fp32 + fp16 operand + bf16 backward copy outputs); add: the residual
    add (and dropout) fused into it, the sum written back over the dense output for the backward."""
    dev = torch.device("cuda")
    d, r = torch.randn(M, H, device=dev), torch.randn(M, H, device=dev)
    gm, bt = torch.randn(H, device=dev), torch.randn(H, device=dev)
    y32 = torch.empty(M, H, device=dev)
    y16, yb = torch.empty(M, H, device=dev, dtype=F16), torch.empty(M, H, device=dev, dtype=BF)
    mean, rstd = torch.empty(M, device=dev), torch.empty(M, device=dev)
    dp = None
    if drop:
        dp = L.Dropout(); dp.step, dp.site, dp.p = step.data_ptr(), 7, 0.1
    lib = L.lib()
    if add:
        fn = lambda: L.check(lib.vb_add_layernorm_fwd(d.data_ptr(), r.data_ptr(), H, C.byref(dp) if dp else None, d.data_ptr(), gm.data_ptr(),
                                                      bt.data_ptr(), 1e-12, y32.data_ptr(), y16.data_ptr(), H, mean.data_ptr(), rstd.data_ptr(),
                                                      M, H, 1, None, yb.data_ptr(), stream()), "vb_add_layernorm_fwd")
    else:
        fn = lambda: L.check(lib.vb_layernorm_fwd(d.data_ptr(), H, gm.data_ptr(), bt.data_ptr(), 1e-12, y32.data_ptr(), y16.data_ptr(), H,
                                                  mean.data_ptr(), rstd.data_ptr(), M, H, None, 1, None, yb.data_ptr(), stream()), "vb_layernorm_fwd")
    return timed(fn)


def ln_bwd_us(M, H, extra):
    """LayerNorm backward of the residual stream (dx fp32 + bf16, dgamma / dbeta / dbias); extra: a second fp32 gradient input."""
    dev = torch.device("cuda")
    dy, e, x = torch.randn(M, H, device=dev), torch.randn(M, H, device=dev), torch.randn(M, H, device=dev)
    gm = torch.randn(H, device=dev)
    mean, rstd = torch.zeros(M, device=dev), torch.ones(M, device=dev)
    dx32, dx16 = torch.empty(M, H, device=dev), torch.empty(M, H, device=dev, dtype=BF)
    dg, db, dbias = torch.zeros(H, device=dev), torch.zeros(H, device=dev), torch.zeros(H, device=dev)
    lib = L.lib()
    if extra:
        fn = lambda: L.check(lib.vb_add_layernorm_bwd(dy.data_ptr(), e.data_ptr(), H, x.data_ptr(), H, gm.data_ptr(), mean.data_ptr(), rstd.data_ptr(),
                                                      dx32.data_ptr(), dx16.data_ptr(), H, None, 0, dg.data_ptr(), db.data_ptr(), dbias.data_ptr(),
                                                      M, H, None, None, stream()), "vb_add_layernorm_bwd")
    else:
        fn = lambda: L.check(lib.vb_layernorm_bwd(dy.data_ptr(), H, x.data_ptr(), H, gm.data_ptr(), mean.data_ptr(), rstd.data_ptr(),
                                                  dx32.data_ptr(), dx16.data_ptr(), H, None, 0, dg.data_ptr(), db.data_ptr(), dbias.data_ptr(),
                                                  M, H, None, None, stream()), "vb_layernorm_bwd")
    return timed(fn)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    torch.cuda.set_device(0)
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    print(f"=== residual / LayerNorm probe  {smi}  {time.ctime()}", flush=True)
    step = torch.ones(1, dtype=torch.int32, device="cuda")
    rows = []
    # config 2 (bert_base_6layer_6conect, batch 64): text 36 x 64 = 2304 rows of 768, image 100 x 64 = 6400 rows of 1024
    fwd = [(2304, 768, 768, "text out-proj"), (2304, 768, 3072, "text FFN2"), (2304, 768, 1024, "conn biOutput text"),
           (6400, 1024, 1024, "image out-proj / FFN2 / biOutput")]
    dgr = [(2304, 768, 2304, "text QKV dgrad"), (2304, 768, 3072, "text FFN1 dgrad"), (6400, 1024, 3072, "image QKV dgrad"),
           (6400, 1024, 1024, "image FFN1 dgrad")]
    for dgrad, shapes in ((False, fwd), (True, dgr)):
        for (M, N, K, name) in shapes:
            r = dict(kind="dgrad" if dgrad else "fwd", name=name, M=M, N=N, K=K)
            for res in (True, False):
                for drop in ((False,) if dgrad else (True, False)):
                    r[f"res{int(res)}_drop{int(drop)}_us"] = gemm_us(M, N, K, dgrad, res, drop, step)
            rows.append(r)
            print(json.dumps(r), flush=True)
    have_add = hasattr(L.lib(), "vb_add_layernorm_fwd")
    for (M, H) in ((2304, 768), (6400, 1024)):
        r = dict(kind="ln", M=M, H=H, ln_fwd_us=ln_us(M, H, False, False, step), ln_bwd_us=ln_bwd_us(M, H, False))
        if have_add:
            r.update(add_ln_fwd_us=ln_us(M, H, True, False, step), add_ln_fwd_drop_us=ln_us(M, H, True, True, step),
                     add_ln_bwd_us=ln_bwd_us(M, H, True))
        rows.append(r)
        print(json.dumps(r), flush=True)
    if a.out:
        with open(a.out, "w") as f:
            json.dump(dict(device=smi, rows=rows), f, indent=1)


if __name__ == "__main__":
    main()
