"""Per-CTA clock64 timeline of one GEMM launch (development tool)."""
import ctypes as C, os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from vilbert_b200 import _lib as L
lib = L.lib(); dev = "cuda"; BF = torch.bfloat16
def run(M, N, K, bn, res=False, a_mn=False, b_mn=False, atomic=False, split_k=1, bf16=False):
    A = (torch.randn(K, M, device=dev) if a_mn else torch.randn(M, K, device=dev)).to(BF)
    B = (torch.randn(K, N, device=dev) if b_mn else torch.randn(N, K, device=dev)).to(BF)
    o16 = torch.empty(M, N, device=dev, dtype=BF)
    out = torch.empty(M, N, device=dev); r = torch.randn(M, N, device=dev)
    nsm = torch.cuda.get_device_properties(0).multi_processor_count
    dbg = torch.zeros(nsm * 10, dtype=torch.int64, device=dev)
    g = L.GemmArgs(); g.M, g.N, g.K = M, N, K
    g.A, g.lda, g.a_mn_major, g.B, g.ldb, g.b_mn_major = A.data_ptr(), (M if a_mn else K), int(a_mn), B.data_ptr(), (N if b_mn else K), int(b_mn)
    g.alpha, g.split_k, g.block_n, g.atomic_out = 1.0, split_k, bn, int(atomic)
    if bf16: g.out_bf16, g.ld_out_bf16 = o16.data_ptr(), N
    else: g.out_f32, g.ld_out_f32 = out.data_ptr(), N
    if res: g.residual, g.ld_res = r.data_ptr(), N
    st = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    for _ in range(3): L.check(lib.vb_gemm_bf16(C.byref(g), st))
    torch.cuda.synchronize()
    g.dbg_timeline = dbg.data_ptr()
    e0, e1 = torch.cuda.Event(True), torch.cuda.Event(True)
    e0.record(); L.check(lib.vb_gemm_bf16(C.byref(g), st)); e1.record(); torch.cuda.synchronize()
    full = dbg.view(nsm, 10).cpu()
    live = full[:, 0] != 0
    full = full[live]
    t = full[:, :8]
    ns0, ns1 = full[:, 8], full[:, 9]
    d = (t - t[:, :1]).float()
    names = ["entry", "setup done", "first TMA issued", "first full_bar", "(not recorded)", "tile 0: k-loop retired", "tile 0: epilogue done", "exit sync"]
    print(f"--- M{M} N{N} K{K} bn{bn} res{int(res)} a_mn{int(a_mn)} b_mn{int(b_mn)} atomic{int(atomic)} split{split_k} bf16out{int(bf16)}: event time {e0.elapsed_time(e1)*1e3:.1f} us, {int(live.sum())} CTAs; cycles since CTA entry (median / max over CTAs):")
    for i, n in enumerate(names):
        print(f"     {n:20s} {d[:, i].median().item():10.0f} {d[:, i].max().item():10.0f}")
    print(f"     globaltimer: CTA start spread {(ns0.max() - ns0.min()).item()} ns, first start -> last end {(ns1.max() - ns0.min()).item()} ns, "
          f"median CTA lifetime {(ns1 - ns0).median().item()} ns")
run(2304, 768, 768, 128, res=True)
run(6400, 1024, 1024, 128, res=True)
run(6400, 1024, 1024, 128, bf16=True)
run(6400, 1024, 3072, 128, res=True, b_mn=True)
run(6400, 1024, 3072, 128, res=True)
run(6400, 1024, 3072, 128, bf16=True, b_mn=True)
run(6400, 1024, 3072, 256, res=True, b_mn=True)
run(3072, 1024, 6400, 128, a_mn=True, b_mn=True, atomic=True)
run(3072, 1024, 6400, 256, a_mn=True, b_mn=True, atomic=True)
run(3072, 1024, 6400, 256, a_mn=True, b_mn=True, atomic=True, split_k=3)
run(3072, 1024, 6400, 256, a_mn=True, b_mn=True, bf16=True)
run(1024, 1024, 6400, 256, a_mn=True, b_mn=True, atomic=True, split_k=4)
run(6400, 3072, 1024, 256, bf16=True)
