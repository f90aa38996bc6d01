"""Launches ONE instance of each representative kernel of the default (fp16 forward / bf16 gradient operand) step, for
`ncu --set full` (keep the report small). Writes the launch order of the GEMM signatures to profiles/ncu_targets_order.json so
that tools/ncu_summary.py can attribute the captured DRAM bytes. Development tool."""
import ctypes as C, json, os, sys
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "tests"))
import torch
from vilbert_b200 import _lib as L
from _gpu_util import gemm_case, attn_case
F = dict(a_fp16=True, b_fp16=True)
order = []
def gemm(M, N, K, tag, **kw):
    # signature key of bench.py's roofline: (M, N, K, a_mn, b_mn, act, residual, atomic)
    order.append(dict(sig=[M, N, K, int(kw.get("a_mn", False)), int(kw.get("b_mn", False)), int(kw.get("act", 0)), int(kw.get("res", False)), int(kw.get("atomic", False))], tag=tag))
    gemm_case(M, N, K, check=False, **kw)
gemm(6400, 1024, 1024, "out-proj / FFN2 (image): fp32 + residual epilogue", bias=True, res=True, **F)
gemm(6400, 3072, 1024, "QKV (image): fp16 output", bias=True, out_bf16=True, out_fp16=True, **F)
gemm(2304, 3072, 768, "FFN1 (text): GELU, fp16 + bf16 copy + gelu' outputs", bias=True, act=L.VB_ACT_GELU, out_bf16=True, out_fp16=True, **F)
gemm(2304, 3072, 768, "dgrad FFN2 (text): DGELU, bf16", b_mn=True, act=L.VB_ACT_DGELU, out_bf16=True)
gemm(1024, 1024, 6400, "wgrad (image), split-K atomics", a_mn=True, b_mn=True, atomic=True, split_k=0)
gemm(6400, 1024, 1024, "dgrad into the residual gradient (image)", b_mn=True, res=True)
gemm(2304, 768, 768, "out-proj (text): fp32 + residual", bias=True, res=True, **F)
gemm(2304, 768, 3072, "FFN2 (text): fp32 + residual", bias=True, res=True, **F)
lib = L.lib(); dev = "cuda"; M, H = 6400, 1024
x = torch.randn(M, H, device=dev); g = torch.randn(H, device=dev); b = torch.randn(H, device=dev)
y32 = torch.empty(M, H, device=dev); y16 = torch.empty(M, H, device=dev, dtype=torch.float16); yb = torch.empty(M, H, device=dev, dtype=torch.bfloat16)
mean = torch.empty(M, device=dev); rstd = torch.empty(M, device=dev)
dy = torch.randn(M, H, device=dev); dx32 = torch.empty(M, H, device=dev); dx16 = torch.empty(M, H, device=dev, dtype=torch.bfloat16)
dg = torch.zeros(H, device=dev); db = torch.zeros(H, device=dev); dbias = torch.zeros(H, device=dev)
st = C.c_void_p(torch.cuda.current_stream().cuda_stream)
lib.vb_layernorm_fwd(x.data_ptr(), H, g.data_ptr(), b.data_ptr(), 1e-12, y32.data_ptr(), y16.data_ptr(), H, mean.data_ptr(), rstd.data_ptr(), M, H, None, 1, None, yb.data_ptr(), st)
lib.vb_layernorm_bwd(dy.data_ptr(), H, x.data_ptr(), H, g.data_ptr(), mean.data_ptr(), rstd.data_ptr(), dx32.data_ptr(), dx16.data_ptr(), H, None, 0,
                     dg.data_ptr(), db.data_ptr(), dbias.data_ptr(), M, H, None, None, st)
torch.cuda.synchronize()
os.makedirs(os.path.join(ROOT, "profiles"), exist_ok=True)
json.dump(order, open(os.path.join(ROOT, "profiles", "ncu_targets_order.json"), "w"))
# attention last (the check inside attn_case also launches torch kernels, which the -k filter ignores)
attn_case(64, 8, 100, 100, 128, False, fp16=True)
attn_case(64, 12, 36, 36, 64, False, fp16=True)
torch.cuda.synchronize()
