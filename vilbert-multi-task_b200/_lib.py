"""ctypes binding of libvilbert_b200.so (C ABI: include/vilbert_b200.h).

The library is the product; there is NO fallback. If the shared object is missing or a call
returns a non-zero status this module raises — nothing here ever routes to a CPU/PyTorch path.
"""
import ctypes as C
import os

import torch

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libvilbert_b200.so")

VB_ACT_NONE, VB_ACT_GELU, VB_ACT_RELU, VB_ACT_DGELU = 0, 1, 2, 3
VB_SCORE_SOFT, VB_SCORE_LABEL, VB_SCORE_THRESHOLD, VB_SCORE_CHOICE = 0, 1, 2, 3
VB_RESULT_ARGMAX, VB_RESULT_SOFTMAX, VB_RESULT_GATHER = 0, 1, 2


class VBError(RuntimeError):
    pass


class DropoutSite(C.Structure):
    """Mirror of ``struct vb_dropout_site`` (the dropout of the GEMM epilogue and of attention)."""

    _fields_ = [("step", C.c_void_p), ("site", C.c_uint32), ("p", C.c_float)]


class Dropout(DropoutSite):
    """Mirror of ``struct vb_dropout`` (the row-wise kernels' descriptor): a DropoutSite with an optional packed-row map. Assigned
    to the dropout field of GemmArgs / AttnArgs it contributes its DropoutSite part."""

    _fields_ = [("row_map", C.c_void_p)]


class GemmArgs(C.Structure):
    """Mirror of ``struct vb_gemm_args`` (include/vilbert_b200.h)."""

    _fields_ = [
        ("M", C.c_int32), ("N", C.c_int32), ("K", C.c_int32),
        ("A", C.c_void_p), ("lda", C.c_int64), ("a_mn_major", C.c_int32),
        ("B", C.c_void_p), ("ldb", C.c_int64), ("b_mn_major", C.c_int32),
        ("alpha", C.c_float),
        ("bias", C.c_void_p),
        ("residual", C.c_void_p), ("ld_res", C.c_int64),
        ("aux", C.c_void_p), ("ld_aux", C.c_int64),
        ("act", C.c_int32),
        ("out_f32", C.c_void_p), ("ld_out_f32", C.c_int64),
        ("out_bf16", C.c_void_p), ("ld_out_bf16", C.c_int64),
        ("out_pre", C.c_void_p), ("ld_out_pre", C.c_int64),
        ("atomic_out", C.c_int32), ("out_colsum", C.c_void_p), ("dropout", DropoutSite), ("split_k", C.c_int32), ("block_n", C.c_int32), ("max_ctas", C.c_int32),
        ("dbg_timeline", C.c_void_p),
        ("a_fp16", C.c_int32), ("b_fp16", C.c_int32), ("out_fp16", C.c_int32),
        ("A_lo", C.c_void_p), ("B_lo", C.c_void_p), ("out_lo", C.c_void_p), ("out_b16", C.c_void_p),
    ]


class AttnArgs(C.Structure):
    """Mirror of ``struct vb_attn_args``."""

    _fields_ = [
        ("B", C.c_int32), ("H", C.c_int32), ("Nq", C.c_int32), ("Nk", C.c_int32), ("D", C.c_int32),
        ("Q", C.c_void_p), ("ldq", C.c_int64), ("K", C.c_void_p), ("ldk", C.c_int64), ("V", C.c_void_p), ("ldv", C.c_int64),
        ("mask", C.c_void_p), ("scale", C.c_float),
        ("O", C.c_void_p), ("ldo", C.c_int64), ("lse", C.c_void_p),
        ("dO", C.c_void_p), ("lddo", C.c_int64), ("dQ", C.c_void_p), ("lddq", C.c_int64),
        ("dK", C.c_void_p), ("lddk", C.c_int64), ("dV", C.c_void_p), ("lddv", C.c_int64),
        ("delta", C.c_void_p),
        ("dbias_q", C.c_void_p), ("dbias_k", C.c_void_p), ("dbias_v", C.c_void_p),
        ("dropout", DropoutSite),
        ("qkv_fp16", C.c_int32), ("Q_lo", C.c_void_p), ("K_lo", C.c_void_p), ("V_lo", C.c_void_p), ("O_lo", C.c_void_p),
        ("O_b16", C.c_void_p),
        ("q_off", C.c_void_p), ("q_len", C.c_void_p), ("k_off", C.c_void_p), ("k_len", C.c_void_p),
    ]


class AdamWGroup(C.Structure):
    """Mirror of ``struct vb_adamw_group``."""

    _fields_ = [("lr", C.c_float), ("beta1", C.c_float), ("beta2", C.c_float), ("eps", C.c_float), ("weight_decay", C.c_float),
                ("correct_bias", C.c_int32)]


_P, _I32, _I64, _F = C.c_void_p, C.c_int32, C.c_int64, C.c_float
# argument types of every entry point of include/vilbert_b200.h (the trailing void* is the stream)
_SIGNATURES = {
    "vb_device_info": [C.POINTER(C.c_int), C.POINTER(C.c_int)],
    "vb_gemm_bf16": [C.POINTER(GemmArgs), _P],
    "vb_gemm_plan": [C.POINTER(GemmArgs), C.c_int32, C.POINTER(C.c_int32), C.POINTER(C.c_int32)],
    "vb_attention_fwd": [C.POINTER(AttnArgs), _P],
    "vb_attention_bwd": [C.POINTER(AttnArgs), _P],
    "vb_attention_probs": [C.POINTER(AttnArgs), _P, _P],
    "vb_layernorm_fwd": [_P, _I64, _P, _P, _F, _P, _P, _I64, _P, _P, _I32, _I32, _P, _I32, _P, _P, _P],
    "vb_layernorm_bwd": [_P, _I64, _P, _I64, _P, _P, _P, _P, _P, _I64, _P, _I64, _P, _P, _P, _I32, _I32, _P, _P, _P],
    "vb_add_layernorm_fwd": [_P, _P, _I64, _P, _P, _P, _P, _F, _P, _P, _I64, _P, _P, _I32, _I32, _I32, _P, _P, _P],
    "vb_add_layernorm_bwd": [_P, _P, _I64, _P, _I64, _P, _P, _P, _P, _P, _I64, _P, _I64, _P, _P, _P, _I32, _I32, _P, _P, _P],
    "vb_cast_f32_to_bf16": [_P, _P, _I64, _I32, _P, _P, _P],
    "vb_cast2d_f32_to_bf16": [_P, _I64, _P, _I64, _I32, _I32, _F, _P],
    "vb_embed_text_fwd": [_P, _P, _P, _P, _P, _P, _P, _P, _I32, _I32, _I32, _P],
    "vb_embed_text_bwd": [_P, _P, _P, _P, _P, _P, _P, _P, _I32, _I32, _I32, _P],
    "vb_loc_proj_fwd": [_P, _P, _P, _P, _I32, _I32, _P],
    "vb_loc_proj_bwd": [_P, _P, _P, _P, _I32, _I32, _P],
    "vb_loc_proj_dx": [_P, _P, _P, _I32, _I32, _P],
    "vb_colsum": [_P, _I32, _I64, _P, _I32, _I32, _P],
    "vb_small_linear_fwd": [_P, _I64, _P, _P, _P, _P, _I32, _I32, _I32, _P, _P],
    "vb_small_linear_bwd": [_P, _P, _I64, _P, _P, _I64, _I32, _P, _P, _I32, _I32, _I32, _P, _P],
    "vb_fuse_pooled_fwd": [_P, _P, _P, _P, _I64, _I32, _P, _I32, _P, _P, _P],
    "vb_fuse_pooled_bwd": [_P, _P, _P, _P, _P, _I64, _I32, _P, _P],
    "vb_step_counter_bump": [_P, _P],
    "vb_broadcast_rows": [_P, _P, _I64, _I32, _P],
    "vb_repeat_rows": [_P, _P, _I64, _I64, _I32, _P],
    "vb_sum_strided": [_P, _P, _I64, _I32, _I64, _I32, _I64, _I32, _P],
    "vb_relu_bwd": [_P, _P, _P, _P, _I64, _P],
    "vb_axpy_f32": [_P, _P, _I64, _F, _P],
    "vb_bce_logits_loss": [_P, _P, _P, _P, _P, _I64, _I32, _I32, _F, _P],
    "vb_mask_to_additive": [_P, _P, _I32, _I32, _I32, _P],
    "vb_memset_zero": [_P, _I64, _P],
    "vb_ce_loss": [_P, _I64, _P, _I64, _P, _P, _I64, _P, _I64, _I32, _I32, _F, _I32, _P],
    "vb_bce_gather_loss": [_P, _I64, _I32, _I32, _P, _P, _I32, _I32, _F, _P, _P, _I32, _P, _I64, _P, _I64, _P],
    "vb_task_score": [_I32, _P, _I64, _I32, _I32, _P, _I32, _P, _I64, _P, _I32, _P, _I32, _P, _P],
    "vb_task_results": [_I32, _P, _I64, _I32, _I32, _P, _I32, _P, _I64, _I32, _P, _P, _I64, _P],
    "vb_retrieval_rank": [_P, _I64, _I32, _I32, _P, _I32, _P, _P, _P],
    "vb_scale_by_device": [_P, _P, _I64, _P, _P],
    "vb_kl_masked_loss": [_P, _P, _P, _P, _P, _P, _I64, _I32, _I32, _I32, _F, _I32, _P],
    "vb_mse_masked_loss": [_P, _P, _P, _I32, _I32, _I32, _F, _P, _P, _I32, _P, _P],
    "vb_nce_region_loss": [_P, _P, _P, _P, _I32, _I32, _I32, _I32, _F, _P, _P, _I32, _P, _P],
    "vb_masked_mean_fwd": [_P, _P, _P, _P, _P, _P, _I32, _I32, _I32, _I32, _P],
    "vb_masked_mean_bwd": [_P, _P, _P, _I32, _I32, _I32, _I32, _P],
    "vb_gate_scale_fwd": [_P, _P, _I64, _P, _I32, _I32, _I32, _I32, _P],
    "vb_gate_scale_bwd": [_P, _I64, _P, _P, _I64, _P, _P, _P, _I32, _I32, _I32, _I32, _P],
    "vb_compact_rows": [_P, _I64, _I32, _I32, _P, _P, _P, _P],
    "vb_compact_rows_mapped": [_P, _I64, _P, _I32, _I32, _P, _P, _P, _P],
    "vb_gather_rows16": [_P, _P, _P, _P, _P, _I32, _I32, _P],
    "vb_scatter_rows_f32": [_P, _P, _P, _I32, _I32, _P, _P, _P],
    "vb_adamw_step": [_P, _P, _P, _P, _P, _P, _P, _I32, _P, _P, _P, _I32, _P, _P, _F, _I32, _P],
    "vb_radam_step": [_P, _P, _P, _P, _P, _P, _P, _I32, _P, _P, _P, _I32, _P, _I32, _P, _I32, _F, _I32, _P],
    "vb_grad_norm": [_P, _P, _P, _I32, _F, _F, _P, _P, _P, _P],
    "vb_adamw_step_clipped": [_P, _P, _P, _P, _P, _P, _P, _I32, _P, _P, _P, _I32, _P, _P, _F, _I32, _P, _P],
    "vb_radam_step_clipped": [_P, _P, _P, _P, _P, _P, _P, _I32, _P, _P, _P, _I32, _P, _I32, _P, _I32, _F, _I32, _P, _P],
    "vb_concat_embed_ln_fwd": [_P, _P, _P, _P, _P, _P, _P, _P, _P, _P, _P, _I32, _P, _P, _I32, _I32, _I32, _I32, _P, _P, _P],
    "vb_concat_embed_ln_bwd": [_P, _P, _P, _P, _P, _P, _P, _P, _P, _P, _P, _P, _P, _P, _P, _P, _P, _I32, _I32, _I32, _I32, _P, _P, _P],
    "vb_embed_text_bwd_padded": [_P, _P, _P, _P, _P, _P, _I32, _I32, _I32, _P],
    "vb_weight_norm_fwd": [_P, _P, _I64, _P, _P, _P, _P, _I32, _P, _P],
    "vb_weight_norm_bwd": [_P, _P, _P, _I64, _P, _P, _P, _P],
    "vb_tanh_fwd": [_P, _P, _P, _P, _P, _I32, _I64, _P],
    "vb_tanh_bwd": [_P, _P, _P, _P, _I32, _I32, _P],
    "vb_mask_concat_additive": [_P, _P, _P, _I32, _I32, _I32, _P],
    "vb_pack_build": [_P, _I32, _I32, _P, _I32, _I32, _I32, _I32, _P, _P, _P, _P, _P, _P, _P],
    "vb_pack_rows_f32": [_P, _P, _P, _I32, _I32, _P],
    "vb_pack_regions": [_P, _P, _I32, _I32, _I32, _P, _P, _P, _P],
    "vb_unpack_rows_f32": [_P, _P, _P, _P, _I32, _I32, _I32, _F, _P],
    "vb_scatter_add_rows_f32": [_P, _P, _P, _I32, _I32, _P],
    "vb_zero_tail_rows": [_P, _P, _P, _I64, _I32, _P, _I32, _P],
    "vb_pack_summary": [_P, _P, _I32, _I32, _I32, _P, _P, _P, _P],
    "vb_reduce_slices": [_P, _I64, _I32, _I64, _P, _P],
    "vb_colsum_det": [_P, _I32, _I64, _P, _I32, _I32, _P, _P],
    "vb_layernorm_bwd_det": [_P, _P, _I64, _P, _I64, _P, _P, _P, _P, _P, _I64, _P, _I64, _P, _P, _P, _I32, _I32, _P, _P, _P, _P],
    "vb_embed_text_bwd_det": [_P, _P, _P, _P, _P, _P, _P, _P, _I32, _I32, _I32, _P],
    "vb_loc_proj_bwd_det": [_P, _P, _P, _P, _I32, _I32, _P, _P],
    "vb_small_linear_bwd_det": [_P, _P, _I64, _P, _P, _I64, _I32, _P, _P, _I32, _I32, _I32, _P, _P, _P],
    "vb_bce_logits_loss_det": [_P, _P, _P, _P, _P, _I64, _I32, _I32, _F, _P, _P],
    "vb_ce_loss_det": [_P, _I64, _P, _I64, _P, _P, _I64, _P, _I64, _I32, _I32, _F, _I32, _P, _P],
    "vb_kl_masked_loss_det": [_P, _P, _P, _P, _P, _P, _I64, _I32, _I32, _I32, _F, _I32, _P, _P],
    "vb_nan_check": [_P, _I32, _P, _I32, _P],
}
# anomaly detection (include/vilbert_b200.h): the dtype codes of a vb_nan_region
VB_NAN_F32, VB_NAN_F16, VB_NAN_BF16 = 0, 1, 2


class NanRegion(C.Structure):
    """Mirror of ``struct vb_nan_region``."""

    _fields_ = [("ptr", C.c_void_p), ("rows", C.c_int64), ("cols", C.c_int64), ("ld", C.c_int64), ("dtype", C.c_int32),
                ("id", C.c_int32)]
# device scratch of one vb_weight_norm_fwd / _bwd launch (include/vilbert_b200.h)
VB_WEIGHT_NORM_SCRATCH = 1024
# deterministic variants (include/vilbert_b200.h): the partials mode of vb_gemm_bf16 and the workspace slices of the _det entry points
VB_GEMM_PARTIALS = 2
VB_DET_SLICES, VB_DET_LN_SLICES, VB_DET_LOSS_SLICES = 64, 256, 1024

_lib = None


def lib():
    """Loads the shared library once; raises VBError if it has not been built."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise VBError(
                f"{LIB_PATH} is missing: run `python -c 'import __graft_entry__ as g; g.build()'` "
                "(there is no CPU or PyTorch fallback for the ViLBERT kernels)")
        _lib = C.CDLL(LIB_PATH)
        _lib.vb_last_error.restype = C.c_char_p
        _lib.vb_version.restype = C.c_int
        for name, argtypes in _SIGNATURES.items():
            fn = getattr(_lib, name)   # AttributeError here = stale build: fail loudly
            fn.argtypes = argtypes
            fn.restype = C.c_int
    return _lib


def check(status, what=""):
    if status != 0:
        msg = lib().vb_last_error().decode("utf-8", "replace")
        raise VBError(f"{what or 'libvilbert_b200'} failed with status {status}: {msg}")


_BYREF = type(C.byref(C.c_int()))


def arg(v):
    """The C value of one launch argument: a tensor's data pointer, a descriptor struct (Dropout, GemmArgs, ...) by reference.
    None, Python and ctypes scalars and byref objects are C values already. Anything else (an Operand passed whole where one of
    its pointers belongs) raises TypeError, so a wrong value fails when the launch is built, not when it first runs."""
    if v is None or isinstance(v, (int, float, C._SimpleCData, _BYREF)):
        return v
    if isinstance(v, torch.Tensor):
        return v.data_ptr()
    if isinstance(v, C.Structure):
        return C.byref(v)
    raise TypeError(f"{type(v).__name__} is not a C launch argument")


def launch_args(fn, *values):
    """The C arguments of one launch of the entry point `fn` without its trailing stream, each converted by arg(). Their count
    is checked against fn's prototype here: ctypes would check it only when the launch first runs."""
    if len(values) != len(fn.argtypes) - 1:
        raise TypeError(f"{fn.__name__} takes {len(fn.argtypes) - 1} arguments before the stream, got {len(values)}")
    return tuple(arg(v) for v in values)


def call(fn, *values, stream=None):
    """One launch of `fn` on `stream` (default: the current stream), outside a plan; raises VBError on a non-zero status."""
    if stream is None:
        stream = torch.cuda.current_stream().cuda_stream
    check(fn(*launch_args(fn, *values), stream), fn.__name__)


def exported_symbols():
    """Names declared in include/vilbert_b200.h (parsed), used by the ABI test."""
    import re
    hdr = os.path.join(_HERE, "..", "include", "vilbert_b200.h")
    with open(hdr) as f:
        text = f.read()
    text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
    return sorted(set(re.findall(r"\b(vb_[a-z0-9_]+)\s*\(", text)))
