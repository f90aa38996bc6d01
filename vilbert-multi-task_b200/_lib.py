"""ctypes binding of libvilbert_b200.so (C ABI: include/vilbert_b200.h).

The header is the one statement of the ABI: it is parsed once at import, every declared function is bound from its prototype,
its integer constants (enum members, #define VB_...) become attributes of this module, and launch_args names each argument
after its parameter. The struct mirrors below are written by hand (tests/test_host_cpu.py checks them against the header).

The library is the product; there is NO fallback. If the shared object is missing or a call
returns a non-zero status this module raises — nothing here ever routes to a CPU/PyTorch path.
"""
import ctypes as C
import os
import re
from collections import namedtuple

import torch

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libvilbert_b200.so")
HEADER_PATH = os.path.normpath(os.path.join(_HERE, "..", "include", "vilbert_b200.h"))


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
                ("correct_bias", C.c_int32), ("one_minus_beta1", C.c_float), ("one_minus_beta2", C.c_float)]


class NanRegion(C.Structure):
    """Mirror of ``struct vb_nan_region``."""

    _fields_ = [("ptr", C.c_void_p), ("rows", C.c_int64), ("cols", C.c_int64), ("ld", C.c_int64), ("dtype", C.c_int32),
                ("id", C.c_int32)]


def header_text():
    """include/vilbert_b200.h without its comments."""
    with open(HEADER_PATH) as f:
        return re.sub(r"/\*.*?\*/", "", f.read(), flags=re.S)


# one declaration of a parameter or struct field: C type (const, base type, optional *) and one or more names
_DECL = re.compile(r"((?:const\s+)?\w+)\s*(\*?)\s*(\w+(?:\s*,\s*\w+)*)")


def _decls(text, what):
    """[(C type, name)] of a declaration such as `const void* A` or `int32_t M, N, K`; anything else raises VBError."""
    m = _DECL.fullmatch(text.strip())
    if m is None:
        raise VBError(f"include/vilbert_b200.h: cannot parse {text.strip()!r} in {what}")
    t = " ".join(m[1].split()) + m[2]
    return [(t, n.strip()) for n in m[3].split(",")]


def _parse_header(text):
    """-> (functions {name: (return type, [(C type, parameter name)])}, integer constants {name: value}, structs {typedef name:
    [(C type, field name)]}) of the header text."""
    consts = {n: int(v) for n, v in re.findall(r"^#define\s+(VB_\w+)\s+(-?\d+)\s*$", text, re.M)}
    for body in re.findall(r"\benum\s*\{([^}]*)\}", text):
        v = -1
        for member in filter(None, (s.strip() for s in body.split(","))):
            name, _, value = member.partition("=")
            v = int(value) if value.strip() else v + 1
            consts[name.strip()] = v
    structs = {name: [d for decl in body.split(";") if decl.strip() for d in _decls(decl, name)]
               for body, name in re.findall(r"\btypedef\s+struct\s+\w+\s*\{([^}]*)\}\s*(\w+)\s*;", text)}
    funcs = {}
    for ret, star, name, params in re.findall(r"((?:const\s+)?\w+)\s*(\*?)\s*\b(vb_\w+)\s*\(([^)]*)\)\s*;", text):
        params = [] if params.strip() == "void" else [d for p in params.split(",") for d in _decls(p, name)]
        funcs[name] = (" ".join(ret.split()) + star, params)
    return funcs, consts, structs


_SCALARS = {"int32_t": C.c_int32, "int64_t": C.c_int64, "uint32_t": C.c_uint32, "int": C.c_int, "float": C.c_float}
_RESTYPES = {"vb_status": C.c_int, "int": C.c_int, "const char*": C.c_char_p}


def ctype(t):
    """The ctypes type of a parameter or field of C type `t`: scalars as themselves, a descriptor pointer as a pointer to its
    mirror (ctypes then checks that one is passed), every other pointer as c_void_p (which also takes byref(...))."""
    if t.endswith("*"):
        return {"vb_gemm_args": C.POINTER(GemmArgs), "vb_attn_args": C.POINTER(AttnArgs)}.get(
            t[:-1].replace("const ", ""), C.c_void_p)
    if t not in _SCALARS:
        raise VBError(f"include/vilbert_b200.h: no ctypes type for {t!r}")
    return _SCALARS[t]


def _bindings(funcs):
    """-> ({name: (restype, argtypes)}, {name: namedtuple of its launch arguments, the parameter names without the trailing
    stream})"""
    types, args = {}, {}
    for name, (ret, params) in funcs.items():
        if ret not in _RESTYPES:
            raise VBError(f"include/vilbert_b200.h: {name} returns {ret!r}, which has no ctypes type here")
        types[name] = (_RESTYPES[ret], [ctype(t) for t, _ in params])
        names = [n for _, n in params]
        args[name] = namedtuple(name, names[:-1] if names[-1:] == ["stream"] else names)
    return types, args


FUNCTIONS, _CONSTANTS, STRUCTS = _parse_header(header_text())
globals().update(_CONSTANTS)
_TYPES, ARGS = _bindings(FUNCTIONS)

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
        for name, (restype, argtypes) in _TYPES.items():
            fn = getattr(_lib, name)   # AttributeError here = stale build: fail loudly
            fn.restype, fn.argtypes = restype, argtypes
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
    """The C arguments of one launch of the entry point `fn` without its trailing stream, each converted by arg(), as the
    namedtuple ARGS[fn.__name__]: readers name an argument after its parameter in the header (its `count` field, where a
    prototype has one, hides tuple.count). Their count is checked against fn's prototype here: ctypes would check it only when
    the launch first runs."""
    cls = ARGS[fn.__name__]
    if len(values) != len(cls._fields):
        raise TypeError(f"{fn.__name__} takes {len(cls._fields)} arguments before the stream, got {len(values)}")
    return cls._make(arg(v) for v in values)


def call(fn, *values, stream=None):
    """One launch of `fn` on `stream` (default: the current stream), outside a plan; raises VBError on a non-zero status."""
    if stream is None:
        stream = torch.cuda.current_stream().cuda_stream
    check(fn(*launch_args(fn, *values), stream), fn.__name__)


def exported_symbols():
    """Names of the functions declared in include/vilbert_b200.h, used by the ABI test."""
    return sorted(FUNCTIONS)
