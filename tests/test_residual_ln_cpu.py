"""The residual add of LN(dropout(dense(a)) + r) lives in the LayerNorm, not in the GEMM epilogue: CPU-built plans of the tiny config
state which GEMMs still read an fp32 residual, forward and backward."""
import json
import os

from oracle import vilbert_oracle as O
from vilbert_b200.config import BertConfig
from vilbert_b200.engine import Engine

NT, NV = 9, 11


def _plan(golden_dir, **kw):
    cfg = BertConfig.from_dict(json.load(open(os.path.join(golden_dir, "tiny_b4.json")))["config"])
    return Engine(cfg, "cpu", _build_only=True).plan(4, NT, NV, **kw)


def _ops(section):
    return [(f.__name__, args) for f, args, _ in section if f is not None]


def test_dense_res_ln_gemms_read_no_residual(golden_dir):
    plan = _plan(golden_dir, grad_outputs=O.HEAD_NAMES, train=True)
    fwd = _ops(plan.fwd)
    adds = [i for i, (n, _) in enumerate(fwd) if n == "vb_add_layernorm_fwd"]
    c = plan.cfg
    assert len(adds) == 2 * c.num_hidden_layers + 2 * c.v_num_hidden_layers + 4 * len(c.v_biattention_id)
    gemm_out = {}
    for n, args in fwd:
        if n == "vb_gemm_bf16":
            g = args[0]._obj
            gemm_out[g.out_f32] = g
    for i in adds:
        args = fwd[i][1]
        assert args.x_out == args.d               # the sum is kept for the backward, over the dense output
        g = gemm_out[args.d]
        assert g.residual is None and g.bias is not None and g.dropout.step is None
        assert args.dropout is not None           # train mode: the hidden dropout moved along with the add
    # the only forward GEMM that still adds a residual is the image embedding's (+ the 5-wide location projection)
    res_fwd = [a[0]._obj for n, a in fwd if n == "vb_gemm_bf16" and a[0]._obj.residual is not None]
    assert [(g.M, g.N) for g in res_fwd] == [(4 * NV, c.v_hidden_size)]


def test_residual_gradients_go_to_the_layernorm_backward(golden_dir):
    plan = _plan(golden_dir, grad_outputs=O.HEAD_NAMES, train=True)
    bwd = _ops(plan.bwd)
    c = plan.cfg
    n_add = sum(1 for n, _ in bwd if n == "vb_add_layernorm_bwd")
    # every residual LayerNorm but those under the last layer of each stream (their output gradient comes from the heads first)
    # takes the residual-path gradient of the block above it as its second input
    n_blocks = 2 * c.num_hidden_layers + 2 * c.v_num_hidden_layers + 4 * len(c.v_biattention_id)
    assert n_add == n_blocks - 2
    # the GEMMs that still read a residual: those that accumulate into a gradient another op wrote first (residual == output, the
    # order of those fp32 sums stays that of the writers), and the dgrads into the two embedding outputs, whose gradient the
    # embedding backward kernels read
    res = [a[0]._obj for n, a in bwd if n == "vb_gemm_bf16" and a[0]._obj.residual is not None]
    assert sum(1 for g in res if g.residual != g.out_f32) == 2
    for n, args in bwd:
        if n == "vb_add_layernorm_bwd":
            assert args.dy2 is not None and args.dy2 != args.dy
