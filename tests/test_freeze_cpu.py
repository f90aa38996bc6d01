"""Frozen parameters (Plan(frozen=...), requires_grad=False on the module surface), checked on CPU-built plans of the tiny config:
the backward writes no range a frozen parameter owns, launches no weight-gradient work for it, stops the gradient where nothing below
needs one, and the all-trainable plan is unchanged."""
import json
import os
import re
import sys

import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from oracle import vilbert_oracle as O
from vilbert_b200.config import BertConfig
from vilbert_b200.engine import LOSS_HEADS, Engine

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tools"))
import plan_dump as PD  # noqa: E402

NT, NV = 9, 11
TRAIN = dict(grad_outputs=O.HEAD_NAMES, train=True)


def _cfg(golden_dir, **over):
    return BertConfig.from_dict(dict(json.load(open(os.path.join(golden_dir, "tiny_b4.json")))["config"], **over))


def patterns(cfg, names):
    """The freezing patterns of the issue-level measurements (tools/freeze_probe.py restates them): name -> frozen entry names."""
    first_t = cfg.t_biattention_id[0]
    text = [n for n in names if n.startswith("bert.embeddings.") or any(n.startswith(f"bert.encoder.layer.{i}.") for i in range(first_t))]
    image = [n for n in names if n.startswith(("bert.v_embeddings.", "bert.encoder.v_layer.")) or
             re.match(r"bert\.encoder\.c_layer\.\d+\.biattention\.(query1|key1|value1)\.", n)]
    return {"text_below_first_connection": frozenset(text), "vision_stream": frozenset(image),
            "heads_only": frozenset(n for n in names if n.startswith("bert."))}


def _listing(plan):
    out = []
    PD.dump_plan(out, "plan", plan)
    return out


def _grad_offsets(plan, section="bwd"):
    """Byte offsets into the flat gradient buffer of every pointer a backward op passes (arguments and struct fields)."""
    offs = []
    for line in _listing(plan):
        if line.startswith(section + " "):
            offs += [int(m) // 4 for m in re.findall(r"\bgrad\+(\d+)", line)]
    return offs


def _entry_at(ps, off):
    for name, (o, shape) in ps.entries.items():
        n = 1
        for d in shape:
            n *= d
        if o <= off < o + n:
            return name
    return None


def _check_frozen_untouched(plan, frozen):
    ps = plan.e.ps
    spans = {n: (ps.entries[n][0], ps.g(n).numel()) for n in frozen}
    for (off, n) in plan.grad_touch:
        for name, (o, m) in spans.items():
            assert off + n <= o or off >= o + m, f"grad_touch range {(off, n)} overlaps frozen {name}"
    for off in _grad_offsets(plan):
        assert _entry_at(ps, off) not in frozen, f"a backward op points into the gradient of frozen {_entry_at(ps, off)}"


def _ops(plan, fn, section="bwd"):
    return [args for f, args, _ in getattr(plan, section) if f is not None and f.__name__ == fn]


def _plan(cfg, frozen=frozenset(), heads="vl", B=4, **kw):
    eng = Engine(cfg, "cpu", heads=heads, _build_only=True)
    return eng.plan(B, NT, NV, frozen=frozen, **(kw or TRAIN))


def test_empty_frozen_set_is_the_default_plan(golden_dir):
    cfg = _cfg(golden_dir)
    for kw in (TRAIN, dict(grad_outputs=LOSS_HEADS["vqa"], loss="vqa", train=True, loss_in_forward=True, score=True)):
        a = Engine(cfg, "cpu", _build_only=True).plan(4, NT, NV, **kw)
        b = Engine(cfg, "cpu", _build_only=True).plan(4, NT, NV, frozen=frozenset(), **kw)
        assert _listing(a) == _listing(b)
    eng = Engine(cfg, "cpu", _build_only=True)
    assert eng.plan(4, NT, NV, **TRAIN) is eng.plan(4, NT, NV, frozen=(), **TRAIN)
    assert eng.plan(4, NT, NV, **TRAIN) is not eng.plan(4, NT, NV, frozen={"vil_logit.bias"}, **TRAIN)    # part of the plan key
    with pytest.raises(ValueError):
        eng.plan(4, NT, NV, frozen={"cls.predictions.decoder.weight"}, **TRAIN)    # the tied decoder is the word-embedding entry


@pytest.mark.parametrize("pattern", ["text_below_first_connection", "vision_stream", "heads_only"])
def test_patterns_write_no_frozen_range(golden_dir, pattern):
    cfg = _cfg(golden_dir)
    names = list(Engine(cfg, "cpu", _build_only=True).ps.entries)
    frozen = patterns(cfg, names)[pattern]
    full, plan = _plan(cfg), _plan(cfg, frozen)
    _check_frozen_untouched(plan, frozen)
    # the forward is the same launch list
    assert [l for l in _listing(plan) if l.startswith("fwd ")] == [l for l in _listing(full) if l.startswith("fwd ")]
    assert plan.n_kernels_bwd < full.n_kernels_bwd
    # every trainable parameter the all-trainable plan gives a gradient still receives it
    ps = plan.e.ps
    for name, (o, _) in ps.entries.items():
        if name not in frozen and any(off <= o < off + n for (off, n) in full.grad_touch):
            assert any(off <= o < off + n for (off, n) in plan.grad_touch), f"{name} lost its gradient"


def test_vision_stream_frozen_uses_the_partial_coattention_backward(golden_dir):
    cfg = _cfg(golden_dir)
    names = list(Engine(cfg, "cpu", _build_only=True).ps.entries)
    plan = _plan(cfg, patterns(cfg, names)["vision_stream"])
    att = [a[0]._obj for a in _ops(plan, "vb_attention_bwd")]
    n_conn = len(cfg.v_biattention_id)
    dq_only = [a for a in att if a.dQ and not a.dK and not a.dV]
    dkv_only = [a for a in att if not a.dQ and a.dK and a.dV]
    # only the first connection layer reads vision states that need no gradient (the later ones read its trainable vision FFN):
    # there, text queries over regions need dQ alone and region queries over text dK / dV alone
    assert len(dq_only) == 1 and len(dkv_only) == 1
    assert all(not a.dbias_k and not a.dbias_v for a in dq_only) and all(not a.dbias_q for a in dkv_only)
    # the image layers here all sit behind a connection layer's trainable vision FFN: they pass the gradient on (dgrad) into it;
    # the image embedding has no backward
    assert len(att) == 2 * n_conn + cfg.num_hidden_layers + cfg.v_num_hidden_layers
    assert not _ops(plan, "vb_loc_proj_bwd")


def test_heads_only_has_no_encoder_backward(golden_dir):
    cfg = _cfg(golden_dir)
    names = list(Engine(cfg, "cpu", _build_only=True).ps.entries)
    plan = _plan(cfg, patterns(cfg, names)["heads_only"])
    for fn in ("vb_attention_bwd", "vb_embed_text_bwd", "vb_loc_proj_bwd", "vb_masked_mean_bwd", "vb_relu_bwd"):
        assert not _ops(plan, fn), fn
    ps = plan.e.ps
    assert all(not _entry_at(ps, off).startswith("bert.") for (off, n) in plan.grad_touch)
    assert all(not plan.out_rg[n] for n in ("sequence_output_t", "sequence_output_v", "pooled_output_t", "pooled_output_v"))
    assert all(plan.out_rg[n] for n in O.HEAD_NAMES)


def test_middle_text_layer_keeps_dgrad_and_drops_wgrad(golden_dir):
    cfg = _cfg(golden_dir)
    names = list(Engine(cfg, "cpu", _build_only=True).ps.entries)
    frozen = frozenset(n for n in names if n.startswith("bert.encoder.layer.1."))
    full, plan = _plan(cfg), _plan(cfg, frozen)
    _check_frozen_untouched(plan, frozen)
    ps = plan.e.ps
    w = ps.entries["bert.embeddings.word_embeddings.weight"][0]
    assert any(off == w for (off, n) in plan.grad_touch)                 # the gradient still reaches the embeddings
    assert len(_ops(plan, "vb_attention_bwd")) == len(_ops(full, "vb_attention_bwd"))
    assert len(_ops(plan, "vb_gemm_bf16")) == len(_ops(full, "vb_gemm_bf16")) - 4    # QKV, out, FFN-in, FFN-out weight gradients


def test_layernorm_parameters_frozen(golden_dir):
    cfg = _cfg(golden_dir)
    names = list(Engine(cfg, "cpu", _build_only=True).ps.entries)
    frozen = frozenset(n for n in names if "LayerNorm" in n or ".logit_fc.2." in n)
    full, plan = _plan(cfg), _plan(cfg, frozen)
    _check_frozen_untouched(plan, frozen)
    ln = _ops(plan, "vb_layernorm_bwd")
    assert len(ln) == len(_ops(full, "vb_layernorm_bwd")) and all(a.dgamma is None and a.dbeta is None for a in ln)
    assert len(_ops(plan, "vb_gemm_bf16")) == len(_ops(full, "vb_gemm_bf16"))


def test_frozen_word_embeddings_with_task_tokens(golden_dir):
    cfg = _cfg(golden_dir, task_specific_tokens=True)
    wn = "bert.embeddings.word_embeddings.weight"
    plan = _plan(cfg, frozenset({wn}))
    _check_frozen_untouched(plan, {wn})
    (emb,) = _ops(plan, "vb_embed_text_bwd")
    assert emb.dword is None and all(a is not None for a in (emb.dpos, emb.dtype, emb.dtask))   # position, type and task tables written
    # the masked-LM decoder tied to it gets no weight gradient either
    assert plan.out_rg["linguisic_prediction"]


def test_pretraining_heads_with_the_tied_decoder_frozen(golden_dir):
    cfg = _cfg(golden_dir)
    wn = "bert.embeddings.word_embeddings.weight"
    for kw in (dict(grad_outputs=LOSS_HEADS["pretraining"], loss="pretraining", train=True, loss_in_forward=True),
               dict(grad_outputs=LOSS_HEADS["pretraining"], loss="pretraining", train=True)):
        full, plan = _plan(cfg, heads="pretraining", **kw), _plan(cfg, frozenset({wn}), heads="pretraining", **kw)
        _check_frozen_untouched(plan, {wn})
        assert len(_ops(plan, "vb_gemm_bf16")) == len(_ops(full, "vb_gemm_bf16")) - 1


@pytest.mark.parametrize("over", [dict(dynamic_attention=True), dict(in_batch_pairs=True)])
def test_dynamic_attention_and_pairs_with_a_frozen_vision_stream(golden_dir, over):
    cfg = _cfg(golden_dir, **over)
    names = list(Engine(cfg, "cpu", _build_only=True).ps.entries)
    frozen = patterns(cfg, names)["vision_stream"]
    full, plan = _plan(cfg), _plan(cfg, frozen)
    _check_frozen_untouched(plan, frozen)
    assert plan.n_kernels_bwd < full.n_kernels_bwd
    if over.get("dynamic_attention"):
        # the image layers' gate Linears are frozen but their input, the pooled text states, needs a gradient: the gate backward
        # still runs for d pool, without the bias sum (dz NULL) and without the gate's weight gradient
        gates = _ops(plan, "vb_gate_scale_bwd")
        assert len(gates) == len(_ops(full, "vb_gate_scale_bwd")) and all(a.dz is None and a.dz16 is not None for a in gates)
        assert _ops(plan, "vb_masked_mean_bwd")


def test_all_frozen_outputs_carry_no_gradient(golden_dir):
    cfg = _cfg(golden_dir)
    eng = Engine(cfg, "cpu", _build_only=True)
    plan = eng.plan(4, NT, NV, frozen=frozenset(eng.ps.entries), **TRAIN)
    assert not any(plan.out_rg.values()) and not plan.grad_touch and plan.n_kernels_bwd == 0


# ------------------------------------------------------------------------------------------------ data parallel
def _worker(rank, world, port, golden_dir, out):
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    sys.path.insert(0, ROOT)
    from vilbert_b200.ddp import FlatGradAllReducer, trainable_ranges
    from vilbert_b200.engine import ParamStore
    dist.init_process_group("gloo", rank=rank, world_size=world)
    cfg = _cfg(golden_dir)
    ps = ParamStore(cfg, "cpu")
    frozen = patterns(cfg, list(ps.entries))["vision_stream"]
    g = torch.Generator().manual_seed(200 + rank)
    ps.grad.copy_(torch.randn(ps.numel, generator=g))
    mine = ps.grad.clone()
    red = FlatGradAllReducer(ps.grad, n_buckets=5)
    full = [(b.data_ptr(), b.numel()) for b in red.buckets]
    red.set_ranges(trainable_ranges(ps, frozenset()))
    same = [(b.data_ptr(), b.numel()) for b in red.buckets] == full
    ranges = trainable_ranges(ps, frozen)
    red.set_ranges(ranges)
    red.allreduce()
    mean = sum(torch.randn(ps.numel, generator=torch.Generator().manual_seed(200 + r)) for r in range(world)) / world
    live = torch.zeros(ps.numel, dtype=torch.bool)
    for lo, hi in ranges:
        live[lo:hi] = True
    ok_live = torch.allclose(ps.grad[live], mean[live], atol=1e-6)
    ok_frozen = torch.equal(ps.grad[~live], mine[~live])
    n_frozen = sum(ps.g(n).numel() for n in frozen)
    out[rank] = (same, ok_live, ok_frozen, int((~live).sum()) >= n_frozen, len(ranges), sum(b.numel() for b in red.buckets) == int(live.sum()))
    dist.barrier()
    dist.destroy_process_group()


def test_reducer_exchanges_only_trainable_ranges_world2(golden_dir):
    world = 2
    port = 31500 + (os.getpid() % 2000)
    mgr = mp.Manager()
    out = mgr.dict()
    mp.spawn(_worker, args=(world, port, golden_dir, out), nprocs=world, join=True)
    for rank in range(world):
        same, ok_live, ok_frozen, covers, n_ranges, sizes = out[rank]
        assert same and ok_live and ok_frozen and covers and sizes
        assert n_ranges >= 2          # the frozen vision stream splits the buffer into coalesced trainable runs
