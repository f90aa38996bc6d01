"""CPU-side checks of the host code: C-ABI exports, config semantics, parameter layout, plan construction."""
import ctypes
import json
import os
import re

import pytest
import torch

from oracle import vilbert_oracle as O
from vilbert_b200 import _lib as L
from vilbert_b200.config import BertConfig
from vilbert_b200.engine import Engine, ParamStore


def test_library_exports_every_header_function_at_abi_v4():
    """v4: vb_adamw_group carries one_minus_beta1 / one_minus_beta2."""
    lib = L.lib()
    declared = L.exported_symbols()
    assert len(declared) >= 20
    for name in declared:
        assert hasattr(lib, name), f"{name} declared in include/vilbert_b200.h but not exported"
    assert lib.vb_version() == 4
    assert ctypes.sizeof(L.GemmArgs) >= 160 and ctypes.sizeof(L.AttnArgs) >= 150


def test_header_parser_reads_every_prototype():
    """The functions bound from the header are every name the header calls like a function: a prototype the parser cannot read
    fails here instead of going unbound. A type without a ctypes counterpart fails the binding."""
    assert set(L.FUNCTIONS) == set(re.findall(r"\b(vb_\w+)\s*\(", L.header_text()))
    funcs, consts, _ = L._parse_header("enum { VB_A = 4, VB_B };\n#define VB_C 7\nvb_status vb_x(int32_t n, void* stream);")
    assert consts == {"VB_A": 4, "VB_B": 5, "VB_C": 7} and L._bindings(funcs)[1]["vb_x"]._fields == ("n",)
    with pytest.raises(L.VBError, match="double"):
        L._bindings(L._parse_header("vb_status vb_x(double d, void* stream);")[0])


# the hand-written ctypes mirrors and the header structs they mirror; the optimizers hold the vb_clip_record as an int32 tensor
MIRRORS = {L.DropoutSite: "vb_dropout_site", L.Dropout: "vb_dropout", L.GemmArgs: "vb_gemm_args", L.AttnArgs: "vb_attn_args",
           L.AdamWGroup: "vb_adamw_group", L.NanRegion: "vb_nan_region"}


def _mirror_fields(cls, prefix=""):
    """(name, ctypes type) of every field of a mirror, base-class fields first, nested structs flattened."""
    out = []
    for c in reversed(cls.__mro__):
        for f, t in c.__dict__.get("_fields_", ()):
            out += _mirror_fields(t, f"{prefix}{f}.") if issubclass(t, ctypes.Structure) else [(prefix + f, t)]
    return out


def _header_fields(struct, prefix=""):
    out = []
    for t, f in L.STRUCTS[struct]:
        out += _header_fields(t, f"{prefix}{f}.") if t in L.STRUCTS else [(prefix + f, L.ctype(t))]
    return out


@pytest.mark.parametrize("cls", list(MIRRORS), ids=[c.__name__ for c in MIRRORS])
def test_struct_mirror_matches_the_header(cls):
    assert _mirror_fields(cls) == _header_fields(MIRRORS[cls])


def test_every_header_struct_but_the_clip_record_has_a_mirror():
    assert set(MIRRORS.values()) == set(L.STRUCTS) - {"vb_clip_record"}


def test_no_fallback_without_gpu():
    """The product must fail loudly when it cannot run on the GPU: no CPU path."""
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    from vilbert_b200 import modeling
    cfg = BertConfig.from_dict(json.load(open(os.path.join(os.path.dirname(__file__), "golden", "tiny_b4.json")))["config"])
    with pytest.raises(L.VBError):
        modeling.VILBertForVLTasks(cfg, num_labels=1)
    with pytest.raises(L.VBError):
        Engine(cfg, "cpu")


def test_config_semantics(tmp_path, golden_dir):
    cfgj = json.load(open(os.path.join(golden_dir, "base_6layer_6conect_b4.json")))["config"]
    p = tmp_path / "c.json"
    p.write_text(json.dumps(cfgj))
    c = BertConfig.from_json_file(str(p))
    assert c.hidden_size == 768 and c.v_hidden_size == 1024 and c.bi_num_attention_heads == 8
    assert c.v_biattention_id == [0, 1, 2, 3, 4, 5] and c.t_biattention_id == [6, 7, 8, 9, 10, 11]
    # defaults the JSON does not carry (vilbert.py:158-184) and post-hoc mutation
    assert c.fusion_method == "mul" and c.task_specific_tokens is False and c.with_coattention is True
    c.task_specific_tokens = True
    assert json.loads(c.to_json_string())["task_specific_tokens"] is True
    c2 = BertConfig(30522, hidden_size=768)
    assert c2.vocab_size == 30522 and c2.v_feature_size == 2048
    with pytest.raises(ValueError):
        BertConfig(3.5)
    BertConfig.from_dict(dict(cfgj, dynamic_attention=True)).check_supported()
    for bad in (dict(cfgj, dynamic_attention=True, in_batch_pairs=True), dict(cfgj, hidden_act="relu")):
        with pytest.raises(NotImplementedError):
            BertConfig.from_dict(bad).check_supported()
    BertConfig.from_dict(dict(cfgj, model="roberta")).check_supported()      # same embeddings as BERT in the reference (tiny_roberta.json)
    with pytest.raises(NotImplementedError):
        BertConfig.from_dict(dict(cfgj, model="roberta", task_specific_tokens=True)).check_supported()


def test_param_store_layout(golden_dir):
    cfgj = json.load(open(os.path.join(golden_dir, "base_6layer_6conect_b4.json")))["config"]
    cfg = BertConfig.from_dict(cfgj)
    ps = ParamStore(cfg, "cpu")
    ref = O.param_shapes(O.make_config(cfgj))
    ref.pop("cls.predictions.decoder.weight")
    assert {k: tuple(v[1]) for k, v in ps.entries.items()} == {k: tuple(v) for k, v in ref.items()}
    # fused QKV views alias the three reference tensors, in order
    p = "bert.encoder.layer.3.attention.self"
    ps.p(p + ".query.weight").fill_(1.0); ps.p(p + ".key.weight").fill_(2.0); ps.p(p + ".value.weight").fill_(3.0)
    w = ps.p(p + ".qkv.weight")
    assert w.shape == (3 * 768, 768)
    assert w[:768].eq(1).all() and w[768:1536].eq(2).all() and w[1536:].eq(3).all()
    for name, (off, shape) in list(ps.entries.items()) + list(ps.fused.items()):
        assert off % 8 == 0, name     # 16-byte aligned bf16 shadow / 32-byte aligned fp32
    assert ps.p("bert.encoder.c_layer.0.biattention.qkv2.weight").shape == (3 * 1024, 768)


@pytest.mark.parametrize("task_tokens,B", [(False, 4), (True, 3)])
def test_plan_builds_on_cpu(golden_dir, task_tokens, B):
    """Plans are pure host data (buffers + C-ABI call records): build them here without a GPU and check structure."""
    cfgj = dict(json.load(open(os.path.join(golden_dir, "tiny_b4.json")))["config"], task_specific_tokens=task_tokens)
    eng = Engine(BertConfig.from_dict(cfgj), "cpu", _build_only=True)
    fwd_only = eng.plan(B, 9, 11)
    assert fwd_only.n_kernels_bwd == 0 and fwd_only.n_kernels_fwd > 50
    full = eng.plan(B, 9, 11, grad_outputs=O.HEAD_NAMES)
    vqa = eng.plan(B, 9, 11, grad_outputs=("vil_prediction",), vqa_loss=True)
    assert full.n_kernels_fwd == fwd_only.n_kernels_fwd == vqa.n_kernels_fwd
    assert full.n_kernels_bwd > vqa.n_kernels_bwd > full.n_kernels_fwd      # dead head branches are not emitted
    assert set(O.HEAD_NAMES) | set(O.BERT_OUT_NAMES) == set(full.outputs)
    nt = 9 + int(task_tokens)
    assert tuple(full.outputs["sequence_output_t"].shape) == (B, nt, cfgj["hidden_size"])
    assert tuple(full.outputs["linguisic_prediction"].shape) == (B, nt, cfgj["vocab_size"])
    assert tuple(full.outputs["vil_binary_prediction"].shape) == ((B // 2, 2) if B % 2 == 0 else (B, 2))
    bert_only = eng.plan(B, 9, 11, heads="none")
    assert set(bert_only.outputs) == set(O.BERT_OUT_NAMES)


def _op_names(ops):
    return [getattr(op[0], "__name__", None) or getattr(op[0], "_name", "") for op in ops if op[0] is not None]


def test_special_mode_plans_build_on_cpu(golden_dir):
    """Structure of the plans of the optional modes, checked without a GPU: dynamic_attention (gate parameters, pooling / gate ops
    in both passes, data-parallel pieces still tile the gradient buffer) and the compacted masked-LM head of the fused pre-training
    objective (no [tokens, vocab] logits output, capacity arithmetic, cache key)."""
    from vilbert_b200.engine import LOSS_HEADS
    tiny = json.load(open(os.path.join(golden_dir, "tiny_b4.json")))["config"]
    cfgj = dict(tiny, dynamic_attention=True)
    eng = Engine(BertConfig.from_dict(cfgj), "cpu", _build_only=True)
    names = set(eng.ps.entries)
    assert names == set(O.param_shapes(O.make_config(cfgj))) - {"cls.predictions.decoder.weight"} | {"bert.embeddings.word_embeddings.weight"}
    p0 = "bert.encoder.v_layer.0.attention.self"
    (wq, sq), (wk, sk) = eng.ps.entries[p0 + ".dyLinear_q.weight"], eng.ps.entries[p0 + ".dyLinear_k.weight"]
    assert sq == sk == (cfgj["v_hidden_size"], cfgj["hidden_size"]) and wk == wq + sq[0] * sq[1]       # contiguous: one fused [2Hv, Ht] GEMM
    assert eng.ps.fused[p0 + ".dy.weight"] == (wq, (2 * sq[0], sq[1]))
    plan = eng.plan(4, 9, 11, grad_outputs=O.HEAD_NAMES, train=True)
    base = Engine(BertConfig.from_dict(tiny), "cpu", _build_only=True).plan(4, 9, 11, grad_outputs=O.HEAD_NAMES, train=True)
    nv = cfgj["v_num_hidden_layers"]
    f, b = _op_names(plan.fwd), _op_names(plan.bwd)
    assert f.count("vb_gate_scale_fwd") == nv and b.count("vb_gate_scale_bwd") == nv
    assert 1 <= f.count("vb_masked_mean_fwd") <= nv and b.count("vb_masked_mean_bwd") == f.count("vb_masked_mean_fwd")
    assert plan.n_kernels_fwd > base.n_kernels_fwd and plan.n_kernels_bwd > base.n_kernels_bwd
    segs = plan.ddp_segments(4)
    assert segs[0][3] == eng.ps.numel and segs[-1][2] == 0 and all(nx[3] == cur[2] for cur, nx in zip(segs, segs[1:]))
    for (lo, hi, glo, ghi) in segs:
        for (off, n), touch in plan.grad_touch.items():
            if glo <= off < ghi:
                assert touch < hi
    # compacted masked-LM head
    engp = Engine(BertConfig.from_dict(tiny), "cpu", heads="pretraining", _build_only=True)
    B, Nt = 64, 20
    pc = engp.plan(B, Nt, 11, grad_outputs=LOSS_HEADS["pretraining"], loss="pretraining")
    assert "linguisic_prediction" not in pc.outputs and pc.lm_c["cap"] == 320 and tuple(pc.lm_c["logits"].shape) == (320, tiny["vocab_size"])
    assert set(pc.loss_inputs) == {"masked_lm_labels", "image_target", "image_label", "next_sentence_label"}
    assert (pc.loss_inputs["masked_lm_labels"] == -1).all()                     # nothing labelled until the caller loads labels
    engp.lm_capacity = 0.5
    assert engp.plan(B, Nt, 11, grad_outputs=LOSS_HEADS["pretraining"], loss="pretraining").lm_c["cap"] == 640
    engp.lm_compact = False
    pf = engp.plan(B, Nt, 11, grad_outputs=LOSS_HEADS["pretraining"], loss="pretraining")
    assert pf.lm_c is None and tuple(pf.outputs["linguisic_prediction"].shape) == (B, Nt, tiny["vocab_size"])
    assert pf is not pc and len(engp.plans) == 3
    small = Engine(BertConfig.from_dict(tiny), "cpu", heads="pretraining", _build_only=True).plan(4, 9, 11, grad_outputs=LOSS_HEADS["pretraining"], loss="pretraining")
    assert small.lm_c["cap"] == 40                                              # never more rows than there are (8-padded)


@pytest.mark.parametrize("precision", ["fp16", "fp32", "bf16"])
@pytest.mark.parametrize("mode", ["base", "dynamic_attention", "in_batch_pairs"])
def test_tensor_core_operands_are_in_the_format_of_their_pass(golden_dir, precision, mode):
    """Every operand pointer a plan hands the GEMM and attention kernels lies in a tensor of the format the kernel reads it
    as: the forward format (fp16, or bf16) for the forward GEMMs and for Q / K / V / O, bf16 for the backward GEMMs, the
    attention gradients and every bf16 copy. An fp16 buffer passed where its bf16 copy belongs would otherwise be read as
    bf16 bits without any error."""
    bf16 = torch.bfloat16
    cfgj = json.load(open(os.path.join(golden_dir, "tiny_b4.json")))["config"]
    if mode != "base":
        cfgj = dict(cfgj, **{mode: True})
    eng = Engine(BertConfig.from_dict(cfgj), "cpu", _build_only=True, precision=precision)
    plan = eng.plan(4, 9, 11, grad_outputs=O.HEAD_NAMES, train=True)
    ps, fwd_dt = eng.ps, eng.op_dtype
    tensors = [t for t in [ps.shadow, ps.shadow_b, ps.shadow_lo] + plan._keep if torch.is_tensor(t)]
    spans = [(t.data_ptr(), t.data_ptr() + t.numel() * t.element_size(), t.dtype) for t in tensors]

    def dtype_at(p):
        return next(dt for lo, hi, dt in spans if lo <= p < hi)

    n_gemm = n_attn = 0
    wrong = []
    for section, ops in (("fwd", plan.fwd), ("bwd", plan.bwd)):
        pass_dt = fwd_dt if section == "fwd" else bf16
        for fn, args, _ in ops:
            name = getattr(fn, "__name__", None)
            if name == "vb_gemm_bf16":
                n_gemm += 1
                s = args[0]._obj
                want = [(f, pass_dt) for f in ("A", "B", "A_lo", "B_lo", "out_bf16", "out_lo")] + [("out_b16", bf16)]
                if precision == "fp32" and section == "fwd":
                    assert s.A_lo and s.B_lo, "split-precision forward GEMM without low parts"
            elif name in ("vb_attention_fwd", "vb_attention_bwd"):
                n_attn += 1
                s = args[0]._obj
                want = [(f, fwd_dt) for f in ("Q", "K", "V", "O", "Q_lo", "K_lo", "V_lo", "O_lo")] + \
                       [(f, bf16) for f in ("dO", "dQ", "dK", "dV", "O_b16")]
            else:
                continue
            wrong += [(section, name, f, dtype_at(getattr(s, f))) for f, dt in want if getattr(s, f) and dtype_at(getattr(s, f)) != dt]
    assert n_gemm > 100 and n_attn > 10
    assert not wrong, wrong


def test_plan_rejects_operands_in_the_wrong_format(golden_dir):
    """Plan.gemm refuses, while the plan is built, a forward operand that is not an Operand of the engine's format and a
    backward operand that is not bf16."""
    from vilbert_b200.engine import Operand
    cfgj = json.load(open(os.path.join(golden_dir, "tiny_b4.json")))["config"]
    plan = Engine(BertConfig.from_dict(cfgj), "cpu", _build_only=True).plan(4, 9, 11)
    a16, ab = torch.zeros(8, 8, dtype=torch.float16), torch.zeros(8, 8, dtype=torch.bfloat16)
    with pytest.raises(TypeError):
        plan.gemm(8, 8, 8, a16, 8, Operand(a16), 8)                     # forward: plain tensor
    with pytest.raises(TypeError):
        plan.gemm(8, 8, 8, Operand(ab, bw=ab), 8, Operand(a16), 8)       # forward: bf16 in an fp16 engine
    plan.cur = plan.bwd
    with pytest.raises(TypeError):
        plan.gemm(8, 8, 8, ab, 8, a16, 8, out_f32=torch.zeros(8, 8))    # backward: fp16 weight copy in place of its bf16 copy
    plan.gemm(8, 8, 8, ab, 8, ab, 8, out_f32=torch.zeros(8, 8))
    assert plan.bwd[-1][0].__name__ == "vb_gemm_bf16"


def test_emit_checks_launch_arguments_while_the_plan_is_built(golden_dir):
    """Plan.emit makes C values of its arguments (a tensor its data pointer, a dropout descriptor a reference to it) and refuses,
    while the plan is built, a launch whose argument count does not match its prototype and an argument with no C form, such as
    an Operand passed whole where one of its pointers belongs. ctypes would only refuse them when the launch first runs."""
    from vilbert_b200.engine import Operand
    cfgj = json.load(open(os.path.join(golden_dir, "tiny_b4.json")))["config"]
    plan = Engine(BertConfig.from_dict(cfgj), "cpu", _build_only=True).plan(4, 9, 11)
    axpy = plan.lib.vb_axpy_f32
    x, y, h = torch.zeros(8), torch.zeros(8), torch.zeros(8, dtype=torch.float16)
    n = len(plan.fwd)
    with pytest.raises(TypeError, match="vb_axpy_f32 takes 4"):
        plan.emit(axpy, x, y, 8)                                    # one short
    with pytest.raises(TypeError, match="vb_axpy_f32 takes 4"):
        plan.emit(axpy, x, y, 8, 1.0, None)                         # a stream: the plan passes the one the op runs on
    with pytest.raises(TypeError, match="Operand"):
        plan.emit(plan.lib.vb_gather_rows16, Operand(h), h, None, None, x, 8, 1)
    assert len(plan.fwd) == n
    plan.emit(axpy, x, y, 8, 1.0)
    assert plan.fwd[-1][1] == (x.data_ptr(), y.data_ptr(), 8, 1.0)
    d = L.Dropout()
    plan.emit(plan.lib.vb_fuse_pooled_bwd, x, x, y, None, y, 8, 1, d)
    assert plan.fwd[-1][1][3] is None and plan.fwd[-1][1][-1]._obj is d


def test_shared_activation_arena_layout(golden_dir):
    """Engine.enable_activation_arena: activation / scratch buffers of every plan are sub-allocated from one arena (plans overlay
    each other), while everything loaded or initialised outside a run (inputs, targets, output gradients) stays private."""
    from vilbert_b200._lib import VBError
    cfgj = json.load(open(os.path.join(golden_dir, "tiny_b4.json")))["config"]
    plain = Engine(BertConfig.from_dict(cfgj), "cpu", _build_only=True).plan(4, 9, 11, grad_outputs=("vil_prediction",), vqa_loss=True)
    eng = Engine(BertConfig.from_dict(cfgj), "cpu", _build_only=True)
    eng.enable_activation_arena(64 << 20)
    a = eng.plan(4, 9, 11, grad_outputs=("vil_prediction",), vqa_loss=True)
    b = eng.plan(6, 20, 33, grad_outputs=("vil_prediction",), vqa_loss=True)
    assert (a.n_kernels_fwd, a.n_kernels_bwd) == (plain.n_kernels_fwd, plain.n_kernels_bwd)
    lo, hi = eng.arena.data_ptr(), eng.arena.data_ptr() + eng.arena.numel()
    inside = lambda t: lo <= t.data_ptr() < hi
    for p in (a, b):
        assert not any(inside(t) for t in (p.in_ids, p.in_tt, p.in_amask, p.in_imask, p.in_feat, p.in_loc, p.vqa_target, p.loss))
        assert all(inside(t) for t in (p.outputs["sequence_output_t"], p.outputs["vil_prediction"], p.mask_t, p.mask_v))
        assert 0 < p.arena_bytes <= eng.arena.numel() and p.arena_bytes % 256 == 0
    assert a.mask_t.data_ptr() == b.mask_t.data_ptr() and b.arena_bytes > a.arena_bytes       # same offsets: the plans overlay
    private = lambda p: sum(t.numel() * t.element_size() for t in p._keep if torch.is_tensor(t))
    assert private(a) < 0.1 * private(plain)
    with pytest.raises(VBError):
        eng.enable_activation_arena(1 << 20)          # only before the first plan
    small = Engine(BertConfig.from_dict(cfgj), "cpu", _build_only=True)
    small.enable_activation_arena(1 << 20)
    with pytest.raises(VBError):
        small.plan(4, 9, 11)


def test_ddp_segments_partition_the_gradient_buffer(golden_dir):
    """Overlapped data-parallel step: backward pieces (each with at least one kernel, no side-stream event recorded in one
    piece and waited for in a later one) release tail ranges of the flat gradient buffer that (a) tile it exactly and (b)
    are never written by a later backward op."""
    cfgj = json.load(open(os.path.join(golden_dir, "tiny_b4.json")))["config"]
    eng = Engine(BertConfig.from_dict(cfgj), "cpu", _build_only=True)
    plan = eng.plan(4, 9, 11, grad_outputs=O.HEAD_NAMES, train=True)
    for k in (1, 3, 8):
        segs = plan.ddp_segments(k)
        assert segs[0][0] == 0 and segs[-1][1] == len(plan.bwd) and segs[0][3] == eng.ps.numel and segs[-1][2] == 0
        for (lo, hi, glo, ghi), nxt in zip(segs, segs[1:] + [None]):
            assert lo < hi and glo <= ghi
            assert any(op[0] is not None for op in plan.bwd[lo:hi])                          # no kernel-less piece
            recs = {op[1][1] for op in plan.bwd[:hi] if op[0] is None and len(op[1]) == 2 and op[1][0] == "rec"}
            late = {op[1][1] for op in plan.bwd[hi:] if op[0] is None and len(op[1]) == 2 and op[1][0] == "wait"}
            assert not (recs & late)                                                          # no event crosses the cut
            if nxt is not None:
                assert nxt[0] == hi and nxt[3] == glo
            for (off, n), touch in plan.grad_touch.items():                              # released ranges are final
                if off >= glo and off < ghi:
                    assert touch < hi, (off, touch, hi)
    # execution-order layout: the tied word-embedding table (written first AND last in backward) sits at offset 0
    assert eng.ps.entries["bert.embeddings.word_embeddings.weight"][0] == 0


def test_gemm_tile_configuration_cost_model():
    """vb_gemm_plan (host only): the (tile width, k splits) vb_gemm_bf16 picks for the model's GEMM shapes on a 132-SM device
    — 256-wide tiles for the large image-stream problems, 128-wide tiles where the tile count binds, split-K only for the
    weight-gradient form; caller-fixed values are honoured, nonsense is rejected."""
    import ctypes as C
    from vilbert_b200 import _lib as L
    lib = L.lib()

    def plan(M, N, K, sms=132, **kw):
        g = L.GemmArgs(); g.M, g.N, g.K, g.alpha = M, N, K, 1.0
        g.A = g.B = 0x1000                                     # never dereferenced by the query
        g.block_n = kw.get("block_n", 0)
        if kw.get("atomic"):
            g.atomic_out, g.out_f32, g.split_k = 1, 0x1000, kw.get("split_k", 0)
        else:
            g.split_k = kw.get("split_k", 1)
            if kw.get("bf16"): g.out_bf16 = 0x1000
            else: g.out_f32 = 0x1000
            if kw.get("res"): g.residual = 0x1000
        bn, sp = C.c_int32(), C.c_int32()
        st = lib.vb_gemm_plan(C.byref(g), sms, C.byref(bn), C.byref(sp))
        return st, (bn.value, sp.value)

    assert plan(6400, 3072, 1024, bf16=True) == (0, (256, 1))             # image QKV: 256-wide tiles
    assert plan(8192, 8192, 8192, bf16=True) == (0, (256, 1))
    assert plan(2304, 768, 768, res=True) == (0, (128, 1))                # text out-proj: 108 tiles on 132 SMs
    st, (bn, sp) = plan(3072, 1024, 6400, atomic=True)                    # image QKV weight gradient
    assert st == 0 and sp > 1
    st, (bn, sp) = plan(768, 768, 2304, atomic=True)
    assert st == 0 and sp > 1                                             # 36 tiles: split K to fill the SMs
    assert plan(6400, 1024, 1024, res=True)[1][1] == 1                    # no split-K outside the atomic form
    assert plan(6400, 3072, 1024, bf16=True, block_n=128) == (0, (128, 1))
    assert plan(3072, 1024, 6400, atomic=True, split_k=5)[1][1] == 5
    assert plan(6400, 1024, 1024, block_n=64)[0] == 1 and b"block_n" in lib.vb_last_error()
    assert plan(6400, 1024, 1024, res=True, split_k=2)[0] == 1 and b"split_k" in lib.vb_last_error()


def test_bench_reference_arm_contract():
    """`bench.py --impl reference` (the CPU arm beside the GPU arm): rank 0 prints ONE JSON line with the contract
    keys for the same metric / workload, other ranks print nothing and exit 0. Runs the oracle port on a 1-sample step here."""
    import subprocess, sys
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    cmd = [sys.executable, os.path.join(root, "bench.py"), "--impl", "reference", "--gpus", "2", "--steps", "1", "--warmup", "1", "--cpu-batch", "1"]
    env = dict(os.environ, RANK="1", WORLD_SIZE="2", LOCAL_RANK="1")
    r = subprocess.run(cmd, env=env, capture_output=True, text=True, timeout=300)
    assert r.returncode == 0 and r.stdout.strip() == ""
    env = dict(os.environ, RANK="0", WORLD_SIZE="2", LOCAL_RANK="0")
    r = subprocess.run(cmd, env=env, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stderr[-2000:]
    lines = [ln for ln in r.stdout.splitlines() if ln.strip()]
    assert len(lines) == 1
    d = json.loads(lines[0])
    assert d["impl"] == "reference" and d["n_gpus"] == 2 and d["unit"] == "pairs/s" and d["higher_is_better"] is True
    assert "bert_base_6layer_6conect" in d["metric"] and "bert_base_6layer_6conect" in d["config"]["workload"]
    assert d["value"] > 0 and d["ms_per_step"] > 0 and d["steps"] >= 1 and d["dtype"] == "f32" and d["data"] == "synthetic"
    assert d["cpu_baseline"]["kind"] == "port"
    assert d["cpu_baseline"]["cores"] >= 1 and d["cpu_baseline"]["value"] == d["value"]
    assert d["e2e"] == {"value": d["value"], "unit": "pairs/s", "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0}

