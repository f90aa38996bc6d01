"""Anomaly detection on the GPU: vb_nan_check against torch.isnan; finite steps unchanged by the checks (bitwise under
torch.use_deterministic_algorithms(True)); a NaN that starts in the backward raises torch's RuntimeError naming the first op that
held it, with the forward's traceback in a warning, before the optimizer step; a NaN the backward never reaches does not raise."""
import gc
import json
import os
import warnings

import pytest
import torch

import _task_oracle as T
from _gpu_util import rel_l2
from oracle import vilbert_oracle as O

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden")
TINY = json.load(open(os.path.join(GOLDEN, "tiny_b4.json")))["config"]
FROZEN_TEXT = ("bert.embeddings.", "bert.encoder.layer.")
NAN = float("nan")


@pytest.fixture(autouse=True)
def release_engines():
    yield
    gc.collect()
    torch.cuda.empty_cache()


@pytest.fixture
def deterministic():
    prev = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(True)
    yield
    torch.use_deterministic_algorithms(prev)


# ------------------------------------------------------------------------------------------ kernel
def _check(regions):
    """vb_nan_check over regions [(tensor 2-D view, id)] -> the flag (INT32_MAX: none)."""
    from vilbert_b200 import _lib as L
    code = {torch.float32: L.VB_NAN_F32, torch.float16: L.VB_NAN_F16, torch.bfloat16: L.VB_NAN_BF16}
    arr = (L.NanRegion * len(regions))()
    for e, (t, rid) in zip(arr, regions):
        e.ptr, e.rows, e.cols, e.ld, e.dtype, e.id = t.data_ptr(), t.shape[0], t.shape[1], t.stride(0), code[t.dtype], rid
    table = torch.frombuffer(bytearray(bytes(arr)), dtype=torch.uint8).cuda()
    flag = torch.zeros(1, dtype=torch.int32, device="cuda")
    L.call(L.lib().vb_nan_check, None, 0, flag, 1)
    L.call(L.lib().vb_nan_check, table, len(regions), flag, 0)
    return int(flag.item())


def _nan_bits(dtype, sign, payload):
    """A NaN of `dtype` with the sign bit and a non-zero mantissa payload, as a tensor element."""
    bits = {torch.float32: (torch.int32, 23, 0xFF), torch.float16: (torch.int16, 10, 0x1F), torch.bfloat16: (torch.int16, 7, 0xFF)}
    it, man, exp = bits[dtype]
    v = (exp << man) | (payload & ((1 << man) - 1) or 1)
    if sign:
        v -= 1 << (31 if it == torch.int32 else 15)
    return torch.tensor([v], dtype=it).view(dtype)


@pytest.mark.parametrize("dtype", [torch.float32, torch.float16, torch.bfloat16])
def test_nan_check_kernel_against_isnan(dtype):
    M = 2 ** 31 - 1
    g = torch.Generator(device="cuda").manual_seed(0)
    base = torch.randn(300, 517, generator=g, device="cuda").to(dtype)
    assert _check([(base, 5)]) == M
    # +-inf and the largest finite values are not NaN
    x = base.clone()
    x[3, 4], x[7, 9], x[0, 0] = float("inf"), float("-inf"), torch.finfo(dtype).max
    assert _check([(x, 1)]) == M and not torch.isnan(x).any()
    # NaN of both signs and several payloads, at unaligned positions and in the tail of a row
    for sign in (0, 1):
        for payload in (1, 2, 0x3F, (1 << 22) - 1):
            y = base.clone()
            y.view(-1)[1 + payload % 1000] = _nan_bits(dtype, sign, payload).cuda()[0]
            assert torch.isnan(y).any() and _check([(y, 2)]) == 2
    # a strided region: NaN in the pitch padding and past the last row are not part of it
    buf = torch.zeros(64, 40, dtype=dtype, device="cuda")
    view = buf[:60, 3:35]
    buf[:, 35:] = NAN
    buf[:, :3] = NAN
    buf[60:] = NAN
    assert not torch.isnan(view).any() and _check([(view, 0)]) == M
    view[59, 31] = NAN
    assert _check([(view, 0)]) == 0
    # many small regions and a large one in one table: the least id holding a NaN wins
    small = [torch.randn(3, 5, generator=g, device="cuda").to(dtype) for _ in range(200)]
    big = torch.randn(4096, 1024, generator=g, device="cuda").to(dtype)
    regs = [(t, i + 1) for i, t in enumerate(small)] + [(big, 0)]
    assert _check(regs) == M
    small[150][2, 4], small[37][0, 0], big[4095, 1023] = NAN, NAN, NAN
    assert _check(regs) == 0
    big[4095, 1023] = 0
    assert _check(regs) == 38
    assert _check([(t, 1000 - i) for i, t in enumerate(small)]) == 850


def test_nan_check_kernel_region_over_2_gib():
    n = (2 ** 31 + 2 ** 20) // 4          # fp32 elements: more than 2^31 bytes
    x = torch.zeros(1, n, device="cuda")
    assert _check([(x, 3)]) == 2 ** 31 - 1
    x[0, n - 1] = NAN
    assert _check([(x, 3)]) == 3
    del x


# ------------------------------------------------------------------------------------------ module surface
def _model(cls="VILBertForVLTasks", **over):
    import vilbert_b200
    task = dict(task_specific_tokens=True, max_position_embeddings=300) if cls == "VILBertForVLTasks" else {}
    cfgj = dict(TINY, **task, **over)
    model = getattr(vilbert_b200, cls)(vilbert_b200.BertConfig.from_dict(cfgj), **({"fused_objective": True} if cls ==
                                                                                   "BertForMultiModalPreTraining" else {}))
    model.load_state_dict(O.synth_params(O.make_config(cfgj), seed=0, device="cuda"), strict=False)
    return model, cfgj


def _inputs(cfgj, B=4, Nv=11, Nt=9, seed=3):
    inp = O.synth_inputs(O.make_config(cfgj), B, Nv, Nt, seed=seed)
    out = {k: inp[k].cuda() for k in ("input_txt", "input_imgs", "image_loc", "token_type_ids", "attention_mask", "image_attention_mask")}
    out["task_ids"] = torch.full((B, 1), 1, dtype=torch.long, device="cuda")
    return out


def _adamw_step(model):
    from vilbert_b200.optim import FusedAdamW
    opt = FusedAdamW([p for p in model.parameters() if p.requires_grad], lr=1e-3, engine=model.engine)
    opt.step()
    torch.cuda.synchronize()


def _vl_step(frozen_text=False):
    model, cfgj = _model()
    model.train()
    if frozen_text:
        for n, p in model.named_parameters():
            p.requires_grad_(not n.startswith(FROZEN_TEXT))
    inp = _inputs(cfgj)
    inp["input_imgs"].requires_grad_(True)
    model.engine.set_dropout_step(5)
    out = model(**inp)
    loss = sum(o.float().square().mean() for o in out[:7] if o.requires_grad)
    loss.backward()
    r = dict(out=torch.cat([o.detach().reshape(-1) for o in out[:9]]), loss=loss.detach(), grad=model.engine.ps.grad.clone(),
             feat_grad=inp["input_imgs"].grad.clone())
    _adamw_step(model)
    r["params"] = model.engine.ps.flat.clone()
    return r


def _task_step(task_id, packed, B=4):
    from vilbert_b200.tasks import ForwardModelsTrain, LoadLosses
    model, cfgj = _model()
    model.train()
    model.engine.pack_padding = packed
    batch = T.make_batch(cfgj, task_id, B, 11, 9)
    model.engine.set_dropout_step(7)
    losses = LoadLosses(None, T.TASK_CFG, [task_id[4:]])
    loss, score = ForwardModelsTrain(None, T.TASK_CFG, torch.device("cuda"), task_id, {task_id: 0}, {}, {task_id: [batch]}, model,
                                     losses)
    loss.backward()
    r = dict(loss=loss.detach(), score=score.detach(), grad=model.engine.ps.grad.clone())
    _adamw_step(model)
    r["params"] = model.engine.ps.flat.clone()
    if packed and task_id == "TASK1":
        assert any(p.packed for p in model.engine.plans.values())
    return r


def _pretraining_step():
    model, cfgj = _model("BertForMultiModalPreTraining", visual_target=2, v_target_size=48)
    model.train()
    torch.manual_seed(0)        # the negatives of visual_target 2 are sampled with torch's generator
    B, Nv, Nt = 4, 11, 9
    inp = _inputs(cfgj, B, Nv, Nt)
    g = torch.Generator().manual_seed(5)
    labels = torch.full((B, Nt), -1, dtype=torch.long)
    labels[:, 2] = torch.randint(1, cfgj["vocab_size"], (B,), generator=g)
    image_label = (torch.rand(B, Nv - 1, generator=g) > 0.6).long()
    target = torch.randn(B, Nv - 1, 48, generator=g)
    model.engine.set_dropout_step(3)
    losses = model(inp["input_txt"], inp["input_imgs"], inp["image_loc"], inp["token_type_ids"], inp["attention_mask"],
                   inp["image_attention_mask"], masked_lm_labels=labels.cuda(), image_label=image_label.cuda(), image_target=target.cuda(),
                   next_sentence_label=torch.tensor([0, 1, 0, 1]).cuda())
    total = losses[0] + losses[1] + losses[2]
    total.backward()
    r = dict(loss=torch.cat([l.detach() for l in losses]), grad=model.engine.ps.grad.clone())
    _adamw_step(model)
    r["params"] = model.engine.ps.flat.clone()
    return r


def _base_step():
    from oracle import basebert_oracle as BO
    from vilbert_b200.basebert import BaseBertForVLTasks
    from vilbert_b200.config import BertConfig
    meta = json.load(open(os.path.join(GOLDEN, "tiny_basebert.json")))
    cfg, labels = O.make_config(meta["config"]), meta["num_labels"]
    model = BaseBertForVLTasks(BertConfig.from_dict(meta["config"]), labels)
    sd = dict(BO.synth_params(cfg, labels, 0, device="cuda", std=0.05))
    sd["cls.predictions.decoder.weight"] = sd["bert.embeddings.word_embeddings.weight"]
    model.load_state_dict(sd)
    model.train()
    inp = BO.synth_inputs(cfg, meta["B"], meta["Nt"], meta["Nv"], 1234, device="cuda")
    model.engine.set_dropout_step(2)
    out = model(**inp)
    loss = sum(o.float().square().mean() for o in out[:7])
    loss.backward()
    r = dict(loss=loss.detach(), grad=model.engine.ps.grad.clone())
    _adamw_step(model)
    r["params"] = model.engine.ps.flat.clone()
    return r


STEPS = {"vl_train": lambda: _vl_step(), "vl_frozen_text": lambda: _vl_step(True), "task_bce_padded": lambda: _task_step("TASK1", False),
         "task_bce_packed": lambda: _task_step("TASK1", True), "task_ce_padded": lambda: _task_step("TASK5", False, 2),
         "task_ce_packed": lambda: _task_step("TASK5", True, 2), "pretraining_vt2": _pretraining_step}


def _on_off(step):
    off = step()
    with torch.autograd.set_detect_anomaly(True):
        on = step()
    return off, on


@pytest.mark.parametrize("name", sorted(STEPS))
def test_finite_step_bitwise_unchanged_under_determinism(name, deterministic):
    off, on = _on_off(STEPS[name])
    diff = [k for k in off if not torch.equal(off[k], on[k])]
    assert not diff, f"anomaly checks changed {diff}"
    assert torch.isfinite(off["grad"]).all()


@pytest.mark.parametrize("name", sorted(STEPS) + ["base"])
def test_finite_step_within_tolerance_default(name):
    off, on = _on_off(_base_step if name == "base" else STEPS[name])
    for k in off:
        assert rel_l2(on[k].float(), off[k].float()) < 1e-4, k


# ------------------------------------------------------------------------------------------ a NaN in the backward
def _raises_at(module_re, fn):
    with pytest.warns(UserWarning, match="Error detected in") as w, pytest.raises(RuntimeError, match=f"Function '{module_re}: vb_\\w+' "
                                                                                                  "returned nan values in its \\d+th output"):
        fn()
    return "".join(str(x.message) for x in w)


def test_nan_gradient_of_a_head_output_is_located():
    model, cfgj = _model()
    model.train()
    inp = _inputs(cfgj)
    with torch.autograd.set_detect_anomaly(True):
        def forward_of_this_test():
            return model(**inp)
        for call in range(3):          # the third call replays the captured graphs
            out = forward_of_this_test()
            vis = out[6]
            g = torch.zeros_like(vis)
            g[1, 4, 0] = NAN           # one region row
            msg = _raises_at("vision_logit", lambda: torch.autograd.backward(vis, grad_tensors=g))
            assert "forward_of_this_test" in msg and "Traceback of forward call" in msg
        plan = model._last_plan
        assert plan.anomaly and plan.graph_fwd is not None and plan.graph_bwd is not None
        out = forward_of_this_test()
        g = torch.zeros_like(out[0])
        g[2, 17] = NAN
        _raises_at("vil_prediction.logit_fc", lambda: torch.autograd.backward(out[0], grad_tensors=g))
        seq_t = model.bert(inp["input_txt"], inp["input_imgs"], inp["image_loc"], inp["token_type_ids"], inp["attention_mask"],
                           inp["image_attention_mask"], task_ids=inp["task_ids"])[0]
        g = torch.zeros_like(seq_t)
        g[3, 2, :] = NAN
        last = f"bert.encoder.layer.{cfgj['num_hidden_layers'] - 1}.output"
        _raises_at(last.replace(".", "\\."), lambda: torch.autograd.backward(seq_t, grad_tensors=g))
        # a finite gradient after a NaN one: the flag is reset by the next forward (the parameter gradients are checked as
        # accumulated, so the NaN the last backward left in them goes first)
        model.zero_grad()
        out = forward_of_this_test()
        torch.autograd.backward(out[6], grad_tensors=torch.ones_like(out[6]))


def test_reference_loop_stops_before_the_optimizer_step():
    """set_detect_anomaly(True), ForwardModelsTrain, loss.backward(), optimizer.step(): a NaN planted in the backward (the bf16 copy
    of one weight, which only the backward reads) stops the loop at loss.backward(); no parameter changes."""
    from vilbert_b200.optim import FusedAdamW
    from vilbert_b200.tasks import ForwardModelsTrain, LoadLosses
    model, cfgj = _model()
    model.train()
    model.engine.pack_padding = True
    opt = FusedAdamW([p for p in model.parameters()], lr=1e-3, engine=model.engine)
    batch = T.make_batch(cfgj, "TASK1", 4, 11, 9)
    losses = LoadLosses(None, T.TASK_CFG, ["1"])
    ps = model.engine.ps
    with torch.autograd.set_detect_anomaly(True):
        loss, score = ForwardModelsTrain(None, T.TASK_CFG, torch.device("cuda"), "TASK1", {"TASK1": 0}, {}, {"TASK1": [batch]}, model,
                                         losses)
        off, _ = ps.span("vil_prediction.logit_fc.3.weight")
        ps.shadow_b[off + 5] = NAN
        before = ps.flat.clone()
        with pytest.raises(RuntimeError, match="Function 'vil_prediction.logit_fc: vb_gemm_bf16' returned nan values"):
            with warnings.catch_warnings():
                warnings.simplefilter("ignore")
                loss.backward()
                opt.step()
    torch.cuda.synchronize()
    assert torch.equal(ps.flat, before)
    assert torch.isnan(ps.grad).any()          # the flat buffer keeps what the backward wrote


def test_nan_root_gradient_on_a_packed_task_step_names_the_objective():
    from vilbert_b200.tasks import ForwardModelsTrain, LoadLosses
    model, cfgj = _model()
    model.train()
    model.engine.pack_padding = True
    batch = T.make_batch(cfgj, "TASK1", 4, 11, 9)
    losses = LoadLosses(None, T.TASK_CFG, ["1"])
    with torch.autograd.set_detect_anomaly(True):
        loss, _ = ForwardModelsTrain(None, T.TASK_CFG, torch.device("cuda"), "TASK1", {"TASK1": 0}, {}, {"TASK1": [batch]}, model, losses)
        assert model.engine.plans and any(p.packed and p.anomaly for p in model.engine.plans.values())
        _raises_at("vqa", lambda: torch.autograd.backward(loss, grad_tensors=torch.tensor(NAN, device="cuda")))


def test_nan_the_backward_never_reaches_does_not_raise():
    model, cfgj = _model()
    model.train()
    with torch.no_grad():
        model.vil_tri_prediction.weight[1, 3] = NAN
    inp = _inputs(cfgj)
    with torch.autograd.set_detect_anomaly(True):
        out = model(**inp)
        assert torch.isnan(out[4]).any()
        out[0].float().square().mean().backward()
    assert torch.isfinite(model.engine.ps.grad).all()


def test_nan_in_the_forward_is_reported_at_the_objective():
    model, cfgj = _model("BertForMultiModalPreTraining")
    model.train()
    B, Nv, Nt = 4, 11, 9
    inp = _inputs(cfgj, B, Nv, Nt)
    inp["input_imgs"][1, 3, 7] = NAN
    labels = torch.full((B, Nt), -1, dtype=torch.long, device="cuda")
    labels[:, 2] = 5
    image_label = torch.zeros(B, Nv - 1, dtype=torch.long, device="cuda")
    image_label[:, 2] = 1
    target = torch.softmax(torch.randn(B, Nv - 1, cfgj["v_target_size"], device="cuda"), -1)
    with torch.autograd.set_detect_anomaly(True):
        losses = model(inp["input_txt"], inp["input_imgs"], inp["image_loc"], inp["token_type_ids"], inp["attention_mask"],
                       inp["image_attention_mask"], masked_lm_labels=labels, image_label=image_label, image_target=target,
                       next_sentence_label=torch.tensor([0, 1, 0, 1], device="cuda"))
        _raises_at("pretraining", lambda: (losses[0] + losses[1] + losses[2]).backward())


# ------------------------------------------------------------------------------------------ the report against an eager replay
def _view(alloc, ptr, rows, cols, ld, dt):
    """The region as a strided tensor view of the plan allocation that holds it."""
    from vilbert_b200 import _lib as L
    dtype = {L.VB_NAN_F32: torch.float32, L.VB_NAN_F16: torch.float16, L.VB_NAN_BF16: torch.bfloat16}[dt]
    t = next(t for t in alloc if t.untyped_storage().data_ptr() <= ptr < t.untyped_storage().data_ptr() + t.untyped_storage().nbytes())
    s = t.untyped_storage()
    base = torch.empty(0, dtype=dtype, device="cuda").set_(s, 0, (s.nbytes() // dtype.itemsize,))
    off = (ptr - s.data_ptr()) // dtype.itemsize
    return base.as_strided((rows, cols), (ld, 1), off)


@pytest.mark.parametrize("precision", ["bf16", "fp16"])
def test_overflowing_gradients_report_the_first_op_an_eager_replay_finds(precision):
    """Output gradients scaled until the bf16 gradients overflow: the backward list replayed one op at a time, each op's declared
    outputs inspected with torch.isnan right after it ran; the first op holding a NaN is the one the checks report."""
    import sys
    sys.path.insert(0, os.path.join(ROOT, "tools"))
    import plan_dump as PD
    from vilbert_b200 import engine as E
    from vilbert_b200.config import BertConfig
    eng = E.Engine(BertConfig.from_dict(TINY), torch.device("cuda"), precision=precision, wgrad_streams=False)
    g = torch.Generator(device="cuda").manual_seed(0)
    eng.ps.flat.normal_(0, 0.02, generator=g)
    eng.refresh_weights()
    plan = eng.plan(4, 9, 11, grad_outputs=("vil_prediction",), train=True, anomaly=True)
    inp = O.synth_inputs(O.make_config(TINY), 4, 11, 9, seed=1)
    plan.load_inputs(*(inp[k] for k in ("input_txt", "input_imgs", "image_loc", "token_type_ids", "attention_mask", "image_attention_mask")))
    plan.gout["vil_prediction"].copy_(torch.randn(plan.gout["vil_prediction"].shape, generator=g, device="cuda") * 3e38)
    eng.zero_grad(force=True)
    plan.run_forward()
    allocs = [t for t in (eng.ps.grad, eng.arena) if t is not None] + [t for t in plan._keep if torch.is_tensor(t)]
    by_op = {}
    for r, reg in zip(plan.nan_records, sorted(plan.nan_regions, key=lambda x: x[5])):
        by_op.setdefault(r.op, []).append((r, reg))
    first = None
    for i, op in enumerate(plan.bwd):
        plan._run([op])
        if first is None and op[0] is not None and i in by_op:
            torch.cuda.synchronize()
            for r, (ptr, rows, cols, ld, dt, rid) in by_op[i]:
                if torch.isnan(_view(allocs, ptr, rows, cols, ld, dt)).any():
                    first = r
                    break
    torch.cuda.synchronize()
    assert first is not None, "the scaled gradients made no NaN: scale them further"
    rep = plan.anomaly_report()
    assert rep is not None and (rep.op, rep.entry, rep.module) == (first.op, first.entry, first.module), (rep, first)
    assert rep.region <= first.region
