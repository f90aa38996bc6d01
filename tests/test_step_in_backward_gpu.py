"""The step in the backward (FusedAdamW / FusedRAdam.step_in_backward) on the GPU.

Kernels: vb_adamw_step_capped and vb_radam_step_capped over the per-bucket chunk tables of the bert_base_6layer_6conect layout, at
several CTA caps, give bitwise the weights, moments, 16-bit copies, zeroed gradient and step counter of one vb_adamw_step /
vb_radam_step over the whole table.

Module surface: under torch.use_deterministic_algorithms(True), N steps with the context equal N steps of backward + step() from
the same parameters, batches and dropout steps bit for bit (flat weights, both moments, every 16-bit copy, the gradient buffer, the
device counter, state_dict steps and the losses), eager and graph-captured pieces: two alternating ForwardModelsTrain tasks in train
mode, the fused pre-training step, FusedRAdam across its rectification switch at t = 6, an lr changed partway, gradient
accumulation, a text stream frozen partway, a packed step, and data parallelism (delay_allreduce=False and True) with a stand-in
reducer of a world of two on one GPU, and config-2 shape on bert_base_6layer_6conect. Without determinism, at config-2 shape, each
step from the same state: the backward's gradient to the last bits of its atomics, and the step bitwise the plain launch over it.
A two-rank NCCL run follows when two GPUs are visible."""
import ctypes as C
import json
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

import _task_oracle as T
from oracle import vilbert_oracle as O

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda")
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BASE66 = os.path.join(ROOT, "vilbert-multi-task_b200", "configs", "bert_base_6layer_6conect.json")


# ============================================================================================ kernels
@pytest.mark.parametrize("kind", ["adamw", "radam"])
def test_capped_entry_points_equal_the_plain_step(kind):
    from vilbert_b200 import _lib as L
    from vilbert_b200.config import BertConfig
    from vilbert_b200.ddp import FlatGradAllReducer, trainable_ranges
    from vilbert_b200.engine import Engine
    from vilbert_b200.optim import _GROUP_DT, bucket_chunks, build_chunks, group_row
    lib = L.lib()
    eng = Engine(BertConfig.from_dict(json.load(open(BASE66))), "cpu", _build_only=True)
    ps = eng.ps
    names = list(ps.entries)
    ranges = [(ps.span(n)[0], ps.span(n)[1], i % 4) for i, n in enumerate(names)]
    red = FlatGradAllReducer(ps.grad, n_buckets=8)
    red.set_ranges(trainable_ranges(ps, frozenset()))
    N = ps.numel
    del eng, ps
    groups = [group_row(lr, (b1, b2), eps, wd, cb) for lr, b1, b2, eps, wd, cb in
              ((1e-3, 0.9, 0.999, 1e-6, 0.01, 1), (2e-4, 0.8, 0.99, 1e-8, 0.0, 0), (5e-4, 0.9, 0.98, 1e-6, 0.1, 1), (1e-4, 0.95, 0.999, 1e-7, 0.0, 0))]
    gtab = torch.from_numpy(np.array(groups, dtype=_GROUP_DT).view(np.uint8).copy()).to(DEV)
    gen = torch.Generator(device=DEV).manual_seed(1)
    init = dict(p=torch.randn(N, generator=gen, device=DEV) * 0.05, g=torch.randn(N, generator=gen, device=DEV) * 1e-2,
                m=torch.randn(N, generator=gen, device=DEV) * 1e-3, v=torch.rand(N, generator=gen, device=DEV) * 1e-5)

    def state():
        s = {k: x.clone() for k, x in init.items()}
        s.update(hi=torch.full((N,), 0x5A5A, dtype=torch.int16, device=DEV), lo=torch.full((N,), 0x5A5A, dtype=torch.int16, device=DEV),
                 b=torch.full((N,), 0x5A5A, dtype=torch.int16, device=DEV), step=torch.full((1,), 5, dtype=torch.int32, device=DEV))
        return s

    def launch(fn, s, tab, extra):
        st, cn, gr = (torch.from_numpy(x).to(DEV) for x in tab)
        args = (s["p"], s["g"], s["m"], s["v"], s["hi"], s["lo"], s["b"], 1, st, cn, gr, len(tab[0]), gtab)
        L.call(fn, *args, *extra)

    def tail(s, advance, cap=None):
        if kind == "adamw":
            return (s["step"], C.c_float(0.5), 1) + (() if cap is None else (cap,))
        return (1, s["step"], advance, C.c_float(0.5), 1) + (() if cap is None else (cap,))
    plain, capped = (lib.vb_adamw_step, lib.vb_adamw_step_capped) if kind == "adamw" else (lib.vb_radam_step, lib.vb_radam_step_capped)
    ref = state()
    if kind == "adamw":
        ref["step"] += 1
    launch(plain, ref, build_chunks(ranges), tail(ref, 1))
    subs = bucket_chunks(ranges, red.table)
    assert len(subs) >= 8
    for caps in ((1,), (7, 132, 0, 1056), (66,)):
        got = state()
        if kind == "adamw":
            got["step"] += 1
        for k, tab in enumerate(subs):
            launch(capped, got, tab, tail(got, 1 if k == 0 else 0, caps[k % len(caps)]))
        torch.cuda.synchronize()
        for key in ref:
            assert torch.equal(ref[key], got[key]), (kind, caps, key)
    assert int(ref["step"].item()) == 6
    assert torch.count_nonzero(ref["g"][torch.from_numpy(_mask(ranges, N)).to(DEV)]) == 0
    with pytest.raises(L.VBError, match="max_ctas"):
        got = state()
        launch(capped, got, subs[0], tail(got, 1, -1))
    assert int(got["step"].item()) == 5          # a refused call moves no counter


def _mask(ranges, N):
    m = np.zeros(N, bool)
    for off, n, _ in ranges:
        m[off:off + n] = True
    return m


# ============================================================================================ module surface
def _tiny(golden_dir, **over):
    return dict(json.load(open(os.path.join(golden_dir, "tiny_b4.json")))["config"], **over)


def _vqa_model(cfgj, params):
    import vilbert_b200
    m = vilbert_b200.VILBertForVLTasks(vilbert_b200.BertConfig.from_dict(cfgj))
    m.load_state_dict(params, strict=False)
    m.train()
    return m


def _snapshot(model, opt, losses):
    ps = model.engine.ps
    out = dict(flat=ps.flat, grad=ps.grad, shadow=ps.shadow, shadow_b=ps.shadow_b, exp_avg=opt.exp_avg, exp_avg_sq=opt.exp_avg_sq,
               step_dev=opt._step_dev)
    if ps.shadow_lo is not None:
        out["shadow_lo"] = ps.shadow_lo
    out = {k: v.clone() for k, v in out.items()}
    out["losses"] = torch.stack([x.detach().reshape(()) for x in losses]).cpu()
    out["host_steps"] = (opt.step_count, sorted({s["step"] for s in opt.state_dict()["state"].values()}))
    return out


def _task_loss(model, cfgj, task_id, B, Nv, Nt, seed):
    from vilbert_b200.tasks import ForwardModelsTrain, LoadLosses
    batch = T.make_batch(cfgj, task_id, B, Nv, Nt, seed=seed)
    model.engine.set_dropout_step(1000 + 17 * seed)
    loss, _ = ForwardModelsTrain(None, T.TASK_CFG, DEV, task_id, {task_id: 0}, {}, {task_id: [batch]}, model,
                                 LoadLosses(None, T.TASK_CFG, [task_id[4:]]))
    return loss


def _run(model, opt, n, loss_fn, in_backward, accumulate=0, lr_change_at=None, freeze_at=None):
    """n optimizer steps: per step `accumulate` plain backwards, then one more backward with the step (the context) or followed
    by step(). -> losses."""
    losses = []
    for s in range(n):
        if lr_change_at == s:
            for g in opt.param_groups:
                g["lr"] *= 0.5
        if freeze_at == s:
            for name, p in model.named_parameters():
                if name.startswith(("bert.embeddings.", "bert.encoder.layer.")):
                    p.requires_grad_(False)
        for a in range(accumulate):
            loss = loss_fn(s, a)
            loss.backward()
            losses.append(loss)
        loss = loss_fn(s, accumulate)
        if in_backward:
            with opt.step_in_backward():
                loss.backward()
        else:
            loss.backward()
            opt.step()
        losses.append(loss)
    torch.cuda.synchronize()
    return losses


def _compare(a, b, exact=True):
    assert a.keys() == b.keys()
    for k in a:
        if k == "host_steps":
            assert a[k] == b[k], k
        elif exact:
            assert torch.equal(a[k], b[k]), k
    return True


@pytest.fixture
def deterministic():
    torch.use_deterministic_algorithms(True)
    try:
        yield
    finally:
        torch.use_deterministic_algorithms(False)


def _two_arms(make, n, loss_fn, **kw):
    """The same n steps with backward + step() and with the context, from the same parameters -> (snapshot, snapshot, models)."""
    out = []
    for in_backward in (False, True):
        model, opt = make()
        losses = _run(model, opt, n, lambda s, a: loss_fn(model, s, a), in_backward, **kw)
        out.append((_snapshot(model, opt, losses), model))
    return out[0][0], out[1][0], out[1][1]


VQA_SHAPES = {"TASK1": (8, 101, 23), "TASK15": (8, 101, 26)}


def _vqa_case(golden_dir, opt_cls="adamw", **okw):
    from vilbert_b200.optim import FusedAdamW, FusedRAdam
    cfgj = _tiny(golden_dir, task_specific_tokens=True, max_position_embeddings=300)
    params = O.synth_params(O.make_config(cfgj), seed=0, device="cuda")

    def make():
        m = _vqa_model(cfgj, params)
        cls = FusedAdamW if opt_cls == "adamw" else FusedRAdam
        kw = dict(lr=1e-3, model=m, **okw)
        if opt_cls == "adamw":
            kw.setdefault("correct_bias", True)
        return m, cls(list(m.parameters()), **kw)
    return cfgj, make


def test_deterministic_two_alternating_tasks_lr_change_and_graphs(golden_dir, deterministic):
    cfgj, make = _vqa_case(golden_dir, weight_decay=0.01)
    tasks = ("TASK1", "TASK15")

    def loss_fn(model, s, a):
        t = tasks[s % 2]
        return _task_loss(model, cfgj, t, *VQA_SHAPES[t], seed=s) * (2.0 if t == "TASK1" else 1.0)
    a, b, model = _two_arms(make, 8, loss_fn, lr_change_at=5)
    _compare(a, b)
    assert a["host_steps"] == (8, [8]) and int(b["step_dev"].item()) == 8
    assert torch.count_nonzero(b["grad"]) == 0
    assert any(p._piece_graphs for p in model.engine.plans.values()), "the pieces were never graph-captured"


def test_deterministic_radam_across_rectification(golden_dir, deterministic):
    cfgj, make = _vqa_case(golden_dir, "radam", weight_decay=0.01)
    a, b, _ = _two_arms(make, 8, lambda m, s, a_: _task_loss(m, cfgj, "TASK1", *VQA_SHAPES["TASK1"], seed=s))
    _compare(a, b)


def test_deterministic_accumulation_and_freezing(golden_dir, deterministic):
    cfgj, make = _vqa_case(golden_dir)
    a, b, _ = _two_arms(make, 4, lambda m, s, k: _task_loss(m, cfgj, "TASK1", *VQA_SHAPES["TASK1"], seed=10 * s + k), accumulate=2)
    _compare(a, b)
    a, b, _ = _two_arms(make, 8, lambda m, s, k: _task_loss(m, cfgj, "TASK1", *VQA_SHAPES["TASK1"], seed=s), freeze_at=3)
    _compare(a, b)


def test_deterministic_packed_step(golden_dir, deterministic):
    cfgj, make = _vqa_case(golden_dir)

    def loss_fn(model, s, a):
        model.engine.pack_padding = True
        loss = _task_loss(model, cfgj, "TASK1", *VQA_SHAPES["TASK1"], seed=s)
        assert model._last_plan.packed is not None
        return loss
    a, b, _ = _two_arms(make, 8, loss_fn)
    _compare(a, b)


def _pretraining_args(pcfg, B, Nv, Nt, seed):
    inp = O.synth_inputs(pcfg, B, Nv, Nt, seed=seed, device=DEV)
    g = torch.Generator().manual_seed(seed)
    lm = torch.full((B, Nt), -1, dtype=torch.long)
    lm[torch.rand(B, Nt, generator=g) < 0.15] = 5
    lm[:, 1] = 7
    il = torch.full((B, Nv - 1), -1, dtype=torch.long)
    il[:, 0] = 1
    it = torch.softmax(torch.randn(B, Nv - 1, pcfg["v_target_size"], generator=g), -1)
    ns = torch.randint(0, 2, (B,), generator=g)
    args = [inp[k] for k in ("input_txt", "input_imgs", "image_loc", "token_type_ids", "attention_mask", "image_attention_mask")]
    return args + [x.to(DEV) for x in (lm, il, it, ns)]


def test_deterministic_pretraining_step(golden_dir, deterministic):
    import vilbert_b200
    from vilbert_b200.optim import FusedAdamW
    pj = _tiny(golden_dir)
    pcfg = O.make_config(pj)
    params = O.synth_params(pcfg, seed=4, device=DEV, with_task_heads=False)

    def make():
        m = vilbert_b200.BertForMultiModalPreTraining(vilbert_b200.BertConfig.from_dict(pj), fused_objective=True)
        m.load_state_dict(params, strict=False)
        m.train()
        return m, FusedAdamW(list(m.parameters()), lr=1e-3, model=m)

    def loss_fn(model, s, a):
        model.engine.set_dropout_step(500 + s)
        return sum(model(*_pretraining_args(pcfg, 4, 37, 12, seed=s))).sum()
    a, b, _ = _two_arms(make, 8, loss_fn)
    _compare(a, b)


@pytest.mark.parametrize("overlap", [True, False], ids=["delay_false", "delay_true"])
def test_deterministic_data_parallel_stand_in(golden_dir, deterministic, monkeypatch, overlap):
    """A stand-in reducer of a world of two doubles each bucket on the communication stream (test_ddp_overlap_gpu): the step of
    a bucket must see its doubled gradient, after the backward (delay_allreduce=True) or during it."""
    from test_ddp_overlap_gpu import _stub_class
    from vilbert_b200 import ddp
    monkeypatch.setattr(ddp, "FlatGradAllReducer", _stub_class())
    cfgj, make0 = _vqa_case(golden_dir)

    def make():
        m, o = make0()
        ddp.DistributedDataParallel(m, delay_allreduce=not overlap, n_buckets=8)
        return m, o
    a, b, model = _two_arms(make, 6, lambda m, s, k: _task_loss(m, cfgj, "TASK1", *VQA_SHAPES["TASK1"], seed=s))
    _compare(a, b)
    assert model._ddp_reducer.calls          # the stand-in exchanged


def _base66_vqa(cfgj, init, **okw):
    import vilbert_b200
    from vilbert_b200.optim import FusedAdamW
    m = vilbert_b200.VILBertForVLTasks(vilbert_b200.BertConfig.from_dict(cfgj))
    m.load_state_dict(init)
    m.train()
    return m, FusedAdamW(list(m.parameters()), correct_bias=False, model=m, **okw)


def test_deterministic_config2_shape(deterministic):
    """bert_base_6layer_6conect, VQA at B = 64, 101 regions x 36 tokens, train mode, under deterministic algorithms: three steps
    with the context equal three steps of backward + step() bit for bit (the second and third replay captured pieces)."""
    import vilbert_b200
    cfgj = dict(json.load(open(BASE66)), task_specific_tokens=True)
    init = {k: v.clone() for k, v in vilbert_b200.VILBertForVLTasks(vilbert_b200.BertConfig.from_dict(cfgj)).state_dict().items()}
    a, b, _ = _two_arms(lambda: _base66_vqa(cfgj, init, lr=1e-4), 3, lambda m, s, k: _task_loss(m, cfgj, "TASK1", 64, 101, 36, seed=s))
    _compare(a, b)


def test_default_mode_config2_shape():
    """The same shape on the default (atomics-ordered) path. Two runs of a backward there differ in the last bits of their
    gradients, and Adam turns such bits into different updates, so two training runs drift apart: the paths are compared step by
    step from the same state instead. Before each step the context's model takes the other's weights, moments and counter. Its
    backward must give the gradient the plain backward gives to the last bits of the atomics (max |difference| / max |g| < 1e-5,
    as tests/test_ddp_overlap_gpu.py holds the overlapped backward): a bucket stepped while a later backward op still read its
    weights would move that gradient by about lr / |w| = 5 %. Its step must be bitwise the plain launch over the gradient the
    backward left (the optimizer keeps the gradient: zero_grad=False), so no bucket was stepped before its gradient was final.
    Steps 3 and 4 replay captured pieces."""
    import vilbert_b200
    cfgj = dict(json.load(open(BASE66)), task_specific_tokens=True)
    init = {k: v.clone() for k, v in vilbert_b200.VILBertForVLTasks(vilbert_b200.BertConfig.from_dict(cfgj)).state_dict().items()}
    mA, oA = _base66_vqa(cfgj, init, lr=1e-3)
    mB, oB = _base66_vqa(cfgj, init, lr=1e-3, zero_grad=False)
    psA, psB = mA.engine.ps, mB.engine.ps
    for s in range(4):
        with torch.no_grad():
            psB.flat.copy_(psA.flat)
            oB.exp_avg.copy_(oA.exp_avg)
            oB.exp_avg_sq.copy_(oA.exp_avg_sq)
            oB._step_dev.copy_(oA._step_dev)
        mB.zero_grad()
        mB.engine.shadow_clean = False           # weights written by hand: refresh the 16-bit copies at the next forward
        pre = (psB.flat.clone(), oB.exp_avg.clone(), oB.exp_avg_sq.clone())
        lossA = _task_loss(mA, cfgj, "TASK1", 64, 101, 36, seed=s)
        lossA.backward()
        gA = psA.grad.clone()
        oA.step()
        lossB = _task_loss(mB, cfgj, "TASK1", 64, 101, 36, seed=s)
        with oB.step_in_backward():
            lossB.backward()
        assert oB._stepped, s
        torch.cuda.synchronize()
        gB = psB.grad.clone()
        post = [t.clone() for t in (psB.flat, oB.exp_avg, oB.exp_avg_sq, psB.shadow, psB.shadow_b)]
        assert torch.allclose(lossA.detach(), lossB.detach(), rtol=1e-5), s
        assert ((gA - gB).abs().max() / gA.abs().max()).item() < 1e-5, s
        with torch.no_grad():                    # the plain launch over the gradient the backward left, from the same state
            for t, x in zip((psB.flat, oB.exp_avg, oB.exp_avg_sq), pre):
                t.copy_(x)
        oB.launch()
        torch.cuda.synchronize()
        for i, (x, t) in enumerate(zip(post, (psB.flat, oB.exp_avg, oB.exp_avg_sq, psB.shadow, psB.shadow_b))):
            assert torch.equal(x, t), (s, i)
    assert oA.step_count == oB.step_count == 4 and torch.equal(oA._step_dev, oB._step_dev)
    assert any(p._piece_graphs for p in mB.engine.plans.values()), "the pieces were never graph-captured"


def test_two_ranks_nccl():
    if torch.cuda.device_count() < 2:
        pytest.skip("needs two GPUs")
    import tempfile
    out = os.path.join(tempfile.mkdtemp(), "res.json")
    subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nproc_per_node=2", "--master_port=29611",
                    os.path.join(ROOT, "tests", "_step_in_backward_ddp_worker.py"), out], check=True, cwd=ROOT, timeout=900)
    res = json.load(open(out))
    assert all(r["params_equal"] and r["ranks_equal"] for r in res), res
