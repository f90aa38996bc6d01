"""vilbert_b200.tasks on the GPU: the fused task-objective kernels against torch, and ForwardModelsTrain / ForwardModelsVal against
the module surface with the objective and score formed as the reference forms them (tests/_task_oracle.py)."""
import ctypes as C
import json
import os

import pytest
import torch

import _task_oracle as T
from oracle import vilbert_oracle as O

pytestmark = pytest.mark.gpu
S = lambda: C.c_void_p(torch.cuda.current_stream().cuda_stream)

TASK_CFG = T.TASK_CFG


def _kind(task_id):
    return T.kind_of(task_id)


def _model(golden_dir, **over):
    import vilbert_b200
    cfgj = dict(json.load(open(os.path.join(golden_dir, "tiny_b4.json")))["config"], task_specific_tokens=True, max_position_embeddings=300, **over)
    model = vilbert_b200.VILBertForVLTasks(vilbert_b200.BertConfig.from_dict(cfgj))
    model.load_state_dict(O.synth_params(O.make_config(cfgj), seed=0, device="cuda"), strict=False)
    return model, cfgj


def _batch(*a, **k):
    return T.make_batch(*a, **k)


def _grads_close(a, b, entries, ps_grad):
    from _gpu_util import rel_l2
    gmax = max(b[k].abs().max().item() for k in entries)
    l2 = sorted(rel_l2(a[k], b[k]) for k in entries if b[k].abs().max().item() > 1e-3 * gmax)
    assert l2 and l2[-1] < 2e-2 and l2[len(l2) // 2] < 1e-2, l2[-3:]


def _train(model, task_id, batch, step=7):
    from vilbert_b200.tasks import ForwardModelsTrain, LoadLosses
    model.engine.set_dropout_step(step)
    losses = LoadLosses(None, TASK_CFG, [task_id[4:]])
    return ForwardModelsTrain(None, TASK_CFG, torch.device("cuda"), task_id, {task_id: 0}, {}, {task_id: [batch]}, model, losses)


def _reference(model, task_id, batch, step=7):
    model.engine.set_dropout_step(step)
    dev = tuple(t.cuda() for t in batch)
    return T.reference_step(_kind(task_id), TASK_CFG[task_id]["process"], task_id, dev, model)


def _snapshot(model):
    eng = model.engine
    return {k: eng.ps.g(k).clone() for k in eng.ps.entries}


# ------------------------------------------------------------------------------------------ kernels
@pytest.mark.parametrize("rows,C,width,masked", [(1, 4, 110, False), (5, 4, 200, False), (3, 204, 306, False), (2, 204, 306, True), (7, 2, 2, False),
                                                 (6, 3, 3, False)])
def test_bce_gather_loss_kernel(rows, C, width, masked):
    from vilbert_b200 import _lib as L
    off = 0 if width == C else T.MC_OFFSET
    x = torch.randn(rows, width, device="cuda") * 3
    if width > 30:
        x[:, width - 30:] = -10000.0
    ids = None
    if off:
        ids = torch.randint(0, width - off, (rows, C), device="cuda")
        ids[:, C // 2:] = width - off - 1                     # padded duplicates
        if masked:
            ids[:] = torch.randint(width - 30 - off, width - off, (rows, C), device="cuda")
    t = torch.rand(rows, C, device="cuda")
    if off:
        t = t.round() * ((ids + off) < width - 30)
    mul = float(C) if off else 1.0
    loss, row_loss = torch.full((1,), 5.0, device="cuda"), torch.empty(rows, device="cuda")
    d32 = torch.full((rows, width), float("nan"), device="cuda")
    d16 = torch.full((rows, width + 8), float("nan"), device="cuda", dtype=torch.bfloat16)
    lib = L.lib()
    for acc in (0, 1):
        L.check(lib.vb_bce_gather_loss(x.data_ptr(), width, off, width, None if ids is None else ids.data_ptr(), t.data_ptr(), rows, C, mul,
                                       row_loss.data_ptr(), loss.data_ptr(), acc, d32.data_ptr(), width, d16.data_ptr(), width + 8, S()))
    ref_loss, ref_d = T.bce_gather_closed_form(x.cpu(), off, None if ids is None else ids.cpu(), t.cpu(), mul)
    got = loss.item() / 2                                      # set, then accumulated once more
    assert abs(got - ref_loss.item()) <= 1e-5 * max(abs(ref_loss.item()), 1e-6)
    assert torch.allclose(d32.cpu().double(), ref_d, rtol=1e-4, atol=1e-7)
    assert torch.equal(d16[:, :width], d32.to(torch.bfloat16))
    if masked:
        assert d32.abs().max().item() == 0 and torch.isfinite(loss).all()
    # the gradient does not depend on how duplicates are scheduled: a second launch is bitwise identical
    again = torch.empty_like(d32)
    L.check(lib.vb_bce_gather_loss(x.data_ptr(), width, off, width, None if ids is None else ids.data_ptr(), t.data_ptr(), rows, C, mul,
                                   row_loss.data_ptr(), loss.data_ptr(), 0, again.data_ptr(), width, None, 0, S()))
    assert torch.equal(again, d32)
    if off:
        bad = ids.clone(); bad[0, 0] = width - off
        L.check(lib.vb_bce_gather_loss(x.data_ptr(), width, off, width, bad.data_ptr(), t.data_ptr(), rows, C, mul, row_loss.data_ptr(),
                                       loss.data_ptr(), 0, again.data_ptr(), width, None, 0, S()))
        assert torch.isnan(loss).all()


def test_task_score_kernel_modes():
    from vilbert_b200 import _lib as L
    lib, nan = L.lib(), float("nan")
    rows, cols = 40, 7
    x = torch.randn(rows, cols, device="cuda").round()        # many ties
    x[0] = -10000.0
    x[1, 2], x[1, 5] = nan, nan
    x[2, 0] = nan
    tgt = torch.rand(rows, cols, device="cuda").round(decimals=1)
    labels = torch.randint(0, cols, (rows,), device="cuda")
    pick = torch.max(x, 1)[1]
    want = {L.VB_SCORE_SOFT: tgt[torch.arange(rows), pick].double().sum().item(), L.VB_SCORE_LABEL: (pick == labels).sum().item(),
            L.VB_SCORE_THRESHOLD: (tgt[torch.arange(rows), pick] > 0.5).sum().item()}
    score, preds = torch.zeros(1, device="cuda"), torch.empty(rows, dtype=torch.int64, device="cuda")
    for mode, w in want.items():
        L.check(lib.vb_task_score(mode, x.data_ptr(), cols, 0, cols, None, 0, tgt.data_ptr(), cols, labels.data_ptr(), rows, score.data_ptr(), 0,
                                  preds.data_ptr(), S()))
        assert torch.equal(preds, pick) and abs(score.item() - w) <= 1e-6 * max(1.0, w), mode
    # V-logit-mc at the GuessWhat shape: gathered logits with padded duplicates (ties at -10000), targets tied at 0
    Nv, Cc, B = 306, 204, 8
    v = torch.randn(B, Nv, device="cuda")
    v[:, 290:] = -10000.0
    ids = torch.randint(0, 204, (B, Cc), device="cuda")
    ids[:, 20:] = 204
    ids[3, :] = 204                                            # every choice masked: ties everywhere
    t = torch.zeros(B, Cc, device="cuda")
    t[:6, 5] = 1.0
    g = v[:, 101:].gather(1, ids)
    want_mc = (torch.max(g, 1)[1] == torch.max(t, 1)[1]).sum().item()
    L.check(lib.vb_task_score(L.VB_SCORE_CHOICE, v.data_ptr(), Nv, 101, Cc, ids.data_ptr(), Nv, t.data_ptr(), Cc, None, B, score.data_ptr(), 0,
                              preds.data_ptr(), S()))
    assert score.item() == want_mc and torch.equal(preds[:B], torch.max(g, 1)[1])
    L.check(lib.vb_task_score(L.VB_SCORE_CHOICE, v.data_ptr(), Nv, 101, Cc, ids.data_ptr(), Nv, t.data_ptr(), Cc, None, B, score.data_ptr(), 1,
                              None, S()))
    assert score.item() == 2 * want_mc


def test_scale_by_device_kernel():
    from vilbert_b200 import _lib as L
    src, dst, s = torch.randn(1000, device="cuda"), torch.empty(1000, device="cuda"), torch.tensor([2.0 / 3.0], device="cuda")
    L.check(L.lib().vb_scale_by_device(src.data_ptr(), dst.data_ptr(), 1000, s.data_ptr(), S()))
    assert torch.equal(dst, src * s)


# ------------------------------------------------------------------------------------------ ForwardModelsTrain / Val
CASES = [("TASK1", 4, 11, 9), ("TASK15", 4, 11, 9), ("TASK5", 2, 11, 9), ("TASK7", 2, 11, 9), ("TASK3", 2, 11, 7), ("TASK9", 4, 11, 9),
         ("TASK4", 4, 110, 9), ("TASK12", 2, 11, 9), ("TASK13", 3, 11, 9)]


@pytest.mark.parametrize("task_id,B,Nv,Nt", CASES)
def test_forward_models_train_matches_module_surface(golden_dir, task_id, B, Nv, Nt):
    """Same parameters, batch and dropout step: loss (1e-5), score (the same argmax of the same head logits) and every parameter
    gradient against VILBertForVLTasks.forward + the reference's torch objective, in train mode."""
    model, cfgj = _model(golden_dir)
    model.train()
    batch = _batch(cfgj, task_id, B, Nv, Nt)
    model.zero_grad()
    ref_loss, ref_score, bs = _reference(model, task_id, batch)
    ref_loss.backward()
    ref_g = _snapshot(model)
    model.zero_grad()
    loss, score = _train(model, task_id, batch)
    assert loss.dim() == 0 and loss.is_cuda and loss.requires_grad and score.dim() == 0 and score.is_cuda
    loss.backward()
    g = _snapshot(model)
    assert abs(loss.item() - ref_loss.item()) <= 1e-5 * abs(ref_loss.item()), (loss.item(), ref_loss.item())
    assert abs(score.item() * bs - ref_score.item()) <= 1e-6 * max(1.0, ref_score.item()), (score.item() * bs, ref_score.item())
    _grads_close(g, ref_g, list(model.engine.ps.entries), None)


@pytest.mark.parametrize("task_id,B,Nv,Nt,C", [("TASK4", 32, 200, 21, 4), ("TASK17", 8, 306, 257, 204)])
def test_vlogit_mc_at_twelve_in_one_shapes(golden_dir, task_id, B, Nv, Nt, C):
    """Visual7w (T4) and GuessWhatPointing (T17, 204 choices padded with region 204) at their 12-in-1 shapes."""
    model, cfgj = _model(golden_dir)
    model.train()
    batch = _batch(cfgj, task_id, B, Nv, Nt, C=C)
    model.zero_grad()
    ref_loss, ref_score, bs = _reference(model, task_id, batch)
    ref_loss.backward()
    ref_g = _snapshot(model)
    model.zero_grad()
    loss, score = _train(model, task_id, batch)
    loss.backward()
    assert abs(loss.item() - ref_loss.item()) <= 1e-5 * abs(ref_loss.item())
    assert score.item() * bs == ref_score.item()
    _grads_close(_snapshot(model), ref_g, list(model.engine.ps.entries), None)


def test_loss_scale_stays_on_the_device(golden_dir):
    """(loss * loss_scale / accumulation).backward(): d(total)/d(loss) reaches the plan as a device scalar that scales the head
    gradient before the backward. A power of two scales every gradient exactly (up to split-K atomics); 2/3 changes the rounding of
    the bf16 gradient operands exactly as it does on the module surface, which the fused path matches."""
    model, cfgj = _model(golden_dir)
    model.train()
    batch = _batch(cfgj, "TASK1", 4, 11, 9)

    def grads(scale, fused=True):
        model.zero_grad()
        loss = _train(model, "TASK1", batch)[0] if fused else _reference(model, "TASK1", batch)[0]
        (loss * scale).backward()
        return model.engine.ps.grad.clone()
    g1 = grads(1.0)
    rel = lambda a, b: ((a - b).norm() / b.norm()).item()
    assert rel(grads(0.5), g1 * 0.5) < 1e-5
    g23 = grads(2 / 3)
    assert rel(g23, g1 * (2 / 3)) < 3e-3                          # bf16 rounding of the scaled gradient operands
    assert rel(g23, grads(2 / 3, fused=False)) < 1e-3               # same, up to which bf16 roundings the fp32 scaling flips


def test_graph_replay_matches_eager(golden_dir):
    """The task plan's passes are captured into CUDA graphs after two eager runs; replays reproduce the eager step."""
    model, cfgj = _model(golden_dir)
    model.train()
    batch = _batch(cfgj, "TASK4", 4, 110, 9)
    res = []
    for _ in range(4):
        model.zero_grad()
        loss, score = _train(model, "TASK4", batch)
        loss.backward()
        res.append((loss.item(), score.item(), model.engine.ps.grad.clone()))
    plan = model._last_plan
    assert plan.graph_fwd is not None and plan.graph_bwd is not None
    (l0, s0, g0), (l3, s3, g3) = res[0], res[3]
    assert l0 == l3 and s0 == s3
    assert ((g3 - g0).abs().max() / g0.abs().max()).item() < 1e-5      # split-K atomics: last-bit order effects only


@pytest.mark.parametrize("task_id", ["TASK1", "TASK7", "TASK9", "TASK4", "TASK12", "TASK13"])
def test_forward_models_val_matches_module_surface(golden_dir, task_id):
    from vilbert_b200.tasks import ForwardModelsVal, LoadLosses
    model, cfgj = _model(golden_dir)
    model.eval()
    Nv = 110 if task_id == "TASK4" else 11
    batch = _batch(cfgj, task_id, 4, Nv, 9)
    with torch.no_grad():
        ref_loss, ref_score, bs = _reference(model, task_id, batch)
    loss, score, n = ForwardModelsVal(None, TASK_CFG, torch.device("cuda"), task_id, batch, model, LoadLosses(None, TASK_CFG, [task_id[4:]]))
    assert isinstance(loss, float) and isinstance(score, float) and n == bs
    assert abs(loss - ref_loss.item()) <= 1e-5 * abs(ref_loss.item()) and abs(score - float(ref_score)) <= 1e-6 * max(1.0, float(ref_score))


@pytest.mark.parametrize("B", [4, 3])
def test_foil_raises_like_the_reference(golden_dir, B):
    """Foil (TASK16, CrossEntropyLoss on int labels): with an even batch the binary head pairs samples and the CE refuses the
    labels (ValueError); with an odd one the head is per sample and compute_score_with_logits raises (IndexError). Both paths
    raise the same error."""
    from vilbert_b200.tasks import ForwardModelsVal, LoadLosses
    model, cfgj = _model(golden_dir)
    batch = _batch(cfgj, "TASK16", B, 11, 9)
    with pytest.raises((ValueError, IndexError)) as ref:
        _reference(model, "TASK16", batch)
    with pytest.raises(ref.type):
        _train(model, "TASK16", batch)
    with pytest.raises(ref.type):
        ForwardModelsVal(None, TASK_CFG, torch.device("cuda"), "TASK16", batch, model, LoadLosses(None, TASK_CFG, ["16"]))


def test_twelve_in_one_iteration_with_fused_adamw_and_arena(golden_dir):
    """One 12-in-1 iteration (train_tasks.py:520-551): every task through ForwardModelsTrain, loss * loss_scale backward, one
    FusedAdamW step, with the plans sharing one activation arena."""
    import vilbert_b200
    from vilbert_b200.optim import FusedAdamW
    cfgj = dict(json.load(open(os.path.join(golden_dir, "tiny_b4.json")))["config"], task_specific_tokens=True, max_position_embeddings=300)
    model = vilbert_b200.VILBertForVLTasks(vilbert_b200.BertConfig.from_dict(cfgj))
    model.engine.enable_activation_arena(1 << 30)
    model.train()
    opt = FusedAdamW(list(model.parameters()), lr=4e-5, correct_bias=False, model=model)
    shapes = [("TASK1", 16, 101, 23), ("TASK4", 32, 200, 20), ("TASK7", 8, 101, 30), ("TASK9", 32, 101, 20), ("TASK12", 16, 101, 40),
              ("TASK13", 32, 101, 56), ("TASK15", 16, 101, 26), ("TASK17", 8, 306, 256)]
    scale = {"TASK1": 2.0, "TASK15": 2.0}
    out = []
    for it in range(2):
        for task_id, B, Nv, Nt in shapes:
            loss, score = _train(model, task_id, _batch(cfgj, task_id, B, Nv, Nt, C=204 if task_id == "TASK17" else 4, seed=it), step=100 * it)
            (loss * scale.get(task_id, 1.0)).backward()
            out.append((loss, score))
        opt.step()
        model.zero_grad()
    vals = torch.stack([torch.stack([l.detach(), s]) for l, s in out]).cpu()
    assert torch.isfinite(vals).all(), vals
    assert torch.isfinite(model.engine.ps.flat).all()
