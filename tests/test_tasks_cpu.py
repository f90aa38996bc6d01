"""Task objectives and scores of the 12-in-1 task table without a GPU: the restatement of task_utils.py against torch autograd and
torch.max, the reference quirks vilbert_b200.tasks reproduces, and the structure of the engine's task-objective plans."""
import json
import math
import os

import pytest
import torch
import torch.nn as nn

import _task_oracle as T
from oracle import vilbert_oracle as O

NT, NV = 9, 11


def _tiny(golden_dir, **over):
    return dict(json.load(open(os.path.join(golden_dir, "tiny_b4.json")))["config"], **over)


def _engine(golden_dir, precision="fp16", **over):
    from vilbert_b200.config import BertConfig
    from vilbert_b200.engine import Engine
    return Engine(BertConfig.from_dict(_tiny(golden_dir, **over)), "cpu", _build_only=True, precision=precision)


def _names(ops):
    return [fn.__name__ for fn, _, _ in ops if fn is not None]


@pytest.mark.parametrize("C,width", [(4, 110), (204, 306)])
def test_bce_gather_closed_form_matches_autograd_with_duplicates_and_masked_regions(C, width):
    """V-logit-mc (task_utils.py:352-360): GuessWhat pads its choices with id 204 (so one region repeats up to 204 times per row),
    masked regions carry about -10000. The closed form the kernel implements, in float64, equals autograd of the reference's
    gather + BCE + mean * C, masked choices give a finite loss and a zero gradient."""
    rows = 3
    x = torch.randn(rows, width, dtype=torch.float64) * 3
    x[:, width - 20:] = -10000.0                                      # masked regions (the mask term of vision_logit)
    ids = torch.randint(0, width - T.MC_OFFSET, (rows, C))
    ids[0, C // 2:] = width - T.MC_OFFSET - 1                        # padded duplicates of one (masked) region
    ids[1, :] = ids[1, 0]                                            # every choice the same region
    t = torch.rand(rows, C, dtype=torch.float64).round()
    t[(ids + T.MC_OFFSET) >= width - 20] = 0.0                      # padded regions have no overlap with the referred box
    xa = x.clone().requires_grad_(True)
    ref = T.bce(xa[:, T.MC_OFFSET:].gather(1, ids).unsqueeze(2), t.unsqueeze(2)) * C
    ref.backward()
    loss, d = T.bce_gather_closed_form(x, T.MC_OFFSET, ids, t, C)
    assert math.isfinite(loss.item()) and abs(loss.item() - ref.item()) <= 1e-12 * abs(ref.item())
    assert torch.allclose(d, xa.grad, rtol=1e-12, atol=1e-15)
    assert d[:, :T.MC_OFFSET].abs().max() == 0 and d[:, width - 20:].abs().max() == 0


def test_bce_gather_closed_form_soft_targets_and_out_of_range_ids():
    """binary / tri with BCEWithLogitLoss (NLVR2, SNLI-VE: soft float targets, loss.mean() without x C) is the same closed form with no
    gather; an id outside the regions poisons the loss with NaN instead of reading out of bounds."""
    x = torch.randn(5, 3, dtype=torch.float64)
    t = torch.rand(5, 3, dtype=torch.float64)
    xa = x.clone().requires_grad_(True)
    ref = T.bce(xa, t)
    ref.backward()
    loss, d = T.bce_gather_closed_form(x, 0, None, t, 1.0)
    assert abs(loss.item() - ref.item()) <= 1e-12 and torch.allclose(d, xa.grad, rtol=1e-12, atol=1e-15)
    ids = torch.tensor([[0, 1, 9, 2]])
    loss, d = T.bce_gather_closed_form(torch.randn(1, 110), T.MC_OFFSET, ids, torch.zeros(1, 4), 4)
    assert math.isnan(loss.item()) and torch.isfinite(d).all()


def test_argmax_rule_follows_torch_max():
    """The score kernel's argmax: torch.max(dim=1) returns the first index among ties and treats NaN as the maximum (first NaN)."""
    nan = float("nan")
    rows = torch.tensor([[1.0, 3.0, 3.0, 2.0], [nan, 5.0, nan, 1.0], [-1e4, -1e4, -1e4, -1e4], [1.0, nan, 9.0, nan], [0.0, -0.0, 0.0, 0.0],
                         [-math.inf, -math.inf, -5.0, -5.0]])
    rows = torch.cat([rows, torch.randn(50, 4).round()])
    want = torch.max(rows, 1)[1]
    assert [T.argmax_torch_rule(r) for r in rows] == want.tolist()
    # V-logit-mc's target argmax over a padded GuessWhat row: ties at 0 pick the first choice
    assert T.argmax_torch_rule(torch.zeros(204)) == torch.max(torch.zeros(1, 204, 1), 1)[1].item() == 0


def test_foil_score_raises_in_the_reference_form():
    """Foil (TASK16: VL-binary-classifier, CrossEntropyLoss) has 1-D int labels: compute_score_with_logits scatters along dim 1 of a
    1-D one-hot and raises. The fused path reproduces the failure instead of inventing an accuracy."""
    logits, labels = torch.randn(4, 2), torch.tensor([0, 1, 1, 0])
    with pytest.raises(IndexError):
        T.score_with_logits(logits, labels)
    heads = [None, None, None, logits, torch.randn(4, 3), None, None, None, None]
    with pytest.raises(IndexError):
        T.objective("binary_ce", heads, labels)
    # the soft-target form is well defined: the label mass at the argmax
    soft = torch.tensor([[0.2, 0.8], [1.0, 0.0], [0.5, 0.5], [0.0, 1.0]])
    pick = torch.max(logits, 1)[1]
    assert T.score_with_logits(logits, soft).sum().item() == pytest.approx(soft[torch.arange(4), pick].sum().item())


def test_task_table_maps_every_type_and_loss():
    """vilbert_tasks.yml (type, loss) -> fused objective kind; the NLVR2 / SNLI-VE rows declare BCEWithLogitLoss on soft targets."""
    from vilbert_b200.tasks import TASK_KINDS, task_kind
    table = {"TASK1": ("VL-classifier", "BCEWithLogitLoss", "vqa"), "TASK3": ("VL-logit", "CrossEntropyLoss", "logit_ce"),
             "TASK4": ("V-logit-mc", "BCEWithLogitLoss", "vlogit_mc"), "TASK9": ("V-logit", "BCEWithLogitLoss", "vlogit_bce"),
             "TASK12": ("VL-binary-classifier", "BCEWithLogitLoss", "binary_bce"), "TASK13": ("VL-tri-classifier", "BCEWithLogitLoss", "tri_bce"),
             "TASK15": ("VL-classifier-GQA", "BCEWithLogitLoss", "gqa"), "TASK16": ("VL-binary-classifier", "CrossEntropyLoss", "binary_ce"),
             "TASK17": ("V-logit-mc", "BCEWithLogitLoss", "vlogit_mc")}
    cfg = {k: {"type": ty, "loss": lo} for k, (ty, lo, _) in table.items()}
    for k, (_, _, kind) in table.items():
        assert task_kind(cfg, k) == kind
    assert len(TASK_KINDS) == 9
    with pytest.raises(NotImplementedError):
        task_kind({"TASK0": {"type": "V-logit", "loss": "CrossEntropyLoss"}}, "TASK0")


def test_task_losses_must_be_the_ones_load_losses_builds():
    from vilbert_b200.tasks import LoadLosses, _check_loss
    cfg = {"TASK1": {"type": "VL-classifier", "loss": "BCEWithLogitLoss"}, "TASK7": {"type": "VL-logit", "loss": "CrossEntropyLoss"}}
    losses = LoadLosses(None, cfg, ["1", "7"])
    for k in cfg:
        _check_loss(cfg, k, losses)
    for bad in (nn.BCEWithLogitsLoss(reduction="sum"), nn.BCEWithLogitsLoss(pos_weight=torch.ones(3)), nn.MSELoss(), None):
        with pytest.raises(NotImplementedError):
            _check_loss(cfg, "TASK1", {"TASK1": bad})
    with pytest.raises(NotImplementedError):
        _check_loss(cfg, "TASK7", {"TASK7": nn.CrossEntropyLoss(label_smoothing=0.1)})


@pytest.mark.parametrize("kind,choices,Nv", [("vqa", None, NV), ("gqa", None, NV), ("logit_ce", 2, NV), ("vlogit_bce", None, NV),
                                              ("vlogit_mc", 4, 110), ("binary_bce", None, NV), ("tri_bce", None, NV)])
def test_task_plan_structure(golden_dir, kind, choices, Nv):
    """loss_in_forward + score: the objective and the score are the last kernels of the forward, the backward starts by scaling the
    stored head gradient by the device scalar loss_grad into the head's gradient buffer; a forward-only plan has both kernels too."""
    from vilbert_b200.engine import LOSS_HEADS
    eng = _engine(golden_dir)
    plan = eng.plan(4, NT, Nv, grad_outputs=LOSS_HEADS[kind], train=True, loss=kind, choices=choices, score=True, loss_in_forward=True)
    f, b = _names(plan.fwd), _names(plan.bwd)
    loss_fn = {"vqa": "vb_bce_logits_loss", "gqa": "vb_bce_logits_loss", "vlogit_bce": "vb_bce_logits_loss", "logit_ce": "vb_ce_loss"}.get(kind, "vb_bce_gather_loss")
    assert f[-2:] == [loss_fn, "vb_task_score"] and b[0] == "vb_scale_by_device"
    assert loss_fn not in b and "vb_task_score" not in b
    assert plan.loss.data_ptr() + 4 == plan.score.data_ptr()          # one device-to-host copy reads both
    assert plan.loss_grad.item() == 1.0 and plan.preds.dtype == torch.int64
    head = LOSS_HEADS[kind][0]
    scale = [op for op in plan.bwd if op[0] is not None][0]
    assert scale[1].dst == plan.gout[head].data_ptr() and scale[1].src == plan.head_grad[head].data_ptr()
    ev = eng.plan(4, NT, Nv, loss=kind, choices=choices, score=True, loss_in_forward=True)
    assert ev is not plan and _names(ev.fwd)[-2:] == [loss_fn, "vb_task_score"] and _names(ev.bwd) == []
    if kind == "vlogit_mc":
        assert set(plan.loss_inputs) == {"multiple_choice_ids", "target"} and tuple(plan.loss_inputs["target"].shape) == (4, choices)
        assert eng.plan(4, NT, Nv, grad_outputs=LOSS_HEADS[kind], train=True, loss=kind, choices=choices + 1, score=True,
                        loss_in_forward=True) is not plan          # C is part of the plan key
    with pytest.raises(ValueError):
        eng.plan(4, NT, Nv, loss="pretraining", score=True, loss_in_forward=True)


def test_task_plans_with_task_tokens_and_arena(golden_dir):
    from vilbert_b200.engine import LOSS_HEADS
    eng = _engine(golden_dir, task_specific_tokens=True)
    eng.enable_activation_arena(64 << 20)
    p = eng.plan(4, NT, 110, grad_outputs=LOSS_HEADS["vlogit_mc"], train=True, loss="vlogit_mc", choices=204, score=True, loss_in_forward=True)
    assert p.Nt == NT + 1 and p.arena_bytes > 0
    for t in (p.objective_out, p.loss_grad, p.preds, *p.loss_inputs.values(), *p.head_grad.values()):   # private, never overlaid
        assert not (eng.arena.data_ptr() <= t.data_ptr() < eng.arena.data_ptr() + eng.arena.numel())


def test_new_objective_options_are_checked(golden_dir):
    eng = _engine(golden_dir)
    with pytest.raises(ValueError):
        eng.plan(4, NT, NV, loss="binary_ce", score=True, loss_in_forward=True)        # no score with int labels (Foil)
    with pytest.raises(ValueError):
        eng.plan(4, NT, 110, loss="vlogit_mc", loss_in_forward=True)                   # choices missing
    with pytest.raises(ValueError):
        eng.plan(4, NT, 101, loss="vlogit_mc", choices=4, loss_in_forward=True)        # no region after the first 101
    p = eng.plan(4, NT, NV, loss="binary_ce", grad_outputs=("vil_binary_prediction",), train=True, loss_in_forward=True)
    assert _names(p.fwd)[-1] == "vb_ce_loss" and p.score is None


@pytest.mark.parametrize("precision", ["fp16", "fp32"])
def test_plans_without_the_new_options_launch_no_new_op(golden_dir, precision):
    from vilbert_b200.engine import LOSS_HEADS
    new = {"vb_bce_gather_loss", "vb_task_score", "vb_scale_by_device"}
    eng = _engine(golden_dir, precision)
    plans = [eng.plan(4, NT, NV, grad_outputs=O.HEAD_NAMES, train=True), eng.plan(4, NT, NV, grad_outputs=("vil_prediction",), vqa_loss=True)]
    plans += [eng.plan(4, NT, NV, grad_outputs=LOSS_HEADS[k], loss=k, train=True) for k in ("gqa", "vlogit_bce", "logit_ce", "binary_ce", "tri_ce")]
    for p in plans:
        p.enable_training_prologue()
        assert not new & set(_names(p.prologue + p.fwd + p.bwd)) and p.score is None and not p.head_grad
