"""Every autograd surface of the module runs its backward at its own forward (modeling._PlanCall): VILBertForVLTasks outputs under a
torch loss, ForwardModelsTrain, and BertForMultiModalPreTraining(fused_objective=True). In train mode a backward after other
forwards gives the gradient of the uninterrupted forward + backward; a forward followed by its own backward writes no dropout
step; every backward ends with one data-parallel all-reduce."""
import json
import os

import pytest
import torch
import torch.nn.functional as F

import _task_oracle as T
from oracle import vilbert_oracle as O

pytestmark = pytest.mark.gpu

# (B, Nv, Nt) of the call under test and of a forward of another shape
SHAPES = {"module": ((4, 11, 9), (6, 13, 10)), "TASK1": ((4, 11, 9), (6, 13, 10)), "TASK4": ((4, 110, 9), (6, 112, 10)),
          "pretraining": ((4, 9, 8), (6, 11, 10))}
SURFACES = list(SHAPES)


def _pretraining_labels(cfg, B, Nv, Nt, seed):
    g = torch.Generator().manual_seed(seed)
    lm = torch.full((B, Nt), -1, dtype=torch.long)
    sel = torch.rand(B, Nt, generator=g) < 0.15
    sel[:, 1] = True
    lm[sel] = torch.randint(0, cfg["vocab_size"], (int(sel.sum()),), generator=g)
    il = torch.full((B, Nv - 1), -1, dtype=torch.long)
    il[torch.rand(B, Nv - 1, generator=g) < 0.15] = 1
    il[:, 0] = 1
    it = torch.randn(B, Nv - 1, cfg["v_target_size"], generator=g) * 0.1
    ns = torch.randint(0, 2, (B,), generator=g)
    return [x.cuda() for x in (lm, il, it, ns)]


def _surface(golden_dir, surface, arena=False):
    """A train-mode model on tiny_b4 (dropout 0.1 everywhere) and `loss(B, Nv, Nt, seed)`: one forward of `surface` on a synthetic
    batch, returning the scalar whose backward() runs the surface's backward."""
    import vilbert_b200
    from vilbert_b200.tasks import ForwardModelsTrain, LoadLosses
    pre = surface == "pretraining"
    over = dict(visual_target=2, v_target_size=48, num_negative=20) if pre else dict(task_specific_tokens=True, max_position_embeddings=300)
    cfgj = dict(json.load(open(os.path.join(golden_dir, "tiny_b4.json")))["config"], **over)
    cfg = O.make_config(cfgj)
    if pre:
        model = vilbert_b200.BertForMultiModalPreTraining(vilbert_b200.BertConfig.from_dict(cfgj), fused_objective=True)
        # every call draws new negatives from torch's CPU generator: a recomputation that drew again would change the gradient
        model.nce_sampler = lambda b, r, dev: O.nce_negative_indices(b, r, cfg["num_negative"]).to(dev)
    else:
        model = vilbert_b200.VILBertForVLTasks(vilbert_b200.BertConfig.from_dict(cfgj))
    model.load_state_dict(O.synth_params(cfg, seed=3, device="cuda", with_task_heads=not pre), strict=False)
    if arena:
        model.engine.enable_activation_arena(256 << 20)
    model.train()

    def loss(B, Nv, Nt, seed):
        if surface.startswith("TASK"):
            batch = T.make_batch(cfgj, surface, B, Nv, Nt, seed=seed)
            return ForwardModelsTrain(None, T.TASK_CFG, torch.device("cuda"), surface, {surface: 0}, {}, {surface: [batch]}, model,
                                      LoadLosses(None, T.TASK_CFG, [surface[4:]]))[0]
        inp = O.synth_inputs(cfg, B, Nv, Nt, seed=seed, device="cuda")
        args = [inp[k] for k in ("input_txt", "input_imgs", "image_loc", "token_type_ids", "attention_mask", "image_attention_mask")]
        if pre:
            return sum(model(*args, *_pretraining_labels(cfg, B, Nv, Nt, seed))).sum()
        tgt = O.synth_vqa_target(B, 3129, seed=seed, device="cuda")
        return F.binary_cross_entropy_with_logits(model(*args, None, inp["task_ids"])[0], tgt)
    return model, loss


@pytest.mark.parametrize("between", ["other_shape", "same_plan"])
@pytest.mark.parametrize("arena", [False, True])
@pytest.mark.parametrize("surface", SURFACES)
def test_backward_after_other_forwards(golden_dir, surface, arena, between):
    """A train-mode forward, then a forward of another shape or of the same plan with other inputs (which moves the dropout step
    and, with the shared arena or the same plan, overwrites the saved activations), then the first forward's backward: the
    gradient is that of the uninterrupted forward + backward at the same dropout step, inputs, targets and negatives."""
    model, loss = _surface(golden_dir, surface, arena)
    eng = model.engine
    first, second = SHAPES[surface]
    other = (*(second if between == "other_shape" else first), 1)

    def grad(interrupted):
        torch.manual_seed(1)
        eng.set_dropout_step(5)
        model.zero_grad()
        total = loss(*first, 0)
        if interrupted:
            loss(*other)
        model.zero_grad()
        total.backward()
        return eng.ps.grad.clone()
    grad(False)             # the module outputs' plan learns its gradient set in the first backward
    want = grad(False)
    got = grad(True)
    assert ((got - want).abs().max() / want.abs().max()).item() < 1e-5     # split-K atomics: last-bit order effects only


@pytest.mark.parametrize("surface", SURFACES)
def test_steady_loop_writes_no_dropout_step(golden_dir, surface, monkeypatch):
    """A forward followed directly by its own backward launches what it launched before: the dropout step is never written."""
    from vilbert_b200.engine import Engine
    model, loss = _surface(golden_dir, surface)
    writes = []
    set_step = Engine.set_dropout_step
    monkeypatch.setattr(Engine, "set_dropout_step", lambda self, step: (writes.append(step), set_step(self, step))[1])
    for i in range(4):       # eager runs, the switch of the module outputs' plan, then both passes as graph replays
        loss(*SHAPES[surface][0], i).backward()
    assert model._last_plan.graph_fwd is not None and model._last_plan.graph_bwd is not None
    assert writes == []


@pytest.mark.parametrize("surface", SURFACES)
def test_backward_ends_with_one_allreduce(golden_dir, surface, monkeypatch):
    """With a data-parallel reducer attached every backward calls allreduce() once, after the plan's backward."""
    from vilbert_b200.engine import Plan
    model, loss = _surface(golden_dir, surface)
    events = []
    run_backward = Plan.run_backward
    monkeypatch.setattr(Plan, "run_backward", lambda self: (run_backward(self), events.append("backward"))[0])

    class Reducer:
        def allreduce(self):
            events.append("allreduce")
    model._ddp_reducer = Reducer()
    for i in range(2):
        events.clear()
        loss(*SHAPES[surface][0], i).backward()
        assert events == ["backward", "allreduce"], i
