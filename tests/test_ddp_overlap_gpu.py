"""The overlapped data-parallel backward of the module surface (DistributedDataParallel(delay_allreduce=False)) on one GPU, against
a stand-in reducer of a world of two: on the stream it is handed it doubles each bucket in place, records (lo, hi) and keeps a copy
of what it doubled. A backward op that wrote into a bucket after its handover would leave the buffer different from that copy, so
the copies must equal the final buffer bitwise, the handovers must be the table in descending order, and the buffers must match the
delayed mode (the stand-in doubles the whole table after the backward): bitwise for a deterministic plan, to the last bits of the
split-K atomics otherwise. Covered: the VQA ForwardModelsTrain step padded and packed, the fused pre-training step, two backwards
accumulated before a clipping FusedAdamW step, a backward that recomputes its forward under the shared arena, a frozen text stream,
a deterministic plan, eager and graph-captured pieces, and no_sync()."""
import json
import os

import pytest
import torch

import _task_oracle as T
from oracle import vilbert_oracle as O

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda")


def _stub_class():
    from vilbert_b200.ddp import FlatGradAllReducer

    class Stub(FlatGradAllReducer):
        def __init__(self, flat_grad, n_buckets=8, group=None):
            super().__init__(flat_grad, n_buckets=n_buckets, group=group)
            self.world = 2
            self.calls, self.copies = [], []

        def broadcast_params(self, flat_params, src=0):
            pass

        def allreduce_range(self, lo, hi, async_op=True):
            self.calls.append((lo, hi))
            t = self.flat[lo:hi]
            t.mul_(2.0)
            self.copies.append((lo, hi, t.clone()))
            return None

        def allreduce(self):
            for lo, hi in self.table:
                self.allreduce_range(lo, hi)
    return Stub


def _wrap(model, overlap, monkeypatch):
    from vilbert_b200 import ddp
    monkeypatch.setattr(ddp, "FlatGradAllReducer", _stub_class())
    return ddp.DistributedDataParallel(model, delay_allreduce=not overlap, n_buckets=8)


def _cfgj(golden_dir, pre):
    over = dict(visual_target=2, v_target_size=48, num_negative=20) if pre else dict(task_specific_tokens=True, max_position_embeddings=300)
    return dict(json.load(open(os.path.join(golden_dir, "tiny_b4.json")))["config"], **over)


def _vqa_model(golden_dir, arena=False):
    import vilbert_b200
    cfgj = _cfgj(golden_dir, False)
    model = vilbert_b200.VILBertForVLTasks(vilbert_b200.BertConfig.from_dict(cfgj))
    model.load_state_dict(O.synth_params(O.make_config(cfgj), seed=3, device="cuda"), strict=False)
    if arena:
        model.engine.enable_activation_arena(256 << 20)
    model.train()
    return model, cfgj


def _vqa_loss(model, cfgj, B, Nv, Nt, seed):
    from vilbert_b200.tasks import ForwardModelsTrain, LoadLosses
    batch = T.make_batch(cfgj, "TASK1", B, Nv, Nt, seed=seed)
    return ForwardModelsTrain(None, T.TASK_CFG, DEV, "TASK1", {"TASK1": 0}, {}, {"TASK1": [batch]}, model,
                              LoadLosses(None, T.TASK_CFG, ["1"]))[0]


def _pretraining_model(golden_dir):
    import vilbert_b200
    cfgj = _cfgj(golden_dir, True)
    cfg = O.make_config(cfgj)
    model = vilbert_b200.BertForMultiModalPreTraining(vilbert_b200.BertConfig.from_dict(cfgj), fused_objective=True)
    model.load_state_dict(O.synth_params(cfg, seed=3, device="cuda", with_task_heads=False), strict=False)
    model.nce_sampler = lambda b, r, dev: O.nce_negative_indices(b, r, cfg["num_negative"]).to(dev)
    model.train()
    return model, cfgj


def _pretraining_loss(model, cfgj, B, Nv, Nt, seed):
    cfg = O.make_config(cfgj)
    inp = O.synth_inputs(cfg, B, Nv, Nt, seed=seed, device="cuda")
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
    args = [inp[k] for k in ("input_txt", "input_imgs", "image_loc", "token_type_ids", "attention_mask", "image_attention_mask")]
    torch.manual_seed(seed)          # the negatives the sampler draws
    return sum(model(*args, *(x.cuda() for x in (lm, il, it, ns)))).sum()


def _freeze_text(model):
    for name, p in model.named_parameters():
        if name.startswith(("bert.embeddings.", "bert.encoder.layer.")):
            p.requires_grad_(False)


# (surface, model options, step options)
CASES = {
    "vqa_padded": ("vqa", {}, {}),
    "vqa_packed": ("vqa", {}, dict(pack=True)),
    "pretraining": ("pretraining", {}, {}),
    "accumulate_two": ("vqa", {}, dict(accumulate=2)),
    "recompute_arena": ("vqa", dict(arena=True), dict(recompute=True)),
    "frozen_text": ("vqa", {}, dict(freeze=True)),
    "deterministic": ("vqa", {}, dict(det=True)),
}
SHAPE = (4, 100, 36)        # the per-GPU shape of config 2 (100 regions x 36 tokens), on the tiny model
OTHER = (6, 37, 20)


def _run(golden_dir, monkeypatch, surface, model_kw, step_kw, overlap, steps=4):
    """`steps` training steps (two eager, then the pieces as graphs) with the stand-in attached; per step the flat gradient buffer
    after the backward(s), the handovers of the last backward and the parameters after a clipping FusedAdamW step."""
    from vilbert_b200.optim import FusedAdamW
    if surface == "pretraining":
        model, cfgj = _pretraining_model(golden_dir)
        loss_fn, shape = _pretraining_loss, (4, 37, 36)
    else:
        model, cfgj = _vqa_model(golden_dir, **model_kw)
        loss_fn, shape = _vqa_loss, SHAPE
    model.engine.pack_padding = step_kw.get("pack", False)
    if step_kw.get("freeze"):
        _freeze_text(model)
    dp = _wrap(model, overlap, monkeypatch)
    red = model._ddp_reducer
    # split-K atomics make the gradients of two runs differ in their last bits, which an AdamW step can magnify where a gradient is
    # near zero: outside a deterministic plan the step keeps the parameters (lr 0) and still clips the averaged buffer
    lr = 1e-3 if torch.are_deterministic_algorithms_enabled() else 0.0
    opt = FusedAdamW([p for p in model.parameters() if p.requires_grad], lr=lr, model=model, max_grad_norm=1.0)
    out = []
    for s in range(steps):
        model.engine.set_dropout_step(11 * s)
        for m in range(step_kw.get("accumulate", 1)):
            loss = loss_fn(dp, cfgj, *shape, 100 * s + m)
            if step_kw.get("recompute"):
                loss_fn(dp, cfgj, *OTHER, 7)          # overwrites the shared arena: the backward recomputes its forward
            red.calls.clear(); red.copies.clear()
            loss.backward()
            torch.cuda.synchronize()
            for lo, hi, c in red.copies:             # nothing landed in a bucket after it was handed over
                assert torch.equal(red.flat[lo:hi], c), (lo, hi)
            assert len(red.calls) == len(red.table)
            if overlap:
                assert red.calls == list(reversed(red.table))
        grad = model.engine.ps.grad.clone()
        opt.step()
        torch.cuda.synchronize()
        out.append((grad, model.engine.ps.flat.clone()))
    plans = list(model.engine.plans.values())
    if not step_kw.get("recompute"):
        assert (model._last_plan.packed is not None) == step_kw.get("pack", False)
    if overlap:
        assert any(p._piece_graphs for p in plans), "the pieces were captured after two eager runs"
        assert all(p.graph_bwd is None for p in plans)       # the whole-backward graph is never used in this mode
    if step_kw.get("freeze"):
        off, _ = model.engine.ps.entries["bert.embeddings.word_embeddings.weight"]
        assert all(not (lo <= off < hi) for lo, hi in red.table)
    return out


@pytest.mark.parametrize("case", list(CASES))
def test_overlapped_matches_delayed(golden_dir, monkeypatch, case):
    surface, model_kw, step_kw = CASES[case]
    det = step_kw.get("det", False)
    prev = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(det)
    try:
        delayed = _run(golden_dir, monkeypatch, surface, model_kw, step_kw, overlap=False)
        overlapped = _run(golden_dir, monkeypatch, surface, model_kw, step_kw, overlap=True)
    finally:
        torch.use_deterministic_algorithms(prev)
    for s, ((g0, p0), (g1, p1)) in enumerate(zip(delayed, overlapped)):
        if det:
            assert torch.equal(g0, g1) and torch.equal(p0, p1), s
        else:
            assert ((g0 - g1).abs().max() / g0.abs().max()).item() < 1e-5, s
            assert ((p0 - p1).abs().max() / p0.abs().max()).item() < 1e-5, s


@pytest.mark.parametrize("overlap", [False, True])
def test_no_sync_issues_no_collective(golden_dir, monkeypatch, overlap):
    model, cfgj = _vqa_model(golden_dir)
    dp = _wrap(model, overlap, monkeypatch)
    red = model._ddp_reducer
    model.zero_grad()
    with dp.no_sync():                  # reachable through the wrapper
        for m in range(3):
            _vqa_loss(dp, cfgj, *SHAPE, m).backward()
    torch.cuda.synchronize()
    assert red.calls == []
    _vqa_loss(dp, cfgj, *SHAPE, 3).backward()
    torch.cuda.synchronize()
    assert sorted(red.calls) == list(red.table)
    assert model._ddp_sync


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs 2 GPUs")
def test_two_ranks_with_other_plans(tmp_path):
    import signal
    import subprocess
    import sys
    out = tmp_path / "ddp_overlap.json"
    worker = os.path.join(os.path.dirname(os.path.abspath(__file__)), "_ddp_overlap_worker.py")
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=2", "--master-addr", "127.0.0.1",
           "--master-port", "29547", worker, str(out)]
    # own process group: on a timeout the launcher and both ranks are ended together, nothing is left running
    proc = subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.PIPE, text=True, start_new_session=True)
    try:
        _, err = proc.communicate(timeout=600)
    except subprocess.TimeoutExpired:
        os.killpg(proc.pid, signal.SIGKILL)
        proc.communicate()
        pytest.fail("the 2-rank overlap worker did not finish within 600 s")
    assert proc.returncode == 0, err[-3000:]
    ranks = json.load(open(out))
    assert ranks[0]["det_packed_rank0"] == [True] * 4 and ranks[1]["det_packed_rank1"] == [False] * 4, ranks
    for res in ranks:
        assert res["det_grad_diff"] == [0.0] * 4 and all(res["det_params_equal"]), res
        assert max(res["default_grad_diff"]) < 1e-5 and all(res["default_params_equal"]), res
        assert res["det_ranks_equal"] and res["default_ranks_equal"], res
        assert res["det_no_sync_l2"] < 1e-6 and res["default_no_sync_l2"] < 1e-6, res
        assert res["pretraining_equal"], res
    for tag in ("det", "default"):     # the tolerances of test_ddp_gpu.py
        assert ranks[0][f"{tag}_vs_one_gpu_l2"] < 2e-3 and ranks[0][f"{tag}_vs_one_gpu_worst_tensor_l2"] < 1e-2, ranks[0]
