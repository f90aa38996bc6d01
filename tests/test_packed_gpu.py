"""Packed task steps (engine.pack_padding) on the GPU: the same batch through the padded and the packed plan gives the same losses,
scores, results and parameter gradients (up to fp32 summation order), batches that cannot be packed run padded and are counted, and
the varlen attention kernels match the padded kernel on the same data."""
import ctypes as C
import json
import math
import os

import pytest
import torch

import _task_oracle as T
from _gpu_util import rel_l2
from oracle import vilbert_oracle as O

pytestmark = pytest.mark.gpu
TASK_CFG = T.TASK_CFG
DEV = torch.device("cuda")


# distinct probabilities per dropout family, so a site that drew another site's mask or probability would show
DROPOUT = dict(hidden_dropout_prob=0.1, attention_probs_dropout_prob=0.15, v_hidden_dropout_prob=0.2, v_attention_probs_dropout_prob=0.25)
HEAD_P = 0.3


def _model(golden_dir, precision=None, **over):
    import vilbert_b200
    cfgj = dict(json.load(open(os.path.join(golden_dir, "tiny_b4.json")))["config"], task_specific_tokens=True, max_position_embeddings=300,
                **over)
    model = vilbert_b200.VILBertForVLTasks(vilbert_b200.BertConfig.from_dict(cfgj), precision=precision)
    model.load_state_dict(O.synth_params(O.make_config(cfgj), seed=0, device="cuda"), strict=False)
    return model, cfgj


def _ragged(mask, seed):
    """Prefix masks of the same shape with random lengths in [1, N], the first row of length 1."""
    g = torch.Generator().manual_seed(seed)
    n = mask.size(-1)
    lens = torch.randint(1, n + 1, mask.shape[:-1], generator=g)
    lens.view(-1)[0] = 1
    return (torch.arange(n) < lens.unsqueeze(-1)).long()


def _batch(cfgj, task_id, B, Nv, Nt, C=4, seed=0):
    b = list(T.make_batch(cfgj, task_id, B, Nv, Nt, C=C, seed=seed))
    kind = T.kind_of(task_id)
    if TASK_CFG[task_id]["process"] == "nlvr":     # two images per sample, each prefix-valid
        b[2] = torch.cat([_ragged(b[2][:, :Nv], seed), _ragged(b[2][:, Nv:], seed + 1)], 1)
    elif kind == "vlogit_mc":                      # keep the first choice and every choice with a non-zero target on valid regions
        keep = b[4].reshape(b[7].shape) != 0
        keep[:, 0] = True
        need = (b[7].long() + T.MC_OFFSET + 1) * keep
        lens = torch.maximum(_ragged(b[2], seed).sum(1), need.max(1).values)
        b[2] = (torch.arange(b[2].size(1)) < lens.unsqueeze(1)).long()
    else:
        b[2] = _ragged(b[2], seed)
    b[5] = _ragged(b[5], seed + 2)
    if kind == "vlogit_bce":
        b[4] = b[4] * b[2].unsqueeze(-1)
    return tuple(b)


def _losses(task_id):
    from vilbert_b200.tasks import LoadLosses
    return LoadLosses(None, TASK_CFG, [task_id[4:]])


KINDS = [("TASK1", 6, 11, 9, 4), ("TASK15", 6, 11, 9, 4), ("TASK5", 4, 11, 9, 4), ("TASK9", 6, 37, 9, 4), ("TASK4", 8, 200, 21, 4),
         ("TASK17", 4, 306, 257, 204), ("TASK12", 4, 11, 9, 4), ("TASK13", 5, 11, 9, 4)]


@pytest.mark.parametrize("task_id,B,Nv,Nt,C", KINDS)
def test_packed_val_and_eval_match_padded(golden_dir, task_id, B, Nv, Nt, C):
    """ForwardModelsVal and EvaluatingModel, packed vs padded on the same batch: equal scores and result dicts, losses to fp32
    reordering."""
    from vilbert_b200.tasks import EvaluatingModel, ForwardModelsVal
    model, cfgj = _model(golden_dir)
    model.eval()
    batch = _batch(cfgj, task_id, B, Nv, Nt, C=C)

    class _DS:
        label2ans = {i: f"a{i}" for i in range(3129)}

    dl = {task_id: type("DL", (), {"dataset": _DS})()}
    out = {}
    for pack in (False, True):
        model.engine.pack_padding = pack
        val = ForwardModelsVal(None, TASK_CFG, DEV, task_id, batch, model, _losses(task_id))
        assert (model._last_plan.packed is not None) == pack
        ev = EvaluatingModel(None, TASK_CFG, DEV, task_id, batch, model, dl, _losses(task_id), [], [])
        out[pack] = val, ev
    assert not model.engine.pack_fallbacks
    (l0, s0, n0), (l1, s1, n1) = out[False][0], out[True][0]
    assert n0 == n1 and s0 == s1 and abs(l0 - l1) <= 1e-5 * max(abs(l0), 1e-6), (l0, l1, s0, s1)
    e0, e1 = out[False][1], out[True][1]
    assert e0[1] == e1[1] and abs(e0[0] - e1[0]) <= 1e-5 * max(abs(e0[0]), 1e-6)
    r0, r1 = e0[3], e1[3]
    assert len(r0) == len(r1)
    for a, b in zip(r0, r1):
        assert a.keys() == b.keys()
        for k in a:
            if isinstance(a[k], list):
                assert max(abs(x - y) for x, y in zip(a[k], b[k])) <= 1e-5, (k, a[k], b[k])
            elif isinstance(a[k], float):
                assert abs(a[k] - b[k]) <= 1e-5, (k, a[k], b[k])
            else:
                assert a[k] == b[k], (k, a[k], b[k])


def _grads(model, task_id, batch, pack, step=7):
    from vilbert_b200.tasks import ForwardModelsTrain
    model.engine.pack_padding = pack
    model.engine.set_dropout_step(step)     # the forward bumps it: both runs draw the masks of step + 1
    model.zero_grad()
    loss, score = ForwardModelsTrain(None, TASK_CFG, DEV, task_id, {task_id: 0}, {}, {task_id: [batch]}, model, _losses(task_id))
    loss.backward()
    assert (model._last_plan.packed is not None) == pack
    eng = model.engine
    return loss.item(), score.item(), {k: eng.ps.g(k).clone() for k in eng.ps.entries}


def _frozen_text(model):
    names = [n for n, p in model.named_parameters() if n.startswith(("bert.embeddings.", "bert.encoder.layer."))]
    for n in names:
        model._params[n].requires_grad_(False)
    return names


def _oracle_grads(cfgj, task_id, batch, step, frozen):
    """The task step in the fp32 oracle with the engine's dropout masks of `step` (oracle.DropMasks): loss and parameter
    gradients (None for a frozen parameter)."""
    kind, proc = T.kind_of(task_id), TASK_CFG[task_id]["process"]
    cfg = O.make_config(cfgj)
    P = O.synth_params(cfg, seed=0, device="cuda")
    Pg = {k: v.clone().requires_grad_(k not in frozen) for k, v in P.items() if k != "cls.predictions.decoder.weight"}
    Pg["cls.predictions.decoder.weight"] = Pg["bert.embeddings.word_embeddings.weight"]
    b = tuple(t.cuda() for t in batch)
    mc = b[7] if task_id in ("TASK4", "TASK17") else None
    features, spatials, image_mask, question, target, input_mask, segment_ids = b[0], b[1], b[2], b[3], b[4], b[5], b[6]
    (features, spatials, image_mask, question, input_mask, segment_ids), target, bs, opts = T.reshape_batch(
        proc, features.size(0), features, spatials, image_mask, question, input_mask, segment_ids, target)
    tasks = question.new_full((question.size(0), 1), int(task_id[4:]))
    _, heads = O.vilbert_for_vl_tasks(Pg, cfg, question, features, spatials, segment_ids, input_mask, image_mask, None, tasks,
                                      drop=O.DropMasks(step, head_p=HEAD_P))
    loss, _ = T.objective(kind, heads, target, mc, bs, opts)
    loss.backward()
    return loss.item(), {k: v.grad for k, v in Pg.items()}


@pytest.mark.parametrize("task_id,B,Nv,Nt,C,precision,freeze", [
    ("TASK1", 6, 37, 9, 4, None, False), ("TASK9", 6, 37, 9, 4, None, False), ("TASK4", 8, 200, 21, 4, None, False),
    ("TASK17", 4, 306, 257, 204, None, False), ("TASK5", 4, 11, 9, 4, None, False), ("TASK12", 4, 11, 9, 4, None, False),
    ("TASK13", 5, 11, 9, 4, None, False), ("TASK9", 6, 37, 9, 4, "fp32", False), ("TASK1", 6, 37, 9, 4, None, True)])
def test_packed_training_step_matches_padded(golden_dir, task_id, B, Nv, Nt, C, precision, freeze):
    """ForwardModelsTrain + backward in train mode with distinct dropout probabilities, packed vs padded at the same dropout step:
    the packed plan draws the padded plan's masks, so the score is equal, the loss equal to fp32 reordering and every parameter
    gradient within a relative L2 of 2e-3 (the oracle contract below is 2e-2). Both are also checked against the fp32 oracle with
    the same masks under the train-mode contract of test_model_gpu.py (rel-L2 with its floor: worst 2e-2, median 1e-2); a frozen
    text stream takes no gradient."""
    model, cfgj = _model(golden_dir, precision, **DROPOUT)
    model.engine.head_dropout_prob = HEAD_P
    model.train()
    frozen = _frozen_text(model) if freeze else []
    batch = _batch(cfgj, task_id, B, Nv, Nt, C=C)
    l0, s0, g0 = _grads(model, task_id, batch, False)
    l1, s1, g1 = _grads(model, task_id, batch, True)
    assert not model.engine.pack_fallbacks
    assert s0 == s1 and abs(l0 - l1) <= 1e-5 * abs(l0), (l0, l1)
    gmax = max(v.abs().max().item() for v in g0.values())
    worst = max((rel_l2(g1[k], g0[k]), k) for k in g0 if g0[k].abs().max().item() > 1e-3 * gmax)
    assert worst[0] < 2e-3, worst
    for n in frozen:
        assert g1[n].abs().max().item() == 0.0, n
    assert all(torch.isfinite(v).all() for v in g1.values())
    # the fp32 oracle with the masks of the step the forward drew (set_dropout_step(7), bumped once)
    lo, go = _oracle_grads(cfgj, task_id, batch, 8, frozen)
    assert abs(l1 - lo) < 1e-3 * abs(lo), (l1, lo)
    gomax = max(v.abs().max().item() for v in go.values() if v is not None)
    floor = 1e-3 * gomax
    l2 = []
    for k, mg in g1.items():
        rg = go[k]
        if rg is None:
            assert mg.abs().max().item() == 0.0, k
            continue
        l2.append((((mg - rg).norm() / max(rg.norm().item(), floor * math.sqrt(rg.numel()) * 0.1)).item(), k))
    l2.sort()
    assert l2[-1][0] < 2e-2 and l2[len(l2) // 2][0] < 1e-2, (l2[-3:], l2[len(l2) // 2])


def test_packed_eval_training_step_matches_padded(golden_dir):
    """The same step in eval mode (no dropout masks at all)."""
    model, cfgj = _model(golden_dir)
    model.eval()
    batch = _batch(cfgj, "TASK9", 6, 37, 9)
    l0, s0, g0 = _grads(model, "TASK9", batch, False)
    l1, s1, g1 = _grads(model, "TASK9", batch, True)
    assert s0 == s1 and abs(l0 - l1) <= 1e-5 * abs(l0), (l0, l1)
    gmax = max(v.abs().max().item() for v in g0.values())
    assert max(rel_l2(g1[k], g0[k]) for k in g0 if g0[k].abs().max().item() > 1e-3 * gmax) < 2e-3


def test_unpackable_batches_run_padded(golden_dir):
    """A non-prefix mask, a V-logit target on a masked region and a V-logit-mc target on a masked region take the padded plan, and
    pack_fallbacks counts them; a train-mode step packs."""
    from vilbert_b200.tasks import ForwardModelsVal
    model, cfgj = _model(golden_dir)
    model.eval()
    model.engine.pack_padding = True
    b = list(_batch(cfgj, "TASK1", 4, 11, 9))
    b[2] = b[2].clone(); b[2][1, 0] = 0; b[2][1, 1] = 1
    ForwardModelsVal(None, TASK_CFG, DEV, "TASK1", tuple(b), model, _losses("TASK1"))
    assert model._last_plan.packed is None and model.engine.pack_fallbacks["mask"] == 1
    b = list(_batch(cfgj, "TASK4", 4, 200, 9))
    b[4] = b[4].clone(); b[4].view(4, -1)[0, 0] = 1.0
    b[2] = b[2].clone(); b[2][0, int(b[7][0, 0]) + T.MC_OFFSET:] = 0
    ForwardModelsVal(None, TASK_CFG, DEV, "TASK4", tuple(b), model, _losses("TASK4"))
    assert model._last_plan.packed is None and model.engine.pack_fallbacks["choice"] == 1
    b = list(_batch(cfgj, "TASK9", 4, 11, 9))
    b[4] = b[4].clone(); b[4][0, -1, 0] = 1.0; b[2] = b[2].clone(); b[2][0, -1] = 0
    ForwardModelsVal(None, TASK_CFG, DEV, "TASK9", tuple(b), model, _losses("TASK9"))
    assert model._last_plan.packed is None and model.engine.pack_fallbacks["target"] == 1
    model.train()
    from vilbert_b200.tasks import ForwardModelsTrain
    ForwardModelsTrain(None, TASK_CFG, DEV, "TASK1", {"TASK1": 0}, {}, {"TASK1": [_batch(cfgj, "TASK1", 4, 11, 9)]}, model, _losses("TASK1"))
    assert model._last_plan.packed is not None and sum(model.engine.pack_fallbacks.values()) == 3


# ------------------------------------------------------------------------------------------ varlen attention kernel
@pytest.mark.parametrize("D", [64, 128])
@pytest.mark.parametrize("Nq,Nk", [(37, 101), (101, 37), (306, 257), (257, 306)])
def test_varlen_attention_matches_padded(D, Nq, Nk):
    """Packed rows with per-sample offsets vs the padded kernel with the additive mask on the same data: O, lse and dQ / dK / dV on
    the valid rows (the single-pass backward for Nq, Nk <= 128, the dq / dkv kernels beyond)."""
    from vilbert_b200 import _lib as L
    lib, S = L.lib(), C.c_void_p(torch.cuda.current_stream().cuda_stream)
    g = torch.Generator(device="cuda").manual_seed(D + Nq)
    B, H = 4, 2
    lq = torch.tensor([1, Nq, max(1, Nq // 3), Nq - 1]); lk = torch.tensor([Nk, 1, max(1, Nk // 2), Nk - 2])
    HD = H * D
    mk = lambda n: (torch.randn(B * n, HD, device="cuda", generator=g) * 0.5).to(torch.bfloat16)
    Q, K, V, dO = mk(Nq), mk(Nk), mk(Nk), mk(Nq)
    mask = torch.where(torch.arange(Nk) < lk.unsqueeze(1), 0.0, -10000.0).float().cuda()
    rq = torch.cat([torch.arange(n) + b * Nq for b, n in enumerate(lq.tolist())]).cuda()
    rk = torch.cat([torch.arange(n) + b * Nk for b, n in enumerate(lk.tolist())]).cuda()
    off = lambda l: torch.cat([torch.zeros(1, dtype=torch.long), l.cumsum(0)]).int().cuda()
    oq, ok, lq32, lk32 = off(lq), off(lk), lq.int().cuda(), lk.int().cuda()

    def run(q, k, v, do, packed):
        a = L.AttnArgs()
        a.B, a.H, a.Nq, a.Nk, a.D, a.scale = B, H, Nq, Nk, D, 1.0 / math.sqrt(D)
        O_ = torch.zeros_like(q); lse = torch.zeros(B, H, Nq, device="cuda")
        dQ, dK, dV = torch.zeros_like(q), torch.zeros_like(k), torch.zeros_like(v)
        delta = torch.zeros(B, H, Nq, device="cuda")
        a.Q, a.K, a.V, a.O, a.ldq, a.ldk, a.ldv, a.ldo = q.data_ptr(), k.data_ptr(), v.data_ptr(), O_.data_ptr(), HD, HD, HD, HD
        a.lse, a.dO, a.lddo, a.dQ, a.lddq, a.dK, a.lddk, a.dV, a.lddv = lse.data_ptr(), do.data_ptr(), HD, dQ.data_ptr(), HD, dK.data_ptr(), HD, dV.data_ptr(), HD
        a.delta = delta.data_ptr()
        if packed:
            a.q_off, a.q_len, a.k_off, a.k_len = oq.data_ptr(), lq32.data_ptr(), ok.data_ptr(), lk32.data_ptr()
        else:
            a.mask = mask.data_ptr()
        L.check(lib.vb_attention_fwd(C.byref(a), S), "fwd")
        L.check(lib.vb_attention_bwd(C.byref(a), S), "bwd")
        torch.cuda.synchronize()
        return O_, lse, dQ, dK, dV

    dead = torch.ones(B * Nq, dtype=torch.bool, device="cuda").index_fill_(0, rq, False)
    dO_masked = dO.clone(); dO_masked[dead] = 0
    P = run(Q, K, V, dO_masked, False)        # the padded plan's masked query rows carry no gradient
    R = run(Q[rq].contiguous(), K[rk].contiguous(), V[rk].contiguous(), dO[rq].contiguous(), True)
    assert torch.equal(R[0], P[0][rq])
    vq = torch.arange(Nq).unsqueeze(0) < lq.unsqueeze(1)
    assert torch.equal(R[1][vq.unsqueeze(1).expand(B, H, Nq).cuda()], P[1][vq.unsqueeze(1).expand(B, H, Nq).cuda()])
    for got, ref in ((R[2], P[2][rq]), (R[3], P[3][rk]), (R[4], P[4][rk])):
        assert rel_l2(got, ref) < 1e-2 and (got.float() - ref.float()).abs().max().item() <= 2e-2 * ref.float().abs().max().item() + 1e-6
