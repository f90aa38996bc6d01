"""vilbert_b200.tasks.EvaluatingModel on the GPU: vb_task_results against torch, pruned plans (Plan(outputs=...)) against the
all-heads plan bit for bit, and EvaluatingModel against the restated reference step (tests/_eval_oracle.py) on the module surface."""
import ctypes as C
import json
import os
import types

import pytest
import torch

import _eval_oracle as E
import _task_oracle as T
from oracle import vilbert_oracle as O

pytestmark = pytest.mark.gpu
S = lambda: C.c_void_p(torch.cuda.current_stream().cuda_stream)
NAN = float("nan")


def _model(golden_dir, cfg_file="tiny_b4.json", **over):
    import vilbert_b200
    cfgj = dict(json.load(open(os.path.join(golden_dir, cfg_file)))["config"], task_specific_tokens=True, max_position_embeddings=300, **over)
    model = vilbert_b200.VILBertForVLTasks(vilbert_b200.BertConfig.from_dict(cfgj))
    model.load_state_dict(O.synth_params(O.make_config(cfgj), seed=0, device="cuda"), strict=False)
    return model, cfgj


def _loader(task_id, n=3129):
    return {task_id: types.SimpleNamespace(dataset=types.SimpleNamespace(label2ans=[f"answer {i}" for i in range(n)]))}


def _same(a, b, rel):
    if isinstance(a, dict):
        return a.keys() == b.keys() and all(_same(a[k], b[k], rel) for k in a)
    if isinstance(a, list):
        return len(a) == len(b) and all(_same(x, y, rel) for x, y in zip(a, b))
    if isinstance(a, float):
        return type(b) is float and ((a != a and b != b) or abs(a - b) <= rel * abs(b))
    return type(a) is type(b) and a == b


# ------------------------------------------------------------------------------------------ vb_task_results
def _rows(rows, cols, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    x = (torch.randn(rows, cols, device="cuda", generator=g) * 3).round(decimals=1)      # ties are common
    x[0, cols // 2:] = x[0].max() + 1.0                                                  # tied maximum
    if rows > 2:
        x[1, cols - 1] = NAN                                                              # NaN row
        x[2, :] = -10000.0                                                               # every column tied
    return x


@pytest.mark.parametrize("rows,cols", [(1, 2), (7, 4), (30, 100), (1024, 3129)])
def test_task_results_kernel_against_torch(rows, cols):
    from vilbert_b200 import _lib as L
    lib = L.lib()
    x = _rows(rows, cols, rows)
    tgt = torch.rand(rows, cols, device="cuda")
    pick = torch.max(x, 1)[1]
    for mode in (L.VB_RESULT_ARGMAX, L.VB_RESULT_SOFTMAX, L.VB_RESULT_GATHER):
        idx = torch.full((rows,), -7, dtype=torch.int64, device="cuda")
        ld = cols + 3 if mode == L.VB_RESULT_SOFTMAX else 1
        vals = torch.full((rows, ld), -7.0, device="cuda")
        L.check(lib.vb_task_results(mode, x.data_ptr(), cols, 0, cols, None, 0, tgt.data_ptr(), cols, rows, idx.data_ptr(), vals.data_ptr(), ld,
                                    S()), "vb_task_results")
        assert torch.equal(idx, pick), mode
        if mode == L.VB_RESULT_SOFTMAX:
            want, got = torch.softmax(x, 1), vals[:, :cols]
            assert torch.equal(torch.isnan(got), torch.isnan(want))
            ok = ~torch.isnan(want)
            assert torch.allclose(got[ok], want[ok], rtol=1e-6, atol=0)
            assert (vals[:, cols:] == -7.0).all()                                         # the row pitch is honoured
        elif mode == L.VB_RESULT_GATHER:
            assert torch.equal(vals[:, 0], tgt.gather(1, pick.view(-1, 1)).view(-1))
    # a row of pitch ld_logits with a column offset, as the V-logit head is read
    wide = _rows(rows, cols + 5, 3)
    idx = torch.empty(rows, dtype=torch.int64, device="cuda")
    L.check(lib.vb_task_results(L.VB_RESULT_ARGMAX, wide.data_ptr(), cols + 5, 5, cols, None, 0, None, 0, rows, idx.data_ptr(), None, 0, S()))
    assert torch.equal(idx, torch.max(wide[:, 5:], 1)[1])


def test_task_results_kernel_gathered_choices():
    """V-logit-mc at the GuessWhatPointing shape: vision_logit[:, 101:].gather(1, ids), padded duplicates on a masked region."""
    from vilbert_b200 import _lib as L
    B, Nv, Cc = 8, 306, 204
    v = torch.randn(B, Nv, device="cuda").round(decimals=1)
    v[:, 290:] = -10000.0
    ids = torch.randint(0, 204, (B, Cc), device="cuda")
    ids[:, 20:] = 204
    ids[3, :] = 204
    idx = torch.empty(B, dtype=torch.int64, device="cuda")
    L.check(L.lib().vb_task_results(L.VB_RESULT_ARGMAX, v.data_ptr(), Nv, 101, Cc, ids.data_ptr(), Nv, None, 0, B, idx.data_ptr(), None, 0, S()))
    assert torch.equal(idx, torch.max(v[:, 101:].gather(1, ids), 1)[1])


def test_task_results_kernel_rejects_bad_arguments():
    from vilbert_b200 import _lib as L
    lib = L.lib()
    x, idx = torch.zeros(4, 4, device="cuda"), torch.zeros(4, dtype=torch.int64, device="cuda")
    assert lib.vb_task_results(3, x.data_ptr(), 4, 0, 4, None, 0, None, 0, 4, idx.data_ptr(), None, 0, S()) != 0
    assert b"vb_task_results" in lib.vb_last_error()
    assert lib.vb_task_results(L.VB_RESULT_SOFTMAX, x.data_ptr(), 4, 0, 4, None, 0, None, 0, 4, idx.data_ptr(), x.data_ptr(), 3, S()) != 0
    assert lib.vb_task_results(L.VB_RESULT_GATHER, x.data_ptr(), 4, 0, 4, None, 0, None, 0, 4, idx.data_ptr(), x.data_ptr(), 1, S()) != 0
    assert lib.vb_task_results(L.VB_RESULT_ARGMAX, x.data_ptr(), 4, 0, 4, None, 0, None, 0, 0, idx.data_ptr(), None, 0, S()) != 0


# ------------------------------------------------------------------------------------------ pruned plans
@pytest.mark.parametrize("train", [False, True])
@pytest.mark.parametrize("B", [4, 3])
def test_kept_head_is_bitwise_the_all_heads_head(golden_dir, train, B):
    model, cfgj = _model(golden_dir)
    eng = model.engine
    Nt, Nv = 9, 11
    batch = T.make_batch(cfgj, "TASK1", B, Nv, Nt)
    inputs = dict(input_txt=batch[3].cuda(), input_imgs=batch[0].cuda(), image_loc=batch[1].cuda(), token_type_ids=batch[6].cuda(),
                  attention_mask=batch[5].cuda(), image_attention_mask=batch[2].cuda(), task_ids=torch.full((B, 1), 1, device="cuda"))
    model._sync_weights()

    def run(plan):
        eng.set_dropout_step(11)
        plan.load_inputs(**inputs)
        plan.run_forward()
        return {k: v.clone() for k, v in plan.outputs.items()}
    full = run(eng.plan(B, Nt, Nv, train=train))
    for head in O.HEAD_NAMES:
        got = run(eng.plan(B, Nt, Nv, train=train, outputs=(head,)))
        assert set(got) == {"sequence_output_t", "sequence_output_v", "pooled_output_t", "pooled_output_v", head}
        assert torch.equal(got[head], full[head]), head
        assert torch.equal(got["pooled_output_v"], full["pooled_output_v"])


# ------------------------------------------------------------------------------------------ EvaluatingModel vs the reference step
CASES = [("TASK1", 4, 11, 9), ("TASK15", 3, 11, 9), ("TASK3", 2, 11, 9), ("TASK5", 2, 11, 9), ("TASK7", 2, 11, 9), ("TASK9", 4, 11, 9),
         ("TASK4", 3, 110, 9), ("TASK12", 2, 11, 9), ("TASK12", 3, 11, 9), ("TASK13", 3, 11, 9), ("BIN_ODD", 3, 11, 9)]
# BIN_ODD: the binary head at an odd model batch (the alignment head of self.cls), which no task of the table reaches
TASK_CFG = dict(T.TASK_CFG, BIN_ODD=dict(type="VL-binary-classifier", loss="BCEWithLogitLoss", process="normal"))


def _eval_both(model, task_cfg, task_id, batch, loader, step=5):
    from vilbert_b200.tasks import EvaluatingModel, LoadLosses
    tid = task_id if task_id.startswith("TASK") else "TASK12"
    cfg = {tid: task_cfg[task_id]}
    losses = LoadLosses(None, cfg, [tid[4:]])
    out = {}
    for name in ("reference", "fused"):
        model.engine.set_dropout_step(step)
        res = []
        try:
            if name == "reference":
                r = E.evaluating_step(cfg, tid, tuple(t.cuda() for t in batch), model, loader[task_id].dataset.label2ans, res, [])
            else:
                r = EvaluatingModel(None, cfg, torch.device("cuda"), tid, batch, model, {tid: loader[task_id]}, losses, res, [])
            out[name] = (r[0], r[1], r[2], res, None)
        except (IndexError, ValueError) as ex:
            out[name] = (None, None, None, res, type(ex))
    return out["reference"], out["fused"]


def _check(ref, got):
    assert got[4] is ref[4], (got[4], ref[4])
    assert _same(got[3], ref[3], 1e-6)
    if ref[4] is None:
        assert got[2] == ref[2] and got[1] == ref[1]
        assert isinstance(got[0], float) and (got[0] == ref[0] == 0.0 or abs(got[0] - ref[0]) <= 1e-5 * abs(ref[0])), (got[0], ref[0])


@pytest.mark.parametrize("train", [False, True])
@pytest.mark.parametrize("task_id,B,Nv,Nt", CASES)
def test_evaluating_model_matches_the_reference_step(golden_dir, task_id, B, Nv, Nt, train):
    """Batch size, results (probabilities to 1e-6), loss (1e-5) and score (exact) against the restated reference step on the module
    surface, in the model's current mode (train mode at the same dropout step). VisDial's batches carry one id per image, so both
    raise IndexError after the same rows; with one id per round both complete."""
    model, cfgj = _model(golden_dir)
    model.train(train)
    bt = task_id if task_id.startswith("TASK") else "TASK13"
    batch = T.make_batch(cfgj, bt, B, Nv, Nt, options=3)
    if task_id.startswith("BIN"):
        batch = batch[:4] + (torch.rand(B, 2).round(),) + batch[5:]
    n = 1533 if task_id == "TASK15" else 3129
    loader = _loader(task_id, n)
    _check(*_eval_both(model, TASK_CFG, task_id, batch, loader))
    if task_id == "TASK3":
        per_round = batch[:-1] + (torch.arange(batch[3].shape[0] * batch[3].shape[1]) + 50,)
        ref, got = _eval_both(model, TASK_CFG, task_id, per_round, loader)
        assert ref[4] is None and len(ref[3]) == B * 2
        _check(ref, got)


def test_evaluating_model_vqa_at_the_twelve_in_one_shape(golden_dir):
    """VQA (TASK1) at B = 64, 101 regions, 23 + 1 tokens on bert_base_6layer_6conect with task tokens."""
    import vilbert_b200
    cfgj = dict(json.load(open(os.path.join(os.path.dirname(golden_dir), "..", "vilbert-multi-task_b200", "configs",
                                            "bert_base_6layer_6conect.json"))), task_specific_tokens=True)
    model = vilbert_b200.VILBertForVLTasks(vilbert_b200.BertConfig.from_dict(cfgj))
    model.eval()
    batch = T.make_batch(cfgj, "TASK1", 64, 101, 23, seed=3)
    ref, got = _eval_both(model, T.TASK_CFG, "TASK1", batch, _loader("TASK1"))
    _check(ref, got)
    assert len(got[3]) == 64


@pytest.mark.parametrize("B", [4, 3])
def test_foil_raises_what_forward_models_val_raises(golden_dir, B):
    from vilbert_b200.tasks import EvaluatingModel, ForwardModelsVal, LoadLosses
    model, cfgj = _model(golden_dir)
    model.eval()
    batch = T.make_batch(cfgj, "TASK16", B, 11, 9)
    losses = LoadLosses(None, T.TASK_CFG, ["16"])
    with pytest.raises((ValueError, IndexError)) as val:
        ForwardModelsVal(None, T.TASK_CFG, torch.device("cuda"), "TASK16", batch, model, losses)
    with pytest.raises(val.type):
        EvaluatingModel(None, T.TASK_CFG, torch.device("cuda"), "TASK16", batch, model, _loader("TASK16"), losses, [], [])


@pytest.mark.parametrize("task_id", ["TASK1", "TASK7", "TASK9", "TASK13"])
def test_one_device_to_host_copy_per_call(golden_dir, task_id):
    """After warm-up (CUDA graphs captured), one call reads loss, score and every result with one device-to-host copy."""
    from torch.profiler import ProfilerActivity, profile
    from vilbert_b200.tasks import EvaluatingModel, LoadLosses
    model, cfgj = _model(golden_dir)
    model.eval()
    batch = T.make_batch(cfgj, task_id, 4, 11, 9, options=3)
    losses = LoadLosses(None, T.TASK_CFG, [task_id[4:]])

    def call():
        return EvaluatingModel(None, T.TASK_CFG, torch.device("cuda"), task_id, batch, model, _loader(task_id), losses, [], [])
    for _ in range(4):
        call()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        call()
        torch.cuda.synchronize()
    names = [e.name for e in prof.events() if "memcpy" in e.name.lower()]
    dtoh = [n for n in names if "dtoh" in n.lower().replace(" ", "")]
    assert len(dtoh) == 1, names
