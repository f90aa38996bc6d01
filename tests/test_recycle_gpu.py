"""Forward-only plans with their buffers placed by lifetime (Engine.recycle_forward_only, Plan(recycle=True)) on the GPU: the same
losses, scores, per-row results and retrieval scores as the plain plans, bitwise under torch.use_deterministic_algorithms(True),
eagerly and as CUDA graphs, from memory filled with NaN before the first run (a read of a byte before its buffer's first write
shows), with the image states of an image-prefix plan kept across another plan's forward, and at batch sizes whose plain plans do
not fit a 40 GiB arena."""
import gc
import json
import math
import os
import types

import pytest
import torch

import _task_oracle as T
from oracle import vilbert_oracle as O

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda")
ARENA = 256 << 20
# EvaluatingModel's task types at the tiny config: (task, B, regions, tokens); BIN_ODD is the binary head at an odd batch
CASES = [("TASK1", 4, 11, 9), ("TASK15", 3, 11, 9), ("TASK7", 2, 11, 9), ("TASK9", 4, 11, 9), ("TASK4", 3, 110, 9), ("TASK12", 2, 11, 9),
         ("TASK13", 3, 11, 9), ("BIN_ODD", 3, 11, 9)]
TASK_CFG = dict(T.TASK_CFG, BIN_ODD=dict(type="VL-binary-classifier", loss="BCEWithLogitLoss", process="normal"))


@pytest.fixture(autouse=True)
def release_engines():
    yield
    gc.collect()
    torch.cuda.empty_cache()


@pytest.fixture(params=[True, False], ids=["deterministic", "default"])
def deterministic(request):
    prev, warn_only = torch.are_deterministic_algorithms_enabled(), torch.is_deterministic_algorithms_warn_only_enabled()
    torch.use_deterministic_algorithms(request.param)
    yield request.param
    torch.use_deterministic_algorithms(prev, warn_only=warn_only)


def _nan_fill(t):
    """Every byte of a uint8 buffer set to the bytes of an fp32 NaN."""
    n = t.numel() // 4 * 4
    t[:n].view(torch.float32).fill_(float("nan"))


def _model(golden_dir, arena=True):
    import vilbert_b200
    cfgj = dict(json.load(open(os.path.join(golden_dir, "tiny_b4.json")))["config"], task_specific_tokens=True, max_position_embeddings=300)
    model = vilbert_b200.VILBertForVLTasks(vilbert_b200.BertConfig.from_dict(cfgj))
    model.load_state_dict(O.synth_params(O.make_config(cfgj), seed=0, device="cuda"), strict=False)
    model.eval()
    if arena:
        model.engine.enable_activation_arena(ARENA)
    return model, cfgj


def _loader(task_id, n=3129):
    return {task_id: types.SimpleNamespace(dataset=types.SimpleNamespace(label2ans=[f"answer {i}" for i in range(n)]))}


def _close(a, b, rel):
    if isinstance(a, dict):
        return a.keys() == b.keys() and all(_close(a[k], b[k], rel) for k in a)
    if isinstance(a, (list, tuple)):
        return len(a) == len(b) and all(_close(x, y, rel) for x, y in zip(a, b))
    if isinstance(a, float):
        return type(b) is float and (a == b or abs(a - b) <= rel * abs(b))
    return type(a) is type(b) and a == b


def _finite(x):
    if isinstance(x, dict):
        return all(_finite(v) for v in x.values())
    if isinstance(x, (list, tuple)):
        return all(_finite(v) for v in x)
    return not isinstance(x, float) or math.isfinite(x)


def _arms(model, call, n=3):
    """(plain, recycled) lists of n calls each; the arena is NaN before each arm's first call. The module surface captures a
    plan's forward into a CUDA graph at its third call, so the last call of each arm is a graph replay."""
    eng = model.engine
    out = {}
    for recycle in (False, True):
        eng.recycle_forward_only = recycle
        _nan_fill(eng.arena)
        out[recycle] = [call() for _ in range(n)]
        assert all(p.recycle == recycle for p in eng.plans.values()), "a forward-only plan of the arm is not of the arm"
        eng.release_plans()
    eng.recycle_forward_only = False
    return out[False], out[True]


@pytest.mark.parametrize("task_id,B,Nv,Nt", CASES, ids=[c[0] for c in CASES])
def test_evaluating_model(golden_dir, deterministic, task_id, B, Nv, Nt):
    from vilbert_b200.tasks import EvaluatingModel, LoadLosses
    model, cfgj = _model(golden_dir)
    tid = task_id if task_id.startswith("TASK") else "TASK12"
    bt = task_id if task_id.startswith("TASK") else "TASK13"
    batch = T.make_batch(cfgj, bt, B, Nv, Nt, options=3)
    if task_id == "BIN_ODD":
        batch = batch[:4] + (torch.rand(B, 2).round(),) + batch[5:]
    cfg = {tid: TASK_CFG[task_id]}
    losses = LoadLosses(None, cfg, [tid[4:]])
    loader = _loader(tid, 1533 if task_id == "TASK15" else 3129)

    def call():
        res = []
        r = EvaluatingModel(None, cfg, DEV, tid, batch, model, loader, losses, res, [])
        return r[:3] + (res,)
    plain, rec = _arms(model, call)
    assert _finite(rec) and len(rec[0][3]) == len(plain[0][3])
    if deterministic:
        assert rec == plain
    else:
        for p, r in zip(plain, rec):
            assert _close(r[3], p[3], 1e-6) and r[1:3] == p[1:3] and _close(r[0], p[0], 1e-5)


@pytest.mark.parametrize("task_id", ["TASK1", "TASK7", "TASK9", "TASK12", "TASK13"])
def test_forward_models_val(golden_dir, deterministic, task_id):
    from vilbert_b200.tasks import ForwardModelsVal, LoadLosses
    model, cfgj = _model(golden_dir)
    batch = T.make_batch(cfgj, task_id, 4 if task_id in ("TASK1", "TASK9", "TASK13") else 2, 11, 9, options=3)
    losses = LoadLosses(None, T.TASK_CFG, [task_id[4:]])
    plain, rec = _arms(model, lambda: ForwardModelsVal(None, T.TASK_CFG, DEV, task_id, batch, model, losses))
    assert _finite(rec)
    if deterministic:
        assert rec == plain
    else:
        for p, r in zip(plain, rec):
            assert r[1:] == p[1:] and _close(r[0], p[0], 1e-5)


def test_module_surface_under_no_grad(golden_dir, deterministic):
    """model(...) under torch.no_grad() with the engine switch set runs the recycled forward-only plan; the heads are the plain
    plan's."""
    model, cfgj = _model(golden_dir)
    inp = O.synth_inputs(O.make_config(cfgj), 4, 11, 9, seed=4, device="cuda", task_id=1)
    args = (inp["input_txt"], inp["input_imgs"], inp["image_loc"], inp["token_type_ids"], inp["attention_mask"], inp["image_attention_mask"])

    def call():
        with torch.no_grad():
            return [t.clone() for t in model(*args, task_ids=inp["task_ids"])[:9]]
    plain, rec = _arms(model, call)
    for p, r in zip(plain, rec):
        for a, b in zip(p, r):
            assert torch.isfinite(b).all()
            assert torch.equal(a, b) if deterministic else torch.allclose(a, b, rtol=1e-5, atol=1e-6)


def test_train_mode_call_under_no_grad_keeps_its_plan(golden_dir):
    """The switch reaches forward-only plans only: a train-mode call under torch.no_grad() takes the plan its training calls
    use, as without the switch (a train-mode plan is never recycled)."""
    model, cfgj = _model(golden_dir)
    model.engine.recycle_forward_only = True
    model.train()
    inp = O.synth_inputs(O.make_config(cfgj), 4, 11, 9, seed=4, device="cuda", task_id=1)
    args = (inp["input_txt"], inp["input_imgs"], inp["image_loc"], inp["token_type_ids"], inp["attention_mask"], inp["image_attention_mask"])
    model(*args, task_ids=inp["task_ids"])[0].sum().backward()
    with torch.no_grad():
        model(*args, task_ids=inp["task_ids"])
    plan = model._last_plan
    assert plan.grad_outputs and not plan.recycle


def _gallery(cfgj, G, Nv, C, Nt, seed):
    cfg = O.make_config(cfgj)
    img = O.synth_inputs(cfg, G, Nv, Nt, seed=seed)
    txt = O.synth_inputs(cfg, C, Nv, Nt, seed=seed + 1)
    return img["input_imgs"], img["image_loc"], img["image_attention_mask"], txt["input_txt"], txt["attention_mask"], txt["token_type_ids"]


@pytest.mark.parametrize("arena", [False, True], ids=["own_region", "arena"])
def test_retrieval_evaluator(golden_dir, deterministic, arena):
    """Scores (bitwise under deterministic algorithms, else to 1e-6) and ranks of RetrievalEvaluator(recycle=True) against
    recycle=False. Each caption after a chunk's first is a graph replay; the recycled plans' bytes are NaN before the first run."""
    from vilbert_b200.retrieval import RetrievalEvaluator
    model, cfgj = _model(golden_dir, arena=arena)
    G, Nv, C, Nt, chunk = 11, 11, 5, 9, 4
    feats, locs, imask, caps, amask, seg = _gallery(cfgj, G, Nv, C, Nt, seed=21)
    target = torch.randint(0, G, (C,))
    out, held = {}, {}
    for recycle in (False, True):
        ev = RetrievalEvaluator(model, feats, locs, imask, chunk=chunk, recycle=recycle)
        plans = [ev._plan(n, Nt) for n in (chunk, G % chunk)]
        assert all(p.recycle == recycle for p in plans)
        for p in plans if recycle else ():
            _nan_fill(p._region)
        scores = ev.score(caps, amask, seg, task_id=8)
        out[recycle] = (scores, *ev.rank(scores, target, k=5))
        held[recycle] = [p.held_bytes for p in plans]
        model.engine.release_plans()
    assert all(r < p for r, p in zip(held[True], held[False]))
    (s0, r0, k0), (s1, r1, k1) = out[False], out[True]
    assert torch.isfinite(s1).all()
    if deterministic:
        assert torch.equal(s0, s1) and torch.equal(r0, r1) and torch.equal(k0, k1)
    else:
        assert (s0 - s1).abs().max().item() <= 1e-6 * s0.abs().max().item()


def test_image_states_survive_another_plan_in_the_arena(golden_dir):
    """A recycled image-prefix plan in the shared arena: another plan's forward between the prefix and the caption replays
    overwrites the arena, the image states are private, and the captions score as without it."""
    model, cfgj = _model(golden_dir)
    eng = model.engine
    model._sync_weights()
    cfg = O.make_config(cfgj)
    B, Nv, Nt = 4, 11, 9
    inp = O.synth_inputs(cfg, B, Nv, Nt, seed=2, device="cuda", task_id=3)
    text = [O.synth_inputs(cfg, 1, Nv, Nt, seed=50 + i, device="cuda", task_id=3) for i in range(4)]
    pre = eng.plan(B, Nt, Nv, outputs=("vil_logit",), fast_mode=True, image_prefix=True, recycle=True)
    other = eng.plan(B, Nt, Nv, outputs=("vil_prediction",), recycle=True)

    def captions():
        got = []
        for t in text:
            pre.load_inputs(t["input_txt"], None, None, t["token_type_ids"], t["attention_mask"], None, t["task_ids"])
            pre.run_forward()
            got.append(pre.outputs["vil_logit"].clone())
        return got
    _nan_fill(eng.arena)
    pre.load_images(inp["input_imgs"], inp["image_loc"], inp["image_attention_mask"])
    pre.run_image_prefix()
    want = captions()
    pre.run_image_prefix()
    _nan_fill(eng.arena)
    other.load_inputs(inp["input_txt"], inp["input_imgs"], inp["image_loc"], inp["token_type_ids"], inp["attention_mask"],
                      inp["image_attention_mask"], inp["task_ids"])
    other.run_forward()
    got = captions()
    for a, b in zip(want, got):
        assert torch.isfinite(a).all() and torch.equal(a, b)


@pytest.mark.parametrize("task_id,Nv,Nt", [("TASK7", 101, 31), ("TASK12", 101, 41)], ids=["VL-logit", "NLVR2"])
def test_evaluating_model_at_b256(golden_dir, task_id, Nv, Nt):
    """VL-logit (4 options: 1,024 rows) and NLVR2 (512 rows) at B = 256 on bert_base_6layer_6conect with task tokens in a 40 GiB
    arena, which their plain plans exceed: the recycled plans fit and give finite losses, scores and results. VL-logit's first 8
    questions get the option probabilities of a B = 8 batch; NLVR2 has no per-row results, and its batch loss and score are means
    over the batch, so it is checked for finite values only."""
    import vilbert_b200
    from vilbert_b200.tasks import EvaluatingModel, LoadLosses
    cfgj = dict(json.load(open(os.path.join(os.path.dirname(golden_dir), "..", "vilbert-multi-task_b200", "configs",
                                            "bert_base_6layer_6conect.json"))), task_specific_tokens=True)
    model = vilbert_b200.VILBertForVLTasks(vilbert_b200.BertConfig.from_dict(cfgj))
    model.eval()
    eng = model.engine
    eng.enable_activation_arena(40 << 30)
    eng.recycle_forward_only = True
    cfg = {task_id: T.TASK_CFG[task_id]}
    losses = LoadLosses(None, cfg, [task_id[4:]])
    batch = T.make_batch(cfgj, task_id, 256, Nv, Nt, options=4, seed=5)     # NLVR2: two images of Nv regions per sample
    res = []
    r = EvaluatingModel(None, cfg, DEV, task_id, batch, model, _loader(task_id), losses, res, [])
    assert _finite(r[:3]) and _finite(res) and r[2] == 256
    assert all(p.recycle and p.arena_bytes <= eng.arena.numel() for p in eng.plans.values())
    small = tuple(t[:8] for t in batch)
    res8 = []
    EvaluatingModel(None, cfg, DEV, task_id, small, model, _loader(task_id), losses, res8, [])
    if task_id == "TASK7":
        assert _close(res[:8], res8, 2e-3)
