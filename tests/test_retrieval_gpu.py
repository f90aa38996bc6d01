"""Caption-to-image retrieval on the GPU: vb_retrieval_rank against np.argsort(-s, kind="stable"), image_prefix plans against the
ordinary fast-mode plan and the fp32 oracle, the image states across caption forwards and other plans, and RetrievalEvaluator /
evaluate_retrieval against the reference loop restated on the module surface."""
import ctypes as C
import json
import os

import numpy as np
import pytest
import torch

from oracle import vilbert_oracle as O

pytestmark = pytest.mark.gpu
S = lambda: C.c_void_p(torch.cuda.current_stream().cuda_stream)
NAN = float("nan")
TOL = 1e-6


def _np_rank(s, t):
    order = np.argsort(-s, kind="stable")
    return (int(np.where(order == t)[0][0]) if 0 <= t < len(s) else -1), order


# ------------------------------------------------------------------------------------------ vb_retrieval_rank
@pytest.mark.parametrize("N", [1, 7, 500, 1000, 5000])
def test_rank_kernel_against_numpy(N):
    from vilbert_b200 import _lib as L
    from vilbert_b200.retrieval import RetrievalEvaluator
    R = 9
    g = torch.Generator().manual_seed(N)
    s = (torch.randn(R, N, generator=g) * 2).round(decimals=1)          # ties are common
    s[1, ::3] = NAN
    s[2, :] = 0.0
    s[2, ::2] = -0.0
    s[3, :] = NAN
    s[4, N // 2:] = s[4].max()
    target = torch.randint(0, N, (R,), generator=g)
    target[5], target[6] = -1, N                                         # outside the gallery
    pitch = N + 5
    buf = torch.full((R, pitch), 7.0)
    buf[:, :N] = s
    dev = buf.cuda()
    for k in sorted({1, 20, min(N + 3, 64), 64}):
        ranks, topk = RetrievalEvaluator.rank(dev[:, :N], target, k=k)
        for r in range(R):
            rk, order = _np_rank(s[r].numpy(), int(target[r]))
            assert int(ranks[r]) == rk, (r, k)
            kk = min(k, N)
            assert topk[r, :kk].tolist() == order[:kk].tolist(), (r, k)
            assert (topk[r, kk:] == -1).all()
    # errors are statuses, not faults
    rk32 = torch.empty(R, dtype=torch.int32, device="cuda")
    tk = torch.empty(R, 65, dtype=torch.int32, device="cuda")
    t64 = target.cuda()
    assert L.lib().vb_retrieval_rank(dev.data_ptr(), pitch, R, N, t64.data_ptr(), 65, rk32.data_ptr(), tk.data_ptr(), S()) != 0
    big = torch.zeros(1, 50001, device="cuda")
    assert L.lib().vb_retrieval_rank(big.data_ptr(), 50001, 1, 50001, t64.data_ptr(), 1, rk32.data_ptr(), tk.data_ptr(), S()) != 0
    assert "50000" in L.lib().vb_last_error().decode()
    torch.cuda.synchronize()


def test_rank_kernel_at_the_largest_gallery():
    from vilbert_b200.retrieval import RetrievalEvaluator
    N = 50000
    s = torch.randn(3, N)
    s[1, 100:200] = 0.5
    t = torch.tensor([3, 150, N - 1])
    ranks, topk = RetrievalEvaluator.rank(s.cuda(), t, k=64)
    for r in range(3):
        rk, order = _np_rank(s[r].numpy(), int(t[r]))
        assert int(ranks[r]) == rk and topk[r].tolist() == order[:64].tolist()


# ------------------------------------------------------------------------------------------ image_prefix plans
def _cfg(golden_dir, base, **over):
    if base:
        path = os.path.join(os.path.dirname(golden_dir), "..", "vilbert-multi-task_b200", "configs", "bert_base_6layer_6conect.json")
        cfgj = json.load(open(path))
    else:
        cfgj = json.load(open(os.path.join(golden_dir, "tiny_b4.json")))["config"]
    return dict(cfgj, **over)


def _fast_inputs(cfg, B, Nv, Nt, seed):
    inp = O.synth_inputs(cfg, B, Nv, Nt, seed=seed, device="cuda", task_id=3 if cfg.get("task_specific_tokens") else None)
    for k in ("input_txt", "token_type_ids", "attention_mask", "task_ids"):
        if inp.get(k) is not None:
            inp[k] = inp[k][:1].contiguous()
    return inp


def _text(plan, inp):
    plan.load_inputs(inp["input_txt"], None, None, inp["token_type_ids"], inp["attention_mask"], None, inp["task_ids"])


@pytest.mark.parametrize("precision", ["fp16", "fp32"])
@pytest.mark.parametrize("base", [False, True], ids=["tiny", "base66"])
def test_prefix_plan_matches_the_ordinary_fast_plan(golden_dir, precision, base):
    from _gpu_util import build_engine, rel
    cfgj = _cfg(golden_dir, base, task_specific_tokens=True, max_position_embeddings=300)
    cfg = O.make_config(cfgj)
    B, Nv, Nt = (6, 101, 31) if base else (4, 11, 9)
    P = O.synth_params(cfg, seed=0, device="cuda")
    eng = build_engine(cfgj, P, "cuda", precision)
    inp = _fast_inputs(cfg, B, Nv, Nt, seed=5)
    kw = dict(outputs=("vil_logit",), fast_mode=True)
    ordinary = eng.plan(B, Nt, Nv, **kw)
    runs = []
    for _ in range(2):
        ordinary.load_inputs(inp["input_txt"], inp["input_imgs"], inp["image_loc"], inp["token_type_ids"], inp["attention_mask"],
                             inp["image_attention_mask"], inp["task_ids"])
        ordinary.run_forward()
        runs.append(ordinary.outputs["vil_logit"].clone())
    pre = eng.plan(B, Nt, Nv, image_prefix=True, **kw)
    pre.load_images(inp["input_imgs"], inp["image_loc"], inp["image_attention_mask"])
    pre.run_image_prefix()
    _text(pre, inp)
    pre.run_forward()
    got = pre.outputs["vil_logit"].clone()
    if torch.equal(runs[0], runs[1]):
        assert torch.equal(got, runs[0]), (got - runs[0]).abs().max()
    else:
        assert ((got - runs[0]).abs().max() / runs[0].abs().max()).item() <= TOL
    if not base and precision == "fp32":
        txt = {k: (v.expand(B, *v.shape[1:]) if v is not None and k in ("input_txt", "token_type_ids", "attention_mask", "task_ids")
                   else v) for k, v in inp.items()}
        _, heads = O.vilbert_for_vl_tasks(P, cfg, txt["input_txt"], txt["input_imgs"], txt["image_loc"], txt["token_type_ids"],
                                          txt["attention_mask"], txt["image_attention_mask"], txt.get("co_attention_mask"), txt["task_ids"])
        assert rel(got, heads[O.HEAD_NAMES.index("vil_logit")].reshape(got.shape)) < 1e-2


@pytest.mark.parametrize("arena", [False, True])
def test_image_states_survive_caption_forwards_and_other_plans(golden_dir, arena):
    from _gpu_util import build_engine
    cfgj = _cfg(golden_dir, False)
    cfg = O.make_config(cfgj)
    eng = build_engine(cfgj, O.synth_params(cfg, seed=1, device="cuda"), "cuda", "fp32")
    if arena:
        eng.enable_activation_arena(256 << 20)
    B, Nv, Nt = 4, 11, 9
    inp = _fast_inputs(cfg, B, Nv, Nt, seed=2)
    pre = eng.plan(B, Nt, Nv, outputs=("vil_logit",), fast_mode=True, image_prefix=True)
    pre.load_images(inp["input_imgs"], inp["image_loc"], inp["image_attention_mask"])
    pre.run_image_prefix()
    states = [t.clone() for t in pre.image_states if t is not None]
    _text(pre, inp)
    pre.run_forward()
    first = pre.outputs["vil_logit"].clone()
    for i in range(12):
        other = _fast_inputs(cfg, B, Nv, Nt, seed=100 + i)
        _text(pre, other)
        pre.run_forward()
    # another plan over the same arena, with other images
    full = eng.plan(B, Nt, Nv)
    o = O.synth_inputs(cfg, B, Nv, Nt, seed=9, device="cuda")
    full.load_inputs(o["input_txt"], o["input_imgs"], o["image_loc"], o["token_type_ids"], o["attention_mask"], o["image_attention_mask"],
                     o["task_ids"])
    full.run_forward()
    for a, b in zip(states, (t for t in pre.image_states if t is not None)):
        assert torch.equal(a, b)
    _text(pre, inp)
    pre.run_forward()
    assert torch.equal(pre.outputs["vil_logit"], first)


# ------------------------------------------------------------------------------------------ RetrievalEvaluator
def _vl_model(golden_dir, task_tokens):
    import vilbert_b200
    cfgj = _cfg(golden_dir, False, task_specific_tokens=task_tokens, max_position_embeddings=300)
    model = vilbert_b200.VILBertForVLTasks(vilbert_b200.BertConfig.from_dict(cfgj))
    model.load_state_dict(O.synth_params(O.make_config(cfgj), seed=0, device="cuda"), strict=False)
    model.eval()
    return model, cfgj


def _pre_model(golden_dir):
    import vilbert_b200
    cfgj = _cfg(golden_dir, False)
    model = vilbert_b200.BertForMultiModalPreTraining(vilbert_b200.BertConfig.from_dict(cfgj))
    sd = O.synth_params(O.make_config(cfgj), seed=0, device="cuda", with_task_heads=False)
    model.load_state_dict(sd, strict=False)
    model.eval()
    return model, cfgj


def _gallery(cfgj, G, Nv, C, Nt, seed):
    cfg = O.make_config(cfgj)
    img = O.synth_inputs(cfg, G, Nv, Nt, seed=seed)
    txt = O.synth_inputs(cfg, C, Nv, Nt, seed=seed + 1)
    return img["input_imgs"], img["image_loc"], img["image_attention_mask"], txt["input_txt"], txt["attention_mask"], txt["token_type_ids"]


def _module_loop(model, feats, locs, imask, caps, amask, seg, task, chunk, zero_shot):
    """eval_retrieval.py:264-313 on the module surface, one call per caption and image chunk with config.fast_mode set."""
    model.config.fast_mode = True
    model.engine.cfg.fast_mode = True
    try:
        G = feats.shape[0]
        out = torch.empty(caps.shape[0], G, device="cuda")
        with torch.no_grad():
            for c in range(caps.shape[0]):
                for lo in range(0, G, chunk):
                    sl = slice(lo, lo + chunk)
                    args = (caps[c:c + 1].cuda(), feats[sl].cuda(), locs[sl].cuda(), seg[c:c + 1].cuda(), amask[c:c + 1].cuda(), imask[sl].cuda())
                    if zero_shot:
                        _, _, logit, _ = model(*args)
                        out[c, sl] = torch.softmax(logit, dim=1)[:, 0]
                    else:
                        tt = None if task is None else torch.full((1, 1), task, dtype=torch.long, device="cuda")
                        out[c, sl] = model(*args, task_ids=tt)[2].view(-1)
        return out
    finally:
        model.config.fast_mode = False
        model.engine.cfg.fast_mode = False


def _check_against_loop(ev, scores, loop, target):
    scale = loop.abs().max().item()
    assert (scores - loop).abs().max().item() <= TOL * scale
    ranks, topk = ev.rank(scores, target, k=5)
    ranks_l, _ = ev.rank(loop, target, k=5)
    for c in range(scores.shape[0]):
        if int(ranks[c]) != int(ranks_l[c]):
            row, t = loop[c], int(target[c])
            gap = (row - row[t]).abs()
            gap[t] = float("inf")
            assert gap.min().item() <= TOL * scale


@pytest.mark.parametrize("task_tokens", [False, True])
def test_evaluator_matches_the_module_loop(golden_dir, task_tokens):
    from vilbert_b200.retrieval import RetrievalEvaluator
    model, cfgj = _vl_model(golden_dir, task_tokens)
    G, Nv, C, Nt, chunk = 11, 11, 5, 9, 4
    feats, locs, imask, caps, amask, seg = _gallery(cfgj, G, Nv, C, Nt, seed=21)
    ev = RetrievalEvaluator(model, feats, locs, imask, chunk=chunk)          # host gallery: pinned staging
    scores = ev.score(caps, amask, seg, task_id="TASK8")
    assert scores.shape == (C, G) and scores.is_cuda
    loop = _module_loop(model, feats, locs, imask, caps, amask, seg, 8 if task_tokens else None, chunk, False)
    target = torch.randint(0, G, (C,))
    _check_against_loop(ev, scores, loop, target)
    # a device gallery gives the same scores
    ev2 = RetrievalEvaluator(model, feats.cuda(), locs.cuda(), imask.cuda(), chunk=chunk)
    assert torch.equal(ev2.score(caps, amask, seg, task_id=8), scores)
    model.train()
    with pytest.raises(ValueError):
        ev.score(caps, amask, seg, task_id=8)
    with pytest.raises(ValueError):
        RetrievalEvaluator(model, feats, locs, imask)


def test_zero_shot_evaluator_matches_the_module_loop(golden_dir):
    from vilbert_b200.retrieval import RetrievalEvaluator
    model, cfgj = _pre_model(golden_dir)
    G, Nv, C, Nt, chunk = 9, 11, 4, 9, 5
    feats, locs, imask, caps, amask, seg = _gallery(cfgj, G, Nv, C, Nt, seed=31)
    ev = RetrievalEvaluator(model, feats, locs, imask, chunk=chunk)
    with pytest.raises(TypeError):
        ev.score(caps, amask, seg, task_id=8)
    scores = ev.score(caps, amask, seg)
    loop = _module_loop(model, feats, locs, imask, caps, amask, seg, None, chunk, True)
    _check_against_loop(ev, scores, loop, torch.randint(0, G, (C,)))
    c = model.config
    plans = [p for p in model.engine.plans.values() if p.image_prefix]
    assert plans
    for p in plans:
        assert "linguisic_prediction" not in p.outputs and "vision_prediction" not in p.outputs
        ns = [args[0]._obj.N for fn, args, _ in p.fwd + p.prefix if fn is not None and fn.__name__ == "vb_gemm_bf16"]
        assert not {c.vocab_size, c.v_target_size} & set(ns)


def test_evaluate_retrieval_end_to_end(golden_dir):
    from test_retrieval_cpu import _FakeDataset
    from vilbert_b200.retrieval import evaluate_retrieval, read_retrieval_dataset, retrieval_metrics
    model, cfgj = _vl_model(golden_dir, True)
    ds = _FakeDataset(6, 5, [[0], [9], [3, 7], [5], [2], [8]], Nv=11, Nt=9, F=cfgj["v_feature_size"])
    ds.feat = torch.relu(ds.feat)
    ds.cap = ds.cap % cfgj["vocab_size"]
    model.train()
    r1, r5, r10, medr, meanr, results = evaluate_retrieval(model, ds, task_id="TASK8", chunk=4, k=20)
    assert not model.training
    feats, locs, imask, caps, amask, seg, target = read_retrieval_dataset(ds)
    loop = _module_loop(model, feats, locs, imask, caps, amask, seg, 8, 4, False).cpu().numpy()
    ranks = [_np_rank(row, int(t))[0] for row, t in zip(loop, target)]
    assert (r1, r5, r10, medr, meanr) == retrieval_metrics(ranks)
    assert len(results) == 6 and all(len(r) == 10 for r in results)
    for r, row in zip(results, loop):
        best = int(np.argsort(-row, kind="stable")[0])
        assert r[0] == best or abs(row[r[0]] - row[best]) <= TOL * np.abs(loop).max()
