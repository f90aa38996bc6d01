"""Packed retrieval on the GPU: vb_pack_segments and vb_broadcast_segment_rows against torch references, and RetrievalEvaluator with
pack=True against the padded evaluation (and the fp32 oracle) on ragged galleries, captions of every length, with and without task
tokens and for the zero-shot pre-training model; with recycled plans, the shared arena, fallbacks mixed in, deterministic
algorithms, and evaluate_retrieval end to end."""
import json
import os

import pytest
import torch

import _packed_ref as P
from oracle import vilbert_oracle as O

pytestmark = pytest.mark.gpu
I32 = torch.int32


def _st():
    return torch.cuda.current_stream().cuda_stream


def _prefix(lens, n):
    return (torch.arange(n) < torch.as_tensor(lens).unsqueeze(1)).long()


# ------------------------------------------------------------------------------------------ kernels
@pytest.mark.parametrize("B,N,has_task,rows", [(1, 30, 1, 31), (1, 9, 0, 9), (500, 101, 0, 31000), (64, 36, 1, 1000), (7, 20, 1, 30)])
def test_pack_segments_against_the_reference_layout(B, N, has_task, rows):
    from vilbert_b200 import _lib as L
    g = torch.Generator().manual_seed(B * N + rows)
    lens = torch.randint(1, N + 1, (B,), generator=g)
    lens[0] = 1
    lens[-1] = N
    mask = _prefix(lens, N)
    off, ln, mp = (torch.full((n,), 7, dtype=I32, device="cuda") for n in (B + 1, B, rows))
    L.call(L.lib().vb_pack_segments, mask.cuda(), N, has_task, B, rows, off, ln, mp)
    ro, rl, rm = P.pack_layout(mask, has_task, rows)          # a capacity below the valid rows clamps, as vb_pack_build does
    assert torch.equal(off.cpu(), ro) and torch.equal(ln.cpu(), rl) and torch.equal(mp.cpu(), rm)


@pytest.mark.parametrize("dtype", [torch.float32, torch.float16, torch.bfloat16])
@pytest.mark.parametrize("Nt_in,has_task,L_in", [(30, 1, 0), (30, 1, 30), (30, 0, 1), (30, 0, 17), (9, 1, 5), (30, 0, 30)])
def test_broadcast_segment_rows_against_torch(dtype, Nt_in, has_task, L_in):
    """The caption's rows from its one-sample segment (built by vb_pack_segments from the mask, task token included) repeated n
    times, bitwise, and every row after n * L zero, whatever the buffer held."""
    from vilbert_b200 import _lib as L
    from vilbert_b200.engine import pack_capacity
    lib = L.lib()
    Nt, H, n = Nt_in + has_task, 768, 37
    m = _prefix([L_in], Nt_in).cuda()
    if L_in == 0:
        m = torch.ones_like(m)                              # L = Nt: every row valid
    Lv = int(m.sum()) + has_task
    off, ln, mp = torch.zeros(2, dtype=I32, device="cuda"), torch.zeros(1, dtype=I32, device="cuda"), torch.zeros(Nt, dtype=I32, device="cuda")
    L.call(lib.vb_pack_segments, m, Nt_in, has_task, 1, Nt, off, ln, mp)
    assert int(ln[0]) == Lv
    rows = pack_capacity(n * Lv, n * Nt)
    src = torch.randn(Nt, H, device="cuda").to(dtype)
    lo = torch.randn(Nt, H, device="cuda").to(dtype)        # a second 16-bit copy (the split-precision low part) in the same launch shape
    for s in (src, lo):
        dst = torch.full((rows, H), 3.0, device="cuda").to(dtype)
        L.call(lib.vb_broadcast_segment_rows, s, dst, H * s.element_size(), ln, n, rows)
        ref = torch.zeros_like(dst)
        ref[:n * Lv] = s[:Lv].repeat(n, 1)
        assert torch.equal(dst.view(torch.int16 if dtype != torch.float32 else torch.int32),
                           ref.view(torch.int16 if dtype != torch.float32 else torch.int32))
    # a capacity below n * L keeps the whole segments that fit and the part of the last one
    small = torch.full((Lv * 2 + 1, H), 3.0, device="cuda").to(dtype)
    L.call(lib.vb_broadcast_segment_rows, src, small, H * src.element_size(), ln, n, small.shape[0])
    assert torch.equal(small, src[:Lv].repeat(3, 1)[:small.shape[0]])
    assert lib.vb_broadcast_segment_rows(src.data_ptr(), small.data_ptr(), 24, ln.data_ptr(), n, 4, _st()) != 0


# ------------------------------------------------------------------------------------------ packed against padded
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _cfgj(golden_dir, base, **over):
    if base:
        cfgj = json.load(open(os.path.join(ROOT, "vilbert-multi-task_b200", "configs", "bert_base_6layer_6conect.json")))
    else:
        cfgj = json.load(open(os.path.join(golden_dir, "tiny_b4.json")))["config"]
    return dict(cfgj, max_position_embeddings=max(cfgj.get("max_position_embeddings", 0), 300), **over)


def _model(cfgj, zero_shot=False, precision="fp16"):
    import vilbert_b200
    cls = vilbert_b200.BertForMultiModalPreTraining if zero_shot else vilbert_b200.VILBertForVLTasks
    model = cls(vilbert_b200.BertConfig.from_dict(cfgj), precision=precision)
    P_ = O.synth_params(O.make_config(cfgj), seed=0, device="cuda", with_task_heads=not zero_shot)
    model.load_state_dict(P_, strict=False)
    model.eval()
    return model, P_


def _gallery(cfgj, G, Nv, Nt, chunk, seed):
    """Ragged prefix-valid image masks with chunk 1 all valid, and one caption of every length 1 .. Nt."""
    cfg = O.make_config(cfgj)
    img = O.synth_inputs(cfg, G, Nv, Nt, seed=seed)
    g = torch.Generator().manual_seed(seed)
    lens = torch.randint(1, Nv + 1, (G,), generator=g)
    lens[chunk:2 * chunk] = Nv
    imask = _prefix(lens, Nv)
    feats = img["input_imgs"] * imask.unsqueeze(-1)
    caps = torch.randint(0, cfgj["vocab_size"], (Nt, Nt), generator=g)
    amask = _prefix(torch.arange(1, Nt + 1), Nt)
    return feats, img["image_loc"], imask, caps, amask, torch.zeros_like(caps)


def _near_ties(row, t, d):
    gap = (row - row[t]).abs()
    gap[t] = float("inf")
    return bool(gap.min() <= 2 * d)


def _compare(ev, packed, padded, bound):
    """max|Δ| / max|padded| within `bound`; ranks and top-k equal except for captions whose target sits within 2 max|Δ| of another
    image's score. -> (relative difference, number of such captions)."""
    d = (packed - padded).abs().max().item()
    r = d / padded.abs().max().item()
    assert r <= bound, r
    C, G = padded.shape
    target = torch.arange(C) % G
    rk_p, tk_p = ev.rank(packed, target, k=min(5, G))
    rk_q, tk_q = ev.rank(padded, target, k=min(5, G))
    near = 0
    for c in range(C):
        t = int(target[c])
        if _near_ties(padded[c], t, d):
            near += 1
            continue
        assert int(rk_p[c]) == int(rk_q[c]), c
    moved = [c for c in range(C) if not torch.equal(tk_p[c], tk_q[c])]
    assert all(any(_near_ties(padded[c], int(j), d) for j in tk_q[c]) for c in moved), moved
    return r, near


@pytest.mark.parametrize("precision", ["fp16", "fp32"])
@pytest.mark.parametrize("task_tokens", [False, True])
@pytest.mark.parametrize("base", [False, True], ids=["tiny", "base66"])
def test_packed_scores_match_the_padded_evaluation(golden_dir, precision, task_tokens, base):
    from _gpu_util import rel
    from vilbert_b200.retrieval import RetrievalEvaluator
    cfgj = _cfgj(golden_dir, base, task_specific_tokens=task_tokens)
    G, Nv, Nt, chunk = (7, 101, 30, 3) if base else (11, 11, 9, 4)        # chunks 3 + 3 + 1 / 4 + 4 + 3: an uneven last chunk
    model, P_ = _model(cfgj, precision=precision)
    feats, locs, imask, caps, amask, seg = _gallery(cfgj, G, Nv, Nt, chunk, seed=41)
    padded = RetrievalEvaluator(model, feats, locs, imask, chunk=chunk, pack=False).score(caps, amask, seg, task_id=8)
    ev = RetrievalEvaluator(model, feats, locs, imask, chunk=chunk, pack=True)
    packed = ev.score(caps, amask, seg, task_id=8)
    assert not model.engine.pack_fallbacks
    assert any(p.packed for p in model.engine.plans.values())
    r, near = _compare(ev, packed, padded, 1e-4 if precision == "fp32" else 1e-3)
    print(f"packed vs padded: max|d|/max|padded| {r:.2e}, {near} of {Nt} captions with a near tie at the target")
    if precision == "fp32":
        # the north-star contract of the fp32 oracle, for both evaluations
        cfg = O.make_config(cfgj)
        cs = range(Nt) if not base else (0, Nt // 2, Nt - 1)
        for c in cs:
            task = torch.full((G, 1), 8, dtype=torch.long, device="cuda") if task_tokens else None
            _, heads = O.vilbert_for_vl_tasks(P_, cfg, caps[c:c + 1].expand(G, -1).cuda(), feats.cuda(), locs.cuda(),
                                              seg[c:c + 1].expand(G, -1).cuda(), amask[c:c + 1].expand(G, -1).cuda(), imask.cuda(),
                                              None, task)
            ref = heads[O.HEAD_NAMES.index("vil_logit")].reshape(-1)
            assert rel(packed[c], ref) < 1e-2 and rel(padded[c], ref) < 1e-2, c


@pytest.mark.parametrize("precision", ["fp16", "fp32"])
def test_zero_shot_packed_scores_match_the_padded_evaluation(golden_dir, precision):
    from vilbert_b200.retrieval import RetrievalEvaluator
    cfgj = _cfgj(golden_dir, False)
    model, _ = _model(cfgj, zero_shot=True, precision=precision)
    feats, locs, imask, caps, amask, seg = _gallery(cfgj, 9, 11, 9, 4, seed=43)
    padded = RetrievalEvaluator(model, feats, locs, imask, chunk=4, pack=False).score(caps, amask, seg)
    ev = RetrievalEvaluator(model, feats, locs, imask, chunk=4, pack=True)
    packed = ev.score(caps, amask, seg)
    plans = [p for p in model.engine.plans.values() if p.packed]
    assert plans and all(list(p.outputs)[-1] == "seq_relationship_score" for p in plans)
    _compare(ev, packed, padded, 1e-4 if precision == "fp32" else 1e-3)


# ------------------------------------------------------------------------------------------ combinations
def test_recycled_packed_plans_and_mixed_fallbacks(golden_dir):
    from vilbert_b200.retrieval import RetrievalEvaluator
    cfgj = _cfgj(golden_dir, False, task_specific_tokens=True)
    model, _ = _model(cfgj)
    feats, locs, imask, caps, amask, seg = _gallery(cfgj, 11, 11, 9, 4, seed=47)
    packed = RetrievalEvaluator(model, feats, locs, imask, chunk=4, pack=True).score(caps, amask, seg, task_id=8)
    recycled = RetrievalEvaluator(model, feats, locs, imask, chunk=4, pack=True, recycle=True).score(caps, amask, seg, task_id=8)
    assert torch.equal(recycled, packed)
    assert any(p.packed and p.recycle for p in model.engine.plans.values())
    # chunk 2 (images 8 .. 10) holds a mask with a hole, caption 3 too: they run padded, everything else packed
    imask2, amask2 = imask.clone(), amask.clone()
    imask2[9] = 1; imask2[9, 2] = 0
    amask2[3] = 1; amask2[3, 1] = 0
    ev = RetrievalEvaluator(model, feats, locs, imask2, chunk=4, pack=True)
    mixed = ev.score(caps, amask2, seg, task_id=8)
    assert model.engine.pack_fallbacks["mask"] == 2
    padded = RetrievalEvaluator(model, feats, locs, imask2, chunk=4, pack=False).score(caps, amask2, seg, task_id=8)
    _compare(ev, mixed, padded, 1e-3)
    assert torch.equal(mixed[3], padded[3]) and torch.equal(mixed[:, 8:], padded[:, 8:])


def test_packed_image_states_survive_caption_forwards_and_another_plan_in_the_arena(golden_dir):
    from _gpu_util import build_engine
    cfgj = _cfgj(golden_dir, False)
    cfg = O.make_config(cfgj)
    eng = build_engine(cfgj, O.synth_params(cfg, seed=1, device="cuda"), "cuda", "fp32")
    eng.enable_activation_arena(256 << 20)
    B, Nv, Nt = 4, 11, 9
    inp = O.synth_inputs(cfg, B, Nv, Nt, seed=2, device="cuda")
    im = inp["image_attention_mask"]
    from vilbert_b200.engine import pack_capacity
    pre = eng.plan(B, Nt, Nv, outputs=("vil_logit",), fast_mode=True, image_prefix=True,
                   packed=(B * Nt, pack_capacity(int(im.sum()), B * Nv)))
    pre.load_images(inp["input_imgs"], inp["image_loc"], im)
    pre.run_image_prefix()
    states = [t.clone() for t in pre.image_states if t is not None]

    def caption(seed):
        o = O.synth_inputs(cfg, 1, Nv, Nt, seed=seed, device="cuda")
        pre.load_inputs(o["input_txt"], None, None, o["token_type_ids"], o["attention_mask"], None, None)
        pre.run_forward()
        return pre.outputs["vil_logit"].clone()
    first = caption(3)
    for i in range(6):
        caption(100 + i)
        full = eng.plan(B, Nt, Nv)             # another plan over the same arena, with other images, between caption forwards
        o = O.synth_inputs(cfg, B, Nv, Nt, seed=9 + i, device="cuda")
        full.load_inputs(o["input_txt"], o["input_imgs"], o["image_loc"], o["token_type_ids"], o["attention_mask"],
                         o["image_attention_mask"], o["task_ids"])
        full.run_forward()
    for a, b in zip(states, (t for t in pre.image_states if t is not None)):
        assert torch.equal(a, b)
    assert torch.equal(caption(3), first)


def test_packed_evaluation_is_bitwise_reproducible_under_deterministic_algorithms(golden_dir):
    from vilbert_b200.retrieval import RetrievalEvaluator
    cfgj = _cfgj(golden_dir, False, task_specific_tokens=True)
    model, _ = _model(cfgj)
    feats, locs, imask, caps, amask, seg = _gallery(cfgj, 11, 11, 9, 4, seed=53)
    prev, warn_only = torch.are_deterministic_algorithms_enabled(), torch.is_deterministic_algorithms_warn_only_enabled()
    try:
        torch.use_deterministic_algorithms(True)
        ev = RetrievalEvaluator(model, feats, locs, imask, chunk=4, pack=True)
        a = ev.score(caps, amask, seg, task_id=8)
        b = ev.score(caps, amask, seg, task_id=8)
        assert all(p.det for p in model.engine.plans.values() if p.packed)
    finally:
        torch.use_deterministic_algorithms(prev, warn_only=warn_only)
    assert torch.equal(a, b)


def test_evaluate_retrieval_packed_end_to_end(golden_dir):
    """evaluate_retrieval(pack=True) against the padded run, on a gallery laid out as tests/golden/retrieval_reference.json's
    (captions_per_image captions per image, caption c -> image c // captions_per_image) with ragged image masks."""
    from test_retrieval_cpu import _FakeDataset
    from vilbert_b200.retrieval import evaluate_retrieval
    g = json.load(open(os.path.join(golden_dir, "retrieval_reference.json")))
    per = g["captions_per_image"]
    cfgj = _cfgj(golden_dir, False, task_specific_tokens=True)
    model, _ = _model(cfgj)
    H = 5
    ds = _FakeDataset(2 * H * per, H, [[c // per] for c in range(2 * H * per)], Nv=11, Nt=9, F=cfgj["v_feature_size"])
    ds.mask = _prefix(torch.randint(1, 12, (2 * H,), generator=torch.Generator().manual_seed(5)), 11)
    ds.feat = torch.relu(ds.feat) * ds.mask.unsqueeze(-1)
    ds.cap = ds.cap % cfgj["vocab_size"]
    padded = evaluate_retrieval(model, ds, task_id="TASK8", chunk=4, k=10, pack=False)
    packed = evaluate_retrieval(model, ds, task_id="TASK8", chunk=4, k=10, pack=True)
    assert any(p.packed for p in model.engine.plans.values()) and not model.engine.pack_fallbacks
    assert packed[:5] == padded[:5]
    assert packed[5] == padded[5]
