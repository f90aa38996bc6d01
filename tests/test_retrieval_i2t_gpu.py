"""Image-to-text retrieval on the GPU: vb_retrieval_rank_sets against the numpy set rank (ties, signed zeros, infinities, NaN, sets of
0 to 7 captions with indices outside the row, up to 50,000 columns), bitwise equal to vb_retrieval_rank on one-element sets, its
refusals, RetrievalEvaluator.rank_captions, and evaluate_retrieval_both against numpy rankings of the score matrix it ranked and
against evaluate_retrieval, on the tiny config and bert_base_6layer_6conect, fine-tuned and zero-shot, padded and packed."""
import ctypes as C
import json
import os

import numpy as np
import pytest
import torch

from oracle import vilbert_oracle as O
from test_retrieval_cpu import _FakeDataset, stable_desc
from test_retrieval_i2t_cpu import set_rank

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
S = lambda: C.c_void_p(torch.cuda.current_stream().cuda_stream)
I32, I64 = torch.int32, torch.int64
SENTINEL = 777


def _scores(R, N, g):
    """Quantised scores (ties) with signed zeros, infinities and NaNs spread over every row, and rows made of them."""
    s = (torch.randn(R, N, generator=g) * 2).round(decimals=1)
    for v in (0.0, -0.0, float("inf"), float("-inf"), float("nan")):
        s[torch.rand(R, N, generator=g) < 0.03] = v
    s[1, ::3] = float("nan")
    s[2, :] = 0.0
    s[2, ::2] = -0.0
    s[3, :] = float("nan")
    s[4, N // 2:] = s[4].nan_to_num(nan=0.0, posinf=0.0).max()
    return s


def _sets(R, N, g):
    """CSR sets of 0 to 7 targets per row, about a fifth of them outside [0, N); row 0 is empty, row 5 out of range only."""
    sizes = torch.randint(0, 8, (R,), generator=g)
    sizes[0], sizes[5], sizes[6] = 0, 3, 7
    off = torch.zeros(R + 1, dtype=I64)
    off[1:] = sizes.cumsum(0)
    idx = torch.randint(0, N, (int(off[-1]),), generator=g)
    bad = torch.rand(len(idx), generator=g) < 0.2
    idx[bad] = torch.tensor([-1, N, N + 100, -7])[torch.randint(0, 4, (int(bad.sum()),), generator=g)]
    idx[off[5]:off[6]] = torch.tensor([-1, N, N + 3])
    return off, idx


def _run_sets(dev, pitch, R, N, off, idx, k):
    from vilbert_b200 import _lib as L
    ranks = torch.full((R,), SENTINEL, dtype=I32, device="cuda")
    topk = torch.full((R, k), SENTINEL, dtype=I32, device="cuda")
    L.call(L.lib().vb_retrieval_rank_sets, dev, pitch, R, N, off.cuda(), idx.cuda(), k, ranks, topk)
    return ranks.cpu(), topk.cpu()


# ------------------------------------------------------------------------------------------ vb_retrieval_rank_sets
@pytest.mark.parametrize("N", [1, 5000, 25000, 50000])
def test_rank_sets_kernel_against_numpy(N):
    R = 16
    g = torch.Generator().manual_seed(N)
    s = _scores(R, N, g)
    off, idx = _sets(R, N, g)
    pitch = N + 3
    buf = torch.full((R, pitch), 7.0)
    buf[:, :N] = s
    dev = buf.cuda()
    sn = s.numpy()
    orders = [stable_desc(row) for row in sn]
    want = [set_rank(sn[r], idx[off[r]:off[r + 1]].numpy()) for r in range(R)]
    assert want[0] == -1 and want[5] == -1
    for k in (1, 20, 64):
        ranks, topk = _run_sets(dev, pitch, R, N, off, idx, k)
        assert ranks.tolist() == want, k
        kk = min(k, N)
        for r in range(R):
            assert topk[r, :kk].tolist() == orders[r][:kk].tolist(), (r, k)
            assert (topk[r, kk:] == -1).all()


@pytest.mark.parametrize("N", [7, 5000])
def test_one_element_sets_equal_vb_retrieval_rank_bitwise(N):
    from vilbert_b200.retrieval import RetrievalEvaluator
    R = 11
    g = torch.Generator().manual_seed(N + 1)
    dev = _scores(R, N, g).cuda()
    target = torch.randint(0, N, (R,), generator=g)
    target[5], target[6], target[7] = -1, N, N + 9
    off = torch.arange(R + 1, dtype=I64)
    for k in (1, 20, 64):
        ranks, topk = RetrievalEvaluator.rank(dev, target, k=k)
        r2, t2 = _run_sets(dev, N, R, N, off, target, k)
        assert torch.equal(ranks.cpu(), r2) and torch.equal(topk.cpu(), t2), k


def test_rank_sets_refusals_write_nothing():
    from vilbert_b200 import _lib as L
    lib = L.lib()
    N, R = 50001, 2
    big = torch.zeros(R, N, device="cuda")
    off = torch.tensor([0, 1, 2], dtype=I64, device="cuda")
    idx = torch.tensor([0, 3], dtype=I64, device="cuda")
    ranks = torch.full((R,), SENTINEL, dtype=I32, device="cuda")
    topk = torch.full((R, 65), SENTINEL, dtype=I32, device="cuda")

    def call(cols, k, o=off):
        return lib.vb_retrieval_rank_sets(big.data_ptr(), N, R, cols, o if o is None else o.data_ptr(), idx.data_ptr(), k,
                                          ranks.data_ptr(), topk.data_ptr(), S())
    assert call(N, 1) != 0 and "50000" in lib.vb_last_error().decode()
    assert call(100, 65) != 0 and "vb_retrieval_rank_sets" in lib.vb_last_error().decode()
    assert call(100, 0) != 0
    assert call(100, 5, None) != 0 and "set_off" in lib.vb_last_error().decode()
    torch.cuda.synchronize()
    assert (ranks == SENTINEL).all() and (topk == SENTINEL).all()
    assert call(50000, 64) == 0                                   # the largest accepted launch, for contrast
    torch.cuda.synchronize()
    assert ranks.tolist() == [0, 3] and topk.view(-1)[:2 * 64].tolist() == list(range(64)) * 2     # rows of k = 64 entries


def test_rank_captions_against_numpy():
    from vilbert_b200.retrieval import RetrievalEvaluator
    Cn, G = 700, 60
    g = torch.Generator().manual_seed(3)
    scores = _scores(Cn, G, g)
    target = torch.randint(0, G - 4, (Cn,), generator=g)          # images G-4 .. G-1 have no caption
    target[:3] = torch.tensor([-1, G, G + 5])                     # captions outside the gallery belong to no image
    dev = scores.cuda()
    ranks, topk = RetrievalEvaluator.rank_captions(dev, target, k=20)
    assert ranks.shape == (G,) and topk.shape == (G, 20) and ranks.dtype == I32 and ranks.is_cuda
    cols = scores.t().contiguous().numpy()
    for i in range(G):
        assert int(ranks[i]) == set_rank(cols[i], np.where(target.numpy() == i)[0]), i
        assert topk[i].tolist() == stable_desc(cols[i])[:20].tolist(), i
    assert (ranks[G - 4:] == -1).all()
    with pytest.raises(ValueError):
        RetrievalEvaluator.rank_captions(dev.t(), target, k=20)     # rows not contiguous
    with pytest.raises(ValueError):
        RetrievalEvaluator.rank_captions(dev, target[:-1], k=20)
    for k in (0, 65):
        with pytest.raises(ValueError):
            RetrievalEvaluator.rank_captions(dev, target, k=k)


# ------------------------------------------------------------------------------------------ evaluate_retrieval_both
G_IMAGES, N_CAPTIONS, PER_IMAGE, CAPTIONLESS, NV, NT, CHUNK = 100, 500, 5, 5, 21, 12, 50


def _cfgj(golden_dir, base):
    if base:
        return json.load(open(os.path.join(ROOT, "vilbert-multi-task_b200", "configs", "bert_base_6layer_6conect.json")))
    return json.load(open(os.path.join(golden_dir, "tiny_b4.json")))["config"]


def _model(cfgj, zero_shot):
    import vilbert_b200
    cfgj = dict(cfgj, task_specific_tokens=not zero_shot)
    cls = vilbert_b200.BertForMultiModalPreTraining if zero_shot else vilbert_b200.VILBertForVLTasks
    model = cls(vilbert_b200.BertConfig.from_dict(cfgj))
    model.load_state_dict(O.synth_params(O.make_config(cfgj), seed=0, device="cuda", with_task_heads=not zero_shot), strict=False)
    return model


class _Dataset(_FakeDataset):
    """The reference's item layout with ragged, prefix-valid caption masks."""

    def __init__(self, *a, lens, **kw):
        super().__init__(*a, **kw)
        self.lens = lens

    def __getitem__(self, i):
        item = list(super().__getitem__(i))
        item[4] = (torch.arange(len(item[3])) < self.lens[i // 2]).long()
        return tuple(item)


def _dataset(cfgj):
    """100 images x 500 captions: five captions for each of images 0 .. 94 except a few that take extra ones, none for the last
    five; ragged image masks and caption lengths."""
    g = torch.Generator().manual_seed(11)
    img = [c // PER_IMAGE for c in range(N_CAPTIONS - 25)]
    img += torch.randint(0, G_IMAGES - CAPTIONLESS, (25,), generator=g).tolist()
    ds = _Dataset(N_CAPTIONS, G_IMAGES // 2, [[i] for i in img], Nv=NV, Nt=NT, F=cfgj["v_feature_size"],
                  lens=torch.randint(1, NT + 1, (N_CAPTIONS,), generator=g).tolist())
    ds.mask = (torch.arange(NV) < torch.randint(1, NV + 1, (G_IMAGES, 1), generator=g)).long()
    ds.feat = torch.relu(ds.feat) * ds.mask.unsqueeze(-1)
    ds.cap = ds.cap % cfgj["vocab_size"]
    return ds, torch.tensor(img)


def _numpy_rankings(scores, target, k):
    """Both directions from the score matrix with np.argsort(-s, kind="stable"): (t2i ranks, t2i top-k, i2t ranks, i2t top-k)."""
    s = scores.cpu().numpy()
    t2i = [int(np.where(stable_desc(row) == int(t))[0][0]) for row, t in zip(s, target)]
    t2i_top = [stable_desc(row)[:k].tolist() for row in s]
    i2t = [set_rank(col, np.where(target.numpy() == i)[0]) for i, col in enumerate(s.T)]
    i2t_top = [stable_desc(col)[:k].tolist() for col in s.T]
    return t2i, t2i_top, i2t, i2t_top


@pytest.mark.parametrize("pack", [False, True], ids=["padded", "packed"])
@pytest.mark.parametrize("zero_shot", [False, True], ids=["finetuned", "zeroshot"])
@pytest.mark.parametrize("base", [False, True], ids=["tiny", "base66"])
def test_evaluate_retrieval_both(golden_dir, monkeypatch, base, zero_shot, pack):
    from vilbert_b200 import retrieval as RT
    cfgj = _cfgj(golden_dir, base)
    model = _model(cfgj, zero_shot)
    ds, target = _dataset(cfgj)
    task_id = None if zero_shot else "TASK8"
    scored = []
    score = RT.RetrievalEvaluator.score
    monkeypatch.setattr(RT.RetrievalEvaluator, "score", lambda self, *a, **kw: scored.append(score(self, *a, **kw)) or scored[-1])
    model.train()
    out = RT.evaluate_retrieval_both(model, ds, task_id=task_id, chunk=CHUNK, k=20, pack=pack)
    assert not model.training
    assert set(out) == {"t2i", "i2t", "rsum", "images_without_caption"}
    assert any(p.packed for p in model.engine.plans.values()) == pack and not model.engine.pack_fallbacks
    assert len(scored) == 1 and scored[0].shape == (N_CAPTIONS, G_IMAGES)
    t2i, t2i_top, i2t, i2t_top = _numpy_rankings(scored[0], target, 20)
    assert out["t2i"][:5] == RT.retrieval_metrics(t2i) and out["t2i"][5] == t2i_top
    assert (out["i2t"][:5], out["images_without_caption"]) == RT.i2t_metrics(i2t) and out["i2t"][5] == i2t_top
    assert out["images_without_caption"] == CAPTIONLESS and len(out["i2t"][5]) == G_IMAGES
    assert out["rsum"] == float(sum(out["t2i"][:3]) + sum(out["i2t"][:3]))
    # caption-to-image is evaluate_retrieval's result for the same arguments
    ref = RT.evaluate_retrieval(model, ds, task_id=task_id, chunk=CHUNK, k=20, pack=pack)
    assert torch.equal(scored[1], scored[0])
    assert out["t2i"] == ref
    print(f"{'base66' if base else 'tiny'} {'zero-shot' if zero_shot else 'fine-tuned'} pack={pack}: t2i r1/r5/r10 "
          f"{out['t2i'][0]:.1f}/{out['t2i'][1]:.1f}/{out['t2i'][2]:.1f}, i2t {out['i2t'][0]:.1f}/{out['i2t'][1]:.1f}/{out['i2t'][2]:.1f}")
