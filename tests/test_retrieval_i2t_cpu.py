"""Image-to-text retrieval without a GPU: the set rank (an image's best-placed ground-truth caption) restated in numpy and checked
against the kernel's key rule, the CSR caption sets built from target_image, the i2t metrics over the images that have a caption,
and the new entry point as the header binds it."""
import numpy as np
import pytest
import torch

from test_retrieval_cpu import key_order, stable_desc
from vilbert_b200 import _lib as L
from vilbert_b200.retrieval import RetrievalEvaluator, caption_sets, i2t_metrics, retrieval_metrics


def set_rank(s, idx):
    """The smallest position in np.argsort(-s, kind="stable") (NaN last) that a target of idx takes; targets outside [0, len(s))
    are ignored, and a set without one gives -1."""
    pos = np.empty(len(s), dtype=np.int64)
    pos[stable_desc(s)] = np.arange(len(s))
    valid = [int(t) for t in idx if 0 <= t < len(s)]
    return int(pos[valid].min()) if valid else -1


def key_set_rank(s, idx):
    """vb_retrieval_rank_sets' rule: the largest key among the targets, then the number of keys above it."""
    order = key_order(s)
    rank_of = {int(j): i for i, j in enumerate(order)}
    valid = [int(t) for t in idx if 0 <= t < len(s)]
    if not valid:
        return -1
    best = max(valid, key=lambda t: -rank_of[t])       # the largest key is the earliest in the descending key order
    return rank_of[best]


def _rows(rng, N):
    s = np.round(rng.normal(size=(8, N)) * 2, 1).astype(np.float32)         # ties are common
    s[1, ::3] = np.nan
    s[2] = 0.0
    s[2, ::2] = -0.0
    s[3] = np.nan
    s[4, rng.integers(0, N, max(1, N // 5))] = np.inf
    s[4, rng.integers(0, N, max(1, N // 5))] = -np.inf
    s[5, N // 2:] = s[5].max()
    s[6, rng.integers(0, N, max(1, N // 4))] = np.nan
    return s


@pytest.mark.parametrize("N", [1, 2, 9, 500])
def test_set_rank_restatement_matches_the_key_rule(N):
    rng = np.random.default_rng(N)
    for row in _rows(rng, N):
        for size in range(8):
            idx = rng.integers(-2, N + 2, size)                             # indices outside [0, N) included
            assert set_rank(row, idx) == key_set_rank(row, idx), (row[:8], idx)
        assert set_rank(row, []) == -1 and set_rank(row, [-1, N, N + 7]) == -1


def test_set_rank_is_the_minimum_single_target_rank():
    s = np.array([0.5, np.nan, 0.5, -0.0, 0.0, 2.0, np.nan], np.float32)
    order = stable_desc(s).tolist()
    assert order == [5, 0, 2, 3, 4, 1, 6]
    assert set_rank(s, [4, 3]) == 3                                          # -0.0 ties with +0.0: column order
    assert set_rank(s, [6, 1]) == 5                                          # NaNs last, in column order
    assert set_rank(s, [2, 9, -1, 0]) == 1
    assert set_rank(s, [3]) == order.index(3)


def test_caption_sets_csr():
    target = torch.tensor([3, 0, 3, -1, 7, 0, 5, 9, 3])
    off, idx = caption_sets(target, 6)
    assert off.dtype == torch.int64 and idx.dtype == torch.int64 and off.tolist() == [1, 3, 3, 3, 6, 6, 7]
    sets = [idx[off[g]:off[g + 1]].tolist() for g in range(6)]
    assert sets == [[1, 5], [], [], [0, 2, 8], [], [6]]                      # captions -1, 7, 9 belong to no image
    # random layouts: every image's set is its captions in ascending order
    rng = np.random.default_rng(0)
    for G, C in [(1, 1), (1, 6), (5, 3), (40, 200), (100, 500)]:
        t = torch.from_numpy(rng.integers(-3, G + 3, C))
        off, idx = caption_sets(t, G)
        assert len(off) == G + 1 and bool((off[1:] >= off[:-1]).all())
        for g in range(G):
            assert idx[off[g]:off[g + 1]].tolist() == [c for c in range(C) if int(t[c]) == g], (G, C, g)
    off, idx = caption_sets(torch.tensor([-1, 4]), 3)
    assert off.tolist() == [1, 1, 1, 1]


def test_i2t_metrics_skip_captionless_images():
    ranks = np.array([0, -1, 3, 12, -1, 1, 0])
    metrics, without = i2t_metrics(ranks)
    assert without == 2 and metrics == retrieval_metrics(np.array([0, 3, 12, 1, 0]))
    assert i2t_metrics(torch.tensor(ranks, dtype=torch.int32)) == (metrics, 2)
    assert i2t_metrics([4, 2]) == (retrieval_metrics([4, 2]), 0)
    with pytest.raises(ValueError):
        i2t_metrics([-1, -1])


def test_rank_captions_refuses_host_scores_and_the_header_binds_the_entry_point():
    with pytest.raises(ValueError, match="device f32"):
        RetrievalEvaluator.rank_captions(torch.zeros(4, 2), torch.zeros(4, dtype=torch.long))
    assert L.ARGS["vb_retrieval_rank_sets"]._fields == ("scores", "ld_scores", "rows", "cols", "set_off", "set_idx", "k", "rank_out",
                                                        "topk_out")
    fn = getattr(L.lib(), "vb_retrieval_rank_sets")
    assert len(fn.argtypes) == 10
