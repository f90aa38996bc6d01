"""Pins the reference dropout masks of tests/_train_ref.py (used by tests/test_train_kernels_gpu.py) before any kernel is compared
with them: bit-identical to the oracle's DropMasks, independent of the element count, index taken mod 2^32, kept fraction 1 - p."""
import numpy as np
import pytest
import torch

import _train_ref as R
from oracle.vilbert_oracle import DropMasks
from vilbert_b200.engine import dropout_site_id

NAMES = ("bert.encoder.layer.0.attention.self.dropout", "bert.encoder.v_layer.3.output.dropout",
         "bert.encoder.c_layer.1.biOutput.dropout1", "bert.embeddings.dropout", "dropout.pooled")
STEPS = (0, 3, 123456, 2 ** 31 + 5)      # 123456 and 2^31 + 5: step * 0x9E3779B9 wraps mod 2^32


def _scalar_keep(site, step, p, i):
    """Plain-Python restatement (arbitrary-precision ints, explicit mod 2^32) of one element's factor."""
    def h(x):
        x &= 0xFFFFFFFF
        x ^= x >> 16; x = (x * 0x7FEB352D) & 0xFFFFFFFF
        x ^= x >> 15; x = (x * 0x846CA68B) & 0xFFFFFFFF
        return x ^ (x >> 16)
    s = h(site + step * 0x9E3779B9)
    thresh = int(float(np.float32(p)) * 2 ** 32)
    return float(np.float32(1) / (np.float32(1) - np.float32(p))) if h((i & 0xFFFFFFFF) ^ s) >= thresh else 0.0


@pytest.mark.parametrize("p", [0.1, 0.15, 0.2, 0.25, 0.3, 0.5])
@pytest.mark.parametrize("step", STEPS)
def test_keep_factor_matches_oracle_masks(step, p):
    shape = (3, 5, 37, 41)
    n = int(np.prod(shape))
    for name in NAMES:
        ref = DropMasks(step).mask(name, p, shape, "cpu")
        mine = R.keep_factor(dropout_site_id(name), step, p, R.flat_index(n).view(shape))
        assert mine.dtype == torch.float32 and torch.equal(mine, ref), (name, step, p)


def test_keep_factor_above_2_24_elements():
    """64 x 12 x 150 x 150 = 17.3M probabilities (> 2^24: an index kept in fp32 anywhere would lose bits)."""
    shape = (64, 12, 150, 150)
    name = NAMES[0]
    ref = DropMasks(123456).mask(name, 0.1, shape, "cpu")
    mine = R.keep_factor(dropout_site_id(name), 123456, 0.1, R.attn_index(*shape))
    assert torch.equal(mine, ref)


@pytest.mark.parametrize("step", STEPS)
def test_keep_factor_scalar_restatement_and_index_mod_2_32(step):
    site = dropout_site_id(NAMES[1])
    idx = torch.cat([torch.arange(0, 300), torch.arange(2 ** 32 - 300, 2 ** 32 + 300), torch.arange(3 * 2 ** 32 + 7, 3 * 2 ** 32 + 100)])
    for p in (0.1, 0.3):
        mine = R.keep_factor(site, step, p, idx)
        assert mine.tolist() == [_scalar_keep(site, step, p, int(i)) for i in idx]
        # the index enters mod 2^32
        assert torch.equal(mine, R.keep_factor(site, step, p, idx & 0xFFFFFFFF))


@pytest.mark.parametrize("p", [0.1, 0.5])
def test_kept_fraction(p):
    f = R.keep_factor(dropout_site_id(NAMES[2]), 7, p, R.flat_index(10 ** 7))
    kept = (f != 0).double().mean().item()
    assert abs(kept - (1 - p)) < 1e-3
    assert set(f.unique().tolist()) == {0.0, float(np.float32(1) / (np.float32(1) - np.float32(p)))}


def test_index_builders():
    B, H, Nq, Nk = 2, 3, 5, 7
    a = R.attn_index(B, H, Nq, Nk)
    assert torch.equal(a.flatten(), torch.arange(B * H * Nq * Nk))            # row-major [B, H, Nq, Nk]
    t = R.attn_index(B, H, Nq, Nk, transposed=True)
    assert t[1, 2, 3, 4].item() == ((1 * H + 2) * Nk + 4) * Nq + 3
    assert torch.equal(R.rowmajor_index(4, 6).flatten(), torch.arange(24))
    assert R.rowmajor_index(4, 6, ld=9)[2, 5].item() == 2 * 9 + 5
    idx, text = R.concat_index(2, 3, 4, 8)
    assert idx.shape == (2, 7, 8) and text[:, :3].all() and not text[:, 3:].any()
    assert idx[1, 1, 5].item() == (1 * 3 + 1) * 8 + 5           # text row 1 of sample 1
    assert idx[1, 5, 2].item() == (1 * 4 + 2) * 8 + 2           # image row 2 of sample 1
