"""tests/_packed_ref.py on the CPU: the packed layout against engine.pack_capacity and a scalar restatement of pack_build_kernel
(vb_pack.cu), the row-mapped dropout index against rowmajor_index and per element, and the padded-coordinate attention index
against _train_ref.attn_index and per element."""
import pytest
import torch

import _packed_ref as P
import _train_ref as R
from vilbert_b200.engine import pack_capacity


def _prefix_mask(B, N, seed):
    g = torch.Generator().manual_seed(seed)
    lens = torch.randint(1, N + 1, (B,), generator=g)
    lens[0], lens[-1] = 1, N
    return (torch.arange(N)[None] < lens[:, None]).long()


def _scalar_layout(mask, has_task, rows):
    """pack_build_kernel one element at a time."""
    B, n_in = mask.shape
    N = n_in + has_task
    lens = [int(sum(int(v != 0) for v in mask[b].tolist())) + has_task for b in range(B)]
    off, used = [], 0
    for b in range(B):
        lens[b] = min(lens[b], rows - used)
        off.append(used)
        used += lens[b]
    off.append(used)
    mp = [-1] * rows
    for b in range(B):
        for i in range(lens[b]):
            mp[off[b] + i] = b * N + i
    return off, lens, mp


@pytest.mark.parametrize("B,N,has_task", [(64, 36, 1), (64, 101, 0), (7, 20, 1), (1, 5, 0)])
def test_pack_layout_against_capacity_and_scalar_restatement(B, N, has_task):
    mask = _prefix_mask(B, N, B * N + has_task)
    count = int(mask.sum()) + B * has_task
    rows = pack_capacity(count, B * (N + has_task))
    off, ln, mp = P.pack_layout(mask, has_task, rows)
    assert off.dtype == ln.dtype == mp.dtype == torch.int32 and mp.shape == (rows,)
    assert int(off[B]) == count <= rows and (mp[count:] == -1).all() and (mp[:count] >= 0).all()
    assert torch.equal(ln.long(), mask.sum(1) + has_task) and torch.equal(off[1:].long() - off[:-1].long(), ln.long())
    so, sl, sm = _scalar_layout(mask, has_task, rows)
    assert off.tolist() == so and ln.tolist() == sl and mp.tolist() == sm
    # map is strictly increasing over the valid rows and lands on padded rows the mask marks valid
    assert (mp[1:count] > mp[:count - 1]).all()
    Np = N + has_task
    b, i = mp[:count].long() // Np, mp[:count].long() % Np
    assert (i < ln.long()[b]).all()


@pytest.mark.parametrize("rows", [1, 40, 100])
def test_pack_layout_clamps_to_capacity(rows):
    mask = _prefix_mask(8, 30, 3)
    off, ln, mp = P.pack_layout(mask, 1, rows)
    assert int(off[-1]) == min(rows, int(mask.sum()) + 8) and int(ln.sum()) == int(off[-1])
    so, sl, sm = _scalar_layout(mask, 1, rows)
    assert off.tolist() == so and ln.tolist() == sl and mp.tolist() == sm


def test_packed_index_identity_map_is_rowmajor_and_wraps():
    rows, H = 333, 768
    ident = torch.arange(rows, dtype=torch.int32)
    assert torch.equal(P.packed_index(ident, H), R.rowmajor_index(rows, H))
    mp = torch.tensor([5, -1, 0, 2 ** 31 - 1], dtype=torch.int32)
    idx = P.packed_index(mp, H)
    for r, m in enumerate(mp.tolist()):
        for c in (0, 1, H - 1):
            assert int(idx[r, c]) == (m * H + c) % 2 ** 32
    # the mask a row draws under the map is the padded row's mask
    mask = _prefix_mask(4, 9, 1)
    _, _, mp = P.pack_layout(mask, 0, 36)
    f_pad = R.keep_factor(7, 11, 0.1, R.rowmajor_index(36, H))
    f_pk = R.keep_factor(7, 11, 0.1, P.packed_index(mp, H))
    valid = mp >= 0
    assert torch.equal(f_pk[valid], f_pad[mp[valid].long()])


def test_packed_attn_index():
    B, H, Nq, Nk = 5, 3, 7, 9
    ql, kl = torch.tensor([1, 7, 6, 3, 2]), torch.tensor([9, 1, 8, 4, 9])
    qoff = torch.cat([torch.zeros(1, dtype=torch.long), ql.cumsum(0)])
    idx, valid = P.packed_attn_index(ql, kl, H, Nq, Nk)
    assert torch.equal(idx, R.attn_index(B, H, Nq, Nk))
    full, fv = P.packed_attn_index(torch.full((B,), Nq), torch.full((B,), Nk), H, Nq, Nk, extent="sample")
    assert torch.equal(full, idx) and bool(fv.all())     # at full lengths the per-sample extents are the padded ones
    sam, _ = P.packed_attn_index(ql, kl, H, Nq, Nk, extent="sample")
    pk, _ = P.packed_attn_index(ql, kl, H, Nq, Nk, extent="packed", q_off=qoff)
    for b in range(B):
        for h in range(H):
            for q in range(Nq):
                for k in range(Nk):
                    assert bool(valid[b, 0, q, k]) == (q < ql[b] and k < kl[b])
                    assert int(idx[b, h, q, k]) == ((b * H + h) * Nq + q) * Nk + k
                    assert int(sam[b, h, q, k]) == ((b * H + h) * int(ql[b]) + q) * int(kl[b]) + k
                    assert int(pk[b, h, q, k]) == ((int(qoff[b]) + q) * H + h) * Nk + k
    # the wrong indices differ from the padded one on the valid pairs of a short sample
    assert (sam != idx)[valid.expand_as(idx)].any() and (pk != idx)[valid.expand_as(idx)].any()
