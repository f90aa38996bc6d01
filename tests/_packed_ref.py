"""Reference layouts and dropout indices of packed rows for the kernel-level packed tests (tests/test_packed_kernels_gpu.py),
pinned by tests/test_packed_kernels_cpu.py.

A packed stream holds the valid rows of a padded [B, N] batch as contiguous per-sample row ranges: sample b owns rows off[b] ..
off[b] + len[b] - 1, rows off[B] .. rows - 1 belong to no sample, and map[r] is the padded row b * N + i of packed row r (-1: none).
A row-indexed dropout site draws, for packed element (r, c), the mask of padded element (map[r], c); attention draws its
probabilities' masks at padded coordinates ((b*H + h)*Nq + q)*Nk + k with Nq / Nk the padded maxima. Plain torch, no kernel."""
import torch

import _train_ref as R

I32, I64 = torch.int32, torch.int64


def pack_layout(mask, has_task, rows):
    """(off int32 [B + 1], len int32 [B], map int32 [rows]) of a packed stream from a prefix-valid 0/1 mask [B, N_in]: the text
    stream counts the task token's row when has_task (padded rows per sample N = N_in + has_task), and a batch with more valid
    rows than `rows` is clamped to it (each sample keeps what still fits, in sample order), as vb_pack_build documents."""
    mask = mask.to("cpu")
    B, n_in = mask.shape
    N = n_in + (1 if has_task else 0)
    want = mask.ne(0).sum(1) + (1 if has_task else 0)
    off, lens, used = torch.zeros(B + 1, dtype=I64), torch.zeros(B, dtype=I64), 0
    for b in range(B):
        lens[b] = min(int(want[b]), rows - used)
        off[b] = used
        used += int(lens[b])
    off[B] = used
    mp = torch.full((rows,), -1, dtype=I64)
    for b in range(B):
        n = int(lens[b])
        mp[int(off[b]):int(off[b]) + n] = b * N + torch.arange(n)
    return off.to(I32), lens.to(I32), mp.to(I32)


def packed_index(row_map, H):
    """[rows, H] element index of a row-indexed dropout site under a row map: map[r] * H + c, mod 2^32 (a row of no sample, map -1,
    gives 2^32 - H + c)."""
    m = row_map.to(I64)
    return (m[:, None] * H + torch.arange(H, dtype=I64, device=m.device)[None, :]) & R.M32


def packed_attn_index(q_len, k_len, H, Nq, Nk, extent="padded", q_off=None):
    """[B, H, Nq, Nk] attention-probability element index of packed (q, k) of each sample and the [B, 1, Nq, Nk] bool of the valid
    (q < q_len[b], k < k_len[b]) pairs. extent="padded" is what the kernels draw: ((b*H + h)*Nq + q)*Nk + k. Wrong indices for the
    sensitivity checks: "sample" takes the per-sample lengths for the extents, ((b*H + h)*q_len[b] + q)*k_len[b] + k; "packed"
    numbers queries by their packed row, ((q_off[b] + q)*H + h)*Nk + k."""
    dev = q_len.device
    B = q_len.numel()
    b = torch.arange(B, dtype=I64, device=dev).view(B, 1, 1, 1)
    h = torch.arange(H, dtype=I64, device=dev).view(1, H, 1, 1)
    q = torch.arange(Nq, dtype=I64, device=dev).view(1, 1, Nq, 1)
    k = torch.arange(Nk, dtype=I64, device=dev).view(1, 1, 1, Nk)
    lq, lk = q_len.to(I64).view(B, 1, 1, 1), k_len.to(I64).view(B, 1, 1, 1)
    if extent == "padded":
        idx = ((b * H + h) * Nq + q) * Nk + k
    elif extent == "sample":
        idx = ((b * H + h) * lq + q) * lk + k
    elif extent == "packed":
        idx = ((q_off[:B].to(I64).view(B, 1, 1, 1) + q) * H + h) * Nk + k
    else:
        raise ValueError(extent)
    return idx, (q < lq) & (k < lk)
