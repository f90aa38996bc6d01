"""Reference dropout masks for the kernel-level train-mode tests (tests/test_train_kernels_gpu.py).

A vectorised int64 restatement of the stateless dropout RNG of include/vilbert_b200.h (vb_dropout):
    keep(index) = hash32(index ^ hash32(site + step * 0x9E3779B9)) >= (uint32)((double)p_f32 * 2^32)
with hash32 = lowbias32 and every sum / product taken mod 2^32; a kept element is scaled by the float32 1 / (1 - p).
The index builders give each kernel's element index of the tensor the reference applies nn.Dropout to.
tests/test_train_kernels_cpu.py pins this module against oracle.vilbert_oracle.DropMasks, so a GPU test that disagrees with it
points at the kernel."""
import numpy as np
import torch

M32 = 0xFFFFFFFF
GOLDEN = 0x9E3779B9


def hash32(x):
    """lowbias32 of an int64 tensor (taken mod 2^32 first); every product stays below 2^63."""
    x = x & M32
    x = x ^ (x >> 16)
    x = (x * 0x7FEB352D) & M32
    x = x ^ (x >> 15)
    x = (x * 0x846CA68B) & M32
    return x ^ (x >> 16)


def seed(site, step):
    return int(hash32(torch.tensor([(int(site) + int(step) * GOLDEN) & M32], dtype=torch.int64))[0])


def threshold(p):
    """(uint32)((double)p_f32 * 2^32), as the kernels' host code computes it."""
    return int(float(np.float32(p)) * 4294967296.0)


def scale(p):
    """float32 1.f / (1.f - p)."""
    return float(np.float32(1.0) / (np.float32(1.0) - np.float32(p)))


def keep_factor(site, step, p, index):
    """float32 tensor shaped like `index` (int64, may exceed 2^32): 1 / (1 - p) where the element is kept, 0 where dropped."""
    keep = hash32((index.to(torch.int64) & M32) ^ seed(site, step)) >= threshold(p)
    return keep.to(torch.float32) * scale(p)


# ------------------------------------------------------------------------------------------ element indices of each site
def rowmajor_index(rows, cols, device="cpu", ld=None):
    """row * ld + col, ld = cols by default: GEMM epilogue (m*N + n), LayerNorm (row*H + col), small linear (m*K + k)."""
    ld = cols if ld is None else ld
    return (torch.arange(rows, dtype=torch.int64, device=device)[:, None] * ld
            + torch.arange(cols, dtype=torch.int64, device=device)[None, :])


def attn_index(B, H, Nq, Nk, device="cpu", transposed=False):
    """[B, H, Nq, Nk] index of the attention probabilities, ((b*H + h)*Nq + q)*Nk + k. transposed=True gives the index of a
    kernel that would walk keys as rows, ((b*H + h)*Nk + k)*Nq + q (a wrong reference for the sensitivity checks)."""
    bh = torch.arange(B * H, dtype=torch.int64, device=device).view(B, H, 1, 1)
    q = torch.arange(Nq, dtype=torch.int64, device=device).view(1, 1, Nq, 1)
    k = torch.arange(Nk, dtype=torch.int64, device=device).view(1, 1, 1, Nk)
    if transposed:
        return (bh * Nk + k) * Nq + q
    return (bh * Nq + q) * Nk + k


def flat_index(n, device="cpu"):
    """i: the fused pooled vector."""
    return torch.arange(n, dtype=torch.int64, device=device)


def concat_index(B, Nt, Nv, H, device="cpu"):
    """Index of each element of the single-stream embedding output [B, Nt + Nv, H] within its modality's dropout (row within
    the modality * H + col), and a [B, Nt + Nv] bool that is True on text rows."""
    pos = torch.arange(Nt + Nv, device=device)
    text = (pos < Nt)[None, :].expand(B, Nt + Nv)
    b = torch.arange(B, dtype=torch.int64, device=device)[:, None]
    row = torch.where(text, b * Nt + pos[None, :], b * Nv + (pos[None, :] - Nt))
    col = torch.arange(H, dtype=torch.int64, device=device)
    return row[..., None] * H + col, text
