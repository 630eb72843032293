"""Reference for attention dropout's keep mask and an fp64 attention with it.

Element (b, h, q, k) is kept iff r >= t, with t = min(rint(p 65536), 65535) and r the 16-bit value
(w[(k & 7) >> 1] >> 16 (k & 1)) & 0xffff of w = Philox4x32-10(counter (k >> 3, q, h, b), key (seed lo, seed hi)).
Kept entries of the softmax are scaled by 1 / (1 - t / 65536).  Written from the definition of Philox4x32-10
(Salmon et al., SC'11), vectorised over numpy uint32 arrays."""
from __future__ import annotations

import numpy as np

M0, M1 = np.uint64(0xD2511F53), np.uint64(0xCD9E8D57)
W0, W1 = 0x9E3779B9, 0xBB67AE85
_LO = np.uint64(0xFFFFFFFF)


def philox4x32_10(c0, c1, c2, c3, k0, k1):
    """Philox4x32-10 of counters (c0..c3, uint32 arrays broadcast together) and key (k0, k1 ints)."""
    c = [np.asarray(x, dtype=np.uint64) for x in np.broadcast_arrays(c0, c1, c2, c3)]
    k0, k1 = int(k0) & 0xFFFFFFFF, int(k1) & 0xFFFFFFFF
    for _ in range(10):
        p0, p1 = M0 * c[0], M1 * c[2]
        hi0, lo0 = p0 >> np.uint64(32), p0 & _LO
        hi1, lo1 = p1 >> np.uint64(32), p1 & _LO
        c = [hi1 ^ c[1] ^ np.uint64(k0), lo1, hi0 ^ c[3] ^ np.uint64(k1), lo0]
        k0, k1 = (k0 + W0) & 0xFFFFFFFF, (k1 + W1) & 0xFFFFFFFF
    return [x.astype(np.uint32) for x in c]


def threshold(p: float) -> int:
    return min(int(np.rint(p * 65536.0)), 65535)


def scale(p: float) -> float:
    """1 / (1 - p_eff) in fp64."""
    return 65536.0 / (65536.0 - threshold(p))


def uniforms(seed: int, B: int, H: int, S: int) -> np.ndarray:
    """The 16-bit values r of every (b, h, q, k): uint32 [B, H, S, S]."""
    b = np.arange(B, dtype=np.uint32)[:, None, None, None]
    h = np.arange(H, dtype=np.uint32)[None, :, None, None]
    q = np.arange(S, dtype=np.uint32)[None, None, :, None]
    k = np.arange(S, dtype=np.uint32)[None, None, None, :]
    w = philox4x32_10(k >> 3, q, h, b, seed & 0xFFFFFFFF, seed >> 32)
    sel = (k & 7) >> 1
    word = np.where(sel == 0, w[0], np.where(sel == 1, w[1], np.where(sel == 2, w[2], w[3])))
    return (word >> (16 * (k & 1))) & 0xFFFF


def keep_mask_head(seed: int, p: float, b: int, h: int, S: int) -> np.ndarray:
    """bool [S, S] keep mask of batch row b and query head h."""
    q = np.arange(S, dtype=np.uint32)[:, None]
    k = np.arange(S, dtype=np.uint32)[None, :]
    w = philox4x32_10(k >> 3, q, np.uint32(h), np.uint32(b), seed & 0xFFFFFFFF, seed >> 32)
    sel = (k & 7) >> 1
    word = np.where(sel == 0, w[0], np.where(sel == 1, w[1], np.where(sel == 2, w[2], w[3])))
    return ((word >> (16 * (k & 1))) & 0xFFFF) >= threshold(p)


def keep_mask_head_torch(seed: int, p: float, b: int, h: int, S: int, device="cpu"):
    """keep_mask_head as a torch bool tensor computed on `device` (the same Philox in int64 arithmetic: products of
    two 32-bit values wrap modulo 2^64, whose low 64 bits are exact, so both halves come out right)."""
    import torch
    M = 0xFFFFFFFF
    q = torch.arange(S, device=device, dtype=torch.int64)[:, None]
    k = torch.arange(S, device=device, dtype=torch.int64)[None, :]
    c0, c1 = (k >> 3).expand(S, S), q.expand(S, S)
    c2 = torch.full((S, S), h, device=device, dtype=torch.int64)
    c3 = torch.full((S, S), b, device=device, dtype=torch.int64)
    k0, k1 = seed & M, (seed >> 32) & M
    for _ in range(10):
        p0, p1 = c0 * 0xD2511F53, c2 * 0xCD9E8D57
        c0, c1, c2, c3 = ((p1 >> 32) & M) ^ c1 ^ k0, p1 & M, ((p0 >> 32) & M) ^ c3 ^ k1, p0 & M
        k0, k1 = (k0 + W0) & M, (k1 + W1) & M
    sel = (k & 7) >> 1
    word = torch.where(sel == 0, c0, torch.where(sel == 1, c1, torch.where(sel == 2, c2, c3)))
    return ((word >> (16 * (k & 1))) & 0xFFFF) >= threshold(p)


def keep_mask(seed: int, p: float, B: int, H: int, S: int) -> np.ndarray:
    """bool [B, H, S, S]: True where the element is kept."""
    return uniforms(seed, B, H, S) >= threshold(p)


def attention64(q, k, v, scale_qk, mask_add, keep, p):
    """fp64 O, LSE of dropout attention.  q [B,S,H,D], k/v [B,S,Hk,D] (float64 numpy or torch), mask_add [B or 1, 1,
    S, S] additive (0 / -inf, with any ALiBi bias), keep bool [B, H, S, S]."""
    import torch
    q, k, v = (torch.as_tensor(x, dtype=torch.float64) for x in (q, k, v))
    H, Hk = q.shape[2], k.shape[2]
    k = k.repeat_interleave(H // Hk, dim=2)
    v = v.repeat_interleave(H // Hk, dim=2)
    s = torch.einsum("bqhd,bkhd->bhqk", q, k) * scale_qk + torch.as_tensor(mask_add, dtype=torch.float64)
    lse = torch.logsumexp(s, dim=-1)
    P = torch.exp(s - lse[..., None])
    Pd = P * torch.as_tensor(keep, dtype=torch.float64) * scale(p)
    return torch.einsum("bhqk,bkhd->bqhd", Pd, v), lse
