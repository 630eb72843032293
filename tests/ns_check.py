"""Stage-by-stage references and checker for the matrix optimizers' GEMM chains: the Newton-Schulz driver
(csrc/newton_schulz.cu: b200_newton_schulz, _allgather, _multi) and Shampoo's bf16x3 statistics and preconditioning
(csrc/shampoo.cu: b200_shampoo_stats, b200_shampoo_precond).  Imports without a GPU.  The families, bounds and
failure messages are those of tests/gemm_check.py; this module only wires them to the drivers' stages.

Newton-Schulz.  The 5-step output is nearly insensitive to the input's scale and damps early errors, so it is checked
one stage at a time, each on the exact bf16 values the kernel itself used.  For iteration s, X = X_{s-1}:
    G1  A_s = sa X X^T         (tall: sa X^T X)          sa = inv_norm^2 on iteration 1, else 1
    G2  B_s = b A_s + c A_s A_s
    G3  X_s = sx (a X + B_s X) (tall: sx (a X + X B_s))  sx = inv_norm on iteration 1, else 1
Every stage has bf16 output and is held to gemm_check's bf16 bound 2^-8 |R| + C32 K 2^-24 P; A_s and B_s must also be
bit-symmetric.  A run with steps = s leaves X_s in x_out and A_s, B_s in the caller's workspace (`ns_slices` says
where); X_{s-1} is the output of the steps = s - 1 run, or the input for s = 1.  If a longer run's inner iterate ever
differed from a shorter run's output, that run's G1 check would fail, so the scheme checks itself.

Shampoo, two input families as in gemm_check:
exact   hi operands are integers in [-8, 8], lo operands integers in [-8, 8] times 2^-8, beta2 and weight (alpha) powers
        of two, K <= 1000.  Every partial sum is a multiple of 2^-8 below 2^16 in magnitude (2^24 units), so fp32
        accumulation is exact in any order and L, R and precond's first product T = PLh m_h + PLh m_l + PLl m_h are
        known bit for bit: any dropped cross term (Gl Gh^T, PLl m_h, ...), any lo operand read from the wrong batch,
        and any padding written, fails.  Precond's second product out = alpha (Th PRh + Th PRl + Tl PRh) mixes the
        granularities of Th (an 8-bit rounding of T) and the 2^-8 lo parts, so it is held to the bound below on the
        kernel's own Th and Tl (read from the workspace, where Th == bf16_rn(T) and Tl == bf16_rn(T - Th) must hold
        bit for bit).  In this family a dropped Th PRl or Tl PRh term is about 2^16 / (2 K^1.5) times the bound: many
        times it at K = k2 <= 264 (tests/test_ns_check.py shows the rejection at the GPU tests' shapes), but only about
        once at K = 1000, where it is not reliably seen.
bound   Gaussian operands (C4's k = 1024).  Three accumulating fp32-output GEMMs: each adds at most C32 K 2^-24 P_i of
        accumulation error and one fp32 rounding of the running sum (<= 2^-24 P), so the chain is checked as one GEMM
        with K + 2 in place of K:  |D - R| <= C32 (K + 2) 2^-24 P,  P = sum of the three |.||.| products (+ |beta C|).
        A dropped lo term is about 2^-8 / sqrt(K) of P: at K = 1024 that is the bound's own size, so only some
        elements exceed it.  This family is relied on for shape, layout and scale faults; missing cross terms are the
        exact family's job.
"""
from __future__ import annotations

from typing import Dict, List, NamedTuple, Sequence

import torch

from tests import gemm_check as gc


# ---- Newton-Schulz workspace layout ---------------------------------------------------------------------------
def _a256(x: int) -> int:
    return (x + 255) // 256 * 256


def g1_k_splits(batch: int, m: int, k: int, sms: int) -> int:
    """The G1 split-K count (g1_k_splits in csrc/newton_schulz.cu): one work item per SM for lone big matrices."""
    if m <= 128 or m % 8 != 0:
        return 1
    t = (m + 127) // 128
    tiles = t * (t + 1) // 2 * batch
    if tiles * 2 > sms:
        return 1
    s = min(sms // tiles, (k + 63) // 64 // 16)
    return 1 if s < 2 else s


class Slices(NamedTuple):
    """Byte offsets of one group's workspace slices: A (bf16 [batch, m, m]), B (same), X_tmp (bf16 [batch, rows,
    cols], only for steps >= 2), the split-K partials (fp32 [splits, batch, m, m], only for splits > 1), and the end."""
    a: int
    b: int
    xtmp: int
    splitk: int
    end: int
    splits: int


def ns_slices(shapes: Sequence[Sequence[int]], steps: int, sms: int) -> List[Slices]:
    """Where each group's A and B sit in the caller's workspace, for b200_newton_schulz (one shape) and for every
    group of b200_newton_schulz_multi, grouped or falling back to one chain per group.  Mirrors ns_layout,
    newton_schulz_workspace_bytes and newton_schulz_multi_workspace_bytes in csrc/newton_schulz.cu: both paths place
    group i at the same offset (the larger of the two layouts' ends of group i - 1), and A at offset 0 of it and B
    after it in either case.  The last slice's `end` is the library's workspace size."""
    out, off = [], 0
    for batch, rows, cols in shapes:
        m = min(rows, cols)
        a = off
        b = a + _a256(batch * m * m * 2)
        xtmp = b + _a256(batch * m * m * 2)
        splitk = xtmp + (_a256(batch * rows * cols * 2) if steps >= 2 else 0)
        splits = g1_k_splits(batch, m, max(rows, cols), sms)
        end = splitk + (_a256(splits * batch * m * m * 4) if splits > 1 else 0)
        out.append(Slices(a, b, xtmp, splitk, end, splits))
        off = end   # single-chain and grouped layouts of one group end at the same byte
    return out


def grouped_ok(shapes: Sequence[Sequence[int]], sms: int) -> bool:
    """Whether b200_newton_schulz_multi runs one grouped launch per stage (multi_grouped_ok); else one chain per group."""
    if not 1 <= len(shapes) <= 6 or sms < 2:
        return False
    return all(min(r, c) > 128 and min(r, c) % 8 == 0 and c % 8 == 0 for _, r, c in shapes)


def ws_view(ws: torch.Tensor, offset: int, shape: Sequence[int], dtype=torch.bfloat16) -> torch.Tensor:
    """A typed view of the byte workspace `ws` at `offset`."""
    n = 1
    for s in shape:
        n *= s
    size = n * torch.tensor([], dtype=dtype).element_size()
    return ws[offset:offset + size].view(dtype).view(*shape)


# ---- Newton-Schulz stage checks -------------------------------------------------------------------------------
def check_symmetric(A: torch.Tensor, what: str) -> None:
    """A [batch, m, m] must equal its transpose bit for bit (the mirrored tiles are copies, not recomputations)."""
    bits = A.view(torch.int16)
    bad = bits != bits.transpose(1, 2)
    if bool(bad.any()):
        i = int(bad.flatten().nonzero()[0])
        raise AssertionError(f"{what}: not bit-symmetric, {int(bad.sum())} elements differ from their mirror; first "
                             f"at {gc.where(A, i)}")


def check_iteration(X: torch.Tensor, A: torch.Tensor, B: torch.Tensor, Xn: torch.Tensor, *, s: int,
                    inv_norm: torch.Tensor, inv_norm_sq: torch.Tensor, coeffs: Sequence[float],
                    what: str = "") -> Dict[str, gc.Bound]:
    """The three stages of iteration s (1-based) on the kernel's own bf16 values: X = X_{s-1} [batch, rows, cols],
    A = A_s, B = B_s [batch, m, m], Xn = X_s.  inv_norm / inv_norm_sq: the fp32 [batch] vectors the kernel was given
    (used on iteration 1 only).  Returns each stage's gemm_check.Bound; raises naming stage, iteration and element."""
    a, b, c = coeffs
    _, rows, cols = X.shape
    tall = rows > cols
    m = min(rows, cols)
    first = s == 1
    tag = f"{what}{': ' if what else ''}iteration {s}"
    out = {}
    check_symmetric(A, f"{tag}, G1 (A = {'X^T X' if tall else 'X X^T'})")
    R, P = gc.reference(X, X, a_mn=tall, b_mn=tall, alpha_vec=inv_norm_sq if first else None)
    out["G1"] = gc.check_bound(A, R, P, max(rows, cols), f"{tag}, G1 (A = {'X^T X' if tall else 'X X^T'})")
    check_symmetric(B, f"{tag}, G2 (B = bA + cAA)")
    R, P = gc.reference(A, A, alpha=c, beta=b, C=A)
    out["G2"] = gc.check_bound(B, R, P, m, f"{tag}, G2 (B = bA + cAA)")
    sx = inv_norm if first else None
    if tall:   # X B^T == X B for the bit-symmetric B
        R, P = gc.reference(X, B, alpha_vec=sx, beta=a, beta_vec=sx, C=X)
    else:
        R, P = gc.reference(B, X, b_mn=True, alpha_vec=sx, beta=a, beta_vec=sx, C=X)
    out["G3"] = gc.check_bound(Xn, R, P, m, f"{tag}, G3 (X' = {'aX + XB' if tall else 'aX + BX'})")
    return out


# ---- Shampoo ---------------------------------------------------------------------------------------------------
def exact_hi(shape, device="cpu", generator=None) -> torch.Tensor:
    """Exact family hi operand: integers in [-8, 8], bf16."""
    return gc.exact_ints(shape, device=device, generator=generator).to(torch.bfloat16)


def exact_lo(shape, device="cpu", generator=None) -> torch.Tensor:
    """Exact family lo operand: integers in [-8, 8] times 2^-8, bf16."""
    return (gc.exact_ints(shape, device=device, generator=generator) * 2.0 ** -8).to(torch.bfloat16)


def split(x: torch.Tensor):
    """Bound family: fp32 x as the kernels split it, hi = bf16_rn(x), lo = bf16_rn(x - hi)."""
    hi = x.to(torch.bfloat16)
    return hi, (x - hi.float()).to(torch.bfloat16)


def reference3(Ah, Al, Bh, Bl, *, a_mn=False, b_mn=False, alpha=1.0, beta=0.0, C=None):
    """fp64 (R, P) of alpha (Ah Bh + Ah Bl + Al Bh) + beta C, gemm3's three accumulating GEMMs (csrc/shampoo.cu);
    a None lo operand drops its term, as a NULL pointer does."""
    R, P = gc.reference(Ah, Bh, a_mn=a_mn, b_mn=b_mn, alpha=alpha, beta=beta, C=C)
    for x, y in ((Ah, Bl), (Al, Bh)):
        if x is not None and y is not None:
            r, p = gc.reference(x, y, a_mn=a_mn, b_mn=b_mn, alpha=alpha)
            R, P = R + r, P + p
    return R, P


def check3(D: torch.Tensor, R: torch.Tensor, P: torch.Tensor, K: int, exact: bool, what: str = "") -> gc.Bound:
    """fp32 output of a three-GEMM chain: bit for bit in the exact family, else the bound with K + 2 (docstring)."""
    if exact:
        gc.check_exact(D, R, what)
        return gc.Bound(0.0, 0.0)
    return gc.check_bound(D, R, P, K + 2, what)


def stats_reference(g_hi, g_lo, L0, R0, k1: int, k2: int, beta2: float, weight: float):
    """fp64 (L, P_L), (R, P_R) of b200_shampoo_stats on the [batch, >= k1, >= k2] gradient halves: L0 / R0 are the
    factors' [:k1, :k1] / [:k2, :k2] blocks before the call."""
    Gh = g_hi[:, :k1, :k2]
    Gl = None if g_lo is None else g_lo[:, :k1, :k2]
    L = reference3(Gh, Gl, Gh, Gl, alpha=weight, beta=beta2, C=L0)
    R = reference3(Gh, Gl, Gh, Gl, a_mn=True, b_mn=True, alpha=weight, beta=beta2, C=R0)
    return L, R


def precond_first_reference(PLh, PLl, m_hi, m_lo, k1: int, k2: int):
    """fp64 (T, P) of precond's first product T = PLh m_h + PLh m_l + PLl m_h over the [:k1, :k2] block."""
    return reference3(PLh[:, :k1, :k1], None if PLl is None else PLl[:, :k1, :k1], m_hi[:, :k1, :k2],
                      None if m_lo is None else m_lo[:, :k1, :k2], b_mn=True)


def check_split(T: torch.Tensor, Th: torch.Tensor, Tl: torch.Tensor, what: str = "") -> None:
    """Th == bf16_rn(T) and Tl == bf16_rn(T - Th), bit for bit (split4_kernel)."""
    gc.check_exact(Th, T.double(), f"{what}: Th = bf16_rn(T)")
    gc.check_exact(Tl, T.double() - Th.double(), f"{what}: Tl = bf16_rn(T - Th)")


def precond_second_reference(Th, Tl, PRh, PRl, k2: int, alpha: float):
    """fp64 (out, P) of precond's second product alpha (Th PRh + Th PRl + Tl PRh) on the kernel's own Th, Tl."""
    return reference3(Th, Tl, PRh[:, :k2, :k2], None if PRl is None else PRl[:, :k2, :k2], b_mn=True, alpha=alpha)


def zero_padding_bits(F: torch.Tensor, k: int, what: str = "") -> None:
    """A [batch, kp, kp] fp32 factor's rows and columns >= k must be +0.0 bit for bit (shampoo_root relies on it)."""
    bits = F.view(torch.int32)
    mask = torch.ones_like(bits, dtype=torch.bool)
    mask[:, :k, :k] = False
    bad = (bits != 0) & mask
    if bool(bad.any()):
        i = int(bad.flatten().nonzero()[0])
        raise AssertionError(f"{what}: padding outside [:{k}, :{k}] is not zero: {int(bad.sum())} elements; first at "
                             f"{gc.where(F, i)}: {float(F.flatten()[i])}")
