"""Truth and checker for Shampoo's inverse 4th root (ShampooParams.inverse_root = "newton").

- `matrix_inverse_root_eigh`: fp64 eigendecomposition truth P0 = (M + ridge I)^(-1/4) with the ridge rule of the
  kernel, ridge = eps * max(lambda_max(M), 1e-6) (Anil et al. 2020, relative ridge).
- `newton_root`: the coupled Newton iteration of b200_shampoo_root_newton restated in torch, with a pluggable
  matrix product: fp64, or `mm6` / `mm3`, emulations of the kernel's 3-way bf16 split (six products) and of the
  2-way hi/lo split used by the literal root (three products).
- `root_errors` / `check_roots`: relative Frobenius error ||P - P0||_F / ||P0||_F and spectral relative error
  ||P0^(-1/2) P P0^(-1/2) - I||_2 per matrix, plus exact-zero padding and the reported iteration counts and
  residuals.  A failure names the matrix.
- `spectrum_matrix`: the test spectra (well-conditioned, kappa 1e4, ridge-limited, rank-deficient, zero, scaled I).
"""
from __future__ import annotations

import math
from contextlib import contextmanager
from typing import Callable, Optional, Sequence

import torch

ROOT_ORDER = 4
SPECTRAL_BOUND = 3e-2    # device and emulation against the fp64 truth
FROBENIUS_BOUND = 1e-2
KINDS = ("well", "kappa1e4", "ridge", "rankdef", "zero", "identity")


def ridge_of(M: torch.Tensor, eps: float) -> float:
    lmax = float(torch.linalg.eigvalsh(M.double())[-1]) if M.numel() else 0.0
    return eps * max(lmax, 1e-6)


def matrix_inverse_root_eigh(M: torch.Tensor, eps: float, r: int = ROOT_ORDER) -> torch.Tensor:
    """(M + ridge I)^(-1/r) in fp64 from the eigendecomposition of the symmetrised M."""
    Md = M.double()
    Md = (Md + Md.T) / 2
    w, Q = torch.linalg.eigh(Md)
    w = w + eps * max(float(w[-1]), 1e-6)
    return (Q * w.clamp_min(1e-300) ** (-1.0 / r)) @ Q.T


# ---- product emulations -------------------------------------------------------------------------------
def split3(x: torch.Tensor):
    h = x.bfloat16().float()
    r = x - h
    m = r.bfloat16().float()
    return h, m, (r - m).bfloat16().float()


def mm6(a: torch.Tensor, b: torch.Tensor) -> torch.Tensor:
    """fp32-output product over 3-way bf16 splits: hh + hm + mh + hl + lh + mm (the kernel's six GEMMs)."""
    ah, am, al = split3(a.float())
    bh, bm, bl = split3(b.float())
    return ah @ bh + ah @ bm + am @ bh + ah @ bl + al @ bh + am @ bm


def mm3(a: torch.Tensor, b: torch.Tensor) -> torch.Tensor:
    """hi/lo split, three products (the literal root's scheme)."""
    ah = a.float().bfloat16().float()
    al = (a.float() - ah).bfloat16().float()
    bh = b.float().bfloat16().float()
    bl = (b.float() - bh).bfloat16().float()
    return ah @ bh + ah @ bl + al @ bh


def mm64(a: torch.Tensor, b: torch.Tensor) -> torch.Tensor:
    return a.double() @ b.double()


def newton_root(M: torch.Tensor, ridge: float, mm: Callable = mm64, max_iters: int = 60, tol: float = 1e-5,
                r: int = ROOT_ORDER, honour_rejection: bool = True):
    """Coupled Newton for (M + ridge I)^(-1/r), exactly the kernel's control flow.  Returns (X, accepted, e)."""
    k = M.shape[0]
    dt = torch.float64 if mm is mm64 else torch.float32
    I = torch.eye(k, dtype=dt)
    Mt = M.to(dt) + ridge * I
    z = (1 + r) / (2 * float(Mt.double().norm()))
    Mc = (Mt * z).to(dt)
    X = I * z ** (1.0 / r)
    e = float((Mc - I).abs().max())
    n = 0
    if e <= tol:
        return X, n, e
    for _ in range(max_iters):
        T = (1 + 1.0 / r) * I - Mc / r
        T2 = mm(T, T).to(dt)
        T4 = mm(T2, T2).to(dt)
        Mn = mm(T4, Mc).to(dt)
        en = float((Mn - I).abs().max())
        if not en <= 1.2 * e and honour_rejection:
            break
        X = mm(X, T).to(dt)
        Mc, e, n = Mn, en, n + 1
        if e <= tol:
            break
    return X, n, e


# ---- checker ----------------------------------------------------------------------------------------------
def root_errors(P: torch.Tensor, M: torch.Tensor, eps: float):
    """(relative Frobenius error, spectral relative error) of P [k, k] against the truth for M [k, k]."""
    Md = M.double()
    Md = (Md + Md.T) / 2
    w, Q = torch.linalg.eigh(Md)
    w = w + eps * max(float(w[-1]), 1e-6)
    P0 = (Q * w ** (-1.0 / ROOT_ORDER)) @ Q.T
    half = (Q * w ** (1.0 / (2 * ROOT_ORDER))) @ Q.T          # P0^(-1/2)
    Pd = P.double()
    fro = float((Pd - P0).norm() / P0.norm())
    E = half @ Pd @ half
    E = (E + E.T) / 2 - torch.eye(M.shape[0], dtype=torch.float64, device=M.device)
    spec = float(torch.linalg.eigvalsh(E).abs().max())
    return fro, spec


def check_roots(P: torch.Tensor, M: torch.Tensor, k: int, eps: float, iters: Optional[torch.Tensor] = None,
                residual: Optional[torch.Tensor] = None, tol: Optional[float] = None,
                max_iters: Optional[int] = None, spectral_bound: float = SPECTRAL_BOUND,
                frobenius_bound: float = FROBENIUS_BOUND):
    """P, M: [batch, kp, kp].  Raises AssertionError naming the first failing matrix; returns the worst errors."""
    assert P.shape == M.shape and P.dim() == 3, (P.shape, M.shape)
    worst = {"fro": 0.0, "spectral": 0.0}
    bad = []
    for b in range(P.shape[0]):
        pad = torch.cat([P[b, k:, :].flatten(), P[b, :k, k:].flatten()])
        if bool((pad != 0).any()):
            bad.append(f"matrix {b}: non-zero padding outside [:{k}, :{k}]")
        Pb = P[b, :k, :k]
        if not bool(torch.isfinite(Pb).all()):
            bad.append(f"matrix {b}: non-finite root")
            continue
        fro, spec = root_errors(Pb, M[b, :k, :k], eps)
        if spec > spectral_bound:
            bad.append(f"matrix {b}: spectral relative error {spec:.3g} > {spectral_bound:g}")
        if fro > frobenius_bound:
            bad.append(f"matrix {b}: relative Frobenius error {fro:.3g} > {frobenius_bound:g}")
        worst["fro"], worst["spectral"] = max(worst["fro"], fro), max(worst["spectral"], spec)
        if residual is not None and not float(residual[b]) <= tol:
            bad.append(f"matrix {b}: residual {float(residual[b]):.3g} > tol {tol:g}")
        if iters is not None and not 0 <= int(iters[b]) <= max_iters:
            bad.append(f"matrix {b}: {int(iters[b])} iterations (max {max_iters})")
    assert not bad, "; ".join(bad)
    return worst


# ---- spectra ------------------------------------------------------------------------------------------------
def spectrum_matrix(kind: str, k: int, seed: int, scale: float = 1.0) -> torch.Tensor:
    """A symmetric PSD fp32 [k, k] matrix with the named spectrum (built in fp64, rounded once)."""
    g = torch.Generator().manual_seed(seed)
    if kind == "zero":
        return torch.zeros(k, k)
    if kind == "identity":
        return torch.eye(k) * 3.7 * scale
    Q, _ = torch.linalg.qr(torch.randn(k, k, generator=g, dtype=torch.float64))
    i = torch.arange(k, dtype=torch.float64)
    t = i / max(k - 1, 1)
    if kind == "well":
        lam = 1.0 + torch.rand(k, generator=g, dtype=torch.float64)
    elif kind == "kappa1e4":
        lam = 10.0 ** (-4.0 * t)
    elif kind == "ridge":                       # down to 1e-6 lambda_max: with the ridge, kappa ~ 5e5
        lam = 10.0 ** (-6.0 * t)
    elif kind == "rankdef":                     # embedding-like: rank k/4, the rest exactly zero
        rank = max(1, k // 4)
        lam = torch.where(i < rank, 10.0 ** (-2.0 * i / max(rank - 1, 1)), torch.zeros_like(i))
    else:
        raise ValueError(kind)
    A = (Q * (lam * scale)) @ Q.T
    return ((A + A.T) / 2).float()


def power_law_statistics(k: int, lmax: float, seed: int = 1, n: int = 2816) -> torch.Tensor:
    """0.05 G G^T of a rank-k gradient with singular values s_i = s_1 i^-1.5, scaled so lambda_max = lmax."""
    g = torch.Generator().manual_seed(seed)
    U, _ = torch.linalg.qr(torch.randn(k, k, generator=g, dtype=torch.float64))
    V, _ = torch.linalg.qr(torch.randn(n, k, generator=g, dtype=torch.float64))
    s = math.sqrt(lmax / 0.05) * torch.arange(1, k + 1, dtype=torch.float64) ** -1.5
    G = (U * s) @ V.T
    M = 0.05 * (G @ G.T)
    return ((M + M.T) / 2).float()


@contextmanager
def oracle_newton_roots(R):
    """Inside the block, the oracle's ShampooOracle computes its preconditioners as the fp64 truth
    (M + ridge I)^(-1/4) instead of the literal formula: the oracle of ShampooParams.inverse_root = "newton"."""
    orig = R.matrix_inverse_pth_root
    R.matrix_inverse_pth_root = lambda M, p, epsilon=1e-6, num_iters=6: matrix_inverse_root_eigh(M, epsilon).float()
    try:
        yield
    finally:
        R.matrix_inverse_pth_root = orig


def batch_of(mats: Sequence[torch.Tensor], kp: int) -> torch.Tensor:
    out = torch.zeros(len(mats), kp, kp)
    for b, m in enumerate(mats):
        out[b, :m.shape[0], :m.shape[1]] = m
    return out
