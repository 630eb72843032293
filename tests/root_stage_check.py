"""Iteration-by-iteration references and checker for Shampoo's two inverse roots in csrc/shampoo.cu:
b200_shampoo_root (the literal MatrixSqrt.matrix_inverse_pth_root, `inverse_root: reference`) and
b200_shampoo_root_newton (the coupled-Newton inverse 4th root, `inverse_root: newton`).  Imports without a GPU or
the package.  Both roots damp or amplify errors over their iterations, so an end-to-end tolerance cannot tell a right
kernel from a subtly wrong one; like tests/ns_check.py, every iteration is checked on the kernel's own operands, read
from its workspace (`literal_views`, `newton_views` mirror the workspace_bytes functions of csrc/shampoo.cu).

u = 2^-24 (fp32 unit roundoff), gamma_n = n u / (1 - n u), kp = round_up(k, 8), K = kp (the GEMMs run over the
zero-padded width).  The library is built without fast-math: divisions and square roots are correctly rounded.

Literal root, a run with iters = s leaves Zb = Z_{s-1} (unscaled, whatever the parity of s), Zh / Zl = its bf16 hi/lo
split, inv_tr, fin, and P = fin (Z_{s-1} + a Z_{s-1} Z_{s-1}^T) with a = fl(1/p).
  tr       root_scalars_kernel sums the (non-negative) diagonal of a PSD M in fixed order: a chain of ceil(k/256)
           per thread, 5 warp levels, 8 partials, then + fl(k eps): every term passes through at most
           D = ceil(k/256) + 5 + 8 + 2 roundings, so |fl(tr) - tr| <= gamma_D tr (fp64 tr = sum diag + k eps).
  inv_tr   one correctly rounded division: rel <= gamma_D / (1 - gamma_D) + u (1 + that).
  fin      powf(tr, e) with the kernel's fp32 exponent e = fl(-1 / fl(p p)): the input error contributes
           max |(1 +- gamma_D)^e - 1| (~ |e| gamma_D), and powf its maximum error, 4 ulp <= 4 2^-23 |fin|
           (CUDA C++ Programming Guide, mathematical functions).
  Z0       fl(fl(M + eps [r == c < k]) inv_tr), bit for bit on the kernel's inv_tr: no row r >= k gets eps.
  Zh, Zl   Zh == bf16_rn(Zb), Zl == bf16_rn(Zb - Zh), bit for bit (ns_check.check_split).
  P        the three accumulating GEMMs of gemm3, Zh Zh^T + Zh Zl^T + Zl Zh^T, with alpha = a fin and C = Zb scaled by
           fin: ns_check's three-GEMM bound |D - R| <= C32 (K + 2) u P, P = fin a (sum |.||.|) + fin |Zb|.
  link     Zb of the s + 1 run (Z_s) against the same product on the s run's operands, unscaled.  With Z0 bit for bit
           this covers every iterate that enters a product.  P_hi / P_lo must be split4(P) bit for bit, and the
           padding of P, P_hi and P_lo must be +0.0.
  A dropped Zh Zl^T term is about 2^-9 |Z||Z| / sqrt(K) against a bound of 2 K u |Z||Z|: it is rejected for K in the
  hundreds and below, not reliably at K = 1024 (tests/test_root_stage_check.py shows where).

Newton root.  Slots: T (region 0) and S (region 1) ping-pong the iteration matrix T, so after a run that executed s
iterations the T used in iteration s sits in region (s - 1) % 2 and the next T in region s % 2.  F = T_s^4 Mc_{s-1},
P = X_s, Xs = split3(X_s).
  ridge    eps max(lambda, 1e-6) with lambda the Rayleigh quotient of 32 power iterations.  With lambda_2 / lambda_1
           <= 1/2 the iteration error (1/2)^62 k is far below fp32, and what is left is arithmetic: the mat-vec and the
           v.w sum each add at most gamma_(k+6) rho lambda_1 (rho = |q|^T |M| |q| / lambda_1 for the top eigenvector q:
           |v|^T |M| |v|, and |v|^T |w| <= |v|^T |M| |v|), the normalisation |v|^2 - 1 at most gamma_(k+6) + 2 ulp of
           rsqrtf, and eps x one rounding: |ridge - eps lambda_1| <= ((2 rho + 1)(k + 8) + 1) u eps lambda_1.  On every
           spectrum the Rayleigh quotient cannot exceed lambda_1 by more than the same arithmetic with rho replaced by
           sigma = || |M| ||_2 / lambda_1.  M = 0 gives fl(eps 1e-6) exactly.
  z        5 / (2 sqrt(fro2)), fro2 = ||M||_F^2 + 2 ridge tr + k ridge^2: sums of non-negative terms.  ||M||_F^2 is a
           chain of ceil(k/32)^2 products per thread, 5 warp levels, 32 partials; tr ceil(k/1024), 5, 32; then three
           more operations: D_z = ceil(k/32)^2 + 1 + 5 + 32 + 4, rel(fro2) <= gamma_(D_z), and the square root
           (halving it, plus u) and the division (u): rel(z) <= gamma_(D_z) / 2 + 2 u (+ second order).
  init     on the kernel's ridge and z: Mc0 = z (M + ridge [diag]) and T = 1.25 [diag] - 0.25 Mc0 bit for bit, zero
           outside [:k, :k] whatever M holds there; X0 = powf(z, 1/4) within 4 ulp.  T (here and after each step) is
           rounded once, as the compiler's contraction fma(-0.25, x, d) does: 0.25 x is exact except in fp32's subnormal
           range, where a separately rounded 0.25 x flushes to +0.0 and fma gives -0.0 off the diagonal (seen on the
           H100 with tol = 0, where off-diagonal elements of F reach 2^-149).  A matrix with e0 = max|Mc0 - I| <= tol freezes at once and iterates on T = I.
  F        three gemm6 products.  One gemm6 product A B: the six kept products over 3-way splits have
           sum |parts| <= (1 + 2^-7) |x| per operand, the hh product over 64-wide K slices and five more add
           C32 K u and kp/64 + 5 roundings of the running sum, the dropped ml, lm, ll terms are below 2 u |A||B|:
           |D - AB| <= gamma |A||B|,  gamma = (1 + 2^-7)^2 C32 (K + 8 + kp/64) u.
           Chained: S1 = T^2 + E1, S2 = S1^2 + E2, F = S2 Mc + E3 with |E1| <= gamma |T|^2, |S1| <= (1 + gamma)|T|^2,
           |E2| <= gamma (1 + gamma)^2 |T|^4, so |S2 - T^4| <= ((1 + gamma)^3 - 1) |T|^4 (the T^2 error enters twice),
           and |F - T^4 Mc| <= ((1 + gamma)^4 - 1) |T|^4 |Mc|  (~ 4 gamma).
           Underflow: with tol = 0 the off-diagonal of Mc shrinks until products fall below fp32's range, where the
           relative model does not hold.  Each of the n = 6 (K + 8 + kp/64) operations behind one gemm6 element can
           lose at most 2^-126 (a flush to zero), eta = n 2^-126 absolute; carried through S1 S1 and S2 Mc it is at
           most eta (1 + K m_Mc (1 + 2 K m_S1)) with m the largest magnitudes, m_S1 <= (1 + gamma) K m_T^2 + eta.
  step     e' = max|F - I| over [:k, :k] (NaN counts as inf); accept iff e' <= fl(1.2f err); freeze iff rejected or
           e' <= tol.  err, iters, frozen, av, bv follow exactly.  Accepted: Mc = split3(F), else Mc keeps its bits.
           The next T is split3(1.25 [diag] - 0.25 F) bit for bit, or exactly I when freezing.
  X        accepted: P against fp64 X_{s-1} T_s within gamma |X||T| + eta (plus X0's 4 ulp at s = 1); rejected or frozen:
           P == X_{s-1} bit for bit.  Xs == split3(P) bit for bit in every run.
  frozen   F == Mc exactly (I times a split is exact), both T regions exactly I, nothing else changes.
  Every run: iters_out == iters, residual_out == err, and the padding of P, Mc, both T regions and Xs is +0.0.

Measured over tests/test_gpu_shampoo_root_stages.py on an H100 80GB HBM3 at a 700 W power limit, the largest error /
bound ratios were: literal P 0.21, literal Z_s 0.16, literal scalars 0.11, Newton F 0.11, Newton X = X T 0.17,
ridge 0.040, z 0.095.  Every bit-for-bit check held.

Failure messages name the root, the iteration, the stage and the matrix, and for matrices the element, as
gemm_check.where does: "(batch b, row r, col c)"; batch b is matrix b.
"""
from __future__ import annotations

import math
from typing import Dict, NamedTuple, Optional

import torch

from tests import gemm_check as gc
from tests import ns_check as nc
from tests import shampoo_root_check as C
from tests.ns_check import _a256

BF16, F32 = torch.bfloat16, torch.float32
U = 2.0 ** -24
POWF_ULP = 4.0          # maximum ulp error of powf, CUDA C++ Programming Guide
ROOT = 4                # the Newton root's r: X -> M^(-1/4)


def rup8(k: int) -> int:
    return (k + 7) // 8 * 8


def gamma(n: float) -> float:
    return n * U / (1.0 - n * U)


def f32(x: float) -> float:
    return float(torch.tensor(x, dtype=F32))


# ---- inputs -----------------------------------------------------------------------------------------------------------
def mixed_batch(k: int, batch: int, seed: int) -> torch.Tensor:
    """The spectra of shampoo_root_check.KINDS in turn, matrix i scaled by 10^(i % 5 - 2), zero padding to kp: with
    equal scales a matrix that read its neighbour's scalar would be invisible."""
    return C.batch_of([C.spectrum_matrix(C.KINDS[i % len(C.KINDS)], k, seed + i, scale=10.0 ** (i % 5 - 2))
                       for i in range(batch)], rup8(k))


def gap_matrix(k: int, seed: int, scale: float = 1.0) -> torch.Tensor:
    """lambda_2 / lambda_1 <= 0.4: a quarter of a well-conditioned matrix (spectrum in [1/4, 1/2]) plus a unit
    rank-one term (Weyl: lambda_1 >= 1.25, lambda_2 <= 1/2), where the power iteration reaches the fp32 floor."""
    g = torch.Generator().manual_seed(seed)
    u = torch.randn(k, 1, generator=g, dtype=torch.float64)
    A = C.spectrum_matrix("well", k, seed).double() / 4 + (u @ u.T) / float(u.norm()) ** 2
    return (((A + A.T) / 2) * scale).float()


def rejecting_matrix() -> torch.Tensor:
    """An 8 x 8 spectrum (log-uniform over 1e-6..1, random basis) whose first Newton step raises max|Mc - I| by 1.32x:
    the coupled iteration rejects it at iteration 1 (found by searching with the fp32 emulation of
    tests/test_root_stage_check.py; convergent spectra only reach the fp32 floor and stay there)."""
    g = torch.Generator().manual_seed(92)
    Q, _ = torch.linalg.qr(torch.randn(8, 8, generator=g, dtype=torch.float64))
    lam = 10 ** (torch.rand(8, generator=g, dtype=torch.float64) * 6 - 6)
    A = (Q * lam) @ Q.T
    return ((A + A.T) / 2).float()


def newton_batch(k: int, seed: int) -> torch.Tensor:
    """mixed_batch's six spectra, a gap-separated matrix (scale 0.1) and, at k = 8, the rejecting matrix."""
    mats = [C.spectrum_matrix(C.KINDS[i], k, seed + i, scale=10.0 ** (i % 5 - 2)) for i in range(len(C.KINDS))]
    mats.append(gap_matrix(k, seed + 6, 0.1))
    if k == 8:
        mats.append(rejecting_matrix())
    return C.batch_of(mats, rup8(k))


# ---- workspace maps ------------------------------------------------------------------------------------------------
class LiteralWs(NamedTuple):
    """Byte offsets in b200_shampoo_root's workspace (shampoo_root_workspace_bytes): Zb fp32 [batch, kp, kp], Zh, Zl
    bf16, inv_tr[batch], fin[batch] (right after inv_tr), end."""
    zb: int
    zh: int
    zl: int
    inv_tr: int
    fin: int
    end: int


def literal_ws(batch: int, k: int) -> LiteralWs:
    n = batch * rup8(k) ** 2
    zh = _a256(n * 4)
    zl = zh + _a256(n * 2)
    inv = zl + _a256(n * 2)
    return LiteralWs(0, zh, zl, inv, inv + 4 * batch, inv + _a256(batch * 8))


class NewtonWs(NamedTuple):
    """Byte offsets in b200_shampoo_root_newton's workspace (shampoo_root_newton_workspace_bytes): F fp32, then four
    3-way bf16 splits (T, S, Mc, Xs; h, m, l each a256(n * 2) apart), then seven [batch] scalar slots, end."""
    f: int
    t: int
    s: int
    mc: int
    xs: int
    ridge: int
    z: int
    err: int
    iters: int
    frozen: int
    av: int
    bv: int
    end: int


def newton_ws(batch: int, k: int) -> NewtonWs:
    n = batch * rup8(k) ** 2
    off = [0, _a256(n * 4)]
    for _ in range(3):
        off.append(off[-1] + 3 * _a256(n * 2))
    off.append(off[-1] + 3 * _a256(n * 2))
    for _ in range(7):
        off.append(off[-1] + _a256(batch * 4))
    return NewtonWs(*off)


def literal_views(ws: torch.Tensor, batch: int, k: int) -> Dict[str, torch.Tensor]:
    kp, w = rup8(k), literal_ws(batch, k)
    sh = (batch, kp, kp)
    return {"Zb": nc.ws_view(ws, w.zb, sh, F32), "Zh": nc.ws_view(ws, w.zh, sh), "Zl": nc.ws_view(ws, w.zl, sh),
            "inv_tr": nc.ws_view(ws, w.inv_tr, (batch,), F32), "fin": nc.ws_view(ws, w.fin, (batch,), F32)}


def newton_views(ws: torch.Tensor, batch: int, k: int) -> Dict[str, object]:
    """T0 / T1: regions 0 (the driver's T) and 1 (its S) as (h, m, l); Mc, Xs likewise; F and the scalar slots."""
    kp, w = rup8(k), newton_ws(batch, k)
    sh, step = (batch, kp, kp), _a256(batch * kp * kp * 2)

    def three(o):
        return tuple(nc.ws_view(ws, o + i * step, sh) for i in range(3))
    out = {"F": nc.ws_view(ws, w.f, sh, F32), "T0": three(w.t), "T1": three(w.s), "Mc": three(w.mc),
           "Xs": three(w.xs)}
    for name in ("ridge", "z", "err", "av", "bv"):
        out[name] = nc.ws_view(ws, getattr(w, name), (batch,), F32)
    for name in ("iters", "frozen"):
        out[name] = nc.ws_view(ws, getattr(w, name), (batch,), torch.int32)
    return out


# ---- exact helpers ---------------------------------------------------------------------------------------------------
def split3(x: torch.Tensor):
    """split3f of csrc/shampoo.cu on fp32 x: h = bf16_rn(x), m = bf16_rn(x - h), l = bf16_rn(x - h - m); h + m + l == x."""
    h = x.to(BF16)
    r = x - h.float()
    m = r.to(BF16)
    return h, m, (r - m.float()).to(BF16)


def value3(s) -> torch.Tensor:
    return s[0].double() + s[1].double() + s[2].double()


def _masks(kp: int, k: int, device):
    i = torch.arange(kp, device=device)
    inside = (i.view(-1, 1) < k) & (i.view(1, -1) < k)
    diag = (i.view(-1, 1) == i.view(1, -1)) & (i.view(-1, 1) < k)
    return inside, diag


def identity(batch: int, kp: int, k: int, device) -> torch.Tensor:
    return _masks(kp, k, device)[1].to(F32).expand(batch, kp, kp).contiguous()


_INT = {BF16: torch.int16, F32: torch.int32, torch.int32: torch.int32}


def same_bits(got: torch.Tensor, exp: torch.Tensor, what: str, sel: Optional[torch.Tensor] = None) -> None:
    """got == exp bit for bit, over the matrices selected by the bool [batch] `sel` (all by default)."""
    it = _INT[got.dtype]
    bad = got.contiguous().view(it) != exp.to(got.dtype).contiguous().view(it)
    if sel is not None:
        bad = bad & sel.view(-1, *([1] * (bad.dim() - 1)))
    if bool(bad.any()):
        i = int(bad.flatten().nonzero()[0])
        loc = gc.where(got, i) if got.dim() == 3 else f"matrix {i}"
        raise AssertionError(f"{what}: {int(bad.sum())} elements differ in their bits; first at {loc}: got "
                             f"{float(got.flatten()[i])!r}, expected {float(exp.flatten()[i])!r}")


def same_split(s, x: torch.Tensor, what: str, sel: Optional[torch.Tensor] = None) -> None:
    """A stored 3-way split (h, m, l) equals split3 of fp32 x bit for bit."""
    for part, want, nm in zip(s, split3(x), "hml"):
        same_bits(part, want, f"{what} ({nm})", sel)


def zero_padding(x: torch.Tensor, k: int, what: str) -> None:
    """+0.0 outside [:k, :k]; bf16 widens exactly to fp32, -0.0 and NaN included."""
    nc.zero_padding_bits(x.float(), k, what)


def check_rel(got: torch.Tensor, ref: torch.Tensor, bound, what: str) -> float:
    """Per matrix |got - ref| <= bound |ref| (bound a float or an fp64 [batch] tensor); returns the worst ratio."""
    err = (got.double() - ref).abs()
    lim = torch.as_tensor(bound, dtype=torch.float64, device=ref.device) * ref.abs()
    ratio = torch.where(err == 0, torch.zeros_like(err), err / lim)
    ratio = torch.where(torch.isfinite(got.double()), ratio, torch.full_like(ratio, math.inf))
    b = int(ratio.argmax())
    if not float(ratio[b]) <= 1.0:
        raise AssertionError(f"{what}: matrix {b}: got {float(got[b])!r}, reference {float(ref[b])!r}, relative error "
                             f"exceeds its bound by {float(ratio[b]):.3g}x")
    return float(ratio.max())


def check_gamma(D, R, P, g: float, what: str, extra=None) -> gc.Bound:
    """|D - R| <= g P (+ extra), element by element."""
    return gc.check_bound(D, R, P, 1, what, c32=g / U, extra=extra)


def _ratio(bounds: Dict[str, float], name: str, b) -> None:
    v = b.ratio if isinstance(b, gc.Bound) else float(b)
    bounds[name] = max(bounds.get(name, 0.0), v)


# ---- literal root ----------------------------------------------------------------------------------------------------
def literal_z0(M: torch.Tensor, k: int, eps: float, inv_tr: torch.Tensor) -> torch.Tensor:
    """root_init_kernel's Z0 in fp32: eps on the diagonal rows r < k only, then times the matrix's inv_tr."""
    _, diag = _masks(M.shape[-1], k, M.device)
    return torch.where(diag, M + torch.tensor(eps, dtype=F32, device=M.device), M) * inv_tr.view(-1, 1, 1)


def literal_reference(Zh, Zl, Zb, p: float, fin=None):
    """fp64 (R, P) of gemm3's fin (a (Zh Zh^T + Zh Zl^T + Zl Zh^T) + Zb), a = fl(1/p); fin None: unscaled."""
    a = f32(1.0 / f32(p))
    R, P = gc.reference(Zh, Zh, alpha=a, alpha_vec=fin, beta=1.0, beta_vec=fin, C=Zb)
    for x, y in ((Zh, Zl), (Zl, Zh)):
        r, q = gc.reference(x, y, alpha=a, alpha_vec=fin)
        R, P = R + r, P + q
    return R, P


def check_literal_scalars(M, k: int, p: float, eps: float, inv_tr, fin, what: str) -> float:
    d = torch.diagonal(M[:, :k, :k].double(), dim1=1, dim2=2)
    tr = d.sum(1) + k * f32(eps)
    g = gamma(-(-k // 256) + 5 + 8 + 2)
    rel_inv = g / (1 - g)
    w = check_rel(inv_tr, 1.0 / tr, rel_inv + U * (1 + rel_inv), f"{what}, inv_tr")
    e = f32(-1.0 / f32(p * p))
    rel_in = max(abs((1 + g) ** e - 1), abs((1 - g) ** e - 1))
    return max(w, check_rel(fin, tr ** e, rel_in + POWF_ULP * 2 * U * (1 + rel_in), f"{what}, fin"))


def check_literal_run(M, k: int, p: float, eps: float, s: int, cur: Dict, nxt: Optional[Dict] = None,
                      what: str = "") -> Dict[str, float]:
    """The state a b200_shampoo_root run with iters = s left: cur = literal_views + "P" (+ "Ph", "Pl"); nxt: the
    iters = s + 1 run's state, whose Zb (= Z_s) is checked on this run's operands.  Returns family -> worst ratio."""
    tag = f"literal root{', ' + what if what else ''}: iteration {s}"
    kp = M.shape[-1]
    out: Dict[str, float] = {}
    _ratio(out, "literal scalars", check_literal_scalars(M, k, p, eps, cur["inv_tr"], cur["fin"], tag))
    if s == 1:
        same_bits(cur["Zb"], literal_z0(M, k, eps, cur["inv_tr"]), f"{tag}, Z0 = (M + eps I) inv_tr")
    nc.check_split(cur["Zb"], cur["Zh"], cur["Zl"], f"{tag}, Zh/Zl split of Z_{s - 1}")
    R, P = literal_reference(cur["Zh"], cur["Zl"], cur["Zb"], p, cur["fin"])
    _ratio(out, "literal P", gc.check_bound(cur["P"], R, P, kp + 2, f"{tag}, P = fin (Z + Z Z / p)"))
    zero_padding(cur["P"], k, f"{tag}, P")
    if cur.get("Ph") is not None:
        nc.check_split(cur["P"], cur["Ph"], cur["Pl"], f"{tag}, P_hi/P_lo")
        zero_padding(cur["Ph"], k, f"{tag}, P_hi")
        zero_padding(cur["Pl"], k, f"{tag}, P_lo")
    if nxt is not None:
        R, P = literal_reference(cur["Zh"], cur["Zl"], cur["Zb"], p)
        _ratio(out, "literal Z_s", gc.check_bound(nxt["Zb"], R, P, kp + 2, f"{tag}, Z_{s} = Z + Z Z / p"))
    return out


# ---- Newton root -----------------------------------------------------------------------------------------------------
def gemm6_gamma(kp: int) -> float:
    return (1 + 2.0 ** -7) ** 2 * gc.C32 * (kp + 8 + kp / 64) * U


def gemm6_eta(kp: int) -> float:
    """Absolute underflow allowance of one gemm6 element (docstring)."""
    return 6 * (kp + 8 + kp / 64) * 2.0 ** -126


def _amax(x: torch.Tensor) -> torch.Tensor:
    return x.abs().flatten(1).max(1).values.view(-1, 1, 1)


def newton_init(M: torch.Tensor, k: int, ridge: torch.Tensor, z: torch.Tensor):
    """newton_init_kernel in fp32 on the kernel's own ridge and z: (Mc0, T, e0)."""
    inside, diag = _masks(M.shape[-1], k, M.device)
    zero = torch.zeros((), dtype=F32, device=M.device)
    add = torch.where(diag, ridge.view(-1, 1, 1), zero)
    mc = torch.where(inside, z.view(-1, 1, 1) * (M + add), zero)
    return mc, next_t(mc, k), max_dev(mc, k)


def max_dev(F: torch.Tensor, k: int) -> torch.Tensor:
    """max |F - I| over [:k, :k] per matrix in fp32, NaN counted as +inf (abs_dev)."""
    d = (F[:, :k, :k] - identity(1, k, k, F.device)).abs()
    d = torch.where(torch.isnan(d), torch.full_like(d, math.inf), d)
    return d.flatten(1).max(1).values


def next_t(F: torch.Tensor, k: int) -> torch.Tensor:
    """1.25 [diag] - 0.25 F rounded once to fp32, as the kernels' contracted fma(-0.25, F, d) does (docstring)."""
    _, diag = _masks(F.shape[-1], k, F.device)
    d = torch.where(diag, torch.tensor(1.25, dtype=torch.float64, device=F.device),
                    torch.zeros((), dtype=torch.float64, device=F.device))
    return (d - 0.25 * F.double()).float()


def check_newton_scalars(M, k: int, eps: float, ridge, z, what: str) -> Dict[str, float]:
    out: Dict[str, float] = {}
    Md = M[:, :k, :k].double()
    lam, Q = torch.linalg.eigh(Md)
    l1 = lam[:, -1]
    e32 = f32(eps)
    zero = (Md == 0).flatten(1).all(1)
    if bool(zero.any()):
        same_bits(ridge, torch.full_like(ridge, f32(e32 * f32(1e-6))), f"{what}, ridge of M = 0", zero)
    sigma = torch.linalg.matrix_norm(Md.abs(), ord=2) / l1.clamp_min(1e-300)
    upper = e32 * torch.maximum(l1, torch.full_like(l1, f32(1e-6))) * (1 + ((2 * sigma + 1) * (k + 8) + 1) * U)
    over = ~(ridge.double() <= upper) & ~zero
    if bool(over.any()):
        b = int(over.nonzero()[0])
        raise AssertionError(f"{what}, ridge: matrix {b}: {float(ridge[b])!r} exceeds eps lambda_max "
                             f"{float(e32 * l1[b]):.9g} by more than its arithmetic")
    gap = (lam[:, -2] <= 0.5 * l1) & (l1 > 1e-6)
    if bool(gap.any()):
        q = Q[:, :, -1:]
        rho = (q.abs().transpose(1, 2) @ Md.abs() @ q.abs()).view(-1) / l1.clamp_min(1e-300)
        bound = ((2 * rho + 1) * (k + 8) + 1) * U
        idx = gap.nonzero().view(-1)
        r = check_rel(ridge[idx], e32 * l1[idx], bound[idx], f"{what}, ridge (gap-separated spectra, indices of "
                                                                f"{idx.tolist()})")
        _ratio(out, "newton ridge", r)
    ss = (Md * Md).flatten(1).sum(1)
    tr = torch.diagonal(Md, dim1=1, dim2=2).sum(1)
    rd = ridge.double()
    zref = (1.0 + ROOT) / (2 * torch.sqrt(ss + 2 * rd * tr + k * rd * rd))
    d = (-(-k // 32)) ** 2 + 1 + 5 + 32 + 4
    _ratio(out, "newton z", check_rel(z, zref, gamma(d) / 2 * (1 + gamma(d)) + 2 * U * (1 + U), f"{what}, z"))
    return out


def _state_same(got, exp, what, name):
    bad = got.view(_INT[got.dtype]) != exp.to(got.dtype).view(_INT[got.dtype])
    if bool(bad.any()):
        b = int(bad.nonzero()[0])
        raise AssertionError(f"{what}, state: matrix {b}: {name} is {got[b].item()!r}, the state machine gives "
                             f"{exp[b].item()!r}")


def check_newton_run(M, k: int, eps: float, tol: float, s: int, cur: Dict, prev: Optional[Dict] = None,
                     what: str = "") -> Dict[str, object]:
    """The state a b200_shampoo_root_newton run that executed s iterations left: cur = newton_views + "P" (+
    "iters_out", "residual_out"); prev: the s - 1 run's (None for s = 1).  Returns {"bounds": family -> worst
    ratio, "branches": branch -> count, "frozen": bool [batch] after iteration s}."""
    tag = f"newton root{', ' + what if what else ''}: iteration {s}"
    batch, kp, _ = M.shape
    dev = M.device
    bounds: Dict[str, float] = {}
    g = gemm6_gamma(kp)
    tol32 = torch.tensor(tol, dtype=F32, device=dev)
    I = identity(batch, kp, k, dev)
    x0_extra = None
    if prev is None:
        bounds.update(check_newton_scalars(M, k, eps, cur["ridge"], cur["z"], tag))
        mc0, t1, e0 = newton_init(M, k, cur["ridge"], cur["z"])
        fz = e0 <= tol32
        err_p, iters_p, frozen_p = e0, torch.zeros(batch, dtype=torch.int32, device=dev), fz
        mc_bits, mc_val = split3(mc0), mc0.double()
        x_ref = cur["z"].double().pow(1.0 / ROOT).view(-1, 1, 1) * I.double()
        x0_extra = POWF_ULP * 2 * U * (1 + 2 * U) * x_ref.abs()
        Ts = cur["T0"]
        same_split(Ts, t1, f"{tag}, init T = 1.25 I - 0.25 Mc0", ~fz)
        same_split(Ts, I, f"{tag}, init T of a matrix frozen at init", fz)
    else:
        err_p, iters_p, frozen_p = prev["err"], prev["iters"], prev["frozen"] != 0
        mc_bits, mc_val = prev["Mc"], value3(prev["Mc"])
        x_ref = prev["P"].double()
        Ts = cur[f"T{(s - 1) % 2}"]
        for a, b, nm in zip(Ts, prev[f"T{(s - 1) % 2}"], "hml"):
            same_bits(a, b, f"{tag}, T_{s} ({nm}) differs from the T the s - 1 run left")
    Tn = cur[f"T{s % 2}"]
    active = ~frozen_p
    F = cur["F"]
    # F = T^4 Mc
    T = value3(Ts)
    R = torch.bmm(torch.bmm(torch.bmm(T, T), torch.bmm(T, T)), mc_val)
    Ta = T.abs()
    T2 = torch.bmm(Ta, Ta)
    P4 = torch.bmm(torch.bmm(T2, T2), mc_val.abs())
    sel = active.view(-1, 1, 1)
    eta = gemm6_eta(kp)
    m_s1 = (1 + g) * kp * _amax(T) ** 2 + eta
    eta_f = (eta * (1 + kp * _amax(mc_val) * (1 + 2 * kp * m_s1))).expand_as(P4)
    _ratio(bounds, "newton F = T^4 Mc",
           check_gamma(F, torch.where(sel, R, F.double()), P4, (1 + g) ** 4 - 1, f"{tag}, F = T^4 Mc", eta_f))
    if bool(frozen_p.any()):
        gc.check_exact(torch.where(sel, mc_val.float(), F), mc_val, f"{tag}, F = I Mc of a frozen matrix")
        same_split(Ts, I, f"{tag}, T of a frozen matrix", frozen_p)
    # the state machine
    e = max_dev(F, k)
    accept = e <= torch.tensor(1.2, dtype=F32, device=dev) * err_p
    freeze = ~accept | (e <= tol32)
    acc = active & accept
    exp = {"err": torch.where(acc, e, err_p), "iters": iters_p + acc.to(torch.int32),
           "frozen": (frozen_p | (active & freeze)).to(torch.int32),
           "av": acc.to(F32), "bv": (~acc).to(F32)}
    for name, v in exp.items():
        _state_same(cur[name], v, tag, name)
    if cur.get("iters_out") is not None:
        _state_same(cur["iters_out"], cur["iters"], tag, "iters_out")
    if cur.get("residual_out") is not None:
        _state_same(cur["residual_out"], cur["err"], tag, "residual_out")
    same_split(cur["Mc"], F, f"{tag}, Mc = split3(F) after an accepted step", acc)
    for a, b, nm in zip(cur["Mc"], mc_bits, "hml"):
        same_bits(a, b, f"{tag}, Mc ({nm}) of a rejected or frozen matrix changed", ~acc)
    same_split(Tn, next_t(F, k), f"{tag}, next T = 1.25 I - 0.25 F", active & ~freeze)
    same_split(Tn, I, f"{tag}, next T of a freezing or frozen matrix", freeze | frozen_p)
    # X
    Pout = cur["P"]
    R, Pb = torch.bmm(x_ref, T), torch.bmm(x_ref.abs(), Ta)
    extra = torch.full_like(Pb, eta) if x0_extra is None else torch.bmm(x0_extra, Ta) + eta
    sa = acc.view(-1, 1, 1)
    _ratio(bounds, "newton X = X T", check_gamma(Pout, torch.where(sa, R, Pout.double()), Pb, g, f"{tag}, X = X T",
                                                  extra))
    if x0_extra is None:
        same_bits(Pout, prev["P"], f"{tag}, X of a rejected or frozen matrix changed", ~acc)
    else:
        check_gamma(Pout, torch.where(sa, Pout.double(), x_ref), torch.zeros_like(x_ref), 0.0,
                    f"{tag}, X0 = z^(1/4) I of a rejected or frozen matrix", x0_extra)
    same_split(cur["Xs"], Pout, f"{tag}, Xs = split3(X)")
    zero_padding(Pout, k, f"{tag}, P")
    for name in ("Mc", "T0", "T1", "Xs"):
        for part, nm in zip(cur[name], "hml"):
            zero_padding(part, k, f"{tag}, {name} ({nm})")
    conv = acc & (e <= tol32)
    branches = {"accept": int((acc & ~conv).sum()), "converge-freeze": int(conv.sum()),
                "reject": int((active & ~accept).sum()),
                "freeze at init": int(frozen_p.sum()) if prev is None else 0}
    return {"bounds": bounds, "branches": branches, "frozen": (cur["frozen"] != 0).clone()}
