"""Element-wise references and checker for the wgmma GEMM engine (csrc/gemm_wgmma.cu).  Imports without a GPU.

Every engine output is checked against D[b] = alpha*av[b] * op(A[b]) op(B[b]) + beta*bv[b] * C[b] computed in
fp64, element by element, in one of two input families:

exact   Operands and C are integers in [-8, 8]; alpha, beta, alpha_vec and beta_vec are powers of two.  Every
        product and partial sum is an integer (times a power of two) below 2^24, so fp32 accumulation is exact in
        any order and the expected output is known bit for bit: D == R for fp32 out, D == bf16_rn(R) for bf16 out.
        Any misplaced chunk, tile, mirror, k-block or batch index, and any rounding other than round-to-nearest-
        even, fails.  (Ties such as 257 -> 256 come up naturally, so truncation is caught too.)
bound   Gaussian operands.  With P = |alpha*av[b]| |op(A)||op(B)| + |beta*bv[b]*C| (fp64), per element
            fp32 out:  |D - R| <= C32 * K * 2^-24 * P
            bf16 out:  |D - R| <= 2^-8 |R| + C32 * K * 2^-24 * P
        C32 covers Hopper's fp32 tensor-core accumulation, which is not IEEE round-to-nearest.

C32 = 2 is the worst case of K-term summation rounded toward zero (unit error 2^-23 per addition).  Measured over
tests/test_gpu_gemm_engine.py on an H100 80GB HBM3 at a 700 W power limit:
    accumulation error, in units of K * 2^-24 * P      at most 0.0032 (fp32 out), 0.0018 (bf16 out, GLU, Newton-Schulz)
    largest |D - R| / bound with C32 = 2               fp32 out 0.0016; bf16 out 0.994 (bf16's half ulp is up to
                                                       2^-8 |R|: the rounding term is tight by design); GLU y 0.74,
                                                       GLU dgu 0.84; Newton-Schulz stages 0.99
So C32 = 2 is about 600x the largest accumulation error seen.  The exact family held bit for bit.

Both families require every element to be finite, and a failure names the worst element's (batch, row, col), its
128 x 128 tile and its 8-element chunk (col % 128 // 8), which is what a swizzle, mirror or raster slip changes.
tests/test_gemm_check.py shows on the CPU that the checker accepts correct outputs and rejects planted faults.

`Guarded` holds an output or operand inside a larger buffer filled with a NaN canary bit pattern (row pitch > row
length, a gap between batch strides, guard elements before and after), so a test can show that the engine writes
only where it should and never reads operand padding.
"""
from __future__ import annotations

from typing import NamedTuple

import torch

C32 = 2.0
TILE = 128
CHUNK = 8
# tanh.approx.f32 has a maximum relative error of about 2^-11 (PTX ISA); sigmoid(x) = 0.5 + 0.5 tanh(x / 2) with
# |tanh| <= 1 is then off by at most 2^-12 plus one fp32 fma rounding: 2^-11 bounds both.
EPS_SIGMA = 2.0 ** -11


def op(X: torch.Tensor, mn: bool) -> torch.Tensor:
    """[batch, rows, K] view of an operand stored K-major ([batch, rows, K]) or MN-major ([batch, K, rows])."""
    return X.transpose(1, 2) if mn else X


def _scale(s: float, vec, batch: int, device) -> torch.Tensor:
    out = torch.full((batch, 1, 1), float(s), dtype=torch.float64, device=device)
    if vec is not None:
        out = out * vec.double().view(-1, 1, 1)
    return out


def reference(A, B, *, a_mn=False, b_mn=False, alpha=1.0, beta=0.0, alpha_vec=None, beta_vec=None, C=None):
    """fp64 (R, P) of D[b] = alpha*av[b] op(A[b]) op(B[b])^T + beta*bv[b] C[b].

    A: [batch, M, K] (a_mn=False) or [batch, K, M]; B: [batch, N, K] (b_mn=False) or [batch, K, N]; C: [batch, M, N].
    Call it with the operands as the kernel read them (bf16 values, fp32 scale vectors)."""
    a, b = op(A.double(), a_mn), op(B.double(), b_mn)
    sa = _scale(alpha, alpha_vec, a.shape[0], a.device)
    R = sa * torch.bmm(a, b.transpose(1, 2))
    P = sa.abs() * torch.bmm(a.abs(), b.abs().transpose(1, 2))
    if C is not None and beta != 0.0:
        cb = _scale(beta, beta_vec, a.shape[0], a.device) * C.double()
        R = R + cb
        P = P + cb.abs()
    return R, P


def bf16_rn(R: torch.Tensor) -> torch.Tensor:
    """Round-to-nearest-even bf16 of R.  Exact for the exact family, whose values are fp32-representable."""
    return R.float().to(torch.bfloat16)


def exact_ints(shape, device="cpu", generator=None) -> torch.Tensor:
    """Integers in [-8, 8] as fp32 (cast to bf16 by the caller: exactly representable)."""
    return torch.randint(-8, 9, shape, device=device, generator=generator).float()


def where(D: torch.Tensor, flat_index: int) -> str:
    """(batch, row, col), tile and chunk of element `flat_index` of a [batch, rows, cols] tensor."""
    _, rows, cols = D.shape
    b, r, c = flat_index // (rows * cols), flat_index // cols % rows, flat_index % cols
    return f"(batch {b}, row {r}, col {c}) in tile ({r // TILE}, {c // TILE}), chunk {c % TILE // CHUNK}"


def _as3(D: torch.Tensor) -> torch.Tensor:
    return D if D.dim() == 3 else D.reshape(1, *D.shape[-2:])


def check_finite(D: torch.Tensor, what: str = "") -> None:
    D = _as3(D)
    bad = ~torch.isfinite(D.float())
    if bool(bad.any()):
        i = int(bad.flatten().nonzero()[0])
        raise AssertionError(f"{what}: {int(bad.sum())} non-finite elements; first at {where(D, i)}")


def check_exact(D: torch.Tensor, R: torch.Tensor, what: str = "") -> None:
    """Exact family: fp32 D must equal R, bf16 D must equal bf16_rn(R), bit for bit."""
    D, R = _as3(D), _as3(R)
    check_finite(D, what)
    exp = R.float() if D.dtype == torch.float32 else bf16_rn(R)
    if torch.equal(D, exp):
        return
    diff = (D.double() - exp.double()).abs()
    i = int(diff.flatten().argmax())
    raise AssertionError(f"{what}: {int((diff != 0).sum())} of {D.numel()} elements differ from the exact result; "
                         f"worst at {where(D, i)}: got {float(D.flatten()[i])}, expected {float(exp.flatten()[i])}")


class Bound(NamedTuple):
    ratio: float   # largest |D - R| / bound
    c32: float     # smallest C32 that would still pass: the accumulation error seen, in units of K 2^-24 P


def check_bound(D: torch.Tensor, R: torch.Tensor, P: torch.Tensor, K: int, what: str = "", c32: float = C32,
                extra=None) -> Bound:
    """Bound family: per-element error bound (module docstring), plus `extra` (an fp64 tensor) where an epilogue
    adds error of its own."""
    D, R, P = _as3(D), _as3(R), _as3(P)
    check_finite(D, what)
    err = (D.double() - R).abs()
    fixed = torch.zeros_like(err)
    if D.dtype == torch.bfloat16:
        fixed = fixed + 2.0 ** -8 * R.abs()
    if extra is not None:
        fixed = fixed + _as3(extra)
    unit = K * 2.0 ** -24 * P
    bound = c32 * unit + fixed
    ratio = torch.where(err == 0, torch.zeros_like(err), err / bound)   # bound == 0 < err -> inf
    i = int(ratio.flatten().argmax())
    worst = float(ratio.flatten()[i])
    if not worst <= 1.0:
        raise AssertionError(f"{what}: |D - R| exceeds its bound by {worst:.3g}x at {where(D, i)}: got "
                             f"{float(D.flatten()[i])}, reference {float(R.flatten()[i])}, bound "
                             f"{float(bound.flatten()[i]):.3g} ({int((ratio > 1).sum())} elements over)")
    acc = (err - fixed).clamp_min(0)
    need = torch.where(acc == 0, torch.zeros_like(acc), acc / unit)
    return Bound(worst, float(need.max()))


def check(D, R, P, K, exact: bool, what: str = "") -> Bound:
    """check_exact or check_bound, by family (the exact family returns Bound(0, 0))."""
    if exact:
        check_exact(D, R, what)
        return Bound(0.0, 0.0)
    return check_bound(D, R, P, K, what)


# ---- canary-guarded buffers ---------------------------------------------------------------------------------
_INT = {torch.bfloat16: torch.int16, torch.float32: torch.int32}
CANARY = {torch.bfloat16: 0x7FB5, torch.float32: 0x7FB5A5A5}   # NaN bit patterns


def round_up(x: int, m: int) -> int:
    return (x + m - 1) // m * m


class Guarded:
    """A [batch, rows, cols] array stored at row pitch `ld` and batch stride `stride` inside a larger buffer that
    starts out as the CANARY (a NaN) everywhere: `guard` elements before and after, columns beyond `cols` up to
    `ld`, rows beyond `rows` up to `stride`.  `ld`, `stride` and `guard` keep 16-byte alignment."""

    def __init__(self, batch, rows, cols, dtype, device, *, ld=None, stride=None, guard=64):
        vec = 16 // torch.tensor([], dtype=dtype).element_size()
        self.batch, self.rows, self.cols, self.dtype = batch, rows, cols, dtype
        self.ld = ld if ld is not None else round_up(cols, vec) + vec
        self.stride = stride if stride is not None else (rows + 2) * self.ld + vec
        assert self.ld % vec == 0 and self.stride % vec == 0 and guard % vec == 0
        self.guard = guard
        size = guard + (batch - 1) * self.stride + rows * self.ld + guard
        self.buf = torch.empty(size, dtype=dtype, device=device)
        self.buf.view(_INT[dtype]).fill_(CANARY[dtype])

    def view(self, cols=None) -> torch.Tensor:
        """The [batch, rows, cols] array (cols defaults to the logical width; wider views reach the padding)."""
        c = self.cols if cols is None else cols
        return self.buf.as_strided((self.batch, self.rows, c), (self.stride, self.ld, 1), self.guard)

    def ptr(self) -> int:
        return self.view().data_ptr()

    def check_canaries(self, cols: int, what: str = "") -> None:
        """Every element outside rows < self.rows, columns < `cols` of each batch must still hold the canary."""
        mask = torch.zeros(self.buf.numel(), dtype=torch.bool, device=self.buf.device)
        mask.as_strided((self.batch, self.rows, cols), (self.stride, self.ld, 1), self.guard).fill_(True)
        bad = (self.buf.view(_INT[self.dtype]) != CANARY[self.dtype]) & ~mask
        if bool(bad.any()):
            o = int(bad.nonzero()[0])
            rel = o - self.guard
            if rel < 0:
                loc = f"{-rel} elements before the array"
            elif rel >= (self.batch - 1) * self.stride + self.rows * self.ld:
                loc = f"{rel - (self.batch - 1) * self.stride - self.rows * self.ld} elements after the array"
            else:
                loc = f"batch {rel // self.stride}, row {rel % self.stride // self.ld}, col {rel % self.ld}"
            raise AssertionError(f"{what}: {int(bad.sum())} canary elements overwritten outside rows < {self.rows}, "
                                 f"cols < {cols}; first at {loc}")
