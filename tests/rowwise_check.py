"""fp64 references with per-element bounds for the memory-bound kernels: RMSNorm / add-RMSNorm and their backward and
dW reductions (csrc/norm_rope.cu), RoPE, the GLU activations, cross entropy, the embedding scatter (csrc/model_fused.cu)
and the flat optimizer updates (first half of csrc/elementwise.cu).  Pure torch, works on any device, does not import
the package.  tests/test_rowwise_check.py shows on the CPU what the checker accepts and rejects;
tests/test_gpu_rowwise_kernels.py feeds it kernel outputs.

Every function takes the kernel's inputs already rounded to their storage type T and returns {name: (ref64, bound)};
`check` asserts |got - ref| <= bound for every element.  A bound of 0 means "this value, exactly".

Notation: u24 = 2^-24 (fp32 unit roundoff), u8 = 2^-8 (one bf16 rounding, the convention of the other checkers),
rnd_T(r) = u8 |r| for bf16 outputs and u24 |r| for fp32 ones, C = 4 (the attention checkers' constant), H the row
length, R the number of rows.

RMSNorm forward (rmsnorm_fwd_kernel / rmsnorm_fwd_warp_kernel).  s = round_T(x + delta) is one fp32 add of two
  T values rounded to T, which torch reproduces: bound 0.  tot = sum s^2 is H products and H adds of non-negative
  terms in any order, relative error <= (H + 1) u24; / H, + eps, sqrt and the reciprocal halve it and add 4 roundings:
      |rstd - R| <= C u24 (H + 2) R              (C = 4 leaves more than the worst case (H/2 + 5) u24)
  y = s rstd w, two more roundings:  |y - R| <= C u24 (H + 4) |R| + [bf16] u8 |R|.
RMSNorm backward (rmsnorm_bwd_kernel / rmsnorm_bwd_warp_kernel), g = dy w, c = rstd^2 mean(g x), taking the kernel's
  own rstd as an input so that the forward's error is not counted twice:
      dx = rstd (g - x c) [+ dres]
      |dx - R| <= C u24 H rstd (|g| + |x| rstd^2 mean|g x|) + [dres] C u24 |dres| + rnd_T(R)
  (the H-term dot product has error <= H u24 mean|g x|; the other five roundings are covered by H >= 8).
  dW[c] = sum_r dy x rstd: two products per term, then R adds split over per-CTA partials and the column reduction,
      |dW - R| <= C u24 R sum_r |dy x rstd|      (+ C u24 |prior| + rnd_T(R) when accumulated into a stored gradient)
  `colsum` is the same bound for b200_rmsnorm_dw_reduce on a given partials buffer.
RoPE (rope_kernel, rope_half_kernel), tables fp32 as given: out_a = x_a c - x_b s, out_b = x_a s + x_b c is two
  products, one sum (or one product and an fma):  |out - R| <= C u24 (|x_a c| + |x_b s|) + rnd_T(R).  The backward is
  the same rotation with s -> -s.
GLU.  sigmoidf_(x) = 1 / (1 + __expf(-x)).  The CUDA programming guide gives __expf a maximum error of
  2 + floor(|1.173 x|) ulp, i.e. relative EXPF(x) = 2 u24 (2 + 1.173 |x|).  With e = exp(-x), d ln sigma / d ln e =
  -(1 - sigma), so  dsig(x) = sigma ((1 - sigma) EXPF(x) + C u24)  bounds |sigma~ - sigma|.  1 - sigma~ (computed as
  1.0f - s) then has absolute error dsig + u24 -- it is 0 for x >= 17 where the true value is e^-x -- so factors
  (1 - sigma) get an absolute, not a relative, term.  Products of factors f_i with errors d_i are bounded by
  sum_i d_i prod_{j != i} |f_j| + C u24 |product| + rnd_T:
      sigmoid2  y  = 2 g sig(u)                    dg = 2 dy sig(u)       du = 2 dy g sig(u) (1 - sig(u))
      silu      y  = g sig(g) u                    du = dy g sig(g)       dg = dy u sig(g) (1 + g (1 - sig(g)))
Cross entropy (ce_fwd_kernel, ce_bwd_kernel), columns < V only.  lse = M + log S.  S is a sum of V terms
  exp(x - m), per-thread chains of V/4096 vectors of 8, then 5 + 16 merges.  The relative error of each term is
  EXPF(x - m) + u24 |x - m|, weighted by p; sum_j p_j (m - x_j) <= entropy <= ln V, so that part is below 40 u24.  A
  relative error of S is an absolute error of lse, and M + log S rounds to u24 (max|x| + ln V):
      |lse - R| <= C u24 (V/512 + 16 + max|x|),   loss = lse - x_t with the same bound, exactly 0 on pad rows.
  Backward, given the kernel's lse: d = bf16(scale (p - [j = t])) with p = exp(x - lse).  x - lse rounds to
  u24 |x - lse|, __expf adds EXPF(x - lse), the subtraction and product two more:
      |d - R| <= u8 |R| + C u24 (2 + |x_j - lse|) |scale| p_j,   exactly 0 for V <= j < ld and on pad rows.
Embedding scatter (embedding_scatter_kernel + embedding_accumulate_kernel): fp32 atomic adds of n_hits rows in any
  order, then one add into the stored gradient:
      |dW - R| <= u24 n_hits sum_hits |dh| + u24 |prior| + rnd_T(R); a row no token hits has bound 0 (unchanged).
Optimizer updates.  The formula of each kernel in fp64 from its fp32 / bf16 inputs.  Each fp32 output is a sum of a
  few products; host-side constants (1 - b1, lr / bc1, rsqrtf(bc2), ...) are themselves rounded.  With K = 8,
      |out - R| <= K u24 (sum of the absolute values of the terms, each error propagated to first order),
  e.g. AdamW: m' = b1 m + (1 - b1) g, v' = b2 v + (1 - b2) g^2, p' = p decay - step m' / (sqrt(v') rs + eps) gets
      K u24 (|p decay| + 2 |upd|) + step / den  K u24 (|b1 m| + |(1 - b1) g|)
  (the second term because m' may cancel).  bf16 shadows are not bounded but compared bit for bit with bf16_rn of the
  fp32 value the kernel wrote (the test does that with torch's round-to-nearest-even cast).
  sumsq: every thread adds 8 squares per pass, `passes` = ceil(n / 8 / (grid 256)) times, then 5 + 3 shuffle steps
  and the fixed-order sum of the per-CTA partials:  |ss - R| <= u24 (8 passes + 16) R  (+ u24 |prior| when accumulating).

Where a measured worst ratio is quoted (DESIGN.md section 5) it was measured, not used to set the bound.
"""
from __future__ import annotations

import math

import numpy as np
import torch

C = 4.0
K = 8.0
U8, U24 = 2.0 ** -8, 2.0 ** -24
TINY = 2.0 ** -133          # bf16 outputs may be subnormal: an absolute floor far below any value of interest
BF16 = torch.bfloat16

WORST = {}


def rnd(ref, dtype):
    """Allowance for the one rounding to the storage type."""
    return (U8 if dtype == BF16 else U24) * ref.abs() + (TINY if dtype == BF16 else 0.0)


def f32(v):
    """The value a C float argument takes."""
    return float(np.float32(v))


def check(got, ref, bound, what, family=None):
    """Asserts |got - ref| <= bound for every element; returns (and records under `family`) the worst ratio."""
    assert tuple(got.shape) == tuple(ref.shape), f"{what}: shape {tuple(got.shape)} vs {tuple(ref.shape)}"
    g = got.detach().double()
    assert bool(torch.isfinite(g).all()), f"{what}: non-finite output"
    err = (g - ref.to(g.device)).abs()
    b = bound.to(g.device).expand_as(err) if torch.is_tensor(bound) else torch.full_like(err, float(bound))
    exact = torch.where(err == 0, torch.zeros_like(err), torch.full_like(err, float("inf")))
    r = torch.where(b > 0, err / b.clamp_min(1e-300), exact)
    worst = float(r.max()) if r.numel() else 0.0
    if family is not None:
        WORST[family] = max(WORST.get(family, 0.0), worst)
    if worst > 1:
        idx = np.unravel_index(int(r.argmax()), r.shape)
        idx = tuple(int(i) for i in idx)
        raise AssertionError(f"{what}: element {idx} got {float(g[idx]):.9e} ref {float(ref[idx]):.9e} "
                             f"bound {float(b[idx]):.3e} ratio {worst:.3g}")
    return worst


def check_all(got: dict, ref: dict, what, family=None):
    """check() for every name in `got` against ref[name] = (ref64, bound)."""
    return max(check(g, *ref[name], f"{what} {name}", None if family is None else f"{family}.{name}")
               for name, g in got.items())


# ----------------------------------------------------------------------------------------------------------------
# guard buffers
# ----------------------------------------------------------------------------------------------------------------
GUARD_BYTE = 0x7B           # bf16 0x7B7B = 1.3e36, fp32 0x7B7B7B7B = 1.3e36, int32 / int64 large positive: never NaN
GUARD_BYTES = 256           # on each side; a multiple of 16, so the payload keeps the allocation's alignment


class Guarded:
    """`numel` elements of `dtype` inside a larger allocation whose every byte is GUARD_BYTE.  `.t` is the payload
    view (16-byte aligned, still holding the sentinel pattern until written); `.intact()` tells whether the bytes on
    both sides still hold the pattern."""

    def __init__(self, shape, dtype, device="cpu"):
        shape = (shape,) if isinstance(shape, int) else tuple(shape)
        n = math.prod(shape)
        item = torch.empty(0, dtype=dtype).element_size()
        self.nbytes = n * item
        tail = GUARD_BYTES + (-self.nbytes) % item      # keep the raw length a whole number of elements
        self.raw = torch.full((GUARD_BYTES + self.nbytes + tail,), GUARD_BYTE, dtype=torch.uint8, device=device)
        self.t = self.raw[GUARD_BYTES:GUARD_BYTES + self.nbytes].view(dtype).view(shape)
        assert self.t.data_ptr() % 16 == 0

    def fill(self, src):
        self.t.copy_(src.reshape(self.t.shape))
        return self

    def intact(self):
        head = self.raw[:GUARD_BYTES]
        tail = self.raw[GUARD_BYTES + self.nbytes:]
        return bool((head == GUARD_BYTE).all()) and bool((tail == GUARD_BYTE).all())

    def untouched(self):
        """The payload still holds the sentinel pattern (nothing was written)."""
        return bool((self.raw == GUARD_BYTE).all())


# ----------------------------------------------------------------------------------------------------------------
# RMSNorm
# ----------------------------------------------------------------------------------------------------------------
def rmsnorm_fwd(x, w, eps, delta=None):
    """x, delta [R, H], w [H] of dtype T.  -> {"sum" (only with delta), "rstd", "y"}."""
    T, H = x.dtype, x.shape[-1]
    out = {}
    s = x
    if delta is not None:
        s = (x.float() + delta.float()).to(T)
        out["sum"] = (s.double(), torch.zeros((), dtype=torch.float64, device=x.device))
    sd = s.double()
    rstd = 1.0 / torch.sqrt((sd * sd).mean(-1) + f32(eps))
    y = sd * rstd[:, None] * w.double()
    out["rstd"] = (rstd, C * U24 * (H + 2) * rstd)
    out["y"] = (y, C * U24 * (H + 4) * y.abs() + (rnd(y, T) if T == BF16 else 0.0))
    return out


def rmsnorm_bwd(dy, x, w, rstd, dres=None, rows_per_chunk=None):
    """dy, x, dres [R, H] and w [H] of dtype T; rstd fp32 [R] as the forward kernel wrote it.  -> {"dx", "dw"}
    (dw: the fp32 column sum before any accumulation)."""
    T, (R, H) = x.dtype, x.shape
    xd, dyd, r = x.double(), dy.double(), rstd.double()[:, None]
    g = dyd * w.double()
    c = r * r * (g * xd).mean(-1, keepdim=True)
    ca = r * r * (g * xd).abs().mean(-1, keepdim=True)
    dx = r * (g - xd * c)
    bdx = C * U24 * H * r * (g.abs() + xd.abs() * ca)
    if dres is not None:
        dx = dx + dres.double()
        bdx = bdx + C * U24 * dres.double().abs()
    t = dyd * xd * r
    return {"dx": (dx, bdx + rnd(dx, T)), "dw": (t.sum(0), C * U24 * R * t.abs().sum(0))}


def colsum(partials, prior=None, out_dtype=torch.float32):
    """b200_rmsnorm_dw_reduce on partials fp32 [P, H]: column sums, optionally accumulated into `prior` of
    out_dtype.  -> {"dw"}."""
    p = partials.double()
    ref, bound = p.sum(0), C * U24 * p.shape[0] * p.abs().sum(0)
    if prior is not None:
        ref = ref + prior.double()
        bound = bound + C * U24 * prior.double().abs()
    if prior is not None or out_dtype == BF16:
        bound = bound + rnd(ref, out_dtype)
    return {"dw": (ref, bound)}


def accumulated(ref_bound, prior, out_dtype):
    """(ref, bound) of a fp32 sum after being added into the stored gradient `prior` of out_dtype."""
    ref, bound = ref_bound
    ref = ref + prior.double()
    return ref, bound + C * U24 * prior.double().abs() + rnd(ref, out_dtype)


# ----------------------------------------------------------------------------------------------------------------
# RoPE
# ----------------------------------------------------------------------------------------------------------------
def rope(x, cos_t, sin_t, pos=None, layout="interleaved", backward=False):
    """x [B, S, NH, D] of dtype T; cos_t / sin_t fp32 [rows, D/2]; pos None or integer [B, S].  -> {"y"}."""
    B, S, NH, D = x.shape
    idx = torch.arange(S, device=x.device).expand(B, S) if pos is None else pos.long()
    c = cos_t.double()[idx][:, :, None, :]                     # [B, S, 1, D/2]
    s = sin_t.double()[idx][:, :, None, :] * (-1.0 if backward else 1.0)
    xd = x.double()
    if layout == "interleaved":
        a, b = xd[..., 0::2], xd[..., 1::2]
    else:
        a, b = xd[..., :D // 2], xd[..., D // 2:]
    oa, ob = a * c - b * s, a * s + b * c
    ba, bb = (a * c).abs() + (b * s).abs(), (a * s).abs() + (b * c).abs()
    if layout == "interleaved":
        y, m = torch.stack([oa, ob], -1).flatten(-2), torch.stack([ba, bb], -1).flatten(-2)
    else:
        y, m = torch.cat([oa, ob], -1), torch.cat([ba, bb], -1)
    return {"y": (y, C * U24 * m + rnd(y, x.dtype))}


# ----------------------------------------------------------------------------------------------------------------
# GLU
# ----------------------------------------------------------------------------------------------------------------
def expf_rel(x):
    """Relative error bound of __expf(x): 2 + floor(|1.173 x|) ulp (CUDA programming guide)."""
    return 2.0 * U24 * (2.0 + 1.173 * x.abs())


def _sig(x):
    s = torch.sigmoid(x)
    one_minus = torch.sigmoid(-x)                               # accurate where 1 - s cancels
    ds = s * (one_minus * expf_rel(x) + C * U24)
    return s, one_minus, ds


def _prod(factors, errs, dtype):
    """Reference and bound of a product of factors with absolute errors errs."""
    ref = torch.ones_like(factors[0])
    for f in factors:
        ref = ref * f
    bound = C * U24 * ref.abs() + rnd(ref, dtype)
    for i, e in enumerate(errs):
        if e is None:
            continue
        t = e
        for j, f in enumerate(factors):
            if j != i:
                t = t * f.abs()
        bound = bound + t
    return ref, bound


def glu_fwd(g, u, act="sigmoid2"):
    """g, u bf16 (any shape).  -> {"y"}."""
    gd, ud = g.double(), u.double()
    if act == "sigmoid2":
        s, _, ds = _sig(ud)
        return {"y": _prod([2 * gd, s], [None, ds], g.dtype)}
    s, _, ds = _sig(gd)
    return {"y": _prod([gd, s, ud], [None, ds, None], g.dtype)}


def glu_bwd(dy, g, u, act="sigmoid2"):
    """-> {"dg", "du"}."""
    dd, gd, ud = dy.double(), g.double(), u.double()
    if act == "sigmoid2":
        s, om, ds = _sig(ud)
        return {"dg": _prod([2 * dd, s], [None, ds], g.dtype),
                "du": _prod([2 * dd * gd, s, om], [None, ds, ds + U24], g.dtype)}
    s, om, ds = _sig(gd)
    f = 1.0 + gd * om
    df = gd.abs() * (ds + U24) + U24 * (1.0 + (gd * om).abs())
    return {"dg": _prod([dd * ud, s, f], [None, ds, df], g.dtype),
            "du": _prod([dd * gd, s], [None, ds], g.dtype)}


# ----------------------------------------------------------------------------------------------------------------
# cross entropy
# ----------------------------------------------------------------------------------------------------------------
def ce_fwd(logits, targets, V, pad):
    """logits bf16 [R, ld] (columns >= V hold anything), targets int64 [R].  -> {"lse", "loss"}."""
    x = logits[:, :V].double()
    lse = torch.logsumexp(x, -1)
    bound = C * U24 * (V / 512.0 + 16.0 + x.abs().amax(-1))
    live = targets != pad
    xt = x.gather(1, targets.clamp(0, V - 1)[:, None])[:, 0]
    loss = torch.where(live, lse - xt, torch.zeros_like(lse))
    return {"lse": (lse, bound), "loss": (loss, torch.where(live, bound, torch.zeros_like(bound)))}


def ce_bwd(logits, targets, V, pad, lse, row_scale):
    """The in-place backward over the whole [R, ld] buffer, given the forward kernel's fp32 lse.  -> {"dlogits"}."""
    R, ld = logits.shape
    x = logits[:, :V].double()
    z = x - lse.double()[:, None]
    p = torch.exp(z)
    live = (targets != pad)[:, None]
    sc = torch.where(live, row_scale.double()[:, None], torch.zeros_like(p[:, :1]))
    onehot = torch.zeros_like(p)
    onehot.scatter_(1, targets.clamp(0, V - 1)[:, None], 1.0)
    onehot = onehot * ((targets >= 0) & (targets < V))[:, None]
    d = sc * (p - onehot)
    b = U8 * d.abs() + C * U24 * (2.0 + z.abs()) * sc.abs() * p + TINY * (sc != 0)
    ref = torch.zeros(R, ld, dtype=torch.float64, device=logits.device)
    bound = torch.zeros_like(ref)
    ref[:, :V], bound[:, :V] = d, b
    return {"dlogits": (ref, bound)}


# ----------------------------------------------------------------------------------------------------------------
# embedding scatter
# ----------------------------------------------------------------------------------------------------------------
def embedding_bwd(dh, tokens, prior, V):
    """dh bf16 [rows, H], tokens int64 [rows] (entries outside [0, V) are skipped), prior [V, H] of the gradient's
    dtype.  -> {"grad"}."""
    ok = (tokens >= 0) & (tokens < V)
    tk, d = tokens[ok], dh[ok].double()
    add = torch.zeros_like(prior, dtype=torch.float64).index_add_(0, tk, d)
    mag = torch.zeros_like(add).index_add_(0, tk, d.abs())
    hits = torch.zeros(V, dtype=torch.float64, device=dh.device).index_add_(0, tk, torch.ones_like(tk, dtype=torch.float64))
    ref = prior.double() + add
    hit = (hits > 0)[:, None]
    bound = U24 * hits[:, None] * mag + hit * (U24 * prior.double().abs() + rnd(ref, prior.dtype))
    return {"grad": (ref, bound)}


# ----------------------------------------------------------------------------------------------------------------
# optimizer updates (flat ranges)
# ----------------------------------------------------------------------------------------------------------------
def _adam_core(g, m, v, lr, b1, b2, eps, bc1, bc2, gscale):
    gj = g.double() * f32(gscale)
    b1, b2 = f32(b1), f32(b2)
    t1, t2 = b1 * m.double(), (1.0 - b1) * gj
    m2 = t1 + t2
    bm = K * U24 * (t1.abs() + t2.abs())
    v2 = b2 * v.double() + (1.0 - b2) * gj * gj
    bv = K * U24 * v2.abs()
    step = f32(lr) / f32(bc1)
    den = torch.sqrt(v2.clamp_min(0)) / math.sqrt(f32(bc2)) + f32(eps)
    upd = step * m2 / den
    bu = 2 * K * U24 * upd.abs() + abs(step) / den * bm
    return m2, bm, v2, bv, upd, bu


def adamw(p, g, m, v, lr, b1, b2, eps, wd, bc1=1.0, bc2=1.0, gscale=1.0):
    """-> {"p", "m", "v"}"""
    m2, bm, v2, bv, upd, bu = _adam_core(g, m, v, lr, b1, b2, eps, bc1, bc2, gscale)
    pd = p.double() * (1.0 - f32(lr) * f32(wd))
    return {"p": (pd - upd, K * U24 * pd.abs() + bu), "m": (m2, bm), "v": (v2, bv)}


def adam_direction(g, m, v, lr, b1, b2, eps, bc1=1.0, bc2=1.0, gscale=1.0):
    """-> {"d", "m", "v"}"""
    m2, bm, v2, bv, upd, bu = _adam_core(g, m, v, lr, b1, b2, eps, bc1, bc2, gscale)
    return {"d": (-upd, bu), "m": (m2, bm), "v": (v2, bv)}


def _momentum(g, buf, mu, nesterov, gscale):
    gj = g.double() * f32(gscale)
    mu = f32(mu)
    t1, t2 = (1.0 - mu) * gj, mu * buf.double()
    b2 = t1 + t2
    ab = t1.abs() + t2.abs()
    if nesterov:
        return b2, ab, gj + mu * b2, gj.abs() + abs(mu) * ab
    return b2, ab, b2, ab


def sgd_momentum(p, g, buf, mu, nesterov, lr, gscale=1.0):
    """-> {"p", "buf"}"""
    b2, ab, u, au = _momentum(g, buf, mu, nesterov, gscale)
    return {"p": (p.double() - f32(lr) * u, K * U24 * (p.double().abs() + abs(f32(lr)) * au)),
            "buf": (b2, K * U24 * ab)}


def muon_momentum(g, buf, mu, nesterov, gscale, passes):
    """g, buf [batch, numel].  -> {"buf", "u" (bf16), "sumsq" [batch] of the unrounded u}."""
    b2, ab, u, au = _momentum(g, buf, mu, nesterov, gscale)
    du = K * U24 * au
    ss = (u * u).sum(-1)
    return {"buf": (b2, K * U24 * ab), "u": (u, du + rnd(u, BF16)),
            "sumsq": (ss, U24 * (8 * passes + 16) * ss + (2 * u.abs() * du).sum(-1))}


def axpy_update(p, x, s):
    """-> {"p"}"""
    t = f32(s) * x.double()
    return {"p": (p.double() + t, K * U24 * (p.double().abs() + t.abs()))}


def clip_accum(g, acc, clip, scale, init):
    """-> {"acc"}"""
    x = g.double()
    if clip > 0:
        x = x.clamp(-f32(clip), f32(clip))
    t = x * f32(scale)
    a = torch.zeros_like(t) if init else acc.double()
    return {"acc": (a + t, K * U24 * (a.abs() + t.abs()))}


def sumsq(x, passes, prior=None):
    """x [batch, numel]; prior fp32 [batch] when accumulating.  -> {"ss"}"""
    ss = (x.double() ** 2).sum(-1)
    bound = U24 * (8 * passes + 16) * ss
    if prior is not None:
        ss = ss + prior.double()
        bound = bound + K * U24 * ss.abs()
    return {"ss": (ss, bound)}


def ns_scales(ss, eps):
    """-> {"inv", "inv2"}"""
    inv = 1.0 / (torch.sqrt(ss.double()) + f32(eps))
    return {"inv": (inv, C * U24 * inv), "inv2": (inv * inv, 2 * C * U24 * inv * inv)}


def _split(x, ax):
    """hi = bf16(x), lo = bf16(x - hi): hi within one bf16 rounding of x, hi + lo within 2^-16 |x|."""
    return {"hi": (x, ax + rnd(x, BF16)), "hi+lo": (x, ax + U8 * U8 * x.abs() + TINY)}


def split_bf16(src, rows, cols, scale=1.0, diag_add=0.0):
    """src fp32 [>= rows, >= cols] (a strided view is fine).  -> {"hi", "hi+lo"} for the [rows, cols] block."""
    s = src[:rows, :cols].double()
    eye = torch.eye(rows, cols, dtype=torch.float64, device=src.device) * f32(diag_add)
    x = (s + eye) * f32(scale)
    return _split(x, K * U24 * (s.abs() + eye.abs()) * abs(f32(scale)))


def ema_split(g, m, beta, gscale, inv_bc, out_scale):
    """-> {"m", "out32", "hi", "hi+lo"}"""
    beta = f32(beta)
    t1, t2 = beta * m.double(), (1.0 - beta) * g.double() * f32(gscale)
    m2 = t1 + t2
    am = K * U24 * (t1.abs() + t2.abs())
    mh = m2 * f32(inv_bc)
    amh = (am + U24 * m2.abs()) * abs(f32(inv_bc))
    out = {"m": (m2, am), "out32": (mh * f32(out_scale), (amh + U24 * mh.abs()) * abs(f32(out_scale)))}
    out.update(_split(mh, amh))
    return out


def graft_update(p, pre, d, coef, coef_d, decay):
    """p, pre, d [batch, numel]; coef, coef_d fp32 [batch].  A zero coefficient drops its term whatever it holds.
    -> {"p"}"""
    c, cd = coef.double()[:, None], coef_d.double()[:, None]
    t0 = p.double() * f32(decay)
    t1 = torch.where(c != 0, c * pre.double(), torch.zeros_like(t0))
    t2 = torch.where(cd != 0, cd * d.double(), torch.zeros_like(t0))
    return {"p": (t0 + t1 + t2, K * U24 * (t0.abs() + t1.abs() + t2.abs()))}
