"""fp64 references with per-element bounds for the sparse MoE MLP's own kernels (csrc/moe.cu): the routing
(b200_moe_route), the combine (b200_moe_combine_fwd), its backward with the router adjoint (b200_moe_combine_bwd),
the un-permutation (b200_moe_unpermute), the router's three fp32 GEMMs (ops._MoeFn) and the expert-segmented GEMMs
(b200_moe_gemm, b200_moe_wgrad).  Pure torch, works on any device, does not import the package.
tests/test_moe_check.py shows on the CPU what the checker accepts and rejects; tests/test_gpu_moe_stages.py and
tests/test_gpu_moe.py feed it kernel outputs.

Each stage is checked on the kernel's own inputs (the probs the routing wrote, the dw the backward wrote, ...), so
an upstream error is not counted twice.  Notation as in tests/rowwise_check.py: u24 = 2^-24, u8 = 2^-8, TINY = 2^-133
(a floor for bf16 outputs); in addition S32 = 2^-149, the smallest fp32 subnormal.  The build has no fast-math flag,
so `expf` is libdevice's (<= 2 ulp, i.e. relative 4 u24) and `/` is IEEE; `-O3` may contract `a += w * f` into an
FMA, and every bound below counts a product and an add as two roundings, so it holds either way.

probs (route_topk_kernel).  d = v - m is one rounding of the exact difference (m, the max, is exact): a relative
  error u24 |d| of exp(d).  With expf's 4 u24, e_i is within (|d_i| + 4) u24 relative.  The warp sum s adds the
  lane's two terms and then 5 shuffle levels: every e_i passes 6 adds of non-negative terms, so s is within
  (sum_i p_i (|d_i| + 4) + 6) u24 relative; the division adds one more:
      |p_e - R| <= u24 R (|d_e| + sum_i p_i |d_i| + 16) + 4 S32
  (the floor: a subnormal expf result is within 2 of its ulps, the division at s >= 1 half of one more).
ids.  Exactly the top k of the kernel's own fp32 probs, larger first and the lower index on an exact tie: the warp
  argmax with candidates -1 for taken experts, so experts whose p underflowed to 0 still rank (lower index first)
  when k exceeds the non-zero count.  On a row whose k + 1 largest fp64 probabilities are separated by more than the
  sum of their two probs bounds the ids are also the fp64 top k.
weights.  sel_j / tot, tot = sum_j sel_j in k - 1 adds, on the kernel's probs: |w - R| <= (k + 2) u24 R + S32.
counts, seg_off, tiles, n_tiles, dest (route_hist / route_scan / route_dest).  Exact: the stable counting sort of
  tests/moe_oracle.py's emulate_routing (`index_ref` is its vectorised form; tests/test_moe_check.py asserts they
  agree).  aux_counts: the assignments of unmasked tokens per expert, exact.
aux_psum.  Per chunk of 64 tokens a sequential fp32 sum of p_e over the unmasked tokens, then a sequential sum over
  the nch chunks: |psum - R| <= (64 + nch) u24 R, exactly 0 when no token is unmasked.
combine forward (combine_kernel with weights).  acc += w_j y_j over j ascending, then one bf16 rounding:
      |out - R| <= u8 |R| + (2 k + 1) u24 sum_j |w_j y_j| + TINY.
combine backward (combine_bwd_kernel).
  dyp:  bf16(fp32(w_j dout)) bit for bit: one IEEE product (nothing to contract), one round to nearest even, which
        torch's fp32 multiply and bf16 cast reproduce.  Every pad row of every segment is +0.0 bit for bit, and rows
        from seg_off[E] on are not written.
  dw:   thread-local sums of 8 products per vector, ceil(H / 1024) vectors per thread, 5 shuffle levels, 3 adds of the
        warp partials: each term meets at most 16 + ceil(H / 1024) roundings,
            |dw - R| <= (16 + ceil(H / 1024)) u24 sum_i |dout_i y_i|.
  dlogits, given the kernel's dw, p, w, ids, aux_grad and mask:
        c = sum_j dw_j w_j,  S = sum_j p_{e_j},  dp_e = aux_grad_e [mask_t] + (dw_j - c) / S  (e = e_j),
        q = sum_f p_f dp_f,  dlogits_e = p_e (dp_e - q).
        dw_j - c cancels, so the magnitudes are  A_e = |aux_grad_e [mask_t]| + (|dw_j| + sum_i |dw_i w_i|) / S and
        Q = sum_f p_f A_f.  c takes 2k roundings of sum |dw_i w_i|, the difference, S (k - 1 adds) and the division
        k + 1 of A_e, the add into dp one: dp_e is within kappa u24 A_e, kappa = 3 k + 3.  q adds 2E roundings of Q,
        and the difference and the product two more:
            |dlogits_e - R| <= u24 p_e ((kappa + 2) A_e + (kappa + 2 E + 2) Q) + (E + 2) S32 [p_e > 0].
        Exactly 0 where p_e = 0, and +0.0 bit for bit for k = 1 without aux_grad (w = sel / sel = 1, so
        dw - c = 0 exactly).
un-permutation (combine_kernel without weights).  acc += 1.f * y_j is exact as a product or an FMA, so the kernel
  computes the fp32 sum of the k bf16 rows, j ascending, then + addend, then one round to nearest even: bit for bit.
router GEMMs (torch fp32 matmuls): logits = x Wr^T, addend = dlogits Wr, dWr = dlogits^T x.  Any order of a K-term
  fp32 dot product is within K u24 of its absolute terms:  |c - R| <= K u24 (|A| |B|)  (+ u8 |R| + TINY when the
  result is stored as bf16).  TF32 (10-bit products) would break it by orders of magnitude.
expert-segmented GEMMs (`gemm_ratio`, `seg_gemm`).  Inputs are bf16 and the fp64 reference is computed from the same
  bf16 values, so the kernel's only errors are (a) its fp32 accumulation over K terms, at most K 2^-24 (|A| |B|) to
  first order, <= 2^-10 mag for K <= 2^14, where mag is the same product evaluated on absolute values, and (b) the
  final rounding to bf16, at most 2^-9 |c|.  An activation epilogue computed from the fp32 accumulators multiplies
  (a) by the activation's partial derivatives (|d act / d g|, |d act / d u|) and adds its own fp32 evaluation error
  (a few 2^-24 relative, absorbed in the 2^-9 term).  The checker allows twice each term:
      |got - ref| <= 2^-8 |ref| + 2^-9 mag_eff + 2^-133,
  with mag_eff = mag for plain outputs and the derivative-weighted mags for activation outputs.  A ratio above 1
  names the element.

Where a measured worst ratio is quoted (DESIGN.md section 5) it was measured, not used to set the bound.
"""
from __future__ import annotations

import math

import numpy as np
import torch

from tests import moe_oracle as mo
from tests.rowwise_check import TINY, U8, U24, check

CHUNK = 64
SEG = mo.SEG
S32 = 2.0 ** -149
BF16 = torch.bfloat16


def _where(t: torch.Tensor):
    idx = torch.nonzero(t)[0]
    return tuple(int(i) for i in idx)


def exact(got, want, what, names=("token", "slot")):
    """Asserts got == want element for element (integer tensors, or floats compared by value); names the first
    differing element."""
    got = torch.as_tensor(got).to(want.device)
    assert tuple(got.shape) == tuple(want.shape), f"{what}: shape {tuple(got.shape)} vs {tuple(want.shape)}"
    bad = got != want
    if bool(bad.any()):
        idx = _where(bad)
        lab = ", ".join(f"{n} {i}" for n, i in zip(names, idx))
        raise AssertionError(f"{what}: {lab}: got {got[idx].item()} want {want[idx].item()} "
                             f"({int(bad.sum())} elements differ)")


def bitwise(got, want, what, names=("row", "element")):
    """Asserts got and want (same floating dtype) have the same bits."""
    assert got.dtype == want.dtype, f"{what}: dtype {got.dtype} vs {want.dtype}"
    iv = {2: torch.int16, 4: torch.int32}[got.element_size()]
    exact(got.contiguous().view(iv), want.to(got.device).contiguous().view(iv), what, names)


# ---- routing -----------------------------------------------------------------------------------------------------
def probs(logits):
    """logits fp32 [T, E] -> (ref, bound) of the kernel's fp32 softmax."""
    v = logits.double()
    d = v - v.amax(-1, keepdim=True)
    p = torch.softmax(v, -1)
    spread = (p * d.abs()).sum(-1, keepdim=True)
    return p, U24 * p * (d.abs() + spread + 16.0) + 4 * S32


def topk_ids(p, k):
    """ids [T, k] (int64): the top k of p [T, E], larger first, the lower index on an exact tie."""
    return torch.sort(-p, dim=-1, stable=True).indices[:, :k]


def clear_rows(p64, bound, k):
    """bool [T]: rows whose k + 1 largest fp64 probabilities are pairwise separated beyond their bounds."""
    T, E = p64.shape
    ps, order = torch.sort(-p64, dim=-1, stable=True)
    ps, bs = -ps, bound.gather(-1, order)
    n = min(k, E - 1)
    if n == 0:
        return torch.ones(T, dtype=torch.bool, device=p64.device)
    return ((ps[:, :n] - ps[:, 1:n + 1]) > (bs[:, :n] + bs[:, 1:n + 1])).all(-1)


def weights(p, ids):
    """p: the kernel's fp32 probs.  -> (ref, bound) of the renormalised top-k weights."""
    top = p.double().gather(-1, ids.long())
    w = top / top.sum(-1, keepdim=True)
    return w, (ids.shape[1] + 2) * U24 * w + S32


def index_ref(ids, E):
    """Vectorised emulate_routing: (counts [E], seg_off [E + 1], tiles [n_tiles], dest [T, k]), int64."""
    T, k = ids.shape
    flat = ids.reshape(-1).long()
    oh = torch.nn.functional.one_hot(flat, E)
    counts = oh.sum(0)
    padded = (counts + SEG - 1) // SEG * SEG
    seg_off = torch.cat([torch.zeros(1, dtype=torch.long, device=ids.device), torch.cumsum(padded, 0)])
    rank = (oh.cumsum(0) - 1).gather(1, flat[:, None])[:, 0]     # stable: assignments before this one, same expert
    dest = (seg_off[flat] + rank).view(T, k)
    tiles = torch.repeat_interleave(torch.arange(E, device=ids.device), padded // SEG)
    return counts, seg_off, tiles, dest


def aux_ref(p, ids, mask, E):
    """(aux_counts exact, (psum ref, bound)) over the unmasked tokens, from the kernel's probs."""
    T = p.shape[0]
    m = torch.ones(T, dtype=torch.float64, device=p.device) if mask is None else mask.double().to(p.device)
    cnt = (torch.nn.functional.one_hot(ids.long(), E).double().sum(1) * m[:, None]).sum(0)
    ps = (p.double() * m[:, None]).sum(0)
    nch = (T + CHUNK - 1) // CHUNK
    return cnt, (ps, (CHUNK + nch) * U24 * ps)


def check_route(logits, k, mask, out: dict, what, family="route"):
    """out: the kernel's ids, weights, probs, counts, seg_off, tile_expert, n_tiles, dest and, when given,
    aux_counts / aux_psum.  Checks every stage on the kernel's own upstream values; returns the worst ratio."""
    T, E = logits.shape
    p_ref, p_bound = probs(logits)
    worst = check(out["probs"], p_ref, p_bound, f"{what} probs (token, expert)", f"{family}.probs")
    p = out["probs"].to(logits.device)
    ids = out["ids"].long().to(logits.device)
    exact(ids, topk_ids(p, k), f"{what} ids vs the top-k of the kernel's probs")
    clear = clear_rows(p_ref, p_bound, k)
    id64 = topk_ids(p_ref, k)
    bad = clear[:, None] & (ids != id64)
    if bool(bad.any()):
        t, j = _where(bad)
        raise AssertionError(f"{what} ids vs the fp64 top-k: token {t} slot {j}: {ids[t].tolist()} vs "
                             f"{id64[t].tolist()} on a row whose gaps exceed the probs bound")
    worst = max(worst, check(out["weights"], *weights(p, ids), f"{what} weights (token, slot)",
                             f"{family}.weights"))
    counts, seg_off, tiles, dest = index_ref(ids, E)
    exact(out["counts"].long(), counts, f"{what} counts", ("expert",))
    exact(out["seg_off"].long(), seg_off, f"{what} seg_off", ("expert",))
    n = int(seg_off[-1]) // SEG
    exact(out["n_tiles"].long().reshape(-1)[:1], torch.tensor([n], device=seg_off.device), f"{what} n_tiles", ("",))
    exact(out["tile_expert"].long()[:n], tiles, f"{what} tile_expert", ("tile",))
    exact(out["dest"].long(), dest, f"{what} dest")
    if out.get("aux_counts") is not None:
        cnt, psum = aux_ref(p, ids, mask, E)
        exact(out["aux_counts"].double(), cnt, f"{what} aux_counts", ("expert",))
        worst = max(worst, check(out["aux_psum"], *psum, f"{what} aux_psum (expert)", f"{family}.aux_psum"))
    return worst


# ---- combine, its backward and the un-permutation ------------------------------------------------------------
def combine_fwd(yp, dest, w):
    """-> (ref, bound) of out [T, H] = sum_j w_j yp[dest[t, j]] rounded to bf16."""
    k = dest.shape[1]
    ref = torch.zeros(dest.shape[0], yp.shape[1], dtype=torch.float64, device=yp.device)
    mag = torch.zeros_like(ref)
    for j in range(k):
        t = w[:, j, None].double() * yp[dest[:, j].long()].double()
        ref, mag = ref + t, mag + t.abs()
    return ref, U8 * ref.abs() + (2 * k + 1) * U24 * mag + TINY


def dyp_ref(dout, dest, w, seg_off, before):
    """The dyp buffer the backward must leave, given its contents `before` the launch: bf16(fp32(w_j dout)) at every
    destination, +0.0 in every pad row of every segment, `before` from seg_off[E] on.  before = None: only the rows
    up to seg_off[E]."""
    end = int(seg_off[-1])
    want = torch.zeros(end, dout.shape[1], dtype=BF16, device=dout.device) if before is None else before.clone()
    want[:end] = 0
    for j in range(dest.shape[1]):
        want[dest[:, j].long()] = (w[:, j, None].float() * dout.float()).to(BF16)
    return want


def combine_dw(dout, yp, dest):
    """-> (ref, bound) of dw [T, k] = <dout[t], yp[dest[t, j]]>."""
    H = dout.shape[1]
    d = dout.double()
    ref, mag = [], []
    for j in range(dest.shape[1]):
        y = yp[dest[:, j].long()].double()
        ref.append((d * y).sum(-1))
        mag.append((d * y).abs().sum(-1))
    depth = 16 + math.ceil(H / 1024)
    return torch.stack(ref, 1), depth * U24 * torch.stack(mag, 1)


def router_adjoint(dw, p, w, ids, aux_grad, mask):
    """dw, w [T, k] and p [T, E]: the kernel's values; aux_grad [E] or None; mask [T] or None.
    -> (ref, bound) of dlogits [T, E]."""
    T, E = p.shape
    k = ids.shape[1]
    dw, p, w, ids = dw.double(), p.double(), w.double(), ids.long()
    m = torch.zeros(T, E, dtype=torch.float64, device=p.device)
    if aux_grad is not None:
        on = torch.ones(T, dtype=torch.float64, device=p.device) if mask is None else (mask != 0).double()
        m = on[:, None] * aux_grad.double()[None, :]
    c = (dw * w).sum(-1, keepdim=True)
    ac = (dw * w).abs().sum(-1, keepdim=True)
    S = p.gather(1, ids).sum(-1, keepdim=True)
    dp = m.clone().scatter_add_(1, ids, (dw - c) / S)
    A = m.abs().scatter_add_(1, ids, (dw.abs() + ac) / S)
    q = (p * dp).sum(-1, keepdim=True)
    Q = (p * A).sum(-1, keepdim=True)
    kappa = 3 * k + 3
    ref = p * (dp - q)
    bound = U24 * p * ((kappa + 2) * A + (kappa + 2 * E + 2) * Q) + (E + 2) * S32 * (p > 0)
    return ref, bound


def unpermute_ref(dxp, dest, addend):
    """The kernel's dx bit for bit: fp32 sum of the k bf16 rows, j ascending, + addend, one bf16 rounding."""
    acc = torch.zeros(dest.shape[0], dxp.shape[1], dtype=torch.float32, device=dxp.device)
    for j in range(dest.shape[1]):
        acc = acc + dxp[dest[:, j].long()].float()
    if addend is not None:
        acc = acc + addend.float()
    return acc.to(BF16)


def check_combine_bwd(dout, yp, dest, ids, w, p, aux_grad, mask, seg_off, before, dyp, dw, dlogits, what,
                      family="combine_bwd"):
    """Checks the three outputs of b200_moe_combine_bwd (dw / dlogits may be None: not written) on the kernel's
    inputs; dlogits against the kernel's own dw.  before: dyp's contents before the launch, or None to check only
    the rows up to seg_off[E].  Returns the worst ratio."""
    want = dyp_ref(dout, dest, w, seg_off, before)
    bitwise(dyp[:want.shape[0]], want, f"{what} dyp")
    worst = 0.0
    if dw is not None:
        worst = check(dw, *combine_dw(dout, yp, dest), f"{what} dw (token, slot)", f"{family}.dw")
    if dlogits is not None:
        assert dw is not None, "dlogits is checked against the kernel's dw"
        if ids.shape[1] == 1 and aux_grad is None:
            bitwise(dlogits, torch.zeros_like(dlogits), f"{what} dlogits (k = 1, no aux: +0.0)", ("token", "expert"))
        ref, bound = router_adjoint(dw, p, w, ids, aux_grad, mask)
        worst = max(worst, check(dlogits, ref, bound, f"{what} dlogits (token, expert)", f"{family}.dlogits"))
    return worst


# ---- router GEMMs ------------------------------------------------------------------------------------------------
def fp32_gemm(a, b, out_dtype=torch.float32):
    """-> (ref, bound) of a @ b computed by an fp32 matmul (any summation order), stored as out_dtype."""
    ad, bd = a.double(), b.double()
    ref = ad @ bd
    bound = a.shape[-1] * U24 * (ad.abs() @ bd.abs())
    if out_dtype == BF16:
        bound = bound + U8 * ref.abs() + TINY
    return ref, bound


# ---- expert-segmented GEMMs ----------------------------------------------------------------------------------------
def gemm_ratio(got, ref, mag, family, record=None):
    """The segmented-GEMM check: asserts |got - ref| <= 2^-8 |ref| + 2^-9 mag + 2^-133 and names the worst element;
    record(family, worst) is called first."""
    got, ref, mag = got.double().cpu(), ref.double().cpu(), mag.double().cpu()
    bound = 2.0 ** -8 * ref.abs() + 2.0 ** -9 * mag + 2.0 ** -133
    r = (got - ref).abs() / bound
    assert torch.isfinite(got).all(), f"{family}: non-finite output"
    worst = float(r.max()) if r.numel() else 0.0
    if record is not None:
        record(family, worst)
    if worst > 1:
        idx = np.unravel_index(int(r.argmax()), r.shape)
        raise AssertionError(f"{family}: element {tuple(int(i) for i in idx)} got {float(got[idx]):.6e} "
                             f"ref {float(ref[idx]):.6e} ratio {worst:.2f}")
    return worst


def _act_partials(g, u, act):
    """(act(g, u), d act / d g, d act / d u) in closed form."""
    if act == "silu":
        sg = torch.sigmoid(g)
        return g * sg * u, u * sg * (1 + g * (1 - sg)), g * sg
    su = torch.sigmoid(u)
    return 2 * g * su, 2 * su, 2 * g * su * (1 - su)


def seg_gemm(mode, act, a, w0, w1, gu, counts, seg_off):
    """fp64 references of one b200_moe_gemm call on its own operands, per expert over its real rows.
    -> {output name: (rows [n] int64, ref, mag)} with outputs "C" (all modes) and "Y" (gateup); for gateup and
    down_bwd C's two halves are separate entries "C.g" / "C.u" because their magnitudes differ."""
    E = w0.shape[0]
    out = {}

    def add(name, rows, ref, mag):
        r0, f0, m0 = out.get(name, ([], [], []))
        out[name] = (r0 + [rows], f0 + [ref], m0 + [mag])

    for e in range(E):
        n = int(counts[e])
        if n == 0:
            continue
        rows = torch.arange(int(seg_off[e]), int(seg_off[e]) + n, device=a.device)
        A = a[rows].double()
        if mode == "gateup":
            Wg, Wu = w0[e].double(), w1[e].double()
            g, u = A @ Wg.T, A @ Wu.T
            mg, mu = A.abs() @ Wg.abs().T, A.abs() @ Wu.abs().T
            y, dg, du = _act_partials(g, u, act)
            add("C.g", rows, g, mg)
            add("C.u", rows, u, mu)
            add("Y", rows, y, dg.abs() * mg + du.abs() * mu)
        elif mode == "down":
            W = w0[e].double()
            add("C", rows, A @ W.T, A.abs() @ W.abs().T)
        elif mode == "down_bwd":
            W = w0[e].double()
            I = W.shape[1]
            d, md = A @ W, A.abs() @ W.abs()
            gs, us = gu[rows, :I].double(), gu[rows, I:].double()
            _y, cg, cu = _act_partials(gs, us, act)
            add("C.g", rows, cg * d, cg.abs() * md)
            add("C.u", rows, cu * d, cu.abs() * md)
        else:   # gateup_dgrad
            Wg, Wu = w0[e].double(), w1[e].double()
            I = Wg.shape[0]
            add("C", rows, A[:, :I] @ Wg + A[:, I:] @ Wu, A[:, :I].abs() @ Wg.abs() + A[:, I:].abs() @ Wu.abs())
    return {n: (torch.cat(r), torch.cat(f), torch.cat(m)) for n, (r, f, m) in out.items()}
