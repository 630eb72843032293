"""fp64 reference and element-wise checker for the attention backward (b200_attn_bwd).

The backward is tested alone: O and LSE come from an fp64 forward and are rounded to bf16 / fp32, and the reference
uses that same O for delta = rowsum(dO * O).  The per-element bound has the form of tests/gemm_check.py:

  2^-8 * (|P| @ |dO|)  or  2^-8 * s * (|dS| @ |Q|), (|dS| @ |K|)   P^T / dS^T are rounded to bf16 before the MMAs
  C32 * 2^-24 * (D + n) * W                                         fp32 accumulation over n keys or queries and D;
                                                                   W uses |P| * (|dP| + |delta|) for dS, which covers
                                                                   the cancellation in dP - delta, and the logit
                                                                   magnitude s * (|q| @ |k|) that exp2 amplifies
  C32 * 2^-24 * D * |P| * (|dO| @ |V|^T + rowsum(|dO| * |O|))       the fp32 sums over D inside dP and delta: their
                                                                   error does not shrink when dP or delta cancels
                                                                   (a query that sees one key has dS = 0 exactly,
                                                                   the kernel the fp32 rounding of dP - delta)
  2^-8 * |R|                                                        bf16 output

ALiBi (b200_attn_bwd_alibi, `slopes`).  The kernel recomputes P^T = exp2(st * sl2 + (fmaf(ml2, -c, abase) - L2)) with
L2 = fl(LSE log2 e) from the pre-pass and abase = fl(ml2 (key - q0 - cq)) per item and key.  The bias's own roundings
are those of the forward (tests/attn_fwd_check.py): 2^-24 (5 |b| + 63 |m|) per logit in natural units (c <= 63 here),
so amp gains |b|, and 63 |m| sits inside C32 * (D + n) * 1 for |m| <= 2.  The bracket (b - L2) rounds once more,
by 2^-24 |b2 - L2|.  It needs no |LSE| term: |b2 - L2| = |x2 - s sl2| <= |log2 p| + sl2 |s|, where x2 = log2 p is
the exponent.  The sl2 |s| part is amp's.  The |log2 p| part is a relative error 2^-24 |log2 p| <= 2^-24 * 126 of p
(below 2^-126 exp2 flushes to 0, an error under 2^-126); 126 < C32 * (D + n) for every D >= 64, so the (D + n)
terms with amp >= 1 already hold it.  The plain kernel has the same |log2 p| from its own st * sl2 - L2.

bf16x3 (ops.attention_fp32's backward, `x3=True`).  _AttentionX3Fn runs the bf16 kernel on Q' = [qh|ql|qh],
K' = [kh|kh|kl], V' = [vh|vh|vl], dO' = [gh|gl|gh] and the saved O' = [bf16(P vh)|bf16(P vh)|bf16(P vl)], and sums
dq = dQ'[0:D] + dQ'[2D:3D] = dS (kh + kl), dk = dK'[0:D] + dK'[D:2D] = dS^T (qh + ql), dv = dV'[0:D] + dV'[D:2D] =
P^T (gh + gl).  The reference is fp64 of the fp32 q, k, v, dO, with delta from the forward's fp32 output
o = O'[0:D] + O'[2D:3D].  Against it the kernel's terms are:
  logits   Q'K'^T misses ql kl, and x - (xh + xl) is the lo half's own rounding: |s' - s| <= 3 * 2^-16 * scale
           |q|.|k|, a relative error C16 2^-16 amp of p (C16 = 4), without the (D + n) of the fp32 sums
  dP       dO'V'^T misses gl vl and the lo roundings: C16 2^-16 (|dO| @ |V|^T)
  delta    rowsum(dO' O') = gh.o_h + gl.o_h + gh.o_l misses gl.o_l and gl's rounding: C16 2^-16 rowsum(|dO| |O|)
  outputs  each gradient is the fp32 sum of two bf16 outputs; the lo one (2^-8 of the hi one) rounds by 2^-9 of
           itself, and the lo operand halves round by 2^-17: 2 * 2^-16 * (|dS| @ |K|, |dS|^T @ |Q|, |P|^T @ |dO|)
P^T and dS^T still pass through bf16 before the MMAs, so the gradients keep their 2^-8 terms: the x3 backward is a
bf16-accurate gradient of 2^-16-accurate logits.  Consequence: a layout fault that drops a lo part (dQ'[2D:3D] =
dS kl, dV'[D:2D] = P^T gl, the P vl third of O' in delta) moves a gradient by at most 2^-9 of the 2^-8 (|P| @ |dO|)-type
term that admits P's rounding, so no sound element bound on the summed gradient can reject it.  Those faults are
caught part by part instead: `x3_operands` builds Q', K', V', dO' from the definition, `reference` in bf16 mode on
them (with O' from the forward) gives each of dQ', dK', dV' with its own bound, so a dropped part fails against its
own magnitude, and the summed gradient must equal the sum of the parts bit for bit.  x3 mode checks the summed
gradient's accuracy end to end: at logits |s| ~ 40 a backward whose logits use the hi halves only lies outside it.
"""
from __future__ import annotations

import torch

C32 = 4.0
C16 = 4.0
U8, U16, U24 = 2.0 ** -8, 2.0 ** -16, 2.0 ** -24


def _bias(slopes, S, h0, h1, device):
    from tests.attn_fwd_check import MAX_SLOPE, alibi_bias
    if float(slopes.abs().max()) > MAX_SLOPE:
        raise ValueError(f"reference: the bound is derived for ALiBi slopes up to {MAX_SLOPE}")
    return alibi_bias(slopes, S, h0, h1, device)


def forward64(q, k, v, scale, causal, mask=None, slopes=None):
    """fp64 attention forward of bf16 [B,S,H,D] / [B,S,Hk,D] inputs -> (o bf16, lse fp32 [B,H,S]).  mask: an optional
    boolean visibility mask [S, S] or [B, S, S] (tests/attn_fwd_check.visible), intersected with `causal`.  slopes:
    ALiBi's fp32 [H] slopes."""
    B, S, H, D = q.shape
    g = H // k.shape[2]
    qd, kd, vd = (t.double().transpose(1, 2) for t in (q, k, v))
    kd, vd = kd.repeat_interleave(g, 1), vd.repeat_interleave(g, 1)
    s = scale * qd @ kd.transpose(-1, -2)
    if slopes is not None:
        s = s + _bias(slopes, S, 0, H, q.device)[None]
    if causal:
        s = s.masked_fill(torch.ones(S, S, dtype=torch.bool, device=q.device).triu(1), float("-inf"))
    if mask is not None:
        s = s.masked_fill(~(mask[:, None] if mask.dim() == 3 else mask), float("-inf"))
    lse = torch.logsumexp(s, -1)
    o = torch.softmax(s, -1) @ vd
    return o.transpose(1, 2).to(torch.bfloat16).contiguous(), lse.float().contiguous()


def x3_operands(q, k, v, do, kernel_d=None):
    """The bf16 operands of ops.attention_fp32's kernel calls, built from their definition: fp32 x = hi + lo with
    hi = bf16(x), lo = bf16(x - hi); Q' = [qh|ql|qh], K' = [kh|kh|kl], V' = [vh|vh|vl], dO' = [gh|gl|gh], zero-padded
    to kernel_d (default: 64 or 128).  Returns (q3, k3, v3, do3)."""
    D = q.shape[-1]
    Dp = kernel_d or (64 if 3 * D <= 64 else 128)

    def hl(x):
        h = x.float().to(torch.bfloat16)
        return h, (x.float() - h.float()).to(torch.bfloat16)

    def cat3(a, b, c):
        return torch.nn.functional.pad(torch.cat([a, b, c], -1), (0, Dp - 3 * D)).contiguous()
    (qh, ql), (kh, kl), (vh, vl), (gh, gl) = hl(q), hl(k), hl(v), hl(do)
    return cat3(qh, ql, qh), cat3(kh, kh, kl), cat3(vh, vh, vl), cat3(gh, gl, gh)


def reference(q, k, v, o, do, lse, scale, causal, rows=None, mask_shift=0, drop_keys=None, mask=None, slopes=None,
              head_chunk=None, x3=False, kernel_d=None, bias=None):
    """fp64 dq, dk, dv (one batch row at a time) and their element-wise bounds for the batch rows `rows`.
    Returns dict name -> (ref [len(rows),S,heads,D], bound).  mask: an optional boolean visibility mask [S, S] or
    [B, S, S] (documents, windows: tests/attn_fwd_check.visible), intersected with `causal`.  slopes: ALiBi's fp32 [H]
    slopes.  head_chunk: query heads per fp64 pass (a multiple of the GQA group; None: all), so long rows fit in
    memory.  x3: fp32 q, k, v, dO and the bf16x3 path's fp32 o (module docstring); kernel_d: the head dim the kernel
    sums over (x3: the padded 3 D).  Fault tests: `mask_shift` moves the causal diagonal, `drop_keys` (a slice)
    leaves those keys out of P, `bias` (h0, h1) -> fp64 [h1 - h0, S, S] replaces the ALiBi bias in P only (the
    bound stays that of `slopes`)."""
    B, S, H, D = q.shape
    Hk = k.shape[2]
    g = H // Hk
    Dk = kernel_d or D
    hc = H if head_chunk is None else head_chunk
    if hc % g:
        raise ValueError("head_chunk must be a multiple of the GQA group")
    rows = range(B) if rows is None else rows
    out = {n: ([], []) for n in ("dq", "dk", "dv")}
    keep = None
    if causal:
        keep = torch.ones(S, S, dtype=torch.bool, device=q.device).tril(mask_shift)
    n = S
    for b in rows:
        mb = None if mask is None else (mask[b] if mask.dim() == 3 else mask)
        dq_b, bdq_b = [], []
        dk_b = torch.zeros(Hk, S, D, dtype=torch.float64, device=q.device)
        dv_b, bdk_b, bdv_b = torch.zeros_like(dk_b), torch.zeros_like(dk_b), torch.zeros_like(dk_b)
        for h0 in range(0, H, hc):
            h1 = min(H, h0 + hc)
            qd, od, dod = (t[b, :, h0:h1].double().transpose(0, 1) for t in (q, o, do))    # [heads, S, D]
            kd, vd = (t[b, :, h0 // g:h1 // g].double().transpose(0, 1).repeat_interleave(g, 0) for t in (k, v))
            s = scale * qd @ kd.transpose(-1, -2)
            # weights of the fp32 terms; exp2 turns a logit error into a relative one
            amp = 1.0 + scale * qd.abs() @ kd.abs().transpose(-1, -2)
            if slopes is not None:
                bh = _bias(slopes, S, h0, h1, q.device)
                amp = amp + bh.abs()
                s = s + (bh if bias is None else bias(h0, h1))
                del bh
            elif bias is not None:
                s = s + bias(h0, h1)
            # masked before exp: ALiBi's bias m (k - q) is positive on the future keys and can overflow exp
            if keep is not None:
                s = s.masked_fill(~keep, float("-inf"))
            if mb is not None:
                s = s.masked_fill(~mb, float("-inf"))
            p = torch.exp(s - lse[b, h0:h1].double()[..., None])
            del s
            if drop_keys is not None:
                p[..., drop_keys] = 0
            dp = dod @ vd.transpose(-1, -2)
            delta = (dod * od).sum(-1, keepdim=True)
            ds = p * (dp - delta)
            dq = scale * ds @ kd
            dk = scale * ds.transpose(-1, -2) @ qd
            dv = p.transpose(-1, -2) @ dod
            pa = p.abs()
            pw = pa * amp
            dsum = dod.abs() @ vd.abs().transpose(-1, -2) + (dod.abs() * od.abs()).sum(-1, keepdim=True)
            dsw = (Dk + n) * pw * (dp.abs() + delta.abs()) + Dk * pa * dsum
            b_dq = U8 * scale * ds.abs() @ kd.abs() + C32 * U24 * scale * dsw @ kd.abs() + U8 * dq.abs()
            b_dk = U8 * scale * ds.abs().transpose(-1, -2) @ qd.abs() \
                + C32 * U24 * scale * dsw.transpose(-1, -2) @ qd.abs()
            b_dv = U8 * pa.transpose(-1, -2) @ dod.abs() + C32 * U24 * (Dk + n) * pw.transpose(-1, -2) @ dod.abs()
            if x3:
                dsw16 = C16 * U16 * (pw * (dp.abs() + delta.abs()) + pa * dsum) + 2 * U16 * ds.abs()
                b_dq = b_dq + scale * dsw16 @ kd.abs()
                b_dk = b_dk + scale * dsw16.transpose(-1, -2) @ qd.abs()
                b_dv = b_dv + (C16 * U16 * pw + 2 * U16 * pa).transpose(-1, -2) @ dod.abs()
            del p, pa, pw, dp, ds, dsw, dsum, amp
            dq_b.append(dq)
            bdq_b.append(b_dq)
            kv = slice(h0 // g, h1 // g)
            for acc, x in ((dk_b, dk), (dv_b, dv), (bdk_b, b_dk), (bdv_b, b_dv)):
                acc[kv] += x.reshape(-1, g, S, D).sum(1)
        bdk_b, bdv_b = bdk_b + U8 * dk_b.abs(), bdv_b + U8 * dv_b.abs()
        for name, r, bd in (("dq", torch.cat(dq_b), torch.cat(bdq_b)), ("dk", dk_b, bdk_b), ("dv", dv_b, bdv_b)):
            out[name][0].append(r.transpose(0, 1))
            out[name][1].append(bd.transpose(0, 1))
    return {nm: (torch.stack(r), torch.stack(bd)) for nm, (r, bd) in out.items()}


def check(name, got, ref, bound, tiny=1e-30):
    """Element-wise |got - ref| <= bound; returns the largest error / bound ratio, raises naming the worst element.
    A non-finite ratio (a NaN reference or bound) fails too."""
    err = (got.double() - ref).abs()
    ratio = err / (bound + tiny)
    worst = float(ratio.max())
    if not torch.isfinite(got).all() or not torch.isfinite(ratio).all() or worst > 1.0:
        i = int(torch.nan_to_num(ratio, nan=float("inf")).flatten().argmax())
        idx = list(torch.unravel_index(torch.tensor(i), ratio.shape))
        idx = [int(x) for x in idx]
        raise AssertionError(f"{name}: worst error/bound {worst:.3g} at [row, token, head, d] = {idx} "
                             f"(token {idx[1]} is in key/query tile {idx[1] // 128}/{idx[1] // 64}): "
                             f"got {float(got.flatten()[i]):.6g} ref {float(ref.flatten()[i]):.6g} "
                             f"bound {float(bound.flatten()[i]):.3g}")
    return worst
