"""fp64 reference and element-wise checker for the attention backward (b200_attn_bwd).

The backward is tested alone: O and LSE come from an fp64 forward and are rounded to bf16 / fp32, and the reference
uses that same O for delta = rowsum(dO * O).  The per-element bound has the form of tests/gemm_check.py:

  2^-8 * (|P| @ |dO|)  or  2^-8 * s * (|dS| @ |Q|), (|dS| @ |K|)   P^T / dS^T are rounded to bf16 before the MMAs
  C32 * 2^-24 * (D + n) * W                                         fp32 accumulation over n keys or queries and D;
                                                                   W uses |P| * (|dP| + |delta|) for dS, which covers
                                                                   the cancellation in dP - delta, and the logit
                                                                   magnitude s * (|q| @ |k|) that exp2 amplifies
  2^-8 * |R|                                                        bf16 output
"""
from __future__ import annotations

import torch

C32 = 4.0
U8, U24 = 2.0 ** -8, 2.0 ** -24


def forward64(q, k, v, scale, causal):
    """fp64 attention forward of bf16 [B,S,H,D] / [B,S,Hk,D] inputs -> (o bf16, lse fp32 [B,H,S])."""
    B, S, H, D = q.shape
    g = H // k.shape[2]
    qd, kd, vd = (t.double().transpose(1, 2) for t in (q, k, v))
    kd, vd = kd.repeat_interleave(g, 1), vd.repeat_interleave(g, 1)
    s = scale * qd @ kd.transpose(-1, -2)
    if causal:
        s = s.masked_fill(torch.ones(S, S, dtype=torch.bool, device=q.device).triu(1), float("-inf"))
    lse = torch.logsumexp(s, -1)
    o = torch.softmax(s, -1) @ vd
    return o.transpose(1, 2).to(torch.bfloat16).contiguous(), lse.float().contiguous()


def reference(q, k, v, o, do, lse, scale, causal, rows=None, mask_shift=0, drop_keys=None):
    """fp64 dq, dk, dv (one batch row at a time) and their element-wise bounds for the batch rows `rows`.
    Returns dict name -> (ref [len(rows),S,heads,D], bound).  Fault tests: `mask_shift` moves the causal diagonal,
    `drop_keys` (a slice) leaves those keys out of P."""
    B, S, H, D = q.shape
    Hk = k.shape[2]
    g = H // Hk
    rows = range(B) if rows is None else rows
    out = {n: ([], []) for n in ("dq", "dk", "dv")}
    keep = None
    if causal:
        keep = torch.ones(S, S, dtype=torch.bool, device=q.device).tril(mask_shift)
    for b in rows:
        qd, kd, vd, od, dod = (t[b].double().transpose(0, 1) for t in (q, k, v, o, do))  # [heads, S, D]
        kd, vd = kd.repeat_interleave(g, 0), vd.repeat_interleave(g, 0)
        s = scale * qd @ kd.transpose(-1, -2)
        p = torch.exp(s - lse[b].double()[..., None])
        if keep is not None:
            p = p * keep
        if drop_keys is not None:
            p[..., drop_keys] = 0
        dp = dod @ vd.transpose(-1, -2)
        delta = (dod * od).sum(-1, keepdim=True)
        ds = p * (dp - delta)
        dq = scale * ds @ kd
        dk = scale * ds.transpose(-1, -2) @ qd
        dv = p.transpose(-1, -2) @ dod
        # weights of the fp32 terms
        amp = 1.0 + scale * qd.abs() @ kd.abs().transpose(-1, -2)  # exp2 turns a logit error into a relative one
        pw = p.abs() * amp
        dsw = p.abs() * amp * (dp.abs() + delta.abs())
        n = S
        b_dq = U8 * scale * ds.abs() @ kd.abs() + C32 * U24 * (D + n) * scale * dsw @ kd.abs() + U8 * dq.abs()
        b_dk = U8 * scale * ds.abs().transpose(-1, -2) @ qd.abs() \
            + C32 * U24 * (D + n) * scale * dsw.transpose(-1, -2) @ qd.abs()
        b_dv = U8 * p.abs().transpose(-1, -2) @ dod.abs() + C32 * U24 * (D + n) * pw.transpose(-1, -2) @ dod.abs()
        dk, dv = dk.reshape(Hk, g, S, D).sum(1), dv.reshape(Hk, g, S, D).sum(1)
        b_dk, b_dv = b_dk.reshape(Hk, g, S, D).sum(1), b_dv.reshape(Hk, g, S, D).sum(1)
        b_dk, b_dv = b_dk + U8 * dk.abs(), b_dv + U8 * dv.abs()
        for name, r, bd in (("dq", dq, b_dq), ("dk", dk, b_dk), ("dv", dv, b_dv)):
            out[name][0].append(r.transpose(0, 1))
            out[name][1].append(bd.transpose(0, 1))
    return {n: (torch.stack(r), torch.stack(bd)) for n, (r, bd) in out.items()}


def check(name, got, ref, bound, tiny=1e-30):
    """Element-wise |got - ref| <= bound; returns the largest error / bound ratio, raises naming the worst element."""
    err = (got.double() - ref).abs()
    ratio = err / (bound + tiny)
    worst = float(ratio.max())
    if not torch.isfinite(got).all() or worst > 1.0:
        i = int(torch.nan_to_num(ratio, nan=float("inf")).flatten().argmax())
        idx = list(torch.unravel_index(torch.tensor(i), ratio.shape))
        idx = [int(x) for x in idx]
        raise AssertionError(f"{name}: worst error/bound {worst:.3g} at [row, token, head, d] = {idx} "
                             f"(token {idx[1]} is in key/query tile {idx[1] // 128}/{idx[1] // 64}): "
                             f"got {float(got.flatten()[i]):.6g} ref {float(ref.flatten()[i]):.6g} "
                             f"bound {float(bound.flatten()[i]):.3g}")
    return worst
