"""fp64 reference and element-wise bounds for attention with dropout (b200_attn_fwd_dropout / b200_attn_bwd_dropout),
built on the derivations of tests/attn_fwd_check.py and tests/attn_bwd_check.py.

With the keep mask Z (tests/dropout_oracle.py) and sc = 1 / (1 - p_eff), the kernels compute O = sc (P o Z) V with
P the dropout-free softmax (its normaliser l sums every visible key), and the LSE of that softmax.  The backward
computes dV = sc (P o Z)^T dO, dS = P o (sc Z o dP - delta) with delta = rowsum(dO o O) of the dropped O, and
dQ = scale dS K, dK = scale dS^T Q.  Each dropout-free bound term carries over with P replaced by the P that enters
the product, and every term of a scaled output is multiplied by sc:

  O    sc [2^-8 (|PZ| @ |V|) + C32 2^-24 (D + n) ((|PZ| o amp) @ |V| + (|PZ| @ |V|) sum_j p_j amp_j)] + 2^-8 |O|
       the last fp32 term is the normaliser's relative error, which sums the dropped keys too
  LSE  the dropout-free bound (Z does not enter it)
  dV   sc [2^-8 (|PZ|^T @ |dO|) + C32 2^-24 (D + n) ((|PZ| o amp)^T @ |dO|)] + 2^-8 |dV|
  dS   the dropout-free weight with dP replaced by sc Z dP: (D + n) |P| amp (sc Z |dP| + |delta|) +
       D |P| (sc Z (|dO| @ |V|^T) + rowsum(|dO| |O|)); dQ and dK as in attn_bwd_check

sc itself is fl(65536 / (65536 - t)), within 2^-24 of its value: inside the C32 2^-24 (D + n) terms.  x3 adds the
bf16x3 path's terms of both modules the same way.  The reference runs one (row, query head) at a time on the
operands' device, so S = 8192 fits.
"""
from __future__ import annotations

import torch

from tests import dropout_oracle as do
from tests.attn_fwd_check import C16, C32, U8, U16, U24, alibi_bias, check  # noqa: F401  (check: re-exported)


def _head(q, k, v, b, h):
    g = q.shape[2] // k.shape[2]
    return (q[b, :, h].double(), k[b, :, h // g].double(), v[b, :, h // g].double())


def reference(q, k, v, o, dout, lse, scale, vis, seed, p, slopes=None, x3=False, kernel_d=None, keep_fn=None,
              sc=None):
    """fp64 references with element-wise bounds: {"o", "lse", "dq", "dk", "dv"} -> (ref, bound), shaped like the
    kernel's outputs ([B, S, heads, D] and lse [B, H, S]).  o / lse: the kernel's forward outputs (delta uses o, as
    the backward does; lse None: the fp64 one).  vis: bool [B, S, S] visibility.  keep_fn(b, h) -> bool [S, S]
    replaces the oracle's mask and sc the oracle's scale (fault tests: the bounds keep the true form, the references
    take the fault)."""
    B, S, H, D = q.shape
    Hk = k.shape[2]
    g = H // Hk
    Dk = kernel_d or D
    n = S
    dev = q.device
    sc_true = do.scale(p)
    sc = sc_true if sc is None else sc
    out = {nm: (torch.zeros(B, S, hh, D, dtype=torch.float64, device=dev),
                torch.zeros(B, S, hh, D, dtype=torch.float64, device=dev))
           for nm, hh in (("o", H), ("dq", H), ("dk", Hk), ("dv", Hk))}
    lse_r = torch.zeros(B, H, S, dtype=torch.float64, device=dev)
    lse_b = torch.zeros_like(lse_r)
    for b in range(B):
        for h in range(H):
            qd, kd, vd = _head(q, k, v, b, h)
            od, dod = o[b, :, h].double(), dout[b, :, h].double()
            s = scale * qd @ kd.T
            amp = 1.0 + scale * qd.abs() @ kd.abs().T
            if slopes is not None:
                bh = alibi_bias(slopes, S, h, h + 1, dev)[0]
                s, amp = s + bh, amp + bh.abs()
                del bh
            s = s.masked_fill(~vis[b], float("-inf"))
            ls = torch.logsumexp(s, -1)
            P = torch.exp(s - ls[:, None])
            del s
            keep = (do.keep_mask_head_torch(seed, p, b, h, S, dev) if keep_fn is None
                    else torch.as_tensor(keep_fn(b, h), device=dev))
            PZ = P * keep
            pw, pzw = P * amp, PZ * amp
            spa = pw.sum(-1, keepdim=True)
            # forward
            o_r = sc * PZ @ vd
            pzv, pzav = PZ @ vd.abs(), pzw @ vd.abs()
            bo = sc_true * (U8 * pzv + C32 * U24 * (Dk + n) * (pzav + pzv * spa)) + U8 * o_r.abs()
            bl = C32 * U24 * ((Dk + n) * spa[:, 0] + ls.abs())
            if x3:
                bo = bo + sc_true * (2 * U16 * pzv + C16 * U16 * (pzav + pzv * spa))
                bl = bl + C16 * U16 * spa[:, 0]
            out["o"][0][b, :, h], out["o"][1][b, :, h] = o_r, bo
            lse_r[b, h], lse_b[b, h] = ls, bl
            # backward (P from the kernel's LSE, as the kernel recomputes it)
            if lse is not None:
                P = P * torch.exp(ls - lse[b, h].double())[:, None]
            PZ = P * keep
            pw, pzw = P * amp, PZ * amp
            dpv = dod @ vd.T
            dp = sc * keep * dpv
            delta = (dod * od).sum(-1, keepdim=True)
            ds = P * (dp - delta)
            dsum = sc_true * keep * (dod.abs() @ vd.abs().T) + (dod.abs() * od.abs()).sum(-1, keepdim=True)
            dsw = (Dk + n) * pw * (sc_true * keep * dpv.abs() + delta.abs()) + Dk * P * dsum
            dq = scale * ds @ kd
            b_dq = U8 * scale * ds.abs() @ kd.abs() + C32 * U24 * scale * dsw @ kd.abs() + U8 * dq.abs()
            dk = scale * ds.T @ qd
            b_dk = U8 * scale * ds.abs().T @ qd.abs() + C32 * U24 * scale * dsw.T @ qd.abs()
            dv = sc * PZ.T @ dod
            b_dv = sc_true * (U8 * PZ.T @ dod.abs() + C32 * U24 * (Dk + n) * pzw.T @ dod.abs())
            if x3:
                dsw16 = C16 * U16 * (pw * (sc_true * keep * dpv.abs() + delta.abs()) + P * dsum) + 2 * U16 * ds.abs()
                b_dq = b_dq + scale * dsw16 @ kd.abs()
                b_dk = b_dk + scale * dsw16.T @ qd.abs()
                b_dv = b_dv + sc_true * (C16 * U16 * pzw + 2 * U16 * PZ).T @ dod.abs()
            out["dq"][0][b, :, h], out["dq"][1][b, :, h] = dq, b_dq
            for nm, x, bx in (("dk", dk, b_dk), ("dv", dv, b_dv)):
                out[nm][0][b, :, h // g] += x
                out[nm][1][b, :, h // g] += bx
            del P, PZ, pw, pzw, dpv, dp, ds, dsw, dsum, amp, keep
    for nm in ("dk", "dv"):
        r, bd = out[nm]
        out[nm] = (r, bd + U8 * r.abs())
    out["lse"] = (lse_r, lse_b)
    return out
