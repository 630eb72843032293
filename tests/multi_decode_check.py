"""fp64 checker of b200_attn_decode_multi (a short chunk of queries per row over a dense KV cache), with
b200_attn_decode's element-wise bound 2^-8 |R| (bf16 outputs) + 64 * 2^-24 * sum |p| |v|.  Query i of row b sits at
position p = start[b] + i, valid iff i < end[b] - start[b], and sees keys max(0, p - window) .. p with ALiBi's
slopes[h] * (k - p).  The reference takes the visible set per query from `visible`, so the self-tests can hand it a
broken rule."""
from __future__ import annotations

import torch

C_BOUND = 64.0


def visible(p: int, n_keys: int, window: int, device):
    """Bool [n_keys]: the keys the query at position p sees (window < 0: none)."""
    k = torch.arange(n_keys, device=device)
    ok = k <= p
    if window >= 0:
        ok = ok & (k >= p - window)
    return ok


def reference(q, kc, vc, starts, ends, window, slopes, rule=visible, bias_pos=None):
    """Per valid (row, query): fp64 (R [H, D], sum |p||v| [H, D], lse [H]) in a dict keyed by (b, i).  rule(p, n, W,
    device) gives the visible keys; bias_pos(b, i, p) the position ALiBi measures distances from (default p)."""
    B, L, H, D = q.shape
    Hk = kc.shape[2]
    scale = D ** -0.5
    out = {}
    for b in range(B):
        for i in range(max(0, ends[b] - starts[b])):
            p = starts[b] + i
            n = kc.shape[1]
            ok = rule(p, n, window, q.device)
            idx = torch.nonzero(ok).flatten()
            k = kc[b, idx].double().repeat_interleave(H // Hk, dim=1)  # [n, H, D]
            v = vc[b, idx].double().repeat_interleave(H // Hk, dim=1)
            s = torch.einsum("hd,nhd->hn", q[b, i].double(), k) * scale
            if slopes is not None:
                at = p if bias_pos is None else bias_pos(b, i, p)
                s = s + slopes.double()[:, None] * (idx.double() - at)[None, :]
            lse = torch.logsumexp(s, dim=-1)
            pr = torch.exp(s - lse[:, None])
            out[(b, i)] = (torch.einsum("hn,nhd->hd", pr, v), torch.einsum("hn,nhd->hd", pr.abs(), v.abs()), lse)
    return out


def check(o, lse, ref, bf16: bool, name: str) -> float:
    """o [B, L, H, D], lse [B, H, L] against reference(); raises AssertionError past the bound; returns the worst
    error / bound ratio."""
    worst = 0.0
    for (b, i), (R, absterm, lse_ref) in ref.items():
        got = o[b, i].double()
        if not torch.isfinite(got).all():
            raise AssertionError(f"{name}: row {b} query {i} has a non-finite output")
        bound = C_BOUND * 2.0 ** -24 * absterm + (2.0 ** -8 * R.abs() if bf16 else 0)
        ratio = float(((got - R).abs() / bound.clamp_min(1e-300)).max())
        if ratio > 1.0:
            raise AssertionError(f"{name}: row {b} query {i} error / bound {ratio:.3g}")
        le = float((lse[b, :, i].double() - lse_ref).abs().max())
        if le > 1e-4 * max(1.0, float(lse_ref.abs().max())):
            raise AssertionError(f"{name}: row {b} query {i} lse off by {le:.3g}")
        worst = max(worst, ratio)
    return worst
