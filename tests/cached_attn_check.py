"""Checker of b200_attn_fwd_cached (a chunk of queries against a KV cache) built on tests/attn_fwd_check.py: row b's
chunk (queries at positions start[b] .. start[b] + n_b - 1) is embedded as the last n_b query rows of a full-length
problem over the cached keys [0, start[b] + n_b), whose fp64 reference and element-wise bounds are the forward's."""
from __future__ import annotations

import torch

from tests import attn_fwd_check as AF


def embed(q, kc, vc, b, start, n, keys=None):
    """(q, k, v) [1, S, heads, D] of row b's chunk as the last n query rows of a problem over S = keys (default
    start + n) cache positions; earlier query rows are zero."""
    S = start + n if keys is None else keys
    qf = torch.zeros((1, S) + tuple(q.shape[2:]), device=q.device, dtype=q.dtype)
    qf[0, start:start + n] = q[b, :n]
    return qf, kc[b:b + 1, :S], vc[b:b + 1, :S]


def check_rows(q, kc, vc, starts, ns, o, lse, window, slopes, name):
    """Each row's valid outputs o [B, L, H, D] and lse [B, H, L] against fp64 (window < 0: none; slopes: ALiBi or
    None); every padding row finite.  Raises AssertionError on a failure; returns the worst error / bound ratio."""
    D = q.shape[-1]
    worst = 0.0
    for b, (s, n) in enumerate(zip(starts, ns)):
        if not (torch.isfinite(o[b]).all() and torch.isfinite(lse[b]).all()):
            raise AssertionError(f"{name}: row {b} has a non-finite output")
        if n == 0:
            continue
        qf, k, v = embed(q, kc, vc, b, s, n)
        mask = AF.visible(s + n, True, window=None if window < 0 else window, device=q.device)
        ref = AF.reference(qf, k, v, D ** -0.5, mask=mask, slopes=slopes)
        (ro, bo), (rl, bl) = ref["o"], ref["lse"]
        worst = max(worst, AF.check(f"{name} row {b} o", o[b:b + 1, :n], ro[:, s:], bo[:, s:]))
        worst = max(worst, AF.check(f"{name} row {b} lse", lse[b:b + 1, :, :n], rl[:, :, s:], bl[:, :, s:]))
    return worst
