"""Checker of the rotating KV cache's kernels (b200_attn_fwd_ring, b200_attn_decode_ring) built on
tests/attn_fwd_check.py.  A row's chunk of queries (positions start .. end - 1) is checked against the fp64 reference of
a compact problem: the key positions the chunk may see (the sinks and the arc, fetched from their ring slots through
ops.ring_slot), each query placed at its own position's index, the mask given by the visibility rule on true positions
and ALiBi's bias m_h (k - q) on true positions.  Every other row of the compact problem sees only itself."""
from __future__ import annotations

import torch

from mlx_cuda_distributed_pretraining_b200.ops import RING_SINKS, ring_slot
from tests import attn_fwd_check as AF


def rule(q, k, M, window=None):
    """Query position q sees key position k (broadcasting int tensors) under max_kv_size M and a window."""
    ok = (k <= q) & ((k < RING_SINKS) | (q - k <= M - 5))
    if window is not None:
        ok &= q - k <= window
    return ok


def held(end, C):
    """Positions whose keys a row holding `end` positions still has: those not overwritten in a ring of C slots."""
    t = torch.arange(end)
    return (t < RING_SINKS) | (t + (C - RING_SINKS) >= end)


def _problem(q_rows, k_ring, v_ring, b, start, end, M):
    """(positions P, q [1, S, H, D], k, v [1, S, Hk, D]) of row b's compact problem."""
    C = k_ring.shape[1]
    lo = max(0, start - (M - 5))
    P = torch.tensor(sorted(set(range(min(RING_SINKS, end))) | set(range(lo, end))), dtype=torch.int64)
    slots = ring_slot(P, C).to(k_ring.device)
    qf = torch.zeros((1, len(P)) + tuple(q_rows.shape[1:]), device=q_rows.device, dtype=q_rows.dtype)
    idx = torch.searchsorted(P, torch.arange(start, end))
    qf[0, idx.to(q_rows.device)] = q_rows[:end - start]
    return P, idx, qf, k_ring[b:b + 1, slots], v_ring[b:b + 1, slots]


def reference(q_rows, k_ring, v_ring, b, start, end, M, window=None, slopes=None, bounds=True):
    """fp64 o [n, H, D] and lse [H, n] of row b's queries (q_rows [n, H, D], n = end - start), with their bounds."""
    D = q_rows.shape[-1]
    P, idx, qf, k, v = _problem(q_rows, k_ring, v_ring, b, start, end, M)
    dev = q_rows.device
    Pd = P.to(dev)
    mask = rule(Pd[:, None], Pd[None, :], M, window)
    own = torch.zeros_like(mask)
    own[idx.to(dev), :] = True
    mask = torch.where(own, mask, torch.eye(len(P), dtype=torch.bool, device=dev))
    bias = None
    if slopes is not None:
        m = slopes.detach().double().to(dev)
        dist = (Pd[None, :] - Pd[:, None]).double()
        bias = lambda h0, h1: m[h0:h1, None, None] * dist[None]  # noqa: E731
    r = AF._run(qf, k, v, D ** -0.5, mask, None, 4, bounds=bounds, bias=bias)
    i = idx.to(dev)
    if not bounds:
        return r[0][0, i], r[1][0][:, i]
    (ro, bo), (rl, bl) = r["o"], r["lse"]
    return (ro[0, i], bo[0, i]), (rl[0][:, i], bl[0][:, i])


def check_rows(q, k_ring, v_ring, starts, ends, o, lse, M, window, slopes, name):
    """Each row's queries o [B, L, H, D] / lse [B, H, L] (q [B, L, H, D]) against fp64; padding rows finite.  Raises
    AssertionError on a failure; returns the worst error / bound ratio."""
    worst = 0.0
    for b, (s, e) in enumerate(zip(starts, ends)):
        if not (torch.isfinite(o[b]).all() and torch.isfinite(lse[b]).all()):
            raise AssertionError(f"{name}: row {b} has a non-finite output")
        n = e - s
        if n == 0:
            continue
        (ro, bo), (rl, bl) = reference(q[b], k_ring, v_ring, b, s, e, M, window, slopes)
        worst = max(worst, AF.check(f"{name} row {b} o", o[b:b + 1, :n], ro[None], bo[None]))
        worst = max(worst, AF.check(f"{name} row {b} lse", lse[b:b + 1, :, :n], rl[None], bl[None]))
    return worst


def emulate(q, k_ring, v_ring, starts, ends, M, window=None, slopes=None, fault=None):
    """fp64 o [B, L, H, D] and lse [B, H, L] computed directly over the ring, rounded to bf16 / fp32 as the kernel
    stores them; `fault` emulates a wrong kernel: "no_sinks", "slot_positions" (window and ALiBi on slot indices),
    "stale" (also reads the slot just past the row's newest key) or "one_more" (q - k <= M - 4)."""
    B, L, H, D = q.shape
    C, Hk = k_ring.shape[1], k_ring.shape[2]
    o = torch.zeros(B, L, H, D, dtype=torch.float64)
    lse = torch.zeros(B, H, L, dtype=torch.float64)
    for b, (s, e) in enumerate(zip(starts, ends)):
        for i in range(e - s):
            p = s + i
            ks = torch.arange(p + 1)
            ok = rule(torch.tensor(p), ks, M + (1 if fault == "one_more" else 0), window)
            if fault == "no_sinks":
                ok &= ks >= RING_SINKS
            slots = ring_slot(ks, C)
            pq, pk = torch.tensor(p), ks
            if fault == "slot_positions":
                pq, pk = ring_slot(pq, C), slots
                ok = (ks <= p) & ((ks < RING_SINKS) | (p - ks <= M - 5))
                if window is not None:
                    ok &= (pq - pk).abs() <= window
            if fault == "stale":
                extra = ring_slot(torch.tensor(e), C)
                slots = torch.cat([slots, extra[None]])
                ok = torch.cat([ok, torch.tensor([True])])
                pk = torch.cat([pk, torch.tensor([e])])
            kk = k_ring[b, slots.to(k_ring.device)].double().cpu()
            vv = v_ring[b, slots.to(k_ring.device)].double().cpu()
            for h in range(H):
                hk = h // (H // Hk)
                sc = (kk[:, hk] @ q[b, i, h].double().cpu()) * D ** -0.5
                if slopes is not None:
                    sc = sc + float(slopes[h]) * (pk - pq).double()
                sc = sc.masked_fill(~ok, float("-inf"))
                ls = torch.logsumexp(sc, 0)
                o[b, i, h] = torch.exp(sc - ls) @ vv[:, hk]
                lse[b, h, i] = ls
    return o.to(torch.bfloat16), lse.float()
