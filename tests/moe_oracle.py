"""fp64 CPU oracle of the sparse MoE block (`model.misc.num_local_experts`, Mixtral's MixtralSparseMoeBlock without
jitter) and of transformers' load_balancing_loss_func, plus the whole model with MoE layers on top of the variant
oracle (tests/llama_variant_oracle.py) and the reference oracle's attention.  Also a CPU emulation of the routing
kernels' index arithmetic (counting sort, segment offsets, tile table, destinations, permutation, combine).
Test infrastructure only; pinned against transformers in tests/test_moe_host.py."""
from __future__ import annotations

from typing import Dict, List, Optional, Sequence

import torch

from oracle import reference_math as rm
from tests import llama_variant_oracle as vo

SEG = 128


def route(logits: torch.Tensor, k: int, ids: Optional[torch.Tensor] = None):
    """(p, ids, w) for logits [T, E]: p = softmax, ids [T, k] = top-k of p, larger first, on an exact tie the lower
    expert index (a stable sort of -p); w = p[ids] / sum p[ids].  ids given: the routing is forced to them."""
    p = torch.softmax(logits, dim=-1)
    if ids is None:
        ids = torch.sort(-p, dim=-1, stable=True).indices[:, :k]
    top = p.gather(-1, ids.long())
    return p, ids.long(), top / top.sum(-1, keepdim=True)


def act_fn(g: torch.Tensor, u: torch.Tensor, act: str) -> torch.Tensor:
    return torch.nn.functional.silu(g) * u if act == "silu" else g * torch.sigmoid(u) * 2


def expert(x, wg, wu, wd, act):
    lin = torch.nn.functional.linear
    return lin(act_fn(lin(x, wg), lin(x, wu), act), wd)


def moe_block(x: torch.Tensor, wr, wg, wu, wd, k: int, act: str = "silu", ids: Optional[torch.Tensor] = None):
    """(out [..., H], router logits [T, E], ids [T, k]): out[t] = sum_j w_j expert_{e_j}(x[t])."""
    H = x.shape[-1]
    x2 = x.reshape(-1, H)
    logits = torch.nn.functional.linear(x2, wr)
    _p, ids, w = route(logits, k, ids)
    out = torch.zeros_like(x2)
    for j in range(k):
        for e in range(wr.shape[0]):
            sel = ids[:, j] == e
            if bool(sel.any()):
                out = out.index_add(0, sel.nonzero()[:, 0], w[sel, j, None] * expert(x2[sel], wg[e], wu[e], wd[e], act))
    return out.view(x.shape), logits, ids


def aux_loss(logits: Sequence[torch.Tensor], k: int, mask: Optional[torch.Tensor] = None,
             ids: Optional[Sequence[torch.Tensor]] = None) -> torch.Tensor:
    """load_balancing_loss_func over the layers' router logits [T, E] (attention_mask = mask [B, S] or None):
    E * sum_e f_e P_e with f_e = assignments to e / (layers x unmasked tokens), P_e = sum of p_e over the same."""
    E = logits[0].shape[-1]
    cnt = torch.zeros(E, dtype=logits[0].dtype)
    ps = torch.zeros(E, dtype=logits[0].dtype)
    n = 0
    for i, lg in enumerate(logits):
        p, sel, _w = route(lg, k, None if ids is None else ids[i])
        m = torch.ones(lg.shape[0], dtype=lg.dtype) if mask is None else mask.reshape(-1).to(lg.dtype)
        cnt = cnt + (torch.nn.functional.one_hot(sel, E).to(lg.dtype).sum(1) * m[:, None]).sum(0)
        ps = ps + (p * m[:, None]).sum(0)
        n = n + m.sum()
    return E * (cnt / n * ps / n).sum()


def forward(params: Dict[str, torch.Tensor], tokens: torch.Tensor, d: rm.LlamaDims, E: int, k: int,
            mask: Optional[torch.Tensor] = None, positions: Optional[torch.Tensor] = None,
            ids: Optional[List[torch.Tensor]] = None):
    """tokens [B, S] -> (logits [B, S, V], router logits per layer, ids per layer) of the mlx_lm variant with every
    MLP a sparse MoE block, on the trainer's flat names.  ids: force each layer's routing (per-layer [B*S, k])."""
    lin = torch.nn.functional.linear
    B, S = tokens.shape
    h = params["embed_tokens.weight"][tokens]
    if mask is None:
        mask = rm.causal_mask(S, dtype=h.dtype)
    rot = lambda t: vo.rope_half(t, d.rope_theta, positions)  # noqa: E731
    router, chosen = [], []
    for i in range(d.num_layers):
        p = f"layers.{i}."
        x = vo.rmsnorm(h, params[p + "input_layernorm.weight"], d.rms_norm_eps)
        q = lin(x, params[p + "self_attn.attn.q_proj.weight"]).reshape(B, S, d.num_heads, d.head_dim)
        kk = lin(x, params[p + "self_attn.attn.k_proj.weight"]).reshape(B, S, d.num_kv_heads, d.head_dim)
        v = lin(x, params[p + "self_attn.attn.v_proj.weight"]).reshape(B, S, d.num_kv_heads, d.head_dim)
        ctx = rm.attention(rot(q), rot(kk), v, d.head_dim ** -0.5, mask).reshape(B, S, d.num_heads * d.head_dim)
        h = h + lin(ctx, params[p + "self_attn.attn.o_proj.weight"])
        x = vo.rmsnorm(h, params[p + "post_attention_layernorm.weight"], d.rms_norm_eps)
        m = p + "block_sparse_moe."
        out, lg, sel = moe_block(x, params[m + "gate.weight"], params[m + "switch_mlp.gate_proj.weight"],
                                 params[m + "switch_mlp.up_proj.weight"], params[m + "switch_mlp.down_proj.weight"], k,
                                 "silu", None if ids is None else ids[i])
        router.append(lg)
        chosen.append(sel)
        h = h + out
    h = vo.rmsnorm(h, params["norm.weight"], d.rms_norm_eps)
    logits = lin(h, params["embed_tokens.weight"] if d.tie_word_embeddings else params["lm_head.weight"])
    return logits, router, chosen


# ---- CPU emulation of the routing kernels' index arithmetic ------------------------------------------------------
def emulate_routing(ids: torch.Tensor, E: int, chunk: int = 64):
    """From ids [T, k]: counts [E], seg_off [E + 1] (each count padded to 128 rows), tile_expert [n_tiles] and
    dest [T, k], computed as the kernels do: per-chunk ranks in (t, j) order, per-expert scans over chunks."""
    T, k = ids.shape
    flat = ids.reshape(-1).tolist()
    nch = (T + chunk - 1) // chunk
    hist = [[0] * E for _ in range(nch)]
    rank = [0] * (T * k)
    for c in range(nch):
        for a in range(c * chunk * k, min(T, (c + 1) * chunk) * k):
            rank[a] = hist[c][flat[a]]
            hist[c][flat[a]] += 1
    base = [[0] * E for _ in range(nch)]
    counts = [0] * E
    for e in range(E):
        run = 0
        for c in range(nch):
            base[c][e] = run
            run += hist[c][e]
        counts[e] = run
    seg_off = [0]
    for e in range(E):
        seg_off.append(seg_off[-1] + (counts[e] + SEG - 1) // SEG * SEG)
    tiles = [e for e in range(E) for _ in range((seg_off[e + 1] - seg_off[e]) // SEG)]
    dest = [seg_off[flat[a]] + base[(a // k) // chunk][flat[a]] + rank[a] for a in range(T * k)]
    return (torch.tensor(counts), torch.tensor(seg_off), torch.tensor(tiles, dtype=torch.long),
            torch.tensor(dest).view(T, k))


def check_routing(ids: torch.Tensor, counts, seg_off, tiles, dest, E: int) -> None:
    """AssertionError unless (counts, seg_off, tiles, dest) is a valid dropless stable routing of ids: segments
    padded to 128 rows in expert order, the tile table covering each segment, every assignment of expert e at a
    distinct row inside e's segment, and tokens in order inside each segment."""
    T, k = ids.shape
    counts, seg_off, tiles, dest = (torch.as_tensor(v).long().cpu() for v in (counts, seg_off, tiles, dest))
    want = torch.bincount(ids.reshape(-1).long(), minlength=E)
    assert torch.equal(counts, want), f"counts {counts.tolist()} != {want.tolist()}"
    exp_off = torch.cat([torch.zeros(1, dtype=torch.long), torch.cumsum((want + SEG - 1) // SEG * SEG, 0)])
    assert torch.equal(seg_off, exp_off), f"seg_off {seg_off.tolist()} != {exp_off.tolist()}"
    n_tiles = int(exp_off[-1]) // SEG
    exp_tiles = torch.repeat_interleave(torch.arange(E), (want + SEG - 1) // SEG)
    assert torch.equal(tiles[:n_tiles], exp_tiles), "tile table does not follow the segments"
    for e in range(E):
        rows = dest[ids.long() == e]            # in token order: a token picks an expert at most once
        want_rows = torch.arange(int(exp_off[e]), int(exp_off[e]) + int(want[e]))
        assert torch.equal(rows, want_rows), f"expert {e}: rows {rows.tolist()[:8]}... not stable in token order"


def check_topk(p: torch.Tensor, ids: torch.Tensor) -> None:
    """AssertionError unless every row of ids [T, k] lists the k experts of p [T, E] in the kernels' order: larger
    probability first and, on an exact tie, the lower index first; no unselected expert ranks before the last one."""
    T, k = ids.shape
    for t in range(T):
        key = [(-float(p[t, e]), e) for e in range(p.shape[1])]
        want = [e for _, e in sorted(key)][:k]
        assert ids[t].tolist() == want, f"token {t}: ids {ids[t].tolist()} are not the top-k {want}"


def check_permute(x: torch.Tensor, dest: torch.Tensor, counts, seg_off, xp: torch.Tensor) -> None:
    """AssertionError unless xp holds x[t] at every dest[t, j] and zeros in every pad row of every segment."""
    for j in range(dest.shape[1]):
        assert torch.equal(xp[dest[:, j].long()], x), f"slot {j}: a token row is not at its destination"
    for e in range(len(counts)):
        pad = xp[int(seg_off[e]) + int(counts[e]):int(seg_off[e + 1])]
        assert not bool(pad.ne(0).any()), f"expert {e}: a pad row is not zero"


def check_combine(yp: torch.Tensor, dest: torch.Tensor, p: torch.Tensor, ids: torch.Tensor, out: torch.Tensor,
                  tol: float = 1e-12) -> None:
    """AssertionError unless out[t] = sum_j w_j yp[dest[t, j]] with w the top-k probabilities renormalised."""
    top = p.gather(1, ids.long())
    want = emulate_combine(yp, dest, top / top.sum(1, keepdim=True))
    err = float((out.double() - want).abs().max())
    assert err <= tol * float(want.abs().max().clamp_min(1e-300)), f"combine differs by {err:.3e}"


def emulate_permute(x: torch.Tensor, dest: torch.Tensor, seg_off: torch.Tensor) -> torch.Tensor:
    """The permuted buffer [seg_off[-1], H]: rows at their destinations, every pad row zero."""
    xp = torch.zeros(int(seg_off[-1]), x.shape[1], dtype=x.dtype)
    T, k = dest.shape
    for j in range(k):
        xp[dest[:, j].long()] = x
    return xp


def emulate_combine(yp: torch.Tensor, dest: torch.Tensor, w: torch.Tensor) -> torch.Tensor:
    out = torch.zeros(dest.shape[0], yp.shape[1], dtype=torch.float64)
    for j in range(dest.shape[1]):
        out += w[:, j, None].double() * yp[dest[:, j].long()].double()
    return out
