"""CPU: tests/moe_check.py accepts an fp32 emulation of the MoE kernels' arithmetic (routing, combine, combine backward
with the router adjoint, un-permutation, the router GEMMs) and rejects single seeded faults of the kind those kernels
can have, each with a message that names the stage and the element."""
import math

import pytest
import torch

from tests import moe_check as mc
from tests import moe_oracle as mo

BF16, F32 = torch.bfloat16, torch.float32


def _gen(seed):
    return torch.Generator().manual_seed(seed)


# ---- fp32 emulations in the kernels' order of operations --------------------------------------------------------
def _softmax(lg, skip_high=False):
    """route_topk_kernel's softmax: lane l holds experts l and l + 32, a butterfly warp sum, one division."""
    T, E = lg.shape
    v = torch.full((T, 64), -math.inf)
    v[:, :E] = lg
    m = v.amax(-1, keepdim=True)
    e = torch.exp(v - m)
    lane = e[:, :32] + (0.0 if skip_high else e[:, 32:])
    idx = torch.arange(32)
    for o in (16, 8, 4, 2, 1):
        lane = lane + lane[:, idx ^ o]
    return (e / lane[:, :1])[:, :E]


def _weights(p, ids):
    sel = p.gather(1, ids)
    tot = torch.zeros(p.shape[0])
    for j in range(ids.shape[1]):
        tot = tot + sel[:, j]
    return sel / tot[:, None]


def _psum(p, mask, extra=None):
    """route_hist_kernel's per-chunk sequential sums, then route_scan_kernel's sum over the chunks."""
    T, E = p.shape
    parts = []
    for c in range(0, T, mc.CHUNK):
        s = torch.zeros(E)
        for t in range(c, min(T, c + mc.CHUNK)):
            if mask is None or mask[t]:
                s = s + p[t]
        if extra is not None and c <= extra < c + mc.CHUNK:
            s = s + p[extra]
        parts.append(s)
    tot = torch.zeros(E)
    for s in parts:
        tot = tot + s
    return tot


def _route(lg, k, mask):
    T, E = lg.shape
    p = _softmax(lg)
    ids = mc.topk_ids(p, k)
    counts, seg_off, tiles, dest = mo.emulate_routing(ids, E)
    cnt = (torch.nn.functional.one_hot(ids, E).sum(1) * mask[:, None]).sum(0).float()
    return {"ids": ids.int(), "weights": _weights(p, ids), "probs": p, "counts": counts.int(), "seg_off": seg_off.int(),
            "tile_expert": tiles.int(), "n_tiles": torch.tensor([int(seg_off[-1]) // 128]).int(), "dest": dest.int(),
            "aux_counts": cnt, "aux_psum": _psum(p, mask)}


def _dw(dout, yp, dest, drop_warp=None, drop_last_vector=False):
    """combine_bwd_kernel's dw: 8-product sums per vector, per-thread sums over its vectors (v = thread + 128 i), a
    butterfly warp sum, then ((w0 + w1) + w2) + w3."""
    T, H = dout.shape
    nv = H // 8
    out = []
    for j in range(dest.shape[1]):
        prod = (dout.float() * yp[dest[:, j].long()].float()).view(T, nv, 8)
        s = torch.zeros(T, nv)
        for i in range(8):
            s = s + prod[:, :, i]
        if drop_last_vector:
            s[:, -1] = 0
        per = -(-nv // 128)
        s = torch.cat([s, torch.zeros(T, per * 128 - nv)], 1).view(T, per, 128)
        part = torch.zeros(T, 128)
        for i in range(per):
            part = part + s[:, i]
        lane = part.view(T, 4, 32)
        idx = torch.arange(32)
        for o in (16, 8, 4, 2, 1):
            lane = lane + lane[:, :, idx ^ o]
        red = lane[:, :, 0]
        if drop_warp is not None:
            red[:, drop_warp] = 0
        out.append(((red[:, 0] + red[:, 1]) + red[:, 2]) + red[:, 3])
    return torch.stack(out, 1)


def _dlogits(dw, p, w, ids, aux_grad, mask, fault=None):
    """combine_bwd_kernel's router adjoint in fp32, in the kernel's order."""
    T, E = p.shape
    k = ids.shape[1]
    on = mask.bool() if fault != "aux_on_masked" else torch.ones(T, dtype=torch.bool)
    dp = torch.zeros(T, E)
    if aux_grad is not None and fault != "aux_dropped":
        dp = torch.where(on[:, None], aux_grad[None, :].expand(T, E), dp)
    S, c = torch.zeros(T), torch.zeros(T)
    for j in range(k):
        S = S + p.gather(1, ids[:, j:j + 1].long())[:, 0]
        c = c + dw[:, j] * w[:, j]
    if fault == "no_c":
        c = torch.zeros(T)
    if fault == "no_S":
        S = torch.ones(T)
    for j in range(k):
        dp.scatter_add_(1, ids[:, j:j + 1].long(), ((dw[:, j] - c) / S)[:, None])
    q = torch.zeros(T)
    for e in range(E):
        q = q + p[:, e] * dp[:, e]
    if fault == "no_q":
        q = torch.zeros(T)
    return p * (dp - q[:, None])


def _case(T=150, E=8, k=2, H=264, aux=True, seed=0, logits=None):
    g = _gen(seed)
    lg = torch.randn(T, E, generator=g) * 2.0 if logits is None else logits
    mask = (torch.rand(T, generator=g) > 0.3).to(torch.uint8)
    r = _route(lg, k, mask)
    rows = int(r["seg_off"][-1]) + 128           # a buffer longer than the segments, as the layer allocates
    yp = torch.randn(rows, H, generator=g).to(BF16)
    dout = torch.randn(T, H, generator=g).to(BF16)
    aux_grad = torch.randn(E, generator=g) * 0.1 if aux else None
    before = torch.full((rows, H), float("nan"), dtype=BF16)
    dest, w = r["dest"], r["weights"]
    dyp = before.clone()
    dyp[:int(r["seg_off"][-1])] = 0
    for j in range(k):
        dyp[dest[:, j].long()] = (w[:, j, None] * dout.float()).to(BF16)
    dw = _dw(dout, yp, dest)
    dl = _dlogits(dw, r["probs"], w, r["ids"], aux_grad, mask)
    out = torch.zeros(T, H)
    for j in range(k):
        out = out + w[:, j, None] * yp[dest[:, j].long()].float()
    addend = torch.randn(T, H, generator=g)
    return dict(lg=lg, mask=mask, k=k, r=r, yp=yp, dout=dout, aux_grad=aux_grad, before=before, dyp=dyp, dw=dw,
                dl=dl, comb=out.to(BF16), addend=addend, dx=mc.unpermute_ref(yp, dest, addend))


def _check_route(c, **override):
    out = dict(c["r"], **override)
    return mc.check_route(c["lg"], c["k"], c["mask"], out, "emulation")


def _check_bwd(c, **override):
    v = dict(dyp=c["dyp"], dw=c["dw"], dl=c["dl"], aux_grad=c["aux_grad"], before=c["before"])
    v.update(override)
    r = c["r"]
    return mc.check_combine_bwd(c["dout"], c["yp"], r["dest"], r["ids"], r["weights"], r["probs"], v["aux_grad"],
                                c["mask"], r["seg_off"], v["before"], v["dyp"], v["dw"], v["dl"],
                                "emulation")


def _check_comb(c, got):
    r = c["r"]
    return mc.check(got, *mc.combine_fwd(c["yp"], r["dest"], r["weights"]), "emulation combine (token, element)")


# ---- acceptance ----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("T,E,k,H", [(150, 8, 2, 264), (1, 2, 2, 8), (65, 64, 8, 1032), (130, 33, 3, 2048),
                                     (70, 5, 1, 16)])
def test_emulation_passes_every_check(T, E, k, H):
    for aux in (True, False):
        c = _case(T, E, k, H, aux, seed=T + E)
        assert _check_route(c) < 1
        assert _check_bwd(c) < 1
        assert _check_comb(c, c["comb"]) < 1
        mc.bitwise(c["dx"], mc.unpermute_ref(c["yp"], c["r"]["dest"], c["addend"]), "unpermute")


def test_integer_and_underflowing_logits_pass():
    g = _gen(3)
    ties = torch.randint(-2, 3, (200, 8), generator=g).float()        # many exact ties
    wide = torch.rand(200, 64, generator=g) * 200.0                   # most probabilities underflow to 0
    wide = wide - 200.0 * (torch.rand(200, 64, generator=g) < 0.9)
    for lg, k in ((ties, 3), (wide, 8)):
        c = _case(200, lg.shape[1], k, 64, True, logits=lg)
        _check_route(c)
        _check_bwd(c)
    assert bool(((c["r"]["probs"] > 0).sum(-1) < 8).any()), "k must exceed the non-zero count on some row"


@pytest.mark.parametrize("T,E,k", [(1, 2, 1), (63, 8, 2), (64, 3, 2), (65, 64, 8), (300, 33, 3), (1000, 4, 4)])
def test_index_ref_is_the_emulation(T, E, k):
    ids = torch.stack([torch.randperm(E, generator=_gen(t))[:k] for t in range(T)])
    got, want = mc.index_ref(ids, E), mo.emulate_routing(ids, E)
    for a, b in zip(got, want):
        assert torch.equal(a, b.long())


def test_k1_router_gradient_is_exactly_zero():
    c = _case(100, 4, 1, 64, aux=False)
    assert bool((c["dl"].view(torch.int32) == 0).all())
    _check_bwd(c)


# ---- rejection -----------------------------------------------------------------------------------------------------
def _rejects(fn, match):
    with pytest.raises(AssertionError, match=match) as e:
        fn()
    return str(e.value)


def test_rejects_neighbour_probs():
    c = _case()
    p = c["r"]["probs"].clone()
    p[40] = p[41]
    msg = _rejects(lambda: _check_route(c, probs=p), "probs")
    assert "element (40," in msg


def test_rejects_softmax_sum_without_upper_half():
    c = _case(100, 64, 8, 64)
    _rejects(lambda: _check_route(c, probs=_softmax(c["lg"], skip_high=True)), "probs")


def test_rejects_tie_toward_higher_index():
    lg = torch.randint(-1, 2, (100, 8), generator=_gen(5)).float()
    c = _case(100, 8, 3, 64, logits=lg)
    p = c["r"]["probs"]
    ids = (7 - mc.topk_ids(torch.flip(p, [1]), 3)).int()           # ties toward the higher index
    assert not torch.equal(ids, c["r"]["ids"])
    msg = _rejects(lambda: _check_route(c, ids=ids), "ids vs the top-k")
    assert "token" in msg and "slot" in msg


def test_rejects_weights_normalised_by_all_of_p():
    c = _case()
    w = c["r"]["probs"].gather(1, c["r"]["ids"].long())
    _rejects(lambda: _check_route(c, weights=w), "weights")


def test_rejects_psum_with_a_masked_token():
    c = _case()
    t = int((c["mask"] == 0).nonzero()[0, 0])
    ps = _psum(c["r"]["probs"], c["mask"], extra=t)
    _rejects(lambda: _check_route(c, aux_psum=ps), "aux_psum")


def test_rejects_chunk_boundary_token_counted_twice():
    c = _case()
    mask = c["mask"].clone()
    mask[64] = 1
    c["mask"] = mask
    c["r"] = dict(c["r"], aux_psum=_psum(c["r"]["probs"], mask),
                  aux_counts=(torch.nn.functional.one_hot(c["r"]["ids"].long(), 8).sum(1) * mask[:, None]).sum(0).float())
    _check_route(c)
    ps = _psum(c["r"]["probs"], mask, extra=64)                    # token 64 added to chunk 1 a second time
    _rejects(lambda: _check_route(c, aux_psum=ps), "aux_psum")


def test_rejects_combine_with_the_next_slot_weight():
    c = _case()
    r = c["r"]
    w = r["weights"]
    out = torch.zeros_like(c["dout"], dtype=F32)
    for j in range(2):
        out = out + w[:, (j + 1) % 2, None] * c["yp"][r["dest"][:, j].long()].float()
    msg = _rejects(lambda: _check_comb(c, out.to(BF16)), "combine")
    assert "element (" in msg


def test_rejects_unscaled_dyp():
    c = _case()
    dyp = c["dyp"].clone()
    dyp[c["r"]["dest"][:, 0].long()] = c["dout"]
    msg = _rejects(lambda: _check_bwd(c, dyp=dyp), "dyp")
    assert "row" in msg


def test_rejects_nan_pad_row():
    c = _case()
    r = c["r"]
    pad = int(r["seg_off"][0]) + int(r["counts"][0])
    assert pad < int(r["seg_off"][1])
    dyp = c["dyp"].clone()
    dyp[pad] = float("nan")
    msg = _rejects(lambda: _check_bwd(c, dyp=dyp), "dyp")
    assert f"row {pad}" in msg


def test_rejects_row_past_the_last_segment():
    c = _case()
    dyp = c["dyp"].clone()
    dyp[int(c["r"]["seg_off"][-1])] = 0
    _rejects(lambda: _check_bwd(c, dyp=dyp), "dyp")


def test_rejects_dw_missing_a_warp():
    c = _case(100, 8, 2, 2048)
    dw = _dw(c["dout"], c["yp"], c["r"]["dest"], drop_warp=3)
    msg = _rejects(lambda: _check_bwd(c, dw=dw), "dw")
    assert "element (" in msg


def test_rejects_dw_missing_the_last_vector():
    c = _case(100, 8, 2, 1032)
    dw = _dw(c["dout"], c["yp"], c["r"]["dest"], drop_last_vector=True)
    _rejects(lambda: _check_bwd(c, dw=dw), "dw")


@pytest.mark.parametrize("fault", ["no_S", "no_c", "no_q", "aux_on_masked", "aux_dropped"])
def test_rejects_router_adjoint_faults(fault):
    c = _case()
    r = c["r"]
    dl = _dlogits(c["dw"], r["probs"], r["weights"], r["ids"], c["aux_grad"], c["mask"], fault)
    msg = _rejects(lambda: _check_bwd(c, dl=dl), "dlogits")
    assert "element (" in msg


def test_rejects_nonzero_k1_router_gradient():
    c = _case(100, 4, 1, 64, aux=False)
    r = c["r"]
    w = r["weights"] * (1 - 2.0 ** -24)                      # a weight one ulp below 1: dw - c no longer cancels
    dl = _dlogits(c["dw"], r["probs"], w, r["ids"], None, c["mask"])
    assert bool((dl != 0).any())
    _rejects(lambda: _check_bwd(c, dl=dl), r"dlogits \(k = 1")


@pytest.mark.parametrize("fault", ["dropped", "twice", "slot"])
def test_rejects_unpermute_faults(fault):
    c = _case()
    dest = c["r"]["dest"]
    want = mc.unpermute_ref(c["yp"], dest, c["addend"])
    if fault == "dropped":
        got = mc.unpermute_ref(c["yp"], dest, None)
    elif fault == "twice":
        got = mc.unpermute_ref(c["yp"], dest, c["addend"] * 2)
    else:
        got = mc.unpermute_ref(c["yp"], dest[:, :1], c["addend"])
    msg = _rejects(lambda: mc.bitwise(got, want, "unpermute dx", ("token", "element")), "unpermute")
    assert "token" in msg


def test_router_gemm_bound_rejects_tf32():
    g = _gen(9)
    x = torch.randn(300, 256, generator=g).to(BF16).float()
    dl = torch.randn(300, 8, generator=g) * 1e-2
    wr = torch.randn(8, 256, generator=g).to(BF16).float()
    mc.check(dl @ wr, *mc.fp32_gemm(dl, wr), "addend")
    mc.check(dl.t() @ x, *mc.fp32_gemm(dl.t(), x), "dWr")
    tf32 = (dl.view(torch.int32) & ~0x1FFF).view(F32)              # 10 explicit mantissa bits
    _rejects(lambda: mc.check(tf32 @ wr, *mc.fp32_gemm(dl, wr), "addend"), "addend")
    _rejects(lambda: mc.check(tf32.t() @ x, *mc.fp32_gemm(dl.t(), x), "dWr"), "dWr")
