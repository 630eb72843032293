"""-m gpu: the sparse MoE MLP's own kernels (csrc/moe.cu) element by element against fp64 (tests/moe_check.py, which
derives every bound), then the MoE layer's backward stage by stage on the operands each stage actually received.

The routing runs at token counts that cross the counting sort's 64-token chunks, at expert counts on both sides of
the warp's lane + 32 half and with k = E, on Gaussian logits, integer logits full of exact ties, logits spread so wide
that most probabilities underflow to 0 (k can exceed the non-zero count), and the skewed loads of
tests/test_gpu_moe.py; with no mask, a random mask and an all-zero mask.  The combine, its backward and the
un-permutation are called directly on random rows at hidden sizes with one active thread, a ragged last vector and
several vectors per thread.  Every buffer a kernel writes is NaN- (or sentinel-) prefilled inside guard bytes that
must survive the launch."""
import pytest
import torch

from tests import moe_check as mc
from tests import rowwise_check as rc

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(900)]

BF16, F32, I32, U8T = torch.bfloat16, torch.float32, torch.int32, torch.uint8
DEV = "cuda"
NAN = float("nan")
_GUARDS = []


@pytest.fixture(scope="module")
def ops():
    from mlx_cuda_distributed_pretraining_b200 import ops
    ops.require_device()
    return ops


@pytest.fixture(autouse=True)
def guards_intact():
    """Every buffer made by G() in a test must still be framed by its sentinel bytes after it."""
    _GUARDS.clear()
    yield
    torch.cuda.synchronize()
    broken = [i for i, g in enumerate(_GUARDS) if not g.intact()]
    _GUARDS.clear()
    assert not broken, f"guard bytes overwritten around buffers {broken}"


def G(shape, dtype, fill=None):
    """A guarded device buffer; floating payloads are NaN unless `fill` is given."""
    g = rc.Guarded(shape, dtype, DEV)
    _GUARDS.append(g)
    if fill is not None:
        g.fill(fill)
    elif dtype.is_floating_point:
        g.t.fill_(NAN)
    return g


def _rec(family, r):
    rc.WORST[family] = max(rc.WORST.get(family, 0.0), r)


def _gen(seed):
    return torch.Generator(device=DEV).manual_seed(seed)


# ---- routing ---------------------------------------------------------------------------------------------------
FAMILIES = ["gauss", "ints", "wide", "one", "half_empty"]


def _logits(T, E, family, gen):
    if family == "gauss":
        return torch.randn((T, E), device=DEV, generator=gen) * 2.0
    if family == "ints":          # exact ties everywhere
        return torch.randint(-2, 3, (T, E), device=DEV, generator=gen).float()
    if family == "wide":          # a spread of ~200: most probabilities underflow to 0
        lg = torch.rand((T, E), device=DEV, generator=gen) * 200.0
        return lg - 200.0 * (torch.rand((T, E), device=DEV, generator=gen) < 0.9)
    lg = torch.randn((T, E), device=DEV, generator=gen) * 3.0
    if family == "one":
        lg[:, 1] += 40.0
    else:
        lg[:, E // 2:] -= 60.0
    return lg


def _mask(T, kind, gen):
    if kind == "none":
        return None
    if kind == "zero":
        return torch.zeros(T, device=DEV, dtype=U8T)
    return (torch.rand(T, device=DEV, generator=gen) > 0.3).to(U8T)


def _route_direct(ops, lg, k, mask, aux):
    """b200_moe_route into guarded buffers; -> dict of the outputs (payload views)."""
    L = ops.lib()
    T, E = lg.shape
    mt = int(L.b200_moe_max_tiles(T, E, k))
    b = {"ids": G((T, k), I32), "weights": G((T, k), F32), "probs": G((T, E), F32), "counts": G(E, I32),
         "seg_off": G(E + 1, I32), "tile_expert": G(max(mt, 1), I32), "n_tiles": G(1, I32), "dest": G((T, k), I32),
         "aux_counts": G(E, F32) if aux else None, "aux_psum": G(E, F32) if aux else None}
    nws = int(L.b200_moe_route_workspace_bytes(T, E, k))
    ws = G(nws, U8T)
    ptr = {n: (None if v is None else v.t.data_ptr()) for n, v in b.items()}
    ops.check(L.b200_moe_route(lg.data_ptr(), None if mask is None else mask.data_ptr(), T, E, k, ptr["ids"],
                               ptr["weights"], ptr["probs"], ptr["counts"], ptr["seg_off"], ptr["tile_expert"],
                               ptr["n_tiles"], ptr["dest"], ptr["aux_counts"], ptr["aux_psum"], ws.t.data_ptr(), nws,
                               ops._stream()), "b200_moe_route")
    out = {n: (None if v is None else v.t) for n, v in b.items()}
    out["max_tiles"] = mt
    return out


@pytest.mark.parametrize("E,k", [(2, 1), (2, 2), (3, 2), (8, 2), (8, 8), (31, 4), (32, 8), (33, 3), (64, 1), (64, 8)])
@pytest.mark.parametrize("T", [1, 63, 64, 65, 4097, 16384])
def test_routing_stages(ops, T, E, k):
    for fam in FAMILIES:
        for mk in ("none", "random", "zero"):
            gen = _gen(T * 7919 + E * 131 + k * 17 + FAMILIES.index(fam) * 3 + len(mk))
            lg = rc.Guarded((T, E), F32, DEV).fill(_logits(T, E, fam, gen)).t
            mask = _mask(T, mk, gen)
            what = f"T={T} E={E} k={k} {fam} mask={mk}"
            out = _route_direct(ops, lg, k, mask, aux=True)
            torch.cuda.synchronize()
            mc.check_route(lg, k, mask, out, what, f"route.{fam}")
            if mk == "zero":
                assert bool((out["aux_psum"] == 0).all()) and bool((out["aux_counts"] == 0).all()), what
            if mk == "none":       # without the aux partials: the same routing, bit for bit
                plain = _route_direct(ops, lg, k, None, aux=False)
                torch.cuda.synchronize()
                for n in ("ids", "weights", "probs", "counts", "seg_off", "n_tiles", "dest"):
                    assert torch.equal(plain[n].view(I32), out[n].view(I32)), f"{what}: {n} changes without aux"


def test_routing_k_beyond_nonzero_probs(ops):
    """The wide family must produce rows where k exceeds the number of non-zero probabilities."""
    lg = _logits(4097, 64, "wide", _gen(5))
    out = _route_direct(ops, lg, 8, None, aux=True)
    torch.cuda.synchronize()
    assert bool(((out["probs"] > 0).sum(-1) < 8).any())
    mc.check_route(lg, 8, None, out, "wide, k beyond the non-zero count")


@pytest.mark.parametrize("T,E,k,H", [(516, 8, 2, 1032), (1032, 64, 8, 256)])
def test_adversarial_counts_fill_every_tile(ops, T, E, k, H):
    """Every expert receives 129 = 1 (mod 128) rows, so the routing uses all b200_moe_max_tiles tiles and the
    permuted buffers are full to r.rows; the permutation and the combine backward must stay inside them."""
    L, st = ops.lib(), ops._stream()
    t = torch.arange(T, device=DEV)
    lg = torch.full((T, E), -10.0, device=DEV)
    for j in range(k):
        lg[t, (k * t + j) % E] = 10.0 - j
    out = _route_direct(ops, lg, k, None, aux=True)
    torch.cuda.synchronize()
    mc.check_route(lg, k, None, out, "adversarial")
    assert bool((out["counts"] == 129).all())
    assert int(out["n_tiles"]) == out["max_tiles"]
    rows = out["max_tiles"] * mc.SEG
    assert int(out["seg_off"][-1]) == rows
    gen = _gen(T)
    x = torch.randn((T, H), device=DEV, generator=gen).to(BF16)
    xp = G((rows, H), BF16)
    ops.check(L.b200_moe_permute(x.data_ptr(), out["dest"].data_ptr(), out["counts"].data_ptr(),
                                 out["seg_off"].data_ptr(), T, H, k, E, xp.t.data_ptr(), st), "b200_moe_permute")
    dout = torch.randn((T, H), device=DEV, generator=gen).to(BF16)
    yp = torch.randn((rows, H), device=DEV, generator=gen).to(BF16)
    dyp, dw, dl = G((rows, H), BF16), G((T, k), F32), G((T, E), F32)
    before = dyp.t.clone()
    ops.check(L.b200_moe_combine_bwd(dout.data_ptr(), yp.data_ptr(), out["dest"].data_ptr(), out["ids"].data_ptr(),
                                     out["weights"].data_ptr(), out["probs"].data_ptr(), None, None,
                                     out["counts"].data_ptr(), out["seg_off"].data_ptr(), T, H, E, k,
                                     dyp.t.data_ptr(), dw.t.data_ptr(), dl.t.data_ptr(), st), "b200_moe_combine_bwd")
    torch.cuda.synchronize()
    want = torch.zeros((rows, H), device=DEV, dtype=BF16)
    for j in range(k):
        want[out["dest"][:, j].long()] = x
    mc.bitwise(xp.t, want, "adversarial permute")
    mc.check_combine_bwd(dout, yp, out["dest"], out["ids"], out["weights"], out["probs"], None, None, out["seg_off"],
                         before, dyp.t, dw.t, dl.t, "adversarial")


# ---- combine, combine backward and un-permutation, called directly -----------------------------------------------
COMBINE_CASES = [(300, 8, 2), (100, 64, 8), (40, 5, 1), (129, 33, 3)]


@pytest.mark.parametrize("T,E,k", COMBINE_CASES)
@pytest.mark.parametrize("H", [8, 1024, 1032, 2048, 4096])
def test_combine_stages(ops, H, T, E, k):
    L, st = ops.lib(), ops._stream()
    gen = _gen(H * 31 + T + E)
    lg = torch.randn((T, E), device=DEV, generator=gen) * 2.0
    mask = (torch.rand(T, device=DEV, generator=gen) > 0.3).to(U8T)
    r = ops.moe_route(lg, k, mask, aux=True)
    rows = r.rows
    yp = torch.randn((rows, H), device=DEV, generator=gen).to(BF16)
    dout = torch.randn((T, H), device=DEV, generator=gen).to(BF16)
    dxp = torch.randn((rows, H), device=DEV, generator=gen).to(BF16)
    addend = torch.randn((T, H), device=DEV, generator=gen) * 0.5
    aux_grad = torch.randn(E, device=DEV, generator=gen) * 0.3
    what = f"H={H} T={T} E={E} k={k}"
    # forward combine
    out = G((T, H), BF16)
    ops.check(L.b200_moe_combine_fwd(yp.data_ptr(), r.dest.data_ptr(), r.weights.data_ptr(), T, H, k,
                                     out.t.data_ptr(), st), "b200_moe_combine_fwd")
    torch.cuda.synchronize()
    rc.check(out.t, *mc.combine_fwd(yp, r.dest, r.weights), f"{what} combine (token, element)", "combine_fwd")
    # un-permutation with and without the fp32 addend
    for add in (addend, None):
        dx = G((T, H), BF16)
        ops.check(L.b200_moe_unpermute(dxp.data_ptr(), r.dest.data_ptr(), None if add is None else add.data_ptr(), T,
                                       H, k, dx.t.data_ptr(), st), "b200_moe_unpermute")
        torch.cuda.synchronize()
        mc.bitwise(dx.t, mc.unpermute_ref(dxp, r.dest, add), f"{what} unpermute (addend {add is not None})",
                   ("token", "element"))

    def bwd(ag, with_dw=True, with_dl=True):
        dyp, dw, dl = G((rows, H), BF16), G((T, k), F32), G((T, E), F32)
        before = dyp.t.clone()
        ops.check(L.b200_moe_combine_bwd(dout.data_ptr(), yp.data_ptr(), r.dest.data_ptr(), r.ids.data_ptr(),
                                         r.weights.data_ptr(), r.probs.data_ptr(),
                                         None if ag is None else ag.data_ptr(), mask.data_ptr(), r.counts.data_ptr(),
                                         r.seg_off.data_ptr(), T, H, E, k, dyp.t.data_ptr(),
                                         dw.t.data_ptr() if with_dw else None, dl.t.data_ptr() if with_dl else None,
                                         st), "b200_moe_combine_bwd")
        torch.cuda.synchronize()
        return before, dyp, dw, dl

    for ag in (aux_grad, None):
        before, dyp, dw, dl = bwd(ag)
        mc.check_combine_bwd(dout, yp, r.dest, r.ids, r.weights, r.probs, ag, mask, r.seg_off, before, dyp.t, dw.t,
                             dl.t, f"{what} aux={ag is not None}")
    # dw_out NULL, then dlogits NULL: the other outputs keep their bits and the NULL output's buffer stays NaN
    ref_b, ref_dyp, ref_dw, ref_dl = bwd(aux_grad)
    _b, dyp2, dw2, dl2 = bwd(aux_grad, with_dw=False)
    _b, dyp3, dw3, dl3 = bwd(aux_grad, with_dl=False)
    assert bool(torch.isnan(dw2.t).all()), f"{what}: dw written with dw_out NULL"
    assert bool(torch.isnan(dl3.t).all()), f"{what}: dlogits written with dlogits NULL"
    assert torch.equal(dl2.t.view(I32), ref_dl.t.view(I32)), f"{what}: dlogits differ with dw_out NULL"
    assert torch.equal(dw3.t.view(I32), ref_dw.t.view(I32)), f"{what}: dw differs with dlogits NULL"
    for d in (dyp2, dyp3):
        assert torch.equal(d.t.view(torch.int16), ref_dyp.t.view(torch.int16)), f"{what}: dyp differs"


# ---- the layer backward, stage by stage ------------------------------------------------------------------------------
class _Stages:
    """Wraps the ops functions _MoeFn calls by module-global name and checks every call on the operands it received:
    the router GEMMs, the routing, the permutation, each expert-segmented GEMM, the combine, the combine backward with
    the router adjoint, each weight gradient and the un-permutation.  aux_grads / aux_counts keep what each layer's
    backward received and each layer's routing wrote."""

    def __init__(self, ops, monkeypatch):
        self.aux_grads, self.aux_counts, self.dlogits, self.n = [], [], [], {}
        self._pending = None
        o = {n: getattr(ops, n) for n in ("moe", "moe_permute", "moe_gemm", "moe_combine", "moe_combine_bwd",
                                         "moe_wgrad", "moe_unpermute")}
        init = ops.MoeRouting.__init__

        def count(name):
            self.n[name] = self.n.get(name, 0) + 1

        def moe(x, w_router, *a, **kw):
            self._pending = (x.reshape(-1, x.shape[-1]), w_router)
            return o["moe"](x, w_router, *a, **kw)

        def route(obj, logits, k, mask, aux):
            init(obj, logits, k, mask, aux)
            x2, wr = self._pending
            obj._stage = {"x": x2, "wr": wr}
            torch.cuda.synchronize()
            rc.check(logits, *mc.fp32_gemm(x2, wr.t()), "router logits = x Wr^T (token, expert)", "router.logits")
            out = {n: getattr(obj, n) for n in ("ids", "weights", "probs", "counts", "seg_off", "tile_expert",
                                                "n_tiles", "dest", "aux_counts", "aux_psum")}
            mc.check_route(logits, k, mask, out, "layer routing", "layer.route")
            if aux:
                self.aux_counts.append(obj.aux_counts.double().clone())
            count("route")

        def permute(x2, r):
            xp = o["moe_permute"](x2, r)
            end = int(r.seg_off[-1])
            want = torch.zeros((end, x2.shape[1]), device=DEV, dtype=BF16)
            for j in range(r.k):
                want[r.dest[:, j].long()] = x2
            mc.bitwise(xp[:end], want, "layer permute")
            count("permute")
            return xp

        def gemm(mode, act, a, w0, w1, r, gu=None):
            c, y = o["moe_gemm"](mode, act, a, w0, w1, r, gu)
            torch.cuda.synchronize()
            refs = mc.seg_gemm(mode, act, a, w0, w1, gu, r.counts, r.seg_off)
            I = w0.shape[1] if mode in ("gateup", "gateup_dgrad") else w0.shape[2]
            for name, (rows, ref, mag) in refs.items():
                got = {"C": c, "Y": y, "C.g": c[:, :I], "C.u": c[:, I:]}[name][rows]
                mc.gemm_ratio(got, ref, mag, f"layer {mode} {name}", _rec)
            end = int(r.seg_off[-1])
            real = torch.zeros(end, dtype=torch.bool, device=DEV)
            real[r.dest.reshape(-1).long()] = True
            for name, t in (("C", c), ("Y", y)):
                if t is not None:
                    pad = t[:end][~real]
                    assert bool((pad == 0).all()), f"layer {mode} {name}: a pad row is not zero"
            count(mode)
            return c, y

        def combine(yp, r):
            out = o["moe_combine"](yp, r)
            torch.cuda.synchronize()
            rc.check(out, *mc.combine_fwd(yp, r.dest, r.weights), "layer combine (token, element)", "layer.combine")
            count("combine")
            return out

        def combine_bwd(dout, yp, r, aux_grad):
            dyp, dw, dl = o["moe_combine_bwd"](dout, yp, r, aux_grad)
            torch.cuda.synchronize()
            mc.check_combine_bwd(dout, yp, r.dest, r.ids, r.weights, r.probs, aux_grad, r.mask, r.seg_off, None, dyp,
                                 dw, dl, "layer combine_bwd", "layer.combine_bwd")
            r._stage["dlogits"] = dl
            self.dlogits.append(dl)
            self.aux_grads.append(None if aux_grad is None else aux_grad.double().clone())
            count("combine_bwd")
            return dyp, dw, dl

        def wgrad(p, ldp, q, ldq, g, r):
            prior = g.clone()
            o["moe_wgrad"](p, ldp, q, ldq, g, r)
            torch.cuda.synchronize()
            E, R, Cc = g.shape
            for e in range(E):
                n, off = int(r.counts[e]), int(r.seg_off[e])
                if n == 0:
                    assert torch.equal(g[e].view(torch.int16), prior[e].view(torch.int16)), f"empty expert {e} written"
                    continue
                P, Q = p[off:off + n, :R].double(), q[off:off + n, :Cc].double()
                mc.gemm_ratio(g[e], prior[e].double() + P.t() @ Q, prior[e].double().abs() + P.abs().t() @ Q.abs(),
                              "layer wgrad", _rec)
            count("wgrad")

        def unpermute(dxp, r, addend=None):
            dx = o["moe_unpermute"](dxp, r, addend)
            torch.cuda.synchronize()
            mc.bitwise(dx, mc.unpermute_ref(dxp, r.dest, addend), "layer unpermute", ("token", "element"))
            st = r._stage
            if addend is not None:
                rc.check(addend, *mc.fp32_gemm(st["dlogits"], st["wr"]),
                         "router dgrad addend = dlogits Wr (token, element)",
                         "router.addend")
            count("unpermute")
            return dx

        for n, f in (("moe", moe), ("moe_permute", permute), ("moe_gemm", gemm), ("moe_combine", combine),
                     ("moe_combine_bwd", combine_bwd), ("moe_wgrad", wgrad), ("moe_unpermute", unpermute)):
            monkeypatch.setattr(ops, n, f)
        monkeypatch.setattr(ops.MoeRouting, "__init__", route)


LAYER_CASES = [(300, 8, 2, 256, 128), (200, 64, 8, 256, 128), (5, 4, 1, 256, 128), (2048, 8, 2, 1024, 1408)]


@pytest.mark.parametrize("aux", ["off", "on", "masked"])
@pytest.mark.parametrize("act", ["silu", "sigmoid2"])
@pytest.mark.parametrize("T,E,k,H,I", LAYER_CASES)
def test_layer_backward_stages(ops, monkeypatch, T, E, k, H, I, act, aux):
    gen = _gen(T + E + H)
    x = torch.randn((T, H), device=DEV, generator=gen).to(BF16)
    wr = (torch.randn((E, H), device=DEV, generator=gen) * 4 * H ** -0.5).to(BF16)
    w2 = (torch.randn((2 * E, I, H), device=DEV, generator=gen) * H ** -0.5).to(BF16).requires_grad_(True)
    wd = (torch.randn((E, H, I), device=DEV, generator=gen) * I ** -0.5).to(BF16)
    dout = torch.randn((T, H), device=DEV, generator=gen)
    mask = (torch.rand(T, device=DEV, generator=gen) > 0.3) if aux == "masked" else None
    st = _Stages(ops, monkeypatch)
    leaves = [t.clone().requires_grad_(True) for t in (x, wr, wd)]
    out, counts, psum = ops.moe(leaves[0], leaves[1], w2[:E], w2[E:], leaves[2], k, act, pad_mask=mask,
                                aux=aux != "off")
    loss = (out.float() * dout).sum()
    if aux != "off":
        n = float(mask.sum()) if mask is not None else float(T)
        loss = loss + 0.5 * E * (counts * psum).sum() / (n * n)
    loss.backward()
    torch.cuda.synchronize()
    assert st.n == {"route": 1, "permute": 1, "gateup": 1, "down": 1, "combine": 1, "combine_bwd": 1, "wgrad": 3,
                    "down_bwd": 1, "gateup_dgrad": 1, "unpermute": 1}, st.n
    # the router's weight gradient dWr = dlogits^T x, returned in bf16
    rc.check(leaves[1].grad, *mc.fp32_gemm(st.dlogits[0].t(), x, BF16), "router dWr = dlogits^T x (expert, element)",
             "router.dWr")
    if aux != "off":
        want = 0.5 * E * st.aux_counts[0] / (n * n)
        rc.check(st.aux_grads[0], want, 8 * rc.U24 * want.abs(), "aux_grad = c E counts / n^2 (expert)")
    else:
        assert st.aux_grads == [None]


def test_model_aux_grad_and_stages(ops, monkeypatch):
    """Through the MoE model (E = 4, k = 2, two layers): every stage of both layers checks, and the aux_grad each
    layer's backward receives is c E counts_total / n^2 with n = unmasked tokens x layers."""
    from tests.test_gpu_moe import _moe_model
    model = _moe_model()
    toks = torch.randint(0, 256, (3, 97), generator=torch.Generator().manual_seed(11))
    toks[0, 70:] = 256                               # padding: masked tokens
    toks[2, :9] = 256
    toks = toks.to(DEV)
    st = _Stages(ops, monkeypatch)
    tmask = toks != 256
    out = model(toks, token_mask=tmask).float()
    coef = 0.01
    (out.square().mean() + coef * model.moe_aux_loss()).backward()
    torch.cuda.synchronize()
    layers, E = model.args.num_hidden_layers, model.args.num_local_experts
    assert len(st.aux_grads) == layers and len(st.aux_counts) == layers
    n = float(tmask.sum()) * layers
    counts = sum(st.aux_counts)
    want = rc.f32(coef) * E * counts / (n * n)
    for i, g in enumerate(st.aux_grads):
        rc.check(g, want, 8 * rc.U24 * want.abs(), f"layer {i} aux_grad = c E counts / n^2 (expert)", "model.aux_grad")


def test_print_worst_ratios():
    """Runs last in this file: the worst |got - ref| / bound per family seen above."""
    for name in sorted(rc.WORST):
        print(f"worst ratio {name}: {rc.WORST[name]:.4f}")
    assert rc.WORST and all(v <= 1.0 for v in rc.WORST.values())
