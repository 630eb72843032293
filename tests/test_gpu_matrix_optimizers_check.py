"""-m gpu: the matrix optimizers' GEMM chains element by element against fp64 (tests/ns_check.py).

Newton-Schulz (b200_newton_schulz, _allgather, _multi) is checked stage by stage: every iteration s = 1..5 of every
matrix, on the kernel's own bf16 iterate X_{s-1} and its own A_s, B_s read from the caller's workspace, with inputs at
the front of NaN-filled allocations, a workspace filled with a NaN bit pattern before each run and outputs inside
canaries.  Batches carry distinct norms (scales 1, 3, 1/4, 7), so a matrix scaled by its neighbour's 1/||G|| fails.
The Muon step must equal, bit for bit, the grouped chain run one group at a time plus `p += -lr max(1, r/c)^0.5 X`.

Shampoo's statistics and preconditioning are checked bit for bit in the exact family and within the three-GEMM bound
at C4's size (k = 1024); factor padding must stay +0.0 and every element outside the block must keep its bits.
The worst ratio per family is printed by the last test.
"""
import ctypes

import pytest
import torch

from tests import gemm_check as gc
from tests import ns_check as nc
from tests.gemm_check import Guarded

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(900)]

BF16, F32 = torch.bfloat16, torch.float32
SCALES = (1.0, 3.0, 0.25, 7.0)
WORST = {}   # family -> largest |D - R| / bound


@pytest.fixture(scope="module")
def ops():
    from mlx_cuda_distributed_pretraining_b200 import ops
    ops.require_device()
    return ops


@pytest.fixture(scope="module")
def L(ops):
    return ops.lib()


@pytest.fixture(scope="module")
def S():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _stream():
    return torch.cuda.current_stream().cuda_stream


def _ok(rc, L):
    from mlx_cuda_distributed_pretraining_b200._lib import check
    check(rc, "call")


def _record(family, bounds):
    for b in [bounds] if isinstance(bounds, gc.Bound) else bounds:
        WORST[family] = max(WORST.get(family, 0.0), b.ratio)


def _nan_front(src):
    """src copied into the front of a NaN-filled allocation (a kernel reading past it sees NaN)."""
    n = src.numel()
    buf = torch.full((n + 4096,), float("nan"), device="cuda", dtype=src.dtype)
    buf[:n].copy_(src.reshape(-1))
    return buf[:n].view(src.shape)


def _nan_ws(nbytes):
    """A byte workspace filled with the bf16 NaN canary bit pattern."""
    ws = torch.empty(gc.round_up(max(nbytes, 256), 256), device="cuda", dtype=torch.uint8)
    ws.view(torch.int16).fill_(gc.CANARY[BF16])
    return ws


def _ns_inputs(ops, batch, rows, cols, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    sc = torch.tensor([SCALES[i % len(SCALES)] for i in range(batch)], device="cuda").view(-1, 1, 1)
    x = (torch.randn(batch, rows, cols, device="cuda", generator=g) * 0.02 * sc).to(BF16)
    inv, inv2 = ops.ns_scales(ops.sumsq(x))
    return _nan_front(x), _nan_front(inv), _nan_front(inv2)


def _out(batch, rows, cols):
    return Guarded(batch, rows, cols, BF16, "cuda", ld=cols, stride=rows * cols)


def _stages(ws, sl, prev, out, s, inv, inv2, ops, what):
    """Stage checks of iteration s for one group whose workspace slices are `sl`; also X_tmp == X_{s-1}."""
    batch, rows, cols = prev.shape
    m = min(rows, cols)
    A = nc.ws_view(ws, sl.a, (batch, m, m))
    B = nc.ws_view(ws, sl.b, (batch, m, m))
    if s >= 2:   # the ping-pong buffer holds X_{s-1}: the shorter run's output, bit for bit
        xt = nc.ws_view(ws, sl.xtmp, (batch, rows, cols))
        assert torch.equal(xt.view(torch.int16), prev.view(torch.int16)), f"{what}: X_tmp of run {s} != X_{s - 1}"
    r = nc.check_iteration(prev, A, B, out, s=s, inv_norm=inv, inv_norm_sq=inv2, coeffs=ops.NS_COEFFS, what=what)
    _record("Newton-Schulz G1", r["G1"])
    _record("Newton-Schulz G2", r["G2"])
    _record("Newton-Schulz G3", r["G3"])


# ------------------------------------------------------------------------------------------------------------------
# Newton-Schulz, single chain
# ------------------------------------------------------------------------------------------------------------------
SINGLE = [(2, 256, 512), (2, 512, 256), (1, 384, 384), (3, 256, 640), (3, 640, 256), (1, 136, 72),
          (1, 32003, 1024), (1, 5000, 512), (1, 384, 9000), (1, 2048, 5632)]


@pytest.mark.parametrize("shape", SINGLE, ids=lambda s: "x".join(map(str, s)))
def test_single_chain_every_iteration(ops, L, S, shape):
    """steps = 1..5 (odd and even counts, so x_out and X_tmp swap roles), each iteration's three stages."""
    batch, rows, cols = shape
    a, b, c = ops.NS_COEFFS
    x, inv, inv2 = _ns_inputs(ops, batch, rows, cols, 100 + rows + cols)
    prev = x
    for s in range(1, 6):
        sl = nc.ns_slices([shape], s, S)[0]
        need = ops.ns_workspace_bytes(batch, rows, cols, s)
        assert need == sl.end, f"workspace layout: library {need} bytes, ns_slices {sl.end}"
        ws = _nan_ws(need)
        out = _out(batch, rows, cols)
        _ok(L.b200_newton_schulz(x.data_ptr(), out.ptr(), batch, rows, cols, s, a, b, c, inv.data_ptr(),
                                 inv2.data_ptr(), ws.data_ptr(), ws.numel(), _stream()), L)
        torch.cuda.synchronize()
        out.check_canaries(cols, f"{shape} steps {s}: x_out")
        _stages(ws, sl, prev, out.view(), s, inv, inv2, ops, f"{shape}")
        prev = out.view().clone()
    print(f"{shape}: G1 split-K {sl.splits} on {S} SMs")


# ------------------------------------------------------------------------------------------------------------------
# Newton-Schulz, grouped chain
# ------------------------------------------------------------------------------------------------------------------
def _entry(x_ptr, out_ptr, batch, rows, cols, inv_ptr, inv2_ptr, peers=None):
    from mlx_cuda_distributed_pretraining_b200._lib import NsGroup
    e = NsGroup()
    e.x_in, e.x_out, e.batch, e.rows, e.cols = x_ptr, out_ptr, batch, rows, cols
    e.inv_norm, e.inv_norm_sq = inv_ptr, inv2_ptr
    if peers:
        arr = (ctypes.c_void_p * len(peers))(*peers)
        e.peer_out, e.n_peers = ctypes.cast(arr, ctypes.POINTER(ctypes.c_void_p)), len(peers)
        e._keep = arr
    else:
        e.peer_out, e.n_peers = None, 0
    return e


def _run_multi(ops, L, entries, steps):
    from mlx_cuda_distributed_pretraining_b200._lib import NsGroup
    arr = (NsGroup * len(entries))(*entries)
    need = int(L.b200_newton_schulz_multi_workspace_bytes(arr, len(entries), steps))
    ws = _nan_ws(need)
    a, b, c = ops.NS_COEFFS
    _ok(L.b200_newton_schulz_multi(arr, len(entries), steps, a, b, c, ws.data_ptr(), ws.numel(), _stream()), L)
    torch.cuda.synchronize()
    return ws, need


MULTI = {
    "wide-tall-square-splitk": [(2, 256, 512), (2, 512, 256), (1, 384, 384), (1, 5000, 512)],
    "six-groups": [(1, 256, 256), (2, 256, 384), (1, 384, 256), (4, 256, 512), (1, 640, 256), (1, 1000, 256)],
    "fallback": [(2, 256, 512), (1, 136, 72), (3, 512, 256), (1, 32003, 1024)],
}


@pytest.mark.parametrize("case", list(MULTI))
def test_grouped_chain_every_group_every_iteration(ops, L, S, case):
    shapes = MULTI[case]
    assert nc.grouped_ok(shapes, S) == (case != "fallback")
    ins = [_ns_inputs(ops, *sh, 200 + 7 * i) for i, sh in enumerate(shapes)]
    prev = [x for x, _, _ in ins]
    for s in range(1, 6):
        sl = nc.ns_slices(shapes, s, S)
        outs = [_out(*sh) for sh in shapes]
        entries = [_entry(x.data_ptr(), o.ptr(), *sh, inv.data_ptr(), inv2.data_ptr())
                   for (x, inv, inv2), o, sh in zip(ins, outs, shapes)]
        ws, need = _run_multi(ops, L, entries, s)
        assert need == sl[-1].end, f"workspace layout: library {need} bytes, ns_slices {sl[-1].end}"
        for i, (sh, o, (x, inv, inv2)) in enumerate(zip(shapes, outs, ins)):
            what = f"{case} group {i} {sh}"
            o.check_canaries(sh[2], f"{what} steps {s}: x_out")
            _stages(ws, sl[i], prev[i], o.view(), s, inv, inv2, ops, what)
        prev = [o.view().clone() for o in outs]
    print(f"{case}: {'grouped' if nc.grouped_ok(shapes, S) else 'per-group fallback'}, G1 split-K "
          f"{[q.splits for q in sl]} on {S} SMs")


def _outside_canary(G, owned, what):
    """Every element of Guarded G outside the matrices [lo, hi) of `owned` still holds the canary."""
    rc = G.rows * G.cols
    mask = torch.zeros(G.buf.numel(), dtype=torch.bool, device=G.buf.device)
    for lo, hi in owned:
        mask[G.guard + lo * rc:G.guard + hi * rc] = True
    bad = (G.buf.view(torch.int16) != gc.CANARY[BF16]) & ~mask
    if bool(bad.any()):
        o = int(bad.nonzero()[0]) - G.guard
        raise AssertionError(f"{what}: {int(bad.sum())} elements written outside the owned matrices; first at "
                             f"element {o} (matrix {o // rc})")


def test_owner_ranges_with_peer_stores(ops, L, S):
    """Muon's data-parallel layout on one GPU: entries whose x_in, x_out and inv_norm point at matrix `lo` of a
    larger batch, with peer_out pointing at one or two other buffers that stand in for other ranks."""
    full = [(4, 256, 512), (3, 768, 256)]
    ins = [_ns_inputs(ops, *sh, 300 + i) for i, sh in enumerate(full)]
    # (group, lo, hi, number of peers)
    owned = [(0, 1, 3, 1), (1, 2, 3, 2), (0, 3, 4, 0)]
    prev = {k: ins[g][0][lo:hi] for k, (g, lo, hi, _) in enumerate(owned)}
    for s in range(1, 6):
        outs = [_out(*sh) for sh in full]
        peers = [[_out(*full[g]) for _ in range(n)] for g, _, _, n in owned]
        entries, shapes = [], []
        for (g, lo, hi, n), pl in zip(owned, peers):
            _, rows, cols = full[g]
            x, inv, inv2 = ins[g]
            off = 2 * lo * rows * cols
            entries.append(_entry(x.data_ptr() + off, outs[g].ptr() + off, hi - lo, rows, cols,
                                  inv.data_ptr() + 4 * lo, inv2.data_ptr() + 4 * lo, [p.ptr() + off for p in pl]))
            shapes.append((hi - lo, rows, cols))
        ws, need = _run_multi(ops, L, entries, s)
        sl = nc.ns_slices(shapes, s, S)
        assert need == sl[-1].end
        for k, ((g, lo, hi, n), pl) in enumerate(zip(owned, peers)):
            what = f"owner entry {k} (group {g}, matrices {lo}..{hi - 1})"
            x, inv, inv2 = ins[g]
            got = outs[g].view()[lo:hi]
            _stages(ws, sl[k], prev[k], got, s, inv[lo:hi], inv2[lo:hi], ops, what)
            for j, p in enumerate(pl):
                assert torch.equal(p.view()[lo:hi].view(torch.int16), got.view(torch.int16)), f"{what}: peer {j}"
                _outside_canary(p, [(lo, hi)], f"{what}: peer {j}")
            prev[k] = got.clone()
        for g in range(len(full)):
            _outside_canary(outs[g], [(lo, hi) for gg, lo, hi, _ in owned if gg == g], f"group {g} x_out")


def test_allgather_owner_slice(ops, L, S):
    """b200_newton_schulz_allgather on matrices 1..2 of a batch of 3, storing into two stand-in peer buffers."""
    batch, rows, cols = 3, 384, 640
    lo, hi = 1, 3
    a, b, c = ops.NS_COEFFS
    x, inv, inv2 = _ns_inputs(ops, batch, rows, cols, 400)
    off = 2 * lo * rows * cols
    prev = x[lo:hi]
    for s in range(1, 6):
        sl = nc.ns_slices([(hi - lo, rows, cols)], s, S)[0]
        ws = _nan_ws(sl.end)
        out = _out(batch, rows, cols)
        peers = [_out(batch, rows, cols) for _ in range(2)]
        arr = (ctypes.c_void_p * 2)(*[p.ptr() + off for p in peers])
        _ok(L.b200_newton_schulz_allgather(x.data_ptr() + off, out.ptr() + off, hi - lo, rows, cols, s, a, b, c,
                                           inv.data_ptr() + 4 * lo, inv2.data_ptr() + 4 * lo, ws.data_ptr(),
                                           ws.numel(), arr, 2, _stream()), L)
        torch.cuda.synchronize()
        got = out.view()[lo:hi]
        _outside_canary(out, [(lo, hi)], f"allgather steps {s}: x_out")
        _stages(ws, sl, prev, got, s, inv[lo:hi], inv2[lo:hi], ops, "allgather")
        for j, p in enumerate(peers):
            assert torch.equal(p.view()[lo:hi].view(torch.int16), got.view(torch.int16)), f"steps {s}: peer {j}"
            _outside_canary(p, [(lo, hi)], f"allgather steps {s}: peer {j}")
        prev = got.clone()


# ------------------------------------------------------------------------------------------------------------------
# The Muon step
# ------------------------------------------------------------------------------------------------------------------
# name -> (shape, gradient scale); parameters of one shape form one group, in this order.  Groups 0..5 go through one
# grouped launch, groups 6 and 7 (min(rows, cols) <= 128) through the second launch's per-group fallback.
MUON_PARAMS = {
    "q0": ((256, 384), 1.0), "q1": ((256, 384), 3.0), "q2": ((256, 384), 0.25), "q3": ((256, 384), 7.0),
    "tall": ((768, 256), 1.0),
    "sq": ((256, 256), 2.0),
    "w": ((384, 640), 0.5),
    "down": ((640, 256), 1.0),
    "big": ((512, 1024), 1.0),
    "small": ((64, 128), 1.0),
    "narrow": ((136, 72), 4.0),
}


def test_muon_step_is_the_grouped_chain_and_the_update(ops, L):
    from mlx_cuda_distributed_pretraining_b200.flat import ParamStore
    from mlx_cuda_distributed_pretraining_b200.optimizers.muon import Muon

    gen = torch.Generator().manual_seed(500)

    class Net(torch.nn.Module):
        def __init__(self):
            super().__init__()
            for n, (shape, _) in MUON_PARAMS.items():
                setattr(self, n, torch.nn.Parameter(torch.randn(*shape, generator=gen) * 0.02))

    model = Net().cuda()
    model._b200_store = ParamStore(model, torch.bfloat16)
    store = model._b200_store
    assert store.mixed and len(store.mat_groups) == 7 + 1
    lr = 0.02
    opt = Muon(learning_rate=lr, momentum=0.9, nesterov=True, ns_steps=5)
    a, b, c = ops.NS_COEFFS

    def grads():
        return {n: (torch.randn(*shape, generator=gen) * s).cuda() for n, (shape, s) in MUON_PARAMS.items()}

    opt.update(model, grads())
    p_before = store.master.clone()
    opt.update(model, grads())
    torch.cuda.synchronize()
    for gi, g in enumerate(store.mat_groups):
        what = f"group {gi} {g.batch}x{g.rows}x{g.cols}"
        sl = slice(g.offset, g.offset + g.numel)
        ref = torch.full((g.numel + 4096,), float("nan"), device="cuda", dtype=BF16)
        o = opt._boff[gi]
        e = _entry(opt._u.data_ptr() + 2 * g.offset, ref.data_ptr(), g.batch, g.rows, g.cols,
                   opt._inv.data_ptr() + 4 * o, opt._inv2.data_ptr() + 4 * o)
        _run_multi(ops, L, [e], 5)
        x = opt._x[sl]
        gc.check_finite(x.view(g.batch, g.rows, g.cols), f"{what}: X")
        assert torch.equal(x.view(torch.int16), ref[:g.numel].view(torch.int16)), \
            f"{what}: the step's Newton-Schulz output differs from the same chain run alone"
        # fmaf(s, x, p) in fp32 with s = fp32(-lr max(1, r/c)^0.5): s x is exact in fp64 and the fp64 sum is rounded
        # once more to fp32 (a double rounding would need the sum within 2^-53 of an fp32 midpoint)
        s = torch.tensor(-lr * max(1.0, g.rows / g.cols) ** 0.5, dtype=F32).double()
        exp = (s * x.double() + p_before[sl].double()).float()
        got = store.master[sl]
        if not torch.equal(got, exp):
            i = int((got != exp).nonzero()[0])
            raise AssertionError(f"{what}: master element {i} is {float(got[i])!r}, fmaf gives {float(exp[i])!r}")
        assert torch.equal(store.shadow[sl].view(torch.int16), got.to(BF16).view(torch.int16)), f"{what}: shadow"


# ------------------------------------------------------------------------------------------------------------------
# Shampoo
# ------------------------------------------------------------------------------------------------------------------
def _factor(batch, k, start, exact, gen):
    """[batch, kp, kp] fp32 factor inside canaries: [:k, :k] = start values (or 0), padding +0.0."""
    kp = (k + 7) // 8 * 8
    G = Guarded(batch, kp, kp, F32, "cuda", ld=kp, stride=kp * kp)
    G.view().zero_()
    if start:
        v = gc.exact_ints((batch, k, k), device="cuda", generator=gen) if exact else \
            torch.randn(batch, k, k, device="cuda", generator=gen)
        G.view()[:, :k, :k] = v
    return G


def _grad(batch, rows, ldg, k1, k2, exact, with_lo, gen):
    """hi (and lo) bf16 [batch, rows, ldg] gradients: the [:k1, :k2] block holds the family's values, the rest NaN."""
    hi = torch.full((batch, rows, ldg), float("nan"), device="cuda", dtype=BF16)
    lo = torch.full_like(hi, float("nan")) if with_lo else None
    if exact:
        hi[:, :k1, :k2] = nc.exact_hi((batch, k1, k2), device="cuda", generator=gen)
        if with_lo:
            lo[:, :k1, :k2] = nc.exact_lo((batch, k1, k2), device="cuda", generator=gen)
    else:
        h, l = nc.split(torch.randn(batch, k1, k2, device="cuda", generator=gen))
        hi[:, :k1, :k2] = h
        if with_lo:
            lo[:, :k1, :k2] = l
    return hi, lo


def _stats_case(ops, batch, rows, ldg, k1, k2, exact, with_lo, start, beta2, weight, seed):
    gen = torch.Generator(device="cuda").manual_seed(seed)
    gh, gl = _grad(batch, rows, ldg, k1, k2, exact, with_lo, gen)
    Lf = _factor(batch, k1, start in ("L", "both"), exact, gen)
    Rf = _factor(batch, k2, start in ("R", "both"), exact, gen)
    L0, R0 = Lf.view()[:, :k1, :k1].clone(), Rf.view()[:, :k2, :k2].clone()
    ops.shampoo_stats(gh, gl, ldg, rows * ldg, Lf.view(), Rf.view(), batch, k1, k2, beta2, weight)
    torch.cuda.synchronize()
    (RL, PL), (RR, PR) = nc.stats_reference(gh, gl, L0, R0, k1, k2, beta2, weight)
    tag = f"stats k1={k1} k2={k2} ldg={ldg} lo={with_lo} start={start}"
    out = []
    for F, k, R, P, K, nm in ((Lf, k1, RL, PL, k2, "L"), (Rf, k2, RR, PR, k1, "R")):
        F.check_canaries(F.cols, f"{tag}: {nm}")
        nc.zero_padding_bits(F.view(), k, f"{tag}: {nm}")
        out.append(nc.check3(F.view()[:, :k, :k], R, P, K, exact, f"{tag}: {nm}"))
    return out


@pytest.mark.parametrize("start", ["zero", "L", "R", "both"])
@pytest.mark.parametrize("with_lo", [True, False], ids=["g_lo", "no_g_lo"])
@pytest.mark.parametrize("k1,k2", [(37, 259), (259, 37), (1000, 264), (136, 1000)])
def test_shampoo_stats_exact(ops, k1, k2, with_lo, start):
    """Bit for bit; the block sits inside a wider gradient (ldg > k2, rows > k1) whose other elements are NaN."""
    ldg = (k2 + 7) // 8 * 8 + 16
    _stats_case(ops, 2, k1 + 5, ldg, k1, k2, True, with_lo, start, 0.5, 0.25, 600 + k1 + k2)


@pytest.mark.parametrize("with_lo", [True, False], ids=["g_lo", "no_g_lo"])
def test_shampoo_stats_bound_c4_size(ops, with_lo):
    r = _stats_case(ops, 2, 1024, 2816, 1024, 1024, False, with_lo, "both", 0.95, 0.05, 700)
    _record("Shampoo stats (bound)", r)


def _precond_case(ops, batch, k1, k2, rows, ldo, exact, drop, alpha, seed):
    gen = torch.Generator(device="cuda").manual_seed(seed)
    k1p = (k1 + 7) // 8 * 8
    mk = (lambda s: (nc.exact_hi(s, device="cuda", generator=gen), nc.exact_lo(s, device="cuda", generator=gen))) \
        if exact else (lambda s: nc.split(torch.randn(*s, device="cuda", generator=gen)))
    PL = [torch.full((batch, k1p, k1p), float("nan"), device="cuda", dtype=BF16) for _ in range(2)]
    for t, v in zip(PL, mk((batch, k1, k1))):
        t[:, :k1, :k1] = v
    PRh, PRl = mk((batch, k2, k2))
    ldm = ldo - 8
    m = [torch.full((batch, rows, ldm), float("nan"), device="cuda", dtype=BF16) for _ in range(2)]
    for t, v in zip(m, mk((batch, k1, k2))):
        t[:, :k1, :k2] = v
    PLh, PLl = PL[0], None if drop == "PL_lo" else PL[1]
    PRl = None if drop == "PR_lo" else PRl
    mh, ml = m[0], None if drop == "m_lo" else m[1]
    out = Guarded(batch, rows, ldo, F32, "cuda", ld=ldo, stride=rows * ldo)
    out.view().copy_(torch.randn(batch, rows, ldo, device="cuda", generator=gen))
    before = out.view().clone()
    need = int(ops.lib().b200_shampoo_precond_workspace_bytes(batch, k1, k2))
    ws = _nan_ws(need)
    ops.shampoo_precond(PLh, PLl, PRh, PRl, mh, ml, ldm, rows * ldm, out.view(), ldo, rows * ldo, batch, k1, k2,
                        alpha, workspace=ws)
    torch.cuda.synchronize()
    tag = f"precond k1={k1} k2={k2} ldo={ldo} {'no ' + drop if drop else 'all lo'}"
    out.check_canaries(ldo, tag)
    keep = torch.ones_like(before, dtype=torch.bool)
    keep[:, :k1, :k2] = False
    assert torch.equal(out.view().view(torch.int32)[keep], before.view(torch.int32)[keep]), \
        f"{tag}: pass-through region changed"
    n = batch * k1 * k2
    T = nc.ws_view(ws, 0, (batch, k1, k2), F32)
    Th = nc.ws_view(ws, gc.round_up(n * 4, 256), (batch, k1, k2))
    Tl = nc.ws_view(ws, gc.round_up(n * 4, 256) + gc.round_up(n * 2, 256), (batch, k1, k2))
    R, P = nc.precond_first_reference(PLh, PLl, mh, ml, k1, k2)
    b1 = nc.check3(T, R, P, k1, exact, f"{tag}: T = PL m")
    nc.check_split(T, Th, Tl, tag)
    R, P = nc.precond_second_reference(Th, Tl, PRh, PRl, k2, alpha)
    b2 = nc.check3(out.view()[:, :k1, :k2], R, P, k2, False, f"{tag}: out = alpha T PR")
    return b1, b2


@pytest.mark.parametrize("k1,k2,drop", [(37, 264, None), (259, 136, None), (37, 64, None), (259, 136, "PL_lo"),
                                        (37, 264, "PR_lo"), (259, 136, "m_lo")])
def test_shampoo_precond_exact(ops, k1, k2, drop):
    """T bit for bit, its split bit for bit, out within the bound (tests/test_ns_check.py shows each dropped term
    exceeds it at these shapes); out is wider than k2 and has more rows than k1."""
    _, b2 = _precond_case(ops, 2, k1, k2, k1 + 3, k2 + 24, True, drop, -0.5, 800 + k1 + k2)
    _record("Shampoo precond out (exact-family operands)", b2)


def test_shampoo_precond_bound_c4_size(ops):
    b1, b2 = _precond_case(ops, 2, 1024, 1024, 1024, 2816, False, None, -0.01, 900)
    _record("Shampoo precond T (bound)", b1)
    _record("Shampoo precond out (bound)", b2)


def test_print_worst_ratios():
    for k, v in sorted(WORST.items()):
        print(f"WORST {k}: {v:.4f}")
