"""-m gpu: conformance of the persistent wgmma GEMM engine (csrc/gemm_wgmma.cu), element by element.

Every mode of the engine -- the four operand layouts, fp32/bf16 output, C / C aliasing D, per-batch alpha/beta
vectors, symmetric output, split-K, grouped launches, peer stores and the two fused MLP epilogues -- is checked with
tests/gemm_check.py against an fp64 reference: bit for bit in the exact (small-integer) family, within a per-element
bound in the Gaussian family.  Each output lives in a canary-filled buffer (row pitch > N, gaps between batches,
guard elements around it) and every operand's padding is NaN, so the tests also show that the engine writes only
rows < M, columns < round_up(N, 16 bytes), and never reads padding.

Shapes that target the persistent schedule are derived from the SM count S: work items in {1, S-1, S, S+1, 2S+1,
~8S}, so CTAs run one to eight tiles, both consumer warpgroups run, and with 2S+1 items they get unequal counts.
"""
import ctypes
import itertools

import pytest
import torch

from tests import gemm_check as gc
from tests.gemm_check import Guarded, round_up

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(180)]

BF16, F32 = torch.bfloat16, torch.float32
NS_A, NS_B, NS_C = 3.4445, -4.7750, 2.0315
RATIOS = {}   # largest |D - R| / bound per bound family, printed at the end of the module


@pytest.fixture(scope="module")
def L():
    from mlx_cuda_distributed_pretraining_b200 import ops
    ops.require_device()
    yield ops.lib()
    if RATIOS:
        print("\nbound family, C32 = %g: largest |D - R| / bound, and the accumulation error in units of K 2^-24 P: "
              "%s" % (gc.C32, "; ".join(f"{k} {r:.3g}, {c:.3g}" for k, (r, c) in sorted(RATIOS.items()))))


@pytest.fixture(scope="module")
def S():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _stream():
    return torch.cuda.current_stream().cuda_stream


def _note(family, b):
    r, c = RATIOS.get(family, (0.0, 0.0))
    RATIOS[family] = (max(r, b.ratio), max(c, b.c32))


def _fill(view, exact):
    src = gc.exact_ints(view.shape, device=view.device) if exact else torch.randn(view.shape, device=view.device)
    view.copy_(src.to(view.dtype))


def _sym_fill(view, exact):
    """A bit-symmetric [batch, m, m] matrix."""
    src = gc.exact_ints(view.shape, device=view.device) if exact else torch.randn(view.shape, device=view.device)
    t = torch.triu(src)
    view.copy_((t + torch.triu(src, 1).transpose(1, 2)).to(view.dtype))


def _bits(t):
    return t.view(torch.int16 if t.dtype == BF16 else torch.int32).clone()


def _raises(rc, L):
    from mlx_cuda_distributed_pretraining_b200._lib import B200Error, check
    with pytest.raises(B200Error):
        check(rc, "expected rejection")


class Prob:
    """One engine problem on guarded buffers: operands with NaN padding, D (and peers) inside canaries, fp64 R/P.

    form: "plain" (A [M,K], B [N,K] or their MN-major transposes), "xxt" (A = B = X: D = X X^T, or X^T X when
    a_mn = b_mn = True), "g2" (A = B = C = a symmetric matrix: D = beta A + alpha A A, Newton-Schulz's G2)."""

    def __init__(self, M, N, K, batch, *, a_mn=False, b_mn=False, out_f32=False, cmode="none", vec=False,
                 exact=True, form="plain", symmetric=False, splits=1, n_peers=0, ld_extra=8, seed=0):
        torch.manual_seed(seed)
        dev = "cuda"
        self.M, self.N, self.K, self.batch = M, N, K, batch
        self.a_mn, self.b_mn, self.out_f32, self.exact = a_mn, b_mn, out_f32, exact
        self.symmetric, self.splits, self.cmode = symmetric, splits, cmode
        self.odt = F32 if out_f32 else BF16
        self.n_store = round_up(N, 4 if out_f32 else 8)
        ldd = round_up(self.n_store + ld_extra, 8)
        if form == "plain":
            self.GA = Guarded(batch, K if a_mn else M, M if a_mn else K, BF16, dev)
            self.GB = Guarded(batch, K if b_mn else N, N if b_mn else K, BF16, dev)
            _fill(self.GA.view(), exact)
            _fill(self.GB.view(), exact)
        elif form == "xxt":
            self.GA = self.GB = Guarded(batch, K if a_mn else M, M if a_mn else K, BF16, dev)
            _fill(self.GA.view(), exact)
        else:  # g2
            assert M == N == K
            self.GA = self.GB = Guarded(batch, M, M, BF16, dev)
            _sym_fill(self.GA.view(), exact)
            cmode = self.cmode = "A"
        self.GD = Guarded(batch, M, N, self.odt, dev, ld=ldd)
        self.alpha, self.beta = (2.0, 0.25) if vec else (0.5, 2.0)
        if form == "g2" and not exact:
            self.alpha, self.beta = NS_C, NS_B
        self.av = torch.tensor([0.5, 2.0, 0.25, 1.0] * batch, device=dev)[:batch] if vec else None
        self.bv = torch.tensor([4.0, 0.5, 1.0, 0.25] * batch, device=dev)[:batch] if vec else None
        self.Cvals, self.C_ptr, self.ldc, self.strideC = None, None, 0, 0
        if cmode == "none":
            self.beta = 0.0
        elif cmode == "c":
            self.GC = Guarded(batch, M, self.n_store, self.odt, dev)
            _fill(self.GC.view(), exact)
            self.Cvals = self.GC.view().clone()
            self.C_ptr, self.ldc, self.strideC = self.GC.ptr(), self.GC.ld, self.GC.stride
        elif cmode == "alias":   # C aliases D: the in-place accumulate of the bf16x3 Shampoo products
            _fill(self.GD.view(self.n_store), exact)
            self.Cvals = self.GD.view(self.n_store).clone()
            self.C_ptr, self.ldc, self.strideC = self.GD.ptr(), self.GD.ld, self.GD.stride
        else:  # "A": C is the A operand (g2)
            self.Cvals = self.GA.view().clone()
            self.C_ptr, self.ldc, self.strideC = self.GA.ptr(), self.GA.ld, self.GA.stride
        self.ws = torch.empty(splits * batch * M * N, device=dev, dtype=F32) if splits > 1 else None
        self.peers = [Guarded(batch, M, N, BF16, dev, ld=ldd, stride=self.GD.stride) for _ in range(n_peers)]
        self._peer_arr = (ctypes.c_void_p * max(n_peers, 1))(*[p.ptr() for p in self.peers])
        self.items = None

    def work_items(self):
        tm, tn = -(-self.M // 128), -(-self.N // 128)
        tiles = tm * (tm + 1) // 2 if self.symmetric else tm * tn
        return tiles * self.batch * self.splits

    def launch_plain(self, L, force_bn=0):
        """Through b200_gemm_bf16 (force_bn = 1256: symmetric output)."""
        return L.b200_gemm_bf16(int(self.a_mn), int(self.b_mn), self.M, self.N, self.K, self.batch, self.GA.ptr(),
                                self.GA.ld, self.GA.stride, self.GB.ptr(), self.GB.ld, self.GB.stride, self.C_ptr,
                                self.ldc, self.strideC, self.GD.ptr(), self.GD.ld, self.GD.stride, int(self.out_f32),
                                self.alpha, self.beta, _ptr(self.av), _ptr(self.bv), force_bn, _stream())

    def problem(self):
        from mlx_cuda_distributed_pretraining_b200._lib import GemmProblem
        assert not self.out_f32
        p = GemmProblem()
        p.a_mn, p.b_mn, p.M, p.N, p.K, p.batch = int(self.a_mn), int(self.b_mn), self.M, self.N, self.K, self.batch
        p.A, p.lda, p.strideA = self.GA.ptr(), self.GA.ld, self.GA.stride
        p.B, p.ldb, p.strideB = self.GB.ptr(), self.GB.ld, self.GB.stride
        p.C, p.ldc, p.strideC = self.C_ptr, self.ldc, self.strideC
        p.D, p.ldd, p.strideD = self.GD.ptr(), self.GD.ld, self.GD.stride
        p.alpha, p.beta, p.alpha_vec, p.beta_vec = self.alpha, self.beta, _ptr(self.av), _ptr(self.bv)
        p.symmetric, p.k_splits, p.splitk_ws = int(self.symmetric), self.splits, _ptr(self.ws)
        p.peer_D = ctypes.cast(self._peer_arr, ctypes.POINTER(ctypes.c_void_p)) if self.peers else None
        p.n_peers = len(self.peers)
        return p

    def reset(self):
        """Canaries back into D and the peers (and C back into D when it aliases)."""
        for G in [self.GD] + self.peers:
            G.buf.view(torch.int16 if G.dtype == BF16 else torch.int32).fill_(gc.CANARY[G.dtype])
        if self.cmode == "alias":
            self.GD.view(self.n_store).copy_(self.Cvals)

    def verify(self, what):
        """Canaries, the padded columns, the checker, the peer copies; returns the bound ratio."""
        torch.cuda.synchronize()
        self.GD.check_canaries(self.n_store, what)
        c = self.Cvals
        R, P = gc.reference(self.GA.view(), self.GB.view(), a_mn=self.a_mn, b_mn=self.b_mn, alpha=self.alpha,
                            beta=self.beta, alpha_vec=self.av, beta_vec=self.bv,
                            C=None if c is None else c[..., :self.N])
        if self.n_store > self.N:  # padded columns: alpha * 0 + beta * C (exact: powers of two)
            pad = self.GD.view(self.n_store)[..., self.N:]
            exp = torch.zeros_like(pad) if c is None else (
                gc._scale(self.beta, self.bv, self.batch, c.device) * c[..., self.N:].double()).to(self.odt)
            assert torch.equal(pad, exp), f"{what}: padded columns are not beta * C"
        D = self.GD.view()
        bound = gc.check(D, R, P, self.K, self.exact, what)
        if not self.exact:
            _note(("fp32 out" if self.out_f32 else "bf16 out"), bound)
        for i, G in enumerate(self.peers):
            G.check_canaries(self.n_store, f"{what}: peer {i}")
            assert torch.equal(G.view(), D), f"{what}: peer {i} differs from D"


def _ptr(t):
    return None if t is None else t.data_ptr()


def _grouped(L, probs):
    from mlx_cuda_distributed_pretraining_b200._lib import GemmProblem
    arr = (GemmProblem * len(probs))(*[p.problem() if isinstance(p, Prob) else p for p in probs])
    return L.b200_gemm_grouped(arr, len(probs), _stream())


def _ok(rc, L):
    if rc != 0:
        raise AssertionError(f"rc={rc}: {L.b200_last_error().decode()}")


# ------------------------------------------------------------------------------------------------------------
# plain engine through b200_gemm_bf16
# ------------------------------------------------------------------------------------------------------------
def _shapes(S):
    """(M, N, K, batch, ld_extra, label); work items = ceil(M/128) ceil(N/128) batch."""
    return [
        (100, 120, 8, 1, 8, "1 item"),
        (128 * (S - 2) + 1, 72, 40, 1, 8, "S-1 items, M%128=1"),
        (128 * (S - 1) + 8, 64, 64, 1, 8, "S items, M%128=8"),
        (128 * S + 127, 128, 64, 1, 8, "S+1 items, M%128=127"),
        (128 * 2 * S + 5, 48, 1000, 1, 8, "2S+1 items: consumer 1 of CTA 0 gets one item fewer"),
        (1024, 128 * (S // 3), 4096, 3, 8, "~8S items, batch 3"),
        (259, 259, 64, 1, 0, "N%8 != 0, ldd = round_up(N, 8) (Shampoo's 259 -> 264)"),
        (8, 8, 8, 1, 8, "one 8x8 corner"),
    ]


LAYOUTS = [(False, False), (False, True), (True, False), (True, True)]
MODES = list(itertools.product(LAYOUTS, (False, True), ("none", "c", "alias"), (False, True)))   # 48 combinations


@pytest.mark.parametrize("i", range(len(MODES)))
def test_plain_engine_exact(L, S, i):
    """Every layout x output type x C mode x scalar/vector combination, with the shape list cycled under it."""
    (a_mn, b_mn), out_f32, cmode, vec = MODES[i]
    M, N, K, batch, ld_extra, label = _shapes(S)[i % len(_shapes(S))]
    p = Prob(M, N, K, batch, a_mn=a_mn, b_mn=b_mn, out_f32=out_f32, cmode=cmode, vec=vec, ld_extra=ld_extra,
             seed=i)
    what = f"{label}: M={M} N={N} K={K} b={batch} a_mn={a_mn} b_mn={b_mn} f32={out_f32} C={cmode} vec={vec}"
    _ok(p.launch_plain(L), L)
    p.verify(what)
    first = _bits(p.GD.buf)
    p.reset()
    _ok(p.launch_plain(L), L)
    torch.cuda.synchronize()
    assert torch.equal(_bits(p.GD.buf), first), f"{what}: a repeated launch changed the result"


@pytest.mark.parametrize("a_mn,b_mn", LAYOUTS)
@pytest.mark.parametrize("out_f32", [False, True])
def test_plain_engine_bound(L, S, a_mn, b_mn, out_f32):
    """Gaussian operands at the largest K and ~8S work items, every layout and output type."""
    M, N, K, batch, _, label = _shapes(S)[5]
    p = Prob(M, N, K, batch, a_mn=a_mn, b_mn=b_mn, out_f32=out_f32, cmode="c", vec=True, exact=False,
             seed=100 + 2 * a_mn + b_mn)
    _ok(p.launch_plain(L), L)
    p.verify(f"{label}: a_mn={a_mn} b_mn={b_mn} f32={out_f32}")


def test_plain_engine_bound_ragged(L):
    p = Prob(259, 259, 1000, 2, out_f32=False, cmode="alias", vec=True, exact=False, ld_extra=0, seed=7)
    _ok(p.launch_plain(L), L)
    p.verify("259 x 259, C aliasing D, bound family")


# ------------------------------------------------------------------------------------------------------------
# symmetric output
# ------------------------------------------------------------------------------------------------------------
def _upper_tiles(m, device):
    t = torch.arange(m, device=device) // 128
    return t[:, None] <= t[None, :]


@pytest.mark.parametrize("m,K", [(200, 64), (1000, 1000), (2048, 512)])
@pytest.mark.parametrize("form", ["xxt", "g2"])
@pytest.mark.parametrize("exact", [True, False])
def test_symmetric_output(L, S, m, K, form, exact):
    tiles = -(-m // 128)
    batch = 2 * S // (tiles * (tiles + 1) // 2) + 1   # upper-triangle work items > 2S
    kw = dict(form=form, exact=exact, vec=(form == "xxt"), seed=m + K)
    K = m if form == "g2" else K
    sym = Prob(m, m, K, batch, symmetric=True, **kw)
    assert sym.work_items() > 2 * S
    what = f"symmetric {form} m={m} K={K} batch={batch} ({sym.work_items()} items, S={S})"
    _ok(sym.launch_plain(L, force_bn=1256), L)
    sym.verify(what)
    D = sym.GD.view()
    assert torch.equal(D, D.transpose(1, 2)), f"{what}: D is not bit-symmetric"
    full = Prob(m, m, K, batch, **kw)   # same seed: same operands
    _ok(full.launch_plain(L, force_bn=0), L)
    torch.cuda.synchronize()
    up = _upper_tiles(m, D.device).expand_as(D)
    assert torch.equal(D[up], full.GD.view()[up]), f"{what}: upper tiles differ from the non-symmetric launch"
    # the same through the grouped entry
    sym.reset()
    _ok(_grouped(L, [sym]), L)
    sym.verify(what + " (grouped entry)")
    assert torch.equal(sym.GD.view(), D)


def test_symmetric_rejects_ragged_n(L):
    """Symmetric output needs M == N % 8 == 0: that is what lets the mirror store whole 8-row pieces."""
    p = Prob(260, 260, 64, 1, ld_extra=8)
    rc = p.launch_plain(L, force_bn=1256)
    _raises(rc, L)
    q = Prob(260, 260, 64, 1, form="xxt", symmetric=True)
    _raises(_grouped(L, [q]), L)


# ------------------------------------------------------------------------------------------------------------
# split-K (grouped entry)
# ------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("splits", [2, 3, 4, 7])
@pytest.mark.parametrize("exact", [True, False])
def test_split_k_plain(L, splits, exact):
    """K = 576 is 9 k-blocks: 4 splits of 3 leave the last one empty, 7 splits of 2 leave the last two empty."""
    p = Prob(384, 512, 576, 2, b_mn=True, vec=True, splits=splits, exact=exact, seed=splits)
    what = f"split-K {splits}: {p.work_items()} items"
    _ok(_grouped(L, [p]), L)
    p.verify(what)
    first = _bits(p.GD.buf)
    p.reset()
    _ok(_grouped(L, [p]), L)
    torch.cuda.synchronize()
    assert torch.equal(_bits(p.GD.buf), first), f"{what}: the split-K finalize is not deterministic"


@pytest.mark.parametrize("exact", [True, False])
def test_split_k_symmetric(L, exact):
    p = Prob(768, 768, 1000, 2, form="xxt", a_mn=True, b_mn=True, vec=True, symmetric=True, splits=3, exact=exact,
             seed=11)
    what = f"symmetric split-K 3: {p.work_items()} items"
    _ok(_grouped(L, [p]), L)
    p.verify(what)
    D = p.GD.view()
    assert torch.equal(D, D.transpose(1, 2)), f"{what}: D is not bit-symmetric"
    first = _bits(p.GD.buf)
    p.reset()
    _ok(_grouped(L, [p]), L)
    torch.cuda.synchronize()
    assert torch.equal(_bits(p.GD.buf), first), f"{what}: not deterministic"


def test_split_k_with_beta_falls_back_to_one_split(L):
    p = Prob(384, 512, 576, 2, cmode="c", vec=True, splits=3, seed=12)
    _ok(_grouped(L, [p]), L)
    p.verify("split-K requested with beta != 0")


# ------------------------------------------------------------------------------------------------------------
# grouped launches and peer stores
# ------------------------------------------------------------------------------------------------------------
def _mix():
    """Six problems: K in {64, 1000, 4096} (the heaviest-K-first reorder permutes them), every layout, batch,
    symmetric, split-K and a peer problem."""
    return [
        Prob(300, 264, 64, 2, b_mn=True, seed=21),
        Prob(512, 384, 4096, 1, a_mn=True, cmode="c", vec=True, seed=22),
        Prob(640, 640, 1000, 3, form="xxt", vec=True, symmetric=True, seed=23),
        Prob(256, 512, 4096, 1, a_mn=True, b_mn=True, splits=3, vec=True, seed=24),
        Prob(200, 136, 1000, 2, n_peers=2, cmode="c", seed=25),
        Prob(1000, 72, 1000, 1, a_mn=True, b_mn=True, seed=26),
    ]


@pytest.mark.parametrize("n", [2, 4, 6])
def test_grouped_matches_lone_launches(L, S, n):
    """Each problem of a grouped launch is bit-identical to the same problem launched alone, although its tiles land
    on other CTAs and warpgroups (DESIGN 4.1: results do not depend on the schedule)."""
    probs = _mix()[6 - n:] if n < 6 else _mix()
    total = sum(p.work_items() for p in probs)
    _ok(_grouped(L, probs), L)
    torch.cuda.synchronize()
    together = [_bits(p.GD.buf) for p in probs]
    for i, p in enumerate(probs):
        p.verify(f"grouped problem {i} of {n} ({total} items, S={S})")
    for p in probs:
        p.reset()
    _ok(_grouped(L, probs), L)
    torch.cuda.synchronize()
    for i, p in enumerate(probs):
        assert torch.equal(_bits(p.GD.buf), together[i]), f"problem {i}: repeated grouped launch differs"
    for i, p in enumerate(probs):
        p.reset()
        _ok(_grouped(L, [p]), L)
        torch.cuda.synchronize()
        assert torch.equal(_bits(p.GD.buf), together[i]), f"problem {i}: grouped result differs from a lone launch"


def test_grouped_rejects_bad_arguments(L):
    probs = _mix()
    _raises(_grouped(L, probs + [Prob(128, 128, 64, 1)]), L)                 # 7 problems
    p = Prob(128, 128, 64, 1, n_peers=7)
    _ok(_grouped(L, [p]), L)
    p.verify("7 peers")
    bad = p.problem()
    bad.n_peers = 8
    _raises(_grouped(L, [bad]), L)
    sym = Prob(256, 256, 64, 1, form="xxt", symmetric=True, n_peers=1)
    _raises(_grouped(L, [sym]), L)                                           # peers + symmetric
    spl = Prob(256, 256, 1024, 1, splits=2, n_peers=1)
    _raises(_grouped(L, [spl]), L)                                           # peers + split-K
    q = Prob(256, 256, 1024, 1, splits=2)
    bad = q.problem()
    bad.splitk_ws = None
    _raises(_grouped(L, [bad]), L)                                           # split-K without a workspace
    bad = q.problem()
    bad.D = bad.D + 2
    _raises(_grouped(L, [bad]), L)                                           # misaligned D
    bad = q.problem()
    bad.ldd = 248
    _raises(_grouped(L, [bad]), L)                                           # ldd < N
    bad = q.problem()
    bad.strideD = q.GD.stride + 4
    _raises(_grouped(L, [bad]), L)                                           # batch stride breaks alignment


@pytest.mark.parametrize("n_peers", [1, 7])
def test_grouped_peer_stores(L, n_peers):
    p = Prob(300, 264, 1000, 2, cmode="c", vec=True, n_peers=n_peers, seed=30 + n_peers)
    _ok(_grouped(L, [p]), L)
    p.verify(f"{n_peers} peers")


def _ns_inputs(batch, rows, cols, seed):
    from mlx_cuda_distributed_pretraining_b200 import ops
    torch.manual_seed(seed)
    x = (torch.randn(batch, rows, cols, device="cuda") * 0.02).to(BF16)
    inv, inv2 = ops.ns_scales(ops.sumsq(x))
    return x, inv, inv2


def test_newton_schulz_allgather_peers(L):
    from mlx_cuda_distributed_pretraining_b200 import ops
    batch, rows, cols = 2, 384, 640
    x, inv, inv2 = _ns_inputs(batch, rows, cols, 40)
    ref = ops.zeropower_via_newtonschulz5(x, 5)   # the same chain without peers
    out = Guarded(batch, rows, cols, BF16, "cuda", ld=cols, stride=rows * cols)
    peers = [Guarded(batch, rows, cols, BF16, "cuda", ld=cols, stride=rows * cols) for _ in range(3)]
    arr = (ctypes.c_void_p * 3)(*[p.ptr() for p in peers])
    ws = torch.empty(ops.ns_workspace_bytes(batch, rows, cols, 5), device="cuda", dtype=torch.uint8)
    _ok(L.b200_newton_schulz_allgather(x.data_ptr(), out.ptr(), batch, rows, cols, 5, NS_A, NS_B, NS_C,
                                       inv.data_ptr(), inv2.data_ptr(), ws.data_ptr(), ws.numel(), arr, 3,
                                       _stream()), L)
    torch.cuda.synchronize()
    out.check_canaries(cols, "x_out")
    assert torch.equal(out.view(), ref)
    for i, p in enumerate(peers):
        p.check_canaries(cols, f"peer {i}")
        assert torch.equal(p.view(), out.view()), f"peer {i}"


def test_newton_schulz_multi_peers(L):
    from mlx_cuda_distributed_pretraining_b200 import ops
    from mlx_cuda_distributed_pretraining_b200._lib import NsGroup
    shapes = [(2, 256, 512), (1, 768, 256)]
    groups, keep = (NsGroup * 2)(), []
    for i, (b, r, c) in enumerate(shapes):
        x, inv, inv2 = _ns_inputs(b, r, c, 41 + i)
        out = Guarded(b, r, c, BF16, "cuda", ld=c, stride=r * c)
        peers = [Guarded(b, r, c, BF16, "cuda", ld=c, stride=r * c) for _ in range(2 + i)]
        arr = (ctypes.c_void_p * len(peers))(*[p.ptr() for p in peers])
        keep.append((x, inv, inv2, out, peers, arr))
        g = groups[i]
        g.x_in, g.x_out, g.batch, g.rows, g.cols = x.data_ptr(), out.ptr(), b, r, c
        g.inv_norm, g.inv_norm_sq = inv.data_ptr(), inv2.data_ptr()
        g.peer_out, g.n_peers = ctypes.cast(arr, ctypes.POINTER(ctypes.c_void_p)), len(peers)
    need = int(L.b200_newton_schulz_multi_workspace_bytes(groups, 2, 5))
    ws = torch.empty(need, device="cuda", dtype=torch.uint8)
    _ok(L.b200_newton_schulz_multi(groups, 2, 5, NS_A, NS_B, NS_C, ws.data_ptr(), need, _stream()), L)
    torch.cuda.synchronize()
    outs = ops.zeropower_groups([k[0] for k in keep])
    for (x, _, _, out, peers, _), ref, (b, r, c) in zip(keep, outs, shapes):
        out.check_canaries(c, "x_out")
        assert torch.equal(out.view(), ref)
        for j, p in enumerate(peers):
            p.check_canaries(c, f"peer {j}")
            assert torch.equal(p.view(), out.view()), f"peer {j}"


# ------------------------------------------------------------------------------------------------------------
# fused MLP epilogues
# ------------------------------------------------------------------------------------------------------------
def _guarded_2d(rows, cols, dtype, fill=None):
    """[rows, cols] contiguous inside canaries, with four rows' worth of guard after (rows beyond M)."""
    G = Guarded(1, rows, cols, dtype, "cuda", ld=cols, stride=rows * cols, guard=4 * cols)
    if fill is not None:
        fill(G.view())
    return G


@pytest.mark.parametrize("M,K,I", [(1, 256, 256), (129, 512, 384), (300, 1024, 256),
                                   (16384, 1024, 2816), (4096, 2048, 5632)])
@pytest.mark.parametrize("exact", [True, False])
def test_mlp_gateup_glu_fwd(L, M, K, I, exact):
    def fill_w(v):   # bound family: u ~ N(0, 1), so the sigmoid is not saturated
        _fill(v, exact)
        if not exact:
            v.mul_(K ** -0.5)

    x = _guarded_2d(M, K, BF16, lambda v: _fill(v, exact))
    W2 = _guarded_2d(2 * I, K, BF16, fill_w)
    gu = _guarded_2d(M, 2 * I, BF16)
    y = _guarded_2d(M, I, BF16)
    what = f"gate/up M={M} K={K} I={I} ({-(-M // 128) * I // 64} items)"
    args = (x.ptr(), W2.ptr(), gu.ptr(), y.ptr(), M, K, I, _stream())
    _ok(L.b200_mlp_gateup_glu_fwd(*args), L)
    torch.cuda.synchronize()
    gu.check_canaries(2 * I, what + ": gu")
    y.check_canaries(I, what + ": y")
    R, P = gc.reference(x.view(), W2.view())
    bound = gc.check(gu.view(), R, P, K, exact, what + ": gu")
    if not exact:
        _note("bf16 out", bound)
        g, u, Pg, Pu = R[..., :I], R[..., I:], P[..., :I], P[..., I:]
        s = torch.sigmoid(u)
        Ry = 2 * g * s
        # g and u come from the fp32 accumulators; sigmoid's slope is at most 1/4
        Py = 2 * (Pg * s + g.abs() * Pu / 4)
        _note("glu y", gc.check_bound(y.view(), Ry, Py, K, what + ": y", extra=2 * g.abs() * gc.EPS_SIGMA))
    first = (_bits(gu.buf), _bits(y.buf))
    _ok(L.b200_mlp_gateup_glu_fwd(*args), L)
    torch.cuda.synchronize()
    assert torch.equal(_bits(gu.buf), first[0]) and torch.equal(_bits(y.buf), first[1]), what + ": not deterministic"


@pytest.mark.parametrize("M,H,I", [(1, 256, 136), (129, 512, 136), (300, 256, 384),
                                   (16384, 1024, 2816), (4096, 2048, 5632)])
def test_mlp_down_glu_bwd(L, M, H, I):
    """dgu against fp64 on the stored bf16 gu, as the kernel reads it."""
    dy = _guarded_2d(M, H, BF16, lambda v: _fill(v, False))
    Wd = _guarded_2d(H, I, BF16, lambda v: v.copy_((torch.randn(v.shape, device="cuda") * H ** -0.5).to(BF16)))
    gu = _guarded_2d(M, 2 * I, BF16, lambda v: v.copy_((torch.randn(v.shape, device="cuda") * 2).to(BF16)))
    dgu = _guarded_2d(M, 2 * I, BF16)
    what = f"down dgrad M={M} H={H} I={I} ({-(-M // 128) * -(-I // 128)} items)"
    args = (dy.ptr(), Wd.ptr(), gu.ptr(), dgu.ptr(), M, H, I, _stream())
    _ok(L.b200_mlp_down_glu_bwd(*args), L)
    torch.cuda.synchronize()
    dgu.check_canaries(2 * I, what)
    R, P = gc.reference(dy.view(), Wd.view(), b_mn=True)   # d = dy Wd, Wd stored [K = H, N = I]
    g, u = gu.view()[..., :I].double(), gu.view()[..., I:].double()
    s = torch.sigmoid(u)
    ds = s * (1 - s)
    Rdgu = torch.cat([2 * R * s, 2 * R * g * ds], dim=-1)
    Pdgu = torch.cat([2 * P * s, 2 * P * g.abs() * ds], dim=-1)
    extra = torch.cat([2 * R.abs(), 2 * R.abs() * g.abs()], dim=-1) * gc.EPS_SIGMA
    _note("glu dgu", gc.check_bound(dgu.view(), Rdgu, Pdgu, H, what, extra=extra))
    first = _bits(dgu.buf)
    _ok(L.b200_mlp_down_glu_bwd(*args), L)
    torch.cuda.synchronize()
    assert torch.equal(_bits(dgu.buf), first), what + ": not deterministic"


# ------------------------------------------------------------------------------------------------------------
# Newton-Schulz, stage by stage, on the kernel's own intermediates
# ------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("shape", [(2, 256, 512), (2, 512, 256), (1, 384, 384), (1, 5000, 512), (1, 32003, 1024)])
@pytest.mark.parametrize("steps", [1, 2])
def test_newton_schulz_stages(L, shape, steps):
    """Workspace layout (newton_schulz.cu): A at 0, B at align256(batch m m 2), X_tmp after it.  After steps = 1 the
    workspace holds iteration 1 (alpha/beta vectors 1/||X||, 1/||X||^2); after steps = 2, iteration 2 (no vectors),
    whose input X_1 is in X_tmp.  Each stage is checked against fp64 on the kernel's own inputs to that stage."""
    from mlx_cuda_distributed_pretraining_b200 import ops
    batch, rows, cols = shape
    tall = rows > cols
    m = min(rows, cols)
    x, inv, inv2 = _ns_inputs(batch, rows, cols, 50 + rows)
    out = torch.empty_like(x)
    ws = torch.zeros(ops.ns_workspace_bytes(batch, rows, cols, steps), device="cuda", dtype=torch.uint8)
    ops.newton_schulz_raw(x, out, inv, inv2, ws, steps)
    torch.cuda.synchronize()
    mm = batch * m * m * 2
    off_b = (mm + 255) // 256 * 256
    A = ws[:mm].view(BF16).view(batch, m, m)
    B = ws[off_b:off_b + mm].view(BF16).view(batch, m, m)
    if steps == 1:
        X, s1, s2 = x, inv, inv2
    else:
        X = ws[2 * off_b:2 * off_b + batch * rows * cols * 2].view(BF16).view(batch, rows, cols)
        s1 = s2 = None
    tag = f"{shape} iteration {steps}"
    R, P = gc.reference(X, X, a_mn=tall, b_mn=tall, alpha_vec=s2)
    _note("ns stage", gc.check_bound(A, R, P, max(rows, cols), tag + ": A = X X^T"))
    R, P = gc.reference(A, A, alpha=NS_C, beta=NS_B, C=A)
    _note("ns stage", gc.check_bound(B, R, P, m, tag + ": B = bA + cAA"))
    if tall:
        R, P = gc.reference(X, B, alpha_vec=s1, beta=NS_A, beta_vec=s1, C=X)
    else:
        R, P = gc.reference(B, X, b_mn=True, alpha_vec=s1, beta=NS_A, beta_vec=s1, C=X)
    _note("ns stage", gc.check_bound(out, R, P, m, tag + ": X' = aX + BX"))
