"""-m gpu: the wgmma engine's epilogue inputs and outputs move by TMA (csrc/gemm_wgmma.cu).  C (beta != 0) and the
saved GLU activations are loaded into the staging tile as 64 x 64 boxes and D / dgu leave it as bulk tensor stores.

Each input here sits inside NaN-filled rows and columns beyond M and the stored width, so a box that read past the
problem would poison an output, and each output sits inside canaries, so a box that wrote past round_up(N, 8) or M
would show.  Results are checked bit for bit in the exact family (tests/gemm_check.py), the GLU adjoint within its
fp64 bound."""
import pytest
import torch

from tests import gemm_check as gc
from tests.gemm_check import Guarded, round_up

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(180)]

BF16 = torch.bfloat16


@pytest.fixture(scope="module")
def L():
    from mlx_cuda_distributed_pretraining_b200 import ops
    ops.require_device()
    return ops.lib()


def _stream():
    return torch.cuda.current_stream().cuda_stream


def _ok(rc, L):
    if rc != 0:
        raise AssertionError(f"rc={rc}: {L.b200_last_error().decode()}")


def _ints(view, gen):
    view.copy_(gc.exact_ints(view.shape, device=view.device, generator=gen).to(view.dtype))


class Case:
    """D = alpha A B^T + beta C (K-major operands) with C and D at a row pitch 72 columns past the stored width and
    NaN rows between batches.  symmetric: A = B = C = one bit-symmetric matrix (Newton-Schulz's B = bA + cAA)."""

    def __init__(self, M, N, K, batch, *, symmetric=False, alpha=0.5, beta=2.0, seed=0):
        gen = torch.Generator(device="cuda").manual_seed(seed)
        self.M, self.N, self.K, self.batch, self.symmetric = M, N, K, batch, symmetric
        self.alpha, self.beta = alpha, beta
        self.n_store = round_up(N, 8)
        ld = self.n_store + 72
        if symmetric:
            assert M == N == K
            self.GA = self.GB = self.GC = Guarded(batch, M, M, BF16, "cuda", ld=ld)
            src = gc.exact_ints((batch, M, M), device="cuda", generator=gen)
            self.GA.view().copy_((torch.triu(src) + torch.triu(src, 1).transpose(1, 2)).to(BF16))
        else:
            self.GA = Guarded(batch, M, K, BF16, "cuda")
            self.GB = Guarded(batch, N, K, BF16, "cuda")
            self.GC = Guarded(batch, M, self.n_store, BF16, "cuda", ld=ld)
            for G in (self.GA, self.GB, self.GC):
                _ints(G.view(), gen)
        self.GD = Guarded(batch, M, N, BF16, "cuda", ld=ld)

    def problem(self):
        from mlx_cuda_distributed_pretraining_b200._lib import GemmProblem
        p = GemmProblem()
        p.a_mn, p.b_mn, p.M, p.N, p.K, p.batch = 0, 0, self.M, self.N, self.K, self.batch
        p.A, p.lda, p.strideA = self.GA.ptr(), self.GA.ld, self.GA.stride
        p.B, p.ldb, p.strideB = self.GB.ptr(), self.GB.ld, self.GB.stride
        p.C, p.ldc, p.strideC = self.GC.ptr(), self.GC.ld, self.GC.stride
        p.D, p.ldd, p.strideD = self.GD.ptr(), self.GD.ld, self.GD.stride
        p.alpha, p.beta, p.alpha_vec, p.beta_vec = self.alpha, self.beta, None, None
        p.symmetric, p.k_splits, p.splitk_ws, p.peer_D, p.n_peers = int(self.symmetric), 1, None, None, 0
        return p

    def launch(self, L):
        return L.b200_gemm_bf16(0, 0, self.M, self.N, self.K, self.batch, self.GA.ptr(), self.GA.ld, self.GA.stride,
                                self.GB.ptr(), self.GB.ld, self.GB.stride, self.GC.ptr(), self.GC.ld, self.GC.stride,
                                self.GD.ptr(), self.GD.ld, self.GD.stride, 0, self.alpha, self.beta, None, None,
                                1256 if self.symmetric else 0, _stream())

    def verify(self, what):
        torch.cuda.synchronize()
        self.GD.check_canaries(self.n_store, what)
        C = self.GC.view(self.n_store)
        R, P = gc.reference(self.GA.view(), self.GB.view(), alpha=self.alpha, beta=self.beta, C=C[..., :self.N])
        gc.check(self.GD.view(), R, P, self.K, True, what)
        if self.n_store > self.N:  # padded columns: alpha * 0 + beta * C
            pad = self.GD.view(self.n_store)[..., self.N:]
            assert torch.equal(pad, (self.beta * C[..., self.N:].double()).to(BF16)), f"{what}: padded columns"


@pytest.mark.parametrize("M,N,K,batch", [(300, 259, 64, 2), (1000, 200, 128, 1), (129, 72, 1000, 3),
                                         (8, 8, 16, 1)])
def test_beta_c_inside_nan_padding(L, M, N, K, batch):
    c = Case(M, N, K, batch, seed=M + N)
    _ok(c.launch(L), L)
    c.verify(f"beta C M={M} N={N} K={K} batch={batch}")


def test_grouped_ns_stage_symmetric_and_tall(L):
    """One grouped launch shaped like a Newton-Schulz stage: a symmetric B = bA + cAA next to a tall X' = aX + XB
    with ragged M, both reading C through the prefetch."""
    sym = Case(384, 384, 384, 2, symmetric=True, alpha=0.25, beta=-2.0, seed=1)
    tall = Case(1000, 256, 256, 1, alpha=0.5, beta=4.0, seed=2)
    from mlx_cuda_distributed_pretraining_b200._lib import GemmProblem
    arr = (GemmProblem * 2)(sym.problem(), tall.problem())
    _ok(L.b200_gemm_grouped(arr, 2, _stream()), L)
    sym.verify("grouped: symmetric")
    tall.verify("grouped: tall")


@pytest.mark.parametrize("M,H,I", [(300, 256, 136), (129, 512, 392), (1, 256, 8)])
def test_glu_bwd_inside_nan_padding(L, M, H, I):
    """dgu from gu stored inside NaN guards before and after (rows beyond M), with I not a multiple of 128, so the
    tile's last column boxes are partly or wholly past I."""
    gen = torch.Generator(device="cuda").manual_seed(M + I)
    G = lambda r, c: Guarded(1, r, c, BF16, "cuda", ld=c, stride=r * c, guard=4 * c)  # noqa: E731
    dy, Wd, gu, dgu = G(M, H), G(H, I), G(M, 2 * I), G(M, 2 * I)
    dy.view().copy_(torch.randn(dy.view().shape, device="cuda", generator=gen).to(BF16))
    Wd.view().copy_((torch.randn(Wd.view().shape, device="cuda", generator=gen) * H ** -0.5).to(BF16))
    gu.view().copy_((torch.randn(gu.view().shape, device="cuda", generator=gen) * 2).to(BF16))
    what = f"down dgrad M={M} H={H} I={I}"
    _ok(L.b200_mlp_down_glu_bwd(dy.ptr(), Wd.ptr(), gu.ptr(), dgu.ptr(), M, H, I, _stream()), L)
    torch.cuda.synchronize()
    dgu.check_canaries(2 * I, what)
    R, P = gc.reference(dy.view(), Wd.view(), b_mn=True)
    g, u = gu.view()[..., :I].double(), gu.view()[..., I:].double()
    s = torch.sigmoid(u)
    ds = s * (1 - s)
    Rdgu = torch.cat([2 * R * s, 2 * R * g * ds], dim=-1)
    Pdgu = torch.cat([2 * P * s, 2 * P * g.abs() * ds], dim=-1)
    extra = torch.cat([2 * R.abs(), 2 * R.abs() * g.abs()], dim=-1) * gc.EPS_SIGMA
    gc.check_bound(dgu.view(), Rdgu, Pdgu, H, what, extra=extra)
