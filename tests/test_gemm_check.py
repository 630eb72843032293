"""CPU self-test of tests/gemm_check.py: the checker accepts correct GEMM outputs of both input families and rejects
the outputs that plausible engine bugs would produce.  Without it nothing shows that the GPU conformance tests
(tests/test_gpu_gemm_engine.py) could fail."""
import pytest
import torch

from tests import gemm_check as gc


def _operands(batch, M, N, K, exact, seed, a_mn=False, b_mn=False):
    g = torch.Generator().manual_seed(seed)
    mk = (lambda *s: gc.exact_ints(s, generator=g)) if exact else (lambda *s: torch.randn(*s, generator=g))
    A = mk(batch, K, M) if a_mn else mk(batch, M, K)
    B = mk(batch, K, N) if b_mn else mk(batch, N, K)
    C = mk(batch, M, N)
    return A.bfloat16(), B.bfloat16(), C.bfloat16()


def _engine_like(A, B, C, out_dtype, *, a_mn=False, b_mn=False, alpha=1.0, beta=0.0, av=None, bv=None):
    """What a correct engine produces: fp32 accumulation (a different order from the reference), fp32 epilogue,
    one rounding to the output type."""
    a, b = gc.op(A.float(), a_mn), gc.op(B.float(), b_mn)
    sa = torch.full((a.shape[0], 1, 1), alpha) * (av.view(-1, 1, 1) if av is not None else 1.0)
    D = sa * torch.bmm(a, b.transpose(1, 2))
    if beta != 0.0:
        D = D + torch.full((a.shape[0], 1, 1), beta) * (bv.view(-1, 1, 1) if bv is not None else 1.0) * C.float()
    return D.to(out_dtype)


def _assert_rejects(D, R, P, K, exact):
    with pytest.raises(AssertionError):
        gc.check(D, R, P, K, exact, "planted fault")


FAMILIES = [pytest.param(True, id="exact"), pytest.param(False, id="bound")]
OUTS = [pytest.param(torch.float32, id="f32"), pytest.param(torch.bfloat16, id="bf16")]


@pytest.mark.parametrize("exact", FAMILIES)
@pytest.mark.parametrize("out", OUTS)
@pytest.mark.parametrize("a_mn,b_mn", [(False, False), (True, True)])
def test_checker_accepts_correct_outputs(exact, out, a_mn, b_mn):
    batch, M, N, K = 3, 200, 264, 1000
    A, B, C = _operands(batch, M, N, K, exact, 1, a_mn, b_mn)
    av, bv = torch.tensor([0.5, 2.0, 0.25]), torch.tensor([4.0, 0.5, 1.0])
    kw = dict(a_mn=a_mn, b_mn=b_mn, alpha=2.0, beta=0.25)
    D = _engine_like(A, B, C, out, av=av, bv=bv, **kw)
    R, P = gc.reference(A, B, alpha_vec=av, beta_vec=bv, C=C, **kw)
    ratio, c32 = gc.check(D, R, P, K, exact, "correct output")
    assert 0.0 <= ratio <= 1.0 and 0.0 <= c32 <= gc.C32


@pytest.mark.parametrize("exact", FAMILIES)
@pytest.mark.parametrize("out", OUTS)
def test_checker_rejects_swizzle_chunk_swap(exact, out):
    """One 8-element chunk swapped with its XOR-swizzle neighbour (chunk k <-> k ^ 1 in one row)."""
    A, B, C = _operands(1, 256, 256, 64, exact, 2)
    R, P = gc.reference(A, B)
    D = _engine_like(A, B, C, out)
    r, k = 129, 5   # tile (1, 0)
    lo, hi = 8 * k, 8 * (k ^ 1)
    D[0, r, lo:lo + 8], D[0, r, hi:hi + 8] = D[0, r, hi:hi + 8].clone(), D[0, r, lo:lo + 8].clone()
    _assert_rejects(D, R, P, 64, exact)


@pytest.mark.parametrize("exact", FAMILIES)
def test_checker_rejects_untransposed_mirror_tile(exact):
    """Symmetric output D = X X^T with one off-diagonal tile written untransposed."""
    X, _, _ = _operands(1, 384, 1, 96, exact, 3)
    R, P = gc.reference(X, X)
    D = _engine_like(X, X, X, torch.bfloat16)
    D[0, 256:384, 128:256] = D[0, 128:256, 256:384]       # should be its transpose
    _assert_rejects(D, R, P, 96, exact)


@pytest.mark.parametrize("exact", FAMILIES)
@pytest.mark.parametrize("out", OUTS)
def test_checker_rejects_dropped_last_k_block(exact, out):
    """K = 1000: one tile lost its last k-block, which is only 40 wide (k in [960, 1000))."""
    K = 1000
    A, B, C = _operands(1, 256, 256, K, exact, 4)
    R, P = gc.reference(A, B)
    D = _engine_like(A, B, C, out)
    short = _engine_like(A[..., :960], B[..., :960], C, out)
    D[0, 128:256, 0:128] = short[0, 128:256, 0:128]
    _assert_rejects(D, R, P, K, exact)


@pytest.mark.parametrize("exact", FAMILIES)
@pytest.mark.parametrize("out", OUTS)
def test_checker_rejects_rows_shifted_by_8(exact, out):
    A, B, C = _operands(1, 256, 256, 64, exact, 5)
    R, P = gc.reference(A, B)
    D = _engine_like(A, B, C, out)
    D[0, 128:248, 128:256] = D[0, 136:256, 128:256].clone()
    _assert_rejects(D, R, P, 64, exact)


def test_checker_rejects_round_toward_zero():
    """Exact family: bf16 truncation instead of round-to-nearest-even."""
    A, B, C = _operands(1, 128, 128, 64, True, 6)
    R, P = gc.reference(A, B)
    D = _engine_like(A, B, C, torch.bfloat16)
    gc.check(D, R, P, 64, True)
    bits = R.float().view(torch.int32) & ~0xFFFF                  # drop the low 16 bits: toward zero
    D_rz = (bits >> 16).to(torch.int16).view(torch.bfloat16)
    assert not torch.equal(D_rz, D)
    _assert_rejects(D_rz, R, P, 64, True)


@pytest.mark.parametrize("exact", FAMILIES)
@pytest.mark.parametrize("which", ["alpha_vec", "beta_vec", "C"])
def test_checker_rejects_wrong_batch_epilogue_input(exact, which):
    """alpha_vec, beta_vec or C taken from batch b + 1 for one batch."""
    batch, K = 3, 64
    A, B, C = _operands(batch, 128, 136, K, exact, 7)
    av, bv = torch.tensor([0.5, 2.0, 0.25]), torch.tensor([4.0, 0.5, 1.0])
    kw = dict(alpha=1.0, beta=2.0)
    R, P = gc.reference(A, B, alpha_vec=av, beta_vec=bv, C=C, **kw)
    D = _engine_like(A, B, C, torch.bfloat16, av=av, bv=bv, **kw)
    gc.check(D, R, P, K, exact)
    perm = torch.tensor([1, 1, 2])                                # batch 0 reads batch 1's input
    args = dict(av=av[perm] if which == "alpha_vec" else av, bv=bv[perm] if which == "beta_vec" else bv)
    D_bad = _engine_like(A, B, C[perm] if which == "C" else C, torch.bfloat16, **args, **kw)
    _assert_rejects(D_bad, R, P, K, exact)


@pytest.mark.parametrize("out", OUTS)
def test_guard_rejects_canary_past_n_store(out):
    """A write inside rows < M, cols < round_up(N, 16 bytes) passes; one word past n_store fails."""
    N = 259
    n_store = gc.round_up(N, 16 // torch.tensor([], dtype=out).element_size())
    G = gc.Guarded(2, 100, N, out, "cpu")
    G.view(n_store).fill_(1.0)
    G.check_canaries(n_store)
    G.view(n_store + 1)[1, 50, n_store] = 0.0
    with pytest.raises(AssertionError, match="batch 1, row 50"):
        G.check_canaries(n_store)


def test_guard_rejects_writes_around_the_array():
    G = gc.Guarded(1, 4, 8, torch.bfloat16, "cpu")
    G.view().fill_(0.0)
    G.check_canaries(8)
    G.buf[G.guard - 1] = 0.0
    with pytest.raises(AssertionError, match="before"):
        G.check_canaries(8)
    G2 = gc.Guarded(1, 4, 8, torch.float32, "cpu")
    G2.buf[-1] = 0.0
    with pytest.raises(AssertionError, match="after"):
        G2.check_canaries(8)


def test_checker_names_the_tile_and_chunk():
    A, B, C = _operands(1, 256, 256, 64, True, 8)
    R, P = gc.reference(A, B)
    D = _engine_like(A, B, C, torch.float32)
    D[0, 130, 200] += 1.0
    with pytest.raises(AssertionError, match=r"row 130, col 200\) in tile \(1, 1\), chunk 9"):
        gc.check_exact(D, R)
    D[0, 3, 4] = float("nan")
    with pytest.raises(AssertionError, match="non-finite"):
        gc.check_bound(D, R, P, 64)
