"""CPU self-test of tests/ns_check.py: the stage checker accepts an emulation of the Newton-Schulz driver and of
Shampoo's bf16x3 chains, and rejects the outputs that plausible driver faults would produce.  Without it nothing
shows that tests/test_gpu_matrix_optimizers_check.py could fail.

The Newton-Schulz emulation does what csrc/newton_schulz.cu asks of the engine: fp32-accumulated products, the
epilogue alpha*av*acc + beta*bv*C in fp32, one rounding to bf16, and the symmetric outputs mirrored from the upper
triangle.  Its inputs give each matrix of a batch a clearly different norm (scales 1, 3, 1/4, 7): with equal norms a
matrix that reads its neighbour's 1/||G|| would be invisible."""
import pytest
import torch

from mlx_cuda_distributed_pretraining_b200.ops import NS_COEFFS as COEFFS, NS_EPS as EPS
from tests import gemm_check as gc
from tests import ns_check as nc

SCALES = (1.0, 3.0, 0.25, 7.0)
STEPS = 5


def _inputs(rows, cols, seed):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(len(SCALES), rows, cols, generator=g) * 0.02 * torch.tensor(SCALES).view(-1, 1, 1)
    x = x.bfloat16()
    inv = 1.0 / (x.float().pow(2).sum((1, 2)).sqrt() + EPS)
    return x, inv, inv * inv


def _bf16(D):
    return D.to(torch.bfloat16)


def _mirror(A):
    """The engine computes tiles on and above the diagonal and copies them below."""
    return torch.triu(A) + torch.triu(A, 1).transpose(1, 2)


def _g1(X, tall, s2, k_keep=None):
    x = X.float()
    if k_keep is not None:   # only these K indices contribute
        x = x[:, k_keep, :] if tall else x[:, :, k_keep]
    acc = x.transpose(1, 2) @ x if tall else x @ x.transpose(1, 2)
    return _bf16(acc * s2.view(-1, 1, 1))


def emulate(x, inv, inv2, steps=STEPS, fault=None, coeffs=COEFFS):
    """X[0..steps], A[1..steps], B[1..steps] of the driver (index 0 of A, B unused).  `fault` plants one bug."""
    a, b, c = coeffs
    if fault == "b_c_exchanged":
        b, c = c, b
    batch, rows, cols = x.shape
    tall = rows > cols
    one = torch.ones(batch)
    X, A, B = [x], [None], [None]
    for s in range(1, steps + 1):
        first = s == 1
        s1, s2 = (inv, inv2) if first else (one, one)
        if fault == "neighbour_inv_norm" and first:
            s1, s2 = inv.roll(-1), inv2.roll(-1)
        if fault == "renormalised_on_iteration_2" and s == 2:
            s1, s2 = inv, inv2
        cur = X[s - 1]
        Am = _mirror(_g1(cur, tall, s2).float())
        if fault == "split_k_partial_dropped" and first:
            # G1 with 4 K-splits: tile (0, 1) (and its mirror) lost the partial over the third quarter of K
            K = rows if tall else cols
            keep = [k for k in range(K) if not K // 2 <= k < 3 * K // 4]
            short = _g1(cur, tall, s2, keep).float()
            Am[:, :128, 128:256] = short[:, :128, 128:256]
            Am[:, 128:256, :128] = short[:, :128, 128:256].transpose(1, 2)
        if fault == "mirror_not_transposed" and s == 2:
            Am[:, 128:256, :128] = Am[:, :128, 128:256]
        A.append(_bf16(Am))
        Af = A[-1].float()
        B.append(_bf16(_mirror((c * (Af @ Af) + b * Af))))
        src = X[s - 2] if (fault == "stale_ping_pong" and s == 3) else cur
        xf, Bf = src.float(), B[-1].float()
        acc = xf @ Bf if tall else Bf @ xf
        beta = a * s1.view(-1, 1, 1)
        if fault == "norm_missing_from_beta_vec" and first:
            beta = a * one.view(-1, 1, 1)
        X.append(_bf16(acc * s1.view(-1, 1, 1) + beta * xf))
    return X, A, B


def check_chain(X, A, B, inv, inv2, what=""):
    worst = {}
    for s in range(1, len(X)):
        r = nc.check_iteration(X[s - 1], A[s], B[s], X[s], s=s, inv_norm=inv, inv_norm_sq=inv2, coeffs=COEFFS,
                               what=what)
        for k, v in r.items():
            worst[k] = max(worst.get(k, 0.0), v.c32)
    return worst


SHAPES = [pytest.param((256, 384), id="wide"), pytest.param((384, 256), id="tall")]


@pytest.mark.parametrize("shape", SHAPES)
def test_checker_accepts_emulated_chain(shape):
    x, inv, inv2 = _inputs(*shape, 1)
    X, A, B = emulate(x, inv, inv2)
    c32 = check_chain(X, A, B, inv, inv2)
    # the accumulation error of the fp32 emulation is far inside C32 (gemm_check's margin, not a new one)
    assert all(v < gc.C32 / 8 for v in c32.values()), c32


FAULTS = [
    ("neighbour_inv_norm", 1, "G1"),
    ("renormalised_on_iteration_2", 2, "G1"),
    ("norm_missing_from_beta_vec", 1, "G3"),
    ("mirror_not_transposed", 2, "G1"),
    ("split_k_partial_dropped", 1, "G1"),
    ("stale_ping_pong", 3, "G3"),
    ("b_c_exchanged", 1, "G2"),
]


@pytest.mark.parametrize("shape", SHAPES)
@pytest.mark.parametrize("fault,iteration,stage", FAULTS, ids=[f[0] for f in FAULTS])
def test_checker_rejects_planted_fault(shape, fault, iteration, stage):
    """Each fault fails at its own stage and iteration, and the message names the element's tile and chunk."""
    x, inv, inv2 = _inputs(*shape, 2)
    X, A, B = emulate(x, inv, inv2, fault=fault)
    with pytest.raises(AssertionError, match=rf"group 0: iteration {iteration}, {stage} .*\(batch \d+, row \d+, "
                                             rf"col \d+\) in tile \(\d+, \d+\), chunk \d+"):
        check_chain(X, A, B, inv, inv2, "group 0")


def test_neighbour_inv_norm_is_invisible_with_equal_norms_after_five_steps():
    """Why the inputs need distinct norms: the 5-step outputs of the faulty and the correct chain are then close."""
    x, inv, inv2 = _inputs(256, 384, 3)
    x = (x.float() / torch.tensor(SCALES).view(-1, 1, 1)).bfloat16()
    inv = 1.0 / (x.float().pow(2).sum((1, 2)).sqrt() + EPS)
    inv2 = inv * inv
    good = emulate(x, inv, inv2)[0][-1].double()
    bad = emulate(x, inv, inv2, fault="neighbour_inv_norm")[0][-1].double()
    assert float((good - bad).norm() / good.norm()) < 3e-2


def test_ns_slices_single_and_grouped():
    """The helper's offsets: A at the group's base, B one aligned A later, X_tmp only for steps >= 2, split-K
    partials only for a lone big matrix, groups back to back."""
    sl = nc.ns_slices([(3, 256, 512)], 1, 132)
    assert sl == [nc.Slices(0, 393216, 786432, 786432, 786432, 1)]
    sl = nc.ns_slices([(1, 32003, 1024), (2, 136, 72)], 2, 132)
    assert sl[0].splits == nc.g1_k_splits(1, 1024, 32003, 132) > 1
    assert sl[0].end == sl[0].splitk + sl[0].splits * 1024 * 1024 * 4
    assert sl[1].a == sl[0].end and sl[1].b == sl[1].a + nc._a256(2 * 72 * 72 * 2)
    assert nc.grouped_ok([(1, 32003, 1024)], 132) and not nc.grouped_ok([(1, 32003, 1024), (2, 136, 72)], 132)


# ---- Shampoo ----------------------------------------------------------------------------------------------------
def _f32_chain(terms, C=None, beta=0.0, alpha=1.0):
    """gemm3 as the kernels run it: one fp32 GEMM per term, each added to the running fp32 output."""
    D = None
    for i, (x, y) in enumerate(terms):
        p = alpha * (x.float() @ y.float())
        D = (p + beta * C.float() if C is not None else p) if i == 0 else D + p
    return D


def _stats_inputs(batch, k1, k2, seed, exact=True):
    g = torch.Generator().manual_seed(seed)
    if exact:
        Gh, Gl = nc.exact_hi((batch, k1, k2), generator=g), nc.exact_lo((batch, k1, k2), generator=g)
        L0 = gc.exact_ints((batch, k1, k1), generator=g)
    else:
        Gh, Gl = nc.split(torch.randn(batch, k1, k2, generator=g))
        L0 = torch.randn(batch, k1, k1, generator=g)
    return Gh, Gl, L0


def _stats_L(Gh, Gl, L0, beta2, weight, fault=None):
    t = Gh.transpose(1, 2)
    terms = [(Gh, t), (Gh, Gl.transpose(1, 2)), (Gl, t)]
    if fault == "Gl_Gh^T_dropped":
        terms = terms[:2]
    if fault == "g_lo_from_next_batch":
        Glr = Gl.roll(1, 0)
        terms = [(Gh, t), (Gh, Glr.transpose(1, 2)), (Glr, t)]
    return _f32_chain(terms, L0, beta2, weight)


@pytest.mark.parametrize("fault", [None, "Gl_Gh^T_dropped", "g_lo_from_next_batch"])
@pytest.mark.parametrize("k", [37, 264, 1000])
def test_stats_exact_family(fault, k):
    """L = beta2 L + weight (Gh Gh^T + Gh Gl^T + Gl Gh^T) is known bit for bit; a dropped or misread lo term fails."""
    beta2, weight = 0.5, 0.25
    Gh, Gl, L0 = _stats_inputs(2, k, 136, 10 + k)
    (R, P), _ = nc.stats_reference(Gh, Gl, L0, torch.zeros(2, 136, 136), k, 136, beta2, weight)
    D = _stats_L(Gh, Gl, L0, beta2, weight, fault)
    if fault is None:
        nc.check3(D, R, P, 136, True, "L")
    else:
        with pytest.raises(AssertionError, match=r"L: .* differ from the exact result; worst at \(batch"):
            nc.check3(D, R, P, 136, True, "L")


def test_stats_bound_family_accepts_c4_size():
    beta2, weight = 0.95, 0.05
    Gh, Gl, L0 = _stats_inputs(1, 1024, 1024, 11, exact=False)
    (R, P), _ = nc.stats_reference(Gh, Gl, L0, torch.zeros(1, 1024, 1024), 1024, 1024, beta2, weight)
    b = nc.check3(_stats_L(Gh, Gl, L0, beta2, weight), R, P, 1024, False, "L")
    assert b.ratio <= 1.0


def _precond_inputs(batch, k1, k2, seed):
    g = torch.Generator().manual_seed(seed)
    PLh, PLl = nc.exact_hi((batch, k1, k1), generator=g), nc.exact_lo((batch, k1, k1), generator=g)
    PRh, PRl = nc.exact_hi((batch, k2, k2), generator=g), nc.exact_lo((batch, k2, k2), generator=g)
    mh, ml = nc.exact_hi((batch, k1, k2), generator=g), nc.exact_lo((batch, k1, k2), generator=g)
    return PLh, PLl, PRh, PRl, mh, ml


PRECOND_SHAPES = [(37, 264), (259, 136), (37, 64)]   # those of the GPU tests' exact family


@pytest.mark.parametrize("fault", [None, "PLl_m_h_dropped", "m_lo_from_next_batch", "Tl_zero"])
@pytest.mark.parametrize("k1,k2", PRECOND_SHAPES)
def test_precond_first_product_and_split_exact(fault, k1, k2):
    PLh, PLl, PRh, PRl, mh, ml = _precond_inputs(2, k1, k2, 20 + k1)
    R, P = nc.precond_first_reference(PLh, PLl, mh, ml, k1, k2)
    terms = [(PLh, mh), (PLh, ml.roll(1, 0) if fault == "m_lo_from_next_batch" else ml), (PLl, mh)]
    if fault == "PLl_m_h_dropped":
        terms = terms[:2]
    T = _f32_chain(terms)
    Th, Tl = nc.split(T)
    if fault == "Tl_zero":
        Tl = torch.zeros_like(Tl)
    if fault is None:
        nc.check3(T, R, P, k1, True, "T")
        nc.check_split(T, Th, Tl, "T")
    elif fault == "Tl_zero":
        nc.check3(T, R, P, k1, True, "T")
        with pytest.raises(AssertionError, match=r"Tl = bf16_rn\(T - Th\): .* worst at \(batch"):
            nc.check_split(T, Th, Tl, "T")
    else:
        with pytest.raises(AssertionError, match=r"T: .* differ from the exact result; worst at \(batch"):
            nc.check3(T, R, P, k1, True, "T")


@pytest.mark.parametrize("fault", [None, "Th_PRl_dropped", "Tl_PRh_dropped", "PRl_from_next_batch"])
@pytest.mark.parametrize("k1,k2", PRECOND_SHAPES)
def test_precond_second_product_sees_each_dropped_term(fault, k1, k2):
    """The second product is held to the bound on the kernel's own Th / Tl.  In the exact family every dropped or
    misread lo term exceeds that bound at the GPU tests' shapes (k2 <= 264), so the bound check still rejects it."""
    alpha = -0.5
    PLh, PLl, PRh, PRl, mh, ml = _precond_inputs(2, k1, k2, 30 + k1)
    T = _f32_chain([(PLh, mh), (PLh, ml), (PLl, mh)])
    Th, Tl = nc.split(T)
    R, P = nc.precond_second_reference(Th, Tl, PRh, PRl, k2, alpha)
    terms = [(Th, PRh), (Th, PRl.roll(1, 0) if fault == "PRl_from_next_batch" else PRl), (Tl, PRh)]
    if fault == "Th_PRl_dropped":
        terms = [terms[0], terms[2]]
    if fault == "Tl_PRh_dropped":
        terms = terms[:2]
    out = _f32_chain(terms, alpha=alpha)
    if fault is None:
        b = nc.check3(out, R, P, k2, False, "out")
        assert b.c32 < gc.C32 / 8
    else:
        with pytest.raises(AssertionError, match=r"out: \|D - R\| exceeds its bound .* at \(batch \d+, row \d+"):
            nc.check3(out, R, P, k2, False, "out")


def test_zero_padding_check():
    F = torch.zeros(2, 40, 40)
    F[:, :37, :37] = torch.randn(2, 37, 37)
    nc.zero_padding_bits(F, 37, "L")
    F[1, 38, 3] = -0.0       # a negative zero is a write, and not +0.0
    with pytest.raises(AssertionError, match=r"padding .* \(batch 1, row 38, col 3\)"):
        nc.zero_padding_bits(F, 37, "L")
