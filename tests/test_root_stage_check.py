"""CPU self-test of tests/root_stage_check.py: the iteration checker accepts an fp32 emulation of both Shampoo roots
and rejects the outputs that plausible driver faults would produce.  Without it nothing shows that
tests/test_gpu_shampoo_root_stages.py could fail.

The emulations do what csrc/shampoo.cu does: split products accumulated in fp32 (one fp32 product per split pair,
added to the running fp32 sum in the driver's order), the same epilogues and the same Newton state machine.  The
matrices of a batch get clearly different scales, 10^(i % 5 - 2): with equal scales a matrix that reads its
neighbour's scalar would be invisible."""
import pytest
import torch

from tests import root_stage_check as rc
from tests import shampoo_root_check as C

F32 = torch.float32
EPS = 1e-6


# ---- literal root emulation ------------------------------------------------------------------------------------------
def _split(x):
    h = x.bfloat16()
    return h, (x - h.float()).bfloat16()


def emulate_literal(M, k, p, eps, iters, fault=None):
    """The state a b200_shampoo_root run with `iters` iterations leaves (workspace slots, P, P_hi, P_lo)."""
    kp = M.shape[-1]
    tr = torch.diagonal(M[:, :k, :k], dim1=1, dim2=2).sum(1) + torch.tensor(k * rc.f32(eps), dtype=F32)
    inv_tr = 1.0 / tr
    fin = tr ** rc.f32(-1.0 / rc.f32(p * p))
    s_inv = inv_tr.roll(1) if fault == "neighbour_inv_tr" else inv_tr
    s_fin = fin.roll(1) if fault == "neighbour_fin" else fin
    if fault in ("eps_on_padded_rows", "eps_everywhere"):
        i = torch.arange(kp)
        add = (i.view(-1, 1) == i.view(1, -1)) if fault == "eps_on_padded_rows" else torch.ones(kp, kp, dtype=bool)
        Z = torch.where(add, M + torch.tensor(eps, dtype=F32), M) * s_inv.view(-1, 1, 1)
    else:
        Z = rc.literal_z0(M, k, eps, s_inv)
    Zh, Zl = _split(Z)
    a = rc.f32(1.0 / rc.f32(p))
    prev = Z
    for it in range(iters):
        last = it == iters - 1
        h, l = Zh.float(), Zl.float()
        acc = h @ h.transpose(1, 2)
        acc = acc + h @ l.transpose(1, 2)          # gemm3's second GEMM (dropped by the fault below)
        if fault == "gemm3_drops_Zh_Zl":
            acc = h @ h.transpose(1, 2)
        acc = acc + l @ h.transpose(1, 2)
        sa = s_fin.view(-1, 1, 1) if last else torch.ones(1)
        sb = s_fin.view(-1, 1, 1) if last and fault != "fin_on_product_only" else torch.ones(1)
        if last and fault == "fin_on_C_only":
            sa = torch.ones(1)
        prev, Z = Z, (a * sa) * acc + sb * Z
        if not last and fault != "stale_split":
            Zh, Zl = _split(Z)
    P = Z
    if fault == "parity_swapped":
        P, prev = prev, P
    Ph, Pl = _split(P)
    return {"Zb": prev, "Zh": Zh, "Zl": Zl, "inv_tr": inv_tr, "fin": fin, "P": P, "Ph": Ph, "Pl": Pl}


def check_literal_chain(M, k, p, fault=None, runs=6, what=""):
    states = [emulate_literal(M, k, p, EPS, s, fault) for s in range(1, runs + 1)]
    worst = {}
    for s in range(1, runs + 1):
        r = rc.check_literal_run(M, k, p, EPS, s, states[s - 1], states[s] if s < runs else None, what)
        for f, v in r.items():
            worst[f] = max(worst.get(f, 0.0), v)
    return worst


@pytest.mark.parametrize("p", [0.5, 0.75])
@pytest.mark.parametrize("k", [8, 37, 259])
def test_literal_checker_accepts_emulation(k, p):
    M = rc.mixed_batch(k, 6, 10 + k)
    worst = check_literal_chain(M, k, p)
    assert all(v <= 1.0 for v in worst.values()), worst


LITERAL_FAULTS = [
    ("neighbour_inv_tr", 1, "Z0"),
    ("neighbour_fin", 1, "P = fin"),
    ("eps_on_padded_rows", 1, "Z0"),
    ("eps_everywhere", 1, "Z0"),
    ("fin_on_product_only", 1, "P = fin"),
    ("fin_on_C_only", 1, "P = fin"),
    ("stale_split", 2, "Zh/Zl split"),
    ("parity_swapped", 1, "Z0"),
    ("gemm3_drops_Zh_Zl", 1, "P = fin"),
]


@pytest.mark.parametrize("k", [37, 259])
@pytest.mark.parametrize("fault,iteration,stage", LITERAL_FAULTS, ids=[f[0] for f in LITERAL_FAULTS])
def test_literal_checker_rejects_planted_fault(fault, iteration, stage, k):
    M = rc.mixed_batch(k, 6, 20 + k)
    with pytest.raises(AssertionError, match=rf"literal root, b: iteration {iteration}, {stage}.*\(batch \d+, row "
                                             rf"\d+, col \d+\)"):
        check_literal_chain(M, k, 0.75, fault, what="b")


def test_literal_dropped_lo_term_visibility():
    """Where the dropped Zh Zl^T product exceeds the three-GEMM bound, on the first iterate (Z0 = M / tr): at
    every k up to 259 by a wide margin; at 1024 on these spectra not reliably (so the GPU tests rely on k <= 259
    for it)."""
    for k in (8, 37, 136, 259):
        M = rc.mixed_batch(k, 6, 30 + k)
        with pytest.raises(AssertionError, match=r"P = fin .* exceeds its bound"):
            check_literal_chain(M, k, 0.75, "gemm3_drops_Zh_Zl", runs=1)


# ---- Newton root emulation -------------------------------------------------------------------------------------------
def mm6(A3, B3, drop=None):
    """gemm6 on 3-way splits: hh, hm, mh, hl, lh, mm, each one fp32 product added to the running fp32 sum."""
    (ah, am, al), (bh, bm, bl) = [[t.float() for t in s] for s in (A3, B3)]
    terms = {"hh": (ah, bh), "hm": (ah, bm), "mh": (am, bh), "hl": (ah, bl), "lh": (al, bh), "mm": (am, bm)}
    D = None
    for name, (x, y) in terms.items():
        if name == drop:
            continue
        p = x @ y
        D = p if D is None else D + p
    return D


def emulate_newton(M, k, eps, tol, iters, fault=None):
    """States after iterations 1..iters of b200_shampoo_root_newton (each the state a run with max_iters = s leaves
    while some matrix is still iterating), keyed as root_stage_check.newton_views."""
    batch, kp, _ = M.shape
    e32 = torch.tensor(eps, dtype=F32)
    Mk = M[:, :k, :k]
    v = torch.rand(batch, k, 1, generator=torch.Generator().manual_seed(0)) * 2 - 1
    v = v / v.norm(dim=1, keepdim=True)
    lam = torch.zeros(batch)
    for _ in range(32):
        w = Mk @ v
        lam = (v * w).sum((1, 2))
        n = w.norm(dim=1, keepdim=True)
        v = torch.where(n > 0, w / n.clamp_min(1e-30), v)
    ridge = e32 * torch.maximum(lam, torch.tensor(1e-6))
    ss = (Mk * Mk).sum((1, 2))
    tr = torch.diagonal(Mk, dim1=1, dim2=2).sum(1)
    fro2 = ss + (0 if fault == "z_without_ridge_tr" else 2.0 * ridge * tr) + k * ridge * ridge
    z = 5.0 / (2.0 * torch.sqrt(fro2))
    r_in = ridge.roll(1) if fault == "neighbour_ridge" else ridge
    z_in = z.roll(1) if fault == "neighbour_z" else z
    mc, t, err = rc.newton_init(M, k, r_in, z_in)
    I = rc.identity(batch, kp, k, "cpu")
    frozen = err <= tol
    t = torch.where(frozen.view(-1, 1, 1), I, t)
    X = (z ** 0.25).view(-1, 1, 1) * I
    n_it = torch.full((batch,), 1 if fault == "iters_off_by_one" else 0, dtype=torch.int32)
    T3, S3, Mc3 = rc.split3(t), None, rc.split3(mc)
    slots = [T3, rc.split3(torch.zeros_like(t))]
    drop = {"gemm6_drops_hm": "hm", "gemm6_drops_mh": "mh"}.get(fault)
    factor = torch.tensor(1.0 if fault == "accept_factor_1" else 1.2, dtype=F32)
    out = []
    for s in range(1, iters + 1):
        cur, nxt = (s - 1) % 2, s % 2
        T3 = slots[cur]
        S3 = rc.split3(mm6(T3, T3, drop))
        S3 = rc.split3(mm6(S3, S3, drop))
        F = mm6(S3, Mc3, drop)
        e = rc.max_dev(F, k)
        accept = (e <= factor * err) & ~frozen
        freeze = (~accept | (e <= tol)) & ~frozen
        nt = rc.split3(torch.where(freeze.view(-1, 1, 1) & (fault != "frozen_T_not_reset"), I, rc.next_t(F, k)))
        slots[nxt] = tuple(torch.where(frozen.view(-1, 1, 1), a, b) for a, b in zip(S3, nt))
        Mc3 = tuple(torch.where(accept.view(-1, 1, 1), a, b) for a, b in zip(rc.split3(F), Mc3))
        upd = accept | (~frozen & (fault == "x_updated_on_reject"))
        X = torch.where(upd.view(-1, 1, 1), mm6(rc.split3(X), T3), X)
        err = torch.where(accept, e, err)
        n_it = n_it + accept.to(torch.int32)
        frozen = frozen | freeze
        out.append({"F": F, "T0": slots[0], "T1": slots[1], "Mc": Mc3, "Xs": rc.split3(X), "ridge": ridge, "z": z,
                    "err": err, "iters": n_it, "frozen": frozen.to(torch.int32), "av": accept.to(F32),
                    "bv": (~accept).to(F32), "P": X, "iters_out": n_it, "residual_out": err})
        if bool(frozen.all()):
            break
    return out


def check_newton_chain(M, k, tol, fault=None, iters=40, eps=EPS, what=""):
    states = emulate_newton(M, k, eps, tol, iters, fault)
    worst, branches = {}, {}
    for s, st in enumerate(states, 1):
        r = rc.check_newton_run(M, k, eps, tol, s, st, states[s - 2] if s > 1 else None, what)
        for f, v in r["bounds"].items():
            worst[f] = max(worst.get(f, 0.0), v)
        for b, n in r["branches"].items():
            branches[b] = branches.get(b, 0) + n
    return worst, branches, len(states)


NEWTON_CASES = [(8, 1e-5), (8, 0.0), (37, 0.0), (136, 1e-5)]


@pytest.mark.parametrize("k,tol", NEWTON_CASES)
def test_newton_checker_accepts_emulation(k, tol):
    M = rc.newton_batch(k, 40 + k)
    worst, _, _ = check_newton_chain(M, k, tol)
    assert all(v <= 1.0 for v in worst.values()), worst


def test_newton_branches_all_reached():
    """At k = 8 the rejecting matrix is rejected at iteration 1, tol = 1e-5 freezes converged matrices, and tol = 0.2
    freezes the scaled identity (Mc0 = 2.5 / sqrt(8) I, e0 = 0.116) at init."""
    seen = {}
    for tol in (1e-5, 0.2):
        _, branches, _ = check_newton_chain(rc.newton_batch(8, 50), 8, tol)
        for b, n in branches.items():
            seen[b] = seen.get(b, 0) + n
    assert all(seen[b] > 0 for b in ("accept", "converge-freeze", "reject", "freeze at init")), seen


NEWTON_FAULTS = [
    ("neighbour_ridge", 1, "init T"),
    ("neighbour_z", 1, "init T"),
    ("z_without_ridge_tr", 1, "z"),
    ("accept_factor_1", None, "state"),
    ("x_updated_on_reject", 1, "X0 = z"),
    ("frozen_T_not_reset", 1, "next T of a freezing"),
    ("iters_off_by_one", 1, "state"),
    ("gemm6_drops_hm", 1, "F = T\\^4 Mc"),
    ("gemm6_drops_mh", 1, "F = T\\^4 Mc"),
]


@pytest.mark.parametrize("fault,iteration,stage", NEWTON_FAULTS, ids=[f[0] for f in NEWTON_FAULTS])
def test_newton_checker_rejects_planted_fault(fault, iteration, stage):
    eps = 1e-3 if fault == "z_without_ridge_tr" else EPS
    it = rf"{iteration}" if iteration else r"\d+"
    elem = r"matrix \d+" if stage in ("z", "state") else r"\(batch \d+, row \d+, col \d+\)"
    with pytest.raises(AssertionError, match=rf"newton root, b: iteration {it}, {stage}.*{elem}"):
        check_newton_chain(rc.newton_batch(8, 60), 8, 1e-5, fault, eps=eps, what="b")


@pytest.mark.parametrize("k", [8, 37, 136, 259])
@pytest.mark.parametrize("drop", ["hm", "mh"])
def test_newton_dropped_term_visibility(drop, k):
    """Where a gemm6 that drops its hm or mh product exceeds the chained F bound at iteration 1."""
    with pytest.raises(AssertionError, match=r"iteration 1, F = T\^4 Mc: .* exceeds its bound"):
        check_newton_chain(rc.newton_batch(k, 70 + k), k, 1e-5, "gemm6_drops_" + drop, iters=1)
