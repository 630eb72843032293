"""-m gpu: Shampoo's two inverse roots iteration by iteration against fp64 (tests/root_stage_check.py).

b200_shampoo_root (the literal root) runs with iters = s for s = 1..6 and b200_shampoo_root_newton with max_iters = s
for s = 1..N; each run's workspace is read through the maps of root_stage_check and checked on the kernel's own
operands.  Inputs sit at the front of NaN-filled allocations, the workspace is filled with a NaN bit pattern before
each run and P sits inside canaries.  The Newton root gets NaN in M's padding, which it must not propagate.  The fp64
references run on the GPU (cuBLAS DGEMM).  The last test asserts that every Newton branch was taken and prints the
worst error / bound ratio per family.
"""
import pytest
import torch

from tests import root_stage_check as rc
from tests.gemm_check import Guarded
from tests.test_gpu_matrix_optimizers_check import _nan_front, _nan_ws

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(900)]

BF16, F32 = torch.bfloat16, torch.float32
EPS = 1e-6
WORST = {}      # family -> largest ratio
BRANCHES = {}   # Newton branch -> times taken


@pytest.fixture(scope="module")
def ops():
    from mlx_cuda_distributed_pretraining_b200 import ops
    ops.require_device()
    return ops


@pytest.fixture(scope="module")
def L(ops):
    return ops.lib()


def _stream():
    return torch.cuda.current_stream().cuda_stream


def _ok(rc_):
    from mlx_cuda_distributed_pretraining_b200._lib import check
    check(rc_, "call")


def _record(bounds):
    for f, v in bounds.items():
        WORST[f] = max(WORST.get(f, 0.0), v)


def _branch(name, n=1):
    BRANCHES[name] = BRANCHES.get(name, 0) + n


def _guarded(batch, kp, dtype):
    return Guarded(batch, kp, kp, dtype, "cuda", ld=kp, stride=kp * kp)


def _clone(d):
    return {n: tuple(t.clone() for t in v) if isinstance(v, tuple) else v.clone() for n, v in d.items()}


def test_workspace_maps_match_the_library(L):
    for batch, k in [(1, 1), (1, 8), (3, 37), (6, 259), (7, 264), (2, 1024), (5, 1000)]:
        assert int(L.b200_shampoo_root_workspace_bytes(batch, k)) == rc.literal_ws(batch, k).end, (batch, k)
        assert int(L.b200_shampoo_root_newton_workspace_bytes(batch, k)) == rc.newton_ws(batch, k).end, (batch, k)


# ------------------------------------------------------------------------------------------------------------------
# the literal root
# ------------------------------------------------------------------------------------------------------------------
def _literal(L, M, k, p, s, split=True):
    batch, kp, _ = M.shape
    ws = _nan_ws(int(L.b200_shampoo_root_workspace_bytes(batch, k)))
    P = _guarded(batch, kp, F32)
    Ph, Pl = (_guarded(batch, kp, BF16), _guarded(batch, kp, BF16)) if split else (None, None)
    _ok(L.b200_shampoo_root(M.data_ptr(), P.ptr(), Ph.ptr() if split else None, Pl.ptr() if split else None, batch,
                            k, p, EPS, s, ws.data_ptr(), ws.numel(), _stream()))
    torch.cuda.synchronize()
    for G, nm in ((P, "P"), (Ph, "P_hi"), (Pl, "P_lo")):
        if G is not None:
            G.check_canaries(kp, f"literal root k={k} iters={s}: {nm}")
    st = _clone(rc.literal_views(ws, batch, k))
    st["P"] = P.view().clone()
    if split:
        st["Ph"], st["Pl"] = Ph.view().clone(), Pl.view().clone()
    return st


@pytest.mark.parametrize("p", [0.5, 0.75])
@pytest.mark.parametrize("k", [8, 37, 259, 1024])
def test_literal_root_every_iteration(L, k, p):
    """iters = 1..6 (both parities of the P / workspace ping-pong), mixed spectra and scales; P without P_hi/P_lo is
    the same bits; each matrix alone gives the same bits as in the batch (the split kernels' grid follows the batch)."""
    batch = 6
    M = _nan_front(rc.mixed_batch(k, batch, 300 + k).cuda())
    runs = [_literal(L, M, k, p, s) for s in range(1, 7)]
    for s, st in enumerate(runs, 1):
        _record(rc.check_literal_run(M, k, p, EPS, s, st, runs[s] if s < 6 else None, f"k={k} p={p}"))
        rc.same_bits(_literal(L, M, k, p, s, split=False)["P"], st["P"], f"k={k} p={p} iters={s}: P without P_hi/lo")
    for s in (5, 6):
        for b in range(batch):
            alone = _literal(L, _nan_front(M[b:b + 1].clone()), k, p, s)
            rc.same_bits(alone["P"], runs[s - 1]["P"][b:b + 1], f"k={k} p={p} iters={s}: matrix {b} alone")


# ------------------------------------------------------------------------------------------------------------------
# the coupled-Newton root
# ------------------------------------------------------------------------------------------------------------------
def _newton(L, M, k, tol, max_iters):
    batch, kp, _ = M.shape
    ws = _nan_ws(int(L.b200_shampoo_root_newton_workspace_bytes(batch, k)))
    P = _guarded(batch, kp, F32)
    it = torch.full((batch + 16,), -7, dtype=torch.int32, device="cuda")
    res = torch.full((batch + 16,), -7.0, dtype=F32, device="cuda")
    _ok(L.b200_shampoo_root_newton(M.data_ptr(), P.ptr(), None, None, batch, k, EPS, max_iters, tol, it.data_ptr(),
                                   res.data_ptr(), ws.data_ptr(), ws.numel(), _stream()))
    torch.cuda.synchronize()
    P.check_canaries(kp, f"newton root k={k} max_iters={max_iters}: P")
    assert bool((it[batch:] == -7).all()) and bool((res[batch:] == -7.0).all()), "iters_out / residual_out overrun"
    st = _clone(rc.newton_views(ws, batch, k))
    st.update(P=P.view().clone(), iters_out=it[:batch].clone(), residual_out=res[:batch].clone())
    return st


def _nan_padding(M, k):
    M = M.clone()
    M[:, k:, :] = float("nan")
    M[:, :, k:] = float("nan")
    return _nan_front(M)


NEWTON_CASES = [(8, 1e-5), (8, 0.2), (37, 0.0), (37, 1e-5), (259, 1e-5), (1024, 1e-5)]
MAX_ITERS = 40


@pytest.mark.parametrize("k,tol", NEWTON_CASES)
def test_newton_root_every_iteration(L, k, tol):
    """max_iters = s for s = 1.. until every matrix is frozen (the host's early exit cannot have cut a run short
    before that), then the early exit: max_iters = 40 and max_iters = last freeze + 1 give the same bits."""
    M = _nan_padding(rc.newton_batch(k, 400 + k).cuda(), k)
    prev, last = None, None
    for s in range(1, MAX_ITERS + 1):
        cur = _newton(L, M, k, tol, s)
        r = rc.check_newton_run(M, k, EPS, tol, s, cur, prev, f"k={k} tol={tol}")
        _record(r["bounds"])
        for b, n in r["branches"].items():
            _branch(b, n)
        prev, last = cur, s
        if bool(r["frozen"].all()):
            break
    print(f"k={k} tol={tol}: {last} iterations checked, iters {prev['iters'].tolist()}, frozen "
          f"{prev['frozen'].tolist()}")
    if not bool((prev["frozen"] != 0).all()):
        return
    # the host checks every 4 iterations whether every matrix is frozen; it stops at the first check at or after the
    # last freeze, while a run of last + 1 iterations runs them all
    assert last < MAX_ITERS - 4
    _branch("early exit")
    full, short = _newton(L, M, k, tol, MAX_ITERS), _newton(L, M, k, tol, last + 1)
    for nm in ("P", "iters_out", "residual_out"):
        rc.same_bits(full[nm], short[nm], f"k={k} tol={tol}: {nm} of max_iters {MAX_ITERS} vs {last + 1}")
        rc.same_bits(full[nm], prev[nm], f"k={k} tol={tol}: {nm} of max_iters {MAX_ITERS} vs {last}")


def test_print_worst_ratios_and_branches():
    for f, v in sorted(WORST.items()):
        print(f"WORST {f}: {v:.4f}")
    print("BRANCHES", BRANCHES)
    assert all(v <= 1.0 for v in WORST.values())
    missing = [b for b in ("accept", "reject", "converge-freeze", "freeze at init", "early exit")
               if BRANCHES.get(b, 0) == 0]
    assert not missing, f"Newton branches never taken: {missing} ({BRANCHES})"
