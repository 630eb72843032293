"""-m gpu: b200_shampoo_root_newton (ShampooParams.inverse_root = "newton") against the fp64 eigendecomposition
truth of tests/shampoo_root_check.py, its determinism, and Shampoo / the Trainer running with it."""
import pytest
import torch

from tests import shampoo_root_check as C

pytestmark = pytest.mark.gpu

EPS = 1e-6
MAX_ITERS = 40
TOL = 1e-5


@pytest.fixture(scope="module")
def ops():
    from mlx_cuda_distributed_pretraining_b200 import ops as _ops
    _ops.require_device()
    return _ops


def run_root(ops, M, k, with_split=True):
    P = torch.full_like(M, float("nan"))      # every element must be written, padding included
    Ph = torch.empty(M.shape, dtype=torch.bfloat16, device=M.device) if with_split else None
    Pl = torch.empty(M.shape, dtype=torch.bfloat16, device=M.device) if with_split else None
    iters, res = ops.shampoo_root_newton(M, P, Ph, Pl, k, EPS, MAX_ITERS, TOL)
    torch.cuda.synchronize()
    return P, Ph, Pl, iters, res


def mixed_batch(k, batch, seed):
    return C.batch_of([C.spectrum_matrix(C.KINDS[i % len(C.KINDS)], k, seed + i, scale=10.0 ** (i % 5 - 2))
                       for i in range(batch)], ops_rup8(k))


def ops_rup8(k):
    return (k + 7) // 8 * 8


@pytest.mark.parametrize("k,batch", [(8, 64), (37, 12), (64, 64), (259, 6), (1024, 6)])
def test_newton_root_matches_fp64_truth(ops, k, batch):
    """Six spectra (well-conditioned, kappa 1e4, ridge-limited, rank-deficient, zero, scaled identity), each at
    several scales: spectral and Frobenius error bounds, residual <= tol within max_iters, zero padding, and the
    bf16 hi/lo pair carrying P."""
    M = mixed_batch(k, batch, seed=100 * k)
    P, Ph, Pl, iters, res = run_root(ops, M.cuda(), k)
    worst = C.check_roots(P, M.cuda(), k, EPS, iters=iters.cpu(), residual=res.cpu(), tol=TOL, max_iters=MAX_ITERS)
    carried = (Ph.float() + Pl.float() - P).abs().max() / P.abs().max()
    assert float(carried) <= 1e-5, float(carried)
    print(f"k={k} batch={batch}: worst fro {worst['fro']:.3g} spectral {worst['spectral']:.3g}, "
          f"iterations {int(iters.min())}..{int(iters.max())}, residual max {float(res.max()):.3g}")


def test_newton_root_on_c4_like_statistics(ops):
    """The power-law statistics of the issue's CPU table (lambda_max 0.45 and 45) at k = 1024."""
    M = torch.stack([C.power_law_statistics(1024, 0.45), C.power_law_statistics(1024, 45.0)])
    P, _, _, iters, res = run_root(ops, M.cuda(), 1024, with_split=False)
    worst = C.check_roots(P, M.cuda(), 1024, EPS, iters=iters.cpu(), residual=res.cpu(), tol=TOL,
                          max_iters=MAX_ITERS)
    print("power-law statistics:", worst, iters.tolist(), res.tolist())


def test_newton_root_is_deterministic_and_batch_independent(ops):
    """Repeated launches give the same bits; every matrix of a batch that mixes fast (scaled identity, well
    conditioned) and slow (ridge-limited, rank-deficient) matrices gives the same bits launched alone."""
    k = 264
    M = mixed_batch(k, 6, seed=7).cuda()
    P1, Ph1, Pl1, it1, r1 = run_root(ops, M, k)
    P2, Ph2, Pl2, it2, r2 = run_root(ops, M, k)
    assert torch.equal(P1, P2) and torch.equal(Ph1, Ph2) and torch.equal(Pl1, Pl2)
    assert torch.equal(it1, it2) and torch.equal(r1, r2)
    assert int(it1.min()) < int(it1.max())           # the batch really mixes convergence speeds
    for b in range(M.shape[0]):
        Pb, _, _, itb, rb = run_root(ops, M[b:b + 1].contiguous(), k)
        assert torch.equal(Pb[0], P1[b]), b
        assert int(itb[0]) == int(it1[b]) and float(rb[0]) == float(r1[b]), b


def test_newton_root_rejects_bad_arguments(ops):
    M = torch.zeros(1, 8, 8, device="cuda")
    with pytest.raises(ops.B200Error):
        ops.shampoo_root_newton(M, M, None, None, 8, EPS)          # M and P must be distinct
    with pytest.raises(ops.B200Error):
        ops.shampoo_root_newton(M, torch.zeros_like(M), None, None, 0, EPS)
    lib = ops.lib()
    P = torch.zeros_like(M)
    need = int(lib.b200_shampoo_root_newton_workspace_bytes(1, 8))
    ws = torch.empty(need - 256, dtype=torch.uint8, device="cuda")
    rc = lib.b200_shampoo_root_newton(M.data_ptr(), P.data_ptr(), None, None, 1, 8, EPS, 4, TOL, None, None,
                                      ws.data_ptr(), ws.numel(), ops._stream())
    assert rc != 0 and b"workspace" in lib.b200_last_error()


def test_shampoo_newton_steps_track_oracle(tmp_path):
    """Shampoo(inverse_root="newton") through the Trainer against ShampooOracle computing its own roots as the fp64
    truth, fed the device's own gradients from a copy of the device state before each step.  Every preconditioned
    step is finite and non-zero (the literal root's fp32 norm overflow does not happen)."""
    from oracle import reference_math as R
    from tests.test_gpu_training import make_trainer, masters, rel
    over = {"training__optimization": {"optimizer": "shampoo", "start_preconditioning_step": 2, "update_period": 2,
                                       "beta2": 0.95, "inverse_root": "newton"}}
    tr = make_trainer(tmp_path, **over)
    assert tr.optimizer.params.inverse_root == "newton"
    hp = R.ShampooParams(beta2=0.95, update_period=2, start_preconditioning_step=2)
    captured = {}
    inner_update = tr.optimizer.update

    def capturing_update(model, gradients=None):
        captured["g"] = {n: tr.store.view(tr.store.grad, n).detach().float().cpu().clone()
                         for n in tr.store.named_master()}
        return inner_update(model, gradients)
    tr.optimizer.update = capturing_update

    worst, compared = 0.0, 0
    so = None
    for step in range(5):
        batch = tr.data_manager.generate_batch(step)
        before = masters(tr)
        if step:   # the oracle continues from the device's state (its roots included) before this step
            so.count = tr.optimizer.count
            for n, st in tr.optimizer.state.items():
                s = so.state[n]
                for key in ("momentum", "graft_m", "graft_v"):
                    s[key] = st[key].detach().cpu().clone()
                if "statistics.0" in st:
                    s["statistics"] = [st["statistics.0"].detach().cpu().clone(),
                                       st["statistics.1"].detach().cpu().clone()]
                    if so.count >= hp.start_preconditioning_step:
                        s["preconditioners"] = [st["preconditioners.0"].detach().cpu().clone(),
                                                st["preconditioners.1"].detach().cpu().clone()]
        else:
            so = R.ShampooOracle(tr.lr_schedule, hp)
        tr.train_step(step, batch)
        after_ref = dict(before)
        with C.oracle_newton_roots(R):
            so.update(after_ref, captured["g"])
        after = masters(tr)
        for n in before:
            d, ds = after[n] - before[n], after_ref[n] - before[n]
            assert bool(torch.isfinite(d).all()), (step, n)
            if before[n].dim() == 2 and tr.optimizer.count >= hp.start_preconditioning_step:
                assert float(d.norm()) > 0.0, (step, n)
                compared += 1
                worst = max(worst, rel(d, ds))
                assert rel(d, ds) < 5e-2, (step, n, rel(d, ds))
    print(f"shampoo newton step parity: worst rel {worst:.3g} over {compared} preconditioned steps")
    assert compared > 0


def test_trainer_newton_root_steps_and_resume(tmp_path):
    """A C4-shaped trainer (Shampoo, preconditioning from step 2, roots every 2 steps) with inverse_root: newton:
    no grafted step is zeroed, and a resume from the step-3 checkpoint reproduces the next step bit for bit."""
    from mlx_cuda_distributed_pretraining_b200.core.training import Config, Trainer
    from tests.smoke_check import tiny_config
    from tests.test_gpu_training import make_trainer, masters
    opt_cfg = {"optimizer": "shampoo", "start_preconditioning_step": 2, "update_period": 2, "beta2": 0.95,
               "inverse_root": "newton"}
    over = {"training__optimization": opt_cfg, "hp__iters": 8,
            "logging__steps": {"logging_interval": 10 ** 9, "checkpoint_interval": 3, "validation_interval": 0}}
    tr = make_trainer(tmp_path, **over)
    for step in range(3):
        before = masters(tr)
        tr.train_step(step, tr.data_manager.generate_batch(step))
        after = masters(tr)
        for n in before:
            d = after[n] - before[n]
            assert bool(torch.isfinite(d).all()) and float(d.norm()) > 0.0, (step, n)
    tr.save_checkpoint(3)
    tr.train_step(3, tr.data_manager.generate_batch(3))
    want = masters(tr)

    cfg = tiny_config(**over)
    cfg["resume"] = {"checkpoint": str(tmp_path / "smoke" / "checkpoints" / "step_3")}
    tr2 = Trainer(Config.from_dict(cfg), synthetic=True, quiet=True, run_root=str(tmp_path / "resumed"))
    tr2._accum_step, tr2._accum_tokens = 0, 0
    assert tr2.load_checkpoint(cfg["resume"]["checkpoint"]) == 3
    tr2.train_step(3, tr2.data_manager.generate_batch(3))
    got = masters(tr2)
    assert all(torch.equal(got[n], want[n]) for n in want), [n for n in want if not torch.equal(got[n], want[n])][:3]
