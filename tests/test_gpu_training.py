"""-m gpu: whole-step parity through the public surface (Trainer / optimizer.update) against the
oracle's restatement of the reference step, plus checkpoint round trip and the 2-GPU DP path.

Per-step tolerances (DESIGN.md "Parity"): loss |d| < 2e-2 absolute (bf16 forward vs fp32 oracle),
per-tensor parameter delta after one optimizer step < 0.15 relative (bf16 gradients propagated
through five Newton-Schulz iterations; SURVEY 8c asks <= 3e-2 for NS given identical inputs, which
test_gpu_parity.py checks directly)."""
import json
import os
import subprocess
import sys
from pathlib import Path

import pytest
import torch

pytestmark = pytest.mark.gpu

ROOT = Path(__file__).resolve().parents[1]

from oracle import reference_math as R  # noqa: E402
from tests.smoke_check import tiny_config  # noqa: E402

DIMS = R.LlamaDims(128, 256, 2, 4, 2, 32, 259)


def rel(a, b):
    a, b = a.detach().double().cpu(), b.detach().double().cpu()
    return float((a - b).norm() / (b.norm() + 1e-30))


def make_trainer(tmp_path, **kw):
    from mlx_cuda_distributed_pretraining_b200.core.training import Config, Trainer
    cfg = tiny_config(**kw)
    tr = Trainer(Config.from_dict(cfg), synthetic=True, quiet=True, run_root=str(tmp_path))
    tr._accum_step, tr._accum_tokens = 0, 0
    return tr


def masters(tr):
    return {n: t.detach().cpu().clone() for n, t in tr.store.named_master().items()}


def test_smoke_entry():
    from tests import smoke_check
    smoke_check.smoke(verbose=False)


def test_muon_steps_track_oracle(tmp_path):
    tr = make_trainer(tmp_path, optimizer="muon")
    ref = masters(tr)
    opt = R.MuonOracle(tr.lr_schedule)
    for step in range(3):
        batch = tr.data_manager.generate_batch(step)
        before = masters(tr)
        loss, _, did = tr.train_step(step, batch)
        assert did
        # oracle step from the SAME starting weights (no drift accumulation in the comparison)
        loss_ref, _, grads = R.loss_and_grads(before, batch, DIMS, pad_token=256)
        o2 = R.MuonOracle(tr.lr_schedule)
        o2.count = step
        o2.state = {n: {"momentum_buffer": s["momentum_buffer"].detach().cpu().clone()}
                    for n, s in prev_state.items()} if step else {}
        after_ref = dict(before)
        o2.update(after_ref, grads)
        prev_state = {n: {"momentum_buffer": s["momentum_buffer"].clone()} for n, s in tr.optimizer.state.items()}
        assert abs(float(loss) - float(loss_ref)) < 2e-2
        after = masters(tr)
        worst = max(rel(after[n] - before[n], after_ref[n] - before[n]) for n in before)
        assert worst < 0.15, (step, worst)
    assert tr.optimizer.count == 3


def test_adamw_fp32_steps_track_oracle(tmp_path):
    # lr 2e-3: at the tiny config's default 2e-2 this model diverges within three AdamW steps (attention scores
    # reach +-170, loss goes up), and a per-step comparison of a chaotic trajectory measures rounding luck
    tr = make_trainer(tmp_path, optimizer="adamw", mixed=False, hp__learning_rate=2e-3)
    for step in range(4):
        batch = tr.data_manager.generate_batch(step)
        before = masters(tr)
        opt = R.AdamWOracle(tr.lr_schedule, betas=(0.9, 0.999), eps=1e-8, weight_decay=0.01)
        opt.count = step
        if step:  # oracle continues from a copy of the CUDA optimizer's moments
            opt.state = {n: {"m": s["m"].detach().cpu().clone(), "v": s["v"].detach().cpu().clone()}
                         for n, s in tr.optimizer.state.items()}
        loss, _, _ = tr.train_step(step, batch)
        loss_ref, _, grads = R.loss_and_grads(before, batch, DIMS, pad_token=256)
        after_ref = dict(before)
        opt.update(after_ref, grads)
        assert abs(float(loss) - float(loss_ref)) < 2e-2, step
        after = masters(tr)
        # Adam's step m/(sqrt(v)+eps) is ~sign(g) for small-|g| elements, so bf16-attention noise on
        # near-zero gradients flips whole-lr steps; the elementwise update formula itself is checked to
        # 1e-6 in test_gpu_parity.py::test_adamw_sgd_axpy_clip.  Here: the moments (linear in g) must
        # track the oracle tightly and the step must be small-angle for every tensor.
        for n, s in tr.optimizer.state.items():
            # q/k projections see the bf16 attention noise most (measured 3e-2); v is quadratic in g
            assert rel(s["m"], opt.state[n]["m"]) < 1e-1, (step, n)
            assert rel(s["v"], opt.state[n]["v"]) < 2e-1, (step, n)
            d, dr = (after[n] - before[n]).flatten().double(), (after_ref[n] - before[n]).flatten().double()
            cos = float(d @ dr / (d.norm() * dr.norm() + 1e-30))
            assert cos > 0.9, (step, n, cos)


def test_shampoo_steps_track_oracle(tmp_path):
    """Two comparisons per step, both from a copy of the CUDA optimizer's state before the step:
    (a) the oracle fed the GPU's OWN gradients -- isolates optimizers/shampoo.py:316-377 (statistics, root, precondition,
        graft, write) behind `optimizer.update`, tight;
    (b) the oracle fed its own fp32 CPU gradients -- the whole step; loose, because the graft norm
        ||m / (sqrt(v) + eps)|| puts +-1 on every element whatever its size, so bf16 noise on near-zero gradient
        elements moves a tensor's step norm by several percent (seen 0.04 ... 0.09 run to run: dQ's fp32 atomics
        make the bf16 gradients themselves vary in the last bit).
    The oracle's preconditioners are the device's own (state `preconditioners.0/1`): the reference's literal "inverse
    root" (SURVEY D10) blows up to ~1e19 on this tiny model, where whether ||step||^2 overflows fp32 (=> the grafted step is
    zeroed, shampoo.py:300-310) flips on the last bits of the root -- an earlier version of this test that let the
    oracle recompute its own roots saw the device zero a step the oracle kept.  Root parity itself is
    test_gpu_parity.py's job (golden vectors, C4 sizes).  Measured: same-gradient step error 3e-6 over 38 preconditioned
    tensors, 7 zeroed steps agreeing exactly; full-step norm ratio within 2e-3, cosine 0.999."""
    over = {"training__optimization": {"optimizer": "shampoo", "start_preconditioning_step": 2, "update_period": 2,
                                       "beta2": 0.95}}
    tr = make_trainer(tmp_path, **over)
    assert type(tr.optimizer).__name__ == "Shampoo"
    hp = R.ShampooParams(beta2=0.95, update_period=2, start_preconditioning_step=2)
    captured = {}
    inner_update = tr.optimizer.update

    def capturing_update(model, gradients=None):
        captured["g"] = {n: tr.store.view(tr.store.grad, n).detach().float().cpu().clone()
                         for n in tr.store.named_master()}
        return inner_update(model, gradients)
    tr.optimizer.update = capturing_update

    def oracle_from_state(before, first):
        so = R.ShampooOracle(tr.lr_schedule, hp)
        so.count = tr.optimizer.count
        has_roots = so.count >= hp.start_preconditioning_step
        for n in (() if first else before):
            st = tr.optimizer.state[n]
            so.state[n] = {"momentum": st["momentum"].detach().cpu().clone(),
                           "graft_m": st["graft_m"].detach().cpu().clone(),
                           "graft_v": st["graft_v"].detach().cpu().clone(), "statistics": None,
                           "preconditioners": None}
            if "statistics.0" in st:
                so.state[n]["statistics"] = [st["statistics.0"].detach().cpu().clone(),
                                             st["statistics.1"].detach().cpu().clone()]
                # roots exist on the device once count reached start_preconditioning_step (update_period divides it)
                so.state[n]["preconditioners"] = ([st["preconditioners.0"].detach().cpu().clone(),
                                                   st["preconditioners.1"].detach().cpu().clone()]
                                                  if has_roots else [None, None])
        return so

    worst = {"norm_same": 0.0, "rel_same": 0.0, "norm_full": 0.0, "cos_full": 1.0, "zero_steps": 0,
             "preconditioned_compared": 0}
    for step in range(4):
        batch = tr.data_manager.generate_batch(step)
        before = masters(tr)
        so_same, so_full = oracle_from_state(before, step == 0), oracle_from_state(before, step == 0)
        loss, _, _ = tr.train_step(step, batch)
        loss_ref, _, grads = R.loss_and_grads(before, batch, DIMS, pad_token=256)
        assert abs(float(loss) - float(loss_ref)) < 2e-2
        after_same, after_full = dict(before), dict(before)
        so_same.update(after_same, captured["g"])
        so_full.update(after_full, grads)
        after = masters(tr)
        for n in before:
            d, ds, df = after[n] - before[n], after_same[n] - before[n], after_full[n] - before[n]
            if float(ds.norm()) == 0.0:
                assert float(d.norm()) == 0.0, (step, n)
                worst["zero_steps"] += 1
                continue
            if before[n].dim() == 2 and tr.optimizer.count >= hp.start_preconditioning_step:
                worst["preconditioned_compared"] += 1
            worst["norm_same"] = max(worst["norm_same"], abs(float(d.norm() / ds.norm()) - 1))
            worst["rel_same"] = max(worst["rel_same"], rel(d, ds))
            assert abs(float(d.norm() / ds.norm()) - 1) < 1e-2, (step, n, float(d.norm() / ds.norm()))
            assert rel(d, ds) < 5e-2, (step, n, rel(d, ds))
            if float(df.norm()) > 0.0:
                cos = float(d.flatten().double() @ df.flatten().double() / (d.norm().double() * df.norm().double()))
                worst["norm_full"] = max(worst["norm_full"], abs(float(d.norm() / df.norm()) - 1))
                worst["cos_full"] = min(worst["cos_full"], cos)
                assert abs(float(d.norm() / df.norm()) - 1) < 0.2, (step, n, float(d.norm() / df.norm()))
                assert cos > 0.9, (step, n, cos)
    print("shampoo step parity (worst over 4 steps):", {k: (v if isinstance(v, int) else float(f"{v:.3g}"))
                                                         for k, v in worst.items()})
    assert worst["preconditioned_compared"] > 0      # the preconditioned branch was really compared


def test_clip_and_accumulation_semantics(tmp_path):
    """core/training.py:1664-1696: clamp each micro-batch's grads, divide by k, sum, update once."""
    clip = 2e-3   # clamps the large entries only, so the clamp is exercised but not everywhere
    tr = make_trainer(tmp_path, optimizer="adamw", mixed=False, hp__gradient_accumulation_steps=2,
                      hp__gradient_clip=clip)
    params = masters(tr)
    acc = None
    for step in range(2):
        batch = tr.data_manager.generate_batch(step)
        _, _, did = tr.train_step(step, batch)
        _, _, grads = R.loss_and_grads(params, batch, DIMS, pad_token=256)
        g = {k: v / 2 for k, v in R.clip_elementwise(grads, clip).items()}
        acc = g if acc is None else {k: acc[k] + g[k] for k in g}
        assert did == (step == 1)
    # the fp32 accumulation buffer the optimizer consumed == sum_k clamp(g_k)/2 of the oracle
    clamped = 0
    for n in params:
        got = tr.store.view(tr.store.acc, n).detach().cpu()
        assert rel(got, acc[n]) < 3e-2, n
        assert float(got.abs().max()) <= clip * (1 + 1e-6)
        clamped += int((got.abs() >= clip * 0.999).sum())
    assert clamped > 0
    assert tr.optimizer.count == 1   # one update for two micro-batches


def test_optimizer_update_accepts_reference_style_gradient_dict(tmp_path):
    """opt.update(model, gradients) with a nested pytree, the call core/training.py:1700 makes."""
    from mlx_cuda_distributed_pretraining_b200.optimizers import Muon
    tr = make_trainer(tmp_path, optimizer="muon")
    model, store = tr.model, tr.store
    grads_flat = {n: torch.randn(s, generator=torch.Generator().manual_seed(i)) * 0.01
                  for i, (n, (_, s)) in enumerate(store.index.items())}
    nested = {}
    for name, g in grads_flat.items():
        d = nested
        parts = name.split(".")
        for p in parts[:-1]:
            d = d.setdefault(p, {})
        d[parts[-1]] = g
    before = masters(tr)
    opt = Muon(learning_rate=0.02)
    opt.update(model, nested)
    ref = dict(before)
    R.MuonOracle(0.02).update(ref, {n: g.to(torch.bfloat16).float() for n, g in grads_flat.items()})
    after = masters(tr)
    assert max(rel(after[n] - before[n], ref[n] - before[n]) for n in before) < 3e-2
    assert set(opt.state) == set(before) and opt.count == 1
    x = opt.zeropower_via_newtonschulz5(torch.randn(64, 128, device="cuda"), 5)
    assert x.shape == (64, 128)


def test_checkpoint_roundtrip_and_log_format(tmp_path):
    tr = make_trainer(tmp_path, hp__iters=6,
                      logging__steps={"logging_interval": 2, "checkpoint_interval": 3, "validation_interval": 0})
    tr.train()
    ck = tmp_path / "smoke" / "checkpoints"
    for stem in ("step_3", "step_6", "step_final"):
        for suffix in ("_model.safetensors", "_optimizer.safetensors", "_state.json"):
            assert (ck / f"{stem}{suffix}").exists(), stem + suffix
    meta = json.loads((tmp_path / "smoke" / "metadata.json").read_text())
    assert [c["step"] for c in meta["checkpoints"]] == [3, 6, "final"]
    log = (tmp_path / "smoke" / "log.txt").read_text()
    assert "Step 0: loss=" in log and " | tokens_per_sec=" in log and " | lr=" in log   # utils/plotting.py format
    from safetensors.torch import load_file
    w = load_file(str(ck / "step_final_model.safetensors"))
    assert set(w) == set(R.param_shapes(DIMS))
    cur = masters(tr)
    assert all(torch.equal(w[n], cur[n]) for n in w)
    # resume: weights + optimizer state + step come back
    cfg = tiny_config(hp__iters=8)
    cfg["resume"] = {"checkpoint": str(ck / "step_3")}
    from mlx_cuda_distributed_pretraining_b200.core.training import Config, Trainer
    tr2 = Trainer(Config.from_dict(cfg), synthetic=True, quiet=True, run_root=str(tmp_path / "resumed"))
    assert tr2.load_checkpoint(str(ck / "step_3")) == 3
    w3 = load_file(str(ck / "step_3_model.safetensors"))
    assert all(torch.equal(w3[n], t.cpu()) for n, t in tr2.store.named_master().items())
    assert tr2.optimizer.count == 3


@pytest.mark.parametrize("mixed", [False, True])
def test_model_and_loss_match_reference_golden(tmp_path, mixed):
    """The product model + Trainer.compute_loss against what the REFERENCE's own arch/llama.py and
    core/training.py:1195-1234 produced for the same weights and tokens (tests/golden/make_golden.py)."""
    import numpy as np
    from mlx_cuda_distributed_pretraining_b200.core.training import Config, Trainer
    g = np.load(ROOT / "tests" / "golden" / "reference_vectors.npz")
    cfg = tiny_config(optimizer="adamw", mixed=mixed)
    cfg["data"]["tokenizer"]["normal_vocab_size"] = 64                     # 64 + pad/bos/eos = the golden model's 67
    cfg["model"]["dimensions"] = {"hidden_size": 64, "intermediate_size": 96, "num_layers": 2}
    cfg["model"]["attention"] = {"num_heads": 4, "num_kv_heads": 2, "head_dim": 16, "max_position_embeddings": 64}
    params = {k.split("::", 1)[1]: torch.from_numpy(g[k]) for k in g.files if k.startswith("model_param::")}
    tr = Trainer(Config.from_dict(cfg), synthetic=True, quiet=True, run_root=str(tmp_path), init_params=params)
    tokens = torch.from_numpy(g["model_tokens"]).cuda()
    with torch.no_grad():
        logits = tr.model(tokens).float()
    assert rel(logits, torch.from_numpy(g["model_logits"])) < (2e-2 if mixed else 5e-3)
    tr.tokenizer.PAD_TOKEN = 66                                            # the pad id the golden batch uses
    batch = torch.from_numpy(g["loss_batch"]).cuda()
    with torch.no_grad():
        loss, ntoks = tr.compute_loss(tr.model, batch[:, :-1], batch[:, 1:])
    assert int(ntoks) == int(g["loss_ntoks"])
    assert abs(float(loss) - float(g["loss_value"])) < (3e-2 if mixed else 5e-3)


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs 2 GPUs")
def test_two_gpu_data_parallel_matches_mean_of_gradients(tmp_path):
    """2 ranks x batch 2 (NCCL all-reduce of the flat gradient buffer, 1/world folded into the
    optimizer) == one process accumulating the same two batches with weight 1/2 each."""
    out = tmp_path / "dp"
    out.mkdir()
    env = dict(os.environ, PYTHONPATH=str(ROOT))
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=2", "--master-addr",
           "127.0.0.1", "--master-port", "29611", str(ROOT / "tests" / "dp_worker.py"), str(out)]
    subprocess.run(cmd, check=True, env=env, timeout=600)
    dpw = torch.load(out / "dp_rank0.pt")
    dpw1 = torch.load(out / "dp_rank1.pt")
    # owner-computes Newton-Schulz: every matrix is orthogonalised on one rank and gathered, so the
    # replicas stay bit-identical
    assert all(torch.equal(dpw[n], dpw1[n]) for n in dpw)
    tr = make_trainer(tmp_path, optimizer="muon", hp__gradient_accumulation_steps=2)
    for micro, rank in enumerate((0, 1)):
        tr.train_step(micro, R.synthetic_batch(0, rank, 2, 128, 256))
    got = masters(tr)
    # DP sums bf16 gradients over NCCL; the single-process twin accumulates them in fp32
    assert max(rel(dpw[n], got[n]) for n in got) < 5e-3


@pytest.mark.parametrize("optimizer", ["hybrid", "shampoo"])
def test_resume_restores_full_optimizer_state(tmp_path, optimizer):
    """Save at step 3, resume in a fresh Trainer: every optimizer tensor (momentum / Adam moments / Shampoo
    statistics AND preconditioners), both step counters of the hybrid optimizer, and -- the point of saving the
    preconditioners (reference state: optimizers/shampoo.py:180-208, saved by core/training.py:1354-1356) -- the
    next step of the resumed run equals the next step of the uninterrupted run bit for bit."""
    from safetensors.torch import load_file
    from mlx_cuda_distributed_pretraining_b200.core.training import Config, Trainer
    opt_cfg = {"optimizer": optimizer}
    if optimizer == "shampoo":
        opt_cfg.update(start_preconditioning_step=2, update_period=2, beta2=0.95)   # roots at t = 2; t = 3, 4 reuse/refresh
    over = {"training__optimization": opt_cfg, "hp__iters": 8,
            "logging__steps": {"logging_interval": 10 ** 9, "checkpoint_interval": 3, "validation_interval": 0}}
    tr = make_trainer(tmp_path, **over)
    for step in range(3):
        tr.train_step(step, tr.data_manager.generate_batch(step))
    tr.save_checkpoint(3)
    saved = load_file(str(tmp_path / "smoke" / "checkpoints" / "step_3_optimizer.safetensors"))
    if optimizer == "shampoo":
        assert any(k.endswith("preconditioners.0") for k in saved) and any(k.endswith("statistics.1") for k in saved)
        assert any(float(v.abs().sum()) > 0 for k, v in saved.items() if k.endswith("preconditioners.0"))
    else:
        assert "alt_count" in saved and int(saved["alt_count"]) == 3
    tr.train_step(3, tr.data_manager.generate_batch(3))          # the uninterrupted run's 4th step
    want = masters(tr)

    cfg = tiny_config(**over)
    cfg["resume"] = {"checkpoint": str(tmp_path / "smoke" / "checkpoints" / "step_3")}
    tr2 = Trainer(Config.from_dict(cfg), synthetic=True, quiet=True, run_root=str(tmp_path / "resumed"))
    tr2._accum_step, tr2._accum_tokens = 0, 0
    assert tr2.load_checkpoint(cfg["resume"]["checkpoint"]) == 3
    assert tr2.optimizer.count == 3
    own = tr2.optimizer.state_dict()
    for n, t in saved.items():
        if n in own and own[n].is_cuda:
            assert torch.equal(own[n].detach().cpu(), t), n
    if optimizer == "hybrid":
        assert tr2.optimizer.non_matrix_optimizer.count == 3
    tr2.train_step(3, tr2.data_manager.generate_batch(3))
    got = masters(tr2)
    assert all(torch.equal(got[n], want[n]) for n in want), [n for n in want if not torch.equal(got[n], want[n])][:3]


def test_explicit_batch_path_never_reuses_a_pinned_buffer_in_flight(tmp_path):
    """Trainer._to_device (validation and the B200_PREFETCH=0 path): back-to-back host batches, no sync in
    between, must reach the device intact even when the CPU runs ahead of the GPU."""
    tr = make_trainer(tmp_path, optimizer="adamw")
    batches = [tr.data_manager.generate_batch(s) for s in range(12)]
    spin = torch.empty(64 << 20, device="cuda")
    devs = []
    for b in batches:
        for _ in range(4):
            spin.add_(1.0)              # keep the stream busy so the copies queue up behind compute
        devs.append(tr._to_device(b))
    torch.cuda.synchronize()
    assert all(torch.equal(d.cpu(), b) for d, b in zip(devs, batches))


@pytest.mark.parametrize("data,lr", [("uniform", None), ("markov", None), ("markov", 1e-3)])
def test_c1_loss_curve_matches_oracle(tmp_path, data, lr):
    """BASELINE configs[0]: Llama 2M + AdamW (configs/c1-llama2m-adamw.yaml), fp32 config, "1k iters synthetic
    tokens ... plumbing + loss parity".  The product Trainer runs the schedule on the GPU; the oracle's curves (CPU
    fp32, tests/golden/make_c1_curve.py, ~5 s/step on 4 cores, committed as tests/golden/c1_curve_*.json) are compared
    step by step.
      uniform          the BASELINE token stream (optimum ln 256: a fast decay onto a plateau)
      markov           a learnable stream (the loss keeps falling), config hyperparameters
      markov, lr 1e-3  control: same stream with a learning rate that does NOT blow up in the first steps
    With the config's own lr 2e-2 (AdamW without bias correction, no warm-up) the loss explodes to 9-10 around steps
    3-8; that transient is chaotic (the fp32 and fp64 ORACLES differ by 1-2 there, a 1e-6 weight perturbation moves
    step 6 by 3.9), so step-by-step agreement is
    asserted before it (steps 0-2) and after it has died out; on the learnable stream the two runs then sit in
    different basins and agree as trajectories (smoothed), not step by step.  The lr-1e-3 control has no such
    transient and must agree step by step throughout."""
    import yaml
    from mlx_cuda_distributed_pretraining_b200.core.training import Config, Trainer
    tag = data + (f"_lr{lr:g}" if lr is not None else "")
    fx = ROOT / "tests" / "golden" / f"c1_curve_{tag}.json"
    if not fx.exists():
        pytest.skip(f"{fx.name} not generated yet")
    ref = json.loads(fx.read_text())
    d = yaml.safe_load((ROOT / "configs" / "c1-llama2m-adamw.yaml").read_text())
    d["name"] = f"c1-curve-{tag}"
    d["data"]["input_file"] = "synthetic" if data == "uniform" else "synthetic:markov"
    d["training"]["hyperparameters"]["iters"] = ref["total_steps"]
    if lr is not None:
        d["training"]["hyperparameters"]["learning_rate"] = lr
    d["logging"]["steps"] = {"logging_interval": 10 ** 9, "checkpoint_interval": 0, "validation_interval": 0}
    tr = Trainer(Config.from_dict(d), synthetic=True, quiet=True, run_root=str(tmp_path))
    tr._accum_step, tr._accum_tokens = 0, 0
    n = min(ref["steps"], len(ref["loss"]))
    losses = []
    for step in range(n):
        loss, _, _ = tr.train_step(step, tr.data_manager.generate_batch(step))
        losses.append(loss)
    got = torch.stack(losses).float().cpu()
    want = torch.tensor(ref["loss"][:n])
    diff = (got - want).abs()
    k = 25
    smooth = lambda t: torch.nn.functional.avg_pool1d(t[None, None], k, 1)[0, 0] if len(t) >= k else t   # noqa: E731
    sdiff = (smooth(got) - smooth(want)).abs()
    (tmp_path / f"c1_curve_{tag}.json").write_text(json.dumps({
        "steps": n, "max_abs_diff": float(diff.max()), "argmax": int(diff.argmax()), "mean_abs_diff": float(diff.mean()),
        "head_0_2": float(diff[:3].max()), "max_30_99": float(diff[30:100].max()) if n > 100 else None,
        "max_from_100": float(diff[100:].max()) if n > 100 else None,
        "smoothed25_max_from_30": float(sdiff[30:].max()) if len(sdiff) > 30 else None,
        "final_gpu": float(got[-1]), "final_oracle": float(want[-1]), "first_gpu": float(got[0]),
        "first_oracle": float(want[0]), "loss_gpu": [round(float(x), 5) for x in got]}))
    assert torch.isfinite(got).all()
    assert float(diff[:3].max()) < C1_TOL["head"], diff[:3]          # before the blow-up: tight
    if lr is not None:                                                 # control: step by step, whole curve
        assert float(diff.max()) < C1_TOL["control"], (float(diff.max()), int(diff.argmax()))
    elif data == "uniform" and n > 200:
        assert float(diff[40:100].max()) < C1_TOL["settling"], float(diff[40:100].max())
        assert float(diff[100:].max()) < C1_TOL["settled"], (float(diff[100:].max()), int(diff[100:].argmax()) + 100)
        # SURVEY 8c's 1e-2, on the 25-step running mean of the signed difference (single steps sit on minibatch noise
        # of two runs whose weights parted in the transient)
        sm = (got - want)[100:].unfold(0, 25, 1).mean(dim=1).abs()
        assert float(sm.max()) < C1_TOL["tail"], (float(sm.max()), int(sm.argmax()) + 100)
    elif n > 100:
        # learnable stream at the config's lr: after the chaotic start the two runs are different realisations of the
        # same (still noisy: lr 2e-2) optimisation -- measured: per-step |d| up to 0.66, final 4.29 vs 3.65 at step 425.
        # Nothing step-wise can be asserted beyond "both learn"; the lr-1e-3 control below is the parity statement.
        assert float(got[-25:].mean()) < float(got[0]) - 1.0 and float(want[-25:].mean()) < float(want[0]) - 1.0


# |loss_gpu - loss_oracle| bounds.  The GPU run is itself not bit-reproducible (dQ is accumulated with fp32 atomics) and
# the config's chaotic first ~30 steps amplify that, so where the transient ends differs run to run.  One run on an
# H100 80GB HBM3 (700 W): uniform stream head 9.5e-3 (steps 0-2), steps 30-99 up to 0.023, steps >= 100 single-step
# 0.0048; lr-1e-3 control (no transient): 5.9e-4 over the whole curve, single steps.
C1_TOL = {"head": 3e-2, "settling": 0.15, "settled": 2e-2, "tail": 1e-2, "control": 1e-2}
