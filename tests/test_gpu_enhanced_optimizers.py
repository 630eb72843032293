"""-m gpu: b200_lion / b200_sgd against the fp32 oracle of tests/enhanced_optim_check.py, the optimizer classes
against the reference's own vectors, and Lion / SGD / SGDEnhanced / hybrid+Lion through the Trainer (tracking,
resume bit for bit, determinism, the CLI)."""
import json
import os
import subprocess
import sys
from pathlib import Path

import numpy as np
import pytest
import torch
import yaml

from oracle import reference_math as R
from tests import enhanced_optim_check as E
from tests.smoke_check import tiny_config

pytestmark = pytest.mark.gpu

ROOT = Path(__file__).resolve().parents[1]
DIMS = R.LlamaDims(128, 256, 2, 4, 2, 32, 259)
PAD = 8          # canary elements each side: keeps the view 16-byte aligned for fp32 and bf16
CANARY = 1024.0  # exact in bf16 and fp32
EPS32 = torch.finfo(torch.float32).eps


def _ops():
    from mlx_cuda_distributed_pretraining_b200 import ops
    ops.require_device()
    return ops


class Guarded:
    """A CUDA buffer of n + 2*PAD elements filled with CANARY; `.v` is the [PAD, PAD+n) view handed to a kernel."""

    def __init__(self, t: torch.Tensor, dtype):
        n = t.numel()
        self.full = torch.full((n + 2 * PAD,), CANARY, dtype=dtype, device="cuda")
        self.full[PAD:PAD + n] = t.to(dtype).cuda()
        self.v = self.full[PAD:PAD + n]

    def canary_ok(self) -> bool:
        return bool((self.full[:PAD] == CANARY).all()) and bool((self.full[-PAD:] == CANARY).all())

    def cpu(self) -> torch.Tensor:
        return self.v.float().cpu()


def _rel_ok(got, want, tol):
    """|got - want| <= tol * max(|want|, rms(want)) elementwise."""
    scale = torch.maximum(want.abs(), want.pow(2).mean().sqrt().expand_as(want))
    err = (got.double() - want.double()).abs()
    return bool((err <= tol * scale.double() + 1e-30).all()), float((err / (scale.double() + 1e-30)).max())


KINDS = ["lion_reference", "lion_paper", "sgd", "sgd_enhanced_nesterov", "sgd_enhanced"]


def _oracle(kind, lr, clip, ema):
    if kind.startswith("lion"):
        return E.LionOracle(lr, betas=(0.9, 0.99), weight_decay=0.1, grad_clip_norm=clip, ema_momentum=ema,
                            variant=kind.split("_")[1]), "exp_avg"
    if kind == "sgd":
        return None, None
    return E.SGDEnhancedOracle(lr, momentum=0.9, weight_decay=0.1, nesterov=kind.endswith("nesterov"),
                               grad_clip_norm=clip, ema_momentum=ema), "momentum_buffer"


def _launch(ops, kind, p, p16, g, st, ema, lr, gscale, ss, clip, ema_decay, ema_mode):
    common = dict(gscale=gscale, clip_ss=ss, max_norm=clip, ema=ema, ema_decay=ema_decay, ema_mode=ema_mode)
    if kind.startswith("lion"):
        paper = kind == "lion_paper"
        ops.lion(p, p16, g, st, lr, 0.9, 0.99 if paper else 0.9, 1.0 - lr * 0.1 if paper else 1.0, **common)
    elif kind == "sgd":
        ops.sgd(p, p16, g, None, lr, **common)
    else:
        ops.sgd(p, p16, g, st, lr, 0.9, 0.0, kind.endswith("nesterov"), lr * 0.1, **common)


def _check_master(kind, got, want, c_ref):
    if not kind.startswith("lion"):
        ok, worst = _rel_ok(got, want, 1e-6)
        assert ok, (kind, worst)
        return
    # a sign update: exact up to rounding wherever the oracle's sign argument is not tiny
    near0 = c_ref.abs() < 1e-6 * c_ref.pow(2).mean().sqrt()
    bad = (got - want).abs() > 4 * EPS32 * want.abs().clamp_min(1e-30)
    assert not bool((bad & ~near0).any()), (kind, int((bad & ~near0).sum()))
    assert int((bad & near0).sum()) <= max(1, got.numel() // 1000)


@pytest.mark.parametrize("shadow", [True, False])
@pytest.mark.parametrize("gdt", [torch.bfloat16, torch.float32])
@pytest.mark.parametrize("n", [1, 7, 8, 4099, (1 << 20) + 3])
@pytest.mark.parametrize("kind", KINDS)
def test_kernel_matches_oracle(kind, n, gdt, shadow):
    """Two steps (EMA initialised, then decayed) on canary-guarded buffers, gradient scale 0.5."""
    ops = _ops()
    gen = torch.Generator().manual_seed(n)
    p0 = torch.randn(n, generator=gen)
    lrs, gscale, ema_d = (3e-3, 2e-3), 0.5, 0.9
    P, P16 = Guarded(p0, torch.float32), (Guarded(p0, torch.bfloat16) if shadow else None)
    ST, EM = Guarded(torch.zeros(n), torch.float32), Guarded(torch.zeros(n), torch.float32)
    opt, key = _oracle(kind, lambda s: lrs[s], None, ema_d)
    params = {"w": p0.clone()}
    # The ABI carries the betas as fp32, so the kernel forms 1 - b from the rounded b: for b = 0.99 that complement
    # is 9e-7 off the exact one the oracle (like the reference) uses, and Lion's moment inherits it.
    state_tol = 1e-5 if kind.startswith("lion") else 1e-6
    for step in range(2):
        graw = torch.randn(n, generator=gen).to(gdt)
        G = Guarded(graw.float(), gdt)
        g_eff = graw.float() * gscale
        ema_prev = EM.cpu()
        _launch(ops, kind, P.v, P16.v if P16 else None, G.v, ST.v, EM.v, lrs[step], gscale, None, None, ema_d,
                1 if step == 0 else 2)
        c_ref = None
        if opt is None:
            E.mlx_sgd_step(params, {"w": g_eff}, lrs[step])
        else:
            m_prev = opt.state["w"][key].clone() if opt.state else torch.zeros(n)
            c_ref = 0.9 * m_prev + (1 - 0.9) * g_eff
            opt.update(params, {"w": g_eff})
        torch.cuda.synchronize()
        got = P.cpu()
        _check_master(kind, got, params["w"], c_ref)
        if opt is not None:
            ok, worst = _rel_ok(ST.cpu(), opt.state["w"][key], state_tol)
            assert ok, ("state", worst)
        # the EMA recurrence on the kernel's own weights (a Lion sign flip near zero legitimately moves the master)
        ema_ref = got if step == 0 else ema_d * ema_prev + (1 - ema_d) * got
        ok, worst = _rel_ok(EM.cpu(), ema_ref, 1e-6)
        assert ok, ("ema", worst)
        if P16 is not None:
            assert torch.equal(P16.v.cpu(), P.v.cpu().to(torch.bfloat16))
        for b in (P, P16, ST, EM, G):
            assert b is None or b.canary_ok()


@pytest.mark.parametrize("kind", ["lion_reference", "lion_paper", "sgd_enhanced_nesterov"])
@pytest.mark.parametrize("max_norm", [5.0, 1e4])   # below / above the gradient norm (~ 0.5 * sqrt(n))
def test_global_norm_clip_matches_oracle(kind, max_norm):
    ops = _ops()
    n = 10007
    gen = torch.Generator().manual_seed(3)
    p0, graw = torch.randn(n, generator=gen), torch.randn(n, generator=gen).to(torch.bfloat16)
    P, G, ST = Guarded(p0, torch.float32), Guarded(graw.float(), torch.bfloat16), Guarded(torch.zeros(n), torch.float32)
    ss = ops.sumsq(G.v)
    _launch(ops, kind, P.v, None, G.v, ST.v, None, 1e-3, 0.5, ss, max_norm, 0.0, 0)
    opt, key = _oracle(kind, 1e-3, max_norm, None)
    params, g_eff = {"w": p0.clone()}, graw.float() * 0.5
    clipped = E.global_norm_clip({"w": g_eff}, max_norm)["w"]
    assert (clipped is g_eff) == (max_norm > 1e3)
    opt.update(params, {"w": g_eff})
    torch.cuda.synchronize()
    _check_master(kind, P.cpu(), params["w"], 0.9 * torch.zeros(n) + (1 - 0.9) * clipped)
    ok, worst = _rel_ok(ST.cpu(), opt.state["w"][key], 1e-5)   # the norm's summation order differs
    assert ok, worst
    assert P.canary_ok() and G.canary_ok()


def _flat_module(shapes):
    root = torch.nn.Module()
    for name, shape in shapes.items():
        *path, leaf = name.split(".")
        m = root
        for part in path:
            if not hasattr(m, part):
                m.add_module(part, torch.nn.Module())
            m = getattr(m, part)
        m.register_parameter(leaf, torch.nn.Parameter(torch.zeros(shape, device="cuda")))
    return root


@pytest.mark.parametrize("case", ["lion", "sgd_nesterov", "sgd_plain"])
def test_optimizer_classes_match_reference_vectors(case):
    """The reference's own LionEnhanced / SGDEnhanced outputs (tests/golden/enhanced_optimizer_vectors.npz): flat
    names with `*.bias`, `.ln`, `norm.weight` and `input_layernorm.weight` (so SGDEnhanced splits its launch by decay
    flag), clipping on and off, EMA, a schedule; the whole update runs with host synchronisation forbidden."""
    _ops()
    from mlx_cuda_distributed_pretraining_b200.flat import get_store
    from mlx_cuda_distributed_pretraining_b200.optimizers import Lion, SGDEnhanced
    vec = np.load(ROOT / "tests" / "golden" / "enhanced_optimizer_vectors.npz")
    cfg = json.loads(str(vec[f"{case}_cfg"]))
    names = [str(x) for x in vec["names"]]
    model = _flat_module({n: vec[f"{case}_param0::{n}"].shape for n in names})
    base, k = cfg["lr"]
    kw = dict(cfg["kwargs"])
    if cfg["class"] == "LionEnhanced":
        opt, key = Lion(lambda s: base * (1.0 + k * s), **{**kw, "betas": tuple(kw["betas"])}), "exp_avg"
    else:
        opt, key = SGDEnhanced(lambda s: base * (1.0 + k * s), **kw), "momentum_buffer"
    store = get_store(model)
    with torch.no_grad():
        for n in names:
            store.view(store.master, n).copy_(torch.from_numpy(vec[f"{case}_param0::{n}"]))
    opt.init(model)
    if key == "momentum_buffer":
        assert len(opt._runs) > 1
    for s in range(cfg["steps"]):
        with torch.no_grad():
            for n in names:
                store.view(store.grad, n).copy_(torch.from_numpy(vec[f"{case}_s{s}_grad::{n}"]))
        torch.cuda.synchronize()
        torch.cuda.set_sync_debug_mode("error")
        try:
            opt.update(model)
        finally:
            torch.cuda.set_sync_debug_mode("default")
        ema = opt.get_ema_params()
        for n in names:
            want = torch.from_numpy(vec[f"{case}_s{s}_param::{n}"])
            got = store.view(store.master, n).cpu()
            if key == "exp_avg":
                assert float((got - want).abs().max()) <= 4 * EPS32 * float(want.abs().max()), (s, n)
            else:
                ok, worst = _rel_ok(got, want, 1e-5)
                assert ok, (s, n, worst)
            for what, t in (("state", opt.state[n][key]), ("ema", ema[n])):
                ok, worst = _rel_ok(t.cpu(), torch.from_numpy(vec[f"{case}_s{s}_{what}::{n}"]), 1e-5)
                assert ok, (s, n, what, worst)
    assert opt.count == cfg["steps"]


# ---- through the Trainer -------------------------------------------------------------------------
def make_trainer(tmp_path, **kw):
    from mlx_cuda_distributed_pretraining_b200.core.training import Config, Trainer
    tr = Trainer(Config.from_dict(tiny_config(**kw)), synthetic=True, quiet=True, run_root=str(tmp_path))
    tr._accum_step, tr._accum_tokens = 0, 0
    return tr


def masters(tr):
    return {n: t.detach().cpu().clone() for n, t in tr.store.named_master().items()}


def _cos(a, b):
    a, b = a.flatten().double(), b.flatten().double()
    return float(a @ b / (a.norm() * b.norm() + 1e-30))


TRACK = {
    "lion": {"optimizer": "lion", "betas": [0.9, 0.99], "ema_momentum": 0.9, "grad_clip_norm": 0.5},
    "lion_paper": {"optimizer": "lion", "lion_variant": "paper", "betas": [0.9, 0.99], "ema_momentum": 0.9},
    "sgd": {"optimizer": "sgd"},
    "sgd_enhanced": {"optimizer": "sgd_enhanced", "nesterov": True, "grad_clip_norm": 0.5, "ema_momentum": 0.9},
    "hybrid_lion": {"optimizer": "hybrid", "non_matrix_optimizer": "lion", "ema_momentum": 0.9,
                    "grad_clip_norm": 0.5},
}


@pytest.mark.parametrize("name", list(TRACK))
def test_trainer_steps_track_oracle(tmp_path, name):
    """Each step from the CUDA run's own weights and optimizer state; the oracle is fed fp32 CPU gradients. The
    momentum (linear in g) must track tightly, the step must point the same way for every tensor, and the EMA must
    follow the oracle's recurrence on the CUDA run's weights."""
    opt_cfg = TRACK[name]
    lr = 2e-3 if "lion" in name else 5e-2
    tr = make_trainer(tmp_path, mixed=False, hp__learning_rate=lr, training__optimization=opt_cfg)
    tr.optimizer.init(tr.model)
    core = tr.optimizer.non_matrix_optimizer if name == "hybrid_lion" else tr.optimizer
    own = set(core._names)
    key = core.state_key
    kw = {k: v for k, v in opt_cfg.items() if k in ("grad_clip_norm", "ema_momentum")}
    for step in range(4):
        batch = tr.data_manager.generate_batch(step)
        before = masters(tr)
        ema_before = {n: t.cpu().clone() for n, t in (core.get_ema_params() or {}).items()}
        if name.startswith("lion") or name == "hybrid_lion":
            opt = E.LionOracle(tr.lr_schedule, betas=(0.9, 0.99), weight_decay=0.01,
                               variant=opt_cfg.get("lion_variant", "reference"), **kw)
        elif name == "sgd_enhanced":
            opt = E.SGDEnhancedOracle(tr.lr_schedule, momentum=0.9, weight_decay=0.01, nesterov=True, **kw)
        else:
            opt = None
        if opt is not None:
            opt.count = step
            opt.state = {n: {key: s[key].cpu().clone()} for n, s in core.state.items()}
            if ema_before:
                opt.state["ema_params"] = dict(ema_before)
        loss, _, _ = tr.train_step(step, batch)
        loss_ref, _, grads = R.loss_and_grads(before, batch, DIMS, pad_token=256)
        assert abs(float(loss) - float(loss_ref)) < 2e-2, step
        after_ref = {n: before[n].clone() for n in own}
        if opt is None:
            E.mlx_sgd_step(after_ref, {n: grads[n] for n in own}, tr.lr_schedule(step))
        else:
            opt.update(after_ref, {n: grads[n] for n in own})
        after = masters(tr)
        for n in own:
            if opt is not None:
                assert R_rel(core.state[n][key], opt.state[n][key]) < 0.1, (step, n)
            c = _cos(after[n] - before[n], after_ref[n] - before[n])
            assert c > (0.8 if "lion" in name else 0.9), (step, n, c)
        if "ema_momentum" in opt_cfg:
            ema = core.get_ema_params()
            for n in own:
                want = after[n] if step == 0 else 0.9 * ema_before[n] + (1 - 0.9) * after[n]
                ok, worst = _rel_ok(ema[n].cpu(), want, 1e-6)
                assert ok, (step, n, worst)
    assert core.count == 4


def R_rel(a, b):
    a, b = a.detach().double().cpu(), b.detach().double().cpu()
    return float((a - b).norm() / (b.norm() + 1e-30))


RESUME = {
    "lion": {"optimizer": "lion", "ema_momentum": 0.9, "grad_clip_norm": 0.5},
    "sgd_enhanced": {"optimizer": "sgd_enhanced", "ema_momentum": 0.9, "grad_clip_norm": 0.5, "nesterov": True},
    "sgd": {"optimizer": "sgd"},
    "hybrid_lion": {"optimizer": "hybrid", "non_matrix_optimizer": "lion", "ema_momentum": 0.9,
                    "lion_variant": "paper"},
}


@pytest.mark.parametrize("name", list(RESUME))
def test_resume_is_bit_exact_and_runs_are_deterministic(tmp_path, name):
    from safetensors.torch import load_file
    from mlx_cuda_distributed_pretraining_b200.core.training import Config, Trainer
    over = {"training__optimization": RESUME[name], "hp__iters": 8, "hp__gradient_clip": 1.0,
            "logging__steps": {"logging_interval": 10 ** 9, "checkpoint_interval": 3, "validation_interval": 0}}
    tr = make_trainer(tmp_path / "a", **over)
    for step in range(3):
        tr.train_step(step, tr.data_manager.generate_batch(step))
    tr.save_checkpoint(3)
    saved = load_file(str(tmp_path / "a" / "smoke" / "checkpoints" / "step_3_optimizer.safetensors"))
    if "ema_momentum" in RESUME[name]:
        ema_keys = [k for k in saved if k.startswith("ema_params.")]
        assert ema_keys and all(float(saved[k].abs().sum()) > 0 for k in ema_keys)
    if name == "hybrid_lion":
        assert int(saved["alt_count"]) == 3 and not any(k.startswith("ema_params.layers.0.self_attn") for k in saved)
    tr.train_step(3, tr.data_manager.generate_batch(3))
    want = masters(tr)

    twin = make_trainer(tmp_path / "b", **over)   # an identical run
    for step in range(4):
        twin.train_step(step, twin.data_manager.generate_batch(step))
    assert all(torch.equal(masters(twin)[n], want[n]) for n in want)

    cfg = tiny_config(**over)
    cfg["resume"] = {"checkpoint": str(tmp_path / "a" / "smoke" / "checkpoints" / "step_3")}
    tr2 = Trainer(Config.from_dict(cfg), synthetic=True, quiet=True, run_root=str(tmp_path / "resumed"))
    tr2._accum_step, tr2._accum_tokens = 0, 0
    assert tr2.load_checkpoint(cfg["resume"]["checkpoint"]) == 3
    own = tr2.optimizer.state_dict()
    for n, t in saved.items():
        if n in own and own[n].is_cuda:
            assert torch.equal(own[n].detach().cpu(), t), n
    if name == "hybrid_lion":
        assert tr2.optimizer.non_matrix_optimizer.count == 3
    tr2.train_step(3, tr2.data_manager.generate_batch(3))
    got = masters(tr2)
    assert all(torch.equal(got[n], want[n]) for n in want), [n for n in want if not torch.equal(got[n], want[n])][:3]
    core = tr2.optimizer.non_matrix_optimizer if name == "hybrid_lion" else tr2.optimizer
    ema = core.get_ema_params()
    if "ema_momentum" in RESUME[name]:
        ema_want = tr.optimizer.state_dict()
        assert all(torch.equal(t.cpu(), ema_want[f"ema_params.{n}"].cpu()) for n, t in ema.items())
    else:
        assert ema is None


def test_cli_trains_lion_and_checkpoints_ema(tmp_path):
    cfg = tiny_config(name="lion-cli", training__optimization={"optimizer": "lion", "betas": [0.9, 0.95], "eps": 1e-8,
                                                              "grad_clip_norm": 1.0, "ema_momentum": 0.999},
                      logging__steps={"logging_interval": 5, "checkpoint_interval": 10, "validation_interval": 0})
    path = tmp_path / "lion.yaml"
    path.write_text(yaml.safe_dump(cfg))
    env = dict(os.environ, PYTHONPATH=str(ROOT))
    r = subprocess.run([sys.executable, "-m", "core.training", "--config", str(path), "--synthetic", "--iters", "20"],
                       cwd=tmp_path, env=env, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-2000:]
    ckpts = sorted(tmp_path.rglob("*_optimizer.safetensors"))
    assert ckpts, list(tmp_path.rglob("*"))
    from safetensors.torch import load_file
    st = load_file(str(ckpts[-1]))
    assert any(k.startswith("ema_params.") for k in st) and any(k.endswith(".exp_avg") for k in st)
    assert all(torch.isfinite(v.float()).all() for v in st.values())
