"""CPU: the Lion / SGD oracle against the reference's own outputs, Lion's paper variant against an fp64
statement of Chen et al., and the host logic of the new optimizers (factory, decay runs)."""
import json
from pathlib import Path

import numpy as np
import pytest
import torch

from tests import enhanced_optim_check as E

ROOT = Path(__file__).resolve().parents[1]


@pytest.fixture(scope="module")
def vectors():
    return np.load(ROOT / "tests" / "golden" / "enhanced_optimizer_vectors.npz")


def _oracle_for(cfg):
    kw = dict(cfg["kwargs"])
    base, k = cfg["lr"]
    sched = lambda s: base * (1.0 + k * s)  # noqa: E731
    if cfg["class"] == "LionEnhanced":
        return E.LionOracle(sched, variant="reference", **kw), "exp_avg"
    return E.SGDEnhancedOracle(sched, **kw), "momentum_buffer"


@pytest.mark.parametrize("case", ["lion", "sgd_nesterov", "sgd_plain"])
def test_oracle_matches_reference_vectors(vectors, case):
    cfg = json.loads(str(vectors[f"{case}_cfg"]))
    names = [str(n) for n in vectors["names"]]
    opt, key = _oracle_for(cfg)
    params = {n: torch.from_numpy(vectors[f"{case}_param0::{n}"]) for n in names}
    clipped = []
    for s in range(cfg["steps"]):
        grads = {n: torch.from_numpy(vectors[f"{case}_s{s}_grad::{n}"]) for n in names}
        assert opt.lr(s) == pytest.approx(float(vectors[f"{case}_s{s}_lr"]), rel=1e-15)
        opt.update(params, grads)
        clipped.append(int(vectors[f"{case}_s{s}_clipped"]))
        ema = opt.get_ema_params()
        for n in names:
            for what, got in (("param", params[n]), ("state", opt.state[n][key]), ("ema", ema[n])):
                want = torch.from_numpy(vectors[f"{case}_s{s}_{what}::{n}"])
                err = float((got - want).abs().max())
                assert err <= 5e-5, (case, s, what, n, err)
    assert 0 in clipped and 1 in clipped   # both sides of the clip are exercised


def test_reference_lion_ignores_weight_decay_and_b2(vectors):
    """LionEnhanced :471-472 discards its decayed parameter, and :465 never reads b2: the fixture (wd 0.1) equals the
    oracle run with wd 0 and any b2."""
    cfg = json.loads(str(vectors["lion_cfg"]))
    names = [str(n) for n in vectors["names"]]
    base, k = cfg["lr"]
    opt = E.LionOracle(lambda s: base * (1.0 + k * s), betas=(cfg["kwargs"]["betas"][0], 0.5), weight_decay=0.0,
                       grad_clip_norm=1.0, ema_momentum=0.9)
    params = {n: torch.from_numpy(vectors[f"lion_param0::{n}"]) for n in names}
    for s in range(cfg["steps"]):
        opt.update(params, {n: torch.from_numpy(vectors[f"lion_s{s}_grad::{n}"]) for n in names})
        for n in names:
            assert torch.equal(params[n], torch.from_numpy(vectors[f"lion_s{s}_param::{n}"])), (s, n)


def test_decay_exclusion_matches_only_bias_and_dotted_norm_names():
    assert E.decay_excluded("layers.0.mlp.up_proj.bias")
    assert E.decay_excluded("layers.0.ln_f.weight")
    assert not E.decay_excluded("norm.weight")
    assert not E.decay_excluded("layers.0.input_layernorm.weight")
    assert not E.decay_excluded("layers.0.post_attention_layernorm.weight")
    from mlx_cuda_distributed_pretraining_b200.optimizers.sgd import decay_excluded
    for n in ("a.bias", "x.ln_1.weight", "norm.weight", "layers.1.input_layernorm.weight", "model.norm.weight"):
        assert decay_excluded(n) == E.decay_excluded(n), n


def test_lion_paper_oracle_matches_fp64_chen_et_al():
    torch.manual_seed(0)
    p, g0 = torch.randn(4096), torch.randn(4096)
    opt = E.LionOracle(lambda s: 3e-3 / (1 + s), betas=(0.9, 0.99), weight_decay=0.1, variant="paper")
    params = {"w": p.clone()}
    p64, m64 = p.double(), torch.zeros(4096, dtype=torch.float64)
    for s in range(5):
        g = g0 * (s + 1) * 0.3 + torch.randn(4096)
        opt.update(params, {"w": g})
        p64, m64 = E.lion_paper_fp64(p64, m64, g, 3e-3 / (1 + s), 0.9, 0.99, 0.1)
        assert float((params["w"].double() - p64).abs().max()) < 1e-6
        assert float((opt.state["w"]["exp_avg"].double() - m64).abs().max() / m64.abs().max()) < 1e-6


def test_global_norm_clip_only_scales_down():
    g = {"a": torch.full((4,), 3.0), "b": torch.full((9,), 1.0)}   # ||g|| = sqrt(36 + 9)
    out = E.global_norm_clip(g, 1.0)
    assert float(torch.sqrt(sum((v ** 2).sum() for v in out.values()))) == pytest.approx(1.0, rel=1e-5)
    assert E.global_norm_clip(g, 100.0) is g
    assert E.global_norm_clip(g, None) is g and E.global_norm_clip(g, 0.0) is g


def _mk(opt, hp=None):
    from mlx_cuda_distributed_pretraining_b200.core.training import OptimizationManager, TrainingConfig
    tc = TrainingConfig(hyperparameters=hp or {"learning_rate": 1e-3, "batch_size": 1, "weight_decay": 0.1},
                        scheduler={"type": "cosine", "min_lr_ratio": 0.1}, optimization=opt)
    om = OptimizationManager(tc, 10)
    return om.create_optimizer(om.create_scheduler())


def test_factory_builds_lion_sgd_and_sgd_enhanced():
    from mlx_cuda_distributed_pretraining_b200.optimizers import SGD, HybridOptimizer, Lion, Muon, SGDEnhanced
    lion = _mk({"optimizer": "lion", "betas": [0.9, 0.95], "grad_clip_norm": 1.0, "ema_momentum": 0.999})
    assert isinstance(lion, Lion) and lion.betas == (0.9, 0.95) and lion.weight_decay == 0.1
    assert lion.grad_clip_norm == 1.0 and lion.ema_momentum == 0.999 and lion.lion_variant == "reference"
    assert _mk({"optimizer": "lion", "lion_variant": "paper"}).lion_variant == "paper"
    sgd = _mk({"optimizer": "sgd", "betas": [0.9, 0.95], "eps": 1e-8, "momentum": 0.5})
    assert type(sgd) is SGD and sgd.state_key is None and not sgd.clipping and sgd.ema_momentum is None
    se = _mk({"optimizer": "sgd_enhanced", "momentum": 0.8, "nesterov": True, "betas": [0.9, 0.95], "eps": 1e-8,
              "grad_clip_norm": 0.5, "ema_momentum": 0.99})
    assert isinstance(se, SGDEnhanced) and se.momentum == 0.8 and se.nesterov and se.weight_decay == 0.1
    assert se.dampening == 0.0 and se.grad_clip_norm == 0.5 and se.ema_momentum == 0.99
    d = _mk({"optimizer": "sgd_enhanced"})
    assert d.momentum == 0.9 and not d.nesterov and d.grad_clip_norm is None and d.ema_momentum is None
    h = _mk({"optimizer": "hybrid", "non_matrix_optimizer": "lion", "ema_momentum": 0.9})
    assert isinstance(h, HybridOptimizer) and isinstance(h.matrix_optimizer, Muon)
    assert isinstance(h.non_matrix_optimizer, Lion) and h.matrix_optimizer.alternate_optimizer is h.non_matrix_optimizer
    for nm, cls in (("sgd", SGD), ("sgd_enhanced", SGDEnhanced)):
        assert type(_mk({"optimizer": "hybrid", "non_matrix_optimizer": nm}).non_matrix_optimizer) is cls


def test_factory_rejects_unknown_lion_variant_and_sgd_extras():
    with pytest.raises(ValueError, match="lion_variant"):
        _mk({"optimizer": "lion", "lion_variant": "bogus"})
    for extra in ({"grad_clip_norm": 1.0}, {"ema_momentum": 0.99}):
        with pytest.raises(ValueError, match="sgd_enhanced"):
            _mk({"optimizer": "sgd", **extra})


def test_factory_accepts_the_reference_lion_config():
    """The optimization section of the reference's configs/model-config-1m-lion.yaml, which its own factory cannot
    construct (it forwards eps to LionEnhanced)."""
    from mlx_cuda_distributed_pretraining_b200.optimizers import Lion
    hp = {"learning_rate": 5.0e-4, "weight_decay": 0.01, "batch_size": 32, "gradient_clip": 1.0,
          "gradient_accumulation_steps": 1}
    opt = _mk({"optimizer": "lion", "betas": [0.9, 0.95], "eps": 1.0e-8, "grad_clip_norm": 1.0,
               "ema_momentum": 0.9999}, hp)
    assert isinstance(opt, Lion) and opt.weight_decay == 0.01 and opt.ema_momentum == 0.9999


def test_lion_reference_mode_logs_inert_weight_decay(caplog):
    from mlx_cuda_distributed_pretraining_b200.optimizers import Lion
    with caplog.at_level("WARNING"):
        Lion(1e-4, weight_decay=0.1)
    assert sum("has no effect" in r.message for r in caplog.records) == 1
    caplog.clear()
    with caplog.at_level("WARNING"):
        Lion(1e-4, weight_decay=0.1, lion_variant="paper")
        Lion(1e-4)
    assert not caplog.records


def test_sgd_enhanced_decay_runs_cover_the_range():
    from mlx_cuda_distributed_pretraining_b200.flat import ParamStore
    from mlx_cuda_distributed_pretraining_b200.optimizers.sgd import SGDEnhanced

    class Block(torch.nn.Module):
        def __init__(self):
            super().__init__()
            self.input_layernorm = torch.nn.Linear(8, 1)   # weight [1, 8] is 2-D; its bias [1] a vector
            self.up_bias = torch.nn.Parameter(torch.zeros(5))
            self.ln_f = torch.nn.Module()
            self.ln_f.weight = torch.nn.Parameter(torch.zeros(3))
            self.gain = torch.nn.Parameter(torch.zeros(6))

    m = torch.nn.Module()
    m.layers = torch.nn.ModuleList([Block()])
    m.norm = torch.nn.Module()
    m.norm.weight = torch.nn.Parameter(torch.zeros(4))
    store = ParamStore(m, torch.float32, "cpu")
    runs = SGDEnhanced.decay_runs(store, 0, store.vec_end)
    assert runs[0][0] == 0 and runs[-1][1] == store.vec_end
    assert all(a[1] == b[0] for a, b in zip(runs, runs[1:]))          # contiguous
    assert all(a[2] != b[2] for a, b in zip(runs, runs[1:]))          # maximal
    for name, (o, _s) in store.index.items():
        run = next(r for r in runs if r[0] <= o < r[1])
        assert run[2] == (not E.decay_excluded(name)), name
    no_bias = SGDEnhanced.decay_runs(store, 0, store.mat_end)
    assert no_bias == [(0, store.mat_end, True)]
