"""Generates tests/golden/enhanced_optimizer_vectors.npz by RUNNING THE REFERENCE'S OWN PYTHON: the unmodified
optimizers/enhanced_optimizers.py (LionEnhanced :358-488, SGDEnhanced :200-355) over the NumPy mlx stand-in of
oracle/mlx_numpy_shim, as make_golden.py does.  tests/test_enhanced_optim_oracle.py holds
tests/enhanced_optim_check.py to these vectors.  Needs the reference tree, so it runs where that is available:

    python tests/golden/make_enhanced_golden.py /path/to/reference

Every case runs STEPS updates with a schedule callable on a flat-named module: gradients are passed as a dict keyed
by flat name and the returned updates are added to the parameters by hand (D1, D2).  Gradients alternate between
scale 1 (global norm ~20: the clip at 1.0 is active) and scale 0.02 (norm ~0.4: inactive).  The names include
`*.bias`, `.ln`, `norm.weight` and `layers.0.input_layernorm.weight`, which pin SGDEnhanced's decay exclusion.
"""
import json
import sys
from pathlib import Path

import numpy as np

HERE = Path(__file__).resolve().parent
REPO = HERE.parents[1]
if len(sys.argv) != 2:
    sys.exit("usage: python tests/golden/make_enhanced_golden.py <reference checkout>")
REF = Path(sys.argv[1]).resolve()

sys.path = [p for p in sys.path if p not in ("", str(REPO)) and Path(p or ".").resolve() != REPO]
sys.path.insert(0, str(REF))
sys.path.insert(0, str(REPO / "oracle" / "mlx_numpy_shim"))

import mlx.core as mx  # noqa: E402  (the shim)
import mlx.nn as nn  # noqa: E402

if not hasattr(mx, "sign"):
    # the one primitive enhanced_optimizers.py needs beyond the shim's set (LionEnhanced :475); sign(0) = 0
    mx.sign = lambda a: mx._w(np.sign(a).astype(np.float32))

from optimizers.enhanced_optimizers import LionEnhanced, SGDEnhanced  # noqa: E402

SHAPES = {
    "embed_tokens.weight": (12, 16),
    "layers.0.input_layernorm.weight": (16,),
    "layers.0.mlp.up_proj.bias": (13,),
    "layers.0.self_attn.o_proj.weight": (16, 8),
    "layers.0.ln_f.weight": (7,),
    "norm.weight": (16,),
}
STEPS = 4
GRAD_SCALES = (1.0, 0.02, 1.0, 0.02)

CASES = {
    "lion": (LionEnhanced, dict(betas=(0.9, 0.95), weight_decay=0.1, grad_clip_norm=1.0, ema_momentum=0.9),
             lambda s: 1e-3 * (1.0 + 0.5 * s)),
    "sgd_nesterov": (SGDEnhanced, dict(momentum=0.9, weight_decay=0.05, nesterov=True, grad_clip_norm=1.0,
                                       ema_momentum=0.9), lambda s: 0.05 * (1.0 + 0.5 * s)),
    "sgd_plain": (SGDEnhanced, dict(momentum=0.8, weight_decay=0.05, nesterov=False, grad_clip_norm=1.0,
                                    ema_momentum=0.95), lambda s: 0.05 * (1.0 + 0.5 * s)),
}
LR_FORMULA = {"lion": [1e-3, 0.5], "sgd_nesterov": [0.05, 0.5], "sgd_plain": [0.05, 0.5]}  # base * (1 + k*step)

rng = np.random.default_rng(2024)
out = {"names": np.array(list(SHAPES))}
for case, (cls, kw, sched) in CASES.items():
    params = {k: (rng.standard_normal(s) * 0.5).astype(np.float32) for k, s in SHAPES.items()}
    for k, v in params.items():
        out[f"{case}_param0::{k}"] = v
    model = nn.Module({k: mx.array(v) for k, v in params.items()})
    opt = cls(learning_rate=sched, **kw)
    state_key = "exp_avg" if cls is LionEnhanced else "momentum_buffer"
    for step in range(STEPS):
        grads = {k: (rng.standard_normal(s) * GRAD_SCALES[step]).astype(np.float32) for k, s in SHAPES.items()}
        upd = opt.update(model, {k: mx.array(v) for k, v in grads.items()})
        for k in SHAPES:   # the reference returns updates; applying them is the caller's job (D2)
            setattr(model, k, mx.array(np.asarray(getattr(model, k)) + np.asarray(upd[k])))
        norm = float(np.sqrt(sum(np.sum(np.square(g, dtype=np.float64)) for g in grads.values())))
        out[f"{case}_s{step}_clipped"] = np.array(int(kw["grad_clip_norm"] / (norm + 1e-6) < 1.0))
        out[f"{case}_s{step}_lr"] = np.array(sched(step), dtype=np.float64)
        for k in SHAPES:
            out[f"{case}_s{step}_grad::{k}"] = grads[k]
            out[f"{case}_s{step}_param::{k}"] = np.asarray(getattr(model, k)).astype(np.float32)
            out[f"{case}_s{step}_state::{k}"] = np.asarray(opt.state[k][state_key]).astype(np.float32)
            out[f"{case}_s{step}_ema::{k}"] = np.asarray(opt.get_ema_params()[k]).astype(np.float32)
    out[f"{case}_cfg"] = np.array(json.dumps({"class": cls.__name__, "kwargs": kw, "lr": LR_FORMULA[case],
                                              "steps": STEPS}))

np.savez_compressed(HERE / "enhanced_optimizer_vectors.npz", **out)
print(f"wrote {HERE / 'enhanced_optimizer_vectors.npz'} with {len(out)} arrays")
