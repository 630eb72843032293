"""fp32 torch restatement of the reference's Lion / SGD optimizers (optimizers/enhanced_optimizers.py), the oracle
of the Lion, SGD and SGDEnhanced tests.  Written in the reference's order of operations, with Python-float
hyperparameters applied to fp32 tensors as mlx applies them, so it can be held to the fixture that runs the
reference itself (tests/golden/make_enhanced_golden.py -> enhanced_optimizer_vectors.npz).

Parameters and gradients are dicts keyed by flat name; updates are applied in place to `params` (D1, D2)."""
from __future__ import annotations

from typing import Callable, Dict, Optional, Union

import torch

Tensors = Dict[str, torch.Tensor]


def _value(x, count: int) -> float:
    return float(x(count)) if callable(x) else float(x)


def global_norm_clip(grads: Tensors, max_norm: Optional[float]) -> Tensors:
    """_clip_gradients (enhanced_optimizers.py:417-432, :285-300): scale every gradient by
    max_norm / (||g||_2 + 1e-6) when that is below 1; the norm runs over every gradient passed."""
    if max_norm is None or max_norm <= 0.0:
        return grads
    total = torch.sqrt(sum(torch.sum(torch.square(g)) for g in grads.values() if g is not None))
    coef = max_norm / (total + 1e-6)
    if coef < 1.0:
        grads = {k: (v * coef if v is not None else None) for k, v in grads.items()}
    return grads


def decay_excluded(name: str) -> bool:
    """enhanced_optimizers.py:275"""
    return name.endswith("bias") or ".norm" in name or ".ln" in name


class _EmaMixin:
    """_compute_ema (enhanced_optimizers.py:396-415, :248-267): ema := the post-update parameters on the first
    update, then ema = d*ema + (1-d)*p_new, with d = ema_momentum(count) if callable."""
    ema_momentum = None

    def _compute_ema(self, new_params: Tensors) -> None:
        if self.ema_momentum is None:
            return
        if "ema_params" not in self.state:
            self.state["ema_params"] = {k: v.clone() for k, v in new_params.items()}
        else:
            d = _value(self.ema_momentum, self.count)
            ema = self.state["ema_params"]
            for k, v in new_params.items():
                if k in ema:
                    ema[k] = d * ema[k] + (1 - d) * v

    def get_ema_params(self) -> Optional[Tensors]:
        return self.state.get("ema_params")


class LionOracle(_EmaMixin):
    """LionEnhanced.update (enhanced_optimizers.py:434-484).

    variant "reference" (as written, :465-475): u = b1 m + (1-b1) g ; m := u ; p += -lr sign(u); b2 unused; the weight
    decay of :471-472 is assigned to a discarded local, so it has no effect.
    variant "paper" (Chen et al. 2023): c = b1 m + (1-b1) g ; p = p (1 - lr wd) - lr sign(c) ; m = b2 m + (1-b2) g."""

    def __init__(self, learning_rate: Union[float, Callable] = 1e-4, betas=(0.9, 0.99), weight_decay: float = 0.0,
                 grad_clip_norm: Optional[float] = None, ema_momentum=None, variant: str = "reference"):
        if variant not in ("reference", "paper"):
            raise ValueError(variant)
        self.lr, self.betas, self.wd, self.clip = learning_rate, tuple(betas), weight_decay, grad_clip_norm
        self.ema_momentum, self.variant = ema_momentum, variant
        self.state: Dict = {}
        self.count = 0

    def update(self, params: Tensors, grads: Tensors) -> Tensors:
        if self.clip is not None:
            grads = global_norm_clip(grads, self.clip)
        lr = _value(self.lr, self.count)
        b1, b2 = self.betas
        updates = {}
        for name, p in params.items():
            g = grads.get(name)
            if g is None:
                continue
            st = self.state.setdefault(name, {"exp_avg": torch.zeros_like(p)})
            c = b1 * st["exp_avg"] + (1 - b1) * g
            if self.variant == "reference":
                st["exp_avg"] = c
                updates[name] = -lr * torch.sign(c)
                params[name] = p + updates[name]
            else:
                st["exp_avg"] = b2 * st["exp_avg"] + (1 - b2) * g
                params[name] = p * (1 - lr * self.wd) - lr * torch.sign(c)
                updates[name] = params[name] - p
        self._compute_ema({n: params[n] for n in params})
        self.count += 1
        return updates


class SGDEnhancedOracle(_EmaMixin):
    """SGDEnhanced.update (enhanced_optimizers.py:302-351): clip ; g += (wd*lr) p unless decay_excluded(name) ;
    buf = mu buf + (1-dampening) g ; p += -lr (nesterov ? g + mu buf : buf)."""

    def __init__(self, learning_rate: Union[float, Callable] = 1e-3, momentum: float = 0.9, weight_decay: float = 0.0,
                 nesterov: bool = False, grad_clip_norm: Optional[float] = None, dampening: float = 0.0,
                 ema_momentum=None):
        self.lr, self.mu, self.wd, self.nesterov = learning_rate, momentum, weight_decay, nesterov
        self.clip, self.dampening, self.ema_momentum = grad_clip_norm, dampening, ema_momentum
        self.state: Dict = {}
        self.count = 0

    def update(self, params: Tensors, grads: Tensors) -> Tensors:
        if self.clip is not None:
            grads = global_norm_clip(grads, self.clip)
        lr = _value(self.lr, self.count)
        updates = {}
        for name, p in params.items():
            g = grads.get(name)
            if g is None:
                continue
            if self.wd != 0.0 and not decay_excluded(name):
                g = g + (self.wd * lr) * p
            st = self.state.setdefault(name, {"momentum_buffer": torch.zeros_like(p)})
            buf = self.mu * st["momentum_buffer"] + (1.0 - self.dampening) * g
            st["momentum_buffer"] = buf
            u = -lr * (g + self.mu * buf) if self.nesterov else -lr * buf
            updates[name] = u
            params[name] = p + u
        self._compute_ema({n: params[n] for n in params})
        self.count += 1
        return updates


def mlx_sgd_step(params: Tensors, grads: Tensors, lr: float) -> None:
    """mlx.optimizers.SGD as core/training.py:891-894 builds it (learning rate only, so momentum 0):
    p = p - lr g (third-party behaviour, stated from mlx 0.25's documentation)."""
    for name, g in grads.items():
        if g is not None and name in params:
            params[name] = params[name] - lr * g


def lion_paper_fp64(p, m, g, lr, b1, b2, wd):
    """Chen et al. (2023), Algorithm 2, in fp64, independent of LionOracle: returns (p_new, m_new)."""
    p, m, g = p.double(), m.double(), g.double()
    c = b1 * m + (1.0 - b1) * g
    p_new = p - lr * (torch.sign(c) + wd * p)
    return p_new, b2 * m + (1.0 - b2) * g
