"""SGD for `optimizer: sgd` and `optimizer: sgd_enhanced` (core/training.py:891-894, :809-815), one fused launch
per flat range (b200_sgd).

`SGD` is what the reference's factory builds for `sgd`: mlx.optimizers.SGD given only the learning rate, so
`p -= lr g` with no state (third-party behaviour, stated from mlx 0.25's documentation).

`SGDEnhanced` is optimizers/enhanced_optimizers.py:200-355 as written:

    g += lr*wd*p          (coupled, before the momentum; skipped for names ending in `bias` or containing
                           `.norm` / `.ln` -- with this model's flat names only `*.bias` matches, so
                           `input_layernorm.weight` and `norm.weight` ARE decayed)
    buf = mu buf + (1-dampening) g ;  p -= lr (nesterov ? g + mu buf : buf)

This is not Muon's `(1-mu) g + mu buf` fallback.  The decay exclusion is applied by range: one launch per
maximal run of entries with the same flag (a single launch when the model has no biases).
`grad_clip_norm` and `ema_momentum` follow the reference (see _flat_enhanced).  `betas` / `eps` are accepted
and ignored: the reference's factory forwards them to constructors without such parameters.
"""
from __future__ import annotations

from typing import Callable, List, Optional, Tuple, Union

from .. import ops
from ._flat_enhanced import FlatEnhancedOptimizer


def decay_excluded(name: str) -> bool:
    """SGDEnhanced._apply_weight_decay's name test (enhanced_optimizers.py:275)."""
    return name.endswith("bias") or ".norm" in name or ".ln" in name


class SGD(FlatEnhancedOptimizer):
    def __init__(self, learning_rate: Union[float, Callable] = 1e-3, betas: Optional[Tuple[float, float]] = None,
                 eps: Optional[float] = None):
        super().__init__(learning_rate)

    def _apply(self, store, lo, hi, gsrc, lr, common) -> None:
        p16 = store.shadow[lo:hi] if store.mixed else None
        ops.sgd(store.master[lo:hi], p16, gsrc[lo:hi], None, lr, **common)


class SGDEnhanced(FlatEnhancedOptimizer):
    state_key = "momentum_buffer"

    def __init__(self, learning_rate: Union[float, Callable] = 1e-3, momentum: float = 0.9,
                 weight_decay: float = 0.0, nesterov: bool = False, grad_clip_norm: Optional[float] = None,
                 dampening: float = 0.0, ema_momentum: Optional[Union[float, Callable]] = None,
                 betas: Optional[Tuple[float, float]] = None, eps: Optional[float] = None):
        super().__init__(learning_rate, grad_clip_norm, ema_momentum)
        self.momentum = momentum
        self.weight_decay = weight_decay
        self.nesterov = nesterov
        self.dampening = dampening

    def init_range(self, store, lo: int, hi: int) -> None:
        if self._store is store and self._range == (lo, hi):
            return
        super().init_range(store, lo, hi)
        self._runs = self.decay_runs(store, lo, hi)

    @staticmethod
    def decay_runs(store, lo: int, hi: int) -> List[Tuple[int, int, bool]]:
        """[(a, b, decayed)] covering [lo, hi): maximal runs of consecutive entries with the same decay flag.
        Alignment padding after an entry belongs to that entry's run."""
        entries = sorted((o, not decay_excluded(n)) for n, (o, _s) in store.index.items() if lo <= o < hi)
        runs: List[Tuple[int, int, bool]] = []
        for o, flag in entries:
            if runs and runs[-1][2] == flag:
                continue
            if runs:
                runs[-1] = (runs[-1][0], o, runs[-1][2])
            runs.append((lo if not runs else o, hi, flag))
        return runs or [(lo, hi, True)]

    def _apply(self, store, lo, hi, gsrc, lr, common) -> None:
        wd_c = lr * self.weight_decay
        for a, b, decayed in self._runs:
            p16 = store.shadow[a:b] if store.mixed else None
            ops.sgd(store.master[a:b], p16, gsrc[a:b], self._buf[a:b], lr, self.momentum, self.dampening,
                    self.nesterov, wd_c if decayed else 0.0, ema=self._ema_slice(a, b), **common)
