"""Lion with the surface of the reference's LionEnhanced (optimizers/enhanced_optimizers.py:358-488), built by
core/training.py:816-818 for `optimizer: lion`.  One fused launch per flat range (b200_lion).

`lion_variant="reference"` (default) is the reference as written (:465-475):

    m = b1 m + (1-b1) g ;  p -= lr * sign(m)                    (b2 is never read; sign(0) = 0)

Its weight decay (:471-472) rebinds a local variable that is then discarded, so it reaches neither the
parameters nor the EMA: in this mode `weight_decay` has no effect, and a non-zero value is logged once.
`lion_variant="paper"` is Lion as Chen et al. (2023) state it, the paper the reference's docstring cites:

    c = b1 m + (1-b1) g ;  p = p (1 - lr wd) - lr sign(c) ;  m = b2 m + (1-b2) g

`grad_clip_norm` and `ema_momentum` follow the reference (see _flat_enhanced).  `eps` is accepted and ignored:
the reference's factory forwards it to a constructor without such a parameter.
"""
from __future__ import annotations

import logging
from typing import Callable, Optional, Tuple, Union

from .. import ops
from ._flat_enhanced import FlatEnhancedOptimizer

LION_VARIANTS = ("reference", "paper")


class Lion(FlatEnhancedOptimizer):
    state_key = "exp_avg"

    def __init__(self, learning_rate: Union[float, Callable] = 1e-4, betas: Tuple[float, float] = (0.9, 0.99),
                 weight_decay: float = 0.0, grad_clip_norm: Optional[float] = None,
                 ema_momentum: Optional[Union[float, Callable]] = None, eps: Optional[float] = None,
                 lion_variant: str = "reference"):
        if lion_variant not in LION_VARIANTS:
            raise ValueError(f"lion_variant must be one of {LION_VARIANTS}, got {lion_variant!r}")
        super().__init__(learning_rate, grad_clip_norm, ema_momentum)
        self.betas = tuple(betas)
        self.weight_decay = weight_decay
        self.lion_variant = lion_variant
        if lion_variant == "reference" and weight_decay:
            logging.getLogger(__name__).warning(
                "lion_variant 'reference': weight_decay=%g has no effect, as in the reference's LionEnhanced; "
                "use lion_variant 'paper' for decoupled weight decay", weight_decay)

    def _apply(self, store, lo, hi, gsrc, lr, common) -> None:
        b1, b2 = self.betas
        if self.lion_variant == "reference":
            b_sign, b_mom, decay = b1, b1, 1.0
        else:
            b_sign, b_mom, decay = b1, b2, 1.0 - lr * self.weight_decay
        p16 = store.shadow[lo:hi] if store.mixed else None
        ops.lion(store.master[lo:hi], p16, gsrc[lo:hi], self._buf[lo:hi], lr, b_sign, b_mom, decay,
                 ema=self._ema_slice(lo, hi), **common)
