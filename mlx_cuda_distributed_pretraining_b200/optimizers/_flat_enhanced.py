"""What LionEnhanced, SGDEnhanced and mlx SGD share here: AdamW's flat-range surface (`init`, `init_range`,
`update_range`, `update`, `apply_gradients`, `step`, `state`, `state_dict`, `count`, `learning_rate`,
`grad_scale`, `use_accumulated`), the global-norm clip and the EMA weights of optimizers/enhanced_optimizers.py.

- Clip (:417-432, :285-300): one deterministic `b200_sumsq` launch (batch 1) over the optimizer's own range of the
  gradient source writes sum(g^2) to a device float; the update kernel turns it into min(1, c/(||g*gscale||+1e-6))
  itself.  No host synchronisation, and data-parallel replicas with identical gradients clip identically.
- EMA (:396-415): fp32, fused into the update pass, on the post-update parameters.  It is initialised on the
  optimizer's first update, so `count > 0` says whether it holds data and resume needs no extra field.
  Saved as `ema_params.<name>`; `get_ema_params()` returns it (None before the first update or when off).
"""
from __future__ import annotations

from typing import Callable, Dict, Optional, Union

import torch

from ..flat import ParamStore, get_store


class FlatEnhancedOptimizer:
    state_key: Optional[str] = None   # per-parameter fp32 state buffer ("exp_avg", "momentum_buffer") or none

    def __init__(self, learning_rate: Union[float, Callable], grad_clip_norm: Optional[float] = None,
                 ema_momentum: Optional[Union[float, Callable]] = None):
        self._learning_rate = learning_rate
        self.grad_clip_norm = grad_clip_norm
        self.ema_momentum = ema_momentum
        self.state: Dict[str, Dict[str, torch.Tensor]] = {}
        self.count = 0
        self.grad_scale = 1.0
        self.use_accumulated = False
        self._store: Optional[ParamStore] = None
        self._range = None
        self._buf = self._ema = self._ss = None

    @property
    def learning_rate(self) -> float:
        return self._lr(self.count)

    def _lr(self, count: int) -> float:
        lr = self._learning_rate(count) if callable(self._learning_rate) else self._learning_rate
        return float(lr)

    @property
    def clipping(self) -> bool:
        return self.grad_clip_norm is not None and self.grad_clip_norm > 0.0

    def init_range(self, store: ParamStore, lo: int, hi: int) -> None:
        if self._store is store and self._range == (lo, hi):
            return
        self._store, self._range = store, (lo, hi)
        dev = store.device
        self._buf = torch.zeros(store.total, dtype=torch.float32, device=dev) if self.state_key else None
        self._ema = torch.zeros(store.total, dtype=torch.float32, device=dev) if self.ema_momentum is not None else None
        self._ss = torch.zeros(1, dtype=torch.float32, device=dev) if self.clipping else None
        self._names = [n for n, (o, _s) in store.index.items() if lo <= o < hi]
        self.state = {n: {self.state_key: store.view(self._buf, n)} for n in self._names} if self.state_key else {}

    def init(self, model) -> None:
        store = get_store(model)
        self.init_range(store, 0, store.vec_end)

    @torch.no_grad()
    def update_range(self, store: ParamStore, lo: int, hi: int, gsrc: torch.Tensor, grad_scale: float) -> None:
        from .. import ops
        lr = self._lr(self.count)
        if self.clipping:
            ops.sumsq(gsrc[lo:hi], out=self._ss)
        ema_mode, ema_decay = 0, 0.0
        if self._ema is not None:
            ema_mode = 1 if self.count == 0 else 2
            d = self.ema_momentum
            ema_decay = float(d(self.count) if callable(d) else d)
        common = dict(gscale=grad_scale, clip_ss=self._ss, max_norm=self.grad_clip_norm if self.clipping else None,
                      ema_decay=ema_decay, ema_mode=ema_mode)
        self._apply(store, lo, hi, gsrc, lr, common)
        self.count += 1

    def _apply(self, store: ParamStore, lo: int, hi: int, gsrc: torch.Tensor, lr: float, common: dict) -> None:
        """One or more fused update launches over [lo, hi); `common` holds the gradient scale, clip and EMA
        arguments shared by ops.lion and ops.sgd."""
        raise NotImplementedError

    def _ema_slice(self, lo: int, hi: int) -> Optional[torch.Tensor]:
        return None if self._ema is None else self._ema[lo:hi]

    @torch.no_grad()
    def update(self, model, gradients=None) -> None:
        self.init(model)
        store = self._store
        if gradients is not None:
            store.load_gradients(gradients)
        gsrc = store.acc if self.use_accumulated else store.grad
        lo, hi = self._range
        self.update_range(store, lo, hi, gsrc, self.grad_scale)

    def apply_gradients(self, gradients, model):
        self.update(model, gradients)
        return model

    def step(self, model) -> None:
        self.update(model, None)

    def get_ema_params(self) -> Optional[Dict[str, torch.Tensor]]:
        if self._ema is None or self.count == 0:
            return None
        return {n: self._store.view(self._ema, n) for n in self._names}

    def state_dict(self) -> Dict[str, torch.Tensor]:
        out = {f"{n}.{k}": t for n, s in self.state.items() for k, t in s.items()}
        if self._ema is not None:
            out.update({f"ema_params.{n}": self._store.view(self._ema, n) for n in self._names})
        return out
