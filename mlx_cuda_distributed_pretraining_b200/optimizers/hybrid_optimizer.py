"""HybridOptimizer (optimizers/hybrid_optimizer.py:78-114): 2-D parameters -> matrix optimizer
(Muon), everything else -> non-matrix optimizer (AdamW, Lion, SGD or SGDEnhanced: anything with AdamW's
`init_range` / `update_range` surface).  The reference's factory recursion for
`optimizer: hybrid` crashes (SURVEY D12); the routing it intended is exactly Muon's
`alternate_optimizer` hook, so this class is a thin composition.

Checkpointing: `state_dict()` holds both sub-optimizers' tensors plus `alt_count` (the non-matrix
optimizer's own step counter drives its schedule, bias correction and EMA initialisation); `count` is
settable so the trainer's resume path (`optimizer.count = saved`) restores the matrix optimizer's counter."""
from __future__ import annotations

import torch

from .muon import Muon

_FORWARDED = ("grad_scale", "use_accumulated", "shard_ns")


class HybridOptimizer:
    def __init__(self, learning_rate=None, matrix_optimizer: Muon = None, non_matrix_optimizer=None):
        """non_matrix_optimizer: AdamW-like (AdamW, Lion, SGD, SGDEnhanced)."""
        if matrix_optimizer is None or non_matrix_optimizer is None:
            raise ValueError("HybridOptimizer needs a matrix_optimizer and a non_matrix_optimizer")
        if not isinstance(matrix_optimizer, Muon):
            raise ValueError("matrix_optimizer must be Muon (Newton-Schulz); Shampoo routes all params itself")
        self.matrix_optimizer = matrix_optimizer
        self.non_matrix_optimizer = non_matrix_optimizer
        matrix_optimizer.alternate_optimizer = non_matrix_optimizer

    # -- counters --------------------------------------------------------------------------------
    @property
    def count(self) -> int:
        return self.matrix_optimizer.count

    @count.setter
    def count(self, value: int) -> None:
        self.matrix_optimizer.count = int(value)

    @property
    def learning_rate(self) -> float:
        return self.matrix_optimizer.learning_rate

    @property
    def state(self):
        s = dict(self.matrix_optimizer.state)
        s.update(self.non_matrix_optimizer.state)
        return s

    # data-parallel / accumulation switches set by the trainer apply to the optimizer doing the work
    def __getattr__(self, k):
        if k in _FORWARDED and "matrix_optimizer" in self.__dict__:
            return getattr(self.__dict__["matrix_optimizer"], k)
        raise AttributeError(k)

    def __setattr__(self, k, v):
        if k in _FORWARDED and "matrix_optimizer" in self.__dict__:
            setattr(self.matrix_optimizer, k, v)
            return
        object.__setattr__(self, k, v)

    def owned_ranges_of(self, *a, **kw):
        return self.matrix_optimizer.owned_ranges_of(*a, **kw)

    @property
    def exchange_mode(self) -> str:
        return self.matrix_optimizer.exchange_mode

    # -- reference surface -----------------------------------------------------------------------
    def init(self, model) -> None:
        self.matrix_optimizer.init(model)   # also sizes the alternate optimizer's range

    def update(self, model, gradients=None):
        self.matrix_optimizer.update(model, gradients)

    def apply_gradients(self, gradients, model):
        self.update(model, gradients)
        return model

    def step(self, model):
        self.update(model, None)

    def state_dict(self):
        out = self.matrix_optimizer.state_dict()   # includes the alternate optimizer's m / v
        out["alt_count"] = torch.tensor([self.non_matrix_optimizer.count], dtype=torch.int64)
        return out

    def load_extra_state(self, tensors) -> None:
        """Entries of a saved state dict that are not views of optimizer buffers."""
        if "alt_count" in tensors:
            self.non_matrix_optimizer.count = int(tensors["alt_count"].item())
