"""Shampoo with the reference's surface (optimizers/shampoo.py:20-45,143-378) on the sm_90a GEMM
engine, orchestrated through the C ABI's b200_shampoo_* entry points (include/b200_hotpath.h).

    opt = Shampoo(learning_rate=float|callable, params=ShampooParams(...))
    opt.update(model, gradients)     # core/training.py:1690,1700

Per step (shampoo.py:314-378, with the wiring defects D1/D2/D9 of SURVEY 2.3 fixed):
  count += 1; lr = sched(count)
  grafting direction d = Adam step (mlx Adam, no bias correction) computed WITHOUT applying it
  L = b2 L + (1-b2) G G^T ; R = b2 R + (1-b2) G^T G       on G[:1024,:1024]   (:229-255)  b200_shampoo_stats
  every `update_period` steps after `start_preconditioning_step`:                          b200_shampoo_root
        P = matrix_inverse_pth_root(stat)  -- the reference's literal formula (:88-126):
        Z0 = (M+eps I)/tr ; 6x Z <- Z + Z Z / p ; P = Z * tr^(-1/p^2)        (not a true inverse root)
        or, inverse_root="newton": P = (M + ridge I)^(-1/4) by coupled Newton    b200_shampoo_root_newton
  m = b1 m + (1-b1) g ; mhat = m/(1-b1^t) ; pre = mhat with pre[:1024,:1024] = PL mhat PR   (:257-295)
                                                                                           b200_shampoo_precond
  upd = -lr*pre rescaled to ||d||_F (grafting, :297-312) ; decoupled wd: upd -= lr*wd*p     (:372-373)
                                                                                           b200_shampoo_graft

All matrix products are batched over the same-shape parameters of a flat.ParamStore group and run on
wgmma.  fp32 matrices enter the tensor cores as bf16 hi+lo pairs (hi*hi + hi*lo + lo*hi, three
accumulating GEMMs, ~16 mantissa bits) so statistics/roots stay close to the reference's fp32 matmuls;
bf16 gradients (mixed precision) are used as they are, fp32 gradients are split the same way.
State per parameter mirrors the reference's (:180-208): momentum, statistics.0/1, preconditioners.0/1
(+ the grafting optimizer's moments), all fp32 and all checkpointed; the bf16 hi/lo copies of the
preconditioners are derived data, rebuilt by `after_load()`.
Factor sides that are not multiples of 8 (the byte-level embedding's [259, 259]) are stored zero-padded
to [264, 264]; only a preconditioned COLUMN count that is not a multiple of 8 disables preconditioning
for a group (momentum + grafting only) -- impossible with ParamStore's cols % 8 rule and the default cap.
"""
from __future__ import annotations

from dataclasses import InitVar, dataclass
from typing import Callable, Dict, List, Optional, Union

import torch

from .. import ops
from ..flat import MatGroup, ParamStore, get_store

# inverse_root="newton": the iteration reaches max|Mc - I| ~ 5e-7 from ~6e-4 in one step (fp32 floor ~2.4e-7 at
# k = 1024), so 1e-5 costs no extra iteration; statistics with condition numbers up to the ridge's 1e6 take <= 25.
NEWTON_MAX_ITERS = 40
NEWTON_TOL = 1e-5


@dataclass
class ShampooParams:
    beta1: float = 0.9
    beta2: float = 0.99
    epsilon: float = 1e-8
    weight_decay: float = 0.0
    update_period: int = 1
    start_preconditioning_step: int = 10
    preconditioner_epsilon: float = 1e-6
    max_preconditioner_dim: int = 1024
    exponent_override: float = 0.75
    use_bias_correction: bool = True
    grafting_optimizer: str = "adam"
    use_decoupled_weight_decay: bool = True
    # "reference": the reference's literal matrix_inverse_pth_root (shampoo.py:88-126, not an inverse root);
    # "newton": P = (M + ridge I)^(-1/4), ridge = preconditioner_epsilon * max(lambda_max(M), 1e-6), by the
    # coupled Newton iteration.  exponent_override only parameterises the literal formula; newton ignores it.
    # An init-only argument stored as an attribute, so the dataclass fields stay the reference's ShampooParams:
    # dataclasses.replace() carries it over, but asdict(), repr() and == see the reference's fields only.
    inverse_root: InitVar[str] = "reference"

    def __post_init__(self, inverse_root: str = "reference"):
        self.inverse_root = inverse_root
        assert 0.0 <= self.beta1 < 1.0, "beta1 must be in [0, 1)"
        assert 0.0 <= self.beta2 < 1.0, "beta2 must be in [0, 1)"
        assert self.epsilon > 0.0, "epsilon must be positive"
        assert self.update_period > 0, "update_period must be positive"
        assert self.start_preconditioning_step >= 0, "start_preconditioning_step must be non-negative"
        assert self.max_preconditioner_dim > 0, "max_preconditioner_dim must be positive"
        assert 0.0 < self.exponent_override <= 1.0, "exponent_override must be in (0, 1]"
        assert self.grafting_optimizer in ["sgd", "adam", "momentum"], \
            "grafting_optimizer must be one of 'sgd', 'adam', 'momentum'"
        if self.inverse_root not in ("reference", "newton"):
            raise ValueError(f"inverse_root must be 'reference' or 'newton', got {self.inverse_root!r}")


class _GroupState:
    """Kronecker factors of one shape group: [batch, kp, kp] fp32 (+ bf16 hi/lo of the preconditioners)."""

    def __init__(self, g: MatGroup, cap: int, dev):
        self.k1, self.k2 = min(g.rows, cap), min(g.cols, cap)
        self.k1p, self.k2p = ops.rup8(self.k1), ops.rup8(self.k2)
        self.enabled = self.k2 % 8 == 0
        if not self.enabled:
            return
        b = g.batch
        f32 = dict(dtype=torch.float32, device=dev)
        bf = dict(dtype=torch.bfloat16, device=dev)
        self.L = torch.zeros(b, self.k1p, self.k1p, **f32)
        self.R = torch.zeros(b, self.k2p, self.k2p, **f32)
        self.PL = torch.zeros(b, self.k1p, self.k1p, **f32)
        self.PR = torch.zeros(b, self.k2p, self.k2p, **f32)
        self.PLh, self.PLl = torch.zeros(b, self.k1p, self.k1p, **bf), torch.zeros(b, self.k1p, self.k1p, **bf)
        self.PRh, self.PRl = torch.zeros(b, self.k2p, self.k2p, **bf), torch.zeros(b, self.k2p, self.k2p, **bf)
        self.has_precond = False


class Shampoo:
    def __init__(self, learning_rate: Union[float, Callable] = 0.01, params: Optional[ShampooParams] = None,
                 use_distributed: bool = False):
        self.params = params or ShampooParams()
        self._learning_rate = learning_rate
        self.use_distributed = use_distributed
        self.state: Dict[str, Dict[str, torch.Tensor]] = {}
        self.count = 0
        self.grad_scale = 1.0
        self.use_accumulated = False
        self._store: Optional[ParamStore] = None
        if self.params.weight_decay > 0.0 and not self.params.use_decoupled_weight_decay:
            raise ValueError("coupled weight decay is not supported on the fused path (reference factory "
                             "always sets use_decoupled_weight_decay=True, core/training.py:855)")

    def _lr(self, count: int) -> float:
        lr = self._learning_rate(count) if callable(self._learning_rate) else self._learning_rate
        return float(lr)

    @property
    def learning_rate(self) -> float:
        return self._lr(self.count)

    # ------------------------------------------------------------------------------------------
    def init(self, model) -> None:
        store = get_store(model)
        if self._store is store:
            return
        self._store = store
        dev, n = store.device, store.total
        f32 = dict(dtype=torch.float32, device=dev)
        bf = dict(dtype=torch.bfloat16, device=dev)
        self._mom = torch.zeros(n, **f32)
        self._gm = torch.zeros(n, **f32)
        self._gv = torch.zeros(n, **f32)
        self._d = torch.zeros(n, **f32)
        self._pre = torch.zeros(n, **f32)
        self._mh = torch.zeros(n, **bf)
        self._ml = torch.zeros(n, **bf)
        self._gh = self._gl = None   # bf16 hi/lo of fp32 gradients (allocated on first use)
        cap = self.params.max_preconditioner_dim
        self._gs: List[_GroupState] = [_GroupState(g, cap, dev) for g in store.mat_groups]
        lib = ops.lib()
        ws = 256
        for g, s in zip(store.mat_groups, self._gs):
            ws = max(ws, int(lib.b200_shampoo_graft_workspace_bytes(g.batch)))
            if s.enabled:
                root_ws = (lib.b200_shampoo_root_newton_workspace_bytes if self.params.inverse_root == "newton"
                           else lib.b200_shampoo_root_workspace_bytes)
                ws = max(ws, int(root_ws(g.batch, s.k1)), int(root_ws(g.batch, s.k2)),
                         int(lib.b200_shampoo_precond_workspace_bytes(g.batch, s.k1, s.k2)))
        # non-2-D parameters: consecutive equal-length entries are grafted as one batched call
        self._vec_runs = []
        for e in store.vec_entries:
            run = self._vec_runs[-1] if self._vec_runs else None
            if run is not None and run[1] == e.numel and e.numel % 8 == 0 and run[0] + run[1] * run[2] == e.offset:
                run[2] += 1
            else:
                self._vec_runs.append([e.offset, e.numel, 1])
        for _, _, cnt in self._vec_runs:
            ws = max(ws, int(lib.b200_shampoo_graft_workspace_bytes(cnt)))
        self._ws = torch.empty(ws, dtype=torch.uint8, device=dev)
        self.state = {}
        for name in store.index:
            self.state[name] = {"momentum": store.view(self._mom, name), "graft_m": store.view(self._gm, name),
                                "graft_v": store.view(self._gv, name)}
        for g, s in zip(store.mat_groups, self._gs):
            if s.enabled:
                for i, name in enumerate(g.names):
                    st = self.state[name]
                    st["statistics.0"] = s.L[i, :s.k1, :s.k1]
                    st["statistics.1"] = s.R[i, :s.k2, :s.k2]
                    st["preconditioners.0"] = s.PL[i, :s.k1, :s.k1]
                    st["preconditioners.1"] = s.PR[i, :s.k2, :s.k2]

    def _inverse_pth_root(self, stat: torch.Tensor, P: torch.Tensor, Ph: torch.Tensor, Pl: torch.Tensor,
                          k: int) -> None:
        """Preconditioner of stat [b, kp, kp]: MatrixSqrt.matrix_inverse_pth_root (shampoo.py:88-126) literally, or
        with inverse_root="newton" the true (stat + ridge I)^(-1/4)."""
        hp = self.params
        if hp.inverse_root == "newton":
            ops.shampoo_root_newton(stat, P, Ph, Pl, k, hp.preconditioner_epsilon, NEWTON_MAX_ITERS, NEWTON_TOL,
                                    self._ws)
        else:
            ops.shampoo_root(stat, P, Ph, Pl, k, hp.exponent_override, hp.preconditioner_epsilon, 6, self._ws)

    @torch.no_grad()
    def after_load(self) -> None:
        """Called after a checkpoint's tensors were copied into `state`: rebuilds the derived bf16 hi/lo
        operands of the preconditioners, so a resumed run is preconditioned from its first step
        (reference: preconditioners are part of the saved state, shampoo.py:180-208, core/training.py:1354)."""
        for s in getattr(self, "_gs", []):
            if not s.enabled:
                continue
            for P, Ph, Pl in ((s.PL, s.PLh, s.PLl), (s.PR, s.PRh, s.PRl)):
                ops.check(ops.lib().b200_split_bf16(P.data_ptr(), P.shape[-1], Ph.data_ptr(), Pl.data_ptr(),
                                                    P.shape[-1], P.shape[0] * P.shape[1], P.shape[2], 1.0, 0.0,
                                                    ops._stream()), "b200_split_bf16")
            s.has_precond = bool(s.PL.any().item()) and bool(s.PR.any().item())

    # ------------------------------------------------------------------------------------------
    @torch.no_grad()
    def update(self, model, gradients=None) -> None:
        self.init(model)
        store, hp = self._store, self.params
        if gradients is not None:
            store.load_gradients(gradients)
        gsrc = store.acc if self.use_accumulated else store.grad
        self.count += 1
        t = self.count
        lr = self._lr(t)
        gs = self.grad_scale
        end = store.vec_end
        # grafting direction (shampoo.py:162-178,326): computed, not applied
        if hp.grafting_optimizer == "adam":
            ops.adam_direction(self._d[:end], gsrc[:end], self._gm[:end], self._gv[:end], lr, hp.beta1, hp.beta2,
                               hp.epsilon, 1.0, 1.0, gs)
        elif hp.grafting_optimizer == "momentum":   # mlx SGD momentum: v = mu v + g ; step = -lr v
            self._gm[:end].mul_(hp.beta1).add_(gsrc[:end].float(), alpha=gs)
            torch.mul(self._gm[:end], -lr, out=self._d[:end])
        else:
            torch.mul(gsrc[:end].float(), -lr * gs, out=self._d[:end])
        inv_bc = 1.0 / (1.0 - hp.beta1 ** t) if hp.use_bias_correction else 1.0
        # pre = -lr * mhat (the reference's `update = -lr * preconditioned_grad`, shampoo.py:365); the
        # preconditioned blocks are overwritten below with -lr * PL mhat PR
        ops.ema_split(gsrc[:end], self._mom[:end], self._pre[:end], self._mh[:end], self._ml[:end], hp.beta1, gs,
                      inv_bc, -lr)
        if gsrc.dtype != torch.bfloat16 and store.mat_end > 0:
            if self._gh is None:
                self._gh = torch.empty(store.total, dtype=torch.bfloat16, device=store.device)
                self._gl = torch.empty(store.total, dtype=torch.bfloat16, device=store.device)
            ops.check(ops.lib().b200_split_bf16(gsrc.data_ptr(), 8, self._gh.data_ptr(), self._gl.data_ptr(), 8,
                                                store.mat_end // 8, 8, 1.0, 0.0, ops._stream()), "b200_split_bf16")
            g_hi, g_lo = self._gh, self._gl
        else:
            g_hi, g_lo = gsrc, None
        decay = 1.0 - lr * hp.weight_decay if hp.weight_decay > 0.0 else 1.0
        do_root = t >= hp.start_preconditioning_step and t % hp.update_period == 0
        for g, s in zip(store.mat_groups, self._gs):
            lo, n, rc = g.offset, g.numel, g.rows * g.cols
            b, c = g.batch, g.cols
            if s.enabled:
                k1, k2 = s.k1, s.k2
                tok = ops._t0("shampoo_stats")
                ops.shampoo_stats(g_hi[lo:lo + n], None if g_lo is None else g_lo[lo:lo + n], c, rc, s.L, s.R, b, k1,
                                  k2, hp.beta2, (1.0 - hp.beta2) * gs * gs)
                ops._t1(tok)
                if do_root:
                    tok = ops._t0("shampoo_root")
                    self._inverse_pth_root(s.L, s.PL, s.PLh, s.PLl, k1)
                    self._inverse_pth_root(s.R, s.PR, s.PRh, s.PRl, k2)
                    ops._t1(tok)
                    s.has_precond = True
                if t >= hp.start_preconditioning_step and s.has_precond:
                    # pre[:k1,:k2] = -lr * PL @ mhat[:k1,:k2] @ PR, written straight into the update buffer
                    tok = ops._t0("shampoo_precond")
                    ops.shampoo_precond(s.PLh, s.PLl, s.PRh, s.PRl, self._mh[lo:lo + n], self._ml[lo:lo + n], c, rc,
                                        self._pre[lo:lo + n], c, rc, b, k1, k2, -lr, self._ws)
                    ops._t1(tok)
            self._graft_and_apply(store, lo, rc, b, decay)
        for off, numel, cnt in self._vec_runs:
            self._graft_and_apply(store, off, numel, cnt, decay)

    def _graft_and_apply(self, store: ParamStore, lo: int, numel: int, batch: int, decay: float) -> None:
        """_apply_grafting + parameter write (shampoo.py:297-312,365-373) for `batch` tensors of `numel`."""
        n = numel * batch
        p16 = store.shadow[lo:lo + n] if store.mixed else None
        ops.shampoo_graft(store.master[lo:lo + n], p16, self._pre[lo:lo + n], self._d[lo:lo + n], numel, batch,
                          decay, self._ws)

    def apply_gradients(self, gradients, model):
        self.update(model, gradients)
        return model

    def step(self, model) -> None:
        self.update(model, None)

    def state_dict(self) -> Dict[str, torch.Tensor]:
        out = {}
        for name, st in self.state.items():
            for k, v in st.items():
                out[f"{name}.{k}"] = v
        return out
