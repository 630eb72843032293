"""PyTorch-tensor wrappers over the C ABI (include/b200_hotpath.h).

PyTorch is plumbing here: it owns device memory and streams; all arithmetic below runs in the
hand-written sm_90a kernels.  Every wrapper validates dtype/contiguity and raises on failure --
there is no eager fallback.
"""
from __future__ import annotations

import os
from typing import Optional, Sequence, Tuple

import torch

from ._lib import B200Error, check, lib, require_device

NS_COEFFS = (3.4445, -4.7750, 2.0315)  # optimizers/muon.py:65
NS_EPS = 1e-7                          # optimizers/muon.py:73


def _stream() -> int:
    # raw handle of torch's current stream on the current device; torch.cuda.current_stream() builds a Stream
    # object on every call (~100 calls per C2 step)
    return torch._C._cuda_getCurrentRawStream(torch._C._cuda_getDevice())


class KernelTimer:
    """Optional CUDA-event bracketing of kernel families on the launching stream (bench.py's
    live roofline measurement).  Disabled (None) in normal runs: zero overhead."""

    def __init__(self):
        self.events = {}

    def start(self, name: str):
        e0 = torch.cuda.Event(enable_timing=True)
        e0.record()
        return (name, e0)

    def stop(self, tok) -> None:
        name, e0 = tok
        e1 = torch.cuda.Event(enable_timing=True)
        e1.record()
        self.events.setdefault(name, []).append((e0, e1))

    def totals_ms(self):
        torch.cuda.synchronize()
        return {k: (sum(a.elapsed_time(b) for a, b in v), len(v)) for k, v in self.events.items()}


TIMER: Optional[KernelTimer] = None


def _t0(name: str):
    return TIMER.start(name) if TIMER is not None else None


def _t1(tok) -> None:
    if tok is not None:
        TIMER.stop(tok)


def _ptr(t: Optional[torch.Tensor]) -> Optional[int]:
    return None if t is None else t.data_ptr()


def _need(t: torch.Tensor, dtype, name: str) -> None:
    if not t.is_cuda:
        raise B200Error(f"{name}: expected a CUDA tensor (no CPU fallback)")
    if t.dtype != dtype:
        raise ValueError(f"{name}: expected {dtype}, got {t.dtype}")
    if not t.is_contiguous():
        raise ValueError(f"{name}: tensor must be contiguous")


def _is_bf16(t: torch.Tensor, name: str) -> int:
    if t.dtype == torch.bfloat16:
        return 1
    if t.dtype == torch.float32:
        return 0
    raise ValueError(f"{name}: unsupported dtype {t.dtype} (bf16 or fp32)")


# ------------------------------------------------------------------------------------------------
# dense contraction engine
# ------------------------------------------------------------------------------------------------
def gemm(a: torch.Tensor, b: torch.Tensor, *, a_mn: bool = False, b_mn: bool = False,
         c: Optional[torch.Tensor] = None, alpha: float = 1.0, beta: float = 0.0,
         alpha_vec: Optional[torch.Tensor] = None, beta_vec: Optional[torch.Tensor] = None,
         out: Optional[torch.Tensor] = None, out_dtype: torch.dtype = torch.bfloat16,
         force_bn: int = 0) -> torch.Tensor:
    """D = alpha*op(A) op(B) + beta*C, batched over a leading dim.

    a: [.., M, K] (a_mn=False) or [.., K, M] (a_mn=True); b: [.., N, K] or [.., K, N] (b_mn=True).
    """
    _need(a, torch.bfloat16, "a")
    _need(b, torch.bfloat16, "b")
    a3 = a if a.dim() == 3 else a.unsqueeze(0)
    b3 = b if b.dim() == 3 else b.unsqueeze(0)
    batch = a3.shape[0]
    if b3.shape[0] != batch:
        raise ValueError("gemm: batch mismatch")
    (K, M) = a3.shape[1:] if a_mn else a3.shape[1:][::-1]
    (Kb, N) = b3.shape[1:] if b_mn else b3.shape[1:][::-1]
    if K != Kb:
        raise ValueError(f"gemm: K mismatch {K} vs {Kb}")
    if out is None:
        out = torch.empty((batch, M, N), device=a.device, dtype=out_dtype)
    out_f32 = _is_bf16(out, "out") == 0
    if tuple(out.shape[-2:]) != (M, N) or not out.is_contiguous():
        raise ValueError("gemm: bad out tensor")
    if c is not None:
        if c.dtype != out.dtype or tuple(c.shape[-2:]) != (M, N) or not c.is_contiguous():
            raise ValueError("gemm: c must match out dtype/shape and be contiguous")
    for v, nm in ((alpha_vec, "alpha_vec"), (beta_vec, "beta_vec")):
        if v is not None:
            _need(v, torch.float32, nm)
            if v.numel() != batch:
                raise ValueError(f"gemm: {nm} must have one entry per batch")
    rc = lib().b200_gemm_bf16(
        int(a_mn), int(b_mn), M, N, K, batch,
        a3.data_ptr(), a3.shape[2], a3.shape[1] * a3.shape[2],
        b3.data_ptr(), b3.shape[2], b3.shape[1] * b3.shape[2],
        _ptr(c), N, M * N,
        out.data_ptr(), N, M * N,
        int(out_f32), float(alpha), float(beta), _ptr(alpha_vec), _ptr(beta_vec), int(force_bn),
        _stream())
    check(rc, "b200_gemm_bf16")
    return out.view(M, N) if (a.dim() == 2 and out.dim() == 3) else out


# ------------------------------------------------------------------------------------------------
# Newton-Schulz / Muon pieces
# ------------------------------------------------------------------------------------------------
def ns_workspace_bytes(batch: int, rows: int, cols: int, steps: int) -> int:
    return int(lib().b200_newton_schulz_workspace_bytes(batch, rows, cols, steps))


_REDUCE_WS = {}


def reduce_workspace(device, batch: int) -> torch.Tensor:
    """Scratch of the deterministic grid reductions (b200_reduce_workspace_bytes), one per (device, stream)."""
    key = (str(device), _stream())
    need = int(lib().b200_reduce_workspace_bytes(int(batch)))
    ws = _REDUCE_WS.get(key)
    if ws is None or ws.numel() < need:
        ws = torch.empty(need, device=device, dtype=torch.uint8)
        _REDUCE_WS[key] = ws
    return ws


def sumsq(x: torch.Tensor, out: Optional[torch.Tensor] = None, zero_first: bool = True) -> torch.Tensor:
    """Per-matrix sum of squares of x [batch, ...] -> fp32 [batch]."""
    xb = x if x.dim() >= 2 else x.unsqueeze(0)
    batch = xb.shape[0] if x.dim() == 3 else 1
    numel = x.numel() // batch
    if out is None:
        out = torch.empty(batch, device=x.device, dtype=torch.float32)
    ws = reduce_workspace(x.device, batch)
    check(lib().b200_sumsq(x.data_ptr(), _is_bf16(x, "x"), out.data_ptr(), numel, batch,
                           int(zero_first), ws.data_ptr(), ws.numel(), _stream()), "b200_sumsq")
    return out


def ns_scales(ss: torch.Tensor, eps: float = NS_EPS) -> Tuple[torch.Tensor, torch.Tensor]:
    inv = torch.empty_like(ss)
    inv2 = torch.empty_like(ss)
    check(lib().b200_ns_scales(ss.data_ptr(), inv.data_ptr(), inv2.data_ptr(), ss.numel(), eps,
                               _stream()), "b200_ns_scales")
    return inv, inv2


def newton_schulz_raw(x_in: torch.Tensor, x_out: torch.Tensor, inv_norm: torch.Tensor,
                      inv_norm_sq: torch.Tensor, workspace: torch.Tensor, steps: int = 5,
                      coeffs: Sequence[float] = NS_COEFFS) -> torch.Tensor:
    """x_in/x_out: bf16 [batch, rows, cols]; workspace: uint8 buffer from ns_workspace_bytes."""
    _need(x_in, torch.bfloat16, "x_in")
    _need(x_out, torch.bfloat16, "x_out")
    batch, rows, cols = x_in.shape
    a, b, c = coeffs
    check(lib().b200_newton_schulz(x_in.data_ptr(), x_out.data_ptr(), batch, rows, cols, steps,
                                   float(a), float(b), float(c), inv_norm.data_ptr(),
                                   inv_norm_sq.data_ptr(), workspace.data_ptr(),
                                   workspace.numel() * workspace.element_size(), _stream()),
          "b200_newton_schulz")
    return x_out


def zeropower_via_newtonschulz5(g: torch.Tensor, steps: int = 5, eps: float = NS_EPS,
                                coeffs: Sequence[float] = NS_COEFFS) -> torch.Tensor:
    """Drop-in for Muon.zeropower_via_newtonschulz5 (optimizers/muon.py:54-83).

    g: [rows, cols] or [batch, rows, cols], fp32 or bf16 on an H100. Returns bf16 of the same shape.
    """
    require_device()
    squeeze = g.dim() == 2
    g3 = (g.unsqueeze(0) if squeeze else g).contiguous()
    batch, rows, cols = g3.shape
    x_in = g3 if g3.dtype == torch.bfloat16 else g3.to(torch.bfloat16)
    # Frobenius norm of the (fp32) input, folded into iteration 1 by the kernel
    inv, inv2 = ns_scales(sumsq(g3 if g3.dtype in (torch.float32, torch.bfloat16) else x_in), eps)
    ws = torch.empty(ns_workspace_bytes(batch, rows, cols, steps), device=g.device, dtype=torch.uint8)
    x_out = torch.empty_like(x_in)
    newton_schulz_raw(x_in, x_out, inv, inv2, ws, steps, coeffs)
    return x_out[0] if squeeze else x_out


def zeropower_groups(gs: Sequence[torch.Tensor], steps: int = 5, eps: float = NS_EPS,
                     coeffs: Sequence[float] = NS_COEFFS):
    """Newton-Schulz of several [batch, rows, cols] groups (different shapes) through the whole-model chain:
    every stage of the iteration is ONE grouped launch over all groups (b200_newton_schulz_multi).
    Returns a list of bf16 tensors shaped like the inputs."""
    from ._lib import NsGroup
    require_device()
    if not 1 <= len(gs) <= 6:
        raise ValueError("zeropower_groups takes 1..6 groups")
    keep, arr, outs = [], (NsGroup * len(gs))(), []
    for i, g in enumerate(gs):
        g3 = g.contiguous()
        if g3.dim() != 3:
            raise ValueError("each group must be [batch, rows, cols]")
        x_in = g3 if g3.dtype == torch.bfloat16 else g3.to(torch.bfloat16)
        inv, inv2 = ns_scales(sumsq(g3), eps)
        x_out = torch.empty_like(x_in)
        keep += [x_in, inv, inv2]
        outs.append(x_out)
        e = arr[i]
        e.x_in, e.x_out = x_in.data_ptr(), x_out.data_ptr()
        e.batch, e.rows, e.cols = x_in.shape
        e.inv_norm, e.inv_norm_sq = inv.data_ptr(), inv2.data_ptr()
        e.peer_out, e.n_peers = None, 0
    a, b, c = coeffs
    need = int(lib().b200_newton_schulz_multi_workspace_bytes(arr, len(gs), steps))
    ws = torch.empty(max(need, 256), device=gs[0].device, dtype=torch.uint8)
    check(lib().b200_newton_schulz_multi(arr, len(gs), steps, float(a), float(b), float(c), ws.data_ptr(),
                                         ws.numel(), _stream()), "b200_newton_schulz_multi")
    return outs


def muon_momentum(g: torch.Tensor, buf: torch.Tensor, u: torch.Tensor, sumsq_out: torch.Tensor,
                  mu: float, nesterov: bool, gscale: float = 1.0) -> None:
    """g,buf,u: [batch, rows, cols] (g bf16|fp32, buf fp32, u bf16); sumsq_out fp32 [batch]."""
    _need(buf, torch.float32, "buf")
    _need(u, torch.bfloat16, "u")
    batch = g.shape[0] if g.dim() == 3 else 1
    numel = g.numel() // batch
    ws = reduce_workspace(g.device, batch)
    check(lib().b200_muon_momentum(g.data_ptr(), _is_bf16(g, "g"), buf.data_ptr(), u.data_ptr(),
                                   sumsq_out.data_ptr(), numel, batch, float(mu), int(nesterov),
                                   float(gscale), ws.data_ptr(), ws.numel(), _stream()), "b200_muon_momentum")


def axpy_update(p32: torch.Tensor, p16: Optional[torch.Tensor], x: torch.Tensor, s: float) -> None:
    _need(p32, torch.float32, "p32")
    check(lib().b200_axpy_update(p32.data_ptr(), _ptr(p16), x.data_ptr(), _is_bf16(x, "x"),
                                 p32.numel(), float(s), _stream()), "b200_axpy_update")


def sgd_momentum(p32, p16, g, buf, mu: float, nesterov: bool, lr: float, gscale: float = 1.0) -> None:
    check(lib().b200_sgd_momentum(p32.data_ptr(), _ptr(p16), g.data_ptr(), _is_bf16(g, "g"),
                                  buf.data_ptr(), p32.numel(), float(mu), int(nesterov), float(lr),
                                  float(gscale), _stream()), "b200_sgd_momentum")


def adamw(p32, p16, g, m, v, lr: float, b1: float, b2: float, eps: float, wd: float,
          bc1: float = 1.0, bc2: float = 1.0, gscale: float = 1.0) -> None:
    check(lib().b200_adamw(p32.data_ptr(), _ptr(p16), g.data_ptr(), _is_bf16(g, "g"), m.data_ptr(),
                           v.data_ptr(), p32.numel(), float(lr), float(b1), float(b2), float(eps),
                           float(wd), float(bc1), float(bc2), float(gscale), _stream()),
          "b200_adamw")


def _check_update_operands(what: str, p32, p16, g, state: dict) -> int:
    """Shared checks of the fused optimizer updates: fp32 master, optional bf16 shadow, bf16|fp32 gradient and
    fp32 state buffers, all contiguous CUDA tensors of p32's length starting on a 16-byte boundary."""
    _need(p32, torch.float32, f"{what}: p32")
    if p16 is not None:
        _need(p16, torch.bfloat16, f"{what}: p16")
    if not g.is_cuda or not g.is_contiguous():
        raise ValueError(f"{what}: g must be a contiguous CUDA tensor")
    g_bf16 = _is_bf16(g, f"{what}: g")
    n = p32.numel()
    for name, t in [("p16", p16), ("g", g)] + list(state.items()):
        if t is None:
            continue
        if name not in ("p16", "g"):
            _need(t, torch.float32, f"{what}: {name}")
        if t.numel() != n:
            raise ValueError(f"{what}: {name} has {t.numel()} elements, p32 has {n}")
    for name, t in [("p32", p32), ("p16", p16), ("g", g)] + list(state.items()):
        if t is not None and t.data_ptr() % 16:
            raise ValueError(f"{what}: {name} must start on a 16-byte boundary")
    return g_bf16


def _clip_args(clip_ss: Optional[torch.Tensor], max_norm: Optional[float]):
    if clip_ss is None:
        return None, 0.0
    _need(clip_ss, torch.float32, "clip_ss")
    if max_norm is None:
        raise ValueError("clip_ss needs max_norm")
    return clip_ss.data_ptr(), float(max_norm)


def lion(p32, p16, g, m, lr: float, b_sign: float, b_mom: float, decay: float = 1.0, gscale: float = 1.0,
         clip_ss: Optional[torch.Tensor] = None, max_norm: Optional[float] = None,
         ema: Optional[torch.Tensor] = None, ema_decay: float = 0.0, ema_mode: int = 0) -> None:
    """Fused Lion update in place (b200_lion).  clip_ss: device fp32 sum of squares of g's range (sumsq) to clip
    by global norm against max_norm; ema_mode 0 none, 1 ema := p_new, 2 ema = d*ema + (1-d)*p_new."""
    if ema_mode and ema is None:
        raise ValueError("lion: ema_mode needs an ema buffer")
    g_bf16 = _check_update_operands("lion", p32, p16, g, {"m": m, "ema": ema})
    ss, mn = _clip_args(clip_ss, max_norm)
    check(lib().b200_lion(p32.data_ptr(), _ptr(p16), g.data_ptr(), g_bf16, m.data_ptr(), _ptr(ema), p32.numel(),
                          float(lr), float(b_sign), float(b_mom), float(decay), float(gscale), ss, mn,
                          float(ema_decay), int(ema_mode), _stream()), "b200_lion")


def sgd(p32, p16, g, buf: Optional[torch.Tensor], lr: float, mu: float = 0.0, dampening: float = 0.0,
        nesterov: bool = False, coupled_wd: float = 0.0, gscale: float = 1.0,
        clip_ss: Optional[torch.Tensor] = None, max_norm: Optional[float] = None,
        ema: Optional[torch.Tensor] = None, ema_decay: float = 0.0, ema_mode: int = 0) -> None:
    """Fused SGD update in place (b200_sgd): buf None is plain mlx SGD (p -= lr*g); otherwise SGDEnhanced's
    momentum with coupled weight decay coupled_wd = lr*wd.  Clip and EMA arguments as in lion()."""
    if ema_mode and ema is None:
        raise ValueError("sgd: ema_mode needs an ema buffer")
    g_bf16 = _check_update_operands("sgd", p32, p16, g, {"buf": buf, "ema": ema})
    ss, mn = _clip_args(clip_ss, max_norm)
    check(lib().b200_sgd(p32.data_ptr(), _ptr(p16), g.data_ptr(), g_bf16, _ptr(buf), _ptr(ema), p32.numel(),
                         float(lr), float(mu), float(dampening), int(nesterov), float(coupled_wd), float(gscale),
                         ss, mn, float(ema_decay), int(ema_mode), _stream()), "b200_sgd")


def adam_direction(d, g, m, v, lr, b1, b2, eps, bc1=1.0, bc2=1.0, gscale=1.0) -> None:
    check(lib().b200_adam_direction(d.data_ptr(), g.data_ptr(), _is_bf16(g, "g"), m.data_ptr(),
                                    v.data_ptr(), d.numel(), float(lr), float(b1), float(b2),
                                    float(eps), float(bc1), float(bc2), float(gscale), _stream()),
          "b200_adam_direction")


def clip_accum(g: torch.Tensor, acc: torch.Tensor, clip: float, scale: float, init: bool) -> None:
    _need(acc, torch.float32, "acc")
    check(lib().b200_clip_accum(g.data_ptr(), _is_bf16(g, "g"), acc.data_ptr(), g.numel(),
                                float(clip), float(scale), int(init), _stream()), "b200_clip_accum")


def split_bf16(src: torch.Tensor, rows: int, cols: int, hi: torch.Tensor,
               lo: Optional[torch.Tensor], scale: float = 1.0, diag_add: float = 0.0) -> None:
    """hi(+lo) = bf16 split of (src[:rows,:cols] + diag_add*I)*scale; src fp32 2-D (strided rows)."""
    _need(hi, torch.bfloat16, "hi")
    check(lib().b200_split_bf16(src.data_ptr(), src.stride(0), hi.data_ptr(), _ptr(lo),
                                hi.stride(0), rows, cols, float(scale), float(diag_add), _stream()),
          "b200_split_bf16")


# ------------------------------------------------------------------------------------------------
# RMSNorm / RoPE / attention as autograd functions
# ------------------------------------------------------------------------------------------------
# Deferred RMSNorm weight gradients: a norm's backward leaves its per-CTA partial sums in a workspace; ONE batched
# launch at the end of the backward pass (an autograd-engine callback) folds all of them into the weights' .grad
# buffers in place.  Used when the weight is a leaf with a preallocated contiguous .grad (the flat ParamStore's
# case); any other weight takes the immediate path and gets its gradient from autograd as usual.
_PENDING_DW: list = []
_DW_DEFER = os.environ.get("B200_DEFER_DW", "1") != "0"


def _dw_target(w: torch.Tensor) -> Optional[torch.Tensor]:
    g = w.grad if (_DW_DEFER and w.is_leaf and w.requires_grad) else None
    if g is None or not g.is_contiguous() or g.dtype not in (torch.bfloat16, torch.float32) or g.shape != w.shape:
        return None
    return g


def flush_deferred_dw() -> None:
    """Runs the pending weight-gradient reductions now (normally called by the autograd engine at the end of the
    backward pass that queued them)."""
    if not _PENDING_DW:
        return
    from ._lib import DwJob
    jobs, _PENDING_DW[:] = list(_PENDING_DW), []
    by_h = {}
    for ws, grad, nparts in jobs:
        by_h.setdefault(grad.numel(), []).append((ws, grad, nparts))
    for H, group in by_h.items():
        arr = (DwJob * len(group))()
        for i, (ws, grad, nparts) in enumerate(group):
            arr[i].partials, arr[i].dw, arr[i].n_partials = ws.data_ptr(), grad.data_ptr(), nparts
            arr[i].dw_is_bf16, arr[i].accumulate = int(grad.dtype == torch.bfloat16), 1
        check(lib().b200_rmsnorm_dw_reduce(arr, len(group), H, _stream()), "b200_rmsnorm_dw_reduce")


def _defer_dw(ws: torch.Tensor, grad: torch.Tensor, nparts: int) -> None:
    if not _PENDING_DW:
        torch.autograd.Variable._execution_engine.queue_callback(flush_deferred_dw)
    _PENDING_DW.append((ws, grad, nparts))


class _RMSNormFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, w, eps):
        xs = x.contiguous()
        rows, H = xs.numel() // xs.shape[-1], xs.shape[-1]
        y = torch.empty_like(xs)
        rstd = torch.empty(rows, device=x.device, dtype=torch.float32)
        wc = w.contiguous().to(xs.dtype)
        check(lib().b200_rmsnorm_fwd(xs.data_ptr(), wc.data_ptr(), y.data_ptr(), rstd.data_ptr(),
                                     rows, H, float(eps), _is_bf16(xs, "x"), _stream()),
              "b200_rmsnorm_fwd")
        ctx.save_for_backward(xs, wc, rstd)
        ctx.w_dtype = w.dtype
        ctx.weight = w
        return y

    @staticmethod
    def backward(ctx, dy):
        xs, wc, rstd = ctx.saved_tensors
        dy = dy.contiguous()
        rows, H = xs.numel() // xs.shape[-1], xs.shape[-1]
        dx = torch.empty_like(xs)
        need_w = ctx.needs_input_grad[1]
        target = _dw_target(ctx.weight) if need_w else None
        dw = None if (target is not None or not need_w) else torch.empty(H, device=xs.device, dtype=torch.float32)
        ws = torch.empty(int(lib().b200_rmsnorm_bwd_workspace_bytes(rows, H)), device=xs.device, dtype=torch.uint8)
        check(lib().b200_rmsnorm_bwd(dy.data_ptr(), xs.data_ptr(), wc.data_ptr(), rstd.data_ptr(),
                                     dx.data_ptr(), _ptr(dw), rows, H, _is_bf16(xs, "x"),
                                     ws.data_ptr(), ws.numel(), _stream()), "b200_rmsnorm_bwd")
        if target is not None:
            _defer_dw(ws, target, int(lib().b200_rmsnorm_bwd_partial_rows(rows, H)))
        return dx, (dw.to(ctx.w_dtype) if dw is not None else None), None


def rmsnorm(x: torch.Tensor, w: torch.Tensor, eps: float = 1e-5) -> torch.Tensor:
    return _RMSNormFn.apply(x, w, eps)


class _AddRMSNormFn(torch.autograd.Function):
    """(x, delta) -> (s = x + delta, rmsnorm(s) * w): the residual add of arch/llama.py:316-319 fused with
    the norm that reads its result; backward folds the residual-stream gradient into the norm's dx."""

    @staticmethod
    def forward(ctx, x, delta, w, eps):
        xs, ds = x.contiguous(), delta.contiguous()
        rows, H = xs.numel() // xs.shape[-1], xs.shape[-1]
        s = torch.empty_like(xs)
        y = torch.empty_like(xs)
        rstd = torch.empty(rows, device=x.device, dtype=torch.float32)
        wc = w.contiguous().to(xs.dtype)
        check(lib().b200_add_rmsnorm_fwd(xs.data_ptr(), ds.data_ptr(), wc.data_ptr(), s.data_ptr(), y.data_ptr(),
                                         rstd.data_ptr(), rows, H, float(eps), _is_bf16(xs, "x"), _stream()),
              "b200_add_rmsnorm_fwd")
        ctx.save_for_backward(s, wc, rstd)
        ctx.w_dtype = w.dtype
        ctx.weight = w
        ctx.set_materialize_grads(False)
        return s, y

    @staticmethod
    def backward(ctx, ds, dy):
        s, wc, rstd = ctx.saved_tensors
        if dy is None:
            return ds, ds, None, None
        dy = dy.contiguous()
        rows, H = s.numel() // s.shape[-1], s.shape[-1]
        dx = torch.empty_like(s)
        need_w = ctx.needs_input_grad[2]
        target = _dw_target(ctx.weight) if need_w else None
        dw = None if (target is not None or not need_w) else torch.empty(H, device=s.device, dtype=torch.float32)
        ws = torch.empty(int(lib().b200_rmsnorm_bwd_workspace_bytes(rows, H)), device=s.device, dtype=torch.uint8)
        dres = ds.contiguous() if ds is not None else None
        check(lib().b200_add_rmsnorm_bwd(dy.data_ptr(), dres.data_ptr() if dres is not None else None,
                                         s.data_ptr(), wc.data_ptr(), rstd.data_ptr(), dx.data_ptr(),
                                         _ptr(dw), rows, H, _is_bf16(s, "x"), ws.data_ptr(), ws.numel(),
                                         _stream()), "b200_add_rmsnorm_bwd")
        if target is not None:
            _defer_dw(ws, target, int(lib().b200_rmsnorm_bwd_partial_rows(rows, H)))
        return dx, dx, (dw.to(ctx.w_dtype) if dw is not None else None), None


def add_rmsnorm(x: torch.Tensor, delta: torch.Tensor, w: torch.Tensor, eps: float = 1e-5):
    """Returns (x + delta, rmsnorm(x + delta) * w)."""
    return _AddRMSNormFn.apply(x, delta, w, eps)


def _accumulate_wgrad(w: torch.Tensor, dy2: torch.Tensor, x2: torch.Tensor):
    """dW = dy^T x.  When the weight's .grad is a view of the flat gradient buffer (flat.ParamStore), the
    GEMM accumulates straight into it (beta = 1 epilogue) and autograd gets None: no temporary, no
    separate AccumulateGrad add kernel per parameter."""
    g = w.grad
    if getattr(w, "_b200_flat_grad", False) and g is not None and g.dtype == dy2.dtype:
        g.addmm_(dy2.t(), x2)
        return None
    return dy2.t() @ x2


class _LinearFn(torch.autograd.Function):
    """y = x W^T (bias-free nn.Linear, arch/llama.py projections) through the library GEMM."""

    @staticmethod
    def forward(ctx, x, w):
        ctx.save_for_backward(x, w)
        return torch.nn.functional.linear(x, w)

    @staticmethod
    def backward(ctx, dy):
        x, w = ctx.saved_tensors
        dx = torch.matmul(dy, w) if ctx.needs_input_grad[0] else None
        dw = None
        if ctx.needs_input_grad[1]:
            dw = _accumulate_wgrad(w, dy.reshape(-1, dy.shape[-1]), x.reshape(-1, x.shape[-1]))
        return dx, dw


class _MultiLinearFn(torch.autograd.Function):
    """Several bias-free projections of the same input (q/k/v, gate/up).  Backward accumulates
    dx = sum_i dy_i W_i inside the GEMM epilogues instead of autograd's extra add passes."""

    @staticmethod
    def forward(ctx, x, *ws):
        ctx.save_for_backward(x, *ws)
        ctx.set_materialize_grads(False)
        return tuple(torch.nn.functional.linear(x, w) for w in ws)

    @staticmethod
    def backward(ctx, *dys):
        x, *ws = ctx.saved_tensors
        x2 = x.reshape(-1, x.shape[-1])
        dx2 = None
        dws = []
        fused = _fuse_adjacent(dys, ws)   # e.g. (dq, Wq), ([dk | dv], [Wk ; Wv]) when memory layouts allow
        if fused is not None:
            for dy2, w, wg in fused:
                if ctx.needs_input_grad[0]:
                    if dx2 is None:
                        dx2 = dy2 @ w
                    else:
                        dx2.addmm_(dy2, w)
                wg.addmm_(dy2.t(), x2)
            return (dx2.view(x.shape) if dx2 is not None else None, *([None] * len(ws)))
        for i, (dy, w) in enumerate(zip(dys, ws)):
            if dy is None:
                dws.append(None)
                continue
            dy2 = dy.reshape(-1, dy.shape[-1])
            if ctx.needs_input_grad[0]:
                if dx2 is None:
                    dx2 = dy2 @ w
                else:
                    dx2.addmm_(dy2, w)
            dws.append(_accumulate_wgrad(w, dy2, x2) if ctx.needs_input_grad[1 + i] else None)
        return (dx2.view(x.shape) if dx2 is not None else None, *dws)


def _fuse_adjacent(dys, ws):
    """Backward of projections sharing an input: where two consecutive weights are adjacent in the flat
    parameter buffer (k_proj / v_proj of a layer), their flat .grad views are adjacent too, and their output
    gradients are the two column halves of one row-major buffer (attention backward writes dk | dv that way),
    [dy_a | dy_b] x [W_a ; W_b] is ONE dgrad GEMM and one wgrad GEMM instead of two each.  Returns a list of
    (dy2 [T, n], W [n, in], W.grad [n, in]) covering all projections, or None when nothing can be merged or
    some weight's gradient is not a flat-buffer view."""
    if any(dy is None for dy in dys) or not all(getattr(w, "_b200_flat_grad", False) and w.grad is not None
                                                 and w.grad.dtype == dy.dtype for w, dy in zip(ws, dys)):
        return None
    out, i, merged = [], 0, False
    while i < len(ws):
        w, dy = ws[i], dys[i]
        n, k_in = w.shape
        es = w.element_size()
        if i + 1 < len(ws):
            w2, dy2 = ws[i + 1], dys[i + 1]
            T = dy.numel() // n
            rows_ok = all(d.dim() >= 2 and d.shape[-1] == n and d.stride(-1) == 1 and d.stride(-2) == 2 * n and
                          all(d.stride(j) == d.stride(j + 1) * d.shape[j + 1] for j in range(d.dim() - 2))
                          for d in (dy, dy2))
            if (w2.shape == w.shape and w.is_contiguous() and w2.is_contiguous() and rows_ok and
                    w2.data_ptr() == w.data_ptr() + n * k_in * es and
                    w2.grad.data_ptr() == w.grad.data_ptr() + n * k_in * es and
                    dy2.data_ptr() == dy.data_ptr() + n * dy.element_size() and dy2.shape == dy.shape):
                out.append((torch.as_strided(dy, (T, 2 * n), (2 * n, 1)),
                            torch.as_strided(w, (2 * n, k_in), (k_in, 1)),
                            torch.as_strided(w.grad, (2 * n, k_in), (k_in, 1))))
                i += 2
                merged = True
                continue
        out.append((dy.reshape(-1, n), w, w.grad))
        i += 1
    return out if merged else None


def linear(x: torch.Tensor, w: torch.Tensor) -> torch.Tensor:
    return _LinearFn.apply(x, w)


def multi_linear(x: torch.Tensor, ws) -> tuple:
    return _MultiLinearFn.apply(x, *ws)


def rope_tables(seq_len: int, head_dim: int, theta: float, device) -> Tuple[torch.Tensor, torch.Tensor]:
    """cos/sin [S, D/2] fp32: angle = pos * theta^(-2i/D) (arch/llama_standard.py:74-75,83-84)."""
    freqs = torch.pow(torch.tensor(float(theta), dtype=torch.float32),
                      -torch.arange(0, head_dim, 2, dtype=torch.float32) / head_dim)
    ang = torch.outer(torch.arange(seq_len, dtype=torch.float32), freqs)
    return torch.cos(ang).to(device).contiguous(), torch.sin(ang).to(device).contiguous()


ROPE_LAYOUTS = ("interleaved", "half")
GLU_ACTS = ("sigmoid2", "silu")


def _check_choice(value, allowed, what: str) -> str:
    if not isinstance(value, str) or value not in allowed:
        raise ValueError(f"{what} must be one of {allowed}, got {value!r}")
    return value


def _rope_call(x, y, cos_t, sin_t, pos, backward: int, what: str, layout: str = "interleaved") -> None:
    B, S, NH, D = x.shape
    if layout == "half":
        check(lib().b200_rope_half(x.data_ptr(), y.data_ptr(), cos_t.data_ptr(), sin_t.data_ptr(), _ptr(pos), B, S,
                                   NH, D, backward, _is_bf16(x, "x"), _stream()), what)
    elif pos is None:
        check(lib().b200_rope(x.data_ptr(), y.data_ptr(), cos_t.data_ptr(), sin_t.data_ptr(), B, S,
                              NH, D, backward, _is_bf16(x, "x"), _stream()), what)
    else:
        check(lib().b200_rope_pos(x.data_ptr(), y.data_ptr(), cos_t.data_ptr(), sin_t.data_ptr(), pos.data_ptr(), B,
                                  S, NH, D, backward, _is_bf16(x, "x"), _stream()), what)


class _RopeFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, cos_t, sin_t, pos, layout):
        xs = x.contiguous()
        y = torch.empty_like(xs)
        _rope_call(xs, y, cos_t, sin_t, pos, 0, "b200_rope", layout)
        ctx.save_for_backward(cos_t, sin_t, pos)
        ctx.layout = layout
        return y

    @staticmethod
    def backward(ctx, dy):
        cos_t, sin_t, pos = ctx.saved_tensors
        dy = dy.contiguous()
        dx = torch.empty_like(dy)
        _rope_call(dy, dx, cos_t, sin_t, pos, 1, "b200_rope(bwd)", ctx.layout)
        return dx, None, None, None, None


def _check_pos(pos: torch.Tensor, x: torch.Tensor, what: str) -> torch.Tensor:
    """pos: int32 [B, S] positions within documents on x's device (x: [B, S, ...])."""
    if pos.dtype != torch.int32 or pos.dim() != 2 or tuple(pos.shape) != tuple(x.shape[:2]):
        raise ValueError(f"{what}: pos must be int32 [B, S] = {list(x.shape[:2])}, got {pos.dtype} {list(pos.shape)}")
    if pos.device != x.device:
        raise ValueError(f"{what}: pos is on {pos.device}, the operands on {x.device}")
    return pos.contiguous()


def rope(x: torch.Tensor, cos_t: torch.Tensor, sin_t: torch.Tensor, pos: Optional[torch.Tensor] = None,
         layout: str = "interleaved") -> torch.Tensor:
    """x: [B, S, heads, D]; rotation of token s by the angle of position s, or of pos[b, s] (int32 [B, S], the
    position within its document; the tables must then hold max(pos) + 1 rows) when pos is given.
    layout "interleaved" rotates pairs (x[2i], x[2i+1]) (b200_rope); "half" rotates (x[i], x[i + D/2]), mlx_lm's
    nn.RoPE(traditional=False) (b200_rope_half, D % 16 == 0).  Pair i's angle is pos * theta^(-2i/D) in both."""
    _check_choice(layout, ROPE_LAYOUTS, "rope: layout")
    if layout == "half" and x.shape[-1] % 16 != 0:
        raise ValueError(f"rope: the half layout needs head_dim % 16 == 0, got {x.shape[-1]}")
    if pos is not None:
        pos = _check_pos(pos, x, "rope")
    return _RopeFn.apply(x, cos_t, sin_t, pos, layout)


def _pad_head_dim(D: int) -> int:
    if D <= 64:
        return 64
    if D <= 128:
        return 128
    raise ValueError(f"attention: head_dim {D} > 128 is not supported")


def _check_window(window, what: str) -> int:
    """A sliding-window size: a non-negative int (query q sees keys q - window .. q)."""
    if isinstance(window, bool) or not isinstance(window, int) or window < 0:
        raise ValueError(f"{what}: window must be a non-negative int, got {window!r}")
    return window


def _check_alibi(alibi: torch.Tensor, q: torch.Tensor, causal: bool, what: str) -> torch.Tensor:
    """ALiBi slopes: a contiguous fp32 [H] tensor on q's device (q: [B, S, H, D] or [B, H, D]), causal attention only.
    The values are not checked: that would read the device."""
    if not causal:
        raise ValueError(f"{what}: ALiBi is defined for causal attention only (causal=False given)")
    H = q.shape[-2]
    if not isinstance(alibi, torch.Tensor) or alibi.dtype != torch.float32 or tuple(alibi.shape) != (H,):
        raise ValueError(f"{what}: alibi must be an fp32 [H] = [{H}] tensor of slopes, got "
                         f"{getattr(alibi, 'dtype', type(alibi))} {list(getattr(alibi, 'shape', []))}")
    if alibi.device != q.device or not alibi.is_contiguous():
        raise ValueError(f"{what}: alibi must be contiguous and on {q.device}, got {alibi.device}")
    return alibi


def _check_prefix(prefix: torch.Tensor, q: torch.Tensor, causal: bool, pos, window, alibi, what: str) -> torch.Tensor:
    """Prefix lengths: an int32 [B] tensor on q's device.  The prefix mask is its own causal mask, so it does not
    combine with pos, window, alibi or causal=False.  The values are not checked (that would read the device): the
    kernels clamp them to [0, S]."""
    for name, given in (("pos", pos is not None), ("window", window is not None), ("alibi", alibi is not None),
                        ("causal=False", not causal)):
        if given:
            raise ValueError(f"{what}: prefix does not combine with {name}")
    B = q.shape[0]
    if not isinstance(prefix, torch.Tensor) or prefix.dtype != torch.int32 or tuple(prefix.shape) != (B,):
        raise ValueError(f"{what}: prefix must be an int32 [B] = [{B}] tensor of prefix lengths, got "
                         f"{getattr(prefix, 'dtype', type(prefix))} {list(getattr(prefix, 'shape', []))}")
    if prefix.device != q.device:
        raise ValueError(f"{what}: prefix is on {prefix.device}, the operands on {q.device}")
    return prefix.contiguous()


_MASK64 = (1 << 64) - 1


def splitmix64(x: int) -> int:
    """One step of Steele, Lea and Flood's splitmix64 (OOPSLA 2014): x + golden gamma, then the finaliser."""
    z = (x + 0x9E3779B97F4A7C15) & _MASK64
    z = ((z ^ (z >> 30)) * 0xBF58476D1CE4E5B9) & _MASK64
    z = ((z ^ (z >> 27)) * 0x94D049BB133111EB) & _MASK64
    return z ^ (z >> 31)


def dropout_seed(*parts: int) -> int:
    """The attention-dropout seed chain: x = 0, then x = splitmix64(x ^ part) for each part.  The trainer's per-step
    base is dropout_seed(system.seed, rank, step) and layer i's launch seed dropout_seed(base, i), so seeds are
    deterministic in (seed, rank, step, layer) and nothing of them enters a checkpoint."""
    x = 0
    for part in parts:
        x = splitmix64(x ^ (int(part) & _MASK64))
    return x


def _check_dropout(p, seed, prefix, what: str):
    """(p, seed) of attention dropout, or None when p == 0.  p: a float in [0, 1); seed: an int in [0, 2^64), or None
    for one drawn from torch's CPU generator (a host draw, no device read)."""
    if isinstance(p, bool) or not isinstance(p, (float, int)) or not (0.0 <= float(p) < 1.0):
        raise ValueError(f"{what}: dropout must be a float in [0, 1), got {p!r}")
    if seed is not None and (isinstance(seed, bool) or not isinstance(seed, int) or not 0 <= seed < 1 << 64):
        raise ValueError(f"{what}: seed must be an int in [0, 2^64), got {seed!r}")
    if float(p) == 0.0:
        return None
    if prefix is not None:
        raise ValueError(f"{what}: dropout does not combine with prefix")
    if seed is None:
        seed = int(torch.randint(-(1 << 63), (1 << 63) - 1, (1,), dtype=torch.int64).item()) & _MASK64
    # the C entries quantise their fp32 p; passing p_eff = t / 65536 (exact in fp32) makes t that of the double p
    t = min(round(float(p) * 65536.0), 65535)
    return t / 65536.0, int(seed)


def attention_fwd_raw(q, k, v, scale: float, causal: bool, pos: Optional[torch.Tensor] = None,
                      window: Optional[int] = None, alibi: Optional[torch.Tensor] = None,
                      prefix: Optional[torch.Tensor] = None, drop=None):
    """q [B,S,H,D], k/v [B,S,Hk,D] bf16 contiguous, D in {64,128}. Returns (o, lse[B,H,S]).  With pos (int32 [B,S]
    contiguous, positions within documents) the mask is document-causal and `causal` is ignored.  With window (an
    int >= 0) query s sees keys s - min(pos[s], window) .. s (pos[s] = s without pos), and `causal` is ignored.
    With alibi (fp32 [H] slopes, checked by the caller) the causal / document / window mask gets the ALiBi bias.
    With prefix (int32 [B], checked by the caller) query s of row b sees key k iff k <= s or k < prefix[b].
    With drop = (p, seed) (checked by the caller; not with prefix) the dropout entry computes
    O = (P o Z / (1 - p_eff)) V under the same mask; the LSE is the dropout-free one."""
    for t, nm in ((q, "q"), (k, "k"), (v, "v")):
        _need(t, torch.bfloat16, nm)
    B, S, H, D = q.shape
    Hk = k.shape[2]
    o = torch.empty_like(q)
    lse = torch.empty((B, H, S), device=q.device, dtype=torch.float32)
    tok = _t0("attn_fwd")
    if drop is not None:
        check(lib().b200_attn_fwd_dropout(q.data_ptr(), k.data_ptr(), v.data_ptr(), o.data_ptr(), lse.data_ptr(),
                                          _ptr(pos), -1 if window is None else min(int(window), S), _ptr(alibi),
                                          B, S, H, Hk, D, float(scale), int(causal), drop[0], drop[1], _stream()),
              "b200_attn_fwd_dropout")
    elif prefix is not None:
        check(lib().b200_attn_fwd_prefix(q.data_ptr(), k.data_ptr(), v.data_ptr(), o.data_ptr(), lse.data_ptr(),
                                         prefix.data_ptr(), B, S, H, Hk, D, float(scale), _stream()),
              "b200_attn_fwd_prefix")
    elif alibi is not None:
        check(lib().b200_attn_fwd_alibi(q.data_ptr(), k.data_ptr(), v.data_ptr(), o.data_ptr(), lse.data_ptr(),
                                        _ptr(pos), -1 if window is None else min(int(window), S), alibi.data_ptr(),
                                        B, S, H, Hk, D, float(scale), _stream()), "b200_attn_fwd_alibi")
    elif window is not None:
        check(lib().b200_attn_fwd_window(q.data_ptr(), k.data_ptr(), v.data_ptr(), o.data_ptr(), lse.data_ptr(),
                                         _ptr(pos), min(int(window), S), B, S, H, Hk, D, float(scale), _stream()),
              "b200_attn_fwd_window")
    elif pos is None:
        check(lib().b200_attn_fwd(q.data_ptr(), k.data_ptr(), v.data_ptr(), o.data_ptr(), lse.data_ptr(),
                                  B, S, H, Hk, D, float(scale), int(causal), _stream()), "b200_attn_fwd")
    else:
        check(lib().b200_attn_fwd_doc(q.data_ptr(), k.data_ptr(), v.data_ptr(), o.data_ptr(), lse.data_ptr(),
                                      pos.data_ptr(), B, S, H, Hk, D, float(scale), _stream()), "b200_attn_fwd_doc")
    _t1(tok)
    return o, lse


def attention_bwd_raw(q, k, v, o, do, lse, scale: float, causal: bool, pos: Optional[torch.Tensor] = None,
                      window: Optional[int] = None, alibi: Optional[torch.Tensor] = None,
                      prefix: Optional[torch.Tensor] = None, drop=None):
    B, S, H, D = q.shape
    Hk = k.shape[2]
    dq = torch.empty_like(q)
    # dk and dv share one [B, S, 2*Hk, D] buffer (dk = first Hk heads of every token row, dv = the rest): the
    # k/v projections' backward can then treat [dk | dv] as ONE matrix against the concatenated weight
    dkv = torch.empty((B, S, 2 * Hk, D), device=k.device, dtype=k.dtype)
    dk, dv = dkv[:, :, :Hk], dkv[:, :, Hk:]
    tok = _t0("attn_bwd")
    if drop is not None:
        nbytes = int(lib().b200_attn_bwd_dropout_workspace_bytes(B, S, H, Hk, D))
        ws = torch.empty(max(nbytes, 16), device=q.device, dtype=torch.uint8)
        check(lib().b200_attn_bwd_dropout(q.data_ptr(), k.data_ptr(), v.data_ptr(), o.data_ptr(), do.data_ptr(),
                                          lse.data_ptr(), _ptr(pos), -1 if window is None else min(int(window), S),
                                          _ptr(alibi), dq.data_ptr(), dk.data_ptr(), dv.data_ptr(), B, S, H, Hk, D,
                                          float(scale), int(causal), drop[0], drop[1], 2 * Hk, ws.data_ptr(),
                                          ws.numel(), _stream()), "b200_attn_bwd_dropout")
    elif prefix is not None:
        nbytes = int(lib().b200_attn_bwd_prefix_workspace_bytes(B, S, H, Hk, D))
        ws = torch.empty(max(nbytes, 16), device=q.device, dtype=torch.uint8)
        check(lib().b200_attn_bwd_prefix(q.data_ptr(), k.data_ptr(), v.data_ptr(), o.data_ptr(), do.data_ptr(),
                                         lse.data_ptr(), prefix.data_ptr(), dq.data_ptr(), dk.data_ptr(),
                                         dv.data_ptr(), B, S, H, Hk, D, float(scale), 2 * Hk, ws.data_ptr(),
                                         ws.numel(), _stream()), "b200_attn_bwd_prefix")
    elif alibi is not None:
        nbytes = int(lib().b200_attn_bwd_window_workspace_bytes(B, S, H, Hk, D))
        ws = torch.empty(max(nbytes, 16), device=q.device, dtype=torch.uint8)
        check(lib().b200_attn_bwd_alibi(q.data_ptr(), k.data_ptr(), v.data_ptr(), o.data_ptr(), do.data_ptr(),
                                        lse.data_ptr(), _ptr(pos), -1 if window is None else min(int(window), S),
                                        alibi.data_ptr(), dq.data_ptr(), dk.data_ptr(), dv.data_ptr(), B, S, H, Hk, D,
                                        float(scale), 2 * Hk, ws.data_ptr(), ws.numel(), _stream()),
              "b200_attn_bwd_alibi")
    elif window is not None:
        nbytes = int(lib().b200_attn_bwd_window_workspace_bytes(B, S, H, Hk, D))
        ws = torch.empty(max(nbytes, 16), device=q.device, dtype=torch.uint8)
        check(lib().b200_attn_bwd_window(q.data_ptr(), k.data_ptr(), v.data_ptr(), o.data_ptr(), do.data_ptr(),
                                         lse.data_ptr(), _ptr(pos), min(int(window), S), dq.data_ptr(), dk.data_ptr(),
                                         dv.data_ptr(), B, S, H, Hk, D, float(scale), 2 * Hk, ws.data_ptr(),
                                         ws.numel(), _stream()), "b200_attn_bwd_window")
    elif pos is None:
        nbytes = int(lib().b200_attn_bwd_workspace_bytes(B, S, H, Hk, D))
        ws = torch.empty(max(nbytes, 16), device=q.device, dtype=torch.uint8)
        check(lib().b200_attn_bwd_strided(q.data_ptr(), k.data_ptr(), v.data_ptr(), o.data_ptr(), do.data_ptr(),
                                          lse.data_ptr(), dq.data_ptr(), dk.data_ptr(), dv.data_ptr(), B, S, H,
                                          Hk, D, float(scale), int(causal), 2 * Hk, ws.data_ptr(), ws.numel(),
                                          _stream()), "b200_attn_bwd_strided")
    else:
        nbytes = int(lib().b200_attn_bwd_doc_workspace_bytes(B, S, H, Hk, D))
        ws = torch.empty(max(nbytes, 16), device=q.device, dtype=torch.uint8)
        check(lib().b200_attn_bwd_doc(q.data_ptr(), k.data_ptr(), v.data_ptr(), o.data_ptr(), do.data_ptr(),
                                      lse.data_ptr(), pos.data_ptr(), dq.data_ptr(), dk.data_ptr(), dv.data_ptr(), B,
                                      S, H, Hk, D, float(scale), 2 * Hk, ws.data_ptr(), ws.numel(), _stream()),
              "b200_attn_bwd_doc")
    _t1(tok)
    return dq, dk, dv


class _AttentionFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, q, k, v, scale, causal, pos, window, alibi=None, prefix=None, drop=None):
        D = q.shape[-1]
        Dp = _pad_head_dim(D)
        if Dp != D:  # zero-padding the head dim leaves QK^T and the first D columns of PV unchanged
            q, k, v = (torch.nn.functional.pad(t, (0, Dp - D)) for t in (q, k, v))
        q, k, v = q.contiguous(), k.contiguous(), v.contiguous()
        o, lse = attention_fwd_raw(q, k, v, scale, causal, pos, window, alibi, prefix, drop)
        ctx.save_for_backward(q, k, v, o, lse, pos, alibi, prefix)
        ctx.scale, ctx.causal, ctx.D, ctx.window, ctx.drop = scale, causal, D, window, drop
        return o[..., :D] if Dp != D else o

    @staticmethod
    def backward(ctx, do):
        q, k, v, o, lse, pos, alibi, prefix = ctx.saved_tensors
        Dp = q.shape[-1]
        if Dp != ctx.D:
            do = torch.nn.functional.pad(do, (0, Dp - ctx.D))
        do = do.contiguous()
        dq, dk, dv = attention_bwd_raw(q, k, v, o, do, lse, ctx.scale, ctx.causal, pos, ctx.window, alibi, prefix,
                                       ctx.drop)
        if Dp != ctx.D:
            dq, dk, dv = dq[..., :ctx.D], dk[..., :ctx.D], dv[..., :ctx.D]
        return dq, dk, dv, None, None, None, None, None, None, None


def _hi_lo(x: torch.Tensor):
    hi = x.to(torch.bfloat16)
    return hi, (x - hi.float()).to(torch.bfloat16)


class _AttentionX3Fn(torch.autograd.Function):
    """fp32 attention on the bf16 tensor-core kernels for small head dims (3*D <= 128), used when the config asks
    for full precision (`mixed_precision: false`, e.g. BASELINE C1 with D = 16).  Each fp32 operand x = hi + lo
    (two bf16) is laid along the head dimension so that ONE bf16 kernel call evaluates the three-term products:

        Q' = [qh | ql | qh]   K' = [kh | kh | kl]   ->  Q'K'^T = qh kh + ql kh + qh kl  ~=  q k^T   (~16 bits)
        V' = [vh | vh | vl]                         ->  O' = [P vh | P vh | P vl],  o = O'[0:D] + O'[2D:3D]
        dO' = [gh | gl | gh]  ->  dP = gh vh + gl vh + gh vl ;  dq = dQ'[0:D] + dQ'[2D:3D],
                                  dk = dK'[0:D] + dK'[D:2D],    dv = dV'[0:D] + dV'[D:2D]

    The logits (where bf16 operand rounding hurts most: an error of |s| * 2^-9 in the exponent) are thus computed
    to fp32-like accuracy; P and the kernel outputs still pass through one bf16 rounding each.

    Dropout needs no kernel of its own here: the keep mask acts on P, which the three concatenated segments share
    (one softmax per (query, key) pair, whatever the head dim), so O' = [P~ vh | P~ vh | P~ vl] with P~ = P o Z /
    (1 - p_eff), and the backward's dV' and dS are those of the same P~."""

    @staticmethod
    def forward(ctx, q, k, v, scale, causal, pos, window, alibi=None, prefix=None, drop=None):
        D = q.shape[-1]
        Dp = _pad_head_dim(3 * D)
        (qh, ql), (kh, kl), (vh, vl) = _hi_lo(q), _hi_lo(k), _hi_lo(v)

        def cat3(a, b, c):
            t = torch.cat([a, b, c], dim=-1)
            return (torch.nn.functional.pad(t, (0, Dp - 3 * D)) if Dp != 3 * D else t).contiguous()
        q3, k3, v3 = cat3(qh, ql, qh), cat3(kh, kh, kl), cat3(vh, vh, vl)
        o3, lse = attention_fwd_raw(q3, k3, v3, scale, causal, pos, window, alibi, prefix, drop)
        ctx.save_for_backward(q3, k3, v3, o3, lse, pos, alibi, prefix)
        ctx.scale, ctx.causal, ctx.D, ctx.Dp, ctx.window, ctx.drop = scale, causal, D, Dp, window, drop
        return o3[..., :D].float() + o3[..., 2 * D:3 * D].float()

    @staticmethod
    def backward(ctx, do):
        q3, k3, v3, o3, lse, pos, alibi, prefix = ctx.saved_tensors
        D, Dp = ctx.D, ctx.Dp
        gh, gl = _hi_lo(do.float())
        g3 = torch.cat([gh, gl, gh], dim=-1)
        if Dp != 3 * D:
            g3 = torch.nn.functional.pad(g3, (0, Dp - 3 * D))
        dq3, dk3, dv3 = attention_bwd_raw(q3, k3, v3, o3, g3.contiguous(), lse, ctx.scale, ctx.causal, pos,
                                          ctx.window, alibi, prefix, ctx.drop)
        dq = dq3[..., :D].float() + dq3[..., 2 * D:3 * D].float()
        dk = dk3[..., :D].float() + dk3[..., D:2 * D].float()
        dv = dv3[..., :D].float() + dv3[..., D:2 * D].float()
        return dq, dk, dv, None, None, None, None, None, None, None


def attention_fp32(q: torch.Tensor, k: torch.Tensor, v: torch.Tensor, scale: Optional[float] = None,
                   causal: bool = True, pos: Optional[torch.Tensor] = None, window: Optional[int] = None,
                   alibi: Optional[torch.Tensor] = None, prefix: Optional[torch.Tensor] = None,
                   dropout: float = 0.0, seed: Optional[int] = None) -> torch.Tensor:
    """fp32 in / fp32 out attention with bf16x3 logits (see _AttentionX3Fn); head_dim <= 42.  pos, window, alibi,
    prefix, dropout, seed: as attention."""
    if 3 * q.shape[-1] > 128:
        raise ValueError("attention_fp32: head_dim must be <= 42 (three bf16 copies must fit a 128-wide tile)")
    if scale is None:
        scale = q.shape[-1] ** -0.5
    if pos is not None:
        pos, causal = _check_pos(pos, q, "attention_fp32"), True
    if window is not None:
        window, causal = _check_window(window, "attention_fp32"), True
    if prefix is not None:
        prefix = _check_prefix(prefix, q, causal, pos, window, alibi, "attention_fp32")
    if alibi is not None:
        alibi = _check_alibi(alibi, q, causal, "attention_fp32")
    drop = _check_dropout(dropout, seed, prefix, "attention_fp32")
    return _AttentionX3Fn.apply(q.float(), k.float(), v.float(), float(scale), bool(causal), pos, window, alibi,
                                prefix, drop)


def attention(q: torch.Tensor, k: torch.Tensor, v: torch.Tensor, scale: Optional[float] = None,
              causal: bool = True, pos: Optional[torch.Tensor] = None, window: Optional[int] = None,
              alibi: Optional[torch.Tensor] = None, prefix: Optional[torch.Tensor] = None,
              dropout: float = 0.0, seed: Optional[int] = None) -> torch.Tensor:
    """softmax(q k^T * scale + causal_mask) v with GQA head sharing; [B,S,H,D] layout, bf16.

    pos (int32 [B, S]) packs several documents per row: pos[b, s] is token s's position within its document (0 at a
    document's first token, +1 per token inside it), and query s sees only keys s - pos[b, s] .. s -- the causal
    attention of each document run alone.  It implies causal.

    window (int >= 0) is a sliding causal window: query s sees key k iff 0 <= s - k <= window, at most window + 1
    keys, intersected with the document when pos is given (keys s - min(pos[b, s], window) .. s).  Tiles outside
    every row's window are skipped, so the cost is linear in S.  It implies causal.

    alibi (fp32 [H] slopes on q's device, one per query head; see arch.flash_attention.alibi_slopes) adds ALiBi's
    bias alibi[h] * (k - s) to the scaled score of query s and key k before the mask and the softmax.  k - s is also
    the distance inside a document, so it composes with pos and window.  Causal only: causal=False raises.

    prefix (int32 [B] on q's device) is the prefix-LM mask: query s of row b sees key k iff k <= s or k < prefix[b],
    so each row's prefix attends bidirectionally within itself and the rest of the row is causal.  prefix[b] <= 1 is
    the causal mask and prefix[b] = S full attention; values outside [0, S] act as their clamps.  It implies causal
    for the rest of the row and raises together with pos, window, alibi or causal=False.

    dropout (a float p in [0, 1)) drops attention probabilities as the reference's mx.dropout after the softmax:
    O = (P o Z / (1 - p_eff)) V, with p_eff = min(rint(p 65536), 65535) / 65536 and Z the Philox keep mask of
    (seed, b, h, q, k) stated in include/b200_hotpath.h (b200_attn_fwd_dropout); the backward regenerates it.  seed
    (an int in [0, 2^64)) fixes the mask; None draws one from torch's CPU generator.  It composes with every mask
    except prefix.  dropout = 0 calls the dropout-free kernels exactly as without it.  The caller decides when to
    drop: the model does only in training mode with grad enabled."""
    if scale is None:
        scale = q.shape[-1] ** -0.5
    if prefix is not None:
        prefix = _check_prefix(prefix, q, causal, pos, window, alibi, "attention")
    if pos is not None:
        pos, causal = _check_pos(pos, q, "attention"), True
    if window is not None:
        window, causal = _check_window(window, "attention"), True
    if alibi is not None:
        alibi = _check_alibi(alibi, q, causal, "attention")
    drop = _check_dropout(dropout, seed, prefix, "attention")
    return _AttentionFn.apply(q, k, v, float(scale), bool(causal), pos, window, alibi, prefix, drop)


# ------------------------------------------------------------------------------------------------
# generation: decode attention over a KV cache and the per-token cache append
# ------------------------------------------------------------------------------------------------
def attention_decode_workspace_bytes(B: int, H: int, s_max: int, D: int) -> int:
    return int(lib().b200_attn_decode_workspace_bytes(B, H, s_max, D))


def _check_rows(t, B: int, device, what: str, nm: str) -> None:
    if not isinstance(t, torch.Tensor) or t.dtype != torch.int32 or tuple(t.shape) != (B,) or t.device != device \
            or not t.is_contiguous():
        raise ValueError(f"{what}: {nm} must be a contiguous int32 [{B}] tensor on {device}, got "
                         f"{getattr(t, 'dtype', type(t))} {list(getattr(t, 'shape', []))}")


def _check_scores(q: torch.Tensor, scale, window, alibi, what: str):
    """(window, alibi, scale) of an attention-over-a-cache wrapper: window and ALiBi slopes checked, scale defaulting
    to head_dim ** -0.5."""
    if window is not None:
        window = _check_window(window, what)
    if alibi is not None:
        alibi = _check_alibi(alibi, q, True, what)
    return window, alibi, q.shape[-1] ** -0.5 if scale is None else scale


def _check_workspace(workspace: Optional[torch.Tensor], need: int, device, what: str, align: int = 1) -> torch.Tensor:
    """The decode workspace: allocated when None, else checked to be uint8 on `device`, align-byte aligned, with at
    least `need` bytes."""
    if workspace is None:
        return torch.empty(max(need, 16), device=device, dtype=torch.uint8)
    if workspace.dtype != torch.uint8 or workspace.device != device or workspace.numel() < need \
            or workspace.data_ptr() % align:
        aligned = f"{align}-byte aligned " if align > 1 else ""
        raise ValueError(f"{what}: workspace must be {aligned}uint8 on {device} with >= {need} bytes")
    return workspace


def _check_rope_tables(rope_tables: Optional[Tuple[torch.Tensor, torch.Tensor]], D: int, layout: str, what: str):
    """(cos, sin, half) of a cache-append wrapper: the fp32 [positions, D / 2] tables of rope_tables() (None, None
    without RoPE) and the flag of the half layout (0 without RoPE)."""
    if rope_tables is None:
        return None, None, 0
    cos_t, sin_t = rope_tables
    for t, nm in ((cos_t, "cos"), (sin_t, "sin")):
        _need(t, torch.float32, f"{what}: {nm}")
        if t.dim() != 2 or t.shape[1] != D // 2:
            raise ValueError(f"{what}: RoPE tables must be [positions, {D // 2}]")
    return cos_t, sin_t, int(layout == "half")


def _check_cache(q: torch.Tensor, k_cache: torch.Tensor, v_cache: torch.Tensor, lens: torch.Tensor, what: str):
    _is_bf16(q, "q")
    for t, nm in ((q, "q"), (k_cache, "k_cache"), (v_cache, "v_cache")):
        _need(t, q.dtype, f"{what}: {nm}")
    if q.dim() != 3 or k_cache.dim() != 4 or k_cache.shape != v_cache.shape:
        raise ValueError(f"{what}: expected q [B,H,D] and k_cache == v_cache [B,s_max,Hk,D], got "
                         f"{tuple(q.shape)}, {tuple(k_cache.shape)}, {tuple(v_cache.shape)}")
    B, H, D = q.shape
    Bc, s_max, Hk, Dc = k_cache.shape
    if Bc != B or Dc != D or H % Hk != 0:
        raise ValueError(f"{what}: q {tuple(q.shape)} does not match cache {tuple(k_cache.shape)}")
    _check_rows(lens, B, q.device, what, "lens")
    return B, H, D, s_max, Hk


def attention_decode(q: torch.Tensor, k_cache: torch.Tensor, v_cache: torch.Tensor, lens: torch.Tensor,
                     scale: Optional[float] = None, workspace: Optional[torch.Tensor] = None,
                     return_lse: bool = False, window: Optional[int] = None, alibi: Optional[torch.Tensor] = None):
    """softmax(q K^T * scale) V for one new query per row over its first lens[b] cached keys (b200_attn_decode).

    q [B,H,D]; k_cache, v_cache [B,s_max,Hk,D]; all bf16 or all fp32, D in {16, 32, 64, 128}; lens int32 [B] on the
    device, 1 <= lens[b] <= s_max (not checked here: that would read the device).  `workspace` (uint8, at least
    attention_decode_workspace_bytes(B, H, s_max, D)) is allocated when not given.  Returns o [B,H,D] in q's dtype,
    and the natural-log LSE [B,H] fp32 with return_lse.  window (int >= 0): the query at position p = lens[b] - 1
    sees only keys max(0, p - window) .. p (b200_attn_decode_window), and only those are read.  alibi (fp32 [H]
    slopes on the device): ALiBi's bias alibi[h] * (k - p) on every cached key k (b200_attn_decode_alibi)."""
    B, H, D, s_max, Hk = _check_cache(q, k_cache, v_cache, lens, "attention_decode")
    if D not in (16, 32, 64, 128):
        raise ValueError(f"attention_decode: head_dim {D} unsupported (16, 32, 64 or 128)")
    window, alibi, scale = _check_scores(q, scale, window, alibi, "attention_decode")
    workspace = _check_workspace(workspace, attention_decode_workspace_bytes(B, H, s_max, D), q.device,
                                 "attention_decode")
    o = torch.empty_like(q)
    lse = torch.empty((B, H), device=q.device, dtype=torch.float32) if return_lse else None
    tok = _t0("attn_decode")
    if alibi is not None:
        check(lib().b200_attn_decode_alibi(q.data_ptr(), k_cache.data_ptr(), v_cache.data_ptr(), lens.data_ptr(),
                                           o.data_ptr(), _ptr(lse), -1 if window is None else min(int(window), s_max),
                                           alibi.data_ptr(), B, s_max, H, Hk, D, float(scale), _is_bf16(q, "q"),
                                           workspace.data_ptr(), workspace.numel(), _stream()),
              "b200_attn_decode_alibi")
    elif window is None:
        check(lib().b200_attn_decode(q.data_ptr(), k_cache.data_ptr(), v_cache.data_ptr(), lens.data_ptr(),
                                     o.data_ptr(), _ptr(lse), B, s_max, H, Hk, D, float(scale), _is_bf16(q, "q"),
                                     workspace.data_ptr(), workspace.numel(), _stream()), "b200_attn_decode")
    else:
        check(lib().b200_attn_decode_window(q.data_ptr(), k_cache.data_ptr(), v_cache.data_ptr(), lens.data_ptr(),
                                            o.data_ptr(), _ptr(lse), min(int(window), s_max), B, s_max, H, Hk, D,
                                            float(scale), _is_bf16(q, "q"), workspace.data_ptr(), workspace.numel(),
                                            _stream()),
              "b200_attn_decode_window")
    _t1(tok)
    return (o, lse) if return_lse else o


MULTI_MAX_QUERIES = 16  # queries per row of attention_decode_multi


def attention_decode_multi_workspace_bytes(B: int, L: int, H: int, s_max: int, D: int) -> int:
    return int(lib().b200_attn_decode_multi_workspace_bytes(B, L, H, s_max, D))


def attention_decode_multi(q: torch.Tensor, k_cache: torch.Tensor, v_cache: torch.Tensor, start: torch.Tensor,
                           end: torch.Tensor, scale: Optional[float] = None, workspace: Optional[torch.Tensor] = None,
                           window: Optional[int] = None, alibi: Optional[torch.Tensor] = None,
                           return_lse: bool = False):
    """A short chunk of L <= 16 new queries per row against the dense KV cache that already holds their keys
    (b200_attn_decode_multi): speculative decoding's verify step, split over keys as attention_decode is.

    q [B,L,H,D]; k_cache, v_cache [B,s_max,Hk,D]; all bf16 or all fp32, D in {16, 32, 64, 128}.  start, end: int32
    [B] on the device.  Query i of row b sits at position p = start[b] + i and sees the cached keys max(0, p - window)
    .. p (window None: from 0), with ALiBi's bias alibi[h] * (k - p) when alibi (fp32 [H] slopes) is given.  Rows
    i >= end[b] - start[b] are padding: the kernel does not write them, and o and lse hold 0 there.  Cache positions at or past end[b] are never read.  The values of
    start and end are not checked here (that would read the device): 0 <= start[b] <= end[b] <= s_max.  `workspace`
    (uint8, at least attention_decode_multi_workspace_bytes(B, L, H, s_max, D)) is allocated when not given.  With
    L = 1 the result is bit-equal to attention_decode with lens = end.  Returns o [B,L,H,D] in q's dtype, and the
    natural-log LSE [B,H,L] fp32 with return_lse."""
    what = "attention_decode_multi"
    _is_bf16(q, "q")
    for t, nm in ((q, "q"), (k_cache, "k_cache"), (v_cache, "v_cache")):
        _need(t, q.dtype, f"{what}: {nm}")
    if q.dim() != 4 or k_cache.dim() != 4 or k_cache.shape != v_cache.shape:
        raise ValueError(f"{what}: expected q [B,L,H,D] and k_cache == v_cache [B,s_max,Hk,D], got "
                         f"{tuple(q.shape)}, {tuple(k_cache.shape)}, {tuple(v_cache.shape)}")
    B, L, H, D = q.shape
    Bc, s_max, Hk, Dc = k_cache.shape
    if Bc != B or Dc != D or H % Hk != 0:
        raise ValueError(f"{what}: q {tuple(q.shape)} does not match cache {tuple(k_cache.shape)}")
    if D not in (16, 32, 64, 128):
        raise ValueError(f"{what}: head_dim {D} unsupported (16, 32, 64 or 128)")
    if not 1 <= L <= MULTI_MAX_QUERIES:
        raise ValueError(f"{what}: {L} queries per row, 1 to {MULTI_MAX_QUERIES} supported")
    _check_rows(start, B, q.device, what, "start")
    _check_rows(end, B, q.device, what, "end")
    window, alibi, scale = _check_scores(q, scale, window, alibi, what)
    workspace = _check_workspace(workspace, attention_decode_multi_workspace_bytes(B, L, H, s_max, D), q.device, what)
    o = torch.zeros_like(q)
    lse = torch.zeros((B, H, L), device=q.device, dtype=torch.float32) if return_lse else None
    tok = _t0("attn_decode_multi")
    check(lib().b200_attn_decode_multi(q.data_ptr(), k_cache.data_ptr(), v_cache.data_ptr(), start.data_ptr(),
                                       end.data_ptr(), o.data_ptr(), _ptr(lse),
                                       -1 if window is None else min(int(window), s_max), _ptr(alibi), B, L, s_max, H,
                                       Hk, D, float(scale), _is_bf16(q, "q"), workspace.data_ptr(), workspace.numel(),
                                       _stream()), "b200_attn_decode_multi")
    _t1(tok)
    return (o, lse) if return_lse else o


def kv_append(q: torch.Tensor, k: torch.Tensor, v: torch.Tensor, k_cache: torch.Tensor, v_cache: torch.Tensor,
              lens: torch.Tensor, rope_tables: Optional[Tuple[torch.Tensor, torch.Tensor]] = None,
              layout: str = "interleaved") -> None:
    """Writes each row's new k [B,Hk,D] and v into the caches at pos = lens[b] - 1 (b200_kv_append).  With
    rope_tables = (cos, sin) from rope_tables(), k and, in place, q [B,H,D] get the rotation ops.rope(layout=layout)
    applies at position pos, with the same arithmetic (b200_kv_append_half for the half layout).  The caller keeps
    pos below the tables' length."""
    _check_choice(layout, ROPE_LAYOUTS, "kv_append: layout")
    B, H, D, s_max, Hk = _check_cache(q, k_cache, v_cache, lens, "kv_append")
    for t, nm in ((k, "k"), (v, "v")):
        _need(t, q.dtype, f"kv_append: {nm}")
        if t.shape != (B, Hk, D):
            raise ValueError(f"kv_append: {nm} must be [{B},{Hk},{D}], got {tuple(t.shape)}")
    if D % 8 != 0:
        raise ValueError(f"kv_append: head_dim {D} must be a multiple of 8")
    cos_t, sin_t, half = _check_rope_tables(rope_tables, D, layout, "kv_append")
    if half:
        if D % 16 != 0:
            raise ValueError(f"kv_append: the half layout needs head_dim % 16 == 0, got {D}")
        check(lib().b200_kv_append_half(q.data_ptr(), k.data_ptr(), v.data_ptr(), k_cache.data_ptr(),
                                        v_cache.data_ptr(), lens.data_ptr(), cos_t.data_ptr(), sin_t.data_ptr(), B,
                                        s_max, H, Hk, D, _is_bf16(q, "q"), _stream()), "b200_kv_append_half")
        return
    check(lib().b200_kv_append(q.data_ptr(), k.data_ptr(), v.data_ptr(), k_cache.data_ptr(), v_cache.data_ptr(),
                               lens.data_ptr(), _ptr(cos_t), _ptr(sin_t), B, s_max, H, Hk, D, _is_bf16(q, "q"),
                               _stream()), "b200_kv_append")


def attention_cached(q: torch.Tensor, k_cache: torch.Tensor, v_cache: torch.Tensor, start: torch.Tensor,
                     end: torch.Tensor, scale: Optional[float] = None, window: Optional[int] = None,
                     alibi: Optional[torch.Tensor] = None, return_lse: bool = False):
    """A chunk of L new queries per row against the KV cache that already holds their keys (b200_attn_fwd_cached).

    q [B,L,H,D]; k_cache, v_cache [B,s_max,Hk,D]; all bf16, D in {64, 128}.  start, end: int32 [B] on the device.
    Query i of row b sits at position start[b] + i and sees the cached keys max(0, p - window) .. p (window None: from
    0), with ALiBi's bias alibi[h] * (k - p) when alibi (fp32 [H] slopes) is given.  Rows i >= end[b] - start[b] are
    padding: finite, unspecified.  Cache positions at or past end[b] are never read into the result.  The values of
    start and end are not checked here (that would read the device): 0 <= start[b] <= end[b] <= s_max.  Returns o
    [B,L,H,D] bf16, and the natural-log LSE [B,H,L] fp32 with return_lse."""
    what = "attention_cached"
    for t, nm in ((q, "q"), (k_cache, "k_cache"), (v_cache, "v_cache")):
        if t.dtype != torch.bfloat16:
            raise ValueError(f"{what}: {nm} must be bf16 (an fp32 cache is served by the one-shot prefill only), "
                             f"got {t.dtype}")
        _need(t, torch.bfloat16, f"{what}: {nm}")
    if q.dim() != 4 or k_cache.dim() != 4 or k_cache.shape != v_cache.shape:
        raise ValueError(f"{what}: expected q [B,L,H,D] and k_cache == v_cache [B,s_max,Hk,D], got "
                         f"{tuple(q.shape)}, {tuple(k_cache.shape)}, {tuple(v_cache.shape)}")
    B, L, H, D = q.shape
    Bc, s_max, Hk, Dc = k_cache.shape
    if Bc != B or Dc != D or H % Hk != 0:
        raise ValueError(f"{what}: q {tuple(q.shape)} does not match cache {tuple(k_cache.shape)}")
    if D not in (64, 128):
        raise ValueError(f"{what}: head_dim {D} unsupported (64 or 128)")
    _check_rows(start, B, q.device, what, "start")
    _check_rows(end, B, q.device, what, "end")
    window, alibi, scale = _check_scores(q, scale, window, alibi, what)
    o = torch.empty_like(q)
    lse = torch.empty((B, H, L), device=q.device, dtype=torch.float32) if return_lse else None
    tok = _t0("attn_cached")
    check(lib().b200_attn_fwd_cached(q.data_ptr(), k_cache.data_ptr(), v_cache.data_ptr(), start.data_ptr(),
                                     end.data_ptr(), o.data_ptr(), _ptr(lse),
                                     -1 if window is None else min(int(window), s_max), _ptr(alibi), B, L, s_max, H,
                                     Hk, D, float(scale), _stream()), "b200_attn_fwd_cached")
    _t1(tok)
    return (o, lse) if return_lse else o


# ------------------------------------------------------------------------------------------------
# the rotating KV cache (the reference's max_kv_size; DESIGN §4.2.3): per layer, K and V rings bf16 [B, C, Hk, D]
# ------------------------------------------------------------------------------------------------
RING_SINKS = 4


def ring_slot(pos, slots: int):
    """The slot of position pos in a ring of `slots` slots (include/b200_hotpath.h): pos itself for the sinks
    pos < 4, else 4 + (pos - 4) mod (slots - 4).  pos: an int or an integer tensor."""
    if isinstance(pos, torch.Tensor):
        return torch.where(pos < RING_SINKS, pos, RING_SINKS + (pos - RING_SINKS) % (slots - RING_SINKS))
    return pos if pos < RING_SINKS else RING_SINKS + (pos - RING_SINKS) % (slots - RING_SINKS)


def check_max_kv_size(max_kv_size, what: str = "max_kv_size") -> int:
    if isinstance(max_kv_size, bool) or not isinstance(max_kv_size, int) or max_kv_size < RING_SINKS + 1:
        raise ValueError(f"{what}: max_kv_size must be an int >= {RING_SINKS + 1}, got {max_kv_size!r}")
    return max_kv_size


def _check_ring(q: torch.Tensor, k_ring: torch.Tensor, v_ring: torch.Tensor, max_kv_size, what: str, qdim: int):
    for t, nm in ((q, "q"), (k_ring, "k_ring"), (v_ring, "v_ring")):
        if t.dtype != torch.bfloat16:
            raise ValueError(f"{what}: {nm} must be bf16 (the rotating cache is bf16 only), got {t.dtype}")
        _need(t, torch.bfloat16, f"{what}: {nm}")
    if q.dim() != qdim or k_ring.dim() != 4 or k_ring.shape != v_ring.shape:
        raise ValueError(f"{what}: expected q with {qdim} dims and k_ring == v_ring [B,C,Hk,D], got "
                         f"{tuple(q.shape)}, {tuple(k_ring.shape)}, {tuple(v_ring.shape)}")
    B, H, D = q.shape[0], q.shape[-2], q.shape[-1]
    Bc, C, Hk, Dc = k_ring.shape
    if Bc != B or Dc != D or H % Hk != 0:
        raise ValueError(f"{what}: q {tuple(q.shape)} does not match the ring {tuple(k_ring.shape)}")
    if D not in (64, 128):
        raise ValueError(f"{what}: head_dim {D} unsupported (64 or 128)")
    check_max_kv_size(max_kv_size, what)
    return B, H, D, C, Hk


def attention_decode_ring(q: torch.Tensor, k_ring: torch.Tensor, v_ring: torch.Tensor, end: torch.Tensor,
                          max_kv_size: int, scale: Optional[float] = None, workspace: Optional[torch.Tensor] = None,
                          return_lse: bool = False, window: Optional[int] = None,
                          alibi: Optional[torch.Tensor] = None):
    """attention_decode over a ring of C slots (b200_attn_decode_ring): the query at position p = end[b] - 1 sees
    key positions k <= p with k < 4 or p - k <= max_kv_size - 5 (and p - k <= window), read from slot ring_slot(k, C),
    with ALiBi's bias alibi[h] * (k - p).  q [B,H,D]; k_ring, v_ring [B,C,Hk,D]; all bf16, D in {64, 128};
    C >= max_kv_size; end int32 [B] on the device, end[b] >= 1 (not checked: that would read the device)."""
    what = "attention_decode_ring"
    B, H, D, C, Hk = _check_ring(q, k_ring, v_ring, max_kv_size, what, 3)
    _check_rows(end, B, q.device, what, "end")
    if C < max_kv_size:
        raise ValueError(f"{what}: the ring's {C} slots cannot hold max_kv_size={max_kv_size} keys")
    window, alibi, scale = _check_scores(q, scale, window, alibi, what)
    workspace = _check_workspace(workspace, attention_decode_workspace_bytes(B, H, C, D), q.device, what)
    o = torch.empty_like(q)
    lse = torch.empty((B, H), device=q.device, dtype=torch.float32) if return_lse else None
    tok = _t0("attn_decode_ring")
    check(lib().b200_attn_decode_ring(q.data_ptr(), k_ring.data_ptr(), v_ring.data_ptr(), end.data_ptr(),
                                      o.data_ptr(), _ptr(lse), int(max_kv_size), -1 if window is None else int(window),
                                      _ptr(alibi), B, C, H, Hk, D, float(scale), workspace.data_ptr(),
                                      workspace.numel(), _stream()), "b200_attn_decode_ring")
    _t1(tok)
    return (o, lse) if return_lse else o


def attention_ring(q: torch.Tensor, k_ring: torch.Tensor, v_ring: torch.Tensor, start: torch.Tensor,
                   end: torch.Tensor, max_kv_size: int, scale: Optional[float] = None, window: Optional[int] = None,
                   alibi: Optional[torch.Tensor] = None, return_lse: bool = False):
    """attention_cached over a ring of C slots that already holds the chunk's keys (b200_attn_fwd_ring): query i of
    row b sits at position p = start[b] + i and sees key positions k <= p with k < 4 or p - k <= max_kv_size - 5
    (and p - k <= window), with ALiBi's bias on positions.  q [B,L,H,D]; k_ring, v_ring [B,C,Hk,D] bf16; D in {64,
    128}; C >= max_kv_size + L - 1.  Rows i >= end[b] - start[b] are padding: finite, unspecified.  The values of
    start and end are not checked (0 <= end[b] - start[b] <= L)."""
    what = "attention_ring"
    B, H, D, C, Hk = _check_ring(q, k_ring, v_ring, max_kv_size, what, 4)
    L = q.shape[1]
    if C < max_kv_size + L - 1:
        raise ValueError(f"{what}: the ring's {C} slots are fewer than max_kv_size + L - 1 = "
                         f"{max_kv_size + L - 1}: writing the chunk would overwrite keys its queries see")
    _check_rows(start, B, q.device, what, "start")
    _check_rows(end, B, q.device, what, "end")
    window, alibi, scale = _check_scores(q, scale, window, alibi, what)
    o = torch.empty_like(q)
    lse = torch.empty((B, H, L), device=q.device, dtype=torch.float32) if return_lse else None
    tok = _t0("attn_ring")
    check(lib().b200_attn_fwd_ring(q.data_ptr(), k_ring.data_ptr(), v_ring.data_ptr(), start.data_ptr(),
                                   end.data_ptr(), o.data_ptr(), _ptr(lse), int(max_kv_size),
                                   -1 if window is None else int(window), _ptr(alibi), B, L, C, H, Hk, D,
                                   float(scale), _stream()), "b200_attn_fwd_ring")
    _t1(tok)
    return (o, lse) if return_lse else o


def kv_append_ring(q: torch.Tensor, k: torch.Tensor, v: torch.Tensor, k_ring: torch.Tensor, v_ring: torch.Tensor,
                   end: torch.Tensor, live: Optional[torch.Tensor] = None,
                   rope_tables: Optional[Tuple[torch.Tensor, torch.Tensor]] = None,
                   layout: str = "interleaved") -> None:
    """kv_append into a ring (b200_kv_append_ring): k (rotated at position end[b] - 1 with rope_tables, as is q in
    place) and v go to slot ring_slot(end[b] - 1, C).  live (int32 [B] on the device, optional): rows with live[b]
    == 0 are left alone, q included.  bf16, D in {64, 128}."""
    what = "kv_append_ring"
    _check_choice(layout, ROPE_LAYOUTS, f"{what}: layout")
    B, H, D, C, Hk = _check_ring(q, k_ring, v_ring, RING_SINKS + 1, what, 3)
    _check_rows(end, B, q.device, what, "end")
    if live is not None:
        _check_rows(live, B, q.device, what, "live")
    for t, nm in ((k, "k"), (v, "v")):
        _need(t, torch.bfloat16, f"{what}: {nm}")
        if t.shape != (B, Hk, D):
            raise ValueError(f"{what}: {nm} must be [{B},{Hk},{D}], got {tuple(t.shape)}")
    cos_t, sin_t, half = _check_rope_tables(rope_tables, D, layout, what)
    check(lib().b200_kv_append_ring(q.data_ptr(), k.data_ptr(), v.data_ptr(), k_ring.data_ptr(), v_ring.data_ptr(),
                                    end.data_ptr(), _ptr(live), _ptr(cos_t), _ptr(sin_t), half, B, C, H, Hk, D,
                                    _stream()), "b200_kv_append_ring")


# ------------------------------------------------------------------------------------------------
# beam search over a shared-prompt cache (DESIGN §4.2.4): per layer, the groups' prefix caches [G, s_prefix, Hk, D]
# and the beam tails [S, tail_cap, Hk, D]; `tables` is one int32 device tensor holding, for R rows and G groups,
# [row_group (R) | row_slot (R) | grp_t0 (G) | grp_row0 (G) | grp_rows (G)]
# ------------------------------------------------------------------------------------------------
def attention_decode_beam_workspace_bytes(R: int, H: int, s_prefix: int, tail_cap: int, D: int) -> int:
    return int(lib().b200_attn_decode_beam_workspace_bytes(R, H, s_prefix, tail_cap, D))


def attention_decode_beam_pack(H: int, Hk: int, D: int) -> int:
    """Beam rows of a group that share one read of a prefix chunk."""
    return int(lib().b200_attn_decode_beam_pack(H, Hk, D))


def _check_beam_tables(tables: torch.Tensor, R: int, G: int, device, what: str) -> None:
    if not isinstance(tables, torch.Tensor) or tables.dtype != torch.int32 or tables.device != device \
            or not tables.is_contiguous() or tables.numel() != 2 * R + 3 * G:
        raise ValueError(f"{what}: tables must be a contiguous int32 [2 R + 3 G] = [{2 * R + 3 * G}] tensor on {device}")


def attention_decode_beam(q: torch.Tensor, k_prefix: torch.Tensor, v_prefix: torch.Tensor, k_tail: torch.Tensor,
                          v_tail: torch.Tensor, lens: torch.Tensor, tables: torch.Tensor,
                          scale: Optional[float] = None, workspace: Optional[torch.Tensor] = None,
                          return_lse: bool = False, window: Optional[int] = None,
                          alibi: Optional[torch.Tensor] = None):
    """attention_decode for beam rows over a shared-prompt cache (b200_attn_decode_beam): row b's query at position
    p = lens[b] - 1 sees keys t < T0 from its group's prefix cache and keys T0 <= t <= p from index t - T0 of its tail
    slot (tables above).  q [R,H,D]; k_prefix, v_prefix [G,s_prefix,Hk,D]; k_tail, v_tail [S,tail_cap,Hk,D]; all bf16
    or all fp32, D in {16, 32, 64, 128}, s_prefix and tail_cap multiples of 256.  window and alibi as in
    attention_decode.  The table values are not checked here (that would read the device)."""
    what = "attention_decode_beam"
    _is_bf16(q, "q")
    for t, nm in ((q, "q"), (k_prefix, "k_prefix"), (v_prefix, "v_prefix"), (k_tail, "k_tail"), (v_tail, "v_tail")):
        _need(t, q.dtype, f"{what}: {nm}")
    if q.dim() != 3 or k_prefix.dim() != 4 or k_prefix.shape != v_prefix.shape or k_tail.dim() != 4 \
            or k_tail.shape != v_tail.shape or k_prefix.shape[2:] != k_tail.shape[2:]:
        raise ValueError(f"{what}: expected q [R,H,D], prefix [G,s_prefix,Hk,D] and tails [S,tail_cap,Hk,D], got "
                         f"{tuple(q.shape)}, {tuple(k_prefix.shape)}, {tuple(k_tail.shape)}")
    R, H, D = q.shape
    G, s_prefix, Hk, Dc = k_prefix.shape
    S, tail_cap = k_tail.shape[:2]
    if Dc != D or H % Hk != 0 or D not in (16, 32, 64, 128):
        raise ValueError(f"{what}: q {tuple(q.shape)} does not match the caches {tuple(k_prefix.shape)} "
                         f"(head_dim 16, 32, 64 or 128)")
    _check_rows(lens, R, q.device, what, "lens")
    _check_beam_tables(tables, R, G, q.device, what)
    window, alibi, scale = _check_scores(q, scale, window, alibi, what)
    workspace = _check_workspace(workspace, attention_decode_beam_workspace_bytes(R, H, s_prefix, tail_cap, D),
                                 q.device, what, align=128)
    o = torch.empty_like(q)
    lse = torch.empty((R, H), device=q.device, dtype=torch.float32) if return_lse else None
    tok = _t0("attn_decode_beam")
    check(lib().b200_attn_decode_beam(q.data_ptr(), k_prefix.data_ptr(), v_prefix.data_ptr(), k_tail.data_ptr(),
                                      v_tail.data_ptr(), lens.data_ptr(), tables.data_ptr(), o.data_ptr(), _ptr(lse),
                                      -1 if window is None else int(window), _ptr(alibi), R, G, s_prefix, S, tail_cap,
                                      H, Hk, D, float(scale), _is_bf16(q, "q"), workspace.data_ptr(),
                                      workspace.numel(), _stream()), "b200_attn_decode_beam")
    _t1(tok)
    return (o, lse) if return_lse else o


def kv_append_beam(q: torch.Tensor, k: torch.Tensor, v: torch.Tensor, k_tail: torch.Tensor, v_tail: torch.Tensor,
                   lens: torch.Tensor, tables: torch.Tensor, n_groups: int,
                   rope_tables: Optional[Tuple[torch.Tensor, torch.Tensor]] = None,
                   layout: str = "interleaved") -> None:
    """kv_append into the beam tails (b200_kv_append_beam): k (rotated at position lens[b] - 1 with rope_tables, as
    is q in place) and v go to index lens[b] - 1 - T0 of row b's tail slot."""
    what = "kv_append_beam"
    _check_choice(layout, ROPE_LAYOUTS, f"{what}: layout")
    _is_bf16(q, "q")
    for t, nm in ((q, "q"), (k, "k"), (v, "v"), (k_tail, "k_tail"), (v_tail, "v_tail")):
        _need(t, q.dtype, f"{what}: {nm}")
    R, H, D = q.shape
    if k_tail.dim() != 4 or k_tail.shape != v_tail.shape or k_tail.shape[3] != D or H % k_tail.shape[2]:
        raise ValueError(f"{what}: tails {tuple(k_tail.shape)} do not match q {tuple(q.shape)}")
    tail_cap, Hk = k_tail.shape[1], k_tail.shape[2]
    for t, nm in ((k, "k"), (v, "v")):
        if t.shape != (R, Hk, D):
            raise ValueError(f"{what}: {nm} must be [{R},{Hk},{D}], got {tuple(t.shape)}")
    _check_rows(lens, R, q.device, what, "lens")
    _check_beam_tables(tables, R, n_groups, q.device, what)
    cos_t, sin_t, half = _check_rope_tables(rope_tables, D, layout, what)
    check(lib().b200_kv_append_beam(q.data_ptr(), k.data_ptr(), v.data_ptr(), k_tail.data_ptr(), v_tail.data_ptr(),
                                    lens.data_ptr(), tables.data_ptr(), _ptr(cos_t), _ptr(sin_t), half, R,
                                    tail_cap, H, Hk, D, _is_bf16(q, "q"), _stream()), "b200_kv_append_beam")


def kv_beam_fork(buffers: torch.Tensor, copies: torch.Tensor, max_len: int, tails: Sequence[torch.Tensor]) -> None:
    """Copy-on-fork (b200_kv_beam_fork): copies int32 [n, 3] on the device = (src slot, dst slot, positions) copies
    tail indices [0, positions) from slot src to slot dst in every tail of `tails` (each [S, tail_cap, Hk, D]);
    buffers: int64 device tensor of their data pointers.  max_len >= every copy's positions.  No copies: nothing."""
    n = copies.shape[0] if copies.dim() == 2 else 0
    if n == 0:
        return
    t0 = tails[0]
    if copies.dtype != torch.int32 or copies.shape[1] != 3 or not copies.is_contiguous() or copies.device != t0.device:
        raise ValueError("kv_beam_fork: copies must be a contiguous int32 [n, 3] tensor on the tails' device")
    if buffers.dtype != torch.int64 or buffers.numel() != len(tails) or buffers.device != t0.device:
        raise ValueError("kv_beam_fork: buffers must be an int64 device tensor of the tails' pointers")
    row_bytes = t0.shape[2] * t0.shape[3] * t0.element_size()
    check(lib().b200_kv_beam_fork(buffers.data_ptr(), len(tails), copies.data_ptr(), n, int(max_len), t0.shape[1],
                                  row_bytes, _stream()), "b200_kv_beam_fork")


# ------------------------------------------------------------------------------------------------
# the quantized KV cache (the reference's kv_bits / kv_group_size; DESIGN §4.2.1): per layer, codes uint8
# [B, s_max, Hk, D * bits / 8] and parameters fp32 [B, Hk, s_max, D / group_size, 2] for each of K and V
# ------------------------------------------------------------------------------------------------
KV_BITS = (4, 8)
KV_GROUP_SIZES = (32, 64, 128)


def check_kv_quant(bits, group_size, head_dim: Optional[int] = None, what: str = "kv cache") -> None:
    """Raises ValueError unless bits is 4 or 8, group_size is 32, 64 or 128 and (given head_dim) it divides head_dim,
    which must then be 32, 64 or 128."""
    if isinstance(bits, bool) or bits not in KV_BITS:
        raise ValueError(f"{what}: kv_bits must be 4 or 8, got {bits!r}")
    if isinstance(group_size, bool) or group_size not in KV_GROUP_SIZES:
        raise ValueError(f"{what}: kv_group_size must be 32, 64 or 128, got {group_size!r}")
    if head_dim is not None and (head_dim not in (32, 64, 128) or head_dim % group_size):
        raise ValueError(f"{what}: a quantized KV cache needs head_dim in (32, 64, 128) divisible by kv_group_size "
                         f"{group_size}, got head_dim {head_dim}")


def kv_quant_shapes(B: int, s_max: int, Hk: int, D: int, bits: int, group_size: int):
    """(codes shape, parameters shape) of one K or V buffer of the quantized cache."""
    return (B, s_max, Hk, D * bits // 8), (B, Hk, s_max, D // group_size, 2)


def _check_quant_cache(k_codes, v_codes, k_params, v_params, B: int, Hk: int, D: int, bits: int, group_size: int,
                       device, what: str) -> int:
    """The four buffers of one layer's quantized cache; returns s_max."""
    check_kv_quant(bits, group_size, D, what)
    if k_codes.dim() != 4:
        raise ValueError(f"{what}: k_codes must be [B, s_max, Hk, D * bits / 8], got {tuple(k_codes.shape)}")
    s_max = k_codes.shape[1]
    cshape, pshape = kv_quant_shapes(B, s_max, Hk, D, bits, group_size)
    bufs = ((k_codes, "k_codes", torch.uint8, cshape), (v_codes, "v_codes", torch.uint8, cshape),
            (k_params, "k_params", torch.float32, pshape), (v_params, "v_params", torch.float32, pshape))
    for t, nm, dt, shp in bufs:
        if t.dtype != dt or tuple(t.shape) != shp:
            raise ValueError(f"{what}: {nm} must be {dt} {list(shp)}, got {t.dtype} {list(t.shape)}")
    for t, nm, dt, _ in bufs:
        _need(t, dt, f"{what}: {nm}")
        if t.device != device or t.data_ptr() % 16:
            raise ValueError(f"{what}: {nm} must be 16-byte aligned on {device}")
    if s_max % 2:
        raise ValueError(f"{what}: s_max {s_max} must be even")
    return s_max


def kv_quantize(k: torch.Tensor, v: torch.Tensor, k_codes: torch.Tensor, v_codes: torch.Tensor,
                k_params: torch.Tensor, v_params: torch.Tensor, bits: int, group_size: int,
                n: Optional[int] = None) -> None:
    """Quantizes positions [0, n) (default: all S) of k, v [B, S, Hk, D] (bf16 or fp32) into the cache buffers
    (b200_kv_quantize).  Positions at or past n are not written."""
    _is_bf16(k, "kv_quantize: k")
    if k.dim() != 4 or v.shape != k.shape or v.dtype != k.dtype:
        raise ValueError(f"kv_quantize: k and v must both be [B, S, Hk, D] of one dtype, got {k.dtype} "
                         f"{tuple(k.shape)}, {v.dtype} {tuple(v.shape)}")
    B, S, Hk, D = k.shape
    s_max = _check_quant_cache(k_codes, v_codes, k_params, v_params, B, Hk, D, bits, group_size, k.device,
                               "kv_quantize")
    _need(k, k.dtype, "kv_quantize: k")
    _need(v, k.dtype, "kv_quantize: v")
    n = S if n is None else n
    if isinstance(n, bool) or not isinstance(n, int) or not 0 <= n <= min(S, s_max):
        raise ValueError(f"kv_quantize: n must be an int in [0, min(S={S}, s_max={s_max})], got {n!r}")
    if k.data_ptr() % 16 or v.data_ptr() % 16:
        raise ValueError("kv_quantize: k and v must be 16-byte aligned")
    check(lib().b200_kv_quantize(k.data_ptr(), v.data_ptr(), n, S, k_codes.data_ptr(), v_codes.data_ptr(),
                                 k_params.data_ptr(), v_params.data_ptr(), B, s_max, Hk, D, bits, group_size,
                                 _is_bf16(k, "k"), _stream()), "b200_kv_quantize")


def kv_dequantize(k_codes: torch.Tensor, v_codes: torch.Tensor, k_params: torch.Tensor, v_params: torch.Tensor,
                  end: torch.Tensor, bits: int, group_size: int, out: Optional[Tuple[torch.Tensor, torch.Tensor]] = None,
                  S: Optional[int] = None) -> Tuple[torch.Tensor, torch.Tensor]:
    """Positions [0, end[b]) of row b of a quantized cache as bf16 k, v [B, S, Hk, D] (b200_kv_dequantize): s q + b in
    fp32, rounded once to bf16.  out: bf16 [B, S, Hk, D] buffers to write (else allocated with S positions, default
    s_max).  Positions at or past end[b] are not written."""
    what = "kv_dequantize"
    if k_codes.dim() != 4:
        raise ValueError(f"{what}: k_codes must be [B, s_max, Hk, D * bits / 8], got {tuple(k_codes.shape)}")
    B, _, Hk, Dc = k_codes.shape
    check_kv_quant(bits, group_size, what=what)
    D = Dc * 8 // bits
    s_max = _check_quant_cache(k_codes, v_codes, k_params, v_params, B, Hk, D, bits, group_size, k_codes.device, what)
    _check_rows(end, B, k_codes.device, what, "end")
    if out is None:
        S = s_max if S is None else S
        if isinstance(S, bool) or not isinstance(S, int) or not 1 <= S <= s_max:
            raise ValueError(f"{what}: S must be an int in [1, {s_max}], got {S!r}")
        shape = (B, S, Hk, D)
        out = (torch.empty(shape, device=k_codes.device, dtype=torch.bfloat16),
               torch.empty(shape, device=k_codes.device, dtype=torch.bfloat16))
    k, v = out
    for t, nm in ((k, "k"), (v, "v")):
        _need(t, torch.bfloat16, f"{what}: {nm}")
        if t.dim() != 4 or t.shape[0] != B or t.shape[2:] != (Hk, D) or not 1 <= t.shape[1] <= s_max \
                or t.shape != k.shape or t.data_ptr() % 16:
            raise ValueError(f"{what}: {nm} must be a 16-byte aligned bf16 [{B}, S <= {s_max}, {Hk}, {D}] tensor, "
                             f"got {tuple(t.shape)}")
    check(lib().b200_kv_dequantize(k_codes.data_ptr(), v_codes.data_ptr(), k_params.data_ptr(), v_params.data_ptr(),
                                   end.data_ptr(), k.data_ptr(), v.data_ptr(), k.shape[1], B, s_max, Hk, D, bits,
                                   group_size, _stream()), "b200_kv_dequantize")
    return k, v


def kv_append_quant(q: torch.Tensor, k: torch.Tensor, v: torch.Tensor, k_codes: torch.Tensor, v_codes: torch.Tensor,
                    k_params: torch.Tensor, v_params: torch.Tensor, lens: torch.Tensor, bits: int, group_size: int,
                    rope_tables: Optional[Tuple[torch.Tensor, torch.Tensor]] = None,
                    layout: str = "interleaved") -> None:
    """kv_append into the quantized cache (b200_kv_append_quant): q [B,H,D] is rotated in place exactly as
    kv_append rotates it, and the rotated k [B,Hk,D] and v, rounded to q's dtype, are quantized into position
    lens[b] - 1."""
    _check_choice(layout, ROPE_LAYOUTS, "kv_append_quant: layout")
    _is_bf16(q, "kv_append_quant: q")
    for t, nm in ((q, "q"), (k, "k"), (v, "v")):
        if t.dim() != 3 or t.dtype != q.dtype:
            raise ValueError(f"kv_append_quant: {nm} must be a [B, heads, D] {q.dtype} tensor, got {t.dtype} "
                             f"{tuple(t.shape)}")
    B, H, D = q.shape
    if k.shape != v.shape or k.shape[0] != B or k.shape[2] != D or H % k.shape[1]:
        raise ValueError(f"kv_append_quant: k, v must be [{B}, Hk, {D}] with H % Hk == 0, got {tuple(k.shape)}, "
                         f"{tuple(v.shape)}")
    Hk = k.shape[1]
    s_max = _check_quant_cache(k_codes, v_codes, k_params, v_params, B, Hk, D, bits, group_size, q.device,
                               "kv_append_quant")
    for t, nm in ((q, "q"), (k, "k"), (v, "v")):
        _need(t, q.dtype, f"kv_append_quant: {nm}")
        if t.data_ptr() % 16:
            raise ValueError(f"kv_append_quant: {nm} must be 16-byte aligned")
    _check_rows(lens, B, q.device, "kv_append_quant", "lens")
    cos_t, sin_t, half = _check_rope_tables(rope_tables, D, layout, "kv_append_quant")
    check(lib().b200_kv_append_quant(q.data_ptr(), k.data_ptr(), v.data_ptr(), k_codes.data_ptr(), v_codes.data_ptr(),
                                     k_params.data_ptr(), v_params.data_ptr(), lens.data_ptr(), _ptr(cos_t),
                                     _ptr(sin_t), half, B, s_max, H, Hk, D, bits, group_size, _is_bf16(q, "q"),
                                     _stream()), "b200_kv_append_quant")


def attention_decode_quant(q: torch.Tensor, k_codes: torch.Tensor, v_codes: torch.Tensor, k_params: torch.Tensor,
                           v_params: torch.Tensor, lens: torch.Tensor, bits: int, group_size: int,
                           scale: Optional[float] = None, workspace: Optional[torch.Tensor] = None,
                           return_lse: bool = False, window: Optional[int] = None,
                           alibi: Optional[torch.Tensor] = None):
    """attention_decode over the quantized cache (b200_attn_decode_quant): the same result over the dequantised keys
    and values s q + b, with the same lens, window, alibi, workspace and return_lse semantics.  q [B,H,D] bf16 or
    fp32, D in {32, 64, 128}."""
    _is_bf16(q, "attention_decode_quant: q")
    if q.dim() != 3 or k_codes.dim() != 4:
        raise ValueError(f"attention_decode_quant: expected q [B,H,D] and k_codes [B,s_max,Hk,Dc], got "
                         f"{tuple(q.shape)}, {tuple(k_codes.shape)}")
    B, H, D = q.shape
    Hk = k_codes.shape[2]
    check_kv_quant(bits, group_size, D, "attention_decode_quant")
    if H % Hk:
        raise ValueError(f"attention_decode_quant: H={H} must be a multiple of Hk={Hk}")
    s_max = _check_quant_cache(k_codes, v_codes, k_params, v_params, B, Hk, D, bits, group_size, q.device,
                               "attention_decode_quant")
    _need(q, q.dtype, "attention_decode_quant: q")
    _check_rows(lens, B, q.device, "attention_decode_quant", "lens")
    window, alibi, scale = _check_scores(q, scale, window, alibi, "attention_decode_quant")
    workspace = _check_workspace(workspace, attention_decode_workspace_bytes(B, H, s_max, D), q.device,
                                 "attention_decode_quant")
    o = torch.empty_like(q)
    lse = torch.empty((B, H), device=q.device, dtype=torch.float32) if return_lse else None
    tok = _t0("attn_decode")
    check(lib().b200_attn_decode_quant(q.data_ptr(), k_codes.data_ptr(), v_codes.data_ptr(), k_params.data_ptr(),
                                       v_params.data_ptr(), lens.data_ptr(), o.data_ptr(), _ptr(lse),
                                       -1 if window is None else min(int(window), s_max), _ptr(alibi), B, s_max, H,
                                       Hk, D, bits, group_size, float(scale), _is_bf16(q, "q"), workspace.data_ptr(),
                                       workspace.numel(), _stream()), "b200_attn_decode_quant")
    _t1(tok)
    return (o, lse) if return_lse else o


# ------------------------------------------------------------------------------------------------
# raw strided GEMM + Shampoo elementwise helpers
# ------------------------------------------------------------------------------------------------
def gemm_raw(a_mn: bool, b_mn: bool, M: int, N: int, K: int, batch: int,
             A: torch.Tensor, lda: int, strideA: int, B: torch.Tensor, ldb: int, strideB: int,
             C: Optional[torch.Tensor], ldc: int, strideC: int, D: torch.Tensor, ldd: int, strideD: int,
             alpha: float = 1.0, beta: float = 0.0, alpha_vec: Optional[torch.Tensor] = None,
             beta_vec: Optional[torch.Tensor] = None, force_bn: int = 0) -> None:
    """Strided/batched GEMM on views (sub-blocks of larger matrices): explicit leading dims."""
    if A.dtype != torch.bfloat16 or B.dtype != torch.bfloat16:
        raise ValueError("gemm_raw: A and B must be bf16")
    out_f32 = _is_bf16(D, "D") == 0
    if C is not None and C.dtype != D.dtype:
        raise ValueError("gemm_raw: C and D dtypes differ")
    check(lib().b200_gemm_bf16(int(a_mn), int(b_mn), M, N, K, batch, A.data_ptr(), lda, strideA,
                               B.data_ptr(), ldb, strideB, _ptr(C), ldc, strideC, D.data_ptr(), ldd,
                               strideD, int(out_f32), float(alpha), float(beta), _ptr(alpha_vec),
                               _ptr(beta_vec), int(force_bn), _stream()), "b200_gemm_bf16")


def ema_split(g, m, out32, hi, lo, beta: float, gscale: float, inv_bc: float, out_scale: float = 1.0) -> None:
    check(lib().b200_ema_split(g.data_ptr(), _is_bf16(g, "g"), m.data_ptr(), out32.data_ptr(),
                               hi.data_ptr(), _ptr(lo), g.numel(), float(beta), float(gscale),
                               float(inv_bc), float(out_scale), _stream()), "b200_ema_split")


def graft_update(p32, p16, pre, d, numel: int, batch: int, coef, coef_d, decay: float) -> None:
    check(lib().b200_graft_update(p32.data_ptr(), _ptr(p16), pre.data_ptr(), d.data_ptr(), numel, batch,
                                  coef.data_ptr(), coef_d.data_ptr(), float(decay), _stream()),
          "b200_graft_update")


def sumsq_raw(x: torch.Tensor, out: torch.Tensor, numel: int, batch: int, zero_first: bool = True) -> None:
    ws = reduce_workspace(x.device, batch)
    check(lib().b200_sumsq(x.data_ptr(), _is_bf16(x, "x"), out.data_ptr(), numel, batch, int(zero_first),
                           ws.data_ptr(), ws.numel(), _stream()), "b200_sumsq")


# ------------------------------------------------------------------------------------------------
# Shampoo's Kronecker-factor path through the C ABI (b200_shampoo_*); factor matrices are [batch, kp, kp]
# with kp = round_up(k, 8)
# ------------------------------------------------------------------------------------------------
def rup8(k: int) -> int:
    return (int(k) + 7) // 8 * 8


def shampoo_stats(g_hi: torch.Tensor, g_lo: Optional[torch.Tensor], ldg: int, stride_g: int, L: torch.Tensor,
                  R: torch.Tensor, batch: int, k1: int, k2: int, beta2: float, weight: float) -> None:
    _need(L, torch.float32, "L")
    _need(R, torch.float32, "R")
    check(lib().b200_shampoo_stats(g_hi.data_ptr(), _ptr(g_lo), int(ldg), int(stride_g), L.data_ptr(), R.data_ptr(),
                                   int(batch), int(k1), int(k2), float(beta2), float(weight), _stream()),
          "b200_shampoo_stats")


def shampoo_root(M: torch.Tensor, P: torch.Tensor, P_hi: Optional[torch.Tensor], P_lo: Optional[torch.Tensor],
                 k: int, p: float, eps: float, iters: int = 6, workspace: Optional[torch.Tensor] = None) -> torch.Tensor:
    """matrix_inverse_pth_root (optimizers/shampoo.py:88-126) of M [batch, kp, kp] fp32 -> P (same layout)."""
    _need(M, torch.float32, "M")
    _need(P, torch.float32, "P")
    batch = M.shape[0]
    need = int(lib().b200_shampoo_root_workspace_bytes(batch, int(k)))
    if workspace is None or workspace.numel() < need:
        workspace = torch.empty(need, device=M.device, dtype=torch.uint8)
    check(lib().b200_shampoo_root(M.data_ptr(), P.data_ptr(), _ptr(P_hi), _ptr(P_lo), batch, int(k), float(p),
                                  float(eps), int(iters), workspace.data_ptr(), workspace.numel(), _stream()),
          "b200_shampoo_root")
    return P


def shampoo_root_newton(M: torch.Tensor, P: torch.Tensor, P_hi: Optional[torch.Tensor], P_lo: Optional[torch.Tensor],
                        k: int, eps: float, max_iters: int = 40, tol: float = 1e-5,
                        workspace: Optional[torch.Tensor] = None) -> Tuple[torch.Tensor, torch.Tensor]:
    """True inverse 4th root P = (M + ridge I)^(-1/4), ridge = eps * max(lambda_max(M), 1e-6), of M [batch, kp, kp]
    fp32 by the coupled Newton iteration.  Returns the per-matrix accepted iteration counts (int32) and final
    residuals max|Mc - I| (fp32), both [batch] on the device."""
    _need(M, torch.float32, "M")
    _need(P, torch.float32, "P")
    batch = M.shape[0]
    need = int(lib().b200_shampoo_root_newton_workspace_bytes(batch, int(k)))
    if workspace is None or workspace.numel() < need:
        workspace = torch.empty(need, device=M.device, dtype=torch.uint8)
    iters = torch.empty(batch, device=M.device, dtype=torch.int32)
    residual = torch.empty(batch, device=M.device, dtype=torch.float32)
    check(lib().b200_shampoo_root_newton(M.data_ptr(), P.data_ptr(), _ptr(P_hi), _ptr(P_lo), batch, int(k),
                                         float(eps), int(max_iters), float(tol), iters.data_ptr(), residual.data_ptr(),
                                         workspace.data_ptr(), workspace.numel(), _stream()),
          "b200_shampoo_root_newton")
    return iters, residual


def shampoo_precond(PLh, PLl, PRh, PRl, m_hi, m_lo, ldm: int, stride_m: int, out: torch.Tensor, ldo: int,
                    stride_o: int, batch: int, k1: int, k2: int, alpha: float,
                    workspace: Optional[torch.Tensor] = None) -> None:
    need = int(lib().b200_shampoo_precond_workspace_bytes(int(batch), int(k1), int(k2)))
    if workspace is None or workspace.numel() < need:
        workspace = torch.empty(need, device=out.device, dtype=torch.uint8)
    check(lib().b200_shampoo_precond(PLh.data_ptr(), _ptr(PLl), PRh.data_ptr(), _ptr(PRl), m_hi.data_ptr(),
                                     _ptr(m_lo), int(ldm), int(stride_m), out.data_ptr(), int(ldo), int(stride_o),
                                     int(batch), int(k1), int(k2), float(alpha), workspace.data_ptr(),
                                     workspace.numel(), _stream()), "b200_shampoo_precond")


def shampoo_graft(p32: torch.Tensor, p16: Optional[torch.Tensor], upd: torch.Tensor, graft: torch.Tensor,
                  numel: int, batch: int, decay: float, workspace: Optional[torch.Tensor] = None) -> None:
    need = int(lib().b200_shampoo_graft_workspace_bytes(int(batch)))
    if workspace is None or workspace.numel() < need:
        workspace = torch.empty(need, device=p32.device, dtype=torch.uint8)
    check(lib().b200_shampoo_graft(p32.data_ptr(), _ptr(p16), upd.data_ptr(), graft.data_ptr(), int(numel),
                                   int(batch), float(decay), workspace.data_ptr(), workspace.numel(), _stream()),
          "b200_shampoo_graft")


# ------------------------------------------------------------------------------------------------
# block-adjacent fused elementwise steps (SURVEY 8f row f1)
# ------------------------------------------------------------------------------------------------
class _GluFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, gate, up, act):
        g, u = gate.contiguous(), up.contiguous()
        y = torch.empty_like(g)
        fwd = "b200_silu_glu_fwd" if act == "silu" else "b200_glu_fwd"
        check(getattr(lib(), fwd)(g.data_ptr(), u.data_ptr(), y.data_ptr(), g.numel(), _stream()), fwd)
        ctx.save_for_backward(g, u)
        ctx.act = act
        return y

    @staticmethod
    def backward(ctx, dy):
        g, u = ctx.saved_tensors
        dy = dy.contiguous()
        dg, du = torch.empty_like(g), torch.empty_like(u)
        bwd = "b200_silu_glu_bwd" if ctx.act == "silu" else "b200_glu_bwd"
        check(getattr(lib(), bwd)(dy.data_ptr(), g.data_ptr(), u.data_ptr(), dg.data_ptr(), du.data_ptr(),
                                  g.numel(), _stream()), bwd)
        return dg, du, None


_EMB_WS = {}


class _EmbeddingFn(torch.autograd.Function):
    """h = E[tokens] (arch/llama.py:389).  Backward scatters dh into the weight's flat-buffer gradient with fp32
    accumulation per vocabulary row (b200_embedding_bwd) instead of torch's sort + segmented-sum path
    (3 kernels, 0.44 ms per C2 step); autograd sees None for the weight."""

    @staticmethod
    def forward(ctx, tokens, weight):
        ctx.save_for_backward(tokens)
        ctx.weight = weight
        return torch.nn.functional.embedding(tokens, weight)

    @staticmethod
    def backward(ctx, dh):
        (tokens,) = ctx.saved_tensors
        w = ctx.weight
        V, H = w.shape
        dh2 = dh.reshape(-1, H).contiguous()
        tok = tokens.reshape(-1).contiguous()
        need = int(lib().b200_embedding_bwd_workspace_bytes(V, H))
        key = (str(dh.device), _stream())
        ws = _EMB_WS.get(key)
        if ws is None or ws.numel() < need:
            ws = torch.empty(need, device=dh.device, dtype=torch.uint8)
            _EMB_WS[key] = ws
        check(lib().b200_embedding_bwd(dh2.data_ptr(), tok.data_ptr(), w.grad.data_ptr(), _is_bf16(w.grad, "grad"),
                                       dh2.shape[0], V, H, ws.data_ptr(), ws.numel(), _stream()), "b200_embedding_bwd")
        return None, None


def embedding(tokens: torch.Tensor, weight: torch.Tensor) -> torch.Tensor:
    """Embedding lookup whose backward accumulates straight into a flat-buffer gradient (bf16 activations, int64
    tokens, hidden % 8 == 0); other cases use torch's embedding."""
    g = weight.grad
    if (getattr(weight, "_b200_flat_grad", False) and g is not None and weight.is_cuda and weight.dtype == torch.bfloat16
            and tokens.dtype == torch.int64 and weight.shape[1] % 8 == 0 and g.is_contiguous()):
        return _EmbeddingFn.apply(tokens, weight)
    return torch.nn.functional.embedding(tokens, weight)


def _adjacent_rows(w_a: torch.Tensor, w_b: torch.Tensor) -> bool:
    return (w_a.shape == w_b.shape and w_a.is_contiguous() and w_b.is_contiguous() and
            w_b.data_ptr() == w_a.data_ptr() + w_a.numel() * w_a.element_size())


class _MlpFn(torch.autograd.Function):
    """down( gate(x) * sigmoid(up(x)) * 2 )  (arch/llama.py:142-151) with the activation inside the GEMM epilogues:

      forward   [g | u], y = b200_mlp_gateup_glu_fwd(x, [Wg ; Wu])      one wgmma kernel (in-tree engine)
                out        = y Wd^T                                      library GEMM
      backward  dWd       += dout^T y                                    library GEMM into the flat gradient
                [dg | du]  = b200_mlp_down_glu_bwd(dout, Wd, [g | u])    one wgmma kernel: dout Wd never leaves the chip
                dx         = [dg | du] [Wg ; Wu]                         ONE library GEMM (K = 2I) instead of two
                d[Wg ; Wu] += [dg | du]^T x                              ONE library GEMM into the flat gradient

    Needs gate_proj.weight and up_proj.weight adjacent in memory (flat.ParamStore) with flat-buffer gradients,
    bf16, intermediate size % 128 == 0; `mlp()` falls back to the unfused path otherwise.  act "silu" runs mlx_lm's
    down(silu(gate(x)) * up(x)) through b200_mlp_gateup_silu_fwd / b200_mlp_down_silu_bwd instead."""

    @staticmethod
    def forward(ctx, x, wg, wu, wd, act):
        I, K = wg.shape
        x2 = x.reshape(-1, K).contiguous()
        M = x2.shape[0]
        gu = torch.empty((M, 2 * I), device=x.device, dtype=torch.bfloat16)
        y = torch.empty((M, I), device=x.device, dtype=torch.bfloat16)
        fwd = "b200_mlp_gateup_silu_fwd" if act == "silu" else "b200_mlp_gateup_glu_fwd"
        tok = _t0("mlp_glu_fwd")
        check(getattr(lib(), fwd)(x2.data_ptr(), wg.data_ptr(), gu.data_ptr(), y.data_ptr(), M, K, I, _stream()), fwd)
        _t1(tok)
        out = y @ wd.t()
        ctx.save_for_backward(x2, gu, y, wg, wu, wd)
        ctx.x_shape = x.shape
        ctx.act = act
        return out.view(*x.shape[:-1], wd.shape[0])

    @staticmethod
    def backward(ctx, dout):
        x2, gu, y, wg, wu, wd = ctx.saved_tensors
        I, K = wg.shape
        H = wd.shape[0]
        M = x2.shape[0]
        d2 = dout.reshape(-1, H).contiguous()
        wd.grad.addmm_(d2.t(), y)                                   # dWd
        dgu = torch.empty((M, 2 * I), device=d2.device, dtype=torch.bfloat16)
        bwd = "b200_mlp_down_silu_bwd" if ctx.act == "silu" else "b200_mlp_down_glu_bwd"
        tok = _t0("mlp_glu_bwd")
        check(getattr(lib(), bwd)(d2.data_ptr(), wd.data_ptr(), gu.data_ptr(), dgu.data_ptr(), M, H, I, _stream()), bwd)
        _t1(tok)
        w2 = torch.as_strided(wg, (2 * I, K), (K, 1))               # [Wg ; Wu], adjacent in the flat store
        g2 = torch.as_strided(wg.grad, (2 * I, K), (K, 1))
        dx = dgu @ w2 if ctx.needs_input_grad[0] else None
        g2.addmm_(dgu.t(), x2)
        return (dx.view(ctx.x_shape) if dx is not None else None), None, None, None, None


def mlp_fusable(x: torch.Tensor, wg: torch.Tensor, wu: torch.Tensor, wd: torch.Tensor) -> bool:
    if not (x.is_cuda and x.dtype == torch.bfloat16 and wg.dtype == torch.bfloat16 and wd.dtype == torch.bfloat16):
        return False
    if wg.shape[0] % 128 != 0 or wg.shape[1] % 8 != 0 or wd.shape != (wg.shape[1], wg.shape[0]) or not wd.is_contiguous():
        return False
    flat = all(getattr(w, "_b200_flat_grad", False) and w.grad is not None and w.grad.dtype == torch.bfloat16
               for w in (wg, wu, wd))
    return flat and _adjacent_rows(wg, wu) and _adjacent_rows(wg.grad, wu.grad)


def mlp(x: torch.Tensor, wg: torch.Tensor, wu: torch.Tensor, wd: torch.Tensor, act: str = "sigmoid2") -> torch.Tensor:
    """The reference MLP (arch/llama.py:149-151) on three bias-free projections; act "silu" gives mlx_lm's
    down(silu(gate(x)) * up(x))."""
    _check_choice(act, GLU_ACTS, "mlp: act")
    if mlp_fusable(x, wg, wu, wd) and _MLP_FUSED:
        return _MlpFn.apply(x, wg, wu, wd, act)
    g, u = multi_linear(x, (wg, wu))
    return linear(glu(g, u, act), wd)


# B200_MLP_FUSED=0 restores the library GEMMs + elementwise GLU kernels (A/B switch for measurements; the first
# version of the fused epilogues, with row-per-lane 16-byte stores, LOST to that pair -- see DESIGN.md sections 4.7 and 9)
_MLP_FUSED = os.environ.get("B200_MLP_FUSED", "1") != "0"


def glu(gate: torch.Tensor, up: torch.Tensor, act: str = "sigmoid2") -> torch.Tensor:
    """gate * sigmoid(up) * 2 (arch/llama.py:151), or silu(gate) * up with act "silu" (mlx_lm's Llama MLP).  bf16
    tensors with numel % 8 == 0 take the fused kernel; other dtypes (fp32 configs) use the same formula through
    torch ops."""
    _check_choice(act, GLU_ACTS, "glu: act")
    if gate.dtype == torch.bfloat16 and gate.is_cuda and gate.numel() % 8 == 0:
        return _GluFn.apply(gate, up, act)
    if act == "silu":
        return torch.nn.functional.silu(gate) * up
    return gate * torch.sigmoid(up) * 2


MOE_MODES = {"gateup": 0, "down": 1, "down_bwd": 2, "gateup_dgrad": 3}
_MOE_ACT = {"sigmoid2": 0, "silu": 1}


class MoeRouting:
    """Device-side result of b200_moe_route for T tokens: ids / weights [T, k], probs [T, E], counts [E],
    seg_off [E + 1], tile_expert [max_tiles], n_tiles [1], dest [T, k], and with aux the load-balancing partials
    aux_counts / aux_psum [E] over the unmasked tokens.  rows = max_tiles * 128 bounds the permuted buffer."""

    def __init__(self, logits: torch.Tensor, k: int, mask: Optional[torch.Tensor], aux: bool):
        _need(logits, torch.float32, "logits")
        T, E = logits.shape
        dev = logits.device
        L = lib()
        self.T, self.E, self.k = T, E, k
        self.max_tiles = int(L.b200_moe_max_tiles(T, E, k))
        self.rows = self.max_tiles * 128
        i32 = dict(device=dev, dtype=torch.int32)
        self.ids = torch.empty((T, k), **i32)
        self.dest = torch.empty((T, k), **i32)
        self.weights = torch.empty((T, k), device=dev, dtype=torch.float32)
        self.probs = torch.empty((T, E), device=dev, dtype=torch.float32)
        self.counts = torch.empty(E, **i32)
        self.seg_off = torch.empty(E + 1, **i32)
        self.tile_expert = torch.empty(max(self.max_tiles, 1), **i32)
        self.n_tiles = torch.empty(1, **i32)
        self.mask = mask
        self.aux_counts = torch.empty(E, device=dev, dtype=torch.float32) if aux else None
        self.aux_psum = torch.empty(E, device=dev, dtype=torch.float32) if aux else None
        ws = torch.empty(int(L.b200_moe_route_workspace_bytes(T, E, k)), device=dev, dtype=torch.uint8)
        tok = _t0("moe_route")
        check(L.b200_moe_route(logits.data_ptr(), _ptr(mask), T, E, k, self.ids.data_ptr(), self.weights.data_ptr(),
                               self.probs.data_ptr(), self.counts.data_ptr(), self.seg_off.data_ptr(),
                               self.tile_expert.data_ptr(), self.n_tiles.data_ptr(), self.dest.data_ptr(),
                               _ptr(self.aux_counts), _ptr(self.aux_psum), ws.data_ptr(), ws.numel(), _stream()),
              "b200_moe_route")
        _t1(tok)


def moe_route(logits: torch.Tensor, k: int, mask: Optional[torch.Tensor] = None, aux: bool = False) -> MoeRouting:
    return MoeRouting(logits, k, mask, aux)


def moe_permute(x2: torch.Tensor, r: MoeRouting) -> torch.Tensor:
    """[r.rows, H] bf16: token rows at their destinations, pad rows of every segment zero (rows past the last
    segment are not written and never read)."""
    T, H = x2.shape
    xp = torch.empty((r.rows, H), device=x2.device, dtype=torch.bfloat16)
    tok = _t0("moe_permute")
    check(lib().b200_moe_permute(x2.data_ptr(), r.dest.data_ptr(), r.counts.data_ptr(), r.seg_off.data_ptr(), T, H,
                                 r.k, r.E, xp.data_ptr(), _stream()), "b200_moe_permute")
    _t1(tok)
    return xp


def moe_gemm(mode: str, act: str, a: torch.Tensor, w0: torch.Tensor, w1: Optional[torch.Tensor], r: MoeRouting,
             gu: Optional[torch.Tensor] = None) -> Tuple[torch.Tensor, Optional[torch.Tensor]]:
    """One expert-segmented GEMM (include/b200_hotpath.h b200_moe_gemm).  Returns (C, Y); Y only for "gateup"."""
    m = MOE_MODES[mode]
    if mode in ("gateup", "gateup_dgrad"):
        E, I, H = w0.shape
    else:
        E, H, I = w0.shape
    rows = r.rows
    ncol = {"gateup": 2 * I, "down": H, "down_bwd": 2 * I, "gateup_dgrad": H}[mode]
    c = torch.empty((rows, ncol), device=a.device, dtype=torch.bfloat16)
    y = torch.empty((rows, I), device=a.device, dtype=torch.bfloat16) if mode == "gateup" else None
    tok = _t0(f"moe_{mode}")
    check(lib().b200_moe_gemm(m, _MOE_ACT[act], a.data_ptr(), w0.data_ptr(), _ptr(w1), _ptr(gu), c.data_ptr(),
                              _ptr(y), r.tile_expert.data_ptr(), r.n_tiles.data_ptr(), r.max_tiles, H, I, E,
                              _stream()),
          "b200_moe_gemm")
    _t1(tok)
    return c, y


def moe_wgrad(p: torch.Tensor, ldp: int, q: torch.Tensor, ldq: int, g: torch.Tensor, r: MoeRouting) -> None:
    """g[e] ([E, R, C] bf16, contiguous) += p[rows_e]^T q[rows_e] for every expert (the pad rows of p or q are zero)."""
    E, R, Cc = g.shape
    tok = _t0("moe_wgrad")
    check(lib().b200_moe_wgrad(p.data_ptr(), ldp, q.data_ptr(), ldq, g.data_ptr(), R, Cc, E, r.rows,
                               r.counts.data_ptr(), r.seg_off.data_ptr(), _stream()), "b200_moe_wgrad")
    _t1(tok)


def moe_combine(yp: torch.Tensor, r: MoeRouting) -> torch.Tensor:
    H = yp.shape[1]
    out = torch.empty((r.T, H), device=yp.device, dtype=torch.bfloat16)
    tok = _t0("moe_combine")
    check(lib().b200_moe_combine_fwd(yp.data_ptr(), r.dest.data_ptr(), r.weights.data_ptr(), r.T, H, r.k,
                                     out.data_ptr(), _stream()), "b200_moe_combine_fwd")
    _t1(tok)
    return out


def moe_combine_bwd(dout: torch.Tensor, yp: torch.Tensor, r: MoeRouting, aux_grad: Optional[torch.Tensor]):
    """(dyp [rows, H] bf16 (pad rows zero), dw [T, k] fp32, dlogits [T, E] fp32)."""
    T, H = dout.shape
    dyp = torch.empty_like(yp)
    dw = torch.empty((T, r.k), device=dout.device, dtype=torch.float32)
    dlogits = torch.empty((T, r.E), device=dout.device, dtype=torch.float32)
    tok = _t0("moe_combine_bwd")
    check(lib().b200_moe_combine_bwd(dout.data_ptr(), yp.data_ptr(), r.dest.data_ptr(), r.ids.data_ptr(),
                                     r.weights.data_ptr(), r.probs.data_ptr(), _ptr(aux_grad), _ptr(r.mask),
                                     r.counts.data_ptr(), r.seg_off.data_ptr(), T, H, r.E, r.k, dyp.data_ptr(),
                                     dw.data_ptr(), dlogits.data_ptr(), _stream()),
          "b200_moe_combine_bwd")
    _t1(tok)
    return dyp, dw, dlogits


def moe_unpermute(dxp: torch.Tensor, r: MoeRouting, addend: Optional[torch.Tensor] = None) -> torch.Tensor:
    H = dxp.shape[1]
    dx = torch.empty((r.T, H), device=dxp.device, dtype=torch.bfloat16)
    tok = _t0("moe_unpermute")
    check(lib().b200_moe_unpermute(dxp.data_ptr(), r.dest.data_ptr(), _ptr(addend), r.T, H, r.k, dx.data_ptr(),
                                   _stream()), "b200_moe_unpermute")
    _t1(tok)
    return dx


def _grad_sink(w: torch.Tensor) -> Tuple[torch.Tensor, bool]:
    """(buffer the expert wgrad accumulates into, whether it is the flat-store .grad itself)."""
    if getattr(w, "_b200_flat_grad", False) and w.grad is not None and w.grad.dtype == torch.bfloat16:
        return w.grad, True
    return torch.zeros_like(w, dtype=torch.bfloat16), False


class _MoeFn(torch.autograd.Function):
    """Mixtral's sparse MoE block on the expert-segmented kernels:

      forward   logits   = x Wr^T                      fp32 library GEMM (bf16 operands, fp32 accumulation and output)
                routing  = b200_moe_route(logits)      softmax, top-k, renormalised weights, stable counting sort
                xp       = b200_moe_permute(x)         rows grouped by expert, segments padded to 128 rows
                gu, y    = b200_moe_gemm(gateup)       x Wg_e^T | x Wu_e^T and the activation, per 128-row tile
                yo       = b200_moe_gemm(down)         y Wd_e^T
                out      = b200_moe_combine_fwd        sum_j w_j yo[dest[t, j]]
      backward  b200_moe_combine_bwd (dyo, router adjoint), b200_moe_wgrad into the experts' flat gradients,
                b200_moe_gemm(down_bwd), b200_moe_gemm(gateup_dgrad), b200_moe_unpermute (+ the router's dgrad).

    Returns (out, aux_counts, aux_psum); the last two are the load-balancing partials over the unmasked tokens (zeros
    when aux is off), and aux_psum carries a gradient."""

    @staticmethod
    def forward(ctx, x, wr, wg, wu, wd, k, act, mask, aux):
        H = x.shape[-1]
        x2 = x.reshape(-1, H).contiguous()
        logits = torch.matmul(x2.float(), wr.float().t())
        r = MoeRouting(logits, k, mask, aux)
        xp = moe_permute(x2, r)
        gu, y = moe_gemm("gateup", act, xp, wg, wu, r)
        yo, _ = moe_gemm("down", act, y, wd, None, r)
        out = moe_combine(yo, r)
        ctx.save_for_backward(x2, xp, gu, y, yo, wr, wg, wu, wd)
        ctx.routing, ctx.act, ctx.x_shape = r, act, x.shape
        E = wr.shape[0]
        counts = r.aux_counts if aux else torch.zeros(E, device=x.device, dtype=torch.float32)
        psum = r.aux_psum if aux else torch.zeros(E, device=x.device, dtype=torch.float32)
        ctx.mark_non_differentiable(counts)
        ctx.aux = aux
        return out.view(*x.shape[:-1], H), counts, psum

    @staticmethod
    def backward(ctx, dout, _dcounts, dpsum):
        x2, xp, gu, y, yo, wr, wg, wu, wd = ctx.saved_tensors
        r, act = ctx.routing, ctx.act
        H = x2.shape[1]
        I = wg.shape[1]
        d2 = dout.reshape(-1, H).contiguous().to(torch.bfloat16)
        aux_grad = dpsum.float().contiguous() if (ctx.aux and dpsum is not None) else None
        dyo, _dw, dlogits = moe_combine_bwd(d2, yo, r, aux_grad)
        gwd, flat_d = _grad_sink(wd)
        moe_wgrad(dyo, H, y, I, gwd, r)                                   # dWd_e += dyo^T y
        dgu, _ = moe_gemm("down_bwd", act, dyo, wd, None, r, gu=gu)
        gwg, flat_g = _grad_sink(wg)
        gwu, flat_u = _grad_sink(wu)
        moe_wgrad(dgu, 2 * I, xp, H, gwg, r)                              # dWg_e += dg^T x
        moe_wgrad(dgu[:, I:], 2 * I, xp, H, gwu, r)                       # dWu_e += du^T x
        dxp, _ = moe_gemm("gateup_dgrad", act, dgu, wg, wu, r)
        dx = None
        if ctx.needs_input_grad[0]:
            dx = moe_unpermute(dxp, r, torch.matmul(dlogits, wr.float())).view(ctx.x_shape)
        dwr = torch.matmul(dlogits.t(), x2.float())
        if getattr(wr, "_b200_flat_grad", False) and wr.grad is not None:
            wr.grad.copy_(wr.grad.float() + dwr)
            dwr = None
        else:
            dwr = dwr.to(wr.dtype)
        return (dx, dwr, None if flat_g else gwg, None if flat_u else gwu, None if flat_d else gwd,
                None, None, None, None)


def moe(x: torch.Tensor, w_router: torch.Tensor, wg: torch.Tensor, wu: torch.Tensor, wd: torch.Tensor, k: int,
        act: str = "sigmoid2", pad_mask: Optional[torch.Tensor] = None, aux: bool = False):
    """Mixtral's sparse MoE block (no jitter): x [..., H] bf16, w_router [E, H], wg / wu [E, I, H], wd [E, H, I], all
    bf16 and contiguous.  Each token goes to the top-k experts of softmax(x Wr^T) with the renormalised weights;
    expert e computes down_e(act(gate_e x, up_e x)).  pad_mask (bool [...], optional) selects the tokens of the
    load-balancing partials; aux=False skips them and their gradient.  Returns (out [..., H], aux_counts [E],
    aux_psum [E])."""
    _check_choice(act, GLU_ACTS, "moe: act")
    for t, nm in ((x, "x"), (w_router, "w_router"), (wg, "wg"), (wu, "wu"), (wd, "wd")):
        _need(t, torch.bfloat16, nm)
    H = x.shape[-1]
    if w_router.dim() != 2 or w_router.shape[1] != H:
        raise ValueError(f"w_router must be [E, {H}], got {list(w_router.shape)}")
    E = w_router.shape[0]
    if not 2 <= E <= 64:
        raise ValueError(f"w_router: number of experts must lie in 2..64, got {E}")
    if wg.dim() != 3 or wg.shape[0] != E or wg.shape[2] != H:
        raise ValueError(f"wg must be [{E}, I, {H}], got {list(wg.shape)}")
    I = wg.shape[1]
    if wu.shape != wg.shape:
        raise ValueError(f"wu must be {list(wg.shape)}, got {list(wu.shape)}")
    if tuple(wd.shape) != (E, H, I):
        raise ValueError(f"wd must be {[E, H, I]}, got {list(wd.shape)}")
    if H % 8 != 0 or I % 64 != 0:
        raise ValueError(f"x: hidden {H} must be a multiple of 8 and the intermediate size {I} of 64")
    step = I * H * wg.element_size()
    d = wu.data_ptr() - wg.data_ptr()
    if d <= 0 or d % step or d // step < E:
        raise ValueError("wu must lie E or more whole [I, hidden] matrices after wg in memory (one tensor map "
                         "addresses both; flat.ParamStore lays a layer's gate and up experts out that way)")
    if isinstance(k, bool) or not isinstance(k, int) or not 1 <= k <= min(E, 8):
        raise ValueError(f"k must be an integer in 1..{min(E, 8)}, got {k!r}")
    mask = None
    if pad_mask is not None:
        if tuple(pad_mask.shape) != tuple(x.shape[:-1]):
            raise ValueError(f"pad_mask must be {list(x.shape[:-1])}, got {list(pad_mask.shape)}")
        mask = pad_mask.reshape(-1).to(device=x.device, dtype=torch.uint8).contiguous()
    if x.numel() == 0:
        raise ValueError("x: no tokens")
    return _MoeFn.apply(x, w_router, wg, wu, wd, k, act, mask, bool(aux))


class _CrossEntropyFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, logits2d, targets, V, pad_token):
        rows, ld = logits2d.shape
        row_loss = torch.empty(rows, device=logits2d.device, dtype=torch.float32)
        row_lse = torch.empty(rows, device=logits2d.device, dtype=torch.float32)
        check(lib().b200_ce_fwd(logits2d.data_ptr(), ld, targets.data_ptr(), rows, V, int(pad_token),
                                row_loss.data_ptr(), row_lse.data_ptr(), _stream()), "b200_ce_fwd")
        ctx.save_for_backward(logits2d, targets, row_lse)
        ctx.V, ctx.pad = V, int(pad_token)
        return row_loss

    @staticmethod
    def backward(ctx, d_row_loss):
        logits2d, targets, row_lse = ctx.saved_tensors
        rows, ld = logits2d.shape
        scale = d_row_loss.contiguous().float()
        # in place: the logits buffer becomes d(loss)/d(logits); its producer (the logits GEMM) does
        # not need its own output for backward
        check(lib().b200_ce_bwd(logits2d.data_ptr(), ld, targets.data_ptr(), rows, ctx.V, ctx.pad,
                                row_lse.data_ptr(), scale.data_ptr(), _stream()), "b200_ce_bwd")
        return logits2d, None, None, None


def cross_entropy_rows(logits2d: torch.Tensor, targets: torch.Tensor, V: int, pad_token: int) -> torch.Tensor:
    """Per-row masked cross entropy of bf16 logits [rows, ld>=V] (contiguous, ld % 8 == 0), fp32 math;
    rows whose target is pad_token contribute 0 (the pad mask of core/training.py:1230-1232)."""
    _need(logits2d, torch.bfloat16, "logits")
    if targets.dtype != torch.int64 or not targets.is_contiguous():
        raise ValueError("targets must be contiguous int64")
    return _CrossEntropyFn.apply(logits2d, targets, int(V), int(pad_token))
