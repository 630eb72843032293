"""Shape-grouped flat storage for parameters, gradients and fp32 masters.

HBM layout (one allocation each, sized for one 80 GB H100 -- nothing is sharded or offloaded):

    master  fp32  [ group(r0,c0): batch0 x r0 x c0 | group(r1,c1): ... | all non-2-D params ]
    shadow  bf16  same layout (only with mixed precision): what forward/backward read
    grad    bf16/fp32 same layout: `param.grad` of every parameter is a view into it
    acc     fp32  same layout (only with gradient accumulation / clipping)

Every 2-D parameter of a given shape sits in one contiguous [batch, rows, cols] block, so the
optimizer runs ONE batched kernel sequence per shape (Newton-Schulz over 24 q_proj/o_proj matrices
is a single batched GEMM chain) and the data-parallel all-reduce is a single NCCL call on `grad`.  A 3-D parameter
[E, r, c] (a MoE layer's stacked expert weights) enters the (r, c) group as E consecutive matrices, so each expert
is orthogonalised on its own; the parameter and its .grad stay single [E, r, c] views.
The reference keeps a Python dict of separate arrays and loops over it (optimizers/muon.py:91).
"""
from __future__ import annotations

from collections import OrderedDict
from dataclasses import dataclass, field
from typing import Dict, List, Optional, Tuple

import torch
from torch import nn

ALIGN = 128  # elements; keeps every group 256-byte aligned in bf16 and 512-byte in fp32
ROW_PAD = 64  # single-matrix groups are followed by zero rows up to a multiple of this


@dataclass
class MatGroup:
    rows: int
    cols: int
    names: List[str] = field(default_factory=list)
    offset: int = 0

    @property
    def batch(self) -> int:
        return len(self.names)

    @property
    def numel(self) -> int:
        return self.batch * self.rows * self.cols


@dataclass
class VecEntry:
    name: str
    shape: Tuple[int, ...]
    offset: int
    numel: int


def _round_up(x: int, a: int) -> int:
    return (x + a - 1) // a * a


class ParamStore:
    def __init__(self, model: nn.Module, compute_dtype: torch.dtype = torch.bfloat16,
                 device: Optional[torch.device] = None):
        named = [(n, p) for n, p in model.named_parameters() if p.requires_grad]
        if not named:
            raise ValueError("model has no trainable parameters")
        self.device = torch.device(device) if device is not None else named[0][1].device
        self.compute_dtype = compute_dtype
        self.mixed = compute_dtype != torch.float32

        groups: "OrderedDict[Tuple[int, int], MatGroup]" = OrderedDict()
        vec_named = []
        for name, p in named:
            if p.dim() == 2 and not getattr(p, "_b200_elementwise", False):
                r, c = p.shape
                if c % 8 != 0:
                    raise ValueError(
                        f"2-D parameter {name} has {c} columns; the tensor-core path needs a multiple of 8 "
                        "(16-byte TMA rows)")
                groups.setdefault((r, c), MatGroup(r, c)).names.append(name)
            elif p.dim() == 3:
                # stacked expert weights [E, r, c]: E consecutive matrices of the (r, c) group, one entry per matrix
                # (the name repeated), so Newton-Schulz treats every expert as its own matrix
                nb, r, c = p.shape
                if c % 8 != 0:
                    raise ValueError(
                        f"3-D parameter {name} has {c} columns; the tensor-core path needs a multiple of 8")
                groups.setdefault((r, c), MatGroup(r, c)).names.extend([name] * nb)
            else:
                vec_named.append((name, p))
        off = 0
        for g in groups.values():
            g.offset = off
            # single matrices whose row count is not a multiple of 64 (the [V, hidden] embedding with
            # V = 32003) get zero tail rows reserved, so the tied logits GEMM can read a [V_pad, hidden]
            # view with an aligned N instead of falling off cuBLAS's fast path (see tied_logits_weight)
            tail = (_round_up(g.rows, ROW_PAD) - g.rows) * g.cols if g.batch == 1 else 0
            off = _round_up(off + g.numel + tail, ALIGN)
        self.mat_groups: List[MatGroup] = list(groups.values())
        self.mat_end = off
        self.vec_entries: List[VecEntry] = []
        self.vec_offset = off
        for name, p in vec_named:
            self.vec_entries.append(VecEntry(name, tuple(p.shape), off, p.numel()))
            off = _round_up(off + p.numel(), 8)
        self.vec_end = off
        self.total = _round_up(off, ALIGN)

        dev = self.device
        self.master = torch.zeros(self.total, dtype=torch.float32, device=dev)
        self.shadow = torch.zeros(self.total, dtype=compute_dtype, device=dev) if self.mixed else None
        self.grad = torch.zeros(self.total, dtype=compute_dtype, device=dev)
        self.acc: Optional[torch.Tensor] = None

        self.index: Dict[str, Tuple[int, Tuple[int, ...]]] = {}
        params_by_name = dict(named)
        for g in self.mat_groups:
            for i, n in enumerate(g.names):
                if n in self.index:
                    continue
                shape = tuple(params_by_name[n].shape)
                self.index[n] = (g.offset + i * g.rows * g.cols, shape)
        for e in self.vec_entries:
            self.index[e.name] = (e.offset, e.shape)

        params = dict(named)
        compute = self.shadow if self.mixed else self.master
        with torch.no_grad():
            for name, (o, shape) in self.index.items():
                p = params[name]
                n = p.numel()
                self.master[o:o + n].view(shape).copy_(p.detach().to(dev, torch.float32))
                if self.mixed:
                    self.shadow[o:o + n].view(shape).copy_(self.master[o:o + n].view(shape))
                p.data = compute[o:o + n].view(shape)
                p.grad = self.grad[o:o + n].view(shape)
                p._b200_flat_grad = True   # ops._accumulate_wgrad may GEMM straight into this view
        self.params = params
        model._b200_store = self

    # ---------------------------------------------------------------------------------------
    def view(self, buf: torch.Tensor, name: str) -> torch.Tensor:
        o, shape = self.index[name]
        n = 1
        for s in shape:
            n *= s
        return buf[o:o + n].view(shape)

    def padded_rows_view(self, buf: torch.Tensor, name: str) -> torch.Tensor:
        """[rows_pad, cols] view of a single-matrix group including its reserved zero tail rows."""
        o, (r, c) = self.index[name]
        g = next(g for g in self.mat_groups if name in g.names)
        if g.batch != 1:
            raise ValueError(f"{name} is part of a batched group; no tail rows reserved")
        return buf[o:o + _round_up(r, ROW_PAD) * c].view(_round_up(r, ROW_PAD), c)

    def tied_logits_weight(self, name: str = "embed_tokens.weight") -> Optional[torch.Tensor]:
        """Autograd leaf aliasing the (row-padded) embedding for the tied logits GEMM h @ E^T
        (arch/llama.py:401-403).  Its .grad aliases the same flat gradient memory as the
        parameter's, so both uses of E accumulate into one buffer.  None if no padding is needed."""
        if name not in self.index:
            return None
        o, (r, c) = self.index[name]
        if r % 8 == 0:
            return None
        try:
            w = self.padded_rows_view(self.shadow if self.mixed else self.master, name)
        except ValueError:
            return None
        leaf = w.detach().requires_grad_(True)
        leaf.grad = self.padded_rows_view(self.grad, name)
        return leaf

    def group_view(self, buf: torch.Tensor, g: MatGroup) -> torch.Tensor:
        return buf[g.offset:g.offset + g.numel].view(g.batch, g.rows, g.cols)

    def vec_range(self, buf: torch.Tensor) -> torch.Tensor:
        return buf[self.vec_offset:self.vec_end]

    def ensure_acc(self) -> torch.Tensor:
        if self.acc is None:
            self.acc = torch.zeros(self.total, dtype=torch.float32, device=self.device)
        return self.acc

    def zero_grad(self) -> None:
        self.grad.zero_()

    def named_master(self) -> Dict[str, torch.Tensor]:
        return {n: self.view(self.master, n) for n in self.index}

    @torch.no_grad()
    def load_gradients(self, grads: Dict[str, torch.Tensor]) -> None:
        """Drop-in path for `optimizer.update(model, gradients)` with an explicit (flat or nested)
        gradient dict, as the reference's trainer passes (core/training.py:1690,1700)."""
        flat = flatten_tree(grads)
        for name, g in flat.items():
            if name not in self.index:
                raise KeyError(f"gradient for unknown parameter {name}")
            self.view(self.grad, name).copy_(g.to(self.device, self.grad.dtype))

    @torch.no_grad()
    def refresh_shadow(self) -> None:
        if self.mixed:
            self.shadow.copy_(self.master)


def flatten_tree(tree, prefix: str = "") -> Dict[str, torch.Tensor]:
    """mlx.utils.tree_flatten for nested dict / list pytrees -> {'a.b.0.c': tensor}."""
    out: Dict[str, torch.Tensor] = {}
    if isinstance(tree, dict):
        for k, v in tree.items():
            out.update(flatten_tree(v, f"{prefix}.{k}" if prefix else str(k)))
    elif isinstance(tree, (list, tuple)):
        for i, v in enumerate(tree):
            out.update(flatten_tree(v, f"{prefix}.{i}" if prefix else str(i)))
    elif tree is not None:
        out[prefix] = tree
    return out


def get_store(model: nn.Module, compute_dtype: Optional[torch.dtype] = None) -> ParamStore:
    store = getattr(model, "_b200_store", None)
    if store is None:
        p0 = next(model.parameters())
        store = ParamStore(model, compute_dtype or p0.dtype, p0.device)
    return store
