"""Muon with the reference's surface (optimizers/muon.py:7-141), running on the sm_90a kernels.

    opt = Muon(learning_rate=float|callable, momentum=0.95, nesterov=True, ns_steps=5,
               alternate_optimizer=None, betas=None, eps=None, weight_decay=None)
    opt.update(model, gradients)      # the one call the trainer makes (core/training.py:1690,1700)
    opt.state[name]["momentum_buffer"], opt.count, opt.zeropower_via_newtonschulz5(G, steps)

Semantics follow the reference's intended math with its wiring defects fixed (SURVEY D1, D2):
gradients are matched by flattened name and the update is applied to the model in place.
Per 2-D shape group the step is: fused momentum+Nesterov+sum-of-squares pass -> batched
Newton-Schulz on wgmma -> fused `p += -lr*max(1,r/c)^0.5 * X` pass (fp32 master + bf16 shadow).
Non-2-D parameters go to `alternate_optimizer` if given, else to the SGD-momentum fallback
(muon.py:119-138).  `betas/eps/weight_decay` are accepted and ignored, as in the reference (:41-52).

Data parallel (`shard_ns=True`, set by the trainer when world > 1): gradients are already
all-reduced, so every rank holds the same momentum; each rank then orthogonalises only its slice
of every shape group (owner computes) and the results are exchanged with one in-place all-gather
per group (a broadcast for groups with fewer matrices than ranks), issued asynchronously so the
gather of group g overlaps the Newton-Schulz GEMMs of group g+1.  When the ranks can map each
other's memory (torch symmetric memory over NVLink; `B200_NS_P2P=0` disables) the gather is not a
separate collective at all: the gather buffers are peer-mapped and the LAST GEMM of each chain
stores its output tiles into every rank's buffer from its epilogue
(`b200_newton_schulz_allgather`), followed by one cross-rank barrier before the apply kernels.  Communication volume equals
the gradient all-reduce's all-gather half; Newton-Schulz work per rank drops by ~1/world
(SURVEY 8e "fused mode", modal/modal_cuda_utils.py:468-490 for the size-balanced ownership idea).
"""
from __future__ import annotations

import ctypes
import os
from typing import Callable, Dict, Optional, Tuple, Union

import torch

from .. import ops
from .._lib import NsGroup
from ..distributed import dp
from ..flat import ParamStore, get_store


class Muon:
    def __init__(self, learning_rate: Union[float, Callable] = 0.02, momentum: float = 0.95,
                 nesterov: bool = True, ns_steps: int = 5, alternate_optimizer=None,
                 betas: Optional[Tuple[float, float]] = None, eps: Optional[float] = None,
                 weight_decay: Optional[float] = None):
        self._learning_rate = learning_rate
        self.momentum = momentum
        self.nesterov = nesterov
        self.ns_steps = ns_steps
        self.alternate_optimizer = alternate_optimizer
        self.state: Dict[str, Dict[str, torch.Tensor]] = {}
        self.count = 0
        self.grad_scale = 1.0        # e.g. 1/world_size for the data-parallel mean
        self.use_accumulated = False  # read gradients from store.acc (fp32) instead of store.grad
        self.shard_ns = False         # owner-computes Newton-Schulz across data-parallel ranks
        self._store: Optional[ParamStore] = None
        self._buf = None
        self._exchange = "auto"       # see set_exchange()
        self._xg = self._xg_handles = None
        self._use_multicast = False

    def set_exchange(self, mode: str) -> str:
        """Select the owner-computes exchange at run time (bench.py's cross-check of the implementations):
        "auto" (peer stores; NVSwitch multicast from 4 ranks up), "unicast", "multicast", or "nccl" (equal-chunk
        ownership + all_gather_into_tensor).  Returns the mode actually in effect."""
        if mode not in ("auto", "unicast", "multicast", "nccl"):
            raise ValueError(f"unknown exchange mode {mode}")
        self._exchange = mode
        self._plan_world = None
        if self._xg_handles is not None and mode != "nccl":
            world = dp.world_size()
            mc_ok = all(int(getattr(h, "multicast_ptr", 0) or 0) != 0 for h in self._xg_handles)
            self._use_multicast = mc_ok and (mode == "multicast" or (mode == "auto" and world >= 4))
        return self.exchange_mode

    # -- reference surface ---------------------------------------------------------------------
    @property
    def learning_rate(self) -> float:
        return self._lr(self.count)

    def _lr(self, count: int) -> float:
        lr = self._learning_rate(count) if callable(self._learning_rate) else self._learning_rate
        return float(lr)

    def zeropower_via_newtonschulz5(self, G: torch.Tensor, steps: int) -> torch.Tensor:
        return ops.zeropower_via_newtonschulz5(G, steps)

    # -- state -----------------------------------------------------------------------------------
    def init(self, model) -> None:
        store = get_store(model)
        if self._store is store:
            return
        self._store = store
        dev = store.device
        self._buf = torch.zeros(store.total, dtype=torch.float32, device=dev)  # momentum buffers
        n_mat = max(store.mat_end, 8)
        total_batch = max(sum(g.batch for g in store.mat_groups), 1)
        # u = Nesterov momentum (Newton-Schulz input) and x = its orthogonalisation, for ALL shape groups at once
        # (same flat layout as the parameters): the groups advance through the chain together, see update()
        self._u = torch.empty(n_mat, dtype=torch.bfloat16, device=dev)
        self._x = torch.empty(n_mat, dtype=torch.bfloat16, device=dev)
        self._xg = None  # per-group gather buffers of the sharded mode (allocated on first use)
        self._xg_handles = None  # symmetric-memory handles when the buffers are peer-mapped
        self._use_multicast = False
        self._ws = torch.empty(256, dtype=torch.uint8, device=dev)   # grown on demand (update())
        self._ss = torch.empty(total_batch, dtype=torch.float32, device=dev)
        self._inv = torch.empty(total_batch, dtype=torch.float32, device=dev)
        self._inv2 = torch.empty(total_batch, dtype=torch.float32, device=dev)
        self._boff = []   # first matrix index of every group inside _ss / _inv / _inv2
        o = 0
        for g in store.mat_groups:
            self._boff.append(o)
            o += g.batch
        self.state = {}
        for g in store.mat_groups:
            for n in g.names:
                self.state[n] = {"momentum_buffer": store.view(self._buf, n)}
        if self.alternate_optimizer is None:
            for e in store.vec_entries:
                self.state[e.name] = {"momentum_buffer": store.view(self._buf, e.name)}
        else:
            self.alternate_optimizer.init_range(store, store.vec_offset, store.vec_end)

    # -- step --------------------------------------------------------------------------------------
    @torch.no_grad()
    def update(self, model, gradients=None) -> None:
        self.init(model)
        store = self._store
        if gradients is not None:
            store.load_gradients(gradients)
        gsrc = store.acc if self.use_accumulated else store.grad
        lr = self._lr(self.count)
        lib = ops.lib()
        stream = ops._stream()
        a, b, c = ops.NS_COEFFS
        world = dp.world_size() if self.shard_ns else 1
        rank = dp.env_rank_world()[0] if world > 1 else 0
        if world > 1 and self._xg is None:
            self._alloc_gather_buffers(store, world)
        p2p = world > 1 and self._xg_handles is not None and self._exchange != "nccl"
        groups = store.mat_groups
        if groups:
            # 1. momentum + Nesterov + per-matrix sum of squares for every group (muon.py:101,105), then ONE launch
            #    turns all sums of squares into 1/(||u||+eps) and its square (muon.py:72-73)
            for gi, g in enumerate(groups):
                n, rc = g.numel, g.rows * g.cols
                gg = gsrc[g.offset:g.offset + n]
                rws = ops.reduce_workspace(store.device, g.batch)
                ops.check(lib.b200_muon_momentum(gg.data_ptr(), ops._is_bf16(gg, "grad"),
                                                 self._buf.data_ptr() + 4 * g.offset, self._u.data_ptr() + 2 * g.offset,
                                                 self._ss.data_ptr() + 4 * self._boff[gi], rc, g.batch,
                                                 float(self.momentum), int(self.nesterov), float(self.grad_scale),
                                                 rws.data_ptr(), rws.numel(), stream), "b200_muon_momentum")
            ops.check(lib.b200_ns_scales(self._ss.data_ptr(), self._inv.data_ptr(), self._inv2.data_ptr(),
                                         self._ss.numel(), ops.NS_EPS, stream), "b200_ns_scales")
            # 2. Newton-Schulz on the matrices this rank owns, all groups advancing together: every stage of the
            #    iteration is one grouped wgmma launch (b200_newton_schulz_multi)
            entries, keep = [], []
            for gi, g in enumerate(groups):
                rc = g.rows * g.cols
                xbase = self._x.data_ptr() + 2 * g.offset if world == 1 else self._xg[gi].data_ptr()
                for lo, hi in self.owned_ranges_of(gi, world, rank):
                    if hi <= lo:
                        continue
                    peers, n_peers = None, 0
                    if p2p:   # GEMM -> all-gather in one kernel: the last GEMM stores into every rank's buffer
                        hdl = self._xg_handles[gi]
                        if self._use_multicast:
                            # one store to the NVSwitch multicast address reaches every rank's replica: per-rank
                            # NVLink egress is its own share, not (world - 1) copies of it
                            ptrs = [int(hdl.multicast_ptr) + 2 * lo * rc]
                        else:
                            ptrs = [int(bp) + 2 * lo * rc for r, bp in enumerate(hdl.buffer_ptrs) if r != rank]
                        peers = (ctypes.c_void_p * len(ptrs))(*ptrs)
                        keep.append(peers)
                        n_peers = len(ptrs)
                    e = NsGroup()
                    e.x_in = self._u.data_ptr() + 2 * (g.offset + lo * rc)
                    e.x_out = xbase + 2 * lo * rc
                    e.batch, e.rows, e.cols = hi - lo, g.rows, g.cols
                    e.inv_norm = self._inv.data_ptr() + 4 * (self._boff[gi] + lo)
                    e.inv_norm_sq = self._inv2.data_ptr() + 4 * (self._boff[gi] + lo)
                    e.peer_out = ctypes.cast(peers, ctypes.POINTER(ctypes.c_void_p)) if peers is not None else None
                    e.n_peers = n_peers
                    entries.append(e)
            tok = ops._t0("newton_schulz")
            for i in range(0, len(entries), 6):   # one grouped launch takes up to 6 problems
                chunk = entries[i:i + 6]
                arr = (NsGroup * len(chunk))(*chunk)
                need = int(lib.b200_newton_schulz_multi_workspace_bytes(arr, len(chunk), self.ns_steps))
                if self._ws.numel() < need:
                    self._ws = torch.empty(need, dtype=torch.uint8, device=store.device)
                ops.check(lib.b200_newton_schulz_multi(arr, len(chunk), self.ns_steps, a, b, c, self._ws.data_ptr(),
                                                       self._ws.numel(), stream), "b200_newton_schulz_multi")
            ops._t1(tok)
            # 3. exchange (data parallel) and apply
            pending = []
            for gi, g in enumerate(groups):
                rc = g.rows * g.cols
                x = self._x[g.offset:g.offset + g.numel] if world == 1 else self._xg[gi]
                works = []
                if world > 1 and not p2p:
                    chunk_len = dp.chunk_ranges(g.batch, world)[0]
                    if g.batch >= world:
                        works.append(dp.all_gather_chunks_(x, chunk_len * rc, async_op=True))
                    else:
                        works += [dp.broadcast_async_(x[i * rc:(i + 1) * rc], dp.small_group_owner(i, world))
                                  for i in range(g.batch)]
                pending.append((g, x, works))
            if p2p:
                # every rank's peer stores are stream-ordered before its barrier arrival
                self._xg_handles[0].barrier()
            for g, x, works in pending:
                for wk in works:
                    if wk is not None:
                        wk.wait()   # orders the current stream after the collective
                self._apply(store, g, x, lr, lib, stream)
        self._update_vectors(store, gsrc, lr)
        self.count += 1

    def _update_vectors(self, store, gsrc, lr) -> None:
        if store.vec_end > store.vec_offset:
            lo, hi = store.vec_offset, store.vec_end
            if self.alternate_optimizer is not None:
                self.alternate_optimizer.update_range(store, lo, hi, gsrc, self.grad_scale)
            else:
                p16 = store.shadow[lo:hi] if store.mixed else None
                ops.sgd_momentum(store.master[lo:hi], p16, gsrc[lo:hi], self._buf[lo:hi], self.momentum,
                                 self.nesterov, lr, self.grad_scale)

    def _alloc_gather_buffers(self, store, world: int) -> None:
        """One padded buffer per shape group: world * ceil(batch/world) matrices, so exchanges can stay in
        flight.  Peer-mapped (symmetric memory) when possible, plain device memory + NCCL otherwise."""
        sizes = [max(g.batch, world * dp.chunk_ranges(g.batch, world)[0]) * g.rows * g.cols for g in store.mat_groups]
        if os.environ.get("B200_NS_P2P", "1") != "0" and world <= 8:
            try:
                import torch.distributed as dist
                import torch.distributed._symmetric_memory as symm
                bufs = [symm.empty(n, dtype=torch.bfloat16, device=store.device) for n in sizes]
                self._xg_handles = [symm.rendezvous(t, group=dist.group.WORLD) for t in bufs]
                self._xg = bufs
                # multicast pays off once a unicast exchange would send several copies; B200_NS_MULTICAST=1/0 forces
                # it on/off
                mc_env = os.environ.get("B200_NS_MULTICAST", "auto")
                mc_ok = all(int(getattr(h, "multicast_ptr", 0) or 0) != 0 for h in self._xg_handles)
                self._use_multicast = mc_ok and (mc_env == "1" or (mc_env == "auto" and world >= 4))
                return
            except Exception as e:  # no peer mapping on this machine: NCCL exchange instead
                self._xg_handles = None
                if os.environ.get("B200_NS_P2P") == "1":
                    raise
                print(f"[muon] symmetric memory unavailable ({type(e).__name__}: {e}); using NCCL all-gather")
        self._xg = [torch.empty(n, dtype=torch.bfloat16, device=store.device) for n in sizes]

    @property
    def exchange_mode(self) -> str:
        if not self.shard_ns or self._xg is None:
            return "replicated" if not self.shard_ns else "sharded (not started)"
        if self._xg_handles is None or self._exchange == "nccl":
            return "NCCL all-gather"
        return ("fused GEMM+all-gather, NVSwitch multicast stores" if self._use_multicast
                else "fused GEMM+all-gather, unicast peer stores")

    def owned_ranges_of(self, gi: int, world: int, rank: int):
        """[lo, hi) ranges of shape group `gi` this rank orthogonalises.  With the peer-memory exchange any
        ownership works, so the split is flop-balanced over ALL matrices (dp.balanced_ranges: at 8 ranks a
        rank runs one or two long batched chains instead of 3-matrix slivers of every group); the NCCL
        exchange needs the equal-chunk split of `owned_ranges`."""
        g = self._store.mat_groups[gi]
        if world <= 1 or self._xg_handles is None or self._exchange == "nccl":
            return self.owned_ranges(g.batch, world, rank)
        if getattr(self, "_plan_world", None) != world:
            def cost(r, c):
                m, n = min(r, c), max(r, c)
                return 4.0 * m * m * n + 2.0 * m ** 3
            self._plan = dp.balanced_ranges([(q.batch, cost(q.rows, q.cols)) for q in self._store.mat_groups], world)
            self._plan_world = world
        return [(lo, hi) for (gg, lo, hi) in self._plan[rank] if gg == gi]

    @staticmethod
    def owned_ranges(batch: int, world: int, rank: int):
        """[lo, hi) matrix ranges of a shape group that `rank` orthogonalises in the sharded mode."""
        if world <= 1:
            return [(0, batch)]
        if batch >= world:
            return [dp.chunk_ranges(batch, world)[1][rank]]
        return [(i, i + 1) for i in range(batch) if dp.small_group_owner(i, world) == rank]

    @staticmethod
    def _apply(store, g, x, lr, lib, stream) -> None:
        """p += -lr * max(1, rows/cols)^0.5 * X  (muon.py:111-114), fp32 master + bf16 shadow in one pass."""
        n = g.numel
        scaling = max(1.0, g.rows / g.cols) ** 0.5
        p32 = store.master[g.offset:g.offset + n]
        p16 = store.shadow[g.offset:g.offset + n] if store.mixed else None
        ops.check(lib.b200_axpy_update(p32.data_ptr(), ops._ptr(p16), x.data_ptr(), 1, n,
                                       float(-lr * scaling), stream), "b200_axpy_update")

    # MLX-style aliases kept so callers written against mlx.optimizers.Optimizer keep working
    def apply_gradients(self, gradients, model):
        self.update(model, gradients)
        return model

    def step(self, model) -> None:
        """torch-style: consume the gradients autograd left in the flat store."""
        self.update(model, None)

    def state_dict(self) -> Dict[str, torch.Tensor]:
        out = {f"{n}.momentum_buffer": s["momentum_buffer"] for n, s in self.state.items()}
        if self.alternate_optimizer is not None:
            out.update(self.alternate_optimizer.state_dict())
        return out
