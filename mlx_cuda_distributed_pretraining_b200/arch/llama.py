"""Llama-style decoder with the reference's structure and parameter names (arch/llama.py), hosted
on PyTorch modules whose hot ops are the sm_90a kernels:

  RMSNorm            arch/llama.py:44-56   -> ops.rmsnorm (fused fwd/bwd)
  MLP                arch/llama.py:142-151 -> down(gate(x) * sigmoid(up(x)) * 2)  (sic, SURVEY D7)
  AttentionModule    arch/llama.py:154-252 -> FlashAttention (fused causal/GQA kernels)
  TransformerBlock   arch/llama.py:255-319 pre-norm residual
  Model              arch/llama.py:322-412 causal mask, tied logits h @ E^T

Flattened parameter names equal mlx's tree_flatten(model.parameters()) names, e.g.
`layers.0.self_attn.attn.q_proj.weight`, so checkpoints and optimizer state keys line up.
RoPE: arch/llama.py constructs a RotaryPositionEncoding and never applies it (SURVEY D6); the
faithful default is therefore no positional rotation.  `ModelArgs.apply_rope=True` enables the
interleaved-pair rotation of arch/llama_standard.py:213-215 through ops.rope.

`ModelArgs.variant = "mlx_lm"` builds the block the reference's trainer actually runs (mlx_lm.models.llama, DESIGN
D4): MLP down(silu(gate(x)) * up(x)), and RoPE always on q and k, half-split pairs (x[i], x[i + D/2]) unless
rope_traditional.  Parameter names are unchanged.
"""
from __future__ import annotations

from dataclasses import dataclass
from typing import Any, Dict, Optional

import torch
from torch import nn

from .. import ops
from .flash_attention import (BeamKV, CausalMask, DenseKV, DocumentCausalMask, FlashAttention, PrefixCausalMask,
                              QuantizedKV, RingKV)

VARIANTS = (None, "reference", "mlx_lm")


@dataclass
class ModelArgs:
    model_type: str
    hidden_size: int
    num_hidden_layers: int
    intermediate_size: int
    num_attention_heads: int
    head_dim: Optional[int] = None
    vocab_size: int = 32000
    num_key_value_heads: Optional[int] = None
    rope_theta: float = 10000.0
    rope_traditional: bool = False
    rope_scaling: Optional[Dict[str, Any]] = None
    rms_norm_eps: float = 1e-5
    max_position_embeddings: int = 4096
    attention_bias: bool = False
    attention_dropout: float = 0.0
    tie_word_embeddings: bool = False
    logit_scale: Optional[float] = None
    mlp_bias: bool = False
    use_flash_attention: bool = True
    use_flex_attention: bool = False
    flash_block_size: int = 128
    num_local_experts: int = 0
    num_experts_per_tok: int = 0
    apply_rope: bool = False  # extension; see module docstring
    sliding_window: Optional[int] = None  # extension: query q sees keys q - W .. q in every layer (None: causal)
    alibi: bool = False  # extension: ALiBi's bias slope_h * (k - q) on every layer's attention scores
    prefix_lm: bool = False  # extension: prefix-LM models (the prompt is the bidirectional prefix in prefill)
    variant: Optional[str] = None  # extension: None / "reference" (this block) or "mlx_lm" (module docstring)
    router_aux_loss_coef: float = 0.001  # with num_local_experts > 0: weight of the load-balancing loss


class RMSNorm(nn.Module):
    def __init__(self, dims: int, eps: float = 1e-5):
        super().__init__()
        self.weight = nn.Parameter(torch.ones(dims))
        self.eps = eps

    def forward(self, x: torch.Tensor) -> torch.Tensor:
        return ops.rmsnorm(x, self.weight, self.eps)


class MLP(nn.Module):
    def __init__(self, hidden_size: int, intermediate_size: int, use_bias: bool = False, act: str = "sigmoid2"):
        """act: "sigmoid2" (the reference's gate * sigmoid(up) * 2) or "silu" (mlx_lm's silu(gate) * up)."""
        super().__init__()
        self.act = act
        self.gate_proj = nn.Linear(hidden_size, intermediate_size, bias=use_bias)
        self.up_proj = nn.Linear(hidden_size, intermediate_size, bias=use_bias)
        self.down_proj = nn.Linear(intermediate_size, hidden_size, bias=use_bias)

    def forward(self, x: torch.Tensor) -> torch.Tensor:
        if self.gate_proj.bias is not None:
            return self.down_proj(ops.glu(self.gate_proj(x), self.up_proj(x), self.act))
        return ops.mlp(x, self.gate_proj.weight, self.up_proj.weight, self.down_proj.weight, self.act)


class _ExpertLinear(nn.Module):
    """E bias-free projections stacked as one [E, out, in] weight (mlx-lm's SwitchLinear)."""

    def __init__(self, num_experts: int, in_features: int, out_features: int):
        super().__init__()
        self.weight = nn.Parameter(torch.empty(num_experts, out_features, in_features))
        bound = in_features ** -0.5
        nn.init.uniform_(self.weight, -bound, bound)


class SwitchGLU(nn.Module):
    def __init__(self, hidden_size: int, intermediate_size: int, num_experts: int):
        super().__init__()
        self.gate_proj = _ExpertLinear(num_experts, hidden_size, intermediate_size)
        self.up_proj = _ExpertLinear(num_experts, hidden_size, intermediate_size)
        self.down_proj = _ExpertLinear(num_experts, intermediate_size, hidden_size)


class SparseMoeBlock(nn.Module):
    """Mixtral's sparse MoE block without jitter (model.misc.num_local_experts): the router `gate` [E, hidden] picks
    each token's top-k experts by softmax probability, their weights renormalised to sum 1, and the token's output is
    the weighted sum of those experts' MLPs (the block's activation, per-expert width intermediate_size).  Dropless.
    Parameter names follow mlx-lm's Mixtral (block_sparse_moe.gate / block_sparse_moe.switch_mlp.*).

    `last_aux` holds the (assignment counts, probability sums) [E] over the unmasked tokens of the last forward that
    asked for them (Model.moe_aux_loss), else None."""

    def __init__(self, hidden_size: int, intermediate_size: int, num_experts: int, top_k: int, act: str):
        super().__init__()
        self.num_experts, self.top_k, self.act = num_experts, top_k, act
        self.gate = nn.Linear(hidden_size, num_experts, bias=False)
        if num_experts % 8:
            # a router with E % 8 != 0 rows cannot go through Newton-Schulz (its GEMMs need N % 8 == 0): the flat
            # store keeps it with the elementwise parameters, so Muon / hybrid update it with their non-matrix rule
            self.gate.weight._b200_elementwise = True
        self.switch_mlp = SwitchGLU(hidden_size, intermediate_size, num_experts)
        self.last_aux = None

    def forward(self, x: torch.Tensor, token_mask: Optional[torch.Tensor] = None, aux: bool = False) -> torch.Tensor:
        s = self.switch_mlp
        out, counts, psum = ops.moe(x, self.gate.weight, s.gate_proj.weight, s.up_proj.weight, s.down_proj.weight,
                                    self.top_k, self.act, pad_mask=token_mask, aux=aux)
        self.last_aux = (counts, psum) if aux else None
        return out


class AttentionModule(nn.Module):
    def __init__(self, hidden_size: int, num_heads: int, num_kv_heads: Optional[int] = None,
                 head_dim: Optional[int] = None, max_positions: int = 4096, rope_theta: float = 10000.0,
                 rope_traditional: bool = False, rope_scaling: Optional[Dict[str, Any]] = None,
                 use_bias: bool = False, use_flash_attention: bool = True, use_flex_attention: bool = False,
                 flash_block_size: int = 128, apply_rope: bool = False, rope_layout: str = "interleaved",
                 alibi: bool = False, dropout: float = 0.0, layer_idx: int = 0):
        super().__init__()
        self.rope_layout = rope_layout
        if use_flex_attention:
            raise NotImplementedError("FlexAttention (arch/flex_attention.py) is out of scope of the hot path")
        self.hidden_size = hidden_size
        self.num_heads = num_heads
        self.num_kv_heads = num_kv_heads or num_heads
        self.head_dim = head_dim or (hidden_size // num_heads)
        # SimpleAttention (use_flash_attention=False) computes the same function; one kernel serves both
        self.attn = FlashAttention(hidden_size, num_heads, self.num_kv_heads, self.head_dim,
                                   dropout=dropout, use_bias=use_bias, flash_block_size=flash_block_size, alibi=alibi,
                                   layer_idx=layer_idx)
        self.scale = self.head_dim ** -0.5
        self.apply_rope = apply_rope
        self.max_positions = max_positions
        self.rope_theta = rope_theta

    def forward(self, x: torch.Tensor, mask=None, position_ids=None,
                dropout_seed: Optional[int] = None) -> torch.Tensor:
        if self.apply_rope and self.attn.rope_tables is None:
            self.attn.rope_tables = ops.rope_tables(self.max_positions, self.head_dim, self.rope_theta, x.device)
        return self.attn(x, mask=mask, rope_layout=self.rope_layout, dropout_seed=dropout_seed)

    def cached(self, x: torch.Tensor, cache: "KVCache", layer: int, window: Optional[int] = None,
               prefix: Optional[torch.Tensor] = None, chunk: Optional["CacheChunk"] = None) -> torch.Tensor:
        """This layer's attention against the KV cache: prefill when x is [B, S, hidden], one decode step when x is
        [B, hidden], a chunk appended at the cache's current lengths when chunk is given (x [B, L, hidden]).
        window: the model's sliding window (None: causal).  prefix (int32 [B], prefill only): the prefix-LM mask's
        prefix lengths."""
        if self.apply_rope and self.attn.rope_tables is None:
            self.attn.rope_tables = ops.rope_tables(self.max_positions, self.head_dim, self.rope_theta, x.device)
        kv = cache.layer(layer)
        if chunk is not None:
            return self.attn.forward_extend(x, kv, chunk, window, self.rope_layout)
        if x.dim() == 3:
            mask = CausalMask(x.shape[1], window) if prefix is None else PrefixCausalMask(prefix, x.shape[1])
            return self.attn.forward_prefill(x, mask, kv, self.rope_layout)
        return self.attn.forward_decode(x, kv, cache, window, self.rope_layout)


class TransformerBlock(nn.Module):
    def __init__(self, args: ModelArgs, layer_idx: int = 0):
        super().__init__()
        inter = args.intermediate_size or 4 * args.hidden_size
        if args.variant not in VARIANTS:
            raise ValueError(f"ModelArgs.variant must be one of {VARIANTS}, got {args.variant!r}")
        mlx_lm = args.variant == "mlx_lm"
        self.input_layernorm = RMSNorm(args.hidden_size, eps=args.rms_norm_eps)
        self.self_attn = AttentionModule(
            hidden_size=args.hidden_size, num_heads=args.num_attention_heads,
            num_kv_heads=args.num_key_value_heads, head_dim=args.head_dim,
            max_positions=args.max_position_embeddings, rope_theta=args.rope_theta,
            rope_traditional=args.rope_traditional, rope_scaling=args.rope_scaling,
            use_bias=args.attention_bias, use_flash_attention=args.use_flash_attention,
            use_flex_attention=args.use_flex_attention, flash_block_size=args.flash_block_size,
            apply_rope=args.apply_rope or mlx_lm,
            rope_layout="half" if mlx_lm and not args.rope_traditional else "interleaved", alibi=args.alibi,
            dropout=args.attention_dropout, layer_idx=layer_idx)
        self.post_attention_layernorm = RMSNorm(args.hidden_size, eps=args.rms_norm_eps)
        act = "silu" if mlx_lm else "sigmoid2"
        self.moe = bool(args.num_local_experts)
        if self.moe:
            if args.mlp_bias:
                raise ValueError("ModelArgs.mlp_bias is not supported with num_local_experts > 0")
            self.block_sparse_moe = SparseMoeBlock(args.hidden_size, inter, args.num_local_experts,
                                                   args.num_experts_per_tok, act)
        else:
            self.mlp = MLP(args.hidden_size, inter, use_bias=args.mlp_bias, act=act)

    def _ffn(self, y: torch.Tensor, token_mask=None, aux: bool = False) -> torch.Tensor:
        if self.moe:
            return self.block_sparse_moe(y, token_mask, aux)
        return self.mlp(y)

    def forward(self, x: torch.Tensor, mask=None, position_ids=None) -> torch.Tensor:
        x = x + self.self_attn(self.input_layernorm(x), mask=mask, position_ids=position_ids)
        return x + self._ffn(self.post_attention_layernorm(x))

    def forward_fused(self, h: torch.Tensor, pending, mask=None, position_ids=None, token_mask=None,
                      aux: bool = False, dropout_seed: Optional[int] = None):
        """Same block with every residual add fused into the norm that consumes it.  `pending` is the
        previous block's MLP output not yet added to the stream h (None for the first block); returns
        (h after the attention residual, this block's MLP output still to be added)."""
        n1, n2 = self.input_layernorm, self.post_attention_layernorm
        if pending is None:
            y = n1(h)
        else:
            h, y = ops.add_rmsnorm(h, pending, n1.weight, n1.eps)
        a = self.self_attn(y, mask=mask, position_ids=position_ids, dropout_seed=dropout_seed)
        h, y = ops.add_rmsnorm(h, a, n2.weight, n2.eps)
        return h, self._ffn(y, token_mask, aux)

    def forward_cached(self, h: torch.Tensor, pending, cache: "KVCache", layer: int, window: Optional[int] = None,
                       prefix: Optional[torch.Tensor] = None, chunk: Optional["CacheChunk"] = None):
        """forward_fused with the attention run against the KV cache (AttentionModule.cached)."""
        n1, n2 = self.input_layernorm, self.post_attention_layernorm
        if pending is None:
            y = n1(h)
        else:
            h, y = ops.add_rmsnorm(h, pending, n1.weight, n1.eps)
        a = self.self_attn.cached(y, cache, layer, window, prefix, chunk)
        h, y = ops.add_rmsnorm(h, a, n2.weight, n2.eps)
        return h, self._ffn(y)


def check_cache_options(model: "Model", kv_bits: Optional[int] = None, kv_group_size: int = 64,
                        quantized_kv_start: int = 0, max_kv_size: Optional[int] = None, what: str = "KVCache",
                        head_dim: Optional[int] = None) -> None:
    """Raises ValueError, naming `what`, for KV-cache options KVCache cannot serve: a bad max_kv_size, a rotating cache
    with kv_bits, for a prefix-LM model or for a model Model.extend cannot serve, and bad kv_bits / kv_group_size
    (given head_dim, one that does not divide it) or quantized_kv_start.  The model is read only for a rotating
    cache."""
    if max_kv_size is not None:
        ops.check_max_kv_size(max_kv_size, what)
        if kv_bits is not None:
            raise ValueError(f"{what}: max_kv_size does not combine with kv_bits (mlx_lm's rotating cache does not "
                             "quantize)")
        if model.args.prefix_lm:
            raise ValueError(f"{what}: a prefix-LM model cannot use a rotating cache (max_kv_size): its prompt is one "
                             "prefix")
        model.check_extend(None)
    if kv_bits is not None:
        ops.check_kv_quant(kv_bits, kv_group_size, head_dim, what)
        if isinstance(quantized_kv_start, bool) or not isinstance(quantized_kv_start, int) or quantized_kv_start < 0:
            raise ValueError(f"{what}: quantized_kv_start must be a non-negative int, got {quantized_kv_start!r}")


class KVCache:
    """Per-layer KV caches (`layers`, one DenseKV, QuantizedKV or RingKV per layer; flash_attention) and the number of
    valid positions per row: `lens` on the device (read by the kernels) and `host_lens` (so sizing a launch never
    reads the device).  A DenseKV holds K and V [B, s_max, Hk, D] in the model's activation dtype.  s_max is rounded
    up to a multiple of 256, the decode kernel's chunk.

    kv_bits (4 or 8), kv_group_size (32, 64 or 128) and quantized_kv_start are the reference's quantized cache
    (core/generation_lite.py:75-90, :100-108): once the longest row holds more than quantized_kv_start positions,
    after prefill or after a decode step, every layer converts to a QuantizedKV and the unquantized buffers are
    released.  When the prompt already passes the start, prefill writes the quantized cache directly and no
    unquantized buffer is ever allocated; otherwise those buffers hold quantized_kv_start + 1 positions (rounded up to
    256), all they can hold before conversion.  The layers are allocated by the first set_lengths (prefill).

    max_kv_size = M (an int >= 5) makes the cache rotate, as the reference's make_prompt_cache(model, max_kv_size)
    (core/generation_lite.py:103, :120) gives every layer mlx_lm's RotatingKVCache(max_size=M, keep=4): each row keeps
    C = M + max_chunk - 1 slots (rounded up to 256; s_max is then C), position t in slot ops.ring_slot(t, C), and a
    query at position q sees key k iff k <= q and (k < 4 or q - k <= M - 5) (DESIGN §2).  A row's length is then
    unbounded.  max_chunk (default 512) is the longest chunk Model.extend may append; the cache is filled by
    Model.extend only, cannot be truncated (overwritten slots cannot be restored) and is bf16 with head_dim 64 or
    128, not quantized and not for prefix-LM models."""

    max_kv_size: Optional[int] = None
    max_chunk: Optional[int] = None
    live: Optional[torch.Tensor] = None  # rotating: the rows the current decode step appends to (None: all)

    def __init__(self, model: "Model", batch: int, s_max: int, kv_bits: Optional[int] = None,
                 kv_group_size: int = 64, quantized_kv_start: int = 0, max_kv_size: Optional[int] = None,
                 max_chunk: Optional[int] = None):
        a = model.args
        attn = model.layers[0].self_attn
        check_cache_options(model, kv_bits, kv_group_size, quantized_kv_start, max_kv_size, "KVCache", attn.head_dim)
        self.max_kv_size = max_kv_size
        self.max_chunk = max_chunk
        if max_kv_size is not None:
            self.max_chunk = 512 if max_chunk is None else max_chunk
            if isinstance(self.max_chunk, bool) or not isinstance(self.max_chunk, int) or self.max_chunk < 1:
                raise ValueError(f"KVCache: max_chunk must be an int >= 1, got {max_chunk!r}")
            s_max = max_kv_size + self.max_chunk - 1
        elif max_chunk is not None:
            raise ValueError("KVCache: max_chunk is for a rotating cache (max_kv_size)")
        self.kv_bits, self.kv_group_size, self.quantized_kv_start = kv_bits, kv_group_size, quantized_kv_start
        w = model.embed_tokens.weight
        self._layers, self._device, self._dtype = a.num_hidden_layers, w.device, w.dtype
        self._batch, self._heads = batch, (attn.num_kv_heads, attn.head_dim)
        self.s_max = max(256, -(-s_max // 256) * 256)
        self.layers = None
        self.quantized = False
        if kv_bits is None:
            self._allocate(self.s_max)
        self.lens = torch.zeros(batch, device=w.device, dtype=torch.int32)
        self.host_lens = [0] * batch
        nbytes = ops.attention_decode_workspace_bytes(batch, attn.num_heads, self.s_max, attn.head_dim)
        self.workspace = torch.empty(max(nbytes, 16), device=w.device, dtype=torch.uint8)

    def _allocate(self, positions: int) -> None:
        """Unquantized layers of `positions` positions: RingKV when the cache rotates, else DenseKV."""
        shape = (self._batch, positions) + self._heads

        def zeros():
            return torch.zeros(shape, device=self._device, dtype=self._dtype)

        if self.rotating:
            self.layers = [RingKV(zeros(), zeros(), self.max_kv_size) for _ in range(self._layers)]
        else:
            self.layers = [DenseKV(zeros(), zeros()) for _ in range(self._layers)]

    def _allocate_quantized(self) -> None:
        self.layers = [QuantizedKV(self._batch, self.s_max, *self._heads, self.kv_bits, self.kv_group_size,
                                   self._device) for _ in range(self._layers)]
        self.quantized = True

    @property
    def rotating(self) -> bool:
        return self.max_kv_size is not None

    def layer(self, i: int):
        """Layer i's cache object (DenseKV, QuantizedKV or RingKV)."""
        return self.layers[i]

    def set_lengths(self, lengths) -> None:
        if self.rotating:
            raise ValueError("a rotating KV cache is filled in chunks by Model.extend, not by Model.prefill")
        if any(n < 1 or n > self.s_max for n in lengths):
            raise ValueError(f"lengths must lie in [1, {self.s_max}], got {list(lengths)}")
        self.host_lens = [int(n) for n in lengths]
        self.lens.copy_(torch.tensor(self.host_lens, dtype=torch.int32))
        if self.layers is None:  # kv_bits: the prefill decides the first format
            if max(self.host_lens) > self.quantized_kv_start:
                self._allocate_quantized()
            else:
                self._allocate(min(self.s_max, -(-(self.quantized_kv_start + 1) // 256) * 256))

    def extend_lengths(self, counts) -> None:
        """counts[b] >= 0 more positions for row b (one Model.extend chunk): host_start keeps the lengths before it.
        Until the cache is quantized, the unquantized buffers grow (copied into larger ones, at most s_max positions)
        when the chunk needs room; a kv_bits cache that holds nothing yet starts unquantized, because the reference
        attends a chunk over the unquantized cache and converts afterwards (maybe_quantize)."""
        counts = [int(n) for n in counts]
        if len(counts) != self._batch or any(n < 0 for n in counts):
            raise ValueError(f"counts must be {self._batch} non-negative ints, got {counts}")
        ends = [n + c for n, c in zip(self.host_lens, counts)]
        if self.rotating and max(counts) > self.max_chunk:
            raise ValueError(f"a chunk of {max(counts)} tokens exceeds the rotating cache's max_chunk "
                             f"({self.max_chunk}): its keys would overwrite keys its queries see")
        if not self.rotating and max(ends) > self.s_max:
            raise ValueError(f"KV cache full: rows would hold {max(ends)} positions, the cache has {self.s_max}")
        if not self.quantized and not self.rotating:  # a ring is allocated whole by __init__
            have = 0 if self.layers is None else self.layers[0].k.shape[1]
            if max(ends) > have:
                old = self.layers
                self._allocate(min(self.s_max, -(-max(ends) // 256) * 256))
                if old is not None:
                    for new, o in zip(self.layers, old):
                        new.k[:, :have].copy_(o.k)
                        new.v[:, :have].copy_(o.v)
        self.host_start = list(self.host_lens)
        self.host_lens = ends
        self.lens.copy_(torch.tensor(ends, dtype=torch.int32))

    def truncate(self, lengths) -> None:
        """Shortens row b to lengths[b] <= its current length: later positions are left as they are and never read."""
        if self.rotating:
            raise ValueError("a rotating KV cache cannot be truncated: the slots of dropped positions may hold keys "
                             "that are already overwritten")
        lengths = [int(n) for n in lengths]
        if len(lengths) != self._batch or any(not 0 <= n <= m for n, m in zip(lengths, self.host_lens)):
            raise ValueError(f"truncate: lengths must lie in [0, current lengths {self.host_lens}], got {lengths}")
        self.host_lens = lengths
        self.lens.copy_(torch.tensor(lengths, dtype=torch.int32))

    def advance(self, live=None) -> None:
        """One more position per row (the token a decode step is about to append).  live (rotating caches; a bool
        per row): only those rows advance, and the decode step writes nothing into the others (self.live)."""
        if live is not None:
            if not self.rotating:
                raise ValueError("advance: live is for a rotating cache (an unbounded one is truncated instead)")
            live = [bool(x) for x in live]
            if len(live) != self._batch:
                raise ValueError(f"advance: live must have {self._batch} entries, got {len(live)}")
            self.host_lens = [n + int(x) for n, x in zip(self.host_lens, live)]
            self.live = torch.tensor(live, dtype=torch.int32).to(self._device)
            self.lens.add_(self.live)
            return
        if not self.rotating and max(self.host_lens) + 1 > self.s_max:
            raise ValueError(f"KV cache full ({self.s_max} positions)")
        self.host_lens = [n + 1 for n in self.host_lens]
        self.lens.add_(1)
        self.live = None

    def maybe_quantize(self) -> None:
        """maybe_quantize_kv_cache (core/generation_lite.py:75-90): with kv_bits, the first time the longest row
        holds more than quantized_kv_start positions, convert every layer and release the unquantized buffers."""
        if self.kv_bits is None or self.quantized or max(self.host_lens) <= self.quantized_kv_start:
            return
        n = max(self.host_lens)
        dense = self.layers
        self._allocate_quantized()
        for d, qkv in zip(dense, self.layers):
            qkv.store(d.k, d.v, n)

    def nbytes(self) -> int:
        """Bytes held by the layers' buffers."""
        return 0 if self.layers is None else sum(kv.nbytes() for kv in self.layers)


class BeamKVCache:
    """The cache of a beam search (core.generation.beam_search; DESIGN §4.2.4).  `prefix` is an ordinary KVCache of
    batch G that Model.prefill filled with the G prompts (the groups), stored and read once per group.  Group g's fork
    point is T0_g = 256 floor(P_g / 256) for its prompt length P_g: positions below it are read from the prefix, and a
    beam's positions t >= T0_g live at index t - T0_g of the beam's tail slot, per layer (a BeamKV over the prefix
    layer's DenseKV) K and V tails [S = G n_beams, tail_cap, Hk, D] with tail_cap = 255 + max_tokens rounded up to
    256.  Group g owns slots [g n_beams, (g + 1) n_beams); prompt positions [T0_g, P_g) start in slot g n_beams.

    The decode batch is the live beam rows, set by set_rows (group, slot and length per row; a group's rows are
    contiguous and equally long).  fork copies tails between slots.  Model.decode_step runs on it unchanged."""

    def __init__(self, model: "Model", prefix: KVCache, n_beams: int, max_tokens: int):
        if prefix.quantized or prefix.rotating or prefix.kv_bits is not None:
            raise ValueError("BeamKVCache: the prefix must be an unquantized, non-rotating KVCache filled by prefill")
        attn = model.layers[0].self_attn
        self.prefix, self.n_beams = prefix, n_beams
        self.n_groups = prefix._batch
        self.t0 = [256 * (n // 256) for n in prefix.host_lens]
        self.tail_cap = -(-(255 + max_tokens) // 256) * 256
        self.layers = [BeamKV(kv, n_beams, self.tail_cap, self.t0, prefix.host_lens) for kv in prefix.layers]
        self._tails = [kv.k_tail for kv in self.layers] + [kv.v_tail for kv in self.layers]
        dev = prefix._device
        self._buffers = torch.tensor([t.data_ptr() for t in self._tails], dtype=torch.int64).to(dev)
        nbytes = ops.attention_decode_beam_workspace_bytes(self.n_groups * n_beams, attn.num_heads, prefix.s_max,
                                                           self.tail_cap, attn.head_dim)
        self.workspace = torch.empty(max(nbytes, 16), device=dev, dtype=torch.uint8)
        self.set_rows(list(range(self.n_groups)), [g * n_beams for g in range(self.n_groups)], prefix.host_lens)

    def set_rows(self, groups, slots, lengths) -> None:
        """The decode batch: row b belongs to group groups[b] (ascending), holds lengths[b] positions and keeps its
        tail in slot slots[b].  One host-to-device copy."""
        groups, slots, lengths = [int(g) for g in groups], [int(s) for s in slots], [int(n) for n in lengths]
        R, G = len(groups), self.n_groups
        if R < 1 or len(slots) != R or len(lengths) != R or any(b < a for a, b in zip(groups, groups[1:])):
            raise ValueError("set_rows: one group, slot and length per row, groups ascending, at least one row")
        row0, rows = [0] * G, [0] * G
        for b, g in enumerate(groups):
            if rows[g] == 0:
                row0[g] = b
            rows[g] += 1
        t = torch.tensor(lengths + groups + slots + self.t0 + row0 + rows, dtype=torch.int32).to(self.prefix._device)
        self.host_lens, self.groups, self.slots = lengths, groups, slots
        self.lens, self.tables = t[:R], t[R:]

    def fork(self, copies) -> None:
        """copies: (src slot, dst slot, positions) triples: tail indices [0, positions) of every layer's K and V tail
        go from src to dst, in one launch.  No destination may be a source."""
        if not copies:
            return
        c = torch.tensor(copies, dtype=torch.int32).to(self.prefix._device)
        ops.kv_beam_fork(self._buffers, c, max(n for _, _, n in copies), self._tails)

    def layer(self, i: int):
        """Layer i's BeamKV."""
        return self.layers[i]

    def advance(self, live=None) -> None:
        if live is not None:
            raise ValueError("advance: live is for a rotating cache")
        if any(n + 1 - self.t0[g] > self.tail_cap for n, g in zip(self.host_lens, self.groups)):
            raise ValueError(f"beam cache full: the tails hold {self.tail_cap} positions past the fork point")
        self.host_lens = [n + 1 for n in self.host_lens]
        self.lens.add_(1)

    def maybe_quantize(self) -> None:
        pass

    def nbytes(self) -> int:
        """Bytes held by the prefix and the tails."""
        return self.prefix.nbytes() + sum(kv.nbytes() for kv in self.layers)


class CacheChunk:
    """The positions one Model.extend call appends, as the layers read them: row b's tokens i < n_b of the chunk
    [B, L] go to cache positions start[b] + i.  start / end: int32 [B] on the device (the lengths before and after);
    pos: int32 [B, L] rotation positions (padding tokens take their row's last position, so that no rotation reads
    past the tables); rows / src / dst: int64 indices of the valid tokens (row, index in the chunk, cache position);
    scratch: a quantized cache's bf16 K / V for the call, made by its first layer.  slots (a rotating cache's C): dst
    are the ring slots ops.ring_slot(start[b] + i, C).  verify / workspace: set by Model.verify, whose chunks the
    layers attend with DenseKV.verify over that decode workspace."""

    verify = False
    workspace: Optional[torch.Tensor] = None

    def __init__(self, start, counts, L: int, device, slots: Optional[int] = None):
        ends = [a + n for a, n in zip(start, counts)]
        self.start = torch.tensor(start, dtype=torch.int32).to(device)
        self.end = torch.tensor(ends, dtype=torch.int32).to(device)
        self.max_end = max(ends)
        rows = [b for b, n in enumerate(counts) for _ in range(n)]
        src = [i for n in counts for i in range(n)]
        self.rows = torch.tensor(rows, dtype=torch.int64).to(device)
        self.src = torch.tensor(src, dtype=torch.int64).to(device)
        dst = [start[b] + i for b, i in zip(rows, src)]
        if slots is not None:
            dst = [ops.ring_slot(t, slots) for t in dst]
        self.dst = torch.tensor(dst, dtype=torch.int64).to(device)
        last = torch.tensor([max(e - 1, 0) for e in ends], dtype=torch.int64)
        pos = torch.minimum(torch.tensor(start, dtype=torch.int64)[:, None] + torch.arange(L)[None], last[:, None])
        self.pos = pos.to(torch.int32).to(device)
        self.scratch = None


class Model(nn.Module):
    def __init__(self, args: ModelArgs):
        super().__init__()
        self.args = args
        self.vocab_size = args.vocab_size
        self.embed_tokens = nn.Embedding(args.vocab_size, args.hidden_size)
        self.layers = nn.ModuleList([TransformerBlock(args, i) for i in range(args.num_hidden_layers)])
        self.norm = RMSNorm(args.hidden_size, eps=args.rms_norm_eps)
        self.logit_scale = args.logit_scale
        self._tied_w = None  # padded alias of the embedding for the logits GEMM (set lazily)
        self.lm_head = None if args.tie_word_embeddings else nn.Linear(args.hidden_size, args.vocab_size, bias=False)

    def hidden_states(self, inputs: torch.Tensor, position_ids=None, attention_mask=None,
                      token_mask: Optional[torch.Tensor] = None,
                      prefix_lens: Optional[torch.Tensor] = None,
                      dropout_seed: Optional[int] = None) -> torch.Tensor:
        """position_ids (int [B, S], optional): packed rows, each token's position within its document (0 at the
        document's first token).  It selects the document-causal mask and, with RoPE on, the rotation angles, so
        every document is computed as if it ran alone.  None keeps the causal mask over whole rows.  Both masks carry
        args.sliding_window.  token_mask (bool [B, S], optional; MoE models): the tokens the load-balancing loss
        counts; given, every MoE layer keeps its partials for moe_aux_loss().  prefix_lens (int32 [B] on the device,
        optional): prefix-LM rows, query q of row b sees key k iff k <= q or k < prefix_lens[b] (PrefixCausalMask);
        it does not combine with position_ids or a sliding window.  dropout_seed (an int in [0, 2^64), optional): the
        base of the attention-dropout masks when args.attention_dropout > 0 and the model trains with grad enabled;
        layer i draws with ops.dropout_seed(dropout_seed, i).  None draws fresh seeds from torch's CPU generator."""
        B, S = inputs.shape
        if prefix_lens is not None:
            if position_ids is not None or attention_mask is not None:
                raise ValueError("prefix_lens does not combine with position_ids or attention_mask")
            if self.args.sliding_window is not None or self.args.alibi:
                raise ValueError("prefix_lens does not combine with a sliding window or ALiBi")
            if tuple(prefix_lens.shape) != (B,):
                raise ValueError(f"prefix_lens must be [B] = [{B}], got {list(prefix_lens.shape)}")
            mask = PrefixCausalMask(prefix_lens, S)
        elif attention_mask is not None:
            mask = attention_mask
        elif position_ids is not None:
            if tuple(position_ids.shape) != (B, S):
                raise ValueError(f"position_ids must be [B, S] = {[B, S]}, got {list(position_ids.shape)}")
            mask = DocumentCausalMask(position_ids, self.args.sliding_window)
        else:
            mask = CausalMask(S, self.args.sliding_window)
        h = ops.embedding(inputs, self.embed_tokens.weight)
        pending = None
        if self.args.num_local_experts:
            aux = token_mask is not None
            self._moe_tokens = token_mask.sum() if aux else None
            for layer in self.layers:
                h, pending = layer.forward_fused(h, pending, mask=mask, position_ids=position_ids,
                                                 token_mask=token_mask, aux=aux, dropout_seed=dropout_seed)
        else:
            for layer in self.layers:
                h, pending = layer.forward_fused(h, pending, mask=mask, position_ids=position_ids,
                                                 dropout_seed=dropout_seed)
        if pending is None:
            return self.norm(h)
        return ops.add_rmsnorm(h, pending, self.norm.weight, self.norm.eps)[1]

    def moe_aux_loss(self) -> Optional[torch.Tensor]:
        """transformers' load_balancing_loss_func over all layers' router logits of the last hidden_states call that
        had a token_mask, with attention_mask = token_mask: E * sum_e f_e P_e, f_e = assignments to expert e and P_e =
        the sum of its router probabilities, both over (layers x unmasked tokens) and divided by their number.  The
        gradient flows through P only.  None for a dense model or when no partials were kept."""
        if not self.args.num_local_experts or any(l.block_sparse_moe.last_aux is None for l in self.layers):
            return None
        counts = torch.stack([l.block_sparse_moe.last_aux[0] for l in self.layers]).sum(0)
        psum = torch.stack([l.block_sparse_moe.last_aux[1] for l in self.layers]).sum(0)
        n = self._moe_tokens.float() * len(self.layers)
        return self.args.num_local_experts * (counts * psum).sum() / (n * n)

    def _logits_weight(self) -> torch.Tensor:
        """[V or V_pad, hidden] weight of the logits GEMM: lm_head, or the embedding (tied,
        arch/llama.py:401-403) through its zero-row-padded alias when V is not a multiple of 8 (with N = 32003
        cuBLAS falls off its fast path; same values, same gradients, padded classes dropped afterwards)."""
        if self.lm_head is not None:
            return self.lm_head.weight
        store = getattr(self, "_b200_store", None)
        if store is not None and self._tied_w is None:
            w = store.tied_logits_weight()
            self._tied_w = w if w is not None else False
        if self._tied_w is not None and self._tied_w is not False:
            return self._tied_w
        return self.embed_tokens.weight

    def padded_logits(self, inputs: torch.Tensor, position_ids=None, token_mask=None, prefix_lens=None,
                      dropout_seed=None):
        """(logits [B*S, ld], V) with ld >= V, ld % 8 == 0 when the fused cross-entropy can take them
        (bf16 weights, tied + row-padded embedding alias or an aligned vocabulary); else (None, V).
        Eligibility is decided BEFORE the forward pass, so an ineligible config (fp32, logit_scale,
        unaligned untied vocabulary) never pays for hidden states it then throws away."""
        if self.logit_scale is not None:
            return None, self.vocab_size
        w = self._logits_weight()
        if w.shape[0] % 8 != 0 or w.dtype != torch.bfloat16:
            return None, self.vocab_size
        h = self.hidden_states(inputs, position_ids, token_mask=token_mask, prefix_lens=prefix_lens,
                               dropout_seed=dropout_seed)
        logits = torch.nn.functional.linear(h, w)
        return logits.view(-1, logits.shape[-1]), self.vocab_size

    def forward(self, inputs: torch.Tensor, position_ids=None, attention_mask=None, token_mask=None,
                prefix_lens=None, dropout_seed=None) -> torch.Tensor:
        h = self.hidden_states(inputs, position_ids, attention_mask, token_mask, prefix_lens, dropout_seed)
        logits = torch.nn.functional.linear(h, self._logits_weight())[..., :self.vocab_size]
        if self.logit_scale is not None:
            logits = logits * self.logit_scale
        return logits

    # -- generation: prefill and decode steps against a KVCache ---------------------------------------------------
    def _row_logits(self, h: torch.Tensor, pending: Optional[torch.Tensor]) -> torch.Tensor:
        """Final norm and fp32 logits [B, V] of one hidden row per sequence (forward's arithmetic)."""
        y = self.norm(h) if pending is None else ops.add_rmsnorm(h, pending, self.norm.weight, self.norm.eps)[1]
        logits = torch.nn.functional.linear(y, self._logits_weight())[..., :self.vocab_size]
        if self.logit_scale is not None:
            logits = logits * self.logit_scale
        return logits.float()

    @torch.no_grad()
    def prefill(self, tokens: torch.Tensor, lengths, cache: KVCache) -> torch.Tensor:
        """Runs the right-padded prompts tokens [B, S] (row b valid in [0, lengths[b])) through the block stack as
        training does, fills cache positions [0, S) and sets the cache lengths.  Returns the fp32 logits [B, V] at
        each row's last prompt position only.  Padding is harmless: under the causal mask no valid position sees it,
        and the decode steps never read cache positions at or past a row's length.  A prefix-LM model (args.prefix_lm)
        runs the prompt as its prefix, P_b = lengths[b]: valid positions see the whole prompt and no padding, and
        every later (decoded) query sees all cached keys, which is the prefix mask's rule for it."""
        B, S = tokens.shape
        cache.set_lengths(lengths)
        prefix = None
        if self.args.prefix_lm:
            prefix = torch.tensor([int(n) for n in lengths], dtype=torch.int32).to(tokens.device)
        h = ops.embedding(tokens, self.embed_tokens.weight)
        pending = None
        for i, layer in enumerate(self.layers):
            h, pending = layer.forward_cached(h, pending, cache, i, self.args.sliding_window, prefix)
        cache.maybe_quantize()
        rows = torch.arange(B, device=tokens.device)
        last = torch.tensor([n - 1 for n in lengths], device=tokens.device)
        return self._row_logits(h[rows, last], None if pending is None else pending[rows, last])

    def check_extend(self, cache: KVCache, counts=None) -> None:
        """Raises ValueError when Model.extend cannot serve this model and cache (counts: the tokens per row)."""
        attn = self.layers[0].self_attn
        if self.embed_tokens.weight.dtype != torch.bfloat16:
            raise ValueError(f"chunked prefill needs a bf16 model and cache, got {self.embed_tokens.weight.dtype} "
                             "(the one-shot prefill serves other dtypes)")
        if attn.head_dim not in (64, 128):
            raise ValueError(f"chunked prefill needs head_dim 64 or 128, got {attn.head_dim} (the one-shot prefill "
                             "serves other head dims)")
        if self.args.prefix_lm and counts is not None \
                and any(n > 0 and m == 0 for n, m in zip(counts, cache.host_lens)):
            raise ValueError("a prefix-LM model's first prompt cannot be split into chunks: its prefix attends to the "
                             "keys of later chunks (give it whole to Model.prefill)")

    @torch.no_grad()
    def extend(self, tokens: torch.Tensor, lengths, cache: KVCache) -> torch.Tensor:
        """Appends the right-padded tokens [B, L] (row b valid in [0, lengths[b]), lengths[b] may be 0) at each row's
        current cache length, each token attending over its row's cache as in decoding, and returns the fp32 logits
        [B, V] after each row's last new token (a row with no new token gets its padding's logits).  The quantized
        cache converts afterwards, as after a prefill (maybe_quantize)."""
        B, L = tokens.shape
        counts = [int(n) for n in lengths]
        if B != cache._batch:
            raise ValueError(f"tokens have {B} rows, the cache {cache._batch}")
        if len(counts) != B or any(not 0 <= n <= L for n in counts) or max(counts) < 1:
            raise ValueError(f"lengths must be {B} ints in [0, {L}], at least one positive, got {counts}")
        self.check_extend(cache, counts)
        cache.extend_lengths(counts)
        chunk = CacheChunk(cache.host_start, counts, L, tokens.device, cache.s_max if cache.rotating else None)
        h = ops.embedding(tokens, self.embed_tokens.weight)
        pending = None
        for i, layer in enumerate(self.layers):
            h, pending = layer.forward_cached(h, pending, cache, i, self.args.sliding_window, chunk=chunk)
        cache.maybe_quantize()
        rows = torch.arange(B, device=tokens.device)
        last = torch.tensor([max(n - 1, 0) for n in counts], device=tokens.device)
        return self._row_logits(h[rows, last], None if pending is None else pending[rows, last])

    @torch.no_grad()
    def verify(self, tokens: torch.Tensor, lengths, cache: KVCache) -> torch.Tensor:
        """Model.extend for a short chunk, tokens [B, L] with L <= 16 (speculative decoding's verify step and the
        draft's catch-up): the same appends, absolute-position RoPE, window, ALiBi and MoE, with the chunk attended by
        the split-KV multi-query decode kernel (DenseKV.verify), so any dtype and head dim the decode step serves.
        Returns the fp32 logits [B, L, V] after every token of the chunk (a row's padding positions get unspecified
        logits).  The cache must be an unquantized, non-rotating KVCache holding at least one position per row with
        new tokens (a prefix-LM model's decoded queries are causal)."""
        B, L = tokens.shape
        counts = [int(n) for n in lengths]
        if B != cache._batch:
            raise ValueError(f"tokens have {B} rows, the cache {cache._batch}")
        if not 1 <= L <= ops.MULTI_MAX_QUERIES:
            raise ValueError(f"verify: chunks of 1 to {ops.MULTI_MAX_QUERIES} tokens per row, got {L}")
        if len(counts) != B or any(not 0 <= n <= L for n in counts) or max(counts) < 1:
            raise ValueError(f"lengths must be {B} ints in [0, {L}], at least one positive, got {counts}")
        if cache.rotating or cache.kv_bits is not None or cache.layers is None:
            raise ValueError("verify needs an unquantized, non-rotating KV cache that a prefill has filled")
        if any(n > 0 and m == 0 for n, m in zip(counts, cache.host_lens)):
            raise ValueError("verify appends to a prefilled cache: a row with new tokens holds no position")
        cache.extend_lengths(counts)
        chunk = CacheChunk(cache.host_start, counts, L, tokens.device)
        attn = self.layers[0].self_attn
        chunk.verify = True
        chunk.workspace = torch.empty(max(16, ops.attention_decode_multi_workspace_bytes(
            B, L, attn.num_heads, cache.s_max, attn.head_dim)), device=tokens.device, dtype=torch.uint8)
        h = ops.embedding(tokens, self.embed_tokens.weight)
        pending = None
        for i, layer in enumerate(self.layers):
            h, pending = layer.forward_cached(h, pending, cache, i, self.args.sliding_window, chunk=chunk)
        return self._row_logits(h, pending)

    @torch.no_grad()
    def decode_step(self, tokens: torch.Tensor, cache: KVCache, live=None) -> torch.Tensor:
        """Appends one token per row (tokens [B]) at position cache.host_lens[b] and returns the fp32 logits [B, V]
        that follow it.  live (a rotating cache only; a bool per row): rows with False neither advance nor write, and
        their logits are unspecified."""
        cache.advance(live)
        h = ops.embedding(tokens, self.embed_tokens.weight)
        pending = None
        for i, layer in enumerate(self.layers):
            h, pending = layer.forward_cached(h, pending, cache, i, self.args.sliding_window)
        cache.maybe_quantize()
        return self._row_logits(h, pending)

    # mlx nn.Module-style accessors used by the optimizers' update(model, grads) surface
    def parameters_dict(self) -> Dict[str, torch.Tensor]:
        return dict(self.named_parameters())

    @torch.no_grad()
    def load_parameters(self, params: Dict[str, torch.Tensor], strict: bool = True) -> None:
        own = dict(self.named_parameters())
        for name, value in params.items():
            if name not in own:
                if strict:
                    raise KeyError(f"unexpected parameter {name}")
                continue
            own[name].copy_(value.to(own[name].dtype))
        if strict:
            missing = set(own) - set(params)
            if missing:
                raise KeyError(f"missing parameters: {sorted(missing)[:5]}...")
