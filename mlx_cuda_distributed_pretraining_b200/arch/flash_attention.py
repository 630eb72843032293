"""FlashAttention module with the reference's constructor and call surface
(arch/flash_attention.py:32-41,158-194), running the fused sm_90a kernels.

The reference materialises softmax(QK^T*scale + mask)V un-tiled (:97-156); here the same result
comes from `ops.attention` (tensor-core forward + backward, online softmax, GQA head sharing).
"""
from __future__ import annotations

from typing import Optional

import torch
from torch import nn

from .. import ops


def alibi_slopes(num_heads: int) -> torch.Tensor:
    """ALiBi's per-head slopes (Press et al., "Train Short, Test Long"), fp32 [num_heads] on the CPU.  For H a power
    of two, m_i = 2^(-8 i / H), i = 1 .. H.  Otherwise, with n = 2^floor(log2 H): the n slopes of the rule for n,
    then the odd-indexed slopes (i = 1, 3, 5, ...) of the rule for 2n, the first H - n of them."""
    if isinstance(num_heads, bool) or not isinstance(num_heads, int) or num_heads < 1:
        raise ValueError(f"alibi_slopes: num_heads must be a positive int, got {num_heads!r}")

    def pow2(n: int):
        return [2.0 ** (-8.0 * i / n) for i in range(1, n + 1)]

    n = 1 << (num_heads.bit_length() - 1)
    slopes = pow2(n) + pow2(2 * n)[0::2][:num_heads - n]
    return torch.tensor(slopes, dtype=torch.float32)


def _window(window: Optional[int]) -> Optional[int]:
    if window is not None and (isinstance(window, bool) or not isinstance(window, int) or window < 0):
        raise ValueError(f"sliding window must be None or a non-negative int, got {window!r}")
    return window


class CausalMask:
    """Marker for the additive causal mask the reference builds in arch/llama.py:384-387
    (-inf strictly above the diagonal).  The fused kernel applies it implicitly.

    window (optional int >= 0): the sliding causal window of the reference's FlexAttention example
    (README-FlexAttention.md:47-59): query q sees key k iff 0 <= q - k <= window."""

    def __init__(self, seq_len: int, window: Optional[int] = None):
        self.seq_len = seq_len
        self.window = _window(window)

    def dense(self, dtype=torch.float32, device="cpu") -> torch.Tensor:
        m = torch.full((self.seq_len, self.seq_len), float("-inf"), dtype=dtype, device=device)
        m = torch.triu(m, diagonal=1)
        if self.window is not None:
            m = m + torch.tril(torch.full_like(m, float("-inf")), diagonal=-self.window - 1)
        return m[None, None]


class DocumentCausalMask:
    """Marker for the document-causal mask of packed rows: pos (int32 [B, S]) is each token's position within its
    document (0 at a document's first token, +1 per token inside it), and query q sees key k iff
    q - pos[q] <= k <= q -- the causal mask of every document run alone.  The fused document kernels apply it
    implicitly, and RoPE rotates by pos.

    window (optional int >= 0) intersects it with the sliding window 0 <= q - k <= window, which is the same mask
    with pos clamped at window.  RoPE still rotates by the unclamped pos."""

    def __init__(self, pos: torch.Tensor, window: Optional[int] = None):
        if pos.dim() != 2:
            raise ValueError(f"DocumentCausalMask: pos must be [B, S], got {list(pos.shape)}")
        self.pos = pos.to(torch.int32).contiguous()
        self.seq_len = pos.shape[1]
        self.window = _window(window)

    def dense(self, dtype=torch.float32, device="cpu") -> torch.Tensor:
        """The additive [B, 1, S, S] mask (0 where visible, -inf elsewhere)."""
        pos = self.pos.to(device=device, dtype=torch.int64)
        s = torch.arange(self.seq_len, device=device)
        q, k = s[:, None], s[None, :]
        ok = (k <= q) & (k >= (s - pos)[:, :, None])
        if self.window is not None:
            ok = ok & (q - k <= self.window)
        m = torch.zeros(ok.shape, dtype=dtype, device=device).masked_fill(~ok, float("-inf"))
        return m[:, None]


class PrefixCausalMask:
    """Marker for the prefix-LM mask: prefix (int32 [B]) holds each row's prefix length P_b, and query q sees key k
    iff k <= q or k < P_b -- the prefix attends bidirectionally within itself and every later token is causal over
    everything before it.  P_b <= 1 is the causal mask and P_b = S full attention; the fused kernels clamp P_b to
    [0, S], and dense() does the same."""

    def __init__(self, prefix: torch.Tensor, seq_len: int):
        if prefix.dim() != 1:
            raise ValueError(f"PrefixCausalMask: prefix must be [B], got {list(prefix.shape)}")
        self.prefix = prefix.to(torch.int32).contiguous()
        self.seq_len = seq_len

    def dense(self, dtype=torch.float32, device="cpu") -> torch.Tensor:
        """The additive [B, 1, S, S] mask (0 where visible, -inf elsewhere)."""
        P = self.prefix.to(device=device, dtype=torch.int64).clamp(0, self.seq_len)
        s = torch.arange(self.seq_len, device=device)
        q, k = s[:, None], s[None, :]
        ok = (k <= q)[None] | (k[None] < P[:, None, None])
        m = torch.zeros(ok.shape, dtype=dtype, device=device).masked_fill(~ok, float("-inf"))
        return m[:, None]


# -- one layer's KV cache, one class per format --------------------------------------------------------------------
# Each format owns its buffers and the ops calls that write and read them, for the generation phases it serves:
#   store(k, v)                                       prefill: k, v [B, S, Hk, D] into positions [0, S)
#   decode(q, k, v, step, attn, window, rope_layout)  q [B, H, D], k, v [B, Hk, D] appended at step.lens - 1 (rotated
#                                                     there with attn.rope_tables), then attended -> ctx [B, H, D]
#   extend(q, k, v, chunk, attn, window)              a llama.CacheChunk's rotated q [B, L, H, D], k, v [B, L, Hk, D]
#                                                     written, then attended -> ctx [B, L, H, D]
#   verify(q, k, v, chunk, attn, window)              extend for a short chunk (chunk.verify, L <= 16: speculative
#                                                     decoding), attended split over keys (DenseKV only)
# step is the model-wide cache (llama.KVCache / BeamKVCache), which holds the per-step state: lens, workspace and,
# per format, the ring's live mask or the beam tables.  attn is the FlashAttention module: scale, rope_tables and
# alibi_slopes().
def _nbytes(*tensors) -> int:
    return sum(t.numel() * t.element_size() for t in tensors)


class DenseKV:
    """One layer's K and V [B, s_max, Hk, D] in the model's activation dtype."""

    def __init__(self, k: torch.Tensor, v: torch.Tensor):
        self.k, self.v = k, v

    def nbytes(self) -> int:
        return _nbytes(self.k, self.v)

    def store(self, k: torch.Tensor, v: torch.Tensor) -> None:
        S = k.shape[1]
        self.k[:, :S].copy_(k)
        self.v[:, :S].copy_(v)

    def decode(self, q, k, v, step, attn, window, rope_layout):
        ops.kv_append(q, k, v, self.k, self.v, step.lens, attn.rope_tables, layout=rope_layout)
        return ops.attention_decode(q, self.k, self.v, step.lens, attn.scale, step.workspace, window=window,
                                    alibi=attn.alibi_slopes(q.device))

    def extend(self, q, k, v, chunk, attn, window):
        r, src, dst = chunk.rows, chunk.src, chunk.dst
        self.k[r, dst] = k[r, src]
        self.v[r, dst] = v[r, src]
        return ops.attention_cached(q, self.k, self.v, chunk.start, chunk.end, attn.scale, window=window,
                                    alibi=attn.alibi_slopes(q.device))

    def verify(self, q, k, v, chunk, attn, window):
        r, src, dst = chunk.rows, chunk.src, chunk.dst
        self.k[r, dst] = k[r, src]
        self.v[r, dst] = v[r, src]
        return ops.attention_decode_multi(q, self.k, self.v, chunk.start, chunk.end, attn.scale, chunk.workspace,
                                          window=window, alibi=attn.alibi_slopes(q.device))


class QuantizedKV:
    """One layer's quantized KV cache (the reference's QuantizedKVCache; DESIGN §4.2.1): for K and for V, codes uint8
    [B, s_max, Hk, D * bits / 8] and fp32 (scale, bias) parameters [B, Hk, s_max, D / group_size, 2]."""

    def __init__(self, batch: int, s_max: int, num_kv_heads: int, head_dim: int, bits: int, group_size: int,
                 device):
        self.bits, self.group_size = bits, group_size
        cshape, pshape = ops.kv_quant_shapes(batch, s_max, num_kv_heads, head_dim, bits, group_size)
        self.k_codes = torch.zeros(cshape, device=device, dtype=torch.uint8)
        self.v_codes = torch.zeros(cshape, device=device, dtype=torch.uint8)
        self.k_params = torch.zeros(pshape, device=device, dtype=torch.float32)
        self.v_params = torch.zeros(pshape, device=device, dtype=torch.float32)

    def buffers(self):
        """(k_codes, v_codes, k_params, v_params), the argument order of the ops.*_quant wrappers."""
        return self.k_codes, self.v_codes, self.k_params, self.v_params

    def nbytes(self) -> int:
        return _nbytes(*self.buffers())

    def store(self, k: torch.Tensor, v: torch.Tensor, n: Optional[int] = None) -> None:
        """Quantizes positions [0, n) (default: all) of k, v [B, S, Hk, D]: a prefill, or the conversion of a
        DenseKV's buffers."""
        ops.kv_quantize(k.contiguous(), v.contiguous(), *self.buffers(), self.bits, self.group_size, n=n)

    def decode(self, q, k, v, step, attn, window, rope_layout):
        bits, g = self.bits, self.group_size
        ops.kv_append_quant(q, k, v, *self.buffers(), step.lens, bits, g, attn.rope_tables, layout=rope_layout)
        return ops.attention_decode_quant(q, *self.buffers(), step.lens, bits, g, attn.scale, step.workspace,
                                          window=window, alibi=attn.alibi_slopes(q.device))

    def extend(self, q, k, v, chunk, attn, window):
        """The chunk is quantized into a temporary cache and its valid positions copied in; the queries then attend
        over the cache's dequantised [0, end) in chunk.scratch (bf16 K / V made by the call's first layer)."""
        B, L, Hk, D = k.shape
        bits, g = self.bits, self.group_size
        r, src, dst = chunk.rows, chunk.src, chunk.dst
        tmp = QuantizedKV(B, L + L % 2, Hk, D, bits, g, k.device)
        ops.kv_quantize(k, v, *tmp.buffers(), bits, g)
        for t, u in zip(self.buffers()[:2], tmp.buffers()[:2]):
            t[r, dst] = u[r, src]
        for t, u in zip(self.buffers()[2:], tmp.buffers()[2:]):
            t[r, :, dst] = u[r, :, src]
        if chunk.scratch is None:
            shape = (B, chunk.max_end, Hk, D)
            chunk.scratch = (torch.empty(shape, device=k.device, dtype=torch.bfloat16),
                             torch.empty(shape, device=k.device, dtype=torch.bfloat16))
        k_att, v_att = ops.kv_dequantize(*self.buffers(), chunk.end, bits, g, out=chunk.scratch)
        return ops.attention_cached(q, k_att, v_att, chunk.start, chunk.end, attn.scale, window=window,
                                    alibi=attn.alibi_slopes(q.device))


class RingKV:
    """One layer's rotating KV cache (mlx_lm's RotatingKVCache; DESIGN §4.2.3): K and V rings bf16 [B, C, Hk, D],
    position t in slot ops.ring_slot(t, C), read under max_kv_size.  Filled by extend only (chunk.dst are ring
    slots); a decode step appends to the rows of step.live (int32 [B], None: all)."""

    def __init__(self, k: torch.Tensor, v: torch.Tensor, max_kv_size: int):
        self.k, self.v, self.max_kv_size = k, v, max_kv_size

    def nbytes(self) -> int:
        return _nbytes(self.k, self.v)

    def decode(self, q, k, v, step, attn, window, rope_layout):
        ops.kv_append_ring(q, k, v, self.k, self.v, step.lens, step.live, attn.rope_tables, rope_layout)
        return ops.attention_decode_ring(q, self.k, self.v, step.lens, self.max_kv_size, attn.scale, step.workspace,
                                         window=window, alibi=attn.alibi_slopes(q.device))

    def extend(self, q, k, v, chunk, attn, window):
        r, src, dst = chunk.rows, chunk.src, chunk.dst
        self.k[r, dst] = k[r, src]
        self.v[r, dst] = v[r, src]
        return ops.attention_ring(q, self.k, self.v, chunk.start, chunk.end, self.max_kv_size, attn.scale,
                                  window=window, alibi=attn.alibi_slopes(q.device))


class BeamKV:
    """One layer of a beam search's cache (llama.BeamKVCache; DESIGN §4.2.4): the DenseKV `prefix` [G, s_prefix, Hk,
    D] holding the G prompts, and beam tails k_tail, v_tail [G n_beams, tail_cap, Hk, D].  Group g's positions
    [t0[g], lens[g]) start at index 0 of slot g n_beams.  Decode only; step.tables are the cache's int32 device
    tables (ops.attention_decode_beam)."""

    def __init__(self, prefix: DenseKV, n_beams: int, tail_cap: int, t0, lens):
        self.prefix, self.n_groups = prefix, len(t0)
        p = prefix.k
        shape = (self.n_groups * n_beams, tail_cap) + tuple(p.shape[2:])
        self.k_tail = torch.zeros(shape, device=p.device, dtype=p.dtype)
        self.v_tail = torch.zeros(shape, device=p.device, dtype=p.dtype)
        for g, (s, n) in enumerate(zip(t0, lens)):
            self.k_tail[g * n_beams, :n - s].copy_(prefix.k[g, s:n])
            self.v_tail[g * n_beams, :n - s].copy_(prefix.v[g, s:n])

    def nbytes(self) -> int:
        """Bytes of the tails (the prefix belongs to its own cache)."""
        return _nbytes(self.k_tail, self.v_tail)

    def decode(self, q, k, v, step, attn, window, rope_layout):
        ops.kv_append_beam(q, k, v, self.k_tail, self.v_tail, step.lens, step.tables, self.n_groups,
                           attn.rope_tables, rope_layout)
        return ops.attention_decode_beam(q, self.prefix.k, self.prefix.v, self.k_tail, self.v_tail, step.lens,
                                         step.tables, attn.scale, step.workspace, window=window,
                                         alibi=attn.alibi_slopes(q.device))


class FlashAttention(nn.Module):
    """alibi: add ALiBi's bias alibi_slopes(num_heads)[h] * (k - q) to every causal score (the slopes are not
    parameters: a device tensor made on first use, like rope_tables).  dropout: the probability p of dropping an
    attention weight after the softmax (arch/flash_attention.py:146-148 of the reference), applied only in training
    mode with grad enabled; layer_idx (the layer's index in the model) derives the layer's mask seed from the
    forward's dropout_seed."""

    def __init__(self, hidden_size: int, num_heads: int, num_kv_heads: Optional[int] = None,
                 head_dim: Optional[int] = None, dropout: float = 0.0, use_bias: bool = False,
                 flash_block_size: int = 128, alibi: bool = False, layer_idx: int = 0):
        super().__init__()
        self.hidden_size = hidden_size
        self.num_heads = num_heads
        self.num_kv_heads = num_kv_heads or num_heads
        self.head_dim = head_dim or (hidden_size // num_heads)
        if isinstance(dropout, bool) or not isinstance(dropout, (int, float)) or not 0.0 <= float(dropout) < 1.0:
            raise ValueError(f"attention dropout must be a float in [0, 1), got {dropout!r}")
        self.dropout = float(dropout)
        self.layer_idx = int(layer_idx)
        self.flash_block_size = flash_block_size  # accepted for config compatibility (kernel tiles are 128)
        self.q_proj = nn.Linear(hidden_size, self.num_heads * self.head_dim, bias=use_bias)
        self.k_proj = nn.Linear(hidden_size, self.num_kv_heads * self.head_dim, bias=use_bias)
        self.v_proj = nn.Linear(hidden_size, self.num_kv_heads * self.head_dim, bias=use_bias)
        self.o_proj = nn.Linear(self.num_heads * self.head_dim, hidden_size, bias=use_bias)
        self.scale = self.head_dim ** -0.5
        self.rope_tables = None  # (cos, sin) set by the parent when RoPE is enabled
        self.alibi = bool(alibi)
        self._alibi_slopes = None  # fp32 [num_heads] on the device, made on first use

    def alibi_slopes(self, device) -> Optional[torch.Tensor]:
        """The ALiBi slopes on `device` (None without ALiBi)."""
        if not self.alibi:
            return None
        if self._alibi_slopes is None or self._alibi_slopes.device != torch.device(device):
            self._alibi_slopes = alibi_slopes(self.num_heads).to(device)
        return self._alibi_slopes

    def drops(self) -> bool:
        """Whether a forward drops: p > 0, training mode and grad enabled (validation, prefill, decode and export
        never drop)."""
        return self.dropout > 0.0 and self.training and torch.is_grad_enabled()

    def _flash_attention(self, q: torch.Tensor, k: torch.Tensor, v: torch.Tensor, mask=None,
                         dropout_seed: Optional[int] = None, drop: bool = False) -> torch.Tensor:
        """q [B,S,H,D], k/v [B,S,Hk,D] -> [B,S,H,D].  drop: apply self.dropout, with the layer's seed
        ops.dropout_seed(dropout_seed, layer_idx) (dropout_seed None: a seed drawn by ops.attention)."""
        pos = window = prefix = None
        if mask is None:
            causal = False
        elif isinstance(mask, CausalMask):
            causal, window = True, mask.window
        elif isinstance(mask, DocumentCausalMask):
            causal, pos, window = True, mask.pos, mask.window
        elif isinstance(mask, PrefixCausalMask):
            causal, prefix = True, mask.prefix
        else:
            raise NotImplementedError(
                "the fused kernel supports mask=None, the causal mask (CausalMask), the document-causal mask of "
                "packed rows (DocumentCausalMask) or the prefix-LM mask (PrefixCausalMask); arbitrary additive masks "
                "are outside the reference's training path")
        alibi = self.alibi_slopes(q.device)
        p = self.dropout if drop else 0.0
        seed = None if not drop or dropout_seed is None else ops.dropout_seed(dropout_seed, self.layer_idx)
        dt = q.dtype
        if dt == torch.float32 and 3 * self.head_dim <= 128:
            # full-precision configs (mixed_precision: false, e.g. BASELINE C1, head_dim 16): logits through
            # three-term bf16 products (hi/lo split operands), ~fp32-accurate scores on the same kernels
            return ops.attention_fp32(q, k, v, self.scale, causal, pos=pos, window=window, alibi=alibi,
                                      prefix=prefix, dropout=p, seed=seed)
        if dt != torch.bfloat16:  # larger head dims: bf16 operands with fp32 accumulation (stated in DESIGN.md)
            q, k, v = q.to(torch.bfloat16), k.to(torch.bfloat16), v.to(torch.bfloat16)
        o = ops.attention(q, k, v, self.scale, causal, pos=pos, window=window, alibi=alibi, prefix=prefix,
                          dropout=p, seed=seed)
        return o if dt == torch.bfloat16 else o.to(dt)

    def _qkv(self, x: torch.Tensor):
        """q [..., H, D] and k, v [..., Hk, D] projected from x [..., hidden]."""
        lead = x.shape[:-1]
        if self.q_proj.bias is None and self.k_proj.bias is None and self.v_proj.bias is None:
            q, k, v = ops.multi_linear(x, (self.q_proj.weight, self.k_proj.weight, self.v_proj.weight))
        else:
            q, k, v = self.q_proj(x), self.k_proj(x), self.v_proj(x)
        return (q.reshape(*lead, self.num_heads, self.head_dim), k.reshape(*lead, self.num_kv_heads, self.head_dim),
                v.reshape(*lead, self.num_kv_heads, self.head_dim))

    def _out(self, ctx: torch.Tensor) -> torch.Tensor:
        """o_proj of ctx [..., H, D]."""
        ctx = ctx.reshape(*ctx.shape[:-2], self.num_heads * self.head_dim)
        return ops.linear(ctx, self.o_proj.weight) if self.o_proj.bias is None else self.o_proj(ctx)

    def forward(self, x: torch.Tensor, mask=None, rope_layout: str = "interleaved",
                dropout_seed: Optional[int] = None) -> torch.Tensor:
        """rope_layout: ops.rope's pair layout when RoPE is on ("interleaved" or mlx_lm's "half").  dropout_seed: the
        model's per-step dropout base (see drops() for when it applies)."""
        S = x.shape[1]
        q, k, v = self._qkv(x)
        if self.rope_tables is not None:
            cos_t, sin_t = self.rope_tables
            pos = mask.pos if isinstance(mask, DocumentCausalMask) else None  # packed rows: position in document
            q = ops.rope(q, cos_t[:S], sin_t[:S], pos, rope_layout)
            k = ops.rope(k, cos_t[:S], sin_t[:S], pos, rope_layout)
        # the dropout arguments go only to dropping calls: without them the call is exactly the dropout-free one
        ctx = (self._flash_attention(q, k, v, mask, dropout_seed, True) if self.drops()
               else self._flash_attention(q, k, v, mask))
        return self._out(ctx)

    # -- generation: the same layer against one layer of a KV cache (a DenseKV, QuantizedKV, RingKV or BeamKV) ------
    def forward_prefill(self, x: torch.Tensor, mask, kv, rope_layout: str = "interleaved") -> torch.Tensor:
        """forward(x, mask) over a right-padded prompt batch x [B, S, hidden] that also stores the (rotated) keys and
        values in positions [0, S) of kv (kv.store).  Attention runs through _flash_attention on the unquantized k and
        v, so the numerics are the training forward's."""
        S = x.shape[1]
        q, k, v = self._qkv(x)
        if self.rope_tables is not None:
            cos_t, sin_t = self.rope_tables
            q = ops.rope(q, cos_t[:S], sin_t[:S], layout=rope_layout)
            k = ops.rope(k, cos_t[:S], sin_t[:S], layout=rope_layout)
        kv.store(k, v)
        return self._out(self._flash_attention(q, k, v, mask))

    def forward_decode(self, x: torch.Tensor, kv, step, window: Optional[int] = None,
                       rope_layout: str = "interleaved") -> torch.Tensor:
        """One new token per row, x [B, hidden]: its k and v go to cache position step.lens[b] - 1 (rotated there
        when RoPE is on), then its query attends over the row's first lens[b] cached keys (the last window + 1 of them
        with a sliding window), with the ALiBi bias when the module has it (kv.decode; step: the model-wide cache)."""
        q, k, v = (t.contiguous() for t in self._qkv(x))
        return self._out(kv.decode(q, k, v, step, self, window, rope_layout))

    def forward_extend(self, x: torch.Tensor, kv, chunk, window: Optional[int] = None,
                       rope_layout: str = "interleaved") -> torch.Tensor:
        """A chunk of new tokens per row, x [B, L, hidden] right-padded, appended at each row's current cache length
        (chunk: the llama.CacheChunk of the call).  Token i of row b sits at position p = chunk.start[b] + i: its q
        and k are rotated there (ops.rope at absolute positions), then kv.extend writes its k and v to the cache and
        its query attends over the row's cached keys up to p (max(0, p - window) .. p with a sliding window).  A
        chunk made for Model.verify (chunk.verify) goes through kv.verify instead."""
        q, k, v = self._qkv(x)
        if self.rope_tables is not None:
            cos_t, sin_t = self.rope_tables
            q = ops.rope(q, cos_t, sin_t, chunk.pos, rope_layout)
            k = ops.rope(k, cos_t, sin_t, chunk.pos, rope_layout)
        q, k, v = q.contiguous(), k.contiguous(), v.contiguous()
        attend = kv.verify if chunk.verify else kv.extend
        return self._out(attend(q, k, v, chunk, self, window))
