"""fp64 / fp32 CPU oracle of the `model.misc.variant: mlx_lm` block (mlx_lm.models.llama as documented): the
reference oracle's RMSNorm and attention (oracle/reference_math.py) with mlx_lm's SiLU-gated MLP and half-split
RoPE.  Test infrastructure only; pinned against transformers' LlamaForCausalLM in tests/test_llama_variant_host.py."""
from __future__ import annotations

from typing import Dict, Optional

import torch

from oracle import reference_math as rm


def rope_half(x: torch.Tensor, theta: float = 10000.0, positions: Optional[torch.Tensor] = None) -> torch.Tensor:
    """x [B,S,NH,D]: for i < D/2 the pair (x[i], x[i + D/2]) rotated by pos * theta^(-2i/D), in x's dtype.
    positions: [S] or [B, S] (position within the document)."""
    B, S, NH, D = x.shape
    pos = torch.arange(S, dtype=x.dtype) if positions is None else positions.to(x.dtype)
    freqs = torch.pow(torch.tensor(float(theta), dtype=x.dtype), -torch.arange(0, D, 2, dtype=x.dtype) / D)
    ang = pos[..., None] * freqs                                   # [S, D/2] or [B, S, D/2]
    ang = ang[None, :, None, :] if ang.dim() == 2 else ang[:, :, None, :]
    cos, sin = torch.cos(ang), torch.sin(ang)
    x0, x1 = x[..., : D // 2], x[..., D // 2:]
    return torch.cat([x0 * cos - x1 * sin, x0 * sin + x1 * cos], dim=-1)


def rmsnorm(x: torch.Tensor, w: torch.Tensor, eps: float) -> torch.Tensor:
    """oracle rmsnorm's formula in x's own dtype (the reference oracle's upcasts to fp32 only)."""
    return x / torch.sqrt(torch.mean(x * x, dim=-1, keepdim=True) + eps) * w


def mlp_silu(x, w_gate, w_up, w_down):
    """mlx_lm.models.llama.MLP: down(silu(gate(x)) * up(x))."""
    lin = torch.nn.functional.linear
    return lin(torch.nn.functional.silu(lin(x, w_gate)) * lin(x, w_up), w_down)


def forward(params: Dict[str, torch.Tensor], tokens: torch.Tensor, d: rm.LlamaDims, mask: Optional[torch.Tensor] = None,
            positions: Optional[torch.Tensor] = None, traditional: bool = False) -> torch.Tensor:
    """tokens [B,S] -> logits [B,S,V] of the variant, on the trainer's flat parameter names.  mask: additive
    [1 or B, 1, S, S] (default causal); positions: RoPE positions [B, S] (packed rows), default 0..S-1."""
    lin = torch.nn.functional.linear
    B, S = tokens.shape
    h = params["embed_tokens.weight"][tokens]
    if mask is None:
        mask = rm.causal_mask(S, dtype=h.dtype)
    rot = (lambda t: rm.rope(t, d.rope_theta, positions)) if traditional else (
        lambda t: rope_half(t, d.rope_theta, positions))
    for i in range(d.num_layers):
        p = f"layers.{i}."
        x = rmsnorm(h, params[p + "input_layernorm.weight"], d.rms_norm_eps)
        q = lin(x, params[p + "self_attn.attn.q_proj.weight"]).reshape(B, S, d.num_heads, d.head_dim)
        k = lin(x, params[p + "self_attn.attn.k_proj.weight"]).reshape(B, S, d.num_kv_heads, d.head_dim)
        v = lin(x, params[p + "self_attn.attn.v_proj.weight"]).reshape(B, S, d.num_kv_heads, d.head_dim)
        ctx = rm.attention(rot(q), rot(k), v, d.head_dim ** -0.5, mask).reshape(B, S, d.num_heads * d.head_dim)
        h = h + lin(ctx, params[p + "self_attn.attn.o_proj.weight"])
        x = rmsnorm(h, params[p + "post_attention_layernorm.weight"], d.rms_norm_eps)
        h = h + mlp_silu(x, params[p + "mlp.gate_proj.weight"], params[p + "mlp.up_proj.weight"],
                         params[p + "mlp.down_proj.weight"])
    h = rmsnorm(h, params["norm.weight"], d.rms_norm_eps)
    return lin(h, params["embed_tokens.weight"] if d.tie_word_embeddings else params["lm_head.weight"])


def loss_and_grads(params, batch, d, pad_token, **kw):
    leaves = {k: v.detach().clone().requires_grad_(True) for k, v in params.items()}
    logits = forward(leaves, batch[:, :-1], d, **kw)
    loss, ntoks = rm.compute_loss(logits, batch[:, 1:], pad_token)
    loss.backward()
    return loss.detach(), int(ntoks), {k: v.grad for k, v in leaves.items()}
