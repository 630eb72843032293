"""CPU oracle of the quantized KV cache format (DESIGN §4.2.1), in torch fp32 on the CPU.

Each group of g consecutive elements of a head vector is stored as x ~ s q + b: n = 2^bits - 1, mn / mx the group's
extremes, s = max((mx - mn) / n, 1e-7), b = mn (a -0 minimum stored as +0), q = min(n, rint((x - b) / s)) with IEEE
division and round-half-to-even.  Codes are uint8 [..., D * bits / 8] (4 bits: element 2j in the low nibble of byte
j); parameters [..., D / g, 2] hold (s, b)."""
from __future__ import annotations

import torch


def quantize(x: torch.Tensor, bits: int, group_size: int):
    """x [..., D] (any float dtype; its fp32 value is quantized) -> (codes int64 [..., D], s fp32 [..., D / g],
    b fp32 [..., D / g])."""
    n = (1 << bits) - 1
    xf = x.float()
    grp = xf.reshape(*xf.shape[:-1], xf.shape[-1] // group_size, group_size)
    mn = grp.amin(-1)
    mx = grp.amax(-1)
    s = torch.maximum((mx - mn) / n, torch.tensor(1e-7, dtype=torch.float32))
    b = mn + 0.0
    q = torch.clamp(torch.round((grp - b[..., None]) / s[..., None]), max=n)
    return q.to(torch.int64).reshape(xf.shape), s, b


def dequantize(codes: torch.Tensor, s: torch.Tensor, b: torch.Tensor, group_size: int) -> torch.Tensor:
    """s q + b in fp32, [..., D]."""
    grp = codes.float().reshape(*codes.shape[:-1], codes.shape[-1] // group_size, group_size)
    return (s[..., None] * grp + b[..., None]).reshape(codes.shape)


def pack(codes: torch.Tensor, bits: int) -> torch.Tensor:
    """codes [..., D] -> uint8 [..., D * bits / 8]."""
    if bits == 8:
        return codes.to(torch.uint8)
    return (codes[..., 0::2] | (codes[..., 1::2] << 4)).to(torch.uint8)


def unpack(packed: torch.Tensor, bits: int) -> torch.Tensor:
    """uint8 [..., D * bits / 8] -> int64 codes [..., D]."""
    p = packed.to(torch.int64)
    if bits == 8:
        return p
    return torch.stack((p & 0xF, p >> 4), dim=-1).reshape(*p.shape[:-1], 2 * p.shape[-1])


def cache_layout(x: torch.Tensor, bits: int, group_size: int):
    """x [B, S, Hk, D] -> (codes uint8 [B, S, Hk, D * bits / 8], params fp32 [B, Hk, S, D / g, 2]) as the kernels
    lay them out."""
    q, s, b = quantize(x, bits, group_size)
    params = torch.stack((s, b), dim=-1).permute(0, 2, 1, 3, 4).contiguous()
    return pack(q, bits), params


def dequantize_cache(codes: torch.Tensor, params: torch.Tensor, bits: int, group_size: int) -> torch.Tensor:
    """The inverse view of cache_layout: [B, S, Hk, D] fp32 values s q + b."""
    p = params.permute(0, 2, 1, 3, 4)
    return dequantize(unpack(codes, bits), p[..., 0], p[..., 1], group_size)
