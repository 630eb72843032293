"""Quantized KV cache, host side: the CPU oracle's properties, the wrappers' rejections (raised before any launch),
the CLI flags and generate()'s argument checks."""
from __future__ import annotations

from types import SimpleNamespace

import pytest
import torch

from tests import kv_quant_oracle as KQ


@pytest.mark.parametrize("bits", [4, 8])
@pytest.mark.parametrize("g", [32, 64, 128])
def test_error_bound_and_code_range(bits, g):
    gen = torch.Generator().manual_seed(bits * 1000 + g)
    x = (torch.randn(64, 128, generator=gen) * torch.rand(64, 1, generator=gen) * 10).to(torch.bfloat16)
    q, s, b = KQ.quantize(x, bits, g)
    assert int(q.min()) >= 0 and int(q.max()) <= (1 << bits) - 1
    xr = KQ.dequantize(q, s, b, g)
    err = (x.double() - xr.double()).abs().reshape(64, 128 // g, g)
    # |x - (s q + b)| <= s / 2, up to the fp32 roundings: (x - b) / s (relative 2^-24 of a quotient up to n, which can
    # move a near-tie to the other code) and s q + b (2^-24 of each term)
    n = (1 << bits) - 1
    mag = x.double().abs().reshape(64, 128 // g, g) + b.double().abs()[..., None]
    bound = s.double()[..., None] / 2 * (1 + n * 2 ** -21) + mag * 2 ** -23
    assert bool((err <= bound).all())
    # the group's extremes: the minimum is exact, the maximum code is n
    assert bool((KQ.quantize(x, bits, g)[0].reshape(64, -1, g).amax(-1) == (1 << bits) - 1).all())


def test_constant_group_and_signed_zero():
    x = torch.full((1, 64), 3.25)
    q, s, b = KQ.quantize(x, 8, 64)
    assert bool((q == 0).all()) and float(s) == pytest.approx(1e-7) and float(b) == 3.25
    assert bool((KQ.dequantize(q, s, b, 64) == 3.25).all())
    z = torch.zeros(1, 64)
    z[0, ::2] = -0.0
    q, s, b = KQ.quantize(z, 4, 64)
    assert bool((q == 0).all())
    assert not torch.signbit(b).any(), "a -0 minimum is stored as +0"


def test_round_half_to_even_ties():
    # mn = 0, mx = 15 * 0.5 gives s = 0.5 exactly at 4 bits; x = 0.25 (q = 0.5) and 0.75 (1.5) are exact ties
    x = torch.zeros(1, 32)
    x[0, 1] = 7.5
    x[0, 2] = 0.25
    x[0, 3] = 0.75
    x[0, 4] = 1.25
    q, s, b = KQ.quantize(x, 4, 32)
    assert float(s) == 0.5 and float(b) == 0.0
    assert q[0, :5].tolist() == [0, 15, 0, 2, 2]


def test_nibble_order_and_layout():
    codes = torch.arange(16, dtype=torch.int64).repeat(2)[None]  # [1, 32]
    packed = KQ.pack(codes, 4)
    assert packed.shape == (1, 16)
    assert packed[0, 0].item() == 0x10 and packed[0, 1].item() == 0x32  # element 2j low nibble, 2j + 1 high
    assert torch.equal(KQ.unpack(packed, 4), codes)
    x = torch.randn(2, 5, 3, 64)
    c, p = KQ.cache_layout(x, 8, 32)
    assert c.shape == (2, 5, 3, 64) and p.shape == (2, 3, 5, 2, 2)
    assert (KQ.dequantize_cache(c, p, 8, 32) - x).abs().max() <= p[..., 0].max() / 2 * 1.001


# -- wrapper rejections: raised before any launch, so they run on CPU tensors --------------------------------------
def _bufs(B=2, s_max=64, Hk=2, D=64, bits=8, g=64):
    from mlx_cuda_distributed_pretraining_b200 import ops
    cs, ps = ops.kv_quant_shapes(B, s_max, Hk, D, bits, g)
    return (torch.zeros(cs, dtype=torch.uint8), torch.zeros(cs, dtype=torch.uint8), torch.zeros(ps),
            torch.zeros(ps))


@pytest.mark.parametrize("bits,g,D,match", [(3, 64, 64, "kv_bits"), (8, 48, 64, "kv_group_size"),
                                            (8, 32, 16, "head_dim"), (4, 128, 64, "head_dim")])
def test_wrappers_reject_bad_format(bits, g, D, match):
    from mlx_cuda_distributed_pretraining_b200 import ops
    q = torch.zeros(2, 4, D, dtype=torch.bfloat16)
    k = torch.zeros(2, 2, D, dtype=torch.bfloat16)
    lens = torch.ones(2, dtype=torch.int32)
    bufs = _bufs(D=64)
    with pytest.raises(ValueError, match=match):
        ops.attention_decode_quant(q, *bufs, lens, bits, g)
    with pytest.raises(ValueError, match=match):
        ops.kv_append_quant(q, k, k, *bufs, lens, bits, g)
    with pytest.raises(ValueError, match=match):
        ops.kv_quantize(k[:, None].expand(2, 8, 2, D).contiguous(), k[:, None].expand(2, 8, 2, D).contiguous(),
                        *bufs, bits, g)


def test_wrappers_reject_mismatched_shapes_and_dtypes():
    from mlx_cuda_distributed_pretraining_b200 import ops
    q = torch.zeros(2, 4, 64, dtype=torch.bfloat16)
    k = torch.zeros(2, 2, 64, dtype=torch.bfloat16)
    lens = torch.ones(2, dtype=torch.int32)
    kc, vc, kp, vp = _bufs()
    with pytest.raises(ValueError, match="v_codes"):
        ops.attention_decode_quant(q, kc, vc[:, :32], kp, vp, lens, 8, 64)
    with pytest.raises(ValueError, match="k_params"):
        ops.attention_decode_quant(q, kc, vc, kp.double(), vp, lens, 8, 64)
    with pytest.raises(ValueError, match="k_codes"):
        ops.attention_decode_quant(q, kc, vc, kp, vp, lens, 4, 64)  # 8-bit buffers given as 4-bit
    with pytest.raises(ValueError, match="v_params"):
        ops.attention_decode_quant(q, kc, vc, kp, vp[..., :1], lens, 8, 64)
    with pytest.raises(ValueError, match="k, v"):
        ops.kv_append_quant(q, k, k[:, :1], kc, vc, kp, vp, lens, 8, 64)
    with pytest.raises(ValueError, match="v must be"):
        ops.kv_append_quant(q, k, k.float(), kc, vc, kp, vp, lens, 8, 64)
    src = torch.zeros(2, 8, 2, 64, dtype=torch.bfloat16)
    with pytest.raises(ValueError, match="one dtype"):
        ops.kv_quantize(src, src.float(), kc, vc, kp, vp, 8, 64)
    with pytest.raises(ValueError, match="unsupported dtype"):
        ops.kv_quantize(src.half(), src.half(), kc, vc, kp, vp, 8, 64)
    with pytest.raises(ValueError, match="k_codes"):
        ops.kv_quantize(torch.zeros(3, 8, 2, 64), torch.zeros(3, 8, 2, 64), kc, vc, kp, vp, 8, 64)


# -- CLI and generate() --------------------------------------------------------------------------------------------
def test_cli_kv_flags():
    from mlx_cuda_distributed_pretraining_b200.core.generation import parse_args
    a = parse_args(["--run", "r", "--prompt", "p"])
    assert (a.kv_bits, a.kv_group_size, a.quantized_kv_start) == (None, 64, 0)
    a = parse_args(["--run", "r", "--prompt", "p", "--kv-bits", "4", "--kv-group-size", "32",
                    "--quantized-kv-start", "100"])
    assert (a.kv_bits, a.kv_group_size, a.quantized_kv_start) == (4, 32, 100)
    for bad in (["--kv-bits", "3"], ["--kv-group-size", "48"], ["--quantized-kv-start", "-1"]):
        with pytest.raises(SystemExit):
            parse_args(["--run", "r", "--prompt", "p"] + bad)


class _NoDevice:
    """A model stand-in that fails on any attribute generate() would touch after its argument checks."""

    def __getattr__(self, name):
        raise AssertionError(f"generate() touched model.{name} before rejecting its arguments")


@pytest.mark.parametrize("kw,match", [(dict(kv_bits=3), "kv_bits"), (dict(kv_bits=2), "kv_bits"),
                                      (dict(kv_bits=8, kv_group_size=16), "kv_group_size"),
                                      (dict(kv_bits=4, quantized_kv_start=-1), "quantized_kv_start")])
def test_generate_rejects_bad_kv_arguments_before_the_device(kw, match):
    from mlx_cuda_distributed_pretraining_b200.core.generation import generate
    with pytest.raises(ValueError, match=match):
        generate(_NoDevice(), [[1, 2, 3]], max_tokens=4, **kw)


def test_kv_cache_refuses_head_dim_16():
    from mlx_cuda_distributed_pretraining_b200.arch.llama import KVCache
    attn = SimpleNamespace(head_dim=16, num_kv_heads=8, num_heads=8)
    model = SimpleNamespace(args=SimpleNamespace(num_hidden_layers=1), layers=[SimpleNamespace(self_attn=attn)])
    with pytest.raises(ValueError, match="head_dim in \\(32, 64, 128\\)"):
        KVCache(model, 1, 64, kv_bits=8)
