"""Each KV-cache format (arch.flash_attention DenseKV, QuantizedKV, RingKV, BeamKV) makes exactly the ops calls a
generation step makes on it, with the same arguments in the same order: ops is replaced by a recorder that binds
every call to the real wrapper's signature, and the formats are driven on CPU tensors with a stand-in attention
module.  The expected calls are written out as the wrappers' literal calls."""
from __future__ import annotations

import inspect
from types import SimpleNamespace

import pytest
import torch

from mlx_cuda_distributed_pretraining_b200 import ops as real_ops
from mlx_cuda_distributed_pretraining_b200.arch import flash_attention as fa

B, L, H, HK, D = 2, 3, 4, 2, 64
ATTN = object()  # the attention wrappers' result


def _bind(name, *args, **kwargs):
    b = inspect.signature(getattr(real_ops, name)).bind(*args, **kwargs)
    b.apply_defaults()
    return name, dict(b.arguments)


class _Recorder:
    """Stands in for ops: shape helpers pass through, every other wrapper is recorded (with the module's
    alibi_slopes() calls, which read the device) and returns ATTN, its `out`, or None."""

    def __init__(self):
        self.calls = []

    def __getattr__(self, name):
        if name == "kv_quant_shapes":
            return real_ops.kv_quant_shapes

        def record(*args, **kwargs):
            call = _bind(name, *args, **kwargs)
            self.calls.append(call)
            if name == "kv_dequantize":
                return call[1]["out"]
            return ATTN if name.startswith("attention") else None
        return record


def _same(a, b) -> bool:
    if isinstance(a, torch.Tensor) or isinstance(b, torch.Tensor):
        return a is b
    if isinstance(a, (tuple, list)) and isinstance(b, (tuple, list)):
        return len(a) == len(b) and all(_same(x, y) for x, y in zip(a, b))
    return a == b


def _assert_calls(got, want):
    assert [n for n, _ in got] == [n for n, _ in want]
    for (name, g), (_, w) in zip(got, want):
        assert g.keys() == w.keys(), name
        for key in w:
            assert _same(g[key], w[key]), f"{name}: argument {key}"


@pytest.fixture
def rec(monkeypatch):
    r = _Recorder()
    monkeypatch.setattr(fa, "ops", r)
    return r


def _attn(rec, rope=True):
    slopes = torch.ones(H)

    def alibi_slopes(device):
        rec.calls.append(("alibi_slopes", {"device": device}))
        return slopes

    tables = (torch.zeros(16, D // 2), torch.zeros(16, D // 2)) if rope else None
    return SimpleNamespace(scale=0.125, rope_tables=tables, alibi_slopes=alibi_slopes), slopes


def _decode_inputs():
    return torch.randn(B, H, D), torch.randn(B, HK, D), torch.randn(B, HK, D)


def _extend_inputs():
    return torch.randn(B, L, H, D).bfloat16(), torch.randn(B, L, HK, D).bfloat16(), torch.randn(B, L, HK, D).bfloat16()


def _chunk():
    from mlx_cuda_distributed_pretraining_b200.arch.llama import CacheChunk
    return CacheChunk([5, 0], [3, 1], L, "cpu")


def _step(**kw):
    return SimpleNamespace(lens=torch.tensor([7, 3], dtype=torch.int32), workspace=torch.empty(64, dtype=torch.uint8),
                           **kw)


def _dense(s=256):
    return fa.DenseKV(torch.ones(B, s, HK, D).bfloat16(), torch.ones(B, s, HK, D).bfloat16())


def _scattered(buf, chunk, src):
    """buf's chunk destinations hold src's chunk tokens and nothing else changed (buf was all ones)."""
    want = torch.ones_like(buf)
    want[chunk.rows, chunk.dst] = src[chunk.rows, chunk.src]
    return torch.equal(buf, want)


# -- DenseKV ---------------------------------------------------------------------------------------------------------
def test_dense_kv_calls(rec):
    attn, slopes = _attn(rec)
    kv, step = _dense(), _step()
    q, k, v = _decode_inputs()
    assert kv.decode(q, k, v, step, attn, 9, "half") is ATTN
    _assert_calls(rec.calls, [
        _bind("kv_append", q, k, v, kv.k, kv.v, step.lens, attn.rope_tables, layout="half"),
        ("alibi_slopes", {"device": q.device}),
        _bind("attention_decode", q, kv.k, kv.v, step.lens, 0.125, step.workspace, window=9, alibi=slopes),
    ])

    rec.calls.clear()
    kv, chunk = _dense(), _chunk()
    q, k, v = _extend_inputs()
    assert kv.extend(q, k, v, chunk, attn, None) is ATTN
    _assert_calls(rec.calls, [
        ("alibi_slopes", {"device": q.device}),
        _bind("attention_cached", q, kv.k, kv.v, chunk.start, chunk.end, 0.125, window=None, alibi=slopes),
    ])
    assert _scattered(kv.k, chunk, k) and _scattered(kv.v, chunk, v)

    rec.calls.clear()
    kv = _dense()
    kv.store(k, v)
    assert rec.calls == []
    assert torch.equal(kv.k[:, :L], k) and torch.equal(kv.v[:, :L], v) and bool((kv.k[:, L:] == 1).all())


# -- QuantizedKV -----------------------------------------------------------------------------------------------------
def _quant(bits=4, g=32, s=256):
    return fa.QuantizedKV(B, s, HK, D, bits, g, "cpu")


def test_quantized_kv_calls(rec):
    attn, slopes = _attn(rec, rope=False)
    kv, step = _quant(), _step()
    q, k, v = _decode_inputs()
    assert kv.decode(q, k, v, step, attn, None, "interleaved") is ATTN
    _assert_calls(rec.calls, [
        _bind("kv_append_quant", q, k, v, *kv.buffers(), step.lens, 4, 32, None, layout="interleaved"),
        ("alibi_slopes", {"device": q.device}),
        _bind("attention_decode_quant", q, *kv.buffers(), step.lens, 4, 32, 0.125, step.workspace, window=None,
              alibi=slopes),
    ])

    rec.calls.clear()
    q, k, v = _extend_inputs()
    kv.store(k, v)
    _assert_calls(rec.calls, [_bind("kv_quantize", k, v, *kv.buffers(), 4, 32)])

    rec.calls.clear()
    kv, chunk = _quant(bits=8, g=64), _chunk()
    for t in kv.buffers():
        t.fill_(1)
    assert kv.extend(q, k, v, chunk, attn, 20) is ATTN
    tmp = [rec.calls[0][1][n] for n in ("k_codes", "v_codes", "k_params", "v_params")]
    cshape, pshape = real_ops.kv_quant_shapes(B, L + L % 2, HK, D, 8, 64)  # the temporary: an even position count
    assert [tuple(t.shape) for t in tmp] == [cshape, cshape, pshape, pshape]
    assert chunk.scratch is not None and [tuple(t.shape) for t in chunk.scratch] == [(B, chunk.max_end, HK, D)] * 2
    assert all(t.dtype == torch.bfloat16 for t in chunk.scratch)
    k_att, v_att = chunk.scratch
    _assert_calls(rec.calls, [
        _bind("kv_quantize", k, v, *tmp, 8, 64),
        _bind("kv_dequantize", *kv.buffers(), chunk.end, 8, 64, out=chunk.scratch),
        ("alibi_slopes", {"device": q.device}),
        _bind("attention_cached", q, k_att, v_att, chunk.start, chunk.end, 0.125, window=20, alibi=slopes),
    ])
    # the chunk's valid tokens were copied from the temporary (zeros) into the cache, nothing else
    r, src, dst = chunk.rows, chunk.src, chunk.dst
    for t in kv.buffers()[:2]:
        assert int((t == 0).sum()) == len(r) * HK * t.shape[-1] and bool((t[r, dst] == 0).all())
    for t in kv.buffers()[2:]:
        assert int((t == 0).sum()) == len(r) * HK * t.shape[-2] * 2 and bool((t[r, :, dst] == 0).all())
    scratch = chunk.scratch
    kv.extend(q, k, v, chunk, attn, 20)
    assert chunk.scratch is scratch, "the call's scratch is made once, by its first layer"


def test_kv_cache_conversion_calls(rec):
    from mlx_cuda_distributed_pretraining_b200.arch.llama import KVCache
    c = KVCache.__new__(KVCache)
    c._layers, c._device, c._dtype, c._batch, c._heads = 2, torch.device("cpu"), torch.bfloat16, B, (HK, D)
    c.s_max, c.kv_bits, c.kv_group_size, c.quantized_kv_start = 256, 8, 64, 4
    c.layers, c.quantized = None, False
    c._allocate(256)
    dense = c.layers
    c.host_lens = [4, 3]
    c.maybe_quantize()
    assert rec.calls == [] and not c.quantized
    c.host_lens = [6, 3]
    c.maybe_quantize()
    assert c.quantized and c.layers is not dense
    _assert_calls(rec.calls, [_bind("kv_quantize", d.k, d.v, *qkv.buffers(), 8, 64, n=6)
                              for d, qkv in zip(dense, c.layers)])


# -- RingKV ----------------------------------------------------------------------------------------------------------
def test_ring_kv_calls(rec):
    attn, slopes = _attn(rec)
    kv = fa.RingKV(torch.ones(B, 256, HK, D).bfloat16(), torch.ones(B, 256, HK, D).bfloat16(), 64)
    step = _step(live=torch.tensor([1, 0], dtype=torch.int32))
    q, k, v = _decode_inputs()
    assert kv.decode(q, k, v, step, attn, None, "half") is ATTN
    _assert_calls(rec.calls, [
        _bind("kv_append_ring", q, k, v, kv.k, kv.v, step.lens, step.live, attn.rope_tables, "half"),
        ("alibi_slopes", {"device": q.device}),
        _bind("attention_decode_ring", q, kv.k, kv.v, step.lens, 64, 0.125, step.workspace, window=None,
              alibi=slopes),
    ])

    rec.calls.clear()
    from mlx_cuda_distributed_pretraining_b200.arch.llama import CacheChunk
    chunk = CacheChunk([254, 0], [3, 2], L, "cpu", slots=256)
    q, k, v = _extend_inputs()
    assert kv.extend(q, k, v, chunk, attn, 7) is ATTN
    _assert_calls(rec.calls, [
        ("alibi_slopes", {"device": q.device}),
        _bind("attention_ring", q, kv.k, kv.v, chunk.start, chunk.end, 64, 0.125, window=7, alibi=slopes),
    ])
    assert chunk.dst.tolist()[:3] == [254, 255, 4], "the chunk wraps past the sinks"
    assert _scattered(kv.k, chunk, k) and _scattered(kv.v, chunk, v)


# -- BeamKV ----------------------------------------------------------------------------------------------------------
def test_beam_kv_calls(rec):
    attn, slopes = _attn(rec)
    prefix = fa.DenseKV(torch.randn(2, 512, HK, D), torch.randn(2, 512, HK, D))
    t0, lens = [256, 0], [300, 40]
    kv = fa.BeamKV(prefix, 3, 256, t0, lens)
    assert kv.n_groups == 2 and tuple(kv.k_tail.shape) == (6, 256, HK, D) and kv.k_tail.dtype == prefix.k.dtype
    for g, slot in ((0, 0), (1, 3)):  # each prompt's positions past its fork point, in the group's first slot
        n = lens[g] - t0[g]
        assert torch.equal(kv.k_tail[slot, :n], prefix.k[g, t0[g]:lens[g]])
        assert torch.equal(kv.v_tail[slot, :n], prefix.v[g, t0[g]:lens[g]])
        assert bool((kv.k_tail[slot, n:] == 0).all())
    assert bool((kv.k_tail[[1, 2, 4, 5]] == 0).all())
    assert kv.nbytes() == 2 * 6 * 256 * HK * D * 4
    assert rec.calls == []

    step = _step(tables=torch.zeros(2 * B + 3 * 2, dtype=torch.int32))
    q, k, v = _decode_inputs()
    assert kv.decode(q, k, v, step, attn, 5, "interleaved") is ATTN
    _assert_calls(rec.calls, [
        _bind("kv_append_beam", q, k, v, kv.k_tail, kv.v_tail, step.lens, step.tables, 2, attn.rope_tables,
              "interleaved"),
        ("alibi_slopes", {"device": q.device}),
        _bind("attention_decode_beam", q, prefix.k, prefix.v, kv.k_tail, kv.v_tail, step.lens, step.tables, 0.125,
              step.workspace, window=5, alibi=slopes),
    ])
