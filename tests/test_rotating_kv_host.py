"""The rotating KV cache (max_kv_size), host side: the slot map and the visibility rule, chunk destinations,
refusals raised before anything is allocated, the CLI flag, and self-tests of tests/rotating_kv_check.py against
emulated faulty kernels."""
from __future__ import annotations

import itertools
from types import SimpleNamespace

import pytest
import torch

from mlx_cuda_distributed_pretraining_b200.ops import ring_slot
from tests import rotating_kv_check as RK


# -- slot map and rule ------------------------------------------------------------------------------------------------
def test_slot_map():
    assert [ring_slot(t, 10) for t in range(16)] == [0, 1, 2, 3, 4, 5, 6, 7, 8, 9, 4, 5, 6, 7, 8, 9]
    t = torch.arange(40)
    assert ring_slot(t, 12).tolist() == [ring_slot(int(x), 12) for x in t]


@pytest.mark.parametrize("M", [5, 6, 9, 64])
def test_decoded_token_sees_sinks_and_recent(M):
    for n in range(M - 1, M + 40):
        seen = torch.nonzero(RK.rule(torch.tensor(n), torch.arange(n + 1), M)).flatten().tolist()
        assert seen == list(range(4)) + list(range(n - M + 5, n + 1)) and len(seen) == M


def _ring_holds(M, C, L, start, n):
    """Write a chunk of n keys from `start` into a ring of C slots (positions written so far: all before start), and
    return whether every key a query of the chunk sees still sits in its slot."""
    owner = {}
    for t in range(start + n):
        owner[ring_slot(t, C)] = t
    for q in range(start, start + n):
        for k in range(q + 1):
            if bool(RK.rule(torch.tensor(q), torch.tensor(k), M)) and owner[ring_slot(k, C)] != k:
                return False
    return True


def test_ring_of_m_plus_l_minus_1_slots_keeps_every_visible_key():
    # with each chunk of <= L keys written before it attends, a ring of C = M + L - 1 slots still holds every key a
    # query of the chunk sees, wherever the chunk starts
    for M, L in itertools.product([5, 6, 9], [1, 2, 3, 5]):
        C = M + L - 1
        for start in range(0, 3 * C):
            for n in range(1, L + 1):
                assert _ring_holds(M, C, L, start, n), (M, L, C, start, n)


def test_ring_one_slot_short_overwrites_a_visible_key():
    found = False
    for M, L in itertools.product([5, 6, 9], [2, 3, 5]):
        C = M + L - 2
        found |= any(not _ring_holds(M, C, L, start, L) for start in range(0, 3 * C))
    assert found


def test_cache_chunk_destinations_are_ring_slots():
    from mlx_cuda_distributed_pretraining_b200.arch.llama import CacheChunk
    c = CacheChunk([2, 300], [4, 3], 4, "cpu", slots=256)
    assert c.dst.tolist() == [2, 3, 4, 5, ring_slot(300, 256), ring_slot(301, 256), ring_slot(302, 256)]
    assert c.start.tolist() == [2, 300] and c.end.tolist() == [6, 303]
    assert c.pos.tolist()[1] == [300, 301, 302, 302], "rotation stays on true positions"


# -- refusals ---------------------------------------------------------------------------------------------------------
def _model(**kw):
    args = SimpleNamespace(prefix_lm=False, alibi=False, apply_rope=False, variant="default",
                           max_position_embeddings=4096, sliding_window=None, num_hidden_layers=1)
    args.__dict__.update(kw.pop("args", {}))
    dtype = kw.pop("dtype", torch.bfloat16)
    head_dim = kw.pop("head_dim", 64)
    attn = SimpleNamespace(num_kv_heads=2, head_dim=head_dim, num_heads=4)

    def check_extend(cache, counts=None):
        from mlx_cuda_distributed_pretraining_b200.arch.llama import Model
        Model.check_extend(m, cache, counts)

    m = SimpleNamespace(args=args, layers=[SimpleNamespace(self_attn=attn)],
                        embed_tokens=SimpleNamespace(weight=torch.zeros(1, dtype=dtype)), check_extend=check_extend)
    return m


@pytest.mark.parametrize("bad", [4, 0, -3, True, 5.0, "8"])
def test_max_kv_size_refused(bad):
    from mlx_cuda_distributed_pretraining_b200.arch.llama import KVCache
    from mlx_cuda_distributed_pretraining_b200.core.generation import generate
    with pytest.raises(ValueError, match="max_kv_size"):
        KVCache(_model(), 2, 64, max_kv_size=bad)
    with pytest.raises(ValueError, match="max_kv_size"):
        generate(_model(), [[1, 2]], max_tokens=2, max_kv_size=bad)


@pytest.mark.parametrize("case,match", [
    (dict(kv_bits=8), "kv_bits"),
    (dict(args=dict(prefix_lm=True)), "prefix-LM"),
    (dict(dtype=torch.float32), "bf16"),
    (dict(head_dim=32), "head_dim"),
])
def test_rotating_cache_refusals(case, match):
    from mlx_cuda_distributed_pretraining_b200.arch.llama import KVCache
    from mlx_cuda_distributed_pretraining_b200.core.generation import generate
    kv_bits = case.pop("kv_bits", None)
    m = _model(**case)
    with pytest.raises(ValueError, match=match):
        KVCache(m, 2, 64, kv_bits=kv_bits, max_kv_size=64)
    with pytest.raises(ValueError, match=match):
        generate(m, [[1, 2]], max_tokens=2, kv_bits=kv_bits, max_kv_size=64)


def _ring_cache(max_kv_size=64, max_chunk=128):
    from mlx_cuda_distributed_pretraining_b200.arch.llama import KVCache
    c = KVCache.__new__(KVCache)
    c._layers, c._device, c._dtype, c._batch, c._heads = 1, torch.device("cpu"), torch.bfloat16, 2, (2, 64)
    c.kv_bits, c.quantized, c.max_kv_size, c.max_chunk = None, False, max_kv_size, max_chunk
    c.s_max = -(-(max_kv_size + max_chunk - 1) // 256) * 256
    c._allocate(c.s_max)
    c.lens = torch.zeros(2, dtype=torch.int32)
    c.host_lens, c.live = [0, 0], None
    return c


def test_ring_cache_layers_bookkeeping_and_refusals():
    c = _ring_cache()
    nbytes = c.nbytes()
    assert nbytes == 2 * 2 * 256 * 2 * 64 * 2
    rings = [c.layer(0).k, c.layer(0).v]
    for _ in range(5):
        c.extend_lengths([128, 100])  # rows grow past the ring's slots
    assert c.host_lens == [640, 500] and c.nbytes() == nbytes
    assert c.layer(0).k is rings[0] and c.layer(0).v is rings[1], "the ring is never reallocated"
    with pytest.raises(ValueError, match="max_chunk"):
        c.extend_lengths([129, 0])
    with pytest.raises(ValueError, match="truncated"):
        c.truncate([10, 10])
    with pytest.raises(ValueError, match="Model.extend"):
        c.set_lengths([3, 3])
    c.advance([True, False])
    assert c.host_lens == [641, 500] and c.lens.tolist() == [641, 500] and c.live.tolist() == [1, 0]
    c.advance()
    assert c.host_lens == [642, 501] and c.live is None


def test_generate_refuses_mismatched_prompt_cache():
    from mlx_cuda_distributed_pretraining_b200.arch import llama
    from mlx_cuda_distributed_pretraining_b200.core.generation import generate
    c = _ring_cache()
    c.__class__ = llama.KVCache
    with pytest.raises(ValueError, match="max_kv_size"):
        generate(_model(), [[1], [2]], max_tokens=2, prompt_cache=c, max_kv_size=32)
    with pytest.raises(ValueError, match="max_chunk"):
        generate(_model(), [[1], [2]], max_tokens=2, prompt_cache=c, prefill_step_size=129)


def test_cli_flag_parses():
    from mlx_cuda_distributed_pretraining_b200.core.generation import parse_args
    assert parse_args(["--run", "r", "--prompt", "p", "--max-kv-size", "64"]).max_kv_size == 64
    assert parse_args(["--run", "r", "--prompt", "p"]).max_kv_size is None
    with pytest.raises(SystemExit):
        parse_args(["--run", "r", "--prompt", "p", "--max-kv-size", "4"])


# -- checker self-tests -----------------------------------------------------------------------------------------------
def _inputs(alibi=False, seed=0):
    g = torch.Generator().manual_seed(seed)
    B, L, H, Hk, D, M, C = 2, 6, 4, 2, 64, 12, 20
    starts, ends = [30, 9], [36, 12]
    q = torch.randn(B, L, H, D, generator=g).to(torch.bfloat16)
    k = torch.randn(B, C, Hk, D, generator=g).to(torch.bfloat16)
    v = torch.randn(B, C, Hk, D, generator=g).to(torch.bfloat16)
    k[1, 12:] = float("nan")  # row 1 has never written slots 12..: stale
    v[1, 12:] = float("nan")
    slopes = torch.tensor([0.5, 0.25, 0.125, 0.0625]) if alibi else None
    return q, k, v, starts, ends, M, slopes


@pytest.mark.parametrize("alibi", [False, True])
@pytest.mark.parametrize("window", [None, 7])
def test_checker_accepts_the_rule(alibi, window):
    q, k, v, starts, ends, M, slopes = _inputs(alibi)
    o, lse = RK.emulate(q, k, v, starts, ends, M, window, slopes)
    RK.check_rows(q, k, v, starts, ends, o, lse, M, window, slopes, "emulated")


@pytest.mark.parametrize("fault,alibi,window", [("no_sinks", False, None), ("slot_positions", True, None),
                                               ("slot_positions", False, 20), ("stale", False, None),
                                               ("one_more", False, None)])
def test_checker_rejects_faulty_kernels(fault, alibi, window):
    q, k, v, starts, ends, M, slopes = _inputs(alibi)
    if fault == "stale":  # a stale but finite slot in row 0
        k[0, ring_slot(36, 20)] = 3.0
    o, lse = RK.emulate(q, k, v, starts, ends, M, window, slopes, fault=fault)
    with pytest.raises(AssertionError):
        RK.check_rows(q, k, v, starts, ends, o, lse, M, window, slopes, fault)
