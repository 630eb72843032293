"""Chunked prefill and prompt caches, host side: argument checks and refusals (raised before any launch), chunk
scheduling for ragged rows, KVCache length bookkeeping, and self-tests of the cached-attention checker
(tests/cached_attn_check.py) against emulated faulty kernels."""
from __future__ import annotations

from types import SimpleNamespace

import pytest
import torch

from tests import attn_fwd_check as AF
from tests import cached_attn_check as CA


# -- scheduling -------------------------------------------------------------------------------------------------------
def test_prefill_chunks_ragged_rows():
    from mlx_cuda_distributed_pretraining_b200.core.generation import prefill_chunks
    prompts = [list(range(10)), list(range(3)), list(range(7))]
    chunks = prefill_chunks(prompts, 4)
    assert [[len(t) for t in c] for c in chunks] == [[4, 3, 4], [4, 0, 3], [2, 0, 0]]
    for b, p in enumerate(prompts):
        assert sum((c[b] for c in chunks), []) == p
    assert prefill_chunks(prompts, 100) == [prompts]
    assert [[len(t) for t in c] for c in prefill_chunks(prompts, 1)][9] == [1, 0, 0]


def test_cache_chunk_positions_and_indices():
    from mlx_cuda_distributed_pretraining_b200.arch.llama import CacheChunk
    c = CacheChunk([5, 0, 9], [3, 1, 0], 4, "cpu")
    assert c.start.tolist() == [5, 0, 9] and c.end.tolist() == [8, 1, 9] and c.max_end == 9
    assert c.rows.tolist() == [0, 0, 0, 1] and c.src.tolist() == [0, 1, 2, 0] and c.dst.tolist() == [5, 6, 7, 0]
    # padding tokens rotate at their row's last position, never past it
    assert c.pos.tolist() == [[5, 6, 7, 7], [0, 0, 0, 0], [8, 8, 8, 8]]
    assert c.pos.dtype == torch.int32


# -- KVCache bookkeeping ---------------------------------------------------------------------------------------------
def _cache(batch=2, s_max=512, positions=None, kv_bits=None):
    from mlx_cuda_distributed_pretraining_b200.arch.llama import KVCache
    c = KVCache.__new__(KVCache)
    c._layers, c._device, c._dtype, c._batch, c._heads = 2, torch.device("cpu"), torch.bfloat16, batch, (2, 64)
    c.s_max, c.kv_bits, c.kv_group_size, c.quantized_kv_start = s_max, kv_bits, 64, 0
    c.layers, c.quantized = None, False
    if positions:
        c._allocate(positions)
    c.lens = torch.zeros(batch, dtype=torch.int32)
    c.host_lens = [0] * batch
    return c


def test_kv_cache_layers_extend_truncate_and_grow():
    c = _cache()
    c.extend_lengths([3, 0])
    assert c.host_start == [0, 0] and c.host_lens == [3, 0] and c.lens.tolist() == [3, 0]
    assert c.layers[0].k.shape[1] == 256  # allocated on first use, rounded up to 256
    c.layers[1].k[0, :3] = 1.5
    c.layers[1].v[1, :2] = -2.0
    c.extend_lengths([300, 2])
    assert c.host_start == [3, 0] and c.host_lens == [303, 2]
    assert c.layers[0].k.shape[1] == 512 and c.layers[0].v.shape[1] == 512
    assert bool((c.layers[1].k[0, :3] == 1.5).all()) and bool((c.layers[1].v[1, :2] == -2.0).all()), \
        "growth keeps the cached positions"
    c.truncate([100, 2])
    assert c.host_lens == [100, 2] and c.lens.tolist() == [100, 2]
    layers = c.layers
    with pytest.raises(ValueError, match="truncate"):
        c.truncate([101, 2])
    with pytest.raises(ValueError, match="KV cache full"):
        c.extend_lengths([413, 0])
    with pytest.raises(ValueError, match="non-negative"):
        c.extend_lengths([1, -1])
    with pytest.raises(ValueError):
        c.extend_lengths([1])
    assert c.host_lens == [100, 2] and c.layers is layers, "a refused extend changes nothing"


# -- refusals ---------------------------------------------------------------------------------------------------------
def _model(dtype=torch.bfloat16, head_dim=64, prefix_lm=False):
    from mlx_cuda_distributed_pretraining_b200.arch.llama import Model
    attn = SimpleNamespace(head_dim=head_dim)
    m = SimpleNamespace(embed_tokens=SimpleNamespace(weight=torch.zeros(1, dtype=dtype)),
                           layers=[SimpleNamespace(self_attn=attn)],
                           args=SimpleNamespace(prefix_lm=prefix_lm, apply_rope=False, variant=None, alibi=False,
                                                max_position_embeddings=1024))
    m.check_extend = lambda cache, counts=None: Model.check_extend(m, cache, counts)
    return m


@pytest.mark.parametrize("kw,match", [
    (dict(dtype=torch.float32), "bf16"),
    (dict(head_dim=32), "head_dim 64 or 128"),
    (dict(head_dim=16), "head_dim 64 or 128"),
])
def test_check_extend_refuses(kw, match):
    from mlx_cuda_distributed_pretraining_b200.arch.llama import Model
    with pytest.raises(ValueError, match=match):
        Model.check_extend(_model(**kw), _cache())


def test_check_extend_refuses_split_prefix_lm_first_prompt():
    from mlx_cuda_distributed_pretraining_b200.arch.llama import Model
    c = _cache()
    with pytest.raises(ValueError, match="prefix-LM"):
        Model.check_extend(_model(prefix_lm=True), c, [3, 0])
    c.host_lens = [5, 0]
    Model.check_extend(_model(prefix_lm=True), c, [3, 0])   # a later turn is causal
    with pytest.raises(ValueError, match="prefix-LM"):
        Model.check_extend(_model(prefix_lm=True), c, [3, 1])


@pytest.mark.parametrize("step", [0, -1, 1.5, "4", True])
def test_generate_refuses_bad_step_sizes(step):
    from mlx_cuda_distributed_pretraining_b200.core.generation import generate
    with pytest.raises(ValueError, match="prefill_step_size"):
        generate(_model(), [[1, 2]], prefill_step_size=step)


def test_generate_refuses_bad_prompt_caches():
    from mlx_cuda_distributed_pretraining_b200.core.generation import generate
    with pytest.raises(ValueError, match="KVCache"):
        generate(_model(), [[1, 2]], prompt_cache=object())
    with pytest.raises(ValueError, match="conflicts"):
        generate(_model(), [[1, 2]], prompt_cache=_cache(batch=1), kv_bits=8)
    with pytest.raises(ValueError, match="holds 2 rows"):
        generate(_model(), [[1, 2]], prompt_cache=_cache(batch=2))
    c = _cache(batch=1, s_max=256)
    c.host_lens = [200]
    with pytest.raises(ValueError, match="256 positions"):
        generate(_model(), [[1] * 50], max_tokens=10, prompt_cache=c)
    c.host_lens = [1000]
    with pytest.raises(ValueError, match="max_position_embeddings"):
        generate(_model(), [[1] * 20], max_tokens=10, prompt_cache=c)


@pytest.mark.parametrize("kw,match", [
    (dict(dtype=torch.float32), "bf16"),
    (dict(head_dim=32), "head_dim"),
    (dict(prefix_lm=True), "prefix-LM"),
])
def test_generate_refuses_chunked_prefill_it_cannot_serve(kw, match):
    from mlx_cuda_distributed_pretraining_b200.core.generation import generate
    with pytest.raises(ValueError, match=match):
        generate(_model(**kw), [[1] * 10], prefill_step_size=4)


def test_cli_prefill_step_size_flag():
    from mlx_cuda_distributed_pretraining_b200.core.generation import parse_args
    assert parse_args(["--run", "r", "--prompt", "p"]).prefill_step_size is None
    assert parse_args(["--run", "r", "--prompt", "p", "--prefill-step-size", "512"]).prefill_step_size == 512
    with pytest.raises(SystemExit):
        parse_args(["--run", "r", "--prompt", "p", "--prefill-step-size", "0"])


def test_ops_wrappers_refuse_before_launch():
    from mlx_cuda_distributed_pretraining_b200 import ops
    q = torch.zeros(1, 4, 2, 64)
    with pytest.raises(ValueError, match="bf16"):
        ops.attention_cached(q, q, q, torch.zeros(1, dtype=torch.int32), torch.zeros(1, dtype=torch.int32))


# -- checker self-tests ------------------------------------------------------------------------------------------------
def _problem(seed=0):
    """Three rows of a 70-query chunk (valid 70, 33, 0) at positions 100, 5, 40 of an 8-head / 2-kv-head, D 64 cache;
    q padding and positions past each end NaN."""
    g = torch.Generator().manual_seed(seed)
    starts, ns, L, H, Hk, D = [100, 5, 40], [70, 33, 0], 70, 8, 2, 64
    s_max = max(s + n for s, n in zip(starts, ns)) + 130
    q = torch.randn(3, L, H, D, generator=g).to(torch.bfloat16)
    kc = torch.randn(3, s_max, Hk, D, generator=g).to(torch.bfloat16)
    vc = torch.randn(3, s_max, Hk, D, generator=g).to(torch.bfloat16)
    for b, (s, n) in enumerate(zip(starts, ns)):
        q[b, n:] = float("nan")
        kc[b, s + n:] = float("nan")
        vc[b, s + n:] = float("nan")
    return q, kc, vc, starts, ns


def _emulate(q, kc, vc, starts, ns, window, visible, keys_past_end=0, stale=None):
    """The kernel's arithmetic (AF.emulate_kernel) on each row's embedded problem over end + keys_past_end cache
    positions, under visible(S) [S, S]; stale replaces the cache past end (else it stays NaN).  Padding rows get
    zeros."""
    B, L, H, D = q.shape
    o = torch.zeros(B, L, H, D, dtype=torch.bfloat16)
    lse = torch.zeros(B, H, L)
    for b, (s, n) in enumerate(zip(starts, ns)):
        if n == 0:
            continue
        S = s + n + keys_past_end
        qf, k, v = CA.embed(q, kc, vc, b, s, n, keys=S)
        qf = torch.nan_to_num(qf)
        if stale is not None:
            k, v = k.clone(), v.clone()
            k[0, s + n:] = stale
            v[0, s + n:] = stale
        ob, lb = AF.emulate_kernel(qf, k, v, D ** -0.5, mask=visible(S))
        o[b, :n] = ob[0, s:s + n]
        lse[b, :, :n] = lb[0, :, s:s + n]
    return o, lse


def _causal(window):
    return lambda S: AF.visible(S, True, window=window)


def test_checker_accepts_the_kernel_arithmetic():
    q, kc, vc, starts, ns = _problem()
    for window in (-1, 20):
        o, lse = _emulate(q, kc, vc, starts, ns, window, _causal(None if window < 0 else window))
        assert CA.check_rows(q, kc, vc, starts, ns, o, lse, window, None, "exact") <= 1.0


def test_checker_rejects_query_seeing_next_key():
    q, kc, vc, starts, ns = _problem(1)
    one_ahead = lambda S: torch.ones(S, S, dtype=torch.bool).tril(1)  # noqa: E731
    o, lse = _emulate(q, kc, vc, starts, ns, -1, one_ahead, keys_past_end=1, stale=0.5)
    with pytest.raises(AssertionError):
        CA.check_rows(q, kc, vc, starts, ns, o, lse, -1, None, "p sees p + 1")


def test_checker_rejects_a_dropped_window_start():
    q, kc, vc, starts, ns = _problem(2)
    o, lse = _emulate(q, kc, vc, starts, ns, 20, _causal(None))
    with pytest.raises(AssertionError):
        CA.check_rows(q, kc, vc, starts, ns, o, lse, 20, None, "no window start")


def test_checker_rejects_ignoring_end():
    """A kernel that takes every row's keys through start + L (the padded chunk) instead of end[b]: the short row
    sees stale keys."""
    q, kc, vc, starts, ns = _problem(3)
    L = q.shape[1]

    def run():
        B, _, H, D = q.shape
        o = torch.zeros(B, L, q.shape[2], q.shape[3], dtype=torch.bfloat16)
        lse = torch.zeros(B, H, L)
        for b, (s, n) in enumerate(zip(starts, ns)):
            if n == 0:
                continue
            oo, ll = _emulate(q[b:b + 1], kc[b:b + 1], vc[b:b + 1], [s], [n], -1,
                              lambda S, n=n: AF.visible(S, True) | (torch.arange(S)[None, :] >= S - (L - n)),
                              keys_past_end=L - n, stale=0.25)
            o[b], lse[b] = oo[0], ll[0]
        return o, lse

    o, lse = run()
    with pytest.raises(AssertionError):
        CA.check_rows(q, kc, vc, starts, ns, o, lse, -1, None, "ignores end")


def test_checker_rejects_nan_past_end():
    """A kernel whose last key tile runs past end with the scores masked: P = 0 there, but 0 * NaN reaches O."""
    q, kc, vc, starts, ns = _problem(4)
    past = lambda S: AF.visible(S, True)  # noqa: E731  (keys past end masked, their NaN V loaded)
    o, lse = _emulate(q, kc, vc, starts, ns, -1, past, keys_past_end=128)
    with pytest.raises(AssertionError):
        CA.check_rows(q, kc, vc, starts, ns, o, lse, -1, None, "NaN past end")
