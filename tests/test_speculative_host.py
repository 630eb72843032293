"""Speculative decoding without a GPU: the accept / rewind / next-draft-input step against a literal restatement of
mlx_lm's speculative_generate_step loop, the exact output distribution of the procedure against plain sampling on
tiny table models, self-tests of the multi-query attention checker, and the refusals of generate and the CLI."""
from __future__ import annotations

import itertools
from functools import lru_cache
from types import SimpleNamespace

import pytest
import torch

from mlx_cuda_distributed_pretraining_b200.core import generation as G
from tests import multi_decode_check as MC


# -- the accept step against mlx_lm's loop --------------------------------------------------------------------------
def mlx_round(drafted, sampled, base, draft_base, ntoks, max_tokens, eos):
    """mlx_lm's round, restated: yield accepted drafts while t_n == d_n (stopping at max_tokens), then t_n; the caller
    stops at EOS.  Rewind the target by num_draft - n and the draft by max(num_draft - n - 1, 0); the draft's next
    input is [d_k, t_n] when every draft was accepted.  Returns (yielded, stopped, target len, draft len, next)."""
    num_draft = len(drafted)
    out, n = [], 0
    while n < num_draft:
        if sampled[n] != drafted[n]:
            break
        n += 1
        ntoks += 1
        out.append(drafted[n - 1])
        if ntoks == max_tokens:
            break
    if ntoks < max_tokens:
        ntoks += 1
        out.append(sampled[n])
    stopped = ntoks == max_tokens
    if eos in out:
        out, stopped = out[:out.index(eos) + 1], True
    target_len = base + num_draft + 1 - (num_draft - n)
    draft_len = draft_base + num_draft - max(num_draft - n - 1, 0)
    nxt = [sampled[n]] if n < num_draft else [drafted[-1], sampled[n]]
    return out, stopped, target_len, draft_len, nxt


CASES = [  # drafted, target samples, tokens emitted before, max_tokens, eos
    ([4, 5, 6], [9, 5, 6, 1], 1, 20, None),        # first-token mismatch
    ([4, 5, 6], [4, 5, 6, 1], 1, 20, None),        # all accepted: two-token catch-up
    ([4, 5, 6], [4, 5, 0, 1], 3, 20, None),        # mismatch at the last draft
    ([4, 2, 6], [4, 2, 6, 1], 1, 20, 2),           # EOS inside the accepted drafts
    ([4, 5, 6], [4, 5, 2, 1], 1, 20, 2),           # EOS as the target's token
    ([4, 5, 6], [4, 5, 6, 1], 2, 4, None),         # max_tokens ends mid-round (k = 2 of K = 3 is the caller's)
    ([4, 5], [4, 5, 1], 2, 4, None),               # k = max_tokens - emitted: bonus cut
    ([4], [4, 7], 9, 10, None),                    # last token of the budget
]


@pytest.mark.parametrize("drafted,sampled,before,max_tokens,eos", CASES)
def test_accept_and_rewind_match_mlx_lm_loop(drafted, sampled, before, max_tokens, eos):
    base = 50 + before - 1
    k = len(drafted)
    ref = mlx_round(drafted, sampled, base, base, before, max_tokens, eos)
    emitted, n, stopped = G.accept_drafts(drafted, sampled, max_tokens - before, eos)
    assert (emitted, stopped) == (ref[0], ref[1])
    if not stopped:
        assert G.rewind(base, k, emitted, drafted) == ref[2:]


def test_draft_counts_and_finished_rows():
    assert G.draft_counts([1, 5, 9, 3], [False, False, False, True], 3, 10) == [3, 3, 1, 0]
    assert G.draft_counts([2], [False], 15, 2) == [0]
    assert G.draft_counts([1, 1], [True, True], 3, 10) == [0, 0]


def test_repetition_windows_follow_the_drafts():
    assert G.repetition_windows([1, 2, 3], [4, 5], 2) == [[1, 2], [2, 3], [3, 4]]
    assert G.repetition_windows([7], [8], 5) == [[], [7]]


# -- exact distribution on table models -----------------------------------------------------------------------------
V = 5


def _table(seed):
    g = torch.Generator().manual_seed(seed)
    return torch.randn(V, V, V, generator=g, dtype=torch.float64) * 1.5   # logits from the last two tokens


T_TARGET, T_DRAFT = _table(1), _table(2)


def _dist(table, seq, sampler):
    temp, min_p, top_p, pen, ctx = sampler
    lg = table[seq[-2], seq[-1]][None].clone()
    if pen != 1.0 and ctx > 0:
        lg = G.apply_repetition_penalty(lg, [G.repetition_window(seq, ctx)], pen)
    return G.token_probs(lg, temp, min_p, top_p)[0].tolist()


def _plain(prompt, n, sampler):
    dist = lru_cache(None)(lambda s: _dist(T_TARGET, list(s), sampler))
    out = {}
    for toks in itertools.product(range(V), repeat=n):
        p, seq = 1.0, list(prompt)
        for t in toks:
            p *= dist(tuple(seq))[t]
            seq.append(t)
        out[toks] = p
    return out


def _speculative(prompt, n, K, sampler):
    td = lru_cache(None)(lambda s: _dist(T_TARGET, list(s), sampler))
    dd = lru_cache(None)(lambda s: _dist(T_DRAFT, list(s), sampler))
    out = {}

    def rounds(seq, emitted, p):
        if len(emitted) == n:
            out[tuple(emitted)] = out.get(tuple(emitted), 0.0) + p
            return
        k = G.draft_counts([len(emitted)], [False], K, n)[0]
        for drafted in itertools.product(range(V), repeat=k):
            pd = 1.0
            for j, d in enumerate(drafted):
                pd *= dd(tuple(seq + list(drafted[:j])))[d]
            if pd == 0.0:
                continue
            for sampled in itertools.product(range(V), repeat=k + 1):
                pt = 1.0
                for i, t in enumerate(sampled):
                    pt *= td(tuple(seq + list(drafted[:i])))[t]
                if pt == 0.0:
                    continue
                e, _, _ = G.accept_drafts(list(drafted), list(sampled), n - len(emitted))
                rounds(seq + e, emitted + e, p * pd * pt)

    first = td(tuple(prompt))
    for t in range(V):
        rounds(list(prompt) + [t], [t], first[t])
    return out


@pytest.mark.parametrize("sampler", [(0.8, None, None, 1.0, 0), (1.0, 0.2, None, 1.3, 2), (0.7, None, 0.8, 1.3, 3),
                                     (1.2, None, None, 1.5, 1)], ids=["temp", "min_p+pen", "top_p+pen", "temp+pen"])
def test_speculative_distribution_is_plain(sampler):
    prompt = [0, 3]
    plain = _plain(prompt, 3, sampler)
    spec = _speculative(prompt, 3, 2, sampler)
    assert abs(sum(spec.values()) - 1.0) < 1e-12
    for toks, p in plain.items():
        assert abs(spec.get(toks, 0.0) - p) < 1e-12, toks


# -- checker self-tests ---------------------------------------------------------------------------------------------
def _problem():
    g = torch.Generator().manual_seed(0)
    starts, counts = [250, 3, 500], [9, 4, 0]
    ends = [s + n for s, n in zip(starts, counts)]
    q = torch.randn(3, 9, 4, 16, generator=g)
    kc = torch.randn(3, 520, 2, 16, generator=g)
    vc = torch.randn(3, 520, 2, 16, generator=g)
    return q, kc, vc, starts, ends


def _as_kernel(ref, B, L, H, D):
    o = torch.full((B, L, H, D), float("nan"), dtype=torch.float64)
    lse = torch.full((B, H, L), float("nan"), dtype=torch.float64)
    for (b, i), (R, _, l) in ref.items():
        o[b, i], lse[b, :, i] = R, l
    return o, lse


@pytest.mark.parametrize("broken", [None, "sees_next", "window_off_by_one", "straddle", "alibi_at_chunk"])
def test_checker_rejects_broken_references(broken):
    from mlx_cuda_distributed_pretraining_b200.arch.flash_attention import alibi_slopes
    q, kc, vc, starts, ends = _problem()
    window, slopes = 100, alibi_slopes(4)
    rule, bias = MC.visible, None
    if broken == "sees_next":
        rule = lambda p, n, W, dev: MC.visible(p + 1, n, W + 1, dev)  # noqa: E731
    elif broken == "window_off_by_one":
        rule = lambda p, n, W, dev: MC.visible(p, n, W + 1, dev)  # noqa: E731
    elif broken == "straddle":   # a query below a 256 boundary also takes the next chunk's keys up to the row's end
        def rule(p, n, W, dev):
            ok = MC.visible(p, n, W, dev)
            row_end = next(e for s, e in zip(starts, ends) if s <= p < e)
            k = torch.arange(n)
            return ok | ((k >= (p // 256 + 1) * 256) & (k < row_end))
    elif broken == "alibi_at_chunk":
        bias = lambda b, i, p: (p // 256) * 256  # noqa: E731
    kern = MC.reference(q, kc, vc, starts, ends, window, slopes, rule=rule, bias_pos=bias)
    o, lse = _as_kernel(kern, *q.shape)
    ref = MC.reference(q, kc, vc, starts, ends, window, slopes)
    if broken is None:
        assert MC.check(o, lse, ref, False, "exact") == 0.0
    else:
        with pytest.raises(AssertionError):
            MC.check(o, lse, ref, False, broken)


# -- refusals -------------------------------------------------------------------------------------------------------
def _fake(vocab=259, limit=1024):
    args = SimpleNamespace(max_position_embeddings=limit, apply_rope=True, alibi=False, variant="default")
    return SimpleNamespace(vocab_size=vocab, args=args)


@pytest.mark.parametrize("kw,msg", [
    (dict(draft_model=_fake(vocab=300)), "vocabulary"),
    (dict(draft_model=_fake(), num_draft_tokens=0), "num_draft_tokens"),
    (dict(draft_model=_fake(), num_draft_tokens=16), "num_draft_tokens"),
    (dict(draft_model=_fake(), kv_bits=8), "kv_bits"),
    (dict(draft_model=_fake(), max_kv_size=64), "max_kv_size"),
    (dict(draft_model=_fake(), prompt_cache=object()), "prompt_cache"),
    (dict(draft_model=_fake(), on_step=print), "on_step"),
    (dict(draft_model=_fake(limit=40)), "max_position_embeddings"),
])
def test_generate_refuses_before_allocating(kw, msg):
    with pytest.raises(ValueError, match=msg):
        G.generate(_fake(), [[1] * 20], max_tokens=30, **kw)


def test_draft_prefill_step():
    def fake(extends, prefix_lm=False):
        def check_extend(cache):
            if not extends:
                raise ValueError("chunked prefill needs a bf16 model")
        return SimpleNamespace(check_extend=check_extend, args=SimpleNamespace(prefix_lm=prefix_lm))

    assert G.draft_prefill_step(fake(True), 64, 500) == 64
    assert G.draft_prefill_step(fake(True), None, 500) is None
    assert G.draft_prefill_step(fake(False), 64, 500) is None       # e.g. a C1 draft: fp32, head_dim 16
    assert G.draft_prefill_step(fake(True, True), 64, 500) is None  # a prefix-LM prompt cannot be split
    assert G.draft_prefill_step(fake(True, True), 64, 50) == 64


def test_check_draft_refuses_num_beams():
    with pytest.raises(ValueError, match="num_beams"):
        G.check_draft(_fake(), _fake(), 3, 10, num_beams=4)


def _tok(n=256, path=None):
    cfg = SimpleNamespace(tokenizer={"normal_vocab_size": n}, tokenizer_path=path)
    return SimpleNamespace(config=cfg, external_tokenizer=None if path is None else object(), VOCAB_SIZE=n + 3,
                           EOS_TOKEN=n + 2)


def test_tokenizer_check(tmp_path):
    G.check_draft_tokenizer(_tok(), _tok())
    with pytest.raises(ValueError):
        G.check_draft_tokenizer(_tok(), _tok(255))
    for d, text in (("a", "{}"), ("b", '{"x": 1}')):
        (tmp_path / d).mkdir()
        (tmp_path / d / "tokenizer.json").write_text(text)
    with pytest.raises(ValueError):
        G.check_draft_tokenizer(_tok(path=str(tmp_path / "a")), _tok(path=str(tmp_path / "b")))


@pytest.mark.parametrize("argv", [["--draft-run", "d", "--num-beams", "2"], ["--draft-run", "d", "--kv-bits", "8"],
                                  ["--draft-run", "d", "--max-kv-size", "64"],
                                  ["--draft-run", "d", "--num-draft-tokens", "0"],
                                  ["--draft-run", "d", "--num-draft-tokens", "16"], ["--draft-checkpoint", "s"]])
def test_cli_refusals(argv):
    with pytest.raises(SystemExit):
        G.parse_args(["--run", "r", "--prompt", "x"] + argv)


def test_cli_accepts_draft_flags():
    a = G.parse_args(["--run", "r", "--prompt", "x", "--draft-run", "d", "--num-draft-tokens", "5"])
    assert (a.draft_run, a.num_draft_tokens, a.draft_checkpoint) == ("d", 5, None)
