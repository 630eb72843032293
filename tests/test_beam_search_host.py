"""Beam search's host side without a GPU: the selection rules (DESIGN §2) replaying the reference's own beam_search
(tests/golden/beam_vectors.npz, made by tests/golden/make_beam_golden.py); the slot planner's invariants; the
refusals and the CLI flags."""
from __future__ import annotations

import math
import random
import zlib
from pathlib import Path

import numpy as np
import pytest
import torch

from mlx_cuda_distributed_pretraining_b200.core.generation import (beam_result, beam_search, parse_args, plan_slots,
                                                                   select_beams)

GOLDEN = Path(__file__).resolve().parent / "golden" / "beam_vectors.npz"


def _logits_of(seq, seed, V):
    """tests/golden/make_beam_golden.py's fake model: fp32 logits after `seq`."""
    r = np.random.default_rng(zlib.crc32(np.asarray([seed] + list(seq), dtype=np.int64).tobytes()))
    return (np.round(r.uniform(-3.0, 3.0, V) * 4) / 4).astype(np.float32)


def _top(seq, seed, V, n):
    lp = torch.log_softmax(torch.from_numpy(_logits_of(seq, seed, V)), -1)
    order = torch.sort(lp, descending=True, stable=True).indices[:n]
    return order.tolist(), lp[order].tolist()


def _driven(prompt, n, max_tokens, stops, seed, V):
    """select_beams / beam_result driven from one beam per prompt, as beam_search drives them."""
    if max_tokens == 0:
        return [([], 0.0)] * n
    beams, finished = [([], 0.0)], []
    for _ in range(max_tokens):
        tops = [_top(list(prompt) + b, seed, V, n) for b, _ in beams]
        scores = sorted({s + l for (_, s), (_, lps) in zip(beams, tops) for l in lps})
        assert all(b - a >= 1e-4 for a, b in zip(scores, scores[1:])), "candidate scores closer than 1e-4"
        chosen, done, n = select_beams(beams, [t for t, _ in tops], [l for _, l in tops], n, stops)
        finished += done
        beams = [(beams[i][0] + [t], s) for i, t, s in chosen]
        if not beams:
            break
    return beam_result(beams, finished)


def test_selection_replays_reference_beam_search():
    z = np.load(GOLDEN)
    V = int(z["V"])
    for c in range(int(z["n_cases"])):
        n_beams, max_tokens, seed = (int(x) for x in z[f"c{c}_args"])
        stops = [int(t) for t in z[f"c{c}_stops"]] or None
        got = _driven([int(t) for t in z[f"c{c}_prompt"]], n_beams, max_tokens, stops, seed, V)
        assert len(got) == int(z[f"c{c}_n"]), f"case {c}"
        for i, (toks, score) in enumerate(got):
            assert toks == [int(t) for t in z[f"c{c}_b{i}_tokens"]], f"case {c} beam {i}"
            want = float(z[f"c{c}_b{i}_score"])
            assert score == want or abs(score - want) <= 1e-6, f"case {c} beam {i}: {score} vs {want}"


def test_eos_first_token_scores_minus_inf_and_shrinks_n():
    beams = [([], 0.0)]
    chosen, done, n = select_beams(beams, [[9, 4, 2]], [[-0.1, -0.5, -0.7]], 3, [9])
    assert done == [([], -math.inf)] and n == 2 and [c[1] for c in chosen] == [4, 2]
    chosen, done, n = select_beams([([4], -0.5), ([2], -0.7)], [[9, 1], [3, 9]], [[-0.1, -0.2], [-0.1, -0.3]], 2, [9])
    assert done == [([4], pytest.approx(-0.6))] and n == 1 and chosen == [(0, 1, pytest.approx(-0.7))]


def test_ties_keep_beam_major_rank_order():
    chosen, _, _ = select_beams([([1], -1.0), ([2], -1.0)], [[5, 6], [7, 8]], [[-1.0, -1.0], [-1.0, -1.0]], 2)
    assert [(i, t) for i, t, _ in chosen] == [(0, 5), (0, 6)]


def test_slot_planner_invariants():
    r = random.Random(0)
    for _ in range(500):
        n = r.randint(1, 8)
        slots = r.sample(range(n), r.randint(1, n))
        free = [s for s in range(n) if s not in slots]
        k = r.randint(0, n)
        parents = sorted(r.choice(range(len(slots))) for _ in range(k))
        r.shuffle(parents)
        out, copies, left = plan_slots(slots, free, parents)
        assert len(set(out)) == len(out) and set(out) | set(left) <= set(range(n))
        assert not set(out) & set(left)
        first = {}
        for p, s in zip(parents, out):
            if p not in first:
                first[p] = s
                assert s == slots[p]  # the first child keeps its parent's slot
        assert len(copies) == len(parents) - len(set(parents))  # copies only for the extra children
        srcs = {s for s, _ in copies}
        dsts = {d for _, d in copies}
        live_with_children = {slots[p] for p in parents}
        assert srcs <= live_with_children and not dsts & live_with_children  # live sources, free destinations


def test_refusals_name_the_constraint():
    class _M:
        class args:
            max_position_embeddings = 64
    with pytest.raises(ValueError, match="n_beams"):
        beam_search(_M(), [[1]], n_beams=0)
    with pytest.raises(ValueError, match="kv_bits"):
        beam_search(_M(), [[1]], kv_bits=8)
    with pytest.raises(ValueError, match="max_kv_size"):
        beam_search(_M(), [[1]], max_kv_size=64)
    with pytest.raises(ValueError, match="prompt_cache"):
        beam_search(_M(), [[1]], prompt_cache=object())
    with pytest.raises(ValueError, match="at least one token"):
        beam_search(_M(), [[]])
    assert beam_search(_M(), [[1], [2]], n_beams=3, max_tokens=0) == [[([], 0.0)] * 3] * 2


def test_cli_num_beams():
    a = parse_args(["--run", "r", "--prompt", "p", "--num-beams", "4"])
    assert a.num_beams == 4
    assert parse_args(["--run", "r", "--prompt", "p"]).num_beams is None
    for extra in (["--num-samples", "2"], ["--kv-bits", "8"], ["--max-kv-size", "64"], ["--prefill-step-size", "8"],
                  ["--num-beams", "0"]):
        with pytest.raises(SystemExit):
            parse_args(["--run", "r", "--prompt", "p", "--num-beams", "4", *extra])
