"""Generates tests/golden/beam_vectors.npz by RUNNING THE REFERENCE'S OWN PYTHON: the unmodified
generate_lite.beam_search (:400-484) over the NumPy mlx stand-in of oracle/mlx_numpy_shim, driven by scripted fake
models.  tests/test_beam_search_host.py replays every case through core/generation.py's host selection.  Needs the
reference tree, so it runs where that is available:

    python tests/golden/make_beam_golden.py /path/to/reference

Importing generate_lite needs, at run time: mx.Stream / mx.new_stream / mx.default_device stubs, a stable mx.argsort,
mx.take_along_axis, nn.log_softmax and a stub module mlx_lm.models.cache with make_prompt_cache.  A fake model's
logits over V tokens are a seeded function of the whole token sequence, rounded to multiples of 1/4 so that exact ties
occur; the replay recomputes them with the same function.  Each case takes the first seed for which the distinct
candidate scores of every step differ by at least 1e-4 (the fake model checks each call), so that no order hangs on
an ulp; the replay checks the gap again.
"""
import sys
import types
import zlib
from pathlib import Path

import numpy as np

HERE = Path(__file__).resolve().parent
REPO = HERE.parents[1]
if len(sys.argv) != 2:
    sys.exit("usage: python tests/golden/make_beam_golden.py <reference checkout>")
REF = Path(sys.argv[1]).resolve()

sys.path = [p for p in sys.path if p not in ("", str(REPO)) and Path(p or ".").resolve() != REPO]
sys.path.insert(0, str(REF))
sys.path.insert(0, str(REPO / "oracle" / "mlx_numpy_shim"))

import mlx.core as mx  # noqa: E402  (the shim)
import mlx.nn as nn  # noqa: E402

mx.Stream = type("Stream", (), {})
mx.new_stream = lambda *a, **k: None
mx.default_device = lambda *a, **k: None
mx.argsort = lambda a, axis=-1: mx._w(np.argsort(np.asarray(a), axis=axis, kind="stable"))
mx.take_along_axis = lambda a, idx, axis=-1: mx._w(np.take_along_axis(np.asarray(a), np.asarray(idx), axis=axis))


def _log_softmax(x, axis=-1):
    x = np.asarray(x, dtype=np.float32)
    m = np.max(x, axis=axis, keepdims=True)
    return mx._w((x - m - np.log(np.sum(np.exp(x - m), axis=axis, keepdims=True))).astype(np.float32))


nn.log_softmax = _log_softmax
for name in ("mlx_lm", "mlx_lm.models", "mlx_lm.models.cache"):
    sys.modules.setdefault(name, types.ModuleType(name))
sys.modules["mlx_lm.models.cache"].make_prompt_cache = lambda *a, **k: None
sys.modules["mlx_lm"].models = sys.modules["mlx_lm.models"]
sys.modules["mlx_lm.models"].cache = sys.modules["mlx_lm.models.cache"]

import generate_lite  # noqa: E402

V = 16


def logits_of(seq, seed):
    """The fake model's fp32 logits after `seq`: multiples of 1/4 in [-3, 3] from a hash of (seed, seq)."""
    r = np.random.default_rng(zlib.crc32(np.asarray([seed] + list(seq), dtype=np.int64).tobytes()))
    return (np.round(r.uniform(-3.0, 3.0, V) * 4) / 4).astype(np.float32)


def _lp(seq, seed):
    return np.asarray(_log_softmax(logits_of(seq, seed)))


class FakeModel:
    """Returns logits_of for each beam; checks that the step's distinct candidate scores (each beam's score replayed
    as the reference sums it, plus its top len(beams) log-probabilities) differ by at least 1e-4."""

    def __init__(self, seed, l_prefix):
        self.seed, self.l_prefix = seed, l_prefix

    def __call__(self, beams):
        b = np.asarray(beams)
        out = np.zeros((b.shape[0], b.shape[1], V), dtype=np.float32)
        scores = set()
        for i, row in enumerate(b.tolist()):
            out[i, -1] = logits_of(row, self.seed)
            score = 0
            for j in range(self.l_prefix, len(row)):
                score = score + float(_lp(row[:j], self.seed)[row[j]])
            lp = _lp(row, self.seed)
            for t in np.argsort(-lp, kind="stable")[:len(beams)]:
                scores.add(score + float(lp[t]))
        s = sorted(scores)
        if any(y - x < 1e-4 for x, y in zip(s, s[1:])):
            raise ValueError("candidate scores closer than 1e-4")
        return mx._w(out)


out = {"V": np.int64(V)}
c = 0
for n_beams in (1, 2, 4, 8):
    for max_tokens in (0, 1, 7, 20):
        for stops in ([], [0], [0, 1, 2], list(range(V // 2))):
            for k in range(2):
                prompt = [3, 5, 7][: 1 + c % 3]
                seed = 1000 * c
                while True:  # the first seed whose every step keeps distinct scores 1e-4 apart
                    try:
                        res = generate_lite.beam_search(FakeModel(seed, len(prompt)), prompt, max_tokens=max_tokens,
                                                        n_beams=n_beams, stop_tokens=stops or None)
                        break
                    except ValueError:
                        seed += 1
                out[f"c{c}_args"] = np.asarray([n_beams, max_tokens, seed], dtype=np.int64)
                out[f"c{c}_prompt"] = np.asarray(prompt, dtype=np.int64)
                out[f"c{c}_stops"] = np.asarray(stops, dtype=np.int64)
                out[f"c{c}_n"] = np.int64(len(res))
                for i, (toks, score) in enumerate(res):
                    out[f"c{c}_b{i}_tokens"] = np.asarray(list(toks), dtype=np.int64)
                    out[f"c{c}_b{i}_score"] = np.float64(score)
                c += 1
out["n_cases"] = np.int64(c)
np.savez_compressed(HERE / "beam_vectors.npz", **out)
print(f"wrote {c} cases to {HERE / 'beam_vectors.npz'}")
