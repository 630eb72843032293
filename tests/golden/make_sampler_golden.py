"""Generates tests/golden/sampler_vectors.npz by RUNNING THE REFERENCE'S OWN PYTHON: the unmodified
mlx_lm_utils.make_sampler (:57-107) and make_logits_processors (:109-142) over the NumPy mlx stand-in of
oracle/mlx_numpy_shim.  tests/test_generation_host.py holds core/generation.py's filters to these vectors.  Needs the
reference tree, so it runs where that is available:

    python tests/golden/make_sampler_golden.py /path/to/reference

The shim lacks argsort, cumsum, log, where, logsumexp and random.categorical; they are added at run time (argsort is
stable, so ties keep index order).  The patched categorical records the log-distribution it is handed and returns its
argmax, so the fixture pins the FILTERED DISTRIBUTIONS, not random draws: for min-p / top-p in sorted order (with the
argsort order that produced it), for plain sampling the scaled logits.  The repetition processor is called in its
declared order processor(logits, tokens, idx) with idx = len(tokens) - 1.
"""
import sys
from pathlib import Path

import numpy as np

HERE = Path(__file__).resolve().parent
REPO = HERE.parents[1]
if len(sys.argv) != 2:
    sys.exit("usage: python tests/golden/make_sampler_golden.py <reference checkout>")
REF = Path(sys.argv[1]).resolve()

sys.path = [p for p in sys.path if p not in ("", str(REPO)) and Path(p or ".").resolve() != REPO]
sys.path.insert(0, str(REF))
sys.path.insert(0, str(REPO / "oracle" / "mlx_numpy_shim"))

import mlx.core as mx  # noqa: E402  (the shim)

_recorded = {}


def _argsort(a, axis=-1):
    idx = np.argsort(np.asarray(a), axis=axis, kind="stable")
    _recorded["order"] = idx
    return mx._w(idx)


def _categorical(logits, axis=-1):
    lg = np.asarray(logits, dtype=np.float32)
    _recorded["dist"] = lg.copy()
    return int(np.argmax(lg))


def _logsumexp(a, axis=None, keepdims=False):
    a = np.asarray(a, dtype=np.float32)
    m = np.max(a, axis=axis, keepdims=True)
    r = (m + np.log(np.sum(np.exp(a - m), axis=axis, keepdims=True))).astype(np.float32)
    return mx._w(r if keepdims else np.squeeze(r, axis=axis))


mx.argsort = _argsort
mx.cumsum = lambda a, axis=None: mx._w(np.cumsum(np.asarray(a), axis=axis if axis is not None else 0))
mx.log = lambda a: mx._w(np.log(np.asarray(a, dtype=np.float32)))
mx.where = lambda c, x, y: mx._w(np.where(c, x, y).astype(np.float32))
mx.logsumexp = _logsumexp
mx.random.categorical = staticmethod(_categorical)

from mlx_lm_utils import make_logits_processors, make_sampler  # noqa: E402

np.seterr(divide="ignore")
rng = np.random.default_rng(7)
V = 64
LOGIT_CASES = {
    "randn": (rng.standard_normal(V) * 2.0).astype(np.float32),
    "peaked": np.where(np.arange(V) == 5, 12.0, rng.standard_normal(V)).astype(np.float32),  # min_p keeps only 5
    "ties": np.repeat(rng.standard_normal(V // 4).astype(np.float32), 4)[rng.permutation(V)].astype(np.float32),
    "flat": np.zeros(V, dtype=np.float32),
}
SAMPLERS = [("min_p", dict(min_p=0.05)), ("min_p", dict(min_p=0.3)), ("top_p", dict(top_p=0.5)),
            ("top_p", dict(top_p=0.9)), ("top_p", dict(top_p=1e-4)), ("plain", {})]
TEMPS = (0.5, 1.0, 1.7)

out = {}
n = 0
for lname, lg in LOGIT_CASES.items():
    # the sampler is handed log-probabilities (generate_lite.py:237)
    logprobs = np.asarray(lg - _logsumexp(lg, axis=-1, keepdims=True), dtype=np.float32)
    for kind, kw in SAMPLERS:
        for temp in TEMPS:
            _recorded.clear()
            make_sampler(temp=temp, **kw)(mx.array(logprobs))
            key = f"s{n:03d}"
            out[f"{key}_logprobs"] = logprobs
            out[f"{key}_kind"] = np.array(kind)
            out[f"{key}_temp"] = np.array(temp, dtype=np.float64)
            out[f"{key}_param"] = np.array(kw.get("min_p", kw.get("top_p", 0.0)), dtype=np.float64)
            out[f"{key}_dist"] = _recorded["dist"]
            out[f"{key}_order"] = _recorded.get("order", np.arange(V))
            out[f"{key}_case"] = np.array(lname)
            n += 1

# repetition processor, intended argument order, windows shorter and longer than R, repeated tokens
m = 0
for penalty, R in ((1.1, 20), (1.5, 4), (0.8, 6)):
    (proc,) = make_logits_processors(repetition_penalty=penalty, repetition_context_size=R)
    for length in (1, 3, R, R + 1, 2 * R + 5):
        toks = [int(t) for t in rng.integers(0, 8, size=length)]  # small alphabet: many repeats
        lg = (rng.standard_normal(V) * 3.0).astype(np.float32)
        res = proc(mx.array(lg), toks, len(toks) - 1)
        key = f"r{m:03d}"
        out[f"{key}_logits"] = lg
        out[f"{key}_tokens"] = np.array(toks, dtype=np.int64)
        out[f"{key}_penalty"] = np.array(penalty, dtype=np.float64)
        out[f"{key}_context"] = np.array(R, dtype=np.int64)
        out[f"{key}_out"] = np.asarray(res, dtype=np.float32)
        m += 1

np.savez_compressed(HERE / "sampler_vectors.npz", **out)
print(f"wrote {HERE / 'sampler_vectors.npz'}: {n} sampler cases, {m} processor cases")
