"""Chunked prefill and prompt caches on the GPU: b200_attn_fwd_cached element by element against fp64 (the forward's
own checker, tests/attn_fwd_check.py, with each chunk embedded as the last rows of a full-length problem),
b200_kv_dequantize bit for bit against the CPU oracle, and Model.extend / generate(prefill_step_size, prompt_cache)
against the one-shot prefill, the full forward and the fp64 oracle."""
from __future__ import annotations

import os
import subprocess
import sys
import tempfile
from pathlib import Path

import pytest
import torch
import yaml

from tests import attn_fwd_check as AF
from tests import cached_attn_check as CA
from tests import kv_quant_oracle as KQ

pytestmark = pytest.mark.gpu

ROOT = Path(__file__).resolve().parents[1]
CANARY = 4096.0     # bf16-exact, far outside any output
FRAME = 4096        # canary elements on each side of an output


def _ops():
    from mlx_cuda_distributed_pretraining_b200 import ops
    ops.require_device()
    return ops


def _framed(shape, dtype):
    """(view of `shape` inside a canary-filled allocation, the allocation)."""
    n = 1
    for s in shape:
        n *= s
    buf = torch.full((n + 2 * FRAME,), CANARY, device="cuda", dtype=dtype)
    return buf[FRAME:FRAME + n].view(shape), buf


def _frame_intact(buf):
    return bool((buf[:FRAME] == CANARY).all()) and bool((buf[-FRAME:] == CANARY).all())


def _cached_raw(q, kc, vc, start, end, window=-1, slopes=None, scale=None):
    """b200_attn_fwd_cached into canary-framed o / lse; returns (o, lse, frames intact)."""
    from mlx_cuda_distributed_pretraining_b200._lib import check, lib
    from mlx_cuda_distributed_pretraining_b200.ops import _ptr, _stream
    B, L, H, D = q.shape
    s_max, Hk = kc.shape[1], kc.shape[2]
    o, ob = _framed((B, L, H, D), torch.bfloat16)
    lse, lb = _framed((B, H, L), torch.float32)
    scale = D ** -0.5 if scale is None else scale
    check(lib().b200_attn_fwd_cached(q.data_ptr(), kc.data_ptr(), vc.data_ptr(), start.data_ptr(), end.data_ptr(),
                                     o.data_ptr(), lse.data_ptr(), window, _ptr(slopes), B, L, s_max, H, Hk, D,
                                     float(scale), _stream()), "b200_attn_fwd_cached")
    torch.cuda.synchronize()
    return o.clone(), lse.clone(), _frame_intact(ob) and _frame_intact(lb)


STARTS = [0, 1, 127, 128, 129, 1000, 4000, 50]


def _inputs(L, H, Hk, D, seed, starts=STARTS):
    """Rows at STARTS with different valid counts (the last row none); q padding and cache positions past each end
    are NaN."""
    g = torch.Generator().manual_seed(seed)
    ns = [L, max(1, L - 1), max(1, L // 2), 1, L, max(1, L // 3), L, 0][:len(starts)]
    ends = [s + n for s, n in zip(starts, ns)]
    B, s_max = len(starts), max(ends) + 3
    q = torch.randn(B, L, H, D, generator=g).to(torch.bfloat16)
    kc = torch.randn(B, s_max, Hk, D, generator=g).to(torch.bfloat16)
    vc = torch.randn(B, s_max, Hk, D, generator=g).to(torch.bfloat16)
    for b, (s, e) in enumerate(zip(starts, ends)):
        q[b, e - s:] = float("nan")
        kc[b, e:] = float("nan")
        vc[b, e:] = float("nan")
    dev = lambda t: t.cuda()  # noqa: E731
    return (dev(q), dev(kc), dev(vc), dev(torch.tensor(starts, dtype=torch.int32)),
            dev(torch.tensor(ends, dtype=torch.int32)), ns)


HEADS = [(8, 8), (8, 4), (8, 1), (12, 4), (1, 1), (2, 1)]   # H / Hk = 1, 2, 8, 3 and single heads
MODES = [(-1, False), (0, True), (1, False), (127, True), (1000, False), (-1, True)]   # (window, ALiBi)


@pytest.mark.parametrize("mode", range(len(MODES)))
@pytest.mark.parametrize("D", [64, 128])
@pytest.mark.parametrize("L", [1, 63, 128, 129, 512])
def test_cached_attention_matches_fp64(L, D, mode):
    from mlx_cuda_distributed_pretraining_b200.arch.flash_attention import alibi_slopes
    window, alibi = MODES[mode]
    H, Hk = HEADS[(L + D // 64 + mode) % len(HEADS)]
    q, kc, vc, start, end, ns = _inputs(L, H, Hk, D, seed=L * 7 + D + mode)
    slopes = alibi_slopes(H).cuda() if alibi else None
    o, lse, intact = _cached_raw(q, kc, vc, start, end, window, slopes)
    assert intact, "a write landed outside o / lse"
    worst = CA.check_rows(q, kc, vc, STARTS, ns, o, lse, window, slopes, f"L{L} D{D} H{H}/{Hk} w{window} a{alibi}")
    print(f"L={L} D={D} H={H}/{Hk} window={window} alibi={alibi}: worst error/bound {worst:.3f}")


def test_cached_attention_bit_identical_repeat_and_alone():
    from mlx_cuda_distributed_pretraining_b200.arch.flash_attention import alibi_slopes
    q, kc, vc, start, end, ns = _inputs(300, 8, 2, 128, seed=3)
    slopes = alibi_slopes(8).cuda()
    o1, l1, _ = _cached_raw(q, kc, vc, start, end, 200, slopes)
    o2, l2, _ = _cached_raw(q, kc, vc, start, end, 200, slopes)
    assert torch.equal(o1, o2) and torch.equal(l1, l2)
    for b in range(q.shape[0]):
        one = [t[b:b + 1].contiguous() for t in (q, kc, vc, start, end)]
        oa, la, _ = _cached_raw(*one, 200, slopes)
        n = ns[b]
        assert torch.equal(oa[0, :n], o1[b, :n]) and torch.equal(la[0, :, :n], l1[b, :, :n]), f"row {b}"


@pytest.mark.parametrize("S", [512, 300])
@pytest.mark.parametrize("D", [64, 128])
def test_cached_from_zero_equals_causal_forward(S, D):
    """start = 0, L = S is the causal forward: bit-equal when S is a multiple of 128 (the same key tiles from 0),
    within the fp64 bound otherwise (the last query tile's key tiles are anchored at S instead)."""
    from mlx_cuda_distributed_pretraining_b200._lib import check, lib
    from mlx_cuda_distributed_pretraining_b200.ops import _stream
    g = torch.Generator().manual_seed(S + D)
    B, H, Hk = 2, 8, 4
    q, k, v = (torch.randn(B, S, h, D, generator=g).to(torch.bfloat16).cuda() for h in (H, Hk, Hk))
    z = torch.zeros(B, dtype=torch.int32, device="cuda")
    e = torch.full((B,), S, dtype=torch.int32, device="cuda")
    o, lse, _ = _cached_raw(q, k, v, z, e)
    oc = torch.empty_like(q)
    lc = torch.empty(B, H, S, device="cuda")
    check(lib().b200_attn_fwd(q.data_ptr(), k.data_ptr(), v.data_ptr(), oc.data_ptr(), lc.data_ptr(), B, S, H, Hk, D,
                              D ** -0.5, 1, _stream()), "b200_attn_fwd")
    torch.cuda.synchronize()
    ref = AF.reference(q, k, v, D ** -0.5, mask=AF.visible(S, True, device="cuda"))
    AF.check("cached o", o, *ref["o"])
    AF.check("cached lse", lse, *ref["lse"])
    same = torch.equal(o, oc) and torch.equal(lse, lc)
    print(f"S={S} D={D}: bit-equal to b200_attn_fwd causal: {same}")
    if S % 128 == 0:
        assert same


def test_cached_attention_errors_are_returned():
    from mlx_cuda_distributed_pretraining_b200._lib import lib
    from mlx_cuda_distributed_pretraining_b200.ops import _stream
    q, kc, vc, start, end, _ = _inputs(64, 4, 2, 64, seed=1)
    o = torch.empty_like(q)
    args = lambda **kw: dict(dict(B=q.shape[0], L=64, s_max=kc.shape[1], H=4, Hk=2, D=64), **kw)  # noqa: E731
    for bad in (args(D=32), args(H=3), args(L=0)):
        rc = lib().b200_attn_fwd_cached(q.data_ptr(), kc.data_ptr(), vc.data_ptr(), start.data_ptr(), end.data_ptr(),
                                        o.data_ptr(), None, -1, None, bad["B"], bad["L"], bad["s_max"], bad["H"],
                                        bad["Hk"], bad["D"], 0.125, _stream())
        assert rc != 0
    rc = lib().b200_attn_fwd_cached(q.data_ptr(), kc.data_ptr(), vc.data_ptr(), None, end.data_ptr(), o.data_ptr(),
                                    None, -1, None, q.shape[0], 64, kc.shape[1], 4, 2, 64, 0.125, _stream())
    assert rc != 0


def test_attention_cached_wrapper_lse_optional():
    ops = _ops()
    q, kc, vc, start, end, ns = _inputs(129, 4, 2, 64, seed=4)
    o, lse = ops.attention_cached(q, kc, vc, start, end, return_lse=True)
    o2 = ops.attention_cached(q, kc, vc, start, end)
    for b, n in enumerate(ns):
        assert torch.equal(o[b, :n], o2[b, :n])
    with pytest.raises(ValueError):
        ops.attention_cached(q.float(), kc.float(), vc.float(), start, end)
    with pytest.raises(ValueError):
        ops.attention_cached(q, kc, vc, start.long(), end)


# -- b200_kv_dequantize ----------------------------------------------------------------------------------------------
@pytest.mark.parametrize("bits", [4, 8])
@pytest.mark.parametrize("D,g", [(64, 32), (64, 64), (128, 32), (128, 64), (128, 128)])
def test_kv_dequantize_bit_exact(bits, D, g):
    ops = _ops()
    B, s_max, Hk = 3, 258, 2
    gen = torch.Generator().manual_seed(bits * D + g)
    ends = [1, 257, 130]
    codes, params = [], []
    for _ in range(2):
        x = torch.randn(B, s_max, Hk, D, generator=gen) * 3
        c, p = KQ.cache_layout(x, bits, g)
        codes.append(c)
        params.append(p)
    S = 257
    k, kb = _framed((B, S, Hk, D), torch.bfloat16)
    v, vb = _framed((B, S, Hk, D), torch.bfloat16)
    end = torch.tensor(ends, dtype=torch.int32, device="cuda")
    ops.kv_dequantize(codes[0].cuda(), codes[1].cuda(), params[0].cuda(), params[1].cuda(), end, bits, g, out=(k, v))
    torch.cuda.synchronize()
    assert _frame_intact(kb) and _frame_intact(vb)
    for got, c, p in ((k, codes[0], params[0]), (v, codes[1], params[1])):
        want = KQ.dequantize_cache(c, p, bits, g).to(torch.bfloat16)
        for b, e in enumerate(ends):
            assert torch.equal(got[b, :e].cpu().view(torch.int16), want[b, :e].view(torch.int16)), f"row {b}"
            assert bool((got[b, e:] == CANARY).all()), f"row {b}: written past end"


# -- model level -----------------------------------------------------------------------------------------------------
KINDS = ["bf16_gqa", "bf16_rope", "mlx_lm_half", "mlx_lm_interleaved", "window", "alibi", "moe"]


def _trainer(kind):
    from mlx_cuda_distributed_pretraining_b200.core.training import Config, Trainer
    from tests.test_gpu_generation import _cfg
    c = _cfg("bf16_gqa" if kind in ("bf16_gqa", "alibi") else "bf16_rope")
    if kind.startswith("mlx_lm") or kind == "moe":
        c["model"]["misc"]["variant"] = "mlx_lm"
        c["model"]["rope"]["traditional"] = kind == "mlx_lm_interleaved"
    if kind == "moe":
        c["model"]["misc"].update(num_local_experts=4, num_experts_per_tok=2)
    if kind == "window":
        c["model"]["attention"]["sliding_window"] = 64
    if kind == "alibi":
        c["model"]["attention"]["alibi"] = True
    return Trainer(Config.from_dict(c), for_training=False, synthetic=True, quiet=True,
                   run_root=tempfile.mkdtemp(prefix="chunk_runs_"))


def _tol(kind):
    from tests.test_gpu_generation import TOL
    return TOL.get(kind, TOL["bf16_rope"])


def _chunked(model, prompts, step, cache, steps_after=None):
    from mlx_cuda_distributed_pretraining_b200.core.generation import _prefill
    out = [_prefill(model, prompts, cache, step)]
    for t in (steps_after if steps_after is not None else []):
        out.append(model.decode_step(t, cache))
    return torch.stack(out, 1)


@pytest.mark.parametrize("kind", KINDS)
def test_chunked_prefill_matches_one_shot(kind):
    from mlx_cuda_distributed_pretraining_b200.arch.llama import KVCache
    from tests.test_gpu_generation import _oracle_logits, _rel_rows
    tr = _trainer(kind)
    model = tr.model
    g = torch.Generator().manual_seed(11)
    T = 300
    tokens = torch.randint(0, 256, (2, T + 3), generator=g)
    prompts = [tokens[0, :T].tolist(), tokens[1, :217].tolist()]
    after = [torch.tensor([tokens[0, T + i], tokens[1, 217 + i]]).cuda() for i in range(3)]
    one = _chunked(model, prompts, None, KVCache(model, 2, T + 8), after)
    tol = _tol(kind)
    oracle = None
    if kind in ("bf16_gqa", "bf16_rope"):
        seq = [prompts[0] + [int(t[0]) for t in after], prompts[1] + [int(t[1]) for t in after]]
        full = [_oracle_logits(tr, torch.tensor([s]))[0] for s in seq]
        oracle = torch.stack([torch.stack([full[b][len(prompts[b]) - 1 + i] for i in range(4)]) for b in range(2)])
    for step in (1, 100, 128, 256):
        got = _chunked(model, prompts, step, KVCache(model, 2, T + 8), after)
        err = _rel_rows(got, one)
        msg = f"{kind} step {step}: vs one-shot {err:.2e}"
        assert err < tol, msg
        if oracle is not None:
            e_orc = _rel_rows(got, oracle)
            msg += f", vs fp64 oracle {e_orc:.2e}"
            assert e_orc < tol, msg
        print(msg)


@pytest.mark.parametrize("kind", ["bf16_rope", "window"])
def test_continuation_matches_whole_prefill_and_ragged_rows_alone(kind):
    from mlx_cuda_distributed_pretraining_b200.arch.llama import KVCache
    from tests.test_gpu_generation import _rel_rows
    model = _trainer(kind).model
    g = torch.Generator().manual_seed(4)
    A, Bn = [200, 37, 130], [90, 129, 1]
    seqs = [torch.randint(0, 256, (a + b,), generator=g) for a, b in zip(A, Bn)]

    def pad(rows):
        w = max(len(r) for r in rows)
        t = torch.zeros(len(rows), w, dtype=torch.int64)
        for i, r in enumerate(rows):
            t[i, :len(r)] = r
        return t.cuda()

    def continued(idx):
        cache = KVCache(model, len(idx), 512)
        model.prefill(pad([seqs[i][:A[i]] for i in idx]), [A[i] for i in idx], cache)
        lg = model.extend(pad([seqs[i][A[i]:] for i in idx]), [Bn[i] for i in idx], cache)
        assert cache.host_lens == [A[i] + Bn[i] for i in idx]
        return lg

    whole_cache = KVCache(model, 3, 512)
    whole = model.prefill(pad(seqs), [len(s) for s in seqs], whole_cache)
    batch = continued([0, 1, 2])
    err = _rel_rows(batch, whole)
    print(f"{kind}: prefill(A) + extend(B) vs prefill(A + B) {err:.2e}")
    assert err < _tol(kind)
    for r in range(3):
        alone = continued([r])
        e = _rel_rows(batch[r:r + 1], alone)
        assert e < _tol(kind) / 4, f"row {r}: batch vs alone {e:.2e}"


def _greedy_check(model, seq, out, tol):
    """out continues seq greedily under the full forward, near-ties skipped; returns the number skipped."""
    seq, skipped = list(seq), 0
    for i, t in enumerate(out):
        with torch.no_grad():
            logits = model(torch.tensor([seq], device="cuda")).float()[0, -1]
        top2 = torch.topk(logits, 2).values
        if float(top2[0] - top2[1]) <= tol * float(logits.abs().max()):
            skipped += 1
        else:
            assert t == int(torch.argmax(logits)), f"step {i}"
        seq.append(t)
    return skipped


def test_two_turn_greedy_with_prompt_cache():
    from mlx_cuda_distributed_pretraining_b200.arch.llama import KVCache
    from mlx_cuda_distributed_pretraining_b200.core.generation import generate
    tr = _trainer("bf16_gqa")
    model = tr.model
    bos = tr.tokenizer.BOS_TOKEN
    turn1 = [[bos] + list(range(40, 80)), [bos] + list(range(100, 117))]
    turn2 = [list(range(60, 90)), list(range(5, 8))]
    kw = dict(temperature=0, repetition_penalty=1.0, min_p=None)
    cache = KVCache(model, 2, 400)
    out1 = generate(model, turn1, max_tokens=20, prompt_cache=cache, **kw)
    assert cache.host_lens == [len(p) + len(o) for p, o in zip(turn1, out1)]
    out2 = generate(model, turn2, max_tokens=24, prompt_cache=cache, prefill_step_size=16, **kw)
    assert cache.host_lens == [len(a) + len(b) + len(c) + len(d) for a, b, c, d in zip(turn1, out1, turn2, out2)]
    skipped = 0
    for b in range(2):
        skipped += _greedy_check(model, turn1[b] + out1[b] + turn2[b], out2[b], _tol("bf16_gqa"))
        fresh = generate(model, [turn1[b] + out1[b] + turn2[b]], max_tokens=24, **kw)[0]
        agree = sum(x == y for x, y in zip(fresh, out2[b]))
        print(f"row {b}: two-turn vs fresh generate on the concatenation: {agree}/{len(fresh)} tokens agree")
    assert skipped < 24


@pytest.mark.parametrize("bits", [4, 8])
@pytest.mark.parametrize("qstart", [0, 150, 1000])
def test_chunked_prefill_quantized_cache(bits, qstart):
    from mlx_cuda_distributed_pretraining_b200.arch.llama import KVCache
    from mlx_cuda_distributed_pretraining_b200.core.generation import prefill_chunks
    from tests.test_gpu_generation import _rel_rows
    from tests.test_gpu_kv_quant import _quant_tol
    model = _trainer("bf16_rope").model
    g = torch.Generator().manual_seed(bits + qstart)
    T = 300
    tokens = torch.randint(0, 256, (2, T + 3), generator=g)
    prompts = [tokens[0, :T].tolist(), tokens[1, :217].tolist()]
    after = [torch.tensor([tokens[0, T + i], tokens[1, 217 + i]]).cuda() for i in range(3)]
    dense = _chunked(model, prompts, None, KVCache(model, 2, T + 8), after)
    for step in (100, 256):
        cache = KVCache(model, 2, T + 8, kv_bits=bits, kv_group_size=64, quantized_kv_start=qstart)
        # conversion follows the reference: after the first chunk that takes the longest row past quantized_kv_start
        seen = 0
        for c, chunk in enumerate(prefill_chunks(prompts, step)):
            counts = [len(t) for t in chunk]
            toks = torch.zeros(2, max(counts), dtype=torch.int64)
            for b, t in enumerate(chunk):
                toks[b, :len(t)] = torch.tensor(t)
            (model.prefill if c == 0 else model.extend)(toks.cuda(), counts, cache)
            seen += max(counts)
            assert cache.quantized == (max(cache.host_lens) > qstart), f"chunk {c}"
        got = _chunked(model, prompts, step,
                       KVCache(model, 2, T + 8, kv_bits=bits, kv_group_size=64, quantized_kv_start=qstart), after)
        err = _rel_rows(got, dense)
        tol = _quant_tol("bf16_rope", bits)
        print(f"{bits}-bit start {qstart} step {step}: vs bf16 one-shot {err:.2e} (tolerance {tol:.2e})")
        assert err < tol


def test_cli_prefill_step_size_end_to_end():
    env = dict(os.environ, PYTHONPATH=str(ROOT) + os.pathsep + os.environ.get("PYTHONPATH", ""))
    with tempfile.TemporaryDirectory(prefix="chunk_e2e_") as tmp:
        cfg = yaml.safe_load((ROOT / "configs" / "c1-llama2m-adamw.yaml").read_text())
        cfg["name"] = "chunk-e2e"
        cfg["data"]["input_file"] = "synthetic:markov"
        cfg["data"]["preprocessing"]["max_context_size"] = 128
        cfg["training"]["hyperparameters"]["iters"] = 3
        cfg["model"]["attention"].update(num_heads=4, num_kv_heads=2, head_dim=64)
        cfg["system"]["mixed_precision"] = True
        cfg_path = Path(tmp) / "cfg.yaml"
        cfg_path.write_text(yaml.safe_dump(cfg))
        subprocess.run([sys.executable, "-m", "core.training", "--config", str(cfg_path)], cwd=tmp, env=env,
                       check=True, timeout=600)
        out = subprocess.run([sys.executable, "-m", "core.generation", "--run", "chunk-e2e", "--runs-dir",
                              str(Path(tmp) / "runs"), "--prompt", "hello there", "--max-tokens", "16", "--seed", "0",
                              "--prefill-step-size", "3", "--num-samples", "2"],
                             cwd=ROOT, env=env, check=True, capture_output=True, text=True, timeout=600).stdout
        assert sum(l.startswith("Greedy Output: ") for l in out.splitlines()) == 2
