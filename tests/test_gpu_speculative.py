"""Speculative decoding on the GPU: b200_attn_decode_multi against fp64, its bit-equality with b200_attn_decode at one
query and its batch / launch invariance; Model.verify's logits against decode steps and Model.forward; speculative
greedy output against Model.forward's argmax; and the sampled distribution against plain generation."""
from __future__ import annotations

import pytest
import torch

from tests import multi_decode_check as MC

pytestmark = pytest.mark.gpu

STARTS = [0, 1, 240, 250, 255, 256, 257, 1000, 4090]
S_MAX = 4352
CANARY = 64


def _ops():
    from mlx_cuda_distributed_pretraining_b200 import ops
    ops.require_device()
    return ops


def _problem(L, counts, H, Hk, D, dtype, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    B = len(STARTS)
    q = torch.randn(B, L, H, D, device="cuda", generator=g).to(dtype)
    kc = torch.randn(B, S_MAX, Hk, D, device="cuda", generator=g).to(dtype)
    vc = torch.randn(B, S_MAX, Hk, D, device="cuda", generator=g).to(dtype)
    ends = [s + n for s, n in zip(STARTS, counts)]
    for b, (e, n) in enumerate(zip(ends, counts)):
        kc[b, e:] = float("nan")   # nothing at or past a row's end may be read
        vc[b, e:] = float("nan")
        q[b, n:] = float("nan")    # nor a padding query
    return q, kc, vc, ends


def _multi_raw(q, kc, vc, starts, ends, window=-1, slopes=None):
    """b200_attn_decode_multi with o and lse inside canary-filled buffers: (o, lse, canaries intact)."""
    from mlx_cuda_distributed_pretraining_b200._lib import check, lib
    ops = _ops()
    B, L, H, D = q.shape
    Hk = kc.shape[2]
    st = torch.tensor(starts, device="cuda", dtype=torch.int32)
    en = torch.tensor(ends, device="cuda", dtype=torch.int32)
    obuf = torch.full((B * L * H * D + 2 * CANARY,), 1234.5, device="cuda", dtype=q.dtype)
    lbuf = torch.full((B * H * L + 2 * CANARY,), 1234.5, device="cuda", dtype=torch.float32)
    ws = torch.empty(ops.attention_decode_multi_workspace_bytes(B, L, H, kc.shape[1], D), device="cuda",
                     dtype=torch.uint8)
    check(lib().b200_attn_decode_multi(q.data_ptr(), kc.data_ptr(), vc.data_ptr(), st.data_ptr(), en.data_ptr(),
                                       obuf[CANARY:].data_ptr(), lbuf[CANARY:].data_ptr(), window,
                                       0 if slopes is None else slopes.data_ptr(), B, L, kc.shape[1], H, Hk, D,
                                       float(D ** -0.5), int(q.dtype == torch.bfloat16), ws.data_ptr(), ws.numel(),
                                       torch.cuda.current_stream().cuda_stream), "b200_attn_decode_multi")
    o = obuf[CANARY:CANARY + B * L * H * D].view(B, L, H, D)
    lse = lbuf[CANARY:CANARY + B * H * L].view(B, H, L)
    intact = all(bool((t[:CANARY] == 1234.5).all() and (t[-CANARY:] == 1234.5).all()) for t in (obuf, lbuf))
    return o, lse, intact


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float32], ids=["bf16", "fp32"])
@pytest.mark.parametrize("D", [16, 32, 64, 128])
@pytest.mark.parametrize("H,Hk", [(1, 1), (2, 1), (3, 1), (16, 2)])
def test_decode_multi_matches_fp64(dtype, D, H, Hk):
    from mlx_cuda_distributed_pretraining_b200.arch.flash_attention import alibi_slopes
    g = torch.Generator().manual_seed(D * 7 + H)
    worst = 0.0
    for j, L in enumerate([1, 2, 3, 5, 8, 16]):
        counts = [int(x) for x in torch.randint(0, L + 1, (len(STARTS),), generator=g)]
        counts[j % len(counts)] = L
        counts[(j + 3) % len(counts)] = 0
        counts[-1] = min(counts[-1], 6)   # start 4090: stays below s_max
        for window, alibi in ((-1, False), (0, True), (1, False), (255, True), (1000, False), (-1, True)):
            slopes = alibi_slopes(H).cuda() if alibi else None
            q, kc, vc, ends = _problem(L, counts, H, Hk, D, dtype, seed=L + D + H + window)
            o, lse, intact = _multi_raw(q, kc, vc, STARTS, ends, window, slopes)
            torch.cuda.synchronize()
            name = f"{dtype} D{D} H{H}/{Hk} L{L} W{window} alibi={alibi}"
            assert intact, f"{name}: wrote outside o / lse"
            ref = MC.reference(q, kc, vc, STARTS, ends, window, slopes)
            worst = max(worst, MC.check(o, lse, ref, dtype == torch.bfloat16, name))
            for b, n in enumerate(counts):   # padding queries are not written
                assert bool((o[b, n:] == 1234.5).all()) and bool((lse[b, :, n:] == 1234.5).all()), name
    print(f"max error / bound {worst:.3f}")


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float32], ids=["bf16", "fp32"])
@pytest.mark.parametrize("mode", ["plain", "window", "alibi"])
def test_decode_multi_one_query_bit_equal_decode(dtype, mode):
    from mlx_cuda_distributed_pretraining_b200.arch.flash_attention import alibi_slopes
    ops = _ops()
    for D, H, Hk in ((16, 8, 8), (64, 16, 8), (128, 4, 1), (32, 3, 3)):
        ends = [1, 2, 255, 256, 257, 1000, 2048, 4095]
        g = torch.Generator(device="cuda").manual_seed(D)
        B = len(ends)
        q = torch.randn(B, H, D, device="cuda", generator=g).to(dtype)
        kc = torch.randn(B, 4096, Hk, D, device="cuda", generator=g).to(dtype)
        vc = torch.randn(B, 4096, Hk, D, device="cuda", generator=g).to(dtype)
        en = torch.tensor(ends, device="cuda", dtype=torch.int32)
        window = 300 if mode == "window" else None
        alibi = alibi_slopes(H).cuda() if mode == "alibi" else None
        o1, l1 = ops.attention_decode(q, kc, vc, en, return_lse=True, window=window, alibi=alibi)
        o2, l2 = ops.attention_decode_multi(q[:, None], kc, vc, en - 1, en, window=window, alibi=alibi,
                                            return_lse=True)
        assert torch.equal(o1, o2[:, 0]) and torch.equal(l1, l2[:, :, 0]), (dtype, mode, D, H, Hk)


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float32], ids=["bf16", "fp32"])
def test_decode_multi_batch_and_launch_invariant(dtype):
    ops = _ops()
    H, Hk, D, L = 16, 8, 64, 5
    counts = [5, 3, 0, 5, 1, 4, 5, 2, 5]
    q, kc, vc, ends = _problem(L, counts, H, Hk, D, dtype, seed=4)
    st = torch.tensor(STARTS, device="cuda", dtype=torch.int32)
    en = torch.tensor(ends, device="cuda", dtype=torch.int32)
    o, lse = ops.attention_decode_multi(q, kc, vc, st, en, window=700, return_lse=True)
    o2, lse2 = ops.attention_decode_multi(q, kc, vc, st, en, window=700, return_lse=True)
    for b, n in enumerate(counts):
        assert torch.equal(o[b, :n], o2[b, :n]) and torch.equal(lse[b, :, :n], lse2[b, :, :n])
        if n == 0:
            continue
        oa, la = ops.attention_decode_multi(q[b:b + 1].contiguous(), kc[b:b + 1].contiguous(),
                                            vc[b:b + 1].contiguous(), st[b:b + 1], en[b:b + 1], window=700,
                                            return_lse=True)
        assert torch.equal(o[b, :n], oa[0, :n]) and torch.equal(lse[b, :, :n], la[0, :, :n]), f"row {b}"


# -- model level ----------------------------------------------------------------------------------------------------
def _trainer(kind):
    if kind == "c1_fp32":
        from tests.test_gpu_generation import _trainer as gen_trainer
        return gen_trainer("c1_fp32")
    from tests.test_gpu_cached_attention import _trainer as chunk_trainer
    return chunk_trainer(kind)


def _tol(kind):
    from tests.test_gpu_generation import TOL
    return TOL.get(kind, TOL["bf16_rope"])


VERIFY_KINDS = ["bf16_gqa", "bf16_rope", "mlx_lm_half", "mlx_lm_interleaved", "window", "alibi", "moe", "c1_fp32"]


def _rel_rows(a, b):
    a, b = a.double().cpu(), b.double().cpu()
    return float(((a - b).abs().amax(-1) / b.abs().amax(-1).clamp_min(1e-6)).max())


@pytest.mark.parametrize("kind", VERIFY_KINDS)
def test_verify_logits_match_decode_and_forward(kind):
    from mlx_cuda_distributed_pretraining_b200.arch.llama import KVCache
    model = _trainer(kind).model
    g = torch.Generator().manual_seed(3)
    P = [300, 250, 40]          # 250 + 7 crosses a 256-key chunk inside the chunk
    L = 7
    counts = [7, 5, 0]
    prompts = [torch.randint(0, 256, (n,), generator=g).tolist() for n in P]
    chunk = torch.randint(0, 256, (3, L), generator=g)
    S = max(P)
    toks = torch.zeros((3, S), dtype=torch.int64)
    for b, p in enumerate(prompts):
        toks[b, :len(p)] = torch.tensor(p)

    cache = KVCache(model, 3, S + L)
    model.prefill(toks.cuda(), P, cache)
    got = model.verify(chunk.cuda(), counts, cache)          # [3, L, V]
    assert cache.host_lens == [p + n for p, n in zip(P, counts)]

    ref_cache = KVCache(model, 3, S + L)
    model.prefill(toks.cuda(), P, ref_cache)
    steps = torch.stack([model.decode_step(chunk[:, i].cuda(), ref_cache) for i in range(L)], 1)
    tol = _tol(kind)
    for b, n in enumerate(counts):
        if n == 0:
            continue
        e_dec = _rel_rows(got[b, :n], steps[b, :n])
        with torch.no_grad():
            full = model(torch.tensor([prompts[b] + chunk[b, :n].tolist()], device="cuda")).float()[0, -n:]
        e_fwd = _rel_rows(got[b, :n], full)
        print(f"{kind} row {b}: verify vs decode steps {e_dec:.2e}, vs forward {e_fwd:.2e}")
        assert e_dec < tol / 4 and e_fwd < tol


def _greedy_check(model, prompts, outs, tol):
    """Each token against Model.forward's argmax over the emitted prefix, near-ties skipped; returns skipped."""
    skipped = 0
    for p, out in zip(prompts, outs):
        seq = list(p)
        for t in out:
            with torch.no_grad():
                logits = model(torch.tensor([seq], device="cuda")).float()[0, -1]
            top2 = torch.topk(logits, 2).values
            if float(top2[0] - top2[1]) <= tol * float(logits.abs().max()):
                skipped += 1
            else:
                assert t == int(torch.argmax(logits))
            seq.append(t)
    return skipped


def test_speculative_greedy_self_draft_rejects_only_near_ties():
    """The target as its own draft: the draft cache is rewound and caught up each round, so a draft differs from the
    target's choice only where the two cached paths' rounding can swap the top two logits.  Every round that accepted
    fewer drafts than it proposed is checked against Model.forward over its prefix: the top two logits there must lie
    within twice the logits tolerance.  An off-by-one in the draft's cache would make it draft wrong tokens at clear
    margins."""
    from mlx_cuda_distributed_pretraining_b200.core.generation import generate
    model = _trainer("bf16_rope").model
    tol = _tol("bf16_rope")
    g = torch.Generator().manual_seed(21)
    prompts = [torch.randint(0, 256, (n,), generator=g).tolist() for n in (60, 3, 250)]
    rounds = [[] for _ in prompts]

    def on_round(emitted, drafted):
        for b, (e, d) in enumerate(zip(emitted, drafted)):
            if d:
                rounds[b].append((e, d))

    outs = generate(model, prompts, max_tokens=40, temperature=0, repetition_penalty=1.0, min_p=None,
                    draft_model=model, num_draft_tokens=4, on_round=on_round)
    n_rounds = rejected = 0
    for b, (p, out) in enumerate(zip(prompts, outs)):
        assert len(out) == 40
        pos = 1                       # the first token comes from the prefill, before any round
        for e, d in rounds[b]:
            n_rounds += 1
            n = 0
            while n < min(len(e), len(d)) and e[n] == d[n]:
                n += 1
            if n < len(d) and n < len(e):   # the target chose e[n], the draft d[n]: a rejection, not a cut
                rejected += 1
                with torch.no_grad():
                    logits = model(torch.tensor([p + out[:pos + n]], device="cuda")).float()[0, -1]
                top2 = torch.topk(logits, 2).values
                gap = float(top2[0] - top2[1]) / float(logits.abs().max())
                assert gap <= 2 * tol, f"row {b}: draft {d[n]} rejected for {e[n]} at a clear margin ({gap:.2e})"
            assert out[pos:pos + len(e)] == e
            pos += len(e)
        assert pos == len(out)
    print(f"self draft: {n_rounds} rounds, {rejected} rejections, all at near-ties")
    assert n_rounds >= 3 * 40 // 5 and rejected <= n_rounds // 4
    assert _greedy_check(model, prompts, outs, tol) < 40


@pytest.mark.parametrize("target_kind,draft_kind", [("bf16_rope", "c1_fp32"), ("alibi", "bf16_gqa"),
                                                    ("moe", "window")])
def test_speculative_greedy_random_draft_is_target_greedy(target_kind, draft_kind):
    from mlx_cuda_distributed_pretraining_b200.core.generation import generate
    model = _trainer(target_kind).model
    draft = _trainer(draft_kind).model
    g = torch.Generator().manual_seed(8)
    prompts = [torch.randint(0, 256, (n,), generator=g).tolist() for n in (5, 270, 33)]
    eos, max_tokens = 7, 23    # 23 tokens end mid-round for K = 3
    cache_lens = []
    outs = generate(model, prompts, max_tokens=max_tokens, temperature=0, repetition_penalty=1.0, min_p=None,
                    eos_token=eos, draft_model=draft, num_draft_tokens=3)
    for o in outs:
        assert len(o) == max_tokens or (o[-1] == eos and eos not in o[:-1])
        assert len(o) <= max_tokens
    skipped = _greedy_check(model, prompts, outs, _tol(target_kind))
    print(f"{target_kind} drafted by {draft_kind}: {[len(o) for o in outs]} tokens, {skipped} near-ties skipped")
    assert skipped < sum(len(o) for o in outs) // 2


def test_speculative_cache_ends_at_prompt_and_output():
    from mlx_cuda_distributed_pretraining_b200.arch import llama
    from mlx_cuda_distributed_pretraining_b200.core.generation import generate
    model = _trainer("bf16_gqa").model
    draft = _trainer("c1_fp32").model
    made = []
    orig = llama.KVCache.__init__

    def spy(self, *a, **k):
        orig(self, *a, **k)
        made.append(self)

    prompts = [[1, 2, 3], list(range(10, 60))]
    llama.KVCache.__init__ = spy
    try:
        outs = generate(model, prompts, max_tokens=10, temperature=0.8, seed=3, draft_model=draft,
                        num_draft_tokens=5)
    finally:
        llama.KVCache.__init__ = orig
    target = made[0]
    assert target.host_lens == [len(p) + len(o) - 1 for p, o in zip(prompts, outs)]


def _tiny(seed):
    """A bf16 model with a 16-token vocabulary (13 byte-level + 3 special tokens)."""
    from mlx_cuda_distributed_pretraining_b200.core.training import Config, Trainer
    from tests.test_gpu_generation import _cfg
    import tempfile
    c = _cfg("bf16_rope")
    c["data"]["tokenizer"]["normal_vocab_size"] = 13
    c["system"]["seed"] = seed
    return Trainer(Config.from_dict(c), for_training=False, synthetic=True, quiet=True,
                   run_root=tempfile.mkdtemp(prefix="spec_runs_")).model


def test_speculative_sampling_matches_plain_distribution():
    from scipy.stats import chi2_contingency
    from mlx_cuda_distributed_pretraining_b200.core.generation import generate

    model, draft = _tiny(1), _tiny(2)
    assert model.vocab_size == 16
    with torch.no_grad():   # sharper target distributions than the random init gives
        model._logits_weight().mul_(8.0)
    N, n_tok = 8192, 4
    prompts = [[1, 5, 2]] * N
    kw = dict(max_tokens=n_tok, temperature=0.9, min_p=None, top_p=0.95, repetition_penalty=1.3,
              repetition_context_size=3)
    plain = torch.tensor(generate(model, prompts, seed=11, **kw))
    spec = torch.tensor(generate(model, prompts, seed=12, draft_model=draft, num_draft_tokens=2, **kw))
    for i in range(n_tok):
        table = torch.stack([torch.bincount(plain[:, i], minlength=16), torch.bincount(spec[:, i], minlength=16)])
        table = table[:, table.sum(0) > 0].numpy()
        p = chi2_contingency(table)[1] if table.shape[1] > 1 else 1.0
        print(f"token {i}: p = {p:.3g}")
        assert p > 1e-3


def test_speculative_sampling_never_reads_padding(monkeypatch):
    """Ragged rounds at temperature > 0 (rows finishing at EOS, k_b cut by max_tokens) leave padding positions in the
    draft's and the target's verify calls.  With every padding output of the attention poisoned with NaN, the run must
    complete and give exactly the tokens of the unpoisoned run with the same seed."""
    from mlx_cuda_distributed_pretraining_b200 import ops
    from mlx_cuda_distributed_pretraining_b200.core.generation import generate
    model, draft = _tiny(3), _tiny(4)
    g = torch.Generator().manual_seed(5)
    prompts = [torch.randint(0, 13, (n,), generator=g).tolist() for n in (1, 4, 9, 2, 30, 7, 3, 12)]
    kw = dict(max_tokens=26, temperature=1.0, min_p=None, repetition_penalty=1.2, eos_token=5, seed=9,
              draft_model=draft, num_draft_tokens=3)
    clean = generate(model, prompts, **kw)
    real = ops.attention_decode_multi
    poisoned = [0]

    def poison(q, k_cache, v_cache, start, end, *a, **k):
        out = real(q, k_cache, v_cache, start, end, *a, **k)
        o = out[0] if isinstance(out, tuple) else out
        for b, n in enumerate((end - start).tolist()):
            if n < q.shape[1]:
                o[b, n:] = float("nan")
                poisoned[0] += 1
        return out

    monkeypatch.setattr(ops, "attention_decode_multi", poison)
    dirty = generate(model, prompts, **kw)
    print(f"{poisoned[0]} padded rows poisoned; lengths {[len(o) for o in clean]}")
    assert poisoned[0] > 0 and any(len(o) < 26 for o in clean)
    assert dirty == clean
    for o in clean:
        assert len(o) == 26 or (o[-1] == 5 and 5 not in o[:-1])


def test_speculative_fp32_draft_with_chunked_prefill():
    """A C1-shaped draft (fp32, head_dim 16), which Model.extend does not serve, is prefilled in one piece when the
    target is prefilled in chunks; the output is still the target's greedy sequence."""
    from mlx_cuda_distributed_pretraining_b200.core.generation import generate
    model = _trainer("bf16_gqa").model
    draft = _trainer("c1_fp32").model
    g = torch.Generator().manual_seed(13)
    prompts = [torch.randint(0, 256, (n,), generator=g).tolist() for n in (40, 5)]
    outs = generate(model, prompts, max_tokens=12, temperature=0, repetition_penalty=1.0, min_p=None,
                    prefill_step_size=16, draft_model=draft, num_draft_tokens=3)
    assert [len(o) for o in outs] == [12, 12]
    assert _greedy_check(model, prompts, outs, _tol("bf16_gqa")) < 12


def test_decode_multi_refuses_a_grid_past_65535():
    from mlx_cuda_distributed_pretraining_b200._lib import B200Error
    ops = _ops()
    B, L = 4096, 16
    q = torch.zeros(B, L, 1, 16, device="cuda")
    kc = torch.zeros(B, 32, 1, 16, device="cuda")
    st = torch.zeros(B, device="cuda", dtype=torch.int32)
    with pytest.raises(B200Error, match="65535"):
        ops.attention_decode_multi(q, kc, kc, st, st + L)
