"""The rotating KV cache (max_kv_size) on the GPU: b200_attn_fwd_ring and b200_attn_decode_ring element by element
against fp64 (tests/rotating_kv_check.py) with never-written slots NaN and outputs canary-framed, bit-identical on
repeat and alone, b200_kv_append_ring against b200_kv_append(_half), and the model and generate() over a ring."""
from __future__ import annotations

import pytest
import torch

from mlx_cuda_distributed_pretraining_b200.ops import ring_slot
from tests import rotating_kv_check as RK
from tests.test_gpu_cached_attention import _frame_intact, _framed, _ops, _tol, _trainer

pytestmark = pytest.mark.gpu


def _ring_inputs(B, L, H, Hk, D, M, ends, ns, seed):
    """q [B, L, H, D] and rings of C = M + L - 1 (rounded to 256) slots holding positions [0, ends[b]) of random keys,
    never-written slots NaN; also the true-position keys."""
    g = torch.Generator().manual_seed(seed)
    C = -(-(M + L - 1) // 256) * 256
    q = torch.randn(B, L, H, D, generator=g).to(torch.bfloat16)
    k = torch.full((B, C, Hk, D), float("nan"), dtype=torch.bfloat16)
    v = torch.full((B, C, Hk, D), float("nan"), dtype=torch.bfloat16)
    for b, e in enumerate(ends):
        pos = torch.arange(e)[RK.held(e, C)]  # the positions not yet overwritten, one per written slot
        slots = ring_slot(pos, C)
        k[b, slots] = torch.randn(len(pos), Hk, D, generator=g).to(torch.bfloat16)
        v[b, slots] = torch.randn(len(pos), Hk, D, generator=g).to(torch.bfloat16)
        q[b, ns[b]:] = float("nan")
    return q.cuda(), k.cuda(), v.cuda(), C


def _fwd_ring(q, k, v, start, end, M, window=-1, slopes=None):
    from mlx_cuda_distributed_pretraining_b200._lib import check, lib
    from mlx_cuda_distributed_pretraining_b200.ops import _ptr, _stream
    B, L, H, D = q.shape
    C, Hk = k.shape[1], k.shape[2]
    o, ob = _framed((B, L, H, D), torch.bfloat16)
    lse, lb = _framed((B, H, L), torch.float32)
    check(lib().b200_attn_fwd_ring(q.data_ptr(), k.data_ptr(), v.data_ptr(), start.data_ptr(), end.data_ptr(),
                                   o.data_ptr(), lse.data_ptr(), M, window, _ptr(slopes), B, L, C, H, Hk, D,
                                   float(D ** -0.5), _stream()), "b200_attn_fwd_ring")
    torch.cuda.synchronize()
    return o.clone(), lse.clone(), _frame_intact(ob) and _frame_intact(lb)


def _dec_ring(q, k, v, end, M, window=-1, slopes=None):
    from mlx_cuda_distributed_pretraining_b200._lib import check, lib
    from mlx_cuda_distributed_pretraining_b200.ops import _ptr, _stream, attention_decode_workspace_bytes
    B, H, D = q.shape
    C, Hk = k.shape[1], k.shape[2]
    o, ob = _framed((B, H, D), torch.bfloat16)
    lse, lb = _framed((B, H), torch.float32)
    ws = torch.empty(attention_decode_workspace_bytes(B, H, C, D), device="cuda", dtype=torch.uint8)
    check(lib().b200_attn_decode_ring(q.data_ptr(), k.data_ptr(), v.data_ptr(), end.data_ptr(), o.data_ptr(),
                                      lse.data_ptr(), M, window, _ptr(slopes), B, C, H, Hk, D, float(D ** -0.5),
                                      ws.data_ptr(), ws.numel(), _stream()), "b200_attn_decode_ring")
    torch.cuda.synchronize()
    return o.clone(), lse.clone(), _frame_intact(ob) and _frame_intact(lb)


def _ends(M, L):
    """Row ends before the wrap, exactly at it, and many times around."""
    C = -(-(M + L - 1) // 256) * 256
    return [min(L, 3) + 2, C - 1, C, C + 1, 3 * C + 7, 9 * C + 100]


CASES = [(5, 1, 64, 1), (64, 17, 128, 2), (300, 128, 64, 4), (1000, 129, 128, 8), (64, 512, 64, 2),
         (1000, 512, 128, 1)]


@pytest.mark.parametrize("M,L,D,G", CASES)
@pytest.mark.parametrize("mode", ["plain", "window", "alibi", "window_alibi"])
def test_fwd_ring_matches_fp64(M, L, D, G, mode):
    ops = _ops()
    ends = _ends(M, L)
    ns = [min(L, e, 1 + (7 * i) % L) for i, e in enumerate(ends)]
    Hk = 2
    H = Hk * G
    q, k, v, C = _ring_inputs(len(ends), L, H, Hk, D, M, ends, ns, seed=M + L + D)
    starts = [e - n for e, n in zip(ends, ns)]
    st = torch.tensor(starts, dtype=torch.int32, device="cuda")
    en = torch.tensor(ends, dtype=torch.int32, device="cuda")
    window = 40 if "window" in mode else -1
    slopes = None
    if "alibi" in mode:
        from mlx_cuda_distributed_pretraining_b200.arch.flash_attention import alibi_slopes
        slopes = alibi_slopes(H).float().cuda()
    o, lse, intact = _fwd_ring(q, k, v, st, en, M, window, slopes)
    assert intact, "write outside o / lse"
    RK.check_rows(q.cpu(), k.cpu(), v.cpu(), starts, ends, o.cpu(), lse.cpu(), M, None if window < 0 else window,
                  None if slopes is None else slopes.cpu(), f"fwd_ring M={M} L={L} {mode}")
    o2, lse2, _ = _fwd_ring(q, k, v, st, en, M, window, slopes)
    assert torch.equal(o, o2) and torch.equal(lse, lse2), "not bit-identical on repeat"
    for b in (1, len(ends) - 1):
        ob, lb, _ = _fwd_ring(q[b:b + 1].contiguous(), k[b:b + 1].contiguous(), v[b:b + 1].contiguous(),
                              st[b:b + 1].contiguous(), en[b:b + 1].contiguous(), M, window, slopes)
        n = ns[b]
        assert torch.equal(ob[0, :n], o[b, :n]) and torch.equal(lb[0, :, :n], lse[b, :, :n]), f"row {b} alone"


@pytest.mark.parametrize("M", [5, 64, 300, 1000])
@pytest.mark.parametrize("D,G", [(64, 1), (128, 4), (64, 8)])
@pytest.mark.parametrize("mode", ["plain", "window", "alibi"])
def test_decode_ring_matches_fp64(M, D, G, mode):
    _ops()
    C = -(-M // 256) * 256
    ends = [1, 3, 5, M - 1, C - 1, C, C + 1, 4 * C + 3, 11 * C + 250]
    Hk = 2
    H = Hk * G
    q, k, v, C2 = _ring_inputs(len(ends), 1, H, Hk, D, M, ends, [1] * len(ends), seed=M + D + G)
    assert C2 == C
    q = q[:, 0].contiguous()
    en = torch.tensor(ends, dtype=torch.int32, device="cuda")
    window = 40 if mode == "window" else -1
    slopes = None
    if mode == "alibi":
        from mlx_cuda_distributed_pretraining_b200.arch.flash_attention import alibi_slopes
        slopes = alibi_slopes(H).float().cuda()
    o, lse, intact = _dec_ring(q, k, v, en, M, window, slopes)
    assert intact, "write outside o / lse"
    RK.check_rows(q.cpu()[:, None], k.cpu(), v.cpu(), [e - 1 for e in ends], ends, o.cpu()[:, None],
                  lse.cpu()[:, :, None], M, None if window < 0 else window, None if slopes is None else slopes.cpu(),
                  f"decode_ring M={M} {mode}")
    o2, lse2, _ = _dec_ring(q, k, v, en, M, window, slopes)
    assert torch.equal(o, o2) and torch.equal(lse, lse2), "not bit-identical on repeat"
    b = len(ends) - 1
    ob, lb, _ = _dec_ring(q[b:b + 1].contiguous(), k[b:b + 1].contiguous(), v[b:b + 1].contiguous(),
                          en[b:b + 1].contiguous(), M, window, slopes)
    assert torch.equal(ob[0], o[b]) and torch.equal(lb[0], lse[b]), "row alone"


@pytest.mark.parametrize("layout", ["none", "interleaved", "half"])
def test_kv_append_ring_bit_equal(layout):
    ops = _ops()
    B, H, Hk, D, C = 3, 8, 2, 128, 256
    g = torch.Generator().manual_seed(5)
    q = torch.randn(B, H, D, generator=g).to(torch.bfloat16).cuda()
    k = torch.randn(B, Hk, D, generator=g).to(torch.bfloat16).cuda()
    v = torch.randn(B, Hk, D, generator=g).to(torch.bfloat16).cuda()
    ends = [3, 700, 1000]
    tables = None if layout == "none" else ops.rope_tables(1024, D, 10000.0, "cuda")
    lay = "half" if layout == "half" else "interleaved"
    # the reference: b200_kv_append(_half) into an unbounded cache at the same positions
    kc = torch.zeros(B, 1024, Hk, D, dtype=torch.bfloat16, device="cuda")
    vc = torch.zeros_like(kc)
    q_ref = q.clone()
    ops.kv_append(q_ref, k, v, kc, vc, torch.tensor(ends, dtype=torch.int32, device="cuda"), tables, lay)
    kr = torch.full((B, C, Hk, D), float("nan"), dtype=torch.bfloat16, device="cuda")
    vr = torch.full_like(kr, float("nan"))
    q_ring = q.clone()
    live = torch.tensor([1, 0, 1], dtype=torch.int32, device="cuda")
    ops.kv_append_ring(q_ring, k, v, kr, vr, torch.tensor(ends, dtype=torch.int32, device="cuda"), live, tables, lay)
    torch.cuda.synchronize()
    for b in (0, 2):
        s = ring_slot(ends[b] - 1, C)
        assert torch.equal(kr[b, s], kc[b, ends[b] - 1]) and torch.equal(vr[b, s], vc[b, ends[b] - 1])
        assert torch.equal(q_ring[b], q_ref[b])
        others = torch.ones(C, dtype=torch.bool)
        others[s] = False
        assert bool(torch.isnan(kr[b, others.cuda()]).all()), "wrote outside its slot"
    assert bool(torch.isnan(kr[1]).all() and torch.isnan(vr[1]).all()), "a stopped row was written"
    assert torch.equal(q_ring[1], q[1]), "a stopped row's q was rotated"


# -- model level -----------------------------------------------------------------------------------------------------
def _teacher(model, prompts, cache, after, step):
    from mlx_cuda_distributed_pretraining_b200.core.generation import _prefill
    out = [_prefill(model, prompts, cache, step)]
    for t in after:
        out.append(model.decode_step(t, cache))
    return torch.stack(out, 1)


@pytest.mark.parametrize("kind", ["bf16_rope", "window", "alibi"])
def test_model_ring_matches_unbounded(kind):
    from mlx_cuda_distributed_pretraining_b200.arch.llama import KVCache
    from tests.test_gpu_generation import _rel_rows
    model = _trainer(kind).model
    g = torch.Generator().manual_seed(3)
    T = 300
    tokens = torch.randint(0, 256, (2, T + 40), generator=g)
    prompts = [tokens[0, :T].tolist(), tokens[1, :217].tolist()]
    after = [torch.tensor([tokens[0, T + i], tokens[1, 217 + i]]).cuda() for i in range(40)]
    ref = _teacher(model, prompts, KVCache(model, 2, T + 48), after, 128)
    tol = _tol(kind)
    # a ring at least as long as every row sees what the unbounded cache shows; steps 64 and 512 agree
    for step in (64, 512):
        got = _teacher(model, prompts, KVCache(model, 2, 0, max_kv_size=T + 41, max_chunk=step), after, step)
        assert _rel_rows(got, ref) < tol, f"{kind} step {step}"
    if kind == "window":  # W = 64: a ring of W + 5 keeps exactly the window
        got = _teacher(model, prompts, KVCache(model, 2, 0, max_kv_size=69, max_chunk=64), after, 64)
        assert _rel_rows(got, ref) < tol, "window ring"


def test_two_turns_through_rotating_prompt_cache_equal_one_pass():
    # M = 64 in a ring of 256 slots: every row wraps, and in turn 2 a row stops at EOS while the other goes on
    import copy
    from mlx_cuda_distributed_pretraining_b200.arch.llama import KVCache
    from mlx_cuda_distributed_pretraining_b200.core.generation import _prefill, generate
    from tests.test_gpu_generation import _rel_rows
    model = _trainer("alibi").model
    g = torch.Generator().manual_seed(9)
    p1 = [torch.randint(0, 256, (n,), generator=g).tolist() for n in (300, 270)]
    p2 = [torch.randint(0, 256, (n,), generator=g).tolist() for n in (30, 70)]
    kw = dict(max_tokens=24, temperature=0, repetition_penalty=1.0, prefill_step_size=64)
    cache = KVCache(model, 2, 0, max_kv_size=64, max_chunk=64)
    nbytes = cache.nbytes()
    out1 = generate(model, p1, prompt_cache=cache, **kw)
    assert cache.host_lens == [len(p) + len(o) for p, o in zip(p1, out1)]
    assert min(cache.host_lens) > cache.s_max, "every row must wrap the ring"
    # an EOS that stops some row early: a token the undisturbed turn 2 yields late in some row
    dry = generate(model, p2, prompt_cache=copy.deepcopy(cache), **kw)
    eos = None
    for b, o in enumerate(dry):
        firsts = [i for i, t in enumerate(o) if t not in o[:i]]
        if len(firsts) > 1:
            eos = o[firsts[-1]]
            break
    if eos is None:
        eos = dry[1][0]
    out2 = generate(model, p2, prompt_cache=cache, eos_token=eos, **kw)
    assert any(len(o) < kw["max_tokens"] for o in out2), "no row stopped early"
    assert cache.nbytes() == nbytes
    whole = [a + b + c + d for a, b, c, d in zip(p1, out1, p2, out2)]
    assert cache.host_lens == [len(w) for w in whole]
    # one pass over each row's whole sequence, then the same fresh token into both caches
    one = KVCache(model, 2, 0, max_kv_size=64, max_chunk=64)
    _prefill(model, whole, one, 64)
    fresh = torch.tensor([7, 11], device="cuda")
    got, ref = model.decode_step(fresh, cache), model.decode_step(fresh, one)
    err = _rel_rows(got, ref)
    assert err < _tol("alibi"), f"two turns vs one pass {err:.2e}"


def _fp64_logits(model, seq, M):
    """fp64 logits [T, V] after every position of seq under the rotating cache's rule: a restatement of a
    non-RoPE ALiBi dense model (RMSNorm, the sigmoid2 MLP, tied or untied logits) in torch fp64 on the CPU."""
    from mlx_cuda_distributed_pretraining_b200.arch.flash_attention import alibi_slopes
    a = model.args
    P = {n: t.detach().double().cpu() for n, t in model.named_parameters()}
    H, Hk = a.num_attention_heads, a.num_key_value_heads
    D = model.layers[0].self_attn.head_dim
    T = len(seq)

    def norm(x, w):
        return x * torch.rsqrt((x * x).mean(-1, keepdim=True) + a.rms_norm_eps) * w

    pos = torch.arange(T)
    mask = RK.rule(pos[:, None], pos[None, :], M, a.sliding_window)
    m = alibi_slopes(H).double()
    bias = m[:, None, None] * (pos[None, :] - pos[:, None]).double()[None]
    x = P["embed_tokens.weight"][torch.tensor(seq)]
    for i in range(a.num_hidden_layers):
        pre = f"layers.{i}."
        y = norm(x, P[pre + "input_layernorm.weight"])
        at = pre + "self_attn.attn."
        q = (y @ P[at + "q_proj.weight"].T).view(T, H, D).transpose(0, 1)
        k = (y @ P[at + "k_proj.weight"].T).view(T, Hk, D).transpose(0, 1).repeat_interleave(H // Hk, 0)
        v = (y @ P[at + "v_proj.weight"].T).view(T, Hk, D).transpose(0, 1).repeat_interleave(H // Hk, 0)
        sc = (q @ k.transpose(-1, -2)) * D ** -0.5 + bias
        sc = sc.masked_fill(~mask[None], float("-inf"))
        ctx = (torch.softmax(sc, -1) @ v).transpose(0, 1).reshape(T, H * D)
        x = x + ctx @ P[at + "o_proj.weight"].T
        y = norm(x, P[pre + "post_attention_layernorm.weight"])
        gt, up = y @ P[pre + "mlp.gate_proj.weight"].T, y @ P[pre + "mlp.up_proj.weight"].T
        x = x + (gt * torch.sigmoid(up) * 2) @ P[pre + "mlp.down_proj.weight"].T
    w = P["lm_head.weight"] if "lm_head.weight" in P else P["embed_tokens.weight"]
    return norm(x, P["norm.weight"]) @ w[:a.vocab_size].T


def test_alibi_long_generation_constant_memory_tracks_fp64():
    from mlx_cuda_distributed_pretraining_b200.arch.llama import KVCache
    from mlx_cuda_distributed_pretraining_b200.core.generation import _prefill
    from tests.test_gpu_generation import _rel_rows
    model = _trainer("alibi").model
    assert not model.args.apply_rope and model.logit_scale is None and not model.args.num_local_experts
    M = 64
    cache = KVCache(model, 1, 0, max_kv_size=M, max_chunk=64)
    nbytes = cache.nbytes()
    g = torch.Generator().manual_seed(2)
    seq = torch.randint(0, 256, (100,), generator=g).tolist()
    logits = [_prefill(model, [seq], cache, 64)[0]]
    for _ in range(4 * cache.s_max):
        t = int(torch.argmax(logits[-1]))
        seq.append(t)
        logits.append(model.decode_step(torch.tensor([t], device="cuda"), cache)[0])
        assert cache.nbytes() == nbytes
    assert cache.host_lens == [len(seq)] and len(seq) > 4 * cache.s_max
    ref = _fp64_logits(model, seq, M)[99:]
    got = torch.stack(logits)
    errs = [_rel_rows(got[i:i + 1], ref[i:i + 1]) for i in range(0, len(got), 64)]
    err = _rel_rows(got, ref)
    print(f"fp64 restatement over {len(seq)} positions: worst {err:.2e}, every 64th step {errs}")
    assert err < _tol("alibi"), f"decode over a ring vs fp64 restatement {err:.2e}"


def test_cli_max_kv_size_end_to_end():
    import os
    import subprocess
    import sys
    import tempfile
    from pathlib import Path

    import yaml
    root = Path(__file__).resolve().parents[1]
    env = dict(os.environ, PYTHONPATH=str(root) + os.pathsep + os.environ.get("PYTHONPATH", ""))
    with tempfile.TemporaryDirectory(prefix="ring_e2e_") as tmp:
        cfg = yaml.safe_load((root / "configs" / "c1-llama2m-adamw.yaml").read_text())
        cfg["name"] = "ring-e2e"
        cfg["data"]["input_file"] = "synthetic:markov"
        cfg["data"]["preprocessing"]["max_context_size"] = 128
        cfg["training"]["hyperparameters"]["iters"] = 3
        cfg["model"]["attention"].update(num_heads=4, num_kv_heads=2, head_dim=64)
        cfg["system"]["mixed_precision"] = True
        cfg_path = Path(tmp) / "cfg.yaml"
        cfg_path.write_text(yaml.safe_dump(cfg))
        subprocess.run([sys.executable, "-m", "core.training", "--config", str(cfg_path)], cwd=tmp, env=env,
                       check=True, timeout=600)
        out = subprocess.run([sys.executable, "-m", "core.generation", "--run", "ring-e2e", "--runs-dir",
                              str(Path(tmp) / "runs"), "--prompt", "hello there", "--max-tokens", "100", "--seed", "0",
                              "--max-kv-size", "64", "--num-samples", "2"],
                             cwd=root, env=env, check=True, capture_output=True, text=True, timeout=600).stdout
        assert sum(l.startswith("Greedy Output: ") for l in out.splitlines()) == 2
