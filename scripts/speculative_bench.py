"""Speculative decoding's verify kernel and end-to-end rounds.  Prints one JSON line per measurement, with the card's
name and power limit.

  kernel: ops.attention_decode_multi (L queries per row) against ops.attention_cached on the same chunk (bf16, D 64 /
          128 only) and against L calls of ops.attention_decode; contexts 512 / 2048 / 8192, B 1 / 8 / 32, C2 heads
          (H16 / Hk8, D 64) and C5 heads (H32 / Hk8, D 64 at hidden 2048).  CUDA events over 50 launches, median of
          3 rounds.  GB/s counts the K and V bytes of positions [0, end) once per row.
  e2e:    a C2-shaped target (24 layers, hidden 1024, bf16, random weights) and a small draft of the same width (2
          layers), B 1 and 8, a 512-token prompt, 128 tokens, K = 3: plain decode step, draft step, verify step, and
          tokens/s with the target as its own draft (every draft accepted) and with the random draft.  speedup(a) =
          derived from the measured step times for acceptance rate a, not measured.

    python scripts/speculative_bench.py [--quick]
"""
from __future__ import annotations

import argparse
import json
import subprocess
import sys
import time
from pathlib import Path

import torch

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))

from mlx_cuda_distributed_pretraining_b200 import ops  # noqa: E402
from mlx_cuda_distributed_pretraining_b200.arch import llama  # noqa: E402
from mlx_cuda_distributed_pretraining_b200.core import generation as gen  # noqa: E402

PEAK = 3.35e12


def card():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip().splitlines()
    return out[0] if out else "unknown"


def ms(fn, n=50, rounds=3):
    fn()
    torch.cuda.synchronize()
    res = []
    for _ in range(rounds):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        for _ in range(n):
            fn()
        b.record()
        torch.cuda.synchronize()
        res.append(a.elapsed_time(b) / n)
    return sorted(res)[len(res) // 2]


def kernels(quick):
    H_sets = {"c2": (16, 8, 64), "c5": (32, 8, 64)}
    for heads, (H, Hk, D) in H_sets.items():
        for ctx in ((2048,) if quick else (512, 2048, 8192)):
            for B in ((1, 8) if quick else (1, 8, 32)):
                s_max = ctx + 256
                kc = torch.randn(B, s_max, Hk, D, device="cuda", dtype=torch.bfloat16)
                vc = torch.randn_like(kc)
                for L in (1, 2, 4, 8, 16):
                    q = torch.randn(B, L, H, D, device="cuda", dtype=torch.bfloat16)
                    st = torch.full((B,), ctx - L, device="cuda", dtype=torch.int32)
                    en = torch.full((B,), ctx, device="cuda", dtype=torch.int32)
                    ws = torch.empty(ops.attention_decode_multi_workspace_bytes(B, L, H, s_max, D), device="cuda",
                                     dtype=torch.uint8)
                    dws = torch.empty(ops.attention_decode_workspace_bytes(B, H, s_max, D), device="cuda",
                                      dtype=torch.uint8)
                    lens = [torch.full((B,), ctx - L + i + 1, device="cuda", dtype=torch.int32) for i in range(L)]
                    qs = [q[:, i].contiguous() for i in range(L)]
                    t_multi = ms(lambda: ops.attention_decode_multi(q, kc, vc, st, en, workspace=ws))
                    t_cached = ms(lambda: ops.attention_cached(q, kc, vc, st, en))
                    t_dec = ms(lambda: [ops.attention_decode(qs[i], kc, vc, lens[i], workspace=dws)
                                        for i in range(L)])
                    nbytes = 2 * B * ctx * Hk * D * 2
                    print(json.dumps({"kind": "kernel", "heads": heads, "ctx": ctx, "B": B, "L": L,
                                      "multi_ms": round(t_multi, 4), "cached_ms": round(t_cached, 4),
                                      "L_decode_ms": round(t_dec, 4),
                                      "multi_GBps": round(nbytes / t_multi / 1e6, 1),
                                      "multi_frac_peak": round(nbytes / (t_multi * 1e-3) / PEAK, 3),
                                      "card": card()}), flush=True)


def model(layers, seed):
    a = llama.ModelArgs(model_type="llama", hidden_size=1024, num_hidden_layers=layers, intermediate_size=2816,
                        num_attention_heads=16, num_key_value_heads=8, head_dim=64, vocab_size=32000,
                        max_position_embeddings=4096, variant="mlx_lm", tie_word_embeddings=True)
    torch.manual_seed(seed)
    m = llama.Model(a).cuda().to(torch.bfloat16).eval()
    with torch.no_grad():
        for p in m.parameters():
            p.normal_(0, 0.02)
    return m


def timed(fn):
    torch.cuda.synchronize()
    t = time.perf_counter()
    r = fn()
    torch.cuda.synchronize()
    return r, time.perf_counter() - t


def e2e(quick):
    target, draft = model(24, 0), model(2, 1)
    P, N, K = 512, (32 if quick else 128), 3
    for B in (1, 8):
        prompts = [[(7 * b + i) % 30000 for i in range(P)] for b in range(B)]
        kw = dict(max_tokens=N, temperature=0, repetition_penalty=1.0, min_p=None)
        steps = {}
        for name, m in (("decode", target), ("draft", draft)):
            cache = llama.KVCache(m, B, P + N + 16)
            tok = torch.tensor([p for p in prompts], device="cuda")
            m.prefill(tok, [P] * B, cache)
            nxt = torch.zeros(B, dtype=torch.int64, device="cuda")
            steps[name] = ms(lambda: (m.decode_step(nxt, cache), cache.truncate([P] * B)), n=20)
        cache = llama.KVCache(target, B, P + N + 16)
        target.prefill(torch.tensor(prompts, device="cuda"), [P] * B, cache)
        vt = torch.zeros((B, K + 1), dtype=torch.int64, device="cuda")
        steps["verify"] = ms(lambda: (target.verify(vt, [K + 1] * B, cache), cache.truncate([P] * B)), n=20)
        gen.generate(target, prompts, **dict(kw, max_tokens=8))
        _, t_plain = timed(lambda: gen.generate(target, prompts, **kw))
        res = {"kind": "e2e", "B": B, "prompt": P, "tokens": N, "K": K,
               "decode_step_ms": round(steps["decode"], 3), "draft_step_ms": round(steps["draft"], 3),
               "verify_step_ms": round(steps["verify"], 3), "plain_tok_s": round(B * N / t_plain, 1)}
        for label, d in (("self", target), ("random", draft)):
            acc = [0, 0]

            def on_round(e, dr):
                for x, y in zip(e, dr):
                    n = 0
                    while n < min(len(x), len(y)) and x[n] == y[n]:
                        n += 1
                    acc[0] += n
                    acc[1] += len(y)

            gen.generate(target, prompts, draft_model=d, num_draft_tokens=K, **dict(kw, max_tokens=8))
            _, t = timed(lambda: gen.generate(target, prompts, draft_model=d, num_draft_tokens=K,
                                              on_round=on_round, **kw))
            res[f"{label}_draft_tok_s"] = round(B * N / t, 1)
            res[f"{label}_draft_acceptance"] = round(acc[0] / max(acc[1], 1), 3)
        # derived: a round costs 1 catch-up + (K - 1) draft steps + 1 verify and emits 1 + (accepted) tokens
        rnd = K * steps["draft"] + steps["verify"]
        res["derived_speedup"] = {str(a): round((1 + sum(a ** i for i in range(1, K + 1))) * steps["decode"] / rnd, 2)
                                  for a in (0.0, 0.5, 0.7, 0.9, 1.0)}
        res["card"] = card()
        print(json.dumps(res), flush=True)


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("--quick", action="store_true")
    ap.add_argument("--skip-kernels", action="store_true")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("speculative_bench: no GPU")
    if not a.skip_kernels:
        kernels(a.quick)
    e2e(a.quick)
