"""Beam search on a C2-shaped model: 24 layers, hidden 1024, H16 / Hk8, D 64, bf16 (K+V 48 KiB per position), random
weights, a 2048-token prompt and 128 steps, for G in {1, 8} prompts and n in {4, 8} beams.  Prints one JSON line per
configuration and one for the kernels.

  step_ms          beam_search's time per step after prefill (decode step + read-back + host selection + fork)
  greedy_step_ms   greedy generate's time per step at batch G over the same prompts
  fork_ms, forks, fork_bytes   per step: the kv_beam_fork launches' device time, copies and bytes copied
  select_ms        per step: host time from the logits to the next decode (read-back, selection, slot plan)
  cache_bytes / naive_bytes    the BeamKVCache against n full caches per prompt
  kernels: b200_attn_decode_beam against b200_attn_decode over G n materialised full caches and greedy at batch G,
           one layer, CUDA events over 200 launches (median of 5 rounds)

The card's name and power limit are printed with the numbers.

    python scripts/beam_bench.py [--steps 128] [--prompt 2048]
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


def card():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip().splitlines()
    return out[0] if out else "unknown"


def model_c2():
    a = llama.ModelArgs(model_type="llama", hidden_size=1024, num_hidden_layers=24, intermediate_size=2816,
                        num_attention_heads=16, num_key_value_heads=8, head_dim=64, vocab_size=32000,
                        max_position_embeddings=4096, variant="mlx_lm", tie_word_embeddings=True)
    torch.manual_seed(0)
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


def run_config(model, G, n, P, steps):
    g = torch.Generator().manual_seed(G * 100 + n)
    prompts = [torch.randint(0, 32000, (P,), generator=g).tolist() for _ in range(G)]
    stats = {"fork_ms": 0.0, "forks": 0, "fork_bytes": 0, "cache": 0, "select": 0.0, "mark": None}
    fork0 = llama.BeamKVCache.fork
    row_bytes = 2 * 24 * 8 * 64 * 2  # K and V, 24 layers, Hk 8, D 64, bf16

    def fork(self, copies):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        fork0(self, copies)
        e1.record()
        e1.synchronize()
        stats["fork_ms"] += e0.elapsed_time(e1)
        stats["forks"] += len(copies)
        stats["fork_bytes"] += sum(c[2] for c in copies) * row_bytes
        stats["cache"] = self.nbytes()

    def on_step(rows, logits):
        torch.cuda.synchronize()
        stats["mark"] = time.perf_counter()

    decode0 = model.decode_step

    def decode(tokens, cache, live=None):
        if stats["mark"] is not None:
            stats["select"] += time.perf_counter() - stats["mark"]
            stats["mark"] = None
        return decode0(tokens, cache, live)

    llama.BeamKVCache.fork = fork
    model.decode_step = decode
    try:
        gen.beam_search(model, prompts, n_beams=n, max_tokens=2)  # warm-up
        stats.update(fork_ms=0.0, forks=0, fork_bytes=0, select=0.0)
        _, t_pre = timed(lambda: gen.beam_search(model, prompts, n_beams=n, max_tokens=1))
        _, t_all = timed(lambda: gen.beam_search(model, prompts, n_beams=n, max_tokens=steps + 1, on_step=on_step))
    finally:
        llama.BeamKVCache.fork = fork0
        del model.decode_step
    gen.generate(model, prompts, max_tokens=2, temperature=0, repetition_penalty=1.0, min_p=None)
    _, g_pre = timed(lambda: gen.generate(model, prompts, max_tokens=1, temperature=0, repetition_penalty=1.0,
                                          min_p=None))
    _, g_all = timed(lambda: gen.generate(model, prompts, max_tokens=steps + 1, temperature=0,
                                          repetition_penalty=1.0, min_p=None))
    naive = G * n * 2 * 24 * (-(-(P + steps + 1) // 256) * 256) * 8 * 64 * 2
    return {"G": G, "n": n, "prompt": P, "steps": steps,
            "step_ms": round((t_all - t_pre) / steps * 1e3, 3),
            "greedy_step_ms": round((g_all - g_pre) / steps * 1e3, 3),
            "fork_ms": round(stats["fork_ms"] / steps, 4), "forks": round(stats["forks"] / steps, 2),
            "fork_bytes": int(stats["fork_bytes"] / steps), "select_ms": round(stats["select"] / steps * 1e3, 3),
            "cache_bytes": stats["cache"], "naive_bytes": naive}


def median_ms(fn, iters=200, rounds=5):
    fn()
    res = []
    for _ in range(rounds):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(iters):
            fn()
        e1.record()
        e1.synchronize()
        res.append(e0.elapsed_time(e1) / iters)
    return sorted(res)[len(res) // 2]


def kernels(G, n, P, steps):
    H, Hk, D = 16, 8, 64
    L = P + steps // 2
    t0 = 256 * (P // 256)
    s_prefix = -(-P // 256) * 256
    tail_cap = -(-(255 + steps) // 256) * 256
    R = G * n
    bf = dict(device="cuda", dtype=torch.bfloat16)
    q = torch.randn(R, H, D, **bf)
    kp, vp = torch.randn(G, s_prefix, Hk, D, **bf), torch.randn(G, s_prefix, Hk, D, **bf)
    kt, vt = torch.randn(R, tail_cap, Hk, D, **bf), torch.randn(R, tail_cap, Hk, D, **bf)
    groups = [r // n for r in range(R)]
    tables = torch.tensor(groups + list(range(R)) + [t0] * G + [g * n for g in range(G)] + [n] * G,
                          dtype=torch.int32, device="cuda")
    lens = torch.full((R,), L, dtype=torch.int32, device="cuda")
    ws = torch.empty(ops.attention_decode_beam_workspace_bytes(R, H, s_prefix, tail_cap, D), device="cuda",
                     dtype=torch.uint8)
    beam = median_ms(lambda: ops.attention_decode_beam(q, kp, vp, kt, vt, lens, tables, workspace=ws))
    s_max = -(-L // 256) * 256
    kc, vc = torch.randn(R, s_max, Hk, D, **bf), torch.randn(R, s_max, Hk, D, **bf)
    wsd = torch.empty(ops.attention_decode_workspace_bytes(R, H, s_max, D), device="cuda", dtype=torch.uint8)
    naive = median_ms(lambda: ops.attention_decode(q, kc, vc, lens, workspace=wsd))
    greedy = median_ms(lambda: ops.attention_decode(q[:G].contiguous(), kc[:G], vc[:G], lens[:G].contiguous(),
                                                    workspace=wsd))
    return {"G": G, "n": n, "keys": L, "beam_ms": round(beam, 4), "naive_n_caches_ms": round(naive, 4),
            "greedy_batch_G_ms": round(greedy, 4)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=128)
    ap.add_argument("--prompt", type=int, default=2048)
    a = ap.parse_args()
    ops.require_device()
    gpu = card()
    for G in (1, 8):
        for n in (4, 8):
            print(json.dumps({"kind": "attention", "gpu": gpu, **kernels(G, n, a.prompt, a.steps)}), flush=True)
    model = model_c2()
    for G in (1, 8):
        for n in (4, 8):
            print(json.dumps({"kind": "beam_step", "gpu": gpu, **run_config(model, G, n, a.prompt, a.steps)}),
                  flush=True)


if __name__ == "__main__":
    main()
