"""Times chunked prefill and prompt-cache continuation on the GPU and prints one JSON line per measurement.

1. b200_attn_fwd_cached alone against b200_attn_fwd causal: C2 heads (H16/Hk8, D64) and C5 heads (H16/Hk16, D128),
   B 1 and 16, start 0 and 2048, chunk L 128, 512 and 2048.  Each shape alternates the two kernels over --rounds
   rounds (CUDA events over --iters calls each) and reports the medians.  The causal forward runs its own square
   problem, S = L (start 0) or S = start + L (start 2048, all rows, of which the chunk is the last L).  FLOPs are
   4 D x (visible query-key pairs) computed from shapes.
2. Generation, C2-shaped model (random weights), B16, a 3968-token prompt: one-shot prefill against
   prefill_step_size 512 and 2048, bf16 and 4-bit caches: time and peak torch.cuda.max_memory_allocated.
3. Multi-turn: a 128-token turn continuing that 3968-token cache (4096 in all) against re-prefilling all 4096 tokens.

    python scripts/prefill_chunk_bench.py [--iters 20] [--rounds 5] [--skip-model]
"""
from __future__ import annotations

import argparse
import json
import statistics
import subprocess
import sys
import tempfile
import time
from pathlib import Path

import torch

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))


def gpu_info():
    return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                          capture_output=True, text=True, timeout=30, check=True).stdout.strip().splitlines()[0]


def time_ms(fn, iters):
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters


def causal_pairs(start, L):
    """Query-key pairs visible to queries start .. start + L - 1 under the causal mask."""
    return L * start + L * (L + 1) // 2


def bench_kernels(iters, rounds):
    from mlx_cuda_distributed_pretraining_b200 import ops
    for heads, H, Hk, D in (("C2", 16, 8, 64), ("C5", 16, 16, 128)):
        for B in (1, 16):
            for start in (0, 2048):
                for L in (128, 512, 2048):
                    S = start + L
                    q = torch.randn(B, L, H, D, device="cuda", dtype=torch.bfloat16)
                    kc = torch.randn(B, S, Hk, D, device="cuda", dtype=torch.bfloat16)
                    vc = torch.randn_like(kc)
                    qf = torch.randn(B, S, H, D, device="cuda", dtype=torch.bfloat16)
                    st = torch.full((B,), start, device="cuda", dtype=torch.int32)
                    en = torch.full((B,), S, device="cuda", dtype=torch.int32)
                    cached = lambda: ops.attention_cached(q, kc, vc, st, en)  # noqa: E731
                    causal = lambda: ops.attention_fwd_raw(qf, kc, vc, D ** -0.5, True)  # noqa: E731
                    tc, tf = [], []
                    for _ in range(rounds):
                        tc.append(time_ms(cached, iters))
                        tf.append(time_ms(causal, iters))
                    mc, mf = statistics.median(tc), statistics.median(tf)
                    fc = 4 * D * causal_pairs(start, L) * B * H
                    ff = 4 * D * causal_pairs(0, S) * B * H
                    print(json.dumps({"bench": "attn_cached", "heads": heads, "B": B, "start": start, "L": L,
                                      "cached_ms": round(mc, 4), "cached_TFLOPs": round(fc / mc / 1e9, 1),
                                      "causal_S": S, "causal_ms": round(mf, 4),
                                      "causal_TFLOPs": round(ff / mf / 1e9, 1)}), flush=True)
                    del q, kc, vc, qf
                    torch.cuda.empty_cache()


def bench_model():
    import yaml
    from mlx_cuda_distributed_pretraining_b200.arch.llama import KVCache
    from mlx_cuda_distributed_pretraining_b200.core.generation import _prefill
    from mlx_cuda_distributed_pretraining_b200.core.training import Config, Trainer
    cfg = yaml.safe_load((ROOT / "configs" / "c2-llama80m-muon.yaml").read_text())
    cfg["data"]["input_file"] = "synthetic"
    with tempfile.TemporaryDirectory() as tmp:
        tr = Trainer(Config.from_dict(cfg), for_training=False, quiet=True, run_root=tmp)
    model = tr.model
    B, prompt, turn = 16, 3968, 128
    tokens = torch.randint(0, 256, (B, prompt + turn), generator=torch.Generator().manual_seed(0))
    prompts = [tokens[b, :prompt].tolist() for b in range(B)]
    turns = [tokens[b, prompt:].tolist() for b in range(B)]
    whole = [tokens[b].tolist() for b in range(B)]

    def timed(fn):
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats()
        base = torch.cuda.memory_allocated()
        t0 = time.perf_counter()
        out = fn()
        torch.cuda.synchronize()
        return out, (time.perf_counter() - t0) * 1e3, (torch.cuda.max_memory_allocated() - base) / 1e6

    for rnd in range(2):  # the second round is reported; the first warms every shape
        for bits in (None, 4):
            row = {"bench": "prefill", "model": "C2-shaped", "B": B, "prompt": prompt, "kv_bits": bits}
            for step in (None, 512, 2048):
                cache = KVCache(model, B, prompt + turn, kv_bits=bits)
                _, ms, mb = timed(lambda: _prefill(model, prompts, cache, step))
                key = "one_shot" if step is None else f"step{step}"
                row[f"{key}_ms"], row[f"{key}_peak_MB"] = round(ms, 2), round(mb, 1)
                if step == 512:  # continue this conversation with a 128-token turn
                    _, ms_turn, _ = timed(lambda: _prefill(model, turns, cache, None))
                    row["turn128_ms"] = round(ms_turn, 2)
                del cache
                torch.cuda.empty_cache()
            cache = KVCache(model, B, prompt + turn, kv_bits=bits)
            _, ms, _ = timed(lambda: _prefill(model, whole, cache, None))
            row["reprefill4096_ms"] = round(ms, 2)
            del cache
            torch.cuda.empty_cache()
            if rnd == 1:
                print(json.dumps(row), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--skip-model", action="store_true")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("prefill_chunk_bench.py needs a CUDA device")
    print(json.dumps({"gpu": gpu_info()}), flush=True)
    with torch.no_grad():
        bench_kernels(a.iters, a.rounds)
        if not a.skip_model:
            bench_model()


if __name__ == "__main__":
    main()
