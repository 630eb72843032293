"""Times the rotating KV cache (max_kv_size) on the GPU and prints one JSON line per measurement.

1. Decode attention alone: b200_attn_decode_ring against b200_attn_decode over the same number of visible keys M.
   C2 heads (H16/Hk8, D64) and C5 heads (H16/Hk16, D128), B32, M in {4096, 8192}.  The ring has C = M + 511 slots
   (rounded up to 256, the default step's ring) and every row has wrapped it several times (end = 3.5 C); the plain
   cache holds M positions.  Both are timed in alternating rounds (CUDA events over --iters calls each) and the
   medians reported.
2. Per-token generation time and cache bytes of a C2-shaped model (random weights, max_position_embeddings raised to
   8192) at B32: a 3968-token prompt in 512-token chunks, then --gen-tokens greedy decode steps, with M = 2048 and
   with the unbounded cache.
3. Cache bytes for C5 (16 layers) at B32 x 32768, from shapes, with and without M = 4096.

    python scripts/rotating_kv_bench.py [--iters 50] [--rounds 5] [--gen-tokens 4096] [--skip-model]
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


def ring_slots(M, step=512):
    return -(-(M + step - 1) // 256) * 256


def bench_attention(iters, rounds):
    from mlx_cuda_distributed_pretraining_b200 import ops
    B = 32
    for name, H, Hk, D in (("C2", 16, 8, 64), ("C5", 16, 16, 128)):
        for M in (4096, 8192):
            C = ring_slots(M)
            q = torch.randn(B, H, D, device="cuda", dtype=torch.bfloat16)
            kr = torch.randn(B, C, Hk, D, device="cuda", dtype=torch.bfloat16)
            vr = torch.randn(B, C, Hk, D, device="cuda", dtype=torch.bfloat16)
            end = torch.full((B,), int(3.5 * C), device="cuda", dtype=torch.int32)
            kp = torch.randn(B, M, Hk, D, device="cuda", dtype=torch.bfloat16)
            vp = torch.randn(B, M, Hk, D, device="cuda", dtype=torch.bfloat16)
            lens = torch.full((B,), M, device="cuda", dtype=torch.int32)
            ws = torch.empty(ops.attention_decode_workspace_bytes(B, H, C, D), device="cuda", dtype=torch.uint8)
            calls = {"plain": lambda: ops.attention_decode(q, kp, vp, lens, workspace=ws),
                     "ring": lambda: ops.attention_decode_ring(q, kr, vr, end, M, workspace=ws)}
            times = {f: [] for f in calls}
            for _ in range(rounds):
                for f, fn in calls.items():
                    times[f].append(time_ms(fn, iters))
            nbytes = B * 2 * M * Hk * D * 2
            row = {"bench": "attn_decode_ring", "shape": name, "B": B, "max_kv_size": M, "slots": C,
                   "end": int(3.5 * C)}
            for f in calls:
                ms = statistics.median(times[f])
                row[f"{f}_ms"] = round(ms, 4)
                row[f"{f}_TB_s"] = round(nbytes / ms / 1e9, 3)
                row[f"{f}_spread_ms"] = round(max(times[f]) - min(times[f]), 4)
            row["ring_over_plain"] = round(row["ring_ms"] / row["plain_ms"], 3)
            print(json.dumps(row), flush=True)
            del q, kr, vr, kp, vp, ws
            torch.cuda.empty_cache()


def bench_model(gen_tokens):
    import yaml
    from mlx_cuda_distributed_pretraining_b200.arch.llama import KVCache
    from mlx_cuda_distributed_pretraining_b200.core.generation import _prefill
    from mlx_cuda_distributed_pretraining_b200.core.training import Config, Trainer
    cfg = yaml.safe_load((ROOT / "configs" / "c2-llama80m-muon.yaml").read_text())
    cfg["data"]["input_file"] = "synthetic"
    cfg["model"]["attention"]["max_position_embeddings"] = 8192
    with tempfile.TemporaryDirectory() as tmp:
        tr = Trainer(Config.from_dict(cfg), for_training=False, quiet=True, run_root=tmp)
    model = tr.model
    B, prompt = 32, 3968
    g = torch.Generator().manual_seed(0)
    prompts = torch.randint(0, 256, (B, prompt), generator=g).tolist()
    for M in (2048, None):
        cache = (KVCache(model, B, 0, max_kv_size=M, max_chunk=512) if M
                 else KVCache(model, B, prompt + gen_tokens))
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        logits = _prefill(model, prompts, cache, 512)
        torch.cuda.synchronize()
        prefill_s = time.perf_counter() - t0
        nxt = torch.argmax(logits, -1)
        seg, marks = [], [time.perf_counter()]
        for i in range(gen_tokens):
            nxt = torch.argmax(model.decode_step(nxt, cache), -1)
            if (i + 1) % 1024 == 0 or i + 1 == gen_tokens:
                torch.cuda.synchronize()
                marks.append(time.perf_counter())
                seg.append(round((marks[-1] - marks[-2]) / ((i % 1024) + 1) * 1e3, 3))
        row = {"bench": "generate", "model": "C2-shaped", "B": B, "prompt": prompt, "gen_tokens": gen_tokens,
               "max_kv_size": M, "prefill_s": round(prefill_s, 3),
               "decode_ms_per_token": round((marks[-1] - marks[0]) / gen_tokens * 1e3, 3),
               "decode_ms_per_token_by_1024": seg, "cache_MB": round(cache.nbytes() / 1e6, 1)}
        print(json.dumps(row), flush=True)
        del cache
        torch.cuda.empty_cache()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--gen-tokens", type=int, default=4096)
    ap.add_argument("--skip-model", action="store_true")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("rotating_kv_bench.py needs a CUDA device")
    print(json.dumps({"gpu": gpu_info()}), flush=True)
    layers, B, ctx, Hk, D, M = 16, 32, 32768, 16, 128, 4096
    per_pos = layers * B * 2 * Hk * D * 2
    print(json.dumps({"bench": "cache_bytes", "shape": "C5 (16 layers)", "B": B, "context": ctx,
                      "unbounded_GB": round(per_pos * ctx / 1e9, 1),
                      f"max_kv_size_{M}_GB": round(per_pos * ring_slots(M) / 1e9, 1)}), flush=True)
    bench_attention(a.iters, a.rounds)
    if not a.skip_model:
        bench_model(a.gen_tokens)
    print(json.dumps({"gpu_after": gpu_info()}), flush=True)


if __name__ == "__main__":
    main()
