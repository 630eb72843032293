"""Times the quantized KV cache on the GPU and prints one JSON line per measurement.

1. Decode attention alone: b200_attn_decode (bf16 cache) against b200_attn_decode_quant at 8 and 4 bits (group 64),
   C2 heads (H16/Hk8, D64) and C5 heads (H16/Hk16, D128), B32 at contexts 8192 and 32768, plus a 1024-key window at
   32768.  The three formats are timed in alternating rounds (CUDA events over --iters calls each) and the medians
   reported.  Bytes read are computed from shapes: the visible keys' K and V codes plus their (scale, bias) pairs.
2. b200_kv_append_quant (one token, B32, C5 heads) and b200_kv_quantize (B32 x 8192, C5 heads) times.
3. Per-token generation time of a C2-shaped model (random weights) at B32 with a 3968-token prompt: bf16, 8- and
   4-bit caches, plus the bytes each cache holds.
4. Cache bytes per format for C5 (16 layers) at B32 x 32768, computed from shapes.

    python scripts/kv_quant_bench.py [--iters 50] [--rounds 5] [--skip-model]
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

G = 64
FORMATS = ("bf16", 8, 4)


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True, timeout=30, check=True).stdout.strip().splitlines()[0]
    return q


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


def cache_bytes(fmt, tokens, Hk, D):
    """K + V bytes of `tokens` cached positions of one layer."""
    if fmt == "bf16":
        return 2 * tokens * Hk * D * 2
    return 2 * tokens * Hk * (D * fmt // 8 + D // G * 8)


def bench_attention(iters, rounds):
    from mlx_cuda_distributed_pretraining_b200 import ops
    B = 32
    cases = [("C2", 16, 8, 64, 8192, None), ("C2", 16, 8, 64, 32768, None), ("C2", 16, 8, 64, 32768, 1024),
             ("C5", 16, 16, 128, 8192, None), ("C5", 16, 16, 128, 32768, None), ("C5", 16, 16, 128, 32768, 1024)]
    for name, H, Hk, D, ctx, window in cases:
        q = torch.randn(B, H, D, device="cuda", dtype=torch.bfloat16)
        k = torch.randn(B, ctx, Hk, D, device="cuda", dtype=torch.bfloat16)
        v = torch.randn(B, ctx, Hk, D, device="cuda", dtype=torch.bfloat16)
        lens = torch.full((B,), ctx, device="cuda", dtype=torch.int32)
        ws = torch.empty(ops.attention_decode_workspace_bytes(B, H, ctx, D), device="cuda", dtype=torch.uint8)
        quant = {}
        for bits in (8, 4):
            cs, ps = ops.kv_quant_shapes(B, ctx, Hk, D, bits, G)
            bufs = (torch.empty(cs, device="cuda", dtype=torch.uint8), torch.empty(cs, device="cuda", dtype=torch.uint8),
                    torch.empty(ps, device="cuda"), torch.empty(ps, device="cuda"))
            ops.kv_quantize(k, v, *bufs, bits, G)
            quant[bits] = bufs
        calls = {"bf16": lambda: ops.attention_decode(q, k, v, lens, workspace=ws, window=window)}
        for bits in (8, 4):
            calls[bits] = (lambda b=bits: ops.attention_decode_quant(q, *quant[b], lens, b, G, workspace=ws,
                                                                     window=window))
        times = {f: [] for f in FORMATS}
        for _ in range(rounds):
            for f in FORMATS:
                times[f].append(time_ms(calls[f], iters))
        visible = ctx if window is None else window + 1
        row = {"bench": "attn_decode", "shape": name, "B": B, "context": ctx, "window": window, "group": G}
        for f in FORMATS:
            ms = statistics.median(times[f])
            nbytes = B * cache_bytes(f, visible, Hk, D)
            row[f"{f}_ms"] = round(ms, 4)
            row[f"{f}_TB_s"] = round(nbytes / ms / 1e9, 3)
            row[f"{f}_spread_ms"] = round(max(times[f]) - min(times[f]), 4)
        row["speedup_8bit"] = round(row["bf16_ms"] / row["8_ms"], 3)
        row["speedup_4bit"] = round(row["bf16_ms"] / row["4_ms"], 3)
        print(json.dumps(row), flush=True)
        del q, k, v, quant, ws
        torch.cuda.empty_cache()


def bench_writes(iters):
    from mlx_cuda_distributed_pretraining_b200 import ops
    B, H, Hk, D, ctx = 32, 16, 16, 128, 8192
    q = torch.randn(B, H, D, device="cuda", dtype=torch.bfloat16)
    k1 = torch.randn(B, Hk, D, device="cuda", dtype=torch.bfloat16)
    v1 = torch.randn(B, Hk, D, device="cuda", dtype=torch.bfloat16)
    lens = torch.full((B,), ctx // 2, device="cuda", dtype=torch.int32)
    tables = ops.rope_tables(ctx, D, 10000.0, "cuda")
    k = torch.randn(B, ctx, Hk, D, device="cuda", dtype=torch.bfloat16)
    v = torch.randn(B, ctx, Hk, D, device="cuda", dtype=torch.bfloat16)
    kc = torch.zeros_like(k)
    vc = torch.zeros_like(v)
    row = {"bench": "cache_writes", "shape": "C5", "B": B, "append_ms_bf16": round(
        time_ms(lambda: ops.kv_append(q, k1, v1, kc, vc, lens, tables), iters), 4)}
    for bits in (8, 4):
        cs, ps = ops.kv_quant_shapes(B, ctx, Hk, D, bits, G)
        bufs = (torch.empty(cs, device="cuda", dtype=torch.uint8), torch.empty(cs, device="cuda", dtype=torch.uint8),
                torch.empty(ps, device="cuda"), torch.empty(ps, device="cuda"))
        row[f"append_ms_{bits}bit"] = round(
            time_ms(lambda: ops.kv_append_quant(q, k1, v1, *bufs, lens, bits, G, tables), iters), 4)
        ms = time_ms(lambda: ops.kv_quantize(k, v, *bufs, bits, G), iters)
        nbytes = 2 * k.numel() * 2 + cache_bytes(bits, B * ctx, Hk, D)
        row[f"quantize_{ctx}_ms_{bits}bit"] = round(ms, 4)
        row[f"quantize_TB_s_{bits}bit"] = round(nbytes / ms / 1e9, 3)
    print(json.dumps(row), flush=True)


def bench_model():
    import yaml
    from mlx_cuda_distributed_pretraining_b200.arch.llama import KVCache
    from mlx_cuda_distributed_pretraining_b200.core.training import Config, Trainer
    cfg = yaml.safe_load((ROOT / "configs" / "c2-llama80m-muon.yaml").read_text())
    cfg["data"]["input_file"] = "synthetic"
    with tempfile.TemporaryDirectory() as tmp:
        tr = Trainer(Config.from_dict(cfg), for_training=False, quiet=True, run_root=tmp)
    model = tr.model
    B, prompt, steps = 32, 3968, 64
    tokens = torch.randint(0, 256, (B, prompt), device="cuda")
    for rnd in range(2):  # the second round is reported; the first warms every shape
        row = {"bench": "generate", "model": "C2-shaped", "B": B, "prompt": prompt, "decode_steps": steps}
        for f in FORMATS:
            cache = KVCache(model, B, prompt + steps, kv_bits=None if f == "bf16" else f)
            logits = model.prefill(tokens, [prompt] * B, cache)
            nxt = torch.argmax(logits, -1)
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            for _ in range(steps):
                nxt = torch.argmax(model.decode_step(nxt, cache), -1)
            torch.cuda.synchronize()
            row[f"{f}_decode_step_ms"] = round((time.perf_counter() - t0) / steps * 1e3, 3)
            row[f"{f}_cache_MB"] = round(cache.nbytes() / 1e6, 1)
            del cache
            torch.cuda.empty_cache()
        if rnd == 1:
            print(json.dumps(row), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--skip-model", action="store_true")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("kv_quant_bench.py needs a CUDA device")
    print(json.dumps({"gpu": gpu_info()}), flush=True)
    layers, B, ctx, Hk, D = 16, 32, 32768, 16, 128
    print(json.dumps({"bench": "cache_bytes", "shape": "C5 (16 layers)", "B": B, "context": ctx, "group": G,
                      **{f"{f}_GB": round(layers * B * cache_bytes(f, ctx, Hk, D) / 1e9, 1) for f in FORMATS}}),
          flush=True)
    bench_attention(a.iters, a.rounds)
    bench_writes(a.iters)
    if not a.skip_model:
        bench_model()
    print(json.dumps({"gpu_after": gpu_info()}), flush=True)


if __name__ == "__main__":
    main()
