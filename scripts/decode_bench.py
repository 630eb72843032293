"""Times the decode path on the GPU and prints one JSON line per measurement.

1. Decode attention alone (b200_attn_decode, K/V cache bf16) at the C2 (H16/Hk8, D64) and C5 (H16/Hk16, D128) head
   shapes for B in {1, 8, 32} and context in {512, 2048, 8192}: CUDA-event time per call and K/V bytes over time,
   next to torch's scaled_dot_product_attention on the same inputs as a sanity baseline (it is not used anywhere).
2. Generation on a C2-shaped model (random weights): B in {1, 16}, a 128-token prompt, 256 new tokens, greedy.
   Prefill time and per-token decode time (host clock around synchronised work).

    python scripts/decode_bench.py [--iters 50] [--skip-model]
"""
from __future__ import annotations

import argparse
import json
import subprocess
import sys
import time
from pathlib import Path

import torch

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))


def gpu_info():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        return q
    except Exception as e:  # noqa: BLE001
        return f"unknown ({e})"


def time_ms(fn, iters):
    for _ in range(5):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters


def bench_kernel(iters):
    from mlx_cuda_distributed_pretraining_b200 import ops
    for name, H, Hk, D in (("C2", 16, 8, 64), ("C5", 16, 16, 128)):
        for B in (1, 8, 32):
            for ctx in (512, 2048, 8192):
                q = torch.randn(B, H, D, device="cuda", dtype=torch.bfloat16)
                kc = torch.randn(B, ctx, Hk, D, device="cuda", dtype=torch.bfloat16)
                vc = torch.randn(B, ctx, Hk, D, device="cuda", dtype=torch.bfloat16)
                lens = torch.full((B,), ctx, device="cuda", dtype=torch.int32)
                ws = torch.empty(ops.attention_decode_workspace_bytes(B, H, ctx, D), device="cuda", dtype=torch.uint8)
                ms = time_ms(lambda: ops.attention_decode(q, kc, vc, lens, workspace=ws), iters)
                qs = q[:, :, None]                                    # [B, H, 1, D]
                ks = kc.transpose(1, 2).contiguous()                  # [B, Hk, ctx, D]
                vs = vc.transpose(1, 2).contiguous()
                sdpa = time_ms(lambda: torch.nn.functional.scaled_dot_product_attention(qs, ks, vs, enable_gqa=True),
                               iters)
                nbytes = 2 * B * ctx * Hk * D * 2
                print(json.dumps({"bench": "attn_decode", "shape": name, "B": B, "context": ctx, "ms": round(ms, 4),
                                  "kv_TB_s": round(nbytes / ms / 1e9, 3),
                                  "frac_of_3.35TB_s": round(nbytes / ms / 1e9 / 3.35, 3),
                                  "sdpa_ms": round(sdpa, 4)}), flush=True)
                del q, kc, vc, ks, vs


def bench_model():
    from mlx_cuda_distributed_pretraining_b200.core.generation import generate
    from mlx_cuda_distributed_pretraining_b200.core.training import Config, Trainer
    import yaml
    cfg = yaml.safe_load((ROOT / "configs" / "c2-llama80m-muon.yaml").read_text())
    cfg["data"]["input_file"] = "synthetic"
    import tempfile
    with tempfile.TemporaryDirectory() as tmp:
        tr = Trainer(Config.from_dict(cfg), for_training=False, quiet=True, run_root=tmp)
    model = tr.model
    a = tr.model_args
    for B in (1, 16):
        prompts = [[(7 * i + 3 * b) % 256 for i in range(128)] for b in range(B)]
        generate(model, prompts, max_tokens=8, temperature=0, min_p=None)  # warm-up
        torch.cuda.synchronize()
        from mlx_cuda_distributed_pretraining_b200.arch.llama import KVCache
        tokens = torch.tensor(prompts, device="cuda")
        cache = KVCache(model, B, 128 + 256)
        t0 = time.perf_counter()
        logits = model.prefill(tokens, [128] * B, cache)
        torch.cuda.synchronize()
        prefill = time.perf_counter() - t0
        nxt = torch.argmax(logits, -1)
        t0 = time.perf_counter()
        for _ in range(255):
            logits = model.decode_step(nxt, cache)
            nxt = torch.argmax(logits, -1)
        torch.cuda.synchronize()
        per_tok = (time.perf_counter() - t0) / 255
        t0 = time.perf_counter()
        generate(model, prompts, max_tokens=256, temperature=0, min_p=None, repetition_penalty=1.0)
        torch.cuda.synchronize()
        total = time.perf_counter() - t0
        print(json.dumps({"bench": "generate", "model": "C2-shaped", "layers": a.num_hidden_layers,
                          "hidden": a.hidden_size, "B": B, "prompt": 128, "new_tokens": 256,
                          "prefill_ms": round(prefill * 1e3, 3), "decode_step_ms": round(per_tok * 1e3, 3),
                          "generate_256_ms": round(total * 1e3, 1)}), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--skip-model", action="store_true")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("decode_bench.py needs a CUDA device")
    print(json.dumps({"gpu": gpu_info()}), flush=True)
    bench_kernel(a.iters)
    if not a.skip_model:
        bench_model()


if __name__ == "__main__":
    main()
