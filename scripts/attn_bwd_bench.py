"""Time the attention backward alone (b200_attn_bwd_strided, as the training step calls it) at the C2, C3 and C5
layer shapes with CUDA events over many launches after warm-up.

Reports ms per call, executed-MMA TFLOP/s (the five 128-key x 64-query x D products of every work item the causal
schedule runs) and full-count TFLOP/s (2.5 x 4 B H S^2 D, the figure bench.py's kernel block uses).  Prints one JSON
line per shape, headed by the card name and power limit.

    python scripts/attn_bwd_bench.py [--iters 50] [--warmup 10]
"""
import argparse
import ctypes
import json
import subprocess
import sys
from pathlib import Path

import torch

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))

SHAPES = {"c2": (16, 1024, 16, 8, 64), "c3": (16, 2048, 16, 8, 64), "c5": (16, 2048, 16, 16, 128)}


def executed_mma_flops(B, S, H, Hk, D, causal=True):
    n_kt, n_qt = -(-S // 128), -(-S // 64)
    items = sum(n_qt - (kt * 2 if causal else 0) for kt in range(n_kt)) * H * B
    return items * 5 * 2 * 128 * 64 * D


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=10)
    args = ap.parse_args()
    from mlx_cuda_distributed_pretraining_b200 import ops
    ops.require_device()
    L = ops.lib()
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip()
    print(json.dumps({"gpu": card}), flush=True)
    for tag, (B, S, H, Hk, D) in SHAPES.items():
        torch.manual_seed(0)
        q = torch.randn(B, S, H, D, device="cuda").to(torch.bfloat16)
        k, v = (torch.randn(B, S, Hk, D, device="cuda").to(torch.bfloat16) for _ in range(2))
        o, do = (torch.randn(B, S, H, D, device="cuda").to(torch.bfloat16) for _ in range(2))
        lse = torch.randn(B, H, S, device="cuda") + 8.0
        dq = torch.empty_like(q)
        dkv = torch.empty(B, S, 2 * Hk, D, device="cuda", dtype=torch.bfloat16)
        ws = torch.empty(int(L.b200_attn_bwd_workspace_bytes(B, S, H, Hk, D)), device="cuda", dtype=torch.uint8)
        st = torch.cuda.current_stream().cuda_stream

        def call():
            rc = L.b200_attn_bwd_strided(q.data_ptr(), k.data_ptr(), v.data_ptr(), o.data_ptr(), do.data_ptr(),
                                         lse.data_ptr(), dq.data_ptr(), dkv.data_ptr(), dkv[:, :, Hk:].data_ptr(),
                                         B, S, H, Hk, D, ctypes.c_float(D ** -0.5), 1, 2 * Hk, ws.data_ptr(),
                                         ws.numel(), st)
            assert rc == 0, L.b200_last_error()

        for _ in range(args.warmup):
            call()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(args.iters):
            call()
        e1.record()
        torch.cuda.synchronize()
        ms = e0.elapsed_time(e1) / args.iters
        full = 2.5 * 4 * B * H * S * S * D
        print(json.dumps({"shape": tag, "B": B, "S": S, "H": H, "Hk": Hk, "D": D, "ms": round(ms, 4),
                          "tflops_executed_mma": round(executed_mma_flops(B, S, H, Hk, D) / ms / 1e9, 1),
                          "tflops_full_count": round(full / ms / 1e9, 1)}), flush=True)


if __name__ == "__main__":
    main()
