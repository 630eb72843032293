"""Time Shampoo's two preconditioner roots on C4's factor groups: the reference's literal formula
(b200_shampoo_root, 6 iterations) and the true inverse 4th root (b200_shampoo_root_newton).

C4 (configs/c4-llama256m-shampoo-dp4.yaml: hidden 1024, intermediate 2816, 16 layers, 16 heads of 64, tied byte-level
embedding of 259 rows) groups its matrices as q/k/v/o [1024, 1024] x 64, gate/up [2816, 1024] x 32,
down [1024, 2816] x 16 and the embedding [259, 1024] x 1; with max_preconditioner_dim 1024 every factor is
1024 wide except the embedding's 259-wide left factor.  The statistics come from a seeded low-rank-plus-noise
gradient model, M = 0.05 G G^T with singular values of G decaying as i^-1.5.

Per factor group: ms per call (CUDA events, median of --reps after one warm-up), iterations used, executed-GEMM
TFLOP/s (six bf16 GEMMs per fp32 product, 4 products per executed iteration), and the cost of one recompute
amortised over update_period = 100 steps.  The card name and power limit are read in the same run.

    python scripts/shampoo_root_bench.py [--reps 3] [--out results.json]
"""
from __future__ import annotations

import argparse
import json
import math
import subprocess
import sys
from pathlib import Path

import torch

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))

from mlx_cuda_distributed_pretraining_b200 import ops  # noqa: E402
from mlx_cuda_distributed_pretraining_b200.optimizers.shampoo import NEWTON_MAX_ITERS, NEWTON_TOL  # noqa: E402

# (name, batch, k) for each root C4 recomputes: the left and right factor of every shape group
C4_FACTORS = [("qkvo L", 64, 1024), ("qkvo R", 64, 1024), ("gate/up L", 32, 1024), ("gate/up R", 32, 1024),
              ("down L", 16, 1024), ("down R", 16, 1024), ("embed L", 1, 259), ("embed R", 1, 1024)]
UPDATE_PERIOD = 100
EPS = 1e-6


def statistics(batch: int, k: int, seed: int, n: int = 2816, rank: int = 256) -> torch.Tensor:
    g = torch.Generator(device="cuda").manual_seed(seed)
    kp = ops.rup8(k)
    s = torch.arange(1, rank + 1, device="cuda", dtype=torch.float32) ** -1.5
    U = torch.randn(batch, k, rank, device="cuda", generator=g) / math.sqrt(k)
    V = torch.randn(batch, rank, n, device="cuda", generator=g) / math.sqrt(n)
    G = (U * s) @ V + 1e-3 * torch.randn(batch, k, n, device="cuda", generator=g) / math.sqrt(n)
    M = torch.zeros(batch, kp, kp, device="cuda")
    M[:, :k, :k] = 0.05 * (G @ G.transpose(1, 2))
    return (M + M.transpose(1, 2)) / 2


def timed(fn, reps: int) -> float:
    fn()
    torch.cuda.synchronize()
    ms = []
    for _ in range(reps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        fn()
        e1.record()
        torch.cuda.synchronize()
        ms.append(e0.elapsed_time(e1))
    return sorted(ms)[len(ms) // 2]


def card() -> dict:
    out = {"device": torch.cuda.get_device_name(0)}
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i",
                            "0"], capture_output=True, text=True, timeout=30)
        out["nvidia_smi"] = q.stdout.strip()
    except (OSError, subprocess.SubprocessError) as e:
        out["nvidia_smi"] = f"unavailable: {e}"
    return out


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--out", type=str, default=None)
    args = ap.parse_args()
    ops.require_device()
    rows = []
    tot = {"reference_ms": 0.0, "newton_ms": 0.0}
    for i, (name, batch, k) in enumerate(C4_FACTORS):
        kp = ops.rup8(k)
        M = statistics(batch, k, seed=i)
        P = torch.empty_like(M)
        Ph = torch.empty(M.shape, dtype=torch.bfloat16, device="cuda")
        Pl = torch.empty_like(Ph)
        ws = torch.empty(max(int(ops.lib().b200_shampoo_root_workspace_bytes(batch, k)),
                             int(ops.lib().b200_shampoo_root_newton_workspace_bytes(batch, k))),
                         dtype=torch.uint8, device="cuda")
        ref_ms = timed(lambda: ops.shampoo_root(M, P, Ph, Pl, k, 0.75, EPS, 6, ws), args.reps)
        res = {}

        def newton():
            res["it"], res["r"] = ops.shampoo_root_newton(M, P, Ph, Pl, k, EPS, NEWTON_MAX_ITERS, NEWTON_TOL, ws)
        new_ms = timed(newton, args.reps)
        it, r = res["it"].cpu(), res["r"].cpu()
        # iterations the host loop executed: it stops at the first multiple of 4 after every matrix froze
        # (a matrix freezes one iteration after its last accepted step when that step did not reach tol)
        last = int((it + (r > NEWTON_TOL).int()).max())
        executed = min(NEWTON_MAX_ITERS, 4 * math.ceil(max(last, 1) / 4))
        gemm_flop = 2.0 * kp ** 3 * batch
        new_flop = executed * 4 * 6 * gemm_flop
        ref_flop = 6 * 3 * gemm_flop
        row = {"factor": name, "batch": batch, "k": k, "reference_ms": round(ref_ms, 3),
               "reference_tflops": round(ref_flop / ref_ms / 1e9, 1), "newton_ms": round(new_ms, 3),
               "newton_iters_min": int(it.min()), "newton_iters_max": int(it.max()), "newton_loop_iters": executed,
               "newton_residual_max": float(r.max()), "newton_tflop": round(new_flop / 1e12, 2),
               "newton_tflops": round(new_flop / new_ms / 1e9, 1),
               "newton_amortised_ms_per_step": round(new_ms / UPDATE_PERIOD, 3)}
        tot["reference_ms"] += ref_ms
        tot["newton_ms"] += new_ms
        rows.append(row)
        print(json.dumps(row), flush=True)
        del M, P, Ph, Pl, ws
        torch.cuda.empty_cache()
    summary = {"c4_recompute_reference_ms": round(tot["reference_ms"], 1),
               "c4_recompute_newton_ms": round(tot["newton_ms"], 1),
               "newton_amortised_ms_per_step": round(tot["newton_ms"] / UPDATE_PERIOD, 2), **card()}
    print(json.dumps(summary), flush=True)
    if args.out:
        Path(args.out).parent.mkdir(parents=True, exist_ok=True)
        Path(args.out).write_text(json.dumps({"factors": rows, "summary": summary}, indent=1))


if __name__ == "__main__":
    main()
