"""Prefix-LM attention (`model.attention.prefix_lm`): what the bidirectional prefix costs.

1. Attention forward + backward as the training step calls them, at the layer shapes of C2 (B16 S1024 H16/Hk8 D64),
   C3 (B16 S2048 H16/Hk8 D64) and C5 (B16 S2048 H16/Hk16 D128): b200_attn_fwd_prefix + b200_attn_bwd_prefix with every
   row's P in {0, S/4, S/2, S}, against b200_attn_fwd + b200_attn_bwd_strided with causal = 1 and causal = 0.  The
   calls alternate in rounds inside one process; each line reports the median round.  Each line also gives the key
   tiles the forward executes (128 x 128) and TFLOP/s counted on the visible (query, key) pairs only: 4 D flops per
   pair forward (QK^T, PV) and 10 D backward (QK^T, dO V^T, P^T dO, dS^T Q, dS K).
2. A C2-shaped trainer step (C2's config, synthetic rows with uniform split points) with and without `prefix_lm`,
   alternating rounds of steps.

CUDA events over many launches after warm-up; the card name and power limit head the output.  One JSON line per
measurement.

    python scripts/prefix_lm_bench.py [--iters 20] [--rounds 5] [--warmup 3] [--steps 10]
"""
import argparse
import ctypes
import json
import statistics
import subprocess
import sys
import tempfile
from pathlib import Path

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))

SHAPES = {"c2": (16, 1024, 16, 8, 64), "c3": (16, 2048, 16, 8, 64), "c5": (16, 2048, 16, 16, 128)}
BT = 128


def _time(call, iters):
    import torch
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        call()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters


def _alternate(calls, iters, rounds, warmup):
    """calls: name -> callable.  Warm every call, then `rounds` rounds timing each in turn; median ms per call."""
    for c in calls.values():
        for _ in range(warmup):
            c()
    times = {n: [] for n in calls}
    for _ in range(rounds):
        for n, c in calls.items():
            times[n].append(_time(c, iters))
    return {n: statistics.median(t) for n, t in times.items()}


def fwd_tiles(S, P):
    """Key tiles the forward runs per (row, head): each 128-query tile runs to max(causal end, ceil(P / 128));
    P = None is the non-causal launch."""
    n = -(-S // BT)
    if P is None:
        return n * n
    return sum(min(n, max(qt + 1, -(-P // BT))) for qt in range(n))


def visible_pairs(S, P):
    """(query, key) pairs the mask leaves visible in one row: k <= q or k < P."""
    if P is None:
        return S * S
    P = min(max(P, 0), S)
    return P * P + (S * (S + 1) // 2 - P * (P + 1) // 2)


def attention_part(args, L):
    import torch
    st = torch.cuda.current_stream().cuda_stream
    for tag, (B, S, H, Hk, D) in SHAPES.items():
        torch.manual_seed(0)
        q = torch.randn(B, S, H, D, device="cuda").to(torch.bfloat16)
        k, v = (torch.randn(B, S, Hk, D, device="cuda").to(torch.bfloat16) for _ in range(2))
        do = torch.randn(B, S, H, D, device="cuda").to(torch.bfloat16)
        o, dq = torch.empty_like(q), torch.empty_like(q)
        lse = torch.empty(B, H, S, device="cuda")
        dkv = torch.empty(B, S, 2 * Hk, D, device="cuda", dtype=torch.bfloat16)
        ws = torch.empty(int(L.b200_attn_bwd_prefix_workspace_bytes(B, S, H, Hk, D)), device="cuda",
                         dtype=torch.uint8)
        sc = ctypes.c_float(D ** -0.5)
        dk, dv = dkv.data_ptr(), dkv[:, :, Hk:].data_ptr()

        def plain(causal):
            def call():
                assert L.b200_attn_fwd(q.data_ptr(), k.data_ptr(), v.data_ptr(), o.data_ptr(), lse.data_ptr(),
                                       B, S, H, Hk, D, sc, causal, st) == 0
                assert L.b200_attn_bwd_strided(q.data_ptr(), k.data_ptr(), v.data_ptr(), o.data_ptr(), do.data_ptr(),
                                               lse.data_ptr(), dq.data_ptr(), dk, dv, B, S, H, Hk, D, sc, causal,
                                               2 * Hk, ws.data_ptr(), ws.numel(), st) == 0
            return call

        def prefixed(P):
            pre = torch.full((B,), P, dtype=torch.int32, device="cuda")

            def call():
                assert L.b200_attn_fwd_prefix(q.data_ptr(), k.data_ptr(), v.data_ptr(), o.data_ptr(), lse.data_ptr(),
                                              pre.data_ptr(), B, S, H, Hk, D, sc, st) == 0
                assert L.b200_attn_bwd_prefix(q.data_ptr(), k.data_ptr(), v.data_ptr(), o.data_ptr(), do.data_ptr(),
                                              lse.data_ptr(), pre.data_ptr(), dq.data_ptr(), dk, dv, B, S, H, Hk, D,
                                              sc, 2 * Hk, ws.data_ptr(), ws.numel(), st) == 0
            return call

        Ps = {"P0": 0, "PS/4": S // 4, "PS/2": S // 2, "PS": S}
        calls = {"causal": plain(1), "noncausal": plain(0), **{n: prefixed(P) for n, P in Ps.items()}}
        ms = _alternate(calls, args.iters, args.rounds, args.warmup)
        for n in calls:
            P = {"causal": 0, "noncausal": None}.get(n, Ps.get(n))
            pairs = B * H * visible_pairs(S, P)
            tflops = pairs * 14 * D / (ms[n] * 1e-3) / 1e12
            print(json.dumps({"part": "attention", "shape": tag, "B": B, "S": S, "H": H, "Hk": Hk, "D": D,
                              "launch": n, "P": P, "fwd_bwd_ms": round(ms[n], 4),
                              "over_causal": round(ms[n] / ms["causal"], 4),
                              "fwd_key_tiles_per_head": fwd_tiles(S, P),
                              "visible_tflops": round(tflops, 1)}), flush=True)


def trainer_part(args):
    import torch
    from mlx_cuda_distributed_pretraining_b200.core.training import Config, Trainer
    trainers, dirs = {}, []
    for name, prefix_lm in (("base", None), ("prefix_lm", True)):
        cfg = Config.from_yaml(str(ROOT / "configs" / "c2-llama80m-muon.yaml"))
        cfg.name = f"prefix_bench_{name}"
        cfg.model.attention = {**cfg.model.attention, "prefix_lm": prefix_lm}
        cfg.training.hyperparameters["iters"] = args.warmup + args.steps * args.rounds
        cfg.system.distributed = False
        d = tempfile.TemporaryDirectory(prefix="prefix_bench_")
        dirs.append(d)
        tr = Trainer(cfg, synthetic=True, quiet=True, run_root=d.name)
        tr._accum_step, tr._accum_tokens = 0, 0
        trainers[name] = tr
    B = trainers["base"].config.training.hyperparameters["batch_size"]
    S = trainers["base"].config.data.preprocessing["max_context_size"]
    step = {n: 0 for n in trainers}

    def run(n, k):
        for _ in range(k):
            trainers[n].train_step(step[n])
            step[n] += 1

    for n in trainers:
        run(n, args.warmup)
    torch.cuda.synchronize()
    times = {n: [] for n in trainers}
    for _ in range(args.rounds):
        for n in trainers:
            times[n].append(_time(lambda: run(n, 1), args.steps))
    ms = {n: statistics.median(t) for n, t in times.items()}
    print(json.dumps({"part": "trainer", "config": "c2", "B": B, "S": S, "step_ms_base": round(ms["base"], 2),
                      "step_ms_prefix_lm": round(ms["prefix_lm"], 2),
                      "prefix_lm_over_base": round(ms["prefix_lm"] / ms["base"], 4)}), flush=True)
    for d in dirs:
        d.cleanup()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--skip-attention", action="store_true")
    ap.add_argument("--skip-trainer", action="store_true")
    args = ap.parse_args()
    from mlx_cuda_distributed_pretraining_b200 import ops
    ops.require_device()
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip()
    print(json.dumps({"gpu": card}), flush=True)
    if not args.skip_attention:
        attention_part(args, ops.lib())
    if not args.skip_trainer:
        trainer_part(args)


if __name__ == "__main__":
    main()
