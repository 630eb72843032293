"""Attention dropout (`model.attention.dropout`): what the Philox keep masks cost.

1. The causal attention forward and backward, timed separately, at the layer shapes of C2 (B16 S1024 H16/Hk8 D64),
   C3 (B16 S2048 H16/Hk8 D64) and C5 (B16 S2048 H16/Hk16 D128): b200_attn_fwd / b200_attn_bwd_strided (p = 0, the
   dropout-free kernels) against b200_attn_fwd_dropout / b200_attn_bwd_dropout at p = 0.1.  The launches alternate
   in rounds inside one process; each line reports the median round.
2. A C2-shaped trainer step (C2's config, synthetic rows) without and with `dropout: 0.1`, alternating rounds.

CUDA events over many launches after warm-up; the card name and power limit head the output.  One JSON line per
measurement.

    python scripts/dropout_bench.py [--iters 20] [--rounds 5] [--warmup 3] [--steps 10]
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
P = 0.1


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
        ws = torch.empty(int(L.b200_attn_bwd_dropout_workspace_bytes(B, S, H, Hk, D)), device="cuda",
                         dtype=torch.uint8)
        sc, pc = ctypes.c_float(D ** -0.5), ctypes.c_float(P)
        dk, dv = dkv.data_ptr(), dkv[:, :, Hk:].data_ptr()
        seed = 0x1234_5678_9ABC_DEF0

        def fwd0():
            assert L.b200_attn_fwd(q.data_ptr(), k.data_ptr(), v.data_ptr(), o.data_ptr(), lse.data_ptr(),
                                   B, S, H, Hk, D, sc, 1, st) == 0

        def bwd0():
            assert L.b200_attn_bwd_strided(q.data_ptr(), k.data_ptr(), v.data_ptr(), o.data_ptr(), do.data_ptr(),
                                           lse.data_ptr(), dq.data_ptr(), dk, dv, B, S, H, Hk, D, sc, 1, 2 * Hk,
                                           ws.data_ptr(), ws.numel(), st) == 0

        def fwd1():
            assert L.b200_attn_fwd_dropout(q.data_ptr(), k.data_ptr(), v.data_ptr(), o.data_ptr(), lse.data_ptr(),
                                           None, -1, None, B, S, H, Hk, D, sc, 1, pc, seed, st) == 0

        def bwd1():
            assert L.b200_attn_bwd_dropout(q.data_ptr(), k.data_ptr(), v.data_ptr(), o.data_ptr(), do.data_ptr(),
                                           lse.data_ptr(), None, -1, None, dq.data_ptr(), dk, dv, B, S, H, Hk, D, sc,
                                           1, pc, seed, 2 * Hk, ws.data_ptr(), ws.numel(), st) == 0

        fwd0()
        ms = _alternate({"fwd_p0": fwd0, "fwd_p0.1": fwd1, "bwd_p0": bwd0, "bwd_p0.1": bwd1},
                        args.iters, args.rounds, args.warmup)
        print(json.dumps({"part": "attention", "shape": tag, "B": B, "S": S, "H": H, "Hk": Hk, "D": D,
                          **{f"{n}_ms": round(t, 4) for n, t in ms.items()},
                          "fwd_dropout_over_plain": round(ms["fwd_p0.1"] / ms["fwd_p0"], 4),
                          "bwd_dropout_over_plain": round(ms["bwd_p0.1"] / ms["bwd_p0"], 4)}), flush=True)


def trainer_part(args):
    import torch
    from mlx_cuda_distributed_pretraining_b200.core.training import Config, Trainer
    trainers, dirs = {}, []
    for name, p in (("p0", None), ("p0.1", P)):
        cfg = Config.from_yaml(str(ROOT / "configs" / "c2-llama80m-muon.yaml"))
        cfg.name = f"dropout_bench_{name}"
        cfg.model.attention = {**cfg.model.attention, "dropout": p}
        cfg.training.hyperparameters["iters"] = args.warmup + args.steps * args.rounds
        cfg.system.distributed = False
        d = tempfile.TemporaryDirectory(prefix="dropout_bench_")
        dirs.append(d)
        tr = Trainer(cfg, synthetic=True, quiet=True, run_root=d.name)
        tr._accum_step, tr._accum_tokens = 0, 0
        trainers[name] = tr
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
    print(json.dumps({"part": "trainer", "config": "c2", "step_ms_p0": round(ms["p0"], 2),
                      "step_ms_p0.1": round(ms["p0.1"], 2),
                      "dropout_over_plain": round(ms["p0.1"] / ms["p0"], 4)}), flush=True)
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
