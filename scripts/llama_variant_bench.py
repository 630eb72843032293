"""Cost of `model.misc.variant: mlx_lm` on the H100, in one call:

  mlp      the fused MLP GEMMs with the SiLU epilogues against the reference activation (sigmoid(u) * 2) at the C2, C3
           and C5 layer shapes, alternating the two launches in rounds (CUDA events).
  rope     b200_rope_half against b200_rope on q-shaped C2 activations, in bytes/s (one read + one write per element).
  trainer  the C2-shaped trainer step (configs/c2-llama80m-muon.yaml, synthetic tokens) without and with the variant.

Prints one JSON line per measurement, headed by the card name, power limit and maximum SM clock.

    python scripts/llama_variant_bench.py [--iters 60] [--warmup 10] [--steps 10] [--repeats 3]
"""
import argparse
import json
import subprocess
import sys
import tempfile
from pathlib import Path

import torch

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))

# name: (M tokens per micro-batch, hidden H, intermediate I)
MLP_SHAPES = {"c2": (16 * 1024, 1024, 2816), "c3": (16 * 2048, 1024, 4096), "c5": (8 * 2048, 2048, 5632)}


def time_rounds(calls, iters, warmup, rounds=5):
    """calls: {tag: fn}; each round times iters // rounds launches of each in turn.  Returns {tag: [ms per call]}."""
    for fn in calls.values():
        for _ in range(warmup):
            fn()
    torch.cuda.synchronize()
    per = max(iters // rounds, 1)
    out = {tag: [] for tag in calls}
    for _ in range(rounds):
        for tag, fn in calls.items():
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(per):
                fn()
            e1.record()
            torch.cuda.synchronize()
            out[tag].append(e0.elapsed_time(e1) / per)
    return out


def summary(ts):
    return {"ms": round(sum(ts) / len(ts), 4), "min": round(min(ts), 4), "max": round(max(ts), 4)}


def ok(L, rc, what):
    if rc != 0:
        raise RuntimeError(f"{what}: rc={rc}: {L.b200_last_error().decode()}")


def mlp_part(args, L):
    st = torch.cuda.current_stream().cuda_stream
    bf = torch.bfloat16
    for shape, (M, H, I) in MLP_SHAPES.items():
        g = torch.Generator(device="cuda").manual_seed(1)
        x = torch.randn(M, H, device="cuda", generator=g).to(bf)
        W2 = (torch.randn(2 * I, H, device="cuda", generator=g) * H ** -0.5).to(bf)
        Wd = (torch.randn(H, I, device="cuda", generator=g) * I ** -0.5).to(bf)
        dy = torch.randn(M, H, device="cuda", generator=g).to(bf)
        gu, y, dgu = (torch.empty(M, 2 * I, device="cuda", dtype=bf), torch.empty(M, I, device="cuda", dtype=bf),
                      torch.empty(M, 2 * I, device="cuda", dtype=bf))
        for kind in ("fwd", "bwd"):
            if kind == "fwd":
                calls = {act: (lambda f=f: ok(L, f(x.data_ptr(), W2.data_ptr(), gu.data_ptr(), y.data_ptr(), M, H, I,
                                                   st), "gateup"))
                         for act, f in (("sigmoid2", L.b200_mlp_gateup_glu_fwd), ("silu", L.b200_mlp_gateup_silu_fwd))}
            else:
                calls = {act: (lambda f=f: ok(L, f(dy.data_ptr(), Wd.data_ptr(), gu.data_ptr(), dgu.data_ptr(), M, H,
                                                   I, st), "down"))
                         for act, f in (("sigmoid2", L.b200_mlp_down_glu_bwd), ("silu", L.b200_mlp_down_silu_bwd))}
            t = time_rounds(calls, args.iters, args.warmup)
            line = {"part": "mlp", "kernel": f"gateup_{kind}" if kind == "fwd" else "down_bwd", "shape": shape,
                    "M": M, "H": H, "I": I, **{a: summary(v) for a, v in t.items()}}
            line["silu_over_sigmoid2"] = round(line["silu"]["ms"] / line["sigmoid2"]["ms"], 4)
            print(json.dumps(line), flush=True)
        del x, W2, Wd, dy, gu, y, dgu
        torch.cuda.empty_cache()


def rope_part(args, L):
    from mlx_cuda_distributed_pretraining_b200 import ops
    B, S, NH, D = 16, 1024, 16, 64   # C2's q: 16 heads of 64
    st = torch.cuda.current_stream().cuda_stream
    for dtype in (torch.bfloat16, torch.float32):
        x = torch.randn(B, S, NH, D, device="cuda").to(dtype)
        y = torch.empty_like(x)
        cos_t, sin_t = ops.rope_tables(S, D, 10000.0, "cuda")
        bf = int(dtype == torch.bfloat16)
        calls = {
            "interleaved": lambda: ok(L, L.b200_rope(x.data_ptr(), y.data_ptr(), cos_t.data_ptr(), sin_t.data_ptr(),
                                                     B, S, NH, D, 0, bf, st), "rope"),
            "half": lambda: ok(L, L.b200_rope_half(x.data_ptr(), y.data_ptr(), cos_t.data_ptr(), sin_t.data_ptr(),
                                                   None, B, S, NH, D, 0, bf, st), "rope_half"),
        }
        t = time_rounds(calls, args.iters, args.warmup)
        nbytes = 2 * x.numel() * x.element_size()
        line = {"part": "rope", "dtype": str(dtype).split(".")[1], "shape": [B, S, NH, D]}
        for k, v in t.items():
            line[k] = {**summary(v), "GB_per_s": round(nbytes / (sum(v) / len(v)) / 1e6, 1)}
        print(json.dumps(line), flush=True)


def trainer_part(args):
    from mlx_cuda_distributed_pretraining_b200.core.training import Config, Trainer
    trainers = {}
    for variant in (None, "mlx_lm"):
        cfg = Config.from_yaml(str(ROOT / "configs" / "c2-llama80m-muon.yaml"))
        cfg.name = "variant_bench"
        cfg.model.misc = {**cfg.model.misc, "variant": variant}
        cfg.training.hyperparameters["iters"] = args.warmup + args.steps * args.repeats + 1
        cfg.system.distributed = False
        tr = Trainer(cfg, synthetic=True, quiet=True, run_root=tempfile.mkdtemp(prefix="variant_bench_"))
        tr._accum_step, tr._accum_tokens = 0, 0
        for s in range(args.warmup):
            tr.train_step(s)
        trainers[variant] = tr
    torch.cuda.synchronize()
    times = {v: [] for v in trainers}
    step = args.warmup
    for _ in range(args.repeats):   # alternate the two models in rounds
        for v, tr in trainers.items():
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for s in range(step, step + args.steps):
                tr.train_step(s)
            e1.record()
            torch.cuda.synchronize()
            times[v].append(e0.elapsed_time(e1) / args.steps)
        step += args.steps
    line = {"part": "trainer", "config": "c2", "steps_per_round": args.steps}
    for v, t in times.items():
        line["reference" if v is None else v] = summary(t)
    line["variant_over_reference"] = round(line["mlx_lm"]["ms"] / line["reference"]["ms"], 4)
    print(json.dumps(line), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=60)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--skip-trainer", action="store_true")
    args = ap.parse_args()
    from mlx_cuda_distributed_pretraining_b200 import ops
    ops.require_device()
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip()
    print(json.dumps({"gpu": card}), flush=True)
    mlp_part(args, ops.lib())
    rope_part(args, ops.lib())
    if not args.skip_trainer:
        trainer_part(args)


if __name__ == "__main__":
    main()
