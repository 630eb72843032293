"""Time the fused optimizer updates on flat ranges of C2's and C5's parameter counts: b200_lion (reference and
paper variants), b200_sgd (plain mlx SGD and SGDEnhanced's momentum) and, as the yardstick, b200_adamw.

Every update writes the fp32 master and the bf16 shadow, as in mixed-precision training.  Cases: gradients in bf16
(`store.grad`) or fp32 (`store.acc`), with and without the EMA weights (steady state: read and written) and the
global-norm clip (its b200_sumsq launch is inside the timed window).  Reported per case: ms per update (CUDA events
around --reps back-to-back updates, median of 5 windows after a warm-up), the bytes the algorithm must move, and
those bytes over the time.  The card name and power limit are read in the same run.

    python scripts/optimizer_bench.py [--reps 20] [--configs c2,c5] [--out results.json]
"""
from __future__ import annotations

import argparse
import json
import statistics
import subprocess
import sys
from pathlib import Path

import torch
import yaml

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))

from mlx_cuda_distributed_pretraining_b200 import ops  # noqa: E402

CONFIGS = {"c2": "configs/c2-llama80m-muon.yaml", "c5": "configs/c5-llama1b-adamw-dp8.yaml"}


def param_count(path: Path) -> int:
    """Parameters of the Llama a config describes (tied embeddings, no biases)."""
    c = yaml.safe_load(path.read_text())
    dims, att = c["model"]["dimensions"], c["model"]["attention"]
    tok = c["data"]["tokenizer"]
    V = tok["normal_vocab_size"] + len(tok.get("special_tokens", {}))
    H, I, L = dims["hidden_size"], dims["intermediate_size"], dims["num_layers"]
    hd, nh, nkv = att["head_dim"], att["num_heads"], att["num_kv_heads"]
    attn = H * nh * hd * 2 + H * nkv * hd * 2
    return V * H + L * (attn + 3 * H * I + 2 * H) + H


def update_bytes(kind: str, gbytes: int, ema: bool, clip: bool) -> int:
    """Bytes per parameter: master read+write (8), shadow write (2), gradient read, state read+write."""
    state = {"adamw": 16, "lion": 8, "lion_paper": 8, "sgd": 0, "sgd_enhanced": 8}[kind]
    return 8 + 2 + gbytes + state + (8 if ema else 0) + (gbytes if clip else 0)


def card() -> dict:
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power, clock = [s.strip() for s in out.split(",")]
        return {"name": name, "power_limit": power, "max_sm_clock": clock}
    except Exception as e:  # the numbers are still measured; the card is then named by torch only
        return {"name": torch.cuda.get_device_name(), "power_limit": f"unknown ({type(e).__name__})"}


def time_ms(fn, reps: int) -> float:
    fn()
    torch.cuda.synchronize()
    windows = []
    for _ in range(5):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(reps):
            fn()
        e1.record()
        e1.synchronize()
        windows.append(e0.elapsed_time(e1) / reps)
    return statistics.median(windows)


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--configs", default="c2,c5")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    ops.require_device()
    info = {"card": card(), "results": []}
    print(json.dumps(info["card"]))
    for cname in a.configs.split(","):
        n = param_count(ROOT / CONFIGS[cname])
        n8 = (n + 7) // 8 * 8
        dev = "cuda"
        p32 = torch.randn(n8, device=dev) * 0.02
        p16 = p32.to(torch.bfloat16)
        st1, st2 = torch.zeros(n8, device=dev), torch.zeros(n8, device=dev)
        ema = p32.clone()
        ss = torch.zeros(1, device=dev)
        for gdt in (torch.bfloat16, torch.float32):
            g = (torch.randn(n8, device=dev) * 1e-3).to(gdt)
            gb = g.element_size()
            cases = [("adamw", False, False)]
            for kind in ("lion", "lion_paper", "sgd", "sgd_enhanced"):
                cases += [(kind, False, False), (kind, True, False), (kind, False, True), (kind, True, True)]
            for kind, use_ema, clip in cases:
                def step(kind=kind, use_ema=use_ema, clip=clip):
                    common = dict(gscale=1.0, clip_ss=ss if clip else None, max_norm=1.0 if clip else None,
                                  ema=ema if use_ema else None, ema_decay=0.999, ema_mode=2 if use_ema else 0)
                    if clip:
                        ops.sumsq(g, out=ss)
                    if kind == "adamw":
                        ops.adamw(p32, p16, g, st1, st2, 1e-4, 0.9, 0.999, 1e-8, 0.01)
                    elif kind == "lion":
                        ops.lion(p32, p16, g, st1, 1e-4, 0.9, 0.9, 1.0, **common)
                    elif kind == "lion_paper":
                        ops.lion(p32, p16, g, st1, 1e-4, 0.9, 0.99, 1.0 - 1e-6, **common)
                    elif kind == "sgd":
                        ops.sgd(p32, p16, g, None, 1e-4, **common)
                    else:
                        ops.sgd(p32, p16, g, st1, 1e-4, 0.9, 0.0, True, 1e-6, **common)
                ms = time_ms(step, a.reps)
                nbytes = update_bytes(kind, gb, use_ema, clip) * n
                row = {"config": cname, "params": n, "kernel": kind, "grad": str(gdt).split(".")[-1],
                       "ema": use_ema, "clip": clip, "ms": round(ms, 4), "bytes": nbytes,
                       "GB/s": round(nbytes / ms / 1e6, 1)}
                info["results"].append(row)
                print(json.dumps(row), flush=True)
            del g
        del p32, p16, st1, st2, ema
        torch.cuda.empty_cache()
    if a.out:
        Path(a.out).parent.mkdir(parents=True, exist_ok=True)
        Path(a.out).write_text(json.dumps(info, indent=1))


if __name__ == "__main__":
    main()
