"""Sliding-window attention (`model.attention.sliding_window`): what skipping the tiles outside the window buys, measured.

1. Attention forward + backward as the training step calls them (b200_attn_fwd + b200_attn_bwd_strided for the full
   causal mask, b200_attn_fwd_window + b200_attn_bwd_window with pos = NULL for a window W) at C3's layer shape
   (B16 S2048 H16/Hk8 D64), C5's (B16 S2048 H16/Hk16 D128) and long-context rows at the same tokens per batch
   (B4 S8192, B2 S16384, at D64 H16/Hk8 and D128 H16/Hk16).  Reports the 128x128 score tiles executed, computed from
   the shapes (forward key tiles per 128-query tile; backward 64-query items, two per tile), ms per fwd+bwd,
   executed-MMA TFLOP/s (4 * 128 * 128 * D per forward tile, 10 * 128 * 64 * D per backward item) and useful
   TFLOP/s (14 * visible query-key pairs * D: 4 forward, 10 backward).
2. Decode attention (b200_attn_decode vs b200_attn_decode_window, bf16 cache, C2 heads H16/Hk8 D64, B32) at contexts
   8192 and 32768, W = 1024 against the full context, with the K/V bytes each reads.
3. A C2-shaped trainer at max_context_size 8192 (B2, synthetic tokens), W = 1024 against full causal: ms per step
   and tok/s.

CUDA events over many launches after warm-up; the card name and power limit head the output.  One JSON line per
measurement.

    python scripts/window_bench.py [--iters 10] [--warmup 3] [--steps 10]
"""
import argparse
import ctypes
import json
import subprocess
import sys
import tempfile
from pathlib import Path

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))

SHAPES = {"c3": (16, 2048, 16, 8, 64), "c5": (16, 2048, 16, 16, 128),
          "s8k_d64": (4, 8192, 16, 8, 64), "s16k_d64": (2, 16384, 16, 8, 64),
          "s8k_d128": (4, 8192, 16, 16, 128), "s16k_d128": (2, 16384, 16, 16, 128)}
WINDOWS = (None, 128, 512, 1024, 4096)
BQ_FWD, BKV, BQ_BWD, DEC_TILE = 128, 128, 64, 32


def fwd_tiles(S, W):
    """Forward key tiles per (row, head): each 128-query tile runs from the tile of its first query's window start to
    the causal tile."""
    n = 0
    for q0 in range(0, S, BQ_FWD):
        j0 = 0 if W is None else max(0, q0 - W) // BKV
        n += min(-(-S // BKV), (q0 + BQ_FWD - 1) // BKV + 1) - j0
    return n


def bwd_items(S, W):
    """Backward 64-query items per (row, query head): key tile kt covers query tiles k0 / 64 up to the tile of its
    last reachable query, min(S - 1, k0 + 127 + W)."""
    n = 0
    for kt in range(-(-S // BKV)):
        k0 = kt * BKV
        last = S - 1 if W is None else min(S - 1, k0 + BKV - 1 + W)
        n += last // BQ_BWD + 1 - k0 // BQ_BWD
    return n


def visible_pairs(S, W):
    return sum(q + 1 if W is None else min(q, W) + 1 for q in range(S))


def _time(call, iters, warmup):
    import torch
    for _ in range(warmup):
        call()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        call()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters


def attention_part(args, L):
    import torch
    st = None if args.count_only else torch.cuda.current_stream().cuda_stream
    for tag, (B, S, H, Hk, D) in SHAPES.items():
        if args.count_only:
            for W in WINDOWS:
                print(json.dumps({"part": "attention", "shape": tag, "B": B, "S": S, "D": D,
                                  "window": W if W is not None else "off", "tiles_fwd_per_row_head": fwd_tiles(S, W),
                                  "tiles_bwd_per_row_head": bwd_items(S, W) / 2}), flush=True)
            continue
        torch.manual_seed(0)
        q = torch.randn(B, S, H, D, device="cuda").to(torch.bfloat16)
        k, v = (torch.randn(B, S, Hk, D, device="cuda").to(torch.bfloat16) for _ in range(2))
        do = torch.randn(B, S, H, D, device="cuda").to(torch.bfloat16)
        o = torch.empty_like(q)
        lse = torch.empty(B, H, S, device="cuda")
        dq = torch.empty_like(q)
        dkv = torch.empty(B, S, 2 * Hk, D, device="cuda", dtype=torch.bfloat16)
        ws = torch.empty(int(L.b200_attn_bwd_window_workspace_bytes(B, S, H, Hk, D)), device="cuda",
                         dtype=torch.uint8)
        sc = ctypes.c_float(D ** -0.5)
        for W in WINDOWS:
            if W is None:
                def call():
                    assert L.b200_attn_fwd(q.data_ptr(), k.data_ptr(), v.data_ptr(), o.data_ptr(), lse.data_ptr(),
                                           B, S, H, Hk, D, sc, 1, st) == 0
                    assert L.b200_attn_bwd_strided(q.data_ptr(), k.data_ptr(), v.data_ptr(), o.data_ptr(),
                                                   do.data_ptr(), lse.data_ptr(), dq.data_ptr(), dkv.data_ptr(),
                                                   dkv[:, :, Hk:].data_ptr(), B, S, H, Hk, D, sc, 1, 2 * Hk,
                                                   ws.data_ptr(), ws.numel(), st) == 0
            else:
                def call():
                    assert L.b200_attn_fwd_window(q.data_ptr(), k.data_ptr(), v.data_ptr(), o.data_ptr(),
                                                  lse.data_ptr(), None, W, B, S, H, Hk, D, sc, st) == 0
                    assert L.b200_attn_bwd_window(q.data_ptr(), k.data_ptr(), v.data_ptr(), o.data_ptr(),
                                                  do.data_ptr(), lse.data_ptr(), None, W, dq.data_ptr(),
                                                  dkv.data_ptr(), dkv[:, :, Hk:].data_ptr(), B, S, H, Hk, D, sc,
                                                  2 * Hk, ws.data_ptr(), ws.numel(), st) == 0
            tf, tb = fwd_tiles(S, W), bwd_items(S, W)
            executed = B * H * (tf * 4 * BQ_FWD * BKV * D + tb * 10 * BQ_BWD * BKV * D)
            useful = 14 * B * H * visible_pairs(S, W) * D
            ms = _time(call, args.iters, args.warmup)
            print(json.dumps({"part": "attention", "shape": tag, "B": B, "S": S, "H": H, "Hk": Hk, "D": D,
                              "window": W if W is not None else "off", "tiles_fwd_per_row_head": tf,
                              "tiles_bwd_per_row_head": tb / 2, "tiles_total": int(B * H * (tf + tb / 2)),
                              "ms_fwd_bwd": round(ms, 4), "executed_tflops": round(executed / ms / 1e9, 1),
                              "useful_tflops": round(useful / ms / 1e9, 1)}), flush=True)
        del q, k, v, do, o, lse, dq, dkv, ws
        torch.cuda.empty_cache()


def decode_part(args, L):
    import torch
    from mlx_cuda_distributed_pretraining_b200 import ops
    B, H, Hk, D, W = 32, 16, 8, 64, 1024
    for ctx in (8192, 32768):
        g = torch.Generator(device="cuda").manual_seed(0)
        q = torch.randn(B, H, D, device="cuda", generator=g).to(torch.bfloat16)
        kc = torch.randn(B, ctx, Hk, D, device="cuda", generator=g).to(torch.bfloat16)
        vc = torch.randn(B, ctx, Hk, D, device="cuda", generator=g).to(torch.bfloat16)
        lens = torch.full((B,), ctx, device="cuda", dtype=torch.int32)
        ws = torch.empty(ops.attention_decode_workspace_bytes(B, H, ctx, D), device="cuda", dtype=torch.uint8)
        for win in (None, W):
            keys = ctx if win is None else ctx - (max(0, ctx - 1 - win) // DEC_TILE * DEC_TILE)
            nbytes = 2 * B * keys * Hk * D * 2
            ms = _time(lambda: ops.attention_decode(q, kc, vc, lens, workspace=ws, window=win),
                       args.iters * 10, args.warmup)
            print(json.dumps({"part": "decode", "B": B, "H": H, "Hk": Hk, "D": D, "context": ctx,
                              "window": win if win is not None else "off", "kv_bytes_read": nbytes,
                              "us": round(ms * 1e3, 1), "TB_per_s": round(nbytes / ms / 1e9, 2)}), flush=True)
        del q, kc, vc, ws
        torch.cuda.empty_cache()


def trainer_part(args):
    import torch
    from mlx_cuda_distributed_pretraining_b200.core.training import Config, Trainer
    S, B, W = 8192, 2, 1024
    for win in (None, W):
        cfg = Config.from_yaml(str(ROOT / "configs" / "c2-llama80m-muon.yaml"))
        cfg.name = "window_bench"
        cfg.data.preprocessing = {**cfg.data.preprocessing, "max_context_size": S}
        cfg.model.attention = {**cfg.model.attention, "max_position_embeddings": S, "sliding_window": win}
        cfg.training.hyperparameters["batch_size"] = B
        cfg.training.hyperparameters["iters"] = args.warmup + args.steps
        cfg.system.distributed = False
        with tempfile.TemporaryDirectory(prefix="window_bench_") as run_root:
            tr = Trainer(cfg, synthetic=True, quiet=True, run_root=run_root)
            tr._accum_step, tr._accum_tokens = 0, 0
            for s in range(args.warmup):
                tr.train_step(s)
            torch.cuda.synchronize()
            ms = _time_steps(tr, args.warmup, args.steps)
            print(json.dumps({"part": "trainer", "config": "c2", "B": B, "S": S,
                              "window": win if win is not None else "off", "step_ms": round(ms, 2),
                              "tokens_per_s": round(B * S / (ms / 1e3))}), flush=True)
            del tr
            torch.cuda.empty_cache()


def _time_steps(tr, start, steps):
    import torch
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for s in range(start, start + steps):
        tr.train_step(s)
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / steps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--count-only", action="store_true", help="print the tile counts and exit (no GPU needed)")
    ap.add_argument("--skip-attention", action="store_true")
    ap.add_argument("--skip-decode", action="store_true")
    ap.add_argument("--skip-trainer", action="store_true")
    args = ap.parse_args()
    if args.count_only:
        attention_part(args, None)
        return
    from mlx_cuda_distributed_pretraining_b200 import ops
    ops.require_device()
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip()
    print(json.dumps({"gpu": card}), flush=True)
    if not args.skip_attention:
        attention_part(args, ops.lib())
    if not args.skip_decode:
        decode_part(args, ops.lib())
    if not args.skip_trainer:
        trainer_part(args)


if __name__ == "__main__":
    main()
