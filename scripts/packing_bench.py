"""Packed sequences: what the document-causal kernels and `pack_sequences` buy, measured.

1. Attention forward + backward (b200_attn_fwd_doc + b200_attn_bwd_doc, as the training step calls them) at the C2,
   C3 and C5 layer shapes for several document layouts: one document per row (also through the causal kernels),
   fixed 512 / 256 / 128-token documents and a seeded log-normal mix.  Reports ms per fwd+bwd, the 128x128
   score tiles executed (forward key tiles per 128-query tile; backward 64-query items, two per tile), and TFLOP/s
   over the useful flop count 14 * (visible query-key pairs) * H * D (4 forward, 10 backward).
2. End to end: a seeded synthetic JSONL corpus (document lengths in bytes ~ exp(N(6.0, 1.0)), clipped to
   [16, 8000], lower-case letters and spaces; nothing is downloaded) written to --out, and a C2-shaped trainer run
   on it unpacked and packed.  The padded share of input positions over the steps run is counted and printed before
   any GPU work; then step ms and useful (non-PAD target) tokens/s.

CUDA events over many launches after warm-up; the card name and power limit head the output.  One JSON line per
measurement.

    python scripts/packing_bench.py [--iters 20] [--warmup 5] [--steps 20] [--out DIR]
"""
import argparse
import ctypes
import json
import random
import subprocess
import sys
import tempfile
from pathlib import Path

import numpy as np
import torch

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))

SHAPES = {"c2": (16, 1024, 16, 8, 64), "c3": (16, 2048, 16, 8, 64), "c5": (16, 2048, 16, 16, 128)}


def layout_rows(kind, B, S, seed=0):
    """Document lengths of each row (summing to S)."""
    rng = np.random.default_rng(seed)
    rows = []
    for _ in range(B):
        if kind == "one_doc":
            lens = [S]
        elif kind.startswith("fixed"):
            n = int(kind[5:])
            lens = [n] * (S // n) + ([S % n] if S % n else [])
        else:  # log-normal mix, the corpus distribution below in tokens
            lens = []
            while sum(lens) < S:
                lens.append(int(min(max(rng.lognormal(6.0, 1.0), 16), S - sum(lens))) or 1)
        rows.append(lens)
    return rows


def pos_of(rows, S):
    return torch.stack([torch.cat([torch.arange(n, dtype=torch.int32) for n in lens]) for lens in rows])


def tile_counts(pos, S):
    """(forward 128x128 tiles, backward 128x128 tiles) the document kernels execute, per head."""
    n_kt = -(-S // 128)
    fwd = bwd = 0
    for p in pos.tolist():
        start = [s - p[s] for s in range(S)]
        for q0 in range(0, S, 128):
            fwd += min(n_kt, (q0 + 127) // 128 + 1) - start[q0] // 128
        ends = [0] * n_kt
        for s in range(S):
            if s == S - 1 or p[s + 1] == 0:
                hi = n_kt - 1 if s == S - 1 else (s + 1) // 128 - 1
                for kt in range(start[s] // 128, hi + 1):
                    ends[kt] = s // 64 + 1
        bwd += sum(ends[kt] - 2 * kt for kt in range(n_kt)) / 2
    return fwd, bwd


def attention_part(args, L, ops):
    for tag, (B, S, H, Hk, D) in SHAPES.items():
        torch.manual_seed(0)
        q = torch.randn(B, S, H, D, device="cuda").to(torch.bfloat16)
        k, v = (torch.randn(B, S, Hk, D, device="cuda").to(torch.bfloat16) for _ in range(2))
        do = torch.randn(B, S, H, D, device="cuda").to(torch.bfloat16)
        o = torch.empty_like(q)
        lse = torch.empty(B, H, S, device="cuda")
        dq = torch.empty_like(q)
        dkv = torch.empty(B, S, 2 * Hk, D, device="cuda", dtype=torch.bfloat16)
        ws = torch.empty(int(L.b200_attn_bwd_doc_workspace_bytes(B, S, H, Hk, D)), device="cuda", dtype=torch.uint8)
        st = torch.cuda.current_stream().cuda_stream
        sc = ctypes.c_float(D ** -0.5)
        for kind in ("causal", "one_doc", "fixed512", "fixed256", "fixed128", "lognormal"):
            rows = layout_rows("one_doc" if kind == "causal" else kind, B, S, seed=1)
            pos = pos_of(rows, S).cuda()
            pairs = sum(n * (n + 1) // 2 for lens in rows for n in lens)
            if kind == "causal":
                def call():
                    assert L.b200_attn_fwd(q.data_ptr(), k.data_ptr(), v.data_ptr(), o.data_ptr(), lse.data_ptr(),
                                           B, S, H, Hk, D, sc, 1, st) == 0
                    assert L.b200_attn_bwd_strided(q.data_ptr(), k.data_ptr(), v.data_ptr(), o.data_ptr(),
                                                   do.data_ptr(), lse.data_ptr(), dq.data_ptr(), dkv.data_ptr(),
                                                   dkv[:, :, Hk:].data_ptr(), B, S, H, Hk, D, sc, 1, 2 * Hk,
                                                   ws.data_ptr(), ws.numel(), st) == 0
                fwd_t, bwd_t = tile_counts(pos[:1].cpu(), S)
                fwd_t, bwd_t = fwd_t * B, bwd_t * B
            else:
                def call():
                    assert L.b200_attn_fwd_doc(q.data_ptr(), k.data_ptr(), v.data_ptr(), o.data_ptr(), lse.data_ptr(),
                                               pos.data_ptr(), B, S, H, Hk, D, sc, st) == 0
                    assert L.b200_attn_bwd_doc(q.data_ptr(), k.data_ptr(), v.data_ptr(), o.data_ptr(), do.data_ptr(),
                                               lse.data_ptr(), pos.data_ptr(), dq.data_ptr(), dkv.data_ptr(),
                                               dkv[:, :, Hk:].data_ptr(), B, S, H, Hk, D, sc, 2 * Hk, ws.data_ptr(),
                                               ws.numel(), st) == 0
                fwd_t, bwd_t = tile_counts(pos.cpu(), S)
            for _ in range(args.warmup):
                call()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(args.iters):
                call()
            e1.record()
            torch.cuda.synchronize()
            ms = e0.elapsed_time(e1) / args.iters
            print(json.dumps({"part": "attention", "shape": tag, "B": B, "S": S, "H": H, "Hk": Hk, "D": D,
                              "layout": kind, "ms_fwd_bwd": round(ms, 4), "tiles_fwd": int(fwd_t * H),
                              "tiles_bwd": int(bwd_t * H), "useful_tflops": round(14 * pairs * H * D / ms / 1e9, 1)}),
                  flush=True)


def write_corpus(path, n_docs=6000, seed=0):
    rng = np.random.default_rng(seed)
    letters = np.frombuffer(b"abcdefghijklmnopqrstuvwxyz     ", dtype=np.uint8)
    with open(path, "w") as f:
        for n in np.clip(rng.lognormal(6.0, 1.0, n_docs), 16, 8000).astype(int):
            f.write(json.dumps({"text": letters[rng.integers(0, len(letters), n)].tobytes().decode()}) + "\n")


def c2_config(corpus, pack, steps):
    from mlx_cuda_distributed_pretraining_b200.core.training import Config
    cfg = Config.from_yaml(str(ROOT / "configs" / "c2-llama80m-muon.yaml"))
    cfg.name = "packing_bench"
    cfg.overwrite = True
    cfg.data.input_file = str(corpus)
    cfg.data.validation_file = None
    cfg.data.tokenizer_path = None
    cfg.data.preprocessing = {**cfg.data.preprocessing, "chunk_overlap": 0, "pack_sequences": pack}
    cfg.training.epochs = None
    cfg.training.hyperparameters["iters"] = steps
    cfg.system.distributed = False
    return cfg


def end_to_end_part(args, out):
    from mlx_cuda_distributed_pretraining_b200.core.training import DataManager, TokenizerManager, Trainer
    corpus = out / "synthetic_corpus.jsonl"
    write_corpus(corpus)
    n_steps = args.warmup + args.steps
    shares = {}
    for pack in (False, True):   # host-only count of the batches the runs below consume
        cfg = c2_config(corpus, pack, n_steps)
        random.seed(cfg.system.seed)
        np.random.seed(cfg.system.seed)
        dm = DataManager(cfg.data, TokenizerManager(cfg.data), cfg.training.hyperparameters["batch_size"])
        pad = tot = 0
        for s in range(n_steps):
            b = dm.generate_batch(s)[:, :-1]
            pad += int((b == dm.tokenizer.PAD_TOKEN).sum())
            tot += b.numel()
        shares[pack] = pad / tot
        print(json.dumps({"part": "end_to_end", "packed": pack, "padded_share_of_positions": round(pad / tot, 4),
                          "positions": tot, "batches_per_epoch": dm.num_train_batches}), flush=True)
    for pack in (False, True):
        with tempfile.TemporaryDirectory(prefix="packing_bench_") as run_root:
            tr = Trainer(c2_config(corpus, pack, n_steps), quiet=True, run_root=run_root)
            tr._accum_step, tr._accum_tokens = 0, 0
            for s in range(args.warmup):
                tr.train_step(s)
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            toks = torch.zeros((), device="cuda", dtype=torch.int64)
            e0.record()
            for s in range(args.warmup, n_steps):
                _, ntoks, _ = tr.train_step(s)
                toks += ntoks
            e1.record()
            torch.cuda.synchronize()
            ms = e0.elapsed_time(e1) / args.steps
            print(json.dumps({"part": "end_to_end", "packed": pack, "step_ms": round(ms, 2),
                              "useful_tokens_per_s": round(int(toks) / (ms * args.steps / 1e3)),
                              "useful_tokens_per_step": round(int(toks) / args.steps)}), flush=True)
            del tr
            torch.cuda.empty_cache()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--out", type=str, default=None, help="directory for the generated corpus (default: a temp dir)")
    ap.add_argument("--skip-attention", action="store_true")
    ap.add_argument("--skip-end-to-end", action="store_true")
    args = ap.parse_args()
    from mlx_cuda_distributed_pretraining_b200 import ops
    ops.require_device()
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip()
    print(json.dumps({"gpu": card}), flush=True)
    if not args.skip_attention:
        attention_part(args, ops.lib(), ops)
    if not args.skip_end_to_end:
        if args.out:
            Path(args.out).mkdir(parents=True, exist_ok=True)
            end_to_end_part(args, Path(args.out))
        else:
            with tempfile.TemporaryDirectory(prefix="packing_corpus_") as d:
                end_to_end_part(args, Path(d))


if __name__ == "__main__":
    main()
