"""ALiBi attention (`model.attention.alibi`): what the bias costs, and what it buys past the training length.

1. Attention forward + backward as the training step calls them: b200_attn_fwd + b200_attn_bwd_strided (causal)
   against b200_attn_fwd_alibi + b200_attn_bwd_alibi (pos = NULL, no window, the standard slopes) at the layer shapes
   of C2 (B16 S1024 H16/Hk8 D64), C3 (B16 S2048 H16/Hk8 D64) and C5 (B16 S2048 H16/Hk16 D128), plus packed ALiBi
   (documents of 100-900 tokens) and windowed ALiBi (W = 512) at C3's shape against the document / window entries.
   Causal and ALiBi calls alternate in rounds inside one process; each line reports the median round.
2. Decode attention (bf16 cache, C2 heads H16/Hk8 D64, B32) at contexts 8192 and 32768: b200_attn_decode against
   b200_attn_decode_alibi, alternating.
3. A C2-shaped trainer step (C2's config: B16 S1024) with and without `alibi`, alternating rounds of steps.
4. Length extrapolation: a small model (hidden 128, 2 layers, 4 heads of 32, fp32) trained for a fixed number of
   AdamW steps at context S on a seeded stream of random 16-token spans (vocabulary 64) each followed by its repeat,
   evaluated (mean cross-entropy on held-out rows; ln 64 = 4.16 knows nothing, about 2.08 copies every repeat
   perfectly) at S, 2S and 4S, for the reference block with no positions, with RoPE and with
   ALiBi.  RoPE's tables end at max_position_embeddings = S, so its longer rows are reported as not run.

CUDA events over many launches after warm-up; the card name and power limit head the output.  One JSON line per
measurement.

    python scripts/alibi_bench.py [--iters 20] [--rounds 5] [--warmup 3] [--steps 10] [--train-steps 1500]
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


def _doc_positions(B, S, seed):
    import torch
    g = torch.Generator().manual_seed(seed)
    rows = []
    for _ in range(B):
        p, n = [], 0
        while n < S:
            L = min(int(torch.randint(100, 900, (1,), generator=g)), S - n)
            p += list(range(L))
            n += L
        rows.append(p)
    return torch.tensor(rows, dtype=torch.int32, device="cuda")


def attention_part(args, L):
    import torch
    from mlx_cuda_distributed_pretraining_b200.arch.flash_attention import alibi_slopes
    st = torch.cuda.current_stream().cuda_stream
    cases = [(tag, shape, "rows") for tag, shape in SHAPES.items()] + [("c3", SHAPES["c3"], "packed"),
                                                                        ("c3", SHAPES["c3"], "window512")]
    for tag, (B, S, H, Hk, D), kind in cases:
        torch.manual_seed(0)
        q = torch.randn(B, S, H, D, device="cuda").to(torch.bfloat16)
        k, v = (torch.randn(B, S, Hk, D, device="cuda").to(torch.bfloat16) for _ in range(2))
        do = torch.randn(B, S, H, D, device="cuda").to(torch.bfloat16)
        o, dq = torch.empty_like(q), torch.empty_like(q)
        lse = torch.empty(B, H, S, device="cuda")
        dkv = torch.empty(B, S, 2 * Hk, D, device="cuda", dtype=torch.bfloat16)
        ws = torch.empty(int(L.b200_attn_bwd_window_workspace_bytes(B, S, H, Hk, D)), device="cuda",
                         dtype=torch.uint8)
        slopes = alibi_slopes(H).cuda()
        sc = ctypes.c_float(D ** -0.5)
        pos = _doc_positions(B, S, 1) if kind == "packed" else None
        pp = None if pos is None else pos.data_ptr()
        W = 512 if kind == "window512" else -1
        dk, dv = dkv.data_ptr(), dkv[:, :, Hk:].data_ptr()

        def base():
            if kind == "rows":
                assert L.b200_attn_fwd(q.data_ptr(), k.data_ptr(), v.data_ptr(), o.data_ptr(), lse.data_ptr(),
                                       B, S, H, Hk, D, sc, 1, st) == 0
                assert L.b200_attn_bwd_strided(q.data_ptr(), k.data_ptr(), v.data_ptr(), o.data_ptr(), do.data_ptr(),
                                               lse.data_ptr(), dq.data_ptr(), dk, dv, B, S, H, Hk, D, sc, 1, 2 * Hk,
                                               ws.data_ptr(), ws.numel(), st) == 0
            else:
                assert L.b200_attn_fwd_window(q.data_ptr(), k.data_ptr(), v.data_ptr(), o.data_ptr(), lse.data_ptr(),
                                              pp, W if W >= 0 else S, B, S, H, Hk, D, sc, st) == 0
                assert L.b200_attn_bwd_window(q.data_ptr(), k.data_ptr(), v.data_ptr(), o.data_ptr(), do.data_ptr(),
                                              lse.data_ptr(), pp, W if W >= 0 else S, dq.data_ptr(), dk, dv, B, S, H,
                                              Hk, D, sc, 2 * Hk, ws.data_ptr(), ws.numel(), st) == 0

        def alibi():
            assert L.b200_attn_fwd_alibi(q.data_ptr(), k.data_ptr(), v.data_ptr(), o.data_ptr(), lse.data_ptr(), pp,
                                         W, slopes.data_ptr(), B, S, H, Hk, D, sc, st) == 0
            assert L.b200_attn_bwd_alibi(q.data_ptr(), k.data_ptr(), v.data_ptr(), o.data_ptr(), do.data_ptr(),
                                         lse.data_ptr(), pp, W, slopes.data_ptr(), dq.data_ptr(), dk, dv, B, S, H, Hk,
                                         D, sc, 2 * Hk, ws.data_ptr(), ws.numel(), st) == 0

        t = _alternate({"base": base, "alibi": alibi}, args.iters, args.rounds, args.warmup)
        print(json.dumps({"part": "attention", "shape": tag, "layout": kind, "B": B, "S": S, "H": H, "Hk": Hk,
                          "D": D, "baseline": "causal" if kind == "rows" else kind.replace("512", "") + " (no bias)",
                          "ms_fwd_bwd_base": round(t["base"], 4), "ms_fwd_bwd_alibi": round(t["alibi"], 4),
                          "alibi_over_base": round(t["alibi"] / t["base"], 4)}), flush=True)
        del q, k, v, do, o, dq, lse, dkv, ws
        torch.cuda.empty_cache()


def decode_part(args):
    import torch
    from mlx_cuda_distributed_pretraining_b200 import ops
    from mlx_cuda_distributed_pretraining_b200.arch.flash_attention import alibi_slopes
    B, H, Hk, D = 32, 16, 8, 64
    slopes = alibi_slopes(H).cuda()
    for ctx in (8192, 32768):
        g = torch.Generator(device="cuda").manual_seed(0)
        q = torch.randn(B, H, D, device="cuda", generator=g).to(torch.bfloat16)
        kc = torch.randn(B, ctx, Hk, D, device="cuda", generator=g).to(torch.bfloat16)
        vc = torch.randn(B, ctx, Hk, D, device="cuda", generator=g).to(torch.bfloat16)
        lens = torch.full((B,), ctx, device="cuda", dtype=torch.int32)
        ws = torch.empty(ops.attention_decode_workspace_bytes(B, H, ctx, D), device="cuda", dtype=torch.uint8)
        t = _alternate({"base": lambda: ops.attention_decode(q, kc, vc, lens, workspace=ws),
                        "alibi": lambda: ops.attention_decode(q, kc, vc, lens, workspace=ws, alibi=slopes)},
                       args.iters * 10, args.rounds, args.warmup)
        nbytes = 2 * B * ctx * Hk * D * 2
        print(json.dumps({"part": "decode", "B": B, "H": H, "Hk": Hk, "D": D, "context": ctx,
                          "us_base": round(t["base"] * 1e3, 1), "us_alibi": round(t["alibi"] * 1e3, 1),
                          "TB_per_s_alibi": round(nbytes / t["alibi"] / 1e9, 2)}), flush=True)
        del q, kc, vc, ws
        torch.cuda.empty_cache()


def trainer_part(args):
    import torch
    from mlx_cuda_distributed_pretraining_b200.core.training import Config, Trainer
    trainers, dirs = {}, []
    for name, alibi in (("base", None), ("alibi", True)):
        cfg = Config.from_yaml(str(ROOT / "configs" / "c2-llama80m-muon.yaml"))
        cfg.name = f"alibi_bench_{name}"
        cfg.model.attention = {**cfg.model.attention, "alibi": alibi}
        cfg.training.hyperparameters["iters"] = args.warmup + args.steps * args.rounds
        cfg.system.distributed = False
        d = tempfile.TemporaryDirectory(prefix="alibi_bench_")
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
                      "step_ms_alibi": round(ms["alibi"], 2), "alibi_over_base": round(ms["alibi"] / ms["base"], 4),
                      "tokens_per_s_alibi": round(B * S / (ms["alibi"] / 1e3))}), flush=True)
    for d in dirs:
        d.cleanup()


VOCAB, SPAN = 64, 16


def repeat_stream(B, S, seed, span=SPAN, vocab=VOCAB):
    """[B, S + 1] int64 tokens: random spans of `span` tokens, each followed by its repeat.  Half of every row is
    predictable only by looking `span` positions back."""
    import torch
    g = torch.Generator().manual_seed(seed)
    n = -(-(S + 1) // (2 * span))
    x = torch.randint(0, vocab, (B, n, span), generator=g)
    return torch.cat([x, x], dim=2).reshape(B, -1)[:, :S + 1]


def extrapolation_part(args):
    import torch
    from mlx_cuda_distributed_pretraining_b200.arch.llama import Model, ModelArgs
    from mlx_cuda_distributed_pretraining_b200.core.training import init_model_
    S = args.train_context
    for name, rope, alibi in (("no_positions", False, False), ("rope", True, False), ("alibi", False, True)):
        args_m = ModelArgs(model_type="llama", hidden_size=128, num_hidden_layers=2, intermediate_size=256,
                           num_attention_heads=4, num_key_value_heads=4, head_dim=32, vocab_size=VOCAB,
                           max_position_embeddings=S, tie_word_embeddings=True, apply_rope=rope, alibi=alibi)
        model = Model(args_m)
        init_model_(model, args_m, seed=0)
        model = model.cuda()
        opt = torch.optim.AdamW(model.parameters(), lr=3e-3, weight_decay=0.0)
        for step in range(args.train_steps):
            toks = repeat_stream(16, S, seed=1000 + step).cuda()
            logits = model(toks[:, :-1]).float()
            loss = torch.nn.functional.cross_entropy(logits.reshape(-1, VOCAB), toks[:, 1:].reshape(-1))
            opt.zero_grad(set_to_none=True)
            loss.backward()
            opt.step()
        row = {"part": "extrapolation", "model": name, "train_context": S, "train_steps": args.train_steps,
               "final_train_loss": round(float(loss.detach()), 4)}
        with torch.no_grad():
            for mult in (1, 2, 4):
                L = S * mult
                if rope and L > S:
                    row[f"eval_loss_{mult}S"] = "not run: the RoPE tables end at max_position_embeddings"
                    continue
                toks = repeat_stream(8, L, seed=7).cuda()
                logits = model(toks[:, :-1]).float()
                row[f"eval_loss_{mult}S"] = round(float(torch.nn.functional.cross_entropy(
                    logits.reshape(-1, VOCAB), toks[:, 1:].reshape(-1))), 4)
        print(json.dumps(row), flush=True)
        del model, opt
        torch.cuda.empty_cache()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--train-steps", type=int, default=1500)
    ap.add_argument("--train-context", type=int, default=256)
    ap.add_argument("--skip-attention", action="store_true")
    ap.add_argument("--skip-decode", action="store_true")
    ap.add_argument("--skip-trainer", action="store_true")
    ap.add_argument("--skip-extrapolation", action="store_true")
    args = ap.parse_args()
    from mlx_cuda_distributed_pretraining_b200 import ops
    ops.require_device()
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip()
    print(json.dumps({"gpu": card}), flush=True)
    if not args.skip_attention:
        attention_part(args, ops.lib())
    if not args.skip_decode:
        decode_part(args)
    if not args.skip_trainer:
        trainer_part(args)
    if not args.skip_extrapolation:
        extrapolation_part(args)


if __name__ == "__main__":
    main()
