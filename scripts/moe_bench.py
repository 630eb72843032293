"""Sparse MoE MLP measurements on one GPU (CUDA events, median of timed rounds after warm-up; dense and MoE rounds
alternate so clock drift hits both alike):

  step      a C2-shaped trainer step (hidden 1024, 12 layers, seq 1024, batch 16) with E = 8, k = 2, I = 1408 per
            expert (the active MLP FLOPs of dense C2's I = 2816) against dense C2: ms and tok/s
  gemm      the four expert-segmented GEMMs + weight gradients of one layer (T = 16384 tokens) against the dense fused
            MLP GEMMs at equal active FLOPs: ms and TFLOP/s
  routing   router GEMM + route + permute + combine (forward) and combine backward + un-permute
  skew      the expert GEMMs with balanced routing against 90 % of the tokens sent to one expert
  decode    one MoE layer's forward at T = 1 and 16 tokens (each active expert pads to 128 rows)

Prints one JSON line per measurement.  Usage: python scripts/moe_bench.py [--rounds 15] [--skip-step]"""
import argparse
import json
import os
import sys
import tempfile

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from mlx_cuda_distributed_pretraining_b200 import ops  # noqa: E402

BF16 = torch.bfloat16


def _time(fn, rounds, warmup=3):
    for _ in range(warmup):
        fn()
    ts = []
    for _ in range(rounds):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        ts.append(a.elapsed_time(b))
    ts.sort()
    return ts[len(ts) // 2]


def _emit(**kw):
    print(json.dumps(kw), flush=True)


def _layer(T, E, k, H, I, skew=False, seed=0):
    g = torch.Generator(device="cuda").manual_seed(seed)
    x = torch.randn((T, H), device="cuda", generator=g).to(BF16)
    wr = (torch.randn((E, H), device="cuda", generator=g) * H ** -0.5).to(BF16)
    if skew:   # 90 % of the tokens prefer expert 0
        x[: int(0.9 * T)] += wr[0].float().sign().to(BF16) * 2
    w2 = (torch.randn((2 * E, I, H), device="cuda", generator=g) * H ** -0.5).to(BF16)   # gate, then up experts
    wd = (torch.randn((E, H, I), device="cuda", generator=g) * I ** -0.5).to(BF16)
    return x, wr, w2[:E], w2[E:], wd


def bench_gemms(rounds, T=16384, E=8, k=2, H=1024, I=1408, skew=False):
    x, wr, wg, wu, wd = _layer(T, E, k, H, I, skew)
    r = ops.moe_route(torch.matmul(x.float(), wr.float().t()), k)
    xp = ops.moe_permute(x, r)
    gu, y = ops.moe_gemm("gateup", "silu", xp, wg, wu, r)
    dyo = torch.randn((r.rows, H), device="cuda").to(BF16)
    gwg, gwu, gwd = (torch.zeros_like(w) for w in (wg, wu, wd))

    def run():
        gu_, y_ = ops.moe_gemm("gateup", "silu", xp, wg, wu, r)
        ops.moe_gemm("down", "silu", y_, wd, None, r)
        dgu, _ = ops.moe_gemm("down_bwd", "silu", dyo, wd, None, r, gu=gu_)
        ops.moe_gemm("gateup_dgrad", "silu", dgu, wg, wu, r)
        ops.moe_wgrad(dyo, H, y_, I, gwd, r)
        ops.moe_wgrad(dgu, 2 * I, xp, H, gwg, r)
        ops.moe_wgrad(dgu[:, I:], 2 * I, xp, H, gwu, r)
    ms = _time(run, rounds)
    flops = 2.0 * T * k * H * I * 3 * 3   # three projections, forward + dgrad + wgrad
    counts = r.counts.cpu().tolist()
    return ms, flops / ms / 1e9, counts


def bench_dense(rounds, T=16384, H=1024, I=2816):
    """The dense fused MLP's GEMMs (b200_mlp_gateup_silu_fwd, down, b200_mlp_down_silu_bwd, dgrad, wgrads)."""
    g = torch.Generator(device="cuda").manual_seed(1)
    x = torch.randn((T, H), device="cuda", generator=g).to(BF16)
    w2 = (torch.randn((2 * I, H), device="cuda", generator=g) * H ** -0.5).to(BF16)
    g2 = torch.zeros_like(w2)
    wg, wu = w2[:I], w2[I:]      # adjacent rows and adjacent gradients, as the flat store lays them out
    wd = (torch.randn((H, I), device="cuda", generator=g) * I ** -0.5).to(BF16)
    for w, gr in ((wg, g2[:I]), (wu, g2[I:]), (wd, torch.zeros_like(wd))):
        w.grad = gr
        w._b200_flat_grad = True
    xx = x.clone().requires_grad_(True)
    d = torch.randn((T, H), device="cuda").to(BF16)

    def run():
        out = ops._MlpFn.apply(xx, wg, wu, wd, "silu")
        out.backward(d)
    ms = _time(run, rounds)
    return ms, 2.0 * T * H * I * 3 * 3 / ms / 1e9


def bench_routing(rounds, T=16384, E=8, k=2, H=1024, I=1408):
    x, wr, wg, wu, wd = _layer(T, E, k, H, I)
    lg = torch.matmul(x.float(), wr.float().t())
    r = ops.moe_route(lg, k)
    xp = ops.moe_permute(x, r)
    gu, y = ops.moe_gemm("gateup", "silu", xp, wg, wu, r)
    yo, _ = ops.moe_gemm("down", "silu", y, wd, None, r)
    dout = torch.randn((T, H), device="cuda").to(BF16)

    def fwd():
        rr = ops.moe_route(torch.matmul(x.float(), wr.float().t()), k)
        ops.moe_permute(x, rr)
        ops.moe_combine(yo, rr)

    def bwd():
        dyo, _, dl = ops.moe_combine_bwd(dout, yo, r, None)
        ops.moe_unpermute(dyo, r, torch.matmul(dl, wr.float()))
    return _time(fwd, rounds), _time(bwd, rounds)


def bench_decode(rounds, B, E=8, k=2, H=1024, I=1408):
    x, wr, wg, wu, wd = _layer(B, E, k, H, I)
    with torch.no_grad():
        return _time(lambda: ops.moe(x, wr, wg, wu, wd, k, "silu"), rounds)


def bench_step(rounds):
    from mlx_cuda_distributed_pretraining_b200.core.training import Config, Trainer
    import yaml
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    base = yaml.safe_load(open(os.path.join(root, "configs", "c2-llama80m-muon.yaml")))
    base["system"]["mixed_precision"] = True
    base["system"]["precision"] = "bfloat16"
    moe = json.loads(json.dumps(base))
    moe["model"]["misc"].update(variant="mlx_lm", num_local_experts=8, num_experts_per_tok=2)
    moe["model"]["dimensions"]["intermediate_size"] = 1408
    moe["model"]["rope"].pop("enabled", None)
    base["model"]["misc"]["variant"] = "mlx_lm"
    base["model"]["rope"].pop("enabled", None)
    trainers = {}
    for name, d in (("dense", base), ("moe", moe)):
        d["name"] = f"moe-bench-{name}"
        trainers[name] = Trainer(Config.from_dict(d), synthetic=True, quiet=True, run_root=tempfile.mkdtemp())
    for tr in trainers.values():
        tr._accum_step, tr._accum_tokens = 0, 0
    times = {n: [] for n in trainers}
    step = {n: 0 for n in trainers}
    for rnd in range(rounds + 3):
        for n, tr in trainers.items():
            batch = tr.data_manager.generate_batch(step[n])
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            tr.train_step(step[n], batch)
            b.record()
            b.synchronize()
            step[n] += 1
            if rnd >= 3:
                times[n].append(a.elapsed_time(b))
    for n, tr in trainers.items():
        ts = sorted(times[n])
        ms = ts[len(ts) // 2]
        hp = tr.config.training.hyperparameters
        toks = hp["batch_size"] * tr.config.data.preprocessing["max_context_size"]
        _emit(measure="step", model=n, ms=round(ms, 3), tok_per_s=round(toks / ms * 1e3))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=15)
    ap.add_argument("--skip-step", action="store_true")
    a = ap.parse_args()
    ops.require_device()
    _emit(device=torch.cuda.get_device_name(), note="median of CUDA-event rounds")
    ms, tf, counts = bench_gemms(a.rounds)
    _emit(measure="gemm", kind="moe_E8_k2_I1408_T16384", ms=round(ms, 3), tflops=round(tf, 1), counts=counts)
    ms, tf = bench_dense(a.rounds)
    _emit(measure="gemm", kind="dense_fused_I2816_T16384", ms=round(ms, 3), tflops=round(tf, 1))
    ms, tf, counts = bench_gemms(a.rounds, skew=True)
    _emit(measure="skew", kind="90pct_to_one_expert", ms=round(ms, 3), tflops=round(tf, 1), counts=counts)
    f, b = bench_routing(a.rounds)
    _emit(measure="routing", fwd_ms=round(f, 3), bwd_ms=round(b, 3))
    for B in (1, 16):
        _emit(measure="decode", tokens=B, layer_ms=round(bench_decode(a.rounds, B), 4))
    if not a.skip_step:
        bench_step(a.rounds)


if __name__ == "__main__":
    main()
