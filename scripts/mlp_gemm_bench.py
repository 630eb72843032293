"""Compare two builds of the library on the wgmma engine's flagship launches: the fused MLP GEMMs
(b200_mlp_gateup_glu_fwd, b200_mlp_down_glu_bwd) at the C2 and C3 layer shapes, and one grouped 5-step
Newton-Schulz over C2's five parameter shape groups (b200_newton_schulz_multi).

On the same seeded inputs it asserts that both builds produce bit-identical gu, y, dgu and Newton-Schulz outputs,
then times each launch with CUDA events, alternating the two builds in rounds, over --iters launches per build
after warm-up.  Prints one JSON line per launch: ms per call for each build, per-step totals (C2: 12 layers; C3: 16
layers x 8 accumulation micro-batches), algorithmic TFLOP/s and GB/s.  The output is headed by the card name,
power limit and maximum SM clock.

    python scripts/mlp_gemm_bench.py --base path/to/other/libb200hotpath.so [--iters 60] [--warmup 10]
"""
import argparse
import ctypes
import json
import subprocess
import sys
from pathlib import Path

import torch

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))

# name: (M tokens per micro-batch, hidden H, intermediate I, GLU launches of each kind per optimizer step)
MLP_SHAPES = {"c2": (16 * 1024, 1024, 2816, 12), "c3": (16 * 2048, 1024, 4096, 16 * 8)}
# C2's Muon shape groups [batch, rows, cols]: q/o, k/v, gate/up, down, embedding
NS_GROUPS = [(24, 1024, 1024), (24, 512, 1024), (24, 2816, 1024), (12, 1024, 2816), (1, 32003, 1024)]
NS_STEPS = 5
NS_COEFFS = (3.4445, -4.7750, 2.0315)


def load(path):
    from mlx_cuda_distributed_pretraining_b200._lib import SIGNATURES
    handle = ctypes.CDLL(str(path))
    for name, (res, args) in SIGNATURES.items():
        if not hasattr(handle, name):  # an older build: entries added since are not compared
            continue
        fn = getattr(handle, name)
        fn.restype, fn.argtypes = res, args
    return handle


def ok(L, rc, what):
    if rc != 0:
        raise RuntimeError(f"{what}: rc={rc}: {L.b200_last_error().decode()}")


def time_pair(calls, iters, warmup, rounds=5):
    """calls: {tag: fn}; each round times iters // rounds launches of every build in turn.  Returns ms per call."""
    for fn in calls.values():
        for _ in range(warmup):
            fn()
    torch.cuda.synchronize()
    per = max(iters // rounds, 1)
    total = {tag: 0.0 for tag in calls}
    for _ in range(rounds):
        for tag, fn in calls.items():
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(per):
                fn()
            e1.record()
            torch.cuda.synchronize()
            total[tag] += e0.elapsed_time(e1)
    return {tag: t / (per * rounds) for tag, t in total.items()}


def report(kernel, shape, ms, flops, nbytes, per_step):
    line = {"kernel": kernel, "shape": shape}
    for tag, t in ms.items():
        line[tag] = {"ms": round(t, 4), "ms_per_step": round(t * per_step, 2),
                     "tflops": round(flops / t / 1e9, 1), "gbps": round(nbytes / t / 1e6, 1)}
    line["speedup"] = round(ms["base"] / ms["new"], 3)
    print(json.dumps(line), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--base", required=True, help="the other build of libb200hotpath.so")
    ap.add_argument("--iters", type=int, default=60)
    ap.add_argument("--warmup", type=int, default=10)
    args = ap.parse_args()
    from mlx_cuda_distributed_pretraining_b200 import _lib, ops
    ops.require_device()
    libs = {"base": load(args.base), "new": load(_lib.LIB_PATH)}
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip()
    print(json.dumps({"gpu": card, "base": str(args.base), "new": str(_lib.LIB_PATH)}), flush=True)
    st = torch.cuda.current_stream().cuda_stream
    bf = torch.bfloat16

    for shape, (M, H, I, per_step) in MLP_SHAPES.items():
        g = torch.Generator(device="cuda").manual_seed(1234)
        x = (torch.randn(M, H, device="cuda", generator=g)).to(bf)
        W2 = (torch.randn(2 * I, H, device="cuda", generator=g) * H ** -0.5).to(bf)
        Wd = (torch.randn(H, I, device="cuda", generator=g) * I ** -0.5).to(bf)
        dy = torch.randn(M, H, device="cuda", generator=g).to(bf)
        out = {tag: (torch.empty(M, 2 * I, device="cuda", dtype=bf), torch.empty(M, I, device="cuda", dtype=bf),
                     torch.empty(M, 2 * I, device="cuda", dtype=bf)) for tag in libs}

        def fwd(tag):
            gu, y, _ = out[tag]
            return lambda: ok(libs[tag], libs[tag].b200_mlp_gateup_glu_fwd(x.data_ptr(), W2.data_ptr(), gu.data_ptr(),
                                                                         y.data_ptr(), M, H, I, st), "gateup")

        def bwd(tag):  # both builds read the base build's gu, so dgu is compared on identical inputs
            gu, dgu = out["base"][0], out[tag][2]
            return lambda: ok(libs[tag], libs[tag].b200_mlp_down_glu_bwd(dy.data_ptr(), Wd.data_ptr(), gu.data_ptr(),
                                                                       dgu.data_ptr(), M, H, I, st), "down")

        for tag in libs:
            fwd(tag)()
        for tag in libs:
            bwd(tag)()
        torch.cuda.synchronize()
        for i, name in enumerate(("gu", "y", "dgu")):
            assert torch.equal(out["base"][i], out["new"][i]), f"{shape}: {name} differs between the builds"
        print(json.dumps({"shape": shape, "bit_identical": ["gu", "y", "dgu"]}), flush=True)
        report("mlp_gateup_glu_fwd", shape, time_pair({t: fwd(t) for t in libs}, args.iters, args.warmup),
               2 * M * H * 2 * I, 2 * (M * H + 2 * I * H + 3 * M * I), per_step)
        report("mlp_down_glu_bwd", shape, time_pair({t: bwd(t) for t in libs}, args.iters, args.warmup),
               2 * M * H * I, 2 * (M * H + H * I + 4 * M * I), per_step)
        del x, W2, Wd, dy, out

    from mlx_cuda_distributed_pretraining_b200._lib import NsGroup
    g = torch.Generator(device="cuda").manual_seed(99)
    xs = [(torch.randn(b, r, c, device="cuda", generator=g) * 0.02).to(bf) for b, r, c in NS_GROUPS]
    scales = [ops.ns_scales(ops.sumsq(x)) for x in xs]
    ns_out, arrs = {}, {}
    for tag in libs:
        ns_out[tag] = [torch.empty_like(x) for x in xs]
        arr = (NsGroup * len(xs))()
        for e, x, o, (inv, inv2) in zip(arr, xs, ns_out[tag], scales):
            e.x_in, e.x_out = x.data_ptr(), o.data_ptr()
            e.batch, e.rows, e.cols = x.shape
            e.inv_norm, e.inv_norm_sq = inv.data_ptr(), inv2.data_ptr()
            e.peer_out, e.n_peers = None, 0
        arrs[tag] = arr
    need = max(int(L.b200_newton_schulz_multi_workspace_bytes(arrs[t], len(xs), NS_STEPS)) for t, L in libs.items())
    ws = torch.empty(need, device="cuda", dtype=torch.uint8)

    def ns(tag):
        L = libs[tag]
        return lambda: ok(L, L.b200_newton_schulz_multi(arrs[tag], len(xs), NS_STEPS, *NS_COEFFS, ws.data_ptr(), need,
                                                        st), "newton_schulz_multi")

    for tag in libs:
        ns(tag)()
    torch.cuda.synchronize()
    for i, (a, b) in enumerate(zip(ns_out["base"], ns_out["new"])):
        assert torch.equal(a, b), f"Newton-Schulz group {NS_GROUPS[i]} differs between the builds"
    print(json.dumps({"shape": "c2 muon groups", "bit_identical": ["newton_schulz"]}), flush=True)
    flops = sum(NS_STEPS * b * (4 * min(r, c) ** 2 * max(r, c) + 2 * min(r, c) ** 3) for b, r, c in NS_GROUPS)
    report("newton_schulz_multi", "c2", time_pair({t: ns(t) for t in libs}, args.iters, args.warmup), flops, 0, 1)


if __name__ == "__main__":
    main()
