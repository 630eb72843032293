"""Quantized KV cache on the GPU: b200_kv_quantize and b200_kv_append_quant bit for bit against the CPU oracle
(tests/kv_quant_oracle.py), b200_attn_decode_quant against fp64 attention over the dequantised cache, determinism,
and the model / generate() / CLI paths with kv_bits."""
from __future__ import annotations

import os
import subprocess
import sys
import tempfile
from pathlib import Path

import pytest
import torch
import yaml

from tests import kv_quant_oracle as KQ

pytestmark = pytest.mark.gpu

ROOT = Path(__file__).resolve().parents[1]
CODE_CANARY = 0xAB
PAR_CANARY = 1234.5


def _ops():
    from mlx_cuda_distributed_pretraining_b200 import ops
    ops.require_device()
    return ops


def _in_nan(x: torch.Tensor, extra: int = 4096) -> torch.Tensor:
    """x copied to the front of a NaN-filled allocation (a view of the same shape)."""
    buf = torch.full((x.numel() + extra,), float("nan"), device="cuda", dtype=x.dtype)
    buf[:x.numel()].copy_(x.reshape(-1))
    return buf[:x.numel()].view(x.shape)


def _canary_bufs(B, s_max, Hk, D, bits, g):
    from mlx_cuda_distributed_pretraining_b200 import ops
    cs, ps = ops.kv_quant_shapes(B, s_max, Hk, D, bits, g)
    return (torch.full(cs, CODE_CANARY, device="cuda", dtype=torch.uint8),
            torch.full(cs, CODE_CANARY, device="cuda", dtype=torch.uint8),
            torch.full(ps, PAR_CANARY, device="cuda"), torch.full(ps, PAR_CANARY, device="cuda"))


def _special_groups(x: torch.Tensor, bits: int, g: int) -> None:
    """Constant, single-outlier, signed-zero and half-way-tie groups in place of some random ones (x [B, S, Hk, D])."""
    n = (1 << bits) - 1
    x[0, 0, 0, :g] = 3.0
    x[0, 1, 0, :g] = 0.01 * torch.arange(g, dtype=torch.float32, device=x.device).sin()
    x[0, 1, 0, g // 2] = 100.0
    z = torch.zeros(g, device=x.device)
    z[::2] = -0.0
    x[0, 2, 0, :g] = z
    # mn = 0, mx = n / 2 gives s = 0.5 exactly; 0.25, 0.75, 1.25, 2.25 are exact ties of (x - b) / s
    t = torch.zeros(g, device=x.device)
    t[1], t[2], t[3], t[4], t[5] = n * 0.5, 0.25, 0.75, 1.25, 2.25
    x[0, 3, 0, :g] = t
    x[-1, 4, -1, -g:] = -0.0


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float32], ids=["bf16", "fp32"])
@pytest.mark.parametrize("bits", [4, 8])
@pytest.mark.parametrize("D,g", [(32, 32), (64, 32), (64, 64), (128, 32), (128, 64), (128, 128)])
def test_kv_quantize_bit_exact(dtype, bits, D, g):
    ops = _ops()
    B, S, Hk, s_max, n = 3, 45, 3, 64, 41
    gen = torch.Generator(device="cuda").manual_seed(D * 10 + g + bits)
    x = [torch.randn(B, S, Hk, D, device="cuda", generator=gen) * 3 for _ in range(2)]
    for t in x:
        _special_groups(t, bits, g)
    k, v = (_in_nan(t.to(dtype)) for t in x)
    kc, vc, kp, vp = _canary_bufs(B, s_max, Hk, D, bits, g)
    ops.kv_quantize(k, v, kc, vc, kp, vp, bits, g, n=n)
    torch.cuda.synchronize()
    for src, codes, par in ((k, kc, kp), (v, vc, vp)):
        c_ref, p_ref = KQ.cache_layout(src[:, :n].cpu(), bits, g)
        assert torch.equal(codes[:, :n].cpu(), c_ref)
        assert torch.equal(par[:, :, :n].cpu().view(torch.int32), p_ref.view(torch.int32))  # bits, incl. +0
        assert bool((codes[:, n:] == CODE_CANARY).all()), "codes written at or past n"
        assert bool((par[:, :, n:] == PAR_CANARY).all()), "parameters written at or past n"


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float32], ids=["bf16", "fp32"])
@pytest.mark.parametrize("bits,g", [(8, 64), (4, 32), (4, 128)])
@pytest.mark.parametrize("rope", ["none", "interleaved", "half"])
def test_kv_append_quant_matches_bf16_append(dtype, bits, g, rope):
    ops = _ops()
    B, H, Hk, D, s_max = 4, 8, 2, 128, 300
    pos = [0, 7, 299, 128]
    gen = torch.Generator(device="cuda").manual_seed(bits + g)
    q = torch.randn(B, H, D, device="cuda", generator=gen).to(dtype)
    k = torch.randn(B, Hk, D, device="cuda", generator=gen).to(dtype) * 2
    v = torch.randn(B, Hk, D, device="cuda", generator=gen).to(dtype)
    lens = torch.tensor([p + 1 for p in pos], device="cuda", dtype=torch.int32)
    tables = ops.rope_tables(512, D, 10000.0, "cuda") if rope != "none" else None
    layout = "half" if rope == "half" else "interleaved"
    q_ref, q_got = q.clone(), q.clone()
    kc16 = torch.zeros(B, s_max, Hk, D, device="cuda", dtype=dtype)
    vc16 = torch.zeros_like(kc16)
    ops.kv_append(q_ref, k, v, kc16, vc16, lens, tables, layout=layout)
    kc, vc, kp, vp = _canary_bufs(B, s_max, Hk, D, bits, g)
    ops.kv_append_quant(q_got, k, v, kc, vc, kp, vp, lens, bits, g, tables, layout=layout)
    torch.cuda.synchronize()
    assert torch.equal(q_got.view(torch.uint8), q_ref.view(torch.uint8)), "q differs from the bf16 path's"
    written = torch.zeros(B, s_max, dtype=torch.bool)
    for b, p in enumerate(pos):
        written[b, p] = True
        for src, codes, par in ((kc16, kc, kp), (vc16, vc, vp)):
            c_ref, p_ref = KQ.cache_layout(src[b:b + 1, p:p + 1].cpu(), bits, g)
            assert torch.equal(codes[b, p].cpu(), c_ref[0, 0])
            assert torch.equal(par[b, :, p].cpu().view(torch.int32), p_ref[0, :, 0].view(torch.int32))
    rest = ~written.cuda()
    for codes, par in ((kc, kp), (vc, vp)):
        assert bool((codes[rest] == CODE_CANARY).all()), "codes written outside [b, lens[b] - 1]"
        assert bool((par.transpose(1, 2)[rest] == PAR_CANARY).all()), "parameters written outside [b, lens[b] - 1]"


# -- decode attention ----------------------------------------------------------------------------------------------
def _quant_cache(lens, s_max, H, Hk, D, dtype, bits, g, seed):
    """q, the quantized cache (parameters NaN at and past each row's length) and its dequantised fp64 values."""
    ops = _ops()
    gen = torch.Generator(device="cuda").manual_seed(seed)
    B = len(lens)
    q = torch.randn(B, H, D, device="cuda", generator=gen).to(dtype)
    k = torch.randn(B, s_max, Hk, D, device="cuda", generator=gen).to(dtype)
    v = torch.randn(B, s_max, Hk, D, device="cuda", generator=gen).to(dtype)
    bufs = _canary_bufs(B, s_max, Hk, D, bits, g)
    ops.kv_quantize(k, v, *bufs, bits, g)
    kc, vc, kp, vp = bufs
    for b, n in enumerate(lens):  # never read
        kp[b, :, n:] = float("nan")
        vp[b, :, n:] = float("nan")
    kd = KQ.dequantize_cache(kc.cpu(), kp.cpu(), bits, g).double()
    vd = KQ.dequantize_cache(vc.cpu(), vp.cpu(), bits, g).double()
    # per element s |c| + |b|: the magnitude the kernel's s (q . c) + b (sum q) and (p s) c + p b forms work with
    def mag(codes, par):
        p = par.cpu().permute(0, 2, 1, 3, 4).double()
        c = KQ.unpack(codes.cpu(), bits).double()
        c = c.reshape(*c.shape[:-1], D // g, g)
        return (p[..., 0:1].abs() * c + p[..., 1:2].abs()).reshape(B, s_max, Hk, D)
    return q, bufs, torch.tensor(lens, device="cuda", dtype=torch.int32), kd, vd, mag(kc, kp), mag(vc, vp)


def _reference(q, kd, vd, km, vm, lens, scale, window=None, slopes=None):
    """fp64 attention of each row's query over its visible dequantised keys: o, lse, sum_j p_j vm_j and the largest
    score magnitude sum_d |q_d| km_jd * scale (the error bound's inputs)."""
    B, H, D = q.shape
    Hk = kd.shape[2]
    out, absterm, lses, smag = [], [], [], []
    for b, n in enumerate(lens):
        lo = 0 if window is None else max(0, n - 1 - window)
        rep = lambda t: t[b, lo:n].repeat_interleave(H // Hk, dim=1)  # noqa: E731
        k, v, kmb, vmb = rep(kd), rep(vd), rep(km), rep(vm)
        qb = q[b].double().cpu()
        s = torch.einsum("hd,nhd->hn", qb, k) * scale
        if slopes is not None:
            s = s + slopes.double().cpu()[:, None] * (torch.arange(lo, n, dtype=torch.float64) - (n - 1))[None]
        lse = torch.logsumexp(s, dim=-1)
        p = torch.exp(s - lse[:, None])
        out.append(torch.einsum("hn,nhd->hd", p, v))
        absterm.append(torch.einsum("hn,nhd->hd", p, vmb))
        smag.append((torch.einsum("hd,nhd->hn", qb.abs(), kmb) * scale).amax(-1))
        lses.append(lse)
    return torch.stack(out), torch.stack(absterm), torch.stack(lses), torch.stack(smag)


# The bound follows tests/test_gpu_generation.py: 2^-8 |R| for a bf16 output's rounding plus C 2^-24 (1 + E) sum p m,
# where m = s |c| + |b| per value element and E the largest score magnitude built from the same terms (an fp32 error
# of the scores moves p by that relative amount).
C_BOUND = 64.0
LENS = [1, 31, 32, 33, 255, 256, 257, 1000, 1024]
S_MAX = 1024


def _decode_raw(q, bufs, lens, bits, g, scale, window=-1, slopes=None, ws_bytes=None):
    """b200_attn_decode_quant into canary-filled o / lse buffers: (rc, o, lse, canaries intact)."""
    from mlx_cuda_distributed_pretraining_b200._lib import lib
    ops = _ops()
    B, H, D = q.shape
    kc = bufs[0]
    Hk, s_max = kc.shape[2], kc.shape[1]
    can = 64
    obuf = torch.full((B * H * D + 2 * can,), 1234.5, device="cuda", dtype=q.dtype)
    lbuf = torch.full((B * H + 2 * can,), 1234.5, device="cuda", dtype=torch.float32)
    need = ops.attention_decode_workspace_bytes(B, H, s_max, D)
    ws = torch.empty(max(need, 16), device="cuda", dtype=torch.uint8)
    rc = lib().b200_attn_decode_quant(q.data_ptr(), *[t.data_ptr() for t in bufs], lens.data_ptr(),
                                      obuf[can:].data_ptr(), lbuf[can:].data_ptr(), window,
                                      None if slopes is None else slopes.data_ptr(), B, s_max, H, Hk, D, bits, g,
                                      float(scale), int(q.dtype == torch.bfloat16), ws.data_ptr(),
                                      need if ws_bytes is None else ws_bytes, torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    intact = bool((obuf[:can] == 1234.5).all() and (obuf[-can:] == 1234.5).all() and
                  (lbuf[:can] == 1234.5).all() and (lbuf[-can:] == 1234.5).all())
    return rc, obuf[can:can + B * H * D].view(B, H, D), lbuf[can:can + B * H].view(B, H), intact


def _check_decode(dtype, bits, D, g, H, Hk, window=None, alibi=False, seed=0):
    from mlx_cuda_distributed_pretraining_b200.arch.flash_attention import alibi_slopes
    scale = D ** -0.5
    q, bufs, lens, kd, vd, km, vm = _quant_cache(LENS, S_MAX, H, Hk, D, dtype, bits, g, seed)
    slopes = alibi_slopes(H).cuda() if alibi else None
    rc, o, lse, intact = _decode_raw(q, bufs, lens, bits, g, scale, -1 if window is None else window, slopes)
    assert rc == 0 and intact, "decode attention failed or wrote outside o / lse"
    R, absterm, lse_ref, smag = _reference(q, kd, vd, km, vm, LENS, scale, window, slopes)
    err = (o.double().cpu() - R).abs()
    bound = C_BOUND * 2.0 ** -24 * (1 + smag[..., None]) * absterm
    if dtype == torch.bfloat16:
        bound = bound + 2.0 ** -8 * R.abs()
    ratio = float((err / bound).max())
    lse_err = float(((lse.double().cpu() - lse_ref).abs() / (C_BOUND * 2.0 ** -24 * (1 + smag) + 1e-6)).max())
    print(f"max error/bound {ratio:.3f}, lse {lse_err:.3f} ({dtype}, bits={bits}, D={D}, g={g}, H={H}, Hk={Hk}, "
          f"window={window}, alibi={alibi})")
    assert torch.isfinite(o).all()
    assert ratio <= 1.0 and lse_err <= 1.0


GROUPS = [(8, 8), (8, 4), (12, 4), (16, 4), (16, 2), (8, 1)]  # G = 1, 2, 3, 4, 8, 8


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float32], ids=["bf16", "fp32"])
@pytest.mark.parametrize("bits", [4, 8])
@pytest.mark.parametrize("D,g", [(32, 32), (64, 64), (128, 64), (128, 32), (64, 32), (128, 128)])
def test_decode_quant_matches_fp64(dtype, bits, D, g):
    i = [(32, 32), (64, 64), (128, 64), (128, 32), (64, 32), (128, 128)].index((D, g))
    H, Hk = GROUPS[(i + bits) % len(GROUPS)]
    _check_decode(dtype, bits, D, g, H, Hk, seed=i * 10 + bits)


@pytest.mark.parametrize("bits", [4, 8])
@pytest.mark.parametrize("window", [0, 1, 100, 5000])
@pytest.mark.parametrize("alibi", [False, True], ids=["plain", "alibi"])
def test_decode_quant_window_and_alibi(bits, window, alibi):
    _check_decode(torch.bfloat16, bits, 64, 64, 12, 4, window=window, alibi=alibi, seed=window + bits)


def test_decode_quant_alibi_fp32_all_group_sizes():
    for G, (H, Hk) in enumerate(GROUPS):
        _check_decode(torch.float32, 8, 128, 32, H, Hk, window=None if G % 2 else 300, alibi=True, seed=G)


def test_decode_quant_errors_are_returned_not_launched():
    from mlx_cuda_distributed_pretraining_b200._lib import lib
    q, bufs, lens, *_ = _quant_cache([40, 7], 64, 4, 2, 64, torch.bfloat16, 8, 64, seed=1)
    need = _ops().attention_decode_workspace_bytes(2, 4, 64, 64)
    for kw, code in ((dict(ws_bytes=need - 1), -4), (dict(bits=3), -1), (dict(g=48), -1), (dict(g=128), -1)):
        bits, g = kw.pop("bits", 8), kw.pop("g", 64)
        rc, o, lse, intact = _decode_raw(q, bufs, lens, bits, g, 0.125, **kw)
        assert rc == code, (bits, g, kw, rc)
        assert intact and bool((o == 1234.5).all()) and bool((lse == 1234.5).all()), "an error launched a kernel"
        assert lib().b200_last_error()


@pytest.mark.parametrize("bits", [4, 8])
def test_decode_quant_batch_invariant_and_repeatable(bits):
    ops = _ops()
    H, Hk, D, g = 16, 8, 64, 64
    lens = [1000, 5, 257, 1024, 256, 31]
    q, (kc, vc, kp, vp), lt, *_ = _quant_cache(lens, S_MAX, H, Hk, D, torch.bfloat16, bits, g, seed=3)
    o = ops.attention_decode_quant(q, kc, vc, kp, vp, lt, bits, g)
    assert torch.equal(o, ops.attention_decode_quant(q, kc, vc, kp, vp, lt, bits, g))
    for b in range(len(lens)):
        one = [t[b:b + 1].contiguous() for t in (q, kc, vc, kp, vp, lt)]
        alone = ops.attention_decode_quant(*one, bits, g)
        assert torch.equal(alone[0], o[b]), f"row {b} differs alone vs in the batch"


# -- model level ---------------------------------------------------------------------------------------------------
def _trainer(kind):
    from tests.test_gpu_generation import _trainer as make
    return make(kind)


# Logit tolerance, relative to the row's largest |logit|: the bf16 cache's own (tests/test_gpu_generation.py TOL)
# plus, per layer, the relative change of a cached value, at most s / 2 = range / (2 n) of its group.  Two layers.
def _quant_tol(kind, bits):
    from tests.test_gpu_generation import TOL
    return TOL[kind] + 2 * 1.0 / (2 * ((1 << bits) - 1))


@pytest.mark.parametrize("bits", [4, 8])
@pytest.mark.parametrize("kind", ["bf16_gqa", "bf16_rope"])
def test_prefill_decode_quantized_layers(kind, bits):
    from mlx_cuda_distributed_pretraining_b200.arch.llama import KVCache
    from mlx_cuda_distributed_pretraining_b200.arch.flash_attention import QuantizedKV
    from tests.test_gpu_generation import _rel_rows
    model = _trainer(kind).model
    T, t0 = 300, 260
    tokens = torch.randint(0, 256, (2, T), generator=torch.Generator().manual_seed(5))
    with torch.no_grad():
        full = model(tokens.cuda()).float()[:, t0 - 1:T - 1]

    def run(**kw):
        cache = KVCache(model, 2, T, **kw)
        got = [model.prefill(tokens[:, :t0].cuda(), [t0, t0], cache)]
        for t in range(t0, T - 1):
            got.append(model.decode_step(tokens[:, t].cuda(), cache))
        return torch.stack(got, 1), cache

    dense, _ = run()
    quant, cache = run(kv_bits=bits)
    assert cache.quantized and all(isinstance(kv, QuantizedKV) for kv in cache.layers)
    e_dense, e_full = _rel_rows(quant, dense), _rel_rows(quant, full)
    tol = _quant_tol(kind, bits)
    print(f"{kind} {bits}-bit cache: vs bf16 cache {e_dense:.2e}, vs forward {e_full:.2e} (tolerance {tol:.2e})")
    assert e_dense < tol and e_full < tol


@pytest.mark.parametrize("kind", ["bf16_rope", "c1_fp32_d32"])
def test_conversion_equals_direct_quantized_layers(kind):
    from mlx_cuda_distributed_pretraining_b200.arch.llama import KVCache
    from mlx_cuda_distributed_pretraining_b200.arch.flash_attention import QuantizedKV
    if kind == "c1_fp32_d32":  # fp32 activations, head_dim 32
        from mlx_cuda_distributed_pretraining_b200.core.training import Config, Trainer
        from tests.test_gpu_generation import _cfg
        c = _cfg("c1_fp32")
        c["model"]["attention"].update(num_heads=4, num_kv_heads=2, head_dim=32)
        model = Trainer(Config.from_dict(c), for_training=False, synthetic=True, quiet=True,
                        run_root=tempfile.mkdtemp(prefix="kvq_")).model
    else:
        model = _trainer(kind).model
    t0, start = 40, 43
    tokens = torch.randint(0, 256, (2, t0 + 8), generator=torch.Generator().manual_seed(2)).cuda()
    direct = KVCache(model, 2, t0 + 8, kv_bits=4, kv_group_size=32)
    model.prefill(tokens[:, :t0], [t0, t0 - 9], direct)
    assert direct.quantized and all(isinstance(kv, QuantizedKV) for kv in direct.layers)
    late = KVCache(model, 2, t0 + 8, kv_bits=4, kv_group_size=32, quantized_kv_start=start)
    model.prefill(tokens[:, :t0], [t0, t0 - 9], late)
    assert not late.quantized and late.layers[0].k.shape[1] == 256  # start + 1 rounded up to 256
    steps = 0
    while not late.quantized:
        model.decode_step(tokens[:, t0 + steps], late)
        steps += 1
    assert steps == start + 1 - t0 and all(isinstance(kv, QuantizedKV) for kv in late.layers)
    for a, b in zip(direct.layers, late.layers):  # each row's prompt positions (the decode steps wrote past them)
        for x, y in zip(a.buffers(), b.buffers()):
            for row, n in enumerate((t0, t0 - 9)):
                if x.dtype == torch.uint8:
                    assert torch.equal(x[row, :n], y[row, :n])
                else:
                    assert torch.equal(x[row, :, :n].view(torch.int32), y[row, :, :n].view(torch.int32))


def test_greedy_8bit_matches_full_forward():
    from mlx_cuda_distributed_pretraining_b200.core.generation import generate
    tr = _trainer("bf16_gqa")
    model = tr.model
    prompt = [tr.tokenizer.BOS_TOKEN] + list(range(40, 80))
    n = 48
    out = generate(model, [prompt], max_tokens=n, temperature=0, repetition_penalty=1.0, min_p=None, kv_bits=8)[0]
    tol = _quant_tol("bf16_gqa", 8)
    seq, skipped = list(prompt), 0
    for i, t in enumerate(out):
        with torch.no_grad():
            logits = model(torch.tensor([seq], device="cuda")).float()[0, -1]
        top2 = torch.topk(logits, 2).values
        if float(top2[0] - top2[1]) <= tol * float(logits.abs().max()):
            skipped += 1
        else:
            assert t == int(torch.argmax(logits)), f"step {i}"
        seq.append(t)
    print(f"greedy 8-bit: {n} steps, {skipped} skipped as near-ties")
    assert skipped < n // 2


def test_cli_kv_bits_end_to_end():
    env = dict(os.environ, PYTHONPATH=str(ROOT) + os.pathsep + os.environ.get("PYTHONPATH", ""))
    with tempfile.TemporaryDirectory(prefix="kvq_e2e_") as tmp:
        cfg = yaml.safe_load((ROOT / "configs" / "c1-llama2m-adamw.yaml").read_text())
        cfg["name"] = "kvq-e2e"
        cfg["data"]["input_file"] = "synthetic:markov"
        cfg["data"]["preprocessing"]["max_context_size"] = 128
        cfg["training"]["hyperparameters"]["iters"] = 3
        cfg["model"]["attention"].update(num_heads=4, num_kv_heads=4, head_dim=32)
        cfg_path = Path(tmp) / "cfg.yaml"
        cfg_path.write_text(yaml.safe_dump(cfg))
        subprocess.run([sys.executable, "-m", "core.training", "--config", str(cfg_path)], cwd=tmp, env=env,
                       check=True, timeout=600)
        out = subprocess.run([sys.executable, "-m", "core.generation", "--run", "kvq-e2e", "--runs-dir",
                              str(Path(tmp) / "runs"), "--prompt", "hello", "--max-tokens", "24", "--seed", "0",
                              "--kv-bits", "4", "--kv-group-size", "32", "--num-samples", "2"],
                             cwd=ROOT, env=env, check=True, capture_output=True, text=True, timeout=600).stdout
        assert sum(l.startswith("Greedy Output: ") for l in out.splitlines()) == 2
