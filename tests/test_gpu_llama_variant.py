"""-m gpu: `model.misc.variant: mlx_lm` on the sm_90a kernels -- the SiLU GEMM epilogues, the unfused SiLU-GLU, the
half-split RoPE and KV append, the variant model against its fp64 oracle (tests/llama_variant_oracle.py), generation,
and a trainer run exported to and reloaded by transformers' LlamaForCausalLM."""
import json
import tempfile

import numpy as np
import pytest
import torch

from tests import gemm_check as gc
from tests import llama_variant_oracle as vo
from tests.gemm_check import Guarded
from tests.test_gpu_packed_attention import _loss_and_grads

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(600)]

BF16 = torch.bfloat16
# rel_sigmoid: ex2.approx and rcp.approx (about 2^-22 relative each) and the rounding of -g log2(e), which adds
# |g| 2^-24 ln 2 (|g| <= 16 here); with the epilogue's few fp32 products, 2^-18 relative covers the activation.
EPS_SILU = 2.0 ** -18


@pytest.fixture(scope="module")
def L():
    from mlx_cuda_distributed_pretraining_b200 import ops
    ops.require_device()
    return ops.lib()


def _stream():
    return torch.cuda.current_stream().cuda_stream


def _ok(rc, L):
    if rc != 0:
        raise AssertionError(f"rc={rc}: {L.b200_last_error().decode()}")


def _g2(rows, cols, fill=None):
    G = Guarded(1, rows, cols, BF16, "cuda", ld=cols, stride=rows * cols, guard=4 * cols)
    if fill is not None:
        G.view().copy_(fill(G.view().shape).to(BF16))
    return G


def _gate_spread(shape, gen):
    """Gate pre-activations from -10 to +10 across columns (plus noise), so the negative tail is exercised."""
    ramp = torch.linspace(-10, 10, shape[-1], device="cuda", dtype=torch.float64)
    return ramp + 0.5 * torch.randn(shape, device="cuda", generator=gen, dtype=torch.float64)


SHAPES = [(300, 1024, 2816), (129, 1024, 4096), (200, 2048, 5632), (1, 256, 256), (4096, 1024, 2816)]


@pytest.mark.parametrize("M,K,I", SHAPES)
def test_gateup_silu_fwd_vs_fp64(L, M, K, I):
    """x = [1, 0, ...] times a scale picks W2's first column, so the gate spans -10..10; the rest is N(0, 1) noise
    at 1/sqrt(K) so the accumulation term is realistic."""
    gen = torch.Generator(device="cuda").manual_seed(M + I)
    x = _g2(M, K, lambda s: torch.randn(s, device="cuda", generator=gen) * 0.05)
    x.view()[..., 0] = 1.0
    W = torch.randn(2 * I, K, device="cuda", generator=gen) * 0.05
    W[:I, 0] = _gate_spread((I,), gen).float()
    W2 = _g2(2 * I, K, lambda s: W)
    gu, y = _g2(M, 2 * I), _g2(M, I)
    what = f"silu gate/up M={M} K={K} I={I}"
    _ok(L.b200_mlp_gateup_silu_fwd(x.ptr(), W2.ptr(), gu.ptr(), y.ptr(), M, K, I, _stream()), L)
    torch.cuda.synchronize()
    gu.check_canaries(2 * I, what + ": gu")
    y.check_canaries(I, what + ": y")
    R, P = gc.reference(x.view(), W2.view())
    gc.check_bound(gu.view(), R, P, K, what + ": gu")
    g, u, Pg, Pu = R[..., :I], R[..., I:], P[..., :I], P[..., I:]
    s = torch.sigmoid(g)
    Ry = g * s * u
    # the fp32 accumulators' error propagates through dy/dg = u s (1 + g (1 - s)) and dy/du = silu(g)
    Py = Pg * (u.abs() * s * (1 + g.abs() * (1 - s))) + Pu * (g * s).abs()
    b = gc.check_bound(y.view(), Ry, Py, K, what + ": y", extra=Ry.abs() * EPS_SILU)
    assert float(g.min()) < -9 and float(g.max()) > 9
    print(f"{what}: y worst ratio {b.ratio:.3f}")


@pytest.mark.parametrize("M,H,I", [(300, 1024, 2816), (129, 1024, 4096), (200, 2048, 5632), (1, 256, 136),
                                   (4096, 1024, 2816)])
def test_down_silu_bwd_vs_fp64(L, M, H, I):
    gen = torch.Generator(device="cuda").manual_seed(M + H + I)
    dy = _g2(M, H, lambda s: torch.randn(s, device="cuda", generator=gen))
    Wd = _g2(H, I, lambda s: torch.randn(s, device="cuda", generator=gen) * H ** -0.5)
    half = (1, M, I)
    gu = _g2(M, 2 * I, lambda s: torch.cat([_gate_spread(half, gen).float(),
                                            2 * torch.randn(half, device="cuda", generator=gen)], -1))
    dgu = _g2(M, 2 * I)
    what = f"silu down dgrad M={M} H={H} I={I}"
    _ok(L.b200_mlp_down_silu_bwd(dy.ptr(), Wd.ptr(), gu.ptr(), dgu.ptr(), M, H, I, _stream()), L)
    torch.cuda.synchronize()
    dgu.check_canaries(2 * I, what)
    R, P = gc.reference(dy.view(), Wd.view(), b_mn=True)
    g, u = gu.view()[..., :I].double(), gu.view()[..., I:].double()
    s = torch.sigmoid(g)
    fg = u * s * (1 + g * (1 - s))
    fabs = u.abs() * s * (1 + g.abs() * (1 - s))
    Rd = torch.cat([R * fg, R * g * s], -1)
    Pd = torch.cat([P * fabs, P * (g * s).abs()], -1)
    extra = torch.cat([R.abs() * fabs, R.abs() * (g * s).abs()], -1) * EPS_SILU
    b = gc.check_bound(dgu.view(), Rd, Pd, H, what, extra=extra)
    print(f"{what}: worst ratio {b.ratio:.3f}")


def test_silu_glu_elementwise_vs_fp64(L):
    from mlx_cuda_distributed_pretraining_b200 import ops
    gen = torch.Generator(device="cuda").manual_seed(7)
    n = 8 * 4099
    g = _gate_spread((n,), gen).to(BF16)
    u = (2 * torch.randn(n, device="cuda", generator=gen)).to(BF16)
    gd, ud = g.double().requires_grad_(True), u.double().requires_grad_(True)
    yr = torch.nn.functional.silu(gd) * ud
    gk, uk = g.clone().requires_grad_(True), u.clone().requires_grad_(True)
    y = ops.glu(gk, uk, "silu")
    dy = torch.randn(n, device="cuda", generator=gen).to(BF16)
    y.backward(dy)
    yr.backward(dy.double())
    gx, ux, dx = g.double(), u.double(), dy.double()
    s_ = torch.sigmoid(gx)
    scale = {"y": (gx * s_ * ux).abs(), "dg": dx.abs() * ux.abs() * s_ * (1 + gx.abs() * (1 - s_)),
             "du": (dx * gx * s_).abs()}
    for got, want, nm in ((y, yr, "y"), (gk.grad, gd.grad, "dg"), (uk.grad, ud.grad, "du")):
        want = want.detach()
        err = (got.double() - want).abs()
        bound = 2.0 ** -8 * want.abs() + EPS_SILU * scale[nm]
        ratio = torch.where(err == 0, torch.zeros_like(err), err / bound)
        assert float(ratio.max()) <= 1.0, (nm, float(ratio.max()))


def _rope_ref(x, pos, backward):
    y = vo.rope_half(x.double().cpu(), 10000.0, pos.cpu() if pos is not None else None)
    if backward:  # the inverse rotation: rotate by -angle
        B, S, NH, D = x.shape
        p = torch.arange(S, dtype=torch.float64) if pos is None else pos.cpu().double()
        freqs = 10000.0 ** (-torch.arange(0, D, 2, dtype=torch.float64) / D)
        ang = p[..., None] * freqs
        ang = ang[None, :, None] if ang.dim() == 2 else ang[:, :, None]
        x0, x1 = x.double().cpu()[..., :D // 2], x.double().cpu()[..., D // 2:]
        y = torch.cat([x0 * ang.cos() + x1 * ang.sin(), -x0 * ang.sin() + x1 * ang.cos()], -1)
    return y


@pytest.mark.parametrize("dtype", [BF16, torch.float32], ids=["bf16", "fp32"])
@pytest.mark.parametrize("D", [16, 64, 128])
@pytest.mark.parametrize("packed", [False, True])
def test_rope_half_vs_fp64_and_adjoint(L, dtype, D, packed):
    from mlx_cuda_distributed_pretraining_b200 import ops
    B, S, NH = 2, 300, 3
    gen = torch.Generator(device="cuda").manual_seed(D)
    x = torch.randn(B, S, NH, D, device="cuda", generator=gen).to(dtype)
    pos = None
    if packed:
        pos = torch.stack([torch.cat([torch.arange(n) for n in lens]) for lens in ([S], [5, 100, S - 105])]).int().cuda()
    cos_t, sin_t = ops.rope_tables(S, D, 10000.0, "cuda")
    xr = x.clone().requires_grad_(True)
    y = ops.rope(xr, cos_t, sin_t, pos, layout="half")
    dy = torch.randn_like(x)
    y.backward(dy)
    # bf16: output rounding.  fp32: the tables' angles pos * theta^(-2i/D) are rounded to fp32, up to S 2^-24 absolute
    tol = 2.0 ** -7 if dtype == BF16 else 4 * S * 2.0 ** -24
    for got, want in ((y, _rope_ref(x, pos, False)), (xr.grad, _rope_ref(dy, pos, True))):
        err = float((got.double().cpu() - want).abs().max() / want.abs().max())
        assert err < tol, err
    if dtype == torch.float32:  # the backward is the adjoint: <rope(x), dy> = <x, rope_bwd(dy)>
        lhs = float((y.double() * dy.double()).sum())
        rhs = float((x.double() * xr.grad.double()).sum())
        assert abs(lhs - rhs) < 1e-4 * (abs(lhs) + 1)


@pytest.mark.parametrize("dtype", [BF16, torch.float32], ids=["bf16", "fp32"])
@pytest.mark.parametrize("D", [16, 64, 128])
def test_kv_append_half_bit_equal_to_rope(L, dtype, D):
    from mlx_cuda_distributed_pretraining_b200 import ops
    B, H, Hk, s_max = 3, 4, 2, 256
    gen = torch.Generator(device="cuda").manual_seed(D + 1)
    q = torch.randn(B, H, D, device="cuda", generator=gen).to(dtype)
    k = torch.randn(B, Hk, D, device="cuda", generator=gen).to(dtype)
    v = torch.randn(B, Hk, D, device="cuda", generator=gen).to(dtype)
    kc = torch.zeros(B, s_max, Hk, D, device="cuda", dtype=dtype)
    vc = torch.zeros_like(kc)
    lens = torch.tensor([1, 77, 256], device="cuda", dtype=torch.int32)
    tabs = ops.rope_tables(s_max, D, 10000.0, "cuda")
    qa = q.clone()
    ops.kv_append(qa, k, v, kc, vc, lens, tabs, layout="half")
    for b, n in enumerate([1, 77, 256]):
        p = torch.tensor([[n - 1]], device="cuda", dtype=torch.int32)
        assert torch.equal(qa[b], ops.rope(q[b][None, None], *tabs, p, layout="half")[0, 0])
        assert torch.equal(kc[b, n - 1], ops.rope(k[b][None, None], *tabs, p, layout="half")[0, 0])
        assert torch.equal(vc[b, n - 1], v[b])


# ---- model level ------------------------------------------------------------------------------------------------
def _model(dtype, hidden, layers, heads, kv_heads, head_dim, window=None, tied=True, vocab=259):
    from mlx_cuda_distributed_pretraining_b200.arch.llama import Model, ModelArgs
    from mlx_cuda_distributed_pretraining_b200.core.training import init_model_
    args = ModelArgs(model_type="llama", hidden_size=hidden, num_hidden_layers=layers, intermediate_size=2 * hidden,
                     num_attention_heads=heads, num_key_value_heads=kv_heads, head_dim=head_dim, vocab_size=vocab,
                     tie_word_embeddings=tied, sliding_window=window, variant="mlx_lm")
    m = Model(args)
    init_model_(m, args, seed=3)
    return m.to("cuda", dtype)


def _dims(m):
    from oracle import reference_math as rm
    a = m.args
    return rm.LlamaDims(hidden_size=a.hidden_size, intermediate_size=a.intermediate_size,
                        num_layers=a.num_hidden_layers, num_heads=a.num_attention_heads,
                        num_kv_heads=a.num_key_value_heads, head_dim=a.head_dim, vocab_size=a.vocab_size,
                        rms_norm_eps=a.rms_norm_eps, rope_theta=a.rope_theta, use_rope=True,
                        tie_word_embeddings=a.tie_word_embeddings)


def _rel(a, b):
    a, b = a.double().cpu(), b.double().cpu()
    return float((a - b).norm() / b.norm().clamp_min(1e-30))


KINDS = {"bf16_gqa": (BF16, 256, 2, 8, 2, 64, 5e-3, 3e-2), "c1_fp32": (torch.float32, 128, 4, 8, 8, 16, 1e-3, 8e-3)}


@pytest.mark.parametrize("kind", list(KINDS))
@pytest.mark.parametrize("window", [None, 40])
def test_variant_model_matches_fp64_oracle(L, kind, window):
    from mlx_cuda_distributed_pretraining_b200.arch.flash_attention import CausalMask
    dtype, hid, layers, heads, kvh, hd, tol_loss, tol_grad = KINDS[kind]
    model = _model(dtype, hid, layers, heads, kvh, hd, window, tied=kind == "c1_fp32")
    toks = torch.randint(0, 256, (2, 201), generator=torch.Generator().manual_seed(4))
    loss_k, g_k = _loss_and_grads(model, toks[:, :-1].cuda(), toks[:, 1:].cuda(), None)
    params = {n: p.detach().double().cpu() for n, p in model.named_parameters()}
    mask = CausalMask(200, window).dense(torch.float64)
    loss_r, ntoks, g_r = vo.loss_and_grads(params, toks, _dims(model), 256, mask=mask)
    loss_r, g_r = loss_r * ntoks, {n: g * ntoks for n, g in g_r.items()}   # _loss_and_grads sums over tokens
    worst = max(_rel(g_k[n], g_r[n]) for n in g_r)
    print(f"{kind} window={window}: loss kernel {loss_k:.6f} fp64 {float(loss_r):.6f}, worst grad rel {worst:.2e}")
    assert abs(loss_k - float(loss_r)) < tol_loss * abs(float(loss_r))
    assert worst < tol_grad


@pytest.mark.parametrize("kind", list(KINDS))
def test_packed_variant_rows_match_documents_alone(L, kind):
    from mlx_cuda_distributed_pretraining_b200.core.training import document_positions, pack_first_fit
    dtype, hid, layers, heads, kvh, hd, tol_loss, tol_grad = KINDS[kind]
    model = _model(dtype, hid, layers, heads, kvh, hd)
    PAD, BOS_ID, EOS, Lr = 256, 257, 258, 257
    rng = np.random.default_rng(12)
    docs = [[BOS_ID] + rng.integers(0, 256, int(n)).tolist() + [EOS]
            for n in np.clip(rng.lognormal(3.5, 1.0, 16), 1, Lr - 2).astype(int)]
    rows = pack_first_fit([len(d) for d in docs], Lr)
    packed = torch.full((len(rows), Lr), PAD, dtype=torch.int64)
    for r, row in enumerate(rows):
        t = [x for i in row for x in docs[i]]
        packed[r, :len(t)] = torch.tensor(t)
    packed = packed.cuda()
    inputs, targets = packed[:, :-1], packed[:, 1:]
    pos = document_positions(inputs, BOS_ID)
    targets = targets.masked_fill(targets == BOS_ID, PAD)
    alone = torch.full((len(docs), max(len(d) for d in docs)), PAD, dtype=torch.int64)
    for i, d in enumerate(docs):
        alone[i, :len(d)] = torch.tensor(d)
    alone = alone.cuda()
    loss_p, g_p = _loss_and_grads(model, inputs, targets, pos)
    loss_a, g_a = _loss_and_grads(model, alone[:, :-1], alone[:, 1:], None)
    worst = max(_rel(g_p[n], g_a[n]) for n in g_a)
    print(f"{kind}: loss packed {loss_p:.6f} alone {loss_a:.6f}, worst grad rel {worst:.2e}")
    assert abs(loss_p - loss_a) < tol_loss * abs(loss_a)
    assert worst < tol_grad


def _variant_cfg(kind):
    from tests.test_gpu_generation import _cfg
    c = _cfg(kind)
    c["model"]["misc"]["variant"] = "mlx_lm"
    c["model"]["rope"].pop("enabled", None)
    return c


@pytest.mark.parametrize("kind", ["bf16_gqa", "c1_fp32"])
def test_prefill_decode_match_forward_under_variant(kind):
    from mlx_cuda_distributed_pretraining_b200.arch.llama import KVCache
    from mlx_cuda_distributed_pretraining_b200.core.generation import generate
    from mlx_cuda_distributed_pretraining_b200.core.training import Config, Trainer
    from tests.test_gpu_generation import TOL, _rel_rows
    tr = Trainer(Config.from_dict(_variant_cfg(kind)), for_training=False, synthetic=True, quiet=True,
                 run_root=tempfile.mkdtemp(prefix="variant_runs_"))
    model = tr.model
    assert model.args.variant == "mlx_lm" and model.layers[0].self_attn.rope_layout == "half"
    T, t0 = 200, 150
    tokens = torch.randint(0, 256, (2, T), generator=torch.Generator().manual_seed(5))
    with torch.no_grad():
        full = model(tokens.cuda()).float()
    cache = KVCache(model, 2, T)
    got = [model.prefill(tokens[:, :t0].cuda(), [t0, t0], cache)]
    for t in range(t0, T - 1):
        got.append(model.decode_step(tokens[:, t].cuda(), cache))
    e = _rel_rows(torch.stack(got, dim=1), full[:, t0 - 1:T - 1])
    print(f"{kind}: cached vs forward {e:.2e}")
    assert e < TOL["c1_fp32" if kind == "c1_fp32" else "bf16_rope"]
    out = generate(model, [tokens[0, :t0].tolist()], max_tokens=12, temperature=0)[0]
    assert len(out) == 12


def test_variant_trainer_run_generates_and_exports(tmp_path):
    """Short synthetic bf16 run with the variant -> core.generation rebuilds it -> tools/convert-to-mlx-lm.py exports
    it -> transformers (CPU, fp32) reproduces Model.forward's logits from the export."""
    transformers = pytest.importorskip("transformers")
    import os
    import subprocess
    import sys
    import yaml
    from pathlib import Path
    from mlx_cuda_distributed_pretraining_b200.core.generation import generate, load_run
    from mlx_cuda_distributed_pretraining_b200.core.training import Config, Trainer
    from tests.smoke_check import tiny_config
    cfg = tiny_config(name="variant", hp__iters=6)
    cfg["model"]["misc"]["variant"] = "mlx_lm"
    cfg["model"]["rope"].pop("enabled", None)
    cfg["logging"]["steps"]["checkpoint_interval"] = 0
    tr = Trainer(Config.from_dict(cfg), quiet=True, run_root=str(tmp_path))
    assert tr.model.args.variant == "mlx_lm"
    tr.train()
    run = tmp_path / "variant"
    assert yaml.safe_load((run / "config.yaml").read_text())["model"]["misc"]["variant"] == "mlx_lm"
    loaded = load_run("variant", str(tmp_path))
    assert loaded.model.args.variant == "mlx_lm" and loaded.model.layers[0].mlp.act == "silu"
    out = generate(loaded.model, [[loaded.tokenizer.BOS_TOKEN] + list(range(40, 100))], max_tokens=6, temperature=0)
    assert len(out[0]) == 6
    root = Path(__file__).resolve().parents[1]
    r = subprocess.run([sys.executable, str(root / "tools" / "convert-to-mlx-lm.py"), "--run", "variant",
                        "--out-path", str(tmp_path / "hf"), "--runs-dir", str(tmp_path)],
                       capture_output=True, text=True, env=dict(os.environ, HF_HUB_OFFLINE="1"))
    assert r.returncode == 0, r.stderr
    assert json.loads((tmp_path / "hf" / "config.json").read_text())["hidden_act"] == "silu"
    toks = torch.randint(0, 256, (2, 64), generator=torch.Generator().manual_seed(9))
    with torch.no_grad():
        ours = loaded.model(toks.cuda()).float().cpu()
        hf = transformers.LlamaForCausalLM.from_pretrained(str(tmp_path / "hf")).eval()
        theirs = hf(toks).logits.float()
    e = float((ours - theirs).abs().max() / theirs.abs().max())
    print(f"export: Model.forward vs transformers fp32 logits, max error / max |logit| = {e:.2e}")
    # the run's activations are bf16 (Model.forward) against transformers' fp32: bf16 rounding through the layers
    assert e < 3e-2
