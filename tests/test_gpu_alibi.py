"""-m gpu: ALiBi attention (`model.attention.alibi`, b200_attn_{fwd,bwd,decode}_alibi): the score of query q and key k
gets the bias m_h (k - q) of query head h's slope before the mask and the softmax.

The fp64 reference and the tolerances are those of tests/test_gpu_sliding_window.py: o / dq / dk / dv relative
Frobenius error < 1e-2, lse max abs error < 1e-3; model level bf16 loss 5e-3 / gradients 3e-2, fp32 (bf16x3
attention) 1e-3 / 8e-3; decode the bound of tests/test_gpu_generation.py."""
import tempfile
from pathlib import Path

import numpy as np
import pytest
import torch

from tests.test_gpu_generation import C_BOUND
from tests.test_gpu_packed_attention import _loss_and_grads, layouts, positions
from tests.test_gpu_sliding_window import _inputs, dense_mask, reference, rel

pytestmark = pytest.mark.gpu

ROOT = Path(__file__).resolve().parents[1]


@pytest.fixture(scope="module")
def ops():
    from mlx_cuda_distributed_pretraining_b200 import ops as o
    o.require_device()
    return o


def std_slopes(H):
    from mlx_cuda_distributed_pretraining_b200.arch.flash_attention import alibi_slopes
    return alibi_slopes(H).cuda()


def mixed_slopes(H):
    """0 (no bias), 1/256 (a gentle one) and 0.5 (the steepest standard slope), cycled over the heads."""
    return torch.tensor([(0.0, 1 / 256, 0.5)[h % 3] for h in range(H)], dtype=torch.float32, device="cuda")


def bias(slopes, S, device="cuda"):
    """fp64 [1, H, S, S] ALiBi bias m_h (k - q)."""
    s = torch.arange(S, device=device, dtype=torch.float64)
    return (slopes.double().to(device)[:, None, None] * (s[None, :] - s[:, None]))[None]


def _pos(packed, S, seed, rows=None):
    if not packed:
        return None
    ls = layouts(S, seed=seed)
    return torch.stack([positions(l, S) for l in (ls if rows is None else ls[:rows])]).int().cuda()


def _check(ops, q, k, v, do, pos, W, slopes, fp32=False):
    S, D = q.shape[1], q.shape[-1]
    q.grad = k.grad = v.grad = None
    f = ops.attention_fp32 if fp32 else ops.attention
    o = f(q, k, v, D ** -0.5, pos=pos, window=W, alibi=slopes)
    o.backward(do)
    o_r, lse_r, dq_r, dk_r, dv_r = reference(q, k, v, do, dense_mask(pos, W, S, "cuda") + bias(slopes, S), D ** -0.5)
    for b in range(q.shape[0]):
        errs = (rel(o[b], o_r[b]), rel(q.grad[b], dq_r[b]), rel(k.grad[b], dk_r[b]), rel(v.grad[b], dv_r[b]))
        assert max(errs) < 1e-2, (W, b, errs)
    if not fp32:
        _, lse = ops.attention_fwd_raw(q.detach(), k.detach(), v.detach(), D ** -0.5, True, pos, W, slopes)
        assert float((lse.double() - lse_r.detach()).abs().max()) < 1e-3, W
    assert torch.isfinite(o).all() and torch.isfinite(q.grad).all() and torch.isfinite(k.grad).all(), W


# ---- kernels against fp64 -------------------------------------------------------------------------------------------
@pytest.mark.parametrize("layout", ["rows", "packed", "window", "packed_window"])
@pytest.mark.parametrize("S,H,Hk,D", [(1000, 16, 8, 64), (2048, 2, 1, 64), (1000, 2, 1, 128), (1024, 4, 4, 128)])
def test_alibi_attention_vs_fp64(ops, S, H, Hk, D, layout):
    """Standard and mixed (0, 1/256, 0.5) slopes; unpacked rows, the packed layouts of the document tests, and
    windows of several widths, alone and intersected with the documents."""
    pos = _pos("packed" in layout, S, seed=D)
    B = pos.shape[0] if pos is not None else 2
    q, k, v, do = _inputs(B, S, H, Hk, D, torch.bfloat16, S + D + H)
    Ws = (0, 1, 127, 129, 300) if "window" in layout else (None,)
    for slopes in (std_slopes(H), mixed_slopes(H)):
        for W in Ws:
            _check(ops, q, k, v, do, pos, W, slopes)


@pytest.mark.parametrize("layout", ["rows", "packed", "window"])
def test_alibi_attention_fp32_path(ops, layout):
    """attention_fp32 (bf16x3, C1's head dim 16) with ALiBi."""
    S, H, Hk, D = 1000, 8, 8, 16
    pos = _pos(layout == "packed", S, seed=3, rows=3)
    B = 3 if pos is not None else 2
    q, k, v, do = _inputs(B, S, H, Hk, D, torch.float32, 7)
    for slopes in (std_slopes(H), mixed_slopes(H)):
        _check(ops, q, k, v, do, pos, 129 if layout == "window" else None, slopes, fp32=True)


def test_long_row_steep_and_gentle_slopes(ops):
    """S = 8192.  Slope 0.5: every key more than a few hundred positions back underflows to an exact 0 in the
    softmax, and nothing turns into NaN.  Slope 1/256: keys thousands of positions back still carry weight, so
    the output differs from the same slope cut to a 512-key window."""
    S, H, Hk, D = 8192, 2, 1, 64
    q, k, v, do = _inputs(1, S, H, Hk, D, torch.bfloat16, 11)
    steep = torch.full((H,), 0.5, device="cuda")
    _check(ops, q, k, v, do, None, None, steep)
    # the bias reaches -0.5 * 8191: far keys give exp(...) == 0 exactly, so a covering window changes nothing in o
    o_full, _ = ops.attention_fwd_raw(q.detach(), k.detach(), v.detach(), D ** -0.5, True, None, None, steep)
    o_win, _ = ops.attention_fwd_raw(q.detach(), k.detach(), v.detach(), D ** -0.5, True, None, 1024, steep)
    assert torch.isfinite(o_full).all()
    assert rel(o_full, o_win) < 1e-6
    gentle = torch.full((H,), 1 / 256, device="cuda")
    _check(ops, q, k, v, do, None, None, gentle)
    o_g, _ = ops.attention_fwd_raw(q.detach(), k.detach(), v.detach(), D ** -0.5, True, None, None, gentle)
    o_g512, _ = ops.attention_fwd_raw(q.detach(), k.detach(), v.detach(), D ** -0.5, True, None, 512, gentle)
    assert rel(o_g[:, 4096:], o_g512[:, 4096:]) > 5e-2


@pytest.mark.parametrize("layout", ["rows", "packed", "window", "packed_window"])
@pytest.mark.parametrize("S,H,Hk,D", [(1024, 16, 8, 64), (1000, 4, 2, 128)])
def test_zero_slopes_match_window_doc_and_causal_bit_for_bit(ops, S, H, Hk, D, layout):
    """All-zero slopes: the ALiBi entries give b200_attn_fwd / _doc / _window's o and lse, and the backward's dk and
    dv, bit for bit (dq by tolerance: its fp32 reduction order is not reproducible)."""
    pos = _pos("packed" in layout, S, seed=1, rows=3)
    B = 3 if pos is not None else 2
    W = 200 if "window" in layout else None
    q, k, v, do = (t.detach() for t in _inputs(B, S, H, Hk, D, torch.bfloat16, 5))
    zero = torch.zeros(H, device="cuda")
    o_c, lse_c = ops.attention_fwd_raw(q, k, v, D ** -0.5, True, pos, W)
    dq_c, dk_c, dv_c = ops.attention_bwd_raw(q, k, v, o_c, do, lse_c, D ** -0.5, True, pos, W)
    o_a, lse_a = ops.attention_fwd_raw(q, k, v, D ** -0.5, True, pos, W, zero)
    assert torch.equal(o_c, o_a) and torch.equal(lse_c, lse_a)
    dq_a, dk_a, dv_a = ops.attention_bwd_raw(q, k, v, o_c, do, lse_c, D ** -0.5, True, pos, W, zero)
    assert torch.equal(dk_c, dk_a) and torch.equal(dv_c, dv_a)
    assert rel(dq_a, dq_c) < 1e-3


def test_bad_alibi_is_rejected(ops):
    q = torch.zeros(1, 64, 2, 64, device="cuda", dtype=torch.bfloat16)
    good = torch.zeros(2, device="cuda")
    with pytest.raises(ValueError, match="causal"):
        ops.attention(q, q, q, causal=False, alibi=good)
    for bad in (torch.zeros(2, device="cuda", dtype=torch.float64), torch.zeros(3, device="cuda"),
                torch.zeros(2), torch.zeros(4, device="cuda")[::2], [0.0, 0.0]):
        with pytest.raises(ValueError):
            ops.attention(q, q, q, alibi=bad)
        with pytest.raises(ValueError):
            ops.attention_decode(q[:, 0].contiguous(), q, q, torch.ones(1, device="cuda", dtype=torch.int32),
                                 alibi=bad)
    from mlx_cuda_distributed_pretraining_b200._lib import B200Error
    L = ops.lib()
    with pytest.raises(B200Error):  # null slopes
        ops.check(L.b200_attn_fwd_alibi(q.data_ptr(), q.data_ptr(), q.data_ptr(), q.data_ptr(), good.data_ptr(), None,
                                        -1, None, 1, 64, 2, 2, 64, 0.125, None), "b200_attn_fwd_alibi")


# ---- decode ---------------------------------------------------------------------------------------------------------
DEC_LENS = [1, 255, 256, 257, 1000, 4095]
DEC_SMAX = 4160


def _cache(lens, H, Hk, D, dtype, seed):
    """Positions at or past lens hold NaN: a read past a row's length would show."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    B = len(lens)
    q = torch.randn(B, H, D, device="cuda", generator=g).to(dtype)
    kc = torch.randn(B, DEC_SMAX, Hk, D, device="cuda", generator=g).to(dtype)
    vc = torch.randn(B, DEC_SMAX, Hk, D, device="cuda", generator=g).to(dtype)
    for b, n in enumerate(lens):
        kc[b, n:] = float("nan")
        vc[b, n:] = float("nan")
    return q, kc, vc, torch.tensor(lens, device="cuda", dtype=torch.int32)


def _decode_reference(q, kc, vc, lens, W, slopes, scale):
    H, Hk = q.shape[1], kc.shape[2]
    out, absterm = [], []
    for b, n in enumerate(lens):
        kv0 = 0 if W is None else max(0, n - 1 - W)
        k, v = (t[b, kv0:n].double().repeat_interleave(H // Hk, dim=1) for t in (kc, vc))
        dist = torch.arange(kv0, n, device="cuda", dtype=torch.float64) - (n - 1)
        s = torch.einsum("hd,nhd->hn", q[b].double(), k) * scale + slopes.double()[:, None] * dist[None]
        p = torch.softmax(s, dim=-1)
        out.append(torch.einsum("hn,nhd->hd", p, v))
        absterm.append(torch.einsum("hn,nhd->hd", p, v.abs()))
    return torch.stack(out), torch.stack(absterm)


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float32], ids=["bf16", "fp32"])
@pytest.mark.parametrize("D", [16, 32, 64, 128])
def test_decode_alibi_matches_fp64(ops, dtype, D):
    H, Hk, scale = 6, 2, D ** -0.5
    for slopes in (std_slopes(H), mixed_slopes(H)):
        for W in (None, 100, 300):
            q, kc, vc, lens = _cache(DEC_LENS, H, Hk, D, dtype, seed=D + (W or 0))
            o = ops.attention_decode(q, kc, vc, lens, scale, window=W, alibi=slopes)
            R, absterm = _decode_reference(q, kc, vc, DEC_LENS, W, slopes, scale)
            bound = C_BOUND * 2.0 ** -24 * absterm + (2.0 ** -8 * R.abs() if dtype == torch.bfloat16 else 0)
            assert torch.isfinite(o).all(), W
            assert float(((o.double() - R).abs() / bound).max()) <= 1.0, (W, float(((o.double() - R).abs() / bound).max()))


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float32], ids=["bf16", "fp32"])
def test_decode_alibi_batch_invariant_and_zero_slopes(ops, dtype):
    """Each row alone is bit-identical to the same row in the batch; zero slopes give b200_attn_decode's and
    b200_attn_decode_window's bits."""
    H, Hk, D = 16, 8, 64
    lens = [2048, 5, 257, 1000, 4095, 256, 31, 301]
    q, kc, vc, lt = _cache(lens, H, Hk, D, dtype, seed=3)
    for W in (None, 300):
        o = ops.attention_decode(q, kc, vc, lt, window=W, alibi=std_slopes(H))
        assert torch.equal(o, ops.attention_decode(q, kc, vc, lt, window=W, alibi=std_slopes(H)))
        for b in range(len(lens)):
            alone = ops.attention_decode(q[b:b + 1].contiguous(), kc[b:b + 1].contiguous(), vc[b:b + 1].contiguous(),
                                         lt[b:b + 1].contiguous(), window=W, alibi=std_slopes(H))
            assert torch.equal(alone[0], o[b]), (W, b)
        zero = torch.zeros(H, device="cuda")
        o0, lse0 = ops.attention_decode(q, kc, vc, lt, window=W, alibi=zero, return_lse=True)
        oc, lsec = ops.attention_decode(q, kc, vc, lt, window=W, return_lse=True)
        assert torch.equal(o0, oc) and torch.equal(lse0, lsec), W


# ---- model level ----------------------------------------------------------------------------------------------------
def _model(dtype, rope, hidden, layers, heads, kv_heads, head_dim, vocab=259, window=None):
    from mlx_cuda_distributed_pretraining_b200.arch.llama import Model, ModelArgs
    from mlx_cuda_distributed_pretraining_b200.core.training import init_model_
    args = ModelArgs(model_type="llama", hidden_size=hidden, num_hidden_layers=layers, intermediate_size=2 * hidden,
                     num_attention_heads=heads, num_key_value_heads=kv_heads, head_dim=head_dim, vocab_size=vocab,
                     tie_word_embeddings=True, apply_rope=rope, sliding_window=window, alibi=True)
    m = Model(args)
    init_model_(m, args, seed=3)
    return m.to("cuda", dtype)


def _dense_alibi_attention(self, q, k, v, mask=None):
    """FlashAttention._flash_attention replaced by fp64 softmax(q k^T scale + mask.dense() + bias) v."""
    H, Hk, S = q.shape[2], k.shape[2], q.shape[1]
    kx, vx = (t.double().repeat_interleave(H // Hk, dim=2) for t in (k, v))
    s = torch.einsum("bqhd,bkhd->bhqk", q.double(), kx) * self.scale + mask.dense(torch.float64, q.device)
    s = s + bias(self.alibi_slopes(q.device), S, q.device)
    return torch.einsum("bhqk,bkhd->bqhd", torch.softmax(s, dim=-1), vx).to(q.dtype)


@pytest.mark.parametrize("kind,rope", [("bf16_gqa", False), ("bf16_gqa", True), ("c1_fp32", False)])
def test_alibi_model_matches_dense_reference(ops, monkeypatch, kind, rope):
    from mlx_cuda_distributed_pretraining_b200.arch.flash_attention import FlashAttention
    if kind == "bf16_gqa":
        model, tol_loss, tol_grad = _model(torch.bfloat16, rope, 256, 2, 8, 2, 64), 5e-3, 3e-2
    else:
        model, tol_loss, tol_grad = _model(torch.float32, rope, 128, 4, 8, 8, 16), 1e-3, 8e-3
    g = torch.Generator().manual_seed(4)
    toks = torch.randint(0, 256, (2, 301), generator=g).cuda()
    inputs, targets = toks[:, :-1], toks[:, 1:]
    loss_k, g_k = _loss_and_grads(model, inputs, targets, None)
    monkeypatch.setattr(FlashAttention, "_flash_attention", _dense_alibi_attention)
    loss_r, g_r = _loss_and_grads(model, inputs, targets, None)
    worst = max(rel(g_k[n], g_r[n]) for n in g_r)
    print(f"{kind} rope={rope}: loss kernel {loss_k:.6f} dense {loss_r:.6f}, worst grad rel {worst:.2e}")
    assert abs(loss_k - loss_r) < tol_loss * abs(loss_r)
    assert worst < tol_grad


@pytest.mark.parametrize("kind", ["bf16_gqa", "c1_fp32"])
def test_packed_alibi_rows_match_documents_alone(ops, kind):
    from mlx_cuda_distributed_pretraining_b200.core.training import document_positions, pack_first_fit
    if kind == "bf16_gqa":
        model, tol_loss, tol_grad = _model(torch.bfloat16, False, 256, 2, 8, 2, 64), 5e-3, 3e-2
    else:
        model, tol_loss, tol_grad = _model(torch.float32, False, 128, 4, 8, 8, 16), 1e-3, 8e-3
    PAD, BOS_ID, EOS, L = 256, 257, 258, 385
    rng = np.random.default_rng(12)
    docs = [[BOS_ID] + rng.integers(0, 256, int(n)).tolist() + [EOS]
            for n in np.clip(rng.lognormal(4.0, 1.0, 24), 1, L - 2).astype(int)]
    rows = pack_first_fit([len(d) for d in docs], L)
    packed = torch.full((len(rows), L), PAD, dtype=torch.int64)
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
    worst = max(rel(g_p[n], g_a[n]) for n in g_a)
    print(f"{kind}: loss packed {loss_p:.6f} alone {loss_a:.6f}, worst grad rel {worst:.2e}")
    assert abs(loss_p - loss_a) < tol_loss * abs(loss_a)
    assert worst < tol_grad


def _alibi_trainer(kind, max_pos):
    from mlx_cuda_distributed_pretraining_b200.core.training import Config, Trainer
    from tests.test_gpu_generation import _cfg
    c = _cfg(kind)
    c["model"]["attention"].update(alibi=True, max_position_embeddings=max_pos)
    return Trainer(Config.from_dict(c), for_training=False, synthetic=True, quiet=True,
                   run_root=tempfile.mkdtemp(prefix="alibi_runs_"))


@pytest.mark.parametrize("kind", ["bf16_gqa", "c1_fp32", "bf16_rope"])
def test_prefill_decode_match_forward_past_max_positions(kind):
    """A 200-token prompt and 99 decode steps against Model.forward (the tolerances of tests/test_gpu_generation.py).
    Without RoPE, max_position_embeddings is 256, so the last 44 steps run past it; generate() goes there too.  With
    RoPE the limit stays."""
    from mlx_cuda_distributed_pretraining_b200.arch.llama import KVCache
    from mlx_cuda_distributed_pretraining_b200.core.generation import generate
    from tests.test_gpu_generation import TOL, _rel_rows
    rope = kind == "bf16_rope"
    tr = _alibi_trainer(kind, 512 if rope else 256)
    model = tr.model
    assert model.args.alibi and model.args.apply_rope == rope
    T, t0 = 300, 200
    tokens = torch.randint(0, 256, (2, T), generator=torch.Generator().manual_seed(5))
    with torch.no_grad():
        full = model(tokens.cuda()).float()
    cache = KVCache(model, 2, T)
    got = [model.prefill(tokens[:, :t0].cuda(), [t0, t0], cache)]
    for t in range(t0, T - 1):
        got.append(model.decode_step(tokens[:, t].cuda(), cache))
    e = _rel_rows(torch.stack(got, dim=1), full[:, t0 - 1:T - 1])
    print(f"{kind}: cached vs forward {e:.2e}")
    assert e < TOL[kind]
    prompt = tokens[0, :t0].tolist()
    if rope:
        with pytest.raises(ValueError, match="max_position_embeddings"):
            generate(model, [prompt], max_tokens=400, temperature=0)
    else:
        out = generate(model, [prompt], max_tokens=99, temperature=0, repetition_penalty=1.0, min_p=None)[0]
        assert len(out) == 99


# ---- trainer --------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kind", ["c1_fp32", "bf16"])
def test_alibi_trainer_run_reloads_for_generation(tmp_path, kind):
    """C1 on its control stream (fp32, the bf16x3 attention path) and a bf16 run: the loss stays finite and falls,
    the run's config.yaml carries the key, and the model reloaded through the generation path gives the in-memory
    model's logits."""
    import yaml
    from mlx_cuda_distributed_pretraining_b200.core.generation import load_run
    from mlx_cuda_distributed_pretraining_b200.core.training import Config, Trainer
    from tests.smoke_check import tiny_config
    if kind == "c1_fp32":
        d = yaml.safe_load((ROOT / "configs" / "c1-llama2m-adamw.yaml").read_text())
        d["data"]["input_file"] = "synthetic:markov"
        d["training"]["hyperparameters"].update(iters=40, learning_rate=1e-3)
    else:
        d = tiny_config(hp__iters=40)
    d["name"] = "alibi"
    d["model"]["attention"]["alibi"] = True
    d["logging"]["steps"] = {"logging_interval": 1, "checkpoint_interval": 0, "validation_interval": 0}
    tr = Trainer(Config.from_dict(d), synthetic=True, quiet=True, run_root=str(tmp_path))
    assert tr.model.args.alibi
    tr.train()
    run = tmp_path / "alibi"
    losses = [float(line.split("loss=")[1].split()[0].rstrip("|"))
              for line in (run / "log.txt").read_text().splitlines() if "loss=" in line]
    print(f"{kind}: loss {losses[0]:.4f} -> {losses[-1]:.4f}")
    assert len(losses) >= 10 and all(np.isfinite(losses))
    assert np.mean(losses[-5:]) < np.mean(losses[:5])
    assert yaml.safe_load((run / "config.yaml").read_text())["model"]["attention"]["alibi"] is True
    loaded = load_run("alibi", str(tmp_path))
    assert loaded.model.args.alibi
    tokens = torch.randint(0, 256, (2, 100), generator=torch.Generator().manual_seed(1)).cuda()
    tr.model.eval()
    with torch.no_grad():
        a, b = tr.model(tokens).float(), loaded.model(tokens).float()
    assert rel(b, a) < 1e-6
