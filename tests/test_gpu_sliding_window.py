"""-m gpu: sliding-window attention (`model.attention.sliding_window`, b200_attn_{fwd,bwd,decode}_window): query q sees
key k iff 0 <= q - k <= W, intersected with the document of packed rows.

Tolerances are the packed-attention ones (tests/test_gpu_packed_attention.py): o / dq / dk / dv relative Frobenius
error < 1e-2 against an fp64 dense-mask reference, lse max abs error < 1e-3; model level bf16 loss 5e-3 / gradients
3e-2, fp32 (bf16x3 attention) 1e-3 / 8e-3.  Decode: the bound of tests/test_gpu_generation.py."""
import tempfile
from pathlib import Path

import numpy as np
import pytest
import torch

from tests.test_gpu_generation import C_BOUND
from tests.test_gpu_packed_attention import _loss_and_grads, layouts, positions

pytestmark = pytest.mark.gpu

ROOT = Path(__file__).resolve().parents[1]


@pytest.fixture(scope="module")
def ops():
    from mlx_cuda_distributed_pretraining_b200 import ops as o
    o.require_device()
    return o


def rel(a, b):
    """Relative Frobenius error; the floor keeps an all-but-zero reference (dq, dk at W = 0, where every query sees
    only itself) from dividing fp32 rounding by nothing."""
    a, b = a.detach().double(), b.detach().double().to(a.device)
    return float((a - b).norm() / max(float(b.norm()), 1e-3 * b.numel() ** 0.5))


def dense_mask(pos, window, S, device):
    from mlx_cuda_distributed_pretraining_b200.arch.flash_attention import CausalMask, DocumentCausalMask
    if pos is None:
        return CausalMask(S, window).dense(torch.float64, device)
    return DocumentCausalMask(pos, window).dense(torch.float64, device)


def reference(q, k, v, do, mask, scale):
    """fp64 softmax(q k^T * scale + mask) v, its lse, and dq / dk / dv (GQA by repeat)."""
    H, Hk = q.shape[2], k.shape[2]
    qr, kr, vr = (t.detach().double().requires_grad_(True) for t in (q, k, v))
    kx, vx = (t.repeat_interleave(H // Hk, dim=2) for t in (kr, vr))
    s = torch.einsum("bqhd,bkhd->bhqk", qr, kx) * scale + mask
    lse = torch.logsumexp(s, dim=-1)
    o = torch.einsum("bhqk,bkhd->bqhd", torch.softmax(s, dim=-1), vx)
    o.backward(do.double())
    return o, lse, qr.grad, kr.grad, vr.grad


def windows(S):
    return [0, 1, 63, 64, 65, 127, 128, 129, 300, S - 2, S - 1, S + 5]


def _inputs(B, S, H, Hk, D, dtype, seed):
    torch.manual_seed(seed)
    q = torch.randn(B, S, H, D, device="cuda").to(dtype).requires_grad_(True)
    k = torch.randn(B, S, Hk, D, device="cuda").to(dtype).requires_grad_(True)
    v = torch.randn(B, S, Hk, D, device="cuda").to(dtype).requires_grad_(True)
    do = torch.randn(B, S, H, D, device="cuda").to(dtype)
    return q, k, v, do


# ---- kernels against fp64 -------------------------------------------------------------------------------------------
@pytest.mark.parametrize("packed", [False, True], ids=["rows", "packed"])
@pytest.mark.parametrize("S,H,Hk,D", [(1000, 16, 8, 64), (2048, 2, 1, 64), (1000, 2, 1, 128), (2048, 4, 4, 128)])
def test_window_attention_vs_fp64(ops, S, H, Hk, D, packed):
    """Every W of windows(S); unpacked rows (pos = None), or the packed layouts of the document tests (boundaries at
    tile offsets, 1-3 token documents, length-1 documents, a trailing PAD run, a log-normal mix)."""
    pos = torch.stack([positions(l, S) for l in layouts(S, seed=D)]).int().cuda() if packed else None
    B = pos.shape[0] if packed else 2
    q, k, v, do = _inputs(B, S, H, Hk, D, torch.bfloat16, S + D + H)
    for W in windows(S):
        q.grad = k.grad = v.grad = None
        o = ops.attention(q, k, v, D ** -0.5, pos=pos, window=W)
        o.backward(do)
        _, lse = ops.attention_fwd_raw(q.detach(), k.detach(), v.detach(), D ** -0.5, True, pos, W)
        o_r, lse_r, dq_r, dk_r, dv_r = reference(q, k, v, do, dense_mask(pos, W, S, "cuda"), D ** -0.5)
        for b in range(B):
            errs = (rel(o[b], o_r[b]), rel(q.grad[b], dq_r[b]), rel(k.grad[b], dk_r[b]), rel(v.grad[b], dv_r[b]))
            assert max(errs) < 1e-2, (W, b, errs)
        assert float((lse.double() - lse_r.detach()).abs().max()) < 1e-3, W
        assert torch.isfinite(o).all() and torch.isfinite(q.grad).all() and torch.isfinite(k.grad).all(), W


@pytest.mark.parametrize("packed", [False, True], ids=["rows", "packed"])
def test_window_attention_fp32_path(ops, packed):
    """attention_fp32 (bf16x3, C1's head dim 16) with a window."""
    S, H, Hk, D = 1000, 8, 8, 16
    pos = torch.stack([positions(l, S) for l in layouts(S, seed=3)[:3]]).int().cuda() if packed else None
    B = 3 if packed else 2
    q, k, v, do = _inputs(B, S, H, Hk, D, torch.float32, 7)
    for W in (0, 1, 64, 129, 300, S - 1):
        q.grad = k.grad = v.grad = None
        o = ops.attention_fp32(q, k, v, D ** -0.5, pos=pos, window=W)
        o.backward(do)
        o_r, _, dq_r, dk_r, dv_r = reference(q, k, v, do, dense_mask(pos, W, S, "cuda"), D ** -0.5)
        errs = (rel(o, o_r), rel(q.grad, dq_r), rel(k.grad, dk_r), rel(v.grad, dv_r))
        assert max(errs) < 1e-2, (W, errs)


@pytest.mark.parametrize("packed", [False, True], ids=["rows", "packed"])
@pytest.mark.parametrize("S,H,Hk,D", [(1024, 16, 8, 64), (1000, 4, 2, 128)])
def test_covering_window_matches_causal_bit_for_bit(ops, S, H, Hk, D, packed):
    """W >= S - 1 is the causal (or document-causal) mask: the same o, lse, dk and dv bits (dq by tolerance: its fp32
    reduction order is not reproducible)."""
    pos = torch.stack([positions(l, S) for l in layouts(S, seed=1)[:3]]).int().cuda() if packed else None
    B = 3 if packed else 2
    q, k, v, do = (t.detach() for t in _inputs(B, S, H, Hk, D, torch.bfloat16, 5))
    o_c, lse_c = ops.attention_fwd_raw(q, k, v, D ** -0.5, True, pos)
    dq_c, dk_c, dv_c = ops.attention_bwd_raw(q, k, v, o_c, do, lse_c, D ** -0.5, True, pos)
    for W in (S - 1, S, S + 5, 1 << 30):
        o_w, lse_w = ops.attention_fwd_raw(q, k, v, D ** -0.5, True, pos, W)
        assert torch.equal(o_c, o_w) and torch.equal(lse_c, lse_w), W
        dq_w, dk_w, dv_w = ops.attention_bwd_raw(q, k, v, o_c, do, lse_c, D ** -0.5, True, pos, W)
        assert torch.equal(dk_c, dk_w) and torch.equal(dv_c, dv_w), W
        assert rel(dq_w, dq_c) < 1e-3, W


def test_bad_window_is_rejected(ops):
    q = torch.zeros(1, 64, 2, 64, device="cuda", dtype=torch.bfloat16)
    for bad in (-1, 1.5, True, "64"):
        with pytest.raises(ValueError):
            ops.attention(q, q, q, window=bad)
    from mlx_cuda_distributed_pretraining_b200._lib import B200Error
    with pytest.raises(B200Error):
        ops.attention_fwd_raw(q, q, q, 0.125, True, None, -1)
    L = ops.lib()
    assert int(L.b200_attn_bwd_window_workspace_bytes(2, 1000, 16, 8, 64)) == \
        int(L.b200_attn_bwd_doc_workspace_bytes(2, 1000, 16, 8, 64))


# ---- decode ---------------------------------------------------------------------------------------------------------
DEC_LENS = [1, 2, 255, 256, 257, 1000, 2048, 4095]
DEC_WINDOWS = [0, 1, 100, 255, 256, 257, 1000, 5000]
DEC_SMAX = 4160


def _window_cache(lens, W, H, D, dtype, seed):
    """MHA cache where every key below a row's window start is 4 q (a score of 4 |q|^2 scale, far above the rest) with
    V = 1e4: any such key that leaked into the softmax would dominate the output.  Positions at or past lens hold NaN."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    B = len(lens)
    q = torch.randn(B, H, D, device="cuda", generator=g).to(dtype)
    kc = torch.randn(B, DEC_SMAX, H, D, device="cuda", generator=g).to(dtype)
    vc = torch.randn(B, DEC_SMAX, H, D, device="cuda", generator=g).to(dtype)
    for b, n in enumerate(lens):
        kv0 = max(0, n - 1 - W)
        kc[b, :kv0] = 4 * q[b]
        vc[b, :kv0] = 1e4
        kc[b, n:] = float("nan")
        vc[b, n:] = float("nan")
    return q, kc, vc, torch.tensor(lens, device="cuda", dtype=torch.int32)


def _window_reference(q, kc, vc, lens, W, scale):
    out, absterm = [], []
    for b, n in enumerate(lens):
        kv0 = max(0, n - 1 - W)
        k, v = kc[b, kv0:n].double(), vc[b, kv0:n].double()
        p = torch.softmax(torch.einsum("hd,nhd->hn", q[b].double(), k) * scale, dim=-1)
        out.append(torch.einsum("hn,nhd->hd", p, v))
        absterm.append(torch.einsum("hn,nhd->hd", p, v.abs()))
    return torch.stack(out), torch.stack(absterm)


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float32], ids=["bf16", "fp32"])
@pytest.mark.parametrize("D", [16, 32, 64, 128])
def test_decode_window_matches_fp64(ops, dtype, D):
    H, scale = 4, D ** -0.5
    for W in DEC_WINDOWS:
        q, kc, vc, lens = _window_cache(DEC_LENS, W, H, D, dtype, seed=D + W)
        o = ops.attention_decode(q, kc, vc, lens, scale, window=W)
        R, absterm = _window_reference(q, kc, vc, DEC_LENS, W, scale)
        err = (o.double() - R).abs()
        bound = C_BOUND * 2.0 ** -24 * absterm + (2.0 ** -8 * R.abs() if dtype == torch.bfloat16 else 0)
        assert torch.isfinite(o).all(), W
        assert float((err / bound).max()) <= 1.0, (W, float((err / bound).max()))


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float32], ids=["bf16", "fp32"])
def test_decode_window_gqa_batch_invariant(ops, dtype):
    """GQA rows of mixed lengths under a window: fp64 agreement, and each row bit-identical alone and in the batch."""
    H, Hk, D, W = 16, 8, 64, 300
    lens = [2048, 5, 257, 1000, 4095, 256, 31, 301, 302]
    g = torch.Generator(device="cuda").manual_seed(3)
    q = torch.randn(len(lens), H, D, device="cuda", generator=g).to(dtype)
    kc = torch.randn(len(lens), DEC_SMAX, Hk, D, device="cuda", generator=g).to(dtype)
    vc = torch.randn(len(lens), DEC_SMAX, Hk, D, device="cuda", generator=g).to(dtype)
    lt = torch.tensor(lens, device="cuda", dtype=torch.int32)
    o = ops.attention_decode(q, kc, vc, lt, window=W)
    assert torch.equal(o, ops.attention_decode(q, kc, vc, lt, window=W))
    R, absterm = _window_reference(q, kc.repeat_interleave(2, 2), vc.repeat_interleave(2, 2), lens, W, D ** -0.5)
    bound = C_BOUND * 2.0 ** -24 * absterm + (2.0 ** -8 * R.abs() if dtype == torch.bfloat16 else 0)
    assert float(((o.double() - R).abs() / bound).max()) <= 1.0
    for b in range(len(lens)):
        alone = ops.attention_decode(q[b:b + 1].contiguous(), kc[b:b + 1].contiguous(), vc[b:b + 1].contiguous(),
                                     lt[b:b + 1].contiguous(), window=W)
        assert torch.equal(alone[0], o[b]), b
    # a window that covers every row gives the unwindowed kernel's bits
    assert torch.equal(ops.attention_decode(q, kc, vc, lt, window=DEC_SMAX), ops.attention_decode(q, kc, vc, lt))


# ---- model level ----------------------------------------------------------------------------------------------------
def _model(dtype, rope, hidden, layers, heads, kv_heads, head_dim, window, vocab=259):
    from mlx_cuda_distributed_pretraining_b200.arch.llama import Model, ModelArgs
    from mlx_cuda_distributed_pretraining_b200.core.training import init_model_
    args = ModelArgs(model_type="llama", hidden_size=hidden, num_hidden_layers=layers, intermediate_size=2 * hidden,
                     num_attention_heads=heads, num_key_value_heads=kv_heads, head_dim=head_dim, vocab_size=vocab,
                     tie_word_embeddings=True, apply_rope=rope, sliding_window=window)
    m = Model(args)
    init_model_(m, args, seed=3)
    return m.to("cuda", dtype)


def _dense_attention(self, q, k, v, mask=None):
    """FlashAttention._flash_attention replaced by fp64 softmax(q k^T scale + mask.dense()) v."""
    H, Hk = q.shape[2], k.shape[2]
    kx, vx = (t.double().repeat_interleave(H // Hk, dim=2) for t in (k, v))
    s = torch.einsum("bqhd,bkhd->bhqk", q.double(), kx) * self.scale + mask.dense(torch.float64, q.device)
    return torch.einsum("bhqk,bkhd->bqhd", torch.softmax(s, dim=-1), vx).to(q.dtype)


@pytest.mark.parametrize("kind,rope", [("bf16_gqa", False), ("bf16_gqa", True), ("c1_fp32", True)])
def test_windowed_model_matches_dense_reference(ops, monkeypatch, kind, rope):
    from mlx_cuda_distributed_pretraining_b200.arch.flash_attention import FlashAttention
    W = 70
    if kind == "bf16_gqa":
        model, tol_loss, tol_grad = _model(torch.bfloat16, rope, 256, 2, 8, 2, 64, W), 5e-3, 3e-2
    else:
        model, tol_loss, tol_grad = _model(torch.float32, rope, 128, 4, 8, 8, 16, W), 1e-3, 8e-3
    g = torch.Generator().manual_seed(4)
    toks = torch.randint(0, 256, (2, 301), generator=g).cuda()
    inputs, targets = toks[:, :-1], toks[:, 1:]
    loss_k, g_k = _loss_and_grads(model, inputs, targets, None)
    monkeypatch.setattr(FlashAttention, "_flash_attention", _dense_attention)
    loss_r, g_r = _loss_and_grads(model, inputs, targets, None)
    worst = max(rel(g_k[n], g_r[n]) for n in g_r)
    print(f"{kind} rope={rope}: loss kernel {loss_k:.6f} dense {loss_r:.6f}, worst grad rel {worst:.2e}")
    assert abs(loss_k - loss_r) < tol_loss * abs(loss_r)
    assert worst < tol_grad


@pytest.mark.parametrize("kind", ["bf16_gqa", "c1_fp32"])
def test_packed_windowed_rows_match_documents_alone(ops, kind):
    from mlx_cuda_distributed_pretraining_b200.core.training import document_positions, pack_first_fit
    W = 50
    if kind == "bf16_gqa":
        model, tol_loss, tol_grad = _model(torch.bfloat16, True, 256, 2, 8, 2, 64, W), 5e-3, 3e-2
    else:
        model, tol_loss, tol_grad = _model(torch.float32, True, 128, 4, 8, 8, 16, W), 1e-3, 8e-3
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
    assert max(len(d) for d in docs) > 2 * W   # the window cuts inside documents
    loss_p, g_p = _loss_and_grads(model, inputs, targets, pos)
    loss_a, g_a = _loss_and_grads(model, alone[:, :-1], alone[:, 1:], None)
    worst = max(rel(g_p[n], g_a[n]) for n in g_a)
    print(f"{kind}: loss packed {loss_p:.6f} alone {loss_a:.6f}, worst grad rel {worst:.2e}")
    assert abs(loss_p - loss_a) < tol_loss * abs(loss_a)
    assert worst < tol_grad


def _window_trainer(kind, W):
    from mlx_cuda_distributed_pretraining_b200.core.training import Config, Trainer
    from tests.test_gpu_generation import _cfg
    c = _cfg(kind)
    c["model"]["attention"]["sliding_window"] = W
    return Trainer(Config.from_dict(c), for_training=False, synthetic=True, quiet=True,
                   run_root=tempfile.mkdtemp(prefix="win_runs_"))


@pytest.mark.parametrize("kind", ["bf16_rope", "c1_fp32"])
def test_prefill_decode_match_forward_with_sliding_window(kind):
    """260-token prompt, 39 decode steps, W = 100: the window slides during decoding.  Logits against Model.forward
    (the tolerances of tests/test_gpu_generation.py), then greedy tokens wherever the top-2 margin exceeds them."""
    from mlx_cuda_distributed_pretraining_b200.arch.llama import KVCache
    from mlx_cuda_distributed_pretraining_b200.core.generation import generate
    from tests.test_gpu_generation import TOL, _rel_rows
    tr = _window_trainer(kind, 100)
    model = tr.model
    assert model.args.sliding_window == 100
    T, t0 = 300, 260
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
    out = generate(model, [prompt], max_tokens=39, temperature=0, repetition_penalty=1.0, min_p=None)[0]
    seq, skipped = list(prompt), 0
    for i, t in enumerate(out):
        with torch.no_grad():
            logits = model(torch.tensor([seq], device="cuda")).float()[0, -1]
        top2 = torch.topk(logits, 2).values
        if float(top2[0] - top2[1]) <= TOL[kind] * float(logits.abs().max()):
            skipped += 1
        else:
            assert t == int(torch.argmax(logits)), f"step {i}"
        seq.append(t)
    assert skipped < len(out) // 2


# ---- trainer --------------------------------------------------------------------------------------------------------
def test_packed_windowed_trainer_run_loads_for_generation(tmp_path):
    import yaml
    from mlx_cuda_distributed_pretraining_b200.core.generation import generate, load_run
    from mlx_cuda_distributed_pretraining_b200.core.training import Config, Trainer
    from tests.test_gpu_packed_attention import _packed_cfg
    cfg = _packed_cfg(6)
    cfg["model"]["attention"]["sliding_window"] = 64
    cfg["logging"]["steps"]["checkpoint_interval"] = 0
    tr = Trainer(Config.from_dict(cfg), quiet=True, run_root=str(tmp_path))
    assert tr.data_manager.pack and tr.model.args.sliding_window == 64
    tr.train()
    run = tmp_path / "smoke"
    losses = [float(line.split("loss=")[1].split()[0].rstrip("|"))
              for line in (run / "log.txt").read_text().splitlines() if "loss=" in line]
    assert losses and all(np.isfinite(losses))
    assert yaml.safe_load((run / "config.yaml").read_text())["model"]["attention"]["sliding_window"] == 64
    loaded = load_run("smoke", str(tmp_path))
    assert loaded.model.args.sliding_window == 64
    out = generate(loaded.model, [[loaded.tokenizer.BOS_TOKEN] + list(range(40, 120))], max_tokens=8, temperature=0)
    assert len(out[0]) == 8


def test_covering_window_trainer_matches_causal_on_c1_control():
    """C1 on its control stream (Markov tokens, lr 1e-3: no chaotic transient) with W = max_context_size against the
    same run without the key: the per-step tolerance of the C1 parity tests."""
    import yaml
    from mlx_cuda_distributed_pretraining_b200.core.training import Config, Trainer

    def run(window):
        d = yaml.safe_load((ROOT / "configs" / "c1-llama2m-adamw.yaml").read_text())
        d["name"] = "c1-window"
        d["data"]["input_file"] = "synthetic:markov"
        d["training"]["hyperparameters"].update(iters=40, learning_rate=1e-3)
        d["logging"]["steps"] = {"logging_interval": 10 ** 9, "checkpoint_interval": 0, "validation_interval": 0}
        if window is not None:
            d["model"]["attention"]["sliding_window"] = window
        tr = Trainer(Config.from_dict(d), synthetic=True, quiet=True, run_root=tempfile.mkdtemp(prefix="c1w_"))
        assert tr.model.args.sliding_window == window
        tr._accum_step, tr._accum_tokens = 0, 0
        return torch.stack([tr.train_step(s, tr.data_manager.generate_batch(s))[0] for s in range(40)]).float().cpu()

    d = yaml.safe_load((ROOT / "configs" / "c1-llama2m-adamw.yaml").read_text())
    base, win = run(None), run(d["data"]["preprocessing"]["max_context_size"])
    assert torch.isfinite(win).all()
    assert float((base - win).abs().max()) < 2e-2, (base - win).abs().max()
