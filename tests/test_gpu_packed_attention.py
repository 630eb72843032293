"""-m gpu: packed sequences -- the document-causal attention kernels (b200_attn_fwd_doc / b200_attn_bwd_doc), RoPE by
position within the document (b200_rope_pos), the model with position_ids, and a packed trainer run.

Tolerances: attention o / dq / dk / dv relative Frobenius error < 1e-2 against an fp64 dense-mask reference (the
attention tolerance of test_gpu_parity.py), lse max abs error < 1e-3.  Single-document rows and RoPE are bit-exact.
Model level (packed vs one document per row, relative): bf16 loss 5e-3 / gradients 3e-2; fp32 with bf16x3 attention
1e-3 / 8e-3 (its P and outputs pass one bf16 rounding, and packing changes which keys share a tile)."""
import random
from pathlib import Path

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

ROOT = Path(__file__).resolve().parents[1]
BOS = 1


def rel(a, b):
    a, b = a.detach().double(), b.detach().double().to(a.device)
    return float((a - b).norm() / (b.norm() + 1e-4))


@pytest.fixture(scope="module")
def ops():
    from mlx_cuda_distributed_pretraining_b200 import ops as o
    o.require_device()
    return o


def positions(layout, S):
    """pos [S] of one packed row: documents of the given lengths from position 0, then a PAD run.  pos comes from the
    trainer's BOS rule (a PAD run continues the last document, as it does in the trainer)."""
    from mlx_cuda_distributed_pretraining_b200.core.training import document_positions
    toks = torch.full((S,), 7, dtype=torch.int64)
    at = 0
    for n in layout:
        toks[at] = BOS
        at += n
    assert at <= S
    return document_positions(toks[None], BOS)[0]


def layouts(S, seed=0):
    rng = random.Random(seed)
    bounds = [0, 1] + [o + 128 * (i + 1) for i, o in enumerate((63, 64, 65, 127, 128, 129)) if o + 128 * (i + 1) < S]
    boundary = [b - a for a, b in zip(bounds, bounds[1:] + [S])]
    tiny = []
    while sum(tiny) < S:
        tiny.append(min(rng.randint(1, 3), S - sum(tiny)))
    ones = [1] * 5 + [100] + [1] * 3 + [S - 109]
    trailing_pad = [S // 3, 1, S // 4]           # PAD from S // 3 + 1 + S // 4 to the end
    lognormal = []
    while sum(lognormal) < S:
        lognormal.append(min(max(1, int(rng.lognormvariate(4.5, 1.0))), S - sum(lognormal)))
    return [boundary, tiny, ones, trailing_pad, lognormal]


def reference(q, k, v, do, pos, scale):
    """fp64 softmax(q k^T * scale + DocumentCausalMask(pos).dense()) v, its lse, and dq / dk / dv (GQA by repeat)."""
    from mlx_cuda_distributed_pretraining_b200.arch.flash_attention import DocumentCausalMask
    H, Hk = q.shape[2], k.shape[2]
    qr, kr, vr = (t.detach().double().requires_grad_(True) for t in (q, k, v))
    kx, vx = (t.repeat_interleave(H // Hk, dim=2) for t in (kr, vr))
    s = torch.einsum("bqhd,bkhd->bhqk", qr, kx) * scale + DocumentCausalMask(pos).dense(torch.float64, q.device)
    lse = torch.logsumexp(s, dim=-1)
    o = torch.einsum("bhqk,bkhd->bqhd", torch.softmax(s, dim=-1), vx)
    o.backward(do.double())
    return o, lse, qr.grad, kr.grad, vr.grad


@pytest.mark.parametrize("S,H,Hk,D", [(1000, 16, 8, 64), (2048, 2, 1, 64), (1000, 2, 1, 128), (2048, 16, 8, 128)])
def test_document_attention_vs_fp64(ops, S, H, Hk, D):
    """Every row of the batch a different layout: boundaries at offsets 1, 63, 64, 65, 127, 128, 129 within a tile,
    rows of 1-3 token documents, length-1 documents, a trailing PAD run, a log-normal mix."""
    torch.manual_seed(S + D + H)
    lay = layouts(S, seed=D)
    pos = torch.stack([positions(l, S) for l in lay]).int().cuda()
    B = len(lay)
    q = torch.randn(B, S, H, D, device="cuda").to(torch.bfloat16).requires_grad_(True)
    k = torch.randn(B, S, Hk, D, device="cuda").to(torch.bfloat16).requires_grad_(True)
    v = torch.randn(B, S, Hk, D, device="cuda").to(torch.bfloat16).requires_grad_(True)
    do = torch.randn(B, S, H, D, device="cuda").to(torch.bfloat16)
    o = ops.attention(q, k, v, D ** -0.5, pos=pos)
    o.backward(do)
    _, lse = ops.attention_fwd_raw(q.detach(), k.detach(), v.detach(), D ** -0.5, True, pos)
    o_r, lse_r, dq_r, dk_r, dv_r = reference(q, k, v, do, pos, D ** -0.5)
    for b in range(B):
        errs = (rel(o[b], o_r[b]), rel(q.grad[b], dq_r[b]), rel(k.grad[b], dk_r[b]), rel(v.grad[b], dv_r[b]))
        assert max(errs) < 1e-2, (b, errs)
    assert float((lse.double() - lse_r.detach()).abs().max()) < 1e-3
    assert torch.isfinite(o).all() and torch.isfinite(q.grad).all() and torch.isfinite(k.grad).all()


@pytest.mark.parametrize("S,H,Hk", [(1000, 8, 8), (2048, 4, 2)])
def test_document_attention_fp32_path(ops, S, H, Hk):
    """attention_fp32 (bf16x3, C1's head dim 16) with documents."""
    D = 16
    torch.manual_seed(S + H)
    lay = layouts(S, seed=3)[:3]
    pos = torch.stack([positions(l, S) for l in lay]).int().cuda()
    B = len(lay)
    q = torch.randn(B, S, H, D, device="cuda").requires_grad_(True)
    k = torch.randn(B, S, Hk, D, device="cuda").requires_grad_(True)
    v = torch.randn(B, S, Hk, D, device="cuda").requires_grad_(True)
    do = torch.randn(B, S, H, D, device="cuda")
    o = ops.attention_fp32(q, k, v, D ** -0.5, pos=pos)
    o.backward(do)
    o_r, _, dq_r, dk_r, dv_r = reference(q, k, v, do, pos, D ** -0.5)
    errs = (rel(o, o_r), rel(q.grad, dq_r), rel(k.grad, dk_r), rel(v.grad, dv_r))
    assert max(errs) < 1e-2, errs


@pytest.mark.parametrize("S,H,Hk,D", [(1024, 16, 8, 64), (1000, 4, 2, 128), (2048, 2, 1, 64)])
def test_single_document_rows_match_causal_bit_for_bit(ops, S, H, Hk, D):
    """pos = arange: the document kernels run the causal kernels' arithmetic (dq goes through a different CTA order
    of the fp32 reduction, so it is compared by tolerance)."""
    torch.manual_seed(5)
    B = 2
    q = torch.randn(B, S, H, D, device="cuda").to(torch.bfloat16)
    k = torch.randn(B, S, Hk, D, device="cuda").to(torch.bfloat16)
    v = torch.randn(B, S, Hk, D, device="cuda").to(torch.bfloat16)
    do = torch.randn(B, S, H, D, device="cuda").to(torch.bfloat16)
    pos = torch.arange(S, device="cuda", dtype=torch.int32).expand(B, S).contiguous()
    o_c, lse_c = ops.attention_fwd_raw(q, k, v, D ** -0.5, True)
    o_d, lse_d = ops.attention_fwd_raw(q, k, v, D ** -0.5, True, pos)
    assert torch.equal(o_c, o_d) and torch.equal(lse_c, lse_d)
    dq_c, dk_c, dv_c = ops.attention_bwd_raw(q, k, v, o_c, do, lse_c, D ** -0.5, True)
    dq_d, dk_d, dv_d = ops.attention_bwd_raw(q, k, v, o_c, do, lse_c, D ** -0.5, True, pos)
    assert torch.equal(dk_c, dk_d) and torch.equal(dv_c, dv_d)
    assert rel(dq_d, dq_c) < 1e-3


def test_workspace_sizes(ops):
    L = ops.lib()
    for B, S, H, Hk, D in ((2, 1000, 16, 8, 64), (16, 2048, 16, 16, 128)):
        base = int(L.b200_attn_bwd_workspace_bytes(B, S, H, Hk, D))
        s_pad = -(-S // 64) * 64
        al = lambda x: -(-x // 256) * 256  # noqa: E731
        assert base == al(B * S * H * D * 4) + 2 * al(B * H * s_pad * 4)
        assert int(L.b200_attn_bwd_doc_workspace_bytes(B, S, H, Hk, D)) == \
            base + al(B * s_pad * 4) + al(B * -(-S // 128) * 4)


def test_bad_pos_is_rejected(ops):
    q = torch.zeros(1, 64, 2, 64, device="cuda", dtype=torch.bfloat16)
    with pytest.raises(ValueError):
        ops.attention(q, q, q, pos=torch.zeros(1, 32, device="cuda", dtype=torch.int32))
    with pytest.raises(ValueError):
        ops.attention(q, q, q, pos=torch.zeros(1, 64, device="cuda", dtype=torch.int64))
    from mlx_cuda_distributed_pretraining_b200._lib import B200Error
    with pytest.raises(B200Error):
        ops.attention_fwd_raw(q, q, q, 0.125, True, torch.empty(0, device="cuda", dtype=torch.int32))


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float32])
def test_rope_with_positions_is_rope_per_document(ops, dtype):
    torch.manual_seed(9)
    S, NH, D = 1000, 3, 64
    lay = layouts(S, seed=1)[:3]
    pos = torch.stack([positions(l, S) for l in lay]).int().cuda()
    cos_t, sin_t = ops.rope_tables(S, D, 10000.0, "cuda")
    x = torch.randn(len(lay), S, NH, D, device="cuda").to(dtype).requires_grad_(True)
    y = ops.rope(x, cos_t, sin_t, pos)
    dy = torch.randn_like(y)
    y.backward(dy)
    for b in range(len(lay)):
        starts = (pos[b] == 0).nonzero().flatten().tolist() + [S]
        for a0, a1 in zip(starts, starts[1:]):   # one document (with the PAD run that continues it)
            xs = x[b:b + 1, a0:a1].detach().requires_grad_(True)
            ys = ops.rope(xs, cos_t[:a1 - a0], sin_t[:a1 - a0])
            ys.backward(dy[b:b + 1, a0:a1])
            assert torch.equal(y[b, a0:a1], ys[0]), (b, a0)
            assert torch.equal(x.grad[b, a0:a1], xs.grad[0]), (b, a0)


# ---- model level: packed rows against the same documents one per row ----------------------------------------------
def _model(dtype, rope, hidden, layers, heads, kv_heads, head_dim, vocab=259):
    from mlx_cuda_distributed_pretraining_b200.arch.llama import Model, ModelArgs
    from mlx_cuda_distributed_pretraining_b200.core.training import init_model_
    args = ModelArgs(model_type="llama", hidden_size=hidden, num_hidden_layers=layers, intermediate_size=2 * hidden,
                     num_attention_heads=heads, num_key_value_heads=kv_heads, head_dim=head_dim, vocab_size=vocab,
                     tie_word_embeddings=True, apply_rope=rope)
    m = Model(args)
    init_model_(m, args, seed=3)
    return m.to("cuda", dtype)


def _loss_and_grads(model, inputs, targets, position_ids, pad=256):
    model.zero_grad(set_to_none=True)
    logits = (model(inputs) if position_ids is None else model(inputs, position_ids)).float()
    ce = torch.nn.functional.cross_entropy(logits.reshape(-1, logits.shape[-1]), targets.reshape(-1),
                                           reduction="none").view(targets.shape)
    loss = (ce * (targets != pad)).sum()
    loss.backward()
    return float(loss.detach()), {n: p.grad.detach().double().clone() for n, p in model.named_parameters()}


@pytest.mark.parametrize("kind,rope", [("bf16_gqa", False), ("bf16_gqa", True), ("c1_fp32", False),
                                       ("c1_fp32", True)])
def test_packed_model_matches_documents_run_alone(ops, kind, rope):
    from mlx_cuda_distributed_pretraining_b200.core.training import document_positions, pack_first_fit
    if kind == "bf16_gqa":
        model, tol_loss, tol_grad = _model(torch.bfloat16, rope, 256, 2, 8, 2, 64), 5e-3, 3e-2
    else:
        model, tol_loss, tol_grad = _model(torch.float32, rope, 128, 4, 8, 8, 16), 1e-3, 8e-3
    PAD, BOS_ID, EOS, L = 256, 257, 258, 385   # the byte tokenizer's special ids
    rng = np.random.default_rng(11)
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
    assert int((targets != PAD).sum()) == int((alone[:, 1:] != PAD).sum())
    worst = max(rel(g_p[n], g_a[n]) for n in g_a)
    print(f"{kind} rope={rope}: loss packed {loss_p:.6f} alone {loss_a:.6f}, worst grad rel {worst:.2e}")
    assert abs(loss_p - loss_a) < tol_loss * abs(loss_a), (loss_p, loss_a)
    assert worst < tol_grad, worst
    # negative control: the packed batch without position_ids leaks across documents
    loss_x, g_x = _loss_and_grads(model, inputs, targets, None)
    leak = max(rel(g_x[n], g_a[n]) for n in g_a)
    print(f"  without position_ids: loss {loss_x:.6f}, worst grad rel {leak:.2e}")
    assert leak > 5 * worst and abs(loss_x - loss_a) > 5 * abs(loss_p - loss_a), (leak, worst, loss_x, loss_p, loss_a)


# ---- trainer: packed run on the tiny corpus, resume replays the same batches ---------------------------------------
def _packed_cfg(iters):
    from tests.smoke_check import tiny_config
    cfg = tiny_config(hp__iters=iters)
    cfg["data"]["input_file"] = str(ROOT / "tests" / "golden" / "tiny_corpus.jsonl")
    cfg["data"]["preprocessing"] = {"max_context_size": 128, "chunk_overlap": 0, "pack_sequences": True}
    cfg["model"]["rope"]["enabled"] = True
    cfg["logging"]["steps"] = {"logging_interval": 1, "checkpoint_interval": 3, "validation_interval": 0}
    return cfg


def test_packed_trainer_run_and_resume(tmp_path):
    from mlx_cuda_distributed_pretraining_b200.core.training import Config, Trainer
    tr = Trainer(Config.from_dict(_packed_cfg(6)), quiet=True, run_root=str(tmp_path / "a"))
    assert tr.data_manager.pack and tr.steps_per_epoch == tr.data_manager.num_train_batches
    out = tr.train()
    log = (tmp_path / "a" / "smoke" / "log.txt").read_text()
    losses = [float(line.split("loss=")[1].split()[0].rstrip("|")) for line in log.splitlines() if "loss=" in line]
    assert losses and all(np.isfinite(losses)), log
    assert out is not None
    ck = tmp_path / "a" / "smoke" / "checkpoints" / "step_3"
    cfg = _packed_cfg(6)
    cfg["resume"] = {"checkpoint": str(ck)}
    tr2 = Trainer(Config.from_dict(cfg), quiet=True, run_root=str(tmp_path / "b"))
    assert tr2.load_checkpoint(str(ck)) == 3
    for step in range(8):
        assert torch.equal(tr2.data_manager.generate_batch(step), tr.data_manager.generate_batch(step)), step
