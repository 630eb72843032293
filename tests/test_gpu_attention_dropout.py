"""Attention dropout on the GPU: the kernels' keep masks bit for bit against the Philox oracle, O / LSE / dQ / dK / dV
against an fp64 reference with the oracle's mask, bit identities with the dropout-free kernels, autograd, the model
and the trainer."""
import numpy as np
import pytest
import torch

from tests import dropout_oracle as do

pytestmark = pytest.mark.gpu

CANARY = float("nan")


def _ops():
    from mlx_cuda_distributed_pretraining_b200 import ops
    return ops


def _mask_add(kind, B, S, H, pos=None, window=None, slopes=None):
    """Additive [B, H, S, S] fp64 mask (0 / -inf plus the ALiBi bias) of a kernel family."""
    s = torch.arange(S, dtype=torch.float64)
    qd, kd = s[:, None], s[None, :]
    if kind == "full":
        ok = torch.ones(B, S, S, dtype=torch.bool)
    else:
        start = torch.zeros(B, S, dtype=torch.float64)
        if pos is not None:
            start = s[None] - pos.double().cpu()
        if window is not None:
            start = torch.maximum(start, s[None] - window)
        ok = (kd[None] <= qd[None]) & (kd[None] >= start[:, :, None])
    m = torch.zeros(B, 1, S, S, dtype=torch.float64).masked_fill(~ok[:, None], float("-inf")).expand(B, H, S, S)
    if slopes is not None:
        m = m + slopes.double().cpu()[None, :, None, None] * (kd - qd)[None, None]
    return m


def _family(kind, B, S, H, dev):
    """(kwargs for ops, fp64 additive mask) of one kernel family."""
    kw, pos, window, slopes = {"causal": kind != "full"}, None, None, None
    if kind == "document":
        g = torch.Generator().manual_seed(S)
        pos = torch.zeros(B, S, dtype=torch.int32)
        for b in range(B):
            c = 0
            for t in range(S):
                c = 0 if (t > 0 and torch.rand((), generator=g) < 0.02) else (c + 1 if t > 0 else 0)
                pos[b, t] = c
        kw["pos"] = pos.to(dev)
    if kind == "window":
        window = 77
        kw["window"] = window
    if kind == "alibi":
        slopes = torch.linspace(0.001, 0.01, H, dtype=torch.float32)
        kw["alibi"] = slopes.to(dev)
    return kw, _mask_add(kind, B, S, H, pos, window, slopes)


def _raw_fwd(q, k, v, scale, kw, drop):
    ops = _ops()
    return ops.attention_fwd_raw(q, k, v, scale, kw.get("causal", True), kw.get("pos"), kw.get("window"),
                                 kw.get("alibi"), None, drop)


def _raw_bwd(q, k, v, o, do_, lse, scale, kw, drop):
    ops = _ops()
    return ops.attention_bwd_raw(q, k, v, o, do_, lse, scale, kw.get("causal", True), kw.get("pos"),
                                 kw.get("window"), kw.get("alibi"), None, drop)


PROBES = [  # kind, D, B, S, H, Hk
    ("causal", 128, 2, 129, 4, 4), ("causal", 64, 1, 1000, 8, 1), ("full", 128, 2, 63, 2, 2),
    ("full", 64, 1, 1, 3, 1), ("document", 128, 2, 300, 4, 2), ("window", 64, 2, 1000, 8, 8),
    ("alibi", 128, 1, 1000, 8, 1), ("alibi", 64, 2, 129, 4, 4),
]


@pytest.mark.parametrize("kind,D,B,S,H,Hk", PROBES)
def test_mask_probe_forward(kind, D, B, S, H, Hk):
    """q = 0 makes P positive on every visible key; V one-hot per key of a D-key block makes O[q, c] > 0 iff key
    k0 + c is visible and kept."""
    dev = torch.device("cuda")
    p, seed = 0.5, 0xC0FFEE_1234_5678
    kw, madd = _family(kind, B, S, H, dev)
    keep = do.keep_mask(seed, p, B, H, S)
    visible = torch.isfinite(madd).numpy()
    q = torch.zeros(B, S, H, D, device=dev, dtype=torch.bfloat16)
    k = torch.zeros(B, S, Hk, D, device=dev, dtype=torch.bfloat16)
    for k0 in sorted({0, max(0, (S - 1) // D * D)}):
        n = min(D, S - k0)
        v = torch.zeros(B, S, Hk, D, device=dev, dtype=torch.bfloat16)
        idx = torch.arange(n, device=dev)
        v[:, k0 + idx, :, idx] = 1.0
        o, _ = _raw_fwd(q, k, v, D ** -0.5, kw, (p, seed))
        got = (o.float()[..., :n] > 0).permute(0, 2, 1, 3).cpu().numpy()  # [B, H, S, n]
        want = keep[..., k0:k0 + n] & visible[..., k0:k0 + n]
        assert (got == want).all(), f"{kind} k0={k0}: {(got != want).sum()} mask bits differ"


@pytest.mark.parametrize("kind,D,B,S,H,Hk", PROBES)
def test_mask_probe_backward(kind, D, B, S, H, Hk):
    """dV[k, c] = sum_h (P o Z)[q0 + c, k] / (1 - p_eff) with dO one-hot per query of a D-query block, on one query
    head at a time (so GQA sums hold one term): dV > 0 iff the key is visible to the query and kept."""
    dev = torch.device("cuda")
    p, seed = 0.5, 0x5EED_0000_0000_0042
    kw, madd = _family(kind, B, S, H, dev)
    keep = do.keep_mask(seed, p, B, H, S)
    visible = torch.isfinite(madd).numpy()
    q = torch.zeros(B, S, H, D, device=dev, dtype=torch.bfloat16)
    k = torch.zeros(B, S, Hk, D, device=dev, dtype=torch.bfloat16)
    v = torch.randn(B, S, Hk, D, device=dev).to(torch.bfloat16)
    o, lse = _raw_fwd(q, k, v, D ** -0.5, kw, (p, seed))
    heads = sorted({0, H - 1})
    for h in heads:
        for q0 in sorted({0, max(0, (S - 1) // D * D)}):
            n = min(D, S - q0)
            g = torch.zeros(B, S, H, D, device=dev, dtype=torch.bfloat16)
            idx = torch.arange(n, device=dev)
            g[:, q0 + idx, h, idx] = 1.0
            _, _, dv = _raw_bwd(q, k, v, o, g, lse, D ** -0.5, kw, (p, seed))
            got = (dv.float()[:, :, h // (H // Hk), :n] > 0).cpu().numpy()  # [B, S keys, n queries]
            want = (keep[:, h, q0:q0 + n, :] & visible[:, h, q0:q0 + n, :]).transpose(0, 2, 1)
            assert (got == want).all(), f"{kind} h={h} q0={q0}: {(got != want).sum()} mask bits differ"


def _vis(kind, kw, B, S, dev):
    """bool [B, S, S] visibility of a kernel family (tests/attn_fwd_check.visible)."""
    from tests import attn_fwd_check as fc
    m = fc.visible(S, kind != "full", pos=kw.get("pos"), window=kw.get("window"), device=dev)
    return m.expand(B, S, S) if m.dim() == 2 else m


def _run_canary(q, k, v, g, kw, p, seed):
    """The dropout C entries with every output in a NaN-filled buffer: (o, lse, dq, dk, dv)."""
    ops = _ops()
    B, S, H, D = q.shape
    Hk = k.shape[2]
    L, st = ops.lib(), ops._stream()
    pos, window, slopes = kw.get("pos"), kw.get("window"), kw.get("alibi")
    win = -1 if window is None else window
    o = torch.full_like(q, CANARY)
    lse = torch.full((B, H, S), CANARY, device=q.device)
    ops.check(L.b200_attn_fwd_dropout(q.data_ptr(), k.data_ptr(), v.data_ptr(), o.data_ptr(), lse.data_ptr(),
                                      ops._ptr(pos), win, ops._ptr(slopes), B, S, H, Hk, D, D ** -0.5,
                                      int(kw.get("causal", True)), p, seed, st), "b200_attn_fwd_dropout")
    dq = torch.full_like(q, CANARY)
    dkv = torch.full((B, S, 2 * Hk, D), CANARY, device=q.device, dtype=q.dtype)
    ws = torch.empty(int(L.b200_attn_bwd_dropout_workspace_bytes(B, S, H, Hk, D)), device=q.device,
                     dtype=torch.uint8)
    ops.check(L.b200_attn_bwd_dropout(q.data_ptr(), k.data_ptr(), v.data_ptr(), o.data_ptr(), g.data_ptr(),
                                      lse.data_ptr(), ops._ptr(pos), win, ops._ptr(slopes), dq.data_ptr(),
                                      dkv.data_ptr(), dkv[:, :, Hk:].data_ptr(), B, S, H, Hk, D, D ** -0.5,
                                      int(kw.get("causal", True)), p, seed, 2 * Hk, ws.data_ptr(), ws.numel(), st),
              "b200_attn_bwd_dropout")
    return o, lse, dq, dkv[:, :, :Hk], dkv[:, :, Hk:]


# the probe matrix plus ragged lengths up to 8192
CASES = PROBES + [("causal", 64, 1, 8192, 2, 1), ("document", 128, 1, 4097, 2, 1), ("causal", 128, 2, 63, 4, 1),
                  ("window", 128, 1, 3001, 4, 2)]


@pytest.mark.parametrize("p", [0.1, 0.5])
@pytest.mark.parametrize("kind,D,B,S,H,Hk", CASES)
def test_elementwise_fp64(kind, D, B, S, H, Hk, p):
    """O, LSE, dQ, dK, dV of the dropout entries, written into NaN-filled buffers, element by element against fp64
    with the oracle's mask and the bounds of tests/attn_dropout_check.py."""
    from tests import attn_dropout_check as dc
    dev = torch.device("cuda")
    seed = 0x0123_4567_89AB_CDEF ^ S
    torch.manual_seed(S)
    kw, _ = _family(kind, B, S, H, dev) if S <= 1000 else _family_large(kind, B, S, H, dev)
    q = torch.randn(B, S, H, D, device=dev).to(torch.bfloat16)
    k = torch.randn(B, S, Hk, D, device=dev).to(torch.bfloat16)
    v = torch.randn(B, S, Hk, D, device=dev).to(torch.bfloat16)
    g = torch.randn(B, S, H, D, device=dev).to(torch.bfloat16)
    o, lse, dq, dk, dv = _run_canary(q, k, v, g, kw, p, seed)
    ref = dc.reference(q, k, v, o, g, lse, D ** -0.5, _vis(kind, kw, B, S, dev), seed, p, slopes=kw.get("alibi"))
    for name, got in (("o", o), ("lse", lse), ("dq", dq), ("dk", dk), ("dv", dv)):
        dc.check(f"{kind} S={S} p={p} {name}", got, *ref[name])


def _family_large(kind, B, S, H, dev):
    """_family without the fp64 additive mask (too large at S in the thousands)."""
    kw = {"causal": kind != "full"}
    if kind == "document":
        pos = torch.zeros(B, S, dtype=torch.int32)
        starts = torch.tensor([0, 700, 701, 2000, 4000])
        for t in range(S):
            pos[:, t] = t - int(starts[starts <= t].max())
        kw["pos"] = pos.to(dev)
    if kind == "window":
        kw["window"] = 300
    return kw, None


def test_canary_outputs_fully_written():
    """The dropout entries write every element of O and LSE (outputs start as NaN)."""
    ops = _ops()
    dev = torch.device("cuda")
    B, S, H, D = 2, 200, 4, 64
    q = torch.randn(B, S, H, D, device=dev).to(torch.bfloat16)
    o = torch.full_like(q, CANARY)
    lse = torch.full((B, H, S), CANARY, device=dev)
    ops.check(ops.lib().b200_attn_fwd_dropout(q.data_ptr(), q.data_ptr(), q.data_ptr(), o.data_ptr(), lse.data_ptr(),
                                              None, -1, None, B, S, H, H, D, D ** -0.5, 1, 0.3, 5, ops._stream()),
              "b200_attn_fwd_dropout")
    assert torch.isfinite(o.float()).all() and torch.isfinite(lse).all()
    assert ops.lib().b200_attn_fwd_dropout(q.data_ptr(), q.data_ptr(), q.data_ptr(), o.data_ptr(), lse.data_ptr(),
                                           None, -1, None, B, S, H, H, D, D ** -0.5, 1, 1.0, 5, ops._stream()) != 0


@pytest.mark.parametrize("kind", ["causal", "full", "document", "window", "alibi"])
@pytest.mark.parametrize("D", [64, 128])
def test_bit_identities(kind, D):
    dev = torch.device("cuda")
    B, S, H, Hk = 2, 333, 4, 2
    kw, _ = _family(kind, B, S, H, dev)
    torch.manual_seed(1)
    q = torch.randn(B, S, H, D, device=dev).to(torch.bfloat16)
    k = torch.randn(B, S, Hk, D, device=dev).to(torch.bfloat16)
    v = torch.randn(B, S, Hk, D, device=dev).to(torch.bfloat16)
    g = torch.randn(B, S, H, D, device=dev).to(torch.bfloat16)
    o0, l0 = _raw_fwd(q, k, v, D ** -0.5, kw, None)
    d0 = _raw_bwd(q, k, v, o0, g, l0, D ** -0.5, kw, None)
    o1, l1 = _raw_fwd(q, k, v, D ** -0.5, kw, (0.0, 99))  # the dropout kernels at p = 0
    d1 = _raw_bwd(q, k, v, o1, g, l1, D ** -0.5, kw, (0.0, 99))
    assert torch.equal(o0, o1) and torch.equal(l0, l1)
    assert torch.equal(d0[1], d1[1]) and torch.equal(d0[2], d1[2])
    oa, la = _raw_fwd(q, k, v, D ** -0.5, kw, (0.3, 7))
    assert torch.equal(la, l0)  # the LSE is the dropout-free one at any p
    da = _raw_bwd(q, k, v, oa, g, la, D ** -0.5, kw, (0.3, 7))
    ob, _ = _raw_fwd(q, k, v, D ** -0.5, kw, (0.3, 7))
    db = _raw_bwd(q, k, v, ob, g, la, D ** -0.5, kw, (0.3, 7))
    assert torch.equal(oa, ob) and torch.equal(da[1], db[1]) and torch.equal(da[2], db[2])
    oc, _ = _raw_fwd(q, k, v, D ** -0.5, kw, (0.3, 8))
    assert not torch.equal(oa, oc)


@pytest.mark.parametrize("fp32", [False, True])
def test_autograd_against_fp64(fp32):
    """ops.attention (bf16, D = 64) and ops.attention_fp32 (the bf16x3 path, D = 16) with dropout: outputs and
    gradients against fp64 autograd with the oracle's mask."""
    ops = _ops()
    dev = torch.device("cuda")
    B, S, H, Hk, D = 2, 150, 4, 2, (16 if fp32 else 64)
    p, seed = 0.2, 1234567
    torch.manual_seed(3)
    dt = torch.float32 if fp32 else torch.bfloat16
    q = torch.randn(B, S, H, D, device=dev).to(dt).requires_grad_()
    k = torch.randn(B, S, Hk, D, device=dev).to(dt).requires_grad_()
    v = torch.randn(B, S, Hk, D, device=dev).to(dt).requires_grad_()
    g = torch.randn(B, S, H, D, device=dev).to(dt)
    fn = ops.attention_fp32 if fp32 else ops.attention
    o = fn(q, k, v, D ** -0.5, True, dropout=p, seed=seed)
    o.backward(g)
    from tests import attn_dropout_check as dc
    vis = _vis("causal", {}, B, S, dev)
    ref = dc.reference(q.detach(), k.detach(), v.detach(), o.detach(), g, None, D ** -0.5, vis, seed, p, x3=fp32,
                       kernel_d=64 if fp32 else None)
    for name, got in (("o", o.detach()), ("dq", q.grad), ("dk", k.grad), ("dv", v.grad)):
        dc.check(f"autograd fp32={fp32} {name}", got, *ref[name])


def _fp64_attention(at, base, S_mask_kind="causal"):
    """A drop-in for FlashAttention._flash_attention that runs the fp64 oracle attention with the layer's mask."""
    ops = _ops()

    def run(q, k, v, mask=None, dropout_seed=None, drop=False):
        B, S, H, _ = q.shape
        keep = do.keep_mask(ops.dropout_seed(base, at.layer_idx), at.dropout, B, H, S)
        o, _ = do.attention64(q.double().cpu(), k.double().cpu(), v.double().cpu(), at.scale,
                              _mask_add(S_mask_kind, B, S, H), keep, at.dropout)
        return o.to(q.device, q.dtype)
    return run


@pytest.mark.parametrize("fp32", [True, False])
def test_model_against_fp64_attention(fp32):
    """A tiny GQA model in training mode with dropout (fp32: the C1-style bf16x3 path, head_dim 16; else bf16,
    head_dim 64): loss and every gradient equal the same model whose attention is the fp64 oracle with the product's
    layer seeds ops.dropout_seed(base, i).  no_grad and eval forwards do not drop."""
    from mlx_cuda_distributed_pretraining_b200.arch.llama import Model, ModelArgs
    dev = torch.device("cuda")
    torch.manual_seed(0)
    hd = 16 if fp32 else 64
    args = ModelArgs(model_type="llama", hidden_size=4 * hd, num_hidden_layers=2, intermediate_size=128,
                     num_attention_heads=4, num_key_value_heads=2, head_dim=hd, vocab_size=96,
                     tie_word_embeddings=True, attention_dropout=0.25)
    model = Model(args).to(dev)
    if not fp32:
        model = model.to(torch.bfloat16)
    inputs = torch.randint(0, 96, (2, 40), device=dev)
    base = 0xDEADBEEF

    def loss_and_grads():
        model.zero_grad(set_to_none=True)
        loss = model(inputs, dropout_seed=base).float().logsumexp(-1).mean()
        loss.backward()
        return loss.detach(), [p.grad.detach().clone() for p in model.parameters()]
    model.train()
    l_k, g_k = loss_and_grads()
    for layer in model.layers:
        at = layer.self_attn.attn
        at._flash_attention = _fp64_attention(at, base)
    l_r, g_r = loss_and_grads()
    for layer in model.layers:
        del layer.self_attn.attn._flash_attention
    # this checks the model's plumbing (the layer seeds, which calls drop); the kernels' masks and arithmetic are
    # checked element by element above.  The kernel side rounds P and dS to bf16, also on the bf16x3 path.
    rel = 1e-2 if fp32 else 5e-2
    assert abs(l_k.item() - l_r.item()) <= rel * abs(l_r.item())
    for a, b in zip(g_k, g_r):
        assert (a.float() - b.float()).abs().max().item() <= rel * max(b.float().abs().max().item(), 1e-6)
    with torch.no_grad():
        a = model(inputs, dropout_seed=base)
    model.eval()
    b = model(inputs, dropout_seed=base)
    for layer in model.layers:
        layer.self_attn.attn.dropout = 0.0
    c = model(inputs)
    assert torch.equal(a, b) and torch.equal(b, c)


def test_trainer_run_and_generation(tmp_path):
    """A synthetic run with dropout 0.1: finite, falling loss;
    greedy generation from the run equals generation with p forced to 0."""
    from mlx_cuda_distributed_pretraining_b200.core.generation import generate, load_run
    from mlx_cuda_distributed_pretraining_b200.core.training import Config, Trainer
    from tests.smoke_check import tiny_config
    d = tiny_config(hp__iters=40)
    d["data"]["input_file"] = "synthetic:markov"
    d["name"] = "drop"
    d["model"]["attention"]["dropout"] = 0.1
    d["logging"]["steps"]["logging_interval"] = 1
    tr = Trainer(Config.from_dict(d), synthetic=True, quiet=True, run_root=str(tmp_path))
    assert tr.model.args.attention_dropout == 0.1
    tr.train()
    losses = [float(line.split("loss=")[1].split()[0].rstrip("|"))
              for line in (tmp_path / "drop" / "log.txt").read_text().splitlines() if "loss=" in line]
    assert len(losses) >= 10 and all(np.isfinite(losses))
    assert np.mean(losses[-5:]) < np.mean(losses[:5])
    loaded = load_run("drop", str(tmp_path))
    assert loaded.model.args.attention_dropout == 0.1
    prompts = [[1, 5, 9, 13], [1, 7]]
    out1 = generate(loaded.model, prompts, max_tokens=12, temperature=0.0)
    for layer in loaded.model.layers:
        layer.self_attn.attn.dropout = 0.0
    out0 = generate(loaded.model, prompts, max_tokens=12, temperature=0.0)
    assert out1 == out0


def _masters(tr):
    return {n: t.detach().clone() for n, t in tr.store.named_master().items()}


def test_resume_is_bit_identical(tmp_path):
    """dropout: 0.1, 3 steps, checkpoint, resume for 3 steps: every master weight equals 6 straight steps', since the
    masks depend on (system.seed, rank, step, layer) only.  S = 128 is one key tile per row, so the backward's dQ
    reduction has one term per element and the run is deterministic."""
    from mlx_cuda_distributed_pretraining_b200.core.training import Config, Trainer
    from tests.smoke_check import tiny_config
    d = tiny_config(hp__iters=6)
    d["model"]["attention"]["dropout"] = 0.1
    d["logging"]["steps"]["checkpoint_interval"] = 3
    straight = Trainer(Config.from_dict(d), synthetic=True, quiet=True, run_root=str(tmp_path / "a"))
    straight.train()
    d2 = tiny_config(hp__iters=6)
    d2["model"]["attention"]["dropout"] = 0.1
    d2["resume"] = {"checkpoint": str(tmp_path / "a" / "smoke" / "checkpoints" / "step_3")}
    resumed = Trainer(Config.from_dict(d2), synthetic=True, quiet=True, run_root=str(tmp_path / "b"))
    resumed.train()
    a, b = _masters(straight), _masters(resumed)
    assert set(a) == set(b) and all(torch.equal(a[n], b[n]) for n in a)
    # the masks matter: the same 6 steps without dropout end elsewhere
    d3 = tiny_config(hp__iters=6)
    plain = Trainer(Config.from_dict(d3), synthetic=True, quiet=True, run_root=str(tmp_path / "c"))
    plain.train()
    c = _masters(plain)
    assert any(not torch.equal(a[n], c[n]) for n in a)


def test_validate_does_not_drop(tmp_path):
    """Trainer.validate() of a model with dropout 0.5, in training mode, equals validate() of the same weights with
    every layer's p set to 0."""
    from mlx_cuda_distributed_pretraining_b200.core.training import Config, Trainer
    from tests.smoke_check import tiny_config
    from pathlib import Path
    golden = Path(__file__).resolve().parent / "golden"
    d = tiny_config(hp__iters=2)
    d["data"]["input_file"] = str(golden / "tiny_corpus.jsonl")
    d["data"]["validation_file"] = str(golden / "tiny_val.jsonl")
    d["data"]["tokenizer_path"] = None
    d["model"]["attention"]["dropout"] = 0.5
    tr = Trainer(Config.from_dict(d), quiet=True, run_root=str(tmp_path))
    assert tr.data_manager.has_validation_data
    tr.model.train()
    v1 = tr.validate()
    for layer in tr.model.layers:
        layer.self_attn.attn.dropout = 0.0
    v0 = tr.validate()
    assert v1 == v0


def test_config_off_equals_absent(tmp_path):
    """dropout: 0, dropout: null and no key give identical ModelArgs through the Trainer."""
    from mlx_cuda_distributed_pretraining_b200.core.training import Config, Trainer
    from tests.smoke_check import tiny_config
    args = []
    for i, val in enumerate((0, None, "absent")):
        d = tiny_config(hp__iters=1)
        if val != "absent":
            d["model"]["attention"]["dropout"] = val
        tr = Trainer(Config.from_dict(d), synthetic=True, quiet=True, run_root=str(tmp_path / str(i)))
        args.append(tr.model_args)
    assert args[0] == args[1] == args[2] and args[0].attention_dropout == 0.0
