"""-m gpu: prefix-LM attention (b200_attn_fwd_prefix / b200_attn_bwd_prefix, called directly) element by element
against the fp64 references of tests/attn_fwd_check.py and tests/attn_bwd_check.py, with the prefix mask built from
its definition (query q sees key k iff k <= q or k < clamp(P_b, 0, S)); the bf16x3 path and autograd through
ops.attention / ops.attention_fp32; the model against an fp64 dense-mask model, the prefix's independence from later
tokens, prefill + decode against Model.forward; and the trainer on prompt / completion data and synthetic rows.

O and LSE live inside canary-filled buffers; q, k, v are the leading part of NaN-filled allocations and the prefix
lengths of one filled with 2^30.  The backward writes dk | dv into a [B, S, 2 Hk + 1, D] buffer whose extra head
column must keep its canary, and must repeat dk and dv bit for bit.
"""
import ctypes
import itertools
import tempfile
from pathlib import Path

import numpy as np
import pytest
import torch

from tests import attn_bwd_check as ac
from tests import attn_fwd_check as fc
from tests.test_gpu_attention_fwd import _nan_guarded
from tests.test_gpu_packed_attention import rel

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(900)]

ROOT = Path(__file__).resolve().parents[1]
RATIOS = {}
O_OFF, L_OFF, TAIL = 24, 5, 1000
CANARY = -777.0
HEADS = {"g1": (2, 2), "g2": (4, 2), "g4": (8, 2), "g8": (16, 2), "mqa": (8, 1), "h12": (12, 3)}   # (H, Hk)


@pytest.fixture(scope="module")
def L():
    from mlx_cuda_distributed_pretraining_b200 import ops
    ops.require_device()
    yield ops.lib()
    if RATIOS:
        print("\nprefix-LM attention, largest |got - ref| / bound: "
              + "; ".join(f"{k} {v:.3g}" for k, v in sorted(RATIOS.items())))


def _note(tag, r):
    RATIOS[tag] = max(RATIOS.get(tag, 0.0), r)


def prefix_values(S):
    """Per-row prefix lengths: the tile edges 127 / 128 / 129, the ends 0, 1, S - 1, S, and out-of-range values that
    must act as their clamps (-5 -> 0, S + 7 -> S)."""
    return [0, 1, 127, 128, 129, S - 1, S, -5, S + 7]


def visible(S, prefix, device="cuda"):
    """[B, S, S] boolean prefix-LM mask from its definition, at the clamped prefix lengths."""
    P = prefix.to(device=device, dtype=torch.int64).clamp(0, S)
    s = torch.arange(S, device=device)
    return (s[None, :] <= s[:, None])[None] | (s[None, None, :] < P[:, None, None])


def _bf16(B, S, H, Hk, D, seed):
    torch.manual_seed(seed)
    return tuple(torch.randn(B, S, h, D, device="cuda").to(torch.bfloat16) for h in (H, Hk, Hk))


def _int_guarded(t, extra=4096):
    """t at the front of an allocation whose tail holds 2^30: a read past prefix[B - 1] would open a whole row."""
    buf = torch.full((t.numel() + extra,), 2 ** 30, device="cuda", dtype=t.dtype)
    buf[:t.numel()].copy_(t.reshape(-1))
    return buf[:t.numel()].view(t.shape)


def _fwd(L, q, k, v, scale, prefix):
    B, S, H, D = q.shape
    Hk = k.shape[2]
    qg, kg, vg = (_nan_guarded(t) for t in (q, k, v))
    pg = _int_guarded(prefix)
    n, nl = q.numel(), B * H * S
    ob = torch.full((O_OFF + n + TAIL,), CANARY, device="cuda", dtype=torch.bfloat16)
    lb = torch.full((L_OFF + nl + TAIL,), CANARY, device="cuda", dtype=torch.float32)
    o, lse = ob[O_OFF:O_OFF + n], lb[L_OFF:L_OFF + nl]
    rc = L.b200_attn_fwd_prefix(qg.data_ptr(), kg.data_ptr(), vg.data_ptr(), o.data_ptr(), lse.data_ptr(),
                                pg.data_ptr(), B, S, H, Hk, D, ctypes.c_float(scale),
                                torch.cuda.current_stream().cuda_stream)
    assert rc == 0, L.b200_last_error()
    torch.cuda.synchronize()
    for buf, off, m in ((ob, O_OFF, n), (lb, L_OFF, nl)):
        assert bool((buf[:off] == CANARY).all()) and bool((buf[off + m:] == CANARY).all()), "write outside O / LSE"
    return o.view(q.shape).clone(), lse.view(B, H, S).clone()


def _fwd_causal(L, q, k, v, scale, causal):
    B, S, H, D = q.shape
    o = torch.empty_like(q)
    lse = torch.empty(B, H, S, device="cuda", dtype=torch.float32)
    rc = L.b200_attn_fwd(q.data_ptr(), k.data_ptr(), v.data_ptr(), o.data_ptr(), lse.data_ptr(), B, S, H, k.shape[2],
                         D, ctypes.c_float(scale), int(causal), torch.cuda.current_stream().cuda_stream)
    assert rc == 0, L.b200_last_error()
    torch.cuda.synchronize()
    return o, lse


def _bwd(L, q, k, v, o, do, lse, prefix):
    B, S, H, D = q.shape
    Hk = k.shape[2]
    q, k, v, o, do, lse = (_nan_guarded(t) for t in (q, k, v, o, do, lse))
    pg = _int_guarded(prefix)
    ws = torch.empty(max(int(L.b200_attn_bwd_prefix_workspace_bytes(B, S, H, Hk, D)), 16), device="cuda",
                     dtype=torch.uint8)
    outs = []
    for _ in range(2):
        dq = torch.empty_like(q)
        buf = torch.full((B, S, 2 * Hk + 1, D), float("nan"), device="cuda", dtype=torch.bfloat16)
        dk, dv = buf[:, :, :Hk], buf[:, :, Hk:2 * Hk]
        rc = L.b200_attn_bwd_prefix(q.data_ptr(), k.data_ptr(), v.data_ptr(), o.data_ptr(), do.data_ptr(),
                                    lse.data_ptr(), pg.data_ptr(), dq.data_ptr(), dk.data_ptr(), dv.data_ptr(), B, S,
                                    H, Hk, D, ctypes.c_float(D ** -0.5), 2 * Hk + 1, ws.data_ptr(), ws.numel(),
                                    torch.cuda.current_stream().cuda_stream)
        assert rc == 0, L.b200_last_error()
        torch.cuda.synchronize()
        assert torch.isnan(buf[:, :, 2 * Hk:].float()).all(), "write into the extra head column"
        outs.append((dq, dk, dv))
    assert torch.equal(outs[0][1], outs[1][1]) and torch.equal(outs[0][2], outs[1][2]), "dk / dv not repeatable"
    return outs[0]


def _bwd_causal(L, q, k, v, o, do, lse, causal):
    B, S, H, D = q.shape
    Hk = k.shape[2]
    ws = torch.empty(max(int(L.b200_attn_bwd_workspace_bytes(B, S, H, Hk, D)), 16), device="cuda", dtype=torch.uint8)
    dq = torch.empty_like(q)
    dkv = torch.empty(B, S, 2 * Hk, D, device="cuda", dtype=torch.bfloat16)
    dk, dv = dkv[:, :, :Hk], dkv[:, :, Hk:]
    rc = L.b200_attn_bwd_strided(q.data_ptr(), k.data_ptr(), v.data_ptr(), o.data_ptr(), do.data_ptr(),
                                 lse.data_ptr(), dq.data_ptr(), dk.data_ptr(), dv.data_ptr(), B, S, H, Hk, D,
                                 ctypes.c_float(D ** -0.5), int(causal), 2 * Hk, ws.data_ptr(), ws.numel(),
                                 torch.cuda.current_stream().cuda_stream)
    assert rc == 0, L.b200_last_error()
    torch.cuda.synchronize()
    return dq, dk, dv


def _prefix(vals):
    return torch.tensor(vals, dtype=torch.int32, device="cuda")


def _check_fwd(tag, o, lse, q, k, v, scale, prefix, rows=None, **kw):
    mask = visible(q.shape[1], prefix)
    ref = fc.reference(q, k, v, scale, mask, rows=rows, **kw)
    rows = list(range(q.shape[0])) if rows is None else list(rows)
    for name, got in (("o", o[rows]), ("lse", lse[rows])):
        _note(f"fwd {tag} {name}", fc.check(f"{tag} {name}", got, *ref[name]))


def _bwd_case(L, tag, S, H, Hk, D, prefix, seed, rows=None, head_chunk=None):
    B = prefix.numel()
    mask = visible(S, prefix)
    q, k, v = _bf16(B, S, H, Hk, D, seed)
    do = torch.randn(B, S, H, D, device="cuda").to(torch.bfloat16)
    o, lse = fc.forward64(q, k, v, D ** -0.5, mask, head_chunk=head_chunk or 4)
    o, lse = o.to(torch.bfloat16).contiguous(), lse.float().contiguous()
    got = _bwd(L, q, k, v, o, do, lse, prefix)
    rows = list(range(B)) if rows is None else list(rows)
    ref = ac.reference(q, k, v, o, do, lse, D ** -0.5, False, rows=rows, mask=mask, head_chunk=head_chunk)
    for name, g in zip(("dq", "dk", "dv"), got):
        _note(f"bwd {tag} {name}", ac.check(f"{tag} {name}", g[rows], *ref[name]))


# ---- kernels against fp64 -------------------------------------------------------------------------------------------
@pytest.mark.parametrize("S,D,heads", list(itertools.product((1, 63, 128, 129, 1000), (64, 128), list(HEADS))))
def test_prefix_fwd_small(L, S, D, heads):
    H, Hk = HEADS[heads]
    prefix = _prefix(prefix_values(S))
    q, k, v = _bf16(prefix.numel(), S, H, Hk, D, seed=S * 31 + D + H + Hk)
    o, lse = _fwd(L, q, k, v, D ** -0.5, prefix)
    _check_fwd("rows", o, lse, q, k, v, D ** -0.5, prefix)


@pytest.mark.parametrize("S,D", [(2048, 64), (2048, 128), (8192, 64)])
def test_prefix_fwd_long(L, S, D):
    prefix = _prefix([S // 2, 129, S - 1] if S == 8192 else prefix_values(S))
    H, Hk = (2, 1) if S == 8192 else (4, 2)
    q, k, v = _bf16(prefix.numel(), S, H, Hk, D, seed=S + D)
    o, lse = _fwd(L, q, k, v, D ** -0.5, prefix)
    _check_fwd("long", o, lse, q, k, v, D ** -0.5, prefix, head_chunk=1 if S == 8192 else 4)


@pytest.mark.parametrize("S,D,heads", list(itertools.product((1, 63, 128, 129, 1000), (64, 128), list(HEADS))))
def test_prefix_bwd_small(L, S, D, heads):
    H, Hk = HEADS[heads]
    _bwd_case(L, "rows", S, H, Hk, D, _prefix(prefix_values(S)), seed=S * 17 + D + H)


@pytest.mark.parametrize("S,D", [(2048, 64), (2048, 128), (8192, 64)])
def test_prefix_bwd_long(L, S, D):
    if S == 8192:
        _bwd_case(L, "long", S, 2, 1, D, _prefix([S // 2, S - 1]), seed=S + D, head_chunk=2)
    else:
        _bwd_case(L, "long", S, 4, 2, D, _prefix(prefix_values(S)), seed=S + D)


@pytest.mark.parametrize("S,D", list(itertools.product((1000, 1024), (64, 128))))
def test_prefix_le1_is_the_causal_kernel_bit_for_bit(L, S, D):
    """Every P_b <= 1 (0, 1 and a negative value): O, LSE, dK and dV equal b200_attn_fwd / b200_attn_bwd_strided with
    causal = 1 bit for bit.  S = 1024 has an even key-tile count, where the causal backward runs paired tiles."""
    prefix = _prefix([0, 1, -3])
    q, k, v = _bf16(3, S, 8, 2, D, seed=S + D)
    o, lse = _fwd(L, q, k, v, D ** -0.5, prefix)
    oc, lc = _fwd_causal(L, q, k, v, D ** -0.5, True)
    assert torch.equal(o, oc) and torch.equal(lse, lc)
    do = torch.randn_like(q)
    _, dk, dv = _bwd(L, q, k, v, o, do, lse, prefix)
    _, dkc, dvc = _bwd_causal(L, q, k, v, o, do, lse, True)
    assert torch.equal(dk, dkc) and torch.equal(dv, dvc)


@pytest.mark.parametrize("S,D", list(itertools.product((1000, 1024), (64, 128))))
def test_prefix_full_row_is_the_noncausal_kernel(L, S, D):
    """P_b = S (and S + 7, its clamp) against the causal = 0 launch: the same key tiles in the same order, masked only
    where a tile crosses S, so O, LSE, dK and dV are expected to agree bit for bit."""
    prefix = _prefix([S, S + 7])
    q, k, v = _bf16(2, S, 8, 2, D, seed=S + D + 1)
    o, lse = _fwd(L, q, k, v, D ** -0.5, prefix)
    on, ln = _fwd_causal(L, q, k, v, D ** -0.5, False)
    same_fwd = torch.equal(o, on) and torch.equal(lse, ln)
    do = torch.randn_like(q)
    _, dk, dv = _bwd(L, q, k, v, o, do, lse, prefix)
    _, dkn, dvn = _bwd_causal(L, q, k, v, o, do, lse, False)
    same_bwd = torch.equal(dk, dkn) and torch.equal(dv, dvn)
    print(f"S={S} D={D}: P = S vs causal=0 bit for bit: forward {same_fwd}, backward dK/dV {same_bwd}")
    assert same_fwd and same_bwd


def test_bad_prefix_arguments_are_rejected(L):
    q, k, v = _bf16(2, 64, 4, 2, 64, seed=1)
    o = torch.empty_like(q)
    lse = torch.empty(2, 4, 64, device="cuda")
    rc = L.b200_attn_fwd_prefix(q.data_ptr(), k.data_ptr(), v.data_ptr(), o.data_ptr(), lse.data_ptr(), None, 2, 64,
                                4, 2, 64, ctypes.c_float(0.125), torch.cuda.current_stream().cuda_stream)
    assert rc != 0 and b"prefix" in L.b200_last_error()


# ---- ops: bf16x3 path and autograd ----------------------------------------------------------------------------------
def _dense64(q, k, v, do, prefix, scale):
    H, Hk, S = q.shape[2], k.shape[2], q.shape[1]
    qr, kr, vr = (t.detach().double().requires_grad_(True) for t in (q, k, v))
    kx, vx = (t.repeat_interleave(H // Hk, dim=2) for t in (kr, vr))
    s = torch.einsum("bqhd,bkhd->bhqk", qr, kx) * scale
    s = s.masked_fill(~visible(S, prefix)[:, None], float("-inf"))
    o = torch.einsum("bhqk,bkhd->bqhd", torch.softmax(s, dim=-1), vx)
    o.backward(do.double())
    return o, qr.grad, kr.grad, vr.grad


@pytest.mark.parametrize("path", ["bf16", "fp32"])
def test_ops_attention_prefix_autograd(path):
    from mlx_cuda_distributed_pretraining_b200 import ops
    S, H, Hk = 300, 4, 2
    D = 64 if path == "bf16" else 16
    torch.manual_seed(7)
    dt = torch.bfloat16 if path == "bf16" else torch.float32
    q, k, v = (torch.randn(4, S, h, D, device="cuda").to(dt).requires_grad_(True) for h in (H, Hk, Hk))
    do = torch.randn(4, S, H, D, device="cuda").to(dt)
    prefix = _prefix([0, 37, 128, S])
    fn = ops.attention if path == "bf16" else ops.attention_fp32
    o = fn(q, k, v, prefix=prefix)
    o.backward(do)
    ref = _dense64(q, k, v, do, prefix, D ** -0.5)
    tol = 2e-2 if path == "bf16" else 5e-3   # the bf16x3 path still rounds P and its outputs to bf16 once
    for got, r, nm in zip((o, q.grad, k.grad, v.grad), ref, ("o", "dq", "dk", "dv")):
        e = rel(got, r)
        print(f"{path} {nm}: rel {e:.2e}")
        assert e < tol, (nm, e)


def test_ops_prefix_rejects_combinations():
    from mlx_cuda_distributed_pretraining_b200 import ops
    q, k, v = _bf16(2, 64, 4, 2, 64, seed=2)
    P = _prefix([3, 4])
    pos = torch.zeros(2, 64, dtype=torch.int32, device="cuda")
    slopes = torch.ones(4, device="cuda")
    for kw, word in (({"pos": pos}, "pos"), ({"window": 8}, "window"), ({"alibi": slopes}, "alibi"),
                     ({"causal": False}, "causal")):
        with pytest.raises(ValueError, match=word):
            ops.attention(q, k, v, prefix=P, **kw)
    with pytest.raises(ValueError, match="int32"):
        ops.attention(q, k, v, prefix=P.long())
    with pytest.raises(ValueError, match="prefix"):
        ops.attention(q, k, v, prefix=_prefix([1, 2, 3]))


# ---- model level ----------------------------------------------------------------------------------------------------
def _model(dtype, rope, hidden, layers, heads, kv_heads, head_dim, vocab=259, **kw):
    from mlx_cuda_distributed_pretraining_b200.arch.llama import Model, ModelArgs
    from mlx_cuda_distributed_pretraining_b200.core.training import init_model_
    args = ModelArgs(model_type="llama", hidden_size=hidden, num_hidden_layers=layers, intermediate_size=2 * hidden,
                     num_attention_heads=heads, num_key_value_heads=kv_heads, head_dim=head_dim, vocab_size=vocab,
                     tie_word_embeddings=True, apply_rope=rope, prefix_lm=True, **kw)
    m = Model(args)
    init_model_(m, args, seed=3)
    return m.to("cuda", dtype)


def _dense_attention(self, q, k, v, mask=None):
    """FlashAttention._flash_attention replaced by fp64 softmax(q k^T scale + mask.dense()) v."""
    H, Hk = q.shape[2], k.shape[2]
    kx, vx = (t.double().repeat_interleave(H // Hk, dim=2) for t in (k, v))
    s = torch.einsum("bqhd,bkhd->bhqk", q.double(), kx) * self.scale + mask.dense(torch.float64, q.device)
    return torch.einsum("bhqk,bkhd->bqhd", torch.softmax(s, dim=-1), vx).to(q.dtype)


def _loss_grads_prefix(model, inputs, targets, prefix, pad=256):
    model.zero_grad(set_to_none=True)
    logits = model(inputs, prefix_lens=prefix).float()
    ce = torch.nn.functional.cross_entropy(logits.reshape(-1, logits.shape[-1]), targets.reshape(-1),
                                           reduction="none").view(targets.shape)
    loss = (ce * (targets != pad)).sum()
    loss.backward()
    return float(loss.detach()), {n: p.grad.detach().double().clone() for n, p in model.named_parameters()}


@pytest.mark.parametrize("kind,rope", [("bf16_gqa", False), ("bf16_gqa", True), ("c1_fp32", False), ("mlx_lm", True)])
def test_prefix_model_matches_dense_reference(monkeypatch, kind, rope):
    from mlx_cuda_distributed_pretraining_b200.arch.flash_attention import FlashAttention
    if kind == "bf16_gqa":
        model, tol_loss, tol_grad = _model(torch.bfloat16, rope, 256, 2, 8, 2, 64), 5e-3, 3e-2
    elif kind == "mlx_lm":
        model, tol_loss, tol_grad = _model(torch.bfloat16, rope, 256, 2, 8, 2, 64, variant="mlx_lm"), 5e-3, 3e-2
    else:
        model, tol_loss, tol_grad = _model(torch.float32, rope, 128, 4, 8, 8, 16), 1e-3, 8e-3
    g = torch.Generator().manual_seed(4)
    toks = torch.randint(0, 256, (3, 301), generator=g).cuda()
    inputs, targets = toks[:, :-1], toks[:, 1:]
    prefix = _prefix([0, 150, 300])
    loss_k, g_k = _loss_grads_prefix(model, inputs, targets, prefix)
    monkeypatch.setattr(FlashAttention, "_flash_attention", _dense_attention)
    loss_r, g_r = _loss_grads_prefix(model, inputs, targets, prefix)
    worst = max(rel(g_k[n], g_r[n]) for n in g_r if g_r[n].norm() > 0)
    print(f"{kind} rope={rope}: loss kernel {loss_k:.6f} dense {loss_r:.6f}, worst grad rel {worst:.2e}")
    assert abs(loss_k - loss_r) < tol_loss * abs(loss_r)
    assert worst < tol_grad


def test_prefix_positions_ignore_later_tokens_and_see_later_prefix_tokens():
    model = _model(torch.bfloat16, True, 256, 2, 8, 2, 64)
    P, S = 100, 240
    toks = torch.randint(0, 256, (1, S), generator=torch.Generator().manual_seed(9)).cuda()
    changed_tail = toks.clone()
    changed_tail[0, P:] = (changed_tail[0, P:] + 1) % 256
    changed_prefix = toks.clone()
    changed_prefix[0, P - 1] = (changed_prefix[0, P - 1] + 1) % 256
    pre, causal = _prefix([P]), _prefix([0])
    with torch.no_grad():
        base = model(toks, prefix_lens=pre).float()
        tail = model(changed_tail, prefix_lens=pre).float()
        late = model(changed_prefix, prefix_lens=pre).float()
        base_c = model(toks, prefix_lens=causal).float()
        late_c = model(changed_prefix, prefix_lens=causal).float()
    assert torch.equal(base[:, :P], tail[:, :P]), "a prefix position saw a token at or after P"
    # every position before P - 1 sees the last prefix token: true of the prefix mask only, which the causal
    # control (P = 0, the same inputs) shows
    assert (base[0, :P - 1] - late[0, :P - 1]).abs().amax(-1).min() > 0, "a prefix position missed a later prefix token"
    assert torch.equal(base_c[:, :P - 1], late_c[:, :P - 1]), "the causal control saw a later token"


@pytest.mark.parametrize("kind", ["bf16_gqa", "c1_fp32", "bf16_rope"])
def test_prefix_prefill_decode_match_forward(kind):
    """Ragged prompts in one batch: prefill with P_b = len(prompt_b) and decode steps equal
    Model.forward(prompt + generated, prefix_lens=len(prompt)) at every generated position."""
    from mlx_cuda_distributed_pretraining_b200.arch.llama import KVCache
    from mlx_cuda_distributed_pretraining_b200.core.training import Config, Trainer
    from tests.test_gpu_generation import TOL, _cfg, _rel_rows
    c = _cfg(kind)
    c["model"]["attention"]["prefix_lm"] = True
    tr = Trainer(Config.from_dict(c), for_training=False, synthetic=True, quiet=True,
                 run_root=tempfile.mkdtemp(prefix="prefix_runs_"))
    model = tr.model
    assert model.args.prefix_lm
    lens, T = [150, 97], 200
    tokens = torch.randint(0, 256, (2, T), generator=torch.Generator().manual_seed(5))
    cache = KVCache(model, 2, T)
    prompt = torch.zeros(2, max(lens), dtype=torch.int64)
    for b, n in enumerate(lens):
        prompt[b, :n] = tokens[b, :n]
    first = model.prefill(prompt.cuda(), lens, cache)
    steps = T - max(lens) - 1
    got = [[first[b]] for b in range(2)]
    for t in range(steps):
        nxt = torch.tensor([int(tokens[b, lens[b] + t]) for b in range(2)])
        out = model.decode_step(nxt.cuda(), cache)
        for b in range(2):
            got[b].append(out[b])
    worst = 0.0
    for b, n in enumerate(lens):
        seq = tokens[b:b + 1, :n + steps].cuda()
        with torch.no_grad():
            full = model(seq, prefix_lens=_prefix([n])).float()[0, n - 1:n + steps]
        worst = max(worst, _rel_rows(torch.stack(got[b]), full))
    print(f"{kind}: cached vs forward {worst:.2e}")
    assert worst < TOL[kind]


# ---- trainer --------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kind", ["c1_fp32", "bf16_jsonl", "moe_mlx_lm"])
def test_prefix_trainer_run_reloads_for_generation(tmp_path, kind):
    """C1 on its control stream (fp32, the bf16x3 attention path, random split points), a bf16 run on the
    prompt / completion fixture with validation, and a mixture-of-experts mlx_lm block on synthetic rows: the loss
    stays finite and falls, and the run reloads through the generation path."""
    import yaml
    from mlx_cuda_distributed_pretraining_b200.core.generation import load_run
    from mlx_cuda_distributed_pretraining_b200.core.training import Config, Trainer
    from tests.smoke_check import tiny_config
    if kind == "c1_fp32":
        d = yaml.safe_load((ROOT / "configs" / "c1-llama2m-adamw.yaml").read_text())
        d["data"]["input_file"] = "synthetic:markov"
        d["training"]["hyperparameters"].update(iters=40, learning_rate=1e-3)
        synthetic = True
    else:
        d = tiny_config(hp__iters=60)
        d["data"]["input_file"] = str(ROOT / "tests" / "golden" / "prompt_completion.jsonl")
        d["data"]["validation_file"] = str(ROOT / "tests" / "golden" / "prompt_completion.jsonl")
        d["data"]["tokenizer_path"] = None
        d["logging"]["steps"] = {"logging_interval": 1, "checkpoint_interval": 0, "validation_interval": 20}
        synthetic = False
    if kind == "moe_mlx_lm":
        d = tiny_config(hp__iters=40)
        d["data"]["input_file"] = "synthetic:markov"
        d["model"]["misc"].update(variant="mlx_lm", num_local_experts=4, num_experts_per_tok=2)
        synthetic = True
    d["name"] = "prefix"
    d["model"]["attention"]["prefix_lm"] = True
    d["logging"]["steps"]["logging_interval"] = 1
    d["logging"]["steps"]["checkpoint_interval"] = 0
    d["logging"]["steps"].setdefault("validation_interval", 0)
    tr = Trainer(Config.from_dict(d), synthetic=synthetic, quiet=True, run_root=str(tmp_path))
    assert tr.model.args.prefix_lm
    tr.train()
    run = tmp_path / "prefix"
    losses = [float(line.split("loss=")[1].split()[0].rstrip("|"))
              for line in (run / "log.txt").read_text().splitlines() if "loss=" in line]
    print(f"{kind}: loss {losses[0]:.4f} -> {losses[-1]:.4f}")
    assert len(losses) >= 10 and all(np.isfinite(losses))
    assert np.mean(losses[-5:]) < np.mean(losses[:5])
    loaded = load_run("prefix", str(tmp_path))
    assert loaded.model.args.prefix_lm
