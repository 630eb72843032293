"""-m gpu: the attention forward (attn_fwd_kernel, csrc/attention_fwd.cu) called directly through b200_attn_fwd /
_doc / _window, compared element by element with the fp64 reference of tests/attn_fwd_check.py: O and LSE of every
checked batch row, token and head.

O and LSE live inside canary-filled buffers and q, k, v are the leading part of NaN-filled allocations, so the tests
also show that nothing outside the outputs is written and nothing past the inputs is read.  Families: the plain and
causal matrix over ragged sequence lengths, head dims and GQA ratios; documents and sliding windows; logit regimes
that stress the online softmax; head dims padded by ops.attention (with their backward); the bf16x3 path of
ops.attention_fp32; the C2 / C3 / C5 layer shapes; and work-item counts around the SM count, where each batch row
must be bit-identical alone and inside the batch and a second launch must repeat the bits.
"""
import ctypes
import itertools

import pytest
import torch

from tests import attn_bwd_check as ac
from tests import attn_fwd_check as fc
from tests.test_gpu_packed_attention import layouts, positions
from tests.test_gpu_sliding_window import windows

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(300)]

RATIOS = {}
O_OFF, L_OFF, TAIL = 24, 5, 1000   # O's offset keeps it 16-byte aligned
CANARY = -777.0
HEADS = {"g1": (2, 2), "g2": (4, 2), "g4": (8, 2), "g8": (16, 2), "mqa": (8, 1)}   # (H, Hk)


@pytest.fixture(scope="module")
def L():
    from mlx_cuda_distributed_pretraining_b200 import ops
    ops.require_device()
    yield ops.lib()
    if RATIOS:
        print("\nattention forward, largest |got - ref| / bound: "
              + "; ".join(f"{k} {v:.3g}" for k, v in sorted(RATIOS.items())))


def _nan_guarded(t, extra=4096):
    buf = torch.full((t.numel() + extra,), float("nan"), device="cuda", dtype=t.dtype)
    buf[:t.numel()].copy_(t.reshape(-1))
    return buf[:t.numel()].view(t.shape)


def _fwd(L, q, k, v, scale, causal=True, pos=None, window=None):
    """One raw launch; window / pos select b200_attn_fwd_window / _doc.  Returns (o, lse) after checking the canaries
    around them."""
    B, S, H, D = q.shape
    Hk = k.shape[2]
    qg, kg, vg = (_nan_guarded(t) for t in (q, k, v))
    n, nl = q.numel(), B * H * S
    ob = torch.full((O_OFF + n + TAIL,), CANARY, device="cuda", dtype=torch.bfloat16)
    lb = torch.full((L_OFF + nl + TAIL,), CANARY, device="cuda", dtype=torch.float32)
    o, lse = ob[O_OFF:O_OFF + n], lb[L_OFF:L_OFF + nl]
    head = (qg.data_ptr(), kg.data_ptr(), vg.data_ptr(), o.data_ptr(), lse.data_ptr())
    shape = (B, S, H, Hk, D, ctypes.c_float(scale))
    st = torch.cuda.current_stream().cuda_stream
    pp = None if pos is None else pos.data_ptr()
    if window is not None:
        rc = L.b200_attn_fwd_window(*head, pp, window, *shape, st)
    elif pos is not None:
        rc = L.b200_attn_fwd_doc(*head, pp, *shape, st)
    else:
        rc = L.b200_attn_fwd(*head, *shape, int(causal), st)
    assert rc == 0, L.b200_last_error()
    torch.cuda.synchronize()
    for buf, off, m in ((ob, O_OFF, n), (lb, L_OFF, nl)):
        assert bool((buf[:off] == CANARY).all()) and bool((buf[off + m:] == CANARY).all()), "write outside O / LSE"
    return o.view(q.shape).clone(), lse.view(B, H, S).clone()


def _check(tag, o, lse, q, k, v, scale, mask, rows=None, **kw):
    ref = fc.reference(q, k, v, scale, mask, rows=rows, **kw)
    rows = list(range(q.shape[0])) if rows is None else list(rows)
    for name, got in (("o", o[rows]), ("lse", lse[rows])):
        r = fc.check(f"{tag} {name}", got, *ref[name])
        RATIOS[f"{tag} {name}"] = max(RATIOS.get(f"{tag} {name}", 0.0), r)


def _bf16(B, S, H, Hk, D, seed, scale=1.0):
    torch.manual_seed(seed)
    return tuple((torch.randn(B, S, h, D, device="cuda") * scale).to(torch.bfloat16) for h in (H, Hk, Hk))


# ---- plain and causal -----------------------------------------------------------------------------------------------
@pytest.mark.parametrize("S,D,heads,causal", list(itertools.product(
    (1, 63, 64, 65, 127, 128, 129, 200, 255, 256, 257, 1000), (64, 128), list(HEADS), (True, False))))
def test_fwd_small(L, S, D, heads, causal):
    H, Hk = HEADS[heads]
    q, k, v = _bf16(2, S, H, Hk, D, seed=S * 31 + D + H + Hk)
    o, lse = _fwd(L, q, k, v, D ** -0.5, causal)
    _check("causal" if causal else "plain", o, lse, q, k, v, D ** -0.5, fc.visible(S, causal, device="cuda"))


# ---- documents and windows ------------------------------------------------------------------------------------------
@pytest.mark.parametrize("S,D", list(itertools.product((257, 1000), (64, 128))))
def test_fwd_documents(L, S, D):
    """Every batch row a layout of test_gpu_packed_attention: boundaries at tile offsets, 1-3 token documents,
    length-1 documents, a trailing PAD run, a log-normal mix."""
    pos = torch.stack([positions(lay, S) for lay in layouts(S, seed=D)]).int().cuda()
    q, k, v = _bf16(pos.shape[0], S, 4, 2, D, seed=S + D)
    o, lse = _fwd(L, q, k, v, D ** -0.5, pos=pos)
    _check("document", o, lse, q, k, v, D ** -0.5, fc.visible(S, pos=pos, device="cuda"))


@pytest.mark.parametrize("packed", [False, True], ids=["rows", "packed"])
@pytest.mark.parametrize("D", [64, 128])
def test_fwd_windows(L, D, packed):
    S = 1000
    pos = torch.stack([positions(lay, S) for lay in layouts(S, seed=D)]).int().cuda() if packed else None
    q, k, v = _bf16(5 if packed else 2, S, 4, 2, D, seed=D + packed)
    for W in windows(S):
        o, lse = _fwd(L, q, k, v, D ** -0.5, pos=pos, window=W)
        _check("window", o, lse, q, k, v, D ** -0.5, fc.visible(S, pos=pos, window=W, device="cuda"))


# ---- logit regimes --------------------------------------------------------------------------------------------------
def _regime(kind, B, S, H, Hk, D):
    torch.manual_seed(D + len(kind))
    q = torch.randn(B, S, H, D, device="cuda") * 0.1
    k = torch.randn(B, S, Hk, D, device="cuda") * 0.1
    v = torch.randn(B, S, Hk, D, device="cuda")
    scale = D ** -0.5
    if kind == "rising":        # the row maximum grows in every key tile: every tile rescales
        q[..., 0] = 8.0
        k[..., 0] = torch.linspace(-2.0, 2.0, S, device="cuda")[None, :, None] * D ** 0.5
    elif kind == "underflow":   # the maximum in key tile 0; the logits of later tiles underflow exp2 to exactly 0
        q[..., 0] = 4.0
        k[..., 0] = -60.0
        k[:, :128, :, 0] = 30.0
        scale = 1.0
    elif kind == "uniform":     # q = 0: P uniform over the visible keys, O their mean
        q.zero_()
    elif kind == "large":       # scale 1, |s| ~ 50
        q = torch.randn(B, S, H, D, device="cuda") * (50.0 / D ** 0.5) ** 0.5
        k = torch.randn(B, S, Hk, D, device="cuda") * (50.0 / D ** 0.5) ** 0.5
        scale = 1.0
    return q.to(torch.bfloat16), k.to(torch.bfloat16), v.to(torch.bfloat16), scale


@pytest.mark.parametrize("kind", ["rising", "underflow", "uniform", "large"])
@pytest.mark.parametrize("causal", [True, False])
@pytest.mark.parametrize("D", [64, 128])
def test_fwd_logit_regimes(L, kind, causal, D):
    S = 1000
    q, k, v, scale = _regime(kind, 2, S, 4, 2, D)
    o, lse = _fwd(L, q, k, v, scale, causal)
    _check("regimes", o, lse, q, k, v, scale, fc.visible(S, causal, device="cuda"))
    if kind == "uniform":   # every p is exactly 1 before normalising: O is the fp32 mean of the visible V, rounded
        vd = v.double()
        n = torch.arange(1, S + 1, device="cuda", dtype=torch.float64)[:, None, None]
        mean = (vd.cumsum(1) / n if causal else vd.mean(1, keepdim=True)).repeat_interleave(2, 2)
        assert bool(((o.double() - mean).abs() <= 2 ** -8 * mean.abs() + 2 ** -16).all())


# ---- head dims padded by ops.attention, forward and backward --------------------------------------------------------
@pytest.mark.parametrize("causal", [True, False])
@pytest.mark.parametrize("D", [16, 32, 40, 80, 96])
def test_padded_head_dims(L, D, causal):
    from mlx_cuda_distributed_pretraining_b200 import ops
    B, S, H, Hk = 2, 300, 4, 2
    Dp = 64 if D <= 64 else 128
    q, k, v = (t.requires_grad_(True) for t in _bf16(B, S, H, Hk, D, seed=D + causal))
    do = torch.randn(B, S, H, D, device="cuda").to(torch.bfloat16)
    scale = D ** -0.5
    o = ops.attention(q, k, v, scale, causal)
    o.backward(do)
    pad = [torch.nn.functional.pad(t.detach(), (0, Dp - D)).contiguous() for t in (q, k, v)]
    o_p, lse = ops.attention_fwd_raw(*pad, scale, causal)
    assert torch.equal(o_p[..., :D], o.detach()) and not o_p[..., D:].any()
    _check("padded D", o.detach(), lse, q.detach(), k.detach(), v.detach(), scale,
           fc.visible(S, causal, device="cuda"), kernel_d=Dp)
    ref = ac.reference(q.detach(), k.detach(), v.detach(), o.detach(), do, lse, scale, causal)
    for name, g in (("dq", q.grad), ("dk", k.grad), ("dv", v.grad)):
        r = ac.check(name, g, *ref[name])
        RATIOS[f"padded D {name}"] = max(RATIOS.get(f"padded D {name}", 0.0), r)


# ---- the bf16x3 path (ops.attention_fp32) ---------------------------------------------------------------------------
@pytest.mark.parametrize("mode", ["plain", "causal", "document", "large"])
@pytest.mark.parametrize("D", [16, 40])
def test_fp32_path(L, mode, D):
    from mlx_cuda_distributed_pretraining_b200 import ops
    S, H, Hk = (256, 8, 4) if mode == "large" else (1000, 4, 2)
    pos = torch.stack([positions(lay, S) for lay in layouts(S, seed=D)[:3]]).int().cuda() \
        if mode == "document" else None
    B = 3 if pos is not None else 2
    torch.manual_seed(D + len(mode))
    mul = 4.0 if mode == "large" else 1.0     # |s| ~ 40, as in test_gpu_parity's large-logit case
    q = torch.randn(B, S, H, D, device="cuda") * mul
    k = torch.randn(B, S, Hk, D, device="cuda") * mul
    v = torch.randn(B, S, Hk, D, device="cuda")
    causal = mode != "plain"
    scale = D ** -0.5
    o = ops.attention_fp32(q, k, v, scale, causal, pos=pos)
    # LSE of the same launch: the three-term operands of ops._AttentionX3Fn
    Dp = 64 if 3 * D <= 64 else 128
    (qh, ql), (kh, kl), (vh, vl) = ops._hi_lo(q), ops._hi_lo(k), ops._hi_lo(v)
    cat3 = lambda a, b, c: torch.nn.functional.pad(torch.cat([a, b, c], -1), (0, Dp - 3 * D)).contiguous()  # noqa
    o3, lse = ops.attention_fwd_raw(cat3(qh, ql, qh), cat3(kh, kh, kl), cat3(vh, vh, vl), scale, causal, pos)
    assert torch.equal(o, o3[..., :D].float() + o3[..., 2 * D:3 * D].float())
    _check("bf16x3", o, lse, q, k, v, scale, fc.visible(S, causal, pos=pos, device="cuda"), kernel_d=Dp, x3=True)


# ---- layer shapes ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("B,S,H,Hk,D", [(16, 1024, 16, 8, 64),     # C2 layer
                                        (16, 2048, 16, 8, 64),     # C3 layer micro-batch
                                        (16, 2048, 16, 16, 128)])  # C5 dims
def test_fwd_layer_shapes(L, B, S, H, Hk, D):
    q, k, v = _bf16(B, S, H, Hk, D, seed=S + D + Hk)
    o, lse = _fwd(L, q, k, v, D ** -0.5, True)
    _check("layer", o, lse, q, k, v, D ** -0.5, fc.visible(S, device="cuda"), rows=(0, B - 1))


# ---- work-item counts around the SM count ---------------------------------------------------------------------------
def _items_shape(n):
    """(S, H, Hk, B) with n = (128-query tiles) x H x B work items."""
    if n % 4 == 0:
        return 200, 2, 1, n // 4
    if n % 2 == 0:
        return 256, 1, 1, n // 2
    return 100, 1, 1, n


@pytest.mark.parametrize("D", [64, 128])
@pytest.mark.parametrize("which", ["1", "N-1", "N", "N+1", "2N+1", "8N"])
def test_fwd_schedule_sized_work(L, which, D):
    N = torch.cuda.get_device_properties(0).multi_processor_count
    n = {"1": 1, "N-1": N - 1, "N": N, "N+1": N + 1, "2N+1": 2 * N + 1, "8N": 8 * N}[which]
    S, H, Hk, B = _items_shape(n)
    assert -(-S // 128) * H * B == n
    q, k, v = _bf16(B, S, H, Hk, D, seed=n + D)
    o, lse = _fwd(L, q, k, v, D ** -0.5, True)
    o2, lse2 = _fwd(L, q, k, v, D ** -0.5, True)
    assert torch.equal(o, o2) and torch.equal(lse, lse2), "a second launch changed the bits"
    for b in range(B):
        ob, lb = _fwd(L, q[b:b + 1], k[b:b + 1], v[b:b + 1], D ** -0.5, True)
        assert torch.equal(ob[0], o[b]) and torch.equal(lb[0], lse[b]), f"batch row {b} differs alone"
    _check("schedule", o, lse, q, k, v, D ** -0.5, fc.visible(S, device="cuda"), rows=sorted({0, B - 1}))
