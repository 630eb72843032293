"""-m gpu: ALiBi attention (b200_attn_fwd_alibi / b200_attn_bwd_alibi, called directly) and the bf16x3 backward of
ops.attention_fp32, compared element by element with the fp64 references of tests/attn_fwd_check.py and
tests/attn_bwd_check.py.  The bias m_h (k - q) is built from its definition at the slopes' fp32 values; the bounds
add |b| to the logit magnitude, which the checkers' docstrings derive.

O and LSE live inside canary-filled buffers, q, k, v and the slopes are the leading part of NaN-filled allocations (a
read of slopes[H] would turn a row into NaN).  The backward gets O and LSE from the biased fp64 forward, so it is
tested alone, writes dk | dv into a [B, S, 2 Hk + 1, D] buffer whose extra head column must keep its canary, and must
repeat dk and dv bit for bit.  tests/test_gpu_alibi.py keeps the model, generation, zero-slope and decode tests; its
Frobenius kernel checks stay as a second opinion through the autograd path (ops.attention), which these tests bypass.
"""
import ctypes
import itertools

import pytest
import torch

from tests import attn_bwd_check as ac
from tests import attn_fwd_check as fc
from tests.test_gpu_attention_fwd import _items_shape, _nan_guarded, _regime
from tests.test_gpu_packed_attention import layouts, positions
from tests.test_gpu_sliding_window import windows

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(600)]

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
        print("\nALiBi / bf16x3 attention, largest |got - ref| / bound: "
              + "; ".join(f"{k} {v:.3g}" for k, v in sorted(RATIOS.items())))


def std_slopes(H):
    from mlx_cuda_distributed_pretraining_b200.arch.flash_attention import alibi_slopes
    return alibi_slopes(H).cuda()


def mixed_slopes(H):
    return torch.tensor([(0.0, 1 / 256, 0.5)[h % 3] for h in range(H)], dtype=torch.float32, device="cuda")


def const_slopes(H, m):
    return torch.full((H,), m, dtype=torch.float32, device="cuda")


def _slopes(kind, H):
    return {"std": std_slopes, "mixed": mixed_slopes}[kind](H) if isinstance(kind, str) else const_slopes(H, kind)


def _note(tag, r):
    RATIOS[tag] = max(RATIOS.get(tag, 0.0), r)


def _bf16(B, S, H, Hk, D, seed):
    torch.manual_seed(seed)
    return tuple(torch.randn(B, S, h, D, device="cuda").to(torch.bfloat16) for h in (H, Hk, Hk))


def _fwd(L, q, k, v, scale, slopes, pos=None, window=None):
    """One raw b200_attn_fwd_alibi launch (window None: -1); returns (o, lse) after checking the canaries."""
    B, S, H, D = q.shape
    Hk = k.shape[2]
    qg, kg, vg, sg = (_nan_guarded(t) for t in (q, k, v, slopes))
    n, nl = q.numel(), B * H * S
    ob = torch.full((O_OFF + n + TAIL,), CANARY, device="cuda", dtype=torch.bfloat16)
    lb = torch.full((L_OFF + nl + TAIL,), CANARY, device="cuda", dtype=torch.float32)
    o, lse = ob[O_OFF:O_OFF + n], lb[L_OFF:L_OFF + nl]
    rc = L.b200_attn_fwd_alibi(qg.data_ptr(), kg.data_ptr(), vg.data_ptr(), o.data_ptr(), lse.data_ptr(),
                               None if pos is None else pos.data_ptr(), -1 if window is None else min(window, S),
                               sg.data_ptr(), B, S, H, Hk, D, ctypes.c_float(scale),
                               torch.cuda.current_stream().cuda_stream)
    assert rc == 0, L.b200_last_error()
    torch.cuda.synchronize()
    for buf, off, m in ((ob, O_OFF, n), (lb, L_OFF, nl)):
        assert bool((buf[:off] == CANARY).all()) and bool((buf[off + m:] == CANARY).all()), "write outside O / LSE"
    return o.view(q.shape).clone(), lse.view(B, H, S).clone()


def _check_fwd(tag, o, lse, q, k, v, scale, mask, slopes, rows=None, **kw):
    ref = fc.reference(q, k, v, scale, mask, rows=rows, slopes=slopes, **kw)
    rows = list(range(q.shape[0])) if rows is None else list(rows)
    for name, got in (("o", o[rows]), ("lse", lse[rows])):
        _note(f"fwd {tag} {name}", fc.check(f"{tag} {name}", got, *ref[name]))


# ---- forward --------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("S,D,heads,kind", list(itertools.product(
    (1, 63, 64, 65, 127, 128, 129, 200, 255, 256, 257, 1000), (64, 128), list(HEADS), ("std", "mixed"))))
def test_alibi_fwd_small(L, S, D, heads, kind):
    H, Hk = HEADS[heads]
    q, k, v = _bf16(2, S, H, Hk, D, seed=S * 31 + D + H + Hk)
    sl = _slopes(kind, H)
    o, lse = _fwd(L, q, k, v, D ** -0.5, sl)
    _check_fwd("rows", o, lse, q, k, v, D ** -0.5, fc.visible(S, device="cuda"), sl)


@pytest.mark.parametrize("S,D", list(itertools.product((257, 1000), (64, 128))))
def test_alibi_fwd_documents(L, S, D):
    pos = torch.stack([positions(lay, S) for lay in layouts(S, seed=D)]).int().cuda()
    q, k, v = _bf16(pos.shape[0], S, 8, 2, D, seed=S + D)
    for kind in ("std", "mixed"):
        sl = _slopes(kind, 8)
        o, lse = _fwd(L, q, k, v, D ** -0.5, sl, pos=pos)
        _check_fwd("document", o, lse, q, k, v, D ** -0.5, fc.visible(S, pos=pos, device="cuda"), sl)


@pytest.mark.parametrize("packed", [False, True], ids=["rows", "packed"])
@pytest.mark.parametrize("D", [64, 128])
def test_alibi_fwd_windows(L, D, packed):
    S = 1000
    pos = torch.stack([positions(lay, S) for lay in layouts(S, seed=D)]).int().cuda() if packed else None
    q, k, v = _bf16(5 if packed else 2, S, 4, 2, D, seed=D + packed)
    sl = mixed_slopes(4)
    for W in windows(S):
        o, lse = _fwd(L, q, k, v, D ** -0.5, sl, pos=pos, window=W)
        _check_fwd("window", o, lse, q, k, v, D ** -0.5, fc.visible(S, pos=pos, window=W, device="cuda"), sl)


@pytest.mark.parametrize("m", [1 / 256, 1 / 64, 0.5])
def test_alibi_fwd_long_rows(L, m):
    """S = 8192: at 1/256 and 1/64 keys thousands back still carry weight; at 0.5 they underflow to an exact 0."""
    S, H, Hk, D = 8192, 2, 1, 64
    q, k, v = _bf16(1, S, H, Hk, D, seed=int(1 / m))
    sl = const_slopes(H, m)
    o, lse = _fwd(L, q, k, v, D ** -0.5, sl)
    _check_fwd("long", o, lse, q, k, v, D ** -0.5, fc.visible(S, device="cuda"), sl, head_chunk=1)


@pytest.mark.parametrize("kind", ["rising", "underflow", "uniform", "large"])
@pytest.mark.parametrize("m", [0.5, 1 / 256], ids=["steep", "gentle"])
def test_alibi_fwd_logit_regimes(L, kind, m):
    S, D = 1000, 64
    q, k, v, scale = _regime(kind, 2, S, 4, 2, D)
    sl = const_slopes(4, m)
    o, lse = _fwd(L, q, k, v, scale, sl)
    _check_fwd("regimes", o, lse, q, k, v, scale, fc.visible(S, device="cuda"), sl)


@pytest.mark.parametrize("B,S,H,Hk,D", [(16, 1024, 16, 8, 64),     # C2 layer
                                        (16, 2048, 16, 8, 64),     # C3 layer micro-batch
                                        (16, 2048, 16, 16, 128)])  # C5 dims
def test_alibi_fwd_layer_shapes(L, B, S, H, Hk, D):
    q, k, v = _bf16(B, S, H, Hk, D, seed=S + D + Hk)
    sl = std_slopes(H)
    o, lse = _fwd(L, q, k, v, D ** -0.5, sl)
    _check_fwd("layer", o, lse, q, k, v, D ** -0.5, fc.visible(S, device="cuda"), sl, rows=(0, B - 1))


@pytest.mark.parametrize("D", [64, 128])
@pytest.mark.parametrize("which", ["1", "N-1", "N", "N+1", "2N+1", "8N"])
def test_alibi_fwd_schedule_sized_work(L, which, D):
    N = torch.cuda.get_device_properties(0).multi_processor_count
    n = {"1": 1, "N-1": N - 1, "N": N, "N+1": N + 1, "2N+1": 2 * N + 1, "8N": 8 * N}[which]
    S, H, Hk, B = _items_shape(n)
    q, k, v = _bf16(B, S, H, Hk, D, seed=n + D)
    sl = mixed_slopes(H)
    o, lse = _fwd(L, q, k, v, D ** -0.5, sl)
    o2, lse2 = _fwd(L, q, k, v, D ** -0.5, sl)
    assert torch.equal(o, o2) and torch.equal(lse, lse2), "a second launch changed the bits"
    for b in range(B):
        ob, lb = _fwd(L, q[b:b + 1], k[b:b + 1], v[b:b + 1], D ** -0.5, sl)
        assert torch.equal(ob[0], o[b]) and torch.equal(lb[0], lse[b]), f"batch row {b} differs alone"
    _check_fwd("schedule", o, lse, q, k, v, D ** -0.5, fc.visible(S, device="cuda"), sl, rows=sorted({0, B - 1}))


# ---- backward -------------------------------------------------------------------------------------------------------
def _bwd(L, q, k, v, o, do, lse, slopes, pos=None, window=None):
    """One raw b200_attn_bwd_alibi launch with dk | dv in a [B, S, 2 Hk + 1, D] NaN buffer; checks the extra head
    column kept its canary and that a second launch repeats dk and dv bit for bit."""
    B, S, H, D = q.shape
    Hk = k.shape[2]
    q, k, v, o, do, lse, sg = (_nan_guarded(t) for t in (q, k, v, o, do, lse, slopes))
    ws = torch.empty(max(int(L.b200_attn_bwd_window_workspace_bytes(B, S, H, Hk, D)), 16), device="cuda",
                     dtype=torch.uint8)
    outs = []
    for _ in range(2):
        dq = torch.empty_like(q)
        buf = torch.full((B, S, 2 * Hk + 1, D), float("nan"), device="cuda", dtype=torch.bfloat16)
        dk, dv = buf[:, :, :Hk], buf[:, :, Hk:2 * Hk]
        rc = L.b200_attn_bwd_alibi(q.data_ptr(), k.data_ptr(), v.data_ptr(), o.data_ptr(), do.data_ptr(),
                                   lse.data_ptr(), None if pos is None else pos.data_ptr(),
                                   -1 if window is None else min(window, S), sg.data_ptr(), dq.data_ptr(),
                                   dk.data_ptr(), dv.data_ptr(), B, S, H, Hk, D, ctypes.c_float(D ** -0.5),
                                   2 * Hk + 1, ws.data_ptr(), ws.numel(), torch.cuda.current_stream().cuda_stream)
        assert rc == 0, L.b200_last_error()
        torch.cuda.synchronize()
        assert torch.isnan(buf[:, :, 2 * Hk:].float()).all(), "write into the extra head column"
        outs.append((dq, dk, dv))
    assert torch.equal(outs[0][1], outs[1][1]) and torch.equal(outs[0][2], outs[1][2]), "dk / dv not repeatable"
    return outs[0]


def _bwd_case(L, tag, B, S, H, Hk, D, slopes, seed, pos=None, window=None, rows=None, head_chunk=None):
    mask = fc.visible(S, pos=pos, window=window, device="cuda")
    q, k, v = _bf16(B, S, H, Hk, D, seed)
    do = torch.randn(B, S, H, D, device="cuda").to(torch.bfloat16)
    o, lse = fc.forward64(q, k, v, D ** -0.5, mask, slopes=slopes, head_chunk=head_chunk or 4)
    o, lse = o.to(torch.bfloat16).contiguous(), lse.float().contiguous()
    got = _bwd(L, q, k, v, o, do, lse, slopes, pos, window)
    rows = list(range(B)) if rows is None else list(rows)
    ref = ac.reference(q, k, v, o, do, lse, D ** -0.5, True, rows=rows, mask=mask, slopes=slopes,
                       head_chunk=head_chunk)
    for name, g in zip(("dq", "dk", "dv"), got):
        _note(f"bwd {tag} {name}", ac.check(f"{tag} {name}", g[rows], *ref[name]))


@pytest.mark.parametrize("S,D,group", list(itertools.product(
    (1, 63, 64, 65, 127, 128, 129, 200, 300, 1000), (64, 128), (1, 2, 4, 8))))
def test_alibi_bwd_small(L, S, D, group):
    Hk = 2
    H = Hk * group
    _bwd_case(L, "rows", 2, S, H, Hk, D, std_slopes(H), seed=S * 17 + D + group)


@pytest.mark.parametrize("S,D,group", list(itertools.product((257, 1000), (64, 128), (1, 8))))
def test_alibi_bwd_documents(L, S, D, group):
    pos = torch.stack([positions(lay, S) for lay in layouts(S, seed=D)]).int().cuda()
    _bwd_case(L, "document", pos.shape[0], S, 2 * group, 2, D, mixed_slopes(2 * group), seed=S + D + group, pos=pos)


@pytest.mark.parametrize("packed", [False, True], ids=["rows", "packed"])
@pytest.mark.parametrize("D", [64, 128])
def test_alibi_bwd_windows(L, D, packed):
    S = 1000
    pos = torch.stack([positions(lay, S) for lay in layouts(S, seed=D)]).int().cuda() if packed else None
    for W in windows(S):
        _bwd_case(L, "window", 5 if packed else 2, S, 4, 2, D, mixed_slopes(4), seed=W + D, pos=pos, window=W)


def test_alibi_bwd_documents_c3_shape(L):
    B, S = 16, 2048
    lay = layouts(S, seed=2)
    pos = torch.stack([positions(lay[b % len(lay)], S) for b in range(B)]).int().cuda()
    _bwd_case(L, "document C3", B, S, 16, 8, 64, std_slopes(16), seed=11, pos=pos, rows=(0, B - 1))


def test_alibi_bwd_long_row(L):
    _bwd_case(L, "long", 1, 8192, 2, 1, 64, const_slopes(2, 1 / 256), seed=13, head_chunk=2)


# ---- the bf16x3 path (ops.attention_fp32) ---------------------------------------------------------------------------
def _fp32_inputs(B, S, H, Hk, D, seed, mul=1.0):
    torch.manual_seed(seed)
    q = (torch.randn(B, S, H, D, device="cuda") * mul).requires_grad_(True)
    k = (torch.randn(B, S, Hk, D, device="cuda") * mul).requires_grad_(True)
    v = torch.randn(B, S, Hk, D, device="cuda").requires_grad_(True)
    do = torch.randn(B, S, H, D, device="cuda")
    return q, k, v, do


@pytest.mark.parametrize("D", [8, 16, 32, 42])
def test_x3_fwd_alibi(L, D):
    from mlx_cuda_distributed_pretraining_b200 import ops
    S, H, Hk = 1000, 4, 2
    q, k, v, _ = (t.detach() for t in _fp32_inputs(2, S, H, Hk, D, seed=D))
    sl = mixed_slopes(H)
    o = ops.attention_fp32(q, k, v, D ** -0.5, alibi=sl)
    q3, k3, v3, _ = ac.x3_operands(q, k, v, q)
    o3, lse = ops.attention_fwd_raw(q3, k3, v3, D ** -0.5, True, None, None, sl)
    assert torch.equal(o, o3[..., :D].float() + o3[..., 2 * D:3 * D].float())
    _check_fwd("bf16x3", o, lse, q, k, v, D ** -0.5, fc.visible(S, device="cuda"), sl, kernel_d=q3.shape[-1],
               x3=True)


X3_MODES = ["plain", "causal", "document", "window", "alibi"]


def _x3_backward(tag, B, S, H, Hk, D, mode, seed, mul=1.0):
    """ops.attention_fp32 forward and backward, then: (1) each three-term kernel output dQ', dK', dV' of a raw launch
    on operands built from the definition against its own bf16 reference (a dropped lo part fails here); (2) the
    autograd gradients equal the parts' sums (dk, dv bit for bit; dq, whose fp32 reduction order is not reproducible,
    far closer than its lo part); (3) the summed gradients against the fp32 fp64 reference in x3 mode."""
    from mlx_cuda_distributed_pretraining_b200 import ops
    causal = mode != "plain"
    pos = torch.stack([positions(lay, S) for lay in layouts(S, seed=D)[:B]]).int().cuda() \
        if mode == "document" else None
    W = 129 if mode == "window" else None
    sl = std_slopes(H) if mode == "alibi" else None
    q, k, v, do = _fp32_inputs(B, S, H, Hk, D, seed, mul)
    scale = D ** -0.5
    o = ops.attention_fp32(q, k, v, scale, causal, pos=pos, window=W, alibi=sl)
    o.backward(do)
    q3, k3, v3, g3 = ac.x3_operands(q.detach(), k.detach(), v.detach(), do)
    o3, lse = ops.attention_fwd_raw(q3, k3, v3, scale, causal, pos, W, sl)
    assert torch.equal(o.detach(), o3[..., :D].float() + o3[..., 2 * D:3 * D].float())
    dq3, dk3, dv3 = ops.attention_bwd_raw(q3, k3, v3, o3, g3, lse, scale, causal, pos, W, sl)
    mask = fc.visible(S, causal, pos=pos, window=W, device="cuda")
    parts = ac.reference(q3, k3, v3, o3, g3, lse, scale, causal, mask=mask, slopes=sl)
    for name, g in (("dq", dq3), ("dk", dk3), ("dv", dv3)):
        _note(f"x3 parts {tag} {name}", ac.check(f"{tag} {name}'", g, *parts[name]))
    assert torch.equal(k.grad, dk3[..., :D].float() + dk3[..., D:2 * D].float())
    assert torch.equal(v.grad, dv3[..., :D].float() + dv3[..., D:2 * D].float())
    lo = dq3[..., 2 * D:3 * D].float()
    assert float((q.grad - dq3[..., :D].float() - lo).norm()) <= 0.25 * float(lo.norm()) + 1e-30
    ref = ac.reference(q.detach(), k.detach(), v.detach(), o.detach(), do, lse, scale, causal, mask=mask, slopes=sl,
                       x3=True, kernel_d=q3.shape[-1])
    for name, g in (("dq", q.grad), ("dk", k.grad), ("dv", v.grad)):
        _note(f"x3 {tag} {name}", ac.check(f"{tag} {name}", g, *ref[name]))


@pytest.mark.parametrize("mode", X3_MODES)
@pytest.mark.parametrize("D", [8, 16, 32, 42])
def test_x3_bwd(L, mode, D):
    _x3_backward(mode, 3 if mode == "document" else 2, 1000, 4, 2, D, mode, seed=D + len(mode))


def test_x3_bwd_c1_shape(L):
    """C1's attention (H 8, D 16, S 1024), ALiBi as `model.attention.alibi` gives it."""
    _x3_backward("C1", 2, 1024, 8, 8, 16, "alibi", seed=1)


@pytest.mark.parametrize("mode", ["causal", "alibi"])
def test_x3_bwd_large_logits(L, mode):
    """|s| ~ 40, as test_gpu_parity's large-logit case: the regime the three-term logits exist for."""
    _x3_backward(f"large {mode}", 2, 256, 8, 4, 16, mode, seed=7, mul=4.0)
