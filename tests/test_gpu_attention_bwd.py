"""-m gpu: the attention backward (csrc/attention_bwd.cu) called directly through b200_attn_bwd / _strided, compared
element by element with the fp64 reference of tests/attn_bwd_check.py.

O and LSE come from an fp64 forward (rounded to bf16 / fp32), so the backward is tested alone.  The small-shape
matrix covers single, ragged and exact query / key tiles, every GQA ratio up to 8, both masks, D = 64 and 128, and
odd and even key-tile counts (causal launches with an even count pair key tiles t and n-1-t in one CTA).  The
document and window kernels (b200_attn_bwd_doc / _window) run on the layouts of test_gpu_packed_attention and the
windows of test_gpu_sliding_window, checked with the same reference under the visibility mask of
tests/attn_fwd_check.py.
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


@pytest.fixture(scope="module")
def L():
    from mlx_cuda_distributed_pretraining_b200 import ops
    ops.require_device()
    yield ops.lib()
    if RATIOS:
        print("\nattention backward, largest |got - ref| / bound: "
              + "; ".join(f"{k} {v:.3g}" for k, v in sorted(RATIOS.items())))


def _inputs(B, S, H, Hk, D, causal, seed):
    torch.manual_seed(seed)
    q = torch.randn(B, S, H, D, device="cuda").to(torch.bfloat16)
    k = torch.randn(B, S, Hk, D, device="cuda").to(torch.bfloat16)
    v = torch.randn(B, S, Hk, D, device="cuda").to(torch.bfloat16)
    do = torch.randn(B, S, H, D, device="cuda").to(torch.bfloat16)
    o, lse = ac.forward64(q, k, v, D ** -0.5, causal)
    return q, k, v, o, do, lse


def _run(L, q, k, v, o, do, lse, causal, dk=None, dv=None, row_heads=0):
    B, S, H, D = q.shape
    Hk = k.shape[2]
    dq = torch.empty_like(q)
    if dk is None:
        dk, dv = torch.empty_like(k), torch.empty_like(v)
    ws = torch.empty(max(int(L.b200_attn_bwd_workspace_bytes(B, S, H, Hk, D)), 16), device="cuda", dtype=torch.uint8)
    st = torch.cuda.current_stream().cuda_stream
    args = (q.data_ptr(), k.data_ptr(), v.data_ptr(), o.data_ptr(), do.data_ptr(), lse.data_ptr(), dq.data_ptr(),
            dk.data_ptr(), dv.data_ptr(), B, S, H, Hk, D, ctypes.c_float(D ** -0.5), int(causal))
    if row_heads:
        rc = L.b200_attn_bwd_strided(*args, row_heads, ws.data_ptr(), ws.numel(), st)
    else:
        rc = L.b200_attn_bwd(*args, ws.data_ptr(), ws.numel(), st)
    assert rc == 0, L.b200_last_error()
    torch.cuda.synchronize()
    return dq, dk, dv


def _compare(tag, got, q, k, v, o, do, lse, causal, rows, mask=None):
    ref = ac.reference(q, k, v, o, do, lse, q.shape[-1] ** -0.5, causal, rows=rows, mask=mask)
    for name, g in zip(("dq", "dk", "dv"), got):
        r, bd = ref[name]
        RATIOS[f"{tag} {name}"] = max(RATIOS.get(f"{tag} {name}", 0.0), ac.check(name, g[list(rows)], r, bd))


@pytest.mark.parametrize("S,D,group,causal", list(itertools.product(
    (1, 63, 64, 65, 127, 128, 129, 200, 300, 1000), (64, 128), (1, 2, 4, 8), (True, False))))
def test_attn_bwd_small(L, S, D, group, causal):
    Hk = 2
    B, H = 2, Hk * group
    t = _inputs(B, S, H, Hk, D, causal, seed=S * 17 + D + group)
    got = _run(L, *t, causal)
    _compare(f"D{D}", got, *t, causal, rows=range(B))


@pytest.mark.parametrize("B,S,H,Hk,D", [(16, 1024, 16, 8, 64),     # C2 layer
                                        (16, 2048, 16, 8, 64),     # C3 layer micro-batch
                                        (16, 2048, 16, 16, 128)])  # C5 dims
def test_attn_bwd_layer_shapes(L, B, S, H, Hk, D):
    t = _inputs(B, S, H, Hk, D, True, seed=S + D)
    got = _run(L, *t, True)
    _compare(f"layer D{D}", got, *t, True, rows=(0, B - 1))


@pytest.mark.parametrize("S,D", [(200, 64), (1000, 128)])
def test_attn_bwd_strided_halves_and_canaries(L, S, D):
    """dk | dv as the halves of one [B,S,2Hk+1,D] buffer: each half lands where it should and the extra head column
    of every token row keeps its NaN canary."""
    B, H, Hk = 2, 8, 2
    t = _inputs(B, S, H, Hk, D, True, seed=5)
    buf = torch.full((B, S, 2 * Hk + 1, D), float("nan"), device="cuda", dtype=torch.bfloat16)
    dq, dk, dv = _run(L, *t, True, dk=buf[:, :, :Hk], dv=buf[:, :, Hk:2 * Hk], row_heads=2 * Hk + 1)
    assert torch.isnan(buf[:, :, 2 * Hk:].float()).all()
    dq2, dk2, dv2 = _run(L, *t, True)
    assert torch.equal(buf[:, :, :Hk], dk2) and torch.equal(buf[:, :, Hk:2 * Hk], dv2)
    _compare(f"strided D{D}", (dq, buf[:, :, :Hk], buf[:, :, Hk:2 * Hk]), *t, True, rows=range(B))


@pytest.mark.parametrize("D", [64, 128])
def test_attn_bwd_dk_dv_deterministic(L, D):
    t = _inputs(4, 1024, 16, 8, D, True, seed=9)
    _, dk, dv = _run(L, *t, True)
    for _ in range(2):
        _, dk2, dv2 = _run(L, *t, True)
        assert torch.equal(dk, dk2) and torch.equal(dv, dv2)


# ---- documents and windows: b200_attn_bwd_doc / b200_attn_bwd_window ------------------------------------------------
def _masked_inputs(B, S, H, Hk, D, mask, seed):
    """bf16 q, k, v, dO and the fp64 forward's O / LSE under `mask`, rounded to bf16 / fp32."""
    torch.manual_seed(seed)
    q = torch.randn(B, S, H, D, device="cuda").to(torch.bfloat16)
    k = torch.randn(B, S, Hk, D, device="cuda").to(torch.bfloat16)
    v = torch.randn(B, S, Hk, D, device="cuda").to(torch.bfloat16)
    do = torch.randn(B, S, H, D, device="cuda").to(torch.bfloat16)
    o, lse = fc.forward64(q, k, v, D ** -0.5, mask)
    return q, k, v, o.to(torch.bfloat16).contiguous(), do, lse.float().contiguous()


def _run_masked(L, q, k, v, o, do, lse, pos, window):
    """b200_attn_bwd_doc (window None) or b200_attn_bwd_window."""
    B, S, H, D = q.shape
    Hk = k.shape[2]
    dq, dk, dv = torch.empty_like(q), torch.empty_like(k), torch.empty_like(v)
    ws = torch.empty(max(int(L.b200_attn_bwd_doc_workspace_bytes(B, S, H, Hk, D)), 16), device="cuda",
                     dtype=torch.uint8)
    st = torch.cuda.current_stream().cuda_stream
    ins = (q.data_ptr(), k.data_ptr(), v.data_ptr(), o.data_ptr(), do.data_ptr(), lse.data_ptr())
    outs = (dq.data_ptr(), dk.data_ptr(), dv.data_ptr(), B, S, H, Hk, D, ctypes.c_float(D ** -0.5), 0,
            ws.data_ptr(), ws.numel(), st)
    pp = None if pos is None else pos.data_ptr()
    if window is None:
        rc = L.b200_attn_bwd_doc(*ins, pp, *outs)
    else:
        rc = L.b200_attn_bwd_window(*ins, pp, window, *outs)
    assert rc == 0, L.b200_last_error()
    torch.cuda.synchronize()
    return dq, dk, dv


@pytest.mark.parametrize("S,D,group", list(itertools.product((257, 1000), (64, 128), (1, 2, 8))))
def test_attn_bwd_documents(L, S, D, group):
    pos = torch.stack([positions(lay, S) for lay in layouts(S, seed=D)]).int().cuda()
    B, Hk = pos.shape[0], 2
    mask = fc.visible(S, pos=pos, device="cuda")
    t = _masked_inputs(B, S, Hk * group, Hk, D, mask, seed=S + D + group)
    got = _run_masked(L, *t, pos, None)
    _compare(f"document D{D}", got, *t, True, rows=range(B), mask=mask)


@pytest.mark.parametrize("packed", [False, True], ids=["rows", "packed"])
@pytest.mark.parametrize("D,group", list(itertools.product((64, 128), (1, 2, 8))))
def test_attn_bwd_windows(L, D, group, packed):
    S, Hk = 1000, 2
    pos = torch.stack([positions(lay, S) for lay in layouts(S, seed=D)]).int().cuda() if packed else None
    B = 5 if packed else 2
    for W in windows(S):
        mask = fc.visible(S, pos=pos, window=W, device="cuda")
        t = _masked_inputs(B, S, Hk * group, Hk, D, mask, seed=W + D + group)
        got = _run_masked(L, *t, pos, W)
        _compare(f"window D{D}", got, *t, True, rows=range(B), mask=mask)


def test_attn_bwd_documents_c3_shape(L):
    """A C3 layer micro-batch (B16 S2048 H16/8 D64) of packed rows, the five layouts repeated; rows 0 and 15."""
    B, S, H, Hk, D = 16, 2048, 16, 8, 64
    lay = layouts(S, seed=2)
    pos = torch.stack([positions(lay[b % len(lay)], S) for b in range(B)]).int().cuda()
    mask = fc.visible(S, pos=pos, device="cuda")
    t = _masked_inputs(B, S, H, Hk, D, mask, seed=11)
    got = _run_masked(L, *t, pos, None)
    _compare("document C3", got, *t, True, rows=(0, B - 1), mask=mask)
