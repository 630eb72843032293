"""-m gpu: the attention backward (csrc/attention_bwd.cu) called directly through b200_attn_bwd / _strided, compared
element by element with the fp64 reference of tests/attn_bwd_check.py.

O and LSE come from an fp64 forward (rounded to bf16 / fp32), so the backward is tested alone.  The small-shape
matrix covers single, ragged and exact query / key tiles, every GQA ratio up to 8, both masks, D = 64 and 128, and
odd and even key-tile counts (causal launches with an even count pair key tiles t and n-1-t in one CTA).
"""
import ctypes
import itertools

import pytest
import torch

from tests import attn_bwd_check as ac

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


def _compare(tag, got, q, k, v, o, do, lse, causal, rows):
    ref = ac.reference(q, k, v, o, do, lse, q.shape[-1] ** -0.5, causal, rows=rows)
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
