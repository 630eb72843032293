"""CPU: the attention-backward checker (tests/attn_bwd_check.py) accepts a correct result and rejects planted faults
that a relative Frobenius norm can miss."""
import pytest
import torch

from tests import attn_bwd_check as ac

B, S, H, Hk, D = 1, 300, 4, 2, 64
SCALE = D ** -0.5


@pytest.fixture(scope="module")
def case():
    torch.manual_seed(3)
    q = torch.randn(B, S, H, D).to(torch.bfloat16)
    k = torch.randn(B, S, Hk, D).to(torch.bfloat16)
    v = torch.randn(B, S, Hk, D).to(torch.bfloat16)
    do = torch.randn(B, S, H, D).to(torch.bfloat16)
    o, lse = ac.forward64(q, k, v, SCALE, True)
    ref = ac.reference(q, k, v, o, do, lse, SCALE, True)
    return (q, k, v, o, do, lse), ref


def _bf16(x):
    return x.to(torch.bfloat16)


def _rejects(name, got, ref):
    r, bd = ref[name]
    with pytest.raises(AssertionError):
        ac.check(name, got, r, bd)


def test_accepts_rounded_reference(case):
    _, ref = case
    for name in ("dq", "dk", "dv"):
        r, bd = ref[name]
        assert ac.check(name, _bf16(r), r, bd) <= 1.0


def test_rejects_dropped_key_tile(case):
    _, ref = case
    dk = ref["dk"][0].clone()
    dk[:, 128:256] = 0
    _rejects("dk", _bf16(dk), ref)


def test_rejects_dq_missing_one_key_tile(case):
    """dK and dV right, dQ without the contribution of keys 128..255 (e.g. one pass of a paired CTA never reduced)."""
    t, ref = case
    bad = ac.reference(*t, SCALE, True, drop_keys=slice(128, 256))
    _rejects("dq", _bf16(bad["dq"][0]), ref)


def test_rejects_diagonal_shifted_by_one(case):
    t, ref = case
    bad = ac.reference(*t, SCALE, True, mask_shift=1)
    for name in ("dq", "dk", "dv"):
        _rejects(name, _bf16(bad[name][0]), ref)


def test_rejects_missing_dq_half(case):
    _, ref = case
    dq = ref["dq"][0].clone()
    dq[..., D // 2:] = 0
    _rejects("dq", _bf16(dq), ref)


def test_rejects_scale_applied_twice(case):
    _, ref = case
    for name in ("dq", "dk"):
        _rejects(name, _bf16(ref[name][0] * SCALE), ref)


def test_rejects_wrong_gqa_head(case):
    t, ref = case
    q, k, v, o, do, lse = t
    # query heads 0,1 share kv head 0 and 2,3 kv head 1: a kernel that used kv head 0 for every query head
    k0, v0 = k[:, :, :1].expand(-1, -1, Hk, -1).contiguous(), v[:, :, :1].expand(-1, -1, Hk, -1).contiguous()
    bad = ac.reference(q, k0, v0, o, do, lse, SCALE, True)
    _rejects("dq", _bf16(bad["dq"][0]), ref)
