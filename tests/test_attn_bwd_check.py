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


# ---- documents and windows (b200_attn_bwd_doc / _window): the pre-pass's dstart / qt_end and the n_vis search -------
@pytest.fixture(scope="module")
def packed():
    """One packed row of documents [0, 150), [150, 250), [250, 300): key tile 1 (keys 128..255) spans all three."""
    from tests.attn_fwd_check import visible
    torch.manual_seed(8)
    q = torch.randn(B, S, H, D).to(torch.bfloat16)
    k = torch.randn(B, S, Hk, D).to(torch.bfloat16)
    v = torch.randn(B, S, Hk, D).to(torch.bfloat16)
    do = torch.randn(B, S, H, D).to(torch.bfloat16)
    pos = torch.cat([torch.arange(150), torch.arange(100), torch.arange(50)])[None]
    return (q, k, v, do), pos, visible


def _masked_fault(t, good, bad, names=("dq", "dk", "dv")):
    q, k, v, do = t
    o, lse = ac.forward64(q, k, v, SCALE, True, mask=good)
    ref = ac.reference(q, k, v, o, do, lse, SCALE, True, mask=good)
    for name in ("dq", "dk", "dv"):
        assert ac.check(name, _bf16(ref[name][0]), *ref[name]) <= 1.0
    wrong = ac.reference(q, k, v, o, do, lse, SCALE, True, mask=bad)
    for name in names:
        _rejects(name, _bf16(wrong[name][0]), ref)


def test_rejects_n_vis_one_too_large_at_document_boundary(packed):
    """The first query of a document (150) also sees the last key of the one before."""
    t, pos, visible = packed
    good = visible(S, pos=pos)
    bad = good.clone()
    bad[..., 150, 149] = True
    _masked_fault(t, good, bad)


def test_rejects_n_vis_one_too_small_at_document_boundary(packed):
    """The last query of a document (149) misses its own key."""
    t, pos, visible = packed
    good = visible(S, pos=pos)
    bad = good.clone()
    bad[..., 149, 149] = False
    _masked_fault(t, good, bad)


def test_rejects_qt_end_one_query_tile_short(packed):
    """Key tile 1 spans three documents; its last query tile (queries 256..299, which see keys 250..255) skipped."""
    t, pos, visible = packed
    good = visible(S, pos=pos)
    bad = good.clone()
    bad[..., 256:, 128:256] = False
    _masked_fault(t, good, bad)


@pytest.mark.parametrize("shift", [-1, 1])
@pytest.mark.parametrize("with_pos", [False, True])
def test_rejects_window_edge_off_by_one(packed, shift, with_pos):
    t, pos, visible = packed
    pos = pos if with_pos else None
    _masked_fault(t, visible(S, pos=pos, window=40), visible(S, pos=pos, window=40 + shift))


def test_accepts_fp32_rounding_of_a_cancelling_dp():
    """Window 0: every query sees only its own key, so P = 1, O = V and dS = dP - delta = 0 exactly.  With dO nearly
    orthogonal to V, dP itself cancels; a kernel still leaves the fp32 rounding of its D-term sums,
    2^-24 * |dO| . |V| per query, in dS, which the bound must admit."""
    from tests.attn_fwd_check import visible
    torch.manual_seed(12)
    q = torch.randn(B, S, H, D).to(torch.bfloat16)
    k = torch.randn(B, S, Hk, D).to(torch.bfloat16)
    v = torch.randn(B, S, Hk, D).to(torch.bfloat16)
    vq = v.double().repeat_interleave(H // Hk, 2)
    do = torch.randn(B, S, H, D).double()
    do = (do - (do * vq).sum(-1, keepdim=True) / (vq * vq).sum(-1, keepdim=True) * vq).to(torch.bfloat16)
    mask = visible(S, window=0)
    o, lse = ac.forward64(q, k, v, SCALE, True, mask=mask)
    ref = ac.reference(q, k, v, o, do, lse, SCALE, True, mask=mask)
    eps = 2.0 ** -24 * (do.double().abs() * vq.abs()).sum(-1, keepdim=True)      # [B, S, H, 1]
    dq = ref["dq"][0] + SCALE * eps * k.double().repeat_interleave(H // Hk, 2)
    assert ac.check("dq", dq, *ref["dq"]) < 0.1
