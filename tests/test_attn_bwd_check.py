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


# ---- ALiBi (b200_attn_bwd_alibi): O and LSE from the biased fp64 forward --------------------------------------------
SLOPES = {"steep": 0.5, "gentle": 1 / 256}
HA, HkA = 8, 2


def _alibi(kind):
    if kind == "mixed":
        return torch.tensor([(0.0, 1 / 256, 0.5)[h % 3] for h in range(HA)], dtype=torch.float32)
    return torch.full((HA,), SLOPES[kind], dtype=torch.float32)


@pytest.fixture(scope="module")
def alibi_inputs():
    torch.manual_seed(31)
    q = torch.randn(B, S, HA, D).to(torch.bfloat16)
    k = torch.randn(B, S, HkA, D).to(torch.bfloat16)
    v = torch.randn(B, S, HkA, D).to(torch.bfloat16)
    do = torch.randn(B, S, HA, D).to(torch.bfloat16)
    return q, k, v, do


def _alibi_case(t, kind):
    q, k, v, do = t
    sl = _alibi(kind)
    o, lse = ac.forward64(q, k, v, SCALE, True, slopes=sl)
    return (q, k, v, o, do, lse), sl


@pytest.mark.parametrize("kind", ["steep", "gentle", "mixed"])
def test_alibi_accepts_rounded_reference_and_chunks_agree(alibi_inputs, kind):
    t, sl = _alibi_case(alibi_inputs, kind)
    ref = ac.reference(*t, SCALE, True, slopes=sl)
    chunked = ac.reference(*t, SCALE, True, slopes=sl, head_chunk=4)
    for name in ("dq", "dk", "dv"):
        r, bd = ref[name]
        assert ac.check(name, _bf16(r), r, bd) <= 1.0
        assert torch.allclose(chunked[name][0], r, rtol=1e-12, atol=1e-14)
        assert torch.allclose(chunked[name][1], bd, rtol=1e-12, atol=1e-20)


def _p_bias(sl, fault):
    """The bias the faulty kernel would put into P: unmasked: missing on the items that skip the mask (the 64-key
    warpgroup's last key at or before the item's first query); key_base: keys 8..15 of every 16 with the base of the
    key 8 before (b - 8 m)."""
    pos = torch.arange(S)

    def f(h0, h1):
        from tests.attn_fwd_check import alibi_bias
        b = alibi_bias(sl, S, h0, h1)
        if fault == "unmasked":
            unmasked = (pos // 64 * 64 + 63)[None, :] <= (pos // 64 * 64)[:, None]   # [query, key]
            b = b.masked_fill(unmasked[None], 0.0)
        elif fault == "key_base":
            b = b - 8 * sl[h0:h1].double()[:, None, None] * ((pos % 16) >= 8)[None, None, :]
        return b
    return f


@pytest.mark.parametrize("fault", ["unmasked", "key_base"])
def test_alibi_rejects_bias_fault(alibi_inputs, fault):
    """Gentle slope (1/256).  Records that the relative Frobenius check of tests/test_gpu_alibi.py (< 1e-2) also
    notices both at this shape (errors 0.23-0.28 and 0.017-0.019): here the element check adds the named element."""
    t, sl = _alibi_case(alibi_inputs, "gentle")
    ref = ac.reference(*t, SCALE, True, slopes=sl)
    bad = ac.reference(*t, SCALE, True, slopes=sl, bias=_p_bias(sl, fault))
    frob = {}
    for name in ("dq", "dk", "dv"):
        _rejects(name, _bf16(bad[name][0]), ref)
        r = ref[name][0]
        frob[name] = float((bad[name][0] - r).norm() / r.norm())
    passes = {n for n, e in frob.items() if e < 1e-2}
    assert passes == set(), frob


def test_alibi_rejects_group_first_slope(alibi_inputs):
    """Every query head of a GQA group given the group's first head's slope (slopes[hk * group]), alibi_slopes(8)."""
    from mlx_cuda_distributed_pretraining_b200.arch.flash_attention import alibi_slopes
    from tests.attn_fwd_check import alibi_bias
    q, k, v, do = alibi_inputs
    sl = alibi_slopes(HA)
    o, lse = ac.forward64(q, k, v, SCALE, True, slopes=sl)
    ref = ac.reference(q, k, v, o, do, lse, SCALE, True, slopes=sl)
    g = HA // HkA
    wrong = sl[torch.arange(HA) // g * g]
    bad = ac.reference(q, k, v, o, do, lse, SCALE, True, slopes=sl, bias=lambda h0, h1: alibi_bias(wrong, S, h0, h1))
    for name in ("dq", "dk", "dv"):
        _rejects(name, _bf16(bad[name][0]), ref)


# ---- the bf16x3 backward (ops.attention_fp32) -----------------------------------------------------------------------
D3 = 16


def _x3_case(mul, seed, mask=None, slopes=None):
    """fp32 inputs; the kernel's forward emulated in fp64 on the three-term operands: O' rounded to bf16 part by part,
    LSE of Q'K'^T.  Returns fp32 (q, k, v, do), the x3 operands with O', LSE, and the fp32 o."""
    torch.manual_seed(seed)
    q = torch.randn(B, S, HA, D3) * mul
    k = torch.randn(B, S, HkA, D3) * mul
    v = torch.randn(B, S, HkA, D3)
    do = torch.randn(B, S, HA, D3)
    q3, k3, v3, g3 = ac.x3_operands(q, k, v, do)
    o3, lse = ac.forward64(q3, k3, v3, D3 ** -0.5, True, mask=mask, slopes=slopes)
    o = o3[..., :D3].float() + o3[..., 2 * D3:3 * D3].float()
    return (q, k, v, do), (q3, k3, v3, o3, g3, lse), o


def _x3_emulated(parts, mask=None, slopes=None):
    """The kernel's three-term gradients: the bf16 reference on the x3 operands, each part rounded to bf16, summed in
    fp32 as _AttentionX3Fn sums them."""
    r = ac.reference(*parts, D3 ** -0.5, True, mask=mask, slopes=slopes)
    dq3, dk3, dv3 = (_bf16(r[n][0]).float() for n in ("dq", "dk", "dv"))
    return {"dq": dq3[..., :D3] + dq3[..., 2 * D3:3 * D3], "dk": dk3[..., :D3] + dk3[..., D3:2 * D3],
            "dv": dv3[..., :D3] + dv3[..., D3:2 * D3]}, r


@pytest.mark.parametrize("kind", ["plain", "alibi", "window0"])
def test_x3_accepts_emulated_backward(kind):
    from tests.attn_fwd_check import visible
    mask = visible(S, window=0) if kind == "window0" else None
    sl = _alibi("mixed") if kind == "alibi" else None
    (q, k, v, do), parts, o = _x3_case(1.0, 41, mask, sl)
    got, _ = _x3_emulated(parts, mask, sl)
    ref = ac.reference(q, k, v, o, do, parts[5], D3 ** -0.5, True, mask=mask, slopes=sl, x3=True, kernel_d=64)
    for name in ("dq", "dk", "dv"):
        assert ac.check(name, got[name], *ref[name]) < 0.5


def test_x3_bound_rejects_hi_only_logits_at_large_logits():
    """|s| ~ 40: the plain bf16 backward (logits of the hi halves, bf16 inputs) misses by 2^-9 |s| in the exponent,
    outside the x3 bound; the x3 emulation stays inside it."""
    (q, k, v, do), parts, o = _x3_case(4.0, 42)
    ref = ac.reference(q, k, v, o, do, parts[5], D3 ** -0.5, True, x3=True, kernel_d=64)
    got, _ = _x3_emulated(parts)
    for name in ("dq", "dk", "dv"):
        assert ac.check(name, got[name], *ref[name]) <= 1.0
    qh, kh, vh, gh = (t.to(torch.bfloat16) for t in (q, k, v, do))
    oh, lh = ac.forward64(qh, kh, vh, D3 ** -0.5, True)
    plain = ac.reference(qh, kh, vh, oh, gh, lh, D3 ** -0.5, True)
    rejected = 0
    for name in ("dq", "dk", "dv"):
        try:
            ac.check(name, _bf16(plain[name][0]), *ref[name])
        except AssertionError:
            rejected += 1
    assert rejected >= 2


@pytest.mark.parametrize("fault", ["dq_without_dS_kl", "dv_without_PT_gl", "delta_without_P_vl"])
def test_x3_layout_faults_are_rejected_part_by_part(fault):
    """Each fault drops one lo part.  Against the summed gradient it is at most 2^-9 of the bound's P / dS rounding
    term (module docstring), so it is checked where it lives: the part's own bf16 reference on the x3 operands.
    delta_without_P_vl (O' saved with its P vl third zeroed) shows where dP - delta cancels: window 0, dS = 0."""
    from tests.attn_fwd_check import visible
    mask = visible(S, window=0) if fault == "delta_without_P_vl" else None
    _, parts, _ = _x3_case(1.0, 43, mask)
    ref = ac.reference(*parts, D3 ** -0.5, True, mask=mask)
    dq3, dk3, dv3 = (_bf16(ref[n][0]) for n in ("dq", "dk", "dv"))
    if fault == "dq_without_dS_kl":
        dq3[..., 2 * D3:3 * D3] = 0
        _rejects("dq", dq3, ref)
    elif fault == "dv_without_PT_gl":
        dv3[..., D3:2 * D3] = 0
        _rejects("dv", dv3, ref)
    else:
        q3, k3, v3, o3, g3, lse = parts
        o3b = o3.clone()
        o3b[..., 2 * D3:3 * D3] = 0
        bad = ac.reference(q3, k3, v3, o3b, g3, lse, D3 ** -0.5, True, mask=mask)
        _rejects("dq", _bf16(bad["dq"][0]), ref)
        _rejects("dk", _bf16(bad["dk"][0]), ref)


def test_alibi_reference_stays_finite_where_the_future_bias_overflows():
    """m (k - q) on a masked future key reaches 0.5 * 1499 > 709, where exp overflows fp64: the reference masks
    before exp, and check() fails a NaN reference instead of passing it."""
    S_ = 1500
    torch.manual_seed(44)
    q, k, v, do = (torch.randn(1, S_, 1, D).to(torch.bfloat16) for _ in range(4))
    sl = torch.full((1,), 0.5)
    o, lse = ac.forward64(q, k, v, SCALE, True, slopes=sl)
    ref = ac.reference(q, k, v, o, do, lse, SCALE, True, slopes=sl)
    for name in ("dq", "dk", "dv"):
        r, bd = ref[name]
        assert torch.isfinite(r).all() and torch.isfinite(bd).all()
        assert ac.check(name, _bf16(r), r, bd) <= 1.0
        with pytest.raises(AssertionError):
            ac.check(name, _bf16(r), r * float("nan"), bd)
