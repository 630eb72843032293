"""CPU: the attention-forward checker (tests/attn_fwd_check.py) accepts the right answer, and an emulation of the
kernel's own arithmetic with margin, and rejects faults confined to one CTA that the relative Frobenius check of
tests/test_gpu_parity.py (< 1e-2 on a whole batch row) lets through.  Also: its mask builder is the product's mask."""
import pytest
import torch

from tests import attn_fwd_check as fc
from tests.test_gpu_packed_attention import layouts, positions
from tests.test_gpu_sliding_window import windows

# one batch row at the C3 layer shape; faults go into the CTA (128-query tile QT, head HF)
B, S, H, Hk, D = 1, 2048, 16, 8, 64
SCALE = D ** -0.5
QT, HF = 8, 3
Q0, Q1 = QT * 128, QT * 128 + 128


def _frob(got, ref):
    return float((got.double() - ref).norm() / ref.norm())


@pytest.fixture(scope="module")
def case():
    torch.manual_seed(1)
    q = torch.randn(B, S, H, D).to(torch.bfloat16)
    k = torch.randn(B, S, Hk, D).to(torch.bfloat16)
    v = torch.randn(B, S, Hk, D).to(torch.bfloat16)
    mask = fc.visible(S)
    return (q, k, v), mask, fc.reference(q, k, v, SCALE, mask)


def _head(q, k, v, h, kv=None):
    kv = h // (H // Hk) if kv is None else kv
    return q[:, :, h:h + 1], k[:, :, kv:kv + 1], v[:, :, kv:kv + 1]


def _cta_fault(ref, o_h=None, lse_h=None):
    """The reference with the CTA (QT, HF) replaced by a faulty head-HF result [1, S, 1, D] / [1, 1, S]."""
    o, lse = ref["o"][0].clone(), ref["lse"][0].clone()
    if o_h is not None:
        o[:, Q0:Q1, HF] = o_h[:, Q0:Q1, 0]
    if lse_h is not None:
        lse[:, HF, Q0:Q1] = lse_h[:, 0, Q0:Q1]
    return o, lse


def _rejects(name, got, ref):
    r, bd = ref[name]
    with pytest.raises(AssertionError, match=name):
        fc.check(name, got, r, bd)


# ---- acceptance ----------------------------------------------------------------------------------------------------
def test_accepts_rounded_reference(case):
    _, _, ref = case
    r, bd = ref["o"]
    assert fc.check("o", r.to(torch.bfloat16), r, bd) < 0.5
    r, bd = ref["lse"]
    assert fc.check("lse", r.float(), r, bd) < 0.5


def test_accepts_kernel_emulation_with_margin(case):
    """Tiled online softmax, bf16 P, fp32 accumulators: a different reduction order from the fp64 reference must
    still sit well inside the bound, or a legitimate rewrite of the kernel would fail it."""
    t, mask, ref = case
    o, lse = fc.emulate_kernel(*t, SCALE, mask)
    assert fc.check("o", o, *ref["o"]) < 0.5
    assert fc.check("lse", lse, *ref["lse"]) < 0.5


@pytest.mark.parametrize("window", [None, 0, 100, 129])
def test_accepts_kernel_emulation_documents_and_windows(window):
    """Rows whose first visible key lies tiles above the first key tile (documents beginning mid-row, windows).
    Rows that see one to three keys carry the bf16 roundings of P and of O unaveraged, each up to its own 2^-8 term
    of the bound, so the ratio here may exceed 0.5; it cannot exceed 1 through those roundings, and fp32 reduction
    order only moves the C32 term."""
    S_, H_, Hk_ = 700, 4, 2
    torch.manual_seed(4)
    q = torch.randn(2, S_, H_, D).to(torch.bfloat16)
    k = torch.randn(2, S_, Hk_, D).to(torch.bfloat16)
    v = torch.randn(2, S_, Hk_, D).to(torch.bfloat16)
    pos = torch.stack([positions(lay, S_) for lay in layouts(S_)[:2]])
    mask = fc.visible(S_, pos=pos, window=window)
    ref = fc.reference(q, k, v, SCALE, mask)
    o, lse = fc.emulate_kernel(q, k, v, SCALE, mask)
    assert fc.check("o", o, *ref["o"]) < 0.75
    assert fc.check("lse", lse, *ref["lse"]) < 0.5


# ---- the faults of one CTA that the Frobenius check passes ----------------------------------------------------------
def test_rejects_skipped_diagonal_key_tile(case):
    t, mask, ref = case
    bad = mask.clone()
    bad[Q0:Q1, Q0:Q1] = False
    o, _ = _cta_fault(ref, *fc.forward64(*_head(*t, HF), SCALE, bad))
    assert _frob(o, ref["o"][0]) < 1e-2
    _rejects("o", o.to(torch.bfloat16), ref)


def test_rejects_first_key_of_every_tile_dropped(case):
    t, mask, ref = case
    bad = mask.clone()
    bad[Q0:Q1, ::128] = False
    o, _ = _cta_fault(ref, *fc.forward64(*_head(*t, HF), SCALE, bad))
    assert _frob(o, ref["o"][0]) < 1e-2
    _rejects("o", o.to(torch.bfloat16), ref)


def test_rejects_one_warp_five_percent_off(case):
    """16 rows of one warp scaled by 1.05, e.g. one missed rescale."""
    _, _, ref = case
    o = ref["o"][0].clone()
    o[:, Q0 + 32:Q0 + 48, HF] *= 1.05
    assert _frob(o, ref["o"][0]) < 1e-2
    _rejects("o", o.to(torch.bfloat16), ref)


def test_rejects_row_stored_from_its_neighbour(case):
    _, _, ref = case
    o = ref["o"][0].clone()
    o[:, Q0 + 70, HF] = o[:, Q0 + 71, HF]
    assert _frob(o, ref["o"][0]) < 1e-2
    _rejects("o", o.to(torch.bfloat16), ref)


def test_rejects_wrong_ring_stage(case):
    """Key tile 3 multiplied with key tile 4's V."""
    (q, k, v), mask, ref = case
    vb = v.clone()
    vb[:, 384:512] = v[:, 512:640]
    o, _ = _cta_fault(ref, *fc.forward64(*_head(q, k, vb, HF), SCALE, mask))
    _rejects("o", o.to(torch.bfloat16), ref)


# ---- more faults ----------------------------------------------------------------------------------------------------
def test_rejects_wrong_gqa_kv_head(case):
    t, mask, ref = case
    hk = HF // (H // Hk)
    o, lse = _cta_fault(ref, *fc.forward64(*_head(*t, HF, kv=(hk + 1) % Hk), SCALE, mask))
    _rejects("o", o.to(torch.bfloat16), ref)
    _rejects("lse", lse.float(), ref)


def test_rejects_scale_off_by_one_percent(case):
    t, mask, ref = case
    o, lse = fc.forward64(*t, SCALE * 1.01, mask)
    _rejects("o", o[0].to(torch.bfloat16), ref)
    _rejects("lse", lse[0].float(), ref)


def test_rejects_lse_in_log2_units(case):
    _, _, ref = case
    _rejects("lse", (ref["lse"][0] * fc.LOG2E).float(), ref)


def test_rejects_cta_lse_missing_its_last_key_tile(case):
    """O right, LSE of one CTA without its last (diagonal) key tile."""
    t, mask, ref = case
    bad = mask.clone()
    bad[Q0:Q1, Q0:Q1] = False
    _, lse = _cta_fault(ref, lse_h=fc.forward64(*_head(*t, HF), SCALE, bad)[1])
    _rejects("lse", lse.float(), ref)


# ---- documents and windows -------------------------------------------------------------------------------------------
S2, H2, Hk2 = 600, 4, 2


@pytest.fixture(scope="module")
def packed():
    """Two packed rows; in row 1 a document begins mid-tile at token 200 and runs to 450."""
    torch.manual_seed(6)
    q = torch.randn(2, S2, H2, D).to(torch.bfloat16)
    k = torch.randn(2, S2, Hk2, D).to(torch.bfloat16)
    v = torch.randn(2, S2, Hk2, D).to(torch.bfloat16)
    pos = torch.stack([positions([100, 100, 100, 300], S2), positions([200, 250, 150], S2)])
    return q, k, v, pos


def _mask_fault(packed, good, bad):
    q, k, v, _ = packed
    ref = fc.reference(q, k, v, SCALE, good)
    o, lse = fc.forward64(q, k, v, SCALE, bad)
    _rejects("o", o.to(torch.bfloat16), ref)
    _rejects("lse", lse.float(), ref)


def test_rejects_document_start_off_by_one(packed):
    """The document starting at token 200 (mid key tile 1) also sees key 199."""
    pos = packed[3]
    bad = pos.clone()
    bad[1, 200:450] += 1
    _mask_fault(packed, fc.visible(S2, pos=pos), fc.visible(S2, pos=bad))


@pytest.mark.parametrize("W", [0, 63, 128])
def test_rejects_window_admitting_w_plus_2_keys(packed, W):
    _mask_fault(packed, fc.visible(S2, window=W), fc.visible(S2, window=W + 1))


def test_rejects_packed_row_ignoring_the_window(packed):
    """pos used where min(pos, W) belongs."""
    pos = packed[3]
    _mask_fault(packed, fc.visible(S2, pos=pos, window=90), fc.visible(S2, pos=pos))


# ---- the mask builder -------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("S_", [1, 129, 1000])
def test_visible_matches_product_masks(S_):
    from mlx_cuda_distributed_pretraining_b200.arch.flash_attention import CausalMask, DocumentCausalMask
    pos = torch.stack([positions(lay, S_) for lay in layouts(S_)]) if S_ > 109 else torch.arange(S_)[None]
    for W in [None] + windows(S_):
        if W is not None and W < 0:
            continue
        assert torch.equal(fc.visible(S_, window=W), CausalMask(S_, W).dense(torch.float64)[0, 0] == 0), W
        assert torch.equal(fc.visible(S_, pos=pos, window=W),
                           DocumentCausalMask(pos, W).dense(torch.float64)[:, 0] == 0), W
    assert fc.visible(S_, causal=False).all()


# ---- ALiBi (b200_attn_fwd_alibi) ------------------------------------------------------------------------------------
# one row, GQA group 4; faults go into the CTA (128-query tile QA, head HA).  Every fault below changes the bias only.
SA, HA_, HkA, QA, HA = 1024, 8, 2, 6, 1
QA0, QA1 = QA * 128, QA * 128 + 128
SLOPES = {"steep": [0.5] * HA_, "gentle": [1 / 256] * HA_, "mixed": [(0.0, 1 / 256, 0.5)[h % 3] for h in range(HA_)],
          "zero": [0.0] * HA_}


def _slopes(kind):
    return torch.tensor(SLOPES[kind], dtype=torch.float32)


@pytest.fixture(scope="module")
def alibi_case():
    torch.manual_seed(21)
    q = torch.randn(1, SA, HA_, D).to(torch.bfloat16)
    k = torch.randn(1, SA, HkA, D).to(torch.bfloat16)
    v = torch.randn(1, SA, HkA, D).to(torch.bfloat16)
    return q, k, v


def _alibi_ref(t, kind, mask=None):
    return fc.reference(*t, SCALE, fc.visible(SA) if mask is None else mask, slopes=_slopes(kind))


def _cta(ref, o_bad, lse_bad):
    o, lse = ref["o"][0].clone(), ref["lse"][0].clone()
    o[:, QA0:QA1, HA] = o_bad[:, QA0:QA1, HA]
    lse[:, HA, QA0:QA1] = lse_bad[:, HA, QA0:QA1]
    return o, lse


def _verdict(ref, o, lse):
    """(O rejected, LSE rejected, O's Frobenius error over the row < 1e-2, LSE's max abs error < 1e-3): the last two
    are the kernel checks of tests/test_gpu_alibi.py."""
    out = []
    for name, got in (("o", o.to(torch.bfloat16)), ("lse", lse.float())):
        try:
            fc.check(name, got, *ref[name])
            out.append(False)
        except AssertionError:
            out.append(True)
    return (out[0], out[1], _frob(o, ref["o"][0]) < 1e-2,
            float((lse.double() - ref["lse"][0]).abs().max()) < 1e-3)


@pytest.mark.parametrize("kind", list(SLOPES))
@pytest.mark.parametrize("layout", ["rows", "packed", "window"])
def test_alibi_accepts_rounded_reference_and_kernel_emulation(alibi_case, kind, layout):
    """The emulation forms the bias as the kernel does (fp32 m log2e, a per-row base, fmaf per column): it must sit
    inside the bound with margin for steep, gentle, mixed and zero slopes, on plain, packed and windowed rows."""
    mask = None
    if layout == "packed":
        mask = fc.visible(SA, pos=positions([100, 200, 129, 300, 295], SA)[None])[0]
    elif layout == "window":
        mask = fc.visible(SA, window=129)
    ref = _alibi_ref(alibi_case, kind, mask)
    r, bd = ref["o"]
    assert fc.check("o", r.to(torch.bfloat16), r, bd) < 0.5
    o, lse = fc.emulate_kernel(*alibi_case, SCALE, fc.visible(SA) if mask is None else mask, slopes=_slopes(kind))
    assert fc.check("o", o, *ref["o"]) < 0.75
    assert fc.check("lse", lse, *ref["lse"]) < 0.25


def test_alibi_zero_slopes_are_the_causal_reference(alibi_case):
    a, c = _alibi_ref(alibi_case, "zero"), fc.reference(*alibi_case, SCALE, fc.visible(SA))
    for name in ("o", "lse"):
        assert torch.equal(a[name][0], c[name][0]) and torch.equal(a[name][1], c[name][1])


def _bias_fn(kind, fault):
    sl = _slopes(kind)
    pos = torch.arange(SA, dtype=torch.float64)

    def f(h0, h1):
        b = fc.alibi_bias(sl, SA, h0, h1)
        m = sl[h0:h1].double()[:, None, None]
        if fault == "interior":        # key tiles wholly below the CTA's first query get no bias
            b[:, QA0:QA1, :QA0] = 0
        elif fault == "odd_columns":   # c = 8 nc: the odd keys' bias one key short
            b = b - m * (pos % 2)[None, None, :]
        elif fault == "bf16":          # the log2-unit bias rounded through bf16 before the add
            b = (b * fc.LOG2E).to(torch.bfloat16).double() / fc.LOG2E
        elif fault == "scaled":        # the bias multiplied by the softmax scale
            b = b * SCALE
        elif fault == "row_half":      # rows + 8 of each 16 use the first half's base: b + 8 m
            b = b + 8 * m * ((pos % 16) >= 8)[None, :, None]
        elif fault == "uniform_shift":  # every distance off by one: b + m on every element
            b = b + m
        return b
    return f


# (fault, slopes, O rejected, LSE rejected, O's Frobenius check passes it, LSE's max-abs check passes it).  At this
# shape the max-abs LSE check of tests/test_gpu_alibi.py notices every one of them (|dLSE| >= 2.3e-3); the Frobenius
# check on O passes four, which only the element check of O or LSE sees.
FAULTS = [("interior", "gentle", True, True, False, False),
          ("odd_columns", "gentle", False, True, True, False),
          ("odd_columns", "steep", True, True, False, False),
          ("bf16", "steep", False, True, True, False),
          ("scaled", "gentle", True, True, False, False),
          ("row_half", "gentle", False, True, True, False),
          ("row_half", "steep", False, True, True, False)]


@pytest.mark.parametrize("fault,kind,o_rej,lse_rej,frob_passes,lse_abs_passes", FAULTS)
def test_alibi_rejects_bias_fault_in_one_cta(alibi_case, fault, kind, o_rej, lse_rej, frob_passes, lse_abs_passes):
    """One CTA's bias wrong; at least one of O and LSE rejects it.  interior: the key tiles wholly below the CTA's
    first query without bias (a fast path that skips it); odd_columns: c = 8 nc, the e & 1 term dropped; bf16: the
    log2-unit bias rounded through bf16; scaled: the bias times the softmax scale; row_half: rows 8..15 of every 16
    with the first half's base, a row-uniform shift, so O cannot change and LSE moves by 8 m."""
    ref = _alibi_ref(alibi_case, kind)
    o, lse = _cta(ref, *fc.forward64(*alibi_case, SCALE, fc.visible(SA), bias=_bias_fn(kind, fault)))
    assert _verdict(ref, o, lse) == (o_rej, lse_rej, frob_passes, lse_abs_passes)


@pytest.mark.parametrize("first", [True, False], ids=["group_first", "next_head"])
def test_alibi_rejects_neighbouring_head_slope(alibi_case, first):
    """alibi_slopes(8) and every head of a GQA group given the group's first head's slope, or query head h + 1's."""
    from mlx_cuda_distributed_pretraining_b200.arch.flash_attention import alibi_slopes
    sl = alibi_slopes(HA_)
    g = HA_ // HkA
    idx = torch.arange(HA_) // g * g if first else torch.clamp(torch.arange(HA_) + 1, max=HA_ - 1)
    ref = fc.reference(*alibi_case, SCALE, fc.visible(SA), slopes=sl)
    o, lse = fc.forward64(*alibi_case, SCALE, fc.visible(SA), slopes=sl[idx])
    h = 2 if first else 5    # a head whose slope the fault changes: 1/16 -> 1/4, 1/32 -> 1/64
    o_h, lse_h = ref["o"][0].clone(), ref["lse"][0].clone()
    o_h[..., h, :], lse_h[:, h] = o[0, :, h], lse[0, h]
    assert _verdict(ref, o_h, lse_h)[:2] == (True, True)


def test_alibi_uniform_shift_is_invisible_to_o_by_construction(alibi_case):
    """A bias off by the same amount on every key of a row (distance off by one everywhere) leaves the softmax and O
    unchanged: no checker of O can see it, and this is no gap in the bound.  LSE moves by exactly m, which its check
    catches."""
    for kind in ("steep", "gentle"):
        ref = _alibi_ref(alibi_case, kind)
        o, lse = fc.forward64(*alibi_case, SCALE, fc.visible(SA), bias=_bias_fn(kind, "uniform_shift"))
        assert float((o[0] - ref["o"][0]).abs().max()) < 1e-12
        assert _verdict(ref, o[0], lse[0])[:2] == (False, True), kind


def test_alibi_bf16_bias_at_gentle_slopes_is_below_the_noise():
    """Stated limit.  The bf16-rounded bias errs by up to 2^-9 |b| per key with pseudo-random sign; at slope 1/256
    |b| stays near 1 where P has weight, so O and LSE move by less than P's own bf16 rounding.  Steep slopes (0.5) and
    far-back heavy keys (the underflow regime) are where the fault shows, and the GPU suite runs both."""
    torch.manual_seed(22)
    q = torch.randn(1, SA, HA_, D).to(torch.bfloat16)
    k = torch.randn(1, SA, HkA, D).to(torch.bfloat16)
    v = torch.randn(1, SA, HkA, D).to(torch.bfloat16)
    ref = _alibi_ref((q, k, v), "gentle")
    o, lse = fc.forward64(q, k, v, SCALE, fc.visible(SA), bias=_bias_fn("gentle", "bf16"))
    assert _verdict(ref, o[0], lse[0])[:2] == (False, False)
    # far-back heavy keys: keys 0..127 dominate every later row, 700-900 positions back (test_fwd_logit_regimes)
    q = torch.randn(1, SA, HA_, D) * 0.1
    k = torch.randn(1, SA, HkA, D) * 0.1
    q[..., 0] = 4.0
    k[..., 0] = -60.0
    k[:, :128, :, 0] = 30.0
    t = (q.to(torch.bfloat16), k.to(torch.bfloat16), v)
    ref = fc.reference(*t, 1.0, fc.visible(SA), slopes=_slopes("steep"))
    o, lse = fc.forward64(*t, 1.0, fc.visible(SA), bias=_bias_fn("steep", "bf16"))
    assert _verdict(ref, o[0], lse[0])[:2] == (True, True)
