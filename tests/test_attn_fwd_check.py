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
