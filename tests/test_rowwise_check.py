"""CPU: tests/rowwise_check.py accepts a plain fp32 / bf16 torch emulation of each memory-bound kernel's arithmetic and
rejects single seeded faults of the kind those kernels can have (a dropped vector, row, tail or partial, a wrong row
length, a padding column read or written, a guard byte touched)."""
import pytest
import torch

from tests import rowwise_check as rc

BF16, F32 = torch.bfloat16, torch.float32


def _gen(seed):
    return torch.Generator().manual_seed(seed)


# ---- fp32 emulations of the kernels' arithmetic: name -> (reference dict, outputs dict, inputs) ------------------
def _case_rmsnorm(T=BF16, R=37, H=264, eps=1e-5):
    g = _gen(1)
    x, d = torch.randn(R, H, generator=g).to(T), torch.randn(R, H, generator=g).to(T)
    w = (torch.rand(H, generator=g) + 0.5).to(T)
    s = (x.float() + d.float()).to(T)
    sf = s.float()
    rstd = 1.0 / torch.sqrt((sf * sf).sum(-1) / H + eps)
    y = (sf * rstd[:, None] * w.float()).to(T)
    return rc.rmsnorm_fwd(x, w, eps, d), {"sum": s, "rstd": rstd, "y": y}, dict(x=x, d=d, w=w, H=H, eps=eps, s=s)


def _case_rmsnorm_bwd(T=BF16, R=41, H=520):
    g = _gen(2)
    x, dy, dres = (torch.randn(R, H, generator=g).to(T) for _ in range(3))
    w = (torch.rand(H, generator=g) + 0.5).to(T)
    xf, dyf = x.float(), dy.float()
    rstd = 1.0 / torch.sqrt((xf * xf).sum(-1) / H + 1e-5)
    gg = dyf * w.float()
    c = (gg * xf).sum(-1, keepdim=True) / H * rstd[:, None] ** 2
    dx = (rstd[:, None] * (gg - xf * c) + dres.float()).to(T)
    parts = (dyf * xf * rstd[:, None]).view(R, 1, H).sum(1)          # one partial row per "CTA"
    return rc.rmsnorm_bwd(dy, x, w, rstd, dres), {"dx": dx, "dw": parts.sum(0)}, dict(dres=dres, parts=parts, T=T)


def _case_colsum(P=129, H=72):
    parts = torch.randn(P, H, generator=_gen(3))
    prior = torch.randn(H, generator=_gen(4)).to(BF16)
    got = (parts.sum(0) + prior.float()).to(BF16)
    return rc.colsum(parts, prior, BF16), {"dw": got}, dict(parts=parts, prior=prior)


def _case_rope(layout="interleaved", T=BF16):
    g = _gen(5)
    B, S, NH, D = 2, 9, 3, 16
    x = torch.randn(B, S, NH, D, generator=g).to(T)
    ang = torch.rand(12, D // 2, generator=g) * 6
    cos_t, sin_t = torch.cos(ang), torch.sin(ang)
    pos = torch.randint(0, 12, (B, S), generator=g).int()

    def emul(p):
        idx = p.long()
        c, s = cos_t[idx][:, :, None], sin_t[idx][:, :, None]
        xf = x.float()
        if layout == "interleaved":
            a, b = xf[..., 0::2], xf[..., 1::2]
            return torch.stack([a * c - b * s, a * s + b * c], -1).flatten(-2).to(T)
        a, b = xf[..., :D // 2], xf[..., D // 2:]
        return torch.cat([a * c - b * s, a * s + b * c], -1).to(T)

    return rc.rope(x, cos_t, sin_t, pos, layout), {"y": emul(pos)}, dict(emul=emul, S=S, B=B)


def _case_glu(act="sigmoid2"):
    g = _gen(6)
    n = 2048
    gt, up, dy = ((torch.randn(n, generator=g) * 8).to(BF16) for _ in range(3))
    gt[:16] = torch.linspace(-60, 60, 16).to(BF16)
    up[8:24] = torch.linspace(60, -60, 16).to(BF16)
    gf, uf, df = gt.float(), up.float(), dy.float()
    if act == "sigmoid2":
        s = torch.sigmoid(uf)
        out = {"y": gf * s * 2, "dg": df * s * 2, "du": df * gf * s * (1 - s) * 2}
    else:
        s = torch.sigmoid(gf)
        out = {"y": gf * s * uf, "dg": df * uf * s * (1 + gf * (1 - s)), "du": df * (gf * s)}
    ref = dict(rc.glu_fwd(gt, up, act), **rc.glu_bwd(dy, gt, up, act))
    return ref, {k: v.to(BF16) for k, v in out.items()}, {}


def _case_ce(R=9, V=259, ld=264, pad=7):
    g = _gen(7)
    full = torch.full((R, ld), 3e38).to(BF16)
    full[:, :V] = (torch.randn(R, V, generator=g) * 3).to(BF16)
    full[1, :V] = 0.0
    full[2, V - 1] = 40.0
    t = torch.randint(0, V, (R,), generator=g)
    t[0], t[1], t[2], t[3], t[4] = 0, V - 1, V // 8 * 8, pad, V - 1
    scale = torch.randn(R, generator=g)
    scale[5] = 0.0
    x = full[:, :V].float()
    lse = torch.logsumexp(x, -1)
    tc = t.clamp(0, V - 1)
    loss = torch.where(t != pad, lse - x.gather(1, tc[:, None])[:, 0], torch.zeros(()))
    pr = torch.exp(x - lse[:, None])
    pr[torch.arange(R), tc] -= (t == tc).float()
    d = torch.zeros(R, ld)
    d[:, :V] = pr * torch.where(t != pad, scale, torch.zeros(()))[:, None]
    ref = dict(rc.ce_fwd(full, t, V, pad), **rc.ce_bwd(full, t, V, pad, lse, scale))
    return ref, {"lse": lse, "loss": loss, "dlogits": d.to(BF16)}, dict(full=full, t=t, V=V, x=x, scale=scale, lse=lse)


def _case_embedding(T=BF16):
    g = _gen(8)
    V, H, rows = 19, 24, 300
    dh = torch.randn(rows, H, generator=g).to(BF16)
    tok = torch.randint(0, V - 2, (rows,), generator=g)               # rows V-2, V-1 are never hit
    tok[::17], tok[5::19] = -1, V
    prior = torch.randn(V, H, generator=g).to(T)
    ok = (tok >= 0) & (tok < V)
    scratch = torch.zeros(V, H).index_add_(0, tok[ok], dh[ok].float())
    got = (prior.float() + scratch).to(T)
    return rc.embedding_bwd(dh, tok, prior, V), {"grad": got}, dict(prior=prior, tok=tok, dh=dh, V=V, T=T)


def _case_adamw(n=4099):
    g = _gen(9)
    p, gr, m = (torch.randn(n, generator=g) for _ in range(3))
    v = torch.rand(n, generator=g) * 0.1
    v[:5], gr[:3], m[3] = 0.0, 0.0, 0.0
    lr, b1, b2, eps, wd, bc1, bc2, gs = 1e-2, 0.9, 0.95, 1e-8, 0.1, 1 - 0.9 ** 3, 1 - 0.95 ** 3, 0.5
    f = torch.tensor
    gj = gr * gs
    m2 = f(b1) * m + (1 - f(b1)) * gj
    v2 = f(b2) * v + (1 - f(b2)) * gj * gj
    p2 = p * (1 - f(lr) * f(wd)) - (f(lr) / f(bc1)) * m2 / (v2.sqrt() * torch.rsqrt(f(bc2)) + f(eps))
    return (rc.adamw(p, gr, m, v, lr, b1, b2, eps, wd, bc1, bc2, gs), {"p": p2, "m": m2, "v": v2},
            dict(p=p, n=n))


def _case_elementwise():
    """sgd_momentum, muon_momentum + sumsq, axpy, clip_accum, ns_scales, split_bf16, ema_split, graft_update in one
    reference dict with prefixed names."""
    g = _gen(10)
    n = 1003
    p, gr, buf = (torch.randn(n, generator=g) for _ in range(3))
    f = torch.tensor
    ref, got = {}, {}

    def add(prefix, r, o):
        ref.update({f"{prefix}.{k}": v for k, v in r.items()})
        got.update({f"{prefix}.{k}": v for k, v in o.items()})

    gj = gr * 0.5
    b2 = (1 - f(0.95)) * gj + f(0.95) * buf
    u = gj + f(0.95) * b2
    add("sgd", rc.sgd_momentum(p, gr, buf, 0.95, True, 0.01, 0.5), {"p": p - f(0.01) * u, "buf": b2})
    add("muon", rc.muon_momentum(gr[None], buf[None], 0.95, True, 0.5, 1),
        {"buf": b2[None], "u": u.to(BF16)[None], "sumsq": (u * u).sum()[None]})
    x16 = gr.to(BF16)
    add("axpy", rc.axpy_update(p, x16, -0.1), {"p": p + f(-0.1) * x16.float()})
    add("clip", rc.clip_accum(x16, buf, 1.0, 0.125, False), {"acc": buf + x16.float().clamp(-1, 1) * 0.125})
    add("sumsq", rc.sumsq(gr[None], 1, prior=f([3.0])), {"ss": (gr * gr).sum()[None] + 3.0})
    ss = torch.rand(5, generator=g) * 100
    inv = 1 / (ss.sqrt() + 1e-7)
    add("ns", rc.ns_scales(ss, 1e-7), {"inv": inv, "inv2": inv * inv})
    src = torch.randn(12, 16, generator=g)
    xs = (src[:10, :9] + torch.eye(10, 9) * 0.5) * f(1.5)
    hi = xs.to(BF16)
    lo = (xs - hi.float()).to(BF16)
    add("split", rc.split_bf16(src, 10, 9, 1.5, 0.5), {"hi": hi, "hi+lo": hi.double() + lo.double()})
    m2 = f(0.9) * buf + (1 - f(0.9)) * gr * 0.5
    mh = m2 * f(1.25)
    h2 = mh.to(BF16)
    add("ema", rc.ema_split(gr, buf, 0.9, 0.5, 1.25, -0.01),
        {"m": m2, "out32": mh * f(-0.01), "hi": h2, "hi+lo": h2.double() + (mh - h2.float()).to(BF16).double()})
    pb, pre, d = (torch.randn(3, 40, generator=g) for _ in range(3))
    coef, coef_d = f([0.5, 0.0, -2.0]), f([0.0, 1.5, 0.25])
    pre[1, 3], d[0, 7] = float("nan"), float("inf")                  # dropped with their zero coefficients
    gp = pb * f(0.99)
    gp = gp + torch.where(coef[:, None] != 0, coef[:, None] * pre, torch.zeros(()))
    gp = gp + torch.where(coef_d[:, None] != 0, coef_d[:, None] * d, torch.zeros(()))
    add("graft", rc.graft_update(pb, pre, d, coef, coef_d, 0.99), {"p": gp})
    return ref, got, dict(n=n, gr=gr, buf=buf)


CASES = {
    "rmsnorm_bf16": _case_rmsnorm, "rmsnorm_fp32": lambda: _case_rmsnorm(F32, R=5, H=1032),
    "rmsnorm_bwd_bf16": _case_rmsnorm_bwd, "rmsnorm_bwd_fp32": lambda: _case_rmsnorm_bwd(F32, R=130, H=8),
    "colsum": _case_colsum,
    "rope_interleaved": _case_rope, "rope_half_fp32": lambda: _case_rope("half", F32),
    "glu_sigmoid2": _case_glu, "glu_silu": lambda: _case_glu("silu"),
    "ce": _case_ce, "ce_v1": lambda: _case_ce(R=6, V=1, ld=8, pad=-100),
    "embedding_bf16": _case_embedding, "embedding_fp32": lambda: _case_embedding(F32),
    "adamw": _case_adamw, "elementwise": _case_elementwise,
}


@pytest.mark.parametrize("name", sorted(CASES))
def test_emulation_passes(name):
    ref, got, _ = CASES[name]()
    rc.check_all(got, ref, name)
    # bf16 outputs can sit at the bound (half an ulp is up to 2^-8 |ref|); an honest fp32 evaluation is well inside it
    f32_out = {k: v for k, v in got.items() if v.dtype != BF16}
    if f32_out:
        worst = rc.check_all(f32_out, ref, name)
        assert worst <= 0.5, worst


# ---- single faults: name -> (case, mutation of the outputs) ------------------------------------------------------
def _bump_bf16(t, idx, ulps=2):
    t = t.clone()
    t.view(torch.int16).view(-1)[idx] += ulps
    return t


def _f_two_ulp(got, inp):
    i = int(got["y"].float().abs().view(-1).argmax())
    got["y"] = _bump_bf16(got["y"], i)


def _f_vector_zeroed(got, inp):
    got["y"] = got["y"].clone()
    got["y"][1024:1032] = 0


def _f_last_row(got, inp):
    got["y"] = got["y"].clone()
    got["y"][-1] = rc.Guarded(got["y"].shape[1:], got["y"].dtype).t      # still the sentinel pattern


def _f_tail(got, inp):
    n = inp["n"]
    got["p"] = got["p"].clone()
    got["p"][n // 8 * 8:] = inp["p"][n // 8 * 8:]


def _f_rstd_h8(got, inp):
    sf, H = inp["s"].float(), inp["H"]
    rstd = 1.0 / torch.sqrt((sf * sf).sum(-1) / (H + 8) + inp["eps"])
    got["rstd"] = rstd
    got["y"] = (sf * rstd[:, None] * inp["w"].float()).to(inp["s"].dtype)


def _f_lse_pad_column(got, inp):
    V = inp["V"]
    x = inp["full"][:, :V + 1].float().clone()
    x[:, V] = 0.0                                   # the padding column as the logits GEMM leaves it
    got["lse"] = torch.logsumexp(x, -1)


def _f_target_kept(got, inp):
    d = got["dlogits"].float()
    r = 0
    d[r, inp["t"][r]] += inp["scale"][r]
    got["dlogits"] = d.to(BF16)


def _f_pad_nonzero(got, inp):
    got["dlogits"] = got["dlogits"].clone()
    got["dlogits"][4, inp["V"] + 2] = 1e-30


def _f_pad_row_loss(got, inp):
    got["loss"] = got["loss"].clone()
    got["loss"][3] = 1e-6


def _f_partial_missing(got, inp):
    got["dw"] = (inp["parts"][:-1].sum(0) + inp["prior"].float()).to(BF16)


def _f_s3_dropped(got, inp):
    p = inp["parts"]
    keep = torch.ones(p.shape[0], dtype=torch.bool)
    keep[96:128] = False                             # the fourth accumulator of the unrolled loop
    got["dw"] = (p[keep].sum(0) + inp["prior"].float()).to(BF16)


def _f_dw_row_missing(got, inp):
    got["dw"] = inp["parts"][1:].sum(0)


def _f_dres_dropped(got, inp):
    got["dx"] = (got["dx"].float() - inp["dres"].float()).to(inp["T"])


def _f_rope_pos_ignored(got, inp):
    got["y"] = inp["emul"](torch.arange(inp["S"]).expand(inp["B"], inp["S"]))


def _f_emb_clamped(got, inp):
    tok, V = inp["tok"].clamp(0, inp["V"] - 1), inp["V"]
    scratch = torch.zeros(V, inp["dh"].shape[1]).index_add_(0, tok, inp["dh"].float())
    got["grad"] = (inp["prior"].float() + scratch).to(inp["T"])


def _f_emb_unhit_row(got, inp):
    got["grad"] = _bump_bf16(got["grad"], got["grad"].numel() - 1, 1)    # last row: no token hits it


def _f_sumsq_tail(got, inp):
    n, gr = inp["n"], inp["gr"]
    got["sumsq.ss"] = (gr[:n // 8 * 8] ** 2).sum()[None] + 3.0


def _f_graft_nan_kept(got, inp):
    got["graft.p"] = got["graft.p"].clone()
    got["graft.p"][1, 3] = float("nan")


def _f_shadow_truncated(got, inp):
    u = got["muon.u"].float()
    got["muon.u"] = (u.view(torch.int32) & ~0xFFFF).view(torch.float32).to(BF16) * (1 - 2.0 ** -7)


FAULTS = {
    "one element 2 bf16 ulp off": ("rmsnorm_bf16", _f_two_ulp),
    "one 8-vector zeroed": ("glu_sigmoid2", _f_vector_zeroed),
    "last row not written": ("rmsnorm_bf16", _f_last_row),
    "tail n % 8 not written": ("adamw", _f_tail),
    "rstd with H + 8": ("rmsnorm_bf16", _f_rstd_h8),
    "rstd with H + 8, fp32": ("rmsnorm_fp32", _f_rstd_h8),
    "lse includes a padding column": ("ce", _f_lse_pad_column),
    "target column not subtracted": ("ce", _f_target_kept),
    "padding column non-zero": ("ce", _f_pad_nonzero),
    "pad row with a loss": ("ce", _f_pad_row_loss),
    "dW reduction misses one partial row": ("colsum", _f_partial_missing),
    "dW reduction drops its fourth accumulator": ("colsum", _f_s3_dropped),
    "dW misses one row": ("rmsnorm_bwd_bf16", _f_dw_row_missing),
    "dres not added": ("rmsnorm_bwd_bf16", _f_dres_dropped),
    "rope ignores pos": ("rope_interleaved", _f_rope_pos_ignored),
    "embedding clamps out-of-range tokens": ("embedding_bf16", _f_emb_clamped),
    "embedding disturbs a row no token hits": ("embedding_bf16", _f_emb_unhit_row),
    "sumsq drops the tail": ("elementwise", _f_sumsq_tail),
    "zero coefficient keeps a NaN term": ("elementwise", _f_graft_nan_kept),
    "bf16 output truncated and 1 ulp low": ("elementwise", _f_shadow_truncated),
}


@pytest.mark.parametrize("fault", sorted(FAULTS))
def test_fault_is_rejected(fault):
    case, mutate = FAULTS[fault]
    ref, got, inp = CASES[case]()
    rc.check_all(got, ref, case)                     # the unmutated emulation passes
    mutate(got, inp)
    with pytest.raises(AssertionError):
        rc.check_all(got, ref, fault)


def test_check_reports_element_and_records_ratio():
    ref, bound = torch.zeros(3, 4, dtype=torch.float64), torch.full((3, 4), 1.0, dtype=torch.float64)
    got = torch.zeros(3, 4)
    got[2, 1] = 0.5
    rc.WORST.pop("t", None)
    assert rc.check(got, ref, bound, "t", family="t") == 0.5 and rc.WORST["t"] == 0.5
    got[1, 3] = 2.0
    with pytest.raises(AssertionError, match=r"element \(1, 3\).*ratio 2"):
        rc.check(got, ref, bound, "t")
    with pytest.raises(AssertionError, match="non-finite"):
        rc.check(torch.full((3, 4), float("nan")), ref, bound, "t")
    # a zero bound demands the value itself
    rc.check(torch.zeros(3, 4), ref, 0.0, "t")
    with pytest.raises(AssertionError):
        rc.check(torch.full((3, 4), 1e-30), ref, 0.0, "t")
    with pytest.raises(AssertionError, match="shape"):
        rc.check(torch.zeros(3, 5), ref, bound, "t")


@pytest.mark.parametrize("dtype,n", [(BF16, 7), (F32, 7), (BF16, 4099), (F32, 8), (torch.int64, 3)])
def test_guard_helper(dtype, n):
    g = rc.Guarded(n, dtype)
    assert g.t.numel() == n and g.t.data_ptr() % 16 == 0 and g.intact() and g.untouched()
    if dtype.is_floating_point:
        assert bool(torch.isfinite(g.t.float()).all())               # the sentinel is not a NaN pattern
    g.fill(torch.ones(n).to(dtype))
    assert g.intact() and not g.untouched()
    item = g.t.element_size()
    # one element past the end (what a full 8-vector store over a ragged tail does), and one before the start
    after = g.raw[rc.GUARD_BYTES + n * item:][:item]
    after.zero_()
    assert not g.intact()
    after.fill_(rc.GUARD_BYTE)
    assert g.intact()
    g.raw[rc.GUARD_BYTES - 1] = 0
    assert not g.intact()
