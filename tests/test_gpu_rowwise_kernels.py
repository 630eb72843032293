"""-m gpu: the memory-bound kernels (csrc/norm_rope.cu, csrc/model_fused.cu, the flat updates of csrc/elementwise.cu)
element by element against fp64 (tests/rowwise_check.py, which derives every bound), at sizes that run every loop:
more than one grid-stride pass with a ragged last one, every NVW / NV instantiation edge of the RMSNorm kernels, more
partial rows than one round of the dW reduction, scalar tails, and rows that some warps of the last CTA do not own.
Every output, workspace and in-place buffer sits between sentinel-filled guard bytes that must survive the launch."""
import pytest
import torch

from tests import rowwise_check as rc

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(900)]

BF16, F32 = torch.bfloat16, torch.float32
DEV = "cuda"
ERR_ARG, ERR_WORKSPACE = -1, -4
_GUARDS = []


@pytest.fixture(scope="module")
def ops():
    from mlx_cuda_distributed_pretraining_b200 import ops
    ops.require_device()
    return ops


@pytest.fixture(scope="module")
def sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


@pytest.fixture(autouse=True)
def guards_intact():
    """Every buffer made by G() in a test must still be framed by its sentinel bytes after it."""
    _GUARDS.clear()
    yield
    _check_guards("the end of the test")


def _check_guards(where):
    """Asserts the guards of every buffer made since the last call, and lets the buffers go."""
    torch.cuda.synchronize()
    broken = [i for i, g in enumerate(_GUARDS) if not g.intact()]
    _GUARDS.clear()
    assert not broken, f"guard bytes overwritten around buffers {broken} before {where}"


def G(shape, dtype, src=None):
    g = rc.Guarded(shape, dtype, DEV)
    _GUARDS.append(g)
    return g.fill(src) if src is not None else g


def _gen(seed):
    return torch.Generator(device=DEV).manual_seed(seed)


def _ok(ops, code, what):
    ops.check(code, what)


# ----------------------------------------------------------------------------------------------------------------
# RMSNorm family
# ----------------------------------------------------------------------------------------------------------------
HS = [8, 256, 264, 512, 520, 776, 1024, 1032, 2048, 4096, 4104, 8192]


def _norm_rows(R, H, T, gen):
    """Gaussian rows plus: one 2^10 among 2^-10s, an all-zero row, a constant row."""
    x = torch.randn(R, H, device=DEV, generator=gen)
    if R >= 5:
        x[1] = 2.0 ** -10
        x[1, H // 2] = 2.0 ** 10
        x[2] = 0.0
        x[3] = 3.0
    return x.to(T)


def _over_one_round(ops, sms, H):
    """One row more than a single round of the backward grid holds, so that some CTA loops twice."""
    per_cta = 4 if H <= 1024 else 1
    rows = sms * (5 if H <= 1024 else 4) * per_cta + 1
    assert ops.lib().b200_rmsnorm_bwd_partial_rows(rows, H) * per_cta < rows
    return rows


@pytest.mark.parametrize("T", [BF16, F32], ids=["bf16", "fp32"])
@pytest.mark.parametrize("H", HS)
def test_rmsnorm_family(ops, sms, H, T):
    L, st, isb = ops.lib(), ops._stream(), int(T == BF16)
    eps = 1e-5
    rows_list = [1, 3, 5, 130, _over_one_round(ops, sms, H)] + ([16384] if H <= 1024 or H == 2048 else [])
    for R in rows_list:
        for fused in (False, True):
            gen = _gen(H * 7 + R + fused)
            x = _norm_rows(R, H, T, gen)
            w = (torch.rand(H, device=DEV, generator=gen) + 0.5).to(T)
            delta = (torch.randn(R, H, device=DEV, generator=gen) * 0.5).to(T) if fused else None
            if fused and R >= 5:
                delta[2] = 0.0                       # the all-zero row stays all-zero
            what = f"H={H} rows={R} fused={fused}"
            y, rstd = G((R, H), T), G(R, F32)
            s = G((R, H), T) if fused else None
            if fused:
                _ok(ops, L.b200_add_rmsnorm_fwd(x.data_ptr(), delta.data_ptr(), w.data_ptr(), s.t.data_ptr(),
                                                y.t.data_ptr(), rstd.t.data_ptr(), R, H, eps, isb, st), what)
            else:
                _ok(ops, L.b200_rmsnorm_fwd(x.data_ptr(), w.data_ptr(), y.t.data_ptr(), rstd.t.data_ptr(), R, H, eps,
                                            isb, st), what)
            got = {"y": y.t, "rstd": rstd.t}
            if fused:
                got["sum"] = s.t
            rc.check_all(got, rc.rmsnorm_fwd(x, w, eps, delta), "fwd " + what, "rmsnorm_fwd")
            if R >= 5:
                assert float(rstd.t[2]) == pytest.approx(eps ** -0.5, rel=1e-6) and not bool(y.t[2].any())

            xs = s.t if fused else x                 # what the backward normalises
            dy = torch.randn(R, H, device=DEV, generator=gen).to(T)
            dres = torch.randn(R, H, device=DEV, generator=gen).to(T) if fused else None
            ref = rc.rmsnorm_bwd(dy, xs, w, rstd.t, dres)
            ws_bytes = int(L.b200_rmsnorm_bwd_workspace_bytes(R, H))
            nparts = int(L.b200_rmsnorm_bwd_partial_rows(R, H))
            assert ws_bytes == nparts * H * 4

            def bwd(dx, dw, ws):
                if fused:
                    return L.b200_add_rmsnorm_bwd(dy.data_ptr(), dres.data_ptr(), xs.data_ptr(), w.data_ptr(),
                                                  rstd.t.data_ptr(), dx.t.data_ptr(), dw, R, H, isb, ws.t.data_ptr(),
                                                  ws_bytes, st)
                return L.b200_rmsnorm_bwd(dy.data_ptr(), xs.data_ptr(), w.data_ptr(), rstd.t.data_ptr(),
                                          dx.t.data_ptr(), dw, R, H, isb, ws.t.data_ptr(), ws_bytes, st)

            # immediate path: dx and the fp32 dW
            dx, dw, ws = G((R, H), T), G(H, F32), G(ws_bytes, torch.uint8)
            _ok(ops, bwd(dx, dw.t.data_ptr(), ws), what)
            rc.check_all({"dx": dx.t, "dw": dw.t}, ref, "bwd " + what, "rmsnorm_bwd")
            assert bool(torch.isfinite(dx.t.float()).all())
            # deferred path: partials stay in the workspace, one batched reduction accumulates into a stored gradient
            dx2, ws2 = G((R, H), T), G(ws_bytes, torch.uint8)
            _ok(ops, bwd(dx2, None, ws2), what)
            assert torch.equal(dx2.t, dx.t)
            for gt in (BF16, F32):
                prior = torch.randn(H, device=DEV, generator=gen).to(gt)
                grad = G(H, gt, prior)
                _reduce(ops, [(ws2.t, grad.t, nparts, 1)], H)
                rc.check(grad.t, *rc.accumulated(ref["dw"], prior, gt), f"deferred dW {gt} " + what,
                         "rmsnorm_dw_deferred")


def _reduce(ops, jobs, H):
    from mlx_cuda_distributed_pretraining_b200._lib import DwJob
    arr = (DwJob * len(jobs))()
    for i, (parts, grad, n, acc) in enumerate(jobs):
        arr[i].partials, arr[i].dw, arr[i].n_partials = parts.data_ptr(), grad.data_ptr(), n
        arr[i].dw_is_bf16, arr[i].accumulate = int(grad.dtype == BF16), acc
    _ok(ops, ops.lib().b200_rmsnorm_dw_reduce(arr, len(jobs), H, ops._stream()), "b200_rmsnorm_dw_reduce")


@pytest.mark.parametrize("H", [72, 1024])
def test_rmsnorm_dw_reduce_partial_counts(ops, H):
    """b200_rmsnorm_dw_reduce on synthetic partials: every trip count of the unrolled-by-four loop and its remainder,
    bf16 and fp32 gradients, overwrite and accumulate, and 33 jobs (a second launch) in one call."""
    gen = _gen(H)
    counts = [1, 32, 96, 97, 128, 129, 500]
    jobs, expect = [], []
    for i in range(33):
        P = counts[i % len(counts)]
        gt, acc = (BF16, F32)[i % 2], (i // 2) % 2
        parts = torch.randn(P, H, device=DEV, generator=gen) * (1 + i % 3)
        prior = torch.randn(H, device=DEV, generator=gen).to(gt)
        grad = G(H, gt, prior)
        jobs.append((parts, grad.t, P, acc))
        expect.append((grad, rc.colsum(parts, prior if acc else None, gt), f"job {i} P={P} {gt} acc={acc}"))
    _reduce(ops, jobs, H)
    for grad, ref, what in expect:
        rc.check(grad.t, *ref["dw"], what, "rmsnorm_dw_reduce")


@pytest.mark.parametrize("H", [8200, 12, 0])
def test_rmsnorm_rejects_unsupported_row_length(ops, H):
    L, st = ops.lib(), ops._stream()
    n = max(H, 8) * 2
    x = torch.randn(n, device=DEV).to(BF16)
    y, rstd, ws = G(n, BF16), G(2, F32), G(1 << 20, torch.uint8)
    assert L.b200_rmsnorm_fwd(x.data_ptr(), x.data_ptr(), y.t.data_ptr(), rstd.t.data_ptr(), 2, H, 1e-5, 1, st) == ERR_ARG
    assert L.b200_rmsnorm_bwd(x.data_ptr(), x.data_ptr(), x.data_ptr(), rstd.t.data_ptr(), y.t.data_ptr(), None, 2, H, 1,
                              ws.t.data_ptr(), 1 << 20, st) == ERR_ARG
    torch.cuda.synchronize()
    assert y.untouched() and rstd.untouched() and ws.untouched()


# ----------------------------------------------------------------------------------------------------------------
# RoPE
# ----------------------------------------------------------------------------------------------------------------
def _doc_positions(B, S, table_rows, gen):
    """int32 [B, S]: row 0 counts up to table_rows - 1 (the largest position the tables hold) and restarts; the other
    rows hold documents of random lengths that restart mid-row."""
    pos = torch.empty(B, S, dtype=torch.int32, device=DEV)
    pos[0] = torch.arange(S, device=DEV) % table_rows
    for b in range(1, B):
        cuts = torch.randint(1, max(2, min(S, table_rows)), (8,), device=DEV, generator=gen)
        start = torch.zeros(S, dtype=torch.int64, device=DEV)
        at = torch.cumsum(cuts, 0)
        at = at[at < S]
        start[at] = at
        start = torch.cummax(start, 0).values
        pos[b] = ((torch.arange(S, device=DEV) - start) % table_rows).int()
    return pos


@pytest.mark.parametrize("T", [BF16, F32], ids=["bf16", "fp32"])
@pytest.mark.parametrize("with_pos", [False, True], ids=["seq", "pos"])
@pytest.mark.parametrize("layout,D", [("interleaved", 8), ("interleaved", 16), ("interleaved", 64), ("interleaved", 128),
                                      ("half", 16), ("half", 64), ("half", 128)])
def test_rope(ops, sms, layout, D, with_pos, T):
    B, NH = 2, 3
    over = 2 * sms * 8 * 256 * 16                      # two passes of the half-split kernel, four of the interleaved
    for S in (5, over // (B * NH * D) + 3):
        gen = _gen(D + S)
        table_rows = S if not with_pos else max(4, S // 3)
        cos_t, sin_t = ops.rope_tables(table_rows, D, 10000.0, DEV)
        pos = _doc_positions(B, S, table_rows, gen) if with_pos else None
        if with_pos:
            assert int(pos.max()) == table_rows - 1
        x = torch.randn(B, S, NH, D, device=DEV, generator=gen).to(T)
        dy = torch.randn(B, S, NH, D, device=DEV, generator=gen).to(T)
        what = f"{layout} D={D} S={S} pos={with_pos}"
        y, dx, back = G(x.shape, T), G(x.shape, T), G(x.shape, T)
        ops._rope_call(x, y.t, cos_t, sin_t, pos, 0, what, layout)
        ops._rope_call(dy, dx.t, cos_t, sin_t, pos, 1, what, layout)
        ops._rope_call(y.t, back.t, cos_t, sin_t, pos, 1, what, layout)
        rc.check(y.t, *rc.rope(x, cos_t, sin_t, pos, layout)["y"], "fwd " + what, "rope_fwd")
        rc.check(dx.t, *rc.rope(dy, cos_t, sin_t, pos, layout, backward=True)["y"], "bwd " + what, "rope_bwd")
        # the backward undoes the forward up to the two roundings to the storage type
        xd = x.double().abs()
        pair = (xd[..., 0::2] + xd[..., 1::2]).repeat_interleave(2, -1) if layout == "interleaved" else \
            (xd[..., :D // 2] + xd[..., D // 2:]).repeat(1, 1, 1, 2)
        unit = rc.U8 if T == BF16 else rc.U24
        rc.check(back.t, x.double(), (2.5 * unit + 4 * rc.C * rc.U24) * pair + rc.TINY, "round trip " + what,
                 "rope_round_trip")


# ----------------------------------------------------------------------------------------------------------------
# GLU activations
# ----------------------------------------------------------------------------------------------------------------
def test_glu_elementwise(ops, sms):
    """sigmoid2 and SiLU, forward and backward, at one vector, a ragged single pass and more than two grid passes."""
    for act in ("sigmoid2", "silu"):
        _glu_elementwise(ops, sms, act)
        _check_guards(f"the end of {act}")


def _glu_elementwise(ops, sms, act):
    L, st = ops.lib(), ops._stream()
    fwd, bwd = ("b200_glu_fwd", "b200_glu_bwd") if act == "sigmoid2" else ("b200_silu_glu_fwd", "b200_silu_glu_bwd")
    for n in (8, 2048 * 8 * 3 - 8, 2 * sms * 8 * 256 * 8 + 2048 * 8 + 8):
        gen = _gen(n % 9973)
        g, u, dy = ((torch.randn(n, device=DEV, generator=gen) * 4).to(BF16) for _ in range(3))
        k = min(n, 4096)
        sweep = torch.linspace(-60, 60, k, device=DEV).to(BF16)
        g[:k], u[n - k:] = sweep, sweep.flip(0)        # saturated sigmoids at the head and in the ragged last pass
        if n > 2 * k:
            u[:k] = sweep.flip(0)[torch.randperm(k, device=DEV, generator=gen)]
        y, dg, du = G(n, BF16), G(n, BF16), G(n, BF16)
        _ok(ops, getattr(L, fwd)(g.data_ptr(), u.data_ptr(), y.t.data_ptr(), n, st), fwd)
        _ok(ops, getattr(L, bwd)(dy.data_ptr(), g.data_ptr(), u.data_ptr(), dg.t.data_ptr(), du.t.data_ptr(), n, st), bwd)
        rc.check_all({"y": y.t}, rc.glu_fwd(g, u, act), f"{act} n={n}", f"glu_{act}")
        rc.check_all({"dg": dg.t, "du": du.t}, rc.glu_bwd(dy, g, u, act), f"{act} n={n}", f"glu_{act}")
    bad = G(16, BF16)
    assert getattr(L, fwd)(g.data_ptr(), u.data_ptr(), bad.t.data_ptr(), 12, st) == ERR_ARG
    torch.cuda.synchronize()
    assert bad.untouched()


# ----------------------------------------------------------------------------------------------------------------
# cross entropy
# ----------------------------------------------------------------------------------------------------------------
CE_SHAPES = [(1, 1, 8), (7, 5, 8), (64, 259, 264), (33, 32003, 32064), (16, 4096, 4096), (4096, 512, 512),
             (3, 50257, 50264)]


def _ce_inputs(R, V, ld, fill, gen):
    full = torch.empty(R, ld, device=DEV, dtype=BF16)
    if fill == "nan":                                   # bf16 NaN bit patterns, quiet and signalling, both signs
        pat = torch.tensor([0x7FC0, 0xFFC1 - 0x10000, 0x7F81, 0xFF80 - 0x10000 + 1], dtype=torch.int16, device=DEV)
        full.view(torch.int16)[:] = pat[torch.arange(ld, device=DEV) % 4]
    else:
        full[:] = torch.where(torch.arange(ld, device=DEV) % 2 == 0, 3e38, -3e38).to(BF16)
    x = torch.randn(R, V, device=DEV, generator=gen) * 3
    tail0 = V // 8 * 8 if V // 8 * 8 < V else max(V - 1, 0)
    pad = V - 3 if V > 8 else -100
    t = torch.randint(0, V, (R,), device=DEV, generator=gen)
    for r in range(R):
        k = r % 8
        if k == 0:
            t[r] = 0
        elif k == 1:                                    # one dominant logit, and it is the target: p - 1 cancels
            x[r] = torch.randn(V, device=DEV, generator=gen)
            x[r, V - 1] = 40.0
            t[r] = V - 1
        elif k == 2:                                    # the row maximum sits in the scalar tail
            x[r, tail0] = 30.0
            t[r] = tail0
        elif k == 3:
            t[r] = pad
        elif k == 4:
            x[r] = 1.5                                  # all equal
        elif k == 5:                                    # |x| ~ 80
            x[r] = 80.0 * torch.sign(torch.randn(V, device=DEV, generator=gen)) + torch.randn(V, device=DEV, generator=gen)
    full[:, :V] = x.to(BF16)
    scale = torch.randn(R, device=DEV, generator=gen)
    scale[4::5] = 0.0
    return full, t, pad, scale


@pytest.mark.parametrize("fill", ["huge", "nan"])
@pytest.mark.parametrize("R,V,ld", CE_SHAPES)
def test_cross_entropy(ops, R, V, ld, fill):
    L, st = ops.lib(), ops._stream()
    full, t, pad, scale = _ce_inputs(R, V, ld, fill, _gen(V + R))
    what = f"rows={R} V={V} ld={ld} pad columns {fill}"
    logits, loss, lse = G((R, ld), BF16, full), G(R, F32), G(R, F32)
    _ok(ops, L.b200_ce_fwd(logits.t.data_ptr(), ld, t.data_ptr(), R, V, pad, loss.t.data_ptr(), lse.t.data_ptr(), st), what)
    assert torch.equal(logits.t.view(torch.int16), full.view(torch.int16))      # the forward only reads
    rc.check_all({"lse": lse.t, "loss": loss.t}, rc.ce_fwd(full, t, V, pad), what, "ce_fwd")
    if bool((t == pad).any()):
        assert float(loss.t[t == pad].abs().max()) == 0.0
    _ok(ops, L.b200_ce_bwd(logits.t.data_ptr(), ld, t.data_ptr(), R, V, pad, lse.t.data_ptr(), scale.data_ptr(), st), what)
    rc.check_all({"dlogits": logits.t}, rc.ce_bwd(full, t, V, pad, lse.t, scale), what, "ce_bwd")
    assert torch.count_nonzero(logits.t[:, V:]) == 0 and torch.count_nonzero(logits.t[t == pad]) == 0


# ----------------------------------------------------------------------------------------------------------------
# embedding scatter
# ----------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("gt", [BF16, F32], ids=["bf16grad", "fp32grad"])
@pytest.mark.parametrize("V,H,rows,mode", [(259, 128, 4096, "random"), (32003, 1024, 16384, "random"),
                                           (67, 64, 24, "random"), (67, 64, 16384, "one"), (259, 520, 5000, "skips")])
def test_embedding_scatter(ops, V, H, rows, mode, gt):
    """(32003, 1024): V * H / 8 vectors are more than two passes of the accumulate kernel's grid, 16384 rows more than
    one of the scatter's; "one": every row hits token 5; "skips": tokens -1 and V among the valid ones."""
    L, st = ops.lib(), ops._stream()
    gen = _gen(V + rows)
    dh = torch.randn(rows, H, device=DEV, generator=gen).to(BF16)
    tok = torch.randint(0, V, (rows,), device=DEV, generator=gen)
    if mode == "one":
        tok[:] = 5
    if mode == "skips":
        tok[::7], tok[3::11] = -1, V
    prior = (torch.randn(V, H, device=DEV, generator=gen) * 0.05).to(gt)
    need = int(L.b200_embedding_bwd_workspace_bytes(V, H))
    grad, ws = G((V, H), gt, prior), G(need, torch.uint8)
    args = (dh.data_ptr(), tok.data_ptr(), grad.t.data_ptr(), int(gt == BF16), rows, V, H, ws.t.data_ptr())
    assert L.b200_embedding_bwd(*args, need - 1, st) == ERR_WORKSPACE
    torch.cuda.synchronize()
    assert ws.untouched() and torch.equal(grad.t, prior)
    _ok(ops, L.b200_embedding_bwd(*args, need, st), "b200_embedding_bwd")
    rc.check_all({"grad": grad.t}, rc.embedding_bwd(dh, tok, prior, V), f"V={V} H={H} rows={rows} {mode}",
                 "embedding_bwd")


# ----------------------------------------------------------------------------------------------------------------
# optimizer updates on flat ranges
# ----------------------------------------------------------------------------------------------------------------
def _vals(seed):
    """Seeded host-side draws, so that the first values do not depend on the length asked for."""
    gen = torch.Generator().manual_seed(seed)

    def draw(n, scale=1.0):
        return (torch.randn(max(n, 64), generator=gen)[:n] * scale).to(DEV)
    return draw


def _passes(sms, n, batch=1):
    nvec = max(n // 8, 1)
    gx = min((n // 8 + 1 + 255) // 256, max(1, (sms * 8 + batch - 1) // batch))
    return (nvec + gx * 256 - 1) // (gx * 256)


def _run_adamw(ops, sms, n, gdt, bc=True, shadow=True):
    r = _vals(1)
    p0, g, m0, v0 = r(n), r(n).to(gdt), r(n, 0.1), r(n, 0.1).abs()
    if n > 2:
        v0[1], g[1] = 0.0, 0.0                          # sqrt(v') = 0: the eps path
        g[2] = 0.0
    hp = dict(lr=1e-2, b1=0.9, b2=0.95, eps=1e-8, wd=0.1, bc1=1 - 0.9 ** 3 if bc else 1.0,
              bc2=1 - 0.95 ** 3 if bc else 1.0, gscale=0.5)
    p, m, v, p16 = G(n, F32, p0), G(n, F32, m0), G(n, F32, v0), (G(n, BF16) if shadow else None)
    ops.adamw(p.t, p16.t if shadow else None, g, m.t, v.t, **hp)
    if shadow:
        assert torch.equal(p16.t, p.t.to(BF16)), "bf16 shadow != bf16_rn(p32)"
    return {"p": p.t, "m": m.t, "v": v.t}, rc.adamw(p0, g, m0, v0, **hp)


def _run_adam_direction(ops, sms, n, gdt):
    r = _vals(2)
    g, m0, v0 = r(n).to(gdt), r(n, 0.1), r(n, 0.1).abs()
    hp = dict(lr=3e-3, b1=0.9, b2=0.999, eps=1e-8, bc1=0.19, bc2=0.002, gscale=2.0)
    d, m, v = G(n, F32), G(n, F32, m0), G(n, F32, v0)
    ops.adam_direction(d.t, g, m.t, v.t, **hp)
    return {"d": d.t, "m": m.t, "v": v.t}, rc.adam_direction(g, m0, v0, **hp)


def _run_sgd_momentum(ops, sms, n, gdt, nesterov=True):
    r = _vals(3)
    p0, g, b0 = r(n), r(n).to(gdt), r(n)
    p, buf, p16 = G(n, F32, p0), G(n, F32, b0), G(n, BF16)
    ops.sgd_momentum(p.t, p16.t, g, buf.t, 0.95, nesterov, 0.01, 0.25)
    assert torch.equal(p16.t, p.t.to(BF16))
    return {"p": p.t, "buf": buf.t}, rc.sgd_momentum(p0, g, b0, 0.95, nesterov, 0.01, 0.25)


def _run_axpy(ops, sms, n, gdt):
    r = _vals(4)
    p0, x = r(n), r(n).to(gdt)
    p, p16 = G(n, F32, p0), G(n, BF16)
    ops.axpy_update(p.t, p16.t, x, -0.1)
    assert torch.equal(p16.t, p.t.to(BF16))
    return {"p": p.t}, rc.axpy_update(p0, x, -0.1)


def _run_clip_accum(ops, sms, n, gdt, init=False, clip=1.0):
    r = _vals(5)
    g, a0 = r(n, 2.0).to(gdt), r(n)
    acc = G(n, F32, a0)
    ops.clip_accum(g, acc.t, clip, 0.125, init)
    return {"acc": acc.t}, rc.clip_accum(g, a0, clip, 0.125, init)


def _run_muon(ops, sms, n, gdt, nesterov=True, batch=1):
    r = _vals(6)
    g, b0 = r(n * batch).to(gdt).view(batch, n), r(n * batch).view(batch, n)
    buf, u, ss = G((batch, n), F32, b0), G((batch, n), BF16), G(batch, F32)
    ops.muon_momentum(g.view(batch, 1, n), buf.t, u.t, ss.t, 0.95, nesterov, 0.5)
    return ({"buf": buf.t, "u": u.t, "sumsq": ss.t},
            rc.muon_momentum(g, b0, 0.95, nesterov, 0.5, _passes(sms, n, batch)))


def _run_ema_split(ops, sms, n, gdt, with_lo=True):
    r = _vals(7)
    g, m0 = r(n).to(gdt), r(n)
    m, out32, hi, lo = G(n, F32, m0), G(n, F32), G(n, BF16), (G(n, BF16) if with_lo else None)
    ops.ema_split(g, m.t, out32.t, hi.t, lo.t if with_lo else None, 0.9, 0.5, 1.25, -0.01)
    got = {"m": m.t, "out32": out32.t, "hi": hi.t}
    if with_lo:
        got["hi+lo"] = hi.t.double() + lo.t.double()
    return got, rc.ema_split(g, m0, 0.9, 0.5, 1.25, -0.01)


def _run_graft(ops, sms, n, gdt=None, batch=1):
    r = _vals(8)
    p0, pre, d = (r(n * batch).view(batch, n) for _ in range(3))
    coef, coef_d = r(batch), r(batch)
    if batch >= 3:                                      # a zero coefficient drops its term, even a NaN / inf one
        coef[1], coef_d[2] = 0.0, 0.0
        pre[1, n // 2], d[2, n - 1] = float("nan"), float("inf")
    p, p16 = G((batch, n), F32, p0), G((batch, n), BF16)
    ops.graft_update(p.t, p16.t, pre, d, n, batch, coef, coef_d, 0.99)
    assert torch.equal(p16.t, p.t.to(BF16))
    return {"p": p.t}, rc.graft_update(p0, pre, d, coef, coef_d, 0.99)


def _flat_sizes(sms):
    P = sms * 8 * 256 * 8                               # elements one pass of a full grid covers
    return [1, 7, 8, 9, 4099, P + 8 + 5, 2 * P + 3]


def test_flat_updates(ops, sms):
    """n in {1, 7, 8, 9, 4099, P + 13, 2 P + 3}, P = one pass of a full grid: tail only, body only, body + tail, and
    two grid-stride passes, the second one a single vector or a full one, with a scalar tail; bf16 and fp32
    gradients.  A failure names the kernel, n and the gradient type."""
    for n in _flat_sizes(sms):
        for gdt in (BF16, F32):
            _flat_updates(ops, sms, n, gdt)
            _check_guards(f"the end of n={n} {gdt}")


def _flat_updates(ops, sms, n, gdt):
    runs = [("adamw", _run_adamw, {}), ("adamw", _run_adamw, dict(bc=False, shadow=False)),
            ("adam_direction", _run_adam_direction, {}),
            ("sgd_momentum", _run_sgd_momentum, {}), ("sgd_momentum", _run_sgd_momentum, dict(nesterov=False)),
            ("axpy_update", _run_axpy, {}),
            ("clip_accum", _run_clip_accum, {}), ("clip_accum", _run_clip_accum, dict(init=True, clip=0.0)),
            ("muon_momentum", _run_muon, {}), ("muon_momentum", _run_muon, dict(nesterov=False)),
            ("ema_split", _run_ema_split, {}), ("ema_split", _run_ema_split, dict(with_lo=False)),
            ("graft_update", _run_graft, {})]
    for name, run, kw in runs:
        got, ref = run(ops, sms, n, gdt, **kw)
        rc.check_all(got, ref, f"{name} n={n} {gdt} {kw}", name)
    # sumsq: overwrite and accumulate, and the same bits on a second call (fixed summation order)
    x = _vals(9)(n).to(gdt)
    out, out2 = G(1, F32, torch.tensor([3.0])), G(1, F32)
    ops.sumsq_raw(x, out.t, n, 1, zero_first=False)
    rc.check_all({"ss": out.t}, rc.sumsq(x[None], _passes(sms, n), prior=torch.tensor([3.0], device=DEV)),
                 f"sumsq accumulate n={n} {gdt}", "sumsq")
    ops.sumsq_raw(x, out.t, n, 1, zero_first=True)
    ops.sumsq_raw(x, out2.t, n, 1, zero_first=True)
    rc.check_all({"ss": out.t}, rc.sumsq(x[None], _passes(sms, n)), f"sumsq n={n} {gdt}", "sumsq")
    assert torch.equal(out.t, out2.t), f"sumsq n={n} {gdt}: a second call gave other bits"


@pytest.mark.parametrize("gdt", [BF16, F32], ids=["bf16grad", "fp32grad"])
def test_vector_body_and_scalar_tail_agree_bit_for_bit(ops, sms, gdt):
    """The same seven values as a scalar tail (n = 7) and inside an 8-element vector (n = 8)."""
    differ = []
    for run in (_run_adamw, _run_adam_direction, _run_sgd_momentum, _run_axpy, _run_clip_accum, _run_muon,
                _run_ema_split, _run_graft):
        tail, _ = run(ops, sms, 7, gdt)
        body, _ = run(ops, sms, 8, gdt)
        differ += [(run.__name__, k) for k in tail
                   if k != "sumsq" and not torch.equal(tail[k].reshape(-1)[:7], body[k].reshape(-1)[:7])]
    assert not differ, differ


@pytest.mark.parametrize("batch", [1, 3, 40])
def test_batched_muon_momentum_and_graft_update(ops, sms, batch):
    """grid = (blocks, batch): per-matrix sums of squares and coefficients; numel a multiple of 8 when batched, ragged
    when not; one size large enough that the per-matrix grid is capped and strides."""
    for n in ([4099, 520] if batch == 1 else [520, 8 * 256 * (sms + 5)]):
        for gdt in (BF16, F32):
            got, ref = _run_muon(ops, sms, n, gdt, batch=batch)
            rc.check_all(got, ref, f"muon_momentum batch={batch} n={n}", "muon_momentum")
            again, _ = _run_muon(ops, sms, n, gdt, batch=batch)
            assert torch.equal(got["sumsq"], again["sumsq"])
        got, ref = _run_graft(ops, sms, n, batch=batch)
        rc.check_all(got, ref, f"graft_update batch={batch} n={n}", "graft_update")
        x = _vals(10)(n * batch).view(batch, n)
        out = G(batch, F32)
        ops.sumsq_raw(x, out.t, n, batch)
        rc.check_all({"ss": out.t}, rc.sumsq(x, _passes(sms, n, batch)), f"sumsq batch={batch} n={n}", "sumsq")


def test_ns_scales_and_split_bf16(ops):
    ss = torch.tensor([0.0, 1e-12, 1.0, 123.456, 3e7] * 30, device=DEV)[:129]
    inv, inv2 = G(129, F32), G(129, F32)
    _ok(ops, ops.lib().b200_ns_scales(ss.data_ptr(), inv.t.data_ptr(), inv2.t.data_ptr(), 129, 1e-7, ops._stream()), "ns")
    rc.check_all({"inv": inv.t, "inv2": inv2.t}, rc.ns_scales(ss, 1e-7), "ns_scales", "ns_scales")
    # strided source and destination, a diagonal shift and a scale; only the [rows, cols] block is written
    gen = _gen(77)
    for rows, cols, ld_s, ld_d in [(37, 37, 40, 40), (1, 1, 8, 8), (300, 259, 264, 272), (1100, 1030, 1030, 1030)]:
        src = torch.randn(rows, ld_s, device=DEV, generator=gen)
        hi, lo = G((rows, ld_d), BF16), G((rows, ld_d), BF16)
        ops.split_bf16(src, rows, cols, hi.t, lo.t, scale=1.5, diag_add=0.25)
        got = {"hi": hi.t[:, :cols], "hi+lo": hi.t[:, :cols].double() + lo.t[:, :cols].double()}
        rc.check_all(got, rc.split_bf16(src, rows, cols, 1.5, 0.25), f"split_bf16 {rows}x{cols}", "split_bf16")
        fresh = rc.Guarded((rows, ld_d), BF16, DEV).t
        assert torch.equal(hi.t[:, cols:], fresh[:, cols:]) and torch.equal(lo.t[:, cols:], fresh[:, cols:])
        hi_only = G((rows, ld_d), BF16)
        ops.split_bf16(src, rows, cols, hi_only.t, None, scale=1.5, diag_add=0.25)
        assert torch.equal(hi_only.t, hi.t)


def test_short_workspaces_are_refused_and_nothing_is_written(ops):
    L, st = ops.lib(), ops._stream()
    n = 4099
    x = torch.randn(n, device=DEV)
    need = int(L.b200_reduce_workspace_bytes(1))
    ws, out, buf, u = G(need, torch.uint8), G(1, F32), G(n, F32), G(n, BF16)
    assert L.b200_sumsq(x.data_ptr(), 0, out.t.data_ptr(), n, 1, 1, ws.t.data_ptr(), need - 1, st) == ERR_WORKSPACE
    assert L.b200_muon_momentum(x.data_ptr(), 0, buf.t.data_ptr(), u.t.data_ptr(), out.t.data_ptr(), n, 1, 0.95, 1, 1.0,
                                ws.t.data_ptr(), need - 1, st) == ERR_WORKSPACE
    R, H = 130, 264
    xb = torch.randn(R, H, device=DEV).to(BF16)
    rstd = torch.ones(R, device=DEV)
    nb = int(L.b200_rmsnorm_bwd_workspace_bytes(R, H))
    dx, dw, ws2 = G((R, H), BF16), G(H, F32), G(nb, torch.uint8)
    assert L.b200_rmsnorm_bwd(xb.data_ptr(), xb.data_ptr(), xb.data_ptr(), rstd.data_ptr(), dx.t.data_ptr(),
                              dw.t.data_ptr(), R, H, 1, ws2.t.data_ptr(), nb - 1, st) == ERR_WORKSPACE
    torch.cuda.synchronize()
    assert all(g.untouched() for g in (ws, out, buf, u, dx, dw, ws2))


def test_print_worst_ratios():
    """Runs last in this file: the worst |got - ref| / bound per operation and output seen above."""
    for name in sorted(rc.WORST):
        print(f"worst ratio {name}: {rc.WORST[name]:.4f}")
    assert rc.WORST and all(v <= 1.0 for v in rc.WORST.values())
