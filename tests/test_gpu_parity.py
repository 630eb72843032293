"""-m gpu: the CUDA path, called through the C ABI, against the oracle and the golden vectors.

Tolerances (relative Frobenius error unless noted; see DESIGN.md section 5 "Oracle and parity"):
  fp32 elementwise kernels            1e-6      (same formula, fp32)
  bf16-output kernels                 4e-3      (one bf16 rounding of the result, 2^-8 relative)
  GEMM engine (tests/test_gpu_gemm_engine.py, element by element against fp64, tests/gemm_check.py):
    exact family (integer operands)   bit for bit: D == R (fp32 out), D == bf16_rn(R) (bf16 out)
    bound family (Gaussian operands)  |D - R| <= C32 K 2^-24 P (+ 2^-8 |R| for bf16 out), per element; C32 = 2,
                                      accumulation error seen <= 0.0032 K 2^-24 P (H100 80GB HBM3, 700 W limit)
  attention fwd/bwd (bf16 I/O)        1e-2      through the autograd wrappers (north_star: "stated fp tolerance";
                                                SURVEY 8c 2e-2).  The kernels themselves are checked element by
                                                element against fp64 in tests/test_gpu_attention_fwd.py
                                                (tests/attn_fwd_check.py) and tests/test_gpu_attention_bwd.py
                                                (tests/attn_bwd_check.py), C32 = 4
  Newton-Schulz 5 steps, bf16 operands 3e-2     (SURVEY 8c; measured ~1e-2).  Pins the reference's semantics; every
                                                iteration's three stages, the grouped chain, the Muon step and
                                                Shampoo's bf16x3 statistics / preconditioning are checked element
                                                by element against fp64 in tests/test_gpu_matrix_optimizers_check.py
                                                (tests/ns_check.py)
  RMSNorm, RoPE, GLU, cross entropy, embedding scatter and the flat optimizer updates are checked element by element
  against fp64 in tests/test_gpu_rowwise_kernels.py (tests/rowwise_check.py); only their golden-vector tests stay here
"""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

from oracle import reference_math as R  # noqa: E402


def rel(a, b):
    a, b = a.detach().double().cpu(), torch.as_tensor(np.asarray(b)).double() if not torch.is_tensor(b) else b.detach().double().cpu()
    # the 1e-4 floor keeps exact-zero references (e.g. dQ of a single-key softmax) meaningful
    return float((a - b).norm() / (b.norm() + 1e-4))


@pytest.fixture(scope="module")
def ops():
    from mlx_cuda_distributed_pretraining_b200 import ops as o
    o.require_device()
    return o


# ------------------------------------------------------------------------------------------------
# dense contraction engine
# ------------------------------------------------------------------------------------------------
# The python wrapper ops.gemm, element by element (tests/gemm_check.py); every mode of the engine underneath it, with
# guard buffers and schedule-sized shapes, is in tests/test_gpu_gemm_engine.py.
@pytest.mark.parametrize("a_mn,b_mn", [(False, False), (False, True), (True, True), (True, False)])
@pytest.mark.parametrize("M,N,K,batch,bn", [(128, 256, 64, 1, 0), (200, 328, 136, 3, 0), (256, 512, 1000, 2, 128),
                                           (384, 256, 520, 2, 256), (8, 8, 8, 1, 0), (1000, 64, 72, 1, 0)])
def test_gemm_layouts(ops, a_mn, b_mn, M, N, K, batch, bn):
    from tests import gemm_check as gc
    torch.manual_seed(M + N + K)
    if (a_mn and M % 8) or (b_mn and N % 8) or (not a_mn and K % 8) or (not b_mn and K % 8):
        pytest.skip("leading dimension must be a multiple of 8")
    for exact in (True, False):
        mk = (lambda *s: gc.exact_ints(s, device="cuda")) if exact else (lambda *s: torch.randn(*s, device="cuda"))
        a = mk(*((batch, K, M) if a_mn else (batch, M, K))).to(torch.bfloat16)
        b = mk(*((batch, K, N) if b_mn else (batch, N, K))).to(torch.bfloat16)
        R, P = gc.reference(a, b, a_mn=a_mn, b_mn=b_mn)
        for out_dtype in (torch.float32, torch.bfloat16):
            out = ops.gemm(a, b, a_mn=a_mn, b_mn=b_mn, out_dtype=out_dtype, force_bn=bn)
            gc.check(out, R, P, K, exact, f"exact={exact} out={out_dtype}")


def test_gemm_epilogue(ops):
    torch.manual_seed(0)
    for exact in (True, False):
        _gemm_epilogue_family(ops, exact)


def _gemm_epilogue_family(ops, exact):
    from tests import gemm_check as gc
    batch, M, N, K = 3, 256, 512, 320
    mk = (lambda *s: gc.exact_ints(s, device="cuda")) if exact else (lambda *s: torch.randn(*s, device="cuda"))
    a = mk(batch, M, K).to(torch.bfloat16)
    b = mk(batch, N, K).to(torch.bfloat16)
    c = mk(batch, M, N).to(torch.bfloat16)
    av, bv = torch.tensor([0.5, 2.0, 1.0], device="cuda"), torch.tensor([4.0, 0.25, 1.0], device="cuda")
    out = ops.gemm(a, b, c=c, alpha=0.5, beta=-2.0, alpha_vec=av, beta_vec=bv)
    R, P = gc.reference(a, b, alpha=0.5, beta=-2.0, alpha_vec=av, beta_vec=bv, C=c)
    gc.check(out, R, P, K, exact, "bf16 out, alpha/beta vectors")
    c32 = mk(batch, M, N)
    out = ops.gemm(a, b, c=c32, alpha=2.0, beta=0.5, out_dtype=torch.float32)
    R, P = gc.reference(a, b, alpha=2.0, beta=0.5, C=c32)
    gc.check(out, R, P, K, exact, "fp32 out")
    # in-place accumulate (C aliases D), as the bf16x3 Shampoo products do
    acc = c32.clone()
    ops.gemm(a, b, c=acc, out=acc, alpha=1.0, beta=1.0)
    R, P = gc.reference(a, b, beta=1.0, C=c32)
    gc.check(acc, R, P, K, exact, "fp32 out, C aliasing D")


def test_tensor_map_cache_answers_repeated_launches(ops):
    """The host encodes a TMA descriptor once per (address, shape, strides, box): a repeated launch on the same buffers
    must be served from the cache and compute the same result; a different shape on the same storage must not."""
    import ctypes
    from mlx_cuda_distributed_pretraining_b200._lib import lib

    def stats():
        h, m = ctypes.c_ulonglong(0), ctypes.c_ulonglong(0)
        lib().b200_tensor_map_cache_stats(ctypes.byref(h), ctypes.byref(m))
        return h.value, m.value

    torch.manual_seed(3)
    a = torch.randn(1, 512, 384, device="cuda").to(torch.bfloat16)
    b = torch.randn(1, 256, 384, device="cuda").to(torch.bfloat16)
    out = torch.empty(1, 512, 256, device="cuda", dtype=torch.float32)
    ops.gemm(a, b, out=out)
    first = out.clone()
    h0, m0 = stats()
    ops.gemm(a, b, out=out)
    h1, m1 = stats()
    assert m1 == m0 and h1 >= h0 + 2, (h0, m0, h1, m1)          # both operand maps came from the cache
    assert torch.equal(out, first)
    # same storage viewed with another shape: new descriptors, right answer
    a2, b2 = a.view(1, 256, 768), b.view(1, 128, 768)
    out2 = ops.gemm(a2, b2, out_dtype=torch.float32)
    h2, m2 = stats()
    assert m2 > m1
    assert rel(out2, torch.bmm(a2.float(), b2.float().transpose(1, 2))) < 2e-6


def test_gemm_rejects_bad_arguments(ops):
    from mlx_cuda_distributed_pretraining_b200._lib import B200Error
    a = torch.zeros(16, 12, device="cuda", dtype=torch.bfloat16)   # K = 12: 24-byte rows, not TMA-able
    with pytest.raises(B200Error):
        ops.gemm(a, a)
    with pytest.raises(ValueError):
        ops.gemm(a.float(), a.float())


# ------------------------------------------------------------------------------------------------
# Newton-Schulz
# ------------------------------------------------------------------------------------------------
def test_newton_schulz_golden(ops, golden):
    for tag in ("wide", "tall", "square", "batched"):
        g = torch.from_numpy(golden[f"ns_{tag}_in"])
        if g.shape[-1] % 8:
            continue
        x = ops.zeropower_via_newtonschulz5(g.cuda(), 5)
        assert rel(x, golden[f"ns_{tag}_out"]) < 3e-2, tag


@pytest.mark.parametrize("shape", [(2, 256, 512), (2, 512, 256), (1, 1024, 1024), (3, 512, 1024), (1, 2816, 1024),
                                   (1, 1024, 2816), (1, 1000, 256), (1, 136, 72), (1, 32003, 1024),
                                   (1, 5000, 512), (1, 384, 9000)])   # last three: split-K G1
def test_newton_schulz_vs_oracle(ops, shape):
    torch.manual_seed(1)
    g = torch.randn(*shape) * 0.02
    x = ops.zeropower_via_newtonschulz5(g.cuda())
    assert rel(x, R.newton_schulz5(g.double())) < 3e-2
    # full-size property (SURVEY section 4): singular values of the result in [0.66, 1.16] for
    # full-rank rectangular Gaussians (square Gaussians are near-singular, so skip them)
    if shape[1] != shape[2] and max(shape[1:]) <= 4096:
        sv = torch.linalg.svdvals(x[0].float().cpu())
        assert 0.64 < sv.min() and sv.max() < 1.18, (sv.min(), sv.max())


def test_newton_schulz_transpose_equivariance_and_steps(ops):
    torch.manual_seed(2)
    g = (torch.randn(1, 384, 640) * 0.1).cuda()
    x = ops.zeropower_via_newtonschulz5(g)
    xt = ops.zeropower_via_newtonschulz5(g.transpose(1, 2).contiguous())
    assert rel(xt.transpose(1, 2), x) < 2e-2          # tall path == transpose of wide path
    for steps in (1, 2, 4):
        xs = ops.zeropower_via_newtonschulz5(g, steps=steps)
        assert rel(xs, R.newton_schulz5(g.cpu().double(), steps)) < 3e-2
    z = ops.zeropower_via_newtonschulz5(torch.zeros(1, 64, 128, device="cuda"))
    assert torch.count_nonzero(z) == 0 and torch.isfinite(z.float()).all()   # eps keeps 0/0 away


# ------------------------------------------------------------------------------------------------
# elementwise optimizer kernels
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("gdt", [torch.bfloat16, torch.float32])
def test_muon_momentum_and_scales(ops, gdt):
    torch.manual_seed(3)
    batch, r, c = 3, 64, 136
    g = torch.randn(batch, r, c, device="cuda").to(gdt)
    buf = torch.randn(batch, r, c, device="cuda")
    b0 = buf.clone()
    u = torch.empty(batch, r, c, device="cuda", dtype=torch.bfloat16)
    ss = torch.empty(batch, device="cuda")
    for nesterov in (True, False):
        buf.copy_(b0)
        ops.muon_momentum(g, buf, u, ss, 0.95, nesterov, 0.5)
        gf = g.float() * 0.5
        bref = 0.05 * gf + 0.95 * b0
        uref = gf + 0.95 * bref if nesterov else bref
        assert rel(buf, bref) < 1e-6 and rel(u, uref) < 4e-3 and rel(ss, (uref ** 2).sum(dim=(1, 2))) < 1e-5
    inv, inv2 = ops.ns_scales(ss, 1e-7)
    assert rel(inv, 1 / (ss.sqrt() + 1e-7)) < 1e-6 and rel(inv2, inv * inv) < 1e-6


def test_muon_update_golden(ops, golden):
    """The product's Muon.update(model, gradients) -- momentum, Nesterov, Newton-Schulz on wgmma, scaled apply,
    SGD-momentum fallback for the 1-D parameter -- against two steps of the REFERENCE's own optimizers/muon.py
    (callable learning rate, explicit gradient dict, as the reference trainer calls it)."""
    from mlx_cuda_distributed_pretraining_b200.optimizers.muon import Muon
    names = ("w_wide", "w_tall", "gain")

    class Tiny(torch.nn.Module):
        def __init__(self):
            super().__init__()
            for k in names:
                setattr(self, k, torch.nn.Parameter(torch.from_numpy(golden[f"muon_param_{k}"]).clone()))

    model = Tiny().cuda()
    opt = Muon(learning_rate=lambda step: 0.01 * (step + 1), momentum=0.95, nesterov=True, ns_steps=5)
    for step in range(2):
        before = {k: getattr(model, k).detach().clone() for k in names}
        opt.update(model, {k: torch.from_numpy(golden[f"muon_s{step}_grad_{k}"]).cuda() for k in names})
        for k in names:
            upd = getattr(model, k).detach() - before[k]
            # 2-D updates go through bf16-operand Newton-Schulz (3e-2, like test_newton_schulz_golden); the 1-D one
            # is plain fp32 arithmetic
            assert rel(upd, golden[f"muon_s{step}_upd_{k}"]) < (3e-2 if upd.dim() == 2 else 1e-5), (step, k)
            assert rel(opt.state[k]["momentum_buffer"], golden[f"muon_s{step}_buf_{k}"]) < 1e-6, (step, k)
    assert opt.count == 2


def test_shampoo_statistics_golden(ops, golden):
    """The product Shampoo's Kronecker-factor statistics after two updates (EMA of G G^T and G^T G over the
    top-left 32 x 32 block, beta2 = 0.95) against the REFERENCE's own Shampoo._update_statistics."""
    from mlx_cuda_distributed_pretraining_b200.optimizers.shampoo import Shampoo, ShampooParams

    class Tiny(torch.nn.Module):
        def __init__(self):
            super().__init__()
            self.w = torch.nn.Parameter(torch.zeros(48, 40))

    model = Tiny().cuda()
    opt = Shampoo(learning_rate=0.01, params=ShampooParams(beta2=0.95, start_preconditioning_step=1000,
                                                           update_period=1, max_preconditioner_dim=32))
    for k in ("sh_g1", "sh_g2"):
        opt.update(model, {"w": torch.from_numpy(golden[k]).cuda()})
    # the factor products run on bf16 operands (gradients are bf16 on the training path), fp32 accumulation
    assert rel(opt.state["w"]["statistics.0"], golden["sh_stat0"]) < 1e-2
    assert rel(opt.state["w"]["statistics.1"], golden["sh_stat1"]) < 1e-2


# ------------------------------------------------------------------------------------------------
# RMSNorm / RoPE
# ------------------------------------------------------------------------------------------------
def test_linear_direct_wgrad(ops):
    """ops.linear / ops.multi_linear == nn.functional.linear; with a flat-buffer .grad the weight gradient
    is accumulated in place by the GEMM and autograd sees None."""
    torch.manual_seed(16)
    x = (torch.randn(4, 33, 256, device="cuda") * 0.5).to(torch.bfloat16).requires_grad_(True)
    ws = [(torch.randn(n, 256, device="cuda") * 0.1).to(torch.bfloat16).requires_grad_(True) for n in (128, 64, 64)]
    outs = ops.multi_linear(x, ws)
    dys = [torch.randn_like(o) for o in outs]
    torch.autograd.backward(list(outs), dys)
    xr = x.detach().float().requires_grad_(True)
    wrs = [w.detach().float().requires_grad_(True) for w in ws]
    outs_r = [torch.nn.functional.linear(xr, w) for w in wrs]
    torch.autograd.backward(outs_r, [d.float() for d in dys])
    assert all(rel(o, r) < 4e-3 for o, r in zip(outs, outs_r))
    assert rel(x.grad, xr.grad) < 6e-3
    assert all(rel(w.grad, wr.grad) < 4e-3 for w, wr in zip(ws, wrs))
    # flat-gradient mode: accumulate into the existing .grad, twice
    flat = torch.zeros(128 * 256, device="cuda", dtype=torch.bfloat16)
    w0 = ws[0].detach().clone().requires_grad_(True)
    w0.grad = flat.view(128, 256)
    w0._b200_flat_grad = True
    for _ in range(2):
        ops.linear(x.detach(), w0).backward(dys[0])
    assert w0.grad.data_ptr() == flat.data_ptr()
    assert rel(flat.view(128, 256), 2 * wrs[0].grad) < 6e-3


def test_multi_linear_fused_kv_backward(ops):
    """k/v projections: adjacent weights + [dk | dv] in one buffer -> one dgrad and one wgrad GEMM, same
    numbers as the separate GEMMs (and as fp32 autograd)."""
    torch.manual_seed(17)
    n, k_in, B, S = 64, 128, 2, 48
    wflat = (torch.randn(2 * n * k_in, device="cuda") * 0.1).to(torch.bfloat16)
    gflat = torch.zeros_like(wflat)
    wq = (torch.randn(128, k_in, device="cuda") * 0.1).to(torch.bfloat16).requires_grad_(True)
    gq = torch.zeros_like(wq)
    ws = [wq]
    for i in range(2):
        w = wflat[i * n * k_in:(i + 1) * n * k_in].view(n, k_in).requires_grad_(True)
        w.grad = gflat[i * n * k_in:(i + 1) * n * k_in].view(n, k_in)
        w._b200_flat_grad = True
        ws.append(w)
    wq.grad, wq._b200_flat_grad = gq, True
    x = (torch.randn(B, S, k_in, device="cuda") * 0.5).to(torch.bfloat16).requires_grad_(True)
    q, k, v = ops.multi_linear(x, ws)
    dq = torch.randn_like(q)
    dkv = torch.randn(B, S, 2 * n, device="cuda").to(torch.bfloat16)
    dk, dv = dkv[..., :n], dkv[..., n:]
    fused = ops._fuse_adjacent((dq, dk, dv), ws)
    assert fused is not None and len(fused) == 2 and fused[1][0].shape == (B * S, 2 * n)
    torch.autograd.backward([q, k, v], [dq, dk, dv])
    xr = x.detach().float().requires_grad_(True)
    wr = [w.detach().float().requires_grad_(True) for w in ws]
    outs = [torch.nn.functional.linear(xr, w) for w in wr]
    torch.autograd.backward(outs, [dq.float(), dk.float(), dv.float()])
    assert rel(x.grad, xr.grad) < 6e-3
    assert rel(gq, wr[0].grad) < 4e-3
    assert rel(gflat.view(2 * n, k_in), torch.cat([wr[1].grad, wr[2].grad])) < 4e-3
    # gradients that are NOT two halves of one buffer fall back to per-projection GEMMs
    assert ops._fuse_adjacent((dq, dk.contiguous(), dv.contiguous()), ws) is None


def test_rmsnorm_golden(ops, golden):
    x, w = torch.from_numpy(golden["rms_x"]).cuda(), torch.from_numpy(golden["rms_w"]).cuda()
    assert rel(ops.rmsnorm(x, w, 1e-5), golden["rms_y"]) < 2e-6


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float32])
def test_rmsnorm_deferred_weight_gradients(ops, dtype):
    """Leaf weights with a preallocated .grad (the flat store's case) get their gradient from ONE batched reduction
    at the end of the backward pass, accumulated in place; it must equal the immediate path's autograd result."""
    torch.manual_seed(11)
    rows, H, L = 777, 1024, 5
    x0 = torch.randn(rows, H, device="cuda").to(dtype)
    deltas = [torch.randn(rows, H, device="cuda").to(dtype) * 0.3 for _ in range(L)]

    def run(defer: bool, passes: int):
        ops._DW_DEFER = defer
        try:
            ws = [torch.nn.Parameter((1 + 0.1 * torch.randn(H, generator=torch.Generator().manual_seed(i))).cuda().to(dtype))
                  for i in range(L + 1)]
            for w in ws:
                w.grad = torch.zeros_like(w) if defer else None
            x = x0.clone().requires_grad_(True)
            for _ in range(passes):
                h = ops.rmsnorm(x, ws[0])
                for i in range(L):
                    h, y = ops.add_rmsnorm(h, deltas[i], ws[i + 1])
                    h = h + 0.5 * y
                (h.float() ** 2).mean().backward()
            assert not ops._PENDING_DW
            return [w.grad.float().clone() for w in ws], x.grad.float().clone()
        finally:
            ops._DW_DEFER = True

    tol = 2e-2 if dtype == torch.bfloat16 else 1e-5     # bf16: one rounding (in-place accumulate) vs two (copy + add)
    g_def, dx_def = run(True, 1)
    g_imm, dx_imm = run(False, 1)
    assert torch.equal(dx_def, dx_imm)
    for a, b in zip(g_def, g_imm):
        assert rel(a, b) < tol
    # a frozen weight (requires_grad False) takes no gradient at all
    w = torch.ones(H, device="cuda", dtype=dtype)
    x = x0.clone().requires_grad_(True)
    ops.rmsnorm(x, w).float().sum().backward()
    assert torch.isfinite(x.grad).all() and w.grad is None and not ops._PENDING_DW
    g2, _ = run(True, 2)                                 # a second backward accumulates
    for a, b in zip(g2, g_def):
        assert rel(a, 2 * b) < tol


# ------------------------------------------------------------------------------------------------
# attention
# ------------------------------------------------------------------------------------------------
def _attn_case(ops, B, S, H, Hk, D, causal, seed=7):
    torch.manual_seed(seed)
    q = torch.randn(B, S, H, D, device="cuda").to(torch.bfloat16).requires_grad_(True)
    k = torch.randn(B, S, Hk, D, device="cuda").to(torch.bfloat16).requires_grad_(True)
    v = torch.randn(B, S, Hk, D, device="cuda").to(torch.bfloat16).requires_grad_(True)
    o = ops.attention(q, k, v, D ** -0.5, causal)
    do = torch.randn_like(o)
    o.backward(do)
    qr, kr, vr = (t.detach().float().cpu().requires_grad_(True) for t in (q, k, v))
    orf = R.attention(qr, kr, vr, D ** -0.5, R.causal_mask(S) if causal else None)
    orf.backward(do.float().cpu())
    return (rel(o, orf), rel(q.grad, qr.grad), rel(k.grad, kr.grad), rel(v.grad, vr.grad))


@pytest.mark.parametrize("B,S,H,Hk,D,causal", [
    (2, 16, 4, 4, 32, True), (2, 16, 4, 1, 32, True), (2, 16, 4, 2, 32, True),   # the reference's own test matrix
    (1, 1, 2, 1, 64, True), (1, 127, 2, 2, 64, True), (1, 129, 2, 2, 64, True), (1, 200, 2, 2, 64, False),
    (2, 512, 4, 2, 64, True), (1, 384, 4, 1, 128, True), (1, 300, 2, 2, 128, False), (2, 256, 8, 8, 16, True),
    (1, 1024, 16, 8, 64, True)])
def test_attention_fwd_bwd_vs_oracle(ops, B, S, H, Hk, D, causal):
    errs = _attn_case(ops, B, S, H, Hk, D, causal)
    assert max(errs) < 1e-2, errs


def test_attention_golden(ops, golden):
    for tag in ("mha", "mqa", "gqa"):
        q, k, v = (torch.from_numpy(golden[f"attn_{tag}_{n}"]).cuda().to(torch.bfloat16) for n in "qkv")
        assert rel(ops.attention(q, k, v, 32 ** -0.5, True), golden[f"attn_{tag}_causal"]) < 1e-2, tag
        assert rel(ops.attention(q, k, v, 32 ** -0.5, False), golden[f"attn_{tag}_nomask"]) < 1e-2, tag


def test_attention_properties_full_size(ops):
    """BASELINE sizes (C2 layer: B16 S1024 H16/8 D64), checked through size-independent properties:
    causality (outputs before t do not depend on tokens >= t), GQA == explicit kv repeat,
    softmax rows sum to one (V = 1 gives O = 1), and linearity of dV in dO."""
    torch.manual_seed(8)
    B, S, H, Hk, D = 16, 1024, 16, 8, 64
    q = torch.randn(B, S, H, D, device="cuda").to(torch.bfloat16)
    k = torch.randn(B, S, Hk, D, device="cuda").to(torch.bfloat16)
    v = torch.randn(B, S, Hk, D, device="cuda").to(torch.bfloat16)
    o = ops.attention(q, k, v, D ** -0.5, True)
    k2, v2 = k.clone(), v.clone()
    k2[:, 700:], v2[:, 700:] = torch.randn_like(k2[:, 700:]), torch.randn_like(v2[:, 700:])
    o2 = ops.attention(q, k2, v2, D ** -0.5, True)
    assert torch.equal(o[:, :700], o2[:, :700])                       # causality, bit-exact
    kr, vr = k.repeat_interleave(H // Hk, dim=2), v.repeat_interleave(H // Hk, dim=2)
    assert torch.equal(ops.attention(q, kr, vr, D ** -0.5, True), o)  # GQA head sharing, bit-exact
    ones = ops.attention(q, k, torch.ones_like(v), D ** -0.5, True)
    assert float((ones.float() - 1).abs().max()) < 8e-3               # rows of P sum to 1
    qg, kg, vg = (t.clone().requires_grad_(True) for t in (q, k, v))
    og = ops.attention(qg, kg, vg, D ** -0.5, True)
    d1, d2 = torch.randn_like(og), torch.randn_like(og)
    (g1,) = torch.autograd.grad(og, vg, d1, retain_graph=True)
    (g2,) = torch.autograd.grad(og, vg, d2, retain_graph=True)
    (g12,) = torch.autograd.grad(og, vg, (d1.float() + d2.float()).to(torch.bfloat16))
    assert rel(g12, g1.float() + g2.float()) < 1e-2                   # dV is linear in dO


def test_attention_unsupported_inputs_fail_loudly(ops):
    from mlx_cuda_distributed_pretraining_b200.arch.flash_attention import FlashAttention
    attn = FlashAttention(64, 4, 2, 16).cuda().to(torch.bfloat16)
    x = torch.randn(1, 8, 64, device="cuda", dtype=torch.bfloat16)
    with pytest.raises(NotImplementedError):
        attn(x, mask=torch.zeros(1, 1, 8, 8, device="cuda"))
    with pytest.raises(ValueError):
        ops.attention(torch.zeros(1, 8, 2, 256, device="cuda", dtype=torch.bfloat16),
                      torch.zeros(1, 8, 2, 256, device="cuda", dtype=torch.bfloat16),
                      torch.zeros(1, 8, 2, 256, device="cuda", dtype=torch.bfloat16))


# ------------------------------------------------------------------------------------------------
# block-adjacent fused steps (SURVEY 8f f1): GLU activation and cross entropy
# ------------------------------------------------------------------------------------------------
def test_glu_golden(ops, golden):
    lin = torch.nn.functional.linear
    x = torch.from_numpy(golden["mlp_x"]).cuda().to(torch.bfloat16)
    w = {k: torch.from_numpy(golden[f"mlp_{k}"]).cuda().to(torch.bfloat16) for k in ("gate_proj", "up_proj", "down_proj")}
    y = lin(ops.glu(lin(x, w["gate_proj"]), lin(x, w["up_proj"])), w["down_proj"])
    assert rel(y, golden["mlp_y"]) < 2e-2


# ------------------------------------------------------------------------------------------------
# Shampoo's Kronecker-factor path through the C ABI (b200_shampoo_*) against the REFERENCE's own
# optimizers/shampoo.py outputs (tests/golden/make_golden.py).  Tolerance: fp32 matrices enter the tensor
# cores as bf16 hi+lo pairs (hi*hi + hi*lo + lo*hi, fp32 accumulation): ~2^-16 per product, 1e-4 after the
# six coupled iterations of the root.
# ------------------------------------------------------------------------------------------------
SH_TOL = 1e-4


def _split(x):
    hi = x.to(torch.bfloat16)
    return hi.contiguous(), (x - hi.float()).to(torch.bfloat16).contiguous()


def _padded(m, kp):
    out = torch.zeros(1, kp, kp, device="cuda")
    out[0, :m.shape[0], :m.shape[1]] = m
    return out


@pytest.mark.parametrize("p,key", [(0.75, "root_out_p075"), (0.5, "root_out_p05")])
def test_shampoo_root_golden(ops, golden, p, key):
    """b200_shampoo_root == MatrixSqrt.matrix_inverse_pth_root (optimizers/shampoo.py:88-126) on the
    reference-generated SPD input, both exponents."""
    m = torch.from_numpy(golden["root_in"]).cuda()
    k = m.shape[0]                       # 40: already a multiple of 8
    M = _padded(m, ops.rup8(k))
    P = torch.empty_like(M)
    Ph, Pl = torch.empty_like(M, dtype=torch.bfloat16), torch.empty_like(M, dtype=torch.bfloat16)
    ops.shampoo_root(M, P, Ph, Pl, k, p, 1e-6, 6)
    assert rel(P[0, :k, :k], golden[key]) < SH_TOL
    assert rel(Ph.float() + Pl.float(), P) < 1e-5           # hi+lo carries ~16 bits of P
    # the oracle restatement agrees too (it is what the whole-step tests use)
    assert rel(P[0, :k, :k], R.matrix_inverse_pth_root(m.cpu(), p)) < SH_TOL


def test_shampoo_root_unaligned_dimension(ops):
    """k = 37 (stored zero-padded to 40, like the byte-level embedding's 259 -> 264): same result as the
    oracle on the unpadded matrix, and the padding stays exactly zero."""
    torch.manual_seed(21)
    a = torch.randn(37, 64) * 0.3
    m = a @ a.T
    M = _padded(m.cuda(), 40)
    P = torch.empty_like(M)
    ops.shampoo_root(M, P, None, None, 37, 0.75, 1e-6, 6)
    assert rel(P[0, :37, :37], R.matrix_inverse_pth_root(m, 0.75)) < SH_TOL
    assert float(P[0, 37:].abs().max()) == 0.0 and float(P[0, :, 37:].abs().max()) == 0.0


def test_shampoo_stats_root_precondition_golden(ops, golden):
    """The three entry points chained exactly as Shampoo.update chains them, on the reference's inputs:
    two statistics updates (g1, g2; beta2 0.95; 32 x 32 block of a [48, 40] gradient) -> roots -> PL g2 PR,
    against the reference's statistics / preconditioners / preconditioned gradient."""
    cap, b2 = 32, 0.95
    L, Rm = torch.zeros(1, cap, cap, device="cuda"), torch.zeros(1, cap, cap, device="cuda")
    for key in ("sh_g1", "sh_g2"):
        gh, gl = _split(torch.from_numpy(golden[key]).cuda())
        ops.shampoo_stats(gh, gl, 40, 48 * 40, L, Rm, 1, cap, cap, b2, 1 - b2)
    assert rel(L[0], golden["sh_stat0"]) < 1e-5 and rel(Rm[0], golden["sh_stat1"]) < 1e-5
    PL, PR = torch.empty_like(L), torch.empty_like(Rm)
    hl = [torch.empty(1, cap, cap, device="cuda", dtype=torch.bfloat16) for _ in range(4)]
    ops.shampoo_root(L, PL, hl[0], hl[1], cap, 0.75, 1e-6, 6)
    ops.shampoo_root(Rm, PR, hl[2], hl[3], cap, 0.75, 1e-6, 6)
    assert rel(PL[0], golden["sh_pre0"]) < SH_TOL and rel(PR[0], golden["sh_pre1"]) < SH_TOL
    g2 = torch.from_numpy(golden["sh_g2"]).cuda()
    mh, ml = _split(g2)
    out = g2.clone().contiguous()        # pass-through part (rows >= 32, cols >= 32) must stay untouched
    ops.shampoo_precond(hl[0], hl[1], hl[2], hl[3], mh, ml, 40, 48 * 40, out, 40, 48 * 40, 1, cap, cap, 1.0)
    assert rel(out, golden["sh_preconditioned"]) < SH_TOL
    assert torch.equal(out[cap:], g2[cap:]) and torch.equal(out[:, cap:], g2[:, cap:])


def test_shampoo_graft_golden(ops, golden):
    """b200_shampoo_graft == Shampoo._apply_grafting (shampoo.py:297-312) + the parameter write; edge cases
    of the reference: zero Shampoo step -> grafting step, zero grafting step -> Shampoo step."""
    gu = torch.from_numpy(golden["graft_in_graft"]).cuda().contiguous()
    su = torch.from_numpy(golden["graft_in_shampoo"]).cuda().contiguous()
    p = torch.zeros_like(su)
    ops.shampoo_graft(p, None, su, gu, su.numel(), 1, 1.0)
    assert rel(p, golden["graft_out"]) < 1e-6
    p0 = torch.randn_like(su)
    p = p0.clone()
    p16 = torch.empty_like(p, dtype=torch.bfloat16)
    ops.shampoo_graft(p, p16, torch.zeros_like(su), gu, su.numel(), 1, 0.99)
    assert rel(p, p0 * 0.99 + gu) < 1e-6 and rel(p16, p) < 4e-3
    p = p0.clone()
    ops.shampoo_graft(p, None, su, torch.zeros_like(gu), su.numel(), 1, 1.0)
    assert rel(p, p0 + su) < 1e-6
    # batched: per-matrix norms
    up, gr = torch.randn(3, 16, 24, device="cuda"), torch.randn(3, 16, 24, device="cuda") * 0.1
    p = torch.zeros_like(up)
    ops.shampoo_graft(p, None, up, gr, 16 * 24, 3, 1.0)
    ref = up * (gr.flatten(1).norm(dim=1) / up.flatten(1).norm(dim=1))[:, None, None]
    assert rel(p, ref) < 1e-6
    # deterministic reductions: bit-identical on repetition (replica equality under data parallelism)
    q = torch.zeros_like(up)
    ops.shampoo_graft(q, None, up, gr, 16 * 24, 3, 1.0)
    assert torch.equal(p, q)


def test_shampoo_optimizer_steps_golden_and_oracle(ops, golden):
    """Product Shampoo.update(model, gradients) with fp32 gradients: (1) after the reference's two gradients
    its state holds the reference's statistics AND preconditioners; (2) three further steps against
    ShampooOracle on a well-conditioned case whose grafted step is NON-zero (finite preconditioned norm)."""
    from mlx_cuda_distributed_pretraining_b200.optimizers.shampoo import Shampoo, ShampooParams

    class Tiny(torch.nn.Module):
        def __init__(self):
            super().__init__()
            torch.manual_seed(31)
            self.w = torch.nn.Parameter(torch.randn(48, 40) * 0.1)
            self.gain = torch.nn.Parameter(torch.ones(40))

    model = Tiny().cuda()
    hp = dict(beta2=0.95, start_preconditioning_step=1, update_period=1, max_preconditioner_dim=32)
    opt = Shampoo(learning_rate=0.01, params=ShampooParams(**hp))
    oracle = R.ShampooOracle(0.01, R.ShampooParams(**hp))
    ref = {"w": model.w.detach().cpu().clone(), "gain": model.gain.detach().cpu().clone()}
    torch.manual_seed(32)
    grads = [{"w": torch.from_numpy(golden["sh_g1"]), "gain": torch.randn(40) * 0.05},
             {"w": torch.from_numpy(golden["sh_g2"]), "gain": torch.randn(40) * 0.05}]
    grads += [{"w": torch.randn(48, 40) * 0.05, "gain": torch.randn(40) * 0.05} for _ in range(3)]
    for step, g in enumerate(grads):
        before = {k: v.clone() for k, v in ref.items()}
        got_before = {"w": model.w.detach().cpu().clone(), "gain": model.gain.detach().cpu().clone()}
        opt.update(model, {k: v.cuda() for k, v in g.items()})
        oracle.update(ref, {k: v.clone() for k, v in g.items()})
        if step == 1:
            st = opt.state["w"]
            assert rel(st["statistics.0"], golden["sh_stat0"]) < 1e-5 and rel(st["statistics.1"], golden["sh_stat1"]) < 1e-5
            assert rel(st["preconditioners.0"], golden["sh_pre0"]) < SH_TOL
            assert rel(st["preconditioners.1"], golden["sh_pre1"]) < SH_TOL
        for k in ref:
            d_ref = ref[k] - before[k]
            d_got = getattr(model, k).detach().cpu() - got_before[k]
            assert float(d_ref.norm()) > 0 and torch.isfinite(d_ref).all(), (step, k)   # the step is NOT zeroed
            assert rel(d_got, d_ref) < 2e-3, (step, k, rel(d_got, d_ref))
        # keep the two trajectories glued (compare per-step updates, not accumulated drift)
        with torch.no_grad():
            model.w.copy_(ref["w"].cuda())
            model.gain.copy_(ref["gain"].cuda())
            store = model._b200_store
            store.view(store.master, "w").copy_(ref["w"].cuda())
            store.view(store.master, "gain").copy_(ref["gain"].cuda())
    assert opt.count == len(grads)


def test_shampoo_unaligned_factor_is_preconditioned(ops):
    """A [259, 64]-style block (byte-level embedding): rows 259 -> factor stored [264, 264]; the preconditioned
    step matches the oracle (previous round skipped such blocks)."""
    from mlx_cuda_distributed_pretraining_b200.optimizers.shampoo import Shampoo, ShampooParams

    class Tiny(torch.nn.Module):
        def __init__(self):
            super().__init__()
            torch.manual_seed(33)
            self.emb = torch.nn.Parameter(torch.randn(37, 24) * 0.1)

    model = Tiny().cuda()
    hp = dict(beta2=0.95, start_preconditioning_step=1, update_period=1, max_preconditioner_dim=1024)
    opt = Shampoo(learning_rate=0.01, params=ShampooParams(**hp))
    assert opt is not None
    oracle = R.ShampooOracle(0.01, R.ShampooParams(**hp))
    ref = {"emb": model.emb.detach().cpu().clone()}
    torch.manual_seed(34)
    for step in range(2):
        g = torch.randn(37, 24) * 0.05
        before = ref["emb"].clone()
        opt.update(model, {"emb": g.cuda()})
        oracle.update(ref, {"emb": g.clone()})
        d_ref = ref["emb"] - before
        d_got = model.emb.detach().cpu() - before
        assert float(d_ref.norm()) > 0
        assert rel(d_got, d_ref) < 2e-3, (step, rel(d_got, d_ref))
        with torch.no_grad():
            store = model._b200_store
            store.view(store.master, "emb").copy_(ref["emb"].cuda())
            model.emb.copy_(ref["emb"].cuda())
    assert opt.state["emb"]["statistics.0"].shape == (37, 37)
    assert opt.state["emb"]["preconditioners.1"].shape == (24, 24)


# ------------------------------------------------------------------------------------------------
# BASELINE shapes: attention at S = 2048 (C3 / C4 / C5 dims) and Newton-Schulz at C5's 2048-wide matrices
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("B,S,H,Hk,D", [(16, 2048, 16, 8, 64),    # C3 per-GPU micro-batch (GQA 16/8)
                                        (8, 2048, 16, 16, 64),    # C4 dims (MHA), 1/8 of its batch
                                        (4, 2048, 16, 16, 128)])  # C5 dims (D = 128, 16 key tiles), 1/8 of its batch
def test_attention_baseline_shapes_vs_oracle(ops, B, S, H, Hk, D):
    """Forward and backward at the BASELINE attention shapes (arch/flash_attention.py:78-156 at the C3/C4/C5
    dims).  The kernel runs the FULL launch; the oracle (dense fp32 softmax(QK^T)V + autograd, ~1 GB of scores
    per batch row) is evaluated on the first and last batch rows -- rows are independent, so this checks every
    (tile, head) code path of the full-size grid."""
    torch.manual_seed(40 + D)
    q = torch.randn(B, S, H, D, device="cuda").to(torch.bfloat16).requires_grad_(True)
    k = torch.randn(B, S, Hk, D, device="cuda").to(torch.bfloat16).requires_grad_(True)
    v = torch.randn(B, S, Hk, D, device="cuda").to(torch.bfloat16).requires_grad_(True)
    o = ops.attention(q, k, v, D ** -0.5, True)
    do = torch.randn_like(o)
    o.backward(do)
    mask = R.causal_mask(S)
    for b in (0, B - 1):
        qr, kr, vr = (t[b:b + 1].detach().float().cpu().requires_grad_(True) for t in (q, k, v))
        orf = R.attention(qr, kr, vr, D ** -0.5, mask)
        orf.backward(do[b:b + 1].float().cpu())
        errs = (rel(o[b:b + 1], orf), rel(q.grad[b:b + 1], qr.grad), rel(k.grad[b:b + 1], kr.grad),
                rel(v.grad[b:b + 1], vr.grad))
        assert max(errs) < 1e-2, (b, errs)


@pytest.mark.parametrize("shape", [(1, 2048, 2048), (2, 2048, 5632), (1, 5632, 2048)])
def test_newton_schulz_c5_shapes(ops, shape):
    """m = 2048 (C5's hidden size): X is stored bf16 between iterations, so the error budget is checked at the
    widest matrices of the BASELINE configs too (fp32 oracle; fp64 would take minutes on the host)."""
    torch.manual_seed(50)
    g = torch.randn(*shape) * 0.02
    x = ops.zeropower_via_newtonschulz5(g.cuda())
    assert rel(x, R.newton_schulz5(g)) < 3e-2


def test_newton_schulz_grouped_chain_matches_per_group(ops):
    """b200_newton_schulz_multi (one grouped launch per stage over all shape groups, run-time operand layouts,
    in-launch split-K of a lone tall matrix) against the per-group chain and the oracle: wide, tall, square and a
    split-K group in the same launch.  Same tiles, same accumulation order -> bit-identical to the per-group
    kernels wherever the split-K choice is the same."""
    torch.manual_seed(60)
    shapes = [(3, 256, 512), (2, 768, 256), (2, 512, 512), (1, 5000, 512), (4, 384, 1024)]
    gs = [(torch.randn(*s) * 0.02).cuda() for s in shapes]
    outs = ops.zeropower_groups(gs)
    for g, x, s in zip(gs, outs, shapes):
        single = ops.zeropower_via_newtonschulz5(g)
        assert rel(x, single) < 2e-3, s
        assert rel(x, R.newton_schulz5(g.cpu().double())) < 3e-2, s
    assert torch.equal(outs[0], ops.zeropower_via_newtonschulz5(gs[0]))     # no split-K involved: same bits
    # groups too small for the CTA-pair kernel take the per-group fallback inside the same entry point
    small = [(torch.randn(2, 64, 136) * 0.1).cuda(), (torch.randn(1, 136, 72) * 0.1).cuda()]
    for g, x in zip(small, ops.zeropower_groups(small)):
        assert torch.equal(x, ops.zeropower_via_newtonschulz5(g))


@pytest.mark.parametrize("B,S,H,Hk,D", [(2, 256, 8, 8, 16), (1, 200, 4, 2, 32), (2, 130, 4, 4, 40)])
def test_attention_fp32_path_large_logits(ops, B, S, H, Hk, D):
    """Full-precision configs (mixed_precision: false; BASELINE C1 has head_dim 16): bf16x3 logits.  With LARGE
    scores (|s| ~ 40, the regime a 2e-2-lr AdamW run reaches) plain bf16 operands put an error of |s| * 2^-9 in
    the exponent; the three-term path must stay at the bf16-OUTPUT rounding level, several times better."""
    torch.manual_seed(70 + D)
    q = (torch.randn(B, S, H, D, device="cuda") * 4).requires_grad_(True)
    k = (torch.randn(B, S, Hk, D, device="cuda") * 4).requires_grad_(True)
    v = torch.randn(B, S, Hk, D, device="cuda").requires_grad_(True)
    do = torch.randn(B, S, H, D, device="cuda")
    o = ops.attention_fp32(q, k, v, D ** -0.5, True)
    o.backward(do)
    qr, kr, vr = (t.detach().double().cpu().requires_grad_(True) for t in (q, k, v))
    orf = R.attention(qr, kr, vr, D ** -0.5, R.causal_mask(S, dtype=torch.float64))
    orf.backward(do.double().cpu())
    errs = (rel(o, orf), rel(q.grad, qr.grad), rel(k.grad, kr.grad), rel(v.grad, vr.grad))
    assert max(errs) < 8e-3, errs
    # the plain bf16-operand path on the same inputs, for the record: must be clearly worse on the logits side
    qb, kb, vb = (t.detach().to(torch.bfloat16).requires_grad_(True) for t in (q, k, v))
    ob = ops.attention(qb, kb, vb, D ** -0.5, True)
    assert rel(ob, orf) > 2 * errs[0], (rel(ob, orf), errs[0])


@pytest.mark.parametrize("M,K,I", [(300, 128, 256), (1024, 1024, 2816), (515, 256, 384)])
def test_mlp_fused_glu_epilogues(ops, M, K, I):
    """The MLP block on the in-tree GEMM engine (b200_mlp_gateup_glu_fwd / b200_mlp_down_glu_bwd: gate*sigmoid(up)*2 and
    its adjoint inside the wgmma epilogues, arch/llama.py:149-151) against fp32 autograd of the same formula, and
    against the unfused path (library GEMMs + glu kernels)."""
    torch.manual_seed(80 + I)
    wflat = (torch.randn(2 * I * K, device="cuda") * K ** -0.5).to(torch.bfloat16)
    gflat = torch.zeros_like(wflat)
    ws = []
    for i in range(2):
        w = wflat[i * I * K:(i + 1) * I * K].view(I, K).requires_grad_(True)
        w.grad = gflat[i * I * K:(i + 1) * I * K].view(I, K)
        w._b200_flat_grad = True
        ws.append(w)
    wg, wu = ws
    wd = (torch.randn(K, I, device="cuda") * I ** -0.5).to(torch.bfloat16).requires_grad_(True)
    wd.grad = torch.zeros_like(wd)
    wd._b200_flat_grad = True
    x = torch.randn(2, M // 2 if M % 2 == 0 else M, K, device="cuda").to(torch.bfloat16)
    x = x.reshape(-1, K)[:M].reshape(1, M, K).contiguous().requires_grad_(True)
    assert ops.mlp_fusable(x, wg, wu, wd)
    out = ops.mlp(x, wg, wu, wd)
    dout = torch.randn_like(out)
    out.backward(dout)
    xr = x.detach().float().requires_grad_(True)
    wr = [w.detach().float().requires_grad_(True) for w in (wg, wu, wd)]
    lin = torch.nn.functional.linear
    ref = lin(lin(xr, wr[0]) * torch.sigmoid(lin(xr, wr[1])) * 2, wr[2])
    ref.backward(dout.float())
    assert rel(out, ref) < 8e-3
    assert rel(x.grad, xr.grad) < 1.2e-2
    assert rel(gflat.view(2 * I, K), torch.cat([wr[0].grad, wr[1].grad])) < 1.2e-2
    assert rel(wd.grad, wr[2].grad) < 8e-3
    # raw entry points: [g | u] and y
    gu = torch.empty(M, 2 * I, device="cuda", dtype=torch.bfloat16)
    y = torch.empty(M, I, device="cuda", dtype=torch.bfloat16)
    x2 = x.detach().reshape(M, K)
    ops.check(ops.lib().b200_mlp_gateup_glu_fwd(x2.data_ptr(), wg.data_ptr(), gu.data_ptr(), y.data_ptr(), M, K, I,
                                                ops._stream()), "fwd")
    g_ref, u_ref = lin(x2.float(), wr[0].detach()), lin(x2.float(), wr[1].detach())
    assert rel(gu[:, :I], g_ref) < 4e-3 and rel(gu[:, I:], u_ref) < 4e-3
    assert rel(y, g_ref * torch.sigmoid(u_ref) * 2) < 4e-3


def test_shampoo_root_and_precondition_at_c4_size(ops):
    """BASELINE C4 shapes: the [1024, 1024] Kronecker factors of a [2816, 1024] parameter (max_preconditioner_dim
    1024), batched.  Statistics from bf16 gradients -> roots -> PL m PR against the oracle in fp64/fp32 on the host;
    same 1e-4 (root) / 2e-4 (two chained bf16x3 products) bounds as the small golden cases."""
    torch.manual_seed(95)
    b, rows, cols, k = 2, 2816, 1024, 1024
    G = (torch.randn(b, rows, cols) * 0.02).to(torch.bfloat16)
    Gc = G.cuda()
    L = torch.zeros(b, k, k, device="cuda")
    Rm = torch.zeros(b, k, k, device="cuda")
    ops.shampoo_stats(Gc, None, cols, rows * cols, L, Rm, b, k, k, 0.95, 0.05)
    gf = G.float()[:, :k, :k]
    assert rel(L, 0.05 * gf @ gf.transpose(1, 2)) < 1e-5 and rel(Rm, 0.05 * gf.transpose(1, 2) @ gf) < 1e-5
    PL, PR = torch.empty_like(L), torch.empty_like(Rm)
    hl = [torch.empty(b, k, k, device="cuda", dtype=torch.bfloat16) for _ in range(4)]
    ops.shampoo_root(L, PL, hl[0], hl[1], k, 0.75, 1e-6, 6)
    ops.shampoo_root(Rm, PR, hl[2], hl[3], k, 0.75, 1e-6, 6)
    for i in range(b):
        assert rel(PL[i], R.matrix_inverse_pth_root(L[i].cpu(), 0.75)) < SH_TOL, i
        assert rel(PR[i], R.matrix_inverse_pth_root(Rm[i].cpu(), 0.75)) < SH_TOL, i
    m = torch.randn(b, rows, cols) * 0.01
    mh, ml = _split(m.cuda())
    out = m.cuda().clone().contiguous()
    ops.shampoo_precond(hl[0], hl[1], hl[2], hl[3], mh, ml, cols, rows * cols, out, cols, rows * cols, b, k, k, -0.01)
    ref = m.clone()
    for i in range(b):
        ref[i, :k, :k] = -0.01 * (PL[i].cpu().double() @ m[i, :k, :k].double() @ PR[i].cpu().double()).float()
    assert rel(out, ref) < 2e-4
    assert torch.equal(out[:, k:], m.cuda()[:, k:])          # rows beyond the preconditioned block pass through
