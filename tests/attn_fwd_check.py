"""fp64 reference and element-wise checker for the attention forward (attn_fwd_kernel, csrc/attention_fwd.cu), and
the visibility-mask builder it shares with tests/attn_bwd_check.py.

The kernel computes, per 128-key tile, logits s = q.k in fp32 (bf16 products are exact, the D-term sum is not),
x = s * scale * log2(e), an online softmax in the log2 domain (running max m, normaliser l summed from the unrounded
p = 2^(x - m)), P rounded to bf16 for the PV MMA, O accumulated in fp32 and rescaled by 2^(m_old - m_new), and at the
end O / l rounded to bf16 and LSE = (m + log2 l) / log2(e) in fp32.  With P the exact softmax, R = P V and n = S
(the longest sum any row can run; the backward checker uses the same n):

  logits   |s~ - s| <~ c * 2^-24 * D * scale * |q|.|k| + 2^-24 |s|; exp2 turns an absolute logit error e into a
           relative error e of p, so every p_j carries a relative error c * 2^-24 * D * amp_j, where
           amp = 1 + scale * |q| @ |k|^T is the logit magnitude (the 1 covers the exp2 / rescale roundings)
  l        fp32 sum of n terms: relative error c * 2^-24 * (n + D * sum_j p_j amp_j)
  O        2^-8 * (|P| @ |V|)                     P rounded to bf16 before the PV MMA
         + C32 * 2^-24 * (D + n) * ((|P| o amp) @ |V|)   fp32 logits, fp32 PV over n keys, the normaliser l
         + 2^-8 * |R|                             bf16 output
  LSE      LSE - R = (log2 l~ - log2 l) / log2(e) + rounding = ln(l~ / l) + ..., so
           |LSE - R| <= C32 * 2^-24 * ((D + n) * sum_j p_j amp_j + |R|)
           (the relative error of l becomes an absolute error of LSE; m + log2 l and the division add 2^-24 |R|)

The bf16x3 path (ops.attention_fp32, D <= 42) splits each fp32 operand into hi + lo bf16 halves laid along the head
dimension of one bf16 kernel call.  Its logits qh kh + ql kh + qh kl miss ql kl and the roundings of the lo halves,
about 3 * 2^-16 * |q|.|k|, which adds C16 * 2^-16 * ((|P| o amp) @ |V|) to O and C16 * 2^-16 * sum_j p_j amp_j to LSE.
Its output is bf16(P vh) + bf16(P vl): the second rounding and vl's own rounding add 2 * 2^-16 * (|P| @ |V|).

C32 = 4 (the backward's constant) and C16 = 4.  The largest ratios observed on an H100 are in DESIGN.md section 5.
"""
from __future__ import annotations

import math

import torch

C32 = 4.0
C16 = 4.0
U8, U16, U24 = 2.0 ** -8, 2.0 ** -16, 2.0 ** -24
LOG2E = 1.0 / math.log(2.0)


def visible(S, causal=True, pos=None, window=None, device="cpu"):
    """Boolean visibility mask, [S, S] or [B, S, S] (with pos [B, S]): query q sees key k iff k <= q (causal) and
    k >= q - min(pos[q], W).  pos = None means pos[q] = q; no window means W = S.  Non-causal: every key."""
    if not causal:
        if pos is not None or window is not None:
            raise ValueError("documents and windows are causal")
        return torch.ones(S, S, dtype=torch.bool, device=device)
    s = torch.arange(S, device=device)
    p = s if pos is None else pos.to(device=device, dtype=torch.int64)
    W = S if window is None else window
    start = (s - torch.clamp(p, max=W))[..., None]      # [S, 1] or [B, S, 1]
    return (s[None, :] <= s[:, None]) & (s[None, :] >= start)


def _row_mask(mask, b):
    if mask is None:
        return None
    return mask[b] if mask.dim() == 3 else mask


def _heads(q, k, v, b, h0, h1):
    """fp64 [h, S, D] slices of batch row b for query heads h0..h1-1, their kv heads repeated (GQA)."""
    g = q.shape[2] // k.shape[2]
    qd = q[b, :, h0:h1].double().transpose(0, 1)
    idx = torch.arange(h0, h1, device=q.device) // g
    kd = k[b].double().transpose(0, 1)[idx]
    vd = v[b].double().transpose(0, 1)[idx]
    return qd, kd, vd


def forward64(q, k, v, scale, mask=None, rows=None, head_chunk=4):
    """fp64 O [len(rows), S, H, D] and LSE [len(rows), H, S] of [B,S,H,D] / [B,S,Hk,D] inputs under a visibility
    mask (None: all keys)."""
    return _run(q, k, v, scale, mask, rows, head_chunk, bounds=False)


def reference(q, k, v, scale, mask=None, rows=None, kernel_d=None, x3=False, head_chunk=4):
    """fp64 O and LSE of the batch rows `rows` with their element-wise bounds (module docstring).  kernel_d: the head
    dim the kernel accumulates over (the padded one); x3: the bf16x3 path.  Returns {"o": (ref, bound),
    "lse": (ref, bound)} with o [len(rows), S, H, D] and lse [len(rows), H, S]."""
    return _run(q, k, v, scale, mask, rows, head_chunk, bounds=True, kernel_d=kernel_d, x3=x3)


def _run(q, k, v, scale, mask, rows, head_chunk, bounds, kernel_d=None, x3=False):
    B, S, H, D = q.shape
    Dk = kernel_d or D
    rows = range(B) if rows is None else rows
    o_all, lse_all, bo_all, bl_all = [], [], [], []
    n = S
    for b in rows:
        m = _row_mask(mask, b)
        os_, ls_, bos, bls = [], [], [], []
        for h0 in range(0, H, head_chunk):
            h1 = min(H, h0 + head_chunk)
            qd, kd, vd = _heads(q, k, v, b, h0, h1)
            s = scale * qd @ kd.transpose(-1, -2)
            if m is not None:
                s = s.masked_fill(~m, float("-inf"))
            lse = torch.logsumexp(s, -1)
            p = torch.exp(s - lse[..., None])
            del s
            o = p @ vd
            os_.append(o)
            ls_.append(lse)
            if bounds:
                pa = p * (1.0 + scale * qd.abs() @ kd.abs().transpose(-1, -2))
                pv, pav = p @ vd.abs(), pa @ vd.abs()
                spa = pa.sum(-1)
                del p, pa
                bo = U8 * pv + U8 * o.abs() + C32 * U24 * (Dk + n) * pav
                bl = C32 * U24 * ((Dk + n) * spa + lse.abs())
                if x3:
                    bo = bo + 2 * U16 * pv + C16 * U16 * pav
                    bl = bl + C16 * U16 * spa
                bos.append(bo)
                bls.append(bl)
        o_all.append(torch.cat(os_).transpose(0, 1))
        lse_all.append(torch.cat(ls_))
        if bounds:
            bo_all.append(torch.cat(bos).transpose(0, 1))
            bl_all.append(torch.cat(bls))
    o, lse = torch.stack(o_all), torch.stack(lse_all)
    if not bounds:
        return o, lse
    return {"o": (o, torch.stack(bo_all)), "lse": (lse, torch.stack(bl_all))}


def check(name, got, ref, bound, tiny=1e-30):
    """Element-wise |got - ref| <= bound for O ([row, token, head, d]) or LSE ([row, head, token]); returns the largest
    error / bound ratio and raises naming the worst element, its CTA's 128-query tile and that token's key tile."""
    err = (got.double() - ref).abs()
    ratio = err / (bound + tiny)
    worst = float(ratio.max())
    if not torch.isfinite(got).all() or worst > 1.0:
        i = int(torch.nan_to_num(ratio, nan=float("inf")).flatten().argmax())
        idx = [int(x) for x in torch.unravel_index(torch.tensor(i), ratio.shape)]
        if ratio.dim() == 4:
            where, tok = "[row, token, head, d]", idx[1]
        else:
            where, tok = "[row, head, token]", idx[2]
        raise AssertionError(f"{name}: worst error/bound {worst:.3g} at {where} = {idx} (128-query tile {tok // 128}, "
                             f"the token's own key in 128-key tile {tok // 128}): got {float(got.flatten()[i]):.6g} "
                             f"ref {float(ref.flatten()[i]):.6g} bound {float(bound.flatten()[i]):.3g}")
    return worst


def emulate_kernel(q, k, v, scale, mask=None, tile=128):
    """CPU emulation of the kernel's arithmetic for bf16 inputs: 128-key tiles, online softmax in the log2 domain,
    P rounded to bf16 before PV, l summed from the unrounded P, fp32 throughout.  Returns (o bf16 [B,S,H,D],
    lse fp32 [B,H,S]).  A legitimate kernel (any reduction order) sits within the bound as this does."""
    B, S, H, D = q.shape
    g = H // k.shape[2]
    sl2 = torch.tensor(scale * LOG2E, dtype=torch.float32)
    os_, ls_ = [], []
    for b in range(B):
        qf = q[b].float().transpose(0, 1)
        kf = k[b].float().transpose(0, 1).repeat_interleave(g, 0)
        vf = v[b].float().transpose(0, 1).repeat_interleave(g, 0)
        mk = _row_mask(mask, b)
        m = torch.full((H, S, 1), float("-inf"))
        l = torch.zeros(H, S, 1)
        o = torch.zeros(H, S, D)
        for k0 in range(0, S, tile):
            k1 = min(S, k0 + tile)
            x = (qf @ kf[:, k0:k1].transpose(-1, -2)) * sl2
            if mk is not None:
                x = x.masked_fill(~mk[:, k0:k1], float("-inf"))
            m_new = torch.maximum(m, x.amax(-1, keepdim=True))
            m_use = torch.where(m_new == float("-inf"), torch.zeros_like(m_new), m_new)
            alpha = torch.exp2(m - m_use)
            pe = torch.exp2(x - m_use)
            l = l * alpha + pe.sum(-1, keepdim=True)
            o = o * alpha + pe.to(torch.bfloat16).float() @ vf[:, k0:k1]
            m = m_new
        os_.append((o * (1.0 / l)).to(torch.bfloat16).transpose(0, 1))
        ls_.append(((m + torch.log2(l)) / torch.tensor(LOG2E, dtype=torch.float32))[..., 0])
    return torch.stack(os_), torch.stack(ls_)
