// HBM-bound elementwise / reduction kernels of the optimizer step (one coalesced 128-bit pass each).
//
//  muon_momentum   optimizers/muon.py:101,105  buf=(1-mu)g+mu*buf ; u=g+mu*buf ; + per-matrix sum(u^2)
//  ns_scales       optimizers/muon.py:72-73    1/(||u||_F+eps) and its square
//  axpy_update     optimizers/muon.py:111-114  p += s*X ; bf16 shadow copy refreshed in the same pass
//  sgd_momentum    optimizers/muon.py:123-138  non-2-D fallback
//  adamw           core/training.py:821 (mlx.optimizers.AdamW; formula also enhanced_optimizers.py:157-184)
//  lion            optimizers/enhanced_optimizers.py:358-488 LionEnhanced (+ Chen et al.'s variant)
//  sgd             enhanced_optimizers.py:200-355 SGDEnhanced; mlx.optimizers.SGD (core/training.py:891-894)
//  clip_accum      core/training.py:1664-1666,1671-1680  clamp to +-clip, scale by 1/k, accumulate
//  sumsq           Frobenius norms for Shampoo grafting (optimizers/shampoo.py:300-310)
//
// All kernels work on flat contiguous ranges: the optimizer keeps parameters, gradients and state
// in shape-grouped flat buffers, so a "multi-tensor" update is just one launch over a range.
#include "common.cuh"
#include "host.h"

namespace b200 {

namespace {

constexpr int EW_THREADS = 256;

__device__ __forceinline__ void load8(const float* p, float* f) {
  const float4 a = *reinterpret_cast<const float4*>(p);
  const float4 b = *reinterpret_cast<const float4*>(p + 4);
  f[0] = a.x; f[1] = a.y; f[2] = a.z; f[3] = a.w;
  f[4] = b.x; f[5] = b.y; f[6] = b.z; f[7] = b.w;
}
__device__ __forceinline__ void load8(const __nv_bfloat16* p, float* f) {
  const uint4 a = *reinterpret_cast<const uint4*>(p);
  const float2 v0 = unpack_bf16x2(a.x), v1 = unpack_bf16x2(a.y), v2 = unpack_bf16x2(a.z),
               v3 = unpack_bf16x2(a.w);
  f[0] = v0.x; f[1] = v0.y; f[2] = v1.x; f[3] = v1.y;
  f[4] = v2.x; f[5] = v2.y; f[6] = v3.x; f[7] = v3.y;
}
__device__ __forceinline__ void store8(float* p, const float* f) {
  *reinterpret_cast<float4*>(p) = make_float4(f[0], f[1], f[2], f[3]);
  *reinterpret_cast<float4*>(p + 4) = make_float4(f[4], f[5], f[6], f[7]);
}
__device__ __forceinline__ void store8(__nv_bfloat16* p, const float* f) {
  uint4 o;
  o.x = pack_bf16x2(f[0], f[1]);
  o.y = pack_bf16x2(f[2], f[3]);
  o.z = pack_bf16x2(f[4], f[5]);
  o.w = pack_bf16x2(f[6], f[7]);
  *reinterpret_cast<uint4*>(p) = o;
}
__device__ __forceinline__ float ldf(const float* p) { return *p; }
__device__ __forceinline__ float ldf(const __nv_bfloat16* p) { return __bfloat162float(*p); }
__device__ __forceinline__ void stf(float* p, float v) { *p = v; }
__device__ __forceinline__ void stf(__nv_bfloat16* p, float v) { *p = __float2bfloat16_rn(v); }

// The last, partial vector of a range whose length is not a multiple of 8: `cnt` valid elements, the other lanes 0.
// A kernel that sends it through the same arithmetic as the full vectors gives every element the same bits wherever
// it falls in a flat buffer (the compiler contracts a separate scalar loop's multiply-adds differently).
template <typename T>
__device__ __forceinline__ void load8n(const T* p, float* f, int cnt) {
  if (cnt == 8) return load8(p, f);
#pragma unroll
  for (int j = 0; j < 8; ++j) f[j] = j < cnt ? ldf(p + j) : 0.f;
}
template <typename T>
__device__ __forceinline__ void store8n(T* p, const float* f, int cnt) {
  if (cnt == 8) return store8(p, f);
#pragma unroll
  for (int j = 0; j < 8; ++j)
    if (j < cnt) stf(p + j, f[j]);
}

__device__ __forceinline__ float block_sum(float v) {
  __shared__ float red[EW_THREADS / 32];
  v = warp_sum(v);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
  __syncthreads();
  float t = 0.f;
  if (threadIdx.x < 32) {
    t = threadIdx.x < EW_THREADS / 32 ? red[threadIdx.x] : 0.f;
    t = warp_sum(t);
  }
  __syncthreads();
  return t;  // valid in warp 0
}

// Deterministic grid reduction (no float atomics: data-parallel replicas must compute bit-identical norms,
// or their fp32 masters drift apart).  Every block parks its partial in `partials[batch][gridDim.x]`; the
// block that arrives last at the per-matrix counter sums the partials in a fixed order and owns out[b].
// `tot` must be valid in thread 0.  Counters are zeroed by the host wrapper before the launch.
__device__ __forceinline__ void grid_reduce_finish(float tot, float* __restrict__ partials,
                                                   unsigned* __restrict__ counters, float* __restrict__ out,
                                                   int accumulate) {
  __shared__ bool is_last;
  const int b = blockIdx.y;
  if (threadIdx.x == 0) {
    partials[(long long)b * gridDim.x + blockIdx.x] = tot;
    __threadfence();
    is_last = atomicAdd(counters + b, 1u) == gridDim.x - 1;
  }
  __syncthreads();
  if (!is_last) return;
  __threadfence();
  float s = 0.f;
  for (unsigned i = threadIdx.x; i < gridDim.x; i += EW_THREADS)
    s += *reinterpret_cast<volatile float*>(partials + (long long)b * gridDim.x + i);
  s = block_sum(s);
  if (threadIdx.x == 0) {
    out[b] = accumulate ? out[b] + s : s;
    counters[b] = 0;
  }
}

// grid = (blocks_per_matrix, batch); every block stays inside one matrix so the Frobenius partial
// sum goes to a single accumulator.
template <typename G>
__global__ void __launch_bounds__(EW_THREADS)
muon_momentum_kernel(const G* __restrict__ g, float* __restrict__ buf, __nv_bfloat16* __restrict__ u,
                     float* __restrict__ sumsq, long long numel, float mu, int nesterov,
                     float gscale, float* __restrict__ partials, unsigned* __restrict__ counters) {
  const long long base = (long long)blockIdx.y * numel;
  const G* gp = g + base;
  float* bp = buf + base;
  __nv_bfloat16* up = u + base;
  const float omm = 1.0f - mu;
  float ss = 0.f;
  const long long nvec = numel / 8;
  for (long long i = (long long)blockIdx.x * EW_THREADS + threadIdx.x; i < nvec;
       i += (long long)gridDim.x * EW_THREADS) {
    float gv[8], bv[8], uv[8];
    load8(gp + i * 8, gv);
    load8(bp + i * 8, bv);
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const float gj = gv[j] * gscale;
      bv[j] = omm * gj + mu * bv[j];
      uv[j] = nesterov ? gj + mu * bv[j] : bv[j];
      ss += uv[j] * uv[j];
    }
    store8(bp + i * 8, bv);
    store8(up + i * 8, uv);
  }
  // tail (numel % 8) handled by block 0
  if (blockIdx.x == 0) {
    for (long long i = nvec * 8 + threadIdx.x; i < numel; i += EW_THREADS) {
      const float gj = ldf(gp + i) * gscale;
      const float b = omm * gj + mu * bp[i];
      const float uu = nesterov ? gj + mu * b : b;
      bp[i] = b;
      up[i] = __float2bfloat16_rn(uu);
      ss += uu * uu;
    }
  }
  const float tot = block_sum(ss);
  grid_reduce_finish(tot, partials, counters, sumsq, 0);
}

__global__ void ns_scales_kernel(const float* __restrict__ sumsq, float* __restrict__ inv_norm,
                                 float* __restrict__ inv_norm_sq, int batch, float eps) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < batch) {
    const float inv = 1.0f / (sqrtf(sumsq[i]) + eps);
    inv_norm[i] = inv;
    inv_norm_sq[i] = inv * inv;
  }
}

// p32 += s * x ; p16 = bf16(p32)   (x: bf16 Newton-Schulz output or fp32 direction)
template <typename X>
__global__ void __launch_bounds__(EW_THREADS)
axpy_update_kernel(float* __restrict__ p32, __nv_bfloat16* __restrict__ p16,
                   const X* __restrict__ x, long long n, float s) {
  const long long nvec = n / 8;
  for (long long i = (long long)blockIdx.x * EW_THREADS + threadIdx.x; i < nvec;
       i += (long long)gridDim.x * EW_THREADS) {
    float pv[8], xv[8];
    load8(p32 + i * 8, pv);
    load8(x + i * 8, xv);
#pragma unroll
    for (int j = 0; j < 8; ++j) pv[j] = fmaf(s, xv[j], pv[j]);
    store8(p32 + i * 8, pv);
    if (p16) store8(p16 + i * 8, pv);
  }
  if (blockIdx.x == 0) {
    for (long long i = nvec * 8 + threadIdx.x; i < n; i += EW_THREADS) {
      const float v = fmaf(s, ldf(x + i), p32[i]);
      p32[i] = v;
      if (p16) p16[i] = __float2bfloat16_rn(v);
    }
  }
}

template <typename G>
__global__ void __launch_bounds__(EW_THREADS)
sgd_momentum_kernel(float* __restrict__ p32, __nv_bfloat16* __restrict__ p16,
                    const G* __restrict__ g, float* __restrict__ buf, long long n, float mu,
                    int nesterov, float lr, float gscale) {
  const float omm = 1.0f - mu;
  const long long nvec = n / 8;
  for (long long i = (long long)blockIdx.x * EW_THREADS + threadIdx.x; i < nvec;
       i += (long long)gridDim.x * EW_THREADS) {
    float gv[8], bv[8], pv[8];
    load8(g + i * 8, gv);
    load8(buf + i * 8, bv);
    load8(p32 + i * 8, pv);
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const float gj = gv[j] * gscale;
      bv[j] = omm * gj + mu * bv[j];
      pv[j] -= lr * (nesterov ? gj + mu * bv[j] : bv[j]);
    }
    store8(buf + i * 8, bv);
    store8(p32 + i * 8, pv);
    if (p16) store8(p16 + i * 8, pv);
  }
  if (blockIdx.x == 0) {
    for (long long i = nvec * 8 + threadIdx.x; i < n; i += EW_THREADS) {
      const float gj = ldf(g + i) * gscale;
      const float b = omm * gj + mu * buf[i];
      const float uu = nesterov ? gj + mu * b : b;
      buf[i] = b;
      const float v = p32[i] - lr * uu;
      p32[i] = v;
      if (p16) p16[i] = __float2bfloat16_rn(v);
    }
  }
}

// MLX AdamW semantics: p *= (1 - lr*wd); m,v EMA; p -= (lr/bc1) * m / (sqrt(v)/sqrt(bc2) + eps)
// (bc1 = bc2 = 1 reproduces mlx 0.25's default bias_correction=False).
template <typename G>
__global__ void __launch_bounds__(EW_THREADS)
adamw_kernel(float* __restrict__ p32, __nv_bfloat16* __restrict__ p16, const G* __restrict__ g,
             float* __restrict__ m, float* __restrict__ v, long long n, float lr, float b1,
             float b2, float eps, float wd, float bc1, float bc2, float gscale) {
  const float step = lr / bc1;
  const float rs_bc2 = rsqrtf(bc2);
  const float decay = 1.0f - lr * wd;
  const long long nvec = n / 8;
  for (long long i = (long long)blockIdx.x * EW_THREADS + threadIdx.x; i < nvec;
       i += (long long)gridDim.x * EW_THREADS) {
    float pv[8], gv[8], mv[8], vv[8];
    load8(p32 + i * 8, pv);
    load8(g + i * 8, gv);
    load8(m + i * 8, mv);
    load8(v + i * 8, vv);
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const float gj = gv[j] * gscale;
      mv[j] = b1 * mv[j] + (1.0f - b1) * gj;
      vv[j] = b2 * vv[j] + (1.0f - b2) * gj * gj;
      pv[j] = pv[j] * decay - step * mv[j] / (sqrtf(vv[j]) * rs_bc2 + eps);
    }
    store8(p32 + i * 8, pv);
    store8(m + i * 8, mv);
    store8(v + i * 8, vv);
    if (p16) store8(p16 + i * 8, pv);
  }
  if (blockIdx.x == 0) {
    for (long long i = nvec * 8 + threadIdx.x; i < n; i += EW_THREADS) {
      const float gj = ldf(g + i) * gscale;
      const float mm = b1 * m[i] + (1.0f - b1) * gj;
      const float vv = b2 * v[i] + (1.0f - b2) * gj * gj;
      const float pp = p32[i] * decay - step * mm / (sqrtf(vv) * rs_bc2 + eps);
      m[i] = mm;
      v[i] = vv;
      p32[i] = pp;
      if (p16) p16[i] = __float2bfloat16_rn(pp);
    }
  }
}

// Adam direction without applying it (Shampoo grafting): d = -(lr/bc1) * m/(sqrt(v)/sqrt(bc2)+eps)
template <typename G>
__global__ void __launch_bounds__(EW_THREADS)
adam_direction_kernel(float* __restrict__ d, const G* __restrict__ g, float* __restrict__ m,
                      float* __restrict__ v, long long n, float lr, float b1, float b2, float eps,
                      float bc1, float bc2, float gscale) {
  const float step = lr / bc1;
  const float rs_bc2 = rsqrtf(bc2);
  const long long nvec = n / 8, nvec_all = (n + 7) / 8;   // the tail (n % 8) is one more, partial vector
  for (long long i = (long long)blockIdx.x * EW_THREADS + threadIdx.x; i < nvec_all;
       i += (long long)gridDim.x * EW_THREADS) {
    const int cnt = i < nvec ? 8 : (int)(n - nvec * 8);
    float gv[8], mv[8], vv[8], dv[8];
    load8n(g + i * 8, gv, cnt);
    load8n(m + i * 8, mv, cnt);
    load8n(v + i * 8, vv, cnt);
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const float gj = gv[j] * gscale;
      mv[j] = b1 * mv[j] + (1.0f - b1) * gj;
      vv[j] = b2 * vv[j] + (1.0f - b2) * gj * gj;
      dv[j] = -step * mv[j] / (sqrtf(vv[j]) * rs_bc2 + eps);
    }
    store8n(m + i * 8, mv, cnt);
    store8n(v + i * 8, vv, cnt);
    store8n(d + i * 8, dv, cnt);
  }
}

// ---- Lion / SGD of enhanced_optimizers.py, with global-norm clipping and EMA weights fused in ----
// The arithmetic is written with explicit round-to-nearest products and sums (no fma contraction), in
// the reference's order of operations, so the fp32 results follow the reference's own rounding.

// Factor the reference's _clip_gradients (:417-432, :285-300) applies to gradients of norm ||g*gscale||:
// min(1, max_norm / (||g*gscale|| + 1e-6)).  `clip_ss` is the device sum of squares of the raw range
// (b200_sumsq, batch 1: a fixed grid and summation order), so every thread forms the same factor with no
// host read, and data-parallel replicas holding identical gradients form identical factors.
__device__ __forceinline__ float clip_factor(const float* __restrict__ clip_ss, float max_norm, float gscale) {
  if (clip_ss == nullptr) return 1.0f;
  const float coef = max_norm / (sqrtf(*clip_ss) * gscale + 1e-6f);
  return coef < 1.0f ? coef : 1.0f;
}

// ema_mode 0: none; 1: ema = p_new (first update); 2: ema = d*ema + (1-d)*p_new   (:396-415, :248-267)
__device__ __forceinline__ float ema_step(float e, float p, float d, float omd, int ema_mode) {
  return ema_mode == 1 ? p : __fadd_rn(__fmul_rn(d, e), __fmul_rn(omd, p));
}

// LionEnhanced.update (:434-484).  c = bs*m + (1-bs)*g ; p = p*decay - lr*sign(c) ; m = bm*m + (1-bm)*g.
// bs == bm and decay == 1 is the reference as written (c is the stored momentum; its weight decay is
// discarded); otherwise Chen et al.'s Lion with decoupled decay.  sign(0) = 0.
__device__ __forceinline__ void lion_elem(float& p, float g, float& m, float& e, float lr, float bs, float obs,
                                          float bm, float obm, float decay, float d, float omd, int ema_mode) {
  const float c = __fadd_rn(__fmul_rn(bs, m), __fmul_rn(obs, g));
  const float s = c > 0.f ? 1.0f : (c < 0.f ? -1.0f : 0.0f);
  m = __fadd_rn(__fmul_rn(bm, m), __fmul_rn(obm, g));
  p = __fadd_rn(__fmul_rn(p, decay), -lr * s);
  if (ema_mode) e = ema_step(e, p, d, omd, ema_mode);
}

template <typename G>
__global__ void __launch_bounds__(EW_THREADS)
lion_kernel(float* __restrict__ p32, __nv_bfloat16* __restrict__ p16, const G* __restrict__ g,
            float* __restrict__ m, float* __restrict__ ema, long long n, float lr, float bs, float bm,
            float decay, float gscale, const float* __restrict__ clip_ss, float max_norm, float d,
            int ema_mode) {
  const float cf = clip_factor(clip_ss, max_norm, gscale);
  const float obs = 1.0f - bs, obm = 1.0f - bm, omd = 1.0f - d;
  const long long nvec = n / 8;
  for (long long i = (long long)blockIdx.x * EW_THREADS + threadIdx.x; i < nvec;
       i += (long long)gridDim.x * EW_THREADS) {
    float pv[8], gv[8], mv[8], ev[8];
    load8(p32 + i * 8, pv);
    load8(g + i * 8, gv);
    load8(m + i * 8, mv);
    if (ema_mode == 2) load8(ema + i * 8, ev);
#pragma unroll
    for (int j = 0; j < 8; ++j)
      lion_elem(pv[j], __fmul_rn(__fmul_rn(gv[j], gscale), cf), mv[j], ev[j], lr, bs, obs, bm, obm, decay, d, omd,
                ema_mode);
    store8(p32 + i * 8, pv);
    store8(m + i * 8, mv);
    if (ema_mode) store8(ema + i * 8, ev);
    if (p16) store8(p16 + i * 8, pv);
  }
  if (blockIdx.x == 0) {
    for (long long i = nvec * 8 + threadIdx.x; i < n; i += EW_THREADS) {
      float p = p32[i], mm = m[i], e = ema_mode == 2 ? ema[i] : 0.f;
      lion_elem(p, __fmul_rn(__fmul_rn(ldf(g + i), gscale), cf), mm, e, lr, bs, obs, bm, obm, decay, d, omd,
                ema_mode);
      p32[i] = p;
      m[i] = mm;
      if (ema_mode) ema[i] = e;
      if (p16) p16[i] = __float2bfloat16_rn(p);
    }
  }
}

// SGDEnhanced.update (:302-351) and mlx SGD:  g += wd_c*p (coupled decay, :269-283) ;
// buf = mu*buf + (1-damp)*g ; p += -lr*(nesterov ? g + mu*buf : buf).  buf == NULL: p += -lr*g.
template <typename G>
__global__ void __launch_bounds__(EW_THREADS)
sgd_kernel(float* __restrict__ p32, __nv_bfloat16* __restrict__ p16, const G* __restrict__ g,
           float* __restrict__ buf, float* __restrict__ ema, long long n, float lr, float mu, float damp,
           int nesterov, float wd_c, float gscale, const float* __restrict__ clip_ss, float max_norm, float d,
           int ema_mode) {
  const float cf = clip_factor(clip_ss, max_norm, gscale);
  const float omdamp = 1.0f - damp, omd = 1.0f - d;
  auto elem = [&](float& p, float gj, float& b, float& e) {
    gj = __fmul_rn(__fmul_rn(gj, gscale), cf);
    if (wd_c != 0.f) gj = __fadd_rn(gj, __fmul_rn(wd_c, p));
    float u = gj;
    if (buf) {
      b = __fadd_rn(__fmul_rn(mu, b), __fmul_rn(omdamp, gj));
      u = nesterov ? __fadd_rn(gj, __fmul_rn(mu, b)) : b;
    }
    p = __fadd_rn(p, __fmul_rn(-lr, u));
    if (ema_mode) e = ema_step(e, p, d, omd, ema_mode);
  };
  const long long nvec = n / 8;
  for (long long i = (long long)blockIdx.x * EW_THREADS + threadIdx.x; i < nvec;
       i += (long long)gridDim.x * EW_THREADS) {
    float pv[8], gv[8], bv[8], ev[8];
    load8(p32 + i * 8, pv);
    load8(g + i * 8, gv);
    if (buf) load8(buf + i * 8, bv);
    if (ema_mode == 2) load8(ema + i * 8, ev);
#pragma unroll
    for (int j = 0; j < 8; ++j) elem(pv[j], gv[j], bv[j], ev[j]);
    store8(p32 + i * 8, pv);
    if (buf) store8(buf + i * 8, bv);
    if (ema_mode) store8(ema + i * 8, ev);
    if (p16) store8(p16 + i * 8, pv);
  }
  if (blockIdx.x == 0) {
    for (long long i = nvec * 8 + threadIdx.x; i < n; i += EW_THREADS) {
      float p = p32[i], b = buf ? buf[i] : 0.f, e = ema_mode == 2 ? ema[i] : 0.f;
      elem(p, ldf(g + i), b, e);
      p32[i] = p;
      if (buf) buf[i] = b;
      if (ema_mode) ema[i] = e;
      if (p16) p16[i] = __float2bfloat16_rn(p);
    }
  }
}

// acc = (init ? 0 : acc) + clamp(g, -clip, clip) * scale    (clip <= 0 disables the clamp)
template <typename G>
__global__ void __launch_bounds__(EW_THREADS)
clip_accum_kernel(const G* __restrict__ g, float* __restrict__ acc, long long n, float clip,
                  float scale, int init) {
  const long long nvec = n / 8;
  for (long long i = (long long)blockIdx.x * EW_THREADS + threadIdx.x; i < nvec;
       i += (long long)gridDim.x * EW_THREADS) {
    float gv[8], av[8];
    load8(g + i * 8, gv);
    if (init) {
#pragma unroll
      for (int j = 0; j < 8; ++j) av[j] = 0.f;
    } else {
      load8(acc + i * 8, av);
    }
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      float x = gv[j];
      if (clip > 0.f) x = fminf(fmaxf(x, -clip), clip);
      av[j] = fmaf(x, scale, av[j]);
    }
    store8(acc + i * 8, av);
  }
  if (blockIdx.x == 0) {
    for (long long i = nvec * 8 + threadIdx.x; i < n; i += EW_THREADS) {
      float x = ldf(g + i);
      if (clip > 0.f) x = fminf(fmaxf(x, -clip), clip);
      acc[i] = (init ? 0.f : acc[i]) + x * scale;
    }
  }
}

// out[b] (+)= sum(x[b, :]^2), grid = (blocks, batch); deterministic (see grid_reduce_finish)
template <typename X>
__global__ void __launch_bounds__(EW_THREADS)
sumsq_kernel(const X* __restrict__ x, float* __restrict__ out, long long numel, int accumulate,
             float* __restrict__ partials, unsigned* __restrict__ counters) {
  const X* xp = x + (long long)blockIdx.y * numel;
  float ss = 0.f;
  const long long nvec = numel / 8;
  for (long long i = (long long)blockIdx.x * EW_THREADS + threadIdx.x; i < nvec;
       i += (long long)gridDim.x * EW_THREADS) {
    float xv[8];
    load8(xp + i * 8, xv);
#pragma unroll
    for (int j = 0; j < 8; ++j) ss += xv[j] * xv[j];
  }
  if (blockIdx.x == 0)
    for (long long i = nvec * 8 + threadIdx.x; i < numel; i += EW_THREADS) {
      const float t = ldf(xp + i);
      ss += t * t;
    }
  const float tot = block_sum(ss);
  grid_reduce_finish(tot, partials, counters, out, accumulate);
}

// dst(bf16) = src(fp32) (strided 2-D block copy with cast; used for Shampoo's [:k,:k] sub-blocks
// and hi/lo bf16 splitting: hi = bf16(x), lo = bf16(x - hi))
__global__ void __launch_bounds__(EW_THREADS)
split_bf16_kernel(const float* __restrict__ src, long long ld_src, __nv_bfloat16* __restrict__ hi,
                  __nv_bfloat16* __restrict__ lo, long long ld_dst, int rows, int cols,
                  float scale, float diag_add) {
  const long long total = (long long)rows * cols;
  for (long long i = (long long)blockIdx.x * EW_THREADS + threadIdx.x; i < total;
       i += (long long)gridDim.x * EW_THREADS) {
    const int r = (int)(i / cols), c = (int)(i % cols);
    float x = src[(long long)r * ld_src + c];
    if (r == c) x += diag_add;
    x *= scale;
    const __nv_bfloat16 h = __float2bfloat16_rn(x);
    hi[(long long)r * ld_dst + c] = h;
    if (lo) lo[(long long)r * ld_dst + c] = __float2bfloat16_rn(x - __bfloat162float(h));
  }
}


// Shampoo momentum (optimizers/shampoo.py:351-359): m = beta*m + (1-beta)*g ; mhat = m/bias_corr.
// Emits out_scale*mhat in fp32 (pass-through part of the update, out_scale = -lr) and as a bf16 hi/lo pair (GEMM operands).
template <typename G>
__global__ void __launch_bounds__(EW_THREADS)
ema_split_kernel(const G* __restrict__ g, float* __restrict__ m, float* __restrict__ out32,
                 __nv_bfloat16* __restrict__ hi, __nv_bfloat16* __restrict__ lo, long long n,
                 float beta, float gscale, float inv_bc, float out_scale) {
  const long long nvec = n / 8;
  for (long long i = (long long)blockIdx.x * EW_THREADS + threadIdx.x; i < nvec;
       i += (long long)gridDim.x * EW_THREADS) {
    float gv[8], mv[8], ov[8], hv[8], lv[8];
    load8(g + i * 8, gv);
    load8(m + i * 8, mv);
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      mv[j] = beta * mv[j] + (1.0f - beta) * gv[j] * gscale;
      const float mh = mv[j] * inv_bc;
      ov[j] = mh * out_scale;
      hv[j] = __bfloat162float(__float2bfloat16_rn(mh));
      lv[j] = mh - hv[j];
    }
    store8(m + i * 8, mv);
    store8(out32 + i * 8, ov);
    store8(hi + i * 8, hv);
    if (lo) store8(lo + i * 8, lv);
  }
  if (blockIdx.x == 0) {
    for (long long i = nvec * 8 + threadIdx.x; i < n; i += EW_THREADS) {
      const float mm = beta * m[i] + (1.0f - beta) * ldf(g + i) * gscale;
      m[i] = mm;
      const float mh = mm * inv_bc;
      out32[i] = mh * out_scale;
      const __nv_bfloat16 h = __float2bfloat16_rn(mh);
      hi[i] = h;
      if (lo) lo[i] = __float2bfloat16_rn(mh - __bfloat162float(h));
    }
  }
}

// Grafted Shampoo update (optimizers/shampoo.py:365-373), batched over same-shape matrices:
// p = p*decay + coef[b]*pre + coef_d[b]*d ; grid = (blocks, batch)
__global__ void __launch_bounds__(EW_THREADS)
graft_update_kernel(float* __restrict__ p32, __nv_bfloat16* __restrict__ p16,
                    const float* __restrict__ pre, const float* __restrict__ d, long long numel,
                    const float* __restrict__ coef, const float* __restrict__ coef_d, float decay) {
  const long long base = (long long)blockIdx.y * numel;
  const float c = coef[blockIdx.y], cd = coef_d[blockIdx.y];
  // batched use has numel % 8 == 0 (checked by the host wrapper), so `base` keeps 16-byte alignment
  const long long nvec = numel / 8, nvec_all = (numel + 7) / 8;   // the tail (numel % 8) is one more, partial vector
  for (long long i = (long long)blockIdx.x * EW_THREADS + threadIdx.x; i < nvec_all;
       i += (long long)gridDim.x * EW_THREADS) {
    const int cnt = i < nvec ? 8 : (int)(numel - nvec * 8);
    float pv[8], rv[8], dv[8];
    load8n(p32 + base + i * 8, pv, cnt);
    load8n(pre + base + i * 8, rv, cnt);
    load8n(d + base + i * 8, dv, cnt);
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      // a zero coefficient must drop its term even when the term is inf/nan (overflowed Shampoo step, D10)
      float v = pv[j] * decay;
      if (c != 0.f) v += c * rv[j];
      if (cd != 0.f) v += cd * dv[j];
      pv[j] = v;
    }
    store8n(p32 + base + i * 8, pv, cnt);
    if (p16) store8n(p16 + base + i * 8, pv, cnt);
  }
}

inline int ew_grid(long long n_per_thread_items) {
  long long blocks = (n_per_thread_items + EW_THREADS - 1) / EW_THREADS;
  const long long cap = (long long)num_sms() * 8;
  if (blocks > cap) blocks = cap;
  if (blocks < 1) blocks = 1;
  return (int)blocks;
}

// splits a caller workspace into (partials, counters) and zeroes the counters on `stream`
int reduce_ws(void* ws, size_t ws_bytes, int batch, int gx, float** partials, unsigned** counters,
              cudaStream_t stream) {
  if (ws == nullptr || ws_bytes < b200_reduce_workspace_bytes(batch) ||
      (size_t)gx * batch + batch > b200_reduce_workspace_bytes(batch) / 4) {
    set_error("reduction workspace too small (%zu < %zu bytes for batch %d)", ws_bytes,
              b200_reduce_workspace_bytes(batch), batch);
    return B200_ERR_WORKSPACE;
  }
  *counters = reinterpret_cast<unsigned*>(ws);
  *partials = reinterpret_cast<float*>(ws) + batch;
  B200_CHECK_CUDA(cudaMemsetAsync(*counters, 0, sizeof(unsigned) * batch, stream));
  return B200_OK;
}

}  // namespace
}  // namespace b200

using namespace b200;

extern "C" {

// Scratch of the deterministic grid reductions: one partial per block (at most 8 blocks per SM over the
// whole batch, plus one per matrix) and one arrival counter per matrix.
size_t b200_reduce_workspace_bytes(int batch) {
  if (batch < 1) batch = 1;
  return al256(((size_t)num_sms() * 8 + 2 * (size_t)batch) * 4);
}

int b200_muon_momentum(const void* g, int g_is_bf16, float* buf, void* u_bf16, float* sumsq,
                       long long numel, int batch, float mu, int nesterov, float gscale, void* ws,
                       size_t ws_bytes, void* stream) {
  const cudaStream_t s = static_cast<cudaStream_t>(stream);
  B200_CHECK_ARG(numel > 0 && batch > 0, "muon_momentum: empty");
  B200_CHECK_ARG(al16(g) && al16(buf) && al16(u_bf16),
                 "muon_momentum: buffers must be 16-byte aligned");
  B200_CHECK_ARG(batch == 1 || numel % 8 == 0,
                 "muon_momentum: batched use needs numel %% 8 == 0 (got %lld)", numel);
  int gx = ew_grid(numel / 8 + 1);
  // keep total blocks around 8 per SM across the batch
  const int cap = (num_sms() * 8 + batch - 1) / batch;
  if (gx > cap) gx = cap < 1 ? 1 : cap;
  dim3 grid(gx, batch);
  float* partials;
  unsigned* counters;
  if (int rc = reduce_ws(ws, ws_bytes, batch, gx, &partials, &counters, s)) return rc;
  if (g_is_bf16)
    muon_momentum_kernel<__nv_bfloat16><<<grid, EW_THREADS, 0, s>>>(
        (const __nv_bfloat16*)g, buf, (__nv_bfloat16*)u_bf16, sumsq, numel, mu, nesterov, gscale, partials,
        counters);
  else
    muon_momentum_kernel<float><<<grid, EW_THREADS, 0, s>>>(
        (const float*)g, buf, (__nv_bfloat16*)u_bf16, sumsq, numel, mu, nesterov, gscale, partials, counters);
  B200_CHECK_LAUNCH();
  return B200_OK;
}

int b200_ns_scales(const float* sumsq, float* inv_norm, float* inv_norm_sq, int batch, float eps,
                   void* stream) {
  const cudaStream_t s = static_cast<cudaStream_t>(stream);
  ns_scales_kernel<<<(batch + 127) / 128, 128, 0, s>>>(sumsq, inv_norm, inv_norm_sq, batch, eps);
  B200_CHECK_LAUNCH();
  return B200_OK;
}

int b200_axpy_update(float* p32, void* p16, const void* x, int x_is_bf16, long long n, float s,
                     void* stream) {
  const cudaStream_t st = static_cast<cudaStream_t>(stream);
  B200_CHECK_ARG(n > 0, "axpy_update: empty");
  B200_CHECK_ARG(al16(p32) && al16(p16) && al16(x),
                 "axpy_update: buffers must be 16-byte aligned");
  const int grid = ew_grid(n / 8 + 1);
  if (x_is_bf16)
    axpy_update_kernel<__nv_bfloat16><<<grid, EW_THREADS, 0, st>>>(
        p32, (__nv_bfloat16*)p16, (const __nv_bfloat16*)x, n, s);
  else
    axpy_update_kernel<float><<<grid, EW_THREADS, 0, st>>>(p32, (__nv_bfloat16*)p16,
                                                          (const float*)x, n, s);
  B200_CHECK_LAUNCH();
  return B200_OK;
}

int b200_sgd_momentum(float* p32, void* p16, const void* g, int g_is_bf16, float* buf, long long n,
                      float mu, int nesterov, float lr, float gscale, void* stream) {
  const cudaStream_t s = static_cast<cudaStream_t>(stream);
  B200_CHECK_ARG(n > 0, "sgd_momentum: empty");
  B200_CHECK_ARG(al16(p32) && al16(p16) && al16(g) && al16(buf),
                 "sgd_momentum: buffers must be 16-byte aligned");
  const int grid = ew_grid(n / 8 + 1);
  if (g_is_bf16)
    sgd_momentum_kernel<__nv_bfloat16><<<grid, EW_THREADS, 0, s>>>(
        p32, (__nv_bfloat16*)p16, (const __nv_bfloat16*)g, buf, n, mu, nesterov, lr, gscale);
  else
    sgd_momentum_kernel<float><<<grid, EW_THREADS, 0, s>>>(
        p32, (__nv_bfloat16*)p16, (const float*)g, buf, n, mu, nesterov, lr, gscale);
  B200_CHECK_LAUNCH();
  return B200_OK;
}

int b200_adamw(float* p32, void* p16, const void* g, int g_is_bf16, float* m, float* v, long long n,
               float lr, float b1, float b2, float eps, float wd, float bc1, float bc2, float gscale,
               void* stream) {
  const cudaStream_t s = static_cast<cudaStream_t>(stream);
  B200_CHECK_ARG(n > 0, "adamw: empty");
  B200_CHECK_ARG(al16(p32) && al16(p16) && al16(g) && al16(m) && al16(v),
                 "adamw: buffers must be 16-byte aligned");
  const int grid = ew_grid(n / 8 + 1);
  if (g_is_bf16)
    adamw_kernel<__nv_bfloat16><<<grid, EW_THREADS, 0, s>>>(
        p32, (__nv_bfloat16*)p16, (const __nv_bfloat16*)g, m, v, n, lr, b1, b2, eps, wd, bc1, bc2,
        gscale);
  else
    adamw_kernel<float><<<grid, EW_THREADS, 0, s>>>(p32, (__nv_bfloat16*)p16, (const float*)g,
                                                   m, v, n, lr, b1, b2, eps, wd, bc1, bc2,
                                                   gscale);
  B200_CHECK_LAUNCH();
  return B200_OK;
}

int b200_adam_direction(float* d, const void* g, int g_is_bf16, float* m, float* v, long long n,
                        float lr, float b1, float b2, float eps, float bc1, float bc2, float gscale,
                        void* stream) {
  const cudaStream_t s = static_cast<cudaStream_t>(stream);
  B200_CHECK_ARG(n > 0, "adam_direction: empty");
  B200_CHECK_ARG(al16(d) && al16(g) && al16(m) && al16(v),
                 "adam_direction: buffers must be 16-byte aligned");
  const int grid = ew_grid(n / 8 + 1);
  if (g_is_bf16)
    adam_direction_kernel<__nv_bfloat16><<<grid, EW_THREADS, 0, s>>>(
        d, (const __nv_bfloat16*)g, m, v, n, lr, b1, b2, eps, bc1, bc2, gscale);
  else
    adam_direction_kernel<float><<<grid, EW_THREADS, 0, s>>>(d, (const float*)g, m, v, n, lr,
                                                            b1, b2, eps, bc1, bc2, gscale);
  B200_CHECK_LAUNCH();
  return B200_OK;
}

int b200_lion(float* p32, void* p16, const void* g, int g_is_bf16, float* m, float* ema, long long n, float lr,
              float b_sign, float b_mom, float decay, float gscale, const float* clip_ss, float max_norm,
              float ema_decay, int ema_mode, void* stream) {
  const cudaStream_t s = static_cast<cudaStream_t>(stream);
  B200_CHECK_ARG(n > 0, "lion: empty");
  B200_CHECK_ARG(p32 && g && m, "lion: p32, g and m are required");
  B200_CHECK_ARG(ema_mode >= 0 && ema_mode <= 2 && (ema_mode == 0 || ema), "lion: ema_mode %d needs ema (0..2)",
                 ema_mode);
  B200_CHECK_ARG(al16(p32) && al16(p16) && al16(g) && al16(m) && al16(ema),
                 "lion: buffers must be 16-byte aligned");
  const int grid = ew_grid(n / 8 + 1);
  if (g_is_bf16)
    lion_kernel<__nv_bfloat16><<<grid, EW_THREADS, 0, s>>>(
        p32, (__nv_bfloat16*)p16, (const __nv_bfloat16*)g, m, ema, n, lr, b_sign, b_mom, decay, gscale, clip_ss,
        max_norm, ema_decay, ema_mode);
  else
    lion_kernel<float><<<grid, EW_THREADS, 0, s>>>(p32, (__nv_bfloat16*)p16, (const float*)g, m, ema, n, lr,
                                                  b_sign, b_mom, decay, gscale, clip_ss, max_norm, ema_decay,
                                                  ema_mode);
  B200_CHECK_LAUNCH();
  return B200_OK;
}

int b200_sgd(float* p32, void* p16, const void* g, int g_is_bf16, float* buf, float* ema, long long n, float lr,
             float mu, float dampening, int nesterov, float coupled_wd, float gscale, const float* clip_ss,
             float max_norm, float ema_decay, int ema_mode, void* stream) {
  const cudaStream_t s = static_cast<cudaStream_t>(stream);
  B200_CHECK_ARG(n > 0, "sgd: empty");
  B200_CHECK_ARG(p32 && g, "sgd: p32 and g are required");
  B200_CHECK_ARG(ema_mode >= 0 && ema_mode <= 2 && (ema_mode == 0 || ema), "sgd: ema_mode %d needs ema (0..2)",
                 ema_mode);
  B200_CHECK_ARG(al16(p32) && al16(p16) && al16(g) && al16(buf) && al16(ema),
                 "sgd: buffers must be 16-byte aligned");
  const int grid = ew_grid(n / 8 + 1);
  if (g_is_bf16)
    sgd_kernel<__nv_bfloat16><<<grid, EW_THREADS, 0, s>>>(
        p32, (__nv_bfloat16*)p16, (const __nv_bfloat16*)g, buf, ema, n, lr, mu, dampening, nesterov, coupled_wd,
        gscale, clip_ss, max_norm, ema_decay, ema_mode);
  else
    sgd_kernel<float><<<grid, EW_THREADS, 0, s>>>(p32, (__nv_bfloat16*)p16, (const float*)g, buf, ema, n, lr,
                                                 mu, dampening, nesterov, coupled_wd, gscale, clip_ss,
                                                 max_norm, ema_decay, ema_mode);
  B200_CHECK_LAUNCH();
  return B200_OK;
}

int b200_clip_accum(const void* g, int g_is_bf16, float* acc, long long n, float clip, float scale,
                    int init, void* stream) {
  const cudaStream_t s = static_cast<cudaStream_t>(stream);
  B200_CHECK_ARG(n > 0, "clip_accum: empty");
  B200_CHECK_ARG(al16(g) && al16(acc), "clip_accum: buffers must be 16-byte aligned");
  const int grid = ew_grid(n / 8 + 1);
  if (g_is_bf16)
    clip_accum_kernel<__nv_bfloat16><<<grid, EW_THREADS, 0, s>>>((const __nv_bfloat16*)g, acc,
                                                                n, clip, scale, init);
  else
    clip_accum_kernel<float><<<grid, EW_THREADS, 0, s>>>((const float*)g, acc, n, clip, scale,
                                                        init);
  B200_CHECK_LAUNCH();
  return B200_OK;
}

int b200_sumsq(const void* x, int x_is_bf16, float* out, long long numel, int batch, int zero_first,
               void* ws, size_t ws_bytes, void* stream) {
  const cudaStream_t s = static_cast<cudaStream_t>(stream);
  B200_CHECK_ARG(numel > 0 && batch > 0, "sumsq: empty");
  B200_CHECK_ARG(al16(x) && (batch == 1 || numel % 8 == 0), "sumsq: alignment");
  int gx = ew_grid(numel / 8 + 1);
  const int cap = (num_sms() * 8 + batch - 1) / batch;
  if (gx > cap) gx = cap < 1 ? 1 : cap;
  dim3 grid(gx, batch);
  float* partials;
  unsigned* counters;
  if (int rc = reduce_ws(ws, ws_bytes, batch, gx, &partials, &counters, s)) return rc;
  if (x_is_bf16)
    sumsq_kernel<__nv_bfloat16><<<grid, EW_THREADS, 0, s>>>((const __nv_bfloat16*)x, out, numel,
                                                           zero_first ? 0 : 1, partials, counters);
  else
    sumsq_kernel<float><<<grid, EW_THREADS, 0, s>>>((const float*)x, out, numel, zero_first ? 0 : 1,
                                                   partials, counters);
  B200_CHECK_LAUNCH();
  return B200_OK;
}

int b200_split_bf16(const float* src, long long ld_src, void* hi, void* lo, long long ld_dst, int rows,
                    int cols, float scale, float diag_add, void* stream) {
  B200_CHECK_ARG(rows > 0 && cols > 0, "split_bf16: empty");
  const int grid = ew_grid((long long)rows * cols);
  split_bf16_kernel<<<grid, EW_THREADS, 0, static_cast<cudaStream_t>(stream)>>>(
      src, ld_src, (__nv_bfloat16*)hi, (__nv_bfloat16*)lo, ld_dst, rows, cols, scale, diag_add);
  B200_CHECK_LAUNCH();
  return B200_OK;
}

int b200_ema_split(const void* g, int g_is_bf16, float* m, float* out32, void* hi, void* lo, long long n,
                   float beta, float gscale, float inv_bc, float out_scale, void* stream) {
  const cudaStream_t s = static_cast<cudaStream_t>(stream);
  B200_CHECK_ARG(n > 0, "ema_split: empty");
  B200_CHECK_ARG(al16(g) && al16(m) && al16(out32) && al16(hi) && al16(lo),
                 "ema_split: buffers must be 16-byte aligned");
  const int grid = ew_grid(n / 8 + 1);
  if (g_is_bf16)
    ema_split_kernel<__nv_bfloat16><<<grid, EW_THREADS, 0, s>>>(
        (const __nv_bfloat16*)g, m, out32, (__nv_bfloat16*)hi, (__nv_bfloat16*)lo, n, beta, gscale, inv_bc, out_scale);
  else
    ema_split_kernel<float><<<grid, EW_THREADS, 0, s>>>(
        (const float*)g, m, out32, (__nv_bfloat16*)hi, (__nv_bfloat16*)lo, n, beta, gscale, inv_bc, out_scale);
  B200_CHECK_LAUNCH();
  return B200_OK;
}

int b200_graft_update(float* p32, void* p16, const float* pre, const float* d, long long numel, int batch,
                      const float* coef, const float* coef_d, float decay, void* stream) {
  const cudaStream_t s = static_cast<cudaStream_t>(stream);
  B200_CHECK_ARG(numel > 0 && batch > 0, "graft_update: empty");
  B200_CHECK_ARG(al16(p32) && al16(p16) && al16(pre) && al16(d) &&
                     (batch == 1 || numel % 8 == 0),
                 "graft_update: buffers must be 16-byte aligned (batched: numel %% 8 == 0)");
  int gx = ew_grid(numel / 8 + 1);
  const int cap = (num_sms() * 8 + batch - 1) / batch;
  if (gx > cap) gx = cap < 1 ? 1 : cap;
  dim3 grid(gx, batch);
  graft_update_kernel<<<grid, EW_THREADS, 0, s>>>(p32, (__nv_bfloat16*)p16, pre, d, numel, coef,
                                                  coef_d, decay);
  B200_CHECK_LAUNCH();
  return B200_OK;
}

}  // extern "C"
