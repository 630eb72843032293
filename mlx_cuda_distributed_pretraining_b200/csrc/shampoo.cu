// Shampoo's Kronecker-factor path (reference: optimizers/shampoo.py) as C-ABI orchestration over the
// wgmma GEMM engine, batched over the same-shape parameters of a flat.ParamStore group:
//
//   shampoo_stats    :229-255   L = b2 L + (1-b2) G G^T ; R = b2 R + (1-b2) G^T G   on G[:k1,:k2]
//   shampoo_root     :88-126    MatrixSqrt.matrix_inverse_pth_root, literally:
//                               Z0 = (M + eps I)/tr ; 6x Z <- Z + Z Z / p ; P = Z * tr^(-1/p^2)
//   shampoo_root_newton         not in the reference: a true inverse 4th root, P = (M + ridge I)^(-1/4) with
//                               ridge = eps * max(lambda_max(M), 1e-6), by the coupled Newton iteration
//                               (Guo & Higham 2006; ridge rule of Anil et al. 2020), products at fp32 accuracy
//   shampoo_precond  :257-295   out[:k1,:k2] = alpha * PL @ m[:k1,:k2] @ PR
//   shampoo_graft    :297-312 + :365-373   ||upd||, ||graft|| -> rescale -> p = p*decay + upd
//
// fp32 matrices enter the tensor cores as bf16 hi+lo pairs (hi*hi + hi*lo + lo*hi: three accumulating
// GEMMs with fp32 accumulation, ~16 mantissa bits), so statistics and roots track the reference's
// fp32 matmuls to ~1e-5 instead of bf16's 4e-3.  Factor matrices are stored [batch, kp, kp] with
// kp = round_up(k, 8) (16-byte TMA rows) and zero padding; trace / identity use the true k, so the padding
// stays exactly zero through the iteration (block-diagonal with a zero block).
#include <math.h>

#include <utility>
#include <vector>

#include "common.cuh"
#include "host.h"

namespace b200 {

int gemm_bf16(bool a_mn, bool b_mn, int M, int N, int K, int batch, const void* A, long long lda,
              long long strideA, const void* B, long long ldb, long long strideB, const void* C,
              long long ldc, long long strideC, void* D, long long ldd, long long strideD,
              bool out_f32, float alpha, float beta, const float* alpha_vec, const float* beta_vec,
              int force_bn, cudaStream_t stream);
size_t reduce_workspace_bytes(int batch);
int graft_update(float* p32, void* p16, const float* pre, const float* d, long long numel, int batch,
                 const float* coef, const float* coef_d, float decay, cudaStream_t stream);
int sumsq(const void* x, int x_is_bf16, float* out, long long numel, int batch, int zero_first, void* ws,
          size_t ws_bytes, cudaStream_t stream);

namespace {

constexpr int SH_THREADS = 256;
inline int rup8(int k) { return (k + 7) & ~7; }
inline size_t al256(size_t x) { return (x + 255) & ~size_t(255); }

// one block per matrix: tr = sum_i M[i,i] + k*eps (trace of M + eps I, shampoo.py:103,110) in a fixed order,
// inv_tr = 1/tr, fin = tr^(-1/p^2) (= (tr^(1/p))^(-1/p), shampoo.py:113,124)
__global__ void __launch_bounds__(SH_THREADS)
root_scalars_kernel(const float* __restrict__ M, int k, int kp, float eps, float p, float* __restrict__ inv_tr,
                    float* __restrict__ fin) {
  __shared__ float red[SH_THREADS / 32];
  const float* m = M + (long long)blockIdx.x * kp * kp;
  float s = 0.f;
  for (int i = threadIdx.x; i < k; i += SH_THREADS) s += m[(long long)i * kp + i];
  s = warp_sum(s);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = s;
  __syncthreads();
  if (threadIdx.x == 0) {
    float t = 0.f;
    for (int w = 0; w < SH_THREADS / 32; ++w) t += red[w];
    const float tr = t + (float)k * eps;
    inv_tr[blockIdx.x] = 1.0f / tr;
    fin[blockIdx.x] = powf(tr, -1.0f / (p * p));
  }
}

// Z0 = (M + eps I[:k,:k]) * inv_tr[b] as fp32 and as a bf16 hi/lo pair; 4 elements per thread
__global__ void __launch_bounds__(SH_THREADS)
root_init_kernel(const float* __restrict__ M, float* __restrict__ Z, __nv_bfloat16* __restrict__ Zh,
                 __nv_bfloat16* __restrict__ Zl, int k, int kp, float eps, const float* __restrict__ inv_tr,
                 long long total4) {
  const long long kk4 = (long long)kp * kp / 4;
  for (long long i = (long long)blockIdx.x * SH_THREADS + threadIdx.x; i < total4;
       i += (long long)gridDim.x * SH_THREADS) {
    const int b = (int)(i / kk4);
    const long long e = (i - (long long)b * kk4) * 4;
    const int r = (int)(e / kp), c = (int)(e - (long long)r * kp);
    const float s = inv_tr[b];
    const float4 v = *reinterpret_cast<const float4*>(M + i * 4);
    float f[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      if (r == c + j && r < k) f[j] += eps;
      f[j] *= s;
    }
    *reinterpret_cast<float4*>(Z + i * 4) = make_float4(f[0], f[1], f[2], f[3]);
    float h[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) h[j] = __bfloat162float(__float2bfloat16_rn(f[j]));
    *reinterpret_cast<uint2*>(Zh + i * 4) = make_uint2(pack_bf16x2(h[0], h[1]), pack_bf16x2(h[2], h[3]));
    *reinterpret_cast<uint2*>(Zl + i * 4) =
        make_uint2(pack_bf16x2(f[0] - h[0], f[1] - h[1]), pack_bf16x2(f[2] - h[2], f[3] - h[3]));
  }
}

// contiguous fp32 -> bf16 hi (+ lo) split, 4 elements per thread (n % 4 == 0)
__global__ void __launch_bounds__(SH_THREADS)
split4_kernel(const float* __restrict__ src, __nv_bfloat16* __restrict__ hi, __nv_bfloat16* __restrict__ lo,
              long long n4) {
  for (long long i = (long long)blockIdx.x * SH_THREADS + threadIdx.x; i < n4;
       i += (long long)gridDim.x * SH_THREADS) {
    const float4 v = *reinterpret_cast<const float4*>(src + i * 4);
    const float f[4] = {v.x, v.y, v.z, v.w};
    float h[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) h[j] = __bfloat162float(__float2bfloat16_rn(f[j]));
    *reinterpret_cast<uint2*>(hi + i * 4) = make_uint2(pack_bf16x2(h[0], h[1]), pack_bf16x2(h[2], h[3]));
    if (lo)
      *reinterpret_cast<uint2*>(lo + i * 4) =
          make_uint2(pack_bf16x2(f[0] - h[0], f[1] - h[1]), pack_bf16x2(f[2] - h[2], f[3] - h[3]));
  }
}

// fp32 -> bf16 hi + mid + lo with x == hi + mid + lo exactly (8 + 8 + 8 mantissa bits)
__device__ __forceinline__ void split3f(float x, float& h, float& m, float& l) {
  h = __bfloat162float(__float2bfloat16_rn(x));
  const float r = x - h;
  m = __bfloat162float(__float2bfloat16_rn(r));
  l = r - m;
}

// element e (a multiple of 4) of a [kp, kp] matrix: writes f[0..3] as a 3-way bf16 split
__device__ __forceinline__ void store_split3(const float f[4], __nv_bfloat16* __restrict__ hi,
                                             __nv_bfloat16* __restrict__ mid, __nv_bfloat16* __restrict__ lo,
                                             long long e) {
  float h[4], m[4], l[4];
#pragma unroll
  for (int j = 0; j < 4; ++j) split3f(f[j], h[j], m[j], l[j]);
  *reinterpret_cast<uint2*>(hi + e) = make_uint2(pack_bf16x2(h[0], h[1]), pack_bf16x2(h[2], h[3]));
  *reinterpret_cast<uint2*>(mid + e) = make_uint2(pack_bf16x2(m[0], m[1]), pack_bf16x2(m[2], m[3]));
  *reinterpret_cast<uint2*>(lo + e) = make_uint2(pack_bf16x2(l[0], l[1]), pack_bf16x2(l[2], l[3]));
}

// contiguous fp32 -> bf16 hi + mid + lo, 4 elements per thread (n % 4 == 0)
__global__ void __launch_bounds__(SH_THREADS)
split3_kernel(const float* __restrict__ src, __nv_bfloat16* __restrict__ hi, __nv_bfloat16* __restrict__ mid,
              __nv_bfloat16* __restrict__ lo, long long n4) {
  for (long long i = (long long)blockIdx.x * SH_THREADS + threadIdx.x; i < n4;
       i += (long long)gridDim.x * SH_THREADS) {
    const float4 v = *reinterpret_cast<const float4*>(src + i * 4);
    const float f[4] = {v.x, v.y, v.z, v.w};
    store_split3(f, hi, mid, lo, i * 4);
  }
}

// ---- coupled Newton inverse 4th root: one block per matrix, fixed-order reductions ----------------------
// Every per-matrix quantity is computed by one block in an order that depends only on k, so a matrix gets the
// same bits whatever batch it is launched in (sumsq's grid, by contrast, is sized by the batch).
constexpr int NR_THREADS = 1024;
constexpr int NR_ROOT = 4;            // r of X -> M^(-1/r)
constexpr int NR_POWER_ITERS = 32;    // power iterations for lambda_max (only the ridge depends on it)

__device__ __forceinline__ float block_sum_nr(float v, float* red) {
  v = warp_sum(v);
  __syncthreads();
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
  __syncthreads();
  float t = 0.f;
  for (int w = 0; w < NR_THREADS / 32; ++w) t += red[w];
  return t;
}

__device__ __forceinline__ float block_max_nr(float v, float* red) {
  v = warp_max(v);
  __syncthreads();
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
  __syncthreads();
  float t = 0.f;
  for (int w = 0; w < NR_THREADS / 32; ++w) t = fmaxf(t, red[w]);
  return t;
}

// |x - id| with NaN counted as +inf, so a NaN iterate is never accepted
__device__ __forceinline__ float abs_dev(float x, float id) {
  const float d = fabsf(x - id);
  return d == d ? d : INFINITY;
}

// fixed pseudo-random start vector in [-1, 1): a constant one can be orthogonal to the top eigenvector (the
// statistics of a softmax layer's weight have the all-ones vector in their null space)
__device__ __forceinline__ float start_vec(int i) {
  unsigned x = (unsigned)i * 0x9E3779B9u + 0x7F4A7C15u;
  x ^= x >> 16;
  x *= 0x7FEB352Du;
  x ^= x >> 15;
  x *= 0x846CA68Bu;
  x ^= x >> 16;
  return (float)(x >> 8) * (2.0f / 16777216.0f) - 1.0f;
}

// lambda_max(M) by power iteration (Rayleigh quotient), ridge = eps * max(lambda_max, 1e-6),
// ||Mt||_F^2 = ||M||_F^2 + 2 ridge tr(M) + k ridge^2 and z = (1 + r) / (2 ||Mt||_F).  Dynamic smem: 2 kp floats.
__global__ void __launch_bounds__(NR_THREADS)
newton_scalars_kernel(const float* __restrict__ M, int k, int kp, float eps, float* __restrict__ ridge_out,
                      float* __restrict__ z_out) {
  extern __shared__ float nr_vec[];
  __shared__ float red[NR_THREADS / 32];
  float* v = nr_vec;
  float* w = nr_vec + kp;
  const float* m = M + (long long)blockIdx.x * kp * kp;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  float ss = 0.f, tr = 0.f, vv = 0.f;
  for (int r = warp; r < k; r += NR_THREADS / 32)
    for (int c = lane; c < k; c += 32) {
      const float x = m[(long long)r * kp + c];
      ss += x * x;
    }
  for (int i = threadIdx.x; i < k; i += NR_THREADS) {
    tr += m[(long long)i * kp + i];
    v[i] = start_vec(i);
    vv += v[i] * v[i];
  }
  ss = block_sum_nr(ss, red);
  tr = block_sum_nr(tr, red);
  vv = block_sum_nr(vv, red);
  const float inv_v = rsqrtf(vv);
  for (int i = threadIdx.x; i < k; i += NR_THREADS) v[i] *= inv_v;
  __syncthreads();
  float lam = 0.f;
  for (int it = 0; it < NR_POWER_ITERS; ++it) {
    for (int r = warp; r < k; r += NR_THREADS / 32) {
      float d = 0.f;
      for (int c = lane; c < k; c += 32) d += m[(long long)r * kp + c] * v[c];
      d = warp_sum(d);
      if (lane == 0) w[r] = d;
    }
    __syncthreads();
    float ww = 0.f, vw = 0.f;
    for (int i = threadIdx.x; i < k; i += NR_THREADS) {
      ww += w[i] * w[i];
      vw += v[i] * w[i];
    }
    ww = block_sum_nr(ww, red);
    lam = block_sum_nr(vw, red);
    if (!(ww > 0.f)) break;  // M v == 0 (a zero M): lambda_max = 0
    const float s = rsqrtf(ww);
    for (int i = threadIdx.x; i < k; i += NR_THREADS) v[i] = w[i] * s;
    __syncthreads();
  }
  if (threadIdx.x == 0) {
    const float ridge = eps * fmaxf(lam, 1e-6f);
    const float fro2 = ss + 2.f * ridge * tr + (float)k * ridge * ridge;
    ridge_out[blockIdx.x] = ridge;
    z_out[blockIdx.x] = (1.f + NR_ROOT) / (2.f * sqrtf(fro2));
  }
}

struct NewtonState {
  float* err;    // max |Mc - I| of the last accepted iterate
  int* iters;    // accepted steps
  int* frozen;   // 1 once converged (err <= tol) or after a rejected step
  float* av;     // per-matrix alpha / beta of the X = X T GEMMs: (1, 0) for an accepted step (including the one
                 // that reaches tol), (0, 1) for a rejected step and for every iteration after the freeze
  float* bv;
};

struct Split3 {
  __nv_bfloat16 *h, *m, *l;
};

// writes I[:k,:k] (zero padding) as a 3-way split
__device__ __forceinline__ void store_identity(Split3 s, long long base, int k, int kp) {
  const long long kk4 = (long long)kp * kp / 4;
  for (long long i = threadIdx.x; i < kk4; i += NR_THREADS) {
    const long long e = i * 4;
    const int r = (int)(e / kp), c = (int)(e - (long long)r * kp);
    float f[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) f[j] = (r == c + j && r < k) ? 1.f : 0.f;
    store_split3(f, s.h, s.m, s.l, base + e);
  }
}

// Mc0 = z (M + ridge I), T0 = (1 + 1/r) I - Mc0 / r, X0 = z^(1/r) I (fp32 into X and split), e0 = max |Mc0 - I|.
// Entries outside [:k,:k] are written as zero whatever M holds there.
__global__ void __launch_bounds__(NR_THREADS)
newton_init_kernel(const float* __restrict__ M, int k, int kp, const float* __restrict__ ridge_in,
                   const float* __restrict__ z_in, float tol, Split3 Mc, Split3 T, float* __restrict__ X, Split3 Xs,
                   NewtonState st) {
  __shared__ float red[NR_THREADS / 32];
  const int b = blockIdx.x;
  const long long base = (long long)b * kp * kp, kk4 = (long long)kp * kp / 4;
  const float ridge = ridge_in[b], z = z_in[b], x0 = powf(z, 1.0f / NR_ROOT);
  float e = 0.f;
  for (long long i = threadIdx.x; i < kk4; i += NR_THREADS) {
    const long long g = base + i * 4;
    const int r = (int)(i * 4 / kp), c = (int)(i * 4 - (long long)r * kp);
    const float4 v = *reinterpret_cast<const float4*>(M + g);
    const float mv[4] = {v.x, v.y, v.z, v.w};
    float mc[4], t[4], x[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const bool in = r < k && c + j < k, diag = in && r == c + j;
      mc[j] = in ? z * (mv[j] + (diag ? ridge : 0.f)) : 0.f;
      t[j] = (diag ? 1.f + 1.f / NR_ROOT : 0.f) - mc[j] * (1.f / NR_ROOT);
      x[j] = diag ? x0 : 0.f;
      if (in) e = fmaxf(e, abs_dev(mc[j], diag ? 1.f : 0.f));
    }
    store_split3(mc, Mc.h, Mc.m, Mc.l, g);
    store_split3(t, T.h, T.m, T.l, g);
    store_split3(x, Xs.h, Xs.m, Xs.l, g);
    *reinterpret_cast<float4*>(X + g) = make_float4(x[0], x[1], x[2], x[3]);
  }
  e = block_max_nr(e, red);
  const bool done = e <= tol;
  if (threadIdx.x == 0) {
    st.err[b] = e;
    st.iters[b] = 0;
    st.frozen[b] = done ? 1 : 0;
    st.av[b] = done ? 0.f : 1.f;
    st.bv[b] = done ? 1.f : 0.f;
  }
  // a frozen matrix iterates on T = I, which keeps every product finite and exact
  if (done) store_identity(T, base, k, kp);
}

// After Mc' = T^4 Mc landed in F: e' = max |Mc' - I|; accept iff e' <= 1.2 e.  Accepted: Mc = Mc' and
// Tn = (1 + 1/r) I - Mc'/r (both as splits); freezing (e' <= tol, or a rejected step): Tn = I.  av/bv select
// whether this iteration's X = X T applies.  Frozen matrices are skipped.
__global__ void __launch_bounds__(NR_THREADS)
newton_step_kernel(const float* __restrict__ F, int k, int kp, float tol, Split3 Mc, Split3 Tn, NewtonState st) {
  __shared__ float red[NR_THREADS / 32];
  __shared__ int mode;  // 1: continue, 2: freeze after a rejected step, 3: freeze after an accepted (converged) step
  const int b = blockIdx.x;
  if (st.frozen[b]) {  // uniform over the block; X = X T stops from the iteration after the freeze
    if (threadIdx.x == 0) {
      st.av[b] = 0.f;
      st.bv[b] = 1.f;
    }
    return;
  }
  const long long base = (long long)b * kp * kp, kk4 = (long long)kp * kp / 4;
  float e = 0.f;
  for (long long i = threadIdx.x; i < kk4; i += NR_THREADS) {
    const int r = (int)(i * 4 / kp), c = (int)(i * 4 - (long long)r * kp);
    if (r >= k) break;
    const float4 v = *reinterpret_cast<const float4*>(F + base + i * 4);
    const float f[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
    for (int j = 0; j < 4; ++j)
      if (c + j < k) e = fmaxf(e, abs_dev(f[j], r == c + j ? 1.f : 0.f));
  }
  e = block_max_nr(e, red);
  if (threadIdx.x == 0) {
    const bool accept = e <= 1.2f * st.err[b];
    if (accept) {
      st.err[b] = e;
      st.iters[b] += 1;
    }
    const bool freeze = !accept || e <= tol;
    st.frozen[b] = freeze ? 1 : 0;
    st.av[b] = accept ? 1.f : 0.f;
    st.bv[b] = accept ? 0.f : 1.f;
    mode = freeze ? (accept ? 3 : 2) : 1;
  }
  __syncthreads();
  if (mode >= 2) {
    // a converged step is still accepted: Mc holds the iterate whose residual err records
    if (mode == 3)
      for (long long i = threadIdx.x; i < kk4; i += NR_THREADS) {
        const float4 v = *reinterpret_cast<const float4*>(F + base + i * 4);
        const float f[4] = {v.x, v.y, v.z, v.w};
        store_split3(f, Mc.h, Mc.m, Mc.l, base + i * 4);
      }
    store_identity(Tn, base, k, kp);
    return;
  }
  for (long long i = threadIdx.x; i < kk4; i += NR_THREADS) {
    const long long g = base + i * 4;
    const int r = (int)(i * 4 / kp), c = (int)(i * 4 - (long long)r * kp);
    const float4 v = *reinterpret_cast<const float4*>(F + g);
    const float f[4] = {v.x, v.y, v.z, v.w};
    float t[4];
#pragma unroll
    for (int j = 0; j < 4; ++j)
      t[j] = (r == c + j && r < k ? 1.f + 1.f / NR_ROOT : 0.f) - f[j] * (1.f / NR_ROOT);
    store_split3(f, Mc.h, Mc.m, Mc.l, g);
    store_split3(t, Tn.h, Tn.m, Tn.l, g);
  }
}

// _apply_grafting (shampoo.py:297-312): ||upd|| == 0 -> graft step ; ||graft|| == 0 -> upd ; else upd*(gn/sn).
// fp32 sqrt(sum x^2) overflows to inf exactly like mx.linalg.norm, which scales the step to 0 (DESIGN D10).
__global__ void graft_coef_kernel(const float* __restrict__ n_upd, const float* __restrict__ n_graft,
                                  float* __restrict__ coef, float* __restrict__ coef_d, int batch) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= batch) return;
  const float sn = sqrtf(n_upd[i]), gn = sqrtf(n_graft[i]);
  coef[i] = sn == 0.f ? 0.f : (gn == 0.f ? 1.f : gn / sn);
  coef_d[i] = sn == 0.f ? 1.f : 0.f;
}

// D = A B + beta C as accumulating fp32-output GEMMs over 3-way splits (hh, hm, mh, hl, lh, mm; the dropped
// ml, lm, ll terms are below fp32 rounding).  All operands [batch, kp, kp] row-major; per-matrix av/bv scale the
// product and C exactly as in gemm3.
// The tensor cores' fp32 accumulation over a whole K = 1024 loses about 4x more than round-to-nearest fp32 sums
// (relative error 6.2e-6 against 1.4e-6 for T T at k = 1024), and the error grows with the K one accumulator spans.
// The dominant hh product therefore runs as GEMMs over 64-wide K slices added in the epilogue (fp32 FMA); that
// brings the product to 4.6e-7 and the root on ridge-limited k = 1024 statistics from 0.065 to 0.002 spectral
// error.  The other products are 2^-8 smaller and run over the whole K.
constexpr int NR_HH_KSLICE = 64;

int gemm6(int kp, int batch, Split3 A, Split3 B, const float* C, float beta, float* D, const float* av,
          const float* bv, cudaStream_t stream) {
  const long long kk = (long long)kp * kp;
  bool first = true;
  for (int k0 = 0; k0 < kp; k0 += NR_HH_KSLICE) {
    const int ks = kp - k0 < NR_HH_KSLICE ? kp - k0 : NR_HH_KSLICE;
    // A is K-major: columns [k0, k0 + ks) start at A + k0; B is MN-major: rows [k0, k0 + ks) start at B + k0 kp
    int rc = gemm_bf16(false, true, kp, kp, ks, batch, A.h + k0, kp, kk, B.h + (long long)k0 * kp, kp, kk,
                       first ? C : D, kp, kk, D, kp, kk, true, 1.0f, first ? beta : 1.0f, av, first ? bv : nullptr,
                       0, stream);
    if (rc) return rc;
    first = false;
  }
  const __nv_bfloat16* pa[5] = {A.h, A.m, A.h, A.l, A.m};
  const __nv_bfloat16* pb[5] = {B.m, B.h, B.l, B.h, B.m};
  for (int i = 0; i < 5; ++i) {
    int rc = gemm_bf16(false, true, kp, kp, kp, batch, pa[i], kp, kk, pb[i], kp, kk, D, kp, kk, D, kp, kk, true, 1.0f,
                       1.0f, av, nullptr, 0, stream);
    if (rc) return rc;
  }
  return B200_OK;
}

inline int sh_grid(long long items) {
  long long b = (items + SH_THREADS - 1) / SH_THREADS;
  const long long cap = (long long)num_sms() * 8;
  if (b > cap) b = cap;
  return (int)(b < 1 ? 1 : b);
}

int split4(const float* src, void* hi, void* lo, long long n, cudaStream_t stream) {
  split4_kernel<<<sh_grid(n / 4), SH_THREADS, 0, stream>>>(src, (__nv_bfloat16*)hi, (__nv_bfloat16*)lo, n / 4);
  B200_CHECK_LAUNCH();
  return B200_OK;
}

// D = alpha*(Ah Bh + Ah Bl + Al Bh) + beta*C  (fp32 out); lo operands may be NULL (plain bf16 product)
int gemm3(bool a_mn, bool b_mn, int M, int N, int K, int batch, const void* Ah, const void* Al, long long lda,
          long long sA, const void* Bh, const void* Bl, long long ldb, long long sB, const float* C, long long ldc,
          long long sC, float* D, long long ldd, long long sD, float alpha, float beta, const float* av,
          const float* bv, cudaStream_t stream) {
  int rc = gemm_bf16(a_mn, b_mn, M, N, K, batch, Ah, lda, sA, Bh, ldb, sB, C, ldc, sC, D, ldd, sD, true, alpha,
                     beta, av, bv, 0, stream);
  if (rc || (Al == nullptr && Bl == nullptr)) return rc;
  if (Bl) {
    rc = gemm_bf16(a_mn, b_mn, M, N, K, batch, Ah, lda, sA, Bl, ldb, sB, D, ldd, sD, D, ldd, sD, true, alpha, 1.0f,
                   av, nullptr, 0, stream);
    if (rc) return rc;
  }
  if (Al)
    rc = gemm_bf16(a_mn, b_mn, M, N, K, batch, Al, lda, sA, Bh, ldb, sB, D, ldd, sD, D, ldd, sD, true, alpha, 1.0f,
                   av, nullptr, 0, stream);
  return rc;
}

}  // namespace

// ---- statistics ---------------------------------------------------------------------------------
int shampoo_stats(const void* g_hi, const void* g_lo, long long ldg, long long strideG, float* L, float* R,
                  int batch, int k1, int k2, float beta2, float weight, cudaStream_t stream) {
  B200_CHECK_ARG(batch > 0 && k1 > 0 && k2 > 0, "shampoo_stats: empty (batch=%d k1=%d k2=%d)", batch, k1, k2);
  B200_CHECK_ARG(ldg % 8 == 0 && ldg >= k2, "shampoo_stats: ldg=%lld must be a multiple of 8 and >= k2", ldg);
  const int k1p = rup8(k1), k2p = rup8(k2);
  // L (+)= G G^T : K-major x K-major over the k2 columns;  R (+)= G^T G : both operands MN-major (G as stored)
  int rc = gemm3(false, false, k1, k1, k2, batch, g_hi, g_lo, ldg, strideG, g_hi, g_lo, ldg, strideG, L, k1p,
                 (long long)k1p * k1p, L, k1p, (long long)k1p * k1p, weight, beta2, nullptr, nullptr, stream);
  if (rc) return rc;
  return gemm3(true, true, k2, k2, k1, batch, g_hi, g_lo, ldg, strideG, g_hi, g_lo, ldg, strideG, R, k2p,
               (long long)k2p * k2p, R, k2p, (long long)k2p * k2p, weight, beta2, nullptr, nullptr, stream);
}

// ---- matrix_inverse_pth_root ----------------------------------------------------------------------
size_t shampoo_root_workspace_bytes(int batch, int k) {
  const size_t kk = (size_t)rup8(k) * rup8(k) * (size_t)(batch > 0 ? batch : 1);
  return al256(kk * 4) + 2 * al256(kk * 2) + al256((size_t)(batch > 0 ? batch : 1) * 8);
}

int shampoo_root(const float* M, float* P, void* P_hi, void* P_lo, int batch, int k, float p, float eps, int iters,
                 void* ws, size_t ws_bytes, cudaStream_t stream) {
  B200_CHECK_ARG(batch > 0 && k > 0 && iters > 0 && p > 0.f, "shampoo_root: bad arguments (batch=%d k=%d iters=%d p=%g)",
                 batch, k, iters, (double)p);
  B200_CHECK_ARG(M != P, "shampoo_root: M and P must be distinct buffers");
  if (ws == nullptr || ws_bytes < shampoo_root_workspace_bytes(batch, k)) {
    set_error("shampoo_root: workspace too small (%zu < %zu)", ws_bytes, shampoo_root_workspace_bytes(batch, k));
    return B200_ERR_WORKSPACE;
  }
  const int kp = rup8(k);
  const long long kk = (long long)kp * kp;
  const size_t n = (size_t)kk * batch;
  char* w = reinterpret_cast<char*>(ws);
  float* Zb = reinterpret_cast<float*>(w);
  void* Zh = w + al256(n * 4);
  void* Zl = w + al256(n * 4) + al256(n * 2);
  float* inv_tr = reinterpret_cast<float*>(w + al256(n * 4) + 2 * al256(n * 2));
  float* fin = inv_tr + batch;
  // ping-pong between P and the workspace so that the LAST iterate lands in P
  float* cur = (iters % 2 == 0) ? P : Zb;
  float* nxt = (iters % 2 == 0) ? Zb : P;
  root_scalars_kernel<<<batch, SH_THREADS, 0, stream>>>(M, k, kp, eps, p, inv_tr, fin);
  B200_CHECK_LAUNCH();
  root_init_kernel<<<sh_grid((long long)n / 4), SH_THREADS, 0, stream>>>(
      M, cur, (__nv_bfloat16*)Zh, (__nv_bfloat16*)Zl, k, kp, eps, inv_tr, (long long)n / 4);
  B200_CHECK_LAUNCH();
  for (int it = 0; it < iters; ++it) {
    const bool last = it == iters - 1;
    // Z' = Z + (1/p) Z Z   (Z @ (I - alpha Z), alpha = -1/p); the final tr^(-1/p^2) rides on the last epilogue
    const float* sv = last ? fin : nullptr;
    int rc = gemm3(false, false, kp, kp, kp, batch, Zh, Zl, kp, kk, Zh, Zl, kp, kk, cur, kp, kk, nxt, kp, kk, 1.0f / p,
                   1.0f, sv, sv, stream);
    if (rc) return rc;
    float* t = cur;
    cur = nxt;
    nxt = t;
    if (!last) {
      rc = split4(cur, Zh, Zl, (long long)n, stream);
      if (rc) return rc;
    }
  }
  // cur == P here
  if (P_hi != nullptr) return split4(P, P_hi, P_lo, (long long)n, stream);
  return B200_OK;
}

// ---- true inverse 4th root by the coupled Newton iteration ------------------------------------------------
// Workspace: F (fp32 product), the 3-way splits of T, S (T^2, T^4, then the next T), Mc and X, and per-matrix
// scalars.
size_t shampoo_root_newton_workspace_bytes(int batch, int k) {
  const size_t b = (size_t)(batch > 0 ? batch : 1);
  const size_t kk = (size_t)rup8(k > 0 ? k : 1) * rup8(k > 0 ? k : 1) * b;
  return al256(kk * 4) + 12 * al256(kk * 2) + 7 * al256(b * 4);
}

int shampoo_root_newton(const float* M, float* P, void* P_hi, void* P_lo, int batch, int k, float eps, int max_iters,
                        float tol, int* iters_out, float* residual_out, void* ws, size_t ws_bytes,
                        cudaStream_t stream) {
  B200_CHECK_ARG(batch > 0 && k > 0 && max_iters > 0 && eps > 0.f && tol >= 0.f,
                 "shampoo_root_newton: bad arguments (batch=%d k=%d max_iters=%d eps=%g tol=%g)", batch, k, max_iters,
                 (double)eps, (double)tol);
  B200_CHECK_ARG(M != P, "shampoo_root_newton: M and P must be distinct buffers");
  if (ws == nullptr || ws_bytes < shampoo_root_newton_workspace_bytes(batch, k)) {
    set_error("shampoo_root_newton: workspace too small (%zu < %zu)", ws_bytes,
              shampoo_root_newton_workspace_bytes(batch, k));
    return B200_ERR_WORKSPACE;
  }
  const int kp = rup8(k);
  const size_t n = (size_t)kp * kp * batch;
  char* w = reinterpret_cast<char*>(ws);
  float* F = reinterpret_cast<float*>(w);
  w += al256(n * 4);
  auto take3 = [&]() {
    Split3 s;
    s.h = reinterpret_cast<__nv_bfloat16*>(w);
    s.m = reinterpret_cast<__nv_bfloat16*>(w + al256(n * 2));
    s.l = reinterpret_cast<__nv_bfloat16*>(w + 2 * al256(n * 2));
    w += 3 * al256(n * 2);
    return s;
  };
  Split3 T = take3(), S = take3(), Mc = take3(), Xs = take3();
  auto take = [&]() {
    char* p = w;
    w += al256((size_t)batch * 4);
    return p;
  };
  float* ridge = reinterpret_cast<float*>(take());
  float* z = reinterpret_cast<float*>(take());
  NewtonState st;
  st.err = reinterpret_cast<float*>(take());
  st.iters = reinterpret_cast<int*>(take());
  st.frozen = reinterpret_cast<int*>(take());
  st.av = reinterpret_cast<float*>(take());
  st.bv = reinterpret_cast<float*>(take());

  const size_t vec_smem = (size_t)2 * kp * sizeof(float);
  if (vec_smem > 48 * 1024)
    B200_CHECK_CUDA(
        cudaFuncSetAttribute(newton_scalars_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)vec_smem));
  newton_scalars_kernel<<<batch, NR_THREADS, vec_smem, stream>>>(M, k, kp, eps, ridge, z);
  B200_CHECK_LAUNCH();
  newton_init_kernel<<<batch, NR_THREADS, 0, stream>>>(M, k, kp, ridge, z, tol, Mc, T, P, Xs, st);
  B200_CHECK_LAUNCH();
  const long long n4 = (long long)n / 4;
  std::vector<int> frozen_host(batch);
  for (int it = 0; it < max_iters; ++it) {
    // Mc' = T^4 Mc, with T^2 and T^4 staged through F and S
    int rc = gemm6(kp, batch, T, T, nullptr, 0.f, F, nullptr, nullptr, stream);
    if (rc) return rc;
    split3_kernel<<<sh_grid(n4), SH_THREADS, 0, stream>>>(F, S.h, S.m, S.l, n4);
    B200_CHECK_LAUNCH();
    if ((rc = gemm6(kp, batch, S, S, nullptr, 0.f, F, nullptr, nullptr, stream))) return rc;
    split3_kernel<<<sh_grid(n4), SH_THREADS, 0, stream>>>(F, S.h, S.m, S.l, n4);
    B200_CHECK_LAUNCH();
    if ((rc = gemm6(kp, batch, S, Mc, nullptr, 0.f, F, nullptr, nullptr, stream))) return rc;
    // accept / freeze; the next T goes to S because X = X T below still reads this iteration's T
    newton_step_kernel<<<batch, NR_THREADS, 0, stream>>>(F, k, kp, tol, Mc, S, st);
    B200_CHECK_LAUNCH();
    // X = av X T + bv X in place: a frozen or rejected matrix keeps its X bit for bit
    if ((rc = gemm6(kp, batch, Xs, T, P, 1.0f, P, st.av, st.bv, stream))) return rc;
    split3_kernel<<<sh_grid(n4), SH_THREADS, 0, stream>>>(P, Xs.h, Xs.m, Xs.l, n4);
    B200_CHECK_LAUNCH();
    std::swap(T, S);
    // every 4 iterations the host stops the loop once every matrix is frozen (frozen matrices no longer change,
    // so the result does not depend on where the loop ends)
    if ((it & 3) == 3 && it + 1 < max_iters) {
      B200_CHECK_CUDA(cudaMemcpyAsync(frozen_host.data(), st.frozen, sizeof(int) * batch, cudaMemcpyDeviceToHost,
                                      stream));
      B200_CHECK_CUDA(cudaStreamSynchronize(stream));
      bool all = true;
      for (int f : frozen_host) all = all && f != 0;
      if (all) break;
    }
  }
  if (iters_out)
    B200_CHECK_CUDA(cudaMemcpyAsync(iters_out, st.iters, sizeof(int) * batch, cudaMemcpyDeviceToDevice, stream));
  if (residual_out)
    B200_CHECK_CUDA(
        cudaMemcpyAsync(residual_out, st.err, sizeof(float) * batch, cudaMemcpyDeviceToDevice, stream));
  if (P_hi != nullptr) return split4(P, P_hi, P_lo, (long long)n, stream);
  return B200_OK;
}

// ---- PL m PR ------------------------------------------------------------------------------------------
size_t shampoo_precond_workspace_bytes(int batch, int k1, int k2) {
  const size_t n = (size_t)(batch > 0 ? batch : 1) * k1 * rup8(k2);
  return al256(n * 4) + 2 * al256(n * 2);
}

int shampoo_precond(const void* PL_hi, const void* PL_lo, const void* PR_hi, const void* PR_lo, const void* m_hi,
                    const void* m_lo, long long ldm, long long strideM, float* out, long long ldo, long long strideO,
                    int batch, int k1, int k2, float alpha, void* ws, size_t ws_bytes, cudaStream_t stream) {
  B200_CHECK_ARG(batch > 0 && k1 > 0 && k2 > 0, "shampoo_precond: empty");
  B200_CHECK_ARG(k2 % 8 == 0, "shampoo_precond: k2=%d must be a multiple of 8 (rows k1 may be arbitrary)", k2);
  if (ws == nullptr || ws_bytes < shampoo_precond_workspace_bytes(batch, k1, k2)) {
    set_error("shampoo_precond: workspace too small (%zu < %zu)", ws_bytes,
              shampoo_precond_workspace_bytes(batch, k1, k2));
    return B200_ERR_WORKSPACE;
  }
  const int k1p = rup8(k1), k2p = rup8(k2);
  const size_t n = (size_t)batch * k1 * k2p;
  char* w = reinterpret_cast<char*>(ws);
  float* T = reinterpret_cast<float*>(w);
  void* Th = w + al256(n * 4);
  void* Tl = w + al256(n * 4) + al256(n * 2);
  // T = PL @ m[:k1,:k2]: the momentum block is read in place as an MN-major B operand ([K = k1 rows][N = k2])
  int rc = gemm3(false, true, k1, k2, k1, batch, PL_hi, PL_lo, k1p, (long long)k1p * k1p, m_hi, m_lo, ldm, strideM,
                 nullptr, k2p, (long long)k1 * k2p, T, k2p, (long long)k1 * k2p, 1.0f, 0.0f, nullptr, nullptr, stream);
  if (rc) return rc;
  rc = split4(T, Th, Tl, (long long)n, stream);
  if (rc) return rc;
  // out[:k1,:k2] = alpha * T @ PR, written straight into the update buffer (ldo = cols of the parameter)
  return gemm3(false, true, k1, k2, k2, batch, Th, Tl, k2p, (long long)k1 * k2p, PR_hi, PR_lo, k2p,
               (long long)k2p * k2p, nullptr, ldo, strideO, out, ldo, strideO, alpha, 0.0f, nullptr, nullptr, stream);
}

// ---- grafting + apply ---------------------------------------------------------------------------------
size_t shampoo_graft_workspace_bytes(int batch) {
  return reduce_workspace_bytes(batch) + al256((size_t)(batch > 0 ? batch : 1) * 16);
}

int shampoo_graft(float* p32, void* p16, const float* upd, const float* graft, long long numel, int batch,
                  float decay, void* ws, size_t ws_bytes, cudaStream_t stream) {
  B200_CHECK_ARG(numel > 0 && batch > 0, "shampoo_graft: empty");
  if (ws == nullptr || ws_bytes < shampoo_graft_workspace_bytes(batch)) {
    set_error("shampoo_graft: workspace too small (%zu < %zu)", ws_bytes, shampoo_graft_workspace_bytes(batch));
    return B200_ERR_WORKSPACE;
  }
  char* w = reinterpret_cast<char*>(ws);
  const size_t rws = reduce_workspace_bytes(batch);
  float* n1 = reinterpret_cast<float*>(w + rws);
  float* n2 = n1 + batch;
  float* coef = n2 + batch;
  float* coef_d = coef + batch;
  int rc = sumsq(upd, 0, n1, numel, batch, 1, w, rws, stream);
  if (rc) return rc;
  rc = sumsq(graft, 0, n2, numel, batch, 1, w, rws, stream);
  if (rc) return rc;
  graft_coef_kernel<<<(batch + 127) / 128, 128, 0, stream>>>(n1, n2, coef, coef_d, batch);
  B200_CHECK_LAUNCH();
  return graft_update(p32, p16, upd, graft, numel, batch, coef, coef_d, decay, stream);
}

}  // namespace b200
