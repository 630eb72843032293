// Shampoo's Kronecker-factor path (reference: optimizers/shampoo.py) as C-ABI orchestration over the
// wgmma GEMM engine, batched over the same-shape parameters of a flat.ParamStore group:
//
//   shampoo_stats    :229-255   L = b2 L + (1-b2) G G^T ; R = b2 R + (1-b2) G^T G   on G[:k1,:k2]
//   shampoo_root     :88-126    MatrixSqrt.matrix_inverse_pth_root, literally:
//                               Z0 = (M + eps I)/tr ; 6x Z <- Z + Z Z / p ; P = Z * tr^(-1/p^2)
//   shampoo_precond  :257-295   out[:k1,:k2] = alpha * PL @ m[:k1,:k2] @ PR
//   shampoo_graft    :297-312 + :365-373   ||upd||, ||graft|| -> rescale -> p = p*decay + upd
//
// fp32 matrices enter the tensor cores as bf16 hi+lo pairs (hi*hi + hi*lo + lo*hi: three accumulating
// GEMMs with fp32 accumulation, ~16 mantissa bits), so statistics and roots track the reference's
// fp32 matmuls to ~1e-5 instead of bf16's 4e-3.  Factor matrices are stored [batch, kp, kp] with
// kp = round_up(k, 8) (16-byte TMA rows) and zero padding; trace / identity use the true k, so the padding
// stays exactly zero through the iteration (block-diagonal with a zero block).
#include <math.h>

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
