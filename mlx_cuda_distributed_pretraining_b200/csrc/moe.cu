// Mixture-of-experts MLP (Mixtral's sparse MoE block): top-k routing with a stable counting sort of the
// assignments into 128-row expert segments, the row permutation, and the weighted combine with its router adjoint.
// The expert GEMMs run on the wgmma engine's expert-segmented instantiation (gemm_wgmma.cu: moe_gemm, moe_wgrad),
// whose 128-row tiles read their expert from the device table this routing writes.
//
// Nothing here synchronises with the host and nothing uses atomics: every output element is written by one thread
// with a fixed summation order, so the same inputs give the same bits on every run and at every batch composition.
#include <math.h>

#include "common.cuh"
#include "host.h"

namespace b200 {
namespace {

constexpr int SEG = 128;     // expert segments of the permuted buffer are padded to multiples of this (= GEMM tile M)
constexpr int CHUNK = 64;    // tokens per block of the counting sort
constexpr int MAX_E = 64;
constexpr int MAX_K = 8;

// ---- routing --------------------------------------------------------------------------------------------------
// One warp per token: softmax over the E <= 64 logits (lane l holds experts l and l + 32), then k rounds of a warp
// argmax in which the larger probability wins and, on an exact tie, the lower expert index.
__global__ void route_topk_kernel(const float* __restrict__ logits, int T, int E, int k, int* __restrict__ ids,
                                  float* __restrict__ weights, float* __restrict__ probs) {
  const int t = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (t >= T) return;
  const float* l = logits + (size_t)t * E;
  const bool h0 = lane < E, h1 = lane + 32 < E;
  const float v0 = h0 ? l[lane] : -INFINITY, v1 = h1 ? l[lane + 32] : -INFINITY;
  const float m = warp_max(fmaxf(v0, v1));
  const float e0 = h0 ? expf(v0 - m) : 0.f, e1 = h1 ? expf(v1 - m) : 0.f;
  const float s = warp_sum(e0 + e1);
  const float p0 = e0 / s, p1 = e1 / s;
  if (h0) probs[(size_t)t * E + lane] = p0;
  if (h1) probs[(size_t)t * E + lane + 32] = p1;
  float c0 = h0 ? p0 : -1.f, c1 = h1 ? p1 : -1.f;   // -1: not a candidate (any probability is >= 0)
  float sel[MAX_K];
  int sid[MAX_K];
  float tot = 0.f;
#pragma unroll
  for (int j = 0; j < MAX_K; ++j) {
    if (j >= k) break;
    float bv = c0;
    int bi = lane;
    if (c1 > c0) { bv = c1; bi = lane + 32; }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      const float ov = __shfl_xor_sync(0xffffffffu, bv, o);
      const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
      if (ov > bv || (ov == bv && oi < bi)) { bv = ov; bi = oi; }
    }
    sel[j] = bv;
    sid[j] = bi;
    tot += bv;
    if (bi == lane) c0 = -1.f;
    if (bi == lane + 32) c1 = -1.f;
  }
  if (lane < k) {
#pragma unroll
    for (int j = 0; j < MAX_K; ++j) {
      if (j == lane) {
        ids[(size_t)t * k + j] = sid[j];
        weights[(size_t)t * k + j] = sel[j] / tot;
      }
    }
  }
}

// Per chunk of CHUNK tokens: thread e walks the chunk's assignments (t, j) in order and numbers those of expert e
// (rank within the chunk, so the sort is stable), and sums the aux-loss partials of expert e over unmasked tokens.
__global__ void route_hist_kernel(const int* __restrict__ ids, const float* __restrict__ probs,
                                  const unsigned char* __restrict__ mask, int T, int E, int k, int* __restrict__ rank,
                                  int* __restrict__ hist, int* __restrict__ mhist, float* __restrict__ psum) {
  __shared__ int sid[CHUNK * MAX_K];
  const int c = blockIdx.x, t0 = c * CHUNK, nt = min(CHUNK, T - t0);
  for (int i = threadIdx.x; i < nt * k; i += blockDim.x) sid[i] = ids[(size_t)t0 * k + i];
  __syncthreads();
  const int e = threadIdx.x;
  if (e >= E) return;
  int cnt = 0, mcnt = 0;
  for (int a = 0; a < nt * k; ++a) {
    if (sid[a] == e) {
      rank[(size_t)t0 * k + a] = cnt++;
      if (mask == nullptr || mask[t0 + a / k]) ++mcnt;
    }
  }
  hist[(size_t)c * E + e] = cnt;
  if (psum != nullptr) {
    float s = 0.f;
    for (int t = 0; t < nt; ++t)
      if (mask == nullptr || mask[t0 + t]) s += probs[(size_t)(t0 + t) * E + e];
    psum[(size_t)c * E + e] = s;
    mhist[(size_t)c * E + e] = mcnt;
  }
}

// One block: per-expert exclusive scan over the chunks (hist becomes each chunk's base inside the expert), the
// expert totals, the 128-padded segment offsets, the M-tile -> expert table and the aux-loss totals.
__global__ void route_scan_kernel(int* __restrict__ hist, const int* __restrict__ mhist, const float* __restrict__ psum,
                                  int nch, int E, int* __restrict__ counts, int* __restrict__ seg_off,
                                  int* __restrict__ tile_expert, int* __restrict__ n_tiles,
                                  float* __restrict__ aux_counts, float* __restrict__ aux_psum) {
  __shared__ int off[MAX_E + 1];
  __shared__ int padded[MAX_E];
  const int e = threadIdx.x;
  if (e < E) {
    int run = 0;
    for (int c = 0; c < nch; ++c) {
      const int h = hist[(size_t)c * E + e];
      hist[(size_t)c * E + e] = run;
      run += h;
    }
    counts[e] = run;
    padded[e] = (run + SEG - 1) / SEG * SEG;
    if (aux_counts != nullptr) {
      int mc = 0;
      float ps = 0.f;
      for (int c = 0; c < nch; ++c) {
        mc += mhist[(size_t)c * E + e];
        ps += psum[(size_t)c * E + e];
      }
      aux_counts[e] = (float)mc;
      aux_psum[e] = ps;
    }
  }
  __syncthreads();
  if (e == 0) {
    int o = 0;
    for (int i = 0; i < E; ++i) {
      off[i] = o;
      seg_off[i] = o;
      o += padded[i];
    }
    off[E] = o;
    seg_off[E] = o;
    n_tiles[0] = o / SEG;
  }
  __syncthreads();
  if (e < E)
    for (int tl = off[e] / SEG; tl < off[e + 1] / SEG; ++tl) tile_expert[tl] = e;
}

__global__ void route_dest_kernel(const int* __restrict__ ids, const int* __restrict__ rank,
                                  const int* __restrict__ hist, const int* __restrict__ seg_off, int T, int E, int k,
                                  int* __restrict__ dest) {
  const int a = blockIdx.x * blockDim.x + threadIdx.x;
  if (a >= T * k) return;
  const int e = ids[a], c = (a / k) / CHUNK;
  dest[a] = seg_off[e] + hist[(size_t)c * E + e] + rank[a];
}

// ---- permutation and combine (one block of 128 threads per token; rows move as 16-byte vectors) --------------
// Blocks [0, T) copy token rows to their k destinations; blocks T + e * (SEG - 1) + r zero pad row r of expert e's
// segment, so a GEMM tile never reads an unwritten row.
__global__ void permute_kernel(const __nv_bfloat16* __restrict__ x, const int* __restrict__ dest,
                               const int* __restrict__ counts, const int* __restrict__ seg_off, int T, int H, int k,
                               __nv_bfloat16* __restrict__ xp) {
  const int nv = H / 8;
  if ((int)blockIdx.x < T) {
    const int t = blockIdx.x;
    for (int v = threadIdx.x; v < nv; v += blockDim.x) {
      const uint4 val = ldg128(x + (size_t)t * H + v * 8);
      for (int j = 0; j < k; ++j) stg128(xp + (size_t)dest[(size_t)t * k + j] * H + v * 8, val);
    }
    return;
  }
  const int b = blockIdx.x - T, e = b / (SEG - 1), r = b % (SEG - 1);
  const int row = seg_off[e] + counts[e] + r;
  if (row >= seg_off[e + 1]) return;
  for (int v = threadIdx.x; v < nv; v += blockDim.x) stg128(xp + (size_t)row * H + v * 8, make_uint4(0, 0, 0, 0));
}

__device__ __forceinline__ void unpack8(uint4 u, float* f) {
  const uint32_t w[4] = {u.x, u.y, u.z, u.w};
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const float2 p = unpack_bf16x2(w[i]);
    f[2 * i] = p.x;
    f[2 * i + 1] = p.y;
  }
}
__device__ __forceinline__ uint4 pack8(const float* f) {
  return make_uint4(pack_bf16x2(f[0], f[1]), pack_bf16x2(f[2], f[3]), pack_bf16x2(f[4], f[5]), pack_bf16x2(f[6], f[7]));
}

// out[t] = sum_j w[t,j] * yp[dest[t,j]] in fp32, j ascending; or, with weights == nullptr, the plain sum
// dx[t] = sum_j yp[dest[t,j]] (+ addend[t], fp32) of the backward's un-permutation.
__global__ void combine_kernel(const __nv_bfloat16* __restrict__ yp, const int* __restrict__ dest,
                               const float* __restrict__ weights, const float* __restrict__ addend, int H, int k,
                               __nv_bfloat16* __restrict__ out) {
  const int t = blockIdx.x, nv = H / 8;
  for (int v = threadIdx.x; v < nv; v += blockDim.x) {
    float acc[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
    for (int j = 0; j < k; ++j) {
      float f[8];
      unpack8(ldg128(yp + (size_t)dest[(size_t)t * k + j] * H + v * 8), f);
      const float wj = weights != nullptr ? weights[(size_t)t * k + j] : 1.f;
#pragma unroll
      for (int i = 0; i < 8; ++i) acc[i] += wj * f[i];
    }
    if (addend != nullptr) {
#pragma unroll
      for (int i = 0; i < 8; ++i) acc[i] += addend[(size_t)t * H + v * 8 + i];
    }
    stg128(out + (size_t)t * H + v * 8, pack8(acc));
  }
}

// Backward of the combine and of the router, one block per token:
//   dyp[dest[t,j]] = w_j * dout[t]            dw_j = <dout[t], yp[dest[t,j]]>   (fp32 block reduction, fixed order)
//   dp_e = (dw_j - sum_i dw_i w_i) / S  for e = e_j (S = sum_j p_{e_j}, the renormalisation), 0 otherwise,
//          + aux_grad[e] * mask[t]       (d loss / d psum_e of the load-balancing term)
//   dlogits_e = p_e (dp_e - sum_f p_f dp_f)   (softmax adjoint)
__global__ void combine_bwd_kernel(const __nv_bfloat16* __restrict__ dout, const __nv_bfloat16* __restrict__ yp,
                                   const int* __restrict__ dest, const int* __restrict__ ids,
                                   const float* __restrict__ weights, const float* __restrict__ probs,
                                   const float* __restrict__ aux_grad, const unsigned char* __restrict__ mask,
                                   const int* __restrict__ counts, const int* __restrict__ seg_off, int T, int H,
                                   int E, int k, __nv_bfloat16* __restrict__ dyp, float* __restrict__ dw_out,
                                   float* __restrict__ dlogits) {
  if ((int)blockIdx.x >= T) {  // blocks T + e * (SEG - 1) + r zero pad row r of expert e's segment of dyp: the weight
    const int b = blockIdx.x - T, e = b / (SEG - 1), r = b % (SEG - 1);   // gradient's K blocks read them
    const int row = seg_off[e] + counts[e] + r;
    if (row >= seg_off[e + 1]) return;
    for (int v = threadIdx.x; v < H / 8; v += blockDim.x) stg128(dyp + (size_t)row * H + v * 8, make_uint4(0, 0, 0, 0));
    return;
  }
  __shared__ float red[4][MAX_K];
  __shared__ float dw[MAX_K];
  __shared__ float dp[MAX_E];
  const int t = blockIdx.x, nv = H / 8, warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  float part[MAX_K];
#pragma unroll
  for (int j = 0; j < MAX_K; ++j) part[j] = 0.f;
  for (int v = threadIdx.x; v < nv; v += blockDim.x) {
    float d[8];
    unpack8(ldg128(dout + (size_t)t * H + v * 8), d);
#pragma unroll
    for (int j = 0; j < MAX_K; ++j) {
      if (j >= k) break;
      const size_t row = (size_t)dest[(size_t)t * k + j];
      float y[8], g[8];
      unpack8(ldg128(yp + row * H + v * 8), y);
      const float wj = weights[(size_t)t * k + j];
      float s = 0.f;
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        s += d[i] * y[i];
        g[i] = wj * d[i];
      }
      part[j] += s;
      stg128(dyp + row * H + v * 8, pack8(g));
    }
  }
#pragma unroll
  for (int j = 0; j < MAX_K; ++j) {
    if (j >= k) break;
    const float s = warp_sum(part[j]);
    if (lane == 0) red[warp][j] = s;
  }
  __syncthreads();
  if (threadIdx.x < k) {
    const int j = threadIdx.x;
    dw[j] = ((red[0][j] + red[1][j]) + red[2][j]) + red[3][j];
    if (dw_out != nullptr) dw_out[(size_t)t * k + j] = dw[j];
  }
  __syncthreads();
  if (dlogits == nullptr) return;
  const float* p = probs + (size_t)t * E;
  if (threadIdx.x < E) {
    const float m = (aux_grad != nullptr && (mask == nullptr || mask[t])) ? aux_grad[threadIdx.x] : 0.f;
    dp[threadIdx.x] = m;
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    float S = 0.f, c = 0.f;
    for (int j = 0; j < k; ++j) {
      S += p[ids[(size_t)t * k + j]];
      c += dw[j] * weights[(size_t)t * k + j];
    }
    for (int j = 0; j < k; ++j) dp[ids[(size_t)t * k + j]] += (dw[j] - c) / S;
    float q = 0.f;
    for (int e = 0; e < E; ++e) q += p[e] * dp[e];
    dw[0] = q;   // reuse: sum_f p_f dp_f
  }
  __syncthreads();
  if (threadIdx.x < E) dlogits[(size_t)t * E + threadIdx.x] = p[threadIdx.x] * (dp[threadIdx.x] - dw[0]);
}

size_t route_ws_layout(int T, int E, int k, size_t* o_rank, size_t* o_hist, size_t* o_mhist, size_t* o_psum) {
  const size_t nch = (size_t)(T + CHUNK - 1) / CHUNK;
  size_t o = 0;
  *o_rank = o;
  o += al256((size_t)T * k * 4);
  *o_hist = o;
  o += al256(nch * E * 4);
  *o_mhist = o;
  o += al256(nch * E * 4);
  *o_psum = o;
  o += al256(nch * E * 4);
  return o;
}

}  // namespace
}  // namespace b200

using namespace b200;

extern "C" {

size_t b200_moe_route_workspace_bytes(int T, int E, int k) {
  size_t a, b, c, d;
  return route_ws_layout(T, E, k, &a, &b, &c, &d);
}

int b200_moe_max_tiles(int T, int E, int k) {
  const long long live = (long long)T * k < E ? (long long)T * k : E;   // experts that can receive a row
  return (int)(((long long)T * k + (SEG - 1) * live) / SEG);
}

int b200_moe_route(const float* logits, const unsigned char* mask, int T, int E, int k, int* ids, float* weights,
                   float* probs, int* counts, int* seg_off, int* tile_expert, int* n_tiles, int* dest,
                   float* aux_counts, float* aux_psum, void* workspace, size_t workspace_bytes, void* stream) {
  B200_CHECK_ARG(T >= 1 && E >= 2 && E <= MAX_E && k >= 1 && k <= MAX_K && k <= E,
                 "b200_moe_route: need T >= 1, 2 <= E <= %d, 1 <= k <= min(E, %d) (T=%d E=%d k=%d)", MAX_E, MAX_K, T,
                 E, k);
  B200_CHECK_ARG((aux_counts == nullptr) == (aux_psum == nullptr),
                 "b200_moe_route: aux_counts and aux_psum are both given or both NULL");
  size_t o_rank, o_hist, o_mhist, o_psum;
  const size_t need = route_ws_layout(T, E, k, &o_rank, &o_hist, &o_mhist, &o_psum);
  B200_CHECK_ARG(workspace != nullptr && workspace_bytes >= need, "b200_moe_route: workspace needs %zu bytes, got %zu",
                 need, workspace_bytes);
  char* ws = static_cast<char*>(workspace);
  int* rank = reinterpret_cast<int*>(ws + o_rank);
  int* hist = reinterpret_cast<int*>(ws + o_hist);
  int* mhist = reinterpret_cast<int*>(ws + o_mhist);
  float* psum = reinterpret_cast<float*>(ws + o_psum);
  const bool aux = aux_counts != nullptr;
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  const int nch = (T + CHUNK - 1) / CHUNK;
  route_topk_kernel<<<(T + 7) / 8, 256, 0, s>>>(logits, T, E, k, ids, weights, probs);
  B200_CHECK_LAUNCH();
  route_hist_kernel<<<nch, MAX_E, 0, s>>>(ids, probs, mask, T, E, k, rank, hist, aux ? mhist : nullptr,
                                          aux ? psum : nullptr);
  B200_CHECK_LAUNCH();
  route_scan_kernel<<<1, MAX_E, 0, s>>>(hist, mhist, psum, nch, E, counts, seg_off, tile_expert, n_tiles,
                                        aux ? aux_counts : nullptr, aux ? aux_psum : nullptr);
  B200_CHECK_LAUNCH();
  route_dest_kernel<<<(T * k + 255) / 256, 256, 0, s>>>(ids, rank, hist, seg_off, T, E, k, dest);
  B200_CHECK_LAUNCH();
  return B200_OK;
}

int b200_moe_permute(const void* x, const int* dest, const int* counts, const int* seg_off, int T, int H, int k,
                     int E, void* xp, void* stream) {
  B200_CHECK_ARG(T >= 1 && H % 8 == 0 && H > 0 && k >= 1 && E >= 1, "b200_moe_permute: bad shape T=%d H=%d k=%d E=%d",
                 T, H, k, E);
  permute_kernel<<<T + E * (SEG - 1), 128, 0, static_cast<cudaStream_t>(stream)>>>(
      static_cast<const __nv_bfloat16*>(x), dest, counts, seg_off, T, H, k, static_cast<__nv_bfloat16*>(xp));
  B200_CHECK_LAUNCH();
  return B200_OK;
}

int b200_moe_gemm(int mode, int act, const void* A, const void* W0, const void* W1, const void* gu, void* C, void* Y,
                  const int* tile_expert, const int* n_tiles, int max_tiles, int H, int I, int E, void* stream) {
  B200_CHECK_ARG(mode >= 0 && mode <= 3, "b200_moe_gemm: unknown mode %d", mode);
  B200_CHECK_ARG(act == 0 || act == 1, "b200_moe_gemm: unknown activation %d", act);
  B200_CHECK_ARG(H > 0 && I > 0 && H % 8 == 0 && I % 64 == 0 && E >= 1 && E <= MAX_E,
                 "b200_moe_gemm: need H %% 8 == 0, I %% 64 == 0, 1 <= E <= %d (H=%d I=%d E=%d)", MAX_E, H, I, E);
  B200_CHECK_ARG(max_tiles >= 0, "b200_moe_gemm: max_tiles=%d", max_tiles);
  B200_CHECK_ARG(mode != 0 || Y != nullptr, "b200_moe_gemm: Y is required");
  B200_CHECK_ARG(mode != 2 || gu != nullptr, "b200_moe_gemm: gu is required");
  int up_off = 0;
  if (mode == 0 || mode == 3) {  // gate and up experts through one map: Wu must follow Wg by whole [I, H] matrices
    B200_CHECK_ARG(W1 != nullptr, "b200_moe_gemm: W1 (up_proj) is required");
    const long long mat = 2LL * I * H;
    const long long d = static_cast<const char*>(W1) - static_cast<const char*>(W0);
    B200_CHECK_ARG(d > 0 && d % mat == 0 && d / mat >= E && d / mat <= 4096,
                   "b200_moe_gemm: up_proj must lie E or more whole [I, H] matrices after gate_proj in memory");
    up_off = (int)(d / mat);
  }
  return moe_gemm(mode, act, A, W0, up_off, W0, gu, C, Y, tile_expert, n_tiles, max_tiles, H, I, E,
                  static_cast<cudaStream_t>(stream));
}

int b200_moe_wgrad(const void* P, long long ldp, const void* Q, long long ldq, void* G, int R, int Cc, int E, int rows,
                   const int* counts, const int* seg_off, void* stream) {
  return moe_wgrad(P, ldp, Q, ldq, G, R, Cc, E, rows, counts, seg_off, static_cast<cudaStream_t>(stream));
}

int b200_moe_combine_fwd(const void* yp, const int* dest, const float* weights, int T, int H, int k, void* out,
                         void* stream) {
  B200_CHECK_ARG(T >= 1 && H > 0 && H % 8 == 0 && k >= 1 && k <= MAX_K && weights != nullptr,
                 "b200_moe_combine_fwd: bad shape T=%d H=%d k=%d", T, H, k);
  combine_kernel<<<T, 128, 0, static_cast<cudaStream_t>(stream)>>>(static_cast<const __nv_bfloat16*>(yp), dest,
                                                                     weights, nullptr, H, k,
                                                                     static_cast<__nv_bfloat16*>(out));
  B200_CHECK_LAUNCH();
  return B200_OK;
}

int b200_moe_combine_bwd(const void* dout, const void* yp, const int* dest, const int* ids, const float* weights,
                         const float* probs, const float* aux_grad, const unsigned char* mask, const int* counts,
                         const int* seg_off, int T, int H, int E, int k, void* dyp, float* dw, float* dlogits,
                         void* stream) {
  B200_CHECK_ARG(T >= 1 && H > 0 && H % 8 == 0 && k >= 1 && k <= MAX_K && E >= 2 && E <= MAX_E && k <= E,
                 "b200_moe_combine_bwd: bad shape T=%d H=%d E=%d k=%d", T, H, E, k);
  combine_bwd_kernel<<<T + E * (SEG - 1), 128, 0, static_cast<cudaStream_t>(stream)>>>(
      static_cast<const __nv_bfloat16*>(dout), static_cast<const __nv_bfloat16*>(yp), dest, ids, weights, probs,
      aux_grad, mask, counts, seg_off, T, H, E, k, static_cast<__nv_bfloat16*>(dyp), dw, dlogits);
  B200_CHECK_LAUNCH();
  return B200_OK;
}

int b200_moe_unpermute(const void* dxp, const int* dest, const float* addend, int T, int H, int k, void* dx,
                       void* stream) {
  B200_CHECK_ARG(T >= 1 && H > 0 && H % 8 == 0 && k >= 1 && k <= MAX_K, "b200_moe_unpermute: bad shape T=%d H=%d k=%d",
                 T, H, k);
  combine_kernel<<<T, 128, 0, static_cast<cudaStream_t>(stream)>>>(static_cast<const __nv_bfloat16*>(dxp), dest,
                                                                     nullptr, addend, H, k,
                                                                     static_cast<__nv_bfloat16*>(dx));
  B200_CHECK_LAUNCH();
  return B200_OK;
}

}  // extern "C"
