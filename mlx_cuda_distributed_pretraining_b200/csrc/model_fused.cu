// SURVEY section 8(f) row f1: the elementwise steps either side of the block's GEMMs, fused into
// single HBM passes.
//
//  glu_fwd / glu_bwd   arch/llama.py:151   y = gate * sigmoid(up) * 2            (sic: not SiLU-GLU)
//  silu_glu_fwd / _bwd mlx_lm's Llama MLP  y = silu(gate) * up                   (model.misc.variant: mlx_lm)
//  ce_fwd  / ce_bwd    core/training.py:1226-1234  per-token cross entropy on fp32-upcast logits with
//                      the pad mask; never materialises the fp32 [B,S,V] copy of the logits.  The
//                      backward overwrites the logits buffer with d(loss)/d(logits) in place.
#include <math_constants.h>

#include "common.cuh"
#include "host.h"

namespace b200 {

namespace {

__device__ __forceinline__ void ld8f(const __nv_bfloat16* p, float* f) {
  const uint4 a = *reinterpret_cast<const uint4*>(p);
  const float2 v0 = unpack_bf16x2(a.x), v1 = unpack_bf16x2(a.y), v2 = unpack_bf16x2(a.z), v3 = unpack_bf16x2(a.w);
  f[0] = v0.x; f[1] = v0.y; f[2] = v1.x; f[3] = v1.y;
  f[4] = v2.x; f[5] = v2.y; f[6] = v3.x; f[7] = v3.y;
}
__device__ __forceinline__ void st8f(__nv_bfloat16* p, const float* f) {
  uint4 o;
  o.x = pack_bf16x2(f[0], f[1]);
  o.y = pack_bf16x2(f[2], f[3]);
  o.z = pack_bf16x2(f[4], f[5]);
  o.w = pack_bf16x2(f[6], f[7]);
  *reinterpret_cast<uint4*>(p) = o;
}
__device__ __forceinline__ float sigmoidf_(float x) { return 1.0f / (1.0f + __expf(-x)); }

__global__ void __launch_bounds__(256)
glu_fwd_kernel(const __nv_bfloat16* __restrict__ g, const __nv_bfloat16* __restrict__ u,
               __nv_bfloat16* __restrict__ y, long long nvec) {
  for (long long i = (long long)blockIdx.x * 256 + threadIdx.x; i < nvec; i += (long long)gridDim.x * 256) {
    float gv[8], uv[8], o[8];
    ld8f(g + i * 8, gv);
    ld8f(u + i * 8, uv);
#pragma unroll
    for (int j = 0; j < 8; ++j) o[j] = gv[j] * sigmoidf_(uv[j]) * 2.0f;
    st8f(y + i * 8, o);
  }
}

__global__ void __launch_bounds__(256)
glu_bwd_kernel(const __nv_bfloat16* __restrict__ dy, const __nv_bfloat16* __restrict__ g,
               const __nv_bfloat16* __restrict__ u, __nv_bfloat16* __restrict__ dg,
               __nv_bfloat16* __restrict__ du, long long nvec) {
  for (long long i = (long long)blockIdx.x * 256 + threadIdx.x; i < nvec; i += (long long)gridDim.x * 256) {
    float dv[8], gv[8], uv[8], og[8], ou[8];
    ld8f(dy + i * 8, dv);
    ld8f(g + i * 8, gv);
    ld8f(u + i * 8, uv);
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const float s = sigmoidf_(uv[j]);
      og[j] = dv[j] * s * 2.0f;
      ou[j] = dv[j] * gv[j] * s * (1.0f - s) * 2.0f;
    }
    st8f(dg + i * 8, og);
    st8f(du + i * 8, ou);
  }
}

// silu(g) u and its adjoint dg = d u s (1 + g (1 - s)), du = d g s with s = sigmoid(g).  sigmoidf_ is relatively
// accurate in the negative tail, where silu(g) is small.
__global__ void __launch_bounds__(256)
silu_glu_fwd_kernel(const __nv_bfloat16* __restrict__ g, const __nv_bfloat16* __restrict__ u,
                    __nv_bfloat16* __restrict__ y, long long nvec) {
  for (long long i = (long long)blockIdx.x * 256 + threadIdx.x; i < nvec; i += (long long)gridDim.x * 256) {
    float gv[8], uv[8], o[8];
    ld8f(g + i * 8, gv);
    ld8f(u + i * 8, uv);
#pragma unroll
    for (int j = 0; j < 8; ++j) o[j] = gv[j] * sigmoidf_(gv[j]) * uv[j];
    st8f(y + i * 8, o);
  }
}

__global__ void __launch_bounds__(256)
silu_glu_bwd_kernel(const __nv_bfloat16* __restrict__ dy, const __nv_bfloat16* __restrict__ g,
                    const __nv_bfloat16* __restrict__ u, __nv_bfloat16* __restrict__ dg,
                    __nv_bfloat16* __restrict__ du, long long nvec) {
  for (long long i = (long long)blockIdx.x * 256 + threadIdx.x; i < nvec; i += (long long)gridDim.x * 256) {
    float dv[8], gv[8], uv[8], og[8], ou[8];
    ld8f(dy + i * 8, dv);
    ld8f(g + i * 8, gv);
    ld8f(u + i * 8, uv);
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const float s = sigmoidf_(gv[j]);
      og[j] = dv[j] * uv[j] * s * fmaf(gv[j], 1.0f - s, 1.0f);
      ou[j] = dv[j] * (gv[j] * s);
    }
    st8f(dg + i * 8, og);
    st8f(du + i * 8, ou);
  }
}

// ---- embedding backward (adjoint of the gather in arch/llama.py:389, `h = self.embed_tokens(inputs)`) --------------
// dW[token[t], :] += dh[t, :].  Two passes over a caller-provided fp32 scratch [V, H] (zeroed by the entry point):
// (1) one warp per token row scatters its bf16 gradient row with fp32 red.global (rows hit by many tokens -- a 259-entry
// byte vocabulary sees hundreds of hits per row -- accumulate in fp32, not in the bf16 gradient buffer), (2) the scratch
// is added into the gradient (which already holds the tied-logits wgrad) in one vectorised pass.
__global__ void __launch_bounds__(256)
embedding_scatter_kernel(const __nv_bfloat16* __restrict__ dh, const long long* __restrict__ tokens,
                         float* __restrict__ scratch, long long rows, int H, int V) {
  const int lane = threadIdx.x & 31;
  for (long long r = (long long)blockIdx.x * 8 + (threadIdx.x >> 5); r < rows; r += (long long)gridDim.x * 8) {
    const long long tok = tokens[r];
    if (tok < 0 || tok >= V) continue;
    const __nv_bfloat16* src = dh + r * H;
    float* dst = scratch + tok * H;
    for (int c = lane * 8; c < H; c += 256) {
      float f[8];
      ld8f(src + c, f);
      asm volatile("red.global.add.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(dst + c), "f"(f[0]), "f"(f[1]), "f"(f[2]),
                   "f"(f[3])
                   : "memory");
      asm volatile("red.global.add.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(dst + c + 4), "f"(f[4]), "f"(f[5]), "f"(f[6]),
                   "f"(f[7])
                   : "memory");
    }
  }
}

template <typename G>
__global__ void __launch_bounds__(256)
embedding_accumulate_kernel(const float* __restrict__ scratch, G* __restrict__ grad, long long nvec) {
  for (long long i = (long long)blockIdx.x * 256 + threadIdx.x; i < nvec; i += (long long)gridDim.x * 256) {
    const float4 a = *reinterpret_cast<const float4*>(scratch + i * 8);
    const float4 b = *reinterpret_cast<const float4*>(scratch + i * 8 + 4);
    if constexpr (sizeof(G) == 2) {
      float g[8];
      ld8f(reinterpret_cast<const __nv_bfloat16*>(grad) + i * 8, g);
      g[0] += a.x; g[1] += a.y; g[2] += a.z; g[3] += a.w;
      g[4] += b.x; g[5] += b.y; g[6] += b.z; g[7] += b.w;
      st8f(reinterpret_cast<__nv_bfloat16*>(grad) + i * 8, g);
    } else {
      float4* gp = reinterpret_cast<float4*>(grad) + i * 2;
      float4 g0 = gp[0], g1 = gp[1];
      g0.x += a.x; g0.y += a.y; g0.z += a.z; g0.w += a.w;
      g1.x += b.x; g1.y += b.y; g1.z += b.z; g1.w += b.w;
      gp[0] = g0;
      gp[1] = g1;
    }
  }
}

constexpr int CE_THREADS = 512;

// one CTA per row; online (max, sum) per thread, then a block reduction of the pairs
__global__ void __launch_bounds__(CE_THREADS)
ce_fwd_kernel(const __nv_bfloat16* __restrict__ logits, long long ld, const long long* __restrict__ targets,
              int V, long long pad_token, float* __restrict__ row_loss, float* __restrict__ row_lse) {
  const long long row = blockIdx.x;
  const __nv_bfloat16* lr = logits + row * ld;
  float m = -CUDART_INF_F, s = 0.f;
  const int nvec = V / 8;
  for (int i = threadIdx.x; i < nvec; i += CE_THREADS) {
    float x[8];
    ld8f(lr + i * 8, x);
    float mx = x[0];
#pragma unroll
    for (int j = 1; j < 8; ++j) mx = fmaxf(mx, x[j]);
    const float mn = fmaxf(m, mx);
    float acc = 0.f;
#pragma unroll
    for (int j = 0; j < 8; ++j) acc += __expf(x[j] - mn);
    s = s * __expf(m - mn) + acc;
    m = mn;
  }
  for (int i = nvec * 8 + threadIdx.x; i < V; i += CE_THREADS) {
    const float x = __bfloat162float(lr[i]);
    const float mn = fmaxf(m, x);
    s = s * __expf(m - mn) + __expf(x - mn);
    m = mn;
  }
  __shared__ float sm[CE_THREADS / 32], ss[CE_THREADS / 32];
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const float m2 = __shfl_xor_sync(0xffffffffu, m, o), s2 = __shfl_xor_sync(0xffffffffu, s, o);
    const float mn = fmaxf(m, m2);
    s = (mn == -CUDART_INF_F) ? 0.f : s * __expf(m - mn) + s2 * __expf(m2 - mn);
    m = mn;
  }
  if ((threadIdx.x & 31) == 0) {
    sm[threadIdx.x >> 5] = m;
    ss[threadIdx.x >> 5] = s;
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    float M = sm[0], S = ss[0];
    for (int w = 1; w < CE_THREADS / 32; ++w) {
      if (sm[w] == -CUDART_INF_F) continue;  // warp saw no element of this row
      if (M == -CUDART_INF_F) {
        M = sm[w];
        S = ss[w];
        continue;
      }
      const float mn = fmaxf(M, sm[w]);
      S = S * __expf(M - mn) + ss[w] * __expf(sm[w] - mn);
      M = mn;
    }
    const float lse = M + logf(S);
    const long long t = targets[row];
    row_lse[row] = lse;
    row_loss[row] = (t != pad_token) ? lse - __bfloat162float(lr[t]) : 0.f;
  }
}

// dlogits[row, j] = row_scale[row] * (exp(logit - lse) - [j == target]) for j < V, 0 for V <= j < ld,
// written over the logits (bf16).  row_scale already contains dloss * pad_mask / ntoks.
__global__ void __launch_bounds__(CE_THREADS)
ce_bwd_kernel(__nv_bfloat16* __restrict__ logits, long long ld, const long long* __restrict__ targets,
              int V, long long pad_token, const float* __restrict__ row_lse,
              const float* __restrict__ row_scale) {
  const long long row = blockIdx.x;
  __nv_bfloat16* lr = logits + row * ld;
  const float lse = row_lse[row];
  const long long t = targets[row];
  const float sc = (t != pad_token) ? row_scale[row] : 0.f;  // padded positions carry no loss
  const int nvec = (int)(ld / 8);
  for (int i = threadIdx.x; i < nvec; i += CE_THREADS) {
    float x[8], o[8];
    ld8f(lr + i * 8, x);
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const int col = i * 8 + j;
      float pr = (col < V) ? __expf(x[j] - lse) : 0.f;
      if (col == t) pr -= 1.0f;
      o[j] = sc * pr;
    }
    st8f(lr + i * 8, o);
  }
}

inline int grid_for(long long nvec) {
  long long b = (nvec + 255) / 256;
  const long long cap = (long long)num_sms() * 8;
  return (int)(b > cap ? cap : (b < 1 ? 1 : b));
}

}  // namespace
}  // namespace b200

using namespace b200;

extern "C" {

int b200_glu_fwd(const void* g, const void* u, void* y, long long n, void* stream) {
  const cudaStream_t s = static_cast<cudaStream_t>(stream);
  B200_CHECK_ARG(n > 0 && n % 8 == 0, "glu_fwd: n=%lld must be a positive multiple of 8", n);
  B200_CHECK_ARG(al16(g) && al16(u) && al16(y), "glu_fwd: 16-byte alignment required");
  glu_fwd_kernel<<<grid_for(n / 8), 256, 0, s>>>((const __nv_bfloat16*)g, (const __nv_bfloat16*)u,
                                                (__nv_bfloat16*)y, n / 8);
  B200_CHECK_LAUNCH();
  return B200_OK;
}

int b200_glu_bwd(const void* dy, const void* g, const void* u, void* dg, void* du, long long n, void* stream) {
  const cudaStream_t s = static_cast<cudaStream_t>(stream);
  B200_CHECK_ARG(n > 0 && n % 8 == 0, "glu_bwd: n=%lld must be a positive multiple of 8", n);
  B200_CHECK_ARG(al16(dy) && al16(g) && al16(u) && al16(dg) && al16(du), "glu_bwd: alignment");
  glu_bwd_kernel<<<grid_for(n / 8), 256, 0, s>>>((const __nv_bfloat16*)dy, (const __nv_bfloat16*)g,
                                                (const __nv_bfloat16*)u, (__nv_bfloat16*)dg,
                                                (__nv_bfloat16*)du, n / 8);
  B200_CHECK_LAUNCH();
  return B200_OK;
}

int b200_silu_glu_fwd(const void* g, const void* u, void* y, long long n, void* stream) {
  const cudaStream_t s = static_cast<cudaStream_t>(stream);
  B200_CHECK_ARG(n > 0 && n % 8 == 0, "silu_glu_fwd: n=%lld must be a positive multiple of 8", n);
  B200_CHECK_ARG(al16(g) && al16(u) && al16(y), "silu_glu_fwd: 16-byte alignment required");
  silu_glu_fwd_kernel<<<grid_for(n / 8), 256, 0, s>>>((const __nv_bfloat16*)g, (const __nv_bfloat16*)u,
                                                     (__nv_bfloat16*)y, n / 8);
  B200_CHECK_LAUNCH();
  return B200_OK;
}

int b200_silu_glu_bwd(const void* dy, const void* g, const void* u, void* dg, void* du, long long n, void* stream) {
  const cudaStream_t s = static_cast<cudaStream_t>(stream);
  B200_CHECK_ARG(n > 0 && n % 8 == 0, "silu_glu_bwd: n=%lld must be a positive multiple of 8", n);
  B200_CHECK_ARG(al16(dy) && al16(g) && al16(u) && al16(dg) && al16(du), "silu_glu_bwd: alignment");
  silu_glu_bwd_kernel<<<grid_for(n / 8), 256, 0, s>>>((const __nv_bfloat16*)dy, (const __nv_bfloat16*)g,
                                                     (const __nv_bfloat16*)u, (__nv_bfloat16*)dg,
                                                     (__nv_bfloat16*)du, n / 8);
  B200_CHECK_LAUNCH();
  return B200_OK;
}

size_t b200_embedding_bwd_workspace_bytes(int V, int H) { return (size_t)V * H * sizeof(float); }

int b200_embedding_bwd(const void* dh, const long long* tokens, void* grad, int grad_is_bf16, long long rows, int V,
                       int H, void* ws, size_t ws_bytes, void* stream) {
  const cudaStream_t s = static_cast<cudaStream_t>(stream);
  B200_CHECK_ARG(rows > 0 && V > 0 && H > 0 && H % 8 == 0, "embedding_bwd: bad shape rows=%lld V=%d H=%d", rows, V, H);
  if (ws == nullptr || ws_bytes < b200_embedding_bwd_workspace_bytes(V, H)) {
    set_error("embedding_bwd: workspace too small (%zu < %zu)", ws_bytes, b200_embedding_bwd_workspace_bytes(V, H));
    return B200_ERR_WORKSPACE;
  }
  B200_CHECK_ARG((reinterpret_cast<uintptr_t>(ws) & 15u) == 0 && (reinterpret_cast<uintptr_t>(grad) & 15u) == 0 &&
                     (reinterpret_cast<uintptr_t>(dh) & 15u) == 0,
                 "embedding_bwd: buffers must be 16-byte aligned");
  float* scratch = reinterpret_cast<float*>(ws);
  B200_CHECK_CUDA(cudaMemsetAsync(scratch, 0, (size_t)V * H * sizeof(float), s));
  long long blocks = (rows + 7) / 8;
  const long long cap = (long long)num_sms() * 8;
  if (blocks > cap) blocks = cap;
  embedding_scatter_kernel<<<(int)blocks, 256, 0, s>>>((const __nv_bfloat16*)dh, tokens, scratch, rows, H, V);
  B200_CHECK_LAUNCH();
  const long long nvec = (long long)V * H / 8;
  long long b2 = (nvec + 255) / 256;
  if (b2 > cap) b2 = cap;
  if (grad_is_bf16)
    embedding_accumulate_kernel<__nv_bfloat16><<<(int)b2, 256, 0, s>>>(scratch, (__nv_bfloat16*)grad, nvec);
  else
    embedding_accumulate_kernel<float><<<(int)b2, 256, 0, s>>>(scratch, (float*)grad, nvec);
  B200_CHECK_LAUNCH();
  return B200_OK;
}

int b200_ce_fwd(const void* logits, long long ld, const long long* targets, int rows, int V, long long pad_token,
                float* row_loss, float* row_lse, void* stream) {
  const cudaStream_t s = static_cast<cudaStream_t>(stream);
  B200_CHECK_ARG(rows > 0 && V > 0 && ld >= V && ld % 8 == 0, "ce_fwd: bad shape rows=%d V=%d ld=%lld", rows, V, ld);
  B200_CHECK_ARG(al16(logits), "ce_fwd: logits must be 16-byte aligned");
  ce_fwd_kernel<<<rows, CE_THREADS, 0, s>>>((const __nv_bfloat16*)logits, ld, targets, V, pad_token, row_loss,
                                            row_lse);
  B200_CHECK_LAUNCH();
  return B200_OK;
}

int b200_ce_bwd(void* logits, long long ld, const long long* targets, int rows, int V, long long pad_token,
                const float* row_lse, const float* row_scale, void* stream) {
  const cudaStream_t s = static_cast<cudaStream_t>(stream);
  B200_CHECK_ARG(rows > 0 && V > 0 && ld >= V && ld % 8 == 0, "ce_bwd: bad shape rows=%d V=%d ld=%lld", rows, V, ld);
  B200_CHECK_ARG(al16(logits), "ce_bwd: logits must be 16-byte aligned");
  ce_bwd_kernel<<<rows, CE_THREADS, 0, s>>>((__nv_bfloat16*)logits, ld, targets, V, pad_token, row_lse,
                                            row_scale);
  B200_CHECK_LAUNCH();
  return B200_OK;
}

}  // extern "C"
