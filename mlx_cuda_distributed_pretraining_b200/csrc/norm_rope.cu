// RMSNorm (arch/llama.py:50-56 of the reference), interleaved-pair RoPE (arch/llama_standard.py:74-75,117-127) and
// half-split RoPE (mlx_lm's nn.RoPE(traditional=False)) as single-pass vectorised HBM kernels, forward + backward.
#include "common.cuh"
#include "host.h"

namespace b200 {

namespace {

constexpr int RN_THREADS = 128;
constexpr int RN_MAX_VEC = 8;  // per-thread 8-element vectors held in registers -> H <= 8192

__device__ __forceinline__ void ld8(const __nv_bfloat16* p, float* f) {
  const uint4 a = *reinterpret_cast<const uint4*>(p);
  const float2 v0 = unpack_bf16x2(a.x), v1 = unpack_bf16x2(a.y), v2 = unpack_bf16x2(a.z),
               v3 = unpack_bf16x2(a.w);
  f[0] = v0.x; f[1] = v0.y; f[2] = v1.x; f[3] = v1.y;
  f[4] = v2.x; f[5] = v2.y; f[6] = v3.x; f[7] = v3.y;
}
__device__ __forceinline__ void ld8(const float* p, float* f) {
  const float4 a = *reinterpret_cast<const float4*>(p);
  const float4 b = *reinterpret_cast<const float4*>(p + 4);
  f[0] = a.x; f[1] = a.y; f[2] = a.z; f[3] = a.w;
  f[4] = b.x; f[5] = b.y; f[6] = b.z; f[7] = b.w;
}
__device__ __forceinline__ void st8(__nv_bfloat16* p, const float* f) {
  uint4 o;
  o.x = pack_bf16x2(f[0], f[1]);
  o.y = pack_bf16x2(f[2], f[3]);
  o.z = pack_bf16x2(f[4], f[5]);
  o.w = pack_bf16x2(f[6], f[7]);
  *reinterpret_cast<uint4*>(p) = o;
}
__device__ __forceinline__ void st8(float* p, const float* f) {
  *reinterpret_cast<float4*>(p) = make_float4(f[0], f[1], f[2], f[3]);
  *reinterpret_cast<float4*>(p + 4) = make_float4(f[4], f[5], f[6], f[7]);
}

__device__ __forceinline__ float block_sum_128(float v, float* red) {
  v = warp_sum(v);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
  __syncthreads();
  const float t = red[0] + red[1] + red[2] + red[3];
  __syncthreads();
  return t;
}

__device__ __forceinline__ float round_like(float v, const __nv_bfloat16*) {
  return __bfloat162float(__float2bfloat16(v));
}
__device__ __forceinline__ float round_like(float v, const float*) { return v; }

// ---- block-per-row kernels (any H <= 8192) -----------------------------------------------------------
// Optional fused residual add (arch/llama.py:316-319, h = x + sublayer(norm(x))): with `delta` the row
// normalised is s = round(x + delta) and s is also written to `sum_out`, exactly what the separate add
// produced before.
template <typename T, int NV>
__global__ void __launch_bounds__(RN_THREADS)
rmsnorm_fwd_kernel(const T* __restrict__ x, const T* __restrict__ delta, const T* __restrict__ w,
                   T* __restrict__ sum_out, T* __restrict__ y, float* __restrict__ rstd_out, int rows, int H,
                   float eps) {
  __shared__ float red[4];
  float wv[NV][8];
#pragma unroll
  for (int v = 0; v < NV; ++v) {
    const int col = (v * RN_THREADS + threadIdx.x) * 8;
    if (col < H) ld8(w + col, wv[v]);
  }
  for (int row = blockIdx.x; row < rows; row += gridDim.x) {
    const T* xr = x + (long long)row * H;
    float xv[NV][8];
    float ss = 0.f;
#pragma unroll
    for (int v = 0; v < NV; ++v) {
      const int col = (v * RN_THREADS + threadIdx.x) * 8;
      if (col < H) {
        ld8(xr + col, xv[v]);
        if (delta) {
          float dv[8];
          ld8(delta + (long long)row * H + col, dv);
#pragma unroll
          for (int j = 0; j < 8; ++j) xv[v][j] = round_like(xv[v][j] + dv[j], x);
          st8(sum_out + (long long)row * H + col, xv[v]);
        }
#pragma unroll
        for (int j = 0; j < 8; ++j) ss += xv[v][j] * xv[v][j];
      }
    }
    const float tot = block_sum_128(ss, red);
    // reference: x / sqrt(mean(x^2) + eps) * w, all in fp32, cast back to the input dtype
    const float rstd = 1.0f / sqrtf(tot / (float)H + eps);
    if (threadIdx.x == 0 && rstd_out) rstd_out[row] = rstd;
    T* yr = y + (long long)row * H;
#pragma unroll
    for (int v = 0; v < NV; ++v) {
      const int col = (v * RN_THREADS + threadIdx.x) * 8;
      if (col < H) {
        float o[8];
#pragma unroll
        for (int j = 0; j < 8; ++j) o[j] = xv[v][j] * rstd * wv[v][j];
        st8(yr + col, o);
      }
    }
  }
}

// dx = [dres +] rstd * (dy*w - x * rstd^2 * mean(dy*w*x)) ; dw partials = sum over this CTA's rows of
// dy * x * rstd, written to dw_part[blockIdx.x, :] and summed by rmsnorm_dw_reduce_kernel (no atomics:
// hundreds of CTAs hammering the same H addresses cost 4x the streaming time).  `dres` is the gradient
// that reached the residual stream directly; adding it here removes autograd's separate accumulation pass.
template <typename T, int NV>
__global__ void __launch_bounds__(RN_THREADS)
rmsnorm_bwd_kernel(const T* __restrict__ dy, const T* __restrict__ dres, const T* __restrict__ x,
                   const T* __restrict__ w, const float* __restrict__ rstd_in, T* __restrict__ dx,
                   float* __restrict__ dw_part, int rows, int H) {
  __shared__ float red[4];
  float wv[NV][8], dwv[NV][8];
#pragma unroll
  for (int v = 0; v < NV; ++v) {
    const int col = (v * RN_THREADS + threadIdx.x) * 8;
    if (col < H) ld8(w + col, wv[v]);
#pragma unroll
    for (int j = 0; j < 8; ++j) dwv[v][j] = 0.f;
  }
  for (int row = blockIdx.x; row < rows; row += gridDim.x) {
    const T* xr = x + (long long)row * H;
    const T* dyr = dy + (long long)row * H;
    const float rstd = rstd_in[row];
    float xv[NV][8], gv[NV][8];
    float dot = 0.f;
#pragma unroll
    for (int v = 0; v < NV; ++v) {
      const int col = (v * RN_THREADS + threadIdx.x) * 8;
      if (col < H) {
        ld8(xr + col, xv[v]);
        ld8(dyr + col, gv[v]);
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          dwv[v][j] += gv[v][j] * xv[v][j] * rstd;
          gv[v][j] *= wv[v][j];
          dot += gv[v][j] * xv[v][j];
        }
      }
    }
    const float tot = block_sum_128(dot, red);
    const float c = tot / (float)H * rstd * rstd;
    T* dxr = dx + (long long)row * H;
#pragma unroll
    for (int v = 0; v < NV; ++v) {
      const int col = (v * RN_THREADS + threadIdx.x) * 8;
      if (col < H) {
        float o[8];
#pragma unroll
        for (int j = 0; j < 8; ++j) o[j] = rstd * (gv[v][j] - xv[v][j] * c);
        if (dres) {
          float r[8];
          ld8(dres + (long long)row * H + col, r);
#pragma unroll
          for (int j = 0; j < 8; ++j) o[j] += r[j];
        }
        st8(dxr + col, o);
      }
    }
  }
#pragma unroll
  for (int v = 0; v < NV; ++v) {
    const int col = (v * RN_THREADS + threadIdx.x) * 8;
    if (col < H) st8(dw_part + (long long)blockIdx.x * H + col, dwv[v]);
  }
}

// ---- warp-per-row kernels (H <= 1024): no block barrier per row, four independent rows in flight per
// ---- CTA, so the loads of one row overlap the reduction and stores of its neighbours ------------------
constexpr int RW_WARPS = RN_THREADS / 32;

// Row segments are held PACKED (bf16 rows as uint4) between the two passes and the gain vector is re-read from
// L1 (2 KB) instead of living in registers: ~56 registers, so 8 CTAs (32 warps) per SM keep enough 16-byte loads
// in flight to cover HBM latency (the first version: 94 registers, 4 CTAs, 0.46 of the HBM roofline under ncu).
template <typename T> struct Raw8;
template <> struct Raw8<__nv_bfloat16> { uint4 r; };
template <> struct Raw8<float> { float4 a, b; };
__device__ __forceinline__ void ldraw(const __nv_bfloat16* p, Raw8<__nv_bfloat16>& o) {
  o.r = *reinterpret_cast<const uint4*>(p);
}
__device__ __forceinline__ void ldraw(const float* p, Raw8<float>& o) {
  o.a = *reinterpret_cast<const float4*>(p);
  o.b = *reinterpret_cast<const float4*>(p + 4);
}
__device__ __forceinline__ void unraw(const Raw8<__nv_bfloat16>& i, float* f) {
  const float2 v0 = unpack_bf16x2(i.r.x), v1 = unpack_bf16x2(i.r.y), v2 = unpack_bf16x2(i.r.z),
               v3 = unpack_bf16x2(i.r.w);
  f[0] = v0.x; f[1] = v0.y; f[2] = v1.x; f[3] = v1.y;
  f[4] = v2.x; f[5] = v2.y; f[6] = v3.x; f[7] = v3.y;
}
__device__ __forceinline__ void unraw(const Raw8<float>& i, float* f) {
  f[0] = i.a.x; f[1] = i.a.y; f[2] = i.a.z; f[3] = i.a.w;
  f[4] = i.b.x; f[5] = i.b.y; f[6] = i.b.z; f[7] = i.b.w;
}
__device__ __forceinline__ void toraw(const float* f, Raw8<__nv_bfloat16>& o) {
  o.r.x = pack_bf16x2(f[0], f[1]);
  o.r.y = pack_bf16x2(f[2], f[3]);
  o.r.z = pack_bf16x2(f[4], f[5]);
  o.r.w = pack_bf16x2(f[6], f[7]);
}
__device__ __forceinline__ void toraw(const float* f, Raw8<float>& o) {
  o.a = make_float4(f[0], f[1], f[2], f[3]);
  o.b = make_float4(f[4], f[5], f[6], f[7]);
}
__device__ __forceinline__ void straw(__nv_bfloat16* p, const Raw8<__nv_bfloat16>& i) {
  *reinterpret_cast<uint4*>(p) = i.r;
}
__device__ __forceinline__ void straw(float* p, const Raw8<float>& i) {
  *reinterpret_cast<float4*>(p) = i.a;
  *reinterpret_cast<float4*>(p + 4) = i.b;
}

template <typename T, int NVW>
__global__ void __launch_bounds__(RN_THREADS, (sizeof(T) == 2) ? 8 : 4)
rmsnorm_fwd_warp_kernel(const T* __restrict__ x, const T* __restrict__ delta, const T* __restrict__ w,
                        T* __restrict__ sum_out, T* __restrict__ y, float* __restrict__ rstd_out, int rows,
                        int H, float eps) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  for (int row = blockIdx.x * RW_WARPS + warp; row < rows; row += gridDim.x * RW_WARPS) {
    const long long base = (long long)row * H;
    Raw8<T> xr[NVW], dr[NVW];
#pragma unroll
    for (int v = 0; v < NVW; ++v) {
      const int col = (v * 32 + lane) * 8;
      if (col < H) {
        ldraw(x + base + col, xr[v]);
        if (delta) ldraw(delta + base + col, dr[v]);
      }
    }
    float ss = 0.f;
#pragma unroll
    for (int v = 0; v < NVW; ++v) {
      const int col = (v * 32 + lane) * 8;
      if (col < H) {
        float xv[8];
        unraw(xr[v], xv);
        if (delta) {
          float dv[8];
          unraw(dr[v], dv);
#pragma unroll
          for (int j = 0; j < 8; ++j) xv[j] = round_like(xv[j] + dv[j], x);
          toraw(xv, xr[v]);  // exact: the sum was just rounded to the storage type
          straw(sum_out + base + col, xr[v]);
        }
#pragma unroll
        for (int j = 0; j < 8; ++j) ss += xv[j] * xv[j];
      }
    }
    const float tot = warp_sum(ss);
    const float rstd = 1.0f / sqrtf(tot / (float)H + eps);
    if (lane == 0 && rstd_out) rstd_out[row] = rstd;
#pragma unroll
    for (int v = 0; v < NVW; ++v) {
      const int col = (v * 32 + lane) * 8;
      if (col < H) {
        float xv[8], wv[8], o[8];
        unraw(xr[v], xv);
        ld8(w + col, wv);  // 2 KB gain vector: L1-resident
#pragma unroll
        for (int j = 0; j < 8; ++j) o[j] = xv[j] * rstd * wv[j];
        st8(y + base + col, o);
      }
    }
  }
}

// Backward: x, dy (and the residual-stream gradient, when fused) of the whole row stay packed in registers between
// the two passes; all three are requested up front so that one HBM latency covers them.
template <typename T, int NVW>
__global__ void __launch_bounds__(RN_THREADS, (sizeof(T) == 2) ? 5 : 3)
rmsnorm_bwd_warp_kernel(const T* __restrict__ dy, const T* __restrict__ dres, const T* __restrict__ x,
                        const T* __restrict__ w, const float* __restrict__ rstd_in, T* __restrict__ dx,
                        float* __restrict__ dw_part, int rows, int H) {
  extern __shared__ float dw_s[];  // [RW_WARPS - 1][H]
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  float dwv[NVW][8];
#pragma unroll
  for (int v = 0; v < NVW; ++v) {
#pragma unroll
    for (int j = 0; j < 8; ++j) dwv[v][j] = 0.f;
  }
  for (int row = blockIdx.x * RW_WARPS + warp; row < rows; row += gridDim.x * RW_WARPS) {
    const long long base = (long long)row * H;
    const float rstd = rstd_in[row];
    Raw8<T> xr[NVW], gr[NVW], rr[NVW];
#pragma unroll
    for (int v = 0; v < NVW; ++v) {
      const int col = (v * 32 + lane) * 8;
      if (col < H) {
        ldraw(x + base + col, xr[v]);
        ldraw(dy + base + col, gr[v]);
        if (dres) ldraw(dres + base + col, rr[v]);  // requested with x and dy: no second, serialised HBM latency
      }
    }
    float dot = 0.f;
#pragma unroll
    for (int v = 0; v < NVW; ++v) {
      const int col = (v * 32 + lane) * 8;
      if (col < H) {
        float xv[8], gv[8], wv[8];
        unraw(xr[v], xv);
        unraw(gr[v], gv);
        ld8(w + col, wv);  // 2 KB, L1-resident
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          const float gx = gv[j] * xv[j];
          dwv[v][j] += gx * rstd;
          dot += gx * wv[j];
        }
      }
    }
    const float c = warp_sum(dot) / (float)H * rstd * rstd;
#pragma unroll
    for (int v = 0; v < NVW; ++v) {
      const int col = (v * 32 + lane) * 8;
      if (col < H) {
        float xv[8], gv[8], wv[8], o[8];
        unraw(xr[v], xv);
        unraw(gr[v], gv);
        ld8(w + col, wv);
#pragma unroll
        for (int j = 0; j < 8; ++j) o[j] = rstd * (gv[j] * wv[j] - xv[j] * c);
        if (dres) {
          float r[8];
          unraw(rr[v], r);
#pragma unroll
          for (int j = 0; j < 8; ++j) o[j] += r[j];
        }
        st8(dx + base + col, o);
      }
    }
  }
  // fold the four warps' dw partials through smem, one partial row per CTA
  if (warp > 0) {
#pragma unroll
    for (int v = 0; v < NVW; ++v) {
      const int col = (v * 32 + lane) * 8;
      if (col < H) st8(dw_s + (warp - 1) * H + col, dwv[v]);
    }
  }
  __syncthreads();
  if (warp == 0) {
#pragma unroll
    for (int v = 0; v < NVW; ++v) {
      const int col = (v * 32 + lane) * 8;
      if (col < H) {
#pragma unroll
        for (int u = 0; u < RW_WARPS - 1; ++u) {
          float t[8];
          ld8(dw_s + u * H + col, t);
#pragma unroll
          for (int j = 0; j < 8; ++j) dwv[v][j] += t[j];
        }
        st8(dw_part + (long long)blockIdx.x * H + col, dwv[v]);
      }
    }
  }
}

// dw[c] = sum_b dw_part[b, c].  One CTA per 32 columns: warp r sums partial rows r, r+32, ... (128-byte
// coalesced row segments, independent loads in flight), then the 32 row groups fold through smem.
__global__ void __launch_bounds__(1024)
rmsnorm_dw_reduce_kernel(const float* __restrict__ dw_part, float* __restrict__ dw, int nblocks, int H) {
  __shared__ float part[32][33];
  const int cx = threadIdx.x & 31, ry = threadIdx.x >> 5;
  const int c = blockIdx.x * 32 + cx;
  float s0 = 0.f, s1 = 0.f, s2 = 0.f, s3 = 0.f;
  if (c < H) {
    int b = ry;
    for (; b + 96 < nblocks; b += 128) {
      s0 += dw_part[(long long)b * H + c];
      s1 += dw_part[(long long)(b + 32) * H + c];
      s2 += dw_part[(long long)(b + 64) * H + c];
      s3 += dw_part[(long long)(b + 96) * H + c];
    }
    for (; b < nblocks; b += 32) s0 += dw_part[(long long)b * H + c];
  }
  part[ry][cx] = (s0 + s1) + (s2 + s3);
  __syncthreads();
  if (ry == 0 && c < H) {
    float t = 0.f;
#pragma unroll
    for (int r = 0; r < 32; ++r) t += part[r][cx];
    dw[c] = t;
  }
}

// The same column sum for up to 32 norms in ONE launch (blockIdx.y = job), accumulating straight into the weight's
// gradient in its storage type: a Llama backward has 2 norms per layer, and each used to cost four launches (partials,
// this reduction, a dtype copy and autograd's accumulate) -- ~100 sub-10-us kernels per C2 step, mostly launch latency.
struct DwJobs {
  b200_dw_job j[32];
};
__global__ void __launch_bounds__(1024) rmsnorm_dw_reduce_batched_kernel(const __grid_constant__ DwJobs jobs, int H) {
  __shared__ float part[32][33];
  const b200_dw_job& job = jobs.j[blockIdx.y];
  const float* __restrict__ dw_part = job.partials;
  const int nblocks = job.n_partials;
  const int cx = threadIdx.x & 31, ry = threadIdx.x >> 5;
  const int c = blockIdx.x * 32 + cx;
  float s0 = 0.f, s1 = 0.f, s2 = 0.f, s3 = 0.f;
  if (c < H) {
    int b = ry;
    for (; b + 96 < nblocks; b += 128) {
      s0 += dw_part[(long long)b * H + c];
      s1 += dw_part[(long long)(b + 32) * H + c];
      s2 += dw_part[(long long)(b + 64) * H + c];
      s3 += dw_part[(long long)(b + 96) * H + c];
    }
    for (; b < nblocks; b += 32) s0 += dw_part[(long long)b * H + c];
  }
  part[ry][cx] = (s0 + s1) + (s2 + s3);
  __syncthreads();
  if (ry == 0 && c < H) {
    float t = 0.f;
#pragma unroll
    for (int r = 0; r < 32; ++r) t += part[r][cx];
    if (job.dw_is_bf16) {
      __nv_bfloat16* d = reinterpret_cast<__nv_bfloat16*>(job.dw);
      if (job.accumulate) t += __bfloat162float(d[c]);
      d[c] = __float2bfloat16(t);
    } else {
      float* d = reinterpret_cast<float*>(job.dw);
      if (job.accumulate) t += d[c];
      d[c] = t;
    }
  }
}

// x: [B, S, NH, D]; cos/sin: [S, D/2] fp32. out[2i] = x[2i]*c - x[2i+1]*s ; out[2i+1] = x[2i]*s +
// x[2i+1]*c. The backward pass is the same rotation with sign = -1.  POS: token s of row b is rotated by the angle of
// pos[b, s] (its position within its document) instead of s.
template <typename T, bool POS>
__global__ void __launch_bounds__(256)
rope_kernel(const T* __restrict__ x, T* __restrict__ y, const float* __restrict__ cos_t,
            const float* __restrict__ sin_t, long long nvec, int S, int NH, int D, float sign,
            const int* __restrict__ pos) {
  const int vec_per_head = D / 8;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < nvec;
       i += (long long)gridDim.x * blockDim.x) {
    const int dv = (int)(i % vec_per_head);
    const long long t = i / vec_per_head / NH;  // token index b*S + s
    int s;
    if constexpr (POS) s = __ldg(pos + t);
    else s = (int)(t % S);
    float xv[8], o[8];
    ld8(x + i * 8, xv);
    const float4 c = *reinterpret_cast<const float4*>(cos_t + (long long)s * (D / 2) + dv * 4);
    float4 sn = *reinterpret_cast<const float4*>(sin_t + (long long)s * (D / 2) + dv * 4);
    sn.x *= sign; sn.y *= sign; sn.z *= sign; sn.w *= sign;
    o[0] = xv[0] * c.x - xv[1] * sn.x;  o[1] = xv[0] * sn.x + xv[1] * c.x;
    o[2] = xv[2] * c.y - xv[3] * sn.y;  o[3] = xv[2] * sn.y + xv[3] * c.y;
    o[4] = xv[4] * c.z - xv[5] * sn.z;  o[5] = xv[4] * sn.z + xv[5] * c.z;
    o[6] = xv[6] * c.w - xv[7] * sn.w;  o[7] = xv[6] * sn.w + xv[7] * c.w;
    st8(y + i * 8, o);
  }
}

// Half-split RoPE: pairs (x[i], x[i + D/2]) for i < D/2, angle of pair i as in rope_kernel.  One thread per 8-column
// slice i in [8 dv, 8 dv + 8): it loads the 16-byte vectors at column 8 dv and at 8 dv + D/2, both coalesced across
// the warp, which needs D % 16 == 0.  Backward: sign = -1.
template <typename T, bool POS>
__global__ void __launch_bounds__(256)
rope_half_kernel(const T* __restrict__ x, T* __restrict__ y, const float* __restrict__ cos_t,
                 const float* __restrict__ sin_t, long long nslice, int S, int NH, int D, float sign,
                 const int* __restrict__ pos) {
  const int per_head = D / 16;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < nslice;
       i += (long long)gridDim.x * blockDim.x) {
    const int dv = (int)(i % per_head);
    const long long head = i / per_head;  // (b*S + s)*NH + h
    const long long t = head / NH;        // token index b*S + s
    int s;
    if constexpr (POS) s = __ldg(pos + t);
    else s = (int)(t % S);
    const long long lo = head * D + dv * 8, hi = lo + D / 2;
    float xl[8], xh[8], c[8], sn[8], ol[8], oh[8];
    ld8(x + lo, xl);
    ld8(x + hi, xh);
    ld8(cos_t + (long long)s * (D / 2) + dv * 8, c);
    ld8(sin_t + (long long)s * (D / 2) + dv * 8, sn);
#pragma unroll
    for (int k = 0; k < 8; ++k) sn[k] *= sign;
    rope_half8(xl, xh, c, sn, ol, oh);
    st8(y + lo, ol);
    st8(y + hi, oh);
  }
}

constexpr int RW_MAX_H = 1024;  // NVW <= 4: beyond that the packed row no longer fits 128 registers

template <typename T>
int rmsnorm_fwd_t(const T* x, const T* delta, const T* w, T* sum_out, T* y, float* rstd, int rows, int H,
                  float eps, cudaStream_t stream) {
  if (H <= RW_MAX_H) {
    const int want = (rows + RW_WARPS - 1) / RW_WARPS;
    const int nvw = (H + 255) / 256;
    auto launch = [&](auto kern) -> int {
      // exactly one resident wave: a second, partial wave of these short CTAs costs ~20 % on a 30 us kernel
      static int per_sm = 0;
      if (per_sm == 0) {
        int n = 0;
        B200_CHECK_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&n, kern, RN_THREADS, 0));
        per_sm = n > 0 ? n : 1;
      }
      // one resident wave, BALANCED: with `want` row groups and room for `cap` CTAs every CTA gets the same number of
      // rounds (16384 rows: 1024 CTAs x 4 rounds instead of 1184 CTAs of which 46 % sit out the last round)
      const int cap = num_sms() * per_sm;
      const int rounds = (want + cap - 1) / cap;
      const int grid = (want + rounds - 1) / rounds;
      kern<<<grid, RN_THREADS, 0, stream>>>(x, delta, w, sum_out, y, rstd, rows, H, eps);
      return B200_OK;
    };
    int rc;
    if (nvw <= 1) rc = launch(rmsnorm_fwd_warp_kernel<T, 1>);
    else if (nvw <= 2) rc = launch(rmsnorm_fwd_warp_kernel<T, 2>);
    else if (nvw <= 4) rc = launch(rmsnorm_fwd_warp_kernel<T, 4>);
    else rc = launch(rmsnorm_fwd_warp_kernel<T, 8>);
    if (rc) return rc;
    B200_CHECK_LAUNCH();
    return B200_OK;
  }
  const int nv = (H / 8 + RN_THREADS - 1) / RN_THREADS;
  const int grid = rows < num_sms() * 16 ? rows : num_sms() * 16;
  switch (nv) {
    case 1: case 2: case 3: case 4:
      rmsnorm_fwd_kernel<T, 4><<<grid, RN_THREADS, 0, stream>>>(x, delta, w, sum_out, y, rstd, rows, H, eps); break;
    default:
      rmsnorm_fwd_kernel<T, RN_MAX_VEC><<<grid, RN_THREADS, 0, stream>>>(x, delta, w, sum_out, y, rstd, rows, H, eps); break;
  }
  B200_CHECK_LAUNCH();
  return B200_OK;
}

inline int rmsnorm_bwd_grid(int rows, int H) {
  if (H <= RW_MAX_H) {
    const int want = (rows + RW_WARPS - 1) / RW_WARPS;
    const int cap = num_sms() * 5;
    const int rounds = (want + cap - 1) / cap;   // balanced single wave, as in the forward kernel
    return (want + rounds - 1) / rounds;
  }
  return rows < num_sms() * 4 ? rows : num_sms() * 4;
}

template <typename T>
int rmsnorm_bwd_t(const T* dy, const T* dres, const T* x, const T* w, const float* rstd, T* dx, float* dw,
                  float* dw_part, int rows, int H, cudaStream_t stream) {
  const int grid = rmsnorm_bwd_grid(rows, H);
  if (H <= RW_MAX_H) {
    const int nvw = (H + 255) / 256;
    const size_t smem = (size_t)(RW_WARPS - 1) * H * sizeof(float);
    if (nvw <= 1) rmsnorm_bwd_warp_kernel<T, 1><<<grid, RN_THREADS, smem, stream>>>(dy, dres, x, w, rstd, dx, dw_part, rows, H);
    else if (nvw <= 2) rmsnorm_bwd_warp_kernel<T, 2><<<grid, RN_THREADS, smem, stream>>>(dy, dres, x, w, rstd, dx, dw_part, rows, H);
    else if (nvw <= 4) rmsnorm_bwd_warp_kernel<T, 4><<<grid, RN_THREADS, smem, stream>>>(dy, dres, x, w, rstd, dx, dw_part, rows, H);
    else rmsnorm_bwd_warp_kernel<T, 8><<<grid, RN_THREADS, smem, stream>>>(dy, dres, x, w, rstd, dx, dw_part, rows, H);
  } else {
    const int nv = (H / 8 + RN_THREADS - 1) / RN_THREADS;
    if (nv <= 4) rmsnorm_bwd_kernel<T, 4><<<grid, RN_THREADS, 0, stream>>>(dy, dres, x, w, rstd, dx, dw_part, rows, H);
    else rmsnorm_bwd_kernel<T, RN_MAX_VEC><<<grid, RN_THREADS, 0, stream>>>(dy, dres, x, w, rstd, dx, dw_part, rows, H);
  }
  B200_CHECK_LAUNCH();
  if (dw == nullptr) return B200_OK;   // partials stay in the workspace for rmsnorm_dw_reduce (deferred, batched)
  rmsnorm_dw_reduce_kernel<<<(H + 31) / 32, 1024, 0, stream>>>(dw_part, dw, grid, H);
  B200_CHECK_LAUNCH();
  return B200_OK;
}

int rope_impl(const void* x, void* y, const float* cos_t, const float* sin_t, const int* pos, int B, int S, int NH,
              int D, int backward, int is_bf16, cudaStream_t stream) {
  B200_CHECK_ARG(B > 0 && S > 0 && NH > 0 && D > 0 && D % 8 == 0, "rope: D=%d must be a multiple of 8",
                 D);
  B200_CHECK_ARG(al16(x) && al16(y) && al16(cos_t) && al16(sin_t), "rope: alignment");
  const long long nvec = (long long)B * S * NH * D / 8;
  long long blocks = (nvec + 255) / 256;
  if (blocks > (long long)num_sms() * 8) blocks = (long long)num_sms() * 8;
  const float sign = backward ? -1.0f : 1.0f;
  auto launch = [&](auto kern, auto* xx, auto* yy) {
    kern<<<(int)blocks, 256, 0, stream>>>(xx, yy, cos_t, sin_t, nvec, S, NH, D, sign, pos);
  };
  using bf = __nv_bfloat16;
  if (is_bf16) {
    if (pos) launch(rope_kernel<bf, true>, (const bf*)x, (bf*)y);
    else launch(rope_kernel<bf, false>, (const bf*)x, (bf*)y);
  } else {
    if (pos) launch(rope_kernel<float, true>, (const float*)x, (float*)y);
    else launch(rope_kernel<float, false>, (const float*)x, (float*)y);
  }
  B200_CHECK_LAUNCH();
  return B200_OK;
}

}  // namespace
}  // namespace b200

using namespace b200;

extern "C" {

int b200_add_rmsnorm_fwd(const void* x, const void* delta, const void* w, void* sum_out, void* y, float* rstd,
                         int rows, int H, float eps, int is_bf16, void* stream) {
  const cudaStream_t s = static_cast<cudaStream_t>(stream);
  B200_CHECK_ARG(rows > 0 && H > 0 && H % 8 == 0 && H <= RN_THREADS * 8 * RN_MAX_VEC,
                 "rmsnorm_fwd: unsupported shape rows=%d H=%d (H %% 8 == 0, H <= %d)", rows, H,
                 RN_THREADS * 8 * RN_MAX_VEC);
  B200_CHECK_ARG(al16(x) && al16(w) && al16(y) && al16(delta) && al16(sum_out),
                 "rmsnorm_fwd: 16-byte alignment required");
  B200_CHECK_ARG((delta == nullptr) == (sum_out == nullptr),
                 "add_rmsnorm_fwd: delta and sum_out must be given together");
  if (is_bf16)
    return rmsnorm_fwd_t<__nv_bfloat16>((const __nv_bfloat16*)x, (const __nv_bfloat16*)delta,
                                        (const __nv_bfloat16*)w, (__nv_bfloat16*)sum_out, (__nv_bfloat16*)y,
                                        rstd, rows, H, eps, s);
  return rmsnorm_fwd_t<float>((const float*)x, (const float*)delta, (const float*)w, (float*)sum_out,
                              (float*)y, rstd, rows, H, eps, s);
}

int b200_rmsnorm_fwd(const void* x, const void* w, void* y, float* rstd, int rows, int H, float eps,
                     int is_bf16, void* stream) {
  return b200_add_rmsnorm_fwd(x, nullptr, w, nullptr, y, rstd, rows, H, eps, is_bf16, stream);
}

size_t b200_rmsnorm_bwd_workspace_bytes(int rows, int H) {
  return (size_t)rmsnorm_bwd_grid(rows, H) * H * sizeof(float);
}

int b200_rmsnorm_bwd_partial_rows(int rows, int H) { return rmsnorm_bwd_grid(rows, H); }

int b200_rmsnorm_dw_reduce(const b200_dw_job* jobs, int n_jobs, int H, void* stream) {
  B200_CHECK_ARG(n_jobs >= 0 && H > 0 && (jobs != nullptr || n_jobs == 0), "rmsnorm_dw_reduce: bad arguments");
  for (int i = 0; i < n_jobs; ++i)
    B200_CHECK_ARG(jobs[i].partials != nullptr && jobs[i].dw != nullptr && jobs[i].n_partials > 0,
                   "rmsnorm_dw_reduce: job %d has a null pointer or no partial rows", i);
  for (int i = 0; i < n_jobs; i += 32) {
    DwJobs a;
    const int n = n_jobs - i < 32 ? n_jobs - i : 32;
    for (int k = 0; k < n; ++k) a.j[k] = jobs[i + k];
    rmsnorm_dw_reduce_batched_kernel<<<dim3((H + 31) / 32, n), 1024, 0, static_cast<cudaStream_t>(stream)>>>(a, H);
    B200_CHECK_LAUNCH();
  }
  return B200_OK;
}

int b200_add_rmsnorm_bwd(const void* dy, const void* dres, const void* x, const void* w, const float* rstd,
                         void* dx, float* dw, int rows, int H, int is_bf16, void* ws, size_t ws_bytes,
                         void* stream) {
  const cudaStream_t s = static_cast<cudaStream_t>(stream);
  B200_CHECK_ARG(rows > 0 && H > 0 && H % 8 == 0 && H <= RN_THREADS * 8 * RN_MAX_VEC,
                 "rmsnorm_bwd: unsupported shape rows=%d H=%d", rows, H);
  B200_CHECK_ARG(al16(dy) && al16(x) && al16(w) && al16(dx) && al16(dres), "rmsnorm_bwd: alignment");
  if (ws == nullptr || ws_bytes < b200_rmsnorm_bwd_workspace_bytes(rows, H)) {
    set_error("rmsnorm_bwd: workspace too small (%zu < %zu)", ws_bytes, b200_rmsnorm_bwd_workspace_bytes(rows, H));
    return B200_ERR_WORKSPACE;
  }
  float* part = reinterpret_cast<float*>(ws);
  if (is_bf16)
    return rmsnorm_bwd_t<__nv_bfloat16>((const __nv_bfloat16*)dy, (const __nv_bfloat16*)dres,
                                        (const __nv_bfloat16*)x, (const __nv_bfloat16*)w, rstd,
                                        (__nv_bfloat16*)dx, dw, part, rows, H, s);
  return rmsnorm_bwd_t<float>((const float*)dy, (const float*)dres, (const float*)x, (const float*)w, rstd,
                              (float*)dx, dw, part, rows, H, s);
}

int b200_rmsnorm_bwd(const void* dy, const void* x, const void* w, const float* rstd, void* dx,
                     float* dw, int rows, int H, int is_bf16, void* ws, size_t ws_bytes,
                     void* stream) {
  return b200_add_rmsnorm_bwd(dy, nullptr, x, w, rstd, dx, dw, rows, H, is_bf16, ws, ws_bytes, stream);
}


// pos: nullable int32 [B, S]; D % 16 == 0 (both halves of a slice are 16-byte vectors)
int b200_rope_half(const void* x, void* y, const float* cos_t, const float* sin_t, const int* pos, int B, int S, int NH,
                   int D, int backward, int is_bf16, void* stream) {
  B200_CHECK_ARG(B > 0 && S > 0 && NH > 0 && D > 0 && D % 16 == 0, "rope_half: D=%d must be a multiple of 16", D);
  B200_CHECK_ARG(al16(x) && al16(y) && al16(cos_t) && al16(sin_t) && (reinterpret_cast<uintptr_t>(pos) & 3u) == 0,
                 "rope_half: alignment");
  const long long nslice = (long long)B * S * NH * D / 16;
  long long blocks = (nslice + 255) / 256;
  if (blocks > (long long)num_sms() * 8) blocks = (long long)num_sms() * 8;
  const float sign = backward ? -1.0f : 1.0f;
  auto launch = [&](auto kern, auto* xx, auto* yy) {
    kern<<<(int)blocks, 256, 0, static_cast<cudaStream_t>(stream)>>>(xx, yy, cos_t, sin_t, nslice, S, NH, D, sign, pos);
  };
  using bf = __nv_bfloat16;
  if (is_bf16) {
    if (pos) launch(rope_half_kernel<bf, true>, (const bf*)x, (bf*)y);
    else launch(rope_half_kernel<bf, false>, (const bf*)x, (bf*)y);
  } else {
    if (pos) launch(rope_half_kernel<float, true>, (const float*)x, (float*)y);
    else launch(rope_half_kernel<float, false>, (const float*)x, (float*)y);
  }
  B200_CHECK_LAUNCH();
  return B200_OK;
}

int b200_rope(const void* x, void* y, const float* cos_t, const float* sin_t, int B, int S, int NH,
              int D, int backward, int is_bf16, void* stream) {
  return rope_impl(x, y, cos_t, sin_t, nullptr, B, S, NH, D, backward, is_bf16, static_cast<cudaStream_t>(stream));
}

// pos: int32 [B, S]; the tables must cover max(pos) + 1 rows
int b200_rope_pos(const void* x, void* y, const float* cos_t, const float* sin_t, const int* pos, int B, int S, int NH,
                  int D, int backward, int is_bf16, void* stream) {
  B200_CHECK_ARG(pos != nullptr && (reinterpret_cast<uintptr_t>(pos) & 3u) == 0,
                 "rope_pos: pos must be a non-null, 4-byte aligned int32 [B, S] array");
  return rope_impl(x, y, cos_t, sin_t, pos, B, S, NH, D, backward, is_bf16, static_cast<cudaStream_t>(stream));
}

}  // extern "C"
