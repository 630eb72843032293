// Fused causal / GQA attention backward on Hopper warpgroup MMA (wgmma) fed by TMA through mbarriers: the adjoint
// the reference obtains from MLX autograd of arch/flash_attention.py:123-151 (core/training.py:1580,1650),
// including the sum of dK/dV over the query heads that share a kv head (adjoint of mx.repeat, :107-120).
//
//   delta = rowsum(dO * O)                                  (pre-pass kernel, also zeroes the dQ accumulator)
//   per (128-key tile, kv head, batch) CTA, 256 threads: thread 0 loads K / V once by TMA and prefetches the Q / dO tiles
//   (64 queries) of every query head of the GQA group one item ahead through a 2-stage ring; warpgroups 0-1 own 64 keys
//   each (a separate producer warp would cap the MMA warpgroups at 168 registers and make them spill):
//     S^T  = K Q^T , dP^T = V dO^T          wgmma, both operands K-major in shared memory
//     P^T  = exp2(S^T * scale*log2e - LSE*log2e),  dS^T = P^T * (dP^T - delta)      (registers)
//     dV  += P^T dO , dK += dS^T Q          wgmma with P^T / dS^T as register A operands, dO / Q MN-major in smem
//     dS^T -> shared memory (the 128B-swizzled MN-major layout wgmma reads), then dQ_tile = dS K as wgmma with
//     both operands MN-major, added into the fp32 dq_acc with atomics
//   dq_acc (fp32) * scale -> dq (bf16)                       (post-pass kernel)
// dK and dQ leave the softmax scale out of dS and apply it once at the end.
#include "common.cuh"
#include "host.h"

namespace b200 {

int make_bshd_map(CUtensorMap* tm, const void* base, int B, int S, int heads, int D, int box_rows);

namespace {

constexpr int BWD_THREADS = 256;  // two MMA warpgroups; thread 0 also issues the TMA loads
constexpr int BKV = 128;          // keys per CTA (64 per warpgroup)
constexpr int BQ = 64;            // queries per inner tile
constexpr float kLog2e = 1.4426950408889634f;

template <int D>
struct BwdCfg {
  static constexpr int NB = D / 64;                // 64-column (128-byte) blocks per row
  static constexpr int KV_BYTES = BKV * D * 2;     // K or V
  static constexpr int QS_BYTES = BQ * D * 2;      // one Q or dO stage
  static constexpr int OFF_K = 0;
  static constexpr int OFF_V = OFF_K + KV_BYTES;
  static constexpr int OFF_Q = OFF_V + KV_BYTES;        // 2 stages
  static constexpr int OFF_DO = OFF_Q + 2 * QS_BYTES;   // 2 stages
  static constexpr int OFF_DS = OFF_DO + 2 * QS_BYTES;  // dS^T [128 keys][64 queries] bf16
  static constexpr int OFF_BAR = OFF_DS + BKV * BQ * 2;
  static constexpr int SMEM_BYTES = OFF_BAR + 64 + 1024;
};

struct BwdArgs {
  const float* lse;    // [B,H,S]
  const float* delta;  // [B,H,S]
  float* dq_acc;       // [B,S,H,D] fp32
  __nv_bfloat16* dk;   // [B,S,dkv_rh,D]-strided rows
  __nv_bfloat16* dv;
  int B, S, H, Hk;
  int dkv_rh;          // heads per dk/dv token row (>= Hk)
  float scale;
  int causal;
};

template <int D>
__device__ __forceinline__ void rs_mma(float* acc, const uint32_t* a, uint64_t db) {
  if constexpr (D == 128) wgmma_m64n128k16_rs<1>(acc, a, db);
  else wgmma_m64n64k16_rs<1>(acc, a, db);
}

template <int D>
__global__ void __launch_bounds__(BWD_THREADS, 1)
attn_bwd_kernel(const __grid_constant__ CUtensorMap tmQ, const __grid_constant__ CUtensorMap tmK,
                const __grid_constant__ CUtensorMap tmV, const __grid_constant__ CUtensorMap tmDO, const BwdArgs p) {
  using Cfg = BwdCfg<D>;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  const uint32_t s0 = smem_u32(smem);
  const uint32_t sK = s0 + Cfg::OFF_K, sV = s0 + Cfg::OFF_V, sQ = s0 + Cfg::OFF_Q, sDO = s0 + Cfg::OFF_DO;
  const uint32_t sDS = s0 + Cfg::OFF_DS;
  const uint32_t kv_full = s0 + Cfg::OFF_BAR, q_full0 = kv_full + 8, q_empty0 = kv_full + 24;
  const int kt = blockIdx.x, hk = blockIdx.y, b = blockIdx.z;
  const int k0 = kt * BKV;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int group = p.H / p.Hk;
  const int n_qt = (p.S + BQ - 1) / BQ;
  const int qt_first = p.causal ? k0 / BQ : 0;
  const int per_head = n_qt - qt_first;
  const int n_items = group * per_head;

  if (threadIdx.x == 0) {
    mbar_init(kv_full, 1);
    for (int s = 0; s < 2; ++s) {
      mbar_init(q_full0 + 8 * s, 1);
      mbar_init(q_empty0 + 8 * s, 2);  // one arrival per consumer warpgroup
    }
    fence_mbar_init();
  }
  __syncthreads();

  // one elected thread: K / V once, then the Q / dO tiles of item `it` into stage it % 2 once both warpgroups
  // have released that stage (item it - 2)
  auto issue_item = [&](int it) {
    const int s = it & 1;
    const int h = hk * group + it / per_head;
    const int q0 = (qt_first + it % per_head) * BQ;
    mbar_wait(q_empty0 + 8 * s, ((it >> 1) & 1) ^ 1u);
    const uint32_t full = q_full0 + 8 * s;
    mbar_arrive_expect_tx(full, 2 * Cfg::QS_BYTES);
    for (int nb = 0; nb < Cfg::NB; ++nb) {
      tma_load_4d(sQ + s * Cfg::QS_BYTES + nb * BQ * 128, &tmQ, full, nb * 64, h, q0, b);
      tma_load_4d(sDO + s * Cfg::QS_BYTES + nb * BQ * 128, &tmDO, full, nb * 64, h, q0, b);
    }
  };
  if (threadIdx.x == 0) {
    mbar_arrive_expect_tx(kv_full, 2 * Cfg::KV_BYTES);
    for (int nb = 0; nb < Cfg::NB; ++nb) {
      tma_load_4d(sK + nb * BKV * 128, &tmK, kv_full, nb * 64, hk, k0, b);
      tma_load_4d(sV + nb * BKV * 128, &tmV, kv_full, nb * 64, hk, k0, b);
    }
    if (n_items > 0) issue_item(0);
  }

  const int wg = warp >> 2, wq = warp & 3;
  const int g = lane >> 2, cq = (lane & 3) * 2;
  const int key_a = k0 + wg * 64 + wq * 16 + g;  // this thread's keys: key_a, key_a + 8
  float dk[D / 2], dv[D / 2];
#pragma unroll
  for (int i = 0; i < D / 2; ++i) dk[i] = dv[i] = 0.f;
  const float sl2 = p.scale * kLog2e;
  mbar_wait(kv_full, 0);

  for (int it = 0; it < n_items; ++it) {
    const int s = it & 1;
    const int h = hk * group + it / per_head;
    const int q0 = (qt_first + it % per_head) * BQ;
    if (threadIdx.x == 0 && it + 1 < n_items) issue_item(it + 1);
    mbar_wait(q_full0 + 8 * s, (it >> 1) & 1);
    const uint32_t tQ = sQ + s * Cfg::QS_BYTES, tDO = sDO + s * Cfg::QS_BYTES;

    // S^T = K Q^T and dP^T = V dO^T: 64 keys x 64 queries per warpgroup
    float st[32], dpt[32];
#pragma unroll
    for (int i = 0; i < 32; ++i) st[i] = dpt[i] = 0.f;
    wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < D / 16; ++kk) {
      const uint32_t ka = (kk >> 2) * BKV * 128 + wg * 64 * 128 + (kk & 3) * 32;
      const uint32_t qb = (kk >> 2) * BQ * 128 + (kk & 3) * 32;
      wgmma_m64n64k16_ss<0, 0>(st, make_wgmma_desc_sw128(sK + ka, 16, 1024), make_wgmma_desc_sw128(tQ + qb, 16, 1024));
      wgmma_m64n64k16_ss<0, 0>(dpt, make_wgmma_desc_sw128(sV + ka, 16, 1024), make_wgmma_desc_sw128(tDO + qb, 16, 1024));
    }
    wgmma_commit();
    wgmma_wait<0>();

    // P^T and dS^T (unscaled); masked entries are exactly 0.  Chunk nc holds queries 8 nc + cq + {0, 1}.
    const long long lrow = ((long long)b * p.H + h) * p.S;
#pragma unroll
    for (int nc = 0; nc < 8; ++nc) {
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const int qi = q0 + nc * 8 + cq + (e & 1);
        const int key = key_a + ((e >> 1) << 3);
        const bool ok = qi < p.S && key < p.S && !(p.causal && key > qi);
        const float pv = ok ? exp2f(st[4 * nc + e] * sl2 - p.lse[lrow + qi] * kLog2e) : 0.f;
        st[4 * nc + e] = pv;
        dpt[4 * nc + e] = ok ? pv * (dpt[4 * nc + e] - p.delta[lrow + qi]) : 0.f;
      }
    }
    uint32_t pa[4][4], da[4][4];
#pragma unroll
    for (int kk = 0; kk < 4; ++kk) {
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        pa[kk][i] = pack_bf16x2(st[8 * kk + 2 * i], st[8 * kk + 2 * i + 1]);
        da[kk][i] = pack_bf16x2(dpt[8 * kk + 2 * i], dpt[8 * kk + 2 * i + 1]);
      }
    }
    // dS^T rows of this thread -> [key][64 queries] tile, 128 B per row, 16-byte chunks XOR (row % 8)
    {
      const int r = wg * 64 + wq * 16 + g;
#pragma unroll
      for (int kk = 0; kk < 4; ++kk) {
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          const int row = r + ((i & 1) << 3), chunk = 2 * kk + (i >> 1);
          *reinterpret_cast<uint32_t*>(smem + Cfg::OFF_DS + row * 128 + ((chunk ^ (row & 7)) << 4) + cq * 2) = da[kk][i];
        }
      }
    }
    fence_proxy_async_smem();  // generic-proxy stores -> visible to the wgmma (async proxy) reads below

    // dV += P^T dO, dK += dS^T Q: k = queries (16 rows of 128 B per step), n = head dim (64-column blocks)
    wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < 4; ++kk) rs_mma<D>(dv, pa[kk], make_wgmma_desc_sw128(tDO + kk * 2048, BQ * 128, 1024));
#pragma unroll
    for (int kk = 0; kk < 4; ++kk) rs_mma<D>(dk, da[kk], make_wgmma_desc_sw128(tQ + kk * 2048, BQ * 128, 1024));
    wgmma_commit();
    named_bar_sync(1, 256);  // both warpgroups' dS^T rows are in shared memory

    // dQ[64 queries, head-dim block] = dS K over all 128 keys; at D = 64 warpgroup 0 does the whole tile
    float dq[32];
    const bool do_dq = (D == 128) || wg == 0;
    const int nblk = (D == 128) ? wg : 0;
    if (do_dq) {
#pragma unroll
      for (int i = 0; i < 32; ++i) dq[i] = 0.f;
      wgmma_fence();
#pragma unroll
      for (int kk = 0; kk < BKV / 16; ++kk)
        wgmma_m64n64k16_ss<1, 1>(dq, make_wgmma_desc_sw128(sDS + kk * 2048, 8192, 1024),
                                 make_wgmma_desc_sw128(sK + nblk * BKV * 128 + kk * 2048, BKV * 128, 1024));
      wgmma_commit();
    }
    wgmma_wait<0>();
    if ((threadIdx.x & 127) == 0) mbar_arrive(q_empty0 + 8 * s);
    if (do_dq) {
      float* dqb = p.dq_acc + ((long long)b * p.S * p.H + h) * D + nblk * 64;
#pragma unroll
      for (int r = 0; r < 2; ++r) {
        const int qi = q0 + wq * 16 + g + 8 * r;
        if (qi >= p.S) continue;
        float* row = dqb + (long long)qi * p.H * D + cq;
#pragma unroll
        for (int nc = 0; nc < 8; ++nc) {
          atomicAdd(row + nc * 8, dq[4 * nc + 2 * r]);
          atomicAdd(row + nc * 8 + 1, dq[4 * nc + 2 * r + 1]);
        }
      }
    }
    named_bar_sync(1, 256);  // the dS^T tile is rewritten by the next item
  }

  // dK (scale applied here), dV -> bf16 rows of dkv_rh heads
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    const int key = key_a + 8 * r;
    if (key >= p.S) continue;
    const long long off = ((long long)b * p.S + key) * p.dkv_rh * D + (long long)hk * D + cq;
#pragma unroll
    for (int dc = 0; dc < D / 8; ++dc) {
      *reinterpret_cast<uint32_t*>(p.dk + off + dc * 8) =
          pack_bf16x2(dk[4 * dc + 2 * r] * p.scale, dk[4 * dc + 2 * r + 1] * p.scale);
      *reinterpret_cast<uint32_t*>(p.dv + off + dc * 8) = pack_bf16x2(dv[4 * dc + 2 * r], dv[4 * dc + 2 * r + 1]);
    }
  }
}

// delta[b,h,s] = sum_d o[b,s,h,d] * do[b,s,h,d]; LPR = D/8 lanes cooperate on one row.  The same pass zeroes the
// fp32 dQ accumulator (same [B,S,H,D] index space: each thread clears the 8 floats under the 8 bf16 it reads), so the
// backward needs no separate memset launch over 4*B*S*H*D bytes.
template <int D>
__global__ void __launch_bounds__(256)
attn_delta_kernel(const __nv_bfloat16* __restrict__ o, const __nv_bfloat16* __restrict__ d_o,
                  float* __restrict__ delta, float* __restrict__ dq_acc, int B, int S, int H) {
  constexpr int LPR = D / 8;
  const long long rows = (long long)B * S * H;
  const long long gtid = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const long long r = gtid / LPR;
  const int sub = (int)(gtid % LPR);
  float acc = 0.f;
  if (r < rows) {
    const uint4 a = ldg128(o + r * D + sub * 8);
    const uint4 c = ldg128(d_o + r * D + sub * 8);
    float4* z = reinterpret_cast<float4*>(dq_acc + r * D + sub * 8);
    z[0] = make_float4(0.f, 0.f, 0.f, 0.f);
    z[1] = make_float4(0.f, 0.f, 0.f, 0.f);
    const uint32_t* au = &a.x;
    const uint32_t* cu = &c.x;
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const float2 x = unpack_bf16x2(au[i]), y = unpack_bf16x2(cu[i]);
      acc += x.x * y.x + x.y * y.y;
    }
  }
#pragma unroll
  for (int off = LPR / 2; off > 0; off >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, off);
  if (r < rows && sub == 0) {
    const int hh = (int)(r % H);
    const long long bs = r / H;
    const int s = (int)(bs % S);
    const long long bb = bs / S;
    delta[(bb * H + hh) * S + s] = acc;
  }
}

__global__ void __launch_bounds__(256)
f32_to_bf16_kernel(const float* __restrict__ src, __nv_bfloat16* __restrict__ dst, long long nvec, float mul) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < nvec;
       i += (long long)gridDim.x * blockDim.x) {
    const float4 a = *reinterpret_cast<const float4*>(src + i * 8);
    const float4 c = *reinterpret_cast<const float4*>(src + i * 8 + 4);
    uint4 o4;
    o4.x = pack_bf16x2(a.x * mul, a.y * mul);
    o4.y = pack_bf16x2(a.z * mul, a.w * mul);
    o4.z = pack_bf16x2(c.x * mul, c.y * mul);
    o4.w = pack_bf16x2(c.z * mul, c.w * mul);
    stg128(dst + i * 8, o4);
  }
}

template <int D>
int launch_bwd(const CUtensorMap& tmQ, const CUtensorMap& tmK, const CUtensorMap& tmV, const CUtensorMap& tmDO,
               const BwdArgs& a, cudaStream_t stream) {
  using Cfg = BwdCfg<D>;
  auto kern = attn_bwd_kernel<D>;
  static bool attr_set = false;
  if (!attr_set) {
    B200_CHECK_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg::SMEM_BYTES));
    attr_set = true;
  }
  dim3 grid((a.S + BKV - 1) / BKV, a.Hk, a.B);
  kern<<<grid, BWD_THREADS, Cfg::SMEM_BYTES, stream>>>(tmQ, tmK, tmV, tmDO, a);
  B200_CHECK_LAUNCH();
  return B200_OK;
}

inline size_t al256(size_t x) { return (x + 255) & ~size_t(255); }

}  // namespace

size_t attn_bwd_workspace_bytes(int B, int S, int H, int Hk, int D) {
  (void)Hk;
  return al256((size_t)B * S * H * D * 4) + al256((size_t)B * H * S * 4);
}

int attn_bwd(const void* q, const void* k, const void* v, const void* o, const void* d_o,
             const float* lse, void* dq, void* dk, void* dv, int B, int S, int H, int Hk, int D,
             float scale, int causal, int dkv_row_heads, void* ws, size_t ws_bytes, cudaStream_t stream) {
  // dk / dv rows may be strided: dkv_row_heads heads per token row (0 = Hk, i.e. contiguous [B,S,Hk,D]).
  // With dk = base, dv = base + Hk*D and dkv_row_heads = 2*Hk both land in ONE [B,S,2*Hk*D] buffer, which lets
  // the k/v projections' dgrad and wgrad run as single GEMMs over the concatenated weight.
  if (dkv_row_heads <= 0) dkv_row_heads = Hk;
  B200_CHECK_ARG(dkv_row_heads >= Hk, "attn_bwd: dkv_row_heads=%d < Hk=%d", dkv_row_heads, Hk);
  B200_CHECK_ARG(B > 0 && S > 0 && H > 0 && Hk > 0 && H % Hk == 0,
                 "attn_bwd: bad shape B=%d S=%d H=%d Hk=%d", B, S, H, Hk);
  B200_CHECK_ARG(D == 64 || D == 128, "attn_bwd: head_dim %d unsupported (64 or 128)", D);
  if (ws_bytes < attn_bwd_workspace_bytes(B, S, H, Hk, D)) {
    set_error("attn_bwd: workspace too small (%zu < %zu)", ws_bytes,
              attn_bwd_workspace_bytes(B, S, H, Hk, D));
    return B200_ERR_WORKSPACE;
  }
  B200_CHECK_ARG((reinterpret_cast<uintptr_t>(ws) & 255u) == 0, "attn_bwd: workspace must be 256-byte aligned");
  B200_CHECK_ARG(((reinterpret_cast<uintptr_t>(q) | reinterpret_cast<uintptr_t>(k) | reinterpret_cast<uintptr_t>(v) |
                   reinterpret_cast<uintptr_t>(o) | reinterpret_cast<uintptr_t>(d_o)) & 15u) == 0,
                 "attn_bwd: q/k/v/o/do must be 16-byte aligned");
  float* dq_acc = reinterpret_cast<float*>(ws);
  float* delta = reinterpret_cast<float*>(reinterpret_cast<char*>(ws) + al256((size_t)B * S * H * D * 4));
  const long long n = (long long)B * S * H * D;
  {
    const long long threads = (long long)B * S * H * (D / 8);
    const int blocks = (int)((threads + 255) / 256);
    if (D == 64)
      attn_delta_kernel<64><<<blocks, 256, 0, stream>>>((const __nv_bfloat16*)o, (const __nv_bfloat16*)d_o, delta, dq_acc, B, S, H);
    else
      attn_delta_kernel<128><<<blocks, 256, 0, stream>>>((const __nv_bfloat16*)o, (const __nv_bfloat16*)d_o, delta, dq_acc, B, S, H);
    B200_CHECK_LAUNCH();
  }
  CUtensorMap tmQ, tmK, tmV, tmDO;
  int rc;
  if ((rc = make_bshd_map(&tmQ, q, B, S, H, D, BQ))) return rc;
  if ((rc = make_bshd_map(&tmK, k, B, S, Hk, D, BKV))) return rc;
  if ((rc = make_bshd_map(&tmV, v, B, S, Hk, D, BKV))) return rc;
  if ((rc = make_bshd_map(&tmDO, d_o, B, S, H, D, BQ))) return rc;
  BwdArgs a;
  a.lse = lse;
  a.delta = delta;
  a.dq_acc = dq_acc;
  a.dk = reinterpret_cast<__nv_bfloat16*>(dk);
  a.dv = reinterpret_cast<__nv_bfloat16*>(dv);
  a.B = B;
  a.S = S;
  a.H = H;
  a.Hk = Hk;
  a.dkv_rh = dkv_row_heads;
  a.scale = scale;
  a.causal = causal;
  rc = D == 64 ? launch_bwd<64>(tmQ, tmK, tmV, tmDO, a, stream) : launch_bwd<128>(tmQ, tmK, tmV, tmDO, a, stream);
  if (rc) return rc;
  {
    const long long nvec = n / 8;
    long long blocks = (nvec + 255) / 256;
    if (blocks > (long long)num_sms() * 8) blocks = (long long)num_sms() * 8;
    // the kernel accumulates dS without the softmax scale: applied here
    f32_to_bf16_kernel<<<(int)blocks, 256, 0, stream>>>(dq_acc, reinterpret_cast<__nv_bfloat16*>(dq), nvec, scale);
    B200_CHECK_LAUNCH();
  }
  return B200_OK;
}

}  // namespace b200
