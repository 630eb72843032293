// Fused causal / GQA attention backward on Hopper warpgroup MMA (wgmma) fed by TMA through mbarriers: the adjoint
// the reference obtains from MLX autograd of arch/flash_attention.py:123-151 (core/training.py:1580,1650),
// including the sum of dK/dV over the query heads that share a kv head (adjoint of mx.repeat, :107-120).
//
//   delta = rowsum(dO * O), LSE * log2e                     (pre-pass kernel, also zeroes the dQ accumulator)
//   per CTA: one 128-key tile of one (kv head, batch), or a pair of them (below); 384 threads in 3 roles:
//     warp 0         producer: K / V once per key tile, then the Q / dO tiles (64 queries) of every query head of the
//                    GQA group through a ring of STAGES stages, with the tile's 64 LSE and delta values (bulk copies
//                    on the same mbarrier)
//     warp 1         dQ writer: adds each item's fp32 dQ tile from shared memory into the fp32 dq_acc with TMA
//                    reductions (cp.reduce.async.bulk.tensor .add), then releases the buffer
//     warpgroups 1-2 consumers, 64 keys each:
//       S^T  = K Q^T , dP^T = V dO^T          wgmma, both operands K-major in shared memory
//       P^T  = exp2(S^T * scale*log2e - LSE*log2e),  dS^T = P^T * (dP^T - delta)      (registers; the causal / bounds
//                                             mask only on tiles that cross the diagonal or the sequence end)
//       dV  += P^T dO , dK += dS^T Q          wgmma with P^T / dS^T as register A operands, dO / Q MN-major in smem
//       dS^T -> shared memory (the 128B-swizzled MN-major layout wgmma reads, double-buffered), then
//       dQ_tile = dS K over all 128 keys, split between the warpgroups by head-dim columns, -> a double-buffered
//       fp32 shared tile in the 128B-swizzled layout of the dq_acc tensor map
//   dq_acc (fp32) * scale -> dq (bf16)                       (post-pass kernel)
// dK and dQ leave the softmax scale out of dS and apply it once at the end.
//
// Causal balance: key tile t has work for the queries from t*128 on, so tile 0 has n_kt times the items of the last
// one.  With an even tile count a CTA runs tile t and then tile n_kt-1-t (equal work in every CTA); the n_kt/2 CTAs of
// one (kv head, batch) are adjacent in launch order and share its Q / dO rows in L2.
//
// Document variant (DOC = true, packed sequences; pos[b, s] = position of token s within its document, so query q sees
// keys q - pos[q] .. q).  The pre-pass also writes each token's document start (rows of S_pad ints) and, per (row,
// key tile), the end of the query-tile range: the tile holding the last token of the document that contains the key
// tile's last key.  Query tiles past it see none of the tile's keys and are skipped.  Each item's 64 document starts
// arrive with its LSE and delta; the mask `key >= q - pos[q]` joins the causal one only on items whose queries'
// highest document start lies above the warpgroup's first key.  Document launches use the unpaired order.  DOC = false
// compiles to the causal / non-causal kernels unchanged.
//
// Sliding window (same DOC kernels): query q sees keys q - min(pos[q], W) .. q, the document mask with pos clamped at W
// (pos == nullptr reads as pos[q] = q).  Only the pre-pass knows about W: it writes the clamped starts, and bounds each
// key tile's query range by k0 + BKV - 1 + W as well, since no later query reaches back to the tile.  The starts stay
// monotone, so the kernel's skipping, masked-item test and binary search are unchanged.
//
// ALiBi (ALIBI = true, DOC kernels only): P^T = exp2(S^T * scale*log2e + b - LSE*log2e) with the forward's bias
// b = m_h log2e (k - q) of the item's query head h (slopes[h], read once per item: items run over the GQA group's
// heads), on the masked and the unmasked path alike.  The bias is constant in Q and K, so dS^T = P^T (dP^T - delta) and
// the pre-pass are unchanged.  A thread's queries are q0 + 8 nc + cq + {0, 1}: per item one integer per key is
// converted, base = m log2e (key - q0 - cq), and each element's bias is fmaf(m log2e, -c, base) for the compile-time
// column c.  With m = 0 the bias is exactly 0 and P^T is the DOC kernel's.  ALIBI = false compiles unchanged.
//
// Prefix-LM (PREFIX = true, causal DOC = false kernels only): query q sees key k iff k <= q or k < P_b, with
// P_b = prefix[b] clamped to [0, S].  A key tile below P_b is seen by every query, so its query range starts at query
// tile 0; other key tiles start at the causal k0 / BQ.  An item is masked when the warpgroup's last key exceeds
// max(q0, P_b - 1) or it crosses S, and the element mask is `key > q && key >= P_b` plus the bounds.  The pre-pass is
// unchanged.  Prefix launches use the unpaired order: the causal pairing no longer balances the work.  P_b <= 1 gives
// the causal kernel's items and values.  PREFIX = false compiles unchanged.
//
// Dropout (DROP = true, on the causal / non-causal and the DOC / ALiBi kernels): the adjoint of the forward's
// O = (P o Z / (1 - p_eff)) V, with Z regenerated from (seed, b, h, q, k) by the forward's Philox rule (nothing of size
// S^2 is stored): dV = (P o Z)^T dO / (1 - p_eff) and dS = P o (Z o dP / (1 - p_eff) - delta), where delta =
// rowsum(dO o O) of the dropped O, so the pre-pass is unchanged.  P^T stays the dropout-free softmax for dS; the bf16
// P^T fed to the dV MMA has the dropped entries zeroed, dV gets the scale in fp32 at the store, and dS gets it on dP in
// registers (dS = P (dP zs - delta) with zs the scale or 0; the packed P^T halves are masked after packing, which
// keeps the D = 128 document kernel's masked-item path free of spills).  A thread's element (nc, e) is query
// q0 + 8 nc + cq + (e & 1) against key key_a + 8 (e >> 1): the 8 lanes g = 0..7 of one cq share one Philox call per (query, 8-key chunk) and take bit g of it.  Lane g computes the
// 4 calls of its group's elements (nc = g, e = 0..3) and the group exchanges them with 8 shuffles, so bit 4 nc + e of
// zk is element (nc, e)'s keep bit.  DROP = false compiles unchanged.
#include "common.cuh"
#include "host.h"

namespace b200 {
namespace {

constexpr int BWD_THREADS = 384;  // producer / dQ-writer warpgroup + two MMA warpgroups
constexpr int BKV = 128;          // keys per tile (64 per consumer warpgroup)
constexpr int BQ = 64;            // queries per item
constexpr float kLog2e = 1.4426950408889634f;

template <int D, bool DOC = false>
struct BwdCfg {
  static constexpr int NB = D / 64;                 // 64-column (128-byte) blocks per bf16 row
  static constexpr int STAGES = D == 64 ? 3 : 2;    // Q / dO ring depth (D = 128: two fill the shared memory)
  static constexpr int KV_BYTES = BKV * D * 2;      // K or V
  static constexpr int QS_BYTES = BQ * D * 2;       // one Q or dO stage
  static constexpr int DS_BYTES = BKV * BQ * 2;     // dS^T [128 keys][64 queries] bf16
  static constexpr int DQ_BYTES = BQ * D * 4;       // fp32 dQ tile: D/32 blocks of [64 rows][32 floats], swizzled
  static constexpr int L_BYTES = (DOC ? 3 : 2) * BQ * 4;  // LSE*log2e, delta (and DOC: document starts) of one item
  static constexpr int OFF_K = 0;
  static constexpr int OFF_V = OFF_K + KV_BYTES;
  static constexpr int OFF_Q = OFF_V + KV_BYTES;
  static constexpr int OFF_DO = OFF_Q + STAGES * QS_BYTES;
  static constexpr int OFF_DS = OFF_DO + STAGES * QS_BYTES;  // 2 buffers
  static constexpr int OFF_DQ = OFF_DS + 2 * DS_BYTES;        // 2 buffers
  static constexpr int OFF_L = OFF_DQ + 2 * DQ_BYTES;         // STAGES x L_BYTES
  static constexpr int OFF_BAR = OFF_L + STAGES * L_BYTES;
  static constexpr int SMEM_BYTES = OFF_BAR + 128 + 1024;
  static_assert(SMEM_BYTES <= 232448, "attn_bwd shared memory");
};

struct BwdArgs {
  const float* lse2;   // [B,H,S_pad] LSE * log2e
  const float* delta;  // [B,H,S_pad]
  __nv_bfloat16* dk;   // [B,S,dkv_rh,D]-strided rows
  __nv_bfloat16* dv;
  int B, S, H, Hk;
  int S_pad;           // S rounded up to BQ
  int dkv_rh;          // heads per dk/dv token row (>= Hk)
  float scale;
  int causal;
  int paired;          // CTA x runs key tiles x and n_kt-1-x
  const int* dstart;   // DOC: [B,S_pad] document start of every query
  const int* qt_end;   // DOC: [B,n_kt] end of each key tile's query-tile range
  const float* slopes; // ALIBI: [H] fp32 per-query-head slopes
  const int* prefix;   // PREFIX: [B] int32 prefix lengths (clamped to [0, S])
  uint32_t drop_t;     // DROP: keep threshold t = round(p 65536) on the 16-bit Philox values
  float drop_inv;      // DROP: 1 / (1 - t / 65536)
  unsigned long long drop_seed;  // DROP: Philox key
};

// PREFIX: batch row b's prefix length
__device__ __forceinline__ int prefix_len(const BwdArgs& p, int b) { return min(max(__ldg(p.prefix + b), 0), p.S); }

// The work of one key tile: `group * per_head` items, item j = (query head h0 + j / per_head, query tile
// qt0 + j % per_head).
struct Tile {
  int kt, k0, qt0, per_head, n_items;
};
template <bool DOC, bool PREFIX = false>
__device__ __forceinline__ Tile tile_of(const BwdArgs& p, int pass) {
  Tile t;
  t.kt = pass == 0 ? (int)blockIdx.x : (p.S + BKV - 1) / BKV - 1 - (int)blockIdx.x;
  t.k0 = t.kt * BKV;
  int n_qt = (p.S + BQ - 1) / BQ;
  if constexpr (DOC) n_qt = __ldg(p.qt_end + (long long)blockIdx.z * gridDim.x + t.kt);  // unpaired: x = kt
  t.qt0 = p.causal ? t.k0 / BQ : 0;
  if constexpr (PREFIX) {
    if (t.k0 < prefix_len(p, blockIdx.z)) t.qt0 = 0;  // every query sees the tile's prefix keys
  }
  t.per_head = n_qt - t.qt0;
  t.n_items = (p.H / p.Hk) * t.per_head;
  return t;
}

__device__ __forceinline__ int lds32i(uint32_t addr) {
  int v;
  asm volatile("ld.shared.b32 %0, [%1];" : "=r"(v) : "r"(addr) : "memory");
  return v;
}

template <int D>
__device__ __forceinline__ void rs_mma(float* acc, const uint32_t* a, uint64_t db) {
  if constexpr (D == 128) wgmma_m64n128k16_rs<1>(acc, a, db);
  else wgmma_m64n64k16_rs<1>(acc, a, db);
}

// DROP: keep bits of a consumer thread's 32 elements of the item (query head h, queries from q0, keys from kbase =
// the warp's first key): bit 4 nc + e for query q0 + 8 nc + cq + (e & 1) and key kbase + g + 8 (e >> 1)
__device__ __forceinline__ uint32_t drop_keep_bits(const BwdArgs& p, int kbase, int q0, int h, int b, int lane) {
  const int g = lane >> 2, cq = (lane & 3) * 2;
  const uint32_t sk0 = (uint32_t)p.drop_seed, sk1 = (uint32_t)(p.drop_seed >> 32);
  uint32_t own = 0u;  // byte j: the call of element (nc = g, e = j), bit i for key 8 (kbase / 8 + (j >> 1)) + i
#pragma unroll 1
  for (int j = 0; j < 4; ++j)
    own |= philox_keep8((uint32_t)(kbase >> 3) + (j >> 1), q0 + 8 * g + cq + (j & 1), h, b, sk0, sk1, p.drop_t)
           << (8 * j);
  uint32_t zk = 0u;
#pragma unroll
  for (int m = 0; m < 8; ++m) {  // from lane g ^ m of the group (xor shuffles need no lane-index registers)
    const uint32_t x = (__shfl_xor_sync(0xffffffffu, own, 4 * m) >> g) & 0x01010101u;
    zk |= ((x | (x >> 7) | (x >> 14) | (x >> 21)) & 0xfu) << (4 * (g ^ m));
  }
  return zk;
}

template <int D, bool DOC, bool ALIBI = false, bool PREFIX = false, bool DROP = false>
__global__ void __launch_bounds__(BWD_THREADS, 1)
attn_bwd_kernel(const __grid_constant__ CUtensorMap tmQ, const __grid_constant__ CUtensorMap tmK,
                const __grid_constant__ CUtensorMap tmV, const __grid_constant__ CUtensorMap tmDO,
                const __grid_constant__ CUtensorMap tmDQ, const BwdArgs p) {
  static_assert(!PREFIX || (!DOC && !ALIBI), "the prefix mask is built on the causal kernel");
  static_assert(!PREFIX || !DROP, "dropout is not built on the prefix kernels");
  using Cfg = BwdCfg<D, DOC>;
  constexpr int ST = Cfg::STAGES;
  extern __shared__ uint8_t smem_raw[];
  const uint32_t s0 = (smem_u32(smem_raw) + 1023) & ~1023u;
  const uint32_t sK = s0 + Cfg::OFF_K, sV = s0 + Cfg::OFF_V, sQ = s0 + Cfg::OFF_Q, sDO = s0 + Cfg::OFF_DO;
  const uint32_t sDS = s0 + Cfg::OFF_DS, sDQ = s0 + Cfg::OFF_DQ, sL = s0 + Cfg::OFF_L;
  const uint32_t kv_full = s0 + Cfg::OFF_BAR, kv_empty = kv_full + 8;
  const uint32_t q_full0 = kv_full + 16, q_empty0 = q_full0 + 8 * ST;
  const uint32_t dq_full0 = q_empty0 + 8 * ST, dq_empty0 = dq_full0 + 16;
  const int hk = blockIdx.y, b = blockIdx.z;
  const int group = p.H / p.Hk;
  const int n_pass = p.paired ? 2 : 1;
  const int wg = threadIdx.x >> 7, warp = threadIdx.x >> 5, lane = threadIdx.x & 31;

  if (threadIdx.x == 0) {
    mbar_init(kv_full, 1);
    mbar_init(kv_empty, 2);  // one arrival per consumer warpgroup
    for (int s = 0; s < ST; ++s) {
      mbar_init(q_full0 + 8 * s, 1);
      mbar_init(q_empty0 + 8 * s, 2);
    }
    for (int s = 0; s < 2; ++s) {
      mbar_init(dq_full0 + 8 * s, 8);  // one arrival per consumer warp
      mbar_init(dq_empty0 + 8 * s, 1);
    }
    fence_mbar_init();
  }
  __syncthreads();

  if (wg == 0) {
    setmaxnreg_dec<24>();
    if (warp == 0 && lane == 0) {  // producer
      tma_prefetch_desc(&tmQ);
      tma_prefetch_desc(&tmDO);
      int slot = 0;
      uint32_t phase = 0;
      for (int pass = 0; pass < n_pass; ++pass) {
        const Tile t = tile_of<DOC, PREFIX>(p, pass);
        if (pass > 0) mbar_wait(kv_empty, 0);
        mbar_arrive_expect_tx(kv_full, 2 * Cfg::KV_BYTES);
        for (int nb = 0; nb < Cfg::NB; ++nb) {
          tma_load_4d(sK + nb * BKV * 128, &tmK, kv_full, nb * 64, hk, t.k0, b);
          tma_load_4d(sV + nb * BKV * 128, &tmV, kv_full, nb * 64, hk, t.k0, b);
        }
        for (int j = 0; j < t.n_items; ++j) {
          const int h = hk * group + j / t.per_head;
          const int q0 = (t.qt0 + j % t.per_head) * BQ;
          mbar_wait(q_empty0 + 8 * slot, phase ^ 1u);
          const uint32_t full = q_full0 + 8 * slot;
          mbar_arrive_expect_tx(full, 2 * Cfg::QS_BYTES + Cfg::L_BYTES);
          for (int nb = 0; nb < Cfg::NB; ++nb) {
            tma_load_4d(sQ + slot * Cfg::QS_BYTES + nb * BQ * 128, &tmQ, full, nb * 64, h, q0, b);
            tma_load_4d(sDO + slot * Cfg::QS_BYTES + nb * BQ * 128, &tmDO, full, nb * 64, h, q0, b);
          }
          const long long lrow = ((long long)b * p.H + h) * p.S_pad + q0;
          bulk_load(sL + slot * Cfg::L_BYTES, p.lse2 + lrow, BQ * 4, full);
          bulk_load(sL + slot * Cfg::L_BYTES + BQ * 4, p.delta + lrow, BQ * 4, full);
          if constexpr (DOC) bulk_load(sL + slot * Cfg::L_BYTES + 2 * BQ * 4, p.dstart + (long long)b * p.S_pad + q0,
                                       BQ * 4, full);
          if (++slot == ST) {
            slot = 0;
            phase ^= 1u;
          }
        }
      }
    } else if (warp == 1 && lane == 0) {  // dQ writer
      tma_prefetch_desc(&tmDQ);
      int it = 0;
      for (int pass = 0; pass < n_pass; ++pass) {
        const Tile t = tile_of<DOC, PREFIX>(p, pass);
        for (int j = 0; j < t.n_items; ++j, ++it) {
          const int h = hk * group + j / t.per_head;
          const int q0 = (t.qt0 + j % t.per_head) * BQ;
          const int buf = it & 1;
          mbar_wait(dq_full0 + 8 * buf, (it >> 1) & 1);
#pragma unroll
          for (int blk = 0; blk < D / 32; ++blk)
            tma_reduce_add_4d(sDQ + buf * Cfg::DQ_BYTES + blk * 8192, &tmDQ, blk * 32, h, q0, b);
          bulk_commit();
          bulk_wait_read<0>();
          mbar_arrive(dq_empty0 + 8 * buf);
        }
      }
      bulk_wait<0>();
    }
    return;
  }

  setmaxnreg_inc<240>();
  const int c = wg - 1;  // consumer warpgroup: keys 64c .. 64c+63 of the tile
  const int wq = warp & 3;
  const int g = lane >> 2, cq = (lane & 3) * 2;
  const float sl2 = p.scale * kLog2e;
  int slot = 0;
  uint32_t phase = 0;
  int it = 0;

  for (int pass = 0; pass < n_pass; ++pass) {
    const Tile t = tile_of<DOC, PREFIX>(p, pass);
    const int key_a = t.k0 + c * 64 + wq * 16 + g;  // this thread's keys: key_a, key_a + 8
    const int wkey_hi = t.k0 + c * 64 + 63;          // last key of this warpgroup
    float dk[D / 2], dv[D / 2];
#pragma unroll
    for (int i = 0; i < D / 2; ++i) dk[i] = dv[i] = 0.f;
    mbar_wait_outlined(kv_full, pass & 1);

    for (int j = 0; j < t.n_items; ++j, ++it) {
      const int q0 = (t.qt0 + j % t.per_head) * BQ;
      // DROP: the item's keep bits, made before the wait for its Q / dO, where only dK and dV are live (with the S^T
      // and dP^T fragments live D = 128 spills, and between the MMAs' commit and wait ptxas injects a
      // warpgroup.arrive)
      uint32_t zk = 0u;
      if constexpr (DROP) zk = drop_keep_bits(p, t.k0 + c * 64 + wq * 16, q0, hk * group + j / t.per_head, b, lane);
      mbar_wait_outlined(q_full0 + 8 * slot, phase);
      const uint32_t tQ = sQ + slot * Cfg::QS_BYTES, tDO = sDO + slot * Cfg::QS_BYTES;
      const uint32_t tL = sL + slot * Cfg::L_BYTES, tDlt = tL + BQ * 4;  // LSE*log2e, delta of the 64 queries

      // S^T = K Q^T and dP^T = V dO^T: 64 keys x 64 queries per warpgroup
      float st[32], dpt[32];
#pragma unroll
      for (int i = 0; i < 32; ++i) st[i] = dpt[i] = 0.f;
      wgmma_fence();
#pragma unroll
      for (int kk = 0; kk < D / 16; ++kk) {
        const uint32_t ka = (kk >> 2) * BKV * 128 + c * 64 * 128 + (kk & 3) * 32;
        const uint32_t qb = (kk >> 2) * BQ * 128 + (kk & 3) * 32;
        wgmma_m64n64k16_ss<0, 0>(st, make_wgmma_desc_sw128(sK + ka, 16, 1024), make_wgmma_desc_sw128(tQ + qb, 16, 1024));
        wgmma_m64n64k16_ss<0, 0>(dpt, make_wgmma_desc_sw128(sV + ka, 16, 1024), make_wgmma_desc_sw128(tDO + qb, 16, 1024));
      }
      wgmma_commit();
      wgmma_wait<0>();

      // ALIBI: the item's head slope in log2 units, and the bias of each of this thread's keys against query
      // q0 + cq
      float ml2 = 0.f, abase[2] = {0.f, 0.f};
      if constexpr (ALIBI) {
        ml2 = __ldg(p.slopes + hk * group + j / t.per_head) * kLog2e;
#pragma unroll
        for (int r = 0; r < 2; ++r) abase[r] = ml2 * (float)(key_a + 8 * r - q0 - cq);
      }

      // P^T and dS^T (unscaled).  Chunk nc holds queries 8 nc + cq + {0, 1}.  Only tiles that cross the causal
      // diagonal or the end of the sequence are masked; masked entries are exactly 0.
      const int pfx = PREFIX ? prefix_len(p, b) : 0;  // PREFIX: this row's prefix length
      bool masked;
      // PREFIX: keys below the prefix are visible to every query, so only keys past max(q0, P_b - 1) need the mask
      if constexpr (PREFIX) masked = wkey_hi > max(q0, pfx - 1) || q0 + BQ > p.S || wkey_hi >= p.S;
      else masked = (p.causal && wkey_hi > q0) || q0 + BQ > p.S || wkey_hi >= p.S;
      // DOC: also where the item's highest document start (its last query's; padded rows repeat the last real one)
      // lies above the warpgroup's first key
      if constexpr (DOC) masked = masked || lds32i(tL + 2 * BQ * 4 + (BQ - 1) * 4) > wkey_hi - 63;
      if (masked) {
        // DOC: document starts are monotone over the item's queries, so the queries that may see key k are a prefix
        // of the item; n_vis[r] = its length for this thread's key key_a + 8 r (binary search over the 64 starts)
        int n_vis[2] = {BQ, BQ};
        if constexpr (DOC) {
          const uint32_t tDs = tL + 2 * BQ * 4;
#pragma unroll
          for (int r = 0; r < 2; ++r) {
            const int key = key_a + 8 * r;
            int n = 0;
#pragma unroll
            for (int step = BQ / 2; step > 0; step >>= 1)
              if (lds32i(tDs + (n + step - 1) * 4) <= key) n += step;
            if (lds32i(tDs + n * 4) <= key) ++n;
            n_vis[r] = n;
          }
        }
#pragma unroll
        for (int nc = 0; nc < 8; ++nc) {
#pragma unroll
          for (int e = 0; e < 4; ++e) {
            const int qc = nc * 8 + cq + (e & 1);
            const int qi = q0 + qc;
            const int key = key_a + ((e >> 1) << 3);
            bool ok;
            if constexpr (PREFIX) ok = qi < p.S && key < p.S && (key <= qi || key < pfx);
            else ok = qi < p.S && key < p.S && !(p.causal && key > qi);
            if constexpr (DOC) ok = ok && qc < n_vis[e >> 1];
            float pv;
            if constexpr (ALIBI)
              pv = ok ? exp2f(st[4 * nc + e] * sl2 +
                              (fmaf(ml2, -(float)(nc * 8 + (e & 1)), abase[e >> 1]) - lds32f(tL + qc * 4)))
                      : 0.f;
            else
              pv = ok ? exp2f(st[4 * nc + e] * sl2 - lds32f(tL + qc * 4)) : 0.f;
            st[4 * nc + e] = pv;
            if constexpr (DROP) {
              const float zs = (zk >> (4 * nc + e)) & 1u ? p.drop_inv : 0.f;
              dpt[4 * nc + e] = ok ? pv * (dpt[4 * nc + e] * zs - lds32f(tDlt + qc * 4)) : 0.f;
            } else {
              dpt[4 * nc + e] = ok ? pv * (dpt[4 * nc + e] - lds32f(tDlt + qc * 4)) : 0.f;
            }
          }
        }
      } else {
#pragma unroll
        for (int nc = 0; nc < 8; ++nc) {
          const float2 l = lds64f(tL + (nc * 8 + cq) * 4);
          const float2 d = lds64f(tDlt + (nc * 8 + cq) * 4);
#pragma unroll
          for (int e = 0; e < 4; ++e) {
            float pv;
            if constexpr (ALIBI)
              pv = exp2f(st[4 * nc + e] * sl2 +
                         (fmaf(ml2, -(float)(nc * 8 + (e & 1)), abase[e >> 1]) - ((e & 1) ? l.y : l.x)));
            else
              pv = exp2f(st[4 * nc + e] * sl2 - ((e & 1) ? l.y : l.x));
            st[4 * nc + e] = pv;
            if constexpr (DROP) {
              const float zs = (zk >> (4 * nc + e)) & 1u ? p.drop_inv : 0.f;
              dpt[4 * nc + e] = pv * (dpt[4 * nc + e] * zs - ((e & 1) ? d.y : d.x));
            } else {
              dpt[4 * nc + e] = pv * (dpt[4 * nc + e] - ((e & 1) ? d.y : d.x));
            }
          }
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
      // DROP: P^T for dV with the dropped bf16 halves zeroed (elements 8 kk + 2 i + {0, 1} of pa[kk][i])
      if constexpr (DROP) {
#pragma unroll
        for (int kk = 0; kk < 4; ++kk) {
#pragma unroll
          for (int i = 0; i < 4; ++i) {
            const uint32_t x = zk >> (8 * kk + 2 * i);
            pa[kk][i] &= (x & 1u) * 0xffffu | ((x >> 1) & 1u) * 0xffff0000u;
          }
        }
      }
      // dS^T rows of this thread -> [key][64 queries] tile, 128 B per row, 16-byte chunks XOR (row % 8)
      const uint32_t tDS = sDS + (it & 1) * Cfg::DS_BYTES;
      {
        const int r = c * 64 + wq * 16 + g;
#pragma unroll
        for (int kk = 0; kk < 4; ++kk) {
#pragma unroll
          for (int i = 0; i < 4; ++i) {
            const int row = r + ((i & 1) << 3), chunk = 2 * kk + (i >> 1);
            sts32(tDS + row * 128 + ((chunk ^ (row & 7)) << 4) + cq * 2, da[kk][i]);
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
      // both warpgroups' dS^T rows are in shared memory.  dS^T is double-buffered: this barrier of item it+1 also
      // orders the dQ reads of item it before the rewrite of its buffer by item it+2.
      named_bar_sync(1, 256);
      wgmma_wait<0>();  // P^T / dS^T registers are free before the dQ accumulators are live

      // dQ[64 queries, D/2 head-dim columns of this warpgroup] = dS K over all 128 keys
      constexpr int NQ = D / 4;  // accumulators per thread
      float dq[NQ];
#pragma unroll
      for (int i = 0; i < NQ; ++i) dq[i] = 0.f;
      wgmma_fence();
#pragma unroll
      for (int kk = 0; kk < BKV / 16; ++kk) {
        const uint64_t da_ = make_wgmma_desc_sw128(tDS + kk * 2048, 8192, 1024);
        if constexpr (D == 128)
          wgmma_m64n64k16_ss<1, 1>(dq, da_, make_wgmma_desc_sw128(sK + c * BKV * 128 + kk * 2048, BKV * 128, 1024));
        else  // columns 32c .. 32c+31: half c of each 128-byte K row
          wgmma_m64n32k16_ss<1, 1>(dq, da_, make_wgmma_desc_sw128(sK + kk * 2048 + c * 64, BKV * 128, 1024));
      }
      wgmma_commit();
      wgmma_wait<0>();
      if ((threadIdx.x & 127) == 0) mbar_arrive(q_empty0 + 8 * slot);
      if (++slot == ST) {
        slot = 0;
        phase ^= 1u;
      }

      // dQ fragment -> fp32 tile in the dq_acc map's layout: block of 32 columns = [64 rows][128 B], 16-byte chunk
      // index XOR (row % 8).  Row g / g+8 of a warp hit 8 distinct chunk pairs: conflict-free 8-byte stores.
      const int buf = it & 1;
      mbar_wait_outlined(dq_empty0 + 8 * buf, ((it >> 1) & 1) ^ 1u);
      {
        const uint32_t tDQ = sDQ + buf * Cfg::DQ_BYTES;
#pragma unroll
        for (int nc = 0; nc < NQ / 4; ++nc) {
          // columns c*D/2 + 8 nc + cq + {0, 1}: 32-column block, 16-byte chunk and 8-byte half within it
          const int blk = c * (D / 64) + (nc >> 2);
          const int chunk = 2 * (nc & 3) + (cq >> 2);
#pragma unroll
          for (int r = 0; r < 2; ++r) {
            const int row = wq * 16 + g + 8 * r;  // row % 8 == g
            sts64f(tDQ + blk * 8192 + row * 128 + ((chunk ^ g) << 4) + (cq & 2) * 4, dq[4 * nc + 2 * r],
                   dq[4 * nc + 2 * r + 1]);
          }
        }
      }
      fence_proxy_async_smem();
      __syncwarp();
      if (lane == 0) mbar_arrive(dq_full0 + 8 * buf);
    }
    // every read of this tile's K / V has completed (the last dQ wgmma was waited for)
    if ((threadIdx.x & 127) == 0) mbar_arrive(kv_empty);

    // dK (scale applied here), dV (DROP: with the dropout scale) -> bf16 rows of dkv_rh heads
    const float dv_mul = DROP ? p.drop_inv : 1.f;
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      const int key = key_a + 8 * r;
      if (key >= p.S) continue;
      const long long off = ((long long)b * p.S + key) * p.dkv_rh * D + (long long)hk * D + cq;
#pragma unroll
      for (int dc = 0; dc < D / 8; ++dc) {
        *reinterpret_cast<uint32_t*>(p.dk + off + dc * 8) =
            pack_bf16x2(dk[4 * dc + 2 * r] * p.scale, dk[4 * dc + 2 * r + 1] * p.scale);
        if constexpr (DROP)
          *reinterpret_cast<uint32_t*>(p.dv + off + dc * 8) =
              pack_bf16x2(dv[4 * dc + 2 * r] * dv_mul, dv[4 * dc + 2 * r + 1] * dv_mul);
        else
          *reinterpret_cast<uint32_t*>(p.dv + off + dc * 8) = pack_bf16x2(dv[4 * dc + 2 * r], dv[4 * dc + 2 * r + 1]);
      }
    }
  }
}

// delta[b,h,s] = sum_d o[b,s,h,d] * do[b,s,h,d] and lse2[b,h,s] = lse[b,h,s] * log2e, both in rows of S_pad floats
// (whole 64-query tiles, 16-byte aligned, for the backward's bulk copies); LPR = D/8 lanes cooperate on one row.  The
// same pass zeroes the fp32 dQ accumulator (same [B,S,H,D] index space: each thread clears the 8 floats under the 8
// bf16 it reads), so the backward needs no separate memset launch over 4*B*S*H*D bytes.
//
// DOC: the threads of head 0 also write dstart[b, s] = s - min(pos[b, s], window) (rows of S_pad, the tail repeating
// the last token's start) and, at each document's last token s, the query-tile end min(s, k0 + BKV - 1 + window) / BQ
// + 1 of every key tile (first key k0) whose last key lies in that document: exactly one document holds each key
// tile's last key, so each entry has one writer.  pos == nullptr reads as pos[b, s] = s: one document per row.
template <int D, bool DOC>
__global__ void __launch_bounds__(256)
attn_delta_kernel(const __nv_bfloat16* __restrict__ o, const __nv_bfloat16* __restrict__ d_o,
                  const float* __restrict__ lse, float* __restrict__ delta, float* __restrict__ lse2,
                  float* __restrict__ dq_acc, int B, int S, int H, int S_pad, const int* __restrict__ pos,
                  int* __restrict__ dstart, int* __restrict__ qt_end, int window) {
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
    delta[(bb * H + hh) * S_pad + s] = acc;
    lse2[(bb * H + hh) * S_pad + s] = lse[(bb * H + hh) * S + s] * kLog2e;
    if constexpr (DOC) {
      if (hh == 0) {
        const int* prow = pos ? pos + bb * S : nullptr;
        const int ps = prow ? prow[s] : s;
        const int doc0 = max(0, s - ps);               // document start
        const int start = max(0, s - min(ps, window));  // first visible key
        int* drow = dstart + bb * S_pad;
        drow[s] = start;
        if (s == S - 1)
          for (int x = S; x < S_pad; ++x) drow[x] = start;
        if (s == S - 1 || (prow && prow[s + 1] == 0)) {  // s ends its document
          const int n_kt = (S + BKV - 1) / BKV;
          const int kt_hi = s == S - 1 ? n_kt - 1 : (s + 1) / BKV - 1;  // last key tile whose last key is <= s
          for (int kt = doc0 / BKV; kt <= kt_hi; ++kt)
            qt_end[bb * n_kt + kt] = min(s, kt * BKV + BKV - 1 + window) / BQ + 1;
        }
      }
    }
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

template <int D, bool DOC, bool ALIBI = false, bool PREFIX = false, bool DROP = false>
int launch_bwd(const CUtensorMap& tmQ, const CUtensorMap& tmK, const CUtensorMap& tmV, const CUtensorMap& tmDO,
               const CUtensorMap& tmDQ, const BwdArgs& a, cudaStream_t stream) {
  using Cfg = BwdCfg<D, DOC>;
  auto kern = attn_bwd_kernel<D, DOC, ALIBI, PREFIX, DROP>;
  static bool attr_set = false;
  if (!attr_set) {
    B200_CHECK_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg::SMEM_BYTES));
    attr_set = true;
  }
  const int n_kt = (a.S + BKV - 1) / BKV;
  dim3 grid(a.paired ? n_kt / 2 : n_kt, a.Hk, a.B);
  kern<<<grid, BWD_THREADS, Cfg::SMEM_BYTES, stream>>>(tmQ, tmK, tmV, tmDO, tmDQ, a);
  B200_CHECK_LAUNCH();
  return B200_OK;
}

inline int pad_q(int S) { return (S + BQ - 1) / BQ * BQ; }

// fp32 [B, S, H, D] dQ accumulator -> 4-D tensor map {D, H, S, B}, box {32, 1, 64, 1} (one 128-byte swizzle span)
int make_dq_acc_map(CUtensorMap* tm, const float* base, int B, int S, int H, int D) {
  const uint64_t dims[4] = {(uint64_t)D, (uint64_t)H, (uint64_t)S, (uint64_t)B};
  const uint64_t strides[3] = {(uint64_t)D * 4, (uint64_t)H * D * 4, (uint64_t)S * H * D * 4};
  const uint32_t box[4] = {32, 1, (uint32_t)BQ, 1};
  return make_tensor_map(tm, base, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 4, 4, dims, strides, box, true);
}

// doc selects the document / window kernels; window < 0 means none; slopes (doc only) selects ALiBi; prefix (causal,
// not doc) selects the prefix-LM kernels; drop selects the dropout kernels (not with prefix)
int attn_bwd_impl(const void* q, const void* k, const void* v, const void* o, const void* d_o, const float* lse,
                  bool doc, const int* pos, int window, void* dq, void* dk, void* dv, int B, int S, int H, int Hk,
                  int D, float scale, int causal, int dkv_row_heads, void* ws, size_t ws_bytes, cudaStream_t stream,
                  const float* slopes = nullptr, const int* prefix = nullptr, bool drop = false,
                  uint32_t drop_t = 0, float drop_inv = 1.f, unsigned long long drop_seed = 0) {
  // dk / dv rows may be strided: dkv_row_heads heads per token row (0 = Hk, i.e. contiguous [B,S,Hk,D]).
  // With dk = base, dv = base + Hk*D and dkv_row_heads = 2*Hk both land in ONE [B,S,2*Hk*D] buffer, which lets
  // the k/v projections' dgrad and wgrad run as single GEMMs over the concatenated weight.
  if (dkv_row_heads <= 0) dkv_row_heads = Hk;
  B200_CHECK_ARG(dkv_row_heads >= Hk, "attn_bwd: dkv_row_heads=%d < Hk=%d", dkv_row_heads, Hk);
  B200_CHECK_ARG(B > 0 && S > 0 && H > 0 && Hk > 0 && H % Hk == 0,
                 "attn_bwd: bad shape B=%d S=%d H=%d Hk=%d", B, S, H, Hk);
  B200_CHECK_ARG(D == 64 || D == 128, "attn_bwd: head_dim %d unsupported (64 or 128)", D);
  const size_t need =
      doc ? b200_attn_bwd_doc_workspace_bytes(B, S, H, Hk, D) : b200_attn_bwd_workspace_bytes(B, S, H, Hk, D);
  if (ws_bytes < need) {
    set_error("attn_bwd: workspace too small (%zu < %zu)", ws_bytes, need);
    return B200_ERR_WORKSPACE;
  }
  B200_CHECK_ARG((reinterpret_cast<uintptr_t>(ws) & 255u) == 0, "attn_bwd: workspace must be 256-byte aligned");
  B200_CHECK_ARG(((reinterpret_cast<uintptr_t>(q) | reinterpret_cast<uintptr_t>(k) | reinterpret_cast<uintptr_t>(v) |
                   reinterpret_cast<uintptr_t>(o) | reinterpret_cast<uintptr_t>(d_o)) & 15u) == 0,
                 "attn_bwd: q/k/v/o/do must be 16-byte aligned");
  float* dq_acc = reinterpret_cast<float*>(ws);
  const int S_pad = pad_q(S);
  const int n_kt = (S + BKV - 1) / BKV;
  float* delta = reinterpret_cast<float*>(reinterpret_cast<char*>(ws) + al256((size_t)B * S * H * D * 4));
  float* lse2 = reinterpret_cast<float*>(reinterpret_cast<char*>(delta) + al256((size_t)B * H * S_pad * 4));
  int* dstart = reinterpret_cast<int*>(reinterpret_cast<char*>(lse2) + al256((size_t)B * H * S_pad * 4));
  int* qt_end = reinterpret_cast<int*>(reinterpret_cast<char*>(dstart) + al256((size_t)B * S_pad * 4));
  const long long n = (long long)B * S * H * D;
  {
    const long long threads = (long long)B * S * H * (D / 8);
    const int blocks = (int)((threads + 255) / 256);
    auto delta_kern = D == 64 ? (doc ? attn_delta_kernel<64, true> : attn_delta_kernel<64, false>)
                              : (doc ? attn_delta_kernel<128, true> : attn_delta_kernel<128, false>);
    delta_kern<<<blocks, 256, 0, stream>>>((const __nv_bfloat16*)o, (const __nv_bfloat16*)d_o, lse, delta, lse2,
                                           dq_acc, B, S, H, S_pad, pos, dstart, qt_end,
                                           window < 0 || window > S ? S : window);
    B200_CHECK_LAUNCH();
  }
  CUtensorMap tmQ, tmK, tmV, tmDO, tmDQ;
  int rc;
  if ((rc = make_bshd_map(&tmQ, q, B, S, H, D, BQ))) return rc;
  if ((rc = make_bshd_map(&tmK, k, B, S, Hk, D, BKV))) return rc;
  if ((rc = make_bshd_map(&tmV, v, B, S, Hk, D, BKV))) return rc;
  if ((rc = make_bshd_map(&tmDO, d_o, B, S, H, D, BQ))) return rc;
  if ((rc = make_dq_acc_map(&tmDQ, dq_acc, B, S, H, D))) return rc;
  BwdArgs a;
  a.lse2 = lse2;
  a.delta = delta;
  a.dk = reinterpret_cast<__nv_bfloat16*>(dk);
  a.dv = reinterpret_cast<__nv_bfloat16*>(dv);
  a.B = B;
  a.S = S;
  a.H = H;
  a.Hk = Hk;
  a.S_pad = S_pad;
  a.dkv_rh = dkv_row_heads;
  a.scale = scale;
  a.causal = causal;
  a.paired = causal && !doc && !prefix && n_kt % 2 == 0;
  a.dstart = doc ? dstart : nullptr;
  a.qt_end = doc ? qt_end : nullptr;
  a.slopes = slopes;
  a.prefix = prefix;
  a.drop_t = drop_t;
  a.drop_inv = drop_inv;
  a.drop_seed = drop_seed;
  if (drop && slopes)
    rc = D == 64 ? launch_bwd<64, true, true, false, true>(tmQ, tmK, tmV, tmDO, tmDQ, a, stream)
                 : launch_bwd<128, true, true, false, true>(tmQ, tmK, tmV, tmDO, tmDQ, a, stream);
  else if (drop && doc)
    rc = D == 64 ? launch_bwd<64, true, false, false, true>(tmQ, tmK, tmV, tmDO, tmDQ, a, stream)
                 : launch_bwd<128, true, false, false, true>(tmQ, tmK, tmV, tmDO, tmDQ, a, stream);
  else if (drop)
    rc = D == 64 ? launch_bwd<64, false, false, false, true>(tmQ, tmK, tmV, tmDO, tmDQ, a, stream)
                 : launch_bwd<128, false, false, false, true>(tmQ, tmK, tmV, tmDO, tmDQ, a, stream);
  else if (prefix)
    rc = D == 64 ? launch_bwd<64, false, false, true>(tmQ, tmK, tmV, tmDO, tmDQ, a, stream)
                 : launch_bwd<128, false, false, true>(tmQ, tmK, tmV, tmDO, tmDQ, a, stream);
  else if (slopes)
    rc = D == 64 ? launch_bwd<64, true, true>(tmQ, tmK, tmV, tmDO, tmDQ, a, stream)
                 : launch_bwd<128, true, true>(tmQ, tmK, tmV, tmDO, tmDQ, a, stream);
  else if (doc)
    rc = D == 64 ? launch_bwd<64, true>(tmQ, tmK, tmV, tmDO, tmDQ, a, stream)
                 : launch_bwd<128, true>(tmQ, tmK, tmV, tmDO, tmDQ, a, stream);
  else
    rc = D == 64 ? launch_bwd<64, false>(tmQ, tmK, tmV, tmDO, tmDQ, a, stream)
                 : launch_bwd<128, false>(tmQ, tmK, tmV, tmDO, tmDQ, a, stream);
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

}  // namespace
}  // namespace b200

using namespace b200;

extern "C" {

size_t b200_attn_bwd_workspace_bytes(int B, int S, int H, int Hk, int D) {
  (void)Hk;
  return al256((size_t)B * S * H * D * 4) + 2 * al256((size_t)B * H * pad_q(S) * 4);
}

// the document variant adds the [B, S_pad] document starts and the [B, n_kt] query-tile ends
size_t b200_attn_bwd_doc_workspace_bytes(int B, int S, int H, int Hk, int D) {
  return b200_attn_bwd_workspace_bytes(B, S, H, Hk, D) + al256((size_t)B * pad_q(S) * 4) +
         al256((size_t)B * ((S + BKV - 1) / BKV) * 4);
}

int b200_attn_bwd(const void* q, const void* k, const void* v, const void* o, const void* d_o,
                  const float* lse, void* dq, void* dk, void* dv, int B, int S, int H, int Hk,
                  int D, float scale, int causal, void* ws, size_t ws_bytes, void* stream) {
  return attn_bwd_impl(q, k, v, o, d_o, lse, false, nullptr, -1, dq, dk, dv, B, S, H, Hk, D, scale, causal, 0, ws,
                       ws_bytes, static_cast<cudaStream_t>(stream));
}

int b200_attn_bwd_strided(const void* q, const void* k, const void* v, const void* o, const void* d_o,
                          const float* lse, void* dq, void* dk, void* dv, int B, int S, int H, int Hk,
                          int D, float scale, int causal, int dkv_row_heads, void* ws, size_t ws_bytes, void* stream) {
  return attn_bwd_impl(q, k, v, o, d_o, lse, false, nullptr, -1, dq, dk, dv, B, S, H, Hk, D, scale, causal,
                       dkv_row_heads, ws, ws_bytes, static_cast<cudaStream_t>(stream));
}

// document-causal backward: query s of row b sees keys s - pos[b, s] .. s
int b200_attn_bwd_doc(const void* q, const void* k, const void* v, const void* o, const void* d_o, const float* lse,
                      const int* pos, void* dq, void* dk, void* dv, int B, int S, int H, int Hk, int D, float scale,
                      int dkv_row_heads, void* ws, size_t ws_bytes, void* stream) {
  B200_CHECK_ARG(pos != nullptr && (reinterpret_cast<uintptr_t>(pos) & 3u) == 0,
                 "attn_bwd_doc: pos must be a non-null, 4-byte aligned int32 [B, S] array");
  return attn_bwd_impl(q, k, v, o, d_o, lse, true, pos, -1, dq, dk, dv, B, S, H, Hk, D, scale, 1, dkv_row_heads, ws,
                       ws_bytes, static_cast<cudaStream_t>(stream));
}

// sliding-window backward: query s sees keys s - min(pos[b, s], window) .. s; pos == nullptr means pos[b, s] = s.
// Same workspace as the document variant.
size_t b200_attn_bwd_window_workspace_bytes(int B, int S, int H, int Hk, int D) {
  return b200_attn_bwd_doc_workspace_bytes(B, S, H, Hk, D);
}

int b200_attn_bwd_window(const void* q, const void* k, const void* v, const void* o, const void* d_o, const float* lse,
                         const int* pos, int window, void* dq, void* dk, void* dv, int B, int S, int H, int Hk, int D,
                         float scale, int dkv_row_heads, void* ws, size_t ws_bytes, void* stream) {
  B200_CHECK_ARG((reinterpret_cast<uintptr_t>(pos) & 3u) == 0, "attn_bwd_window: pos must be 4-byte aligned int32");
  B200_CHECK_ARG(window >= 0, "attn_bwd_window: window=%d must be >= 0", window);
  return attn_bwd_impl(q, k, v, o, d_o, lse, true, pos, window, dq, dk, dv, B, S, H, Hk, D, scale, 1, dkv_row_heads,
                       ws, ws_bytes, static_cast<cudaStream_t>(stream));
}

// ALiBi backward: attn_bwd_window (window < 0: none) with the forward's bias slopes[h] * (k - s).  Same workspace.
int b200_attn_bwd_alibi(const void* q, const void* k, const void* v, const void* o, const void* d_o, const float* lse,
                        const int* pos, int window, const float* slopes, void* dq, void* dk, void* dv, int B, int S,
                        int H, int Hk, int D, float scale, int dkv_row_heads, void* ws, size_t ws_bytes, void* stream) {
  B200_CHECK_ARG((reinterpret_cast<uintptr_t>(pos) & 3u) == 0, "attn_bwd_alibi: pos must be 4-byte aligned int32");
  B200_CHECK_ARG(slopes != nullptr && (reinterpret_cast<uintptr_t>(slopes) & 3u) == 0,
                 "attn_bwd_alibi: slopes must be a non-null, 4-byte aligned fp32 [H] array");
  return attn_bwd_impl(q, k, v, o, d_o, lse, true, pos, window, dq, dk, dv, B, S, H, Hk, D, scale, 1, dkv_row_heads,
                       ws, ws_bytes, static_cast<cudaStream_t>(stream), slopes);
}

// prefix-LM backward: query s of row b sees key k iff k <= s or k < prefix[b] (clamped to [0, S] in the kernel).
// Same workspace as the causal backward.
size_t b200_attn_bwd_prefix_workspace_bytes(int B, int S, int H, int Hk, int D) {
  return b200_attn_bwd_workspace_bytes(B, S, H, Hk, D);
}

int b200_attn_bwd_prefix(const void* q, const void* k, const void* v, const void* o, const void* d_o, const float* lse,
                         const int* prefix, void* dq, void* dk, void* dv, int B, int S, int H, int Hk, int D,
                         float scale, int dkv_row_heads, void* ws, size_t ws_bytes, void* stream) {
  B200_CHECK_ARG(prefix != nullptr && (reinterpret_cast<uintptr_t>(prefix) & 3u) == 0,
                 "attn_bwd_prefix: prefix must be a non-null, 4-byte aligned int32 [B] array");
  return attn_bwd_impl(q, k, v, o, d_o, lse, false, nullptr, -1, dq, dk, dv, B, S, H, Hk, D, scale, 1, dkv_row_heads,
                       ws, ws_bytes, static_cast<cudaStream_t>(stream), nullptr, prefix);
}

// dropout backward: the causal / non-causal (pos == nullptr, window < 0, slopes == nullptr), document / window or
// ALiBi backward of attn_fwd_dropout's O = (P o Z / (1 - p_eff)) V, the same p and seed.  Workspace: the document
// variant's when pos, window or slopes select the DOC kernels, else the causal one's.
size_t b200_attn_bwd_dropout_workspace_bytes(int B, int S, int H, int Hk, int D) {
  return b200_attn_bwd_doc_workspace_bytes(B, S, H, Hk, D);
}

int b200_attn_bwd_dropout(const void* q, const void* k, const void* v, const void* o, const void* d_o, const float* lse,
                          const int* pos, int window, const float* slopes, void* dq, void* dk, void* dv, int B, int S,
                          int H, int Hk, int D, float scale, int causal, float p, unsigned long long seed,
                          int dkv_row_heads, void* ws, size_t ws_bytes, void* stream) {
  const cudaStream_t s = static_cast<cudaStream_t>(stream);
  B200_CHECK_ARG(p >= 0.f && p < 1.f, "attn_bwd_dropout: p=%g must lie in [0, 1)", (double)p);
  B200_CHECK_ARG((reinterpret_cast<uintptr_t>(pos) & 3u) == 0, "attn_bwd_dropout: pos must be 4-byte aligned int32");
  B200_CHECK_ARG((reinterpret_cast<uintptr_t>(slopes) & 3u) == 0, "attn_bwd_dropout: slopes must be 4-byte aligned");
  const bool doc = pos != nullptr || window >= 0 || slopes != nullptr;
  B200_CHECK_ARG(!doc || causal, "attn_bwd_dropout: pos, window and slopes need causal=1");
  const uint32_t t = dropout_threshold(p);
  return attn_bwd_impl(q, k, v, o, d_o, lse, doc, pos, window, dq, dk, dv, B, S, H, Hk, D, scale, doc ? 1 : causal,
                       dkv_row_heads, ws, ws_bytes, s, slopes, nullptr, true, t, dropout_scale(t), seed);
}

}  // extern "C"
