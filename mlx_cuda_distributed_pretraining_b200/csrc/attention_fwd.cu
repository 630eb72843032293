// Fused causal / GQA attention forward on Hopper warpgroup MMA (wgmma) fed by TMA through an mbarrier ring.
//
// Computes what FlashAttention._flash_attention (arch/flash_attention.py:97-156 of the reference)
// computes -- O = softmax(Q K^T * scale + mask) V with q-head h reading kv-head h / (H/Hk) -- but
// tiled with an online softmax, so the [B,H,S,S] score tensor the reference materialises (:134)
// never exists.  Also emits LSE = log sum exp(scaled masked scores) for the backward pass.
//
// One CTA per (128-query tile, head, batch), 288 threads:
//   warp 8          TMA producer: the Q tile once, then K / V tiles of 128 keys through a 2-stage ring
//                   (128B-swizzled boxes of 64 head-dim columns, full / empty mbarriers per stage)
//   warpgroups 0-1  64 query rows each: S = Q K^T as wgmma.m64n128k16 with both operands in shared memory,
//                   online softmax on the fp32 accumulators in registers, then O += P V as wgmma with P as the
//                   register A operand (the accumulator fragment packed to bf16) and V read MN-major from smem.
//
// Masks.  In every variant the keys query row r (at position q) sees are one interval [lo, hi] (row_keys):
//   causal / non-causal         [0, min(r, S - 1)] / [0, S - 1]
//   DOC (documents, window)     [r - min(pos[r], W), min(r, S - 1)]   (pos == nullptr reads as pos[r] = r)
//   PREFIX                      [0, min(max(r, P_b - 1), S - 1)],  P_b = prefix[b] clamped to [0, S]
//   CACHED                      [max(0, q - W), q],  q = start[b] + min(r, n_b - 1)
//   RING                        [max(lo_t, q - W_t), q],  lo_t / W_t of the tile's slot range (below)
// Both ends rise with r, so a CTA's key tiles run from its first row's lo to its last row's hi, and a tile is masked
// only when it reaches past a thread's first row's hi or below its second row's lo.  Each score is scaled into the
// log2 domain, gets the ALiBi bias m_h log2e (k - q) (ALIBI), is set to -inf outside its row's interval and then
// enters the online softmax; a row with no visible key in a tile passes through as m_use shows.  ALiBi's bias is
// fmaf(m log2e, c, base) of the compile-time column c, one int -> float conversion per row and tile.  The intervals
// are formed per tile from the rows' positions: CACHED's window starts, held across the key loop, pushed D = 128 into
// spills, and RING's depend on the tile's slot range.
//
// Dropout (DROP = true, on the causal / non-causal and the DOC / ALiBi kernels): O = (P o Z / (1 - p_eff)) V as
// arch/flash_attention.py:146-148 of the reference applies mx.dropout after the softmax.  The softmax P, its row sums
// and the LSE are the dropout-free ones; only the bf16 P fed to the P V MMA has dropped entries zeroed, and O is
// multiplied by 1 / (1 - p_eff) in fp32 after the normalisation.  Z(b, h, q, k) = [r >= t] with r the 16-bit value
// of key k in Philox4x32-10(counter (k >> 3, q, h, b), key (seed lo, seed hi)) (philox_keep8), h the query head: the
// mask depends on positions only, never on the tiling.  A quad's rows are one (row, 8-key chunk) Philox call per
// chunk nc, whose word w[l] holds exactly lane l's keys 8 nc + 2 l + {0, 1}; so each lane computes 8 of the tile's
// 32 calls (both rows, chunks nc = 4 m + l) and the quad exchanges the 8-bit results with 4 shuffles per row.  Bit
// 2 nc + c of keep[r] is this thread's key 8 nc + 2 l + c of row r.
//
// Cached queries (CACHED = true, on the causal kernels, with or without ALiBi): a chunk of L queries per row attends
// over a KV cache [B, s_max, Hk, D] that already holds its own keys; query row i of batch row b sits at position
// start[b] + i, and rows i >= n_b = end[b] - start[b] are padding.  A CTA with only padding rows writes zeros and
// returns.  Otherwise its key tiles are anchored at one past its last valid row's position (<= end[b]), so no cache
// position at or past it is ever loaded (those may hold anything, and 0 * NaN would reach O through the P V MMA);
// keys below 0 are TMA's zero fill and masked.  Padding rows take the last valid row's position and their Q rows are
// zeroed in shared memory, so their outputs are finite whatever Q holds there.
//
// Rotating cache (RING = true, on the CACHED kernels): the cache is a ring of C = s_max slots holding position t in
// slot(t) (common.cuh, ring_slot), and query position q sees key position k iff k <= q, q - k <= W and (k < 4 or
// q - k <= M - 5).  The CTA's queries q_lo .. q_hi see the sinks and the arc A = max(4, q_lo - min(M - 5, W)) .. q_hi,
// whose slots form at most two ranges (the arc wraps at most once, as C >= M + L - 1).  Thread 0 writes a table of
// three slot ranges into shared memory: the sink tile (ending at slot min(4, q_hi + 1)), then the arc's ranges, each
// tiled by 128-slot tiles anchored at the range's end.  Inside a range position = slot + off, and a range's keys are
// masked below its first position lo_t, with W_t = W for the sinks and min(M - 5, W) for the arc.  No slot at or past
// end[b] is loaded before the ring first wraps; after it every slot holds a written key.
//
// Each flag set to false compiles to the kernels without it.
#include "common.cuh"
#include "host.h"

namespace b200 {

namespace {

constexpr int ATT_BQ = 128;
constexpr int ATT_BKV = 128;
constexpr int FWD_THREADS = 288;  // two consumer warpgroups + one producer warp
constexpr float kLog2e = 1.4426950408889634f;

template <int D>
struct FwdCfg {
  static constexpr int NB = D / 64;                 // 64-column (128-byte) blocks per row
  static constexpr int Q_BYTES = ATT_BQ * D * 2;
  static constexpr int KV_BYTES = ATT_BKV * D * 2;  // one K or V stage
  static constexpr int OFF_Q = 0;
  static constexpr int OFF_K = OFF_Q + Q_BYTES;       // 2 stages
  static constexpr int OFF_V = OFF_K + 2 * KV_BYTES;  // 2 stages
  static constexpr int OFF_BAR = OFF_V + 2 * KV_BYTES;
  static constexpr int SMEM_BYTES = OFF_BAR + 64 + 1024;
};

struct FwdArgs {
  __nv_bfloat16* o;
  float* lse;
  int B, S, H, Hk;
  float scale;
  int causal;
  const int* pos;  // [B, S] positions within documents (DOC kernels only; null: pos[q] = q)
  int window;      // query q sees keys from q - min(pos[q], window) (CACHED: q - window); INT_MAX for none
  const float* slopes;  // ALIBI: [H] fp32 per-query-head slopes
  const int* prefix;    // PREFIX: [B] int32 prefix lengths (clamped to [0, S])
  uint32_t drop_t;      // DROP: keep threshold t = round(p 65536) on the 16-bit Philox values
  float drop_inv;       // DROP: 1 / (1 - t / 65536)
  unsigned long long drop_seed;  // DROP: Philox key
  const int* start;     // CACHED: [B] int32 position of each row's first query; S is the chunk length L
  const int* end;       // CACHED: [B] int32 cached positions once the chunk is in (its last query's position + 1)
  int s_max;            // CACHED: positions of the K / V cache (RING: its slots C)
  int ring_m;           // RING: max_kv_size M
};

// RING: the table of slot ranges (see the head of this file), 4 ints per range: the running tile count at its end,
// the slot of its first tile, the offset from slot to position and its first visible position
constexpr int RING_TAB_BYTES = 64;
__device__ __forceinline__ void ring_table(int* tab, int qlo, int qhi, int C, int M, int W) {
  int n = qlo - W <= RING_SINKS - 1 ? 1 : 0;  // some sink is in some query's window
  tab[0] = n;
  tab[1] = min(RING_SINKS, qhi + 1) - ATT_BKV;
  tab[2] = tab[3] = 0;
  const int A = max(RING_SINKS, qlo - min(M - 5, W));
  int lo[2] = {0, 0}, hi[2] = {0, 0}, off[2] = {0, 0};
  if (A <= qhi) {
    const int sa = ring_slot(A, C), sh = ring_slot(qhi, C);
    lo[0] = sa;
    if (sa <= sh) {
      hi[0] = sh + 1;
      off[0] = qhi - sh;
    } else {  // the older positions up to slot C - 1, then the newer ones from slot 4
      hi[0] = C;
      off[0] = A - sa;
      lo[1] = RING_SINKS;
      hi[1] = sh + 1;
      off[1] = qhi - sh;
    }
  }
  for (int r = 0; r < 2; ++r) {
    const int nt = (hi[r] - lo[r] + ATT_BKV - 1) / ATT_BKV;
    n += nt;
    tab[4 * r + 4] = n;
    tab[4 * r + 5] = hi[r] - nt * ATT_BKV;
    tab[4 * r + 6] = off[r];
    tab[4 * r + 7] = lo[r] + off[r];
  }
}
// RING: tile j's first slot, its range (0: the sinks), the range's offset and first visible position
__device__ __forceinline__ int ring_tile(const int* tab, int j, int& r, int& off, int& rlo) {
  r = (j >= tab[0]) + (j >= tab[4]);
  off = tab[4 * r + 2];
  rlo = tab[4 * r + 3];
  return tab[4 * r + 1] + (j - (r == 0 ? 0 : tab[4 * r - 4])) * ATT_BKV;
}

// first key query `row` of batch row b may see: its document start, or its window start when that is later
__device__ __forceinline__ int key_start(const FwdArgs& p, int b, int row) {
  // (the null-pos form max(0, row - window) is row - min(row, window); written so, it keeps D = 128 within 168
  // registers without spills)
  return p.pos ? row - min(__ldg(p.pos + (long long)b * p.S + row), p.window) : max(0, row - p.window);
}

// The position of query row `row`, from which ALiBi measures k - q: the row itself, or for CACHED start[b] + row
// (c_st, c_nv: the batch row's first position and valid rows), where a padding row takes the last valid row's
template <bool CACHED>
__device__ __forceinline__ int row_pos(int row, int c_st, int c_nv) {
  return CACHED ? c_st + min(row, c_nv - 1) : row;
}

// The keys [lo, hi] that the query at position q (row_pos) sees, as in the table at the head of this file.  dstart:
// DOC, the row's key_start; pfx: PREFIX, the batch row's prefix length; ring_lo / ring_w: RING, the first position
// and the window of the tile's slot range (ring_tile).
struct RowKeys {
  int lo, hi;
};
template <bool DOC, bool PREFIX, bool CACHED, bool RING>
__device__ __forceinline__ RowKeys row_keys(const FwdArgs& p, int q, int dstart, int pfx, int ring_lo = 0,
                                            int ring_w = 0) {
  if constexpr (CACHED) return {RING ? max(ring_lo, q - ring_w) : max(0, q - p.window), q};
  const int last = p.S - 1;
  return {DOC ? dstart : 0, PREFIX ? min(max(q, pfx - 1), last) : p.causal ? min(q, last) : last};
}

// DROP: keep bits of a thread's 2 x 32 scores in the key tile from k0 (rows row_a, row_a + 8).  Byte m of lane L's
// `own` is chunk 4 m + L of row r; this lane takes bits 2 (lane % 4) + {0, 1} of every byte.
__device__ __forceinline__ void drop_keep_bits(const FwdArgs& p, int k0, int row_a, int h, int b, int lane,
                                               uint32_t* keep) {
  const uint32_t kc = (uint32_t)(k0 >> 3) + (lane & 3);
  const uint32_t sk0 = (uint32_t)p.drop_seed, sk1 = (uint32_t)(p.drop_seed >> 32);
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    uint32_t own = 0u;
#pragma unroll 1
    for (int m = 0; m < 4; ++m) own |= philox_keep8(kc + 4 * m, row_a + 8 * r, h, b, sk0, sk1, p.drop_t) << (8 * m);
    keep[r] = 0u;
#pragma unroll
    for (int L = 0; L < 4; ++L) {
      const uint32_t w = __shfl_sync(0xffffffffu, own, L, 4);
      keep[r] |= ((w >> (2 * (lane & 3))) & 0x03030303u) << (2 * L);
    }
  }
}

template <int D>
__device__ __forceinline__ void pv_mma(float* o, const uint32_t* a, uint64_t db) {
  if constexpr (D == 128) wgmma_m64n128k16_rs<1>(o, a, db);
  else wgmma_m64n64k16_rs<1>(o, a, db);
}

template <int D, bool DOC, bool ALIBI = false, bool PREFIX = false, bool DROP = false, bool CACHED = false,
          bool RING = false>
__global__ void __launch_bounds__(FWD_THREADS, 1)
attn_fwd_kernel(const __grid_constant__ CUtensorMap tmQ, const __grid_constant__ CUtensorMap tmK,
                const __grid_constant__ CUtensorMap tmV, const FwdArgs p) {
  static_assert(!RING || CACHED, "the ring is built on the cached kernel");
  static_assert(!PREFIX || (!DOC && !ALIBI), "the prefix mask is built on the causal kernel");
  static_assert(!PREFIX || !DROP, "dropout is not built on the prefix kernels");
  static_assert(!CACHED || (!DOC && !PREFIX && !DROP), "cached queries are built on the causal kernel");
  using Cfg = FwdCfg<D>;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  const uint32_t s0 = smem_u32(smem);
  const uint32_t sQ = s0 + Cfg::OFF_Q, sK = s0 + Cfg::OFF_K, sV = s0 + Cfg::OFF_V;
  const uint32_t q_full = s0 + Cfg::OFF_BAR, kv_full0 = q_full + 8, kv_empty0 = q_full + 24;
  int* ring_tab = reinterpret_cast<int*>(smem + Cfg::OFF_BAR + 64);  // RING only
  const int qt = blockIdx.x, h = blockIdx.y, b = blockIdx.z;
  const int hk = h / (p.H / p.Hk);
  const int q0 = qt * ATT_BQ;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int pfx = PREFIX ? min(max(__ldg(p.prefix + b), 0), p.S) : 0;
  // CACHED: the row's first query position and valid rows
  int c_st = 0, c_nv = 0;
  if constexpr (CACHED) {
    c_st = max(__ldg(p.start + b), 0);
    c_nv = min((RING ? __ldg(p.end + b) : min(__ldg(p.end + b), p.s_max)) - c_st, p.S);
    if (q0 >= c_nv) {  // padding rows only
      const int rows = min(ATT_BQ, p.S - q0);
      for (int i = threadIdx.x; i < rows * (D / 8); i += FWD_THREADS) {
        const long long row = (long long)b * p.S + q0 + i / (D / 8);
        stg128(p.o + (row * p.H + h) * D + (i % (D / 8)) * 8, make_uint4(0u, 0u, 0u, 0u));
        if (i % (D / 8) == 0 && p.lse != nullptr) p.lse[((long long)b * p.H + h) * p.S + q0 + i / (D / 8)] = 0.f;
      }
      return;
    }
  }
  // key tiles from the CTA's first row's first key to its last row's last; CACHED: tile j holds keys
  // kbase + 128 j .., anchored at the last one
  const int q_first = row_pos<CACHED>(q0, c_st, c_nv);
  const int q_last = row_pos<CACHED>(min(q0 + ATT_BQ, p.S) - 1, c_st, c_nv);
  const RowKeys first = row_keys<DOC, PREFIX, CACHED, RING>(p, q_first, DOC ? key_start(p, b, q0) : 0, pfx);
  const RowKeys last = row_keys<DOC, PREFIX, CACHED, RING>(p, q_last, 0, pfx);
  int j0 = 0, n_kv = 0, kbase = 0;
  if constexpr (RING) {
    if (threadIdx.x == 0) ring_table(ring_tab, q_first, q_last, p.s_max, p.ring_m, p.window);
  } else if constexpr (CACHED) {
    n_kv = (last.hi + 1 - first.lo + ATT_BKV - 1) / ATT_BKV;
    kbase = last.hi + 1 - n_kv * ATT_BKV;
  } else {
    j0 = max(0, first.lo) / ATT_BKV;
    n_kv = last.hi / ATT_BKV + 1;
  }

  if (threadIdx.x == 0) {
    mbar_init(q_full, 1);
    for (int s = 0; s < 2; ++s) {
      mbar_init(kv_full0 + 8 * s, 1);
      mbar_init(kv_empty0 + 8 * s, 2);  // one arrival per consumer warpgroup
    }
    fence_mbar_init();
  }
  __syncthreads();
  if constexpr (RING) n_kv = ring_tab[8];

  if (warp == 8) {
    if (lane == 0) {
      tma_prefetch_desc(&tmQ);
      tma_prefetch_desc(&tmK);
      tma_prefetch_desc(&tmV);
      mbar_arrive_expect_tx(q_full, Cfg::Q_BYTES);
      for (int nb = 0; nb < Cfg::NB; ++nb) tma_load_4d(sQ + nb * ATT_BQ * 128, &tmQ, q_full, nb * 64, h, q0, b);
      for (int j = j0; j < n_kv; ++j) {
        const int s = (j - j0) & 1;
        mbar_wait(kv_empty0 + 8 * s, (((j - j0) >> 1) & 1) ^ 1u);
        const uint32_t full = kv_full0 + 8 * s;
        mbar_arrive_expect_tx(full, 2 * Cfg::KV_BYTES);
        int slot = kbase + j * ATT_BKV;
        if constexpr (RING) {
          int r, off, rlo;
          slot = ring_tile(ring_tab, j, r, off, rlo);
        }
        for (int nb = 0; nb < Cfg::NB; ++nb) {
          tma_load_4d(sK + s * Cfg::KV_BYTES + nb * ATT_BKV * 128, &tmK, full, nb * 64, hk, slot, b);
          tma_load_4d(sV + s * Cfg::KV_BYTES + nb * ATT_BKV * 128, &tmV, full, nb * 64, hk, slot, b);
        }
      }
    }
    return;
  }

  const int wg = warp >> 2, wq = warp & 3;
  float o[D / 2];
#pragma unroll
  for (int i = 0; i < D / 2; ++i) o[i] = 0.f;
  float m_r[2] = {-INFINITY, -INFINITY}, l_r[2] = {0.f, 0.f};
  const float sl2 = p.scale * kLog2e;
  const int row_a = q0 + wg * 64 + wq * 16 + (lane >> 2);  // this thread's rows: row_a, row_a + 8
  // DOC: document / window start of each of this thread's rows; a row past S takes the last row's, which keeps the
  // starts rising with the row as the edge-tile test needs
  int dstart[2] = {0, 0};
  if constexpr (DOC) {
#pragma unroll
    for (int r = 0; r < 2; ++r) dstart[r] = key_start(p, b, min(row_a + 8 * r, p.S - 1));
  }
  // CACHED: the positions of this thread's rows, held across the key loop (elsewhere a row's position is the row)
  const int qpos[2] = {row_pos<CACHED>(row_a, c_st, c_nv), row_pos<CACHED>(row_a + 8, c_st, c_nv)};
  float ml2 = 0.f;  // ALIBI: this head's slope in log2 units
  if constexpr (ALIBI) ml2 = __ldg(p.slopes + h) * kLog2e;
  mbar_wait(q_full, 0);
  if constexpr (CACHED) {
    // padding rows of Q may hold anything: zero this warpgroup's (each 128-byte row of a 64-column block is one
    // swizzled line) before its S MMAs read them
    const int r0 = q0 + wg * 64;
    if (r0 + 64 > c_nv) {
      for (int i = threadIdx.x & 127; i < Cfg::NB * 64 * 8; i += 128) {
        const int rr = (i >> 3) & 63;
        if (r0 + rr >= c_nv)
          sts128(sQ + (i >> 9) * ATT_BQ * 128 + (wg * 64 + rr) * 128 + (i & 7) * 16, make_uint4(0u, 0u, 0u, 0u));
      }
      fence_proxy_async_smem();
      named_bar_sync(1 + wg, 128);
    }
  }

  for (int j = j0; j < n_kv; ++j) {
    const int s = (j - j0) & 1;
    mbar_wait(kv_full0 + 8 * s, ((j - j0) >> 1) & 1);
    const uint32_t tK = sK + s * Cfg::KV_BYTES, tV = sV + s * Cfg::KV_BYTES;
    int k0 = kbase + j * ATT_BKV;

    int ring_lo = 0, ring_w = 0;
    if constexpr (RING) {  // the tile's first position and its slot range's bounds
      int r, off;
      k0 = ring_tile(ring_tab, j, r, off, ring_lo) + off;
      ring_w = r == 0 ? p.window : min(p.ring_m - 5, p.window);
    }
    // S = Q K^T: 64 rows x 128 keys per warpgroup, both operands K-major (head dim contiguous)
    float sc[64];
#pragma unroll
    for (int i = 0; i < 64; ++i) sc[i] = 0.f;
    wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < D / 16; ++kk) {
      const uint64_t da = make_wgmma_desc_sw128(sQ + (kk >> 2) * ATT_BQ * 128 + wg * 64 * 128 + (kk & 3) * 32, 16, 1024);
      const uint64_t db = make_wgmma_desc_sw128(tK + (kk >> 2) * ATT_BKV * 128 + (kk & 3) * 32, 16, 1024);
      wgmma_m64n128k16_ss<0, 0>(sc, da, db);
    }
    wgmma_commit();
    wgmma_wait<0>();

    // scale (log2 domain), bias, mask, online softmax.  Accumulator chunk nc holds keys k_lane + c, c = 8 nc + {0, 1};
    // row r sees the columns c_lo[r] .. c_hi[r].  Only a tile that some row's range does not cover is masked (edge);
    // both ends of the ranges rise with the row.  The bias gets a pass of its own: in the mask's pass, with the
    // bounds, it pushed the D = 128 ALiBi kernels into spills.
    RowKeys rk[2];
#pragma unroll
    for (int r = 0; r < 2; ++r)
      rk[r] = row_keys<DOC, PREFIX, CACHED, RING>(p, CACHED ? qpos[r] : (row_a + 8 * r), dstart[r], pfx, ring_lo,
                                                  ring_w);
    const bool edge = k0 + ATT_BKV - 1 > rk[0].hi || k0 < rk[1].lo;
    const int k_lane = k0 + (lane & 3) * 2;
    float abase[2] = {0.f, 0.f};  // ALIBI: the bias m log2e (key - q) of column c is fmaf(m log2e, c, abase[r])
    int c_lo[2], c_hi[2];
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      c_lo[r] = rk[r].lo - k_lane;
      c_hi[r] = rk[r].hi - k_lane;
      if constexpr (ALIBI) abase[r] = ml2 * (float)(k_lane - (CACHED ? qpos[r] : (row_a + 8 * r)));
    }
    float mx[2] = {-INFINITY, -INFINITY};
#pragma unroll
    for (int nc = 0; nc < 16; ++nc) {
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const int c = nc * 8 + (e & 1);
        float x = sc[4 * nc + e] * sl2;
        if constexpr (ALIBI) x += fmaf(ml2, (float)c, abase[e >> 1]);
        sc[4 * nc + e] = x;
      }
    }
#pragma unroll
    for (int nc = 0; nc < 16; ++nc) {
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const int c = nc * 8 + (e & 1);
        sc[4 * nc + e] = edge && (c < c_lo[e >> 1] || c > c_hi[e >> 1]) ? -INFINITY : sc[4 * nc + e];
      }
    }
#pragma unroll
    for (int i = 0; i < 64; ++i) mx[(i >> 1) & 1] = fmaxf(mx[(i >> 1) & 1], sc[i]);
    float alpha[2], m_use[2];
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      mx[r] = fmaxf(mx[r], __shfl_xor_sync(0xffffffffu, mx[r], 1));
      mx[r] = fmaxf(mx[r], __shfl_xor_sync(0xffffffffu, mx[r], 2));
      const float m_new = fmaxf(m_r[r], mx[r]);
      m_use[r] = (m_new == -INFINITY) ? 0.f : m_new;
      alpha[r] = exp2f(m_r[r] - m_use[r]);
      m_r[r] = m_new;
      l_r[r] *= alpha[r];
    }
    uint32_t pa[8][4];
#pragma unroll
    for (int nc = 0; nc < 16; ++nc) {
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const float pe = exp2f(sc[4 * nc + e] - m_use[e >> 1]);
        sc[4 * nc + e] = pe;
        l_r[e >> 1] += pe;
      }
    }
    // two adjacent key chunks form one k16 A fragment: (row, k 0-7), (row + 8, k 0-7), (row, k 8-15), (row + 8, k 8-15)
#pragma unroll
    for (int kk = 0; kk < 8; ++kk) {
      pa[kk][0] = pack_bf16x2(sc[8 * kk + 0], sc[8 * kk + 1]);
      pa[kk][1] = pack_bf16x2(sc[8 * kk + 2], sc[8 * kk + 3]);
      pa[kk][2] = pack_bf16x2(sc[8 * kk + 4], sc[8 * kk + 5]);
      pa[kk][3] = pack_bf16x2(sc[8 * kk + 6], sc[8 * kk + 7]);
    }
    // DROP: zero the dropped bf16 halves of P (the row sums above keep every visible key).  The keep bits are made
    // here, where the S fragment is dead: live across the S MMAs or the softmax they push D = 128 into spills.
    // pa[kk][i] holds chunk 2 kk + (i >> 1) of row i & 1.
    if constexpr (DROP) {
      uint32_t keep[2];
      drop_keep_bits(p, k0, row_a, h, b, lane, keep);
#pragma unroll
      for (int kk = 0; kk < 8; ++kk) {
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          const uint32_t x = keep[i & 1] >> (4 * kk + 2 * (i >> 1));
          pa[kk][i] &= (x & 1u) * 0xffffu | ((x >> 1) & 1u) * 0xffff0000u;
        }
      }
    }
#pragma unroll
    for (int dc = 0; dc < D / 8; ++dc) {
      o[4 * dc + 0] *= alpha[0];
      o[4 * dc + 1] *= alpha[0];
      o[4 * dc + 2] *= alpha[1];
      o[4 * dc + 3] *= alpha[1];
    }
    // O += P V: V is the MN-major B operand (keys = k rows of 128 B, head-dim blocks LBO apart)
    wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < 8; ++kk)
      pv_mma<D>(o, pa[kk], make_wgmma_desc_sw128(tV + kk * 2048, ATT_BKV * 128, 1024));
    wgmma_commit();
    wgmma_wait<0>();
    if ((threadIdx.x & 127) == 0) mbar_arrive(kv_empty0 + 8 * s);
  }

  // normalise, store O and LSE (natural log of the scaled scores' sum-exp)
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    l_r[r] += __shfl_xor_sync(0xffffffffu, l_r[r], 1);
    l_r[r] += __shfl_xor_sync(0xffffffffu, l_r[r], 2);
  }
  // DROP: the normaliser carries the fp32 dropout scale 1 / (1 - p_eff)
  const float inv[2] = {(DROP ? p.drop_inv : 1.0f) / l_r[0], (DROP ? p.drop_inv : 1.0f) / l_r[1]};
  const long long q_stride = (long long)p.H * D;
  __nv_bfloat16* ob = p.o + (long long)b * p.S * q_stride + (long long)h * D;
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    const int row = row_a + 8 * r;
    if (row >= p.S) continue;
    __nv_bfloat16* orow = ob + (long long)row * q_stride;
#pragma unroll
    for (int dc = 0; dc < D / 8; ++dc)
      *reinterpret_cast<uint32_t*>(orow + dc * 8 + (lane & 3) * 2) =
          pack_bf16x2(o[4 * dc + 2 * r] * inv[r], o[4 * dc + 2 * r + 1] * inv[r]);
    if ((lane & 3) == 0 && (!CACHED || p.lse != nullptr))
      p.lse[((long long)b * p.H + h) * p.S + row] = (m_r[r] + log2f(l_r[r])) / kLog2e;
  }
}

template <int D, bool DOC, bool ALIBI = false, bool PREFIX = false, bool DROP = false, bool CACHED = false,
          bool RING = false>
int launch_fwd(const CUtensorMap& tmQ, const CUtensorMap& tmK, const CUtensorMap& tmV, const FwdArgs& a,
               cudaStream_t stream) {
  using Cfg = FwdCfg<D>;
  auto kern = attn_fwd_kernel<D, DOC, ALIBI, PREFIX, DROP, CACHED, RING>;
  constexpr int smem_bytes = Cfg::SMEM_BYTES + (RING ? RING_TAB_BYTES : 0);
  static bool attr_set = false;
  if (!attr_set) {
    B200_CHECK_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, smem_bytes));
    attr_set = true;
  }
  dim3 grid((a.S + ATT_BQ - 1) / ATT_BQ, a.H, a.B);
  kern<<<grid, FWD_THREADS, smem_bytes, stream>>>(tmQ, tmK, tmV, a);
  B200_CHECK_LAUNCH();
  return B200_OK;
}

template <bool DOC, bool ALIBI = false, bool PREFIX = false, bool DROP = false, bool CACHED = false, bool RING = false>
int launch_fwd_d(int D, const CUtensorMap& tmQ, const CUtensorMap& tmK, const CUtensorMap& tmV, const FwdArgs& a,
                 cudaStream_t stream) {
  return D == 64 ? launch_fwd<64, DOC, ALIBI, PREFIX, DROP, CACHED, RING>(tmQ, tmK, tmV, a, stream)
                 : launch_fwd<128, DOC, ALIBI, PREFIX, DROP, CACHED, RING>(tmQ, tmK, tmV, a, stream);
}

}  // namespace

// [B, S, heads, D] bf16 tensor -> 4-D tensor map {D, heads, S, B}, box {64, 1, rows, 1}, 128B swizzle
int make_bshd_map(CUtensorMap* tm, const void* base, int B, int S, int heads, int D, int box_rows) {
  const uint64_t dims[4] = {(uint64_t)D, (uint64_t)heads, (uint64_t)S, (uint64_t)B};
  const uint64_t strides[3] = {(uint64_t)D * 2, (uint64_t)heads * D * 2, (uint64_t)S * heads * D * 2};
  const uint32_t box[4] = {64, 1, (uint32_t)box_rows, 1};
  return make_tensor_map(tm, base, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, 4, dims, strides, box, true);
}

namespace {

// doc selects the document / window instantiation; window < 0 means none; slopes selects ALiBi; prefix (causal, not
// doc) the prefix-LM kernels; drop the dropout kernels (not with prefix); start the cached queries (not doc), over a
// K / V cache of s_max positions, and ring_m > 0 their rotating cache of s_max slots
int attn_fwd_impl(const void* q, const void* k, const void* v, void* o, float* lse, bool doc, const int* pos,
                  int window, int B, int S, int H, int Hk, int D, float scale, int causal, cudaStream_t stream,
                  const float* slopes = nullptr, const int* prefix = nullptr, bool drop = false,
                  uint32_t drop_t = 0, float drop_inv = 1.f, unsigned long long drop_seed = 0,
                  const int* start = nullptr, const int* end = nullptr, int s_max = 0, int ring_m = 0) {
  B200_CHECK_ARG(B > 0 && S > 0 && H > 0 && Hk > 0 && H % Hk == 0,
                 "attn_fwd: bad shape B=%d S=%d H=%d Hk=%d", B, S, H, Hk);
  B200_CHECK_ARG(D == 64 || D == 128, "attn_fwd: head_dim %d unsupported (64 or 128; pad smaller dims)", D);
  B200_CHECK_ARG((reinterpret_cast<uintptr_t>(o) & 15u) == 0, "attn_fwd: o must be 16-byte aligned");
  CUtensorMap tmQ, tmK, tmV;
  int rc;
  if ((rc = make_bshd_map(&tmQ, q, B, S, H, D, ATT_BQ))) return rc;
  if ((rc = make_bshd_map(&tmK, k, B, start ? s_max : S, Hk, D, ATT_BKV))) return rc;
  if ((rc = make_bshd_map(&tmV, v, B, start ? s_max : S, Hk, D, ATT_BKV))) return rc;
  FwdArgs a;
  a.o = reinterpret_cast<__nv_bfloat16*>(o);
  a.lse = lse;
  a.B = B;
  a.S = S;
  a.H = H;
  a.Hk = Hk;
  a.scale = scale;
  a.causal = causal;
  a.pos = pos;
  a.window = window < 0 ? INT_MAX : window;
  a.slopes = slopes;
  a.prefix = prefix;
  a.drop_t = drop_t;
  a.drop_inv = drop_inv;
  a.drop_seed = drop_seed;
  a.start = start;
  a.end = end;
  a.s_max = s_max;
  a.ring_m = ring_m;
  if (start && ring_m > 0)
    return slopes ? launch_fwd_d<false, true, false, false, true, true>(D, tmQ, tmK, tmV, a, stream)
                  : launch_fwd_d<false, false, false, false, true, true>(D, tmQ, tmK, tmV, a, stream);
  if (start)
    return slopes ? launch_fwd_d<false, true, false, false, true>(D, tmQ, tmK, tmV, a, stream)
                  : launch_fwd_d<false, false, false, false, true>(D, tmQ, tmK, tmV, a, stream);
  if (drop) {
    if (slopes) return launch_fwd_d<true, true, false, true>(D, tmQ, tmK, tmV, a, stream);
    if (doc) return launch_fwd_d<true, false, false, true>(D, tmQ, tmK, tmV, a, stream);
    return launch_fwd_d<false, false, false, true>(D, tmQ, tmK, tmV, a, stream);
  }
  if (prefix) return launch_fwd_d<false, false, true>(D, tmQ, tmK, tmV, a, stream);
  if (slopes) return launch_fwd_d<true, true>(D, tmQ, tmK, tmV, a, stream);
  if (doc) return launch_fwd_d<true>(D, tmQ, tmK, tmV, a, stream);
  return launch_fwd_d<false>(D, tmQ, tmK, tmV, a, stream);
}

}  // namespace
}  // namespace b200

using namespace b200;

extern "C" {

int b200_attn_fwd(const void* q, const void* k, const void* v, void* o, float* lse, int B, int S, int H,
                  int Hk, int D, float scale, int causal, void* stream) {
  const cudaStream_t s = static_cast<cudaStream_t>(stream);
  return attn_fwd_impl(q, k, v, o, lse, false, nullptr, -1, B, S, H, Hk, D, scale, causal, s);
}

// document-causal: query s of row b sees keys s - pos[b, s] .. s
int b200_attn_fwd_doc(const void* q, const void* k, const void* v, void* o, float* lse, const int* pos, int B, int S,
                      int H, int Hk, int D, float scale, void* stream) {
  B200_CHECK_ARG(pos != nullptr && (reinterpret_cast<uintptr_t>(pos) & 3u) == 0,
                 "attn_fwd_doc: pos must be a non-null, 4-byte aligned int32 [B, S] array");
  return attn_fwd_impl(q, k, v, o, lse, true, pos, -1, B, S, H, Hk, D, scale, 1, static_cast<cudaStream_t>(stream));
}

// sliding window: query s sees keys s - min(pos[b, s], window) .. s; pos == nullptr means pos[b, s] = s
int b200_attn_fwd_window(const void* q, const void* k, const void* v, void* o, float* lse, const int* pos, int window,
                         int B, int S, int H, int Hk, int D, float scale, void* stream) {
  B200_CHECK_ARG((reinterpret_cast<uintptr_t>(pos) & 3u) == 0, "attn_fwd_window: pos must be 4-byte aligned int32");
  B200_CHECK_ARG(window >= 0, "attn_fwd_window: window=%d must be >= 0", window);
  return attn_fwd_impl(q, k, v, o, lse, true, pos, window, B, S, H, Hk, D, scale, 1, static_cast<cudaStream_t>(stream));
}

// ALiBi: attn_fwd_window (window < 0: none) with the bias slopes[h] * (k - s) added to every visible score
int b200_attn_fwd_alibi(const void* q, const void* k, const void* v, void* o, float* lse, const int* pos, int window,
                        const float* slopes, int B, int S, int H, int Hk, int D, float scale, void* stream) {
  const cudaStream_t s = static_cast<cudaStream_t>(stream);
  B200_CHECK_ARG((reinterpret_cast<uintptr_t>(pos) & 3u) == 0, "attn_fwd_alibi: pos must be 4-byte aligned int32");
  B200_CHECK_ARG(slopes != nullptr && (reinterpret_cast<uintptr_t>(slopes) & 3u) == 0,
                 "attn_fwd_alibi: slopes must be a non-null, 4-byte aligned fp32 [H] array");
  return attn_fwd_impl(q, k, v, o, lse, true, pos, window, B, S, H, Hk, D, scale, 1, s, slopes);
}

// prefix-LM: query s of row b sees key k iff k <= s or k < prefix[b] (clamped to [0, S] in the kernel)
int b200_attn_fwd_prefix(const void* q, const void* k, const void* v, void* o, float* lse, const int* prefix, int B,
                         int S, int H, int Hk, int D, float scale, void* stream) {
  const cudaStream_t s = static_cast<cudaStream_t>(stream);
  B200_CHECK_ARG(prefix != nullptr && (reinterpret_cast<uintptr_t>(prefix) & 3u) == 0,
                 "attn_fwd_prefix: prefix must be a non-null, 4-byte aligned int32 [B] array");
  return attn_fwd_impl(q, k, v, o, lse, false, nullptr, -1, B, S, H, Hk, D, scale, 1, s, nullptr, prefix);
}

// dropout: the causal / non-causal (pos == nullptr, window < 0, slopes == nullptr), document / window or ALiBi
// forward with O = (P o Z / (1 - p_eff)) V; t = min(rint(p 65536), 65535), p_eff = t / 65536
int b200_attn_fwd_dropout(const void* q, const void* k, const void* v, void* o, float* lse, const int* pos, int window,
                          const float* slopes, int B, int S, int H, int Hk, int D, float scale, int causal, float p,
                          unsigned long long seed, void* stream) {
  const cudaStream_t s = static_cast<cudaStream_t>(stream);
  B200_CHECK_ARG(p >= 0.f && p < 1.f, "attn_fwd_dropout: p=%g must lie in [0, 1)", (double)p);
  B200_CHECK_ARG((reinterpret_cast<uintptr_t>(pos) & 3u) == 0, "attn_fwd_dropout: pos must be 4-byte aligned int32");
  B200_CHECK_ARG((reinterpret_cast<uintptr_t>(slopes) & 3u) == 0, "attn_fwd_dropout: slopes must be 4-byte aligned");
  const bool doc = pos != nullptr || window >= 0 || slopes != nullptr;
  B200_CHECK_ARG(!doc || causal, "attn_fwd_dropout: pos, window and slopes need causal=1");
  const uint32_t t = dropout_threshold(p);
  return attn_fwd_impl(q, k, v, o, lse, doc, pos, window, B, S, H, Hk, D, scale, doc ? 1 : causal, s, slopes,
                       nullptr, true, t, dropout_scale(t), seed);
}

// cached queries: query i of row b sits at position start[b] + i and sees cached key k iff
// max(0, p - window) <= k <= p for i < end[b] - start[b]; the later rows are padding (finite, unspecified)
int b200_attn_fwd_cached(const void* q, const void* k_cache, const void* v_cache, const int* start, const int* end,
                         void* o, float* lse, int window, const float* slopes, int B, int L, int s_max, int H, int Hk,
                         int D, float scale, void* stream) {
  B200_CHECK_ARG(B > 0 && L > 0 && s_max > 0 && H > 0 && Hk > 0 && H % Hk == 0,
                 "attn_fwd_cached: bad shape B=%d L=%d s_max=%d H=%d Hk=%d", B, L, s_max, H, Hk);
  B200_CHECK_ARG(D == 64 || D == 128, "attn_fwd_cached: head_dim %d unsupported (64 or 128)", D);
  B200_CHECK_ARG(start != nullptr && end != nullptr && (reinterpret_cast<uintptr_t>(start) & 3u) == 0 &&
                     (reinterpret_cast<uintptr_t>(end) & 3u) == 0,
                 "attn_fwd_cached: start and end must be non-null, 4-byte aligned int32 [B] arrays");
  B200_CHECK_ARG(al16(q) && al16(k_cache) && al16(v_cache) && al16(o),
                 "attn_fwd_cached: q, k_cache, v_cache and o must be 16-byte aligned");
  B200_CHECK_ARG((reinterpret_cast<uintptr_t>(slopes) & 3u) == 0 && (reinterpret_cast<uintptr_t>(lse) & 3u) == 0,
                 "attn_fwd_cached: slopes and lse must be 4-byte aligned");
  return attn_fwd_impl(q, k_cache, v_cache, o, lse, false, nullptr, window, B, L, H, Hk, D, scale, 1,
                       static_cast<cudaStream_t>(stream), slopes, nullptr, false, 0, 1.f, 0, start, end, s_max);
}

// The rotating KV cache of the reference's generator (core/generation_lite.py:103, :120): a chunk of queries at
// positions start[b] + i over a ring of C slots that already holds their keys (include/b200_hotpath.h)
int b200_attn_fwd_ring(const void* q, const void* k_ring, const void* v_ring, const int* start, const int* end,
                       void* o, float* lse, int max_kv, int window, const float* slopes, int B, int L, int C, int H,
                       int Hk, int D, float scale, void* stream) {
  B200_CHECK_ARG(B > 0 && L > 0 && H > 0 && Hk > 0 && H % Hk == 0, "attn_fwd_ring: bad shape B=%d L=%d H=%d Hk=%d",
                 B, L, H, Hk);
  B200_CHECK_ARG(D == 64 || D == 128, "attn_fwd_ring: head_dim %d unsupported (64 or 128)", D);
  B200_CHECK_ARG(max_kv >= 5 && (long long)C >= (long long)max_kv + L - 1,
                 "attn_fwd_ring: max_kv=%d must be >= 5 and C=%d >= max_kv + L - 1 (L=%d)", max_kv, C, L);
  B200_CHECK_ARG(start != nullptr && end != nullptr && (reinterpret_cast<uintptr_t>(start) & 3u) == 0 &&
                     (reinterpret_cast<uintptr_t>(end) & 3u) == 0,
                 "attn_fwd_ring: start and end must be non-null, 4-byte aligned int32 [B] arrays");
  B200_CHECK_ARG(al16(q) && al16(k_ring) && al16(v_ring) && al16(o),
                 "attn_fwd_ring: q, k_ring, v_ring and o must be 16-byte aligned");
  B200_CHECK_ARG((reinterpret_cast<uintptr_t>(slopes) & 3u) == 0 && (reinterpret_cast<uintptr_t>(lse) & 3u) == 0,
                 "attn_fwd_ring: slopes and lse must be 4-byte aligned");
  return attn_fwd_impl(q, k_ring, v_ring, o, lse, false, nullptr, window, B, L, H, Hk, D, scale, 1,
                       static_cast<cudaStream_t>(stream), slopes, nullptr, false, 0, 1.f, 0, start, end, C, max_kv);
}

}  // extern "C"
