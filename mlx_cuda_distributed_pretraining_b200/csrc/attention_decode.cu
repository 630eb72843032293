// Decode-time attention over a KV cache, and the per-token cache append.
//
// attn_decode computes what FlashAttention._flash_attention (arch/flash_attention.py:97-156 of the reference) computes
// for the LAST query row of a causal sequence: o = softmax(q K^T * scale) V over the row's lens[b] cached keys, with
// q-head h reading kv-head h / (H/Hk).  One new query per sequence makes this memory-bound, so the kernel is built
// around reading every K/V byte exactly once:
//
//   grid (chunk, kv head, batch row), 128 threads.  A CTA owns keys [256 c, min(256 (c + 1), lens[b])) of one kv head
//   and ALL G = H/Hk query heads that share it.  Chunk boundaries depend on lens[b] alone (not on B, s_max or the SM
//   count), and CTAs past the row's last chunk exit at once.
//   Thread 0 streams the chunk through a 4-stage ring of 32-key K and V tiles (TMA boxes {D, 1, 32, 1} over the
//   [B, s_max, Hk, D] cache, one mbarrier per stage).  The last tile of a chunk is anchored at its end (rows
//   [end - 32, end)), so no key at or beyond lens[b] is ever read; the rows it re-reads from the previous chunk (or
//   the zero rows TMA fills in below position 0) are masked out of the softmax.
//   Per tile: scores (D/8 lanes per key, fp32 dot products, shuffle-reduced), an online softmax per query head (one
//   warp per head, lane = key), then acc += p v with each thread owning (head, 8 columns) x (a fixed subset of keys).
//   A chunk's fp32 partial (m, l, acc) goes to the workspace; attn_decode_combine_kernel merges a row's chunks in
//   chunk order.  Rows with a single chunk are finished by the first kernel.
//
// Every reduction has a fixed order that depends only on the row's own data, so a row's output is bit-identical
// whether it runs alone or inside any batch, and from launch to launch.
//
// Sliding window (attn_decode_window): the query at position len - 1 sees keys kv0 = max(0, len - 1 - W) .. len - 1.
// Chunk boundaries stay at multiples of 256 from position 0; chunks that end at or below kv0 exit at once, the first
// live chunk starts at the 32-key tile holding kv0 and masks the keys below it, and the combine merges the live chunks
// only.  A row's result still depends on lens[b] and W alone.  Without a window W = s_max, so kv0 = 0 and the
// arithmetic is the unwindowed kernel's.
//
// ALiBi (attn_decode_alibi, ALIBI = true): the query at position len - 1 adds m_h log2e (k - (len - 1)) to the score
// of key k, with query head h's slope m_h = slopes[h].  The slopes (times log2e) of the CTA's G heads are read once
// into the reduction buffer, which is free until the key subsets merge.  Per tile each lane converts its key's distance
// start + lane - (len - 1) once for all G heads, and the online-softmax step adds slope * distance to the score; keys
// below the tile start or the window stay -inf.  With zero slopes the scores are the window kernel's.
#include <type_traits>

#include "common.cuh"
#include "host.h"

namespace b200 {

namespace {

constexpr int DEC_CHUNK = 256;    // keys per split
constexpr int DEC_TILE = 32;      // keys per TMA box / ring stage (= warp size: one lane per key in the softmax)
constexpr int DEC_STAGES = 4;
constexpr int DEC_THREADS = 128;
constexpr int DEC_MAX_ITEMS = 2;  // (head, 8-column slice) accumulators per thread: G * D <= 2048
constexpr float kLog2e = 1.4426950408889634f;

__device__ __forceinline__ void ld8(const __nv_bfloat16* p, float* f) {
  const uint4 a = *reinterpret_cast<const uint4*>(p);
  const float2 v0 = unpack_bf16x2(a.x), v1 = unpack_bf16x2(a.y), v2 = unpack_bf16x2(a.z), v3 = unpack_bf16x2(a.w);
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

// Shared-memory layout (offsets from a 128-byte aligned base): the K/V ring, then q [G][D] f32 (pre-scaled by
// scale * log2 e), scores / probabilities [G][32] f32, per-head alpha, m, l, and the cross-thread reduction buffer.
struct DecSmem {
  int ring, q, s, ml, red, bar, total;
  __host__ __device__ DecSmem(int D, int elem, int G) {
    ring = 0;
    q = ring + DEC_STAGES * 2 * DEC_TILE * D * elem;
    s = q + G * D * 4;
    ml = s + G * DEC_TILE * 4;
    red = ml + ((3 * G + 3) & ~3) * 4;
    bar = red + DEC_THREADS * 8 * 4;
    total = bar + DEC_STAGES * 8 + 128;  // + alignment slack of the dynamic base
  }
};

struct DecArgs {
  const void* q;      // [B, H, D]
  void* o;            // [B, H, D]
  float* lse;         // [B, H] or null
  const int* lens;    // [B]
  float* part_acc;    // [B, H, max_chunks, D]
  float* part_ml;     // [B, H, max_chunks, 2]
  int H, G, s_max, max_chunks;
  float scale_log2;   // scale * log2 e
  int window;         // keys len - 1 - window .. len - 1 are visible; s_max without a window
  const float* slopes;  // ALIBI: [H] fp32 per-query-head slopes
  union {  // the struct's size and every field's offset stay those of the kernels without BEAM
    int ring_m;                   // RING: max_kv_size M (s_max is the ring's C slots, window has no s_max bound)
    const struct BeamMaps* beam;  // BEAM: the tails' tensor maps and the tables, in global memory
  };
};

// MULTI (attn_decode_multi): n_q new queries per row, query i of row b at position start[b] + i and valid iff
// i < lens[b] - start[b] (lens is each row's end).  q / o are [B, n_q, H, D], lse [B, H, n_q], and the partials are
// those of B * n_q decode rows.  A separate type, so the kernels without MULTI keep their parameters.
struct DecMultiArgs : DecArgs {
  const int* start;  // [B]
  int n_q;
};
// MULTI: queries per CTA, so that their (query, q head) pairs fit the accumulators: pack * G * D <= 2048
__host__ __device__ __forceinline__ int multi_pack(int G, int D) {
  return max(1, DEC_MAX_ITEMS * DEC_THREADS * 8 / (G * D));
}
template <bool MULTI>
using DecArgsT = std::conditional_t<MULTI, DecMultiArgs, DecArgs>;

// kv0: the first cached key the row's query sees
__device__ __forceinline__ int first_visible_key(const DecArgs& p, int len) { return max(0, len - 1 - p.window); }

// RING: the slots the query at position n = end - 1 sees, in ascending slot order: [lo[i], hi[i]) holds positions
// slot + off[i] (empty ranges have lo == hi).  Range 0 is the sinks max(0, n - W) .. min(3, n); the arc
// A = max(4, n - min(M - 5, W)) .. n is range 1 when its slots do not wrap, else ranges 1 = [4, slot(n)] and
// 2 = [slot(A), C).
struct RingRow {
  int lo[3], hi[3], off[3];
};
__device__ __forceinline__ RingRow ring_row(int end, int M, int C, int W) {
  RingRow r;
#pragma unroll
  for (int i = 0; i < 3; ++i) r.lo[i] = r.hi[i] = r.off[i] = 0;
  const int n = end - 1;
  if (max(0, n - W) < min(RING_SINKS, end)) {
    r.lo[0] = max(0, n - W);
    r.hi[0] = min(RING_SINKS, end);
  }
  const int A = max(RING_SINKS, n - min(M - 5, W));
  if (A <= n) {
    const int sa = ring_slot(A, C), sn = ring_slot(n, C);
    r.lo[1] = sa <= sn ? sa : RING_SINKS;
    r.hi[1] = sn + 1;
    r.off[1] = n - sn;
    if (sa > sn) {
      r.lo[2] = sa;
      r.hi[2] = C;
      r.off[2] = A - sa;
    }
  }
  return r;
}
// the hull [lo, hi) of the visible slots in the 256-slot chunk from c0; false when it holds none
__device__ __forceinline__ bool ring_chunk(const RingRow& r, int c0, int& lo, int& hi) {
  lo = INT_MAX;
  hi = INT_MIN;
#pragma unroll
  for (int i = 0; i < 3; ++i) {
    const int l = max(r.lo[i], c0), h = min(r.hi[i], c0 + DEC_CHUNK);
    if (l < h) {
      lo = min(lo, l);
      hi = max(hi, h);
    }
  }
  return lo < hi;
}
// chunks holding a visible slot (the ranges are ascending and disjoint)
__device__ __forceinline__ int ring_live_chunks(const RingRow& r) {
  int n = 0, last = -1;
#pragma unroll
  for (int i = 0; i < 3; ++i) {
    if (r.lo[i] >= r.hi[i]) continue;
    const int c_hi = (r.hi[i] - 1) / DEC_CHUNK;
    n += max(0, c_hi - max(r.lo[i] / DEC_CHUNK, last + 1) + 1);
    last = max(last, c_hi);
  }
  return n;
}
// whether slot s is visible, and its position's offset from s
__device__ __forceinline__ bool ring_visible(const RingRow& r, int s, int& off) {
  off = 0;
  bool in = false;
#pragma unroll
  for (int i = 0; i < 3; ++i)
    if (s >= r.lo[i] && s < r.hi[i]) {
      in = true;
      off = r.off[i];
    }
  return in;
}

// BEAM (attn_decode_beam): the beam rows of a group share the group's prefix cache [n_groups, s_prefix, Hk, D] below
// its fork point T0 (a multiple of DEC_CHUNK) and keep positions t >= T0 at index t - T0 of their own tail slot
// [n_slots, tail_cap, Hk, D].  A group's rows are contiguous and have the same length.
struct BeamArgs {
  const int* row_group;  // [R] the row's group
  const int* row_slot;   // [R] the row's tail slot
  const int* grp_t0;     // [n_groups] fork point
  const int* grp_row0;   // [n_groups] first row
  const int* grp_rows;   // [n_groups] live rows
  int pack;              // beams per prefix CTA: pack * G * D <= DEC_MAX_ITEMS * DEC_THREADS * 8
};
// BEAM: the tails' tensor maps and the tables, written by the host to the start of the workspace so that the kernel
// keeps attn_decode_kernel's parameters; BEAM_HDR bytes, the partials follow
struct BeamMaps {
  CUtensorMap k_tail, v_tail;
  BeamArgs args;
};
constexpr int BEAM_HDR = 384;
static_assert(sizeof(BeamMaps) <= BEAM_HDR, "BeamMaps exceeds its workspace header");

// ALIBI: at least 4 CTAs per SM (<= 128 registers); left to itself ptxas keeps the ALiBi kernels at 64 registers and
// spills the bf16 D = 32 / 128 ones.  RING takes the same bound (without it the ring kernels spill too).
// ALIBI = RING = false keeps the plain bound (0 = none).
//
// RING (attn_decode_ring): s_max is the ring's C slots and lens[b] the positions the row holds.  The chunks are
// 256-slot chunks of the ring; one holding no visible slot (ring_row) exits at once, and one holding some reads the
// hull of its visible slots, from the 32-slot tile holding the first, with the slots outside the ranges masked.  The
// ALiBi distance is the slot's position (slot + its range's offset) minus the query's.
//
// BEAM: blockIdx.z is a beam row and the chunks are the unwindowed kernel's.  A tail chunk (c0 >= T0) reads the row's
// slot at index pos - T0 (an end-anchored tile below T0 reads TMA's zero fill, masked as below position 0).  A prefix
// chunk is run by the first row of each pack of `pack` consecutive rows of the group only: it reads the prefix tile
// once for the nb <= pack rows, whose nb * G query heads act as the CTA's heads (head e = row e / G, q head e % G).
//
// MULTI: blockIdx.z is (row, pack of multi_pack(G, D) consecutive queries); the CTA's heads are the pack's nb valid
// queries' G q heads (head e = query qi0 + e / G, q head e % G).  The chunks are the unwindowed kernel's, the CTA reads
// the hull from the tile holding its first query's kv0 to the chunk's end as seen by the row's last valid query
// (min(end, c0 + 256), so no position at or past end is read), and each head masks the keys outside its own query's
// view max(0, pos - W) .. pos.  A tile may hold no visible key for some head: its max stays -inf, and the softmax
// step then adds nothing.  A query writes only for the chunks its own view touches, finishing itself when that is one.
template <typename T, int D, bool ALIBI = false, bool RING = false, bool BEAM = false, bool MULTI = false>
__global__ void __launch_bounds__(DEC_THREADS, ALIBI || RING || BEAM || MULTI ? 4 : 0)
attn_decode_kernel(const __grid_constant__ CUtensorMap tmK, const __grid_constant__ CUtensorMap tmV,
                   const DecArgsT<MULTI> p) {
  const BeamMaps* bm = BEAM ? p.beam : nullptr;  // BEAM: tmK / tmV are the prefix caches
  const BeamArgs* bp = BEAM ? &bm->args : nullptr;
  constexpr int L = D / 8;                        // 8-column slices per row
  constexpr int TILE_ELEMS = DEC_TILE * D;
  constexpr int TILE_BYTES = TILE_ELEMS * (int)sizeof(T);
  int n_q = 1, qp = 1, n_packs = 1;  // MULTI: queries per row, per CTA, and query packs per row
  if constexpr (MULTI) {
    n_q = p.n_q;
    qp = multi_pack(p.G, D);
    n_packs = (n_q + qp - 1) / qp;
  }
  const int c = blockIdx.x, hk = blockIdx.y, b = MULTI ? blockIdx.z / n_packs : blockIdx.z;
  const int c0 = c * DEC_CHUNK;
  int len, kv0, lo, end, n_chunks;
  RingRow rr;
  int nb = 1, grp = 0, t0 = 0, slot = 0;  // BEAM: rows in this CTA, the row's group, fork point and tail slot
  bool tail = false;
  int qi0 = 0, qpos0 = 0;  // MULTI: the CTA's first query and its position
  if constexpr (MULTI) {
    len = min(p.lens[b], p.s_max);
    const int s0 = p.start[b];
    qi0 = blockIdx.z % n_packs * qp;
    if (s0 < 0 || qi0 >= min(len - s0, n_q)) return;
    nb = min(qp, min(len - s0, n_q) - qi0);
    qpos0 = s0 + qi0;
    kv0 = max(0, qpos0 - p.window);
    if (c0 > qpos0 + nb - 1 || c0 + DEC_CHUNK <= kv0) return;
    lo = max(c0, kv0 & ~(DEC_TILE - 1));
    end = min(len, c0 + DEC_CHUNK);
    n_chunks = 0;  // per query, below
  } else if constexpr (RING) {
    len = p.lens[b];
    if (len < 1) return;
    rr = ring_row(len, p.ring_m, p.s_max, p.window);
    if (!ring_chunk(rr, c0, kv0, end)) return;
    lo = kv0 & ~(DEC_TILE - 1);
    n_chunks = ring_live_chunks(rr);
  } else {
    len = min(p.lens[b], p.s_max);
    kv0 = first_visible_key(p, len);
    if (c0 >= len || c0 + DEC_CHUNK <= kv0) return;
    if constexpr (BEAM) {
      grp = bp->row_group[b];
      t0 = bp->grp_t0[grp];
      slot = bp->row_slot[b];
      tail = c0 >= t0;
      if (!tail) {
        const int j = b - bp->grp_row0[grp];
        if (j % bp->pack != 0) return;
        nb = min(bp->pack, bp->grp_rows[grp] - j);
      }
    }
    lo = max(c0, kv0 & ~(DEC_TILE - 1));  // the first live chunk starts at the tile holding kv0
    end = min(len, c0 + DEC_CHUNK);
    n_chunks = (len + DEC_CHUNK - 1) / DEC_CHUNK - kv0 / DEC_CHUNK;  // live chunks of the row
  }
  const int n_tiles = (end - lo + DEC_TILE - 1) / DEC_TILE;
  const int G = BEAM || MULTI ? nb * p.G : p.G;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;

  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 127) & ~uintptr_t(127));
  const DecSmem lay(D, (int)sizeof(T), G);
  T* ring = reinterpret_cast<T*>(smem + lay.ring);  // stage st: K at 2 st, V at 2 st + 1 (TILE_ELEMS each)
  float* sq = reinterpret_cast<float*>(smem + lay.q);
  float* ss = reinterpret_cast<float*>(smem + lay.s);
  float* salpha = reinterpret_cast<float*>(smem + lay.ml);
  float* sm = salpha + G;
  float* sl = sm + G;
  float* sred = reinterpret_cast<float*>(smem + lay.red);
  const uint32_t bar0 = smem_u32(smem + lay.bar);

  auto tile_start = [&](int j) { return min(lo + j * DEC_TILE, end - DEC_TILE); };
  auto issue = [&](int j) {
    const int st = j % DEC_STAGES;
    const uint32_t bar = bar0 + 8 * st;
    mbar_arrive_expect_tx(bar, 2 * TILE_BYTES);
    if (BEAM && tail) {
      tma_load_4d(smem_u32(ring + (2 * st) * TILE_ELEMS), &bm->k_tail, bar, 0, hk, tile_start(j) - t0, slot);
      tma_load_4d(smem_u32(ring + (2 * st + 1) * TILE_ELEMS), &bm->v_tail, bar, 0, hk, tile_start(j) - t0, slot);
    } else {
      tma_load_4d(smem_u32(ring + (2 * st) * TILE_ELEMS), &tmK, bar, 0, hk, tile_start(j), BEAM ? grp : b);
      tma_load_4d(smem_u32(ring + (2 * st + 1) * TILE_ELEMS), &tmV, bar, 0, hk, tile_start(j), BEAM ? grp : b);
    }
  };

  if (tid == 0) {
    for (int s = 0; s < DEC_STAGES; ++s) mbar_init(bar0 + 8 * s, 1);
    fence_mbar_init();
    if constexpr (BEAM) {  // the tail maps were written through the generic proxy, possibly over older maps
      asm volatile("fence.proxy.tensormap::generic.acquire.gpu [%0], 128;" ::"l"(&bm->k_tail) : "memory");
      asm volatile("fence.proxy.tensormap::generic.acquire.gpu [%0], 128;" ::"l"(&bm->v_tail) : "memory");
    }
    tma_prefetch_desc(BEAM && tail ? &bm->k_tail : &tmK);
    tma_prefetch_desc(BEAM && tail ? &bm->v_tail : &tmV);
  }
  __syncthreads();
  if (tid == 0)
    for (int j = 0; j < min(n_tiles, DEC_STAGES); ++j) issue(j);

  if constexpr (BEAM || MULTI) {
    // head e of the CTA is q head hk * p.G + e % p.G of row b + e / p.G (MULTI: of query qi0 + e / p.G of row b)
    for (int i = tid; i < G * L; i += DEC_THREADS) {
      const int e = i / L;
      const long long row = MULTI ? (long long)b * n_q + qi0 + e / p.G : b + e / p.G;
      float f[8];
      ld8(reinterpret_cast<const T*>(p.q) + (row * p.H + hk * p.G + e % p.G) * D + (i % L) * 8, f);
#pragma unroll
      for (int x = 0; x < 8; ++x) sq[i * 8 + x] = f[x] * p.scale_log2;
    }
  } else {
    // the G query heads of this kv head are contiguous in [B, H, D]
    const T* qb = reinterpret_cast<const T*>(p.q) + ((long long)b * p.H + (long long)hk * G) * D;
    for (int i = tid; i < G * L; i += DEC_THREADS) {
      float f[8];
      ld8(qb + i * 8, f);
#pragma unroll
      for (int e = 0; e < 8; ++e) sq[i * 8 + e] = f[e] * p.scale_log2;
    }
  }
  for (int g = tid; g < G; g += DEC_THREADS) {
    sm[g] = -INFINITY;
    sl[g] = 0.f;
    if constexpr (ALIBI && !BEAM && !MULTI) sred[g] = __ldg(p.slopes + hk * G + g) * kLog2e;  // G <= DEC_THREADS * 8
    if constexpr (ALIBI && (BEAM || MULTI)) sred[g] = __ldg(p.slopes + hk * p.G + g % p.G) * kLog2e;
  }

  // accumulator ownership: item = (head g, slice) with g = item / L; keys my_ks, my_ks + ks_n, ... of every tile
  const int items = G * L;
  const int ks_n = items <= DEC_THREADS ? DEC_THREADS / items : 1;
  int my_item[DEC_MAX_ITEMS], my_ks;
  if (items <= DEC_THREADS) {
    my_ks = tid / items;
    my_item[0] = my_ks < ks_n ? tid % items : -1;
    my_item[1] = -1;
  } else {
    my_ks = 0;
    my_item[0] = tid;
    my_item[1] = tid + DEC_THREADS < items ? tid + DEC_THREADS : -1;
  }
  float acc[DEC_MAX_ITEMS][8];
#pragma unroll
  for (int r = 0; r < DEC_MAX_ITEMS; ++r)
#pragma unroll
    for (int e = 0; e < 8; ++e) acc[r][e] = 0.f;
  __syncthreads();

  for (int j = 0; j < n_tiles; ++j) {
    const int st = j % DEC_STAGES;
    mbar_wait(bar0 + 8 * st, (j / DEC_STAGES) & 1);
    const T* tK = ring + (2 * st) * TILE_ELEMS;
    const T* tV = ring + (2 * st + 1) * TILE_ELEMS;
    const int start = tile_start(j);
    // rows of an end-anchored tile below lo + 32 j belong to earlier tiles; keys below kv0 are outside the window
    const int first_valid = max(lo + j * DEC_TILE, kv0);

    // scores: L consecutive lanes per key, 8 columns each
    {
      const int kl = tid % L;
      for (int key = tid / L; key < DEC_TILE; key += DEC_THREADS / L) {
        float kf[8];
        ld8(tK + key * D + kl * 8, kf);
        bool valid = start + key >= first_valid;
        if constexpr (RING) {
          int off;
          valid = valid && ring_visible(rr, start + key, off);
        }
        for (int g = 0; g < G; ++g) {
          const float4 qa = *reinterpret_cast<const float4*>(sq + g * D + kl * 8);
          const float4 qc = *reinterpret_cast<const float4*>(sq + g * D + kl * 8 + 4);
          float d = qa.x * kf[0];
          d = fmaf(qa.y, kf[1], d);
          d = fmaf(qa.z, kf[2], d);
          d = fmaf(qa.w, kf[3], d);
          d = fmaf(qc.x, kf[4], d);
          d = fmaf(qc.y, kf[5], d);
          d = fmaf(qc.z, kf[6], d);
          d = fmaf(qc.w, kf[7], d);
#pragma unroll
          for (int off = L / 2; off > 0; off >>= 1) d += __shfl_xor_sync(0xffffffffu, d, off);
          if constexpr (MULTI) {  // the view of head g's query at position qpos
            const int qpos = qpos0 + g / p.G;
            valid = start + key <= qpos && start + key >= max(lo + j * DEC_TILE, qpos - p.window);
          }
          if (kl == 0) ss[g * DEC_TILE + key] = valid ? d : -INFINITY;
        }
      }
    }
    __syncthreads();

    // online softmax (log2 domain): one warp per head, one lane per key; every tile holds at least one valid key
    // (kv0 < end, and kv0 lies in the first tile), except under MULTI.  ALIBI: kd = this lane's key distance,
    // converted once per tile (MULTI: per head, from the head's query)
    float kd = 0.f;
    if constexpr (ALIBI && !MULTI) {
      int off = 0;
      if constexpr (RING) ring_visible(rr, start + lane, off);
      kd = (float)(start + lane + off - (len - 1));
    }
    for (int g = warp; g < G; g += DEC_THREADS / 32) {
      float x = ss[g * DEC_TILE + lane];
      if constexpr (ALIBI && MULTI) kd = (float)(start + lane - (qpos0 + g / p.G));
      if constexpr (ALIBI) x = x + sred[g] * kd;
      const float m_old = sm[g];
      const float m_new = fmaxf(m_old, warp_max(x));
      const float m_use = MULTI && m_new == -INFINITY ? 0.f : m_new;  // no visible key yet: p = 0, alpha = 0
      const float pe = exp2f(x - m_use);
      const float sum = warp_sum(pe);
      ss[g * DEC_TILE + lane] = pe;
      __syncwarp();
      if (lane == 0) {
        const float alpha = exp2f(m_old - m_use);
        salpha[g] = alpha;
        sl[g] = sl[g] * alpha + sum;
        sm[g] = m_new;
      }
    }
    __syncthreads();

    // acc = acc * alpha + sum over this thread's keys of p v
#pragma unroll
    for (int r = 0; r < DEC_MAX_ITEMS; ++r) {
      if (my_item[r] < 0) continue;
      const int g = my_item[r] / L, sc = my_item[r] % L;
      const float a = salpha[g];
#pragma unroll
      for (int e = 0; e < 8; ++e) acc[r][e] *= a;
      for (int key = my_ks; key < DEC_TILE; key += ks_n) {
        const float pe = ss[g * DEC_TILE + key];
        float vf[8];
        ld8(tV + key * D + sc * 8, vf);
#pragma unroll
        for (int e = 0; e < 8; ++e) acc[r][e] = fmaf(pe, vf[e], acc[r][e]);
      }
    }
    __syncthreads();  // stage st and the score buffer are free again
    if (tid == 0 && j + DEC_STAGES < n_tiles) issue(j + DEC_STAGES);
  }

  // merge the key subsets in subset order
  if (ks_n > 1) {
    if (my_item[0] >= 0)
#pragma unroll
      for (int e = 0; e < 8; ++e) sred[(my_ks * items + my_item[0]) * 8 + e] = acc[0][e];
    __syncthreads();
    if (tid < items) {
#pragma unroll
      for (int e = 0; e < 8; ++e) acc[0][e] = sred[tid * 8 + e];
      for (int k = 1; k < ks_n; ++k)
#pragma unroll
        for (int e = 0; e < 8; ++e) acc[0][e] += sred[(k * items + tid) * 8 + e];
      my_item[0] = tid;
    } else {
      my_item[0] = -1;
    }
  }

#pragma unroll
  for (int r = 0; r < DEC_MAX_ITEMS; ++r) {
    if (my_item[r] < 0) continue;
    const int g = my_item[r] / L, sc = my_item[r] % L;
    const int h = BEAM || MULTI ? hk * p.G + g % p.G : hk * G + g;
    const int qi = qi0 + g / p.G;  // MULTI: the head's query
    const long long bh = (MULTI ? (long long)b * n_q + qi : (long long)(BEAM ? b + g / p.G : b)) * p.H + h;
    const float m = sm[g], l = sl[g];
    int nc = n_chunks;
    if constexpr (MULTI) {  // the chunks the query's view touches
      const int qpos = qpos0 + g / p.G;
      const int c_first = max(0, qpos - p.window) / DEC_CHUNK, c_last = qpos / DEC_CHUNK;
      if (c < c_first || c > c_last) continue;
      nc = c_last - c_first + 1;
    }
    if (nc == 1) {
      const float inv = 1.0f / l;
      float f[8];
#pragma unroll
      for (int e = 0; e < 8; ++e) f[e] = acc[r][e] * inv;
      st8(reinterpret_cast<T*>(p.o) + bh * D + sc * 8, f);
      if (p.lse != nullptr && sc == 0) p.lse[MULTI ? ((long long)b * p.H + h) * n_q + qi : bh] = (m + log2f(l)) / kLog2e;
    } else {
      st8(p.part_acc + (bh * p.max_chunks + c) * D + sc * 8, acc[r]);
      if (sc == 0) {
        p.part_ml[(bh * p.max_chunks + c) * 2] = m;
        p.part_ml[(bh * p.max_chunks + c) * 2 + 1] = l;
      }
    }
  }
}

// o = sum_c exp2(m_c - M) acc_c / sum_c exp2(m_c - M) l_c over a row's live chunks, in chunk order; one thread per
// column
// (RING: over the chunks ring_chunk finds live, the others skipped; MULTI: blockIdx.y is (row, query), a query's
// live chunks those of its own view)
template <typename T, int D, bool RING = false, bool MULTI = false>
__global__ void __launch_bounds__(D)
attn_decode_combine_kernel(const DecArgsT<MULTI> p) {
  const int h = blockIdx.x, b = blockIdx.y, d = threadIdx.x;
  int c_lo, n;
  RingRow rr;
  long long lse_i = 0;  // MULTI: the query's LSE in [B, H, n_q]
  if constexpr (MULTI) {
    const int rb = b / p.n_q, qi = b % p.n_q;
    const int s0 = p.start[rb];
    if (s0 < 0 || qi >= min(p.lens[rb], p.s_max) - s0) return;
    const int len = s0 + qi + 1;
    c_lo = max(0, len - 1 - p.window) / DEC_CHUNK;
    n = (len + DEC_CHUNK - 1) / DEC_CHUNK;
    if (n - c_lo <= 1) return;  // finished by attn_decode_kernel
    lse_i = ((long long)rb * p.H + h) * p.n_q + qi;
  } else if constexpr (RING) {
    if (p.lens[b] < 1) return;
    rr = ring_row(p.lens[b], p.ring_m, p.s_max, p.window);
    if (ring_live_chunks(rr) <= 1) return;  // finished by attn_decode_kernel
    c_lo = 0;
    n = p.max_chunks;
  } else {
    const int len = min(p.lens[b], p.s_max);
    c_lo = first_visible_key(p, len) / DEC_CHUNK;
    n = (len + DEC_CHUNK - 1) / DEC_CHUNK;
    if (n - c_lo <= 1) return;  // finished by attn_decode_kernel
  }
  auto live = [&](int c) {
    int lo, hi;
    return !RING || ring_chunk(rr, c * DEC_CHUNK, lo, hi);
  };
  const long long bh = (long long)b * p.H + h;
  const float* ml = p.part_ml + bh * p.max_chunks * 2;
  const float* pa = p.part_acc + bh * p.max_chunks * D + d;
  float M = -INFINITY;
  for (int c = c_lo; c < n; ++c)
    if (live(c)) M = fmaxf(M, ml[2 * c]);
  float l = 0.f, acc = 0.f;
  for (int c = c_lo; c < n; ++c) {
    if (!live(c)) continue;
    const float w = exp2f(ml[2 * c] - M);
    l = fmaf(ml[2 * c + 1], w, l);
    acc = fmaf(pa[(long long)c * D], w, acc);
  }
  const float out = acc / l;
  if constexpr (sizeof(T) == 2) reinterpret_cast<__nv_bfloat16*>(p.o)[bh * D + d] = __float2bfloat16(out);
  else reinterpret_cast<float*>(p.o)[bh * D + d] = out;
  if (p.lse != nullptr && d == 0) p.lse[MULTI ? lse_i : bh] = (M + log2f(l)) / kLog2e;
}

template <typename T, int D, bool ALIBI = false, bool RING = false>
int launch_decode(const CUtensorMap& tmK, const CUtensorMap& tmV, const DecArgs& a, int B, int Hk,
                  cudaStream_t stream) {
  auto kern = attn_decode_kernel<T, D, ALIBI, RING>;
  const DecSmem lay(D, (int)sizeof(T), a.G);
  static int attr_bytes = 0;
  if (lay.total > 48 * 1024 && lay.total > attr_bytes) {
    B200_CHECK_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, lay.total));
    attr_bytes = lay.total;
  }
  kern<<<dim3(a.max_chunks, Hk, B), DEC_THREADS, lay.total, stream>>>(tmK, tmV, a);
  B200_CHECK_LAUNCH();
  if (a.max_chunks > 1) {
    attn_decode_combine_kernel<T, D, RING><<<dim3(a.H, B), D, 0, stream>>>(a);
    B200_CHECK_LAUNCH();
  }
  return B200_OK;
}

template <typename T, bool ALIBI = false>
int launch_decode_d(int D, const CUtensorMap& tmK, const CUtensorMap& tmV, const DecArgs& a, int B, int Hk,
                    cudaStream_t stream) {
  switch (D) {
    case 16: return launch_decode<T, 16, ALIBI>(tmK, tmV, a, B, Hk, stream);
    case 32: return launch_decode<T, 32, ALIBI>(tmK, tmV, a, B, Hk, stream);
    case 64: return launch_decode<T, 64, ALIBI>(tmK, tmV, a, B, Hk, stream);
    default: return launch_decode<T, 128, ALIBI>(tmK, tmV, a, B, Hk, stream);
  }
}

// MULTI: grid z is (row, query pack), the combine's y (row, query)
template <typename T, int D, bool ALIBI>
int launch_decode_multi(const CUtensorMap& tmK, const CUtensorMap& tmV, const DecMultiArgs& a, int B, int Hk,
                        cudaStream_t stream) {
  auto kern = attn_decode_kernel<T, D, ALIBI, false, false, true>;
  const int qp = min(multi_pack(a.G, D), a.n_q);
  const DecSmem lay(D, (int)sizeof(T), a.G * qp);
  static int attr_bytes = 0;
  if (lay.total > 48 * 1024 && lay.total > attr_bytes) {
    B200_CHECK_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, lay.total));
    attr_bytes = lay.total;
  }
  kern<<<dim3(a.max_chunks, Hk, B * ((a.n_q + qp - 1) / qp)), DEC_THREADS, lay.total, stream>>>(tmK, tmV, a);
  B200_CHECK_LAUNCH();
  if (a.max_chunks > 1) {
    attn_decode_combine_kernel<T, D, false, true><<<dim3(a.H, B * a.n_q), D, 0, stream>>>(a);
    B200_CHECK_LAUNCH();
  }
  return B200_OK;
}

template <typename T, bool ALIBI>
int launch_decode_multi_d(int D, const CUtensorMap& tmK, const CUtensorMap& tmV, const DecMultiArgs& a, int B, int Hk,
                          cudaStream_t stream) {
  switch (D) {
    case 16: return launch_decode_multi<T, 16, ALIBI>(tmK, tmV, a, B, Hk, stream);
    case 32: return launch_decode_multi<T, 32, ALIBI>(tmK, tmV, a, B, Hk, stream);
    case 64: return launch_decode_multi<T, 64, ALIBI>(tmK, tmV, a, B, Hk, stream);
    default: return launch_decode_multi<T, 128, ALIBI>(tmK, tmV, a, B, Hk, stream);
  }
}

template <typename T, int D, bool ALIBI>
int launch_decode_beam(const CUtensorMap* tm, const DecArgs& a, int pack, int R, int Hk, cudaStream_t stream) {
  auto kern = attn_decode_kernel<T, D, ALIBI, false, true>;
  const DecSmem lay(D, (int)sizeof(T), a.G * pack);
  static int attr_bytes = 0;
  if (lay.total > 48 * 1024 && lay.total > attr_bytes) {
    B200_CHECK_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, lay.total));
    attr_bytes = lay.total;
  }
  kern<<<dim3(a.max_chunks, Hk, R), DEC_THREADS, lay.total, stream>>>(tm[0], tm[1], a);
  B200_CHECK_LAUNCH();
  if (a.max_chunks > 1) {
    attn_decode_combine_kernel<T, D><<<dim3(a.H, R), D, 0, stream>>>(a);
    B200_CHECK_LAUNCH();
  }
  return B200_OK;
}

template <typename T, bool ALIBI>
int launch_decode_beam_d(int D, const CUtensorMap* tm, const DecArgs& a, int bp, int R, int Hk,
                         cudaStream_t stream) {
  switch (D) {
    case 16: return launch_decode_beam<T, 16, ALIBI>(tm, a, bp, R, Hk, stream);
    case 32: return launch_decode_beam<T, 32, ALIBI>(tm, a, bp, R, Hk, stream);
    case 64: return launch_decode_beam<T, 64, ALIBI>(tm, a, bp, R, Hk, stream);
    default: return launch_decode_beam<T, 128, ALIBI>(tm, a, bp, R, Hk, stream);
  }
}

// b200_rope's interleaved-pair rotation of one 8-column vector, c / sn = the vector's 4 table entries
__device__ __forceinline__ void rope_pairs8(const float* xv, const float* cos4, const float* sin4, float* o) {
  const float4 c = *reinterpret_cast<const float4*>(cos4);
  const float4 sn = *reinterpret_cast<const float4*>(sin4);
  o[0] = xv[0] * c.x - xv[1] * sn.x;  o[1] = xv[0] * sn.x + xv[1] * c.x;
  o[2] = xv[2] * c.y - xv[3] * sn.y;  o[3] = xv[2] * sn.y + xv[3] * c.y;
  o[4] = xv[4] * c.z - xv[5] * sn.z;  o[5] = xv[4] * sn.z + xv[5] * c.z;
  o[6] = xv[6] * c.w - xv[7] * sn.w;  o[7] = xv[6] * sn.w + xv[7] * c.w;
}

// One thread per 8-column vector: q heads (rotated in place, RoPE only), then k heads (rotated when RoPE is on) and
// v heads, both written to cache row pos = lens[b] - 1.  The rotation is b200_rope's arithmetic, statement for
// statement, so a token rotated here equals the same token rotated by the prefill.
// RING (kv_append_ring): s_max is the ring's C slots; the cache row is slot(pos), pos itself unbounded, and a row
// with live[b] == 0 (live non-null) is skipped whole.
// BEAM (kv_append_beam): the caches are the tails [n_slots, s_max = tail_cap, Hk, D]; row b writes index pos - T0 of
// its slot, T0 its group's fork point, and `live` holds the tables [row_group (B) | row_slot (B) | grp_t0].
template <typename T, bool RING = false, bool BEAM = false>
__global__ void __launch_bounds__(256)
kv_append_kernel(T* __restrict__ q, const T* __restrict__ k, const T* __restrict__ v, T* __restrict__ k_cache,
                 T* __restrict__ v_cache, const int* __restrict__ lens, const float* __restrict__ cos_t,
                 const float* __restrict__ sin_t, long long nvec, int s_max, int H, int Hk, int D,
                 const int* __restrict__ live = nullptr) {
  const int L = D / 8;
  const int q_heads = cos_t != nullptr ? H : 0;
  const int heads = q_heads + 2 * Hk;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < nvec; i += (long long)gridDim.x * blockDim.x) {
    const int dv = (int)(i % L);
    const int hh = (int)(i / L % heads);
    const int b = (int)(i / L / heads);
    const int pos = lens[b] - 1;
    int row = pos;  // the cache row
    int cb = b;     // the cache's batch index
    if constexpr (RING) {
      if (pos < 0 || (live != nullptr && live[b] == 0)) continue;
      row = ring_slot(pos, s_max);
    } else if constexpr (BEAM) {
      const int R = (int)(nvec / L / heads);  // live: the tables [row_group (R) | row_slot (R) | grp_t0]
      row = pos - live[2 * R + live[b]];
      cb = live[R + b];
      if (row < 0 || row >= s_max) continue;
    } else {
      if (pos < 0 || pos >= s_max) continue;  // outside the documented 1 <= lens[b] <= s_max: write nothing
    }
    const T* src;
    T* dst;
    bool rotate = cos_t != nullptr;
    if (hh < q_heads) {
      src = dst = q + ((long long)b * H + hh) * D + dv * 8;
    } else if (hh < q_heads + Hk) {
      const int h = hh - q_heads;
      src = k + ((long long)b * Hk + h) * D + dv * 8;
      dst = k_cache + (((long long)cb * s_max + row) * Hk + h) * D + dv * 8;
    } else {
      const int h = hh - q_heads - Hk;
      src = v + ((long long)b * Hk + h) * D + dv * 8;
      dst = v_cache + (((long long)cb * s_max + row) * Hk + h) * D + dv * 8;
      rotate = false;
    }
    float xv[8], o[8];
    ld8(src, xv);
    if (rotate) {
      rope_pairs8(xv, cos_t + (long long)pos * (D / 2) + dv * 4, sin_t + (long long)pos * (D / 2) + dv * 4, o);
      st8(dst, o);
    } else {
      st8(dst, xv);
    }
  }
}

// kv_append_kernel for the half-split layout: one thread per 8-column slice pair (columns [8 dv, 8 dv + 8) and the
// same D/2 later) of a q, k or v head.  q and k are rotated by rope_half8, b200_rope_half's own rotation.
template <typename T, bool RING = false, bool BEAM = false>
__global__ void __launch_bounds__(256)
kv_append_half_kernel(T* __restrict__ q, const T* __restrict__ k, const T* __restrict__ v, T* __restrict__ k_cache,
                      T* __restrict__ v_cache, const int* __restrict__ lens, const float* __restrict__ cos_t,
                      const float* __restrict__ sin_t, long long nslice, int s_max, int H, int Hk, int D,
                      const int* __restrict__ live = nullptr) {
  const int L = D / 16;
  const int heads = H + 2 * Hk;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < nslice; i += (long long)gridDim.x * blockDim.x) {
    const int dv = (int)(i % L);
    const int hh = (int)(i / L % heads);
    const int b = (int)(i / L / heads);
    const int pos = lens[b] - 1;
    int row = pos;  // the cache row
    int cb = b;     // the cache's batch index
    if constexpr (RING) {
      if (pos < 0 || (live != nullptr && live[b] == 0)) continue;
      row = ring_slot(pos, s_max);
    } else if constexpr (BEAM) {
      const int R = (int)(nslice / L / heads);  // live: the tables [row_group (R) | row_slot (R) | grp_t0]
      row = pos - live[2 * R + live[b]];
      cb = live[R + b];
      if (row < 0 || row >= s_max) continue;
    } else {
      if (pos < 0 || pos >= s_max) continue;  // outside the documented 1 <= lens[b] <= s_max: write nothing
    }
    const T* src;
    T* dst;
    bool rotate = true;
    if (hh < H) {
      src = dst = q + ((long long)b * H + hh) * D + dv * 8;
    } else if (hh < H + Hk) {
      const int h = hh - H;
      src = k + ((long long)b * Hk + h) * D + dv * 8;
      dst = k_cache + (((long long)cb * s_max + row) * Hk + h) * D + dv * 8;
    } else {
      const int h = hh - H - Hk;
      src = v + ((long long)b * Hk + h) * D + dv * 8;
      dst = v_cache + (((long long)cb * s_max + row) * Hk + h) * D + dv * 8;
      rotate = false;
    }
    float xl[8], xh[8];
    ld8(src, xl);
    ld8(src + D / 2, xh);
    if (rotate) {
      float c[8], sn[8], ol[8], oh[8];
      ld8(cos_t + (long long)pos * (D / 2) + dv * 8, c);
      ld8(sin_t + (long long)pos * (D / 2) + dv * 8, sn);
      rope_half8(xl, xh, c, sn, ol, oh);
      st8(dst, ol);
      st8(dst + D / 2, oh);
    } else {
      st8(dst, xl);
      st8(dst + D / 2, xh);
    }
  }
}

// Copy-on-fork: copies[3 i .. 3 i + 2] = (src slot, dst slot, n) copies tail indices [0, n) of slot src to slot dst
// in each of the n_bufs tails bufs[z] [n_slots, tail_cap, row_vec x 16 bytes].  One CTA row per (copy, buffer); the
// host makes copies only from live slots to free ones, so no copy reads what another writes.
__global__ void __launch_bounds__(256)
kv_beam_fork_kernel(void* const* __restrict__ bufs, const int* __restrict__ copies, int tail_cap, int row_vec) {
  const int i = blockIdx.y;
  const int src = copies[3 * i], dst = copies[3 * i + 1], n = copies[3 * i + 2];
  uint4* base = static_cast<uint4*>(bufs[blockIdx.z]);
  const uint4* s = base + (long long)src * tail_cap * row_vec;
  uint4* d = base + (long long)dst * tail_cap * row_vec;
  const long long total = (long long)n * row_vec;
  for (long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += (long long)gridDim.x * blockDim.x)
    d[e] = s[e];
}

// ---- quantized KV cache (DESIGN §4.2.1) --------------------------------------------------------------------------
// Group-affine codes, mlx's scheme without its scale nudge: each group of g consecutive elements of a head vector is
// x ~ s q + b with n = 2^BITS - 1, mn / mx the group's extremes, s = max((mx - mn) / n, 1e-7), b = mn (a -0 minimum
// is stored as +0) and q = min(n, rint((x - b) / s)), all IEEE fp32, so |x - (s q + b)| <= s / 2.
// Codes uint8 [B, s_max, Hk, D * BITS / 8] (4 bits: element 2j in the low nibble of byte j); parameters f32
// [B, Hk, s_max, D / g, 2] holding (s, b), so a 32-key tile's parameters are one contiguous block.

// Quantizes one 8-element slice per lane.  The g / 8 slices of a group sit on w = g / 8 consecutive, w-aligned lanes,
// and every lane of the warp calls this (the min / max reductions shuffle over the full warp).  The group's lead lane
// writes the parameters when `par` is non-null.
template <int BITS>
__device__ __forceinline__ void quantize_slice(const float* x, int w, uint8_t* codes, float* par) {
  constexpr float n = (float)((1 << BITS) - 1);
  float mx = x[0], mn = x[0];
#pragma unroll
  for (int e = 1; e < 8; ++e) {
    mx = fmaxf(mx, x[e]);
    mn = fminf(mn, x[e]);
  }
  for (int off = w >> 1; off > 0; off >>= 1) {
    mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, off));
    mn = fminf(mn, __shfl_xor_sync(0xffffffffu, mn, off));
  }
  const float s = fmaxf(__fdiv_rn(mx - mn, n), 1e-7f);
  const float b = mn + 0.f;
  uint32_t q[8];
#pragma unroll
  for (int e = 0; e < 8; ++e) q[e] = (uint32_t)fminf(n, rintf(__fdiv_rn(x[e] - b, s)));
  if (codes != nullptr) {
    if constexpr (BITS == 8) {
      *reinterpret_cast<uint2*>(codes) = make_uint2(q[0] | q[1] << 8 | q[2] << 16 | q[3] << 24,
                                                    q[4] | q[5] << 8 | q[6] << 16 | q[7] << 24);
    } else {
      uint32_t u = 0;
#pragma unroll
      for (int e = 0; e < 8; ++e) u |= q[e] << (4 * e);
      *reinterpret_cast<uint32_t*>(codes) = u;
    }
    if (par != nullptr && (threadIdx.x & (w - 1)) == 0) *reinterpret_cast<float2*>(par) = make_float2(s, b);
  }
}

// the 8 codes of one slice as exact floats 0 .. n (2^23 + c built in the mantissa, then 2^23 subtracted)
template <int BITS>
__device__ __forceinline__ void codes8(const uint8_t* p, float* f) {
  if constexpr (BITS == 8) {
    const uint2 u = *reinterpret_cast<const uint2*>(p);
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      f[e] = __uint_as_float(__byte_perm(u.x, 0x4B000000u, 0x7540 + e)) - 8388608.f;
      f[4 + e] = __uint_as_float(__byte_perm(u.y, 0x4B000000u, 0x7540 + e)) - 8388608.f;
    }
  } else {
    const uint32_t u = *reinterpret_cast<const uint32_t*>(p);
#pragma unroll
    for (int e = 0; e < 8; ++e) f[e] = __uint_as_float(((u >> (4 * e)) & 0xFu) | 0x4B000000u) - 8388608.f;
  }
}

// Positions [0, n) of a [B, S, Hk, D] K and V source into codes and parameters: one thread per 8-element slice, the
// threads of a warp advancing together so that every group's lanes meet in quantize_slice.
template <typename T, int BITS>
__global__ void __launch_bounds__(256)
kv_quantize_kernel(const T* __restrict__ k, const T* __restrict__ v, uint8_t* __restrict__ kc, uint8_t* __restrict__ vc,
                   float* __restrict__ kp, float* __restrict__ vp, int n, int S, int B, int s_max, int Hk, int D,
                   int g) {
  const int L = D / 8, ng = D / g, Dc = D * BITS / 8;
  const long long per = (long long)B * n * Hk * L;  // slices of K (then as many of V)
  const long long stride = (long long)gridDim.x * blockDim.x;
  for (long long i0 = ((long long)blockIdx.x * blockDim.x + threadIdx.x) & ~31LL; i0 < 2 * per; i0 += stride) {
    const long long i = i0 + (threadIdx.x & 31);
    const bool valid = i < 2 * per;
    const int which = valid && i >= per;
    const long long r = valid ? i - which * per : 0;
    const int sl = (int)(r % L);
    const int h = (int)(r / L % Hk);
    const int pos = (int)(r / L / Hk % n);
    const int b = (int)(r / L / Hk / n);
    float x[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
    if (valid) ld8((which ? v : k) + (((long long)b * S + pos) * Hk + h) * D + sl * 8, x);
    uint8_t* codes = valid ? (which ? vc : kc) + (((long long)b * s_max + pos) * Hk + h) * Dc + sl * BITS : nullptr;
    float* par = (which ? vp : kp) + ((((long long)b * Hk + h) * s_max + pos) * ng + sl / (g / 8)) * 2;
    quantize_slice<BITS>(x, g / 8, codes, par);
  }
}

// The inverse for a chunk that attends over a quantized cache: positions [0, end[b]) of row b (and below S) of the
// codes and parameters into bf16 [B, S, Hk, D] K and V, one thread per 8-element slice.  The value is s q + b in fp32
// with the product and the sum rounded separately (no fma, so the bits are those of the format's definition), then
// rounded once to bf16.  Nothing at or past end[b] is written.
template <int BITS>
__global__ void __launch_bounds__(256)
kv_dequantize_kernel(const uint8_t* __restrict__ kc, const uint8_t* __restrict__ vc, const float* __restrict__ kp,
                     const float* __restrict__ vp, const int* __restrict__ end, __nv_bfloat16* __restrict__ k,
                     __nv_bfloat16* __restrict__ v, int S, int B, int s_max, int Hk, int D, int g) {
  const int L = D / 8, ng = D / g, Dc = D * BITS / 8;
  const long long per = (long long)B * S * Hk * L;  // slices of K (then as many of V)
  const long long stride = (long long)gridDim.x * blockDim.x;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < 2 * per; i += stride) {
    const int which = i >= per;
    const long long r = i - which * per;
    const int sl = (int)(r % L);
    const int h = (int)(r / L % Hk);
    const int pos = (int)(r / L / Hk % S);
    const int b = (int)(r / L / Hk / S);
    if (pos >= __ldg(end + b)) continue;
    float f[8];
    codes8<BITS>((which ? vc : kc) + (((long long)b * s_max + pos) * Hk + h) * Dc + sl * BITS, f);
    const float2 sb = *reinterpret_cast<const float2*>(
        (which ? vp : kp) + ((((long long)b * Hk + h) * s_max + pos) * ng + sl / (g / 8)) * 2);
    uint32_t w[4];
#pragma unroll
    for (int e = 0; e < 4; ++e)
      w[e] = pack_bf16x2(__fadd_rn(__fmul_rn(sb.x, f[2 * e]), sb.y), __fadd_rn(__fmul_rn(sb.x, f[2 * e + 1]), sb.y));
    stg128((which ? v : k) + (((long long)b * S + pos) * Hk + h) * D + sl * 8, make_uint4(w[0], w[1], w[2], w[3]));
  }
}

// kv_append for the quantized cache: one CTA per (kv head, row).  Its G query heads are rotated in place and its k
// and v heads rotated / copied exactly as kv_append_kernel (interleaved) or kv_append_half_kernel (half) do, the k and
// v results rounded to T through shared memory; then warp 0 quantizes both into position lens[b] - 1.
template <typename T, int BITS>
__global__ void __launch_bounds__(128)
kv_append_quant_kernel(T* __restrict__ q, const T* __restrict__ k, const T* __restrict__ v, uint8_t* __restrict__ kc,
                       uint8_t* __restrict__ vc, float* __restrict__ kp, float* __restrict__ vp,
                       const int* __restrict__ lens, const float* __restrict__ cos_t, const float* __restrict__ sin_t,
                       int half, int s_max, int H, int Hk, int D, int g) {
  __shared__ __align__(16) T kv[2 * 128];  // [k | v] of this head, rounded to T
  const int hk = blockIdx.x, b = blockIdx.y, G = H / Hk;
  const int pos = lens[b] - 1;
  if (pos < 0 || pos >= s_max) return;  // outside the documented 1 <= lens[b] <= s_max: write nothing
  const bool rope = cos_t != nullptr;
  const int per_head = half ? D / 16 : D / 8;  // threads per head: slice pairs (half) or 8-column vectors
  for (int i = threadIdx.x; i < (G + 2) * per_head; i += blockDim.x) {
    const int dv = i % per_head, hh = i / per_head;  // hh < G: query head hk * G + hh; G: k; G + 1: v
    if (hh < G && !rope) continue;
    const T* src;
    T* dst;
    if (hh < G) {
      src = dst = q + ((long long)b * H + hk * G + hh) * D + dv * 8;
    } else {
      src = (hh == G ? k : v) + ((long long)b * Hk + hk) * D + dv * 8;
      dst = kv + (hh - G) * D + dv * 8;
    }
    const bool rotate = rope && hh <= G;
    if (half) {
      float xl[8], xh[8];
      ld8(src, xl);
      ld8(src + D / 2, xh);
      if (rotate) {
        float c[8], sn[8], ol[8], oh[8];
        ld8(cos_t + (long long)pos * (D / 2) + dv * 8, c);
        ld8(sin_t + (long long)pos * (D / 2) + dv * 8, sn);
        rope_half8(xl, xh, c, sn, ol, oh);
        st8(dst, ol);
        st8(dst + D / 2, oh);
      } else {
        st8(dst, xl);
        st8(dst + D / 2, xh);
      }
    } else {
      float xv[8], o[8];
      ld8(src, xv);
      if (rotate) {
        rope_pairs8(xv, cos_t + (long long)pos * (D / 2) + dv * 4, sin_t + (long long)pos * (D / 2) + dv * 4, o);
        st8(dst, o);
      } else {
        st8(dst, xv);
      }
    }
  }
  __syncthreads();
  if (threadIdx.x >= 32) return;
  const int L = D / 8, lane = threadIdx.x, which = lane / L, sl = lane % L;  // 2 L <= 32 lanes hold k and v
  const bool valid = which < 2;
  float x[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
  if (valid) ld8(kv + which * D + sl * 8, x);
  const int Dc = D * BITS / 8, ng = D / g;
  uint8_t* codes = valid ? (which ? vc : kc) + (((long long)b * s_max + pos) * Hk + hk) * Dc + sl * BITS : nullptr;
  float* par = (which ? vp : kp) + ((((long long)b * Hk + hk) * s_max + pos) * ng + sl / (g / 8)) * 2;
  quantize_slice<BITS>(x, g / 8, codes, par);
}

// Parameter positions per TMA box.  A box's first coordinate is innermost ([B, Hk, s_max * ng * 2] floats) and must
// sit on a 16-byte boundary: with ng even every position does, with ng = 1 the box starts at the even position at or
// below the tile's start and spans 34 positions (the one or two past the tile are fetched, never used).
__host__ __device__ __forceinline__ int qdec_param_positions(int ng) { return ng == 1 ? DEC_TILE + 2 : DEC_TILE; }

// Shared memory of attn_decode_quant_kernel: per ring stage the K codes, V codes, K parameters and V parameters of a
// 32-key tile (each region a multiple of 128 bytes), then attn_decode_kernel's buffers plus the per-slice query sums.
struct QDecSmem {
  int kc, vc, kp, vp, stage, q, qs, s, ml, red, bar, total;
  __host__ __device__ QDecSmem(int Dc, int ng, int D, int G) {
    const int pr = (qdec_param_positions(ng) * ng * 8 + 127) & ~127;
    kc = 0;
    vc = DEC_TILE * Dc;
    kp = 2 * DEC_TILE * Dc;
    vp = kp + pr;
    stage = vp + pr;
    q = DEC_STAGES * stage;
    qs = q + G * D * 4;
    s = qs + G * (D / 8) * 4;
    ml = s + G * DEC_TILE * 4;
    red = ml + ((3 * G + 3) & ~3) * 4;
    bar = red + DEC_THREADS * 8 * 4;
    total = bar + DEC_STAGES * 8 + 128;
  }
};

// attn_decode_kernel over the quantized cache, chunking, ring, softmax, merge and output unchanged.  Per key and
// 8-column slice (inside one group with scale s, bias b) the score part is s (q . codes) + b (sum q), the slice's
// query sum computed once per CTA; the value update is acc += (p s) codes, with the p b terms summed apart and added
// to acc before the key subsets merge.  ALiBi is on when p.slopes is non-null.
template <typename T, int D, int BITS>
__global__ void __launch_bounds__(DEC_THREADS, 4)
attn_decode_quant_kernel(const __grid_constant__ CUtensorMap tmKc, const __grid_constant__ CUtensorMap tmVc,
                         const __grid_constant__ CUtensorMap tmKp, const __grid_constant__ CUtensorMap tmVp,
                         const DecArgs p, const int g) {
  constexpr int L = D / 8;
  constexpr int Dc = D * BITS / 8;
  constexpr int SB = BITS;  // code bytes per 8-column slice
  const int ng = D / g, spg = g / 8;  // groups per head vector, slices per group
  const int c = blockIdx.x, hk = blockIdx.y, b = blockIdx.z;
  const int len = min(p.lens[b], p.s_max);
  const int c0 = c * DEC_CHUNK;
  const int kv0 = first_visible_key(p, len);
  if (c0 >= len || c0 + DEC_CHUNK <= kv0) return;
  const int lo = max(c0, kv0 & ~(DEC_TILE - 1));
  const int end = min(len, c0 + DEC_CHUNK);
  const int n_tiles = (end - lo + DEC_TILE - 1) / DEC_TILE;
  const int n_chunks = (len + DEC_CHUNK - 1) / DEC_CHUNK - kv0 / DEC_CHUNK;
  const int G = p.G;
  const bool alibi = p.slopes != nullptr;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;

  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 127) & ~uintptr_t(127));
  const QDecSmem lay(Dc, ng, D, G);
  float* sq = reinterpret_cast<float*>(smem + lay.q);
  float* sqs = reinterpret_cast<float*>(smem + lay.qs);
  float* ss = reinterpret_cast<float*>(smem + lay.s);
  float* salpha = reinterpret_cast<float*>(smem + lay.ml);
  float* sm = salpha + G;
  float* sl = sm + G;
  float* sred = reinterpret_cast<float*>(smem + lay.red);
  const uint32_t bar0 = smem_u32(smem + lay.bar);
  const int tile_bytes = 2 * (DEC_TILE * Dc + qdec_param_positions(ng) * ng * 8);

  auto tile_start = [&](int j) { return min(lo + j * DEC_TILE, end - DEC_TILE); };
  auto issue = [&](int j) {
    const int st = j % DEC_STAGES;
    const uint32_t bar = bar0 + 8 * st;
    uint8_t* base = smem + st * lay.stage;
    mbar_arrive_expect_tx(bar, tile_bytes);
    tma_load_4d(smem_u32(base + lay.kc), &tmKc, bar, 0, hk, tile_start(j), b);
    tma_load_4d(smem_u32(base + lay.vc), &tmVc, bar, 0, hk, tile_start(j), b);
    const int p0 = ng == 1 ? tile_start(j) & ~1 : tile_start(j);  // a 16-byte aligned first coordinate
    tma_load_3d(smem_u32(base + lay.kp), &tmKp, bar, p0 * ng * 2, hk, b);
    tma_load_3d(smem_u32(base + lay.vp), &tmVp, bar, p0 * ng * 2, hk, b);
  };

  if (tid == 0) {
    for (int s = 0; s < DEC_STAGES; ++s) mbar_init(bar0 + 8 * s, 1);
    fence_mbar_init();
    tma_prefetch_desc(&tmKc);
    tma_prefetch_desc(&tmVc);
    tma_prefetch_desc(&tmKp);
    tma_prefetch_desc(&tmVp);
  }
  __syncthreads();
  if (tid == 0)
    for (int j = 0; j < min(n_tiles, DEC_STAGES); ++j) issue(j);

  const T* qb = reinterpret_cast<const T*>(p.q) + ((long long)b * p.H + (long long)hk * G) * D;
  for (int i = tid; i < G * L; i += DEC_THREADS) {
    float f[8];
    ld8(qb + i * 8, f);
    float sum = 0.f;
#pragma unroll
    for (int e = 0; e < 8; ++e) {
      sq[i * 8 + e] = f[e] * p.scale_log2;
      sum += f[e] * p.scale_log2;
    }
    sqs[i] = sum;
  }
  for (int h = tid; h < G; h += DEC_THREADS) {
    sm[h] = -INFINITY;
    sl[h] = 0.f;
    if (alibi) sred[h] = __ldg(p.slopes + hk * G + h) * kLog2e;
  }

  const int items = G * L;
  const int ks_n = items <= DEC_THREADS ? DEC_THREADS / items : 1;
  int my_item[DEC_MAX_ITEMS], my_ks;
  if (items <= DEC_THREADS) {
    my_ks = tid / items;
    my_item[0] = my_ks < ks_n ? tid % items : -1;
    my_item[1] = -1;
  } else {
    my_ks = 0;
    my_item[0] = tid;
    my_item[1] = tid + DEC_THREADS < items ? tid + DEC_THREADS : -1;
  }
  float acc[DEC_MAX_ITEMS][8], accb[DEC_MAX_ITEMS];
#pragma unroll
  for (int r = 0; r < DEC_MAX_ITEMS; ++r) {
    accb[r] = 0.f;
#pragma unroll
    for (int e = 0; e < 8; ++e) acc[r][e] = 0.f;
  }
  __syncthreads();

  for (int j = 0; j < n_tiles; ++j) {
    const int st = j % DEC_STAGES;
    mbar_wait(bar0 + 8 * st, (j / DEC_STAGES) & 1);
    const uint8_t* base = smem + st * lay.stage;
    const uint8_t* tKc = base + lay.kc;
    const uint8_t* tVc = base + lay.vc;
    const int start = tile_start(j);
    const int poff = ng == 1 ? (start & 1) * 2 : 0;  // floats before the tile's first parameter pair
    const float* tKp = reinterpret_cast<const float*>(base + lay.kp) + poff;
    const float* tVp = reinterpret_cast<const float*>(base + lay.vp) + poff;
    const int first_valid = max(lo + j * DEC_TILE, kv0);

    {
      const int kl = tid % L;
      for (int key = tid / L; key < DEC_TILE; key += DEC_THREADS / L) {
        float kf[8];
        codes8<BITS>(tKc + key * Dc + kl * SB, kf);
        const float2 sb = *reinterpret_cast<const float2*>(tKp + (key * ng + kl / spg) * 2);
        const bool valid = start + key >= first_valid;
        for (int h = 0; h < G; ++h) {
          const float4 qa = *reinterpret_cast<const float4*>(sq + h * D + kl * 8);
          const float4 qc = *reinterpret_cast<const float4*>(sq + h * D + kl * 8 + 4);
          float d = qa.x * kf[0];
          d = fmaf(qa.y, kf[1], d);
          d = fmaf(qa.z, kf[2], d);
          d = fmaf(qa.w, kf[3], d);
          d = fmaf(qc.x, kf[4], d);
          d = fmaf(qc.y, kf[5], d);
          d = fmaf(qc.z, kf[6], d);
          d = fmaf(qc.w, kf[7], d);
          d = fmaf(sb.x, d, sb.y * sqs[h * L + kl]);
#pragma unroll
          for (int off = L / 2; off > 0; off >>= 1) d += __shfl_xor_sync(0xffffffffu, d, off);
          if (kl == 0) ss[h * DEC_TILE + key] = valid ? d : -INFINITY;
        }
      }
    }
    __syncthreads();

    const float kd = (float)(start + lane - (len - 1));
    for (int h = warp; h < G; h += DEC_THREADS / 32) {
      float x = ss[h * DEC_TILE + lane];
      if (alibi) x = x + sred[h] * kd;
      const float m_old = sm[h];
      const float m_new = fmaxf(m_old, warp_max(x));
      const float pe = exp2f(x - m_new);
      const float sum = warp_sum(pe);
      ss[h * DEC_TILE + lane] = pe;
      __syncwarp();
      if (lane == 0) {
        const float alpha = exp2f(m_old - m_new);
        salpha[h] = alpha;
        sl[h] = sl[h] * alpha + sum;
        sm[h] = m_new;
      }
    }
    __syncthreads();

#pragma unroll
    for (int r = 0; r < DEC_MAX_ITEMS; ++r) {
      if (my_item[r] < 0) continue;
      const int h = my_item[r] / L, sc = my_item[r] % L;
      const float a = salpha[h];
      accb[r] *= a;
#pragma unroll
      for (int e = 0; e < 8; ++e) acc[r][e] *= a;
      const int gp = (sc / spg) * 2;
      for (int key = my_ks; key < DEC_TILE; key += ks_n) {
        const float pe = ss[h * DEC_TILE + key];
        const float2 sb = *reinterpret_cast<const float2*>(tVp + key * ng * 2 + gp);
        float vf[8];
        codes8<BITS>(tVc + key * Dc + sc * SB, vf);
        const float ps = pe * sb.x;
        accb[r] = fmaf(pe, sb.y, accb[r]);
#pragma unroll
        for (int e = 0; e < 8; ++e) acc[r][e] = fmaf(ps, vf[e], acc[r][e]);
      }
    }
    __syncthreads();
    if (tid == 0 && j + DEC_STAGES < n_tiles) issue(j + DEC_STAGES);
  }

#pragma unroll
  for (int r = 0; r < DEC_MAX_ITEMS; ++r)
#pragma unroll
    for (int e = 0; e < 8; ++e) acc[r][e] += accb[r];

  if (ks_n > 1) {
    if (my_item[0] >= 0)
#pragma unroll
      for (int e = 0; e < 8; ++e) sred[(my_ks * items + my_item[0]) * 8 + e] = acc[0][e];
    __syncthreads();
    if (tid < items) {
#pragma unroll
      for (int e = 0; e < 8; ++e) acc[0][e] = sred[tid * 8 + e];
      for (int k = 1; k < ks_n; ++k)
#pragma unroll
        for (int e = 0; e < 8; ++e) acc[0][e] += sred[(k * items + tid) * 8 + e];
      my_item[0] = tid;
    } else {
      my_item[0] = -1;
    }
  }

#pragma unroll
  for (int r = 0; r < DEC_MAX_ITEMS; ++r) {
    if (my_item[r] < 0) continue;
    const int h = my_item[r] / L, sc = my_item[r] % L;
    const long long bh = (long long)b * p.H + hk * G + h;
    const float m = sm[h], l = sl[h];
    if (n_chunks == 1) {
      const float inv = 1.0f / l;
      float f[8];
#pragma unroll
      for (int e = 0; e < 8; ++e) f[e] = acc[r][e] * inv;
      st8(reinterpret_cast<T*>(p.o) + bh * D + sc * 8, f);
      if (p.lse != nullptr && sc == 0) p.lse[bh] = (m + log2f(l)) / kLog2e;
    } else {
      st8(p.part_acc + (bh * p.max_chunks + c) * D + sc * 8, acc[r]);
      if (sc == 0) {
        p.part_ml[(bh * p.max_chunks + c) * 2] = m;
        p.part_ml[(bh * p.max_chunks + c) * 2 + 1] = l;
      }
    }
  }
}

template <typename T, int D, int BITS>
int launch_decode_quant(const CUtensorMap* tm, const DecArgs& a, int g, int B, int Hk, cudaStream_t stream) {
  auto kern = attn_decode_quant_kernel<T, D, BITS>;
  const QDecSmem lay(D * BITS / 8, D / g, D, a.G);
  static int attr_bytes = 0;
  if (lay.total > 48 * 1024 && lay.total > attr_bytes) {
    B200_CHECK_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, lay.total));
    attr_bytes = lay.total;
  }
  kern<<<dim3(a.max_chunks, Hk, B), DEC_THREADS, lay.total, stream>>>(tm[0], tm[1], tm[2], tm[3], a, g);
  B200_CHECK_LAUNCH();
  if (a.max_chunks > 1) {
    attn_decode_combine_kernel<T, D><<<dim3(a.H, B), D, 0, stream>>>(a);
    B200_CHECK_LAUNCH();
  }
  return B200_OK;
}

template <typename T, int BITS>
int launch_decode_quant_d(int D, const CUtensorMap* tm, const DecArgs& a, int g, int B, int Hk, cudaStream_t stream) {
  switch (D) {
    case 32: return launch_decode_quant<T, 32, BITS>(tm, a, g, B, Hk, stream);
    case 64: return launch_decode_quant<T, 64, BITS>(tm, a, g, B, Hk, stream);
    default: return launch_decode_quant<T, 128, BITS>(tm, a, g, B, Hk, stream);
  }
}

// the format's argument checks shared by the three quantized-cache entries
int check_quant_format(const char* what, int B, int s_max, int Hk, int D, int bits, int g) {
  B200_CHECK_ARG(bits == 4 || bits == 8, "%s: kv_bits=%d unsupported (4 or 8)", what, bits);
  B200_CHECK_ARG(g == 32 || g == 64 || g == 128, "%s: group size %d unsupported (32, 64 or 128)", what, g);
  B200_CHECK_ARG(D == 32 || D == 64 || D == 128, "%s: head_dim %d unsupported (32, 64 or 128)", what, D);
  B200_CHECK_ARG(D % g == 0, "%s: the group size %d must divide head_dim %d", what, g, D);
  B200_CHECK_ARG(B > 0 && Hk > 0 && s_max > 0 && s_max % 2 == 0, "%s: bad shape B=%d s_max=%d (even) Hk=%d", what, B,
                 s_max, Hk);
  return B200_OK;
}

// window < 0 means none; slopes selects ALiBi
// ring_m > 0: a ring of s_max slots (bf16, D 64 / 128) with max_kv_size ring_m
// start non-null: n_q queries per row from position start[b], lens the rows' ends (attn_decode_multi)
int attn_decode_impl(const void* q, const void* k_cache, const void* v_cache, const int* lens, void* o, float* lse,
                     int window, int B, int s_max, int H, int Hk, int D, float scale, int is_bf16, void* ws,
                     size_t ws_bytes, cudaStream_t stream, const float* slopes = nullptr, int ring_m = 0,
                     const int* start = nullptr, int n_q = 1) {
  B200_CHECK_ARG(B > 0 && H > 0 && Hk > 0 && H % Hk == 0, "attn_decode: bad shape B=%d H=%d Hk=%d", B, H, Hk);
  B200_CHECK_ARG(D == 16 || D == 32 || D == 64 || D == 128, "attn_decode: head_dim %d unsupported (16/32/64/128)", D);
  B200_CHECK_ARG(s_max >= DEC_TILE, "attn_decode: s_max=%d must be >= %d", s_max, DEC_TILE);
  const int G = H / Hk;
  B200_CHECK_ARG(G * D <= DEC_MAX_ITEMS * DEC_THREADS * 8, "attn_decode: (H/Hk) * D = %d exceeds %d", G * D,
                 DEC_MAX_ITEMS * DEC_THREADS * 8);
  B200_CHECK_ARG(al16(q) && al16(o) && lens != nullptr, "attn_decode: q / o must be 16-byte aligned, lens non-null");
  const size_t need = b200_attn_decode_workspace_bytes(B * n_q, H, s_max, D);
  if (ws_bytes < need || (need > 0 && ws == nullptr)) {
    set_error("attn_decode: workspace of %zu bytes, %zu needed", ws_bytes, need);
    return B200_ERR_WORKSPACE;
  }
  const int elem = is_bf16 ? 2 : 4;
  const CUtensorMapDataType dt = is_bf16 ? CU_TENSOR_MAP_DATA_TYPE_BFLOAT16 : CU_TENSOR_MAP_DATA_TYPE_FLOAT32;
  const uint64_t dims[4] = {(uint64_t)D, (uint64_t)Hk, (uint64_t)s_max, (uint64_t)B};
  const uint64_t strides[3] = {(uint64_t)D * elem, (uint64_t)Hk * D * elem, (uint64_t)s_max * Hk * D * elem};
  const uint32_t box[4] = {(uint32_t)D, 1, (uint32_t)DEC_TILE, 1};
  CUtensorMap tmK, tmV;
  int rc;
  if ((rc = make_tensor_map(&tmK, k_cache, dt, elem, 4, dims, strides, box, false))) return rc;
  if ((rc = make_tensor_map(&tmV, v_cache, dt, elem, 4, dims, strides, box, false))) return rc;
  DecMultiArgs a;
  a.q = q;
  a.o = o;
  a.lse = lse;
  a.lens = lens;
  a.max_chunks = (s_max + DEC_CHUNK - 1) / DEC_CHUNK;
  a.part_acc = reinterpret_cast<float*>(ws);
  a.part_ml = a.part_acc + (size_t)B * n_q * H * a.max_chunks * D;
  a.H = H;
  a.G = G;
  a.s_max = s_max;
  a.scale_log2 = scale * kLog2e;
  a.window = window < 0 || window > s_max ? s_max : window;
  a.slopes = slopes;
  a.ring_m = ring_m;
  a.start = start;
  a.n_q = n_q;
  if (start != nullptr) {
    if (slopes)
      return is_bf16 ? launch_decode_multi_d<__nv_bfloat16, true>(D, tmK, tmV, a, B, Hk, stream)
                     : launch_decode_multi_d<float, true>(D, tmK, tmV, a, B, Hk, stream);
    return is_bf16 ? launch_decode_multi_d<__nv_bfloat16, false>(D, tmK, tmV, a, B, Hk, stream)
                   : launch_decode_multi_d<float, false>(D, tmK, tmV, a, B, Hk, stream);
  }
  if (ring_m > 0) {
    a.window = window < 0 ? INT_MAX : window;
    if (slopes)
      return D == 64 ? launch_decode<__nv_bfloat16, 64, true, true>(tmK, tmV, a, B, Hk, stream)
                     : launch_decode<__nv_bfloat16, 128, true, true>(tmK, tmV, a, B, Hk, stream);
    return D == 64 ? launch_decode<__nv_bfloat16, 64, false, true>(tmK, tmV, a, B, Hk, stream)
                   : launch_decode<__nv_bfloat16, 128, false, true>(tmK, tmV, a, B, Hk, stream);
  }
  if (slopes)
    return is_bf16 ? launch_decode_d<__nv_bfloat16, true>(D, tmK, tmV, a, B, Hk, stream)
                   : launch_decode_d<float, true>(D, tmK, tmV, a, B, Hk, stream);
  return is_bf16 ? launch_decode_d<__nv_bfloat16>(D, tmK, tmV, a, B, Hk, stream)
                 : launch_decode_d<float>(D, tmK, tmV, a, B, Hk, stream);
}

}  // namespace
}  // namespace b200

using namespace b200;

extern "C" {

size_t b200_attn_decode_workspace_bytes(int B, int H, int s_max, int D) {
  if (B <= 0 || H <= 0 || s_max <= 0 || D <= 0) return 0;
  const size_t chunks = (size_t)(s_max + DEC_CHUNK - 1) / DEC_CHUNK;
  return (size_t)B * H * chunks * (size_t)(D + 2) * sizeof(float);
}

int b200_attn_decode(const void* q, const void* k_cache, const void* v_cache, const int* lens, void* o, float* lse,
                     int B, int s_max, int H, int Hk, int D, float scale, int is_bf16, void* ws, size_t ws_bytes,
                     void* stream) {
  return attn_decode_impl(q, k_cache, v_cache, lens, o, lse, -1, B, s_max, H, Hk, D, scale, is_bf16, ws, ws_bytes,
                          static_cast<cudaStream_t>(stream));
}

// sliding window: the query at position lens[b] - 1 sees cached keys max(0, lens[b] - 1 - window) .. lens[b] - 1
int b200_attn_decode_window(const void* q, const void* k_cache, const void* v_cache, const int* lens, void* o,
                            float* lse, int window, int B, int s_max, int H, int Hk, int D, float scale, int is_bf16,
                            void* ws, size_t ws_bytes, void* stream) {
  B200_CHECK_ARG(window >= 0, "attn_decode_window: window=%d must be >= 0", window);
  return attn_decode_impl(q, k_cache, v_cache, lens, o, lse, window, B, s_max, H, Hk, D, scale, is_bf16, ws,
                          ws_bytes, static_cast<cudaStream_t>(stream));
}

// ALiBi: attn_decode_window (window < 0: none) with the bias slopes[h] * (k - (lens[b] - 1)) on every cached key k
int b200_attn_decode_alibi(const void* q, const void* k_cache, const void* v_cache, const int* lens, void* o,
                           float* lse, int window, const float* slopes, int B, int s_max, int H, int Hk, int D,
                           float scale, int is_bf16, void* ws, size_t ws_bytes, void* stream) {
  B200_CHECK_ARG(slopes != nullptr && (reinterpret_cast<uintptr_t>(slopes) & 3u) == 0,
                 "attn_decode_alibi: slopes must be a non-null, 4-byte aligned fp32 [H] array");
  return attn_decode_impl(q, k_cache, v_cache, lens, o, lse, window, B, s_max, H, Hk, D, scale, is_bf16, ws,
                          ws_bytes, static_cast<cudaStream_t>(stream), slopes);
}

int b200_kv_append(void* q, const void* k, const void* v, void* k_cache, void* v_cache, const int* lens,
                   const float* cos_t, const float* sin_t, int B, int s_max, int H, int Hk, int D, int is_bf16,
                   void* stream) {
  const cudaStream_t s = static_cast<cudaStream_t>(stream);
  B200_CHECK_ARG(B > 0 && s_max > 0 && H > 0 && Hk > 0 && D > 0 && D % 8 == 0,
                 "kv_append: bad shape B=%d s_max=%d H=%d Hk=%d D=%d (D %% 8 == 0)", B, s_max, H, Hk, D);
  B200_CHECK_ARG((cos_t == nullptr) == (sin_t == nullptr), "kv_append: give both RoPE tables or neither");
  B200_CHECK_ARG(al16(k) && al16(v) && al16(k_cache) && al16(v_cache) && (cos_t == nullptr || (al16(q) && al16(cos_t) && al16(sin_t))),
                 "kv_append: alignment");
  const int heads = (cos_t != nullptr ? H : 0) + 2 * Hk;
  const long long nvec = (long long)B * heads * (D / 8);
  long long blocks = (nvec + 255) / 256;
  if (blocks > (long long)num_sms() * 8) blocks = (long long)num_sms() * 8;
  if (is_bf16)
    kv_append_kernel<__nv_bfloat16><<<(int)blocks, 256, 0, s>>>(
        (__nv_bfloat16*)q, (const __nv_bfloat16*)k, (const __nv_bfloat16*)v, (__nv_bfloat16*)k_cache,
        (__nv_bfloat16*)v_cache, lens, cos_t, sin_t, nvec, s_max, H, Hk, D);
  else
    kv_append_kernel<float><<<(int)blocks, 256, 0, s>>>((float*)q, (const float*)k, (const float*)v,
                                                        (float*)k_cache, (float*)v_cache, lens, cos_t, sin_t,
                                                        nvec, s_max, H, Hk, D);
  B200_CHECK_LAUNCH();
  return B200_OK;
}

// kv_append with the half-split rotation of b200_rope_half; the tables are required and D % 16 == 0
int b200_kv_append_half(void* q, const void* k, const void* v, void* k_cache, void* v_cache, const int* lens,
                        const float* cos_t, const float* sin_t, int B, int s_max, int H, int Hk, int D, int is_bf16,
                        void* stream) {
  const cudaStream_t s = static_cast<cudaStream_t>(stream);
  B200_CHECK_ARG(B > 0 && s_max > 0 && H > 0 && Hk > 0 && D > 0 && D % 16 == 0,
                 "kv_append_half: bad shape B=%d s_max=%d H=%d Hk=%d D=%d (D %% 16 == 0)", B, s_max, H, Hk, D);
  B200_CHECK_ARG(cos_t != nullptr && sin_t != nullptr && lens != nullptr, "kv_append_half: RoPE tables and lens required");
  B200_CHECK_ARG(al16(q) && al16(k) && al16(v) && al16(k_cache) && al16(v_cache) && al16(cos_t) && al16(sin_t),
                 "kv_append_half: alignment");
  const long long nslice = (long long)B * (H + 2 * Hk) * (D / 16);
  long long blocks = (nslice + 255) / 256;
  if (blocks > (long long)num_sms() * 8) blocks = (long long)num_sms() * 8;
  if (is_bf16)
    kv_append_half_kernel<__nv_bfloat16><<<(int)blocks, 256, 0, s>>>(
        (__nv_bfloat16*)q, (const __nv_bfloat16*)k, (const __nv_bfloat16*)v, (__nv_bfloat16*)k_cache,
        (__nv_bfloat16*)v_cache, lens, cos_t, sin_t, nslice, s_max, H, Hk, D);
  else
    kv_append_half_kernel<float><<<(int)blocks, 256, 0, s>>>((float*)q, (const float*)k, (const float*)v,
                                                             (float*)k_cache, (float*)v_cache, lens, cos_t,
                                                             sin_t, nslice, s_max, H, Hk, D);
  B200_CHECK_LAUNCH();
  return B200_OK;
}

// The rotating KV cache of the reference's generator (core/generation_lite.py:103, :120: max_kv_size makes every
// layer's cache an mlx_lm RotatingKVCache): decode attention over a ring of C slots (include/b200_hotpath.h)
int b200_attn_decode_ring(const void* q, const void* k_ring, const void* v_ring, const int* end, void* o, float* lse,
                          int max_kv, int window, const float* slopes, int B, int C, int H, int Hk, int D, float scale,
                          void* ws, size_t ws_bytes, void* stream) {
  B200_CHECK_ARG(max_kv >= 5 && C >= max_kv, "attn_decode_ring: max_kv=%d must be >= 5 and <= C=%d", max_kv, C);
  B200_CHECK_ARG(D == 64 || D == 128, "attn_decode_ring: head_dim %d unsupported (64 or 128)", D);
  B200_CHECK_ARG(al16(k_ring) && al16(v_ring), "attn_decode_ring: k_ring and v_ring must be 16-byte aligned");
  B200_CHECK_ARG((reinterpret_cast<uintptr_t>(slopes) & 3u) == 0, "attn_decode_ring: slopes must be 4-byte aligned");
  return attn_decode_impl(q, k_ring, v_ring, end, o, lse, window, B, C, H, Hk, D, scale, 1, ws, ws_bytes,
                          static_cast<cudaStream_t>(stream), slopes, max_kv);
}

// Speculative decoding's verify step (the reference's mlx_lm generate with a draft_model): n_q <= 16 new queries per
// row over its dense cache, query i at position start[b] + i valid iff i < end[b] - start[b] (include/b200_hotpath.h)
int b200_attn_decode_multi(const void* q, const void* k_cache, const void* v_cache, const int* start, const int* end,
                           void* o, float* lse, int window, const float* slopes, int B, int n_q, int s_max, int H,
                           int Hk, int D, float scale, int is_bf16, void* ws, size_t ws_bytes, void* stream) {
  B200_CHECK_ARG(n_q >= 1 && n_q <= 16, "attn_decode_multi: n_q=%d must lie in [1, 16]", n_q);
  // grid z is (row, query pack) and the combine's grid y (row, query): both at most B * n_q
  B200_CHECK_ARG(B > 0 && (long long)B * n_q <= 65535, "attn_decode_multi: B * n_q = %lld exceeds the grid's 65535",
                 (long long)B * n_q);
  B200_CHECK_ARG(start != nullptr && end != nullptr && (reinterpret_cast<uintptr_t>(start) & 3u) == 0 &&
                     (reinterpret_cast<uintptr_t>(end) & 3u) == 0,
                 "attn_decode_multi: start and end must be non-null, 4-byte aligned int32 [B] arrays");
  B200_CHECK_ARG(slopes == nullptr || (reinterpret_cast<uintptr_t>(slopes) & 3u) == 0,
                 "attn_decode_multi: slopes must be a 4-byte aligned fp32 [H] array");
  return attn_decode_impl(q, k_cache, v_cache, end, o, lse, window, B, s_max, H, Hk, D, scale, is_bf16, ws, ws_bytes,
                          static_cast<cudaStream_t>(stream), slopes, 0, start, n_q);
}

size_t b200_attn_decode_multi_workspace_bytes(int B, int n_q, int H, int s_max, int D) {
  if (n_q <= 0) return 0;
  return b200_attn_decode_workspace_bytes(B * n_q, H, s_max, D);
}

// The token a decode step appends to a ring (core/generation_lite.py:103, :120): rotated at position end[b] - 1,
// stored in slot(end[b] - 1); rows with live[b] == 0 are left alone
int b200_kv_append_ring(void* q, const void* k, const void* v, void* k_ring, void* v_ring, const int* end,
                        const int* live, const float* cos_t, const float* sin_t, int half, int B, int C, int H,
                        int Hk, int D, void* stream) {
  const cudaStream_t s = static_cast<cudaStream_t>(stream);
  B200_CHECK_ARG(B > 0 && C > RING_SINKS && H > 0 && Hk > 0 && H % Hk == 0 && (D == 64 || D == 128),
                 "kv_append_ring: bad shape B=%d C=%d H=%d Hk=%d D=%d (D 64 or 128)", B, C, H, Hk, D);
  B200_CHECK_ARG(end != nullptr && (reinterpret_cast<uintptr_t>(end) & 3u) == 0 &&
                     (reinterpret_cast<uintptr_t>(live) & 3u) == 0,
                 "kv_append_ring: end (non-null) and live must be 4-byte aligned int32 [B] arrays");
  B200_CHECK_ARG((cos_t == nullptr) == (sin_t == nullptr) && (!half || cos_t != nullptr),
                 "kv_append_ring: give both RoPE tables or neither (the half layout needs them)");
  B200_CHECK_ARG(al16(q) && al16(k) && al16(v) && al16(k_ring) && al16(v_ring) &&
                     (cos_t == nullptr || (al16(cos_t) && al16(sin_t))),
                 "kv_append_ring: alignment");
  auto* qq = static_cast<__nv_bfloat16*>(q);
  auto* kk = static_cast<const __nv_bfloat16*>(k);
  auto* vv = static_cast<const __nv_bfloat16*>(v);
  auto* kr = static_cast<__nv_bfloat16*>(k_ring);
  auto* vr = static_cast<__nv_bfloat16*>(v_ring);
  if (half) {
    const long long nslice = (long long)B * (H + 2 * Hk) * (D / 16);
    long long blocks = (nslice + 255) / 256;
    if (blocks > (long long)num_sms() * 8) blocks = (long long)num_sms() * 8;
    kv_append_half_kernel<__nv_bfloat16, true><<<(int)blocks, 256, 0, s>>>(qq, kk, vv, kr, vr, end, cos_t, sin_t,
                                                                           nslice, C, H, Hk, D, live);
  } else {
    const long long nvec = (long long)B * ((cos_t != nullptr ? H : 0) + 2 * Hk) * (D / 8);
    long long blocks = (nvec + 255) / 256;
    if (blocks > (long long)num_sms() * 8) blocks = (long long)num_sms() * 8;
    kv_append_kernel<__nv_bfloat16, true><<<(int)blocks, 256, 0, s>>>(qq, kk, vv, kr, vr, end, cos_t, sin_t, nvec,
                                                                      C, H, Hk, D, live);
  }
  B200_CHECK_LAUNCH();
  return B200_OK;
}

// Beam search over a shared-prompt cache (generate_lite.py:400-484 of the reference runs n_beams full sequences per
// prompt; here each prompt's cache is stored and read once for its beams, include/b200_hotpath.h)
int b200_attn_decode_beam(const void* q, const void* k_prefix, const void* v_prefix, const void* k_tail,
                          const void* v_tail, const int* lens, const int* tables, void* o, float* lse, int window,
                          const float* slopes, int R, int n_groups, int s_prefix, int n_slots, int tail_cap, int H,
                          int Hk, int D, float scale, int is_bf16, void* ws, size_t ws_bytes, void* stream) {
  B200_CHECK_ARG(R > 0 && n_groups > 0 && n_slots > 0 && H > 0 && Hk > 0 && H % Hk == 0,
                 "attn_decode_beam: bad shape R=%d n_groups=%d n_slots=%d H=%d Hk=%d", R, n_groups, n_slots, H, Hk);
  B200_CHECK_ARG(D == 16 || D == 32 || D == 64 || D == 128, "attn_decode_beam: head_dim %d unsupported (16/32/64/128)",
                 D);
  B200_CHECK_ARG(s_prefix >= DEC_CHUNK && s_prefix % DEC_CHUNK == 0 && tail_cap >= DEC_CHUNK &&
                     tail_cap % DEC_CHUNK == 0,
                 "attn_decode_beam: s_prefix=%d and tail_cap=%d must be positive multiples of %d", s_prefix, tail_cap,
                 DEC_CHUNK);
  const int G = H / Hk;
  B200_CHECK_ARG(G * D <= DEC_MAX_ITEMS * DEC_THREADS * 8, "attn_decode_beam: (H/Hk) * D = %d exceeds %d", G * D,
                 DEC_MAX_ITEMS * DEC_THREADS * 8);
  B200_CHECK_ARG(al16(q) && al16(o) && al16(k_prefix) && al16(v_prefix) && al16(k_tail) && al16(v_tail),
                 "attn_decode_beam: q, o and the caches must be 16-byte aligned");
  B200_CHECK_ARG(lens != nullptr && tables != nullptr && (reinterpret_cast<uintptr_t>(tables) & 3u) == 0,
                 "attn_decode_beam: lens and tables must be non-null int32 arrays");
  B200_CHECK_ARG(slopes == nullptr || (reinterpret_cast<uintptr_t>(slopes) & 3u) == 0,
                 "attn_decode_beam: slopes must be a 4-byte aligned fp32 [H] array");
  const size_t need = b200_attn_decode_beam_workspace_bytes(R, H, s_prefix, tail_cap, D);
  if (ws_bytes < need || ws == nullptr || (reinterpret_cast<uintptr_t>(ws) & 127u) != 0) {
    set_error("attn_decode_beam: workspace of %zu bytes (128-byte aligned), %zu needed", ws_bytes, need);
    return B200_ERR_WORKSPACE;
  }
  const int s_max = s_prefix + tail_cap;
  const int elem = is_bf16 ? 2 : 4;
  const CUtensorMapDataType dt = is_bf16 ? CU_TENSOR_MAP_DATA_TYPE_BFLOAT16 : CU_TENSOR_MAP_DATA_TYPE_FLOAT32;
  const uint32_t box[4] = {(uint32_t)D, 1, (uint32_t)DEC_TILE, 1};
  const uint64_t strides[3] = {(uint64_t)D * elem, (uint64_t)Hk * D * elem, (uint64_t)s_prefix * Hk * D * elem};
  const uint64_t dims[4] = {(uint64_t)D, (uint64_t)Hk, (uint64_t)s_prefix, (uint64_t)n_groups};
  const uint64_t tstrides[3] = {(uint64_t)D * elem, (uint64_t)Hk * D * elem, (uint64_t)tail_cap * Hk * D * elem};
  const uint64_t tdims[4] = {(uint64_t)D, (uint64_t)Hk, (uint64_t)tail_cap, (uint64_t)n_slots};
  CUtensorMap tm[2];
  BeamMaps hdr;
  int rc;
  if ((rc = make_tensor_map(&tm[0], k_prefix, dt, elem, 4, dims, strides, box, false))) return rc;
  if ((rc = make_tensor_map(&tm[1], v_prefix, dt, elem, 4, dims, strides, box, false))) return rc;
  if ((rc = make_tensor_map(&hdr.k_tail, k_tail, dt, elem, 4, tdims, tstrides, box, false))) return rc;
  if ((rc = make_tensor_map(&hdr.v_tail, v_tail, dt, elem, 4, tdims, tstrides, box, false))) return rc;
  const int pack = b200_attn_decode_beam_pack(H, Hk, D);
  hdr.args = BeamArgs{tables, tables + R, tables + 2 * R, tables + 2 * R + n_groups, tables + 2 * R + 2 * n_groups,
                      pack};
  const cudaStream_t s = static_cast<cudaStream_t>(stream);
  B200_CHECK_CUDA(cudaMemcpyAsync(ws, &hdr, sizeof(hdr), cudaMemcpyHostToDevice, s));
  DecArgs a;
  a.q = q;
  a.o = o;
  a.lse = lse;
  a.lens = lens;
  a.max_chunks = s_max / DEC_CHUNK;
  a.part_acc = reinterpret_cast<float*>(static_cast<uint8_t*>(ws) + BEAM_HDR);
  a.part_ml = a.part_acc + (size_t)R * H * a.max_chunks * D;
  a.H = H;
  a.G = G;
  a.s_max = s_max;
  a.scale_log2 = scale * kLog2e;
  a.window = window < 0 || window > s_max ? s_max : window;
  a.slopes = slopes;
  a.beam = static_cast<const BeamMaps*>(ws);
  if (slopes)
    return is_bf16 ? launch_decode_beam_d<__nv_bfloat16, true>(D, tm, a, pack, R, Hk, s)
                   : launch_decode_beam_d<float, true>(D, tm, a, pack, R, Hk, s);
  return is_bf16 ? launch_decode_beam_d<__nv_bfloat16, false>(D, tm, a, pack, R, Hk, s)
                 : launch_decode_beam_d<float, false>(D, tm, a, pack, R, Hk, s);
}

size_t b200_attn_decode_beam_workspace_bytes(int R, int H, int s_prefix, int tail_cap, int D) {
  if (R <= 0 || H <= 0 || s_prefix <= 0 || tail_cap <= 0 || D <= 0) return 0;
  return BEAM_HDR + b200_attn_decode_workspace_bytes(R, H, s_prefix + tail_cap, D);
}

int b200_attn_decode_beam_pack(int H, int Hk, int D) {
  if (H <= 0 || Hk <= 0 || D <= 0 || H % Hk != 0) return 0;
  return max(1, DEC_MAX_ITEMS * DEC_THREADS * 8 / (H / Hk * D));
}

// The token a beam step appends: b200_kv_append (half == 0) or b200_kv_append_half (half != 0) rotated at position
// lens[b] - 1 and written to index lens[b] - 1 - T0 of row b's tail slot
int b200_kv_append_beam(void* q, const void* k, const void* v, void* k_tail, void* v_tail, const int* lens,
                        const int* tables, const float* cos_t, const float* sin_t, int half, int R, int tail_cap, int H,
                        int Hk, int D, int is_bf16, void* stream) {
  B200_CHECK_ARG(R > 0 && tail_cap > 0 && H > 0 && Hk > 0 && D > 0 && D % (half ? 16 : 8) == 0,
                 "kv_append_beam: bad shape R=%d tail_cap=%d H=%d Hk=%d D=%d (D %% %d == 0)", R, tail_cap, H, Hk, D,
                 half ? 16 : 8);
  B200_CHECK_ARG((cos_t == nullptr) == (sin_t == nullptr) && (!half || cos_t != nullptr),
                 "kv_append_beam: give both RoPE tables or neither (the half layout needs them)");
  B200_CHECK_ARG(lens != nullptr && tables != nullptr, "kv_append_beam: lens and tables must be non-null");
  B200_CHECK_ARG(al16(k) && al16(v) && al16(k_tail) && al16(v_tail) &&
                     (cos_t == nullptr || (al16(q) && al16(cos_t) && al16(sin_t))),
                 "kv_append_beam: alignment");
  const long long n = half ? (long long)R * (H + 2 * Hk) * (D / 16)
                           : (long long)R * ((cos_t != nullptr ? H : 0) + 2 * Hk) * (D / 8);
  long long blocks = (n + 255) / 256;
  if (blocks > (long long)num_sms() * 8) blocks = (long long)num_sms() * 8;
  const cudaStream_t s = static_cast<cudaStream_t>(stream);
  if (is_bf16) {
    auto* qq = static_cast<__nv_bfloat16*>(q);
    auto* kk = static_cast<const __nv_bfloat16*>(k);
    auto* vv = static_cast<const __nv_bfloat16*>(v);
    auto* kt = static_cast<__nv_bfloat16*>(k_tail);
    auto* vt = static_cast<__nv_bfloat16*>(v_tail);
    if (half)
      kv_append_half_kernel<__nv_bfloat16, false, true><<<(int)blocks, 256, 0, s>>>(
          qq, kk, vv, kt, vt, lens, cos_t, sin_t, n, tail_cap, H, Hk, D, tables);
    else
      kv_append_kernel<__nv_bfloat16, false, true><<<(int)blocks, 256, 0, s>>>(
          qq, kk, vv, kt, vt, lens, cos_t, sin_t, n, tail_cap, H, Hk, D, tables);
  } else {
    auto* qq = static_cast<float*>(q);
    auto* kk = static_cast<const float*>(k);
    auto* vv = static_cast<const float*>(v);
    auto* kt = static_cast<float*>(k_tail);
    auto* vt = static_cast<float*>(v_tail);
    if (half)
      kv_append_half_kernel<float, false, true><<<(int)blocks, 256, 0, s>>>(
          qq, kk, vv, kt, vt, lens, cos_t, sin_t, n, tail_cap, H, Hk, D, tables);
    else
      kv_append_kernel<float, false, true><<<(int)blocks, 256, 0, s>>>(qq, kk, vv, kt, vt, lens, cos_t, sin_t, n,
                                                                       tail_cap, H, Hk, D, tables);
  }
  B200_CHECK_LAUNCH();
  return B200_OK;
}

// The copies of one beam step's fork, for every layer's K and V tail in one launch
int b200_kv_beam_fork(void* const* bufs, int n_bufs, const int* copies, int n_copies, int max_len, int tail_cap,
                      int row_bytes, void* stream) {
  if (n_copies == 0) return B200_OK;
  B200_CHECK_ARG(bufs != nullptr && copies != nullptr && n_bufs > 0 && n_bufs <= 65535 && n_copies > 0 &&
                     n_copies <= 65535,
                 "kv_beam_fork: bad table n_bufs=%d n_copies=%d", n_bufs, n_copies);
  B200_CHECK_ARG(max_len >= 0 && max_len <= tail_cap && row_bytes > 0 && row_bytes % 16 == 0,
                 "kv_beam_fork: max_len=%d must lie in [0, tail_cap=%d], row_bytes=%d a multiple of 16", max_len,
                 tail_cap, row_bytes);
  if (max_len == 0) return B200_OK;
  const int row_vec = row_bytes / 16;
  const long long per = (long long)max_len * row_vec;
  const int bx = (int)(per < 64 * 256 ? (per + 255) / 256 : 64);
  kv_beam_fork_kernel<<<dim3(bx, n_copies, n_bufs), 256, 0, static_cast<cudaStream_t>(stream)>>>(bufs, copies,
                                                                                               tail_cap, row_vec);
  B200_CHECK_LAUNCH();
  return B200_OK;
}

// The quantized KV cache of the reference's generator (core/generation_lite.py:75-90, :100-108, :190-195): the
// conversion maybe_quantize_kv_cache makes, as codes and parameters written in place (DESIGN §4.2.1).
int b200_kv_quantize(const void* k, const void* v, int n, int S, void* k_codes, void* v_codes, float* k_params,
                     float* v_params, int B, int s_max, int Hk, int D, int bits, int group_size, int is_bf16,
                     void* stream) {
  const cudaStream_t s = static_cast<cudaStream_t>(stream);
  int rc;
  if ((rc = check_quant_format("kv_quantize", B, s_max, Hk, D, bits, group_size))) return rc;
  B200_CHECK_ARG(n >= 0 && n <= S && n <= s_max, "kv_quantize: n=%d must lie in [0, min(S=%d, s_max=%d)]", n, S, s_max);
  B200_CHECK_ARG(al16(k) && al16(v) && al16(k_codes) && al16(v_codes) && al16(k_params) && al16(v_params),
                 "kv_quantize: every pointer must be 16-byte aligned");
  if (n == 0) return B200_OK;
  const long long slices = 2LL * B * n * Hk * (D / 8);
  long long blocks = (slices + 255) / 256;
  if (blocks > (long long)num_sms() * 8) blocks = (long long)num_sms() * 8;
  auto* kc = static_cast<uint8_t*>(k_codes);
  auto* vc = static_cast<uint8_t*>(v_codes);
  if (is_bf16) {
    auto* kk = static_cast<const __nv_bfloat16*>(k);
    auto* vv = static_cast<const __nv_bfloat16*>(v);
    if (bits == 8)
      kv_quantize_kernel<__nv_bfloat16, 8><<<(int)blocks, 256, 0, s>>>(kk, vv, kc, vc, k_params, v_params, n, S, B,
                                                                       s_max, Hk, D, group_size);
    else
      kv_quantize_kernel<__nv_bfloat16, 4><<<(int)blocks, 256, 0, s>>>(kk, vv, kc, vc, k_params, v_params, n, S, B,
                                                                       s_max, Hk, D, group_size);
  } else {
    auto* kk = static_cast<const float*>(k);
    auto* vv = static_cast<const float*>(v);
    if (bits == 8)
      kv_quantize_kernel<float, 8><<<(int)blocks, 256, 0, s>>>(kk, vv, kc, vc, k_params, v_params, n, S, B, s_max, Hk,
                                                               D, group_size);
    else
      kv_quantize_kernel<float, 4><<<(int)blocks, 256, 0, s>>>(kk, vv, kc, vc, k_params, v_params, n, S, B, s_max, Hk,
                                                               D, group_size);
  }
  B200_CHECK_LAUNCH();
  return B200_OK;
}

// b200_kv_append / b200_kv_append_half (half != 0) into the quantized cache (core/generation_lite.py:139, :149: the
// decode steps after conversion)
int b200_kv_append_quant(void* q, const void* k, const void* v, void* k_codes, void* v_codes, float* k_params,
                         float* v_params, const int* lens, const float* cos_t, const float* sin_t, int half, int B,
                         int s_max, int H, int Hk, int D, int bits, int group_size, int is_bf16, void* stream) {
  const cudaStream_t s = static_cast<cudaStream_t>(stream);
  int rc;
  if ((rc = check_quant_format("kv_append_quant", B, s_max, Hk, D, bits, group_size))) return rc;
  B200_CHECK_ARG(H > 0 && H % Hk == 0, "kv_append_quant: H=%d must be a multiple of Hk=%d", H, Hk);
  B200_CHECK_ARG((cos_t == nullptr) == (sin_t == nullptr), "kv_append_quant: give both RoPE tables or neither");
  B200_CHECK_ARG(!half || cos_t != nullptr, "kv_append_quant: the half layout needs the RoPE tables");
  B200_CHECK_ARG(lens != nullptr && al16(q) && al16(k) && al16(v) && al16(k_codes) && al16(v_codes) &&
                     al16(k_params) && al16(v_params) && (cos_t == nullptr || (al16(cos_t) && al16(sin_t))),
                 "kv_append_quant: alignment (16 bytes) or null lens");
  const dim3 grid(Hk, B);
  auto* kc = static_cast<uint8_t*>(k_codes);
  auto* vc = static_cast<uint8_t*>(v_codes);
  if (is_bf16) {
    auto* qq = static_cast<__nv_bfloat16*>(q);
    auto* kk = static_cast<const __nv_bfloat16*>(k);
    auto* vv = static_cast<const __nv_bfloat16*>(v);
    if (bits == 8)
      kv_append_quant_kernel<__nv_bfloat16, 8><<<grid, 128, 0, s>>>(qq, kk, vv, kc, vc, k_params, v_params, lens,
                                                                    cos_t, sin_t, half, s_max, H, Hk, D, group_size);
    else
      kv_append_quant_kernel<__nv_bfloat16, 4><<<grid, 128, 0, s>>>(qq, kk, vv, kc, vc, k_params, v_params, lens,
                                                                    cos_t, sin_t, half, s_max, H, Hk, D, group_size);
  } else {
    auto* qq = static_cast<float*>(q);
    auto* kk = static_cast<const float*>(k);
    auto* vv = static_cast<const float*>(v);
    if (bits == 8)
      kv_append_quant_kernel<float, 8><<<grid, 128, 0, s>>>(qq, kk, vv, kc, vc, k_params, v_params, lens, cos_t,
                                                            sin_t, half, s_max, H, Hk, D, group_size);
    else
      kv_append_quant_kernel<float, 4><<<grid, 128, 0, s>>>(qq, kk, vv, kc, vc, k_params, v_params, lens, cos_t,
                                                            sin_t, half, s_max, H, Hk, D, group_size);
  }
  B200_CHECK_LAUNCH();
  return B200_OK;
}

// Positions [0, end[b]) of the quantized cache as bf16 K and V [B, S, Hk, D]: the keys and values a chunk of queries
// attends over once the cache is quantized (QuantizedKVCache.update_and_fetch of the reference quantizes the chunk
// first, core/generation_lite.py:144-154)
int b200_kv_dequantize(const void* k_codes, const void* v_codes, const float* k_params, const float* v_params,
                       const int* end, void* k, void* v, int S, int B, int s_max, int Hk, int D, int bits,
                       int group_size, void* stream) {
  int rc;
  if ((rc = check_quant_format("kv_dequantize", B, s_max, Hk, D, bits, group_size))) return rc;
  B200_CHECK_ARG(S > 0 && S <= s_max, "kv_dequantize: S=%d must lie in [1, s_max=%d]", S, s_max);
  B200_CHECK_ARG(end != nullptr && (reinterpret_cast<uintptr_t>(end) & 3u) == 0,
                 "kv_dequantize: end must be a non-null, 4-byte aligned int32 [B] array");
  B200_CHECK_ARG(al16(k_codes) && al16(v_codes) && al16(k_params) && al16(v_params) && al16(k) && al16(v),
                 "kv_dequantize: every buffer must be 16-byte aligned");
  const long long slices = 2LL * B * S * Hk * (D / 8);
  long long blocks = (slices + 255) / 256;
  if (blocks > (long long)num_sms() * 8) blocks = (long long)num_sms() * 8;
  const cudaStream_t s = static_cast<cudaStream_t>(stream);
  auto* kc = static_cast<const uint8_t*>(k_codes);
  auto* vc = static_cast<const uint8_t*>(v_codes);
  auto* kk = static_cast<__nv_bfloat16*>(k);
  auto* vv = static_cast<__nv_bfloat16*>(v);
  if (bits == 8)
    kv_dequantize_kernel<8><<<(int)blocks, 256, 0, s>>>(kc, vc, k_params, v_params, end, kk, vv, S, B, s_max, Hk, D,
                                                        group_size);
  else
    kv_dequantize_kernel<4><<<(int)blocks, 256, 0, s>>>(kc, vc, k_params, v_params, end, kk, vv, S, B, s_max, Hk, D,
                                                        group_size);
  B200_CHECK_LAUNCH();
  return B200_OK;
}

// b200_attn_decode_alibi (window < 0: none, slopes null: no ALiBi) over the quantized cache (the attention the
// reference's decode steps run once the cache is a QuantizedKVCache, core/generation_lite.py:139)
int b200_attn_decode_quant(const void* q, const void* k_codes, const void* v_codes, const float* k_params,
                           const float* v_params, const int* lens, void* o, float* lse, int window,
                           const float* slopes, int B, int s_max, int H, int Hk, int D, int bits, int group_size,
                           float scale, int is_bf16, void* ws, size_t ws_bytes, void* stream) {
  int rc;
  if ((rc = check_quant_format("attn_decode_quant", B, s_max, Hk, D, bits, group_size))) return rc;
  B200_CHECK_ARG(H > 0 && H % Hk == 0, "attn_decode_quant: H=%d must be a multiple of Hk=%d", H, Hk);
  B200_CHECK_ARG(s_max >= DEC_TILE, "attn_decode_quant: s_max=%d must be >= %d", s_max, DEC_TILE);
  const int G = H / Hk;
  B200_CHECK_ARG(G * D <= DEC_MAX_ITEMS * DEC_THREADS * 8, "attn_decode_quant: (H/Hk) * D = %d exceeds %d", G * D,
                 DEC_MAX_ITEMS * DEC_THREADS * 8);
  B200_CHECK_ARG(al16(q) && al16(o) && lens != nullptr, "attn_decode_quant: q / o must be 16-byte aligned, lens non-null");
  B200_CHECK_ARG(slopes == nullptr || (reinterpret_cast<uintptr_t>(slopes) & 3u) == 0,
                 "attn_decode_quant: slopes must be a 4-byte aligned fp32 [H] array");
  const size_t need = b200_attn_decode_workspace_bytes(B, H, s_max, D);
  if (ws_bytes < need || (need > 0 && ws == nullptr)) {
    set_error("attn_decode_quant: workspace of %zu bytes, %zu needed", ws_bytes, need);
    return B200_ERR_WORKSPACE;
  }
  const int Dc = D * bits / 8, ng = D / group_size;
  const uint64_t cdims[4] = {(uint64_t)Dc, (uint64_t)Hk, (uint64_t)s_max, (uint64_t)B};
  const uint64_t cstrides[3] = {(uint64_t)Dc, (uint64_t)Hk * Dc, (uint64_t)s_max * Hk * Dc};
  const uint32_t cbox[4] = {(uint32_t)Dc, 1, (uint32_t)DEC_TILE, 1};
  // parameters as [B, Hk, s_max * ng * 2] floats: a tile's block is one box (qdec_param_positions)
  const uint64_t pdims[3] = {(uint64_t)s_max * ng * 2, (uint64_t)Hk, (uint64_t)B};
  const uint64_t pstrides[2] = {(uint64_t)s_max * ng * 8, (uint64_t)Hk * s_max * ng * 8};
  const uint32_t pbox[3] = {(uint32_t)(qdec_param_positions(ng) * ng * 2), 1, 1};
  CUtensorMap tm[4];
  if ((rc = make_tensor_map(&tm[0], k_codes, CU_TENSOR_MAP_DATA_TYPE_UINT8, 1, 4, cdims, cstrides, cbox, false))) return rc;
  if ((rc = make_tensor_map(&tm[1], v_codes, CU_TENSOR_MAP_DATA_TYPE_UINT8, 1, 4, cdims, cstrides, cbox, false))) return rc;
  if ((rc = make_tensor_map(&tm[2], k_params, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 4, 3, pdims, pstrides, pbox, false)))
    return rc;
  if ((rc = make_tensor_map(&tm[3], v_params, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 4, 3, pdims, pstrides, pbox, false)))
    return rc;
  DecArgs a;
  a.q = q;
  a.o = o;
  a.lse = lse;
  a.lens = lens;
  a.max_chunks = (s_max + DEC_CHUNK - 1) / DEC_CHUNK;
  a.part_acc = reinterpret_cast<float*>(ws);
  a.part_ml = a.part_acc + (size_t)B * H * a.max_chunks * D;
  a.H = H;
  a.G = G;
  a.s_max = s_max;
  a.scale_log2 = scale * kLog2e;
  a.window = window < 0 || window > s_max ? s_max : window;
  a.slopes = slopes;
  const cudaStream_t s = static_cast<cudaStream_t>(stream);
  if (is_bf16)
    return bits == 8 ? launch_decode_quant_d<__nv_bfloat16, 8>(D, tm, a, group_size, B, Hk, s)
                     : launch_decode_quant_d<__nv_bfloat16, 4>(D, tm, a, group_size, B, Hk, s);
  return bits == 8 ? launch_decode_quant_d<float, 8>(D, tm, a, group_size, B, Hk, s)
                   : launch_decode_quant_d<float, 4>(D, tm, a, group_size, B, Hk, s);
}

}  // extern "C"
