// Batched bf16 GEMM engine on Hopper warpgroup MMA (wgmma) fed by TMA through an mbarrier ring.
//
// Persistent and warp-specialised: the grid is min(work items, SMs) CTAs and CTA c walks work items
// c, c + gridDim.x, ... of the concatenated list of every problem of the launch (grouped GEMM).
//   warpgroup 0     producer: one thread streams A[128 x 64] + B[128 x 64] k-blocks (128B-swizzled TMA boxes)
//                   into a 5-stage ring (32 KB per stage).  Ring slot and phase run on across work items, so the
//                   next tile's loads start while the current one is still being multiplied.
//   warpgroups 1-2  consumers, ping-pong: each owns a whole 128 x 128 tile (two wgmma.m64n128k16 per k16 step,
//                   128 fp32 accumulators per thread) and they take the CTA's work items in turn.  A pair of
//                   named barriers orders their mainloops, so one warpgroup's epilogue runs while the other
//                   keeps the tensor cores busy.  A stage is handed back once the wgmma batch that read it has
//                   retired, so one batch is always in flight behind the next TMA wait.
//   epilogue        bf16 outputs go through a 32 KB shared-memory tile per consumer, laid out as TMA boxes: the
//                   accumulators go in with stmatrix and leave as bulk tensor stores issued by one thread, which
//                   drain while the warpgroup runs its next mainloop.  Epilogue inputs (C for beta != 0, the saved
//                   GLU activations of the adjoint) are loaded into the tile by the producer right after the
//                   tile's k-blocks, so they land while the tile's own MMAs run.  This covers alpha/beta/C, the
//                   symmetric-output mirror (stmatrix.trans), and the two fused MLP epilogues; peer copies are
//                   written from the tile as 16-byte rows.  fp32 outputs and split-K partials are stored straight
//                   from the accumulators.
// Operand layouts (K-major or MN-major for A and for B) are per-problem run-time flags: they select the TMA
// box shape and the transpose bits of the wgmma instruction.  Grouped launches are how the Newton-Schulz chain
// runs each stage over all shape groups at once.
#include "common.cuh"
#include "host.h"

namespace b200 {

namespace {

constexpr int BM = 128, BN = 128, BK = 64;
constexpr int STAGES = 5;
constexpr int THREADS = 384;
constexpr int A_BYTES = BM * BK * 2;  // 16 KB
constexpr int B_BYTES = BN * BK * 2;  // 16 KB
constexpr int STAGE_BYTES = A_BYTES + B_BYTES;
constexpr int OUT_BYTES = BM * BN * 2;  // bf16 staging tile of one consumer warpgroup
constexpr int HALF_BYTES = BM * 128;    // one [128 rows x 64 columns] half of it
constexpr int BOX_BYTES = 64 * 128;     // one [64 x 64] TMA box of the epilogue tensor maps
constexpr int SMEM_BYTES = STAGES * STAGE_BYTES + 2 * OUT_BYTES + 1024 + 256;
static_assert(SMEM_BYTES <= 227 * 1024, "shared memory budget of one block");
constexpr int MAX_PROBLEMS = 6;
constexpr int MAX_PEERS = 7;
constexpr int GROUP_M = 8;  // tile raster: 8 row blocks sweep the columns together (L2 reuse of B)
// named barriers: 1 + c = "consumer c may start its mainloop", 3 + c = consumer c's own warpgroup barrier
constexpr uint32_t BAR_ORDER = 1, BAR_WG = 3;

struct Problem {
  int M, N, K, batch;
  int tiles_m, tiles_n, tiles_per_batch, num_kb;
  int work_begin;  // first work item of this problem in the concatenated list
  int a_mn, b_mn, symmetric, k_splits, n_peers, out_f32;
  int epi;         // 0 plain | 1 gate/up + GLU forward | 2 down dgrad + GLU adjoint
  int n_store;     // columns written per row: N rounded up to the store vector
  float alpha, beta;
  const float* alpha_vec;
  const float* beta_vec;
  const void* C;
  long long ldc, strideC;
  void* D;
  long long ldd, strideD;
  float* ws;  // split-K fp32 slabs [k_splits][batch][M][N]
  void* peer_D[MAX_PEERS];
  int glu_I;
  void* aux;  // epi 1: y [M, I] (written); epi 2: gu [M, 2I] (read)
  long long ld_aux;
};

struct Args {
  int n_problems, total_work;
  Problem p[MAX_PROBLEMS];
  CUtensorMap tmA[MAX_PROBLEMS];
  CUtensorMap tmB[MAX_PROBLEMS];
  CUtensorMap tmD[MAX_PROBLEMS];  // bf16 D (plain), gu (epi 1) or dgu (epi 2); unset for fp32 / split-K outputs
  CUtensorMap tmE[MAX_PROBLEMS];  // C (plain, beta != 0), y (epi 1) or the saved gu (epi 2)
};
// sm_90 with CUDA >= 12.1 takes up to 32764 bytes of kernel parameters (4096 before)
static_assert(sizeof(Args) <= 32764, "kernel parameter block");

__device__ __forceinline__ void tile_coords(const Problem& p, int r, int& mi, int& ni) {
  if (p.symmetric) {  // upper triangle, row by row
    int row = 0, len = p.tiles_n;
    while (r >= len) {
      r -= len;
      ++row;
      --len;
    }
    mi = row;
    ni = row + r;
    return;
  }
  const int per_group = GROUP_M * p.tiles_n;
  const int first_m = (r / per_group) * GROUP_M;
  const int gsize = min(p.tiles_m - first_m, GROUP_M);
  const int rr = r % per_group;
  mi = first_m + rr % gsize;
  ni = rr / gsize;
}

struct Item {
  int pi, split, b, mi, ni, kb_begin, kb_end;
};

__device__ __forceinline__ int problem_of(const Args& g, int w) {
  int pi = 0;
#pragma unroll
  for (int i = 1; i < MAX_PROBLEMS; ++i)
    if (i < g.n_problems && w >= g.p[i].work_begin) pi = i;
  return pi;
}

// k-block range of work item w (split s of its tile covers [s * kb_per, min(num_kb, (s + 1) * kb_per)))
__device__ __forceinline__ void kb_range(const Problem& p, int split, int& kb_begin, int& kb_end) {
  const int kb_per = (p.num_kb + p.k_splits - 1) / p.k_splits;
  kb_begin = split * kb_per;
  kb_end = min(p.num_kb, kb_begin + kb_per);
}

__device__ __forceinline__ Item decode(const Args& g, int w) {
  Item it;
  it.pi = problem_of(g, w);
  const Problem& p = g.p[it.pi];
  int r = w - p.work_begin;
  it.split = r % p.k_splits;
  r /= p.k_splits;
  it.b = r / p.tiles_per_batch;
  tile_coords(p, r - it.b * p.tiles_per_batch, it.mi, it.ni);
  kb_range(p, it.split, it.kb_begin, it.kb_end);
  return it;
}

__device__ __forceinline__ int item_kbs(const Args& g, int w) {
  const Problem& p = g.p[problem_of(g, w)];
  int kb_begin, kb_end;
  kb_range(p, (w - p.work_begin) % p.k_splits, kb_begin, kb_end);
  return max(kb_end - kb_begin, 0);
}

// sigmoid with one special-function op: sigmoid(x) = 0.5 + 0.5 tanh(x / 2)
__device__ __forceinline__ float fast_sigmoid(float x) {
  float t;
  asm("tanh.approx.f32 %0, %1;" : "=f"(t) : "f"(0.5f * x));
  return fmaf(0.5f, t, 0.5f);
}

// One tile's k-blocks [kb_begin, kb_end) from the ring: acc[0, 64) = rows [0, 64), acc[64, 128) = rows [64, 128).
template <int TA, int TB>
__device__ __forceinline__ void mainloop(float* acc, uint32_t sbase, uint32_t full0, uint32_t empty0, int n_kb,
                                         int& slot, uint32_t& phase, bool leader) {
  int prev = -1;
  for (int i = 0; i < n_kb; ++i) {
    mbar_wait(full0 + 8 * slot, phase);
    const uint32_t sA = sbase + slot * STAGE_BYTES, sB = sA + A_BYTES;
    wgmma_fence();
    // per k16 step: K-major operands advance 32 B inside the swizzled row, MN-major ones 16 rows of 128 B
#pragma unroll
    for (int k = 0; k < BK / 16; ++k) {
      const uint64_t db = make_wgmma_desc_sw128(sB + k * (TB ? 2048 : 32), 8192, 1024);
      const uint64_t da0 = make_wgmma_desc_sw128(sA + k * (TA ? 2048 : 32), 8192, 1024);
      const uint64_t da1 = make_wgmma_desc_sw128(sA + 8192 + k * (TA ? 2048 : 32), 8192, 1024);
      wgmma_m64n128k16_ss<TA, TB>(acc, da0, db);
      wgmma_m64n128k16_ss<TA, TB>(acc + 64, da1, db);
    }
    wgmma_commit();
    wgmma_wait<1>();
    if (prev >= 0 && leader) mbar_arrive(empty0 + 8 * prev);
    prev = slot;
    if (++slot == STAGES) {
      slot = 0;
      phase ^= 1u;
    }
  }
  wgmma_wait<0>();
  if (prev >= 0 && leader) mbar_arrive(empty0 + 8 * prev);
}

// Staging tile: two [128 rows x 64 columns] halves of 128-byte rows in the TMA SWIZZLE_128B pattern (16-byte chunk c
// of row r at c ^ (r & 7)), so the epilogue tensor maps load into it and store from it directly, and the eight rows of
// an 8x8 stmatrix / ldmatrix hit distinct banks.  `chunk` in [0, 16) counts 8-column groups across both halves; the
// [64 x 64] box (column half h, row half v) starts at h * HALF_BYTES + v * BOX_BYTES.
__device__ __forceinline__ uint32_t stage_off(int row, int chunk) {
  return (chunk >> 3) * HALF_BYTES + row * 128 + (((chunk & 7) ^ (row & 7)) << 4);
}

// Row addresses of the x4 matrix group (h = 0/1 row halves of 8, column groups j0, j0 + 1) of warp `warp`
// at tile row offset `row0`; lane 8i + rr addresses row rr of matrix i.
__device__ __forceinline__ uint32_t frag_addr(uint32_t stg, int row0, int warp, int j0, int lane) {
  const int mi = lane >> 3, rr = lane & 7;
  return stg + stage_off(row0 + 16 * warp + 8 * (mi & 1) + rr, j0 + (mi >> 1));
}
// The same matrices stored transposed: fragment column 8j + c becomes staging row 8j + c.
__device__ __forceinline__ uint32_t frag_addr_trans(uint32_t stg, int row0, int warp, int j0, int lane) {
  const int mi = lane >> 3, rr = lane & 7;
  return stg + stage_off(8 * (j0 + (mi >> 1)) + rr, (row0 >> 3) + 2 * warp + (mi & 1));
}

// Whether a problem's epilogue reads an input into the staging tile (C of a bf16 output, the saved gu of epi 2).
__device__ __forceinline__ bool epi_input(const Problem& p) { return p.epi == 2 || (p.C != nullptr && !p.out_f32); }

// The whole [128 x 128] tile at column col0, row row0 of batch b as four 64 x 64 boxes (loads complete on `bar`).
__device__ __forceinline__ void tile_load(const CUtensorMap* m, uint32_t stg, uint32_t bar, int col0, int row0, int b) {
#pragma unroll
  for (int h = 0; h < 2; ++h)
#pragma unroll
    for (int v = 0; v < 2; ++v) tma_load_3d(stg + h * HALF_BYTES + v * BOX_BYTES, m, bar, col0 + 64 * h, row0 + 64 * v, b);
}
__device__ __forceinline__ void tile_store(const CUtensorMap* m, uint32_t stg, int col0, int row0, int b) {
#pragma unroll
  for (int h = 0; h < 2; ++h)
#pragma unroll
    for (int v = 0; v < 2; ++v) tma_store_3d(m, stg + h * HALF_BYTES + v * BOX_BYTES, col0 + 64 * h, row0 + 64 * v, b);
}
// Epi 2's half tile: 128 columns from col0 of 64 rows from row0, g in staging rows [0, 64) and u in [64, 128); the
// {I, 2, M} view of gu / dgu clips at column I, so a box never reaches from g into u.
__device__ __forceinline__ void glu_half_load(const CUtensorMap* m, uint32_t stg, uint32_t bar, int col0, int row0) {
#pragma unroll
  for (int h = 0; h < 2; ++h)
#pragma unroll
    for (int gu = 0; gu < 2; ++gu) tma_load_3d(stg + h * HALF_BYTES + gu * BOX_BYTES, m, bar, col0 + 64 * h, gu, row0);
}
__device__ __forceinline__ void glu_half_store(const CUtensorMap* m, uint32_t stg, int col0, int row0) {
#pragma unroll
  for (int h = 0; h < 2; ++h)
#pragma unroll
    for (int gu = 0; gu < 2; ++gu) tma_store_3d(m, stg + h * HALF_BYTES + gu * BOX_BYTES, col0 + 64 * h, gu, row0);
}

// Closes a bulk group of the leader's stores.  `drain` after the warpgroup's last tile: the CTA's shared memory must
// outlive the stores reading it.
__device__ __forceinline__ void commit_stores(bool drain) {
  bulk_commit();
  if (drain) bulk_wait<0>();
}

__global__ void __launch_bounds__(THREADS, 1) gemm_wgmma_kernel(const __grid_constant__ Args g) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  const uint32_t sbase = smem_u32(smem);
  const uint32_t full0 = sbase + STAGES * STAGE_BYTES + 2 * OUT_BYTES;
  const uint32_t empty0 = full0 + STAGES * 8;
  // per consumer c: epi_full0 + 8c = its staging tile holds the epilogue input, epi_empty0 + 8c = the tile may be
  // refilled (the consumer's earlier stores have read it)
  const uint32_t epi_full0 = empty0 + STAGES * 8;
  const uint32_t epi_empty0 = epi_full0 + 16;
  const int wg = threadIdx.x >> 7;

  if (threadIdx.x == 0) {
    for (int s = 0; s < STAGES; ++s) {
      mbar_init(full0 + 8 * s, 1);
      mbar_init(empty0 + 8 * s, 1);  // one arrival by the consumer warpgroup that read the stage
    }
    for (int c = 0; c < 2; ++c) {
      mbar_init(epi_full0 + 8 * c, 1);
      mbar_init(epi_empty0 + 8 * c, 1);
    }
    fence_mbar_init();
  }
  __syncthreads();

  if (wg == 0) {
    setmaxnreg_dec<40>();
    if (threadIdx.x == 0) {
      for (int i = 0; i < g.n_problems; ++i) {
        tma_prefetch_desc(&g.tmA[i]);
        tma_prefetch_desc(&g.tmB[i]);
      }
      int slot = 0;
      uint32_t phase = 0, epi_phase = 0;  // epi_phase bit c: parity of consumer c's next epi_empty completion
      for (int w = blockIdx.x, t = 0; w < g.total_work; w += gridDim.x, ++t) {
        const Item it = decode(g, w);
        const Problem& p = g.p[it.pi];
        const CUtensorMap* tmA = &g.tmA[it.pi];
        const CUtensorMap* tmB = &g.tmB[it.pi];
        const int mi = it.mi, ni = it.ni, b = it.b;
        for (int kb = it.kb_begin; kb < it.kb_end; ++kb) {
          mbar_wait(empty0 + 8 * slot, phase ^ 1u);
          const uint32_t full = full0 + 8 * slot;
          mbar_arrive_expect_tx(full, STAGE_BYTES);
          const uint32_t sA = sbase + slot * STAGE_BYTES, sB = sA + A_BYTES;
          const int k0 = kb * BK;
          if (p.a_mn) {  // two [64 k-rows x 64 m] boxes
            tma_load_3d(sA, tmA, full, mi * BM, k0, b);
            tma_load_3d(sA + 8192, tmA, full, mi * BM + 64, k0, b);
          } else {
            tma_load_3d(sA, tmA, full, k0, mi * BM, b);
          }
          if (p.epi == 1) {  // 64 gate rows of W2, then the same 64 up rows
            tma_load_3d(sB, tmB, full, k0, ni * 64, b);
            tma_load_3d(sB + 8192, tmB, full, k0, p.glu_I + ni * 64, b);
          } else if (p.b_mn) {
            tma_load_3d(sB, tmB, full, ni * BN, k0, b);
            tma_load_3d(sB + 8192, tmB, full, ni * BN + 64, k0, b);
          } else {
            tma_load_3d(sB, tmB, full, k0, ni * BN, b);
          }
          if (++slot == STAGES) {
            slot = 0;
            phase ^= 1u;
          }
        }
        if (epi_input(p)) {  // into the owning consumer's staging tile, once its previous stores have read it
          const int c = t & 1;
          mbar_wait(epi_empty0 + 8 * c, (epi_phase >> c) & 1u);
          epi_phase ^= 1u << c;
          const uint32_t stg = sbase + STAGES * STAGE_BYTES + c * OUT_BYTES, bar = epi_full0 + 8 * c;
          mbar_arrive_expect_tx(bar, OUT_BYTES);
          if (p.epi == 2) glu_half_load(&g.tmE[it.pi], stg, bar, ni * BN, mi * BM);  // first 64-row half
          else tile_load(&g.tmE[it.pi], stg, bar, ni * BN, mi * BM, b);
        }
      }
    }
    return;
  }

  setmaxnreg_inc<232>();
  const int c = wg - 1;
  const int tid = threadIdx.x & 127, lane = threadIdx.x & 31, warp = tid >> 5;
  const uint32_t stg = sbase + STAGES * STAGE_BYTES + c * OUT_BYTES;
  const uint32_t bar_wg = BAR_WG + c;
  const uint32_t epi_full = epi_full0 + 8 * c;
  // thread 0 of the warpgroup hands ring stages back and issues (and so owns) the warpgroup's bulk stores
  const bool leader = tid == 0;
  int slot = 0;
  uint32_t phase = 0, epi_phase = 0;
  for (int w = blockIdx.x, t = 0; w < g.total_work; w += gridDim.x, ++t) {
    if ((t & 1) != c) {  // the other warpgroup's tile: step the ring past its k-blocks
      const int n = slot + item_kbs(g, w);
      phase ^= (uint32_t)(n / STAGES) & 1u;
      slot = n % STAGES;
      continue;
    }
    const Item it = decode(g, w);
    const Problem& p = g.p[it.pi];
    const int mi = it.mi, ni = it.ni, b = it.b;
    const bool last = w + 2 * (int)gridDim.x >= g.total_work;  // this warpgroup's last tile

    float acc[128];
#pragma unroll
    for (int i = 0; i < 128; ++i) acc[i] = 0.f;
    if (t > 0) named_bar_sync(BAR_ORDER + c, 256);  // the other warpgroup's mainloop is done
    if (epi_input(p) && leader) {  // every thread is past the last tile's epilogue: free the staging tile
      bulk_wait_read<0>();
      mbar_arrive(epi_empty0 + 8 * c);
    }
    const int n_kb = max(it.kb_end - it.kb_begin, 0);
    if (p.a_mn) {
      if (p.b_mn) mainloop<1, 1>(acc, sbase, full0, empty0, n_kb, slot, phase, leader);
      else mainloop<1, 0>(acc, sbase, full0, empty0, n_kb, slot, phase, leader);
    } else {
      if (p.b_mn) mainloop<0, 1>(acc, sbase, full0, empty0, n_kb, slot, phase, leader);
      else mainloop<0, 0>(acc, sbase, full0, empty0, n_kb, slot, phase, leader);
    }
    if (w + (int)gridDim.x < g.total_work) named_bar_arrive(BAR_ORDER + (c ^ 1), 256);

    // accumulator fragment: acc[64 hm + 4 j + 2 h + e] = tile (64 hm + 16 warp + 8 h + lane / 4, 8 j + cq + e)
    const int cq = (lane & 3) * 2;
    const int rq = 16 * warp + (lane >> 2);

    if (p.k_splits > 1 || p.out_f32) {  // fp32 results straight from the accumulators
      const float alpha = p.k_splits > 1 ? 1.0f : p.alpha * (p.alpha_vec ? p.alpha_vec[b] : 1.0f);
      const float beta = p.beta * (p.beta_vec ? p.beta_vec[b] : 1.0f);
      float* Db;
      long long ld;
      const float* Cb = nullptr;
      int n_cols;
      if (p.k_splits > 1) {  // raw partial of this K range
        Db = p.ws + ((long long)it.split * p.batch + b) * p.M * (long long)p.N;
        ld = p.N;
        n_cols = p.N;
      } else {
        Db = reinterpret_cast<float*>(p.D) + (long long)b * p.strideD;
        ld = p.ldd;
        n_cols = p.n_store;
        if (p.C) Cb = reinterpret_cast<const float*>(p.C) + (long long)b * p.strideC;
      }
#pragma unroll
      for (int hm = 0; hm < 2; ++hm)
#pragma unroll
        for (int j = 0; j < 16; ++j) {
          const int col = ni * BN + 8 * j + cq;
          if (col >= n_cols) continue;
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            const int row = mi * BM + 64 * hm + rq + 8 * h;
            if (row >= p.M) continue;
            float v0 = acc[64 * hm + 4 * j + 2 * h], v1 = acc[64 * hm + 4 * j + 2 * h + 1];
            if (p.k_splits <= 1) {
              v0 = alpha * v0;
              v1 = alpha * v1;
              if (Cb) {
                const float2 cv = *reinterpret_cast<const float2*>(Cb + (long long)row * p.ldc + col);
                v0 += beta * cv.x;
                v1 += beta * cv.y;
              }
            }
            *reinterpret_cast<float2*>(Db + (long long)row * ld + col) = make_float2(v0, v1);
          }
        }
      if (last) bulk_wait<0>();  // stores of an earlier bf16 tile of a grouped launch
      continue;
    }

    const CUtensorMap* tmD = &g.tmD[it.pi];
    const CUtensorMap* tmE = &g.tmE[it.pi];
    const bool has_input = epi_input(p);
    if (!has_input) {  // this warpgroup's previous stores have left the staging tile
      if (leader) bulk_wait_read<0>();
      named_bar_sync(bar_wg, 128);
    }

    if (p.epi == 1) {  // acc columns [0, 64) = gate, [64, 128) = up of the same 64 output columns
#pragma unroll
      for (int hm = 0; hm < 2; ++hm)
#pragma unroll
        for (int j = 0; j < 16; j += 2) {
          const float* a = acc + 64 * hm + 4 * j;
          stmatrix_x4(frag_addr(stg, 64 * hm, warp, j, lane), pack_bf16x2(a[0], a[1]), pack_bf16x2(a[2], a[3]),
                      pack_bf16x2(a[4], a[5]), pack_bf16x2(a[6], a[7]));
        }
      fence_proxy_async_smem();
      named_bar_sync(bar_wg, 128);
      if (leader) {  // staging half 0 = gate columns, half 1 = the up columns I later
#pragma unroll
        for (int gu = 0; gu < 2; ++gu) {
          tma_store_3d(tmD, stg + gu * HALF_BYTES, ni * 64, gu, mi * BM);
          tma_store_3d(tmD, stg + gu * HALF_BYTES + BOX_BYTES, ni * 64, gu, mi * BM + 64);
          commit_stores(last);
        }
        bulk_wait_read<1>();  // the gate half has been read: y goes there
      }
      named_bar_sync(bar_wg, 128);
#pragma unroll
      for (int hm = 0; hm < 2; ++hm)
#pragma unroll
        for (int j = 0; j < 8; j += 2) {  // y = g sigmoid(u) 2 from the fp32 accumulators
          const float* g = acc + 64 * hm + 4 * j;
          const float* u = g + 32;
          uint32_t yv[4];
#pragma unroll
          for (int q = 0; q < 4; ++q)
            yv[q] = pack_bf16x2(g[2 * q] * fast_sigmoid(u[2 * q]) * 2.0f, g[2 * q + 1] * fast_sigmoid(u[2 * q + 1]) * 2.0f);
          stmatrix_x4(frag_addr(stg, 64 * hm, warp, j, lane), yv[0], yv[1], yv[2], yv[3]);
        }
      fence_proxy_async_smem();
      named_bar_sync(bar_wg, 128);
      if (leader) {
        tma_store_3d(tmE, stg, ni * 64, mi * BM, 0);
        tma_store_3d(tmE, stg + BOX_BYTES, ni * 64, mi * BM + 64, 0);
        commit_stores(last);
      }
      continue;
    }

    if (p.epi == 2) {  // acc = d = dy Wd; dg = d s 2, du = d g s (1 - s) 2 with g, u from the saved gu
#pragma unroll
      for (int hm = 0; hm < 2; ++hm) {  // staging rows [0, 64): g, [64, 128): u of tile rows [64 hm, 64 hm + 64)
        if (hm && leader) {  // the producer loaded the first half; load the second once its stores have read the tile
          bulk_wait_read<0>();
          mbar_arrive_expect_tx(epi_full, OUT_BYTES);
          glu_half_load(tmE, stg, epi_full, ni * BN, mi * BM + 64);
        }
        mbar_wait_outlined(epi_full, epi_phase);
        epi_phase ^= 1u;
#pragma unroll
        for (int j = 0; j < 16; j += 2) {  // each warp reads and rewrites only its own 16 rows: in place
          const uint32_t ga = frag_addr(stg, 0, warp, j, lane), ua = frag_addr(stg, 64, warp, j, lane);
          uint32_t gq[4], uq[4], dg[4], du[4];
          ldmatrix_x4(ga, gq);
          ldmatrix_x4(ua, uq);
#pragma unroll
          for (int q = 0; q < 4; ++q) {  // q = (column group j + q / 2, row half q % 2)
            const float* a = acc + 64 * hm + 4 * (j + (q >> 1)) + 2 * (q & 1);
            const float2 gg = unpack_bf16x2(gq[q]), uu = unpack_bf16x2(uq[q]);
            const float d0 = a[0], d1 = a[1];
            const float s0 = fast_sigmoid(uu.x), s1 = fast_sigmoid(uu.y);
            dg[q] = pack_bf16x2(d0 * s0 * 2.0f, d1 * s1 * 2.0f);
            du[q] = pack_bf16x2(d0 * gg.x * s0 * (1.0f - s0) * 2.0f, d1 * gg.y * s1 * (1.0f - s1) * 2.0f);
          }
          __syncwarp();
          stmatrix_x4(ga, dg[0], dg[1], dg[2], dg[3]);
          stmatrix_x4(ua, du[0], du[1], du[2], du[3]);
        }
        fence_proxy_async_smem();
        named_bar_sync(bar_wg, 128);
        if (leader) {
          glu_half_store(tmD, stg, ni * BN, mi * BM + 64 * hm);
          commit_stores(last);
        }
      }
      continue;
    }

    // ---- plain bf16: D = alpha acc + beta C, optional mirror and peer copies ----
    const float alpha = p.alpha * (p.alpha_vec ? p.alpha_vec[b] : 1.0f);
    const float beta = p.beta * (p.beta_vec ? p.beta_vec[b] : 1.0f);
    if (has_input) {  // C, loaded by the producer under this tile's MMAs
      mbar_wait_outlined(epi_full, epi_phase);
      epi_phase ^= 1u;
    }
    uint32_t dv[2][8][4];  // the tile as packed bf16 pairs, kept for the mirror
#pragma unroll
    for (int hm = 0; hm < 2; ++hm)
#pragma unroll
      for (int jp = 0; jp < 8; ++jp) {  // each warp reads and rewrites only its own 16 rows: in place
        const uint32_t fa = frag_addr(stg, 64 * hm, warp, 2 * jp, lane);
        uint32_t cq4[4];
        if (has_input) ldmatrix_x4(fa, cq4);
#pragma unroll
        for (int q = 0; q < 4; ++q) {
          const float* a = acc + 64 * hm + 4 * (2 * jp + (q >> 1)) + 2 * (q & 1);
          float v0 = alpha * a[0], v1 = alpha * a[1];
          if (has_input) {
            const float2 cv = unpack_bf16x2(cq4[q]);
            v0 += beta * cv.x;
            v1 += beta * cv.y;
          }
          dv[hm][jp][q] = pack_bf16x2(v0, v1);
        }
        __syncwarp();
        stmatrix_x4(fa, dv[hm][jp][0], dv[hm][jp][1], dv[hm][jp][2], dv[hm][jp][3]);
      }
    fence_proxy_async_smem();
    named_bar_sync(bar_wg, 128);
    if (leader) {
      tile_store(tmD, stg, ni * BN, mi * BM, b);
      commit_stores(last);
    }
    if (p.n_peers) {  // peer-mapped copies of D, as 16-byte rows
#pragma unroll 4
      for (int i = 0; i < 16; ++i) {
        const int idx = i * 128 + tid, r = idx >> 4, k = idx & 15;
        const int row = mi * BM + r, col = ni * BN + 8 * k;
        if (row >= p.M || col >= p.n_store) continue;
        const uint4 v = lds128(stg + stage_off(r, k));
        const long long od = (long long)b * p.strideD + (long long)row * p.ldd + col;
        for (int pe = 0; pe < p.n_peers; ++pe) stg128(reinterpret_cast<__nv_bfloat16*>(p.peer_D[pe]) + od, v);
      }
    }
    if (p.symmetric && mi != ni) {  // D == D^T: block (ni, mi) is this tile transposed
      if (leader) bulk_wait_read<0>();
      named_bar_sync(bar_wg, 128);
#pragma unroll
      for (int hm = 0; hm < 2; ++hm)
#pragma unroll
        for (int jp = 0; jp < 8; ++jp)
          stmatrix_x4_trans(frag_addr_trans(stg, 64 * hm, warp, 2 * jp, lane), dv[hm][jp][0], dv[hm][jp][1],
                            dv[hm][jp][2], dv[hm][jp][3]);
      fence_proxy_async_smem();
      named_bar_sync(bar_wg, 128);
      // staging row r = column ni BN + r of D, staging column = row mi BM + col.  Both entries reject symmetric
      // output unless M == N is a multiple of 8, so the map's bounds clip the mirror exactly.
      if (leader) {
        tile_store(tmD, stg, mi * BM, ni * BN, b);
        commit_stores(last);
      }
    }
  }
}

// Split-K epilogue: D = bf16(alpha * sum_s ws[s]) in a fixed summation order (deterministic), with the
// symmetric mode's mirror writes.
__global__ void __launch_bounds__(256)
splitk_finalize_kernel(const float* __restrict__ ws, int splits, int batch, int M, int N, __nv_bfloat16* D,
                       long long ldd, long long strideD, float alpha, const float* __restrict__ alpha_vec,
                       int symmetric) {
  const int b = blockIdx.z;
  const int i = blockIdx.x * 32 + (threadIdx.x & 31);
  const int j0 = (blockIdx.y * 8 + (threadIdx.x >> 5)) * 8;
  if (i >= M || j0 >= N) return;
  const int ti = i / BM, tj = j0 / BN;
  if (symmetric && ti > tj) return;
  float acc[8] = {0, 0, 0, 0, 0, 0, 0, 0};
  for (int s = 0; s < splits; ++s) {
    const float* src = ws + (((long long)s * batch + b) * M + i) * (long long)N + j0;
    const float4 v0 = *reinterpret_cast<const float4*>(src);
    const float4 v1 = *reinterpret_cast<const float4*>(src + 4);
    acc[0] += v0.x; acc[1] += v0.y; acc[2] += v0.z; acc[3] += v0.w;
    acc[4] += v1.x; acc[5] += v1.y; acc[6] += v1.z; acc[7] += v1.w;
  }
  const float a = alpha * (alpha_vec ? alpha_vec[b] : 1.0f);
  uint4 o;
  o.x = pack_bf16x2(a * acc[0], a * acc[1]);
  o.y = pack_bf16x2(a * acc[2], a * acc[3]);
  o.z = pack_bf16x2(a * acc[4], a * acc[5]);
  o.w = pack_bf16x2(a * acc[6], a * acc[7]);
  __nv_bfloat16* dbase = D + (long long)b * strideD;
  stg128(dbase + (long long)i * ldd + j0, o);
  if (symmetric && ti != tj) {
    const uint32_t w[4] = {o.x, o.y, o.z, o.w};
#pragma unroll
    for (int t = 0; t < 8; ++t) {
      const uint16_t h = (t & 1) ? (uint16_t)(w[t >> 1] >> 16) : (uint16_t)(w[t >> 1] & 0xffffu);
      *reinterpret_cast<uint16_t*>(dbase + (long long)(j0 + t) * ldd + i) = h;
    }
  }
}

// TMA map of one bf16 operand: K-major -> dims {K, rows, batch}, box {64, box_rows};
// MN-major -> dims {rows, K, batch}, box {64, 64} (two boxes cover a 128-wide tile).
int operand_map(CUtensorMap* m, const void* base, bool mn, int rows, int K, int batch, long long ld,
                long long stride, int box_rows) {
  const uint64_t dims[3] = {(uint64_t)(mn ? rows : K), (uint64_t)(mn ? K : rows), (uint64_t)batch};
  const uint64_t strides[2] = {(uint64_t)ld * 2, (uint64_t)(batch > 1 ? stride : (long long)dims[1] * ld) * 2};
  const uint32_t box[3] = {64, (uint32_t)(mn ? 64 : box_rows), 1};
  return make_tensor_map(m, base, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, 3, dims, strides, box, true);
}

// TMA map of a bf16 epilogue tile (D, C, y): dims {cols, rows, batch}, 128B-swizzled 64 x 64 boxes, so each half
// of the staging tile is two boxes.  `cols` is the stored width (N rounded up to 8 for D): the padded columns of a
// ragged output are written, and rows >= `rows` are clipped.
int tile_map(CUtensorMap* m, const void* base, int cols, int rows, int batch, long long ld, long long stride) {
  const uint64_t dims[3] = {(uint64_t)cols, (uint64_t)rows, (uint64_t)batch};
  const uint64_t strides[2] = {(uint64_t)ld * 2, (uint64_t)(batch > 1 ? stride : (long long)rows * ld) * 2};
  const uint32_t box[3] = {64, 64, 1};
  return make_tensor_map(m, base, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, 3, dims, strides, box, true);
}
// TMA map of the GLU activations gu / dgu [M, 2I] (row pitch ld) viewed as {I, 2 (gate, up), M}, boxes of 64 columns
// by 64 rows: column I clips a box instead of running into the other half.
int glu_map(CUtensorMap* m, const void* base, int I, int M, long long ld) {
  const uint64_t dims[3] = {(uint64_t)I, 2, (uint64_t)M};
  const uint64_t strides[2] = {(uint64_t)I * 2, (uint64_t)ld * 2};
  const uint32_t box[3] = {64, 1, 64};
  return make_tensor_map(m, base, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, 3, dims, strides, box, true);
}

// The bf16 epilogue's maps of a plain problem: D and, when beta != 0, C.
int plain_epi_maps(Args& a, int i) {
  const Problem& q = a.p[i];
  if (q.out_f32 || q.k_splits > 1) return B200_OK;
  int rc = tile_map(&a.tmD[i], q.D, q.n_store, q.M, q.batch, q.ldd, q.strideD);
  if (rc == B200_OK && q.C) rc = tile_map(&a.tmE[i], q.C, q.n_store, q.M, q.batch, q.ldc, q.strideC);
  return rc;
}

Problem base_problem(int M, int N, int K, int batch, int tiles_n, int epi) {
  Problem q = {};
  q.M = M;
  q.N = N;
  q.K = K;
  q.batch = batch;
  q.tiles_m = (M + BM - 1) / BM;
  q.tiles_n = tiles_n;
  q.tiles_per_batch = q.tiles_m * tiles_n;
  q.num_kb = (K + BK - 1) / BK;
  q.k_splits = 1;
  q.epi = epi;
  q.n_store = N;
  q.alpha = 1.0f;
  return q;
}

int launch(Args& a, int n, cudaStream_t stream) {
  int work = 0;
  for (int i = 0; i < n; ++i) {
    a.p[i].work_begin = work;
    work += a.p[i].tiles_per_batch * a.p[i].batch * a.p[i].k_splits;
  }
  a.n_problems = n;
  a.total_work = work;
  static bool attr_set = false;
  if (!attr_set) {
    B200_CHECK_CUDA(cudaFuncSetAttribute(gemm_wgmma_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM_BYTES));
    attr_set = true;
  }
  gemm_wgmma_kernel<<<work < num_sms() ? work : num_sms(), THREADS, SMEM_BYTES, stream>>>(a);
  B200_CHECK_LAUNCH();
  for (int i = 0; i < n; ++i) {
    const Problem& q = a.p[i];
    if (q.k_splits <= 1) continue;
    const dim3 grid((q.M + 31) / 32, (q.N + 63) / 64, q.batch);
    splitk_finalize_kernel<<<grid, 256, 0, stream>>>(q.ws, q.k_splits, q.batch, q.M, q.N,
                                                     reinterpret_cast<__nv_bfloat16*>(q.D), q.ldd, q.strideD, q.alpha,
                                                     q.alpha_vec, q.symmetric);
    B200_CHECK_LAUNCH();
  }
  return B200_OK;
}

}  // namespace

// Same contract as gemm_bf16 plus the engine's extra modes; arguments are assumed validated by the caller.
// symmetric: D == D^T (M == N, bf16 out): only tiles on/above the diagonal are computed, the rest mirror-written.
// k_splits > 1: K cut into k_splits ranges with fp32 partials in splitk_ws + a deterministic finalize.
// peer_D: peer-mapped copies of D (other GPUs' buffers) written by the same epilogue.
int gemm_bf16_ex(bool a_mn, bool b_mn, int M, int N, int K, int batch, const void* A, long long lda,
                 long long strideA, const void* B, long long ldb, long long strideB, const void* C,
                 long long ldc, long long strideC, void* D, long long ldd, long long strideD, bool out_f32,
                 float alpha, float beta, const float* alpha_vec, const float* beta_vec, int symmetric,
                 int k_splits, float* splitk_ws, const void* const* peer_D, int n_peers, cudaStream_t stream) {
  if (symmetric && (M != N || out_f32)) symmetric = 0;
  B200_CHECK_ARG(n_peers >= 0 && n_peers <= MAX_PEERS, "gemm: n_peers=%d out of range (0..%d)", n_peers, MAX_PEERS);
  B200_CHECK_ARG(n_peers == 0 || (!out_f32 && !symmetric && k_splits <= 1),
                 "gemm: peer stores need a bf16, non-symmetric, non-split-K output");
  // split-K needs a plain alpha-only bf16 epilogue and 16-byte partial rows
  if (k_splits > 1 && (!splitk_ws || out_f32 || beta != 0.0f || (N & 7) != 0)) k_splits = 1;
  if (k_splits < 1) k_splits = 1;
  Args a;
  int rc;
  if ((rc = operand_map(&a.tmA[0], A, a_mn, M, K, batch, lda, strideA, BM))) return rc;
  if ((rc = operand_map(&a.tmB[0], B, b_mn, N, K, batch, ldb, strideB, BN))) return rc;
  const int tiles_n = (N + BN - 1) / BN;
  Problem& q = a.p[0];
  q = base_problem(M, N, K, batch, tiles_n, 0);
  const int vec = out_f32 ? 4 : 8;
  q.n_store = (N + vec - 1) / vec * vec;
  if (symmetric) q.tiles_per_batch = q.tiles_m * (q.tiles_m + 1) / 2;
  q.a_mn = a_mn;
  q.b_mn = b_mn;
  q.symmetric = symmetric;
  q.k_splits = k_splits;
  q.out_f32 = out_f32;
  q.alpha = alpha;
  q.beta = beta;
  q.alpha_vec = alpha_vec;
  q.beta_vec = beta_vec;
  q.C = (beta != 0.0f) ? C : nullptr;
  q.ldc = ldc;
  q.strideC = strideC;
  q.D = D;
  q.ldd = ldd;
  q.strideD = strideD;
  q.ws = splitk_ws;
  q.n_peers = n_peers;
  for (int i = 0; i < n_peers; ++i) q.peer_D[i] = const_cast<void*>(peer_D[i]);
  if ((rc = plain_epi_maps(a, 0))) return rc;
  return launch(a, 1, stream);
}

// Internal C++ entry (also used by the Newton-Schulz / Shampoo drivers).
int gemm_bf16(bool a_mn, bool b_mn, int M, int N, int K, int batch, const void* A, long long lda,
              long long strideA, const void* B, long long ldb, long long strideB, const void* C,
              long long ldc, long long strideC, void* D, long long ldd, long long strideD,
              bool out_f32, float alpha, float beta, const float* alpha_vec, const float* beta_vec,
              int force_bn, cudaStream_t stream) {
  B200_CHECK_ARG(M > 0 && N > 0 && K > 0 && batch > 0, "gemm: empty problem M=%d N=%d K=%d b=%d", M,
                 N, K, batch);
  B200_CHECK_ARG(lda % 8 == 0 && ldb % 8 == 0, "gemm: lda=%lld ldb=%lld must be multiples of 8", lda,
                 ldb);
  const int out_vec = out_f32 ? 4 : 8;
  // N need not be a multiple of the store vector as long as the padded row exists: columns
  // [N, round_up(N, vec)) of D receive alpha*0 + beta*C (B rows >= N are zero-filled by TMA).  Used by
  // Shampoo's [259, 259] factor of the byte-level embedding (stored with ld = 264).
  {
    const long long n_pad = ((long long)N + out_vec - 1) / out_vec * out_vec;
    B200_CHECK_ARG(N % out_vec == 0 || (ldd >= n_pad && (C == nullptr || ldc >= n_pad) && force_bn != 1256),
                   "gemm: N=%d is not a multiple of %d and ldd=%lld/ldc=%lld leave no room for the padded vector",
                   N, out_vec, ldd, ldc);
  }
  B200_CHECK_ARG(ldd % out_vec == 0 && (C == nullptr || ldc % out_vec == 0),
                 "gemm: ldd=%lld ldc=%lld must be multiples of %d", ldd, ldc, out_vec);
  B200_CHECK_ARG((reinterpret_cast<uintptr_t>(D) & 15u) == 0 &&
                     (reinterpret_cast<uintptr_t>(C) & 15u) == 0,
                 "gemm: C/D must be 16-byte aligned");
  B200_CHECK_ARG(strideA % 8 == 0 && strideB % 8 == 0 && strideD % out_vec == 0 &&
                     strideC % out_vec == 0,
                 "gemm: batch strides must keep 16-byte alignment");
  // force_bn: 0 / 128 / 256 = tile-width hints (the engine's tiles are 128 wide) | 1256 = D == D^T asserted
  return gemm_bf16_ex(a_mn, b_mn, M, N, K, batch, A, lda, strideA, B, ldb, strideB, C, ldc, strideC, D, ldd, strideD,
                      out_f32, alpha, beta, alpha_vec, beta_vec, force_bn == 1256 ? 1 : 0, 1, nullptr, nullptr, 0,
                      stream);
}

// ---- fused MLP GEMMs (arch/llama.py:142-151: down(gate(x) * sigmoid(up(x)) * 2)) --------------------------
// gu[M, 2I] = x[M, K] [Wg ; Wu]^T (W2: [2I, K] row-major, gate rows first), y[M, I] = g * sigmoid(u) * 2
int gemm_glu_fwd(const void* x, const void* W2, void* gu, void* y, int M, int K, int I, cudaStream_t stream) {
  B200_CHECK_ARG(M > 0 && K > 0 && I > 0 && K % 8 == 0 && I % 128 == 0,
                 "mlp_glu_fwd: need K %% 8 == 0 and intermediate size %% 128 == 0 (M=%d K=%d I=%d)", M, K, I);
  Args a;
  int rc;
  if ((rc = operand_map(&a.tmA[0], x, false, M, K, 1, K, 0, BM))) return rc;
  if ((rc = operand_map(&a.tmB[0], W2, false, 2 * I, K, 1, K, 0, 64))) return rc;
  Problem& q = a.p[0];
  q = base_problem(M, I, K, 1, I / 64, 1);
  q.D = gu;
  q.ldd = 2LL * I;
  q.glu_I = I;
  q.aux = y;
  q.ld_aux = I;
  if ((rc = glu_map(&a.tmD[0], gu, I, M, q.ldd))) return rc;
  if ((rc = tile_map(&a.tmE[0], y, I, M, 1, I, 0))) return rc;
  return launch(a, 1, stream);
}

// dgu[M, 2I] = GLU adjoint of d = dy[M, H] Wd (Wd: [H, I] row-major = down_proj.weight), gu[M, 2I] the saved
// forward activations: dg = d * sigmoid(u) * 2 ; du = d * g * sigmoid(u) * (1 - sigmoid(u)) * 2
int gemm_glu_bwd(const void* dy, const void* Wd, const void* gu, void* dgu, int M, int H, int I, cudaStream_t stream) {
  B200_CHECK_ARG(M > 0 && H > 0 && I > 0 && H % 8 == 0 && I % 8 == 0, "mlp_glu_bwd: bad shape M=%d H=%d I=%d", M, H, I);
  Args a;
  int rc;
  if ((rc = operand_map(&a.tmA[0], dy, false, M, H, 1, H, 0, BM))) return rc;
  // B[n = i, k = h] = Wd[h, i]: stored [K = H rows][N = I]: MN-major
  if ((rc = operand_map(&a.tmB[0], Wd, true, I, H, 1, I, 0, BN))) return rc;
  Problem& q = a.p[0];
  q = base_problem(M, I, H, 1, (I + BN - 1) / BN, 2);
  q.b_mn = 1;
  q.D = dgu;
  q.ldd = 2LL * I;
  q.glu_I = I;
  q.aux = const_cast<void*>(gu);
  q.ld_aux = 2LL * I;
  if ((rc = glu_map(&a.tmD[0], dgu, I, M, q.ldd))) return rc;
  if ((rc = glu_map(&a.tmE[0], gu, I, M, q.ld_aux))) return rc;
  return launch(a, 1, stream);
}

// ---- grouped launch: up to MAX_PROBLEMS independent batched problems in one grid ----------------------------
// Problems are bf16-out; `k_splits` > 1 requests split-K into fp32 slabs (splitk_ws) + a finalize pass.  Work
// items are ordered heaviest K range first, so the tail of the launch is made of the cheapest tiles.
int gemm_grouped(const GroupedGemm* probs, int n, cudaStream_t stream) {
  B200_CHECK_ARG(n >= 1 && n <= MAX_PROBLEMS, "grouped gemm: %d problems (1..%d supported)", n, MAX_PROBLEMS);
  int order[MAX_PROBLEMS];
  for (int i = 0; i < n; ++i) order[i] = i;
  auto item_kb = [&](int i) {
    const int num_kb = (probs[i].K + BK - 1) / BK;
    const int ks = probs[i].k_splits > 1 ? probs[i].k_splits : 1;
    return (num_kb + ks - 1) / ks;
  };
  for (int i = 1; i < n; ++i)
    for (int j = i; j > 0 && item_kb(order[j]) > item_kb(order[j - 1]); --j) {
      const int t = order[j];
      order[j] = order[j - 1];
      order[j - 1] = t;
    }
  Args a;
  for (int oi = 0; oi < n; ++oi) {
    const GroupedGemm& h = probs[order[oi]];
    B200_CHECK_ARG(h.M > 0 && h.N > 0 && h.K > 0 && h.batch > 0 && h.N % 8 == 0,
                   "grouped gemm: problem %d has an unsupported shape M=%d N=%d K=%d batch=%d", order[oi], h.M, h.N,
                   h.K, h.batch);
    B200_CHECK_ARG(h.lda % 8 == 0 && h.ldb % 8 == 0 && h.ldd % 8 == 0 && (h.C == nullptr || h.ldc % 8 == 0),
                   "grouped gemm: leading dimensions must be multiples of 8");
    B200_CHECK_ARG(h.n_peers >= 0 && h.n_peers <= MAX_PEERS, "grouped gemm: n_peers out of range");
    const int symmetric = (h.symmetric && h.M == h.N) ? 1 : 0;
    int k_splits = h.k_splits > 1 ? h.k_splits : 1;
    if (k_splits > 1 && (h.splitk_ws == nullptr || h.beta != 0.0f)) k_splits = 1;
    B200_CHECK_ARG(h.n_peers == 0 || (!symmetric && k_splits == 1),
                   "grouped gemm: peer stores need a non-symmetric, non-split-K problem");
    int rc;
    if ((rc = operand_map(&a.tmA[oi], h.A, h.a_mn, h.M, h.K, h.batch, h.lda, h.strideA, BM))) return rc;
    if ((rc = operand_map(&a.tmB[oi], h.B, h.b_mn, h.N, h.K, h.batch, h.ldb, h.strideB, BN))) return rc;
    Problem& q = a.p[oi];
    q = base_problem(h.M, h.N, h.K, h.batch, (h.N + BN - 1) / BN, 0);
    if (symmetric) q.tiles_per_batch = q.tiles_m * (q.tiles_m + 1) / 2;
    q.a_mn = h.a_mn;
    q.b_mn = h.b_mn;
    q.symmetric = symmetric;
    q.k_splits = k_splits;
    q.alpha = h.alpha;
    q.beta = h.beta;
    q.alpha_vec = h.alpha_vec;
    q.beta_vec = h.beta_vec;
    q.C = (h.beta != 0.0f) ? h.C : nullptr;
    q.ldc = h.ldc;
    q.strideC = h.strideC;
    q.D = h.D;
    q.ldd = h.ldd;
    q.strideD = h.strideD;
    q.ws = h.splitk_ws;
    q.n_peers = h.n_peers;
    for (int i = 0; i < h.n_peers; ++i) q.peer_D[i] = const_cast<void*>(h.peer_D[i]);
    if ((rc = plain_epi_maps(a, oi))) return rc;
  }
  return launch(a, n, stream);
}

}  // namespace b200
