// Host-side helpers shared by the C-ABI entry points: error reporting, TMA tensor maps, and the one declaration
// of every internal function that a source file other than its own calls.
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/b200_hotpath.h"

namespace b200 {

// thread-local last error message (returned by b200_last_error())
void set_error(const char* fmt, ...);

// error codes: B200_OK / B200_ERR_* macros from the public header

#define B200_CHECK_ARG(cond, ...)          \
  do {                                     \
    if (!(cond)) {                         \
      ::b200::set_error(__VA_ARGS__);      \
      return B200_ERR_ARG;         \
    }                                      \
  } while (0)

#define B200_CHECK_CUDA(expr)                                                              \
  do {                                                                                     \
    cudaError_t e__ = (expr);                                                              \
    if (e__ != cudaSuccess) {                                                              \
      ::b200::set_error("%s failed: %s (%s:%d)", #expr, cudaGetErrorString(e__), __FILE__, \
                        __LINE__);                                                         \
      return B200_ERR_CUDA;                                                        \
    }                                                                                      \
  } while (0)

// every kernel launch of the library is counted (bench.py reports it as gpu_launches)
void count_launch();

#define B200_CHECK_LAUNCH()                  \
  do {                                       \
    ::b200::count_launch();                  \
    B200_CHECK_CUDA(cudaGetLastError());     \
  } while (0)

// Builds a tiled tensor map with 128B swizzle over a row-major array of `elem_bytes`-sized
// elements. dims/strides are listed innermost-first; strides_bytes[i] is the byte stride of
// dims[i+1] (rank-1 entries). Returns 0 on success.
int make_tensor_map(CUtensorMap* out, const void* base, CUtensorMapDataType dtype, int elem_bytes,
                    int rank, const uint64_t* dims, const uint64_t* strides_bytes,
                    const uint32_t* box, bool swizzle128);

int num_sms();

// 16-byte alignment test, 256-byte round-up of workspace slices, round-up to a multiple of 8
inline bool al16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15u) == 0; }
inline size_t al256(size_t x) { return (x + 255) & ~size_t(255); }
inline int rup8(int k) { return (k + 7) & ~7; }

// attention dropout: keep threshold t = min(rint(p 65536), 65535) on 16-bit uniforms (p in [0, 1)), and the fp32
// scale 1 / (1 - p_eff) of p_eff = t / 65536
inline uint32_t dropout_threshold(float p) {
  const double t = __builtin_rint((double)p * 65536.0);
  return t > 65535.0 ? 65535u : (uint32_t)t;
}
inline float dropout_scale(uint32_t t) { return (float)(65536.0 / (65536.0 - (double)t)); }

// ---- the wgmma GEMM engine (gemm_wgmma.cu), shared by the Newton-Schulz, Shampoo and MoE drivers ----
// b200_gemm_bf16 with bool layout flags
int gemm_bf16(bool a_mn, bool b_mn, int M, int N, int K, int batch, const void* A, long long lda,
              long long strideA, const void* B, long long ldb, long long strideB, const void* C,
              long long ldc, long long strideC, void* D, long long ldd, long long strideD,
              bool out_f32, float alpha, float beta, const float* alpha_vec, const float* beta_vec,
              int force_bn, cudaStream_t stream);
// gemm_bf16 plus symmetric tiles, split-K and peer stores, without argument checks
int gemm_bf16_ex(bool a_mn, bool b_mn, int M, int N, int K, int batch, const void* A, long long lda,
                 long long strideA, const void* B, long long ldb, long long strideB, const void* C,
                 long long ldc, long long strideC, void* D, long long ldd, long long strideD, bool out_f32,
                 float alpha, float beta, const float* alpha_vec, const float* beta_vec, int symmetric,
                 int k_splits, float* splitk_ws, const void* const* peer_D, int n_peers, cudaStream_t stream);
// b200_gemm_grouped without the entry's pointer, stride and peer-list validation
int gemm_grouped(const b200_gemm_problem* probs, int n, cudaStream_t stream);
// b200_moe_gemm with Wu at up_off [I, H] matrices after Wg (modes 0 and 3), and b200_moe_wgrad
int moe_gemm(int mode, int silu, const void* A, const void* Wg, int up_off, const void* Wd, const void* gu, void* C,
             void* Y, const int* tile_expert, const int* n_tiles, int max_tiles, int H, int I, int E,
             cudaStream_t stream);
int moe_wgrad(const void* P, long long ldp, const void* Q, long long ldq, void* G, int R, int Cc, int E, int rows,
              const int* counts, const int* seg_off, cudaStream_t stream);

// ---- attention (attention_fwd.cu, also used by attention_bwd.cu) ----
// [B, S, heads, D] bf16 tensor -> 4-D tensor map {D, heads, S, B}, box {64, 1, rows, 1}, 128B swizzle
int make_bshd_map(CUtensorMap* tm, const void* base, int B, int S, int heads, int D, int box_rows);

}  // namespace b200
