// Host-side helpers shared by the C-ABI entry points: error reporting and TMA tensor maps.
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/b200_hotpath.h"

namespace b200 {

// thread-local last error message (returned by b200_last_error())
void set_error(const char* fmt, ...);
const char* last_error();

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
// one deferred RMSNorm weight-gradient reduction (mirrors b200_dw_job of include/b200_hotpath.h)
struct DwJob {
  const float* partials;  // [n_partials][H] fp32, left in the workspace by (add_)rmsnorm_bwd with dw == nullptr
  void* dw;               // [H] bf16 or fp32
  int n_partials;
  int dw_is_bf16;
  int accumulate;         // 1: dw += sum, 0: dw = sum
  int reserved;
};
unsigned long long launch_count();
unsigned long long tensor_map_cache_hits();     // make_tensor_map calls answered from the descriptor cache
unsigned long long tensor_map_cache_misses();   // ... that went to cuTensorMapEncodeTiled

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

// attention dropout: keep threshold t = min(rint(p 65536), 65535) on 16-bit uniforms (p in [0, 1)), and the fp32
// scale 1 / (1 - p_eff) of p_eff = t / 65536
inline uint32_t dropout_threshold(float p) {
  const double t = __builtin_rint((double)p * 65536.0);
  return t > 65535.0 ? 65535u : (uint32_t)t;
}
inline float dropout_scale(uint32_t t) { return (float)(65536.0 / (65536.0 - (double)t)); }

// One problem of a grouped GEMM launch (gemm_wgmma.cu: gemm_grouped): D = alpha*av[b]*op(A)op(B) +
// beta*bv[b]*C, bf16 in/out, batched; layouts as in b200_gemm_bf16.  Mirrors b200_gemm_problem of the public
// header field for field.
struct GroupedGemm {
  int a_mn, b_mn;
  int M, N, K, batch;
  const void* A;
  long long lda, strideA;
  const void* B;
  long long ldb, strideB;
  const void* C;
  long long ldc, strideC;
  void* D;
  long long ldd, strideD;
  float alpha, beta;
  const float* alpha_vec;
  const float* beta_vec;
  int symmetric;     // D == D^T asserted by the caller: compute the upper triangle of tiles, mirror the rest
  int k_splits;      // > 1: split-K into fp32 slabs `splitk_ws` ([k_splits][batch][M][N]) + finalize
  float* splitk_ws;
  const void* const* peer_D;  // GEMM -> all-gather: peer-mapped copies of D (n_peers <= 7)
  int n_peers;
};
int gemm_grouped(const GroupedGemm* probs, int n, cudaStream_t stream);

}  // namespace b200
