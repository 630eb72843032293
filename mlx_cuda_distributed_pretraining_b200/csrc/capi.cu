// extern "C" surface of libb200hotpath.so -- see include/b200_hotpath.h for the contract.
#include "../../include/b200_hotpath.h"

#include "host.h"

namespace b200 {
int gemm_bf16(bool a_mn, bool b_mn, int M, int N, int K, int batch, const void* A, long long lda,
              long long strideA, const void* B, long long ldb, long long strideB, const void* C,
              long long ldc, long long strideC, void* D, long long ldd, long long strideD,
              bool out_f32, float alpha, float beta, const float* alpha_vec, const float* beta_vec,
              int force_bn, cudaStream_t stream);
size_t newton_schulz_workspace_bytes(int batch, int rows, int cols, int steps);
int newton_schulz(const void* x_in, void* x_out, int batch, int rows, int cols, int steps, float a,
                  float b, float c, const float* inv_norm, const float* inv_norm_sq, void* ws,
                  size_t ws_bytes, const void* const* peer_out, int n_peers, cudaStream_t stream);
struct NsGroup {
  const void* x_in;
  void* x_out;
  int batch, rows, cols;
  const float* inv_norm;
  const float* inv_norm_sq;
  const void* const* peer_out;
  int n_peers;
};
size_t newton_schulz_multi_workspace_bytes(const NsGroup* g, int n, int steps);
int newton_schulz_multi(const NsGroup* g, int n, int steps, float a, float b, float c, void* ws, size_t ws_bytes,
                        cudaStream_t stream);
int gemm_glu_fwd(const void* x, const void* W2, void* gu, void* y, int M, int K, int I, int silu, cudaStream_t stream);
int gemm_glu_bwd(const void* dy, const void* Wd, const void* gu, void* dgu, int M, int H, int I, int silu,
                 cudaStream_t stream);
size_t embedding_bwd_workspace_bytes(int V, int H);
int embedding_bwd(const void* dh, const long long* tokens, void* grad, int grad_is_bf16, long long rows, int V, int H,
                  void* ws, size_t ws_bytes, cudaStream_t stream);
size_t reduce_workspace_bytes(int batch);
int muon_momentum(const void* g, int g_is_bf16, float* buf, void* u_bf16, float* sumsq,
                  long long numel, int batch, float mu, int nesterov, float gscale, void* ws,
                  size_t ws_bytes, cudaStream_t stream);
int shampoo_stats(const void* g_hi, const void* g_lo, long long ldg, long long strideG, float* L, float* R,
                  int batch, int k1, int k2, float beta2, float weight, cudaStream_t stream);
size_t shampoo_root_workspace_bytes(int batch, int k);
int shampoo_root(const float* M, float* P, void* P_hi, void* P_lo, int batch, int k, float p, float eps, int iters,
                 void* ws, size_t ws_bytes, cudaStream_t stream);
size_t shampoo_root_newton_workspace_bytes(int batch, int k);
int shampoo_root_newton(const float* M, float* P, void* P_hi, void* P_lo, int batch, int k, float eps, int max_iters,
                        float tol, int* iters_out, float* residual_out, void* ws, size_t ws_bytes,
                        cudaStream_t stream);
size_t shampoo_precond_workspace_bytes(int batch, int k1, int k2);
int shampoo_precond(const void* PL_hi, const void* PL_lo, const void* PR_hi, const void* PR_lo, const void* m_hi,
                    const void* m_lo, long long ldm, long long strideM, float* out, long long ldo, long long strideO,
                    int batch, int k1, int k2, float alpha, void* ws, size_t ws_bytes, cudaStream_t stream);
size_t shampoo_graft_workspace_bytes(int batch);
int shampoo_graft(float* p32, void* p16, const float* upd, const float* graft, long long numel, int batch,
                  float decay, void* ws, size_t ws_bytes, cudaStream_t stream);
int ns_scales(const float* sumsq, float* inv_norm, float* inv_norm_sq, int batch, float eps,
              cudaStream_t stream);
int axpy_update(float* p32, void* p16, const void* x, int x_is_bf16, long long n, float s,
                cudaStream_t stream);
int sgd_momentum(float* p32, void* p16, const void* g, int g_is_bf16, float* buf, long long n,
                 float mu, int nesterov, float lr, float gscale, cudaStream_t stream);
int adamw(float* p32, void* p16, const void* g, int g_is_bf16, float* m, float* v, long long n,
          float lr, float b1, float b2, float eps, float wd, float bc1, float bc2, float gscale,
          cudaStream_t stream);
int adam_direction(float* d, const void* g, int g_is_bf16, float* m, float* v, long long n,
                   float lr, float b1, float b2, float eps, float bc1, float bc2, float gscale,
                   cudaStream_t stream);
int lion(float* p32, void* p16, const void* g, int g_is_bf16, float* m, float* ema, long long n, float lr,
         float b_sign, float b_mom, float decay, float gscale, const float* clip_ss, float max_norm,
         float ema_decay, int ema_mode, cudaStream_t stream);
int sgd(float* p32, void* p16, const void* g, int g_is_bf16, float* buf, float* ema, long long n, float lr,
        float mu, float dampening, int nesterov, float coupled_wd, float gscale, const float* clip_ss,
        float max_norm, float ema_decay, int ema_mode, cudaStream_t stream);
int clip_accum(const void* g, int g_is_bf16, float* acc, long long n, float clip, float scale,
               int init, cudaStream_t stream);
int sumsq(const void* x, int x_is_bf16, float* out, long long numel, int batch, int zero_first,
          void* ws, size_t ws_bytes, cudaStream_t stream);
int split_bf16(const float* src, long long ld_src, void* hi, void* lo, long long ld_dst, int rows,
               int cols, float scale, float diag_add, cudaStream_t stream);
int ema_split(const void* g, int g_is_bf16, float* m, float* out32, void* hi, void* lo, long long n,
              float beta, float gscale, float inv_bc, float out_scale, cudaStream_t stream);
int graft_update(float* p32, void* p16, const float* pre, const float* d, long long numel, int batch,
                 const float* coef, const float* coef_d, float decay, cudaStream_t stream);
int rmsnorm_fwd(const void* x, const void* w, void* y, float* rstd, int rows, int H, float eps,
                int is_bf16, cudaStream_t stream);
size_t rmsnorm_bwd_workspace_bytes(int rows, int H);
int rmsnorm_bwd(const void* dy, const void* x, const void* w, const float* rstd, void* dx,
                float* dw, int rows, int H, int is_bf16, void* ws, size_t ws_bytes,
                cudaStream_t stream);
int rmsnorm_bwd_partial_rows(int rows, int H);
int rmsnorm_dw_reduce(const DwJob* jobs, int n_jobs, int H, cudaStream_t stream);
int add_rmsnorm_fwd(const void* x, const void* delta, const void* w, void* sum_out, void* y, float* rstd,
                    int rows, int H, float eps, int is_bf16, cudaStream_t stream);
int add_rmsnorm_bwd(const void* dy, const void* dres, const void* x, const void* w, const float* rstd,
                    void* dx, float* dw, int rows, int H, int is_bf16, void* ws, size_t ws_bytes,
                    cudaStream_t stream);
int rope(const void* x, void* y, const float* cos_t, const float* sin_t, int B, int S, int NH,
         int D, int backward, int is_bf16, cudaStream_t stream);
int rope_pos(const void* x, void* y, const float* cos_t, const float* sin_t, const int* pos, int B, int S, int NH,
             int D, int backward, int is_bf16, cudaStream_t stream);
int rope_half(const void* x, void* y, const float* cos_t, const float* sin_t, const int* pos, int B, int S, int NH,
              int D, int backward, int is_bf16, cudaStream_t stream);
int silu_glu_fwd(const void* g, const void* u, void* y, long long n, cudaStream_t stream);
int silu_glu_bwd(const void* dy, const void* g, const void* u, void* dg, void* du, long long n, cudaStream_t stream);
int glu_fwd(const void* g, const void* u, void* y, long long n, cudaStream_t stream);
int glu_bwd(const void* dy, const void* g, const void* u, void* dg, void* du, long long n, cudaStream_t stream);
int ce_fwd(const void* logits, long long ld, const long long* targets, int rows, int V, long long pad_token,
           float* row_loss, float* row_lse, cudaStream_t stream);
int ce_bwd(void* logits, long long ld, const long long* targets, int rows, int V, long long pad_token,
           const float* row_lse, const float* row_scale, cudaStream_t stream);
int attn_fwd(const void* q, const void* k, const void* v, void* o, float* lse, int B, int S, int H,
             int Hk, int D, float scale, int causal, cudaStream_t stream);
size_t attn_bwd_workspace_bytes(int B, int S, int H, int Hk, int D);
int attn_bwd(const void* q, const void* k, const void* v, const void* o, const void* d_o,
             const float* lse, void* dq, void* dk, void* dv, int B, int S, int H, int Hk, int D,
             float scale, int causal, int dkv_row_heads, void* ws, size_t ws_bytes, cudaStream_t stream);
int attn_fwd_doc(const void* q, const void* k, const void* v, void* o, float* lse, const int* pos, int B, int S,
                 int H, int Hk, int D, float scale, cudaStream_t stream);
size_t attn_bwd_doc_workspace_bytes(int B, int S, int H, int Hk, int D);
int attn_bwd_doc(const void* q, const void* k, const void* v, const void* o, const void* d_o, const float* lse,
                 const int* pos, void* dq, void* dk, void* dv, int B, int S, int H, int Hk, int D, float scale,
                 int dkv_row_heads, void* ws, size_t ws_bytes, cudaStream_t stream);
int attn_fwd_window(const void* q, const void* k, const void* v, void* o, float* lse, const int* pos, int window,
                    int B, int S, int H, int Hk, int D, float scale, cudaStream_t stream);
int attn_bwd_window(const void* q, const void* k, const void* v, const void* o, const void* d_o, const float* lse,
                    const int* pos, int window, void* dq, void* dk, void* dv, int B, int S, int H, int Hk, int D,
                    float scale, int dkv_row_heads, void* ws, size_t ws_bytes, cudaStream_t stream);
int attn_fwd_alibi(const void* q, const void* k, const void* v, void* o, float* lse, const int* pos, int window,
                   const float* slopes, int B, int S, int H, int Hk, int D, float scale, cudaStream_t stream);
int attn_bwd_alibi(const void* q, const void* k, const void* v, const void* o, const void* d_o, const float* lse,
                   const int* pos, int window, const float* slopes, void* dq, void* dk, void* dv, int B, int S, int H,
                   int Hk, int D, float scale, int dkv_row_heads, void* ws, size_t ws_bytes, cudaStream_t stream);
int attn_fwd_prefix(const void* q, const void* k, const void* v, void* o, float* lse, const int* prefix, int B, int S,
                    int H, int Hk, int D, float scale, cudaStream_t stream);
int attn_bwd_prefix(const void* q, const void* k, const void* v, const void* o, const void* d_o, const float* lse,
                    const int* prefix, void* dq, void* dk, void* dv, int B, int S, int H, int Hk, int D, float scale,
                    int dkv_row_heads, void* ws, size_t ws_bytes, cudaStream_t stream);
int attn_fwd_dropout(const void* q, const void* k, const void* v, void* o, float* lse, const int* pos, int window,
                     const float* slopes, int B, int S, int H, int Hk, int D, float scale, int causal, float p,
                     unsigned long long seed, cudaStream_t stream);
size_t attn_bwd_dropout_workspace_bytes(int B, int S, int H, int Hk, int D);
int attn_bwd_dropout(const void* q, const void* k, const void* v, const void* o, const void* d_o, const float* lse,
                     const int* pos, int window, const float* slopes, void* dq, void* dk, void* dv, int B, int S,
                     int H, int Hk, int D, float scale, int causal, float p, unsigned long long seed,
                     int dkv_row_heads, void* ws, size_t ws_bytes, cudaStream_t stream);
size_t attn_decode_workspace_bytes(int B, int H, int s_max, int D);
int attn_decode_alibi(const void* q, const void* k_cache, const void* v_cache, const int* lens, void* o, float* lse,
                      int window, const float* slopes, int B, int s_max, int H, int Hk, int D, float scale, int is_bf16,
                      void* ws, size_t ws_bytes, cudaStream_t stream);
int attn_decode_window(const void* q, const void* k_cache, const void* v_cache, const int* lens, void* o, float* lse,
                       int window, int B, int s_max, int H, int Hk, int D, float scale, int is_bf16, void* ws,
                       size_t ws_bytes, cudaStream_t stream);
int attn_decode(const void* q, const void* k_cache, const void* v_cache, const int* lens, void* o, float* lse, int B,
                int s_max, int H, int Hk, int D, float scale, int is_bf16, void* ws, size_t ws_bytes,
                cudaStream_t stream);
int kv_append(void* q, const void* k, const void* v, void* k_cache, void* v_cache, const int* lens,
              const float* cos_t, const float* sin_t, int B, int s_max, int H, int Hk, int D, int is_bf16,
              cudaStream_t stream);
int kv_append_half(void* q, const void* k, const void* v, void* k_cache, void* v_cache, const int* lens,
                   const float* cos_t, const float* sin_t, int B, int s_max, int H, int Hk, int D, int is_bf16,
                   cudaStream_t stream);
}  // namespace b200

#define S_(x) reinterpret_cast<cudaStream_t>(x)

extern "C" {

int b200_version(void) { return 4; }
const char* b200_last_error(void) { return b200::last_error(); }

unsigned long long b200_launch_count(void) { return b200::launch_count(); }
void b200_tensor_map_cache_stats(unsigned long long* hits, unsigned long long* misses) {
  if (hits) *hits = b200::tensor_map_cache_hits();
  if (misses) *misses = b200::tensor_map_cache_misses();
}

int b200_device_ok(void) {
  int dev = 0, major = 0, minor = 0;
  if (cudaGetDevice(&dev) != cudaSuccess) return 0;
  if (cudaDeviceGetAttribute(&major, cudaDevAttrComputeCapabilityMajor, dev) != cudaSuccess) return 0;
  if (cudaDeviceGetAttribute(&minor, cudaDevAttrComputeCapabilityMinor, dev) != cudaSuccess) return 0;
  return (major == 9 && minor == 0) ? 1 : 0;  // the library holds sm_90a code only
}

int b200_gemm_bf16(int a_mn, int b_mn, int M, int N, int K, int batch, const void* A,
                   long long lda, long long strideA, const void* B, long long ldb,
                   long long strideB, const void* C, long long ldc, long long strideC, void* D,
                   long long ldd, long long strideD, int out_f32, float alpha, float beta,
                   const float* alpha_vec, const float* beta_vec, int force_bn, void* stream) {
  return b200::gemm_bf16(a_mn != 0, b_mn != 0, M, N, K, batch, A, lda, strideA, B, ldb, strideB, C,
                         ldc, strideC, D, ldd, strideD, out_f32 != 0, alpha, beta, alpha_vec,
                         beta_vec, force_bn, S_(stream));
}

static_assert(sizeof(b200_gemm_problem) == sizeof(b200::GroupedGemm) &&
                  offsetof(b200_gemm_problem, A) == offsetof(b200::GroupedGemm, A) &&
                  offsetof(b200_gemm_problem, alpha) == offsetof(b200::GroupedGemm, alpha) &&
                  offsetof(b200_gemm_problem, symmetric) == offsetof(b200::GroupedGemm, symmetric) &&
                  offsetof(b200_gemm_problem, n_peers) == offsetof(b200::GroupedGemm, n_peers),
              "b200_gemm_problem layout");
// The internal gemm_grouped trusts its callers (the Newton-Schulz drivers); from outside, check what its
// epilogues assume: 16-byte rows and pointers, room for N columns in D, a split-K workspace when one is asked for.
int b200_gemm_grouped(const b200_gemm_problem* problems, int n, void* stream) {
  B200_CHECK_ARG(problems != nullptr && n >= 1, "gemm_grouped: no problems (n=%d)", n);
  auto misaligned = [](const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15u) != 0; };
  for (int i = 0; i < n; ++i) {
    const b200_gemm_problem& h = problems[i];
    B200_CHECK_ARG(h.D != nullptr && h.A != nullptr && h.B != nullptr, "gemm_grouped: problem %d: null operand", i);
    B200_CHECK_ARG(!misaligned(h.D) && !misaligned(h.C), "gemm_grouped: problem %d: C/D must be 16-byte aligned", i);
    B200_CHECK_ARG(h.ldd >= h.N && (h.C == nullptr || h.beta == 0.0f || h.ldc >= h.N),
                   "gemm_grouped: problem %d: ldd=%lld / ldc=%lld shorter than N=%d", i, h.ldd, h.ldc, h.N);
    B200_CHECK_ARG(h.strideA % 8 == 0 && h.strideB % 8 == 0 && h.strideC % 8 == 0 && h.strideD % 8 == 0,
                   "gemm_grouped: problem %d: batch strides must keep 16-byte alignment", i);
    B200_CHECK_ARG(h.k_splits <= 1 || h.splitk_ws != nullptr, "gemm_grouped: problem %d: k_splits=%d needs splitk_ws",
                   i, h.k_splits);
    B200_CHECK_ARG(h.n_peers >= 0 && h.n_peers <= 7 && (h.n_peers == 0 || h.peer_D != nullptr),
                   "gemm_grouped: problem %d: bad peer list (n_peers=%d, 0..7)", i, h.n_peers);
    for (int p = 0; p < h.n_peers; ++p)
      B200_CHECK_ARG(h.peer_D[p] != nullptr && !misaligned(h.peer_D[p]),
                     "gemm_grouped: problem %d: peer %d must be a 16-byte aligned pointer", i, p);
  }
  return b200::gemm_grouped(reinterpret_cast<const b200::GroupedGemm*>(problems), n, S_(stream));
}

size_t b200_newton_schulz_workspace_bytes(int batch, int rows, int cols, int steps) {
  return b200::newton_schulz_workspace_bytes(batch, rows, cols, steps);
}
int b200_newton_schulz(const void* x_in, void* x_out, int batch, int rows, int cols, int steps,
                       float a, float b, float c, const float* inv_norm, const float* inv_norm_sq,
                       void* workspace, size_t workspace_bytes, void* stream) {
  return b200::newton_schulz(x_in, x_out, batch, rows, cols, steps, a, b, c, inv_norm, inv_norm_sq,
                             workspace, workspace_bytes, nullptr, 0, S_(stream));
}
int b200_newton_schulz_allgather(const void* x_in, void* x_out, int batch, int rows, int cols, int steps,
                                 float a, float b, float c, const float* inv_norm, const float* inv_norm_sq,
                                 void* workspace, size_t workspace_bytes, const void* const* peer_out,
                                 int n_peers, void* stream) {
  return b200::newton_schulz(x_in, x_out, batch, rows, cols, steps, a, b, c, inv_norm, inv_norm_sq,
                             workspace, workspace_bytes, peer_out, n_peers, S_(stream));
}
static_assert(sizeof(b200_ns_group) == sizeof(b200::NsGroup), "b200_ns_group layout");
size_t b200_newton_schulz_multi_workspace_bytes(const b200_ns_group* groups, int n_groups, int steps) {
  return b200::newton_schulz_multi_workspace_bytes(reinterpret_cast<const b200::NsGroup*>(groups), n_groups, steps);
}
int b200_newton_schulz_multi(const b200_ns_group* groups, int n_groups, int steps, float a, float b, float c,
                             void* workspace, size_t workspace_bytes, void* stream) {
  return b200::newton_schulz_multi(reinterpret_cast<const b200::NsGroup*>(groups), n_groups, steps, a, b, c, workspace,
                                   workspace_bytes, S_(stream));
}
int b200_mlp_gateup_glu_fwd(const void* x, const void* W2, void* gu, void* y, int M, int K, int I, void* stream) {
  return b200::gemm_glu_fwd(x, W2, gu, y, M, K, I, 0, S_(stream));
}
int b200_mlp_down_glu_bwd(const void* dy, const void* Wd, const void* gu, void* dgu, int M, int H, int I,
                          void* stream) {
  return b200::gemm_glu_bwd(dy, Wd, gu, dgu, M, H, I, 0, S_(stream));
}
int b200_mlp_gateup_silu_fwd(const void* x, const void* W2, void* gu, void* y, int M, int K, int I, void* stream) {
  return b200::gemm_glu_fwd(x, W2, gu, y, M, K, I, 1, S_(stream));
}
int b200_mlp_down_silu_bwd(const void* dy, const void* Wd, const void* gu, void* dgu, int M, int H, int I,
                           void* stream) {
  return b200::gemm_glu_bwd(dy, Wd, gu, dgu, M, H, I, 1, S_(stream));
}
size_t b200_embedding_bwd_workspace_bytes(int V, int H) { return b200::embedding_bwd_workspace_bytes(V, H); }
int b200_embedding_bwd(const void* dh, const long long* tokens, void* grad, int grad_is_bf16, long long rows,
                       int V, int H, void* workspace, size_t workspace_bytes, void* stream) {
  return b200::embedding_bwd(dh, tokens, grad, grad_is_bf16, rows, V, H, workspace, workspace_bytes, S_(stream));
}
size_t b200_reduce_workspace_bytes(int batch) { return b200::reduce_workspace_bytes(batch); }
int b200_muon_momentum(const void* g, int g_is_bf16, float* buf, void* u_bf16, float* sumsq,
                       long long numel, int batch, float mu, int nesterov, float gscale,
                       void* workspace, size_t workspace_bytes, void* stream) {
  return b200::muon_momentum(g, g_is_bf16, buf, u_bf16, sumsq, numel, batch, mu, nesterov, gscale,
                             workspace, workspace_bytes, S_(stream));
}
int b200_shampoo_stats(const void* g_hi, const void* g_lo, long long ldg, long long strideG, float* L,
                       float* R, int batch, int k1, int k2, float beta2, float weight, void* stream) {
  return b200::shampoo_stats(g_hi, g_lo, ldg, strideG, L, R, batch, k1, k2, beta2, weight, S_(stream));
}
size_t b200_shampoo_root_workspace_bytes(int batch, int k) { return b200::shampoo_root_workspace_bytes(batch, k); }
int b200_shampoo_root(const float* M, float* P, void* P_hi, void* P_lo, int batch, int k, float p,
                      float eps, int iters, void* workspace, size_t workspace_bytes, void* stream) {
  return b200::shampoo_root(M, P, P_hi, P_lo, batch, k, p, eps, iters, workspace, workspace_bytes, S_(stream));
}
size_t b200_shampoo_root_newton_workspace_bytes(int batch, int k) {
  return b200::shampoo_root_newton_workspace_bytes(batch, k);
}
int b200_shampoo_root_newton(const float* M, float* P, void* P_hi, void* P_lo, int batch, int k, float eps,
                             int max_iters, float tol, int* iters_out, float* residual_out, void* workspace,
                             size_t workspace_bytes, void* stream) {
  return b200::shampoo_root_newton(M, P, P_hi, P_lo, batch, k, eps, max_iters, tol, iters_out, residual_out,
                                   workspace, workspace_bytes, S_(stream));
}
size_t b200_shampoo_precond_workspace_bytes(int batch, int k1, int k2) {
  return b200::shampoo_precond_workspace_bytes(batch, k1, k2);
}
int b200_shampoo_precond(const void* PL_hi, const void* PL_lo, const void* PR_hi, const void* PR_lo,
                         const void* m_hi, const void* m_lo, long long ldm, long long strideM, float* out,
                         long long ldo, long long strideO, int batch, int k1, int k2, float alpha,
                         void* workspace, size_t workspace_bytes, void* stream) {
  return b200::shampoo_precond(PL_hi, PL_lo, PR_hi, PR_lo, m_hi, m_lo, ldm, strideM, out, ldo, strideO, batch, k1,
                               k2, alpha, workspace, workspace_bytes, S_(stream));
}
size_t b200_shampoo_graft_workspace_bytes(int batch) { return b200::shampoo_graft_workspace_bytes(batch); }
int b200_shampoo_graft(float* p32, void* p16, const float* upd, const float* graft, long long numel,
                       int batch, float decay, void* workspace, size_t workspace_bytes, void* stream) {
  return b200::shampoo_graft(p32, p16, upd, graft, numel, batch, decay, workspace, workspace_bytes, S_(stream));
}
int b200_ns_scales(const float* sumsq, float* inv_norm, float* inv_norm_sq, int batch, float eps,
                   void* stream) {
  return b200::ns_scales(sumsq, inv_norm, inv_norm_sq, batch, eps, S_(stream));
}
int b200_axpy_update(float* p32, void* p16, const void* x, int x_is_bf16, long long n, float s,
                     void* stream) {
  return b200::axpy_update(p32, p16, x, x_is_bf16, n, s, S_(stream));
}
int b200_sgd_momentum(float* p32, void* p16, const void* g, int g_is_bf16, float* buf,
                      long long n, float mu, int nesterov, float lr, float gscale, void* stream) {
  return b200::sgd_momentum(p32, p16, g, g_is_bf16, buf, n, mu, nesterov, lr, gscale, S_(stream));
}
int b200_adamw(float* p32, void* p16, const void* g, int g_is_bf16, float* m, float* v,
               long long n, float lr, float b1, float b2, float eps, float wd, float bc1,
               float bc2, float gscale, void* stream) {
  return b200::adamw(p32, p16, g, g_is_bf16, m, v, n, lr, b1, b2, eps, wd, bc1, bc2, gscale,
                     S_(stream));
}
int b200_adam_direction(float* d, const void* g, int g_is_bf16, float* m, float* v, long long n,
                        float lr, float b1, float b2, float eps, float bc1, float bc2,
                        float gscale, void* stream) {
  return b200::adam_direction(d, g, g_is_bf16, m, v, n, lr, b1, b2, eps, bc1, bc2, gscale,
                              S_(stream));
}
int b200_lion(float* p32, void* p16, const void* g, int g_is_bf16, float* m, float* ema, long long n,
              float lr, float b_sign, float b_mom, float decay, float gscale, const float* clip_ss,
              float max_norm, float ema_decay, int ema_mode, void* stream) {
  return b200::lion(p32, p16, g, g_is_bf16, m, ema, n, lr, b_sign, b_mom, decay, gscale, clip_ss, max_norm,
                    ema_decay, ema_mode, S_(stream));
}
int b200_sgd(float* p32, void* p16, const void* g, int g_is_bf16, float* buf, float* ema, long long n,
             float lr, float mu, float dampening, int nesterov, float coupled_wd, float gscale,
             const float* clip_ss, float max_norm, float ema_decay, int ema_mode, void* stream) {
  return b200::sgd(p32, p16, g, g_is_bf16, buf, ema, n, lr, mu, dampening, nesterov, coupled_wd, gscale, clip_ss,
                   max_norm, ema_decay, ema_mode, S_(stream));
}
int b200_clip_accum(const void* g, int g_is_bf16, float* acc, long long n, float clip,
                    float scale, int init, void* stream) {
  return b200::clip_accum(g, g_is_bf16, acc, n, clip, scale, init, S_(stream));
}
int b200_sumsq(const void* x, int x_is_bf16, float* out, long long numel, int batch,
               int zero_first, void* workspace, size_t workspace_bytes, void* stream) {
  return b200::sumsq(x, x_is_bf16, out, numel, batch, zero_first, workspace, workspace_bytes, S_(stream));
}
int b200_split_bf16(const float* src, long long ld_src, void* hi, void* lo, long long ld_dst,
                    int rows, int cols, float scale, float diag_add, void* stream) {
  return b200::split_bf16(src, ld_src, hi, lo, ld_dst, rows, cols, scale, diag_add, S_(stream));
}
int b200_ema_split(const void* g, int g_is_bf16, float* m, float* out32, void* hi, void* lo,
                   long long n, float beta, float gscale, float inv_bc, float out_scale,
                   void* stream) {
  return b200::ema_split(g, g_is_bf16, m, out32, hi, lo, n, beta, gscale, inv_bc, out_scale,
                         S_(stream));
}
int b200_graft_update(float* p32, void* p16, const float* pre, const float* d, long long numel,
                      int batch, const float* coef, const float* coef_d, float decay, void* stream) {
  return b200::graft_update(p32, p16, pre, d, numel, batch, coef, coef_d, decay, S_(stream));
}
int b200_rmsnorm_fwd(const void* x, const void* w, void* y, float* rstd, int rows, int H,
                     float eps, int is_bf16, void* stream) {
  return b200::rmsnorm_fwd(x, w, y, rstd, rows, H, eps, is_bf16, S_(stream));
}
size_t b200_rmsnorm_bwd_workspace_bytes(int rows, int H) {
  return b200::rmsnorm_bwd_workspace_bytes(rows, H);
}
int b200_rmsnorm_bwd(const void* dy, const void* x, const void* w, const float* rstd, void* dx,
                     float* dw_f32, int rows, int H, int is_bf16, void* workspace,
                     size_t workspace_bytes, void* stream) {
  return b200::rmsnorm_bwd(dy, x, w, rstd, dx, dw_f32, rows, H, is_bf16, workspace, workspace_bytes,
                           S_(stream));
}
int b200_rmsnorm_bwd_partial_rows(int rows, int H) { return b200::rmsnorm_bwd_partial_rows(rows, H); }
static_assert(sizeof(b200_dw_job) == sizeof(b200::DwJob), "b200_dw_job layout");
int b200_rmsnorm_dw_reduce(const b200_dw_job* jobs, int n_jobs, int H, void* stream) {
  return b200::rmsnorm_dw_reduce(reinterpret_cast<const b200::DwJob*>(jobs), n_jobs, H, S_(stream));
}
int b200_add_rmsnorm_fwd(const void* x, const void* delta, const void* w, void* sum_out, void* y,
                         float* rstd, int rows, int H, float eps, int is_bf16, void* stream) {
  return b200::add_rmsnorm_fwd(x, delta, w, sum_out, y, rstd, rows, H, eps, is_bf16, S_(stream));
}
int b200_add_rmsnorm_bwd(const void* dy, const void* dres, const void* x, const void* w,
                         const float* rstd, void* dx, float* dw_f32, int rows, int H, int is_bf16,
                         void* workspace, size_t workspace_bytes, void* stream) {
  return b200::add_rmsnorm_bwd(dy, dres, x, w, rstd, dx, dw_f32, rows, H, is_bf16, workspace,
                               workspace_bytes, S_(stream));
}
int b200_rope(const void* x, void* y, const float* cos_t, const float* sin_t, int B, int S, int NH,
              int D, int backward, int is_bf16, void* stream) {
  return b200::rope(x, y, cos_t, sin_t, B, S, NH, D, backward, is_bf16, S_(stream));
}
int b200_rope_pos(const void* x, void* y, const float* cos_t, const float* sin_t, const int* pos, int B, int S,
                  int NH, int D, int backward, int is_bf16, void* stream) {
  return b200::rope_pos(x, y, cos_t, sin_t, pos, B, S, NH, D, backward, is_bf16, S_(stream));
}
int b200_rope_half(const void* x, void* y, const float* cos_t, const float* sin_t, const int* pos, int B, int S,
                   int NH, int D, int backward, int is_bf16, void* stream) {
  return b200::rope_half(x, y, cos_t, sin_t, pos, B, S, NH, D, backward, is_bf16, S_(stream));
}
int b200_silu_glu_fwd(const void* g, const void* u, void* y, long long n, void* stream) {
  return b200::silu_glu_fwd(g, u, y, n, S_(stream));
}
int b200_silu_glu_bwd(const void* dy, const void* g, const void* u, void* dg, void* du, long long n, void* stream) {
  return b200::silu_glu_bwd(dy, g, u, dg, du, n, S_(stream));
}
int b200_glu_fwd(const void* g, const void* u, void* y, long long n, void* stream) {
  return b200::glu_fwd(g, u, y, n, S_(stream));
}
int b200_glu_bwd(const void* dy, const void* g, const void* u, void* dg, void* du, long long n, void* stream) {
  return b200::glu_bwd(dy, g, u, dg, du, n, S_(stream));
}
int b200_ce_fwd(const void* logits, long long ld, const long long* targets, int rows, int V,
                long long pad_token, float* row_loss, float* row_lse, void* stream) {
  return b200::ce_fwd(logits, ld, targets, rows, V, pad_token, row_loss, row_lse, S_(stream));
}
int b200_ce_bwd(void* logits, long long ld, const long long* targets, int rows, int V, long long pad_token,
                const float* row_lse, const float* row_scale, void* stream) {
  return b200::ce_bwd(logits, ld, targets, rows, V, pad_token, row_lse, row_scale, S_(stream));
}
int b200_attn_fwd(const void* q, const void* k, const void* v, void* o, float* lse, int B, int S,
                  int H, int Hk, int D, float scale, int causal, void* stream) {
  return b200::attn_fwd(q, k, v, o, lse, B, S, H, Hk, D, scale, causal, S_(stream));
}
size_t b200_attn_bwd_workspace_bytes(int B, int S, int H, int Hk, int D) {
  return b200::attn_bwd_workspace_bytes(B, S, H, Hk, D);
}
int b200_attn_bwd(const void* q, const void* k, const void* v, const void* o, const void* d_o,
                  const float* lse, void* dq, void* dk, void* dv, int B, int S, int H, int Hk,
                  int D, float scale, int causal, void* workspace, size_t workspace_bytes,
                  void* stream) {
  return b200::attn_bwd(q, k, v, o, d_o, lse, dq, dk, dv, B, S, H, Hk, D, scale, causal, 0, workspace,
                        workspace_bytes, S_(stream));
}
int b200_attn_bwd_strided(const void* q, const void* k, const void* v, const void* o, const void* d_o,
                          const float* lse, void* dq, void* dk, void* dv, int B, int S, int H, int Hk,
                          int D, float scale, int causal, int dkv_row_heads, void* workspace,
                          size_t workspace_bytes, void* stream) {
  return b200::attn_bwd(q, k, v, o, d_o, lse, dq, dk, dv, B, S, H, Hk, D, scale, causal, dkv_row_heads,
                        workspace, workspace_bytes, S_(stream));
}
int b200_attn_fwd_doc(const void* q, const void* k, const void* v, void* o, float* lse, const int* pos, int B,
                      int S, int H, int Hk, int D, float scale, void* stream) {
  return b200::attn_fwd_doc(q, k, v, o, lse, pos, B, S, H, Hk, D, scale, S_(stream));
}
size_t b200_attn_bwd_doc_workspace_bytes(int B, int S, int H, int Hk, int D) {
  return b200::attn_bwd_doc_workspace_bytes(B, S, H, Hk, D);
}
int b200_attn_bwd_doc(const void* q, const void* k, const void* v, const void* o, const void* d_o, const float* lse,
                      const int* pos, void* dq, void* dk, void* dv, int B, int S, int H, int Hk, int D, float scale,
                      int dkv_row_heads, void* workspace, size_t workspace_bytes, void* stream) {
  return b200::attn_bwd_doc(q, k, v, o, d_o, lse, pos, dq, dk, dv, B, S, H, Hk, D, scale, dkv_row_heads, workspace,
                            workspace_bytes, S_(stream));
}

int b200_attn_fwd_window(const void* q, const void* k, const void* v, void* o, float* lse, const int* pos, int window,
                         int B, int S, int H, int Hk, int D, float scale, void* stream) {
  return b200::attn_fwd_window(q, k, v, o, lse, pos, window, B, S, H, Hk, D, scale, S_(stream));
}
size_t b200_attn_bwd_window_workspace_bytes(int B, int S, int H, int Hk, int D) {
  return b200::attn_bwd_doc_workspace_bytes(B, S, H, Hk, D);
}
int b200_attn_bwd_window(const void* q, const void* k, const void* v, const void* o, const void* d_o, const float* lse,
                         const int* pos, int window, void* dq, void* dk, void* dv, int B, int S, int H, int Hk, int D,
                         float scale, int dkv_row_heads, void* workspace, size_t workspace_bytes, void* stream) {
  return b200::attn_bwd_window(q, k, v, o, d_o, lse, pos, window, dq, dk, dv, B, S, H, Hk, D, scale, dkv_row_heads,
                               workspace, workspace_bytes, S_(stream));
}

int b200_attn_fwd_prefix(const void* q, const void* k, const void* v, void* o, float* lse, const int* prefix, int B,
                         int S, int H, int Hk, int D, float scale, void* stream) {
  return b200::attn_fwd_prefix(q, k, v, o, lse, prefix, B, S, H, Hk, D, scale, S_(stream));
}
size_t b200_attn_bwd_prefix_workspace_bytes(int B, int S, int H, int Hk, int D) {
  return b200::attn_bwd_workspace_bytes(B, S, H, Hk, D);
}
int b200_attn_bwd_prefix(const void* q, const void* k, const void* v, const void* o, const void* d_o, const float* lse,
                         const int* prefix, void* dq, void* dk, void* dv, int B, int S, int H, int Hk, int D,
                         float scale, int dkv_row_heads, void* workspace, size_t workspace_bytes, void* stream) {
  return b200::attn_bwd_prefix(q, k, v, o, d_o, lse, prefix, dq, dk, dv, B, S, H, Hk, D, scale, dkv_row_heads,
                               workspace, workspace_bytes, S_(stream));
}

int b200_attn_fwd_dropout(const void* q, const void* k, const void* v, void* o, float* lse, const int* pos, int window,
                          const float* slopes, int B, int S, int H, int Hk, int D, float scale, int causal, float p,
                          unsigned long long seed, void* stream) {
  return b200::attn_fwd_dropout(q, k, v, o, lse, pos, window, slopes, B, S, H, Hk, D, scale, causal, p, seed,
                                S_(stream));
}
size_t b200_attn_bwd_dropout_workspace_bytes(int B, int S, int H, int Hk, int D) {
  return b200::attn_bwd_dropout_workspace_bytes(B, S, H, Hk, D);
}
int b200_attn_bwd_dropout(const void* q, const void* k, const void* v, const void* o, const void* d_o, const float* lse,
                          const int* pos, int window, const float* slopes, void* dq, void* dk, void* dv, int B, int S,
                          int H, int Hk, int D, float scale, int causal, float p, unsigned long long seed,
                          int dkv_row_heads, void* workspace, size_t workspace_bytes, void* stream) {
  return b200::attn_bwd_dropout(q, k, v, o, d_o, lse, pos, window, slopes, dq, dk, dv, B, S, H, Hk, D, scale, causal,
                                p, seed, dkv_row_heads, workspace, workspace_bytes, S_(stream));
}

int b200_attn_fwd_alibi(const void* q, const void* k, const void* v, void* o, float* lse, const int* pos, int window,
                        const float* slopes, int B, int S, int H, int Hk, int D, float scale, void* stream) {
  return b200::attn_fwd_alibi(q, k, v, o, lse, pos, window, slopes, B, S, H, Hk, D, scale, S_(stream));
}
int b200_attn_bwd_alibi(const void* q, const void* k, const void* v, const void* o, const void* d_o, const float* lse,
                        const int* pos, int window, const float* slopes, void* dq, void* dk, void* dv, int B, int S,
                        int H, int Hk, int D, float scale, int dkv_row_heads, void* workspace, size_t workspace_bytes,
                        void* stream) {
  return b200::attn_bwd_alibi(q, k, v, o, d_o, lse, pos, window, slopes, dq, dk, dv, B, S, H, Hk, D, scale,
                              dkv_row_heads, workspace, workspace_bytes, S_(stream));
}

size_t b200_attn_decode_workspace_bytes(int B, int H, int s_max, int D) {
  return b200::attn_decode_workspace_bytes(B, H, s_max, D);
}
int b200_attn_decode(const void* q, const void* k_cache, const void* v_cache, const int* lens, void* o, float* lse,
                     int B, int s_max, int H, int Hk, int D, float scale, int is_bf16, void* workspace,
                     size_t workspace_bytes, void* stream) {
  return b200::attn_decode(q, k_cache, v_cache, lens, o, lse, B, s_max, H, Hk, D, scale, is_bf16, workspace,
                           workspace_bytes, S_(stream));
}
int b200_attn_decode_window(const void* q, const void* k_cache, const void* v_cache, const int* lens, void* o,
                            float* lse, int window, int B, int s_max, int H, int Hk, int D, float scale, int is_bf16,
                            void* workspace, size_t workspace_bytes, void* stream) {
  return b200::attn_decode_window(q, k_cache, v_cache, lens, o, lse, window, B, s_max, H, Hk, D, scale, is_bf16,
                                  workspace, workspace_bytes, S_(stream));
}
int b200_attn_decode_alibi(const void* q, const void* k_cache, const void* v_cache, const int* lens, void* o,
                           float* lse, int window, const float* slopes, int B, int s_max, int H, int Hk, int D,
                           float scale, int is_bf16, void* workspace, size_t workspace_bytes, void* stream) {
  return b200::attn_decode_alibi(q, k_cache, v_cache, lens, o, lse, window, slopes, B, s_max, H, Hk, D, scale,
                                 is_bf16, workspace, workspace_bytes, S_(stream));
}
int b200_kv_append(void* q, const void* k, const void* v, void* k_cache, void* v_cache, const int* lens,
                   const float* cos_t, const float* sin_t, int B, int s_max, int H, int Hk, int D, int is_bf16,
                   void* stream) {
  return b200::kv_append(q, k, v, k_cache, v_cache, lens, cos_t, sin_t, B, s_max, H, Hk, D, is_bf16, S_(stream));
}
int b200_kv_append_half(void* q, const void* k, const void* v, void* k_cache, void* v_cache, const int* lens,
                        const float* cos_t, const float* sin_t, int B, int s_max, int H, int Hk, int D, int is_bf16,
                        void* stream) {
  return b200::kv_append_half(q, k, v, k_cache, v_cache, lens, cos_t, sin_t, B, s_max, H, Hk, D, is_bf16,
                              S_(stream));
}

}  // extern "C"
