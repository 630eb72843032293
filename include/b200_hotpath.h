/*
 * b200_hotpath.h -- C ABI of the CUDA-native (H100, sm_90a) training-step hot path.
 *
 * The reference (arthurcolle/mlx-cuda-distributed-pretraining) has no native code and no FFI: its
 * hot path is Python over mlx.core ops.  This header is therefore the boundary a maintainer would
 * bind *instead of* those mlx.core call sites; each entry point cites the reference lines whose
 * arithmetic it replaces.  All functions:
 *   - take raw device pointers + explicit sizes/strides + a cudaStream_t (passed as void*),
 *   - never allocate: scratch comes from the caller via *_workspace_bytes() queries,
 *   - return 0 on success, a negative b200 error code otherwise (message: b200_last_error()),
 *   - are asynchronous on `stream` and re-entrant across streams.
 * Element types: "bf16" = __nv_bfloat16, "f32" = float.  Matrices are row-major.
 */
#ifndef B200_HOTPATH_H_
#define B200_HOTPATH_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define B200_OK 0
#define B200_ERR_ARG (-1)
#define B200_ERR_CUDA (-2)
#define B200_ERR_DEVICE (-3)
#define B200_ERR_WORKSPACE (-4)

/* ---- library / device ---------------------------------------------------------------------- */
int b200_version(void);                 /* ABI version (monotonic integer) */
const char* b200_last_error(void);      /* thread-local message of the last failing call */
int b200_device_ok(void);               /* 1 if the current device is compute capability 9.0 */
unsigned long long b200_launch_count(void); /* kernels launched by this library so far (process-wide) */
/* TMA descriptors are cached per (address, shape, strides, box): calls answered from the cache / encoded by the driver */
void b200_tensor_map_cache_stats(unsigned long long* hits, unsigned long long* misses);

/* ---- dense contraction engine (wgmma + TMA) ----------------------------------------------
 * D[b] = alpha*alpha_vec[b] * op(A[b]) op(B[b]) + beta*beta_vec[b] * C[b],  b in [0,batch)
 * replaces: `@` / mx.matmul in optimizers/muon.py:76-78, optimizers/shampoo.py:121,250,254,287-290
 * a_mn=0: A is [M,K] row-major (K-major);  a_mn=1: A is stored [K,M] row-major (MN-major)
 * b_mn=0: B is [N,K] row-major (K-major);  b_mn=1: B is stored [K,N] row-major (MN-major)
 * A,B bf16; C,D bf16 (out_f32=0) or f32 (out_f32=1); accumulate fp32.
 * alpha_vec/beta_vec: optional per-batch device scalars (NULL = 1).
 * force_bn: 0 | 128 | 256 (tile-width hints; tiles are 128 x 128) | 1256 = the caller asserts D == D^T
 * (M == N, bf16 out): only tiles on/above the diagonal are computed, the rest mirror-written.
 * lda/ldb/ldd/ldc multiples of 8 (bf16) / 4 (f32 C,D).  M, K arbitrary (TMA zero-fills); N arbitrary too if
 * ldd/ldc >= round_up(N, 16 bytes): the padded tail columns of D are then written with alpha*0 + beta*C.
 */
int b200_gemm_bf16(int a_mn, int b_mn, int M, int N, int K, int batch,
                   const void* A, long long lda, long long strideA,
                   const void* B, long long ldb, long long strideB,
                   const void* C, long long ldc, long long strideC,
                   void* D, long long ldd, long long strideD,
                   int out_f32, float alpha, float beta,
                   const float* alpha_vec, const float* beta_vec, int force_bn, void* stream);

/* Grouped launch of the same engine: up to 6 independent batched problems in one persistent grid, work items
 * ordered heaviest K range first.  bf16 C/D; per problem, besides the b200_gemm_bf16 arguments:
 *   symmetric=1: D == D^T asserted (M == N): tiles on/above the diagonal computed, the rest mirror-written;
 *   k_splits>1:  K cut into k_splits ranges, fp32 partials in splitk_ws ([k_splits][batch][M][N], required) and a
 *                deterministic finalize; ignored (one split) when beta != 0;
 *   peer_D:      HOST array of n_peers <= 7 extra copies of D (same ldd/strideD) written by the same epilogue;
 *                not combinable with symmetric or split-K.
 * N % 8 == 0, ldd >= N, leading dimensions and batch strides multiples of 8, C/D/peer pointers 16-byte aligned. */
typedef struct b200_gemm_problem {
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
  const float* alpha_vec;       /* [batch] or NULL */
  const float* beta_vec;        /* [batch] or NULL */
  int symmetric;
  int k_splits;
  float* splitk_ws;
  const void* const* peer_D;
  int n_peers;
} b200_gemm_problem;
int b200_gemm_grouped(const b200_gemm_problem* problems, int n, void* stream);

/* ---- Muon (optimizers/muon.py) ---------------------------------------------------------------
 * b200_newton_schulz: Muon.zeropower_via_newtonschulz5 (muon.py:54-83) on a batch of same-shape
 * matrices.  x_in: bf16 [batch,rows,cols], *un-normalised*; inv_norm[b] = 1/(||x_b||_F+eps) and
 * inv_norm_sq[b] = inv_norm[b]^2 (from b200_muon_momentum + b200_ns_scales) fold muon.py:72-73
 * into the first iteration.  x_out: bf16 [batch,rows,cols], must not alias x_in.
 */
size_t b200_newton_schulz_workspace_bytes(int batch, int rows, int cols, int steps);
int b200_newton_schulz(const void* x_in, void* x_out, int batch, int rows, int cols, int steps,
                       float a, float b, float c, const float* inv_norm, const float* inv_norm_sq,
                       void* workspace, size_t workspace_bytes, void* stream);
/* Same chain for the owner-computes data-parallel mode (SURVEY 8e "fused mode"; the reference's size-balanced
 * ownership idea: modal/modal_cuda_utils.py:468-490).  peer_out[i] (HOST array of n_peers <= 7 device
 * pointers) are peer-mapped addresses of the SAME x_out slot in the other ranks' buffers (NVLink peer
 * memory, e.g. torch symmetric memory).  The last X' = aX + BX GEMM writes its tiles to x_out and to every
 * peer from its epilogue -- GEMM and all-gather are one kernel; the caller only needs a cross-rank barrier
 * before reading the gathered buffer. */
int b200_newton_schulz_allgather(const void* x_in, void* x_out, int batch, int rows, int cols, int steps,
                                 float a, float b, float c, const float* inv_norm,
                                 const float* inv_norm_sq, void* workspace, size_t workspace_bytes,
                                 const void* const* peer_out, int n_peers, void* stream);

/* Scratch of the grid reductions below (b200_muon_momentum, b200_sumsq): per-block partials + arrival
 * counters.  The reductions are DETERMINISTIC (fixed summation order, no float atomics), so data-parallel
 * replicas that hold identical gradients compute bit-identical norms and stay bit-identical. */
size_t b200_reduce_workspace_bytes(int batch);
/* Whole-model chain: all shape groups of the optimizer advance through the iteration together and every stage
 * (A = X X^T | B = bA + cAA | X' = aX + BX) is ONE grouped wgmma launch over all groups -- 3 launches per
 * iteration instead of 3 per group (muon.py:91 loops over parameters).  Per group the arguments mean what they
 * mean in b200_newton_schulz / _allgather; n_groups <= 6 takes the grouped path (each group min(rows, cols) > 128),
 * anything else falls back to per-group chains.  Results are identical to per-group calls up to the fp32
 * summation order of split-K partials. */
typedef struct b200_ns_group {
  const void* x_in;            /* bf16 [batch, rows, cols], un-normalised */
  void* x_out;                 /* bf16 [batch, rows, cols] */
  int batch, rows, cols;
  const float* inv_norm;       /* [batch] 1/(||x||_F + eps) */
  const float* inv_norm_sq;    /* [batch] its square */
  const void* const* peer_out; /* HOST array of n_peers peer-mapped copies of x_out (NULL when n_peers == 0) */
  int n_peers;
} b200_ns_group;
size_t b200_newton_schulz_multi_workspace_bytes(const b200_ns_group* groups, int n_groups, int steps);
int b200_newton_schulz_multi(const b200_ns_group* groups, int n_groups, int steps, float a, float b, float c,
                             void* workspace, size_t workspace_bytes, void* stream);

/* muon.py:101,105: buf = (1-mu)*g*gscale + mu*buf ; u = nesterov ? g*gscale + mu*buf : buf.
 * g: [batch,numel] bf16 (g_is_bf16=1) or f32; buf f32; u bf16; sumsq[b] = sum(u_b^2) (overwritten). */
int b200_muon_momentum(const void* g, int g_is_bf16, float* buf, void* u_bf16, float* sumsq,
                       long long numel, int batch, float mu, int nesterov, float gscale,
                       void* workspace, size_t workspace_bytes, void* stream);
/* muon.py:72-73: inv_norm = 1/(sqrt(sumsq)+eps), inv_norm_sq = inv_norm^2 */
int b200_ns_scales(const float* sumsq, float* inv_norm, float* inv_norm_sq, int batch, float eps,
                   void* stream);
/* muon.py:111-114 (and the in-place apply the reference forgot, SURVEY D2):
 * p32 += s*x ; p16 = bf16(p32) if p16 != NULL.  x bf16 (x_is_bf16=1) or f32. */
int b200_axpy_update(float* p32, void* p16, const void* x, int x_is_bf16, long long n, float s,
                     void* stream);
/* muon.py:123-138 non-2-D fallback: momentum as above, p -= lr*u */
int b200_sgd_momentum(float* p32, void* p16, const void* g, int g_is_bf16, float* buf,
                      long long n, float mu, int nesterov, float lr, float gscale, void* stream);

/* ---- AdamW (core/training.py:821 -> mlx.optimizers.AdamW; enhanced_optimizers.py:157-184) ----
 * p *= 1-lr*wd ; m = b1 m + (1-b1) g ; v = b2 v + (1-b2) g^2 ;
 * p -= (lr/bc1) * m / (sqrt(v)/sqrt(bc2) + eps)        (bc1=bc2=1: no bias correction) */
int b200_adamw(float* p32, void* p16, const void* g, int g_is_bf16, float* m, float* v,
               long long n, float lr, float b1, float b2, float eps, float wd, float bc1,
               float bc2, float gscale, void* stream);
/* Adam step direction without applying it (Shampoo grafting, optimizers/shampoo.py:162-167,326) */
int b200_adam_direction(float* d, const void* g, int g_is_bf16, float* m, float* v, long long n,
                        float lr, float b1, float b2, float eps, float bc1, float bc2,
                        float gscale, void* stream);

/* ---- Lion / SGD (optimizers/enhanced_optimizers.py:200-488; core/training.py:809-818,891-894) ------
 * Shared by both entries:
 *   gradient  gj = (g*gscale) * s,  s = min(1, max_norm / (sqrt(*clip_ss)*gscale + 1e-6)) when clip_ss != NULL
 *             (_clip_gradients :417-432 / :285-300; *clip_ss = sum(g^2) over the same range from b200_sumsq with
 *             batch = 1, read on the device: no host synchronisation), else s = 1.
 *   EMA       ema_mode 0: none; 1: ema = p_new; 2: ema = ema_decay*ema + (1-ema_decay)*p_new
 *             (_compute_ema :396-415 / :248-267, on the post-update parameters).
 *   p16 = bf16(p32) when p16 != NULL.  g bf16 (g_is_bf16=1) or f32; every buffer 16-byte aligned; any n.
 * b200_lion (LionEnhanced.update :434-484): c = b_sign*m + (1-b_sign)*gj ; p = p*decay - lr*sign(c) ;
 *   m = b_mom*m + (1-b_mom)*gj ; sign(0) = 0.  b_sign == b_mom and decay = 1 is the reference as written
 *   (b2 unused; its weight decay :471-472 never reaches the parameters); otherwise Chen et al. (2023)
 *   with decay = 1 - lr*wd. */
int b200_lion(float* p32, void* p16, const void* g, int g_is_bf16, float* m, float* ema, long long n,
              float lr, float b_sign, float b_mom, float decay, float gscale, const float* clip_ss,
              float max_norm, float ema_decay, int ema_mode, void* stream);
/* b200_sgd (SGDEnhanced.update :302-351): gj += coupled_wd*p (coupled_wd = lr*wd, :269-283) ;
 *   buf = mu*buf + (1-dampening)*gj ; p += -lr*(nesterov ? gj + mu*buf : buf).
 *   buf == NULL: p += -lr*gj (mlx.optimizers.SGD with momentum 0, what the factory builds for `sgd`). */
int b200_sgd(float* p32, void* p16, const void* g, int g_is_bf16, float* buf, float* ema, long long n,
             float lr, float mu, float dampening, int nesterov, float coupled_wd, float gscale,
             const float* clip_ss, float max_norm, float ema_decay, int ema_mode, void* stream);

/* ---- gradient post-processing (core/training.py:1664-1666,1671-1680) --------------------------
 * acc = (init?0:acc) + clamp(g,-clip,clip)*scale ; clip<=0 disables the clamp */
int b200_clip_accum(const void* g, int g_is_bf16, float* acc, long long n, float clip,
                    float scale, int init, void* stream);
/* out[b] (+)= sum(x[b,:]^2)   (optimizers/shampoo.py:300-301 Frobenius norms); workspace from
 * b200_reduce_workspace_bytes(batch) */
int b200_sumsq(const void* x, int x_is_bf16, float* out, long long numel, int batch,
               int zero_first, void* workspace, size_t workspace_bytes, void* stream);
/* hi = bf16((src + diag_add*I)*scale), lo = bf16(that - hi) (lo may be NULL); strided [rows,cols] */
int b200_split_bf16(const float* src, long long ld_src, void* hi, void* lo, long long ld_dst,
                    int rows, int cols, float scale, float diag_add, void* stream);

/* ---- Shampoo elementwise pieces (optimizers/shampoo.py:351-359, 365-373) ----------------------
 * ema_split: m = beta*m + (1-beta)*g*gscale ; mhat = m*inv_bc -> out32 = out_scale*mhat (f32),
 * hi/lo = bf16 split of mhat */
int b200_ema_split(const void* g, int g_is_bf16, float* m, float* out32, void* hi, void* lo,
                   long long n, float beta, float gscale, float inv_bc, float out_scale,
                   void* stream);
/* p[b] = p[b]*decay + coef[b]*pre[b] + coef_d[b]*d[b] ; p16 = bf16(p) (grafting + decoupled wd) */
int b200_graft_update(float* p32, void* p16, const float* pre, const float* d, long long numel,
                      int batch, const float* coef, const float* coef_d, float decay, void* stream);

/* ---- Shampoo's Kronecker-factor path (optimizers/shampoo.py), batched over same-shape parameters --------
 * Factor matrices (statistics L/R, preconditioners P) are f32 [batch, kp, kp], kp = round_up(k, 8), zero
 * padded; their bf16 hi/lo splits have the same layout.  fp32 operands enter the tensor cores as bf16 hi+lo
 * pairs (three accumulating GEMMs); a NULL lo pointer means "plain bf16 operand".
 *
 * b200_shampoo_stats -- Shampoo._update_statistics (shampoo.py:229-255):
 *   L = beta2*L + weight * G[:k1,:k2] G[:k1,:k2]^T ;  R = beta2*R + weight * G[:k1,:k2]^T G[:k1,:k2]
 *   g_hi (/g_lo): bf16 [batch][rows >= k1][ldg >= k2] (the parameter-shaped gradient, read in place);
 *   weight = (1-beta2) * gscale^2 when the stored gradient still carries a 1/gscale factor. */
int b200_shampoo_stats(const void* g_hi, const void* g_lo, long long ldg, long long strideG, float* L,
                       float* R, int batch, int k1, int k2, float beta2, float weight, void* stream);
/* b200_shampoo_root -- MatrixSqrt.matrix_inverse_pth_root (shampoo.py:88-126), reproduced literally:
 *   Mt = M + eps*I ; Z = Mt/tr(Mt) ; iters x { Z = Z @ (I + Z/p) } ; P = Z * tr(Mt)^(-1/p^2)
 *   M, P: f32 [batch,kp,kp] (distinct); P_hi/P_lo (nullable): bf16 split of P for b200_shampoo_precond. */
size_t b200_shampoo_root_workspace_bytes(int batch, int k);
int b200_shampoo_root(const float* M, float* P, void* P_hi, void* P_lo, int batch, int k, float p,
                      float eps, int iters, void* workspace, size_t workspace_bytes, void* stream);
/* b200_shampoo_root_newton -- a true inverse 4th root, offered next to the literal b200_shampoo_root (which
 * MatrixSqrt.matrix_inverse_pth_root, shampoo.py:88-126, is not: SURVEY D10); selected by ShampooParams.inverse_root:
 *   P = (M + ridge*I_k)^(-1/4),  ridge = eps * max(lambda_max(M), 1e-6)   (lambda_max by power iteration)
 *   coupled Newton, r = 4: Mt = M + ridge I ; z = 5 / (2 ||Mt||_F) ; Mc = z Mt ; X = z^(1/4) I ;
 *   up to max_iters x { T = 1.25 I - Mc/4 ; Mc' = T^4 Mc ; e' = max|Mc' - I| ; accept iff e' <= 1.2 e:
 *   X = X T, Mc = Mc', e = e' } ; a matrix freezes once e <= tol or a step is rejected ; P = X.
 *   Products at fp32 accuracy (3-way bf16 split; hh over 64-wide K slices, five more products).
 *   M, P: f32 [batch,kp,kp] (distinct), padding of P exactly zero; P_hi/P_lo (nullable): bf16 split of P;
 *   iters_out (int) / residual_out (f32, the final e) [batch], nullable.  Bit-identical run to run and independent of the batch a matrix is launched in.
 *   Synchronises `stream` every 4 iterations to stop once every matrix is frozen. */
size_t b200_shampoo_root_newton_workspace_bytes(int batch, int k);
int b200_shampoo_root_newton(const float* M, float* P, void* P_hi, void* P_lo, int batch, int k, float eps,
                             int max_iters, float tol, int* iters_out, float* residual_out, void* workspace,
                             size_t workspace_bytes, void* stream);
/* b200_shampoo_precond -- Shampoo._apply_preconditioners (shampoo.py:257-295):
 *   out[:k1,:k2] = alpha * PL @ m[:k1,:k2] @ PR   (elements of `out` outside the block are left alone)
 *   m_hi/m_lo: bf16 split of the (bias-corrected) momentum, [batch][rows][ldm]; out: f32 [batch][rows][ldo];
 *   k2 % 8 == 0, k1 arbitrary. */
size_t b200_shampoo_precond_workspace_bytes(int batch, int k1, int k2);
int b200_shampoo_precond(const void* PL_hi, const void* PL_lo, const void* PR_hi, const void* PR_lo,
                         const void* m_hi, const void* m_lo, long long ldm, long long strideM, float* out,
                         long long ldo, long long strideO, int batch, int k1, int k2, float alpha,
                         void* workspace, size_t workspace_bytes, void* stream);
/* b200_shampoo_graft -- Shampoo._apply_grafting + the parameter write (shampoo.py:297-312,365-373):
 *   sn = ||upd_b||_F, gn = ||graft_b||_F (f32, overflow to inf like mx.linalg.norm);
 *   step = sn==0 ? graft : (gn==0 ? upd : upd*gn/sn) ;  p = p*decay + step ; p16 = bf16(p) if non-NULL.
 *   upd, graft, p32: f32 [batch, numel]. Deterministic reductions. */
size_t b200_shampoo_graft_workspace_bytes(int batch);
int b200_shampoo_graft(float* p32, void* p16, const float* upd, const float* graft, long long numel,
                       int batch, float decay, void* workspace, size_t workspace_bytes, void* stream);

/* ---- RMSNorm (arch/llama.py:50-56) and RoPE (arch/llama_standard.py:74-75,117-127) ------------ */
int b200_rmsnorm_fwd(const void* x, const void* w, void* y, float* rstd, int rows, int H,
                     float eps, int is_bf16, void* stream);
size_t b200_rmsnorm_bwd_workspace_bytes(int rows, int H);   /* per-CTA dW partials */
int b200_rmsnorm_bwd(const void* dy, const void* x, const void* w, const float* rstd, void* dx,
                     float* dw_f32 /* NULL: deferred, see below */, int rows, int H, int is_bf16, void* workspace,
                     size_t workspace_bytes, void* stream);
/* Deferred weight gradient: (add_)rmsnorm_bwd called with dw_f32 == NULL leaves its per-CTA partial sums
 * [b200_rmsnorm_bwd_partial_rows(rows, H)][H] (fp32) in the workspace; b200_rmsnorm_dw_reduce then folds any number of
 * such workspaces (one job per norm, all of width H) in one launch per 32 jobs, writing or accumulating into each
 * weight's gradient in its storage type -- the backward of an L-layer model reduces its 2L+1 norm weights once, after
 * the last layer, instead of with four small launches per norm. */
typedef struct b200_dw_job {
  const float* partials; /* workspace of the matching (add_)rmsnorm_bwd call */
  void* dw;              /* [H] bf16 or fp32 */
  int n_partials;        /* b200_rmsnorm_bwd_partial_rows(rows, H) of that call */
  int dw_is_bf16;
  int accumulate;        /* 1: dw += sum (autograd semantics), 0: dw = sum */
  int reserved;
} b200_dw_job;
int b200_rmsnorm_bwd_partial_rows(int rows, int H);
int b200_rmsnorm_dw_reduce(const b200_dw_job* jobs, int n_jobs, int H, void* stream);
/* Residual add fused with the norm that follows it (arch/llama.py:316-319: h = x + sublayer(...), then
 * the next norm reads h):  sum_out = x + delta (rounded to the storage type), y = rmsnorm(sum_out) * w.
 * Backward: dx = dres + rmsnorm_bwd(dy) where dres (nullable) is the gradient that reached sum_out
 * directly; dx is the gradient of both x and delta.  Same workspace as b200_rmsnorm_bwd. */
int b200_add_rmsnorm_fwd(const void* x, const void* delta, const void* w, void* sum_out, void* y,
                         float* rstd, int rows, int H, float eps, int is_bf16, void* stream);
int b200_add_rmsnorm_bwd(const void* dy, const void* dres, const void* x, const void* w,
                         const float* rstd, void* dx, float* dw_f32, int rows, int H, int is_bf16,
                         void* workspace, size_t workspace_bytes, void* stream);
/* x,y: [B,S,NH,D]; cos_t,sin_t: f32 [S,D/2]; backward=1 applies the inverse rotation */
int b200_rope(const void* x, void* y, const float* cos_t, const float* sin_t, int B, int S, int NH,
              int D, int backward, int is_bf16, void* stream);
/* b200_rope for packed sequences: token s of row b is rotated by the angle of pos[b, s] (int32 [B,S], its position
 * within its document, 4-byte aligned) instead of s, so each document gets the rotation it would get alone
 * (arch/llama_standard.py:90-131 with position_ids).  The tables must hold max(pos) + 1 rows. */
int b200_rope_pos(const void* x, void* y, const float* cos_t, const float* sin_t, const int* pos, int B, int S,
                  int NH, int D, int backward, int is_bf16, void* stream);
/* Half-split RoPE, mlx_lm's nn.RoPE(traditional=False) (and Hugging Face Llama's rotate_half): for i < D/2 the pair
 * (x[i], x[i + D/2]) is rotated by pos * theta^(-2i/D), with the same cos_t / sin_t tables as b200_rope.  pos is as
 * for b200_rope_pos, or NULL for position s.  D % 16 == 0; backward=1 applies the inverse rotation. */
int b200_rope_half(const void* x, void* y, const float* cos_t, const float* sin_t, const int* pos, int B, int S,
                   int NH, int D, int backward, int is_bf16, void* stream);

/* ---- MLP block on the in-tree GEMM engine with the GLU in the epilogue (SURVEY 8f row f1) ----------------
 * arch/llama.py:142-151: down( gate(x) * sigmoid(up(x)) * 2 ).  gate_proj.weight and up_proj.weight must be
 * adjacent in memory (W2 = [Wg ; Wu], [2I, K] row-major; flat.ParamStore lays them out that way).
 * b200_mlp_gateup_glu_fwd:  gu[M, 2I] = x[M, K] W2^T  (columns [0, I) = gate(x), [I, 2I) = up(x)),
 *                           y[M, I] = gate * sigmoid(up) * 2 from the fp32 accumulators -- one wgmma kernel,
 *                           no separate activation pass.  K % 8 == 0, I % 128 == 0.
 * b200_mlp_down_glu_bwd:    d = dy[M, H] Wd (dgrad of down_proj, Wd = down_proj.weight [H, I]) never leaves the
 *                           chip: dgu[M, 2I] = [ d * sigmoid(u) * 2 | d * g * sigmoid(u) * (1 - sigmoid(u)) * 2 ]
 *                           with g, u read from the saved gu.  [dg | du] is one matrix, so the gate/up dgrad and
 *                           wgrad each run as a single GEMM against W2. */
int b200_mlp_gateup_glu_fwd(const void* x, const void* W2, void* gu, void* y, int M, int K, int I, void* stream);
int b200_mlp_down_glu_bwd(const void* dy, const void* Wd, const void* gu, void* dgu, int M, int H, int I,
                          void* stream);
/* The same pair for mlx_lm's Llama MLP (mlx_lm/models/llama.py: down(silu(gate(x)) * up(x)), model.misc.variant:
 * mlx_lm), with the same arguments, shapes and alignment rules:
 * b200_mlp_gateup_silu_fwd: y = silu(g) * u = g * sigmoid(g) * u from the fp32 accumulators.
 * b200_mlp_down_silu_bwd:   dgu = [ d * u * sigmoid(g) * (1 + g * (1 - sigmoid(g))) | d * silu(g) ].
 * Their sigmoid is accurate relative to its value (not just to 1), so silu stays accurate in the negative tail. */
int b200_mlp_gateup_silu_fwd(const void* x, const void* W2, void* gu, void* y, int M, int K, int I, void* stream);
int b200_mlp_down_silu_bwd(const void* dy, const void* Wd, const void* gu, void* dgu, int M, int H, int I,
                           void* stream);

/* ---- block-adjacent fused elementwise steps (SURVEY 8f row f1) ------------------------------------
 * arch/llama.py:151: y = gate * sigmoid(up) * 2 and its adjoint; bf16, n % 8 == 0 */
int b200_glu_fwd(const void* gate, const void* up, void* y, long long n, void* stream);
int b200_glu_bwd(const void* dy, const void* gate, const void* up, void* dgate, void* dup, long long n,
                 void* stream);
/* mlx_lm's Llama MLP activation: y = silu(gate) * up and its adjoint; bf16, n % 8 == 0 */
int b200_silu_glu_fwd(const void* gate, const void* up, void* y, long long n, void* stream);
int b200_silu_glu_bwd(const void* dy, const void* gate, const void* up, void* dgate, void* dup, long long n,
                      void* stream);
/* Adjoint of the embedding gather (arch/llama.py:389): grad[tokens[r], :] += dh[r, :] for r in [0, rows);
 * dh bf16 [rows, H]; grad bf16 or f32 [V, H] (accumulated into: it may already hold the tied-logits wgrad);
 * fp32 accumulation per vocabulary row in the workspace (V*H floats), tokens outside [0, V) are ignored. */
size_t b200_embedding_bwd_workspace_bytes(int V, int H);
int b200_embedding_bwd(const void* dh, const long long* tokens, void* grad, int grad_is_bf16, long long rows,
                       int V, int H, void* workspace, size_t workspace_bytes, void* stream);
/* core/training.py:1226-1234: per-row cross entropy of bf16 logits [rows, ld] (first V columns valid),
 * computed in fp32: row_lse = logsumexp, row_loss = (target != pad_token) ? lse - logit[target] : 0.
 * ce_bwd overwrites logits with row_scale[row] * (softmax - onehot(target)) (0 in columns >= V and in
 * rows whose target is pad_token). */
int b200_ce_fwd(const void* logits, long long ld, const long long* targets, int rows, int V,
                long long pad_token, float* row_loss, float* row_lse, void* stream);
int b200_ce_bwd(void* logits, long long ld, const long long* targets, int rows, int V, long long pad_token,
                const float* row_lse, const float* row_scale, void* stream);

/* ---- fused causal / GQA attention (arch/flash_attention.py:97-156 + its autograd) --------------
 * q: bf16 [B,S,H,D], k,v: bf16 [B,S,Hk,D] (q head h uses kv head h/(H/Hk), flash_attention.py:102-120)
 * o: bf16 [B,S,H,D]; lse: f32 [B,H,S] (natural-log sum-exp of scaled, masked scores)
 * causal=1 reproduces the additive -inf strictly-upper mask of arch/llama.py:384-387. */
int b200_attn_fwd(const void* q, const void* k, const void* v, void* o, float* lse, int B, int S,
                  int H, int Hk, int D, float scale, int causal, void* stream);
size_t b200_attn_bwd_workspace_bytes(int B, int S, int H, int Hk, int D);
int b200_attn_bwd(const void* q, const void* k, const void* v, const void* o, const void* d_o,
                  const float* lse, void* dq, void* dk, void* dv, int B, int S, int H, int Hk,
                  int D, float scale, int causal, void* workspace, size_t workspace_bytes,
                  void* stream);
/* Same, with dk / dv token rows of dkv_row_heads heads (>= Hk).  dk = base, dv = base + Hk*D,
 * dkv_row_heads = 2*Hk writes both into one [B,S,2*Hk*D] buffer, so the k/v projections' dgrad / wgrad
 * (arch/flash_attention.py:52-53 weights, adjacent in the flat store) each run as ONE GEMM. */
int b200_attn_bwd_strided(const void* q, const void* k, const void* v, const void* o, const void* d_o,
                          const float* lse, void* dq, void* dk, void* dv, int B, int S, int H, int Hk,
                          int D, float scale, int causal, int dkv_row_heads, void* workspace,
                          size_t workspace_bytes, void* stream);
/* Document-causal attention for packed sequences, replacing b200_attn_fwd / b200_attn_bwd_strided with causal=1
 * when a row holds several documents.  pos (int32 [B,S], 4-byte aligned) is each token's position within its
 * document (0 at a document's first token, +1 per token inside it); query s sees keys s - pos[b,s] .. s, the causal
 * mask of each document run alone (the block-diagonal mask the reference would build as an additive [B,1,S,S] mask,
 * arch/flash_attention.py:123-134).  Key / query tiles wholly outside a query's document are skipped.  The backward
 * takes b200_attn_bwd_strided's dk / dv rows and a workspace of b200_attn_bwd_doc_workspace_bytes
 * (b200_attn_bwd_workspace_bytes plus the per-row document bounds). */
int b200_attn_fwd_doc(const void* q, const void* k, const void* v, void* o, float* lse, const int* pos, int B,
                      int S, int H, int Hk, int D, float scale, void* stream);
size_t b200_attn_bwd_doc_workspace_bytes(int B, int S, int H, int Hk, int D);
int b200_attn_bwd_doc(const void* q, const void* k, const void* v, const void* o, const void* d_o, const float* lse,
                      const int* pos, void* dq, void* dk, void* dv, int B, int S, int H, int Hk, int D, float scale,
                      int dkv_row_heads, void* workspace, size_t workspace_bytes, void* stream);
/* Sliding-window causal attention, with or without packed documents: query s sees key k iff
 * 0 <= s - k <= min(pos[b,s], window), i.e. at most window + 1 keys, itself included (the sliding causal window of
 * the reference's FlexAttention example, README-FlexAttention.md:47-59, with its block mask skipping whole tiles,
 * arch/flex_attention.py:90-139).  pos is as for b200_attn_fwd_doc, or NULL for one document per row
 * (pos[b,s] = s); window >= 0, and window >= S - 1 gives the causal / document-causal mask.  Key and query tiles
 * outside every row's window are skipped, so the cost grows linearly in S.  The backward's workspace is
 * b200_attn_bwd_window_workspace_bytes (equal to the document variant's). */
int b200_attn_fwd_window(const void* q, const void* k, const void* v, void* o, float* lse, const int* pos, int window,
                         int B, int S, int H, int Hk, int D, float scale, void* stream);
size_t b200_attn_bwd_window_workspace_bytes(int B, int S, int H, int Hk, int D);
int b200_attn_bwd_window(const void* q, const void* k, const void* v, const void* o, const void* d_o, const float* lse,
                         const int* pos, int window, void* dq, void* dk, void* dv, int B, int S, int H, int Hk, int D,
                         float scale, int dkv_row_heads, void* workspace, size_t workspace_bytes, void* stream);
/* ALiBi (Press et al., "Train Short, Test Long"): b200_attn_fwd_window / b200_attn_bwd_window with the bias
 * slopes[h] * (k - s) <= 0 added to the scaled score of query s, key k, query head h before the mask and the softmax
 * (the order of the reference's FlexAttention score_mod, arch/flex_attention.py:193-235).  slopes: device fp32 [H],
 * one per QUERY head (the heads of a GQA group keep their own slopes), 4-byte aligned and non-null; its values are not
 * checked, since that would read the device.  pos and window as for the window entries (pos NULL: one document per
 * row; window < 0: no window).  k - s is also the distance inside a document, so packed rows need no more input.
 * Causal only.  The backward's workspace is b200_attn_bwd_window_workspace_bytes.  Zero slopes give the window
 * entries' results bit for bit. */
int b200_attn_fwd_alibi(const void* q, const void* k, const void* v, void* o, float* lse, const int* pos, int window,
                        const float* slopes, int B, int S, int H, int Hk, int D, float scale, void* stream);
int b200_attn_bwd_alibi(const void* q, const void* k, const void* v, const void* o, const void* d_o, const float* lse,
                        const int* pos, int window, const float* slopes, void* dq, void* dk, void* dv, int B, int S,
                        int H, int Hk, int D, float scale, int dkv_row_heads, void* workspace, size_t workspace_bytes,
                        void* stream);
/* Prefix-LM: causal attention in which each row's prefix attends bidirectionally within itself.  prefix: device
 * int32 [B], 4-byte aligned and non-null; query s of row b sees key k iff k <= s or k < P_b, with P_b = prefix[b]
 * clamped to [0, S] by the kernels (its values are not checked on the host, since that would read the device, and
 * the clamp keeps any value from reaching past the row).  P_b <= 1 gives b200_attn_fwd / b200_attn_bwd_strided with
 * causal=1 bit for bit (O, LSE, dK, dV); P_b = S is full non-causal attention.  The backward takes
 * b200_attn_bwd_strided's dk / dv rows and a workspace of b200_attn_bwd_prefix_workspace_bytes (equal to
 * b200_attn_bwd_workspace_bytes). */
int b200_attn_fwd_prefix(const void* q, const void* k, const void* v, void* o, float* lse, const int* prefix, int B,
                         int S, int H, int Hk, int D, float scale, void* stream);
size_t b200_attn_bwd_prefix_workspace_bytes(int B, int S, int H, int Hk, int D);
int b200_attn_bwd_prefix(const void* q, const void* k, const void* v, const void* o, const void* d_o, const float* lse,
                         const int* prefix, void* dq, void* dk, void* dv, int B, int S, int H, int Hk, int D,
                         float scale, int dkv_row_heads, void* workspace, size_t workspace_bytes, void* stream);
/* Attention dropout (arch/flash_attention.py:146-148, arch/flex_attention.py:283-285 and 552-554,
 * arch/simple_attention.py:152-154 of the reference: mx.dropout on the softmax weights before @ V):
 * O = (P o Z / (1 - p_eff)) V with P the ordinary softmax (the LSE is the dropout-free one).  t = min(rint(p 65536),
 * 65535), p_eff = t / 65536; element (b, h, q, k) is kept iff r >= t with r = (w[(k & 7) >> 1] >> 16 (k & 1)) &
 * 0xffff of w = Philox4x32-10(counter (k >> 3, q, h, b), key (seed & 0xffffffff, seed >> 32)), b the row of the
 * launch, h the query head, q and k absolute positions.  pos, window and slopes select the mask as in
 * b200_attn_fwd_window / b200_attn_fwd_alibi (pos and slopes may be NULL, window < 0 means none; any of them needs
 * causal = 1); with none of them, causal selects the causal or full mask.  p outside [0, 1) is rejected; t is
 * rounded from the fp32 p received (ops.attention passes p_eff, so t is that of its double p).  The
 * backward takes the same p and seed, b200_attn_bwd_strided's dk / dv rows and a workspace of
 * b200_attn_bwd_dropout_workspace_bytes.  Decode never drops. */
int b200_attn_fwd_dropout(const void* q, const void* k, const void* v, void* o, float* lse, const int* pos, int window,
                          const float* slopes, int B, int S, int H, int Hk, int D, float scale, int causal, float p,
                          unsigned long long seed, void* stream);
size_t b200_attn_bwd_dropout_workspace_bytes(int B, int S, int H, int Hk, int D);
int b200_attn_bwd_dropout(const void* q, const void* k, const void* v, const void* o, const void* d_o, const float* lse,
                          const int* pos, int window, const float* slopes, void* dq, void* dk, void* dv, int B, int S,
                          int H, int Hk, int D, float scale, int causal, float p, unsigned long long seed,
                          int dkv_row_heads, void* workspace, size_t workspace_bytes, void* stream);

/* ---- generation: a chunk of queries against a KV cache (core/generation_lite.py:104-105, :119-122, :144-154: the
 * prompt_cache and prefill_step_size of the reference's generate_step) ------------------------------------------
 * q, o: bf16 [B, L, H, D]; k_cache, v_cache: bf16 [B, s_max, Hk, D] already holding the chunk's own keys; start,
 * end: device int32 [B].  Query i of row b sits at position p = start[b] + i and sees cached key k iff
 * max(0, p - window) <= k <= p (window < 0: no window), for i < end[b] - start[b]; later rows are padding, their
 * outputs finite but unspecified.  Cache positions at or past end[b] may hold anything (NaN included) and never
 * reach the result.  slopes (device fp32 [H], or NULL) adds ALiBi's slopes[h] * (k - p) to every score.  lse: f32
 * [B, H, L] natural-log sum-exp of the scaled scores, or NULL.  D in {64, 128}.  One CTA per (128 queries, head,
 * row) with no split over keys, so a row's output is bit-identical alone or in any batch; no host synchronisation. */
int b200_attn_fwd_cached(const void* q, const void* k_cache, const void* v_cache, const int* start, const int* end,
                         void* o, float* lse, int window, const float* slopes, int B, int L, int s_max, int H, int Hk,
                         int D, float scale, void* stream);

/* ---- generation: decode attention over a KV cache (arch/flash_attention.py:97-156, last query row) ------------
 * One new query per sequence against its cached keys, causal by construction (every cached key precedes it):
 *   q, o: [B,H,D]; k_cache, v_cache: [B,s_max,Hk,D] (the training layout [B,S,Hk,D]); q head h reads kv head
 *   h/(H/Hk).  All bf16 (is_bf16=1) or all f32 (is_bf16=0); softmax and accumulation in f32 either way.
 *   lens: device int32 [B], keys valid per row including the new token, 1 <= lens[b] <= s_max; keys at or beyond
 *   lens[b] are never read.  lse: f32 [B,H] natural-log sum-exp of the scaled scores, or NULL.
 *   D in {16,32,64,128}, (H/Hk)*D <= 2048, s_max >= 32.
 * Keys split into fixed 256-key chunks from position 0, each chunk's f32 partial (m, l, acc) goes to the workspace
 * and a second pass merges them in chunk order: a row's output is bit-identical alone or in any batch.
 * No host synchronisation; the K/V tensor maps are cached per buffer. */
size_t b200_attn_decode_workspace_bytes(int B, int H, int s_max, int D);
int b200_attn_decode(const void* q, const void* k_cache, const void* v_cache, const int* lens, void* o, float* lse,
                     int B, int s_max, int H, int Hk, int D, float scale, int is_bf16, void* workspace,
                     size_t workspace_bytes, void* stream);
/* b200_attn_decode under a sliding window (README-FlexAttention.md:47-59): the query at position p = lens[b] - 1
 * sees cached keys max(0, p - window) .. p only, window >= 0.  Chunks wholly below the window are skipped and
 * never read; chunk boundaries and the merge order depend on lens[b] and window alone, so a row's output is still
 * bit-identical alone or in any batch.  Same workspace as b200_attn_decode. */
int b200_attn_decode_window(const void* q, const void* k_cache, const void* v_cache, const int* lens, void* o,
                            float* lse, int window, int B, int s_max, int H, int Hk, int D, float scale, int is_bf16,
                            void* workspace, size_t workspace_bytes, void* stream);
/* b200_attn_decode_window (window < 0: no window) with ALiBi: the query at position p = lens[b] - 1 adds
 * slopes[h] * (k - p) to the scaled score of cached key k, slopes as for b200_attn_fwd_alibi (device fp32 [H], not
 * checked).  Same workspace as b200_attn_decode; a row's output is still bit-identical alone or in any batch. */
int b200_attn_decode_alibi(const void* q, const void* k_cache, const void* v_cache, const int* lens, void* o,
                           float* lse, int window, const float* slopes, int B, int s_max, int H, int Hk, int D,
                           float scale, int is_bf16, void* workspace, size_t workspace_bytes, void* stream);
/* A short chunk of new queries over the dense cache that already holds their keys (speculative decoding's verify
 * step): q, o [B, n_q, H, D], 1 <= n_q <= 16; query i of row b sits at position p = start[b] + i and is valid iff
 * i < end[b] - start[b]; it sees keys max(0, p - window) .. p (window < 0: none), with slopes[h] * (k - p) added when
 * slopes is non-null.  lse: f32 [B, H, n_q] or NULL.  Invalid queries' o and lse are not written; no position at or
 * past end[b] is read.  Dtypes, D and (H/Hk) * D as b200_attn_decode.  The chunks, the merge order and the tiles
 * depend on (start[b], end[b], window) alone, so a row is bit-identical alone or in any batch, and with n_q = 1 it
 * is bit-equal to b200_attn_decode(_window / _alibi) with lens = end.  0 <= start[b] <= end[b] <= s_max (device
 * values, not checked); B * n_q <= 65535.  Workspace: b200_attn_decode_multi_workspace_bytes(B, n_q, H, s_max, D). */
size_t b200_attn_decode_multi_workspace_bytes(int B, int n_q, int H, int s_max, int D);
int b200_attn_decode_multi(const void* q, const void* k_cache, const void* v_cache, const int* start, const int* end,
                           void* o, float* lse, int window, const float* slopes, int B, int n_q, int s_max, int H,
                           int Hk, int D, float scale, int is_bf16, void* workspace, size_t workspace_bytes,
                           void* stream);
/* Appends one token per row at pos = lens[b] - 1: k_cache[b,pos] = rot(k[b]), v_cache[b,pos] = v[b] (k, v:
 * [B,Hk,D]).  With cos_t/sin_t (f32 [>= max pos + 1, D/2], ops.rope_tables) the interleaved-pair rotation of
 * b200_rope (arch/llama_standard.py:90-131) is applied to k and, in place, to q [B,H,D], with b200_rope's exact
 * arithmetic; with both NULL k is copied and q is untouched.  Same dtype rule as above; D % 8 == 0. */
int b200_kv_append(void* q, const void* k, const void* v, void* k_cache, void* v_cache, const int* lens,
                   const float* cos_t, const float* sin_t, int B, int s_max, int H, int Hk, int D, int is_bf16,
                   void* stream);
/* b200_kv_append with b200_rope_half's half-split rotation, statement for statement, so a token rotated here is
 * bit-equal to the same token rotated by the prefill.  cos_t / sin_t are required; D % 16 == 0. */
int b200_kv_append_half(void* q, const void* k, const void* v, void* k_cache, void* v_cache, const int* lens,
                        const float* cos_t, const float* sin_t, int B, int s_max, int H, int Hk, int D, int is_bf16,
                        void* stream);

/* ---- quantized KV cache (the reference's kv_bits / kv_group_size, core/generation_lite.py:75-90) --------------
 * Each group of g = group_size consecutive elements of a head vector is stored as x ~ s q + b: n = 2^bits - 1,
 * s = max((max - min) / n, 1e-7), b = min (-0 stored as +0), q = min(n, rint((x - b) / s)), IEEE fp32 throughout.
 * Codes uint8 [B, s_max, Hk, D * bits / 8] (4 bits: element 2j in the low nibble of byte j, 2j + 1 in the high one);
 * parameters f32 [B, Hk, s_max, D / g, 2] holding (s, b).  bits in {4, 8}, g in {32, 64, 128}, D in {32, 64, 128},
 * g divides D, s_max even; every pointer 16-byte aligned.
 *
 * b200_kv_quantize: positions [0, n) of the bf16 / f32 (is_bf16) sources k, v [B, S, Hk, D] into the codes and
 *   parameters; nothing else is written. */
int b200_kv_quantize(const void* k, const void* v, int n, int S, void* k_codes, void* v_codes, float* k_params,
                     float* v_params, int B, int s_max, int Hk, int D, int bits, int group_size, int is_bf16,
                     void* stream);
/* b200_kv_append (half == 0) or b200_kv_append_half (half != 0, tables required) into a quantized cache: q is
 *   rotated in place exactly as there, and k (rotated) and v, rounded to the activation dtype, are quantized into
 *   position lens[b] - 1.  Nothing else is written. */
int b200_kv_append_quant(void* q, const void* k, const void* v, void* k_codes, void* v_codes, float* k_params,
                         float* v_params, const int* lens, const float* cos_t, const float* sin_t, int half, int B,
                         int s_max, int H, int Hk, int D, int bits, int group_size, int is_bf16, void* stream);
/* b200_kv_dequantize: positions [0, min(end[b], S)) of row b of the codes and parameters into bf16 k, v
 *   [B, S, Hk, D], each value s q + b in f32 (product and sum rounded separately) rounded once to bf16; nothing at
 *   or past end[b] is written.  end: device int32 [B]; 1 <= S <= s_max. */
int b200_kv_dequantize(const void* k_codes, const void* v_codes, const float* k_params, const float* v_params,
                       const int* end, void* k, void* v, int S, int B, int s_max, int Hk, int D, int bits,
                       int group_size, void* stream);
/* b200_attn_decode_alibi over a quantized cache: window < 0 is no window, slopes NULL is no ALiBi.  q and o bf16 or
 *   f32 [B, H, D]; same chunking, workspace (b200_attn_decode_workspace_bytes) and merge order, so a row's output is
 *   bit-identical alone or in any batch. */
int b200_attn_decode_quant(const void* q, const void* k_codes, const void* v_codes, const float* k_params,
                           const float* v_params, const int* lens, void* o, float* lse, int window,
                           const float* slopes, int B, int s_max, int H, int Hk, int D, int bits, int group_size,
                           float scale, int is_bf16, void* workspace, size_t workspace_bytes, void* stream);

/* ---- rotating KV cache (the reference's max_kv_size, core/generation_lite.py:103, :120) ----------------------
 * Each row keeps C slots, k_ring / v_ring bf16 [B, C, Hk, D].  Slot map: position t lives in slot
 *     slot(t) = t                        for t < 4 (the sinks)
 *     slot(t) = 4 + (t - 4) mod (C - 4)  otherwise.
 * With M = max_kv_size (>= 5), query position q sees key position k iff
 *     k <= q  and  (k < 4  or  q - k <= M - 5)  [and q - k <= window]
 * and ALiBi's bias slopes[h] * (k - q) uses true positions.  end[b] is the number of positions row b holds; a slot
 * whose position under the map was never written (slot >= end[b] before the first wrap) is never read into a result.
 * C >= M (decode) or C >= M + L - 1 (a chunk of L queries), so no key a query sees has been overwritten.
 *
 * b200_attn_decode_ring: b200_attn_decode_alibi over a ring (window < 0: none, slopes NULL: no ALiBi), the query at
 *   position end[b] - 1.  The visible slots are at most three ranges (the sinks and one arc, which may wrap); 256-slot
 *   chunks holding none are not read.  Chunk boundaries and merge order depend on (end[b], M, C, window) alone, so a
 *   row's output is bit-identical alone or in any batch.  Workspace: b200_attn_decode_workspace_bytes(B, H, C, D). */
int b200_attn_decode_ring(const void* q, const void* k_ring, const void* v_ring, const int* end, void* o, float* lse,
                          int max_kv, int window, const float* slopes, int B, int C, int H, int Hk, int D, float scale,
                          void* workspace, size_t workspace_bytes, void* stream);
/* b200_attn_fwd_cached over a ring: query i < end[b] - start[b] of row b sits at position start[b] + i, the ring
 *   already holding the chunk's keys; later query rows are padding (finite, unspecified).  Masking follows the rule
 *   above.  One CTA per (128 queries, head, row), no split over keys: a row is bit-identical alone or in any batch.
 *   Key tiles with no visible key are skipped: a sink tile plus the arc, about M + 128 keys per query tile. */
int b200_attn_fwd_ring(const void* q, const void* k_ring, const void* v_ring, const int* start, const int* end,
                       void* o, float* lse, int max_kv, int window, const float* slopes, int B, int L, int C, int H,
                       int Hk, int D, float scale, void* stream);
/* b200_kv_append (half == 0) or b200_kv_append_half (half != 0, tables required) into a ring: q and k rotated by
 *   position end[b] - 1 with those kernels' own statements, k and v written to slot(end[b] - 1).  live: device int32
 *   [B] or NULL (all live); a row with live[b] == 0 writes nothing, q included. */
int b200_kv_append_ring(void* q, const void* k, const void* v, void* k_ring, void* v_ring, const int* end,
                        const int* live, const float* cos_t, const float* sin_t, int half, int B, int C, int H,
                        int Hk, int D, void* stream);

/* ---- beam search over a shared-prompt cache (the reference's beam_search, generate_lite.py:400-484) -------------
 * R beam rows in n_groups groups (one per prompt), described by one device int32 array
 *     tables = [row_group (R) | row_slot (R) | grp_t0 (n_groups) | grp_row0 (n_groups) | grp_rows (n_groups)].
 * A group's rows are contiguous (grp_row0[g], grp_rows[g] of them) and have the same length lens[b] (positions held,
 * the new token included).  Positions t < T0 = grp_t0[g] (a multiple of 256) live in the group's prefix cache
 * k_prefix / v_prefix [n_groups, s_prefix, Hk, D]; positions t >= T0 of row b at index t - T0 of its tail slot
 * row_slot[b] in k_tail / v_tail [n_slots, tail_cap, Hk, D].
 * Prefix positions >= T0, tail indices >= lens[b] - T0 and slots no row uses are never read.
 *
 * b200_attn_decode_beam: b200_attn_decode_alibi (window < 0: none, slopes NULL: no ALiBi) for each row's query at
 *   position lens[b] - 1 over that layout.  Chunks are 256 positions from 0, as b200_attn_decode's.  A prefix chunk is
 *   read once for each pack of b200_attn_decode_beam_pack(H, Hk, D) consecutive rows of a group, whose query heads
 *   run together; a tail chunk once per row.  Merge order depends on (lens[b], T0, window) alone, so a row's output is
 *   bit-identical in any batch and, with one row per group, equal to b200_attn_decode(_alibi) over the materialised
 *   row.  q and o bf16 or f32 [R, H, D], D in 16/32/64/128.  s_prefix and tail_cap are multiples of 256.
 *   Workspace: b200_attn_decode_beam_workspace_bytes, 128-byte aligned; the call writes the tails' tensor maps to its
 *   start (an asynchronous copy on the stream) and the partials after them. */
int b200_attn_decode_beam(const void* q, const void* k_prefix, const void* v_prefix, const void* k_tail,
                          const void* v_tail, const int* lens, const int* tables, void* o, float* lse, int window,
                          const float* slopes, int R, int n_groups, int s_prefix, int n_slots, int tail_cap, int H,
                          int Hk, int D, float scale, int is_bf16, void* workspace, size_t workspace_bytes,
                          void* stream);
size_t b200_attn_decode_beam_workspace_bytes(int R, int H, int s_prefix, int tail_cap, int D);
/* Beam rows that share one read of a prefix chunk: max(1, 2048 / (H / Hk * D)); 0 for a bad shape. */
int b200_attn_decode_beam_pack(int H, int Hk, int D);
/* b200_kv_append (half == 0) or b200_kv_append_half (half != 0, tables required) into the tails: q and k rotated at
 *   position lens[b] - 1 with those kernels' own statements, k and v written to index lens[b] - 1 - T0 of slot
 *   row_slot[b] (T0 = grp_t0[row_group[b]], tables as above; only its first 2 R + n_groups entries are read). */
int b200_kv_append_beam(void* q, const void* k, const void* v, void* k_tail, void* v_tail, const int* lens,
                        const int* tables, const float* cos_t, const float* sin_t, int half, int R, int tail_cap, int H,
                        int Hk, int D, int is_bf16, void* stream);
/* Copy-on-fork: copies int32 [n_copies, 3] = (src slot, dst slot, n) copies tail indices [0, n <= max_len) from slot
 *   src to slot dst in each of the n_bufs tails bufs (a device array of pointers, every layer's K and V), one launch.
 *   row_bytes = Hk * D * element size, a multiple of 16.  No destination may be a source.  n_copies == 0: nothing. */
int b200_kv_beam_fork(void* const* bufs, int n_bufs, const int* copies, int n_copies, int max_len, int tail_cap,
                      int row_bytes, void* stream);

/* ---- mixture-of-experts MLP (Mixtral's sparse MoE block, model.misc.num_local_experts) -------------------------
 * T tokens, E experts (2..64), k experts per token (1..min(E, 8)), hidden H, per-expert intermediate I (H, I % 8 == 0).
 * Everything stays on the device and nothing uses atomics: the same inputs give the same bits on every run.
 *
 * b200_moe_route: logits f32 [T, E] -> probs = softmax f32 [T, E]; ids int32 [T, k] = the top-k of probs (larger
 *   first; on an exact tie the lower expert index); weights f32 [T, k] = probs of the ids renormalised to sum 1;
 *   counts int32 [E] rows per expert; seg_off int32 [E + 1]: expert e owns rows [seg_off[e], seg_off[e + 1]) of the
 *   permuted buffer, its count padded up to a multiple of 128; tile_expert int32 [b200_moe_max_tiles]: the expert of
 *   each 128-row tile, n_tiles int32 [1]: seg_off[E] / 128; dest int32 [T, k]: each assignment's row, a stable
 *   counting sort (tokens keep their order inside an expert).  With aux_counts / aux_psum (f32 [E], or both NULL to
 *   skip) it also writes the load-balancing loss partials over the tokens whose mask byte is non-zero (mask NULL: all):
 *   assignments per expert and the sum of probs per expert. */
size_t b200_moe_route_workspace_bytes(int T, int E, int k);
int b200_moe_max_tiles(int T, int E, int k);
int b200_moe_route(const float* logits, const unsigned char* mask, int T, int E, int k, int* ids, float* weights,
                   float* probs, int* counts, int* seg_off, int* tile_expert, int* n_tiles, int* dest,
                   float* aux_counts, float* aux_psum, void* workspace, size_t workspace_bytes, void* stream);
/* xp[dest[t, j]] = x[t] (bf16 rows of H); every pad row of every segment is zero-filled. */
int b200_moe_permute(const void* x, const int* dest, const int* counts, const int* seg_off, int T, int H, int k,
                     int E, void* xp, void* stream);
/* Expert-segmented GEMMs over the permuted buffer, on the wgmma engine's expert-segmented instantiation (TMA +
 * wgmma, persistent).  128-row tile x uses expert tile_expert[x] and tiles at or past *n_tiles are skipped, so the
 * work list is sized by max_tiles (b200_moe_max_tiles) without a host round trip.  Weights are expert-stacked:
 * Wg, Wu [E, I, H] with Wu a whole number (>= E) of [I, H] matrices after Wg in memory (one tensor map addresses
 * both; flat.ParamStore lays a layer's experts out that way), Wd [E, H, I]; H % 8 == 0, I % 64 == 0.
 * act 0: gate * sigmoid(up) * 2, 1: silu(gate) * up.
 *   mode 0 (gate/up forward):  A = xp [rows, H], W0 = Wg, W1 = Wu -> C = gu [rows, 2I] (g | u), Y = act(g, u) [rows, I]
 *                               from the fp32 accumulators
 *   mode 1 (down forward):     A = y [rows, I], W0 = Wd -> C [rows, H]
 *   mode 2 (down dgrad + act adjoint): A = dy [rows, H], W0 = Wd, gu -> C = dgu [rows, 2I] (dg | du)
 *   mode 3 (gate/up dgrad):    A = dgu [rows, 2I], W0 = Wg, W1 = Wu -> C = dg Wg_e + du Wu_e [rows, H] */
int b200_moe_gemm(int mode, int act, const void* A, const void* W0, const void* W1, const void* gu, void* C, void* Y,
                  const int* tile_expert, const int* n_tiles, int max_tiles, int H, int I, int E, void* stream);
/* Weight gradient per expert on the same instantiation: G[e] [R, C] += P[rows_e]^T Q[rows_e] over expert e's counts[e]
 * rows from seg_off[e] (P, Q bf16 buffers of `rows` rows with leading dimensions ldp, ldq; K runs in 64-row blocks
 * inside the 128-padded segment, so the pad rows of P or of Q must be zero, as b200_moe_permute and
 * b200_moe_combine_bwd leave them); fp32 accumulation added to the bf16 G (beta = 1); an expert with no rows is
 * skipped and G[e] left untouched. */
int b200_moe_wgrad(const void* P, long long ldp, const void* Q, long long ldq, void* G, int R, int Cc, int E, int rows,
                   const int* counts, const int* seg_off, void* stream);
/* out[t] = sum_j weights[t, j] * yp[dest[t, j]] in f32, j ascending, bf16 out. */
int b200_moe_combine_fwd(const void* yp, const int* dest, const float* weights, int T, int H, int k, void* out,
                         void* stream);
/* Backward of the combine and the router: dyp[dest[t, j]] = weights[t, j] * dout[t] and zeros in every pad row of
 * every segment (counts / seg_off of b200_moe_route); dw[t, j] = <dout[t],
 * yp[dest[t, j]]> (f32, or NULL); dlogits f32 [T, E] (or NULL) through the renormalisation and the softmax, plus
 * aux_grad[e] (d loss / d aux_psum[e], or NULL) on every token whose mask byte is non-zero. */
int b200_moe_combine_bwd(const void* dout, const void* yp, const int* dest, const int* ids, const float* weights,
                         const float* probs, const float* aux_grad, const unsigned char* mask, const int* counts,
                         const int* seg_off, int T, int H, int E, int k, void* dyp, float* dw, float* dlogits,
                         void* stream);
/* dx[t] = sum_j dxp[dest[t, j]] (+ addend[t], f32 [T, H], or NULL) in f32, bf16 out. */
int b200_moe_unpermute(const void* dxp, const int* dest, const float* addend, int T, int H, int k, void* dx,
                       void* stream);

#ifdef __cplusplus
}
#endif
#endif /* B200_HOTPATH_H_ */
