// Newton-Schulz orthogonalisation driver (reference: Muon.zeropower_via_newtonschulz5,
// optimizers/muon.py:54-83):   X0 = G/(||G||_F+eps);  repeat: A = X X^T, B = bA + cAA, X = aX + BX
//
// Formulation: every step is a batched wgmma GEMM (gemm_wgmma.cu) with a fused epilogue
//   G1: A  = X X^T                (wide)   |  A = X^T X   (tall, both operands MN-major)
//   G2: B  = b*A + c*(A A)        (A symmetric -> A A^T, both operands K-major)
//   G3: X' = a*X + B X            (wide, X as MN-major B operand) | X' = a*X + X B (tall)
// so the reference's transpose for tall matrices (muon.py:68-70,80-81) never materialises, and
// the normalisation X0 = G/(||G||+eps) is folded into the first iteration's epilogue scalars
// (per-matrix 1/(norm+eps) vectors produced by the momentum kernel's fused sum of squares).
#include <stdlib.h>

#include "host.h"

namespace b200 {

// G1 of a lone big matrix (the 32003 x 1024 embedding: 36 symmetric 128-tiles, K = 32003) would occupy a
// fraction of the SMs for hundreds of microseconds.  Cut K so that every SM gets a work item.
static int g1_k_splits(int batch, int m, int k) {
  if (m <= 128 || (m & 7) != 0) return 1;
  const int t = (m + 127) / 128;
  const long long tiles = (long long)t * (t + 1) / 2 * batch;
  const int ctas = num_sms();
  if (tiles * 2 > ctas) return 1;
  const int num_kb = (k + 63) / 64;
  int s = (int)(ctas / tiles);
  if (s > num_kb / 16) s = num_kb / 16;
  return s < 2 ? 1 : s;
}

// A = X X^T and B = bA + cAA are symmetric: only tiles on or above the diagonal are computed and
// the rest mirror-written (force_bn code understood by gemm_bf16; ignored when it cannot apply)
static const int kSym = [] {
  const char* e = getenv("B200_NS_NOSYM");  // debug: full (non-symmetric) G1/G2 tiles
  return (e != nullptr && e[0] == '1') ? 0 : 1256;
}();

// peer_out / n_peers: peer-mapped copies of x_out on other GPUs (owner-computes Newton-Schulz under data
// parallelism).  The LAST iteration's X' = aX + BX GEMM then stores its tiles to x_out and to every peer
// from its epilogue (GEMM -> all-gather in one kernel); with n_peers == 0 this is the plain chain.
static int newton_schulz(const void* x_in, void* x_out, int batch, int rows, int cols, int steps, float a,
                         float b, float c, const float* inv_norm, const float* inv_norm_sq, void* ws,
                         size_t ws_bytes, const void* const* peer_out, int n_peers, cudaStream_t stream) {
  B200_CHECK_ARG(n_peers >= 0 && n_peers <= 7 && (n_peers == 0 || peer_out != nullptr),
                 "newton_schulz: bad peer list (n_peers=%d)", n_peers);
  B200_CHECK_ARG(batch > 0 && rows > 0 && cols > 0 && steps > 0,
                 "newton_schulz: bad shape batch=%d rows=%d cols=%d steps=%d", batch, rows, cols,
                 steps);
  B200_CHECK_ARG(cols % 8 == 0, "newton_schulz: cols=%d must be a multiple of 8 (16-byte rows)",
                 cols);
  B200_CHECK_ARG(x_in != x_out, "newton_schulz: x_in and x_out must be distinct buffers");
  if (ws_bytes < b200_newton_schulz_workspace_bytes(batch, rows, cols, steps)) {
    set_error("newton_schulz: workspace too small (%zu < %zu)", ws_bytes,
              b200_newton_schulz_workspace_bytes(batch, rows, cols, steps));
    return B200_ERR_WORKSPACE;
  }
  const bool tall = rows > cols;
  const int m = tall ? cols : rows;
  const long long mm = (long long)m * m;
  const long long rc = (long long)rows * cols;
  char* w = reinterpret_cast<char*>(ws);
  void* Abuf = w;
  void* Bbuf = w + al256((size_t)batch * mm * 2);
  void* Xtmp = w + 2 * al256((size_t)batch * mm * 2);
  const int splits = g1_k_splits(batch, m, tall ? rows : cols);
  float* splitk_ws = reinterpret_cast<float*>(
      w + 2 * al256((size_t)batch * mm * 2) + (steps >= 2 ? al256((size_t)batch * rc * 2) : 0));

  const void* cur = x_in;
  for (int it = 0; it < steps; ++it) {
    void* nxt = ((steps - 1 - it) % 2 == 0) ? x_out : Xtmp;
    const float* s1 = (it == 0) ? inv_norm : nullptr;
    const float* s2 = (it == 0) ? inv_norm_sq : nullptr;
    int rc_;
    // G1
    if (splits > 1)
      rc_ = gemm_bf16_ex(tall, tall, m, m, tall ? rows : cols, batch, cur, cols, rc, cur, cols, rc, nullptr,
                           0, 0, Abuf, m, mm, false, 1.0f, 0.0f, s2, nullptr, 1, splits, splitk_ws,
                           nullptr, 0, stream);
    else if (!tall)
      rc_ = gemm_bf16(false, false, m, m, cols, batch, cur, cols, rc, cur, cols, rc, nullptr, 0, 0,
                      Abuf, m, mm, false, 1.0f, 0.0f, s2, nullptr, kSym, stream);
    else
      rc_ = gemm_bf16(true, true, m, m, rows, batch, cur, cols, rc, cur, cols, rc, nullptr, 0, 0,
                      Abuf, m, mm, false, 1.0f, 0.0f, s2, nullptr, kSym, stream);
    if (rc_) return rc_;
    // G2: B = b*A + c*A*A
    rc_ = gemm_bf16(false, false, m, m, m, batch, Abuf, m, mm, Abuf, m, mm, Abuf, m, mm, Bbuf, m,
                    mm, false, c, b, nullptr, nullptr, kSym, stream);
    if (rc_) return rc_;
    // G3 (the last one carries the peer stores)
    const bool last = it == steps - 1;
    const void* const* peers = last ? peer_out : nullptr;
    const int np = last ? n_peers : 0;
    if (!tall)
      rc_ = gemm_bf16_ex(false, true, m, cols, m, batch, Bbuf, m, mm, cur, cols, rc, cur, cols, rc, nxt, cols, rc,
                         false, 1.0f, a, s1, s1, 0, 1, nullptr, peers, np, stream);
    else
      rc_ = gemm_bf16_ex(false, false, rows, m, m, batch, cur, cols, rc, Bbuf, m, mm, cur, cols, rc, nxt, cols, rc,
                         false, 1.0f, a, s1, s1, 0, 1, nullptr, peers, np, stream);
    if (rc_) return rc_;
    cur = nxt;
  }
  return B200_OK;
}


// ---------------------------------------------------------------------------------------------------------
// Whole-model chain: every shape group of the optimizer advances through the SAME iteration together, so each
// stage (A = X X^T | B = bA + cAA | X' = aX + BX) is ONE grouped launch over all groups (gemm_wgmma.cu) instead
// of one launch per group: 3 launches per iteration (+ one split-K finalize for a lone tall matrix) instead of
// 3 x groups, and the per-launch wave tail is amortised over all groups' tiles.  Falls back to the per-group
// chain for small groups (min(rows, cols) <= 128) or when there are more groups than one launch takes.
// ---------------------------------------------------------------------------------------------------------
static bool multi_grouped_ok(const b200_ns_group* g, int n) {
  static const bool off = [] {
    const char* e = getenv("B200_NS_GROUPED");
    return e != nullptr && e[0] == '0';
  }();
  if (off || n < 1 || n > 6 || num_sms() < 2) return false;
  for (int i = 0; i < n; ++i) {
    const int m = g[i].rows < g[i].cols ? g[i].rows : g[i].cols;
    if (m <= 128 || (m & 7) != 0 || (g[i].cols & 7) != 0) return false;
  }
  return true;
}

struct NsLayout {  // workspace slices of one group
  size_t a, b, xtmp, splitk, end;
  int splits;
};
static NsLayout ns_layout(const b200_ns_group& g, int steps, size_t base) {
  const size_t m = g.rows < g.cols ? g.rows : g.cols;
  NsLayout l;
  l.a = base;
  l.b = l.a + al256((size_t)g.batch * m * m * 2);
  l.xtmp = l.b + al256((size_t)g.batch * m * m * 2);
  l.splitk = l.xtmp + (steps >= 2 ? al256((size_t)g.batch * g.rows * g.cols * 2) : 0);
  l.splits = g1_k_splits(g.batch, (int)m, g.rows < g.cols ? g.cols : g.rows);
  l.end = l.splitk + (l.splits > 1 ? al256((size_t)l.splits * g.batch * m * m * 4) : 0);
  return l;
}

}  // namespace b200

using namespace b200;

extern "C" {

size_t b200_newton_schulz_workspace_bytes(int batch, int rows, int cols, int steps) {
  const size_t m = rows < cols ? rows : cols;
  size_t bytes = 2 * al256((size_t)batch * m * m * 2);
  if (steps >= 2) bytes += al256((size_t)batch * rows * cols * 2);
  const int splits = g1_k_splits(batch, (int)m, rows < cols ? cols : rows);
  if (splits > 1) bytes += al256((size_t)splits * batch * m * m * 4);
  return bytes;
}

int b200_newton_schulz(const void* x_in, void* x_out, int batch, int rows, int cols, int steps,
                       float a, float b, float c, const float* inv_norm, const float* inv_norm_sq,
                       void* workspace, size_t workspace_bytes, void* stream) {
  return newton_schulz(x_in, x_out, batch, rows, cols, steps, a, b, c, inv_norm, inv_norm_sq, workspace,
                       workspace_bytes, nullptr, 0, static_cast<cudaStream_t>(stream));
}

int b200_newton_schulz_allgather(const void* x_in, void* x_out, int batch, int rows, int cols, int steps,
                                 float a, float b, float c, const float* inv_norm, const float* inv_norm_sq,
                                 void* workspace, size_t workspace_bytes, const void* const* peer_out,
                                 int n_peers, void* stream) {
  return newton_schulz(x_in, x_out, batch, rows, cols, steps, a, b, c, inv_norm, inv_norm_sq, workspace,
                       workspace_bytes, peer_out, n_peers, static_cast<cudaStream_t>(stream));
}

size_t b200_newton_schulz_multi_workspace_bytes(const b200_ns_group* g, int n, int steps) {
  size_t off = 0;
  for (int i = 0; i < n; ++i) {
    const size_t grouped_end = ns_layout(g[i], steps, off).end;
    const size_t single_end = off + b200_newton_schulz_workspace_bytes(g[i].batch, g[i].rows, g[i].cols, steps);
    off = grouped_end > single_end ? grouped_end : single_end;
  }
  return off;
}

int b200_newton_schulz_multi(const b200_ns_group* g, int n, int steps, float a, float b, float c, void* ws,
                             size_t ws_bytes, void* stream) {
  const cudaStream_t s = static_cast<cudaStream_t>(stream);
  B200_CHECK_ARG(n >= 1 && g != nullptr && steps > 0, "newton_schulz_multi: bad arguments (n=%d steps=%d)", n, steps);
  for (int i = 0; i < n; ++i) {
    B200_CHECK_ARG(g[i].batch > 0 && g[i].rows > 0 && g[i].cols > 0 && g[i].cols % 8 == 0,
                   "newton_schulz_multi: group %d has a bad shape batch=%d rows=%d cols=%d", i, g[i].batch, g[i].rows,
                   g[i].cols);
    B200_CHECK_ARG(g[i].x_in != g[i].x_out, "newton_schulz_multi: group %d: x_in and x_out must be distinct", i);
    B200_CHECK_ARG(g[i].n_peers >= 0 && g[i].n_peers <= 7 && (g[i].n_peers == 0 || g[i].peer_out != nullptr),
                   "newton_schulz_multi: group %d: bad peer list", i);
  }
  if (ws_bytes < b200_newton_schulz_multi_workspace_bytes(g, n, steps)) {
    set_error("newton_schulz_multi: workspace too small (%zu < %zu)", ws_bytes,
              b200_newton_schulz_multi_workspace_bytes(g, n, steps));
    return B200_ERR_WORKSPACE;
  }
  char* w = reinterpret_cast<char*>(ws);
  if (!multi_grouped_ok(g, n)) {
    size_t off = 0;
    for (int i = 0; i < n; ++i) {
      const size_t grouped_end = ns_layout(g[i], steps, off).end;
      const size_t need = b200_newton_schulz_workspace_bytes(g[i].batch, g[i].rows, g[i].cols, steps);
      int rc = newton_schulz(g[i].x_in, g[i].x_out, g[i].batch, g[i].rows, g[i].cols, steps, a, b, c, g[i].inv_norm,
                             g[i].inv_norm_sq, w + off, need, g[i].peer_out, g[i].n_peers, s);
      if (rc) return rc;
      off = grouped_end > off + need ? grouped_end : off + need;
    }
    return B200_OK;
  }
  NsLayout lay[6];
  const void* cur[6];
  {
    size_t off = 0;
    for (int i = 0; i < n; ++i) {
      lay[i] = ns_layout(g[i], steps, off);
      const size_t single_end = off + b200_newton_schulz_workspace_bytes(g[i].batch, g[i].rows, g[i].cols, steps);
      off = lay[i].end > single_end ? lay[i].end : single_end;
      cur[i] = g[i].x_in;
    }
  }
  b200_gemm_problem pr[6];
  for (int it = 0; it < steps; ++it) {
    const bool first = it == 0, last = it == steps - 1;
    // ---- G1: A = X X^T (wide) / X^T X (tall), symmetric; iteration 1 carries 1/(||G||+eps)^2 ----
    for (int i = 0; i < n; ++i) {
      const bool tall = g[i].rows > g[i].cols;
      const int m = tall ? g[i].cols : g[i].rows;
      const long long rc_ = (long long)g[i].rows * g[i].cols, mm = (long long)m * m;
      b200_gemm_problem& q = pr[i];
      q = b200_gemm_problem{};
      q.a_mn = tall;
      q.b_mn = tall;
      q.M = m;
      q.N = m;
      q.K = tall ? g[i].rows : g[i].cols;
      q.batch = g[i].batch;
      q.A = cur[i];
      q.lda = g[i].cols;
      q.strideA = rc_;
      q.B = cur[i];
      q.ldb = g[i].cols;
      q.strideB = rc_;
      q.D = w + lay[i].a;
      q.ldd = m;
      q.strideD = mm;
      q.alpha = 1.0f;
      q.beta = 0.0f;
      q.alpha_vec = first ? g[i].inv_norm_sq : nullptr;
      q.symmetric = kSym ? 1 : 0;
      q.k_splits = lay[i].splits;
      q.splitk_ws = reinterpret_cast<float*>(w + lay[i].splitk);
    }
    int rc = gemm_grouped(pr, n, s);
    if (rc) return rc;
    // ---- G2: B = b A + c A A (A symmetric: A A^T with both operands K-major) ----
    for (int i = 0; i < n; ++i) {
      const int m = g[i].rows > g[i].cols ? g[i].cols : g[i].rows;
      const long long mm = (long long)m * m;
      b200_gemm_problem& q = pr[i];
      q = b200_gemm_problem{};
      q.M = q.N = q.K = m;
      q.batch = g[i].batch;
      q.A = q.B = q.C = w + lay[i].a;
      q.lda = q.ldb = q.ldc = q.ldd = m;
      q.strideA = q.strideB = q.strideC = q.strideD = mm;
      q.D = w + lay[i].b;
      q.alpha = c;
      q.beta = b;
      q.symmetric = kSym ? 1 : 0;
      q.k_splits = 1;
    }
    rc = gemm_grouped(pr, n, s);
    if (rc) return rc;
    // ---- G3: X' = a X + B X (wide) / a X + X B (tall); the last one carries the peer stores ----
    for (int i = 0; i < n; ++i) {
      const bool tall = g[i].rows > g[i].cols;
      const int m = tall ? g[i].cols : g[i].rows;
      const long long rc_ = (long long)g[i].rows * g[i].cols, mm = (long long)m * m;
      void* nxt = ((steps - 1 - it) % 2 == 0) ? g[i].x_out : static_cast<void*>(w + lay[i].xtmp);
      b200_gemm_problem& q = pr[i];
      q = b200_gemm_problem{};
      if (!tall) {  // [m, cols] = B[m, m] (K-major) x X[m(K), cols] (MN-major)
        q.a_mn = false;
        q.b_mn = true;
        q.M = m;
        q.N = g[i].cols;
        q.K = m;
        q.A = w + lay[i].b;
        q.lda = m;
        q.strideA = mm;
        q.B = cur[i];
        q.ldb = g[i].cols;
        q.strideB = rc_;
      } else {  // [rows, m] = X[rows, m(K)] (K-major) x B[m, m] (symmetric: K-major read of B^T = B)
        q.a_mn = false;
        q.b_mn = false;
        q.M = g[i].rows;
        q.N = m;
        q.K = m;
        q.A = cur[i];
        q.lda = g[i].cols;
        q.strideA = rc_;
        q.B = w + lay[i].b;
        q.ldb = m;
        q.strideB = mm;
      }
      q.batch = g[i].batch;
      q.C = cur[i];
      q.ldc = g[i].cols;
      q.strideC = rc_;
      q.D = nxt;
      q.ldd = g[i].cols;
      q.strideD = rc_;
      q.alpha = 1.0f;
      q.beta = a;
      q.alpha_vec = first ? g[i].inv_norm : nullptr;
      q.beta_vec = first ? g[i].inv_norm : nullptr;
      q.k_splits = 1;
      if (last && g[i].n_peers > 0) {
        q.peer_D = g[i].peer_out;
        q.n_peers = g[i].n_peers;
      }
      cur[i] = nxt;
    }
    rc = gemm_grouped(pr, n, s);
    if (rc) return rc;
  }
  return B200_OK;
}

}  // extern "C"
