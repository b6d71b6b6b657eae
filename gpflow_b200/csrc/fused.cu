// fused.cu — one-call objectives: GPR log marginal likelihood, SGPR ELBO, SVGP ELBO.
// Each function enqueues the whole evaluation on the caller's stream from a caller-provided
// workspace (no allocation, no host synchronisation) and leaves the scalars in device memory.
//   gpk_gpr_lml   : gpflow/models/gpr.py:91-107 + logdensities.py:139-156
//   gpk_sgpr_elbo : gpflow/models/sgpr.py:181-289 (+ the cache of posteriors.py:520-551)
//   gpk_svgp_elbo : gpflow/models/svgp.py:166-181 -> posteriors.py:827-841 -> conditionals/util.py:84-169
//                   -> kullback_leiblers.py:59-165 -> the likelihood's variational expectations (lik.cu)
//   gpk_svgp_mo_elbo_grad : svgp.py:166-181 for multi-output kernels, per latent, with the mixing of
//                           conditionals/util.py:518-563
//   gpk_vgp_elbo_grad : gpflow/models/vgp.py:111-143 (value and gradient; the value alone stays VGP.elbo's operators)
// The gpk.h entry points sit between the helpers they call, at file scope with C linkage, so that the compiler checks
// each definition against its declaration.
#include <stdlib.h>

#include <vector>

#include "internal.cuh"

using namespace gpk;

namespace gpk {

// ---------------------------------------------------------------------------------------------
// GPR
// ---------------------------------------------------------------------------------------------
// Upper bound of max_i K_ii for the expression tree when every leaf has a constant diagonal (stationary, White,
// Constant: the variance); <= 0 when a leaf's diagonal depends on x (Linear, Polynomial): unknown.
static double diag_bound(const gpk_knode* nodes, int idx) {
  const gpk_knode& nd = nodes[idx];
  if (nd.op == GPK_K_SUM || nd.op == GPK_K_PRODUCT) {
    double acc = nd.op == GPK_K_SUM ? 0.0 : 1.0;
    for (int c = 0; c < nd.n_children; ++c) {
      const double v = diag_bound(nodes, nd.child[c]);
      if (!(v > 0.0)) return 0.0;
      acc = nd.op == GPK_K_SUM ? acc + v : acc * v;
    }
    return acc;
  }
  if (nd.op == GPK_K_LINEAR || nd.op == GPK_K_POLYNOMIAL) return 0.0;
  return nd.variance;
}
static double gpr_cond_hint(const gpk_knode* nodes, int n_nodes, double noise_variance) {
  const double d = diag_bound(nodes, n_nodes - 1);
  return (d > 0.0 && noise_variance > 0.0) ? (d + noise_variance) / noise_variance : 0.0;
}

struct GprWs {
  void* A; int64_t lda; void* dinv; int32_t* info; size_t bytes;
};
static GprWs gpr_layout(void* ws, int64_t N, int64_t P, int dtype) {
  Arena a(ws);
  GprWs w;
  w.lda = pad_ld(N);
  w.A = a.take((size_t)(N + P) * w.lda * dtype_size(dtype));
  w.dinv = a.take(potrf_ws_bytes(N, N + P, dtype));
  w.info = (int32_t*)a.take(256);
  w.bytes = a.off;
  return w;
}

__global__ void gpr_finalize_kernel(double* out, const int32_t* info, double N, double P) {
  // logdensities.py:152-154 summed over the P columns (gpr.py:107)
  out[0] = -0.5 * out[1] - 0.5 * N * P * LOG2PI - P * out[2];
  out[3] = (double)info[0];
}

}  // namespace gpk
extern "C" size_t gpk_gpr_lml_ws(int64_t N, int64_t P, int dtype) { return gpr_layout(nullptr, N, P, dtype).bytes; }
namespace gpk {

// The LML's forward pass (gpr.py:91-107), shared by gpk_gpr_lml and gpk_gpr_lml_grad_expr: out[0..3] (out[0 .. n_clear)
// zeroed first), the factor L in w.A with beta^T = L^-1 (Y - m) in its P extra rows, and with need_dinv the block
// inverses of L in w.dinv.
static int gpr_forward(const gpk_knode* nodes, int n_nodes, const int32_t* dims, const double* ard, const void* X,
                       int64_t N, int64_t ldx, int64_t D, const void* Yc, int64_t P, double noise_variance,
                       const void* noise_vec, int dtype, double* out, int n_clear, bool need_dinv, const GprWs& w,
                       cudaStream_t st) {
  const size_t ts = dtype_size(dtype);
  // K(X,X) lower triangle + sigma^2 on the diagonal, no jitter (gpr.py:100-101, model_utils.py:33-50)
  GPK_TRY(kbuild_impl(nodes, n_nodes, dims, ard, X, N, ldx, nullptr, N, ldx, D, w.A, w.lda, dtype, GPK_LOWER,
                      noise_variance, noise_vec, st));
  // (Y - m)^T as P extra rows: the factorisation's panel solves turn them into alpha^T (logdensities.py:150)
  char* Yrows = (char*)w.A + (size_t)N * w.lda * ts;
  GPK_TRY(transpose_impl(Yc, N, P, P, Yrows, w.lda, dtype, st));
  // the block inverses serve the gradient's solves only: the LML needs no trsm on this factor
  GPK_TRY(potrf_any(w.A, N, N + P, w.lda, dtype, w.info, w.dinv, st, need_dinv,
                    noise_vec ? 0.0 : gpr_cond_hint(nodes, n_nodes, noise_variance)));  // gpr.py:102
  GPK_CUDA_OK(cudaMemsetAsync(out, 0, (size_t)n_clear * sizeof(double), st));
  for (int64_t p = 0; p < P; ++p)
    GPK_TRY(reduce_impl(1, Yrows + (size_t)p * w.lda * ts, N, 1, 1.0, 1, out + 1, dtype, st));
  GPK_TRY(reduce_impl(2, w.A, N, w.lda + 1, 1.0, 1, out + 2, dtype, st));
  gpr_finalize_kernel<<<1, 1, 0, st>>>(out, w.info, (double)N, (double)P);
  GPK_LAUNCH_OK();
  return 0;
}

}  // namespace gpk
extern "C" int gpk_gpr_lml(const gpk_knode* nodes, int n_nodes, const int32_t* dims, const double* ard, const void* X,
                           int64_t N, int64_t ldx, int64_t D, const void* Yc, int64_t P, double noise_variance,
                           const void* noise_vec, int dtype, double* out, void* ws, void* stream) {
  const cudaStream_t st = (cudaStream_t)stream;
  GPK_DTYPE_OK("gpr_lml");
  GPK_CHECK_ARG(N > 0 && P > 0 && ws && out && Yc, "gpr_lml: bad arguments");
  return gpr_forward(nodes, n_nodes, dims, ard, X, N, ldx, D, Yc, P, noise_variance, noise_vec, dtype, out, 4, false,
                     gpr_layout(ws, N, P, dtype), st);
}
namespace gpk {

// ---- value + gradient (grad.cu) -----------------------------------------------------------------
struct GprGradWs {
  GprWs f; void* Kinv; void* tmp; void* alpha; size_t alpha_off; size_t bytes;
};
static GprGradWs gpr_grad_layout(void* ws, int64_t N, int64_t P, int dtype) {
  GprGradWs w;
  w.f = gpr_layout(ws, N, P, dtype);
  Arena a(ws);
  a.off = w.f.bytes;
  const size_t ts = dtype_size(dtype);
  const int64_t h = N / 2 + NB;
  w.Kinv = a.take((size_t)N * w.f.lda * ts);
  w.tmp = a.take((size_t)h * h * ts);
  w.alpha_off = a.off;
  w.alpha = a.take((size_t)N * P * ts);
  w.bytes = a.off;
  return w;
}

}  // namespace gpk
extern "C" size_t gpk_gpr_lml_grad_ws(int64_t N, int64_t P, int dtype) {
  return gpr_grad_layout(nullptr, N, P, dtype).bytes;
}
extern "C" size_t gpk_gpr_lml_grad_alpha(int64_t N, int64_t P, int dtype) {
  return gpr_grad_layout(nullptr, N, P, dtype).alpha_off;
}

// out: [0..3] as gpk_gpr_lml; [4] d/dnoise_variance, [5 ...] the leaf slots of build_gradprog (grad.cu)
extern "C" int gpk_gpr_lml_grad_expr(const gpk_knode* nodes, int n_nodes, const int32_t* dims, const double* ard,
                                     const void* X, int64_t N, int64_t ldx, int64_t D, const void* Yc, int64_t P,
                                     double noise_variance, int dtype, double* out, int n_out, void* ws, void* stream) {
  const cudaStream_t st = (cudaStream_t)stream;
  GPK_DTYPE_OK("gpr_lml_grad_expr");
  GPK_CHECK_ARG(dtype == GPK_F64, "gpr_lml_grad_expr: the device backward computes in float64 (dtype %d)", dtype);
  GPK_CHECK_ARG(N > 0 && P > 0 && ws && out && Yc, "gpr_lml_grad_expr: bad arguments");
  const int slots = grad_expr_slots(nodes, n_nodes, dims, ard, D, "gpr_lml_grad_expr");
  if (slots < 0) return slots;
  GPK_CHECK_ARG(n_out >= 5 + slots, "gpr_lml_grad_expr: n_out = %d, the expression needs %d outputs", n_out, 5 + slots);
  GprGradWs w = gpr_grad_layout(ws, N, P, dtype);
  GPK_TRY(gpr_forward(nodes, n_nodes, dims, ard, X, N, ldx, D, Yc, P, noise_variance, nullptr, dtype, out, n_out, true,
                      w.f, st));
  // alpha = L^-T beta  (beta^T = the extra rows)
  GPK_TRY(transpose_impl((const char*)w.f.A + (size_t)N * w.f.lda * sizeof(double), P, N, w.f.lda, w.alpha, P, dtype,
                         st));
  GPK_TRY(trsm_any(1, w.f.A, N, w.f.lda, w.alpha, P, P, dtype, w.f.dinv, st));
  // K^-1 (lower) = L^-T L^-1; the factor is overwritten by its inverse
  GPK_TRY(potri_lower((double*)w.f.A, N, w.f.lda, (const double*)w.f.dinv, (double*)w.Kinv, w.f.lda, (double*)w.tmp, st));
  return gpr_grad_launch(nodes, n_nodes, dims, ard, (const double*)X, N, ldx, D, (const double*)w.alpha, (int)P,
                         (const double*)w.Kinv, w.f.lda, out + 4, st);
}
namespace gpk {

// ---------------------------------------------------------------------------------------------
// SGPR
// ---------------------------------------------------------------------------------------------
// The factors of the collapsed bound, shared by SGPR, the Bayesian GPLVM and CGLB: L = chol(Kuu + jitter I) in Kuu,
// LB = chol(B) in Bm, their block inverses in dinvL / dinvB, c = LB^-1 A' Y / s; info: 0 L, 1 LB.
struct CollapsedWs {
  void *Kuu, *Bm, *dinvL, *dinvB, *c; int64_t ldm, ldn; int32_t* info; double* scal;
};
static CollapsedWs collapsed_layout(Arena& a, int64_t N, int64_t M, int64_t P, int dtype) {
  CollapsedWs w;
  const size_t ts = dtype_size(dtype);
  w.ldm = pad_ld(M);
  w.ldn = pad_ld(N);
  w.Kuu = a.take((size_t)M * w.ldm * ts);
  w.Bm = a.take((size_t)M * w.ldm * ts);
  w.dinvL = a.take(potrf_ws_bytes(M, M, dtype));
  w.dinvB = a.take(potrf_ws_bytes(M, M, dtype));
  w.c = a.take((size_t)M * P * ts);
  w.info = (int32_t*)a.take(256);
  w.scal = (double*)a.take(256);
  return w;
}

// The forward's tail once Bm holds A'A'^T / s (lower), A' [M, ldn]: trace_q = tr(A'A'^T) / s, LB = chol(I + A'A'^T / s),
// half_logdet_b, c = LB^-1 A' Y / s, sum Y^2 / s and |c|^2 into scal[1..4] (sgpr.py:205-207, 262-270).
static int collapsed_tail(const CollapsedWs& w, int64_t N, int64_t M, int64_t P, const void* Ap, const void* Y,
                          double inv_s, int dtype, cudaStream_t st) {
  GPK_TRY(reduce_impl(0, w.Bm, M, w.ldm + 1, 1.0, 1, w.scal + 1, dtype, st));
  GPK_TRY(add_diag_impl(w.Bm, M, w.ldm, 1.0, nullptr, dtype, st));
  GPK_TRY(potrf_any(w.Bm, M, M, w.ldm, dtype, w.info + 1, w.dinvB, st));
  GPK_TRY(reduce_impl(2, w.Bm, M, w.ldm + 1, 1.0, 1, w.scal + 2, dtype, st));
  GPK_TRY(gemm_any(0, 0, M, P, N, inv_s, Ap, w.ldn, Y, P, 0.0, w.c, P, dtype, 0, st));
  GPK_TRY(trsm_any(0, w.Bm, M, w.ldm, w.c, P, P, dtype, w.dinvB, st));
  GPK_TRY(reduce_impl(1, Y, N * P, 1, inv_s, 1, w.scal + 3, dtype, st));
  return reduce_impl(1, w.c, M * P, 1, 1.0, 1, w.scal + 4, dtype, st);
}

struct SgprWs {
  CollapsedWs b; void *Kuf, *kdiag; size_t bytes;
};
static SgprWs sgpr_layout(void* ws, int64_t N, int64_t M, int64_t P, int dtype) {
  Arena a(ws);
  SgprWs w;
  const size_t ts = dtype_size(dtype);
  w.b = collapsed_layout(a, N, M, P, dtype);
  w.Kuf = a.take((size_t)M * w.b.ldn * ts);
  w.kdiag = a.take((size_t)N * ts);
  w.bytes = a.off;
  return w;
}

// scal: 0 trace_k, 1 trace_q, 2 half_logdet_b, 3 sum err^2, 4 sum c^2
__global__ void sgpr_finalize_kernel(double* out, const double* scal, const int32_t* info, double N, double P,
                                     double noise) {
  const double trace_k = scal[0], trace_q = scal[1], half_logdet_b = scal[2];
  const double log_sigma_sq = N * log(noise);
  const double logdet = -P * (half_logdet_b + 0.5 * log_sigma_sq + 0.5 * (trace_k - trace_q));  // sgpr.py:245
  const double quad = -0.5 * (scal[3] - scal[4]);                                              // sgpr.py:270
  const double cst = -0.5 * N * P * LOG2PI;                                                    // sgpr.py:286
  out[0] = cst + logdet + quad;
  out[1] = cst; out[2] = logdet; out[3] = quad; out[4] = trace_k; out[5] = trace_q; out[6] = half_logdet_b;
  out[7] = (double)(info[0] != 0 ? info[0] : info[1]);
}

}  // namespace gpk
extern "C" size_t gpk_sgpr_elbo_ws(int64_t N, int64_t M, int64_t P, int dtype) {
  return sgpr_layout(nullptr, N, M, P, dtype).bytes;
}
namespace gpk {

// The bound's forward pass (sgpr.py:181-289), shared by gpk_sgpr_elbo, gpk_sgpr_elbo_grad and CGLB.  Leaves L in
// w.b.Kuu, A' = L^-1 Kuf in w.Kuf, LB in w.b.Bm, c = LB^-1 A' Yc / s in w.b.c, the scalars in w.b.scal and out[0..7].
static int sgpr_forward(const gpk_knode* nodes, int n_nodes, const int32_t* dims, const double* ard, const void* X,
                        int64_t N, int64_t ldx, int64_t D, const void* Yc, int64_t P, const void* Z, int64_t M,
                        int64_t ldz, double noise, double jitter, int dtype, double* out, const SgprWs& w,
                        cudaStream_t st) {
  const CollapsedWs& b = w.b;
  const double inv_s2 = 1.0 / noise;
  GPK_CUDA_OK(cudaMemsetAsync(b.scal, 0, 8 * sizeof(double), st));
  GPK_CUDA_OK(cudaMemsetAsync(b.info, 0, 2 * sizeof(int32_t), st));
  // kuu = kernel(Z) + jitter I ; L = chol(kuu)   (sgpr.py:200-201)
  GPK_TRY(kbuild_impl(nodes, n_nodes, dims, ard, Z, M, ldz, nullptr, M, ldz, D, b.Kuu, b.ldm, dtype, GPK_LOWER, jitter,
                      nullptr, st));
  GPK_TRY(potrf_any(b.Kuu, M, M, b.ldm, dtype, b.info, b.dinvL, st));
  // kuf = kernel(Z, X) [M,N];  A' = L^-1 kuf  (the 1/sigma of sgpr.py:204 is folded into the scalars below)
  GPK_TRY(kbuild_impl(nodes, n_nodes, dims, ard, Z, M, ldz, X, N, ldx, D, w.Kuf, b.ldn, dtype, GPK_FULL, 0.0, nullptr,
                      st));
  GPK_TRY(trsm_any(0, b.Kuu, M, b.ldm, w.Kuf, N, b.ldn, dtype, b.dinvL, st));
  // trace_k = sum kdiag / sigma^2  (sgpr.py:231-233)
  GPK_TRY(kdiag_impl(nodes, n_nodes, dims, ard, X, N, ldx, D, w.kdiag, dtype, st));
  GPK_TRY(reduce_impl(0, w.kdiag, N, 1, inv_s2, 1, b.scal + 0, dtype, st));
  // AAT = A'A'^T / sigma^2 (lower) ; B = AAT + I = LB LB^T ; c = LB^-1 A' Yc / sigma^2  (sgpr.py:205-207, 262-264)
  GPK_TRY(gemm_any(0, 1, M, M, N, inv_s2, w.Kuf, b.ldn, w.Kuf, b.ldn, 0.0, b.Bm, b.ldm, dtype, GPK_GEMM_LOWER_ONLY, st));
  GPK_TRY(collapsed_tail(b, N, M, P, w.Kuf, Yc, inv_s2, dtype, st));
  sgpr_finalize_kernel<<<1, 1, 0, st>>>(out, b.scal, b.info, (double)N, (double)P, noise);
  GPK_LAUNCH_OK();
  return 0;
}

}  // namespace gpk
extern "C" int gpk_sgpr_elbo(const gpk_knode* nodes, int n_nodes, const int32_t* dims, const double* ard, const void* X,
                             int64_t N, int64_t ldx, int64_t D, const void* Yc, int64_t P, const void* Z, int64_t M,
                             int64_t ldz, double noise, double jitter, int dtype, double* out, void* cache_L,
                             void* cache_LB, void* cache_c, void* ws, void* stream) {
  const cudaStream_t st = (cudaStream_t)stream;
  GPK_DTYPE_OK("sgpr_elbo");
  GPK_CHECK_ARG(N > 0 && M > 0 && P > 0 && ws && out, "sgpr_elbo: bad arguments");
  GPK_CHECK_ARG(noise > 0.0, "sgpr_elbo: noise variance must be positive");
  SgprWs w = sgpr_layout(ws, N, M, P, dtype);
  const size_t ts = dtype_size(dtype);
  GPK_TRY(sgpr_forward(nodes, n_nodes, dims, ard, X, N, ldx, D, Yc, P, Z, M, ldz, noise, jitter, dtype, out, w, st));
  if (cache_L) {
    GPK_TRY(axpby_impl(M, M, 1.0, w.b.Kuu, w.b.ldm, 0.0, cache_L, M, dtype, st));
    GPK_TRY(tril_impl(cache_L, M, M, 0, 1, dtype, st));
  }
  if (cache_LB) {
    GPK_TRY(axpby_impl(M, M, 1.0, w.b.Bm, w.b.ldm, 0.0, cache_LB, M, dtype, st));
    GPK_TRY(tril_impl(cache_LB, M, M, 0, 1, dtype, st));
  }
  if (cache_c) GPK_CUDA_OK(cudaMemcpyAsync(cache_c, w.b.c, (size_t)M * P * ts, cudaMemcpyDeviceToDevice, st));
  return 0;
}
namespace gpk {

// ---- value + gradient of the bound ----------------------------------------------------------------------------
// With s the noise variance, Yc = Y - m(X), K = Kuu + jitter I = L L^T, A' = L^-1 Kuf, B = I + A'A'^T / s = LB LB^T,
// c = LB^-1 A' Yc / s and v = LB^-T c:
//   dF/dKuu   = L^-T [P/2 (I - B^-1) - P/2 (B - I) - 1/2 v v^T] L^-1
//   dF/dKuf   = L^-T [H A' + v Yc^T / s],  H = (P/s)(I - B^-1) - v v^T / s
//   dF/dKdiag = -P / (2s)
//   dF/ds     = [-NP + P (M - tr B^-1) + P trace_k - P trace_q + sum Yc^2 / s - |c|^2 - |v|^2] / (2s)
//   dF/dm     = (Yc - A'^T v) / s
// L^-1 and B^-1 come from potri_lower on the two factors; the O(M^2 N) work added to the forward is the G_uf GEMM and
// the Kuf pass of inducing_grad_launch (grad.cu).

// The backward's M x M scratch, shared by SGPR, the Bayesian GPLVM and CGLB: Guu, Hm and T1 [M, ldm], potri_lower's tmp
// and two M x P vectors, x (SGPR's v, CGLB's Az) and Lx = L^-T x.
struct CollapsedGradWs {
  double *Guu, *Hm, *T1, *tmp, *x, *Lx;
};
static CollapsedGradWs collapsed_grad_layout(Arena& a, int64_t M, int64_t P, int64_t ldm, int dtype) {
  CollapsedGradWs w;
  const size_t ts = dtype_size(dtype);
  const int64_t h = M / 2 + NB;
  w.Guu = (double*)a.take((size_t)M * ldm * ts);
  w.Hm = (double*)a.take((size_t)M * ldm * ts);
  w.T1 = (double*)a.take((size_t)M * ldm * ts);
  w.tmp = (double*)a.take((size_t)h * h * ts);
  w.x = (double*)a.take((size_t)M * P * ts);
  w.Lx = (double*)a.take((size_t)M * P * ts);
  return w;
}

// Guu <- B - I = LB LB^T - I; Hm <- B^-1 (lower), LB^-1 over LB; *trace += tr B^-1
static int collapsed_binv(const CollapsedWs& f, const CollapsedGradWs& g, int64_t M, double* trace, cudaStream_t st) {
  const int64_t ldm = f.ldm;
  GPK_TRY(axpby_impl(M, M, 1.0, f.Bm, ldm, 0.0, g.T1, ldm, GPK_F64, st));
  GPK_TRY(tril_impl(g.T1, M, ldm, 0, 1, GPK_F64, st));
  GPK_TRY(gemm_any(0, 1, M, M, M, 1.0, g.T1, ldm, g.T1, ldm, 0.0, g.Guu, ldm, GPK_F64, 0, st));
  GPK_TRY(add_diag_impl(g.Guu, M, ldm, -1.0, nullptr, GPK_F64, st));
  GPK_TRY(potri_lower((double*)f.Bm, M, ldm, (const double*)f.dinvB, g.Hm, ldm, g.tmp, st));
  return reduce_impl(0, g.Hm, M, ldm + 1, 1.0, 1, trace, GPK_F64, st);
}

// L^-1 over L, its strict upper part zeroed (K^-1 into T1, unused)
static int collapsed_linv(const CollapsedWs& f, const CollapsedGradWs& g, int64_t M, cudaStream_t st) {
  GPK_TRY(potri_lower((double*)f.Kuu, M, f.ldm, (const double*)f.dinvL, g.T1, f.ldm, g.tmp, st));
  return tril_impl(f.Kuu, M, f.ldm, 0, 1, GPK_F64, st);
}

// out = alpha L^-T X L^-1 (Li = L^-1, lower) through T1 = X L^-1; out may be X
static int sandwich(double alpha, const void* Li, const double* X, double* out, double* T1, int64_t M, int64_t ld,
                    cudaStream_t st) {
  GPK_TRY(gemm_any(0, 0, M, M, M, 1.0, X, ld, Li, ld, 0.0, T1, ld, GPK_F64, 0, st));
  return gemm_any(1, 0, M, M, M, alpha, Li, ld, T1, ld, 0.0, out, ld, GPK_F64, 0, st);
}

// Guf = (L^-T H) A' + a (L^-T x) y^T with H in Hm, L^-1 over L, A' [M, ldn], y [N, P]
static int collapsed_guf(const CollapsedWs& f, const CollapsedGradWs& g, int64_t N, int64_t M, int64_t P,
                         const void* Ap, double a, const void* y, double* Guf, cudaStream_t st) {
  const void* Li = f.Kuu;
  const int64_t ldm = f.ldm, ldn = f.ldn;
  GPK_TRY(gemm_any(1, 0, M, M, M, 1.0, Li, ldm, g.Hm, ldm, 0.0, g.T1, ldm, GPK_F64, 0, st));
  GPK_TRY(gemm_any(0, 0, M, N, M, 1.0, g.T1, ldm, Ap, ldn, 0.0, Guf, ldn, GPK_F64, 0, st));
  GPK_TRY(gemm_any(1, 0, M, P, M, 1.0, Li, ldm, g.x, P, 0.0, g.Lx, P, GPK_F64, 0, st));
  return gemm_any(0, 1, M, N, P, a, g.Lx, P, y, P, 1.0, Guf, ldn, GPK_F64, 0, st);
}

struct SgprGradWs {
  SgprWs f; double* Guf; CollapsedGradWs g; double* dm; size_t dm_off, bytes;
};
static SgprGradWs sgpr_grad_layout(void* ws, int64_t N, int64_t M, int64_t P, int dtype) {
  SgprGradWs w;
  w.f = sgpr_layout(ws, N, M, P, dtype);
  Arena a(ws);
  a.off = w.f.bytes;
  const size_t ts = dtype_size(dtype);
  w.Guf = (double*)a.take((size_t)M * w.f.b.ldn * ts);
  w.g = collapsed_grad_layout(a, M, P, w.f.b.ldm, dtype);
  w.dm_off = a.off;
  w.dm = (double*)a.take((size_t)N * P * ts);
  w.bytes = a.off;
  return w;
}

}  // namespace gpk
extern "C" size_t gpk_sgpr_elbo_grad_ws(int64_t N, int64_t M, int64_t P, int dtype) {
  return sgpr_grad_layout(nullptr, N, M, P, dtype).bytes;
}
extern "C" size_t gpk_sgpr_elbo_grad_dm(int64_t N, int64_t M, int64_t P, int dtype) {
  return sgpr_grad_layout(nullptr, N, M, P, dtype).dm_off;
}
namespace gpk {

// In place on the M x M operands: Hm <- H, Guu (holding B - I) <- the bracket of dF/dKuu; Binv holds B^-1 (lower).
__global__ void sgpr_inner_kernel(const double* __restrict__ Binv, double* __restrict__ Guu, double* __restrict__ Hm,
                                  int64_t ld, const double* __restrict__ v, int64_t M, int64_t P, double s) {
  const int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= M * M) return;
  const int64_t i = e / M, j = e % M;
  const double bi = j <= i ? Binv[i * ld + j] : Binv[j * ld + i];
  double vv = 0.0;
  for (int64_t p = 0; p < P; ++p) vv = fma(v[i * P + p], v[j * P + p], vv);
  const double ib = (i == j ? 1.0 : 0.0) - bi;  // (I - B^-1)_ij
  Guu[i * ld + j] = 0.5 * (double)P * (ib - Guu[i * ld + j]) - 0.5 * vv;
  Hm[i * ld + j] = ((double)P * ib - vv) / s;
}

// The backward through G_uu, shared with the Bayesian GPLVM: v = LB^-T c into g.x, |v|^2 into scal[6], tr B^-1 into
// scal[5], Hm <- H, L^-1 over L and Guu <- G_uu = L^-T W L^-1, W = P/2 (I - B^-1) - P/2 (B - I) - v v^T / 2.
static int sgpr_backward(const CollapsedWs& f, const CollapsedGradWs& g, int64_t M, int64_t P, double s,
                         cudaStream_t st) {
  const int64_t ldm = f.ldm;
  GPK_CUDA_OK(cudaMemcpyAsync(g.x, f.c, (size_t)M * P * sizeof(double), cudaMemcpyDeviceToDevice, st));
  GPK_TRY(trsm_any(1, f.Bm, M, ldm, g.x, P, P, GPK_F64, f.dinvB, st));
  GPK_TRY(reduce_impl(1, g.x, M * P, 1, 1.0, 1, f.scal + 6, GPK_F64, st));
  GPK_TRY(collapsed_binv(f, g, M, f.scal + 5, st));
  // the two brackets: Guu <- W ; Hm <- H (B^-1 read from a copy in T1)
  GPK_TRY(axpby_impl(M, M, 1.0, g.Hm, ldm, 0.0, g.T1, ldm, GPK_F64, st));
  sgpr_inner_kernel<<<(unsigned)((M * M + 255) / 256), 256, 0, st>>>(g.T1, g.Guu, g.Hm, ldm, g.x, M, P, s);
  GPK_LAUNCH_OK();
  GPK_TRY(collapsed_linv(f, g, M, st));
  return sandwich(1.0, f.Kuu, g.Guu, g.Guu, g.T1, M, ldm, st);
}

// scal: 0..4 as the forward, 5 tr B^-1, 6 |v|^2
__global__ void sgpr_noise_grad_kernel(double* out, const double* scal, double N, double M, double P, double s) {
  out[8] = (-N * P + P * (M - scal[5]) + P * scal[0] - P * scal[1] + scal[3] - scal[4] - scal[6]) / (2.0 * s);
}

}  // namespace gpk
// out: [0..7] as gpk_sgpr_elbo; [8] d/dnoise_variance, [9 ...] the leaf slots (grad.cu); dZ [M, D] row-major
extern "C" int gpk_sgpr_elbo_grad(const gpk_knode* nodes, int n_nodes, const int32_t* dims, const double* ard,
                                  const void* X, int64_t N, int64_t ldx, int64_t D, const void* Yc, int64_t P,
                                  const void* Z, int64_t M, int64_t ldz, double noise, double jitter, int dtype,
                                  double* out, int n_out, double* dZ, void* ws, void* stream) {
  const cudaStream_t st = (cudaStream_t)stream;
  GPK_DTYPE_OK("sgpr_elbo_grad");
  GPK_CHECK_ARG(dtype == GPK_F64, "sgpr_elbo_grad: the device backward computes in float64 (dtype %d)", dtype);
  GPK_CHECK_ARG(N > 0 && M > 0 && P > 0 && D > 0 && ws && out && Yc && X && Z, "sgpr_elbo_grad: bad arguments");
  GPK_CHECK_ARG(dZ, "sgpr_elbo_grad: dZ [M, D] is required");
  GPK_CHECK_ARG(noise > 0.0, "sgpr_elbo_grad: noise variance must be positive");
  const int slots = grad_expr_slots(nodes, n_nodes, dims, ard, D, "sgpr_elbo_grad");
  if (slots < 0) return slots;
  GPK_CHECK_ARG(n_out >= 9 + slots, "sgpr_elbo_grad: n_out = %d, the expression needs %d outputs", n_out, 9 + slots);
  SgprGradWs w = sgpr_grad_layout(ws, N, M, P, dtype);
  const CollapsedWs& f = w.f.b;
  const double s = noise;
  GPK_CUDA_OK(cudaMemsetAsync(out, 0, (size_t)n_out * sizeof(double), st));
  GPK_CUDA_OK(cudaMemsetAsync(dZ, 0, (size_t)M * D * sizeof(double), st));
  GPK_TRY(sgpr_forward(nodes, n_nodes, dims, ard, X, N, ldx, D, Yc, P, Z, M, ldz, noise, jitter, dtype, out, w.f, st));
  GPK_CUDA_OK(cudaMemsetAsync(f.scal + 5, 0, 2 * sizeof(double), st));
  GPK_TRY(sgpr_backward(f, w.g, M, P, s, st));
  // G_uf = (L^-T H) A' + (L^-T v) Yc^T / s
  GPK_TRY(collapsed_guf(f, w.g, N, M, P, w.f.Kuf, 1.0 / s, Yc, w.Guf, st));
  // dF/dm = (Yc - A'^T v) / s
  GPK_TRY(gemm_any(1, 0, N, P, M, -1.0 / s, w.f.Kuf, f.ldn, w.g.x, P, 0.0, w.dm, P, dtype, 0, st));
  GPK_TRY(axpby_impl(N, P, 1.0 / s, Yc, P, 1.0, w.dm, P, dtype, st));
  sgpr_noise_grad_kernel<<<1, 1, 0, st>>>(out, f.scal, (double)N, (double)M, (double)P, s);
  GPK_LAUNCH_OK();
  return inducing_grad_launch(nodes, n_nodes, dims, ard, (const double*)X, N, ldx, D, (const double*)Z, M, ldz, w.Guf,
                              f.ldn, w.g.Guu, f.ldm, -(double)P / (2.0 * s), nullptr, out + 8, dZ, "sgpr_elbo_grad",
                              st);
}
namespace gpk {

// ---------------------------------------------------------------------------------------------
// Bayesian GPLVM (gplvm.py:162-216): the SGPR bound with Kuf Kuf^T -> psi2, Kuf -> psi1^T, sum Kdiag -> psi0, less
// the KL of q(X) = N(mu, diag S) from the prior N(m0, diag p0)
// ---------------------------------------------------------------------------------------------
struct BgWs {
  CollapsedWs b; void *P1, *P2, *psi, *kl; size_t bytes;
};
static BgWs bgplvm_layout(void* ws, int64_t N, int64_t Q, int64_t M, int64_t P) {
  Arena a(ws);
  BgWs w;
  w.b = collapsed_layout(a, N, M, P, GPK_F64);
  w.P1 = a.take((size_t)M * w.b.ldn * 8);
  w.P2 = a.take((size_t)M * w.b.ldm * 8);
  w.psi = a.take(psi_ws_bytes(N, M));
  w.kl = a.take((size_t)N * Q * 8);
  w.bytes = a.off;
  return w;
}

}  // namespace gpk
extern "C" size_t gpk_bgplvm_elbo_ws(int64_t N, int64_t Q, int64_t M, int64_t P) {
  return bgplvm_layout(nullptr, N, Q, M, P).bytes;
}
namespace gpk {

// scal: 0 psi0 / s, 1 tr(L^-1 psi2 L^-T) / s, 2 half_logdet_b, 3 sum Y^2 / s, 4 |c|^2, 5 tr B^-1, 6 |v|^2, 7 KL
__global__ void bgplvm_finalize_kernel(double* out, const double* scal, const int32_t* info, double N, double P,
                                       double noise) {
  const double trace_k = scal[0], trace_q = scal[1], half_logdet_b = scal[2];
  const double logdet = -P * (half_logdet_b + 0.5 * N * log(noise) + 0.5 * (trace_k - trace_q));  // gplvm.py:208,212
  const double quad = -0.5 * (scal[3] - scal[4]);                                                   // gplvm.py:210-211
  const double cst = -0.5 * N * P * LOG2PI;                                                         // gplvm.py:207
  out[0] = cst + logdet + quad - scal[7];
  out[1] = cst; out[2] = logdet; out[3] = quad; out[4] = trace_k; out[5] = trace_q; out[6] = half_logdet_b;
  out[7] = scal[7];
  out[8] = (double)(info[0] != 0 ? info[0] : info[1]);
}

// The bound's forward (gplvm.py:172-216).  Leaves L in w.b.Kuu, A' = L^-1 psi1^T in w.P1, LB in w.b.Bm, c in w.b.c and
// the scalars in w.b.scal and out[0..8].
static int bgplvm_forward(const gpk_knode* nodes, int n_nodes, const int32_t* dims, const double* ard, const double* mu,
                          const double* S, int64_t N, int64_t Q, const double* Y, int64_t P, const double* Z, int64_t M,
                          int64_t ldz, const double* m0, const double* p0, double noise, double jitter, double* out,
                          double* dmu, double* dS, const BgWs& w, const char* who, cudaStream_t st) {
  const CollapsedWs& b = w.b;
  const double inv_s = 1.0 / noise;
  const int64_t ldm = b.ldm, ldn = b.ldn;
  GPK_CUDA_OK(cudaMemsetAsync(b.scal, 0, 8 * sizeof(double), st));
  GPK_CUDA_OK(cudaMemsetAsync(b.info, 0, 2 * sizeof(int32_t), st));
  // psi0 / s = N sigma^2 / s (the psi statistics check the expression is one SquaredExponential leaf)
  GPK_TRY(fill_impl(b.scal, 1, 1, 1, (double)N * nodes[0].variance * inv_s, GPK_F64, st));
  GPK_TRY(psi_forward(nodes, n_nodes, dims, ard, mu, S, N, Q, Z, M, ldz, (double*)w.P1, 1, ldn, (double*)w.P2, ldm,
                      w.psi, who, st));
  // K = Kuu + jitter I = L L^T (gplvm.py:182-183)
  GPK_TRY(kbuild_impl(nodes, n_nodes, dims, ard, Z, M, ldz, nullptr, M, ldz, Q, b.Kuu, ldm, GPK_F64, GPK_LOWER, jitter,
                      nullptr, st));
  GPK_TRY(potrf_any(b.Kuu, M, M, ldm, GPK_F64, b.info, b.dinvL, st));
  // A' = L^-1 psi1^T ; L^-1 psi2 L^-T as two solves around a transpose, over s (gplvm.py:187-189)
  GPK_TRY(trsm_any(0, b.Kuu, M, ldm, w.P1, N, ldn, GPK_F64, b.dinvL, st));
  GPK_TRY(trsm_any(0, b.Kuu, M, ldm, w.P2, M, ldm, GPK_F64, b.dinvL, st));
  GPK_TRY(transpose_impl(w.P2, M, M, ldm, b.Bm, ldm, GPK_F64, st));
  GPK_TRY(trsm_any(0, b.Kuu, M, ldm, b.Bm, M, ldm, GPK_F64, b.dinvL, st));
  GPK_TRY(axpby_impl(M, M, 0.0, b.Bm, ldm, inv_s, b.Bm, ldm, GPK_F64, st));
  // B = I + AAT / s = LB LB^T, tr(AAT) / s, log det B / 2, c = LB^-1 A' Y / s (gplvm.py:189-193)
  GPK_TRY(collapsed_tail(b, N, M, P, w.P1, Y, inv_s, GPK_F64, st));
  // KL[q(X) || p(X)] (gplvm.py:195-204), with its gradient when dmu / dS are given
  GPK_TRY(kl_diag(mu, S, m0, p0, N * Q, (double*)w.kl, dmu, dS, st));
  GPK_TRY(reduce_impl(0, w.kl, N * Q, 1, 1.0, 1, b.scal + 7, GPK_F64, st));
  bgplvm_finalize_kernel<<<1, 1, 0, st>>>(out, b.scal, b.info, (double)N, (double)P, noise);
  GPK_LAUNCH_OK();
  return 0;
}

static int bgplvm_check(const double* mu, const double* S, int64_t N, int64_t Q, const double* Y, int64_t P,
                        const double* Z, int64_t M, int64_t ldz, const double* m0, const double* p0, double noise,
                        void* ws, double* out, const char* who) {
  GPK_CHECK_ARG(N > 0 && Q > 0 && M > 0 && P > 0 && ldz >= Q, "%s: bad sizes", who);
  GPK_CHECK_ARG(mu && S && Y && Z && m0 && p0 && ws && out, "%s: a required pointer is NULL", who);
  GPK_CHECK_ARG(noise > 0.0, "%s: noise variance must be positive", who);
  return 0;
}

}  // namespace gpk
extern "C" int gpk_bgplvm_elbo(const gpk_knode* nodes, int n_nodes, const int32_t* dims, const double* ard,
                               const double* mu, const double* S, int64_t N, int64_t Q, const double* Y, int64_t P,
                               const double* Z, int64_t M, int64_t ldz, const double* m0, const double* p0,
                               double noise, double jitter, double* out, void* ws, void* stream) {
  const cudaStream_t st = (cudaStream_t)stream;
  GPK_TRY(bgplvm_check(mu, S, N, Q, Y, P, Z, M, ldz, m0, p0, noise, ws, out, "bgplvm_elbo"));
  return bgplvm_forward(nodes, n_nodes, dims, ard, mu, S, N, Q, Y, P, Z, M, ldz, m0, p0, noise, jitter, out, nullptr,
                        nullptr, bgplvm_layout(ws, N, Q, M, P), "bgplvm_elbo", st);
}
namespace gpk {

struct BgGradWs {
  BgWs f; CollapsedGradWs g; double *G1, *G2, *gpar; size_t bytes;
};
static BgGradWs bgplvm_grad_layout(void* ws, int64_t N, int64_t Q, int64_t M, int64_t P) {
  BgGradWs w;
  w.f = bgplvm_layout(ws, N, Q, M, P);
  Arena a(ws);
  a.off = w.f.bytes;
  w.g = collapsed_grad_layout(a, M, P, w.f.b.ldm, GPK_F64);
  w.G1 = (double*)a.take((size_t)M * w.f.b.ldn * 8);
  w.G2 = (double*)a.take((size_t)M * w.f.b.ldm * 8);
  w.gpar = (double*)a.take(64 * 8);
  w.bytes = a.off;
  return w;
}

}  // namespace gpk
extern "C" size_t gpk_bgplvm_elbo_grad_ws(int64_t N, int64_t Q, int64_t M, int64_t P) {
  return bgplvm_grad_layout(nullptr, N, Q, M, P).bytes;
}
namespace gpk {

// out[10] (the variance slot) += gpar[0] - P N / (2s) (psi0 = N sigma^2); the lengthscale slot(s) += gpar[1 + d]
__global__ void bgplvm_kernel_grad_kernel(double* out, const double* gpar, int nd, int ard, double psi0_w) {
  out[10] += gpar[0] + psi0_w;
  for (int d = 0; d < nd; ++d) out[ard ? 11 + d : 11] += gpar[1 + d];
}

}  // namespace gpk
// out: [0..8] as gpk_bgplvm_elbo; [9] d/dnoise_variance, [10 ...] the leaf slots; dmu, dS [N, Q], dZ [M, Q] row-major
extern "C" int gpk_bgplvm_elbo_grad(const gpk_knode* nodes, int n_nodes, const int32_t* dims, const double* ard,
                                    const double* mu, const double* S, int64_t N, int64_t Q, const double* Y, int64_t P,
                                    const double* Z, int64_t M, int64_t ldz, const double* m0, const double* p0,
                                    double noise, double jitter, double* out, int n_out, double* dmu, double* dS,
                                    double* dZ, void* ws, void* stream) {
  const cudaStream_t st = (cudaStream_t)stream;
  const char* who = "bgplvm_elbo_grad";
  GPK_TRY(bgplvm_check(mu, S, N, Q, Y, P, Z, M, ldz, m0, p0, noise, ws, out, who));
  GPK_CHECK_ARG(dmu && dS && dZ, "%s: dmu, dS and dZ are required", who);
  const int slots = grad_expr_slots(nodes, n_nodes, dims, ard, Q, who);
  if (slots < 0) return slots;
  GPK_CHECK_ARG(n_out >= 10 + slots, "%s: n_out = %d, the expression needs %d outputs", who, n_out, 10 + slots);
  BgGradWs w = bgplvm_grad_layout(ws, N, Q, M, P);
  const CollapsedWs& f = w.f.b;
  const double s = noise;
  const int64_t ldm = f.ldm, ldn = f.ldn;
  GPK_CUDA_OK(cudaMemsetAsync(out, 0, (size_t)n_out * sizeof(double), st));
  GPK_CUDA_OK(cudaMemsetAsync(dmu, 0, (size_t)N * Q * sizeof(double), st));
  GPK_CUDA_OK(cudaMemsetAsync(dS, 0, (size_t)N * Q * sizeof(double), st));
  GPK_CUDA_OK(cudaMemsetAsync(dZ, 0, (size_t)M * Q * sizeof(double), st));
  GPK_CUDA_OK(cudaMemsetAsync(w.gpar, 0, 64 * sizeof(double), st));
  GPK_TRY(bgplvm_forward(nodes, n_nodes, dims, ard, mu, S, N, Q, Y, P, Z, M, ldz, m0, p0, noise, jitter, out, dmu, dS,
                         w.f, who, st));
  // dF/dKuu = L^-T W L^-1 into Guu, with H = (P (I - B^-1) - v v^T) / s in Hm
  GPK_TRY(sgpr_backward(f, w.g, M, P, s, st));
  // dF/dpsi2 = L^-T H L^-1 / 2
  GPK_TRY(sandwich(0.5, f.Kuu, w.g.Hm, w.G2, w.g.T1, M, ldm, st));
  // (dF/dpsi1)^T = u Y^T / s, u = L^-T v
  GPK_TRY(gemm_any(1, 0, M, P, M, 1.0, f.Kuu, ldm, w.g.x, P, 0.0, w.g.Lx, P, GPK_F64, 0, st));
  GPK_TRY(gemm_any(0, 1, M, N, P, 1.0 / s, w.g.Lx, P, Y, P, 0.0, w.G1, ldn, GPK_F64, 0, st));
  // d/dnoise: the SGPR formula with sum Kdiag -> psi0 and tr(A'A'^T) -> tr(L^-1 psi2 L^-T), into out[9]
  sgpr_noise_grad_kernel<<<1, 1, 0, st>>>(out + 1, f.scal, (double)N, (double)M, (double)P, s);
  GPK_LAUNCH_OK();
  // Kuu: the square pass of the expression reduction into the leaf slots out[10 ...] and dZ
  GPK_TRY(square_grad_launch(nodes, n_nodes, dims, ard, Z, M, ldz, Q, w.g.Guu, ldm, out + 9, dZ, who, st));
  // psi1, psi2: dmu, dS, dZ and the kernel parameters
  GPK_TRY(psi_backward(nodes, n_nodes, dims, ard, mu, S, N, Q, Z, M, ldz, w.G1, ldn, w.G2, ldm, dmu, dS, dZ, w.gpar,
                       w.f.psi, who, st));
  const gpk_knode& nd = nodes[0];
  bgplvm_kernel_grad_kernel<<<1, 1, 0, st>>>(out, w.gpar, nd.n_dims > 0 ? nd.n_dims : (int)Q, nd.n_ard > 0 ? 1 : 0,
                                             -(double)P * (double)N / (2.0 * s));
  GPK_LAUNCH_OK();
  return 0;
}
namespace gpk {

// ---------------------------------------------------------------------------------------------
// SVGP
// ---------------------------------------------------------------------------------------------
struct SvgpWs {
  void *Kuu, *A, *dinv, *v0, *fvar, *fmu, *tmpM, *tmpP, *kinv; int64_t ldm, ldb; int32_t* info; double* scal;
  size_t bytes, A_off, fvar_off, fmu_off;  // byte offsets (the pointers are null in a layout without a workspace)
};
static SvgpWs svgp_layout(void* ws, int64_t B, int64_t M, int64_t P, int dtype) {
  Arena a(ws);
  SvgpWs w;
  const size_t ts = dtype_size(dtype);
  w.ldm = pad_ld(M);
  w.ldb = pad_ld(B);
  w.Kuu = a.take((size_t)M * w.ldm * ts);
  w.A_off = a.off;
  w.A = a.take((size_t)M * w.ldb * ts);
  w.dinv = a.take(potrf_ws_bytes(M, M, dtype));
  w.v0 = a.take((size_t)B * ts);
  w.fvar_off = a.off;
  w.fvar = a.take((size_t)P * B * ts);   // [P][B]
  w.fmu_off = a.off;
  w.fmu = a.take((size_t)B * P * ts);    // [B][P]
  w.tmpM = a.take((size_t)M * w.ldm * ts);
  w.tmpP = a.take((size_t)M * P * ts);
  w.kinv = a.take((size_t)M * ts);
  w.info = (int32_t*)a.take(256);
  w.scal = (double*)a.take(256);
  w.bytes = a.off;
  return w;
}

// scal: 0 sum var_exp, 1 mahalanobis, 2 logdet_qcov, 3 trace, 4 sum log diag(Lp)^2
__global__ void svgp_finalize_kernel(double* out, const double* scal, const int32_t* info, double M, double Pl,
                                     double scale, int whiten) {
  double twoKL = scal[1] - M * Pl - scal[2] + scal[3];   // kullback_leiblers.py:124-155
  if (!whiten) twoKL += Pl * scal[4];                    // :158-163
  const double kl = 0.5 * twoKL;
  out[0] = scal[0] * scale - kl;                         // svgp.py:181
  out[1] = scal[0];
  out[2] = kl;
  out[3] = (double)info[0];
}

}  // namespace gpk
extern "C" size_t gpk_svgp_elbo_ws(int64_t B, int64_t M, int64_t P, int dtype) {
  return svgp_layout(nullptr, B, M, P, dtype).bytes;
}

// byte offset and leading dimension of A [M, ldb] inside the workspace (for the all-gather between stages 1 and 2)
extern "C" size_t gpk_svgp_elbo_A(int64_t B, int64_t M, int64_t P, int dtype, int64_t* ld) {
  SvgpWs w = svgp_layout(nullptr, B, M, P, dtype);
  if (ld) *ld = w.ldb;
  return w.A_off;
}

// byte offsets of fmean - m(X) [B][Pl] and fvar [Pl][B] inside the workspace, as svgp_forward leaves them
extern "C" int gpk_svgp_elbo_fmu_fvar(int64_t B, int64_t M, int64_t P, int dtype, int64_t* fmu, int64_t* fvar) {
  GPK_DTYPE_OK("svgp_elbo_fmu_fvar");
  GPK_CHECK_ARG(B > 0 && M > 0 && P > 0 && fmu && fvar, "svgp_elbo_fmu_fvar: bad arguments");
  SvgpWs w = svgp_layout(nullptr, B, M, P, dtype);
  *fmu = (int64_t)w.fmu_off;
  *fvar = (int64_t)w.fvar_off;
  return 0;
}
namespace gpk {

// The latent part of the forward for the latents [p_begin, p_end) of q_mu [M, P] / q_sqrt that share one Kuu: after
// stage 0 or 2, L in w.Kuu, A in w.A (L^-1 Kuf with whiten, K^-1 Kuf without), gmean = A^T q_mu in w.fmu [B][Pl] and
// gvar in w.fvar [Pl][B].  Stage 1 stops after the columns [c0, c1) of A.
static int svgp_latents(const gpk_knode* nodes, int n_nodes, const int32_t* dims, const double* ard, const void* Xb,
                        int64_t B, int64_t ldx, int64_t D, int64_t P, const void* Z, int64_t M, int64_t ldz,
                        const void* q_mu, const void* q_sqrt, int q_diag, int whiten, double jitter, int p_begin,
                        int p_end, int dtype, const SvgpWs& w, cudaStream_t st, int stage, int64_t c0, int64_t c1) {
  const size_t ts = dtype_size(dtype);
  const int64_t Pl = p_end - p_begin;
  const char* qmu = (const char*)q_mu;
  const char* qs = (const char*)q_sqrt;
  if (stage != 2) {
    // Kmm = Kuu + jitter ; Lm = chol(Kmm)   (posteriors.py:835, util.py:67)
    GPK_TRY(kbuild_impl(nodes, n_nodes, dims, ard, Z, M, ldz, nullptr, M, ldz, D, w.Kuu, w.ldm, dtype, GPK_LOWER, jitter,
                        nullptr, st));
    GPK_TRY(potrf_any(w.Kuu, M, M, w.ldm, dtype, w.info, w.dinv, st));
    // Kmn = Kuf [M,B] ; A = Lm^-1 Kmn   (posteriors.py:836, util.py:125); columns [c0, c1) only in stage 1
    if (c1 > c0) {
      char* Ac = (char*)w.A + (size_t)c0 * ts;
      GPK_TRY(kbuild_impl(nodes, n_nodes, dims, ard, Z, M, ldz, (const char*)Xb + (size_t)c0 * ldx * ts, c1 - c0, ldx, D,
                          Ac, w.ldb, dtype, GPK_FULL, 0.0, nullptr, st));
      GPK_TRY(trsm_any(0, w.Kuu, M, w.ldm, Ac, c1 - c0, w.ldb, dtype, w.dinv, st));
    }
    if (stage == 1) return 0;
  } else {
    GPK_CUDA_OK(cudaMemsetAsync(w.info, 0, sizeof(int32_t), st));
  }
  // fvar0 = Knn - sum_m A^2   (util.py:133)
  GPK_TRY(kdiag_impl(nodes, n_nodes, dims, ard, Xb, B, ldx, D, w.v0, dtype, st));
  GPK_TRY(colsumsq_impl(w.A, M, B, w.ldb, -1.0, 1, w.v0, dtype, st));
  if (!whiten) GPK_TRY(trsm_any(1, w.Kuu, M, w.ldm, w.A, B, w.ldb, dtype, w.dinv, st));  // util.py:138-139
  // fmean = A^T q_mu[:, p_begin:p_end]   (util.py:144)
  GPK_TRY(gemm_any(1, 0, B, Pl, M, 1.0, w.A, w.ldb, qmu + (size_t)p_begin * ts, P, 0.0, w.fmu, Pl, dtype, 0, st));
  // fvar_p = fvar0 + sum_m (q_sqrt_p^T A)^2   (util.py:149-164) — LTA is never materialised
  // fp32, dense q_sqrt: ALL latents in one batched int8 tensor-core launch (A split into TF32 planes once, one persistent grid
  // over P x tiles instead of P launches with a 2-wave tail each)
  static const bool batch_on = []() { const char* e = getenv("GPK_SVGP_BATCHED"); return !(e && e[0] == '0'); }();
  const bool batched = batch_on && !q_diag && dtype == GPK_F32 && Pl > 1 && M % 256 == 0 &&
                       gemm_tf32_eligible(M, B, M, nullptr, nullptr, nullptr, 0);
  for (int64_t p = p_begin; p < p_end; ++p) {
    char* fv = (char*)w.fvar + (size_t)(p - p_begin) * B * ts;
    GPK_CUDA_OK(cudaMemcpyAsync(fv, w.v0, (size_t)B * ts, cudaMemcpyDeviceToDevice, st));
    if (batched) continue;
    if (q_diag) {
      GPK_TRY(colsumsq_impl(w.A, M, B, w.ldb, 1.0, 1, fv, dtype, st, qs + (size_t)p * ts, P));
    } else {
      GPK_TRY(gemm_any(1, 0, M, B, M, 1.0, qs + (size_t)p * M * M * ts, M, w.A, w.ldb, 0.0, fv, 0, dtype,
                       GPK_GEMM_A_LOWER | GPK_GEMM_COLSUMSQ, st));
    }
  }
  if (batched)
    GPK_TRY(gemm_tf32(1, 0, M, B, M, 1.0f, (const float*)(qs + (size_t)p_begin * M * M * ts), M, (const float*)w.A, w.ldb, 0.0f,
                      (float*)w.fvar, 0, GPK_GEMM_A_LOWER | GPK_GEMM_COLSUMSQ, st, (int)Pl, M * M, B));
  return 0;
}

// KL[q || p] of the latents [p_begin, p_end) (kullback_leiblers.py:59-165), accumulated into w.scal[1..4] (the scalars
// svgp_finalize_kernel reads), with L in w.Kuu as svgp_latents leaves it.
static int svgp_kl(const void* q_mu, const void* q_sqrt, int q_diag, int whiten, int64_t M, int64_t P, int p_begin,
                   int p_end, int dtype, const SvgpWs& w, cudaStream_t st) {
  const size_t ts = dtype_size(dtype);
  const int64_t Pl = p_end - p_begin;
  const char* qmu = (const char*)q_mu;
  const char* qs = (const char*)q_sqrt;
  for (int64_t p = p_begin; p < p_end; ++p) {
    if (q_diag) {
      GPK_TRY(reduce_impl(3, qs + (size_t)p * ts, M, P, 1.0, 1, w.scal + 2, dtype, st));           // :130
    } else {
      GPK_TRY(reduce_impl(3, qs + (size_t)p * M * M * ts, M, M + 1, 1.0, 1, w.scal + 2, dtype, st));
    }
  }
  if (whiten) {
    for (int64_t p = p_begin; p < p_end; ++p)
      GPK_TRY(reduce_impl(1, qmu + (size_t)p * ts, M, P, 1.0, 1, w.scal + 1, dtype, st));           // :124
    if (q_diag) {
      for (int64_t p = p_begin; p < p_end; ++p)
        GPK_TRY(reduce_impl(1, qs + (size_t)p * ts, M, P, 1.0, 1, w.scal + 3, dtype, st));          // :134
    } else {
      GPK_TRY(tril_sumsq_impl(qs + (size_t)p_begin * M * M * ts, M, M, M * M, (int)Pl, 1.0, 1, w.scal + 3, dtype, st));
    }
  } else {
    // alpha = Lp^-1 q_mu  (:114)
    GPK_TRY(axpby_impl(M, Pl, 1.0, qmu + (size_t)p_begin * ts, P, 0.0, w.tmpP, Pl, dtype, st));
    GPK_TRY(trsm_any(0, w.Kuu, M, w.ldm, w.tmpP, Pl, Pl, dtype, w.dinv, st));
    GPK_TRY(reduce_impl(1, w.tmpP, M * Pl, 1, 1.0, 1, w.scal + 1, dtype, st));
    if (q_diag) {
      // K^-1 diagonal = column sums of squares of Lp^-1  (:136-145)
      GPK_TRY(fill_impl(w.tmpM, M, M, w.ldm, 0.0, dtype, st));
      GPK_TRY(add_diag_impl(w.tmpM, M, w.ldm, 1.0, nullptr, dtype, st));
      GPK_TRY(trsm_any(0, w.Kuu, M, w.ldm, w.tmpM, M, w.ldm, dtype, w.dinv, st));
      GPK_TRY(colsumsq_impl(w.tmpM, M, M, w.ldm, 1.0, 0, w.kinv, dtype, st));
      for (int64_t p = p_begin; p < p_end; ++p)
        GPK_TRY(reduce_wsq_impl(w.kinv, qs + (size_t)p * ts, M, P, 1.0, w.scal + 3, dtype, st));
    } else {
      for (int64_t p = p_begin; p < p_end; ++p) {  // trace = sum (Lp^-1 Lq)^2  (:152-153)
        GPK_TRY(axpby_impl(M, M, 1.0, qs + (size_t)p * M * M * ts, M, 0.0, w.tmpM, w.ldm, dtype, st));
        GPK_TRY(tril_impl(w.tmpM, M, w.ldm, 0, 1, dtype, st));
        GPK_TRY(trsm_any(0, w.Kuu, M, w.ldm, w.tmpM, M, w.ldm, dtype, w.dinv, st));
        GPK_TRY(colsumsq_impl(w.tmpM, M, M, w.ldm, 1.0, p == p_begin ? 0 : 1, w.kinv, dtype, st));
      }
      GPK_TRY(reduce_impl(0, w.kinv, M, 1, 1.0, 1, w.scal + 3, dtype, st));
    }
    GPK_TRY(reduce_impl(3, w.Kuu, M, w.ldm + 1, 1.0, 1, w.scal + 4, dtype, st));                   // :159-160
  }
  return 0;
}

// The ELBO's forward pass (svgp.py:166-181), shared by gpk_svgp_elbo_staged and gpk_svgp_elbo_grad: the variational
// expectations of `lik` on the raw targets Y [B, P] (MULTICLASS: the labels [B, 1]; HETEROSKEDASTIC: the targets
// [B, 1]) with m(X) [B, P] (NULL: zero mean) shifting fmean.  After stage 0 or 2: L in w.Kuu, A in w.A (L^-1 Kuf with
// whiten, K^-1 Kuf without), fmean - m(X) in w.fmu [B][Pl], fvar in w.fvar [Pl][B], out[0..3].
static int svgp_forward(const gpk_knode* nodes, int n_nodes, const int32_t* dims, const double* ard, const void* Xb,
                        int64_t B, int64_t ldx, int64_t D, const void* Y, const void* mX, int64_t P, const void* Z,
                        int64_t M, int64_t ldz, const void* q_mu, const void* q_sqrt, int q_diag, int whiten,
                        const gpk_lik* lik, double scale, double jitter, int p_begin, int p_end, int dtype, double* out,
                        const SvgpWs& w, cudaStream_t st, int stage, int64_t c0, int64_t c1) {
  const size_t ts = dtype_size(dtype);
  const int64_t Pl = p_end - p_begin;
  GPK_CUDA_OK(cudaMemsetAsync(w.scal, 0, 8 * sizeof(double), st));
  GPK_TRY(svgp_latents(nodes, n_nodes, dims, ard, Xb, B, ldx, D, P, Z, M, ldz, q_mu, q_sqrt, q_diag, whiten, jitter,
                       p_begin, p_end, dtype, w, st, stage, c0, c1));
  if (stage == 1) return 0;
  // sum of variational expectations (likelihoods/base.py:361-376) over the columns [p_begin, p_end) of Y and m(X)
  // (MULTICLASS, HETEROSKEDASTIC: p_begin = 0, the entries refuse a sub-range)
  GPK_TRY(lik_varexp_impl(lik, w.fmu, w.fvar, (const char*)Y + (size_t)p_begin * ts,
                          mX ? (const char*)mX + (size_t)p_begin * ts : nullptr, B, Pl, lik_ldy(lik, P), P, 1, B, 1.0,
                          1, w.scal + 0, dtype, st));
  GPK_TRY(svgp_kl(q_mu, q_sqrt, q_diag, whiten, M, P, p_begin, p_end, dtype, w, st));
  svgp_finalize_kernel<<<1, 1, 0, st>>>(out, w.scal, w.info, (double)M, (double)Pl, scale, whiten);
  GPK_LAUNCH_OK();
  return 0;
}

}  // namespace gpk
extern "C" int gpk_svgp_elbo_staged(const gpk_knode* nodes, int n_nodes, const int32_t* dims, const double* ard,
                                    const void* Xb, int64_t B, int64_t ldx, int64_t D, const void* Y, const void* mX,
                                    int64_t P, const void* Z, int64_t M, int64_t ldz, const void* q_mu,
                                    const void* q_sqrt, int q_diag, int whiten, const gpk_lik* lik, double scale,
                                    double jitter, int p_begin, int p_end, int stage, int64_t c0, int64_t c1, int dtype,
                                    double* out, void* ws, void* stream) {
  const cudaStream_t st = (cudaStream_t)stream;
  GPK_DTYPE_OK("svgp_elbo_staged");
  // stage 0: the whole evaluation.  Latent sharding over GPUs with a column-sharded triangular solve (SURVEY 8(e)):
  //   stage 1: Kuu, chol, and ONLY the columns [c0, c1) of Kuf / A = Lm^-1 Kuf (written in place in the workspace's
  //            A [M, ldb]; gpk_svgp_elbo_A locates it) -- the caller then all-gathers the column blocks of A;
  //   stage 2: everything after the solve for the latents [p_begin, p_end), A taken complete from the workspace.
  GPK_CHECK_ARG(B > 0 && M > 0 && P > 0 && ws && out && q_mu && q_sqrt, "svgp_elbo: bad arguments");
  GPK_CHECK_ARG(stage >= 0 && stage <= 2, "svgp_elbo: bad stage %d", stage);
  GPK_CHECK_ARG(stage == 0 || whiten, "svgp_elbo: the staged (column-sharded) evaluation covers whiten=True");
  if (stage != 1) { c0 = 0; c1 = B; }
  GPK_CHECK_ARG(0 <= c0 && c0 <= c1 && c1 <= B, "svgp_elbo: bad column range [%lld,%lld) of %lld", (long long)c0,
                (long long)c1, (long long)B);
  GPK_CHECK_ARG(0 <= p_begin && p_begin < p_end && p_end <= P, "svgp_elbo: bad latent range [%d,%d) of %lld", p_begin,
                p_end, (long long)P);
  GPK_TRY(lik_check(lik, P, "svgp_elbo"));
  GPK_CHECK_ARG(lik->type != GPK_LIK_MULTICLASS || (p_begin == 0 && p_end == P),
                "svgp_elbo: MultiClass couples the latents of a row; the latent range [%d,%d) must be [0,%lld)", p_begin,
                p_end, (long long)P);
  GPK_CHECK_ARG(lik->type != GPK_LIK_HETEROSKEDASTIC || (p_begin == 0 && p_end == P),
                "svgp_elbo: the heteroskedastic likelihood couples the latents of a row; the latent range [%d,%d) must "
                "be [0,%lld)", p_begin, p_end, (long long)P);
  return svgp_forward(nodes, n_nodes, dims, ard, Xb, B, ldx, D, Y, mX, P, Z, M, ldz, q_mu, q_sqrt, q_diag, whiten, lik,
                      scale, jitter, p_begin, p_end, dtype, out, svgp_layout(ws, B, M, P, dtype), st, stage, c0, c1);
}

extern "C" int gpk_svgp_elbo(const gpk_knode* nodes, int n_nodes, const int32_t* dims, const double* ard,
                             const void* Xb, int64_t B, int64_t ldx, int64_t D, const void* Y, const void* mX,
                             int64_t P, const void* Z, int64_t M, int64_t ldz, const void* q_mu, const void* q_sqrt,
                             int q_diag, int whiten, const gpk_lik* lik, double scale, double jitter, int p_begin,
                             int p_end, int dtype, double* out, void* ws, void* stream) {
  GPK_DTYPE_OK("svgp_elbo");
  return gpk_svgp_elbo_staged(nodes, n_nodes, dims, ard, Xb, B, ldx, D, Y, mX, P, Z, M, ldz, q_mu, q_sqrt, q_diag,
                              whiten, lik, scale, jitter, p_begin, p_end, 0, 0, 0, dtype, out, ws, stream);
}
namespace gpk {

// ---- value + gradient of the ELBO ------------------------------------------------------------------------------
// With c = num_data / B, the likelihood's adjoints R[n,p] = c dVE/dfmean [B, P] and W[n,p] = c dVE/dfvar
// (lik.cu::lik_grad_kernel), K = Kuu + jitter I = L L^T, S_p = tril(q_sqrt[p]), m = q_mu, Sig = sum_p S_p S_p^T,
// A as the forward leaves it, Phi(T) = tril(T) with its diagonal halved and sym(T) = (T + T^T) / 2:
//   whiten:  Abar = m R^T + 2 sum_p (S_p S_p^T - I) A diag(W_p),  dF/dKuf = L^-T Abar,
//            dF/dKuu = -sym(L^-T Phi(Abar A^T) L^-1)  (the Cholesky adjoint: the whitened ELBO depends on L, not only
//            on K),  dF/dq_mu = A R - m,  dF/dS_p = tril(2 A diag(W_p) A^T S_p - S_p) + diag(1 / diag S_p)
//   otherwise: Abar = m R^T + 2 sum_p S_p S_p^T A diag(W_p),  dF/dKuf = K^-1 Abar - 2 A diag(sum_p W_p),
//            dF/dKuu = sym(-K^-1 Abar A^T) + A diag(sum_p W_p) A^T + 1/2 K^-1 (m m^T + Sig) K^-1 - P/2 K^-1,
//            dF/dq_mu = A R - K^-1 m,  dF/dS_p = tril(2 A diag(W_p) A^T S_p - K^-1 S_p) + diag(1 / diag S_p)
//   both:    dF/dKdiag[n] = sum_p W[n,p],  dF/dm(X) = R
// (svgp.py:166-181 through conditionals/util.py:84-169 and kullback_leiblers.py:59-165).  q_diag restricts the forms to
// the diagonal.  The kernel parameters and Z then go through the three passes of inducing_grad_launch (grad.cu).
// The likelihood picks one of two routes through the middle of the backward:
//   uniform (Gaussian, W = w = -c / (2s) everywhere): the products over latents are shared, Sig A and A A^T formed
//     once; Abar = m R^T + 2w (Sig - [whiten] P I) A, the Kuf term -2wP A, the Kuu term wP A A^T, the Kdiag weight P w;
//   per latent (any other likelihood): per latent p, T = A diag(W_p), U = S_p^T T, Abar += 2 S_p U and G_p = T A^T,
//     through M x B / M x M scratch buffers that only this route's workspace holds.
struct SvgpGradWs {
  SvgpWs f;
  void *R, *Abar, *Guf, *Sig, *T, *AAt, *Guu, *Kinv, *Lc, *St, *tmp, *sig;
  void *Tb, *Ub, *Gp, *Gsum, *Wt, *Wsum;  // the per-latent route's buffers (NULL on the uniform route)
  size_t dm_off, bytes;
};
// the uniform route; a NULL descriptor (refused by the entry) sizes the larger workspace
static bool svgp_uniform_weights(const gpk_lik* lik) { return lik && lik->type == GPK_LIK_GAUSSIAN; }

static SvgpGradWs svgp_grad_layout(void* ws, int64_t B, int64_t M, int64_t P, int dtype, bool per_latent) {
  SvgpGradWs w;
  w.f = svgp_layout(ws, B, M, P, dtype);
  Arena a(ws);
  a.off = w.f.bytes;
  const size_t ts = dtype_size(dtype);
  const size_t mm = (size_t)M * w.f.ldm * ts, mb = (size_t)M * w.f.ldb * ts;
  const int64_t h = M / 2 + NB;
  w.dm_off = a.off;
  w.R = a.take((size_t)B * P * ts);
  w.Abar = a.take(mb);
  w.Guf = a.take(mb);
  w.Sig = a.take(mm);
  w.T = a.take(mm);
  w.AAt = a.take(mm);
  w.Guu = a.take(mm);
  w.Kinv = a.take(mm);
  w.Lc = a.take(mm);
  w.St = a.take(mm > (size_t)P * M * ts ? mm : (size_t)P * M * ts);
  w.tmp = a.take((size_t)h * h * ts);
  w.sig = a.take((size_t)M * ts);
  w.Tb = w.Ub = w.Gp = w.Gsum = w.Wt = w.Wsum = nullptr;
  if (per_latent) {
    w.Tb = a.take(mb);
    w.Ub = a.take(mb);
    w.Gp = a.take(mm);
    w.Gsum = a.take(mm);
    w.Wt = a.take((size_t)P * B * ts);
    w.Wsum = a.take((size_t)B * ts);
  }
  w.bytes = a.off;
  return w;
}

}  // namespace gpk
extern "C" size_t gpk_svgp_elbo_grad_ws(int64_t B, int64_t M, int64_t P, const gpk_lik* lik, int dtype) {
  return svgp_grad_layout(nullptr, B, M, P, dtype, !svgp_uniform_weights(lik)).bytes;
}
extern "C" size_t gpk_svgp_elbo_grad_dm(int64_t B, int64_t M, int64_t P, int dtype) {
  return svgp_grad_layout(nullptr, B, M, P, dtype, false).dm_off;
}
namespace gpk {

// The M x M brackets (the modes are listed at svgp_bracket in internal.cuh)
__global__ void svgp_bracket_kernel(int mode, const double* __restrict__ T, double* G, int64_t M, int64_t ld,
                                    const double* __restrict__ AAt, const double* __restrict__ V,
                                    const double* __restrict__ Kinv, double wP, double P) {
  const int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= M * M) return;
  const int64_t i = e / M, j = e % M, ij = i * ld + j, ji = j * ld + i;
  if (mode == SB_MIRROR) {
    if (j > i) G[ij] = G[ji];
  } else if (mode == SB_PHI) {
    G[ij] = j < i ? T[ij] : (j == i ? 0.5 * T[ij] : 0.0);
  } else {
    double v = -0.5 * (T[ij] + T[ji]);
    if (mode == SB_UNWHITENED) v += wP * AAt[ij] + 0.25 * (V[ij] + V[ji]) - 0.5 * P * Kinv[ij];
    G[ij] = v;
  }
}

// dF/dq_sqrt.  Dense (one latent): T [M, ldt] holds 2w S^T AAt (minus S^T K^-1 without whiten), the transpose of the
// product term, so dS[i,j] = T[j,i] (- S[i,j] with whiten) (+ 1 / S[i,i] on the diagonal) for j <= i, 0 above.
// q_diag: S and dS [M, P], dS = 2w s AAt_mm - (s with whiten, K^-1_mm s without) + 1 / s.
__global__ void svgp_dqsqrt_kernel(int q_diag, int whiten, const double* __restrict__ T, const double* __restrict__ S,
                                   double* __restrict__ dS, int64_t M, int64_t P, const double* __restrict__ AAt,
                                   const double* __restrict__ Kinv, int64_t ldm, double w2) {
  const int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (q_diag) {
    if (e >= M * P) return;
    const int64_t m = e / P;
    const double sv = S[e];
    dS[e] = w2 * sv * AAt[m * ldm + m] - (whiten ? sv : Kinv[m * ldm + m] * sv) + 1.0 / sv;
    return;
  }
  if (e >= M * M) return;
  const int64_t i = e / M, j = e % M;
  if (j > i) {
    dS[e] = 0.0;
    return;
  }
  double v = T[j * ldm + i] - (whiten ? S[e] : 0.0);
  if (i == j) v += 1.0 / S[e];
  dS[e] = v;
}

int svgp_bracket(int mode, const void* T, void* G, int64_t M, int64_t ld, const void* AAt, const void* V,
                 const void* Kinv, double wP, double P, cudaStream_t st) {
  const unsigned g = (unsigned)((M * M + 255) / 256);
  svgp_bracket_kernel<<<g, 256, 0, st>>>(mode, (const double*)T, (double*)G, M, ld, (const double*)AAt,
                                         (const double*)V, (const double*)Kinv, wP, P);
  GPK_LAUNCH_OK();
  return 0;
}

// The whitened Cholesky adjoint G = -sym(L^-T Phi(T) L^-1) of L [n, ld] (lower, with its block inverses dinv); T is
// overwritten.  Not static: gpk_debug_inverse_chain tests it directly.
int chol_adjoint(const void* L, const void* dinv, int64_t n, int64_t ld, void* T, void* G, cudaStream_t st) {
  GPK_TRY(svgp_bracket(SB_PHI, T, G, n, ld, nullptr, nullptr, nullptr, 0.0, 0.0, st));
  GPK_TRY(trsm_any(1, L, n, ld, G, n, ld, GPK_F64, dinv, st));
  GPK_TRY(transpose_impl(G, n, n, ld, T, ld, GPK_F64, st));
  GPK_TRY(trsm_any(1, L, n, ld, T, n, ld, GPK_F64, dinv, st));
  return svgp_bracket(SB_SYMNEG, T, G, n, ld, nullptr, nullptr, nullptr, 0.0, 0.0, st);
}

// Sig [M, ldm] = sum_p S_p S_p^T in full, S_p = tril(q_sqrt[p]) of a dense q_sqrt [P, M, M]; St [M, ldm] is scratch.
static int dense_sig(const void* q_sqrt, int64_t M, int64_t P, void* St, void* Sig, int64_t ldm, int dtype,
                     cudaStream_t st) {
  const char* qs = (const char*)q_sqrt;
  for (int64_t p = 0; p < P; ++p) {
    GPK_TRY(axpby_impl(M, M, 1.0, qs + (size_t)p * M * M * sizeof(double), M, 0.0, St, ldm, dtype, st));
    GPK_TRY(tril_impl(St, M, ldm, 0, 1, dtype, st));
    GPK_TRY(gemm_any(0, 1, M, M, M, 1.0, St, ldm, St, ldm, p ? 1.0 : 0.0, Sig, ldm, dtype,
                     GPK_GEMM_A_LOWER | GPK_GEMM_LOWER_ONLY, st));
  }
  return svgp_bracket(SB_MIRROR, nullptr, Sig, M, ldm, nullptr, nullptr, nullptr, 0.0, 0.0, st);
}

// out[m,b] = beta out[m,b] + alpha A[m,b] c[m,b] over the M x B operand (A, out [M, ld]), with
//   c[m,b] = sum_{p0 <= p < p1} (sd2[m,p] - h) Wt[p,b],  sd2 = Sd[m,p]^2 (Sd [M, P], the q_diag q_sqrt) or 0 without Sd,
// or, when Wt is NULL, c = A (the elementwise square).
__global__ void __launch_bounds__(256)
lik_colmix_kernel(const double* __restrict__ A, int64_t M, int64_t B, int64_t ld, const double* __restrict__ Sd,
                  double h, const double* __restrict__ Wt, int64_t P, int64_t p0, int64_t p1, double alpha, double beta,
                  double* __restrict__ out) {
  for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e < M * B; e += (int64_t)gridDim.x * blockDim.x) {
    const int64_t m = e / B, b = e % B;
    const double a = A[m * ld + b];
    double c = a;
    if (Wt) {
      c = 0.0;
      for (int64_t p = p0; p < p1; ++p) {
        const double sv = Sd ? Sd[m * P + p] : 0.0;
        c = fma(fma(sv, sv, -h), Wt[p * B + b], c);
      }
    }
    const double v = alpha * a * c;
    out[m * ld + b] = beta != 0.0 ? fma(beta, out[m * ld + b], v) : v;
  }
}

static int lik_colmix(const void* A, int64_t M, int64_t B, int64_t ld, const void* Sd, double h, const void* Wt,
                      int64_t P, int64_t p0, int64_t p1, double alpha, double beta, void* out, cudaStream_t st) {
  int64_t g = (M * B + 255) / 256;
  g = g < 4096 ? g : 4096;
  lik_colmix_kernel<<<(unsigned)g, 256, 0, st>>>((const double*)A, M, B, ld, (const double*)Sd, h, (const double*)Wt, P,
                                                 p0, p1, alpha, beta, (double*)out);
  GPK_LAUNCH_OK();
  return 0;
}

// dF/dq_sqrt with q_diag: dS[m,p] = 2 s AAW[m,p] - (s with whiten, K^-1_mm s without) + 1 / s, AAW = (A o A) W [M, P]
__global__ void lik_dqdiag_kernel(int whiten, const double* __restrict__ S, const double* __restrict__ AAW,
                                  const double* __restrict__ Kinv, int64_t ldm, int64_t M, int64_t P,
                                  double* __restrict__ dS) {
  const int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= M * P) return;
  const int64_t m = e / P;
  const double sv = S[e];
  dS[e] = 2.0 * sv * AAW[e] - (whiten ? sv : Kinv[m * ldm + m] * sv) + 1.0 / sv;
}

// The backward of a block of P latents that share one Kuu (the forms above), from R [B, P] (ld P) and, on the
// per-latent route, Wt [P, B]; Wt NULL takes the uniform route with the weight wv.  f holds L, its block inverses and
// A as svgp_latents leaves them; w's scratch buffers are overwritten.  The kernel slots go to gout[1 ...] and dZ
// [M, D], both accumulated (the caller zeroes them); dq_mu [M, P] and dq_sqrt (the shape of q_sqrt) are written.
static int svgp_backward(const gpk_knode* nodes, int n_nodes, const int32_t* dims, const double* ard, const void* Xb,
                         int64_t B, int64_t ldx, int64_t D, const void* Z, int64_t M, int64_t ldz, const void* q_mu,
                         const void* q_sqrt, int q_diag, int whiten, int64_t P, const double* R, const double* Wt,
                         double wv, const SvgpWs& f, const SvgpGradWs& w, double* gout, double* dZ, double* dq_mu,
                         double* dq_sqrt, const char* who, cudaStream_t st) {
  const int dtype = GPK_F64;
  const bool uniform = Wt == nullptr;
  const int64_t ldm = f.ldm, ldb = f.ldb;
  const double wP = (double)P * wv;
  const char* qs = (const char*)q_sqrt;
  const void* A = f.A;
  if (!whiten) {
    // K^-1 (full) from a copy of L
    GPK_TRY(axpby_impl(M, M, 1.0, f.Kuu, ldm, 0.0, w.Lc, ldm, dtype, st));
    GPK_TRY(potri_lower((double*)w.Lc, M, ldm, (const double*)f.dinv, (double*)w.Kinv, ldm, (double*)w.tmp, st));
    GPK_TRY(svgp_bracket(SB_MIRROR, nullptr, w.Kinv, M, ldm, nullptr, nullptr, nullptr, 0.0, 0.0, st));
  }
  // Sig = sum_p S_p S_p^T (full), minus P I with whiten: the uniform route's Sig A, and V without whiten
  if (uniform || !whiten) {
    if (q_diag) {
      GPK_TRY(transpose_impl(q_sqrt, M, P, P, w.St, M, dtype, st));
      GPK_TRY(colsumsq_impl(w.St, P, M, M, 1.0, 0, w.sig, dtype, st));
      GPK_TRY(fill_impl(w.Sig, M, M, ldm, 0.0, dtype, st));
      GPK_TRY(add_diag_impl(w.Sig, M, ldm, whiten ? -(double)P : 0.0, w.sig, dtype, st));
    } else {
      GPK_TRY(dense_sig(q_sqrt, M, P, w.St, w.Sig, ldm, dtype, st));
      if (whiten) GPK_TRY(add_diag_impl(w.Sig, M, ldm, -(double)P, nullptr, dtype, st));
    }
  }
  // Abar, dF/dq_sqrt, and without whiten the Kuu term A diag(sum_p W_p) A^T (AAt scaled by wP, or Gsum)
  if (uniform) {
    // Abar = m R^T + 2w Sig' A (Sig' = Sig - P I with whiten); A A^T (lower, then mirrored)
    GPK_TRY(gemm_any(0, 0, M, B, M, 2.0 * wv, w.Sig, ldm, A, ldb, 0.0, w.Abar, ldb, dtype, 0, st));
    GPK_TRY(gemm_any(0, 1, M, B, P, 1.0, q_mu, P, R, P, 1.0, w.Abar, ldb, dtype, 0, st));
    GPK_TRY(gemm_any(0, 1, M, M, B, 1.0, A, ldb, A, ldb, 0.0, w.AAt, ldm, dtype, GPK_GEMM_LOWER_ONLY, st));
    GPK_TRY(svgp_bracket(SB_MIRROR, nullptr, w.AAt, M, ldm, nullptr, nullptr, nullptr, 0.0, 0.0, st));
    if (q_diag) {
      const unsigned g = (unsigned)((M * P + 255) / 256);
      svgp_dqsqrt_kernel<<<g, 256, 0, st>>>(1, whiten, nullptr, (const double*)q_sqrt, dq_sqrt, M, P,
                                            (const double*)w.AAt, (const double*)w.Kinv, ldm, 2.0 * wv);
      GPK_LAUNCH_OK();
    } else {
      const unsigned g = (unsigned)((M * M + 255) / 256);
      for (int64_t p = 0; p < P; ++p) {
        const char* Sp = qs + (size_t)p * M * M * sizeof(double);
        // T = 2w S_p^T AAt (- S_p^T K^-1) = the transpose of 2w AAt S_p (- K^-1 S_p)
        GPK_TRY(gemm_any(1, 0, M, M, M, 2.0 * wv, Sp, M, w.AAt, ldm, 0.0, w.T, ldm, dtype, GPK_GEMM_A_LOWER, st));
        if (!whiten)
          GPK_TRY(gemm_any(1, 0, M, M, M, -1.0, Sp, M, w.Kinv, ldm, 1.0, w.T, ldm, dtype, GPK_GEMM_A_LOWER, st));
        svgp_dqsqrt_kernel<<<g, 256, 0, st>>>(0, whiten, (const double*)w.T, (const double*)Sp,
                                              dq_sqrt + (size_t)p * M * M, M, P, nullptr, nullptr, ldm, 0.0);
        GPK_LAUNCH_OK();
      }
    }
  } else {
    // Wsum = sum_p W_p; Abar = m R^T + 2 sum_p (S_p S_p^T - [whiten] I) A diag(W_p)
    for (int64_t p = 0; p < P; ++p)
      GPK_TRY(axpby_impl(1, B, 1.0, Wt + p * B, B, p ? 1.0 : 0.0, w.Wsum, B, dtype, st));
    GPK_TRY(gemm_any(0, 1, M, B, P, 1.0, q_mu, P, R, P, 0.0, w.Abar, ldb, dtype, 0, st));
    if (q_diag) {
      GPK_TRY(lik_colmix(A, M, B, ldb, q_sqrt, whiten ? 1.0 : 0.0, Wt, P, 0, P, 2.0, 1.0, w.Abar, st));
      // AAW = (A o A) W [M, P] into St
      GPK_TRY(lik_colmix(A, M, B, ldb, nullptr, 0.0, nullptr, P, 0, 0, 1.0, 0.0, w.Tb, st));
      GPK_TRY(gemm_any(0, 1, M, P, B, 1.0, w.Tb, ldb, Wt, B, 0.0, w.St, P, dtype, 0, st));
      const unsigned g = (unsigned)((M * P + 255) / 256);
      lik_dqdiag_kernel<<<g, 256, 0, st>>>(whiten, (const double*)q_sqrt, (const double*)w.St, (const double*)w.Kinv,
                                           ldm, M, P, dq_sqrt);
      GPK_LAUNCH_OK();
      if (!whiten) {
        GPK_TRY(lik_colmix(A, M, B, ldb, nullptr, -1.0, Wt, P, 0, P, 1.0, 0.0, w.Tb, st));
        GPK_TRY(gemm_any(0, 1, M, M, B, 1.0, w.Tb, ldb, A, ldb, 0.0, w.Gsum, ldm, dtype, GPK_GEMM_LOWER_ONLY, st));
        GPK_TRY(svgp_bracket(SB_MIRROR, nullptr, w.Gsum, M, ldm, nullptr, nullptr, nullptr, 0.0, 0.0, st));
      }
    } else {
      if (whiten) GPK_TRY(lik_colmix(A, M, B, ldb, nullptr, 1.0, Wt, P, 0, P, 2.0, 1.0, w.Abar, st));  // -2 A diag(sum W)
      const unsigned g = (unsigned)((M * M + 255) / 256);
      for (int64_t p = 0; p < P; ++p) {
        const char* Sp = qs + (size_t)p * M * M * sizeof(double);
        GPK_TRY(axpby_impl(M, M, 1.0, Sp, M, 0.0, w.St, ldm, dtype, st));  // S_p = tril(q_sqrt[p])
        GPK_TRY(tril_impl(w.St, M, ldm, 0, 1, dtype, st));
        // T = A diag(W_p); U = S_p^T T; Abar += 2 S_p U
        GPK_TRY(lik_colmix(A, M, B, ldb, nullptr, -1.0, Wt, P, p, p + 1, 1.0, 0.0, w.Tb, st));
        GPK_TRY(gemm_any(1, 0, M, B, M, 1.0, w.St, ldm, w.Tb, ldb, 0.0, w.Ub, ldb, dtype, GPK_GEMM_A_LOWER, st));
        GPK_TRY(gemm_any(0, 0, M, B, M, 2.0, w.St, ldm, w.Ub, ldb, 1.0, w.Abar, ldb, dtype, GPK_GEMM_A_LOWER, st));
        // G_p = A diag(W_p) A^T (full)
        GPK_TRY(gemm_any(0, 1, M, M, B, 1.0, w.Tb, ldb, A, ldb, 0.0, w.Gp, ldm, dtype, GPK_GEMM_LOWER_ONLY, st));
        GPK_TRY(svgp_bracket(SB_MIRROR, nullptr, w.Gp, M, ldm, nullptr, nullptr, nullptr, 0.0, 0.0, st));
        if (!whiten) GPK_TRY(axpby_impl(M, M, 1.0, w.Gp, ldm, p ? 1.0 : 0.0, w.Gsum, ldm, dtype, st));
        // T = 2 S_p^T G_p (- S_p^T K^-1): the transpose of 2 G_p S_p (- K^-1 S_p)
        GPK_TRY(gemm_any(1, 0, M, M, M, 2.0, w.St, ldm, w.Gp, ldm, 0.0, w.T, ldm, dtype, GPK_GEMM_A_LOWER, st));
        if (!whiten)
          GPK_TRY(gemm_any(1, 0, M, M, M, -1.0, w.St, ldm, w.Kinv, ldm, 1.0, w.T, ldm, dtype, GPK_GEMM_A_LOWER, st));
        svgp_dqsqrt_kernel<<<g, 256, 0, st>>>(0, whiten, (const double*)w.T, (const double*)Sp,
                                              dq_sqrt + (size_t)p * M * M, M, P, nullptr, nullptr, ldm, 0.0);
        GPK_LAUNCH_OK();
      }
    }
  }
  const void* Guf;
  if (whiten) {
    // dF/dKuu = the Cholesky adjoint of T = Abar A^T; dF/dKuf = L^-T Abar, in place
    GPK_TRY(gemm_any(0, 1, M, M, B, 1.0, w.Abar, ldb, A, ldb, 0.0, w.T, ldm, dtype, 0, st));
    GPK_TRY(chol_adjoint(f.Kuu, f.dinv, M, ldm, w.T, w.Guu, st));
    GPK_TRY(trsm_any(1, f.Kuu, M, ldm, w.Abar, B, ldb, dtype, f.dinv, st));
    Guf = w.Abar;
    // dF/dq_mu = A R - m
    GPK_TRY(gemm_any(0, 0, M, P, B, 1.0, A, ldb, R, P, 0.0, dq_mu, P, dtype, 0, st));
    GPK_TRY(axpby_impl(M, P, -1.0, q_mu, P, 1.0, dq_mu, P, dtype, st));
  } else {
    // dF/dKuf = K^-1 Abar - 2 A diag(sum_p W_p), with T = (K^-1 Abar) A^T taken on the way
    GPK_TRY(gemm_any(0, 0, M, B, M, 1.0, w.Kinv, ldm, w.Abar, ldb, 0.0, w.Guf, ldb, dtype, 0, st));
    GPK_TRY(gemm_any(0, 1, M, M, B, 1.0, w.Guf, ldb, A, ldb, 0.0, w.T, ldm, dtype, 0, st));
    if (uniform)
      GPK_TRY(axpby_impl(M, B, -2.0 * wP, A, ldb, 1.0, w.Guf, ldb, dtype, st));
    else
      GPK_TRY(lik_colmix(A, M, B, ldb, nullptr, 1.0, Wt, P, 0, P, 2.0, 1.0, w.Guf, st));
    Guf = w.Guf;
    // V = K^-1 (m m^T + Sig) K^-1 into Sig (Lc is free after potri)
    GPK_TRY(gemm_any(0, 1, M, M, P, 1.0, q_mu, P, q_mu, P, 1.0, w.Sig, ldm, dtype, 0, st));
    GPK_TRY(gemm_any(0, 0, M, M, M, 1.0, w.Kinv, ldm, w.Sig, ldm, 0.0, w.Lc, ldm, dtype, 0, st));
    GPK_TRY(gemm_any(0, 0, M, M, M, 1.0, w.Lc, ldm, w.Kinv, ldm, 0.0, w.Sig, ldm, dtype, 0, st));
    // dF/dKuu = sym(-T) + A diag(sum_p W_p) A^T + sym(V) / 2 - P/2 K^-1
    GPK_TRY(svgp_bracket(SB_UNWHITENED, w.T, w.Guu, M, ldm, uniform ? w.AAt : w.Gsum, w.Sig, w.Kinv,
                         uniform ? wP : 1.0, (double)P, st));
    // dF/dq_mu = A R - K^-1 m
    GPK_TRY(gemm_any(0, 0, M, P, B, 1.0, A, ldb, R, P, 0.0, dq_mu, P, dtype, 0, st));
    GPK_TRY(gemm_any(0, 0, M, P, M, -1.0, w.Kinv, ldm, q_mu, P, 1.0, dq_mu, P, dtype, 0, st));
  }
  // the kernel parameters and Z: dF/dKuf, dF/dKuu and the Kdiag weights (P w, or sum_p W[n, p] per element)
  return inducing_grad_launch(nodes, n_nodes, dims, ard, (const double*)Xb, B, ldx, D, (const double*)Z, M, ldz,
                              (const double*)Guf, ldb, (const double*)w.Guu, ldm, uniform ? wP : 0.0,
                              uniform ? nullptr : (const double*)w.Wsum, gout, dZ, who, st);
}

}  // namespace gpk
// out: [0..3] as gpk_svgp_elbo; [4] d/d(likelihood parameter) (Gaussian: the variance, Student-t: the scale, otherwise
// 0), [5 ...] the leaf slots (grad.cu); dZ [M, D], dq_mu [M, P] and dq_sqrt (the shape of q_sqrt) row-major.
extern "C" int gpk_svgp_elbo_grad(const gpk_knode* nodes, int n_nodes, const int32_t* dims, const double* ard,
                                  const void* Xb, int64_t B, int64_t ldx, int64_t D, const void* Y, const void* mX,
                                  int64_t P, const void* Z, int64_t M, int64_t ldz, const void* q_mu,
                                  const void* q_sqrt, int q_diag, int whiten, const gpk_lik* lik, double scale,
                                  double jitter, int dtype, double* out, int n_out, double* dZ, double* dq_mu,
                                  double* dq_sqrt, void* ws, void* stream) {
  const cudaStream_t st = (cudaStream_t)stream;
  GPK_DTYPE_OK("svgp_elbo_grad");
  GPK_CHECK_ARG(dtype == GPK_F64, "svgp_elbo_grad: the device backward computes in float64 (dtype %d)", dtype);
  GPK_CHECK_ARG(B > 0 && M > 0 && P > 0 && D > 0 && ws && out && Y && Xb && Z && q_mu && q_sqrt,
                "svgp_elbo_grad: bad arguments");
  GPK_CHECK_ARG(dZ && dq_mu && dq_sqrt, "svgp_elbo_grad: dZ [M, D], dq_mu [M, P] and dq_sqrt are required");
  GPK_TRY(lik_check(lik, P, "svgp_elbo_grad"));
  const int slots = grad_expr_slots(nodes, n_nodes, dims, ard, D, "svgp_elbo_grad");
  if (slots < 0) return slots;
  GPK_CHECK_ARG(n_out >= 5 + slots, "svgp_elbo_grad: n_out = %d, the expression needs %d outputs", n_out, 5 + slots);
  const bool uniform = svgp_uniform_weights(lik);
  SvgpGradWs w = svgp_grad_layout(ws, B, M, P, dtype, !uniform);
  const SvgpWs& f = w.f;
  const double wv = uniform ? -scale / (2.0 * lik->noise) : 0.0;
  GPK_CUDA_OK(cudaMemsetAsync(out, 0, (size_t)n_out * sizeof(double), st));
  GPK_CUDA_OK(cudaMemsetAsync(dZ, 0, (size_t)M * D * sizeof(double), st));
  GPK_TRY(svgp_forward(nodes, n_nodes, dims, ard, Xb, B, ldx, D, Y, mX, P, Z, M, ldz, q_mu, q_sqrt, q_diag, whiten, lik,
                       scale, jitter, 0, (int)P, dtype, out, f, st, 0, 0, B));
  // R (also dF/dm(X)), out[4], and on the per-latent route W as Wt [P, B]
  GPK_TRY(lik_grad_impl(lik, (const double*)f.fmu, (const double*)f.fvar, (const double*)Y, lik_ldy(lik, P),
                        (const double*)mX, B, P, scale, (double*)w.R, (double*)w.Wt, out + 4, st));
  return svgp_backward(nodes, n_nodes, dims, ard, Xb, B, ldx, D, Z, M, ldz, q_mu, q_sqrt, q_diag, whiten, P,
                       (const double*)w.R, (const double*)w.Wt, wv, f, w, out + 4, dZ, dq_mu, dq_sqrt, "svgp_elbo_grad",
                       st);
}
namespace gpk {

// ---------------------------------------------------------------------------------------------
// Multi-output SVGP: value + gradient of the ELBO for L independent latent GPs g_l, each with its own kernel expression
// k_l and inducing inputs Z_l (or one of either shared by every latent), mixed into P outputs by W [P, L] or not mixed
// (P = L): SharedIndependent / SeparateIndependent / LinearCoregionalization with Shared- / SeparateIndependent
// inducing variables (conditionals/multioutput/conditionals.py:45-152,261-311, posteriors.py:844-901,1050-1086).
// ---------------------------------------------------------------------------------------------
// Per latent l the forward is the single-output forward with P = 1 on K_l = k_l(Z_l, Z_l) + jitter I, A_l, q_mu[:, l]
// and q_sqrt[l]: gmean[:, l], gvar[l, :] and the latent's KL terms.  Without W, fmean = gmean and fvar = gvar; with
// W (conditionals/util.py:518-563)
//   fmean = gmean W^T [B, P],   fvar = gvar^T (W o W)^T [B, P].
// The likelihood step gives R [B, P] = c dVE/dfmean and Wt [P, B] = c dVE/dfvar, and then
//   Rg = R W [B, L] (dF/dgmean),   Wg = (W o W)^T Wt [L, B] (dF/dgvar),   dW = R^T gmean + 2 W o (Wt gvar^T) [P, L]
// (Rg = R and Wg = Wt without W).  The KL is the sum of the latents' KLs (kullback_leiblers.py:31-49 with Kuu
// [L, M, M]).  Each latent's backward is svgp_backward with P = 1, driven by Rg[:, l] and Wg[l]; its kernel slots and
// dZ accumulate into its expression's slot range and its Z's dZ (summed where one is shared).  A Gaussian likelihood
// without W keeps the uniform route per latent (w_l = w); with W, w_l = w sum_p W[p,l]^2 depends on device data, so
// the latents take the per-latent route with Wg[l] (Wt filled by the likelihood step).
// Workspace: the single-output P = 1 layout (latent 0's L, A and block inverses, the shared forward scratch and one
// set of backward scratch buffers), then latents 1..L-1's L, A and block inverses, so O(L M (M + B)) in all, and the
// [B, L] / [P, B] mixing buffers.
struct SvgpMoWs {
  SvgpGradWs g;                     // P = 1: latent 0 and the shared scratch; g.R holds the gathered Rg[:, l]
  void** Kuu; void** A; void** dinv;  // per latent (host arrays of device pointers; null in a size-only layout)
  int32_t* info;                    // [L]
  double *gmT, *gvar, *gm, *fmu, *fvar, *R, *Wt, *Rg, *Wg, *WW, *dWt, *qm, *qs, *dqm, *dqs;
  size_t dm_off, bytes;
};
static SvgpMoWs svgp_mo_layout(void* ws, int64_t B, int64_t M, int64_t L, int64_t P, void** Kuu, void** A,
                               void** dinv) {
  SvgpMoWs w;
  w.g = svgp_grad_layout(ws, B, M, 1, GPK_F64, true);
  Arena a(ws);
  a.off = w.g.bytes;
  const size_t ts = sizeof(double);
  const SvgpWs& f = w.g.f;
  w.Kuu = Kuu; w.A = A; w.dinv = dinv;
  for (int64_t l = 0; l < L; ++l) {
    void* k = l ? a.take((size_t)M * f.ldm * ts) : f.Kuu;
    void* x = l ? a.take((size_t)M * f.ldb * ts) : f.A;
    void* d = l ? a.take(potrf_ws_bytes(M, M, GPK_F64)) : f.dinv;
    if (Kuu) { Kuu[l] = k; A[l] = x; dinv[l] = d; }
  }
  w.info = (int32_t*)a.take((size_t)L * sizeof(int32_t));
  w.gmT = (double*)a.take((size_t)L * B * ts);
  w.gvar = (double*)a.take((size_t)L * B * ts);
  w.gm = (double*)a.take((size_t)B * L * ts);
  w.fmu = (double*)a.take((size_t)B * P * ts);
  w.fvar = (double*)a.take((size_t)P * B * ts);
  w.dm_off = a.off;
  w.R = (double*)a.take((size_t)B * P * ts);
  w.Wt = (double*)a.take((size_t)P * B * ts);
  w.Rg = (double*)a.take((size_t)B * L * ts);
  w.Wg = (double*)a.take((size_t)L * B * ts);
  w.WW = (double*)a.take((size_t)P * L * ts);
  w.dWt = (double*)a.take((size_t)P * L * ts);
  w.qm = (double*)a.take((size_t)M * ts);
  w.qs = (double*)a.take((size_t)M * ts);
  w.dqm = (double*)a.take((size_t)M * ts);
  w.dqs = (double*)a.take((size_t)M * ts);
  w.bytes = a.off;
  return w;
}

}  // namespace gpk
extern "C" size_t gpk_svgp_mo_elbo_grad_ws(int64_t B, int64_t M, int64_t L, int64_t P, const gpk_lik*, int) {
  return svgp_mo_layout(nullptr, B, M, L, P, nullptr, nullptr, nullptr).bytes;
}
extern "C" size_t gpk_svgp_mo_elbo_grad_dm(int64_t B, int64_t M, int64_t L, int64_t P, int) {
  return svgp_mo_layout(nullptr, B, M, L, P, nullptr, nullptr, nullptr).dm_off;
}
namespace gpk {

// out[0..3] from the scalars of L latents (scal as svgp_finalize_kernel; scal[4] already summed over the latents'
// log det K_l) and the first non-zero Cholesky info of the latents
__global__ void svgp_mo_finalize_kernel(double* out, const double* scal, const int32_t* info, int L, double M,
                                        double scale, int whiten) {
  double twoKL = scal[1] - M * L - scal[2] + scal[3];
  if (!whiten) twoKL += scal[4];
  const double kl = 0.5 * twoKL;
  int bad = 0;
  for (int l = 0; l < L && !bad; ++l) bad = info[l];
  out[0] = scal[0] * scale - kl;
  out[1] = scal[0];
  out[2] = kl;
  out[3] = (double)bad;
}

// mode 0: WW = W o W;  mode 1: dW += 2 W o dWt   (n = P L elements)
__global__ void svgp_mo_mix_kernel(int mode, const double* __restrict__ W, const double* __restrict__ dWt, double* out,
                                   int64_t n) {
  const int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= n) return;
  const double v = W[e];
  if (mode == 0) out[e] = v * v;
  else out[e] = fma(2.0 * v, dWt[e], out[e]);
}

}  // namespace gpk
extern "C" int gpk_svgp_mo_elbo_grad(const gpk_kexpr* kernels, int n_kernels, const void* Xb, int64_t B, int64_t ldx,
                                     int64_t D, const void* Y, const void* mX, int64_t P, const void* const* Z, int n_z,
                                     int64_t M, int64_t ldz, int64_t L, const void* q_mu, const void* q_sqrt,
                                     int q_diag, int whiten, const void* W, const gpk_lik* lik, double scale,
                                     double jitter, int dtype, double* out, int n_out, double* const* dZ,
                                     double* dq_mu, double* dq_sqrt, double* dW, void* ws, void* stream) {
  const cudaStream_t st = (cudaStream_t)stream;
  GPK_DTYPE_OK("svgp_mo_elbo_grad");
  const char* who = "svgp_mo_elbo_grad";
  GPK_CHECK_ARG(dtype == GPK_F64, "svgp_mo_elbo_grad: the device backward computes in float64 (dtype %d)", dtype);
  GPK_CHECK_ARG(B > 0 && M > 0 && P > 0 && L > 0 && D > 0 && ws && out && Y && Xb && Z && kernels && q_mu && q_sqrt,
                "svgp_mo_elbo_grad: bad arguments");
  GPK_CHECK_ARG(n_kernels == 1 || n_kernels == L, "svgp_mo_elbo_grad: n_kernels = %d, must be 1 or L = %lld",
                n_kernels, (long long)L);
  GPK_CHECK_ARG(n_z == 1 || n_z == L, "svgp_mo_elbo_grad: n_z = %d, must be 1 or L = %lld", n_z, (long long)L);
  GPK_CHECK_ARG(W || P == L, "svgp_mo_elbo_grad: without a mixing matrix W the outputs are the latents (P = %lld, L = "
                "%lld)", (long long)P, (long long)L);
  GPK_CHECK_ARG(dZ && dq_mu && dq_sqrt && (!W || dW),
                "svgp_mo_elbo_grad: dZ [n_z][M, D], dq_mu [M, L], dq_sqrt and (with W) dW [P, L] are required");
  for (int z = 0; z < n_z; ++z)
    GPK_CHECK_ARG(Z[z] && dZ[z], "svgp_mo_elbo_grad: inducing set %d or its dZ is missing", z);
  GPK_TRY(lik_check(lik, P, who));
  std::vector<int> off(n_kernels + 1, 0);
  for (int k = 0; k < n_kernels; ++k) {
    const int s = grad_expr_slots(kernels[k].nodes, kernels[k].n_nodes, kernels[k].dims, kernels[k].ard, D, who);
    if (s < 0) return s;
    off[k + 1] = off[k] + s;
  }
  GPK_CHECK_ARG(n_out >= 5 + off[n_kernels], "svgp_mo_elbo_grad: n_out = %d, the expressions need %d outputs", n_out,
                5 + off[n_kernels]);
  std::vector<void*> Kuu(L), A(L), dinv(L);
  SvgpMoWs w = svgp_mo_layout(ws, B, M, L, P, Kuu.data(), A.data(), dinv.data());
  const SvgpWs& f0 = w.g.f;
  const size_t ts = sizeof(double);
  const char* qmu = (const char*)q_mu;
  const char* qs = (const char*)q_sqrt;
  GPK_CUDA_OK(cudaMemsetAsync(out, 0, (size_t)n_out * sizeof(double), st));
  for (int z = 0; z < n_z; ++z) GPK_CUDA_OK(cudaMemsetAsync(dZ[z], 0, (size_t)M * D * sizeof(double), st));
  GPK_CUDA_OK(cudaMemsetAsync(f0.scal, 0, 8 * sizeof(double), st));
  // the latents: L_l, A_l, gmean[:, l] (into gmT row l), gvar[l] and the KL terms
  std::vector<SvgpWs> lat(L, f0);
  for (int64_t l = 0; l < L; ++l) {
    SvgpWs& fl = lat[l];
    fl.Kuu = Kuu[l]; fl.A = A[l]; fl.dinv = dinv[l];
    fl.info = w.info + l;
    fl.fmu = w.gmT + l * B;
    fl.fvar = w.gvar + l * B;
    const gpk_kexpr& k = kernels[n_kernels > 1 ? l : 0];
    GPK_TRY(svgp_latents(k.nodes, k.n_nodes, k.dims, k.ard, Xb, B, ldx, D, L, Z[n_z > 1 ? l : 0], M, ldz, q_mu, q_sqrt,
                         q_diag, whiten, jitter, (int)l, (int)l + 1, dtype, fl, st, 0, 0, B));
    GPK_TRY(svgp_kl(q_mu, q_sqrt, q_diag, whiten, M, L, (int)l, (int)l + 1, dtype, fl, st));
  }
  // mixing: fmean = gmean W^T, fvar = (W o W) gvar  (or the latents themselves)
  GPK_TRY(transpose_impl(w.gmT, L, B, B, w.gm, L, dtype, st));
  const double* fmu = w.gm;
  const double* fvar = w.gvar;
  const unsigned gw = (unsigned)((P * L + 255) / 256);
  if (W) {
    svgp_mo_mix_kernel<<<gw, 256, 0, st>>>(0, (const double*)W, nullptr, w.WW, P * L);
    GPK_LAUNCH_OK();
    GPK_TRY(gemm_any(0, 1, B, P, L, 1.0, w.gm, L, W, L, 0.0, w.fmu, P, dtype, 0, st));
    GPK_TRY(gemm_any(0, 0, P, B, L, 1.0, w.WW, L, w.gvar, B, 0.0, w.fvar, B, dtype, 0, st));
    fmu = w.fmu;
    fvar = w.fvar;
  }
  GPK_TRY(lik_varexp_impl(lik, fmu, fvar, Y, mX, B, P, lik_ldy(lik, P), P, 1, B, 1.0, 1, f0.scal + 0, dtype, st));
  svgp_mo_finalize_kernel<<<1, 1, 0, st>>>(out, f0.scal, w.info, (int)L, (double)M, scale, whiten);
  GPK_LAUNCH_OK();
  // R (also dF/dm(X)), out[4], Wt; then the latents' adjoints Rg, Wg and dW
  GPK_TRY(lik_grad_impl(lik, fmu, fvar, (const double*)Y, lik_ldy(lik, P), (const double*)mX, B, P, scale, w.R, w.Wt,
                        out + 4, st));
  const double* Rg = w.R;
  const double* Wg = w.Wt;
  if (W) {
    GPK_TRY(gemm_any(0, 0, B, L, P, 1.0, w.R, P, W, L, 0.0, w.Rg, L, dtype, 0, st));
    GPK_TRY(gemm_any(1, 0, L, B, P, 1.0, w.WW, L, w.Wt, B, 0.0, w.Wg, B, dtype, 0, st));
    GPK_TRY(gemm_any(1, 0, P, L, B, 1.0, w.R, P, w.gm, L, 0.0, dW, L, dtype, 0, st));
    GPK_TRY(gemm_any(0, 1, P, L, B, 1.0, w.Wt, B, w.gvar, B, 0.0, w.dWt, L, dtype, 0, st));
    svgp_mo_mix_kernel<<<gw, 256, 0, st>>>(1, (const double*)W, w.dWt, dW, P * L);
    GPK_LAUNCH_OK();
    Rg = w.Rg;
    Wg = w.Wg;
  }
  const bool uniform = svgp_uniform_weights(lik) && !W;
  const double wv = uniform ? -scale / (2.0 * lik->noise) : 0.0;
  // each latent's backward: gather q_mu[:, l], q_sqrt[l] (a column with q_diag) and Rg[:, l]; scatter dq_mu / dq_sqrt
  for (int64_t l = 0; l < L; ++l) {
    const gpk_kexpr& k = kernels[n_kernels > 1 ? l : 0];
    const int z = n_z > 1 ? (int)l : 0;
    GPK_TRY(axpby_impl(M, 1, 1.0, qmu + l * ts, L, 0.0, w.qm, 1, dtype, st));
    GPK_TRY(axpby_impl(B, 1, 1.0, Rg + l, L, 0.0, w.g.R, 1, dtype, st));
    const void* qsl = qs + (size_t)l * M * M * ts;
    double* dqsl = dq_sqrt + (size_t)l * M * M;
    if (q_diag) {
      GPK_TRY(axpby_impl(M, 1, 1.0, qs + l * ts, L, 0.0, w.qs, 1, dtype, st));
      qsl = w.qs;
      dqsl = w.dqs;
    }
    GPK_TRY(svgp_backward(k.nodes, k.n_nodes, k.dims, k.ard, Xb, B, ldx, D, Z[z], M, ldz, w.qm, qsl, q_diag, whiten, 1,
                          (const double*)w.g.R, uniform ? nullptr : Wg + l * B, wv, lat[l], w.g,
                          out + 4 + off[n_kernels > 1 ? l : 0], dZ[z], w.dqm, dqsl, who, st));
    GPK_TRY(axpby_impl(M, 1, 1.0, w.dqm, 1, 0.0, dq_mu + l, L, dtype, st));
    if (q_diag) GPK_TRY(axpby_impl(M, 1, 1.0, w.dqs, 1, 0.0, dq_sqrt + l, L, dtype, st));
  }
  return 0;
}
namespace gpk {

// ---------------------------------------------------------------------------------------------
// VGP: value + gradient of the ELBO (vgp.py:111-143, Gaussian likelihood, whitened q over f = L v + m(X))
// ---------------------------------------------------------------------------------------------
// With s the noise variance, w = -1/(2s), K = k(X) + jitter I = L L^T, m = q_mu [N, P], S_p = tril(q_sqrt[p]),
// Sig = sum_p S_p S_p^T, R = (Yc - L m) / s [N, P], Phi(T) = tril(T) with its diagonal halved, sym(T) = (T + T^T) / 2:
//   Lbar = tril(R m^T + 2w L Sig)  (dF/dL),   dF/dK = sym(L^-T Phi(L^T Lbar) L^-1)  (the Cholesky adjoint),
//   dF/dq_mu = L^T R - m,   dF/dS_p = tril(2w (L^T L) S_p - S_p) + diag(1 / diag S_p),
//   dF/ds = sum_np [-1/(2s) + ((Yc - L m)^2 + fvar) / (2 s^2)],   dF/dm(X) = R.
// The jitter carries no parameter; the kernel parameters take sum_ij dF/dK_ij dK_ij/dtheta through the square pass of
// square_grad_launch (grad.cu).  This is the whitened SVGP form with A = L^T, c = 1 and no Kuf / Kdiag terms.

struct VgpGradWs {
  void *L, *dinv, *fmu, *fvar, *R, *Sig, *G, *LtL, *Lbar, *T, *St; int32_t* info; double* scal; int64_t ldn;
  size_t dm_off, scratch_bytes, bytes;
};
static VgpGradWs vgp_grad_layout(void* ws, int64_t N, int64_t P, int dtype) {
  Arena a(ws);
  VgpGradWs w;
  const size_t ts = dtype_size(dtype);
  w.ldn = pad_ld(N);
  const size_t nn = (size_t)N * w.ldn * ts;
  w.L = a.take(nn);
  w.dinv = a.take(potrf_ws_bytes(N, N, dtype));
  w.info = (int32_t*)a.take(256);
  w.scal = (double*)a.take(256);
  w.fmu = a.take((size_t)N * P * ts);   // [N][P]
  w.fvar = a.take((size_t)P * N * ts);  // [P][N]
  w.dm_off = a.off;
  w.R = a.take((size_t)N * P * ts);
  w.Sig = a.take(nn);
  w.G = a.take(nn);
  w.LtL = a.take(nn);
  // Lbar, T and St are dead when the square pass runs: their span is its discarded input-derivative scratch
  const size_t s0 = a.off;
  w.Lbar = a.take(nn);
  w.T = a.take(nn);
  w.St = a.take(nn);
  w.scratch_bytes = a.off - s0;
  w.bytes = a.off;
  return w;
}

}  // namespace gpk
extern "C" size_t gpk_vgp_elbo_grad_ws(int64_t N, int64_t P, int dtype) {
  return vgp_grad_layout(nullptr, N, P, dtype).bytes;
}
extern "C" size_t gpk_vgp_elbo_grad_dm(int64_t N, int64_t P, int dtype) {
  return vgp_grad_layout(nullptr, N, P, dtype).dm_off;
}

// out: [0] ELBO, [1] variational expectations, [2] KL, [3] Cholesky info, [4] d/dnoise_variance, [5 ...] the leaf slots
// (grad.cu); dq_mu [N, P] and dq_sqrt [P, N, N] row-major.
extern "C" int gpk_vgp_elbo_grad(const gpk_knode* nodes, int n_nodes, const int32_t* dims, const double* ard,
                                 const void* X, int64_t N, int64_t ldx, int64_t D, const void* Yc, int64_t P,
                                 const void* q_mu, const void* q_sqrt, double noise, double jitter, int dtype,
                                 double* out, int n_out, double* dq_mu, double* dq_sqrt, void* ws, void* stream) {
  const cudaStream_t st = (cudaStream_t)stream;
  GPK_DTYPE_OK("vgp_elbo_grad");
  GPK_CHECK_ARG(dtype == GPK_F64, "vgp_elbo_grad: the device backward computes in float64 (dtype %d)", dtype);
  GPK_CHECK_ARG(N > 0 && P > 0 && D > 0 && ws && out && Yc && X && q_mu && q_sqrt, "vgp_elbo_grad: bad arguments");
  GPK_CHECK_ARG(dq_mu && dq_sqrt, "vgp_elbo_grad: dq_mu [N, P] and dq_sqrt [P, N, N] are required");
  GPK_CHECK_ARG(noise > 0.0, "vgp_elbo_grad: noise variance must be positive");
  const int slots = grad_expr_slots(nodes, n_nodes, dims, ard, D, "vgp_elbo_grad");
  if (slots < 0) return slots;
  GPK_CHECK_ARG(n_out >= 5 + slots, "vgp_elbo_grad: n_out = %d, the expression needs %d outputs", n_out, 5 + slots);
  VgpGradWs w = vgp_grad_layout(ws, N, P, dtype);
  GPK_CHECK_ARG((size_t)N * D * sizeof(double) <= w.scratch_bytes,
                "vgp_elbo_grad: X has %lld columns, the workspace's scratch holds %lld for N = %lld", (long long)D,
                (long long)(w.scratch_bytes / ((size_t)N * sizeof(double))), (long long)N);
  const int64_t ldn = w.ldn;
  const double s = noise, wv = -1.0 / (2.0 * s);
  const char* qs = (const char*)q_sqrt;
  const size_t sq = (size_t)N * N * sizeof(double);
  gpk_lik gauss{};
  gauss.type = GPK_LIK_GAUSSIAN;
  gauss.noise = s;
  GPK_CUDA_OK(cudaMemsetAsync(out, 0, (size_t)n_out * sizeof(double), st));
  GPK_CUDA_OK(cudaMemsetAsync(w.scal, 0, 8 * sizeof(double), st));
  // ---- forward (vgp.py:124-142) ----
  // K = k(X) + jitter I, lower; L = chol(K) with its block inverses, strict upper part zeroed (tf.linalg.cholesky)
  GPK_TRY(kbuild_impl(nodes, n_nodes, dims, ard, X, N, ldx, nullptr, N, ldx, D, w.L, ldn, dtype, GPK_LOWER, jitter,
                      nullptr, st));
  GPK_TRY(potrf_any(w.L, N, N, ldn, dtype, w.info, w.dinv, st));
  GPK_TRY(tril_impl(w.L, N, ldn, 0, 1, dtype, st));
  // fmean - m(X) = L m;  fvar_p = column sums of squares of S_p^T L^T
  GPK_TRY(gemm_any(0, 0, N, P, N, 1.0, w.L, ldn, q_mu, P, 0.0, w.fmu, P, dtype, GPK_GEMM_A_LOWER, st));
  GPK_CUDA_OK(cudaMemsetAsync(w.fvar, 0, (size_t)P * N * sizeof(double), st));
  for (int64_t p = 0; p < P; ++p)
    GPK_TRY(gemm_any(1, 1, N, N, N, 1.0, qs + p * sq, N, w.L, ldn, 0.0, (double*)w.fvar + p * N, 0, dtype,
                     GPK_GEMM_A_LOWER | GPK_GEMM_COLSUMSQ, st));
  GPK_TRY(lik_varexp_impl(&gauss, w.fmu, w.fvar, Yc, nullptr, N, P, P, P, 1, N, 1.0, 1, w.scal + 0, dtype, st));
  // whitened KL (kullback_leiblers.py:124-155): |m|^2, sum log diag(S_p)^2, |tril S_p|^2
  GPK_TRY(reduce_impl(1, q_mu, N * P, 1, 1.0, 1, w.scal + 1, dtype, st));
  for (int64_t p = 0; p < P; ++p) GPK_TRY(reduce_impl(3, qs + p * sq, N, N + 1, 1.0, 1, w.scal + 2, dtype, st));
  GPK_TRY(tril_sumsq_impl(q_sqrt, N, N, N * N, (int)P, 1.0, 1, w.scal + 3, dtype, st));
  svgp_finalize_kernel<<<1, 1, 0, st>>>(out, w.scal, w.info, (double)N, (double)P, 1.0, 1);
  GPK_LAUNCH_OK();
  // ---- backward ----
  // R = (Yc - L m) / s (also dF/dm(X)) and the noise gradient: the Gaussian likelihood's adjoints
  GPK_TRY(lik_grad_impl(&gauss, (const double*)w.fmu, (const double*)w.fvar, (const double*)Yc, P, nullptr, N, P,
                        1.0, (double*)w.R, nullptr, out + 4, st));
  // Lbar = tril(R m^T + 2w L Sig)
  GPK_TRY(dense_sig(q_sqrt, N, P, w.St, w.Sig, ldn, dtype, st));
  GPK_TRY(gemm_any(0, 1, N, N, P, 1.0, w.R, P, q_mu, P, 0.0, w.Lbar, ldn, dtype, 0, st));
  GPK_TRY(gemm_any(0, 0, N, N, N, 2.0 * wv, w.L, ldn, w.Sig, ldn, 1.0, w.Lbar, ldn, dtype,
                   GPK_GEMM_A_LOWER | GPK_GEMM_LOWER_ONLY, st));
  GPK_TRY(tril_impl(w.Lbar, N, ldn, 0, 1, dtype, st));
  // dF/dK = sym(Y), Y = (L^-T Phi(L^T Lbar) L^-1)^T: T = -L^T Lbar (its lower part) makes SB_SYMNEG's -sym a +sym
  GPK_TRY(gemm_any(1, 0, N, N, N, -1.0, w.L, ldn, w.Lbar, ldn, 0.0, w.T, ldn, dtype,
                   GPK_GEMM_A_LOWER | GPK_GEMM_LOWER_ONLY, st));
  GPK_TRY(chol_adjoint(w.L, w.dinv, N, ldn, w.T, w.G, st));
  // dF/dq_mu = L^T R - m
  GPK_TRY(gemm_any(1, 0, N, P, N, 1.0, w.L, ldn, w.R, P, 0.0, dq_mu, P, dtype, GPK_GEMM_A_LOWER, st));
  GPK_TRY(axpby_impl(N, P, -1.0, q_mu, P, 1.0, dq_mu, P, dtype, st));
  // dF/dq_sqrt: T = 2w S_p^T (L^T L), the transpose of 2w (L^T L) S_p
  GPK_TRY(lauum_lower((const double*)w.L, N, ldn, (double*)w.LtL, ldn, st));
  GPK_TRY(svgp_bracket(SB_MIRROR, nullptr, w.LtL, N, ldn, nullptr, nullptr, nullptr, 0.0, 0.0, st));
  {
    const unsigned g = (unsigned)((N * N + 255) / 256);
    for (int64_t p = 0; p < P; ++p) {
      GPK_TRY(gemm_any(1, 0, N, N, N, 2.0 * wv, qs + p * sq, N, w.LtL, ldn, 0.0, w.T, ldn, dtype, GPK_GEMM_A_LOWER,
                       st));
      svgp_dqsqrt_kernel<<<g, 256, 0, st>>>(0, 1, (const double*)w.T, (const double*)(qs + p * sq),
                                            dq_sqrt + (size_t)p * N * N, N, P, nullptr, nullptr, ldn, 0.0);
      GPK_LAUNCH_OK();
    }
  }
  // the kernel parameters: dF/dK over the square K(X, X)
  return square_grad_launch(nodes, n_nodes, dims, ard, (const double*)X, N, ldx, D, (const double*)w.G, ldn, out + 4,
                            (double*)w.Lbar, "vgp_elbo_grad", st);
}
namespace gpk {

// ---------------------------------------------------------------------------------------------
// CGLB (gpflow/models/cglb.py:83-160, 340-420): SGPR's Nystrom factors as the preconditioner of conjugate gradients on
// the exact K^ = K(X, X) + s I, applied through the matrix-free product of kmv.cu; K^ is never formed.
// ---------------------------------------------------------------------------------------------
struct CglbWs {
  SgprWs f; double *V, *R, *Pd, *Ap, *Zd, *t1, *cgs; int32_t* cgi; void* kws; size_t bytes;
};
static CglbWs cglb_layout(void* ws, int64_t N, int64_t M, int64_t P) {
  CglbWs w;
  w.f = sgpr_layout(ws, N, M, P, GPK_F64);
  Arena a(ws);
  a.off = w.f.bytes;
  const size_t np = (size_t)N * P * sizeof(double);
  w.V = (double*)a.take(np);
  w.R = (double*)a.take(np);
  w.Pd = (double*)a.take(np);
  w.Ap = (double*)a.take(np);
  w.Zd = (double*)a.take(np);
  w.t1 = (double*)a.take((size_t)M * P * sizeof(double));
  w.cgs = (double*)a.take(256);  // 0 rz
  w.cgi = (int32_t*)a.take(256); // 0 iterations run, 1 done
  w.kws = a.take(kmv_ws_bytes(N, N, P));
  w.bytes = a.off;
  return w;
}
}  // namespace gpk
extern "C" size_t gpk_cglb_elbo_ws(int64_t N, int64_t M, int64_t P) { return cglb_layout(nullptr, N, M, P).bytes; }
namespace gpk {

constexpr int CG_THREADS = 1024;
// Sum over one CTA in a fixed order (per-thread strided sums, then xor butterflies): the same bits on every run.
__device__ double cg_block_sum(double v, double* red) {
  v = warp_sum(v);
  const int lane = threadIdx.x & 31, wp = threadIdx.x >> 5;
  __syncthreads();  // red is free
  if (lane == 0) red[wp] = v;
  __syncthreads();
  double s = lane < (int)(blockDim.x >> 5) ? red[lane] : 0.0;
  return warp_sum(s);
}

// R = E - KV (elementwise, n = N P); skipped once the loop has converged
__global__ void cg_resid_kernel(int64_t n, const double* __restrict__ E, const double* __restrict__ KV,
                                double* __restrict__ R, const int32_t* __restrict__ done) {
  if (done && *done) return;
  const int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (e < n) R[e] = E[e] - KV[e];
}

// cglb.py:398-401: rz = sum z * r, p = z, i = 0
__global__ void cg_init_kernel(int64_t n, const double* __restrict__ Z, const double* __restrict__ R,
                               double* __restrict__ Pd, double* cgs, int32_t* cgi) {
  __shared__ double red[32];
  double a = 0.0;
  for (int64_t e = threadIdx.x; e < n; e += blockDim.x) {
    a = fma(Z[e], R[e], a);
    Pd[e] = Z[e];
  }
  a = cg_block_sum(a, red);
  if (threadIdx.x == 0) { cgs[0] = a; cgi[0] = 0; cgi[1] = 0; }
}

// cglb.py:382 before each step: stop once 0.5 rz <= tolerance (the host stops at max_cg_iters)
__global__ void cg_gate_kernel(const double* cgs, int32_t* cgi, double tol) {
  if (!cgi[1] && !(0.5 * cgs[0] > tol)) cgi[1] = 1;
}

// cglb.py:385-395: denom = p.Ap, gamma = rz / denom, v += gamma p, and (no restart) r -= gamma Ap
__global__ void cg_step_kernel(int64_t n, const double* __restrict__ Pd, const double* __restrict__ Ap,
                               double* __restrict__ V, double* __restrict__ R, const double* cgs, const int32_t* cgi,
                               int restart) {
  if (cgi[1]) return;
  __shared__ double red[32];
  double a = 0.0;
  for (int64_t e = threadIdx.x; e < n; e += blockDim.x) a = fma(Pd[e], Ap[e], a);
  a = cg_block_sum(a, red);
  const double gamma = cgs[0] / a;
  for (int64_t e = threadIdx.x; e < n; e += blockDim.x) {
    V[e] = V[e] + gamma * Pd[e];
    if (!restart) R[e] = R[e] - gamma * Ap[e];
  }
}

// cglb.py:396-405: new_rz = z.r, p = z (restart) or z + p new_rz / rz, rz = new_rz, i += 1
__global__ void cg_finish_kernel(int64_t n, const double* __restrict__ Z, const double* __restrict__ R,
                                 double* __restrict__ Pd, double* cgs, int32_t* cgi, int restart) {
  if (cgi[1]) return;
  __shared__ double red[32];
  double a = 0.0;
  for (int64_t e = threadIdx.x; e < n; e += blockDim.x) a = fma(Z[e], R[e], a);
  a = cg_block_sum(a, red);
  const double rz = cgs[0];
  for (int64_t e = threadIdx.x; e < n; e += blockDim.x) Pd[e] = restart ? Z[e] : Z[e] + Pd[e] * a / rz;
  __syncthreads();  // every thread has read cgs[0]
  if (threadIdx.x == 0) { cgs[0] = a; cgi[0] += 1; }
}

// cglb.py:147-150 and 83-110: lb = sum v (r + Kv / 2), rz = r^T Q^-1 r, quad = -(lb + rz / 2); the SGPR scalars give
// the logdet term with the tighter log(1 + t / N) trace correction
__global__ void cglb_finalize_kernel(int64_t n, const double* __restrict__ V, const double* __restrict__ R,
                                     const double* __restrict__ KV, const double* __restrict__ Z, const double* scal,
                                     const int32_t* info, const int32_t* cgi, double N, double P, double noise,
                                     double* out) {
  __shared__ double red[32];
  double a = 0.0, b = 0.0;
  for (int64_t e = threadIdx.x; e < n; e += blockDim.x) {
    a = fma(V[e], R[e] + 0.5 * KV[e], a);
    b = fma(Z[e], R[e], b);
  }
  a = cg_block_sum(a, red);
  b = cg_block_sum(b, red);
  if (threadIdx.x != 0) return;
  const double t = scal[0] - scal[1];  // (sum Kdiag - |A'|_F^2) / s
  const double logdet = -P * (scal[2] + 0.5 * N * log(noise) + 0.5 * N * log(1.0 + t / N));
  const double quad = -(a + 0.5 * b);
  const double cst = -0.5 * N * P * LOG2PI;
  out[0] = cst + logdet + quad;
  out[1] = cst; out[2] = logdet; out[3] = quad; out[4] = a; out[5] = b;
  out[6] = cgi ? (double)cgi[0] : 0.0;
  out[7] = (double)(info[0] != 0 ? info[0] : info[1]);
}

// z = Q^-1 r = (r - A'^T B^-1 A' r / s) / s  (NystromPreconditioner, cglb.py:322-340, with A = A' / sqrt s)
static int cglb_precond(const CglbWs& w, int64_t N, int64_t M, int64_t P, double s, const double* R, double* Zd,
                        cudaStream_t st) {
  const CollapsedWs& f = w.f.b;
  GPK_TRY(gemm_any(0, 0, M, P, N, 1.0, w.f.Kuf, f.ldn, R, P, 0.0, w.t1, P, GPK_F64, 0, st));
  GPK_TRY(trsm_any(0, f.Bm, M, f.ldm, w.t1, P, P, GPK_F64, f.dinvB, st));
  GPK_TRY(trsm_any(1, f.Bm, M, f.ldm, w.t1, P, P, GPK_F64, f.dinvB, st));
  GPK_TRY(axpby_impl(N, P, 1.0 / s, R, P, 0.0, Zd, P, GPK_F64, st));
  return gemm_any(1, 0, N, P, M, -1.0 / (s * s), w.f.Kuf, f.ldn, w.t1, P, 1.0, Zd, P, GPK_F64, 0, st);
}

// out: {elbo, const, logdet_term, quad_term, lb, r^T Q^-1 r, cg_iters, info}.  v [P, N] is read, and with run_cg
// replaced by the CG result (P = 1 only: the reference's step does not broadcast over several outputs).
// Leaves, besides out: the SGPR factors in w.f, V = v^T, R = e - K^ V, Zd = Q^-1 R and Ap = K^ V in the workspace.
static int cglb_forward(const gpk_knode* nodes, int n_nodes, const int32_t* dims, const double* ard, const double* X,
                        int64_t N, int64_t ldx, int64_t D, const double* Yc, int64_t P, const double* Z, int64_t M,
                        int64_t ldz, double noise, double jitter, double* v, int run_cg, double cg_tolerance,
                        int max_cg_iters, int restart_cg_iters, double* out, const CglbWs& w, cudaStream_t st) {
  GPK_CHECK_ARG(N > 0 && M > 0 && P > 0 && D > 0 && X && Yc && Z && v && out && w.V, "cglb_elbo: bad arguments");
  GPK_CHECK_ARG(noise > 0.0, "cglb_elbo: noise variance must be positive");
  GPK_CHECK_ARG(!run_cg || P == 1, "cglb_elbo: conjugate gradients run for one output only (P = %lld): the reference's "
                "step size has shape [P] against a [P, N] direction and does not broadcast", (long long)P);
  GPK_CHECK_ARG(!run_cg || (max_cg_iters >= 0 && restart_cg_iters >= 1), "cglb_elbo: max_cg_iters %d, restart_cg_iters %d",
                max_cg_iters, restart_cg_iters);
  const int64_t n = N * P;
  const unsigned eg = (unsigned)((n + 255) / 256);
  GPK_TRY(sgpr_forward(nodes, n_nodes, dims, ard, X, N, ldx, D, Yc, P, Z, M, ldz, noise, jitter, GPK_F64, out, w.f, st));
  GPK_TRY(transpose_impl(v, P, N, N, w.V, P, GPK_F64, st));  // v [P, N] -> V [N, P]
  auto kmv = [&](const double* in, double* o, const int32_t* skip) {
    return kmv_impl(nodes, n_nodes, dims, ard, X, N, ldx, nullptr, N, ldx, D, in, P, P, noise, o, P, w.kws, skip, st);
  };
  if (run_cg) {
    // cglb.py:398-401: r = b - v K^, z = Q^-1 r, p = z
    GPK_TRY(kmv(w.V, w.Ap, nullptr));
    cg_resid_kernel<<<eg, 256, 0, st>>>(n, Yc, w.Ap, w.R, nullptr);
    GPK_LAUNCH_OK();
    GPK_TRY(cglb_precond(w, N, M, P, noise, w.R, w.Zd, st));
    cg_init_kernel<<<1, CG_THREADS, 0, st>>>(n, w.Zd, w.R, w.Pd, w.cgs, w.cgi);
    GPK_LAUNCH_OK();
    // the steps go out in chunks; between chunks one 4-byte read of the done flag.  Once the flag is set the products
    // and every kernel that writes CG state (v, r, p, rz, the counter) return at once; the preconditioner's launches
    // still run to the end of the chunk, but only recompute their scratch (t1, z) from the unchanged r, which the
    // gated kernels never read again.  So the result does not depend on the chunk length.
    constexpr int CHUNK = 8;
    for (int k = 0; k < max_cg_iters; ++k) {
      if (k > 0 && k % CHUNK == 0) {
        int32_t done = 0;
        GPK_CUDA_OK(cudaMemcpyAsync(&done, w.cgi + 1, sizeof(int32_t), cudaMemcpyDeviceToHost, st));
        GPK_CUDA_OK(cudaStreamSynchronize(st));
        if (done) break;
      }
      const int restart = k % restart_cg_iters == restart_cg_iters - 1;
      cg_gate_kernel<<<1, 1, 0, st>>>(w.cgs, w.cgi, cg_tolerance);
      GPK_LAUNCH_OK();
      GPK_TRY(kmv(w.Pd, w.Ap, w.cgi + 1));
      cg_step_kernel<<<1, CG_THREADS, 0, st>>>(n, w.Pd, w.Ap, w.V, w.R, w.cgs, w.cgi, restart);
      GPK_LAUNCH_OK();
      if (restart) {  // cglb.py:389-393: r = b - v K^
        GPK_TRY(kmv(w.V, w.Ap, w.cgi + 1));
        cg_resid_kernel<<<eg, 256, 0, st>>>(n, Yc, w.Ap, w.R, w.cgi + 1);
        GPK_LAUNCH_OK();
      }
      GPK_TRY(cglb_precond(w, N, M, P, noise, w.R, w.Zd, st));
      cg_finish_kernel<<<1, CG_THREADS, 0, st>>>(n, w.Zd, w.R, w.Pd, w.cgs, w.cgi, restart);
      GPK_LAUNCH_OK();
    }
    GPK_TRY(transpose_impl(w.V, N, P, P, v, N, GPK_F64, st));  // v_init.assign(v) (cglb.py:155-156)
  }
  // the bound at the final v (cglb.py:143-150)
  GPK_TRY(kmv(w.V, w.Ap, nullptr));
  cg_resid_kernel<<<eg, 256, 0, st>>>(n, Yc, w.Ap, w.R, nullptr);
  GPK_LAUNCH_OK();
  GPK_TRY(cglb_precond(w, N, M, P, noise, w.R, w.Zd, st));
  cglb_finalize_kernel<<<1, CG_THREADS, 0, st>>>(n, w.V, w.R, w.Ap, w.Zd, w.f.b.scal, w.f.b.info,
                                                 run_cg ? w.cgi : nullptr, (double)N, (double)P, noise, out);
  GPK_LAUNCH_OK();
  return 0;
}

}  // namespace gpk
extern "C" int gpk_cglb_elbo(const gpk_knode* nodes, int n_nodes, const int32_t* dims, const double* ard,
                             const double* X, int64_t N, int64_t ldx, int64_t D, const double* Yc, int64_t P,
                             const double* Z, int64_t M, int64_t ldz, double noise, double jitter, double* v,
                             int run_cg, double cg_tolerance, int max_cg_iters, int restart_cg_iters, double* out,
                             void* ws, void* stream) {
  const cudaStream_t st = (cudaStream_t)stream;
  GPK_CHECK_ARG(ws, "cglb_elbo: null workspace");
  return cglb_forward(nodes, n_nodes, dims, ard, X, N, ldx, D, Yc, P, Z, M, ldz, noise, jitter, v, run_cg,
                      cg_tolerance, max_cg_iters, restart_cg_iters, out, cglb_layout(ws, N, M, P), st);
}
namespace gpk {

// ---- value + gradient of the CGLB bound ------------------------------------------------------------------------
// v is held fixed (the reference's stop_gradient when CG chose it).  With A' = L^-1 Kuf, z = Q^-1 r, Az = A' z,
// t = (sum Kdiag - |A'|_F^2) / s and c_t = -(P/2) / (1 + t/N):
//   dF/dK^     = 1/2 v v^T + 1/2 (z v^T + v z^T)                  (N x N, never formed: grad.cu's low-rank source)
//   dF/dKuf    = L^-T [ (-P/s B^-1 - 2 c_t/s I) A' + Az z^T ]
//   dF/dKuu    = L^-T [ P/2 (I - B^-1) - 1/2 Az Az^T + c_t (B - I) ] L^-1     (A'A'^T = s (B - I))
//   dF/dKdiag  = c_t / s
//   dF/ds      = sum (v^2/2 + z v) - P/2 (N - M + tr B^-1) / s + |z|^2 / 2 - c_t t / s
//   dF/dm      = v + z,   dF/dv (trainable v) = -r + K^ z
struct CglbGradWs {
  CglbWs c; double* Guf; CollapsedGradWs g; double *kdw, *dm; size_t dm_off, bytes;
};
static CglbGradWs cglb_grad_layout(void* ws, int64_t N, int64_t M, int64_t P) {
  CglbGradWs w;
  w.c = cglb_layout(ws, N, M, P);
  Arena a(ws);
  a.off = w.c.bytes;
  w.Guf = (double*)a.take((size_t)M * w.c.f.b.ldn * sizeof(double));
  w.g = collapsed_grad_layout(a, M, P, w.c.f.b.ldm, GPK_F64);
  w.kdw = (double*)a.take((size_t)N * sizeof(double));
  w.dm_off = a.off;
  w.dm = (double*)a.take((size_t)N * P * sizeof(double));
  w.bytes = a.off;
  return w;
}
}  // namespace gpk
extern "C" size_t gpk_cglb_elbo_grad_ws(int64_t N, int64_t M, int64_t P) {
  return cglb_grad_layout(nullptr, N, M, P).bytes;
}
extern "C" size_t gpk_cglb_elbo_grad_dm(int64_t N, int64_t M, int64_t P) {
  return cglb_grad_layout(nullptr, N, M, P).dm_off;
}
namespace gpk {

// scal (SGPR's): 0 trace_k, 1 trace_q; cgs (free after the forward): 1 tr B^-1, 2 |z|^2
__device__ __forceinline__ double cglb_ct(const double* scal, double N, double P) {
  return -0.5 * P / (1.0 + (scal[0] - scal[1]) / N);
}

// Hm <- -P/s B^-1 - 2 c_t/s I (B^-1 read from Hm, full); Guu <- P/2 (I - B^-1) - Az Az^T / 2 + c_t (B - I)
// (B - I read from Guu)
__global__ void cglb_inner_kernel(double* __restrict__ Hm, double* __restrict__ Guu, int64_t ld,
                                  const double* __restrict__ Az, int64_t M, int64_t P, double s, double N,
                                  const double* scal) {
  const int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= M * M) return;
  const int64_t i = e / M, j = e % M;
  const double ct = cglb_ct(scal, N, (double)P);
  const double d = i == j ? 1.0 : 0.0, bi = Hm[i * ld + j];
  double aa = 0.0;
  for (int64_t p = 0; p < P; ++p) aa = fma(Az[i * P + p], Az[j * P + p], aa);
  Hm[i * ld + j] = -(double)P / s * bi - 2.0 * ct / s * d;
  Guu[i * ld + j] = 0.5 * (double)P * (d - bi) - 0.5 * aa + ct * Guu[i * ld + j];
}

__global__ void cglb_fill_kdiag_kernel(double* __restrict__ w, int64_t N, const double* scal, double P, double s) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < N) w[i] = cglb_ct(scal, (double)N, P) / s;
}

// dm = V + Zd; dv^T = Kz - R  (dv [P, N] written transposed)
__global__ void cglb_adj_kernel(int64_t N, int64_t P, const double* __restrict__ V, const double* __restrict__ Zd,
                                const double* __restrict__ R, const double* __restrict__ Kz, double* __restrict__ dm,
                                double* __restrict__ dv) {
  const int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= N * P) return;
  dm[e] = V[e] + Zd[e];
  if (dv) dv[(e % P) * N + e / P] = Kz[e] - R[e];
}

// out[8] (d/ds) already holds sum_i dF/dK^_ii from the N x N pass
__global__ void cglb_noise_grad_kernel(double* out, const double* scal, const double* cgs, double N, double M,
                                       double P, double s) {
  const double t = scal[0] - scal[1], ct = cglb_ct(scal, N, P);
  out[8] += -0.5 * P * (N - M + cgs[1]) / s + 0.5 * cgs[2] - ct * t / s;
}

}  // namespace gpk

// out: [0..7] as gpk_cglb_elbo, [8] d/dnoise_variance, [9 ...] the leaf slots (grad.cu); dZ [M, D]; dv [P, N] or NULL
extern "C" int gpk_cglb_elbo_grad(const gpk_knode* nodes, int n_nodes, const int32_t* dims, const double* ard,
                                  const double* X, int64_t N, int64_t ldx, int64_t D, const double* Yc, int64_t P,
                                  const double* Z, int64_t M, int64_t ldz, double noise, double jitter, double* v,
                                  int run_cg, double cg_tolerance, int max_cg_iters, int restart_cg_iters,
                                  double* out, int n_out, double* dZ, double* dv, void* ws, void* stream) {
  const cudaStream_t st = (cudaStream_t)stream;
  GPK_CHECK_ARG(ws && dZ, "cglb_elbo_grad: null workspace or dZ");
  const int slots = grad_expr_slots(nodes, n_nodes, dims, ard, D, "cglb_elbo_grad");
  if (slots < 0) return slots;
  GPK_CHECK_ARG(n_out >= 9 + slots, "cglb_elbo_grad: n_out = %d, the expression needs %d outputs", n_out, 9 + slots);
  CglbGradWs w = cglb_grad_layout(ws, N, M, P);
  const CglbWs& c = w.c;
  const CollapsedWs& f = c.f.b;
  const double s = noise;
  const int64_t ldm = f.ldm, ldn = f.ldn, n = N * P;
  GPK_CUDA_OK(cudaMemsetAsync(out, 0, (size_t)n_out * sizeof(double), st));
  GPK_CUDA_OK(cudaMemsetAsync(dZ, 0, (size_t)M * D * sizeof(double), st));
  GPK_TRY(cglb_forward(nodes, n_nodes, dims, ard, X, N, ldx, D, Yc, P, Z, M, ldz, noise, jitter, v, run_cg,
                       cg_tolerance, max_cg_iters, restart_cg_iters, out, c, st));
  GPK_CUDA_OK(cudaMemsetAsync(c.cgs + 1, 0, 2 * sizeof(double), st));
  // the N x N pass: sum_ij dF/dK^_ij dK_ij/dtheta into the slots, sum_i dF/dK^_ii into out[8]
  GPK_TRY(gpr_lowrank_grad_launch(nodes, n_nodes, dims, ard, X, N, ldx, D, c.V, c.Zd, (int)P, out + 8, st));
  // Az = A' z into g.x ; |z|^2
  GPK_TRY(gemm_any(0, 0, M, P, N, 1.0, c.f.Kuf, ldn, c.Zd, P, 0.0, w.g.x, P, GPK_F64, 0, st));
  GPK_TRY(reduce_impl(1, c.Zd, n, 1, 1.0, 1, c.cgs + 2, GPK_F64, st));
  // B - I into Guu ; B^-1 into Hm, made full ; tr B^-1
  GPK_TRY(collapsed_binv(f, w.g, M, c.cgs + 1, st));
  GPK_TRY(svgp_bracket(SB_MIRROR, nullptr, w.g.Hm, M, ldm, nullptr, nullptr, nullptr, 0.0, 0.0, st));
  cglb_inner_kernel<<<(unsigned)((M * M + 255) / 256), 256, 0, st>>>(w.g.Hm, w.g.Guu, ldm, w.g.x, M, P, s, (double)N,
                                                                     f.scal);
  GPK_LAUNCH_OK();
  // G_uu = L^-T W L^-1 ; G_uf = (L^-T H) A' + (L^-T Az) z^T
  GPK_TRY(collapsed_linv(f, w.g, M, st));
  GPK_TRY(sandwich(1.0, f.Kuu, w.g.Guu, w.g.Guu, w.g.T1, M, ldm, st));
  GPK_TRY(collapsed_guf(f, w.g, N, M, P, c.f.Kuf, 1.0, c.Zd, w.Guf, st));
  // dm = v + z ; dv = K^ z - r (trainable v: K^ z into Ap, which the forward no longer needs)
  if (dv) GPK_TRY(kmv_impl(nodes, n_nodes, dims, ard, X, N, ldx, nullptr, N, ldx, D, c.Zd, P, P, noise, c.Ap, P, c.kws,
                           nullptr, st));
  cglb_adj_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(N, P, c.V, c.Zd, c.R, c.Ap, w.dm, dv);
  GPK_LAUNCH_OK();
  cglb_fill_kdiag_kernel<<<(unsigned)((N + 255) / 256), 256, 0, st>>>(w.kdw, N, f.scal, (double)P, s);
  GPK_LAUNCH_OK();
  cglb_noise_grad_kernel<<<1, 1, 0, st>>>(out, f.scal, c.cgs, (double)N, (double)M, (double)P, s);
  GPK_LAUNCH_OK();
  return inducing_grad_launch(nodes, n_nodes, dims, ard, X, N, ldx, D, Z, M, ldz, w.Guf, ldn, w.g.Guu, ldm, 0.0,
                              w.kdw, out + 8, dZ, "cglb_elbo_grad", st);
}
