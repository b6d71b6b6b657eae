// fused.cu — one-call objectives: GPR log marginal likelihood, SGPR ELBO, SVGP ELBO.
// Each function enqueues the whole evaluation on the caller's stream from a caller-provided
// workspace (no allocation, no host synchronisation) and leaves the scalars in device memory.
//   gpr_lml   : gpflow/models/gpr.py:91-107 + logdensities.py:139-156
//   sgpr_elbo : gpflow/models/sgpr.py:181-289 (+ the cache of posteriors.py:520-551)
//   svgp_elbo : gpflow/models/svgp.py:166-181 -> posteriors.py:827-841 -> conditionals/util.py:84-169
//               -> kullback_leiblers.py:59-165 -> the likelihood's variational expectations (lik.cu)
//   vgp_elbo_grad : gpflow/models/vgp.py:111-143 (value and gradient; the value alone stays VGP.elbo's operators)
#include <stdlib.h>

#include "internal.cuh"

namespace gpk {

struct Arena {
  char* base;
  size_t off;
  explicit Arena(void* p) : base((char*)p), off(0) {}
  void* take(size_t bytes) {
    void* r = base ? base + off : nullptr;
    off += align_up(bytes, 256);
    return r;
  }
};

static inline int64_t pad_ld(int64_t n) { return (n + 3) / 4 * 4; }

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

size_t gpr_lml_ws(int64_t N, int64_t P, int dtype) { return gpr_layout(nullptr, N, P, dtype).bytes; }

// The LML's forward pass (gpr.py:91-107), shared by gpr_lml and gpr_lml_grad_expr: out[0..3] (out[0 .. n_clear) zeroed
// first), the factor L in w.A with beta^T = L^-1 (Y - m) in its P extra rows, and with need_dinv the block inverses
// of L in w.dinv.
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

int gpr_lml(const gpk_knode* nodes, int n_nodes, const int32_t* dims, const double* ard, const void* X, int64_t N,
            int64_t ldx, int64_t D, const void* Yc, int64_t P, double noise_variance, const void* noise_vec,
            int dtype, double* out, void* ws, cudaStream_t st) {
  GPK_CHECK_ARG(N > 0 && P > 0 && ws && out && Yc, "gpr_lml: bad arguments");
  return gpr_forward(nodes, n_nodes, dims, ard, X, N, ldx, D, Yc, P, noise_variance, noise_vec, dtype, out, 4, false,
                     gpr_layout(ws, N, P, dtype), st);
}

// ---- value + gradient (grad.cu) -----------------------------------------------------------------
int potri_lower(double* L, int64_t n, int64_t ldl, const double* dinv, double* Kinv, int64_t ldk, double* tmp,
                cudaStream_t st);
int grad_expr_slots(const gpk_knode* nodes, int n_nodes, const int32_t* dims, const double* ard, int64_t D,
                    const char* who);
int gpr_grad_launch(const gpk_knode* nodes, int n_nodes, const int32_t* dims, const double* ard, const double* X,
                    int64_t N, int64_t ldx, int64_t D, const double* alpha, int P, const double* Kinv, int64_t ldk,
                    double* gout, cudaStream_t st);

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

size_t gpr_lml_grad_ws(int64_t N, int64_t P, int dtype) { return gpr_grad_layout(nullptr, N, P, dtype).bytes; }
size_t gpr_lml_grad_alpha(int64_t N, int64_t P, int dtype) { return gpr_grad_layout(nullptr, N, P, dtype).alpha_off; }

// out: [0..3] as gpr_lml; [4] d/dnoise_variance, [5 ...] the leaf slots of build_gradprog (grad.cu)
int gpr_lml_grad_expr(const gpk_knode* nodes, int n_nodes, const int32_t* dims, const double* ard, const void* X,
                      int64_t N, int64_t ldx, int64_t D, const void* Yc, int64_t P, double noise_variance, int dtype,
                      double* out, int n_out, void* ws, cudaStream_t st) {
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

// ---------------------------------------------------------------------------------------------
// SGPR
// ---------------------------------------------------------------------------------------------
struct SgprWs {
  void *Kuu, *Kuf, *Bm, *dinvL, *dinvB, *kdiag, *c; int64_t ldm, ldn; int32_t* info; double* scal; size_t bytes;
};
static SgprWs sgpr_layout(void* ws, int64_t N, int64_t M, int64_t P, int dtype) {
  Arena a(ws);
  SgprWs w;
  const size_t ts = dtype_size(dtype);
  w.ldm = pad_ld(M);
  w.ldn = pad_ld(N);
  w.Kuu = a.take((size_t)M * w.ldm * ts);
  w.Kuf = a.take((size_t)M * w.ldn * ts);
  w.Bm = a.take((size_t)M * w.ldm * ts);
  w.dinvL = a.take(potrf_ws_bytes(M, M, dtype));
  w.dinvB = a.take(potrf_ws_bytes(M, M, dtype));
  w.kdiag = a.take((size_t)N * ts);
  w.c = a.take((size_t)M * P * ts);
  w.info = (int32_t*)a.take(256);
  w.scal = (double*)a.take(256);
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

size_t sgpr_elbo_ws(int64_t N, int64_t M, int64_t P, int dtype) { return sgpr_layout(nullptr, N, M, P, dtype).bytes; }

// The bound's forward pass (sgpr.py:181-289), shared by sgpr_elbo and sgpr_elbo_grad.  Leaves L in w.Kuu, A' = L^-1 Kuf
// in w.Kuf, LB in w.Bm, c = LB^-1 A' Yc / s in w.c, the scalars in w.scal and out[0..7].
static int sgpr_forward(const gpk_knode* nodes, int n_nodes, const int32_t* dims, const double* ard, const void* X,
                        int64_t N, int64_t ldx, int64_t D, const void* Yc, int64_t P, const void* Z, int64_t M,
                        int64_t ldz, double noise, double jitter, int dtype, double* out, const SgprWs& w,
                        cudaStream_t st) {
  const double inv_s2 = 1.0 / noise;
  GPK_CUDA_OK(cudaMemsetAsync(w.scal, 0, 8 * sizeof(double), st));
  GPK_CUDA_OK(cudaMemsetAsync(w.info, 0, 2 * sizeof(int32_t), st));
  // kuu = kernel(Z) + jitter I ; L = chol(kuu)   (sgpr.py:200-201)
  GPK_TRY(kbuild_impl(nodes, n_nodes, dims, ard, Z, M, ldz, nullptr, M, ldz, D, w.Kuu, w.ldm, dtype, GPK_LOWER, jitter,
                      nullptr, st));
  GPK_TRY(potrf_any(w.Kuu, M, M, w.ldm, dtype, w.info, w.dinvL, st));
  // kuf = kernel(Z, X) [M,N];  A' = L^-1 kuf  (the 1/sigma of sgpr.py:204 is folded into the scalars below)
  GPK_TRY(kbuild_impl(nodes, n_nodes, dims, ard, Z, M, ldz, X, N, ldx, D, w.Kuf, w.ldn, dtype, GPK_FULL, 0.0, nullptr,
                      st));
  GPK_TRY(trsm_any(0, w.Kuu, M, w.ldm, w.Kuf, N, w.ldn, dtype, w.dinvL, st));
  // AAT = A A^T = A'A'^T / sigma^2 (lower) ; trace_q = tr(AAT) ; B = AAT + I ; LB = chol(B)  (sgpr.py:205-207)
  GPK_TRY(gemm_any(0, 1, M, M, N, inv_s2, w.Kuf, w.ldn, w.Kuf, w.ldn, 0.0, w.Bm, w.ldm, dtype, GPK_GEMM_LOWER_ONLY, st));
  GPK_TRY(reduce_impl(0, w.Bm, M, w.ldm + 1, 1.0, 1, w.scal + 1, dtype, st));
  GPK_TRY(add_diag_impl(w.Bm, M, w.ldm, 1.0, nullptr, dtype, st));
  GPK_TRY(potrf_any(w.Bm, M, M, w.ldm, dtype, w.info + 1, w.dinvB, st));
  GPK_TRY(reduce_impl(2, w.Bm, M, w.ldm + 1, 1.0, 1, w.scal + 2, dtype, st));
  // trace_k = sum kdiag / sigma^2  (sgpr.py:231-233)
  GPK_TRY(kdiag_impl(nodes, n_nodes, dims, ard, X, N, ldx, D, w.kdiag, dtype, st));
  GPK_TRY(reduce_impl(0, w.kdiag, N, 1, inv_s2, 1, w.scal + 0, dtype, st));
  // quad: err = Yc/sigma ; Aerr = A err = A' Yc / sigma^2 ; c = LB^-1 Aerr  (sgpr.py:262-264)
  GPK_TRY(gemm_any(0, 0, M, P, N, inv_s2, w.Kuf, w.ldn, Yc, P, 0.0, w.c, P, dtype, 0, st));
  GPK_TRY(trsm_any(0, w.Bm, M, w.ldm, w.c, P, P, dtype, w.dinvB, st));
  GPK_TRY(reduce_impl(1, Yc, N * P, 1, inv_s2, 1, w.scal + 3, dtype, st));
  GPK_TRY(reduce_impl(1, w.c, M * P, 1, 1.0, 1, w.scal + 4, dtype, st));
  sgpr_finalize_kernel<<<1, 1, 0, st>>>(out, w.scal, w.info, (double)N, (double)P, noise);
  GPK_LAUNCH_OK();
  return 0;
}

int sgpr_elbo(const gpk_knode* nodes, int n_nodes, const int32_t* dims, const double* ard, const void* X, int64_t N,
              int64_t ldx, int64_t D, const void* Yc, int64_t P, const void* Z, int64_t M, int64_t ldz,
              double noise, double jitter, int dtype, double* out, void* cache_L, void* cache_LB, void* cache_c,
              void* ws, cudaStream_t st) {
  GPK_CHECK_ARG(N > 0 && M > 0 && P > 0 && ws && out, "sgpr_elbo: bad arguments");
  GPK_CHECK_ARG(noise > 0.0, "sgpr_elbo: noise variance must be positive");
  SgprWs w = sgpr_layout(ws, N, M, P, dtype);
  const size_t ts = dtype_size(dtype);
  GPK_TRY(sgpr_forward(nodes, n_nodes, dims, ard, X, N, ldx, D, Yc, P, Z, M, ldz, noise, jitter, dtype, out, w, st));
  if (cache_L) {
    GPK_TRY(axpby_impl(M, M, 1.0, w.Kuu, w.ldm, 0.0, cache_L, M, dtype, st));
    GPK_TRY(tril_impl(cache_L, M, M, 0, 1, dtype, st));
  }
  if (cache_LB) {
    GPK_TRY(axpby_impl(M, M, 1.0, w.Bm, w.ldm, 0.0, cache_LB, M, dtype, st));
    GPK_TRY(tril_impl(cache_LB, M, M, 0, 1, dtype, st));
  }
  if (cache_c) GPK_CUDA_OK(cudaMemcpyAsync(cache_c, w.c, (size_t)M * P * ts, cudaMemcpyDeviceToDevice, st));
  return 0;
}

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
int inducing_grad_launch(const gpk_knode* nodes, int n_nodes, const int32_t* dims, const double* ard, const double* X,
                         int64_t N, int64_t ldx, int64_t D, const double* Z, int64_t M, int64_t ldz, const double* Guf,
                         int64_t ldgf, const double* Guu, int64_t ldgu, double kdiag_weight, const double* kdiag_vec,
                         double* gout, double* dZ, const char* who, cudaStream_t st);

struct SgprGradWs {
  SgprWs f; void *Guf, *Guu, *Hm, *T1, *tmp, *v, *Lv, *dm; size_t dm_off, bytes;
};
static SgprGradWs sgpr_grad_layout(void* ws, int64_t N, int64_t M, int64_t P, int dtype) {
  SgprGradWs w;
  w.f = sgpr_layout(ws, N, M, P, dtype);
  Arena a(ws);
  a.off = w.f.bytes;
  const size_t ts = dtype_size(dtype);
  const int64_t h = M / 2 + NB;
  w.Guf = a.take((size_t)M * w.f.ldn * ts);
  w.Guu = a.take((size_t)M * w.f.ldm * ts);
  w.Hm = a.take((size_t)M * w.f.ldm * ts);
  w.T1 = a.take((size_t)M * w.f.ldm * ts);
  w.tmp = a.take((size_t)h * h * ts);
  w.v = a.take((size_t)M * P * ts);
  w.Lv = a.take((size_t)M * P * ts);
  w.dm_off = a.off;
  w.dm = a.take((size_t)N * P * ts);
  w.bytes = a.off;
  return w;
}

size_t sgpr_elbo_grad_ws(int64_t N, int64_t M, int64_t P, int dtype) {
  return sgpr_grad_layout(nullptr, N, M, P, dtype).bytes;
}
size_t sgpr_elbo_grad_dm(int64_t N, int64_t M, int64_t P, int dtype) {
  return sgpr_grad_layout(nullptr, N, M, P, dtype).dm_off;
}

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

// scal: 0..4 as the forward, 5 tr B^-1, 6 |v|^2
__global__ void sgpr_noise_grad_kernel(double* out, const double* scal, double N, double M, double P, double s) {
  out[8] = (-N * P + P * (M - scal[5]) + P * scal[0] - P * scal[1] + scal[3] - scal[4] - scal[6]) / (2.0 * s);
}

// out: [0..7] as sgpr_elbo; [8] d/dnoise_variance, [9 ...] the leaf slots (grad.cu); dZ [M, D] row-major
int sgpr_elbo_grad(const gpk_knode* nodes, int n_nodes, const int32_t* dims, const double* ard, const void* X,
                   int64_t N, int64_t ldx, int64_t D, const void* Yc, int64_t P, const void* Z, int64_t M, int64_t ldz,
                   double noise, double jitter, int dtype, double* out, int n_out, double* dZ, void* ws,
                   cudaStream_t st) {
  GPK_CHECK_ARG(dtype == GPK_F64, "sgpr_elbo_grad: the device backward computes in float64 (dtype %d)", dtype);
  GPK_CHECK_ARG(N > 0 && M > 0 && P > 0 && D > 0 && ws && out && Yc && X && Z, "sgpr_elbo_grad: bad arguments");
  GPK_CHECK_ARG(dZ, "sgpr_elbo_grad: dZ [M, D] is required");
  GPK_CHECK_ARG(noise > 0.0, "sgpr_elbo_grad: noise variance must be positive");
  const int slots = grad_expr_slots(nodes, n_nodes, dims, ard, D, "sgpr_elbo_grad");
  if (slots < 0) return slots;
  GPK_CHECK_ARG(n_out >= 9 + slots, "sgpr_elbo_grad: n_out = %d, the expression needs %d outputs", n_out, 9 + slots);
  SgprGradWs w = sgpr_grad_layout(ws, N, M, P, dtype);
  const SgprWs& f = w.f;
  const double s = noise;
  const int64_t ldm = f.ldm, ldn = f.ldn;
  GPK_CUDA_OK(cudaMemsetAsync(out, 0, (size_t)n_out * sizeof(double), st));
  GPK_CUDA_OK(cudaMemsetAsync(dZ, 0, (size_t)M * D * sizeof(double), st));
  GPK_TRY(sgpr_forward(nodes, n_nodes, dims, ard, X, N, ldx, D, Yc, P, Z, M, ldz, noise, jitter, dtype, out, f, st));
  GPK_CUDA_OK(cudaMemsetAsync(f.scal + 5, 0, 2 * sizeof(double), st));
  // v = LB^-T c ; |v|^2
  GPK_CUDA_OK(cudaMemcpyAsync(w.v, f.c, (size_t)M * P * sizeof(double), cudaMemcpyDeviceToDevice, st));
  GPK_TRY(trsm_any(1, f.Bm, M, ldm, w.v, P, P, dtype, f.dinvB, st));
  GPK_TRY(reduce_impl(1, w.v, M * P, 1, 1.0, 1, f.scal + 6, dtype, st));
  // B - I = LB LB^T - I into Guu (LB's strict upper part zeroed in a copy)
  GPK_TRY(axpby_impl(M, M, 1.0, f.Bm, ldm, 0.0, w.T1, ldm, dtype, st));
  GPK_TRY(tril_impl(w.T1, M, ldm, 0, 1, dtype, st));
  GPK_TRY(gemm_any(0, 1, M, M, M, 1.0, w.T1, ldm, w.T1, ldm, 0.0, w.Guu, ldm, dtype, 0, st));
  GPK_TRY(add_diag_impl(w.Guu, M, ldm, -1.0, nullptr, dtype, st));
  // B^-1 (lower) into Hm, LB^-1 over LB ; tr B^-1
  GPK_TRY(potri_lower((double*)f.Bm, M, ldm, (const double*)f.dinvB, (double*)w.Hm, ldm, (double*)w.tmp, st));
  GPK_TRY(reduce_impl(0, w.Hm, M, ldm + 1, 1.0, 1, f.scal + 5, dtype, st));
  // the two brackets: Guu <- P/2 (I - B^-1) - P/2 (B - I) - v v^T / 2 ; T1 <- H (B^-1 read from Hm first)
  GPK_TRY(axpby_impl(M, M, 1.0, w.Hm, ldm, 0.0, w.T1, ldm, dtype, st));
  {
    const unsigned g = (unsigned)((M * M + 255) / 256);
    sgpr_inner_kernel<<<g, 256, 0, st>>>((const double*)w.T1, (double*)w.Guu, (double*)w.Hm, ldm, (const double*)w.v,
                                         M, P, s);
    GPK_LAUNCH_OK();
  }
  // L^-1 over L (K^-1 into T1, unused), its strict upper part zeroed
  GPK_TRY(potri_lower((double*)f.Kuu, M, ldm, (const double*)f.dinvL, (double*)w.T1, ldm, (double*)w.tmp, st));
  GPK_TRY(tril_impl(f.Kuu, M, ldm, 0, 1, dtype, st));
  const void* Li = f.Kuu;
  // G_uu = L^-T W L^-1  (W in Guu): T1 = W L^-1, Guu = L^-T T1
  GPK_TRY(gemm_any(0, 0, M, M, M, 1.0, w.Guu, ldm, Li, ldm, 0.0, w.T1, ldm, dtype, 0, st));
  GPK_TRY(gemm_any(1, 0, M, M, M, 1.0, Li, ldm, w.T1, ldm, 0.0, w.Guu, ldm, dtype, 0, st));
  // G_uf = (L^-T H) A' + (L^-T v) Yc^T / s
  GPK_TRY(gemm_any(1, 0, M, M, M, 1.0, Li, ldm, w.Hm, ldm, 0.0, w.T1, ldm, dtype, 0, st));
  GPK_TRY(gemm_any(0, 0, M, N, M, 1.0, w.T1, ldm, f.Kuf, ldn, 0.0, w.Guf, ldn, dtype, 0, st));
  GPK_TRY(gemm_any(1, 0, M, P, M, 1.0, Li, ldm, w.v, P, 0.0, w.Lv, P, dtype, 0, st));
  GPK_TRY(gemm_any(0, 1, M, N, P, 1.0 / s, w.Lv, P, Yc, P, 1.0, w.Guf, ldn, dtype, 0, st));
  // dF/dm = (Yc - A'^T v) / s
  GPK_TRY(gemm_any(1, 0, N, P, M, -1.0 / s, f.Kuf, ldn, w.v, P, 0.0, w.dm, P, dtype, 0, st));
  GPK_TRY(axpby_impl(N, P, 1.0 / s, Yc, P, 1.0, w.dm, P, dtype, st));
  sgpr_noise_grad_kernel<<<1, 1, 0, st>>>(out, f.scal, (double)N, (double)M, (double)P, s);
  GPK_LAUNCH_OK();
  return inducing_grad_launch(nodes, n_nodes, dims, ard, (const double*)X, N, ldx, D, (const double*)Z, M, ldz,
                              (const double*)w.Guf, ldn, (const double*)w.Guu, ldm, -(double)P / (2.0 * s), nullptr,
                              out + 8, dZ, "sgpr_elbo_grad", st);
}

// ---------------------------------------------------------------------------------------------
// SVGP
// ---------------------------------------------------------------------------------------------
struct SvgpWs {
  void *Kuu, *A, *dinv, *v0, *fvar, *fmu, *tmpM, *tmpP, *kinv; int64_t ldm, ldb; int32_t* info; double* scal;
  size_t bytes;
};
static SvgpWs svgp_layout(void* ws, int64_t B, int64_t M, int64_t P, int dtype) {
  Arena a(ws);
  SvgpWs w;
  const size_t ts = dtype_size(dtype);
  w.ldm = pad_ld(M);
  w.ldb = pad_ld(B);
  w.Kuu = a.take((size_t)M * w.ldm * ts);
  w.A = a.take((size_t)M * w.ldb * ts);
  w.dinv = a.take(potrf_ws_bytes(M, M, dtype));
  w.v0 = a.take((size_t)B * ts);
  w.fvar = a.take((size_t)P * B * ts);   // [P][B]
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

size_t svgp_elbo_ws(int64_t B, int64_t M, int64_t P, int dtype) { return svgp_layout(nullptr, B, M, P, dtype).bytes; }

// byte offset and leading dimension of A [M, ldb] inside the workspace (for the all-gather between stages 1 and 2)
size_t svgp_elbo_A(int64_t B, int64_t M, int64_t P, int dtype, int64_t* ld) {
  SvgpWs w = svgp_layout(nullptr, B, M, P, dtype);
  if (ld) *ld = w.ldb;
  return (size_t)((char*)w.A - (char*)nullptr);
}

// The ELBO's forward pass (svgp.py:166-181), shared by svgp_elbo and svgp_elbo_grad: the variational expectations
// of `lik` on the raw targets Y [B, P] (MULTICLASS: the labels [B, 1]) with m(X) [B, P] (NULL: zero mean) shifting
// fmean.  After stage 0 or 2: L in w.Kuu, A in w.A (L^-1 Kuf with whiten, K^-1 Kuf without), fmean - m(X) in w.fmu
// [B][Pl], fvar in w.fvar [Pl][B], out[0..3].
static int svgp_forward(const gpk_knode* nodes, int n_nodes, const int32_t* dims, const double* ard, const void* Xb,
                        int64_t B, int64_t ldx, int64_t D, const void* Y, const void* mX, int64_t P, const void* Z,
                        int64_t M, int64_t ldz, const void* q_mu, const void* q_sqrt, int q_diag, int whiten,
                        const gpk_lik* lik, double scale, double jitter, int p_begin, int p_end, int dtype, double* out,
                        const SvgpWs& w, cudaStream_t st, int stage, int64_t c0, int64_t c1) {
  const size_t ts = dtype_size(dtype);
  const int64_t Pl = p_end - p_begin;
  const char* qmu = (const char*)q_mu;
  const char* qs = (const char*)q_sqrt;
  GPK_CUDA_OK(cudaMemsetAsync(w.scal, 0, 8 * sizeof(double), st));
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
  // sum of variational expectations (likelihoods/base.py:361-376) over the columns [p_begin, p_end) of Y and m(X)
  // (MULTICLASS: p_begin = 0, the entries refuse a sub-range)
  GPK_TRY(lik_varexp_impl(lik, w.fmu, w.fvar, (const char*)Y + (size_t)p_begin * ts,
                          mX ? (const char*)mX + (size_t)p_begin * ts : nullptr, B, Pl, lik_ldy(lik, P), P, 1, B, 1.0,
                          1, w.scal + 0, dtype, st));
  // KL[q || p]   (kullback_leiblers.py:59-165)
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
  svgp_finalize_kernel<<<1, 1, 0, st>>>(out, w.scal, w.info, (double)M, (double)Pl, scale, whiten);
  GPK_LAUNCH_OK();
  return 0;
}

int svgp_elbo(const gpk_knode* nodes, int n_nodes, const int32_t* dims, const double* ard, const void* Xb, int64_t B,
              int64_t ldx, int64_t D, const void* Y, const void* mX, int64_t P, const void* Z, int64_t M,
              int64_t ldz, const void* q_mu, const void* q_sqrt, int q_diag, int whiten, const gpk_lik* lik,
              double scale, double jitter, int p_begin, int p_end, int dtype, double* out, void* ws, cudaStream_t st,
              int stage, int64_t c0, int64_t c1) {
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
  return svgp_forward(nodes, n_nodes, dims, ard, Xb, B, ldx, D, Y, mX, P, Z, M, ldz, q_mu, q_sqrt, q_diag, whiten, lik,
                      scale, jitter, p_begin, p_end, dtype, out, svgp_layout(ws, B, M, P, dtype), st, stage, c0, c1);
}

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

size_t svgp_elbo_grad_ws(int64_t B, int64_t M, int64_t P, const gpk_lik* lik, int dtype) {
  return svgp_grad_layout(nullptr, B, M, P, dtype, !svgp_uniform_weights(lik)).bytes;
}
size_t svgp_elbo_grad_dm(int64_t B, int64_t M, int64_t P, int dtype) {
  return svgp_grad_layout(nullptr, B, M, P, dtype, false).dm_off;
}

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

// out: [0..3] as svgp_elbo; [4] d/d(likelihood parameter) (Gaussian: the variance, Student-t: the scale, otherwise 0),
// [5 ...] the leaf slots (grad.cu); dZ [M, D], dq_mu [M, P] and dq_sqrt (the shape of q_sqrt) row-major.
int svgp_elbo_grad(const gpk_knode* nodes, int n_nodes, const int32_t* dims, const double* ard, const void* Xb,
                   int64_t B, int64_t ldx, int64_t D, const void* Y, const void* mX, int64_t P, const void* Z, int64_t M,
                   int64_t ldz, const void* q_mu, const void* q_sqrt, int q_diag, int whiten, const gpk_lik* lik,
                   double scale, double jitter, int dtype, double* out, int n_out, double* dZ, double* dq_mu,
                   double* dq_sqrt, void* ws, cudaStream_t st) {
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
  const int64_t ldm = f.ldm, ldb = f.ldb;
  const double wv = uniform ? -scale / (2.0 * lik->noise) : 0.0, wP = (double)P * wv;
  const char* qs = (const char*)q_sqrt;
  const double* Wt = (const double*)w.Wt;
  GPK_CUDA_OK(cudaMemsetAsync(out, 0, (size_t)n_out * sizeof(double), st));
  GPK_CUDA_OK(cudaMemsetAsync(dZ, 0, (size_t)M * D * sizeof(double), st));
  GPK_TRY(svgp_forward(nodes, n_nodes, dims, ard, Xb, B, ldx, D, Y, mX, P, Z, M, ldz, q_mu, q_sqrt, q_diag, whiten, lik,
                       scale, jitter, 0, (int)P, dtype, out, f, st, 0, 0, B));
  const void* A = f.A;
  // R (also dF/dm(X)), out[4], and on the per-latent route W as Wt [P, B]
  GPK_TRY(lik_grad_impl(lik, (const double*)f.fmu, (const double*)f.fvar, (const double*)Y, lik_ldy(lik, P),
                        (const double*)mX, B, P, scale, (double*)w.R, (double*)w.Wt, out + 4, st));
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
    GPK_TRY(gemm_any(0, 1, M, B, P, 1.0, q_mu, P, w.R, P, 1.0, w.Abar, ldb, dtype, 0, st));
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
    GPK_TRY(gemm_any(0, 1, M, B, P, 1.0, q_mu, P, w.R, P, 0.0, w.Abar, ldb, dtype, 0, st));
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
    GPK_TRY(gemm_any(0, 0, M, P, B, 1.0, A, ldb, w.R, P, 0.0, dq_mu, P, dtype, 0, st));
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
    GPK_TRY(gemm_any(0, 0, M, P, B, 1.0, A, ldb, w.R, P, 0.0, dq_mu, P, dtype, 0, st));
    GPK_TRY(gemm_any(0, 0, M, P, M, -1.0, w.Kinv, ldm, q_mu, P, 1.0, dq_mu, P, dtype, 0, st));
  }
  // the kernel parameters and Z: dF/dKuf, dF/dKuu and the Kdiag weights (P w, or sum_p W[n, p] per element)
  return inducing_grad_launch(nodes, n_nodes, dims, ard, (const double*)Xb, B, ldx, D, (const double*)Z, M, ldz,
                              (const double*)Guf, ldb, (const double*)w.Guu, ldm, uniform ? wP : 0.0,
                              uniform ? nullptr : (const double*)w.Wsum, out + 4, dZ, "svgp_elbo_grad", st);
}

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
int square_grad_launch(const gpk_knode* nodes, int n_nodes, const int32_t* dims, const double* ard, const double* X,
                       int64_t N, int64_t ldx, int64_t D, const double* G, int64_t ldg, double* gout,
                       double* dz_scratch, const char* who, cudaStream_t st);
int lauum_lower(const double* A, int64_t n, int64_t lda, double* C, int64_t ldc, cudaStream_t st);

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

size_t vgp_elbo_grad_ws(int64_t N, int64_t P, int dtype) { return vgp_grad_layout(nullptr, N, P, dtype).bytes; }
size_t vgp_elbo_grad_dm(int64_t N, int64_t P, int dtype) { return vgp_grad_layout(nullptr, N, P, dtype).dm_off; }

// out: [0] ELBO, [1] variational expectations, [2] KL, [3] Cholesky info, [4] d/dnoise_variance, [5 ...] the leaf slots
// (grad.cu); dq_mu [N, P] and dq_sqrt [P, N, N] row-major.
int vgp_elbo_grad(const gpk_knode* nodes, int n_nodes, const int32_t* dims, const double* ard, const void* X,
                  int64_t N, int64_t ldx, int64_t D, const void* Yc, int64_t P, const void* q_mu, const void* q_sqrt,
                  double noise, double jitter, int dtype, double* out, int n_out, double* dq_mu, double* dq_sqrt,
                  void* ws, cudaStream_t st) {
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

}  // namespace gpk
