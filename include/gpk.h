/*
 * gpk.h — C ABI of libgpk.so, the H100 (sm_90a) implementation of GPflow's GP-inference hot
 * path: covariance build -> Cholesky / triangular solves -> GPR LML, SGPR / SVGP ELBO, posterior.
 *
 * The reference (GPflow 2.9.2, /root/reference) has NO FFI boundary: it is pure Python on
 * TensorFlow ops.  Each entry point below therefore replaces a *TensorFlow-op call site* of the
 * reference; the site(s) are cited as `gpflow/...:line`.  The Python package `gpflow_b200`
 * mirrors the reference's Python plugin API (gpflow.kernels.Kernel, covariances.Kuu/Kuf,
 * conditionals, kullback_leiblers, posteriors, models.GPR/SGPR/SVGP) and reaches these symbols
 * through ctypes (gpflow_b200/_lib.py).  INTEGRATION.md shows the stub a GPflow maintainer adds.
 *
 * Conventions
 *  - All matrices are ROW-MAJOR (C order, like NumPy/TF); `ld*` = elements between rows.
 *  - All data pointers are DEVICE pointers (e.g. torch.Tensor.data_ptr()) unless named `host`.
 *    The caller owns all memory; workspaces come from the matching `*_ws` size query.  Two resources
 *    are library-owned, keyed by (device, stream), created on first use and never on the steady-state
 *    path: the side stream + 3 events of the Cholesky look-ahead, and the grow-only TF32 plane scratch
 *    of the fp32 int8 tensor-core GEMM (gpk_gemm has no workspace argument in the reference-shaped ABI).
 *    gpk_warm() creates / reserves them eagerly.
 *  - `dtype`: GPK_F32 or GPK_F64; every array of one call has that dtype (gpflow/base.py:299-311).
 *  - `stream` is a cudaStream_t passed as void*; calls are asynchronous on it.
 *  - Return: 0 = OK; <0 = argument / launch error (text via gpk_last_error()); potrf reports a
 *    non-positive pivot through the device-side `info` word (LAPACK convention, 1-based column).
 */
#ifndef GPK_H_
#define GPK_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define GPK_VERSION 1
#define GPK_API __attribute__((visibility("default")))

enum { GPK_F32 = 0, GPK_F64 = 1 };
enum { GPK_FULL = 0, GPK_LOWER = 1 };

/* Kernel-expression node ops.  Stationary ops follow gpflow/kernels/stationaries.py:209-313,
 * statics gpflow/kernels/statics.py:57-91, linear gpflow/kernels/linears.py:60-68,
 * combinations gpflow/kernels/base.py:305-314. */
enum {
  GPK_K_RBF = 0,      /* sigma^2 exp(-r2/2)                      stationaries.py:209-210 */
  GPK_K_MATERN12 = 1, /* sigma^2 exp(-r)                         stationaries.py:270-271 */
  GPK_K_MATERN32 = 2, /* sigma^2 (1+sqrt3 r) exp(-sqrt3 r)       stationaries.py:290-292 */
  GPK_K_MATERN52 = 3, /* sigma^2 (1+sqrt5 r+5/3 r^2) exp(-sqrt5 r) stationaries.py:311-313 */
  GPK_K_RQ = 4,       /* sigma^2 (1 + r2/(2 alpha))^-alpha       stationaries.py:237-238 */
  GPK_K_EXPONENTIAL = 5, /* sigma^2 exp(-r/2)                    stationaries.py:250-251 */
  GPK_K_LINEAR = 6,   /* (x*sigma^2) . x'                        linears.py:60-64 */
  GPK_K_WHITE = 7,    /* sigma^2 delta_ij iff X2 is NULL, else 0 statics.py:57-63 */
  GPK_K_CONSTANT = 8, /* sigma^2                                 statics.py:78-91 */
  GPK_K_SUM = 9,      /* add_n of children                       base.py:305-308 */
  GPK_K_PRODUCT = 10, /* product of children                     base.py:311-314 */
  GPK_K_POLYNOMIAL = 11 /* ((x*sigma^2) . x' + offset)^degree: offset in `lengthscale`, degree in `alpha`  linears.py:71-112 */
};

#define GPK_MAX_CHILDREN 8

/* One node of a flattened kernel expression tree, children before parents, root LAST.
 * Replaces the Python object graph walked by Kernel.__call__ / ReducingCombination.__call__
 * (gpflow/kernels/base.py:195-214, 281-291): every leaf applies its OWN active_dims to the
 * unsliced X.  `dims` / `ard` index into the side arrays handed to gpk_kbuild. */
typedef struct gpk_knode {
  int32_t op;
  int32_t n_children;
  int32_t child[GPK_MAX_CHILDREN];
  double variance;    /* scalar variance (ignored when LINEAR has ARD variances) */
  double lengthscale; /* scalar lengthscale (ignored when n_ard > 0) */
  double alpha;       /* RationalQuadratic only */
  int32_t n_dims;     /* #active dims; 0 = all D columns (slice(None)) base.py:90-109 */
  int32_t dims_off;   /* offset of this leaf's column indices in `dims` */
  int32_t n_ard;      /* 0 = scalar; else == #active dims: per-dim lengthscales (stationary)
                         or per-dim variances (LINEAR) stationaries.py:60-75, linears.py:38-49 */
  int32_t ard_off;    /* offset in `ard` */
} gpk_knode;

GPK_API int gpk_version(void);
GPK_API const char* gpk_last_error(void);

/* K = kernel(X, X2) [+ diag].  Replaces square_distance + K_r/K_r2 + Sum/Product temporaries
 * (gpflow/utilities/ops.py:105-122, kernels/stationaries.py:77-130, kernels/base.py:281-314) and
 * the diagonal shifts add_noise_cov (utilities/model_utils.py:33-38) / `+ jitter*eye`
 * (covariances/kuus.py:33).
 *   nodes/n_nodes, dims, ard : HOST arrays describing the expression (copied per call)
 *   X [N, D] (ldx), X2 [N2, D] (ldx2) or NULL => symmetric K(X, X) with White active
 *   K [N, N2] (ldk) output
 *   uplo: GPK_FULL, or GPK_LOWER (symmetric only: tiles strictly above the diagonal are skipped)
 *   diag_scalar / diag_vec[N] (device, may be NULL): added to K[i,i] (symmetric only) */
GPK_API int gpk_kbuild(const gpk_knode* nodes, int n_nodes, const int32_t* dims, const double* ard,
               const void* X, int64_t N, int64_t ldx, const void* X2, int64_t N2, int64_t ldx2,
               int64_t D, void* K, int64_t ldk, int dtype, int uplo, double diag_scalar,
               const void* diag_vec, void* stream);

/* out[i] = K_diag(X)[i]  (kernel(X, full_cov=False); stationaries.py:82-83, statics.py:41-42,
 * linears.py:67-68, base.py:296-297). */
GPK_API int gpk_kdiag(const gpk_knode* nodes, int n_nodes, const int32_t* dims, const double* ard,
              const void* X, int64_t N, int64_t ldx, int64_t D, void* out, int dtype, void* stream);

/* In-place lower Cholesky of the leading n x n block of the row-major [rows, n] matrix A; only the
 * lower triangle is read.  The strict upper triangle is scratch: the trailing updates store whole tiles, so its entries
 * inside the 128x128 diagonal blocks are overwritten (ops.cholesky zeroes it afterwards).  Rows n..rows-1 (if any)
 * are overwritten with A[n:, :] L^-T — i.e. appending B^T as extra rows yields (L^-1 B)^T for
 * free.  Replaces tf.linalg.cholesky (gpflow/models/gpr.py:102, posteriors.py:422,533,538,703,
 * models/sgpr.py:201,207, conditionals/util.py:67, kullback_leiblers.py:107) and the
 * triangular_solve of logdensities.py:150.
 *   ws: gpk_potrf_ws(n, rows, dtype) bytes; on return its head holds the inverses of the 128x128
 *       diagonal blocks of L (reused by gpk_trsm via `dinv`); the rest is scratch: the int8 digit planes of the
 *       int8 tensor-core trailing updates (fp64, n >= 256), or -- square fp32 matrices of n >= 512, which are widened,
 *       factored on the fp64 path and rounded back -- the fp64 copy with its own inverse slots and planes.
 *   info (device int32, may be NULL): 0, or 1-based index of the first non-positive pivot. */
GPK_API size_t gpk_potrf_ws(int64_t n, int64_t rows, int dtype);
GPK_API int gpk_potrf(void* A, int64_t n, int64_t rows, int64_t lda, int dtype, int32_t* info, void* ws,
              void* stream);

/* Batched variant: `batch` matrices `stride` elements apart (multi-output Kuu stacks [L, M, M],
 * gpflow/covariances/multioutput/kuus.py:62-122).  n <= 128: the whole batch is ONE launch (one CTA per matrix) and the
 * workspace receives one 128x128 inverse slot per matrix; larger n: the factorisations run back to back on the stream.
 * ws: gpk_potrf_batched_ws(n, batch, dtype) bytes.  info: `batch` device words. */
GPK_API size_t gpk_potrf_batched_ws(int64_t n, int batch, int dtype);
GPK_API int gpk_potrf_batched(void* A, int64_t n, int64_t lda, int64_t stride, int batch, int dtype,
                      int32_t* info, void* ws, void* stream);

/* B <- L^-1 B (trans=0) or L^-T B (trans=1); L [n,n] lower (ldl), B [n, nrhs] (ldb).
 * Replaces tf.linalg.triangular_solve (conditionals/util.py:125,139, models/sgpr.py:204,264,
 * posteriors.py:495-496,534,540,707,710, kullback_leiblers.py:114,152).
 *   dinv: inverses of L's 128x128 diagonal blocks as left by gpk_potrf in its ws, or NULL (then
 *         they are recomputed into ws).  ws: gpk_trsm_ws(n, dtype) bytes. */
GPK_API size_t gpk_trsm_ws(int64_t n, int dtype);
GPK_API int gpk_trsm(int trans, const void* L, int64_t n, int64_t ldl, void* B, int64_t nrhs, int64_t ldb,
             int dtype, const void* dinv, void* ws, void* stream);

/* C[m,n] = alpha * op(A) op(B) + beta * C.  transa=0: A stored [m,k]; 1: stored [k,m].
 * transb=0: B stored [k,n]; 1: stored [n,k].  flags: see below.
 * In place: C may be the same pointer as B when transb = 0, ldb == ldc and m <= 128, or as A when transa = 0,
 * lda == ldc and n <= 128.  One tile then spans the aliased dimension, so each element of the operand is read only by
 * the CTA that overwrites it, before it does.  Any other C == B or C == A (transposed, another leading dimension, a
 * larger m or n, or C == A == B) returns -1.  Partial overlaps are not detected and are not supported.
 * Replaces tf.linalg.matmul (models/sgpr.py:205,263, conditionals/util.py:144,157,
 * posteriors.py:497,535,539,728,734). */
enum {
  GPK_GEMM_LOWER_ONLY = 1,  /* only tiles touching the lower triangle of C (SYRK use) */
  GPK_GEMM_A_LOWER = 2,     /* stored A is lower triangular (band_part(-1,0), util.py:151):
                               entries above its diagonal are treated as zero and never read */
  GPK_GEMM_COLSUMSQ = 4     /* do not store C; instead colsum[j] += sum_i (alpha op(A)op(B))_ij^2
                               into `C` interpreted as a [n] vector (util.py:164 fused) */
};
GPK_API int gpk_gemm(int transa, int transb, int64_t m, int64_t n, int64_t k, double alpha, const void* A,
             int64_t lda, const void* B, int64_t ldb, double beta, void* C, int64_t ldc, int dtype,
             int flags, void* stream);

/* Reductions (device outputs, fp64 accumulators written as `dtype`):
 *   colsumsq: out[j] (+)= scale * sum_i A[i,j]^2      conditionals/util.py:133,164
 *   reduce  : out[0] (+)= scale * sum f(x)            logdensities.py:152-154, sgpr.py:233-243,
 *                                                     kullback_leiblers.py:124,130,134,159
 *             f: 0 sum, 1 sum of squares, 2 sum log, 3 sum log of squares
 *             x: strided vector (n elements, `inc` apart) — inc=ld+1 walks a diagonal.
 *   tril_sumsq: out[0] (+)= scale * sum_{b} sum_{i>=j} A[b,i,j]^2   kullback_leiblers.py:120,134 */
GPK_API int gpk_colsumsq(const void* A, int64_t m, int64_t n, int64_t lda, double scale, int accumulate,
                 void* out, int dtype, void* stream);
GPK_API int gpk_reduce(int f, const void* x, int64_t n, int64_t inc, double scale, int accumulate,
               double* out, int dtype, void* stream);
GPK_API int gpk_tril_sumsq(const void* A, int64_t n, int64_t lda, int64_t stride, int batch, double scale,
                   int accumulate, double* out, int dtype, void* stream);

/* Elementwise helpers used by the Python mirror where the reference has small TF ops:
 *   axpby:    Y[m,n] = a*X + b*Y                      (Y - m(X): gpr.py:103-105; + mean)
 *   scale_cols: A[i,j] *= s[j]  or  /= s[j]           (kuf / sigma: sgpr.py:204)
 *   scale_rows: A[i,j] *= s[i]  or  /= s[i]           (err / sigma[:,None]: sgpr.py:262)
 *   add_diag: A[i,i] += scalar + vec[i]               (add_noise_cov model_utils.py:33-38)
 *   fill / tril (zero strict upper, batched)          (band_part util.py:151) */
GPK_API int gpk_axpby(int64_t m, int64_t n, double a, const void* X, int64_t ldx, double b, void* Y,
              int64_t ldy, int dtype, void* stream);
GPK_API int gpk_scale_cols(void* A, int64_t m, int64_t n, int64_t lda, const void* s, int invert,
                   int dtype, void* stream);
GPK_API int gpk_scale_rows(void* A, int64_t m, int64_t n, int64_t lda, const void* s, int invert,
                   int dtype, void* stream);
GPK_API int gpk_add_diag(void* A, int64_t n, int64_t lda, double scalar, const void* vec, int dtype,
                 void* stream);
GPK_API int gpk_fill(void* A, int64_t m, int64_t n, int64_t lda, double value, int dtype, void* stream);
GPK_API int gpk_tril(void* A, int64_t n, int64_t lda, int64_t stride, int batch, int dtype, void* stream);
GPK_API int gpk_transpose(const void* A, int64_t m, int64_t n, int64_t lda, void* B, int64_t ldb, int dtype,
                  void* stream);

/* ---- Scalar likelihoods (gpflow/likelihoods/scalar_continuous.py, scalar_discrete.py, base.py:279-456) ----------------
 * One descriptor per likelihood.  Quadrature is the reference's NDiagGHQuadrature with n_gh = 20 points
 * (quadrature/gauss_hermite.py): E[g(f)] ~ sum_k w_k g(mu + sqrt(v) z_k), z = sqrt(2) hermgauss nodes, w = weights / sqrt(pi);
 * log-space: logsumexp_k(log w_k + g).  Every element (n, p) is one independent scalar likelihood.
 *   GAUSSIAN      log N(y | f, noise); closed forms throughout (scalar_continuous.py:127-148).
 *   BERNOULLI     probit link with the reference's jitter: p = 0.5 (1 + erf(f / sqrt 2)) (1 - 2e-3) + 1e-3,
 *                 log p(y|f) = log(y == 1 ? p : 1 - p); variational expectations by quadrature, predictions closed
 *                 (p = inv_probit(mu / sqrt(1 + v)); mean p, variance p - p^2).
 *   POISSON       exp link, rate = binsize e^f; variational expectations closed (y mu - binsize e^(mu + v/2) - lgamma(y+1)
 *                 + y log binsize); predictions by quadrature.
 *   STUDENT_T     location f, the given scale and df (logdensities.py:93-102); quadrature throughout; predicted mean and
 *                 variance as quadratures of the conditional mean f and of scale^2 df / (df - 2) + f^2 (base.py:379-400).
 *   MULTICLASS    MultiClass with the RobustMax inverse link (gpflow/likelihoods/multiclass.py:55-243): the P = num_classes
 *                 latents of a row are one likelihood, and Y is [rows, 1], its labels truncated to integers.  With x_k =
 *                 hermgauss(20) nodes, w_k = weights / sqrt(pi), label y, s_y = sqrt(max(2 v_y, 1e-10)), s_c =
 *                 sqrt(max(v_c, 1e-10)) and the squashed CDF cdf_ck = Phi((mu_y + x_k s_y - mu_c) / s_c)(1 - 2e-6) + 1e-6:
 *                   p = sum_k w_k prod_{c != y} cdf_ck,   eps_k1 = epsilon / (num_classes - 1),
 *                   VE = p log(1 - epsilon) + (1 - p) log eps_k1,   density(y) = p (1 - epsilon) + (1 - p) eps_k1;
 *                 a label outside [0, num_classes) has mu_y = v_y = 0 and every class in the product, as the reference's
 *                 all-zero one-hot gives.  Predicted mean [rows, num_classes] = density(c) for every class c, variance
 *                 mean - mean^2; log density log density(y), one value per row.  Requires n_gh = 20, 0 < epsilon < 1,
 *                 2 <= num_classes <= GPK_LIK_MAX_CLASSES and P == num_classes. */
enum { GPK_LIK_GAUSSIAN = 0, GPK_LIK_BERNOULLI = 1, GPK_LIK_POISSON = 2, GPK_LIK_STUDENT_T = 3, GPK_LIK_MULTICLASS = 4 };
#define GPK_LIK_MAX_CLASSES 128
typedef struct gpk_lik {
  int32_t type;         /* GPK_LIK_* */
  int32_t n_gh;         /* quadrature points: 20 */
  double scale;         /* STUDENT_T scale (> 0) */
  double df;            /* STUDENT_T degrees of freedom (> 0) */
  double binsize;       /* POISSON bin size (> 0) */
  double noise;         /* GAUSSIAN variance: > 0; 0 is accepted by the two prediction operators, which add it to Fvar
                           (a heteroskedastic variance passed folded into Fvar) */
  double epsilon;       /* MULTICLASS RobustMax epsilon (0 < epsilon < 1) */
  int32_t num_classes;  /* MULTICLASS classes (2 .. GPK_LIK_MAX_CLASSES) */
} gpk_lik;

/* out[0] (+)= scale * sum_{n,p} E_q[log p(Y[n,p] | f)], f ~ N(Fmu, Fvar).  Fmu, Fvar, Y: [B, P] contiguous
 * (MULTICLASS: Y [B, 1], one expectation per row). */
GPK_API int gpk_lik_varexp_sum(const gpk_lik* lik, const void* Fmu, const void* Fvar, const void* Y, int64_t B, int64_t P,
                               double scale, int accumulate, double* out, int dtype, void* stream);
/* mean, var [N, P] = the mean and variance of y under the predictive distribution; inputs [N, P] contiguous
 * (MULTICLASS: the class probabilities, [N, num_classes]). */
GPK_API int gpk_lik_predict_mean_and_var(const gpk_lik* lik, const void* Fmu, const void* Fvar, int64_t N, int64_t P,
                                         void* mean, void* var, int dtype, void* stream);
/* out[n] = sum_p log E_q[p(Y[n,p] | f)], out [N] of the input dtype (MULTICLASS: Y [N, 1], out[n] = log density(y_n)). */
GPK_API int gpk_lik_predict_log_density(const gpk_lik* lik, const void* Fmu, const void* Fvar, const void* Y, int64_t N,
                                        int64_t P, void* out, int dtype, void* stream);

/* ---- Kernels that are not functions of a Gram term (materialised leaves; the Python layer composes them with
 * Sum / Product / ChangePoints through gpk_axpby / gpk_hadamard / gpk_scale_rows / gpk_scale_cols) ------------------ */
enum {
  GPK_KAUX_COSINE = 0,   /* sigma^2 cos(2 pi sum_d (x_d - x'_d) scale_d), scale = 1 / lengthscale   stationaries.py:316-332 */
  GPK_KAUX_PERIODIC = 1, /* base.K_r(sum_d |sin(pi (x_d - x'_d) / period_d)| scale_d) for bases with K_r (Matern12/32/52,
                            Exponential), base.K_r2(sum_d sin^2(...) scale_d^2) otherwise (RBF, RQ)    periodic.py:28-111 */
  GPK_KAUX_ARCCOS = 2,   /* sigma^2 / pi J_order(theta) |x|^order |x'|^order, |x|^2 = sum_d scale_d x_d^2 + bias
                            (scale = weight variances)                                               misc.py:27-200 */
  GPK_KAUX_COREGION = 3  /* table[int(x), int(x')], table = W W^T + diag(kappa) [table_dim^2 doubles]  misc.py:203-296 */
};
#define GPK_KAUX_MAXD 32
typedef struct gpk_kaux_desc {
  int32_t op;
  int32_t base;      /* PERIODIC: GPK_K_* op code of the base kernel */
  int32_t order;     /* ARCCOS: 0, 1 or 2 */
  int32_t n_dims;    /* active columns (explicit, 1..GPK_KAUX_MAXD) */
  int32_t table_dim; /* COREGION: output_dim */
  int32_t pad_;
  double variance, alpha, bias;
  const void* table; /* COREGION: DEVICE pointer to the [table_dim, table_dim] float64 matrix B */
  int32_t dims[GPK_KAUX_MAXD];
  double scale[GPK_KAUX_MAXD];
  double period[GPK_KAUX_MAXD];
} gpk_kaux_desc;

/* K [N, N2] = kernel(X, X2) (X2 NULL: K(X, X)) and its diagonal for the kernels above. */
GPK_API int gpk_kaux(const gpk_kaux_desc* desc, const void* X, int64_t N, int64_t ldx, const void* X2, int64_t N2,
             int64_t ldx2, void* K, int64_t ldk, int dtype, void* stream);
GPK_API int gpk_kaux_diag(const gpk_kaux_desc* desc, const void* X, int64_t N, int64_t ldx, void* out, int dtype,
                  void* stream);
/* ChangePoints sigmoid weights (gpflow/kernels/changepoints.py:118-137,189-193): out[n] =
 * (has_lo ? sig(steep_lo (x_n - loc_lo)) : 1) * (has_hi ? 1 - sig(steep_hi (x_n - loc_hi)) : 1), x_n = X[n, dim]. */
GPK_API int gpk_changepoint_weights(const void* X, int64_t N, int64_t ldx, int dim, int has_lo, double loc_lo,
                            double steep_lo, int has_hi, double loc_hi, double steep_hi, void* out,
                            int dtype, void* stream);
/* A[m, n] = max(A, lower), then squared (`square` = 1) or square-rooted (2): evaluation of a heteroskedastic
 * Gaussian(variance|scale=Function) (gpflow/likelihoods/scalar_continuous.py:92-102: tf.maximum(f(X), lower_bound) [** 2])
 * and tf.sqrt(cov) of sample_mvn (conditionals/util.py:199). */
GPK_API int gpk_clamp_min(void* A, int64_t m, int64_t n, int64_t lda, double lower, int square, int dtype,
                  void* stream);
/* Y[m, n] *= X elementwise (Product of materialised kernels, base.py:311-314). */
GPK_API int gpk_hadamard(int64_t m, int64_t n, const void* X, int64_t ldx, void* Y, int64_t ldy, int dtype,
                 void* stream);

/* ---- Fused objectives: one call per evaluation ------------------------------------------- */

/* GPR.log_marginal_likelihood (gpflow/models/gpr.py:91-107): K-build(lower)+noise, Cholesky with
 * (Y-m)^T appended as extra rows, log-density reduction.  Yc [N,P] = Y - mean_function(X)
 * (contiguous).  out: device double[4] = {lml, sum alpha^2, sum log diag L, info}.
 * ws: gpk_gpr_lml_ws(N, P, dtype) bytes. */
GPK_API size_t gpk_gpr_lml_ws(int64_t N, int64_t P, int dtype);
GPK_API int gpk_gpr_lml(const gpk_knode* nodes, int n_nodes, const int32_t* dims, const double* ard,
                const void* X, int64_t N, int64_t ldx, int64_t D, const void* Yc, int64_t P,
                double noise_variance, const void* noise_vec, int dtype, double* out, void* ws,
                void* stream);

/* GPR log marginal likelihood AND its gradient w.r.t. every kernel parameter and the likelihood variance: the backward
 * pass that TensorFlow autodiff supplies to the reference's optimiser (gpflow/optimizers/scipy.py:78-228 ->
 * models/training_mixins.py:43-78 -> models/gpr.py:91-107), for ANY expression gpk_kbuild fuses (Sum / Product trees of
 * RBF, Matern12/32/52, Exponential, RationalQuadratic, Linear, Polynomial, White and Constant leaves), float64.
 * Written out as dLML/dK = 1/2 (alpha alpha^T - P K^-1), K^-1 = L^-T L^-1 from the factor of the forward pass, and one
 * K-build-shaped reduction sum_ij (dLML/dK)_ij d leaf_ij / d theta per gradient slot, which re-evaluates every leaf per
 * element of the lower triangle and takes d root / d leaf from the postfix program (Sum passes the adjoint through,
 * Product multiplies it by the siblings' product).  A single RBF / Matern / Exponential leaf runs a dedicated, faster
 * reduction with the same slots.
 *   Slots: leaves in node-array order, each with its gradients w.r.t. the constrained values:
 *     RBF, Matern12/32/52, Exponential: variance, lengthscale (1 or n_ard);  RationalQuadratic: variance,
 *     lengthscale(s), alpha;  Linear: variance (1 or n_ard);  Polynomial: variance (1 or n_ard), offset (the degree is
 *     no parameter);  White, Constant: variance.
 *   Limits (status -1 and gpk_last_error otherwise): at most 32 distinct active columns over the gram groups of the
 *     expression, at most 32 per-dimension (ARD) slots, dtype GPK_F64.
 *   gpk_gpr_lml_grad_slots: the number of slots of an expression (host only, no device needed; <0 and gpk_last_error
 *     for an expression the device backward does not cover).
 *   gpk_gpr_lml_grad_alpha: byte offset of alpha = K^-1 (Y - m) [N, P] (row-major, ld P) inside the workspace,
 *     valid after the call (d LML / d m = alpha: mean-function gradients).
 *   out: device double[n_out]: [0..3] as gpk_gpr_lml, [4] d/dnoise_variance, [5 ...] the slots; n_out >= 5 + slots.
 *   ws:  gpk_gpr_lml_grad_ws(N, P, dtype) bytes. */
GPK_API size_t gpk_gpr_lml_grad_ws(int64_t N, int64_t P, int dtype);
GPK_API int gpk_gpr_lml_grad_slots(const gpk_knode* nodes, int n_nodes, const int32_t* dims, const double* ard,
                                   int64_t D);
GPK_API size_t gpk_gpr_lml_grad_alpha(int64_t N, int64_t P, int dtype);
GPK_API int gpk_gpr_lml_grad_expr(const gpk_knode* nodes, int n_nodes, const int32_t* dims, const double* ard,
                                  const void* X, int64_t N, int64_t ldx, int64_t D, const void* Yc, int64_t P,
                                  double noise_variance, int dtype, double* out, int n_out, void* ws, void* stream);

/* SGPR.elbo (gpflow/models/sgpr.py:181-289).  Yc = Y - m(X) [N,P] contiguous, Z [M,D].
 * out: device double[8] = {elbo, const, logdet, quad, trace_k, trace_q, half_logdet_b, info}.
 * If `cache_L`, `cache_LB`, `cache_c` are non-NULL they receive L [M,M], LB [M,M], c [M,P]
 * (posteriors.py:520-551) for prediction. */
GPK_API size_t gpk_sgpr_elbo_ws(int64_t N, int64_t M, int64_t P, int dtype);
GPK_API int gpk_sgpr_elbo(const gpk_knode* nodes, int n_nodes, const int32_t* dims, const double* ard,
                  const void* X, int64_t N, int64_t ldx, int64_t D, const void* Yc, int64_t P,
                  const void* Z, int64_t M, int64_t ldz, double noise_variance, double jitter,
                  int dtype, double* out, void* cache_L, void* cache_LB, void* cache_c, void* ws,
                  void* stream);

/* SGPR.elbo AND its gradient (gpflow/models/sgpr.py:181-289): the backward pass that TensorFlow autodiff supplies to
 * the reference's optimiser, for every expression gpk_gpr_lml_grad_expr covers, the inducing points included; float64.
 * The same forward as gpk_sgpr_elbo, then with K = Kuu + jitter I = L L^T, A' = L^-1 Kuf, B = I + A'A'^T / s = LB LB^T,
 * c = LB^-1 A' Yc / s, v = LB^-T c (s the noise variance):
 *   dF/dKuu = L^-T [P/2 (I - B^-1) - P/2 (B - I) - v v^T / 2] L^-1,   dF/dKuf = L^-T [H A' + v Yc^T / s],
 *   H = (P/s)(I - B^-1) - v v^T / s,   dF/dKdiag = -P / (2s),   dF/dm = (Yc - A'^T v) / s,
 * and three passes of the expression reduction of gpk_gpr_lml_grad_expr (over Kuf, the Kuu square and the N diagonal
 * elements of K(X, X)) that also accumulate dZ.
 *   out:  device double[n_out]: [0..7] as gpk_sgpr_elbo, [8] d/dnoise_variance, [9 ...] the leaf slots in the layout
 *         gpk_gpr_lml_grad_slots counts; n_out >= 9 + slots.
 *   dZ:   device double[M, D] row-major: dF/dZ, zeros in the columns no leaf reads.
 *   Limits (status -1 and gpk_last_error otherwise): those of gpk_gpr_lml_grad_expr, dtype GPK_F64, dZ non-NULL.
 *   gpk_sgpr_elbo_grad_dm: byte offset of dF/dm [N, P] (row-major, ld P) inside the workspace, valid after the call
 *         (mean-function gradients).
 *   ws:   gpk_sgpr_elbo_grad_ws(N, M, P, dtype) bytes. */
GPK_API size_t gpk_sgpr_elbo_grad_ws(int64_t N, int64_t M, int64_t P, int dtype);
GPK_API size_t gpk_sgpr_elbo_grad_dm(int64_t N, int64_t M, int64_t P, int dtype);
GPK_API int gpk_sgpr_elbo_grad(const gpk_knode* nodes, int n_nodes, const int32_t* dims, const double* ard,
                               const void* X, int64_t N, int64_t ldx, int64_t D, const void* Yc, int64_t P,
                               const void* Z, int64_t M, int64_t ldz, double noise_variance, double jitter,
                               int dtype, double* out, int n_out, double* dZ, void* ws, void* stream);

/* SVGP.elbo (gpflow/models/svgp.py:166-181) for a single-output kernel shared by P latent GPs
 * (posteriors.py:827-841 -> conditionals/util.py:84-169 -> kullback_leiblers.py:59-165 -> the variational
 * expectations of `lik`, as gpk_lik_varexp_sum).  Xb [B,D], Z [M,D], q_mu [M,P], q_sqrt [P,M,M] (q_diag=0) or [M,P]
 * (q_diag=1).  The targets come raw, Y [B, P] contiguous (MULTICLASS: the labels [B, 1]), with mX = m(Xb) [B, P]
 * contiguous apart (NULL: zero mean): m(X) shifts fmean.
 * Latent GPs p in [p_begin, p_end) are evaluated (latent sharding); KL is included for those p.  MULTICLASS couples
 * the latents of a row and takes only [0, P).
 * out: device double[4] = {elbo_partial, sum var_exp (unscaled), kl, info}.
 * Limits (status -1 and gpk_last_error otherwise): a valid descriptor, as gpk_svgp_elbo_grad. */
GPK_API size_t gpk_svgp_elbo_ws(int64_t B, int64_t M, int64_t P, int dtype);
GPK_API int gpk_svgp_elbo(const gpk_knode* nodes, int n_nodes, const int32_t* dims, const double* ard,
                  const void* Xb, int64_t B, int64_t ldx, int64_t D, const void* Y, const void* mX, int64_t P,
                  const void* Z, int64_t M, int64_t ldz, const void* q_mu, const void* q_sqrt,
                  int q_diag, int whiten, const gpk_lik* lik, double num_data_scale,
                  double jitter, int p_begin, int p_end, int dtype, double* out, void* ws,
                  void* stream);

/* The same evaluation in two stages, for latent-GP sharding over GPUs with a COLUMN-SHARDED triangular solve
 * (SURVEY.md 8(e); derived from conditionals/util.py:125-164: every column of A = Lm^-1 Kuf depends on its own x_n only):
 *   stage 1: Kuu, chol(Kuu), Kuf[:, col_begin:col_end] and A[:, col_begin:col_end] = Lm^-1 Kuf[:, ...], left in place in
 *            the workspace matrix A [M, ld] (gpk_svgp_elbo_A returns its byte offset in `ws` and `ld`); the caller
 *            all-gathers the column blocks of A between the ranks (NCCL);
 *   stage 2: everything after the solve (fmean, fvar, variational expectations, KL) for the latents [p_begin, p_end)
 *            with A complete in the workspace.  stage 0 = gpk_svgp_elbo.  whiten = 1 only. */
GPK_API size_t gpk_svgp_elbo_A(int64_t B, int64_t M, int64_t P, int dtype, int64_t* ld);
GPK_API int gpk_svgp_elbo_staged(const gpk_knode* nodes, int n_nodes, const int32_t* dims, const double* ard,
                         const void* Xb, int64_t B, int64_t ldx, int64_t D, const void* Y, const void* mX, int64_t P,
                         const void* Z, int64_t M, int64_t ldz, const void* q_mu, const void* q_sqrt,
                         int q_diag, int whiten, const gpk_lik* lik, double num_data_scale, double jitter,
                         int p_begin, int p_end, int stage, int64_t col_begin, int64_t col_end, int dtype,
                         double* out, void* ws, void* stream);

/* SVGP.elbo AND its gradient (gpflow/models/svgp.py:166-181) for any likelihood gpk_lik describes: the backward pass
 * that TensorFlow autodiff supplies to the reference's optimiser, for every expression gpk_gpr_lml_grad_expr covers, both
 * whiten and both q_diag settings, the inducing points and the variational parameters included; float64, the whole
 * minibatch and every latent (no staging or sharding).  The forward, and its Y and mX, are gpk_svgp_elbo's.
 * With c = num_data_scale, K = Kuu + jitter I = L L^T, S_p = tril(q_sqrt[p]), m = q_mu,
 * Sig = sum_p S_p S_p^T, A = L^-1 Kuf (whiten) or K^-1 Kuf, Phi(T) = tril(T) with its diagonal halved,
 * sym(T) = (T + T^T) / 2, and the per-element adjoints of the variational expectations
 *   R[n,p] = c dVE/dfmean[n,p],   W[n,p] = c dVE/dfvar[n,p]
 * (GAUSSIAN: c (Y - mX - fmean) / s and -c / (2s); POISSON closed: c (y - b e^(mu + v/2)) and -c b e^(mu + v/2) / 2;
 * quadrature: c sum_k w_k g'(f_k) and c sum_k w_k g'(f_k) z_k / (2 sqrt v), the exact derivatives of the 20-point sum;
 * MULTICLASS, with kappa = log(1 - epsilon) - log eps_k1, phi the standard normal density and E_ck = prod_{c' != y, c}
 * cdf_c'k: g_ck = w_k E_ck (1 - 2e-6) phi(d_ck) / s_c, d_ck = (mu_y + x_k s_y - mu_c) / s_c, and for c != y
 * R = -c kappa sum_k g_ck, W = -c kappa sum_k g_ck d_ck / (2 s_c) (0 where v_c <= 1e-10), for the label's own latent
 * R = c kappa sum_k sum_{c != y} g_ck, W = c kappa sum_k x_k sum_{c != y} g_ck / s_y (0 where 2 v_y <= 1e-10)):
 *   whiten:    Abar = m R^T + 2 sum_p (S_p S_p^T - I) A diag(W_p), dF/dKuf = L^-T Abar,
 *              dF/dKuu = -sym(L^-T Phi(Abar A^T) L^-1), dF/dq_mu = A R - m,
 *              dF/dS_p = tril(2 (A diag(W_p) A^T) S_p - S_p) + diag(1 / diag S_p);
 *   otherwise: Abar = m R^T + 2 sum_p S_p S_p^T A diag(W_p),   dF/dKuf = K^-1 Abar - 2 A diag(sum_p W_p),
 *              dF/dKuu = sym(-K^-1 Abar A^T) + A diag(sum_p W_p) A^T + K^-1 (m m^T + Sig) K^-1 / 2 - P K^-1 / 2,
 *              dF/dq_mu = A R - K^-1 m, dF/dS_p = tril(2 (A diag(W_p) A^T) S_p - K^-1 S_p) + diag(1 / diag S_p);
 *   both:      dF/dKdiag[n] = sum_p W[n,p],   dF/dm(X) = R;  q_diag restricts the q_sqrt forms to the diagonal.
 * For GAUSSIAN the weight is one constant w = -c / (2s), and the products over latents are shared: Abar = m R^T +
 * 2w (Sig - [whiten] P I) A, dF/dS_p = tril(2w (A A^T) S_p - ...), dF/dKuf gets -2wP A, dF/dKuu gets wP A A^T and
 * dF/dKdiag = P w.  The kernel parameters and Z then go through the three passes gpk_sgpr_elbo_grad runs (Kuf, Kuu,
 * Kdiag).
 *   out:     device double[n_out]: [0..3] as gpk_svgp_elbo, [4] the gradient of the likelihood's parameter (GAUSSIAN:
 *            noise variance; STUDENT_T: scale; MULTICLASS: epsilon, c sum_n [-p_n / (1 - epsilon) + (1 - p_n) /
 *            epsilon]; else 0), [5 ...] the leaf slots in the layout gpk_gpr_lml_grad_slots counts; n_out >= 5 + slots.
 *   Y:       MULTICLASS: the labels [B, 1], with P == num_classes.
 *   dZ:      device double[M, D] row-major; dq_mu: device double[M, P]; dq_sqrt: the shape of q_sqrt ([P, M, M], its
 *            strict upper parts 0, or [M, P] with q_diag).
 *   Limits (status -1 and gpk_last_error otherwise): those of gpk_gpr_lml_grad_expr, dtype GPK_F64, dZ, dq_mu and
 *            dq_sqrt non-NULL, a valid descriptor (n_gh = 20, positive scale / df / binsize / noise; MULTICLASS as
 *            above).
 *   gpk_svgp_elbo_grad_dm: byte offset of dF/dm(X) [B, P] (row-major, ld P) inside the workspace, valid after the call.
 *   ws:      gpk_svgp_elbo_grad_ws(B, M, P, lik, dtype) bytes: GAUSSIAN needs less, without the per-latent scratch of the
 *            other likelihoods. */
GPK_API size_t gpk_svgp_elbo_grad_ws(int64_t B, int64_t M, int64_t P, const gpk_lik* lik, int dtype);
GPK_API size_t gpk_svgp_elbo_grad_dm(int64_t B, int64_t M, int64_t P, int dtype);
GPK_API int gpk_svgp_elbo_grad(const gpk_knode* nodes, int n_nodes, const int32_t* dims, const double* ard,
                               const void* Xb, int64_t B, int64_t ldx, int64_t D, const void* Y, const void* mX,
                               int64_t P, const void* Z, int64_t M, int64_t ldz, const void* q_mu, const void* q_sqrt,
                               int q_diag, int whiten, const gpk_lik* lik, double num_data_scale, double jitter,
                               int dtype, double* out, int n_out, double* dZ, double* dq_mu, double* dq_sqrt,
                               void* ws, void* stream);

/* VGP.elbo AND its gradient (gpflow/models/vgp.py:111-143, Gaussian likelihood, whitened q(v) over f = L v + m(X)): the
 * backward pass that TensorFlow autodiff supplies to the reference's optimiser, for every expression
 * gpk_gpr_lml_grad_expr covers, the variational parameters included; float64.  The forward builds
 * K = k(X) + jitter I = L L^T (the factorisation ops.cholesky runs), fmean - m(X) = L m and
 * fvar[n,p] = sum_k (L S_p)[n,k]^2; then with s the noise variance, w = -1/(2s), m = q_mu [N, P],
 * S_p = tril(q_sqrt[p]) (the strict upper part of q_sqrt is never read), Sig = sum_p S_p S_p^T, R = (Yc - L m) / s,
 * Phi(T) = tril(T) with its diagonal halved and sym(T) = (T + T^T) / 2:
 *   F        = sum_np [-1/2 log(2 pi s) - ((Yc - L m)^2 + fvar) / (2s)] - KL_white(m, S)
 *   Lbar     = tril(R m^T + 2w L Sig)                        (dF/dL)
 *   dF/dK    = sym(L^-T Phi(L^T Lbar) L^-1)                  (the Cholesky adjoint; the jitter carries no parameter)
 *   dF/dq_mu = L^T R - m
 *   dF/dS_p  = tril(2w (L^T L) S_p - S_p) + diag(1 / diag S_p)
 *   dF/ds    = sum_np [-1/(2s) + ((Yc - L m)^2 + fvar) / (2 s^2)],   dF/dm(X) = R
 * The kernel parameters take sum_ij dF/dK_ij dK_ij/dtheta over the N x N square, the diagonal included (White counts).
 *   out:     device double[n_out]: [0] ELBO, [1] sum of variational expectations, [2] KL, [3] Cholesky info (0, or
 *            the first non-positive pivot), [4] d/dnoise_variance, [5 ...] the leaf slots in the layout
 *            gpk_gpr_lml_grad_slots counts; n_out >= 5 + slots.
 *   dq_mu:   device double[N, P] row-major; dq_sqrt: device double[P, N, N] row-major, its strict upper parts 0.
 *   Limits (status -1 and gpk_last_error otherwise): those of gpk_gpr_lml_grad_expr, dtype GPK_F64, dq_mu and dq_sqrt
 *            non-NULL, D at most about 3 pad4(N) columns of X (the scratch of the square pass).
 *   gpk_vgp_elbo_grad_dm: byte offset of dF/dm(X) [N, P] (row-major, ld P) inside the workspace, valid after the call.
 *   ws:      gpk_vgp_elbo_grad_ws(N, P, dtype) bytes. */
GPK_API size_t gpk_vgp_elbo_grad_ws(int64_t N, int64_t P, int dtype);
GPK_API size_t gpk_vgp_elbo_grad_dm(int64_t N, int64_t P, int dtype);
GPK_API int gpk_vgp_elbo_grad(const gpk_knode* nodes, int n_nodes, const int32_t* dims, const double* ard,
                              const void* X, int64_t N, int64_t ldx, int64_t D, const void* Yc, int64_t P,
                              const void* q_mu, const void* q_sqrt, double noise_variance, double jitter, int dtype,
                              double* out, int n_out, double* dq_mu, double* dq_sqrt, void* ws, void* stream);

/* One natural-gradient step on q(u) = N(m, S S^T) for each of P latent GPs (gpflow/optimizers/natgrad.py:280-367, with
 * the parameter conversions of natgrad.py:429-502 written out), ascending the ELBO F; the reference descends -F and takes
 * the same step.  For latent p: m = q_mu[:, p], S = tril(q_sqrt[p]), Sig = S S^T, gm = dq_mu[:, p] = dF/dm,
 * gS = dq_sqrt[p] = dF/dS (as the gradient entries above return them: constrained values, strict upper parts 0),
 * Phi(T) = the strict lower triangle of T plus half its diagonal, sym(T) = (T + T^T) / 2, J the index reversal and
 *   H = sym(Phi(S^T gS)) = S^T Sigbar S,  Sigbar = sym(S^-T Phi(S^T gS) S^-1) = dF/d(Sig + m m^T):
 *   GPK_XI_NAT (the natural parameters, XiNat):  B = I - 2 gamma H = U U^T with U upper, taken as J B J = C C^T
 *       (lower Cholesky, U = J C J);  S' = S U^-T (lower, S' S'^T = (Sig^-1 - 2 gamma Sigbar)^-1),
 *       m' = m + gamma S' S'^T gm  (= m + gamma S B^-1 S^T gm).  One product S^T gS, one Cholesky and one triangular
 *       solve per latent; neither Sig^-1, S^-1 nor a second Cholesky is formed.
 *   GPK_XI_SQRT_MEAN_VAR (XiSqrtMeanVar, the forward-mode derivative of natural_to_meanvarsqrt):
 *       S' = S + 2 gamma S Phi(H) = S + gamma S Phi(S^T gS),  m' = m + gamma Sig gm.  No factorisation.
 * Sign of diag(S): q_sqrt may hold negative diagonal entries (the triangular transform does not keep them positive).
 * The step follows the chain rule through q_sqrt itself: with D = diag(sign(diag S)), XiNat runs on S D and gS D (H
 * becomes D H D) and returns the factor with a positive diagonal, which is what the reference's Cholesky returns.
 * XiSqrtMeanVar needs no such care.  Both agree with the reference exactly when diag(S) > 0; with negative entries the
 * reference applies gS as though it were the gradient at chol(Sig), which it is not, and the two differ.
 *   q_mu [M, P], q_sqrt [P, M, M] row-major (SVGP with q_diag = 0, VGP); the strict upper part of q_sqrt is never read.
 *   Out of place: q_mu_out [M, P] and q_sqrt_out [P, M, M] must not be the inputs; q_sqrt_out is written in full, zeros
 *   above the diagonal.  A failed step leaves the parameters untouched when the caller discards the outputs.
 *   info: P device words, each 0, k > 0 (XiNat: the 1-based first non-positive pivot of that latent's J B J, the step
 *   is too long for the current q) or -(i + 1) (q_sqrt[p][i, i] == 0, the first such i; S is singular).  The outputs
 *   of a latent with info != 0 are undefined.
 *   Limits (status -1 and gpk_last_error otherwise): dtype GPK_F64, gamma > 0 and finite.
 *   ws: gpk_natgrad_step_ws(M, P, xi, dtype) bytes (three M x M matrices, plus the factorisation's workspace for XiNat).
 * Asynchronous on `stream`. */
enum { GPK_XI_NAT = 0, GPK_XI_SQRT_MEAN_VAR = 1 };
GPK_API size_t gpk_natgrad_step_ws(int64_t M, int64_t P, int xi, int dtype);
GPK_API int gpk_natgrad_step(int xi, int64_t M, int64_t P, const void* q_mu, const void* q_sqrt, const double* dq_mu,
                             const double* dq_sqrt, double gamma, int dtype, void* q_mu_out, void* q_sqrt_out,
                             int32_t* info, void* ws, void* stream);

/* ---- Instrumentation (bench.py / tests; not on the numeric path) ---------------------------- */
/* Number of CUDA kernels launched by this library since the last reset. */
GPK_API int64_t gpk_launch_count(void);
GPK_API void gpk_launch_count_reset(void);
/* Per-kernel-class device timing with CUDA events recorded on the launch stream around every
 * launch (single-threaded diagnostic).  Classes: 0 kbuild, 1 tiled DMMA / SIMT GEMM (small-K trailing
 * updates, TRSM blocks), 2 potrf leaf (128x128 factor+invert; includes its look-ahead spin), 3 skinny
 * GEMM, 4 reductions/elementwise/slicing, 5 int8 tensor-core kernels (int8 digit SYRK, tf32 GEMM), 6 panel solve.
 * gpk_prof_read synchronises, writes summed milliseconds and launch counts for `n` classes and
 * clears the records; gpk_prof_read2 also returns the operations ISSUED per class (class 5: MACs on
 * the tensor pipe, padding tiles included). */
#define GPK_PROF_CLASSES 8
/* Tuning aid: runs ONE fp64 128x128 leaf (factor+invert) and stores clock64() at its phase
 * boundaries into dbg[0..11] (device int64, at least 12 entries; scripts/leaf_timing.py names them). */
GPK_API int gpk_debug_leaf(void* A, int64_t lda, int n, void* dinv, void* dbg, void* stream);
/* Test aid: ONE int8 digit-sliced trailing update as gpk_potrf issues it for rows with row-maximum scales (the GPK_TC_STATIC=0
 * path).  A holds the m operand rows (row-major, lda); their columns [k0, k0 + K) are sliced into S digit planes (S = 6, 7 or 8)
 * stored as rows [r0, r0 + m) of a factorisation's plane store, then
 *     C[m, n] -= A[0 : m, k0 : k0 + K] A[0 : n, k0 : k0 + K]^T
 * runs on the wgmma int8 kernel in clusters of `cluster` CTAs (1, 2 or 4); lower = 1: only the 128 x 32 tiles touching the lower
 * triangle of C.  r0 % 128 == 0, k0 % 32 == 0, K % 32 == 0, k0 + K <= r0, n <= m, K * S * 2^14 < 2^31.
 * rowscale_out (device, m doubles: the row scales 2^(e_i - 6)) and head_flag (device int[2], zeroed by the caller: head tiles
 * published, 32x32 units of C's leading 128x128 block published) may be NULL.  Allocates the planes of the m rows; synchronises. */
GPK_API int gpk_debug_syrk_i8(const void* A, int64_t lda, int64_t r0, int64_t k0, int64_t K, void* C, int64_t ldc,
                              int64_t m, int64_t n, int lower, int S, int cluster, void* rowscale_out, void* head_flag,
                              void* stream);
/* Test aid: one fp64 step of the inverse chain the device gradients run (GPR, SGPR, SVGP, VGP), as they call it.
 * L [n, ld] is a lower factor as gpk_potrf leaves it, dinv the inverses of its 128x128 diagonal blocks from gpk_potrf's ws.
 *   GPK_CHAIN_POTRI:        L <- L^-1 and out <- lower triangle of K^-1 = L^-T L^-1.  Reads only the lower triangle of L.
 *                           Above the diagonal, L's entries inside the 128x128 diagonal blocks become 0 and every other entry
 *                           of L is left as it was.  out's entries above the diagonal inside its 128x128 diagonal blocks
 *                           are scratch; its other entries above the diagonal are not written.
 *                           ws: gpk_debug_inverse_chain_ws bytes.
 *   GPK_CHAIN_LAUUM:        out <- lower triangle of L^T L.  The strict upper part of L's 128x128 diagonal blocks must be
 *                           zero (as POTRI leaves it): the leaf products read those blocks whole as their second operand.
 *                           L's other entries above the diagonal are never read.  out's strict upper triangle as for
 *                           POTRI.  dinv, T and ws unused.
 *   GPK_CHAIN_CHOL_ADJOINT: out <- G = -sym(L^-T Phi(T) L^-1), Phi(T) = strict lower triangle of T plus half its diagonal,
 *                           the whitened Cholesky adjoint of SVGP and VGP.  out is written in full and is exactly
 *                           symmetric; T is overwritten; T and out share ld (ldo == ld).  Reads only the lower triangle of L.
 * Asynchronous on `stream`. */
enum { GPK_CHAIN_POTRI = 0, GPK_CHAIN_LAUUM = 1, GPK_CHAIN_CHOL_ADJOINT = 2 };
GPK_API size_t gpk_debug_inverse_chain_ws(int op, int64_t n);
GPK_API int gpk_debug_inverse_chain(int op, double* L, int64_t n, int64_t ld, const double* dinv, double* T,
                                    double* out, int64_t ldo, void* ws, void* stream);
/* Tuning aid: device timeline of a factorisation.  While `buf` is set, thread 0 of selected CTAs of the leaf (id 1), fused
 * panel (2), plain panel (3) and int8 tensor-core update (4) kernels append (%globaltimer ns, id << 8 | phase) pairs to buf[2 * capacity]
 * (device uint64) through the counter *pos (device uint32).  phase 0 = first CTA started, 1 = inputs ready (leaf) / look-ahead
 * block published (panel, update), 2 = first CTA done, 3 = last CTA done.  buf = NULL switches it off.  scripts/trace_chain.py. */
GPK_API int gpk_debug_trace(void* buf, void* pos, unsigned int capacity);
GPK_API int gpk_prof_enable(int on);
GPK_API int gpk_prof_read(double* ms, int64_t* launches, int n);
GPK_API int gpk_prof_read2(double* ms, int64_t* launches, double* work, int n);
/* Pipe peaks measured in place (operands resident, every SM busy): out_host[0] = wgmma .s8 issue peak in
 * T(int8 op)/s (2 per MAC), out_host[1] = mma.sync.m8n8k4.f64 peak in TFLOP/s, out_host[2] = SM count.  Synchronises.
 * The roofline denominators bench.py reports for syrk_i8_kernel and the DMMA kernels. */
GPK_API int gpk_peak_probe(double* out_host, void* stream);
/* Digit planes S used by the int8 tensor-core trailing updates of the most recent fp64 factorisation on this process (chosen from
 * the conditioning hint of the caller: 6 or 7 base-256 planes; 0 = no update ran on the int8 tensor cores, e.g. n < 512 or fp32). */
GPK_API int gpk_potrf_last_slices(void);
/* Eager creation of the library-owned per-(device, stream) resources (see "Conventions"): the look-ahead side stream and
 * events, and `tf32_scratch_bytes` of TF32 plane scratch (0 = skip; 2 * 4 * (m + n) * k bytes cover an m x n x k product). */
GPK_API int gpk_warm(size_t tf32_scratch_bytes, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* GPK_H_ */
