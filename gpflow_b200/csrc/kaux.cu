// kaux.cu — covariance builders for the kernels that are not functions of a Gram term (SURVEY.md 8(f) rank 4):
//   Cosine      sigma^2 cos(2 pi sum_d (x_d - x'_d) / l_d)                          gpflow/kernels/stationaries.py:316-332
//   Periodic    base.K_r(sum_d |sin(pi (x_d - x'_d) / p_d)| / l_d)  (Matern / Exponential bases) or
//               base.K_r2(sum_d sin^2(pi (x_d - x'_d) / p_d) / l_d^2)  (SquaredExponential / RationalQuadratic)
//                                                                                   gpflow/kernels/periodic.py:28-111
//   ArcCosine   sigma^2 / pi * J_n(theta) |x|^n |x'|^n,  |x|^2 = sum_d w_d x_d^2 + b     gpflow/kernels/misc.py:27-200
//   Coregion    B[int(x), int(x')],  B = W W^T + diag(kappa) (built on the host, O x O)    gpflow/kernels/misc.py:203-296
// and the sigmoid weights of ChangePoints (gpflow/kernels/changepoints.py:26-193), whose K is a sum of
// diag(a_i) K_i diag(a_i') composed from these pieces by the Python layer.
// One thread per output element, the two rows' active columns read straight from global memory (L1/L2 resident: D is
// small); these kernels are plug-in breadth, not the benchmarked path.
#include "internal.cuh"

using namespace gpk;

namespace gpk {

template <typename T>
__device__ __forceinline__ double base_k(int base, double var, double alpha, double r, double r2) {
  // stationaries.py:209-210 (RBF), 237-238 (RQ), 250-251 (Exponential), 270-271, 290-292, 311-313 (Matern)
  switch (base) {
    case GPK_K_RBF: return var * exp(-0.5 * r2);
    case GPK_K_RQ: return var * pow(1.0 + 0.5 * r2 / alpha, -alpha);
    case GPK_K_EXPONENTIAL: return var * exp(-0.5 * r);
    case GPK_K_MATERN12: return var * exp(-r);
    case GPK_K_MATERN32: { const double s3 = 1.7320508075688772935; return var * (1.0 + s3 * r) * exp(-s3 * r); }
    default: { const double s5 = 2.2360679774997896964; return var * (1.0 + s5 * r + (5.0 / 3.0) * r * r) * exp(-s5 * r); }
  }
}

__device__ __forceinline__ double arccos_J(int order, double theta) {  // misc.py:141-157
  const double pi = 3.14159265358979323846;
  if (order == 0) return pi - theta;
  if (order == 1) return sin(theta) + (pi - theta) * cos(theta);
  return 3.0 * sin(theta) * cos(theta) + (pi - theta) * (1.0 + 2.0 * cos(theta) * cos(theta));
}

template <typename T>
__device__ double kaux_eval(const gpk_kaux_desc& d, const T* xa, const T* xb) {
  const double pi = 3.14159265358979323846;
  if (d.op == GPK_KAUX_COSINE) {
    double s = 0.0;
    for (int q = 0; q < d.n_dims; ++q) s += ((double)xa[d.dims[q]] - (double)xb[d.dims[q]]) * d.scale[q];
    return d.variance * cos(2.0 * pi * s);
  }
  if (d.op == GPK_KAUX_PERIODIC) {
    const bool use_r = d.base == GPK_K_EXPONENTIAL || d.base == GPK_K_MATERN12 || d.base == GPK_K_MATERN32 ||
                       d.base == GPK_K_MATERN52;  // kernels with K_r (periodic.py:102-107)
    double acc = 0.0;
    for (int q = 0; q < d.n_dims; ++q) {
      const double sn = sin(pi * ((double)xa[d.dims[q]] - (double)xb[d.dims[q]]) / d.period[q]) * d.scale[q];
      acc += use_r ? fabs(sn) : sn * sn;
    }
    return base_k<T>(d.base, d.variance, d.alpha, acc, acc);
  }
  // ArcCosine
  double num = d.bias, na = d.bias, nb = d.bias;
  for (int q = 0; q < d.n_dims; ++q) {
    const double a = (double)xa[d.dims[q]], b = (double)xb[d.dims[q]], w = d.scale[q];
    num += w * a * b;
    na += w * a * a;
    nb += w * b * b;
  }
  const double da = sqrt(na), db = sqrt(nb);
  const double jitter = 1e-15;
  const double theta = acos(jitter + (1.0 - 2.0 * jitter) * (num / da / db));
  double pw = 1.0;
  for (int o = 0; o < d.order; ++o) pw *= da * db;
  return d.variance * (1.0 / pi) * arccos_J(d.order, theta) * pw;
}

// A Coregion index truncates toward zero like tf.cast(x, tf.int32) (1.7 -> 1, -0.5 -> 0); it is valid when the truncated
// value lies in [0, table_dim).  Tested on the value before the conversion, so that NaN (which converts to 0 on the
// device) and values beyond the int range are invalid too.
__device__ __forceinline__ bool coregion_index_ok(double x, int table_dim) { return x > -1.0 && x < (double)table_dim; }

template <typename T>
__global__ void __launch_bounds__(256)
kaux_kernel(gpk_kaux_desc d, const T* __restrict__ X, int64_t N, int64_t ldx, const T* __restrict__ X2, int64_t N2,
            int64_t ldx2, T* __restrict__ K, int64_t ldk) {
  const int64_t j = (int64_t)blockIdx.x * 32 + (threadIdx.x & 31);
  const int64_t i0 = (int64_t)blockIdx.y * 64 + (threadIdx.x >> 5) * 8;
  if (j >= N2) return;
  for (int u = 0; u < 8; ++u) {
    const int64_t i = i0 + u;
    if (i >= N) return;
    double v;
    if (d.op == GPK_KAUX_COREGION) {
      const double xa = (double)X[i * ldx + d.dims[0]], xb = (double)X2[j * ldx2 + d.dims[0]];
      const bool ok = coregion_index_ok(xa, d.table_dim) && coregion_index_ok(xb, d.table_dim);
      v = ok ? ((const double*)d.table)[(int64_t)(int)xa * d.table_dim + (int)xb] : nan("");
    } else {
      v = kaux_eval<T>(d, X + i * ldx, X2 + j * ldx2);
    }
    K[i * ldk + j] = (T)v;
  }
}

template <typename T>
__global__ void kaux_diag_kernel(gpk_kaux_desc d, const T* __restrict__ X, int64_t N, int64_t ldx, T* __restrict__ out) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= N) return;
  const double pi = 3.14159265358979323846;
  double v;
  if (d.op == GPK_KAUX_COREGION) {
    const double xa = (double)X[i * ldx + d.dims[0]];
    v = coregion_index_ok(xa, d.table_dim) ? ((const double*)d.table)[(int64_t)(int)xa * (d.table_dim + 1)] : nan("");
  } else if (d.op == GPK_KAUX_ARCCOS) {  // misc.py:197-200
    double na = d.bias;
    for (int q = 0; q < d.n_dims; ++q) { const double a = (double)X[i * ldx + d.dims[q]]; na += d.scale[q] * a * a; }
    double pw = 1.0;
    for (int o = 0; o < d.order; ++o) pw *= na;
    v = d.variance * (1.0 / pi) * arccos_J(d.order, 0.0) * pw;
  } else if (d.op == GPK_KAUX_PERIODIC) {
    v = base_k<T>(d.base, d.variance, d.alpha, 0.0, 0.0);  // base_kernel.K_diag = variance (periodic.py:91-93)
  } else {
    v = d.variance;  // Cosine: stationaries.py:82-83
  }
  out[i] = (T)v;
}

// ChangePoints weights: out[n] = (has_lo ? sig_lo(x_n) : 1) * (has_hi ? 1 - sig_hi(x_n) : 1), sig(x) = 1 / (1 + exp(-s (x - x0)))
template <typename T>
__global__ void cp_weights_kernel(const T* __restrict__ X, int64_t N, int64_t ldx, int dim, int has_lo, double loc_lo,
                                  double steep_lo, int has_hi, double loc_hi, double steep_hi, T* __restrict__ out) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= N) return;
  const double x = (double)X[i * ldx + dim];
  double w = 1.0;
  if (has_lo) w *= 1.0 / (1.0 + exp(-steep_lo * (x - loc_lo)));
  if (has_hi) w *= 1.0 - 1.0 / (1.0 + exp(-steep_hi * (x - loc_hi)));
  out[i] = (T)w;
}

template <typename T>
__global__ void hadamard_kernel(int64_t m, int64_t n, const T* __restrict__ X, int64_t ldx, T* __restrict__ Y, int64_t ldy) {
  const int64_t j = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= n) return;
  for (int64_t i = blockIdx.y; i < m; i += gridDim.y) Y[i * ldy + j] *= X[i * ldx + j];
}

// A = max(A, lower) [then squared]: evaluate_parameter_or_function of a heteroskedastic likelihood
// (gpflow/likelihoods/utils.py; scalar_continuous.py:92-102)
template <typename T>
__global__ void clamp_min_kernel(T* __restrict__ A, int64_t m, int64_t n, int64_t lda, T lower, int square) {
  const int64_t j = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= n) return;
  for (int64_t i = blockIdx.y; i < m; i += gridDim.y) {
    T v = A[i * lda + j];
    v = v > lower ? v : lower;
    A[i * lda + j] = square == 1 ? v * v : (square == 2 ? (T)sqrt((double)v) : v);
  }
}

}  // namespace gpk

extern "C" int gpk_clamp_min(void* A, int64_t m, int64_t n, int64_t lda, double lower, int square, int dtype,
                             void* stream) {
  const cudaStream_t st = (cudaStream_t)stream;
  GPK_DTYPE_OK("clamp_min");
  if (m <= 0 || n <= 0) return 0;
  dim3 grid((unsigned)((n + 255) / 256), (unsigned)(m < 65535 ? m : 65535));
  if (dtype == GPK_F64) clamp_min_kernel<double><<<grid, 256, 0, st>>>((double*)A, m, n, lda, lower, square);
  else clamp_min_kernel<float><<<grid, 256, 0, st>>>((float*)A, m, n, lda, (float)lower, square);
  GPK_LAUNCH_OK();
  return 0;
}

extern "C" int gpk_kaux(const gpk_kaux_desc* d, const void* X, int64_t N, int64_t ldx, const void* X2, int64_t N2,
                        int64_t ldx2, void* K, int64_t ldk, int dtype, void* stream) {
  const cudaStream_t st = (cudaStream_t)stream;
  GPK_DTYPE_OK("kaux");
  GPK_CHECK_ARG(d && X && K && N > 0, "kaux: bad arguments");
  GPK_CHECK_ARG(d->op >= GPK_KAUX_COSINE && d->op <= GPK_KAUX_COREGION, "kaux: unknown op %d", d->op);
  GPK_CHECK_ARG(d->n_dims >= 1 && d->n_dims <= GPK_KAUX_MAXD, "kaux: 1..%d active dims", GPK_KAUX_MAXD);
  GPK_CHECK_ARG(d->op != GPK_KAUX_COREGION || (d->table && d->table_dim > 0), "kaux: Coregion needs its B table");
  if (!X2) { X2 = X; N2 = N; ldx2 = ldx; }
  ProfScope ps(PROF_KBUILD, st);
  // grid.y covers 64 rows per block and is limited to 65535: taller K runs as row chunks of X and K (no element
  // depends on its global row index)
  const int64_t rows_max = 65535 * 64;
  const size_t es = dtype == GPK_F64 ? sizeof(double) : sizeof(float);
  for (int64_t r0 = 0; r0 < N; r0 += rows_max) {
    const int64_t n = N - r0 < rows_max ? N - r0 : rows_max;
    const void* Xc = (const char*)X + (size_t)(r0 * ldx) * es;
    void* Kc = (char*)K + (size_t)(r0 * ldk) * es;
    dim3 grid((unsigned)((N2 + 31) / 32), (unsigned)((n + 63) / 64));
    if (dtype == GPK_F64)
      kaux_kernel<double><<<grid, 256, 0, st>>>(*d, (const double*)Xc, n, ldx, (const double*)X2, N2, ldx2, (double*)Kc, ldk);
    else
      kaux_kernel<float><<<grid, 256, 0, st>>>(*d, (const float*)Xc, n, ldx, (const float*)X2, N2, ldx2, (float*)Kc, ldk);
    GPK_LAUNCH_OK();
  }
  return 0;
}

extern "C" int gpk_kaux_diag(const gpk_kaux_desc* d, const void* X, int64_t N, int64_t ldx, void* out, int dtype,
                             void* stream) {
  const cudaStream_t st = (cudaStream_t)stream;
  GPK_DTYPE_OK("kaux_diag");
  GPK_CHECK_ARG(d && X && out && N > 0, "kaux_diag: bad arguments");
  const unsigned grid = (unsigned)((N + 255) / 256);
  if (dtype == GPK_F64) kaux_diag_kernel<double><<<grid, 256, 0, st>>>(*d, (const double*)X, N, ldx, (double*)out);
  else kaux_diag_kernel<float><<<grid, 256, 0, st>>>(*d, (const float*)X, N, ldx, (float*)out);
  GPK_LAUNCH_OK();
  return 0;
}

extern "C" int gpk_changepoint_weights(const void* X, int64_t N, int64_t ldx, int dim, int has_lo, double loc_lo,
                                       double steep_lo, int has_hi, double loc_hi, double steep_hi, void* out,
                                       int dtype, void* stream) {
  const cudaStream_t st = (cudaStream_t)stream;
  GPK_DTYPE_OK("changepoint_weights");
  GPK_CHECK_ARG(X && out && N > 0, "changepoint_weights: bad arguments");
  const unsigned grid = (unsigned)((N + 255) / 256);
  if (dtype == GPK_F64)
    cp_weights_kernel<double><<<grid, 256, 0, st>>>((const double*)X, N, ldx, dim, has_lo, loc_lo, steep_lo, has_hi, loc_hi,
                                                   steep_hi, (double*)out);
  else
    cp_weights_kernel<float><<<grid, 256, 0, st>>>((const float*)X, N, ldx, dim, has_lo, loc_lo, steep_lo, has_hi, loc_hi,
                                                  steep_hi, (float*)out);
  GPK_LAUNCH_OK();
  return 0;
}

extern "C" int gpk_hadamard(int64_t m, int64_t n, const void* X, int64_t ldx, void* Y, int64_t ldy, int dtype,
                            void* stream) {
  const cudaStream_t st = (cudaStream_t)stream;
  GPK_DTYPE_OK("hadamard");
  if (m <= 0 || n <= 0) return 0;
  dim3 grid((unsigned)((n + 255) / 256), (unsigned)(m < 65535 ? m : 65535));
  if (dtype == GPK_F64) hadamard_kernel<double><<<grid, 256, 0, st>>>(m, n, (const double*)X, ldx, (double*)Y, ldy);
  else hadamard_kernel<float><<<grid, 256, 0, st>>>(m, n, (const float*)X, ldx, (float*)Y, ldy);
  GPK_LAUNCH_OK();
  return 0;
}
