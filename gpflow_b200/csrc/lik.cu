// lik.cu — scalar likelihoods: variational expectations, predictive mean / variance and log density, and the per-element
// adjoints of the variational expectations that the SVGP and VGP backwards (fused.cu::svgp_elbo_grad, vgp_elbo_grad)
// consume.
//   Bernoulli : gpflow/likelihoods/scalar_discrete.py:81-117, utils.py::inv_probit, logdensities.py:49-50
//   Poisson   : scalar_discrete.py:29-78, logdensities.py:58-59
//   StudentT  : scalar_continuous.py:177-213, logdensities.py:93-102
//   MultiClass: multiclass.py:55-243 (RobustMax)
//   quadrature: likelihoods/base.py:279-456 -> quadrature/gauss_hermite.py:30-154 (NDiagGHQuadrature, 20 points)
// Every element (n, p) of the scalar likelihoods is one likelihood; one thread per element, fp64 arithmetic whatever the
// storage dtype, sums through warp shuffles and one atomicAdd per CTA.  MultiClass couples
// the latents of a row: one warp per row (below).
#include <math.h>

#include "internal.cuh"

namespace gpk {

// numpy.polynomial.hermite.hermgauss(20) scaled as gauss_hermite.py:42-44: z = sqrt(2) x, w = w / sqrt(pi)
constexpr int GH_N = 20;
__constant__ double GH_Z[GH_N] = {
    -7.619048541679759,  -6.510590157013655,  -5.5787388058932015, -4.734581334046055,  -3.9439673506573163,
    -3.18901481655339,   -2.458663611172368,  -1.745247320814127,  -1.0429453488027511, -0.3469641570813559,
    0.3469641570813559,  1.0429453488027511,  1.745247320814127,   2.458663611172368,   3.18901481655339,
    3.9439673506573163,  4.734581334046055,   5.5787388058932015,  6.510590157013655,   7.619048541679759};
__constant__ double GH_W[GH_N] = {
    1.2578006724379234e-13, 2.4820623623151755e-10, 6.127490259982928e-08, 4.402121090230851e-06,
    0.00012882627996192928, 0.00183010313108049,    0.013997837447101022,  0.0615063720639769,
    0.16173933398399998,    0.2607930634495549,     0.2607930634495549,    0.16173933398399998,
    0.0615063720639769,     0.013997837447101022,   0.00183010313108049,   0.00012882627996192928,
    4.402121090230851e-06,  6.127490259982928e-08,  2.4820623623151755e-10, 1.2578006724379234e-13};

// The descriptor with the host-side constants of its log density.
struct LikD {
  int type;
  double scale, df, binsize, noise;
  double c0;  // Gaussian: -1/2 log(2 pi s);  Student-t: lgamma((df+1)/2) - lgamma(df/2) - 1/2 log(scale^2 df pi);
              // Poisson: log binsize
};

// P: the latents per row the caller passes (MULTICLASS needs P == num_classes).  `predict`: a GAUSSIAN noise of 0 is
// accepted (the predictions add it to Fvar; a heteroskedastic caller folds its variance into Fvar and passes 0).
static int lik_prepare(const gpk_lik* lik, LikD& d, int64_t P, const char* who, bool predict = false) {
  GPK_CHECK_ARG(lik, "%s: the likelihood descriptor is NULL", who);
  GPK_CHECK_ARG(lik->type >= GPK_LIK_GAUSSIAN && lik->type <= GPK_LIK_MULTICLASS, "%s: unknown likelihood type %d", who,
                lik->type);
  GPK_CHECK_ARG(lik->type == GPK_LIK_GAUSSIAN || lik->type == GPK_LIK_POISSON || lik->n_gh == GH_N,
                "%s: %d Gauss-Hermite points; the quadrature has %d", who, lik->n_gh, GH_N);
  if (lik->type == GPK_LIK_MULTICLASS) {
    GPK_CHECK_ARG(lik->epsilon > 0.0 && lik->epsilon < 1.0, "%s: the RobustMax epsilon must lie in (0, 1) (%g)", who,
                  lik->epsilon);
    GPK_CHECK_ARG(lik->num_classes >= 2 && lik->num_classes <= GPK_LIK_MAX_CLASSES,
                  "%s: MultiClass covers 2 to %d classes (num_classes = %d)", who, GPK_LIK_MAX_CLASSES,
                  lik->num_classes);
    GPK_CHECK_ARG(P == lik->num_classes, "%s: MultiClass needs one latent per class (P = %lld, num_classes = %d)", who,
                  (long long)P, lik->num_classes);
  }
  d.type = lik->type;
  d.scale = lik->scale;
  d.df = lik->df;
  d.binsize = lik->binsize;
  d.noise = lik->noise;
  d.c0 = 0.0;
  if (d.type == GPK_LIK_GAUSSIAN) {
    GPK_CHECK_ARG(d.noise > 0.0 || (predict && d.noise == 0.0), "%s: Gaussian noise variance must be %s", who,
                  predict ? "non-negative" : "positive");
    d.c0 = -0.5 * LOG2PI - 0.5 * log(d.noise);
  } else if (d.type == GPK_LIK_POISSON) {
    GPK_CHECK_ARG(d.binsize > 0.0, "%s: Poisson binsize must be positive", who);
    d.c0 = log(d.binsize);
  } else if (d.type == GPK_LIK_STUDENT_T) {
    GPK_CHECK_ARG(d.scale > 0.0 && d.df > 0.0, "%s: Student-t scale and df must be positive", who);
    d.c0 = lgamma(0.5 * (d.df + 1.0)) - lgamma(0.5 * d.df) -
           0.5 * (log(d.scale * d.scale) + log(d.df) + 1.1447298858494001741434273513531);  // log(pi)
  }
  return 0;
}

// ---- MultiClass with RobustMax (multiclass.py:55-243) --------------------------------------------------------------
// One warp per row: class c = 32 j + lane sits in chunk j of lane `lane`, NJ = ceil(num_classes / 32) chunks held in
// registers; the 20 nodes in a loop.  The product over classes is an inclusive shuffle scan per chunk times the chunk
// totals; the gradient's exclusive products E_ck come from a prefix and a suffix scan (never the full product divided
// by cdf_ck, which underflows for many classes).
struct McD {
  int C;
  double eps, eps_k1, log1m, logk1;  // epsilon, epsilon / (C - 1), log(1 - epsilon), log eps_k1
  double inv1m, inveps;              // 1 / (1 - epsilon), 1 / epsilon
};

static McD mc_desc(const gpk_lik* lik) {
  McD m;
  m.C = lik->num_classes;
  m.eps = lik->epsilon;
  m.eps_k1 = lik->epsilon / (lik->num_classes - 1.0);
  m.log1m = log(1.0 - m.eps);
  m.logk1 = log(m.eps_k1);
  m.inv1m = 1.0 / (1.0 - m.eps);
  m.inveps = 1.0 / m.eps;
  return m;
}

constexpr double MC_SQUASH = 1e-6;  // RobustMax._squash
constexpr unsigned FULL_MASK = 0xffffffffu;

// the label of a row, truncated toward zero as to_default_int does; -1 outside [0, C)
__device__ __forceinline__ int mc_label(double y, int C) { return (y > -1.0 && y < (double)C) ? (int)y : -1; }

__device__ __forceinline__ double mc_scan_up(double x, int lane) {  // inclusive prefix product over lanes 0..lane
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const double t = __shfl_up_sync(FULL_MASK, x, o);
    if (lane >= o) x *= t;
  }
  return x;
}

__device__ __forceinline__ double mc_scan_down(double x, int lane) {  // inclusive suffix product over lanes lane..31
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const double t = __shfl_down_sync(FULL_MASK, x, o);
    if (lane + o < 32) x *= t;
  }
  return x;
}

// The row's latents in registers: mu (mean, + m(X)), v and is = 1 / s_c = rsqrt(max(v, 1e-10)) of the lane's classes
// (0, 1 and 1 past C).  The node loop multiplies by is: no fp64 division in it.
template <int NJ>
struct McRow {
  double mu[NJ], is[NJ], v[NJ];
};

template <typename T, int NJ>
__device__ __forceinline__ void mc_load(McRow<NJ>& r, const T* __restrict__ Fmu, const T* __restrict__ mX,
                                        const T* __restrict__ Fvar, int64_t n, int64_t P, int64_t var_sb,
                                        int64_t var_sp, int C, int lane) {
#pragma unroll
  for (int j = 0; j < NJ; ++j) {
    const int c = 32 * j + lane;
    r.mu[j] = 0.0;
    r.v[j] = 1.0;
    if (c < C) {
      r.mu[j] = (double)Fmu[n * P + c] + (mX ? (double)mX[n * P + c] : 0.0);
      r.v[j] = (double)Fvar[n * var_sb + c * var_sp];
    }
    r.is[j] = rsqrt(fmax(r.v[j], 1e-10));
  }
}

// p = sum_k w_k prod_{c != y} cdf_ck for the label y (-1: no class left out; mu_y = v_y = 0), the same in every lane.
// With GRAD also, per chunk, G[j] = sum_k g_ck and H[j] = sum_k g_ck d_ck of the lane's class, gs = sum_k sum_{c != y}
// g_ck and gx = sum_k x_k sum_{c != y} g_ck of the lane's classes (warp-reduce them), g_ck = w_k E_ck (1 - 2 squash)
// phi(d_ck) / s_c.
template <int NJ, bool GRAD>
__device__ __forceinline__ double mc_prob(const McRow<NJ>& r, int y, double mu_y, double s_y, int C, int lane,
                                          double* G, double* H, double& gs, double& gx) {
  double p = 0.0;
  gs = gx = 0.0;
  if (GRAD) {
#pragma unroll
    for (int j = 0; j < NJ; ++j) G[j] = H[j] = 0.0;
  }
  for (int k = 0; k < GH_N; ++k) {
    const double xk = GH_Z[k] * 0.70710678118654752440, wk = GH_W[k];
    const double X = fma(xk, s_y, mu_y);
    double cdf[NJ], d[NJ], incl[NJ], tot[NJ];
#pragma unroll
    for (int j = 0; j < NJ; ++j) {
      const int c = 32 * j + lane;
      d[j] = (X - r.mu[j]) * r.is[j];
      cdf[j] = (c < C && c != y) ? fma(0.5 * (1.0 + erf(d[j] * 0.70710678118654752440)), 1.0 - 2.0 * MC_SQUASH,
                                       MC_SQUASH)
                                 : 1.0;
      incl[j] = mc_scan_up(cdf[j], lane);
      tot[j] = __shfl_sync(FULL_MASK, incl[j], 31);
    }
    double all = 1.0;
#pragma unroll
    for (int j = 0; j < NJ; ++j) all *= tot[j];
    p = fma(wk, all, p);
    if (GRAD) {
      double before = 1.0;  // product of the chunk totals before j
      double gk = 0.0;
#pragma unroll
      for (int j = 0; j < NJ; ++j) {
        double after = 1.0;
#pragma unroll
        for (int i = j + 1; i < NJ; ++i) after *= tot[i];
        const int c = 32 * j + lane;
        const double up = __shfl_up_sync(FULL_MASK, incl[j], 1);
        const double dn = __shfl_down_sync(FULL_MASK, mc_scan_down(cdf[j], lane), 1);
        const double E = before * after * (lane > 0 ? up : 1.0) * (lane < 31 ? dn : 1.0);
        const double g = (c < C && c != y)
                             ? wk * E * (1.0 - 2.0 * MC_SQUASH) * 0.39894228040143267794 * exp(-0.5 * d[j] * d[j]) *
                                   r.is[j]
                             : 0.0;
        G[j] += g;
        H[j] = fma(g, d[j], H[j]);
        gk += g;
        before *= tot[j];
      }
      gs += gk;
      gx = fma(xk, gk, gx);
    }
  }
  return p;
}

__device__ __forceinline__ double inv_probit(double f) {  // utils.py::inv_probit, jitter 1e-3
  return 0.5 * (1.0 + erf(f * 0.70710678118654752440)) * (1.0 - 2e-3) + 1e-3;
}

// log p(y | f) of the quadrature likelihoods, its f-derivative and (Student-t) its scale derivative
__device__ __forceinline__ double lik_logp(const LikD& L, double y, double f) {
  if (L.type == GPK_LIK_BERNOULLI) {
    const double p = inv_probit(f);
    return log(y == 1.0 ? p : 1.0 - p);
  }
  if (L.type == GPK_LIK_POISSON) {
    const double lam = exp(f) * L.binsize;
    return y * log(lam) - lam - lgamma(y + 1.0);
  }
  if (L.type == GPK_LIK_STUDENT_T) {
    const double r = (y - f) / L.scale;
    return L.c0 - 0.5 * (L.df + 1.0) * log(1.0 + r * r / L.df);
  }
  const double r = y - f;  // Gaussian
  return L.c0 - 0.5 * r * r / L.noise;
}

__device__ __forceinline__ double lik_dlogp(const LikD& L, double y, double f, double& dscale) {
  dscale = 0.0;
  if (L.type == GPK_LIK_BERNOULLI) {
    const double p = inv_probit(f);
    const double dp = (1.0 - 2e-3) * 0.39894228040143267794 * exp(-0.5 * f * f);  // (1 - 2 jitter) phi(f)
    return y == 1.0 ? dp / p : -dp / (1.0 - p);
  }
  if (L.type == GPK_LIK_POISSON) return y - exp(f) * L.binsize;
  if (L.type == GPK_LIK_STUDENT_T) {
    const double r = y - f, s2df = L.scale * L.scale * L.df, q = s2df + r * r;
    dscale = -1.0 / L.scale + (L.df + 1.0) * r * r / (L.scale * q);
    return (L.df + 1.0) * r / q;
  }
  return (y - f) / L.noise;  // Gaussian
}

// The variational expectation of one element, and with GRAD its derivatives w.r.t. mu, v and the likelihood parameter
// (Gaussian: the variance; Student-t: the scale).
template <bool GRAD>
__device__ __forceinline__ double lik_ve(const LikD& L, double y, double mu, double v, double& dmu, double& dv,
                                         double& dpar) {
  dmu = dv = dpar = 0.0;
  if (L.type == GPK_LIK_GAUSSIAN) {  // scalar_continuous.py:139-148
    const double r = y - mu, s = L.noise;
    if (GRAD) {
      dmu = r / s;
      dv = -0.5 / s;
      dpar = -0.5 / s + 0.5 * (r * r + v) / (s * s);
    }
    return L.c0 - 0.5 * (r * r + v) / s;
  }
  if (L.type == GPK_LIK_POISSON) {  // scalar_discrete.py:67-78
    const double e = exp(mu + 0.5 * v) * L.binsize;
    if (GRAD) {
      dmu = y - e;
      dv = -0.5 * e;
    }
    return y * mu - e - lgamma(y + 1.0) + y * L.c0;
  }
  const double sd = sqrt(v);
  double ve = 0.0, dz = 0.0;
#pragma unroll 4
  for (int k = 0; k < GH_N; ++k) {
    const double f = fma(sd, GH_Z[k], mu), wk = GH_W[k];
    if (GRAD) {
      double ds;
      const double g1 = lik_dlogp(L, y, f, ds);
      dmu = fma(wk, g1, dmu);
      dz = fma(wk * g1, GH_Z[k], dz);
      dpar = fma(wk, ds, dpar);
    }
    ve = fma(wk, lik_logp(L, y, f), ve);
  }
  if (GRAD) dv = dz / (2.0 * sd);  // d/dv of sqrt(v) z_k: the derivative of the 20-point sum itself
  return ve;
}

__device__ __forceinline__ double block_sum_256(double s, double* sh) {
  s = warp_sum(s);
  if ((threadIdx.x & 31) == 0) sh[threadIdx.x >> 5] = s;
  __syncthreads();
  double t = 0.0;
  if (threadIdx.x < 32) {
    t = threadIdx.x < (blockDim.x >> 5) ? sh[threadIdx.x] : 0.0;
    t = warp_sum(t);
  }
  return t;  // valid in thread 0
}

// Fmu [B, P] contiguous; Fvar[b * var_sb + p * var_sp]; Y[b * ldy + p]; mX[b * ldmx + p] or NULL (added to Fmu)
template <typename T>
__global__ void __launch_bounds__(256)
lik_varexp_kernel(LikD L, const T* __restrict__ Fmu, const T* __restrict__ Fvar, const T* __restrict__ Y,
                  const T* __restrict__ mX, int64_t total, int64_t P, int64_t ldy, int64_t ldmx, int64_t var_sb,
                  int64_t var_sp, double scale, double* out) {
  __shared__ double sh[32];
  double s = 0.0;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t b = i / P, p = i % P;
    const double mu = (double)Fmu[i] + (mX ? (double)mX[b * ldmx + p] : 0.0);
    double d0, d1, d2;
    s += lik_ve<false>(L, (double)Y[b * ldy + p], mu, (double)Fvar[b * var_sb + p * var_sp], d0, d1, d2);
  }
  s = block_sum_256(s, sh);
  if (threadIdx.x == 0) atomicAdd(out, scale * s);
}

// The SVGP backward's per-element adjoints (float64): fmu [B][P], fvar [P][B]; R [B][P] = c dVE/dmu, Wt [P][B] =
// c dVE/dv (not written when Wt is NULL), *gpar += c sum dVE/d(likelihood parameter).
__global__ void __launch_bounds__(256)
lik_grad_kernel(LikD L, const double* __restrict__ fmu, const double* __restrict__ fvar, const double* __restrict__ Y,
                const double* __restrict__ mX, int64_t B, int64_t P, double c, double* __restrict__ R,
                double* __restrict__ Wt, double* __restrict__ gpar) {
  __shared__ double sh[32];
  double s = 0.0;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < B * P; i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t b = i / P, p = i % P;
    const double mu = fmu[i] + (mX ? mX[i] : 0.0);
    double dmu, dv, dpar;
    lik_ve<true>(L, Y[i], mu, fvar[p * B + b], dmu, dv, dpar);
    R[i] = c * dmu;
    if (Wt) Wt[p * B + b] = c * dv;
    s += dpar;
  }
  s = block_sum_256(s, sh);
  if (threadIdx.x == 0 && (L.type == GPK_LIK_GAUSSIAN || L.type == GPK_LIK_STUDENT_T)) atomicAdd(gpar, c * s);
}

// predictive mean and variance of y (one thread per element)
template <typename T>
__global__ void __launch_bounds__(256)
lik_predict_mv_kernel(LikD L, const T* __restrict__ Fmu, const T* __restrict__ Fvar, int64_t total, T* __restrict__ mean,
                      T* __restrict__ var) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= total) return;
  const double mu = (double)Fmu[i], v = (double)Fvar[i];
  double m, vy;
  if (L.type == GPK_LIK_GAUSSIAN) {  // scalar_continuous.py:127-130
    m = mu;
    vy = v + L.noise;
  } else if (L.type == GPK_LIK_BERNOULLI) {  // scalar_discrete.py:93-101
    const double p = inv_probit(mu / sqrt(1.0 + v));
    m = p;
    vy = p - p * p;
  } else {  // base.py:379-400: E[E[y|f]] and E[Var[y|f] + E[y|f]^2] by quadrature
    const double sd = sqrt(v);
    const double cvar = L.type == GPK_LIK_STUDENT_T ? L.scale * L.scale * (L.df / (L.df - 2.0)) : 0.0;
    double ey = 0.0, ey2 = 0.0;
    for (int k = 0; k < GH_N; ++k) {
      const double f = fma(sd, GH_Z[k], mu), wk = GH_W[k];
      double cm, cv;
      if (L.type == GPK_LIK_POISSON) {
        cm = exp(f) * L.binsize;
        cv = cm;
      } else {
        cm = f;
        cv = cvar;
      }
      ey = fma(wk, cm, ey);
      ey2 = fma(wk, cv + cm * cm, ey2);
    }
    m = ey;
    vy = ey2 - ey * ey;
  }
  mean[i] = (T)m;
  var[i] = (T)vy;
}

// out[n] = sum_p log E[p(y | f)] (one thread per row)
template <typename T>
__global__ void __launch_bounds__(256)
lik_predict_ld_kernel(LikD L, const T* __restrict__ Fmu, const T* __restrict__ Fvar, const T* __restrict__ Y, int64_t N,
                      int64_t P, T* __restrict__ out) {
  const int64_t n = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (n >= N) return;
  double acc = 0.0;
  for (int64_t p = 0; p < P; ++p) {
    const int64_t i = n * P + p;
    const double mu = (double)Fmu[i], v = (double)Fvar[i], y = (double)Y[i];
    if (L.type == GPK_LIK_GAUSSIAN) {  // scalar_continuous.py:133-136
      const double tv = v + L.noise, r = y - mu;
      acc += -0.5 * (LOG2PI + log(tv) + r * r / tv);
    } else if (L.type == GPK_LIK_BERNOULLI) {  // scalar_discrete.py:103-108
      const double pr = inv_probit(mu / sqrt(1.0 + v));
      acc += log(y == 1.0 ? pr : 1.0 - pr);
    } else {  // base.py:344-359: logsumexp_k(log w_k + log p(y | f_k))
      const double sd = sqrt(v);
      double gmax = -INFINITY, se = 0.0;  // online: se = sum_k exp(g_k - gmax)
      for (int k = 0; k < GH_N; ++k) {
        const double g = lik_logp(L, y, fma(sd, GH_Z[k], mu)) + log(GH_W[k]);
        if (g > gmax) {
          se = se * exp(gmax - g) + 1.0;
          gmax = g;
        } else {
          se += exp(g - gmax);
        }
      }
      acc += gmax + log(se);
    }
  }
  out[n] = (T)acc;
}

// ---- MultiClass kernels: one warp per row (grid-stride over rows, so every lane of a warp takes the same rows) -------
// Fmu, mX [rows, P] contiguous (mX may be NULL); Fvar[n * var_sb + c * var_sp]; the label Y[n * ldy].
// Four warps per CTA: with one CTA per SM as the register bound, the four-chunk gradient fits in registers (at 256
// threads ptxas caps it at 128 registers and spills).
constexpr int MC_THREADS = 128;

// mu_y (with m(X)), v_y, s_y = sqrt(max(2 v_y, 1e-10)) and is_y = 1 / s_y of the label y; mu_y = v_y = 0 for y = -1
template <typename T>
__device__ __forceinline__ void mc_selected(const T* __restrict__ Fmu, const T* __restrict__ mX,
                                            const T* __restrict__ Fvar, int64_t n, int64_t P, int64_t var_sb,
                                            int64_t var_sp, int y, double& mu_y, double& v_y, double& s_y,
                                            double& is_y) {
  mu_y = v_y = 0.0;
  if (y >= 0) {
    mu_y = (double)Fmu[n * P + y] + (mX ? (double)mX[n * P + y] : 0.0);
    v_y = (double)Fvar[n * var_sb + y * var_sp];
  }
  const double q = fmax(2.0 * v_y, 1e-10);
  is_y = rsqrt(q);
  s_y = q * is_y;
}

__device__ __forceinline__ int64_t mc_first_row() { return ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5; }
__device__ __forceinline__ int64_t mc_row_stride() { return ((int64_t)gridDim.x * blockDim.x) >> 5; }

// *out += scale * sum_n VE_n
template <typename T, int NJ>
__global__ void __launch_bounds__(MC_THREADS, 1)
mc_varexp_kernel(McD L, const T* __restrict__ Fmu, const T* __restrict__ Fvar, const T* __restrict__ Y,
                 const T* __restrict__ mX, int64_t B, int64_t P, int64_t ldy, int64_t var_sb, int64_t var_sp,
                 double scale, double* out) {
  __shared__ double sh[32];
  double s = 0.0;
  const int lane = threadIdx.x & 31;
  for (int64_t n = mc_first_row(); n < B; n += mc_row_stride()) {
    McRow<NJ> r;
    mc_load<T, NJ>(r, Fmu, mX, Fvar, n, P, var_sb, var_sp, L.C, lane);
    const int y = mc_label((double)Y[n * ldy], L.C);
    double mu_y, v_y, s_y, is_y, gs, gx;
    mc_selected(Fmu, mX, Fvar, n, P, var_sb, var_sp, y, mu_y, v_y, s_y, is_y);
    const double p = mc_prob<NJ, false>(r, y, mu_y, s_y, L.C, lane, nullptr, nullptr, gs, gx);
    if (lane == 0) s += p * L.log1m + (1.0 - p) * L.logk1;
  }
  s = block_sum_256(s, sh);
  if (threadIdx.x == 0) atomicAdd(out, scale * s);
}

// mean [N, C] = density(c) for every class c, var = mean - mean^2; inputs [N, C] contiguous
template <typename T, int NJ>
__global__ void __launch_bounds__(MC_THREADS, 1)
mc_predict_mv_kernel(McD L, const T* __restrict__ Fmu, const T* __restrict__ Fvar, int64_t N, T* __restrict__ mean,
                     T* __restrict__ var) {
  const int64_t P = L.C;
  const int lane = threadIdx.x & 31;
  for (int64_t n = mc_first_row(); n < N; n += mc_row_stride()) {
    McRow<NJ> r;
    mc_load<T, NJ>(r, Fmu, (const T*)nullptr, Fvar, n, P, P, 1, L.C, lane);
    for (int y = 0; y < L.C; ++y) {
      double mu_y, v_y, s_y, is_y, gs, gx;
      mc_selected(Fmu, (const T*)nullptr, Fvar, n, P, P, 1, y, mu_y, v_y, s_y, is_y);
      const double p = mc_prob<NJ, false>(r, y, mu_y, s_y, L.C, lane, nullptr, nullptr, gs, gx);
      if (lane == (y & 31)) {
        const double dens = fma(p, 1.0 - L.eps, (1.0 - p) * L.eps_k1);
        mean[n * P + y] = (T)dens;
        var[n * P + y] = (T)(dens - dens * dens);
      }
    }
  }
}

// out[n] = log density(y_n); inputs [N, C] contiguous, Y [N, 1]
template <typename T, int NJ>
__global__ void __launch_bounds__(MC_THREADS, 1)
mc_predict_ld_kernel(McD L, const T* __restrict__ Fmu, const T* __restrict__ Fvar, const T* __restrict__ Y, int64_t N,
                     T* __restrict__ out) {
  const int64_t P = L.C;
  const int lane = threadIdx.x & 31;
  for (int64_t n = mc_first_row(); n < N; n += mc_row_stride()) {
    McRow<NJ> r;
    mc_load<T, NJ>(r, Fmu, (const T*)nullptr, Fvar, n, P, P, 1, L.C, lane);
    const int y = mc_label((double)Y[n], L.C);
    double mu_y, v_y, s_y, is_y, gs, gx;
    mc_selected(Fmu, (const T*)nullptr, Fvar, n, P, P, 1, y, mu_y, v_y, s_y, is_y);
    const double p = mc_prob<NJ, false>(r, y, mu_y, s_y, L.C, lane, nullptr, nullptr, gs, gx);
    if (lane == 0) out[n] = (T)log(fma(p, 1.0 - L.eps, (1.0 - p) * L.eps_k1));
  }
}

// The SVGP backward's adjoints (float64), as lik_grad_kernel: fmu [B][C], fvar [C][B], labels Y[n * ldy]; R [B][C] =
// c dVE/dmu, Wt [C][B] = c dVE/dv (not written when Wt is NULL), *geps += c sum_n dVE_n/d epsilon.
template <int NJ>
__global__ void __launch_bounds__(MC_THREADS, 1)
mc_grad_kernel(McD L, const double* __restrict__ fmu, const double* __restrict__ fvar, const double* __restrict__ Y,
               const double* __restrict__ mX, int64_t B, int64_t ldy, double cs, double* __restrict__ R,
               double* __restrict__ Wt, double* __restrict__ geps) {
  __shared__ double sh[32];
  const int64_t P = L.C;
  const double kappa = L.log1m - L.logk1;
  double se = 0.0;
  const int lane = threadIdx.x & 31;
  for (int64_t n = mc_first_row(); n < B; n += mc_row_stride()) {
    McRow<NJ> r;
    mc_load<double, NJ>(r, fmu, mX, fvar, n, P, 1, B, L.C, lane);
    const int y = mc_label(Y[n * ldy], L.C);
    double mu_y, v_y, s_y, is_y, gs, gx, G[NJ], H[NJ];
    mc_selected(fmu, mX, fvar, n, P, 1, B, y, mu_y, v_y, s_y, is_y);
    const double p = mc_prob<NJ, true>(r, y, mu_y, s_y, L.C, lane, G, H, gs, gx);
    gs = warp_sum(gs);
    gx = warp_sum(gx);
#pragma unroll
    for (int j = 0; j < NJ; ++j) {
      const int c = 32 * j + lane;
      if (c < L.C && c != y) {
        R[n * P + c] = -cs * kappa * G[j];
        if (Wt) Wt[c * B + n] = r.v[j] > 1e-10 ? -0.5 * cs * kappa * H[j] * r.is[j] : 0.0;
      }
    }
    if (lane == 0) {
      if (y >= 0) {
        R[n * P + y] = cs * kappa * gs;
        if (Wt) Wt[y * B + n] = 2.0 * v_y > 1e-10 ? cs * kappa * gx * is_y : 0.0;
      }
      se += -p * L.inv1m + (1.0 - p) * L.inveps;
    }
  }
  se = block_sum_256(se, sh);
  if (threadIdx.x == 0) atomicAdd(geps, cs * se);
}

static_assert(GPK_LIK_MAX_CLASSES == 4 * 32, "the MultiClass kernels hold at most 4 chunks of 32 classes per row");
// calls F(NJ) with the chunk count of C classes as a compile-time constant
#define MC_DISPATCH(C, F)   \
  switch (((C) + 31) / 32) { \
    case 1: F(1); break;     \
    case 2: F(2); break;     \
    case 3: F(3); break;     \
    default: F(4); break;    \
  }

static unsigned lik_grid(int64_t total) {
  int64_t g = (total + 255) / 256;
  if (g < 1) g = 1;
  if (g > 2048) g = 2048;
  return (unsigned)g;
}

static unsigned mc_grid(int64_t rows) {  // one warp per row, grid-stride beyond 8192 CTAs
  int64_t g = (rows + MC_THREADS / 32 - 1) / (MC_THREADS / 32);
  if (g < 1) g = 1;
  if (g > 8192) g = 8192;
  return (unsigned)g;
}

// the MultiClass launches for a storage type T, at the chunk count of the class count
template <typename T>
static void mc_varexp_launch(const McD& M, const void* Fmu, const void* Fvar, const void* Y, const void* mX, int64_t B,
                             int64_t P, int64_t ldy, int64_t var_sb, int64_t var_sp, double scale, double* out,
                             cudaStream_t st) {
#define F(NJ)                                                                                                       \
  mc_varexp_kernel<T, NJ><<<mc_grid(B), MC_THREADS, 0, st>>>(M, (const T*)Fmu, (const T*)Fvar, (const T*)Y,          \
                                                             (const T*)mX, B, P, ldy, var_sb, var_sp, scale, out)
  MC_DISPATCH(M.C, F)
#undef F
}

template <typename T>
static void mc_predict_mv_launch(const McD& M, const void* Fmu, const void* Fvar, int64_t N, void* mean, void* var,
                                 cudaStream_t st) {
#define F(NJ) \
  mc_predict_mv_kernel<T, NJ><<<mc_grid(N), MC_THREADS, 0, st>>>(M, (const T*)Fmu, (const T*)Fvar, N, (T*)mean, (T*)var)
  MC_DISPATCH(M.C, F)
#undef F
}

template <typename T>
static void mc_predict_ld_launch(const McD& M, const void* Fmu, const void* Fvar, const void* Y, int64_t N, void* out,
                                 cudaStream_t st) {
#define F(NJ)                                                                                                   \
  mc_predict_ld_kernel<T, NJ><<<mc_grid(N), MC_THREADS, 0, st>>>(M, (const T*)Fmu, (const T*)Fvar, (const T*)Y, N, \
                                                                 (T*)out)
  MC_DISPATCH(M.C, F)
#undef F
}

int lik_varexp_impl(const gpk_lik* lik, const void* Fmu, const void* Fvar, const void* Y, const void* mX, int64_t B,
                    int64_t P, int64_t ldy, int64_t ldmx, int64_t var_sb, int64_t var_sp, double scale, int accumulate,
                    double* out, int dtype, cudaStream_t st) {
  LikD L;
  GPK_TRY(lik_prepare(lik, L, P, "lik_varexp_sum"));
  GPK_CHECK_ARG(Fmu && Fvar && Y && out, "lik_varexp_sum: null argument");
  // the MultiClass kernels read m(X) with the row stride of Fmu: all the latents of a row
  GPK_CHECK_ARG(L.type != GPK_LIK_MULTICLASS || !mX || ldmx == P, "lik_varexp_sum: MultiClass takes m(X) [B, %lld]",
                (long long)P);
  if (!accumulate) GPK_CUDA_OK(cudaMemsetAsync(out, 0, sizeof(double), st));
  const int64_t tot = B * P;
  if (tot <= 0) return 0;
  if (L.type == GPK_LIK_MULTICLASS) {
    if (dtype == GPK_F64)
      mc_varexp_launch<double>(mc_desc(lik), Fmu, Fvar, Y, mX, B, P, ldy, var_sb, var_sp, scale, out, st);
    else
      mc_varexp_launch<float>(mc_desc(lik), Fmu, Fvar, Y, mX, B, P, ldy, var_sb, var_sp, scale, out, st);
  } else if (dtype == GPK_F64) {
    lik_varexp_kernel<double><<<lik_grid(tot), 256, 0, st>>>(L, (const double*)Fmu, (const double*)Fvar,
                                                             (const double*)Y, (const double*)mX, tot, P, ldy, ldmx,
                                                             var_sb, var_sp, scale, out);
  } else {
    lik_varexp_kernel<float><<<lik_grid(tot), 256, 0, st>>>(L, (const float*)Fmu, (const float*)Fvar, (const float*)Y,
                                                            (const float*)mX, tot, P, ldy, ldmx, var_sb, var_sp, scale,
                                                            out);
  }
  GPK_LAUNCH_OK();
  return 0;
}

// Y [B, ldy]: the targets (ldy = P) of a scalar likelihood, the labels (ldy = 1) of MULTICLASS
int lik_grad_impl(const gpk_lik* lik, const double* fmu, const double* fvar, const double* Y, int64_t ldy,
                  const double* mX, int64_t B, int64_t P, double c, double* R, double* Wt, double* gpar,
                  cudaStream_t st) {
  LikD L;
  GPK_TRY(lik_prepare(lik, L, P, "lik_grad"));
  if (L.type == GPK_LIK_MULTICLASS) {
    const McD M = mc_desc(lik);
#define F(NJ) mc_grad_kernel<NJ><<<mc_grid(B), MC_THREADS, 0, st>>>(M, fmu, fvar, Y, mX, B, ldy, c, R, Wt, gpar)
    MC_DISPATCH(M.C, F)
#undef F
  } else {
    GPK_CHECK_ARG(ldy == P, "lik_grad: the targets of a scalar likelihood are [B, P] (ldy = %lld, P = %lld)",
                  (long long)ldy, (long long)P);
    lik_grad_kernel<<<lik_grid(B * P), 256, 0, st>>>(L, fmu, fvar, Y, mX, B, P, c, R, Wt, gpar);
  }
  GPK_LAUNCH_OK();
  return 0;
}

int lik_check(const gpk_lik* lik, int64_t P, const char* who) {
  LikD L;
  return lik_prepare(lik, L, P, who);
}

int lik_predict_mv_impl(const gpk_lik* lik, const void* Fmu, const void* Fvar, int64_t N, int64_t P, void* mean,
                        void* var, int dtype, cudaStream_t st) {
  LikD L;
  GPK_TRY(lik_prepare(lik, L, P, "lik_predict_mean_and_var", true));
  GPK_CHECK_ARG(Fmu && Fvar && mean && var, "lik_predict_mean_and_var: null argument");
  GPK_CHECK_ARG(L.type != GPK_LIK_STUDENT_T || L.df > 2.0,
                "lik_predict_mean_and_var: the Student-t variance needs df > 2 (df = %g)", L.df);
  const int64_t tot = N * P;
  if (tot <= 0) return 0;
  const unsigned g = (unsigned)((tot + 255) / 256);
  if (L.type == GPK_LIK_MULTICLASS) {
    if (dtype == GPK_F64)
      mc_predict_mv_launch<double>(mc_desc(lik), Fmu, Fvar, N, mean, var, st);
    else
      mc_predict_mv_launch<float>(mc_desc(lik), Fmu, Fvar, N, mean, var, st);
  } else if (dtype == GPK_F64) {
    lik_predict_mv_kernel<double><<<g, 256, 0, st>>>(L, (const double*)Fmu, (const double*)Fvar, tot, (double*)mean,
                                                     (double*)var);
  } else {
    lik_predict_mv_kernel<float><<<g, 256, 0, st>>>(L, (const float*)Fmu, (const float*)Fvar, tot, (float*)mean,
                                                    (float*)var);
  }
  GPK_LAUNCH_OK();
  return 0;
}

int lik_predict_ld_impl(const gpk_lik* lik, const void* Fmu, const void* Fvar, const void* Y, int64_t N, int64_t P,
                        void* out, int dtype, cudaStream_t st) {
  LikD L;
  GPK_TRY(lik_prepare(lik, L, P, "lik_predict_log_density", true));
  GPK_CHECK_ARG(Fmu && Fvar && Y && out, "lik_predict_log_density: null argument");
  if (N <= 0 || P <= 0) return 0;
  const unsigned g = (unsigned)((N + 255) / 256);
  if (L.type == GPK_LIK_MULTICLASS) {
    if (dtype == GPK_F64)
      mc_predict_ld_launch<double>(mc_desc(lik), Fmu, Fvar, Y, N, out, st);
    else
      mc_predict_ld_launch<float>(mc_desc(lik), Fmu, Fvar, Y, N, out, st);
  } else if (dtype == GPK_F64) {
    lik_predict_ld_kernel<double><<<g, 256, 0, st>>>(L, (const double*)Fmu, (const double*)Fvar, (const double*)Y, N,
                                                     P, (double*)out);
  } else {
    lik_predict_ld_kernel<float><<<g, 256, 0, st>>>(L, (const float*)Fmu, (const float*)Fvar, (const float*)Y, N, P,
                                                    (float*)out);
  }
  GPK_LAUNCH_OK();
  return 0;
}

}  // namespace gpk
