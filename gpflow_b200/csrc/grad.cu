// grad.cu — device backward pass of GPR.log_marginal_likelihood (SURVEY.md 8(f) rank 1).
//
// The reference gets d(LML)/d(theta) from TensorFlow autodiff through gpflow/models/gpr.py:91-107 (driven by
// gpflow/optimizers/scipy.py:78-228 via training_loss_closure, models/training_mixins.py:43-78).  Here the adjoint is
// written out:
//     dLML/dK = G = 1/2 (alpha alpha^T - P K^-1),   alpha = K^-1 (Y - m),   K = kernel(X) + sigma_n^2 I
//     dLML/dtheta = sum_ij G_ij dK_ij/dtheta ,      dLML/dsigma_n^2 = tr G
// with K^-1 = L^-T L^-1 from the factor the forward pass leaves behind:
//   1. alpha  = L^-T beta            (beta^T = the extra rows of the factorisation; one trsm)
//   2. L^-1   in place (recursive block inversion [A 0; C D]^-1 = [A^-1 0; -D^-1 C A^-1, D^-1]; the 128x128 diagonal
//             blocks are the block inverses potrf already produced; two triangular x dense GEMMs per level)
//   3. K^-1   = L^-T L^-1, lower triangle (recursive: C11 = lauum(A11) + A21^T A21, C21 = A22^T A21, C22 = lauum(A22))
//   4. one K-build-shaped pass over the lower-triangle tiles that re-evaluates k and dk/ds per element (s = scaled
//      squared distance, by direct differences), forms G_ij on the fly from alpha and K^-1, and reduces
//      sum G (.) dK/dtheta per parameter: registers -> warp shuffles -> one atomicAdd per CTA and parameter.
// Steps 2-3 run on the DMMA GEMM with the triangular operand's zero k-range skipped (GPK_GEMM_A_LOWER): 2 N^3 / 3 flops.
// gpr_grad_expr_kernel covers every expression the fused K-build compiles (compile_kprog): Sum / Product trees of
// stationary, RationalQuadratic, Linear, Polynomial, White and Constant leaves.  gpr_grad_launch runs the faster
// gpr_grad_kernel instead when the expression is a single stationary leaf (SquaredExponential, Matern12/32/52,
// Exponential) with a scalar or ARD lengthscale; both write the same slots.
#include "internal.cuh"
#include "kprog.cuh"

namespace gpk {

constexpr int GR_MAXD = 32;
struct GradKern {
  int type;            // GPK_K_RBF / MATERN12 / MATERN32 / MATERN52 / EXPONENTIAL
  int nd;              // active dims
  int ard;             // 0: scalar lengthscale (one gradient slot), 1: nd slots
  double variance;
  int dims[GR_MAXD];
  double inv_l[GR_MAXD];  // 1 / lengthscale_d
};

__device__ __forceinline__ void k_and_dkds(int type, double s, double var, double& k, double& dkds) {
  // s = scaled squared distance; k(s) and dk/ds as gpflow/kernels/stationaries.py:209-210,250-251,270-271,290-292,311-313
  // (the 1e-36 clip before the square root passes no gradient when active, like tf.maximum)
  if (type == GPK_K_RBF) {
    k = var * exp(-0.5 * s);
    dkds = -0.5 * k;
    return;
  }
  const bool clipped = !(s > 1e-36);
  const double r = sqrt(clipped ? 1e-36 : s);
  if (type == GPK_K_MATERN12) {
    k = var * exp(-r);
    dkds = clipped ? 0.0 : -k / (2.0 * r);
  } else if (type == GPK_K_EXPONENTIAL) {
    k = var * exp(-0.5 * r);
    dkds = clipped ? 0.0 : -k / (4.0 * r);
  } else if (type == GPK_K_MATERN32) {
    const double s3 = 1.7320508075688772935, e = exp(-s3 * r);
    k = var * (1.0 + s3 * r) * e;
    dkds = clipped ? 0.0 : -1.5 * var * e;
  } else {  // MATERN52
    const double s5 = 2.2360679774997896964, e = exp(-s5 * r);
    k = var * (1.0 + s5 * r + (5.0 / 3.0) * r * r) * e;
    dkds = clipped ? 0.0 : -(5.0 / 6.0) * var * (1.0 + s5 * r) * e;
  }
}

// lower-triangular tile index t -> (ti, tj), tj <= ti
__device__ __forceinline__ void tri_tile(int64_t t, int64_t& ti, int64_t& tj) {
  ti = (int64_t)((sqrt(8.0 * (double)t + 1.0) - 1.0) * 0.5);
  while (ti * (ti + 1) / 2 > t) --ti;
  while ((ti + 1) * (ti + 2) / 2 <= t) ++ti;
  tj = t - ti * (ti + 1) / 2;
}

constexpr int GT = 64;  // tile edge

// gout: [0] d/dnoise_variance, [1] d/dvariance, [2 ...] d/dlengthscale (1 slot, or nd slots with ARD): the slots
// build_gradprog assigns to a single stationary leaf
template <int ND>
__global__ void __launch_bounds__(256)
gpr_grad_kernel(GradKern gk, const double* __restrict__ X, int64_t N, int64_t ldx, const double* __restrict__ alpha,
                int P, const double* __restrict__ Kinv, int64_t ldk, double* __restrict__ gout) {
  __shared__ double xa[GT][ND + 1], xb[GT][ND + 1];
  __shared__ double red[8][ND + 2];
  int64_t ti, tj;
  tri_tile(blockIdx.x, ti, tj);
  const int tid = threadIdx.x, tr = tid >> 4, tc = tid & 15;
  const int nd = gk.nd;
  for (int e = tid; e < GT * ND; e += 256) {
    const int r = e / ND, d = e % ND;
    const int64_t ra = ti * GT + r, rb = tj * GT + r;
    const double sc = d < nd ? gk.inv_l[d] : 0.0;
    const int col = d < nd ? gk.dims[d] : 0;
    xa[r][d] = (ra < N && d < nd) ? X[ra * ldx + col] * sc : 0.0;
    xb[r][d] = (rb < N && d < nd) ? X[rb * ldx + col] * sc : 0.0;
  }
  __syncthreads();
  double gv = 0.0, gn = 0.0, gl[ND];
#pragma unroll
  for (int d = 0; d < ND; ++d) gl[d] = 0.0;
  double gls = 0.0;
#pragma unroll 1
  for (int a = 0; a < 4; ++a) {
    const int r = tr + 16 * a;
    const int64_t i = ti * GT + r;
#pragma unroll 1
    for (int b = 0; b < 4; ++b) {
      const int c = tc + 16 * b;
      const int64_t j = tj * GT + c;
      if (i >= N || j > i) continue;
      double s = 0.0;
#pragma unroll
      for (int d = 0; d < ND; ++d) {
        const double df = xa[r][d] - xb[c][d];
        s = fma(df, df, s);
      }
      double k, dkds;
      k_and_dkds(gk.type, s, gk.variance, k, dkds);
      double aa = 0.0;
      for (int p = 0; p < P; ++p) aa = fma(alpha[i * P + p], alpha[j * P + p], aa);
      const double G = 0.5 * (aa - (double)P * Kinv[i * ldk + j]);
      const double Ge = i == j ? G : 2.0 * G;  // the strict lower part stands for both (i,j) and (j,i)
      gv = fma(Ge, k, gv);
      if (i == j) gn += G;
      const double w = Ge * dkds * -2.0;
      if (gk.ard) {
#pragma unroll
        for (int d = 0; d < ND; ++d) {
          const double df = xa[r][d] - xb[c][d];
          gl[d] = fma(w, df * df, gl[d]);   // ds/dl_d = -2 diff_d^2 / l_d^3; the 1/l_d factor is applied at the end
        }
      } else {
        gls = fma(w, s, gls);               // ds/dl = -2 s / l
      }
    }
  }
  // CTA reduction: shuffles, then one atomicAdd per parameter
  const int lane = tid & 31, wp = tid >> 5;
  gv = warp_sum(gv);
  gn = warp_sum(gn);
  gls = warp_sum(gls);
#pragma unroll
  for (int d = 0; d < ND; ++d) gl[d] = warp_sum(gl[d]);
  if (lane == 0) {
    red[wp][0] = gv;
    red[wp][1] = gn;
#pragma unroll
    for (int d = 0; d < ND; ++d) red[wp][2 + d] = gk.ard ? gl[d] : (d == 0 ? gls : 0.0);
  }
  __syncthreads();
  if (tid < ND + 2) {
    double v = 0.0;
    for (int w2 = 0; w2 < 8; ++w2) v += red[w2][tid];
    if (tid == 0) atomicAdd(gout + 1, v / gk.variance);
    else if (tid == 1) atomicAdd(gout + 0, v);
    else {
      const int d = tid - 2;
      if (gk.ard) { if (d < nd) atomicAdd(gout + 2 + d, v * gk.inv_l[d]); }
      else if (d == 0) atomicAdd(gout + 2, v * gk.inv_l[0]);
    }
  }
}

// ---- any fused expression ------------------------------------------------------------------------------------
// Output slots (gout[1 ...], gout[0] is d/dnoise_variance): leaves in node-array order; per leaf the gradients w.r.t.
// the constrained values: stationary: variance, lengthscale(s) [, RQ alpha]; Linear: variance(s); Polynomial:
// variance(s), offset; White / Constant: variance.  Per element each leaf's value is re-evaluated (stationary s by
// direct differences, Linear / Polynomial dot products directly), its adjoint d root / d leaf comes from a forward
// dual-number pass over the postfix program (the root is multilinear in the leaf values: every leaf occurs once, so
// nothing is ever divided by a leaf value), and G_ij adjoint dleaf/dtheta is accumulated per slot.
constexpr int GR_MAXA = 32;             // per-dimension (ARD) slots
constexpr int GR_MAXS = 3 * KB_MAXL;    // scalar slots: at most variance, lengthscale / offset, alpha per leaf
constexpr int GE = 32;                  // tile edge
constexpr int GE_THREADS = 128;         // 8 elements per thread

struct GradProg {
  int n_groups, n_cols, n_leaves, n_ops, n_s, n_a;
  int g_lo[KB_MAXG], g_hi[KB_MAXG];     // staged-column range of each gram group
  int col[GR_MAXD];                     // X column of each staged column
  int c_group[GR_MAXD];                 // gram group of each staged column
  double ws[GR_MAXD], wl[GR_MAXD];      // staged value = X * ws (both sides); dot product weight wl (A side)
  int l_type[KB_MAXL], l_group[KB_MAXL];
  double l_var[KB_MAXL], l_scale[KB_MAXL], l_alpha[KB_MAXL];
  int l_s0[KB_MAXL], l_s1[KB_MAXL], l_a0[KB_MAXL], l_a1[KB_MAXL];  // the leaf's ranges in the scalar / ARD slot lists
  int s_kind[GR_MAXS], s_out[GR_MAXS];  // kind 0: variance, 1: lengthscale or Polynomial offset, 2: RQ alpha
  double s_fac[GR_MAXS];                // applied to the CTA sum (1 / variance, -2 / lengthscale, 1)
  int a_col[GR_MAXA], a_out[GR_MAXA];
  double a_fac[GR_MAXA];
  unsigned char ops[KB_MAXOPS];
};

static bool linear_like_op(int t) { return t == GPK_K_LINEAR || t == GPK_K_POLYNOMIAL; }

// Flattened expression (compile_kprog) -> staging plan and slot lists; *n_slots = leaf slots (outputs after noise).
static int build_gradprog(const gpk_knode* nodes, int n_nodes, const int32_t* dims, const double* ard, int64_t D,
                          GradProg& gp, int* n_slots, const char* who = "gpr_lml_grad_expr") {
  KProg p;
  GPK_TRY(compile_kprog(nodes, n_nodes, dims, ard, D, p));
  memset(&gp, 0, sizeof(gp));
  gp.n_groups = p.n_groups;
  gp.n_leaves = p.n_leaves;
  gp.n_ops = p.n_ops;
  memcpy(gp.ops, p.ops, sizeof(gp.ops));
  int tot = 0;
  for (int g = 0; g < p.n_groups; ++g) tot = p.g_off[g] + p.g_ndims[g] > tot ? p.g_off[g] + p.g_ndims[g] : tot;
  GPK_CHECK_ARG(tot <= GR_MAXD, "%s: the expression stages %d active columns, at most %d", who, tot, GR_MAXD);
  gp.n_cols = tot;
  for (int g = 0; g < p.n_groups; ++g) {
    gp.g_lo[g] = p.g_off[g];
    gp.g_hi[g] = p.g_off[g] + p.g_ndims[g];
    for (int d = gp.g_lo[g]; d < gp.g_hi[g]; ++d) {
      gp.col[d] = p.dims[d];
      gp.c_group[d] = g;
      gp.ws[d] = p.g_weighted[g] == 2 ? p.w[d] : 1.0;
      gp.wl[d] = p.g_weighted[g] == 1 ? p.w[d] : 1.0;
    }
  }
  int slot = 1;  // gout[0] is the noise variance
  auto scalar = [&](int kind, double fac) -> int {
    GPK_CHECK_ARG(gp.n_s < GR_MAXS, "%s: more than %d scalar gradient slots", who, GR_MAXS);
    gp.s_kind[gp.n_s] = kind;
    gp.s_out[gp.n_s] = slot++;
    gp.s_fac[gp.n_s++] = fac;
    return 0;
  };
  auto per_dim = [&](int g, bool stationary) -> int {
    for (int d = gp.g_lo[g]; d < gp.g_hi[g]; ++d) {
      GPK_CHECK_ARG(gp.n_a < GR_MAXA, "%s: more than %d per-dimension gradient slots", who, GR_MAXA);
      gp.a_col[gp.n_a] = d;
      gp.a_out[gp.n_a] = slot++;
      gp.a_fac[gp.n_a++] = stationary ? -2.0 * p.w[d] : 1.0;  // ds/dl_d = -2 diff_d^2 / l_d, diff_d scaled by 1/l_d
    }
    return 0;
  };
  for (int l = 0; l < p.n_leaves; ++l) {
    const int t = p.l_type[l], g = p.l_group[l];
    const bool ard = g >= 0 && p.g_weighted[g] != 0;
    gp.l_type[l] = t;
    gp.l_group[l] = g;
    gp.l_var[l] = p.l_var[l];
    gp.l_scale[l] = p.l_scale[l];
    gp.l_alpha[l] = p.l_alpha[l];
    gp.l_s0[l] = gp.n_s;
    gp.l_a0[l] = gp.n_a;
    if (kprog_stationary(t)) {
      GPK_TRY(scalar(0, p.l_var[l] != 0.0 ? 1.0 / p.l_var[l] : 0.0));
      if (ard) GPK_TRY(per_dim(g, true));
      else GPK_TRY(scalar(1, -2.0 / p.l_len[l]));
      if (t == GPK_K_RQ) GPK_TRY(scalar(2, 1.0));
    } else if (linear_like_op(t)) {
      if (ard) GPK_TRY(per_dim(g, false));
      else GPK_TRY(scalar(0, 1.0));
      if (t == GPK_K_POLYNOMIAL) GPK_TRY(scalar(1, 1.0));
    } else {  // White, Constant
      GPK_TRY(scalar(0, 1.0));
    }
    gp.l_s1[l] = gp.n_s;
    gp.l_a1[l] = gp.n_a;
  }
  *n_slots = slot - 1;
  return 0;
}

__device__ __forceinline__ double sel4(const double (&v)[KB_MAXG], int g) {
  double r = 0.0;
#pragma unroll
  for (int k = 0; k < KB_MAXG; ++k)
    if (g == k) r = v[k];
  return r;
}

// d root / d leaf l at this thread's element: forward dual numbers (value, derivative) through the postfix program,
// seeded 1 at leaf l.  Sum passes the adjoint through, Product multiplies it by the siblings' product.
__device__ __forceinline__ double leaf_adjoint(const GradProg& gp, int l, const double (*sv)[GE_THREADS], int tid) {
  double v0 = 0.0, v1 = 0.0, v2 = 0.0, v3 = 0.0, d0 = 0.0, d1 = 0.0, d2 = 0.0, d3 = 0.0;
  for (int o = 0; o < gp.n_ops; ++o) {
    const int op = gp.ops[o];
    if (op < KB_MAXL) {
      v3 = v2; v2 = v1; v1 = v0; v0 = sv[op][tid];
      d3 = d2; d2 = d1; d1 = d0; d0 = op == l ? 1.0 : 0.0;
    } else {
      if (op == KB_OP_ADD) {
        d0 = d1 + d0;
        v0 = v1 + v0;
      } else {
        d0 = fma(d1, v0, v1 * d0);
        v0 = v1 * v0;
      }
      v1 = v2; v2 = v3; d1 = d2; d2 = d3;
    }
  }
  return d0;
}

// The per-element leaf engine shared by the GPR reduction and the three SGPR passes.  Element k(xr, xc) of the
// expression, xr / xc the staged (scaled) columns of its two points, weighted by Ge = d objective / d element: every
// leaf's value and derivative factor into sv / sd (this thread's column), then per leaf w = Ge x its adjoint, and
// w x d leaf / d theta accumulated into the slot registers.  With DZ, also the per-group factors of
// d element / d (first point): zs[g] multiplies 2 (xr_d - xc_d), zl[g] multiplies wl_d xc_d (then ws_d, the staging
// scale, turns a staged-column derivative into one w.r.t. the raw column).
template <int NS, int NA, bool DZ>
__device__ __forceinline__ void leaf_element(const GradProg& gp, const double* xr, const double* xc, bool diag,
                                             double Ge, double (*sv)[GE_THREADS], double (*sd)[GE_THREADS], int tid,
                                             double* gs, double* ga, double* zs, double* zl) {
  const int nl = gp.n_leaves;
  // per gram group: squared distance of the staged (scaled) columns and the weighted dot product
  double qs[KB_MAXG], ps[KB_MAXG];
#pragma unroll
  for (int g = 0; g < KB_MAXG; ++g) {
    double q = 0.0, pd = 0.0;
    if (g < gp.n_groups) {
      for (int d = gp.g_lo[g]; d < gp.g_hi[g]; ++d) {
        const double xv = xr[d], yv = xc[d], df = xv - yv;
        q = fma(df, df, q);
        pd = fma(gp.wl[d] * xv, yv, pd);
      }
    }
    qs[g] = q;
    ps[g] = pd;
  }
  // leaf values and derivative factors
  for (int l = 0; l < nl; ++l) {
    const int type = gp.l_type[l], g = gp.l_group[l];
    const double var = gp.l_var[l];
    double v, dv = 0.0;
    if (type == GPK_K_RQ) {
      const double al = gp.l_alpha[l], u = gp.l_scale[l] * sel4(qs, g) / (2.0 * al);
      v = var * pow(1.0 + u, -al);
      dv = -0.5 * v / (1.0 + u);
    } else if (kprog_stationary(type)) {
      k_and_dkds(type, gp.l_scale[l] * sel4(qs, g), var, v, dv);
    } else if (type == GPK_K_LINEAR) {
      v = var * sel4(ps, g);
    } else if (type == GPK_K_POLYNOMIAL) {
      const double deg = gp.l_alpha[l], base = fma(var, sel4(ps, g), gp.l_scale[l]);
      v = pow(base, deg);
      dv = deg * pow(base, deg - 1.0);
    } else if (type == GPK_K_WHITE) {
      v = diag ? var : 0.0;
    } else {  // Constant
      v = var;
    }
    sv[l][tid] = v;
    sd[l][tid] = dv;
  }
  for (int l = 0; l < nl; ++l) {
    const double w = Ge * leaf_adjoint(gp, l, sv, tid);
    const int type = gp.l_type[l], g = gp.l_group[l];
    const double v = sv[l][tid], dv = sd[l][tid];
    double c0, c1 = 0.0, c2 = 0.0, ca;  // d leaf / d (variance, lengthscale or offset, alpha), per-dim factor
    if (kprog_stationary(type)) {
      const double s = gp.l_scale[l] * sel4(qs, g);
      c0 = v;       // times 1 / variance at the end
      c1 = dv * s;  // times -2 / lengthscale at the end
      ca = dv;      // times diff_d^2 (scaled), then -2 / l_d at the end
      if (type == GPK_K_RQ) {
        const double u = s / (2.0 * gp.l_alpha[l]);
        c2 = v * (u / (1.0 + u) - log1p(u));
      }
    } else if (type == GPK_K_LINEAR) {
      c0 = sel4(ps, g);
      ca = 1.0;     // times x_d x'_d
    } else if (type == GPK_K_POLYNOMIAL) {
      c0 = dv * sel4(ps, g);
      c1 = dv;
      ca = dv;
    } else {
      c0 = type == GPK_K_WHITE ? (diag ? 1.0 : 0.0) : 1.0;
      ca = 0.0;
    }
    const int s0 = gp.l_s0[l], s1 = gp.l_s1[l], a0 = gp.l_a0[l], a1 = gp.l_a1[l];
#pragma unroll
    for (int q = 0; q < NS; ++q)
      if (q >= s0 && q < s1) {
        const int k = gp.s_kind[q];
        gs[q] = fma(w, k == 0 ? c0 : (k == 1 ? c1 : c2), gs[q]);
      }
    if (NA > 0 && a1 > a0) {
      const double wa = w * ca;
      const bool stat = kprog_stationary(type);
#pragma unroll
      for (int q = 0; q < NA; ++q)
        if (q >= a0 && q < a1) {
          const int d = gp.a_col[q];
          const double xv = xr[d], yv = xc[d], df = xv - yv;
          ga[q] = fma(wa, stat ? df * df : xv * yv, ga[q]);
        }
    }
    if (DZ) {
      // d s / d xr_d = l_scale 2 (xr_d - xc_d);  d (x.x') / d xr_d = wl_d xc_d;  White and Constant: 0
      const double fz = kprog_stationary(type) ? w * dv * gp.l_scale[l]
                        : type == GPK_K_LINEAR   ? w * gp.l_var[l]
                        : type == GPK_K_POLYNOMIAL ? w * dv * gp.l_var[l]
                                                   : 0.0;
      const bool stat = kprog_stationary(type);
#pragma unroll
      for (int k = 0; k < KB_MAXG; ++k)
        if (k == g) {
          if (stat) zs[k] += fz;
          else zl[k] += fz;
        }
    }
  }
}

// The staged columns of the points Pt[r0 .. r0 + GE) (Pt [n, ldp] row-major): s[r][d] = Pt[r0 + r, col[d]] * ws[d],
// zero past row n; with s2, those of Pt[r2 .. r2 + GE) into s2 in the same pass (two independent loads per step).
__device__ __forceinline__ void stage_rows(const GradProg& gp, const double* __restrict__ Pt, int64_t n, int64_t ldp,
                                           int tid, int64_t r0, double (*s)[GR_MAXD + 1], int64_t r2 = 0,
                                           double (*s2)[GR_MAXD + 1] = nullptr) {
  const int nc = gp.n_cols;
  for (int e = tid; e < GE * nc; e += GE_THREADS) {
    const int r = e / nc, d = e % nc;
    const int64_t row = r0 + r, row2 = r2 + r;
    s[r][d] = row < n ? Pt[row * ldp + gp.col[d]] * gp.ws[d] : 0.0;
    if (s2) s2[r][d] = row2 < n ? Pt[row2 * ldp + gp.col[d]] * gp.ws[d] : 0.0;
  }
}

// CTA reduction of the slot registers: shuffles, then red[] (one row per warp), then one thread and one atomicAdd per
// CTA and slot, scaled by s_fac / a_fac.  With NOISE, the last column of red[] carries gn into gout[0].
template <int NS, int NA, bool NOISE>
__device__ __forceinline__ void reduce_slots(const GradProg& gp, double* gs, double* ga, double gn,
                                             double (*red)[NS + NA + NOISE], int tid, double* __restrict__ gout) {
  const int lane = tid & 31, wp = tid >> 5;
  if (NOISE) gn = warp_sum(gn);
#pragma unroll
  for (int q = 0; q < NS; ++q) gs[q] = warp_sum(gs[q]);
#pragma unroll
  for (int q = 0; q < NA; ++q) ga[q] = warp_sum(ga[q]);
  if (lane == 0) {
#pragma unroll
    for (int q = 0; q < NS; ++q) red[wp][q] = gs[q];
#pragma unroll
    for (int q = 0; q < NA; ++q) red[wp][NS + q] = ga[q];
    if (NOISE) red[wp][NS + NA] = gn;
  }
  __syncthreads();
  static_assert(NS + NA + NOISE <= GE_THREADS, "one thread per slot");
  const int k = tid;
  if (k < NS + NA + NOISE) {
    double v = 0.0;
#pragma unroll
    for (int w2 = 0; w2 < GE_THREADS / 32; ++w2) v += red[w2][k];
    if (k < NS) { if (k < gp.n_s) atomicAdd(gout + gp.s_out[k], v * gp.s_fac[k]); }
    else if (k < NS + NA) { if (k - NS < gp.n_a) atomicAdd(gout + gp.a_out[k - NS], v * gp.a_fac[k - NS]); }
    else atomicAdd(gout, v);
  }
}

template <int NS, int NA>
__global__ void __launch_bounds__(GE_THREADS)
gpr_grad_expr_kernel(const __grid_constant__ GradProg gp, const double* __restrict__ X, int64_t N, int64_t ldx,
                     const double* __restrict__ alpha, int P, const double* __restrict__ Kinv, int64_t ldk,
                     double* __restrict__ gout) {
  __shared__ double xa[GE][GR_MAXD + 1], xb[GE][GR_MAXD + 1];
  __shared__ double sv[KB_MAXL][GE_THREADS];  // leaf values of this thread's current element
  __shared__ double sd[KB_MAXL][GE_THREADS];  // their derivative factors (dk/ds, Polynomial d/d(base))
  __shared__ double red[GE_THREADS / 32][NS + NA + 1];
  int64_t ti, tj;
  tri_tile(blockIdx.x, ti, tj);
  const int tid = threadIdx.x, tr = tid >> 4, tc = tid & 15;
  stage_rows(gp, X, N, ldx, tid, ti * GE, xa, tj * GE, xb);
  __syncthreads();
  double gs[NS > 0 ? NS : 1], ga[NA > 0 ? NA : 1], gn = 0.0;
#pragma unroll
  for (int q = 0; q < NS; ++q) gs[q] = 0.0;
#pragma unroll
  for (int q = 0; q < NA; ++q) ga[q] = 0.0;
#pragma unroll 1
  for (int a = 0; a < GE / 8; ++a) {
    const int r = tr + 8 * a;
    const int64_t i = ti * GE + r;
#pragma unroll 1
    for (int b = 0; b < GE / 16; ++b) {
      const int c = tc + 16 * b;
      const int64_t j = tj * GE + c;
      if (i >= N || j > i) continue;
      const bool diag = i == j;
      double aa = 0.0;
      for (int p = 0; p < P; ++p) aa = fma(alpha[i * P + p], alpha[j * P + p], aa);
      const double G = 0.5 * (aa - (double)P * Kinv[i * ldk + j]);
      const double Ge = diag ? G : 2.0 * G;  // the strict lower part stands for both (i,j) and (j,i)
      if (diag) gn += G;
      leaf_element<NS, NA, false>(gp, xa[r], xb[c], diag, Ge, sv, sd, tid, gs, ga, nullptr, nullptr);
    }
  }
  reduce_slots<NS, NA, true>(gp, gs, ga, gn, red, tid, gout);
}

// ---- SGPR / SVGP: the three element sources of an inducing-point objective -------------------------------------
// dF/dtheta = sum_mn G_uf[m,n] dKuf_mn/dtheta + sum_ij G_uu[i,j] dKuu_ij/dtheta + g_d sum_n dKdiag_n/dtheta (SGPR's
// collapsed bound g_d = -P/(2s), SVGP's ELBO g_d = P w), each
// through leaf_element.  A CTA owns 32 rows of the A side (Z; X for the diagonal) and a range of 32-column tiles of the
// B side (X for Kuf, Z for Kuu); thread t owns row t / 4 and the columns t % 4 + 4 b, so its d element / d z_row
// accumulates in registers (dz[ND]) across the whole range and leaves the CTA in one atomicAdd per (row, column).
enum { SG_KUF = 0, SG_KUU = 1, SG_KDIAG = 2 };
struct SgprPass {
  int mode;
  const double* A; int64_t nA, lda;    // row points (Z, or X for the diagonal)
  const double* B; int64_t nB, ldb;    // column points (X for Kuf, Z for Kuu)
  const double* G; int64_t ldg;        // element weights (Kuf, Kuu); the diagonal's is gvec[i], or the constant gconst
  double gconst;                       // when gvec is NULL
  const double* gvec;
  int64_t tiles;                       // column tiles per CTA
  double zfac;                         // Kuf 1, Kuu 2 (G_uu symmetric: both arguments' derivatives of the square)
  double* dZ; int64_t D;               // [nA, D] row-major (Kuf / Kuu)
};

// SH: dz lives in dynamic shared memory (one column of ND per thread) instead of registers, for the instantiation
// whose slot registers leave no room for it.
template <int NS, int NA, int ND, bool SH>
__global__ void __launch_bounds__(GE_THREADS, NS + NA + ND <= 40 ? 3 : 1)
sgpr_grad_kernel(const __grid_constant__ GradProg gp, const SgprPass sp, double* __restrict__ gout) {
  extern __shared__ double dzs[];
  __shared__ double xa[GE][GR_MAXD + 1], xb[GE][GR_MAXD + 1];
  __shared__ double sv[KB_MAXL][GE_THREADS];
  __shared__ double sd[KB_MAXL][GE_THREADS];
  __shared__ double red[GE_THREADS / 32][NS + NA];
  const int tid = threadIdx.x, r = tid >> 2, tc = tid & 3;
  const int nc = gp.n_cols;
  const int64_t ti = blockIdx.x, i = ti * GE + r;
  stage_rows(gp, sp.A, sp.nA, sp.lda, tid, ti * GE, xa);
  double gs[NS > 0 ? NS : 1], ga[NA > 0 ? NA : 1], dzr[SH ? 1 : ND];
  auto dz = [&](int d) -> double& { return SH ? dzs[d * GE_THREADS + tid] : dzr[SH ? 0 : d]; };
#pragma unroll
  for (int q = 0; q < NS; ++q) gs[q] = 0.0;
#pragma unroll
  for (int q = 0; q < NA; ++q) ga[q] = 0.0;
#pragma unroll
  for (int d = 0; d < ND; ++d) dz(d) = 0.0;
  const int64_t ntb = (sp.nB + GE - 1) / GE;
  const int64_t t0 = sp.mode == SG_KDIAG ? ti : (int64_t)blockIdx.y * sp.tiles;
  const int64_t t1 = sp.mode == SG_KDIAG ? ti + 1 : (t0 + sp.tiles < ntb ? t0 + sp.tiles : ntb);
#pragma unroll 1
  for (int64_t tj = t0; tj < t1; ++tj) {
    __syncthreads();  // the previous tile's columns are no longer read
    stage_rows(gp, sp.B, sp.nB, sp.ldb, tid, tj * GE, xb);
    __syncthreads();
    if (i >= sp.nA) continue;
#pragma unroll 1
    for (int b = 0; b < GE / 4; ++b) {
      const int c = tc + 4 * b;
      const int64_t j = tj * GE + c;
      if (j >= sp.nB) break;
      if (sp.mode == SG_KDIAG && c != r) continue;
      const bool diag = sp.mode == SG_KDIAG || (sp.mode == SG_KUU && i == j);
      const double Ge = sp.mode == SG_KDIAG ? (sp.gvec ? sp.gvec[i] : sp.gconst) : sp.G[i * sp.ldg + j];
      double zs[KB_MAXG] = {0.0, 0.0, 0.0, 0.0}, zl[KB_MAXG] = {0.0, 0.0, 0.0, 0.0};
      leaf_element<NS, NA, true>(gp, xa[r], xb[c], diag, Ge, sv, sd, tid, gs, ga, zs, zl);
      if (sp.mode == SG_KDIAG) continue;
      if (gp.n_groups == 1) {
        const double z2 = 2.0 * zs[0], z1 = zl[0];
#pragma unroll
        for (int d = 0; d < ND; ++d)
          if (d < nc) dz(d) = fma(z2, xa[r][d] - xb[c][d], fma(z1 * gp.wl[d], xb[c][d], dz(d)));
      } else {
#pragma unroll
        for (int d = 0; d < ND; ++d)
          if (d < nc) {
            const int g = gp.c_group[d];
            dz(d) = fma(2.0 * sel4(zs, g), xa[r][d] - xb[c][d], fma(sel4(zl, g) * gp.wl[d], xb[c][d], dz(d)));
          }
      }
    }
  }
  // dZ: the four threads of a row, then one row of staged columns per row in shared memory (xb is free)
  __syncthreads();
#pragma unroll
  for (int d = 0; d < ND; ++d) {
    double v = dz(d);
    v += __shfl_xor_sync(0xffffffffu, v, 1);
    v += __shfl_xor_sync(0xffffffffu, v, 2);
    if (tc == 0 && d < nc) xb[r][d] = v * gp.ws[d] * sp.zfac;
  }
  reduce_slots<NS, NA, false>(gp, gs, ga, 0.0, red, tid, gout);  // its barrier also completes the rows of xb
  if (sp.mode == SG_KDIAG) return;
  // a column staged by several groups collects them all in its first staging: one atomicAdd per (row, column)
  for (int e = tid; e < GE * nc; e += GE_THREADS) {
    const int rr = e / nc, d = e % nc;
    const int64_t row = ti * GE + rr;
    const int col = gp.col[d];
    bool first = true;
    for (int d2 = 0; d2 < d; ++d2) first = first && gp.col[d2] != col;
    if (row >= sp.nA || !first) continue;
    double v = xb[rr][d];
    for (int d2 = d + 1; d2 < nc; ++d2)
      if (gp.col[d2] == col) v += xb[rr][d2];
    atomicAdd(sp.dZ + row * sp.D + col, v);
  }
}

// The number of leaf slots of an expression, or -1 with an error message under the caller's name `who`.
int grad_expr_slots(const gpk_knode* nodes, int n_nodes, const int32_t* dims, const double* ard, int64_t D,
                    const char* who) {
  GradProg gp;
  int n = 0;
  GPK_TRY(build_gradprog(nodes, n_nodes, dims, ard, D, gp, &n, who));
  return n;
}

// sum G (.) dK/dtheta, G = 1/2 (alpha alpha^T - P K^-1), into gout[0] (d/dnoise_variance) and the leaf slots
// gout[1 ...].  A single stationary leaf runs gpr_grad_kernel (about twice as fast on C2), every other expression
// gpr_grad_expr_kernel.
int gpr_grad_launch(const gpk_knode* nodes, int n_nodes, const int32_t* dims, const double* ard, const double* X,
                    int64_t N, int64_t ldx, int64_t D, const double* alpha, int P, const double* Kinv, int64_t ldk,
                    double* gout, cudaStream_t st) {
  GradProg gp;
  int n = 0;
  GPK_TRY(build_gradprog(nodes, n_nodes, dims, ard, D, gp, &n));
  const gpk_knode& nd = nodes[0];
  if (n_nodes == 1 && (nd.op == GPK_K_RBF || nd.op == GPK_K_MATERN12 || nd.op == GPK_K_MATERN32 ||
                       nd.op == GPK_K_MATERN52 || nd.op == GPK_K_EXPONENTIAL)) {
    GradKern gk;
    memset(&gk, 0, sizeof(gk));
    gk.type = nd.op;
    gk.variance = nd.variance;
    gk.nd = gp.n_cols;  // the leaf's active dims (at most GR_MAXD: build_gradprog)
    gk.ard = nd.n_ard > 0 ? 1 : 0;
    for (int d = 0; d < gk.nd; ++d) {
      gk.dims[d] = nd.n_dims > 0 ? dims[nd.dims_off + d] : d;
      gk.inv_l[d] = 1.0 / (nd.n_ard > 0 ? ard[nd.ard_off + d] : nd.lengthscale);
    }
    const int64_t nt = (N + GT - 1) / GT;
    const unsigned grid = (unsigned)(nt * (nt + 1) / 2);
    ProfScope ps(PROF_KBUILD, st);
    if (gk.nd <= 8) gpr_grad_kernel<8><<<grid, 256, 0, st>>>(gk, X, N, ldx, alpha, P, Kinv, ldk, gout);
    else if (gk.nd <= 16) gpr_grad_kernel<16><<<grid, 256, 0, st>>>(gk, X, N, ldx, alpha, P, Kinv, ldk, gout);
    else gpr_grad_kernel<32><<<grid, 256, 0, st>>>(gk, X, N, ldx, alpha, P, Kinv, ldk, gout);
    GPK_LAUNCH_OK();
    return 0;
  }
  const int64_t nt = (N + GE - 1) / GE;
  const unsigned grid = (unsigned)(nt * (nt + 1) / 2);
  ProfScope ps(PROF_KBUILD, st);
#define GPK_GE_GO(NS, NA) \
  gpr_grad_expr_kernel<NS, NA><<<grid, GE_THREADS, 0, st>>>(gp, X, N, ldx, alpha, P, Kinv, ldk, gout)
  if (gp.n_a == 0) {
    if (gp.n_s <= 8) GPK_GE_GO(8, 0);
    else if (gp.n_s <= 16) GPK_GE_GO(16, 0);
    else GPK_GE_GO(GR_MAXS, 0);
  } else {
    if (gp.n_s <= 8) GPK_GE_GO(8, GR_MAXA);
    else if (gp.n_s <= 16) GPK_GE_GO(16, GR_MAXA);
    else GPK_GE_GO(GR_MAXS, GR_MAXA);
  }
#undef GPK_GE_GO
  GPK_LAUNCH_OK();
  return 0;
}

// The dynamic shared memory of the instantiation that keeps dz there, granted once; -1 with an error under `who`.
static int dz_smem_bytes(const char* who) {
  const int dz_smem = GR_MAXD * GE_THREADS * (int)sizeof(double);
  static const bool dz_smem_ok = cudaFuncSetAttribute(sgpr_grad_kernel<GR_MAXS, GR_MAXA, GR_MAXD, true>,
                                                      cudaFuncAttributeMaxDynamicSharedMemorySize, dz_smem) ==
                                 cudaSuccess;
  GPK_CHECK_ARG(dz_smem_ok, "%s: %d bytes of dynamic shared memory refused", who, dz_smem);
  return dz_smem;
}

// One element pass of sgpr_grad_kernel on `grid`, the instantiation chosen by the expression's slot and column counts.
static int inducing_pass(const GradProg& gp, const SgprPass& sp, dim3 grid, int dz_smem, double* gout,
                         cudaStream_t st) {
#define GPK_SG_GO(NS, NA, ND, SH) \
  sgpr_grad_kernel<NS, NA, ND, SH><<<grid, GE_THREADS, SH ? dz_smem : 0, st>>>(gp, sp, gout)
  if (gp.n_a == 0) {
    if (gp.n_s <= 8) { if (gp.n_cols <= 16) GPK_SG_GO(8, 0, 16, false); else GPK_SG_GO(8, 0, GR_MAXD, false); }
    else if (gp.n_s <= 16) GPK_SG_GO(16, 0, GR_MAXD, false);
    else GPK_SG_GO(GR_MAXS, 0, GR_MAXD, false);
  } else {
    if (gp.n_s <= 8) GPK_SG_GO(8, GR_MAXA, GR_MAXD, false);
    else if (gp.n_s <= 16) GPK_SG_GO(16, GR_MAXA, GR_MAXD, false);
    else GPK_SG_GO(GR_MAXS, GR_MAXA, GR_MAXD, true);
  }
#undef GPK_SG_GO
  GPK_LAUNCH_OK();
  return 0;
}

// The three passes of an inducing-point objective (Kuf, Kuu, Kdiag) into the leaf slots gout[1 ...] (gout[0], the
// noise, is not touched) and dZ [M, D] (zeroed by the caller): G_uf [M, ldgf] = dF/dKuf, G_uu [M, ldgu] = dF/dKuu full
// and symmetric, and the weight of every diagonal element of K(X, X): the constant kdiag_weight (SGPR -P / (2 s), SVGP
// P w), or per element kdiag_vec [N] when it is not NULL (SVGP with a non-Gaussian likelihood: sum_p W[n, p]).  `who`
// names the caller in error messages.
int inducing_grad_launch(const gpk_knode* nodes, int n_nodes, const int32_t* dims, const double* ard, const double* X,
                         int64_t N, int64_t ldx, int64_t D, const double* Z, int64_t M, int64_t ldz, const double* Guf,
                         int64_t ldgf, const double* Guu, int64_t ldgu, double kdiag_weight, const double* kdiag_vec,
                         double* gout, double* dZ, const char* who, cudaStream_t st) {
  GradProg gp;
  int n = 0;
  GPK_TRY(build_gradprog(nodes, n_nodes, dims, ard, D, gp, &n, who));
  const int64_t tm = (M + GE - 1) / GE, tn = (N + GE - 1) / GE;
  // Kuf: about 2048 CTAs, each a strip of 32 Z rows x `tiles` column tiles of X
  const int64_t ych = tn < (2048 + tm - 1) / tm ? tn : (2048 + tm - 1) / tm;
  SgprPass pass[3];
  pass[0] = SgprPass{SG_KUF, Z, M, ldz, X, N, ldx, Guf, ldgf, 0.0, nullptr, (tn + ych - 1) / ych, 1.0, dZ, D};
  pass[1] = SgprPass{SG_KUU, Z, M, ldz, Z, M, ldz, Guu, ldgu, 0.0, nullptr, 1, 2.0, dZ, D};
  pass[2] = SgprPass{SG_KDIAG, X, N, ldx, X, N, ldx, nullptr, 0, kdiag_weight, kdiag_vec, 1, 0.0, nullptr, D};
  const dim3 grids[3] = {dim3((unsigned)tm, (unsigned)((tn + pass[0].tiles - 1) / pass[0].tiles)),
                         dim3((unsigned)tm, (unsigned)tm), dim3((unsigned)tn, 1)};
  const int dz_smem = dz_smem_bytes(who);
  if (dz_smem < 0) return dz_smem;
  ProfScope ps(PROF_KBUILD, st);
  for (int k = 0; k < 3; ++k) GPK_TRY(inducing_pass(gp, pass[k], grids[k], dz_smem, gout, st));
  return 0;
}

// The square pass alone, over K(X, X): sum_ij G[i,j] dK_ij/dtheta on the full N x N square, the diagonal included (so
// White counts), into the leaf slots gout[1 ...] (gout[0] is not touched).  G [N, ldg] full and symmetric.  The pass
// also accumulates its input derivative into dz_scratch [N, D], which the caller discards (VGP's objective has no
// inducing points).
int square_grad_launch(const gpk_knode* nodes, int n_nodes, const int32_t* dims, const double* ard, const double* X,
                       int64_t N, int64_t ldx, int64_t D, const double* G, int64_t ldg, double* gout,
                       double* dz_scratch, const char* who, cudaStream_t st) {
  GradProg gp;
  int n = 0;
  GPK_TRY(build_gradprog(nodes, n_nodes, dims, ard, D, gp, &n, who));
  const int64_t tn = (N + GE - 1) / GE;
  const SgprPass pass{SG_KUU, X, N, ldx, X, N, ldx, G, ldg, 0.0, nullptr, 1, 2.0, dz_scratch, D};
  const int dz_smem = dz_smem_bytes(who);
  if (dz_smem < 0) return dz_smem;
  ProfScope ps(PROF_KBUILD, st);
  return inducing_pass(gp, pass, dim3((unsigned)tn, (unsigned)tn), dz_smem, gout, st);
}

// ---- L^-1 in place (lower), diagonal 128-blocks taken from the block inverses of the factorisation ------------
__global__ void put_dinv_kernel(double* __restrict__ L, int64_t ldl, int64_t n, const double* __restrict__ dinv) {
  const int64_t b0 = (int64_t)blockIdx.x * NB;
  const double* src = dinv + (size_t)blockIdx.x * NB * NB;
  for (int e = threadIdx.x; e < NB * NB; e += blockDim.x) {
    const int r = e / NB, c = e % NB;
    // the strict upper part of the block is zeroed: lauum reads the block as a dense operand, and the workspace above
    // the diagonal tiles of the K-build is uninitialised (0 x NaN)
    if (b0 + r < n && b0 + c < n) L[(b0 + r) * ldl + b0 + c] = c <= r ? src[r * NB + c] : 0.0;
  }
}

static inline int64_t split128(int64_t n) { return ((n / NB + 1) / 2) * NB; }

static int trtri_rec(double* L, int64_t n, int64_t ldl, double* tmp, cudaStream_t st) {
  if (n <= NB) return 0;  // diagonal blocks are already inverses
  const int64_t n1 = split128(n), n2 = n - n1;
  GPK_TRY(trtri_rec(L, n1, ldl, tmp, st));
  GPK_TRY(trtri_rec(L + n1 * ldl + n1, n2, ldl, tmp, st));
  double* L21 = L + n1 * ldl;
  double* A22 = L + n1 * ldl + n1;
  // Tt [n1, n2] = L11inv^T L21^T   (= (L21 L11inv)^T), the zero k-range of the triangular operand skipped
  GPK_TRY(gemm_t<double>(1, 1, n1, n2, n1, 1.0, L, ldl, L21, ldl, 0.0, tmp, n2, GPK_GEMM_A_LOWER, st));
  // L21 <- - L22inv (Tt)^T
  GPK_TRY(gemm_t<double>(0, 1, n2, n1, n2, -1.0, A22, ldl, tmp, n2, 0.0, L21, ldl, GPK_GEMM_A_LOWER, st));
  return 0;
}

// C (lower) = A^T A for lower-triangular A, out of place
static int lauum_rec(const double* A, int64_t n, int64_t lda, double* C, int64_t ldc, cudaStream_t st) {
  if (n <= NB)
    return gemm_t<double>(1, 0, n, n, n, 1.0, A, lda, A, lda, 0.0, C, ldc, GPK_GEMM_A_LOWER | GPK_GEMM_LOWER_ONLY, st);
  const int64_t n1 = split128(n), n2 = n - n1;
  const double* A21 = A + n1 * lda;
  const double* A22 = A + n1 * lda + n1;
  GPK_TRY(lauum_rec(A, n1, lda, C, ldc, st));
  GPK_TRY(lauum_rec(A22, n2, lda, C + n1 * ldc + n1, ldc, st));
  GPK_TRY(gemm_t<double>(1, 0, n1, n1, n2, 1.0, A21, lda, A21, lda, 1.0, C, ldc, GPK_GEMM_LOWER_ONLY, st));
  GPK_TRY(gemm_t<double>(1, 0, n2, n1, n2, 1.0, A22, lda, A21, lda, 0.0, C + n1 * ldc, ldc, GPK_GEMM_A_LOWER, st));
  return 0;
}

// K^-1 (lower triangle) from the factor L and its block inverses; L is overwritten by L^-1.
// tmp: (n/2 + 128)^2 doubles.
int potri_lower(double* L, int64_t n, int64_t ldl, const double* dinv, double* Kinv, int64_t ldk, double* tmp,
                cudaStream_t st) {
  const unsigned nblk = (unsigned)((n + NB - 1) / NB);
  put_dinv_kernel<<<nblk, 256, 0, st>>>(L, ldl, n, dinv);
  GPK_LAUNCH_OK();
  GPK_TRY(trtri_rec(L, n, ldl, tmp, st));
  return lauum_rec(L, n, ldl, Kinv, ldk, st);
}

// C (lower triangle) = A^T A for lower-triangular A [n, lda] whose strict upper part is zero; C out of place.
int lauum_lower(const double* A, int64_t n, int64_t lda, double* C, int64_t ldc, cudaStream_t st) {
  return lauum_rec(A, n, lda, C, ldc, st);
}

}  // namespace gpk
