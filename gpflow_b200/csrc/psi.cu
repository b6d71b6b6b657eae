// psi.cu — the RBF kernel expectations under a diagonal Gaussian q(x) = N(mu, diag S) (the psi statistics of the
// Bayesian GPLVM, gpflow/expectations/squared_exponentials.py:49-96, 207-292) and their adjoints, float64.
// With sigma^2 the kernel variance, l_d the lengthscales of the leaf's active dims and zbar = (z_m + z_m') / 2:
//   psi1[n,m]  = sigma^2 exp(-u1),  u1 = 1/2 sum_d log(1 + S_nd/l_d^2) + 1/2 sum_d (mu_nd - z_md)^2 / (l_d^2 + S_nd)
//   psi2[m,m'] = sum_n sigma^4 exp(-u2),
//                u2 = sum_d (z_md - z_m'd)^2 / (4 l_d^2) + 1/2 sum_d log(1 + 2 S_nd/l_d^2)
//                     + sum_d (mu_nd - zbar_d)^2 / (l_d^2 + 2 S_nd)
// Both exponents are >= 0 and go through the table-driven exp of the K-build fast path (fastexp.cuh), four at a time.
// The per-point factors (the two log-determinants and 1/(l^2 + S), 1/(l^2 + 2S)) are computed once per point by
// psi_prep_kernel.
//
// psi2 and its adjoint are the O(N M^2 Q) part.  The forward (and the Z side of the adjoint) gives each thread PP pairs
// (m >= m') of the lower triangle and walks a chunk of the points staged in shared memory; the grid splits over the
// points when M is small and the chunks are summed in a fixed order by psi2_reduce_kernel (deterministic).  The point
// side of the adjoint (d/dmu, d/dS) gives each thread one point and walks a chunk of the pairs staged in shared memory,
// so that every accumulator has a single owner and no reduction runs inside the loops.
#include "fastexp.cuh"
#include "internal.cuh"

using namespace gpk;

namespace gpk {

int exp2_table_device(const double** tab);

constexpr int PS_MAXD = 32;   // active latent dims (the limit of the Kuu gradient pass, GR_MAXD)
constexpr int PS_T = 256;     // threads of the pair-owner kernels
constexpr int PS_NB = 32;     // points staged per block
constexpr int PS_PT = 128;    // threads of the point-owner kernels
constexpr int PS_PB = 64;     // pairs staged per block

struct PsiK {
  int nd;                 // active dims
  int col[PS_MAXD];       // latent column of each active dim
  double l2[PS_MAXD];     // lengthscale^2
  double var;             // sigma^2
};

// One SquaredExponential leaf over Q latent columns (all, or its active_dims); -1 and gpk_last_error otherwise.
static int psi_kernel_of(const gpk_knode* nodes, int n_nodes, const int32_t* dims, const double* ard, int64_t Q,
                         PsiK& k, const char* who) {
  GPK_CHECK_ARG(nodes && n_nodes == 1 && nodes[0].op == GPK_K_RBF,
                "%s: the psi statistics cover one SquaredExponential leaf", who);
  const gpk_knode& nd = nodes[0];
  k.nd = nd.n_dims > 0 ? nd.n_dims : (int)Q;
  GPK_CHECK_ARG(k.nd > 0 && k.nd <= PS_MAXD, "%s: %d active latent dims, at most %d", who, k.nd, PS_MAXD);
  GPK_CHECK_ARG(nd.n_ard == 0 || nd.n_ard == k.nd, "%s: %d ARD lengthscales for %d active dims", who, nd.n_ard, k.nd);
  k.var = nd.variance;
  for (int d = 0; d < k.nd; ++d) {
    k.col[d] = nd.n_dims > 0 ? dims[nd.dims_off + d] : d;
    GPK_CHECK_ARG(k.col[d] >= 0 && k.col[d] < Q, "%s: active dim %d outside the %lld latent columns", who, k.col[d],
                  (long long)Q);
    const double l = nd.n_ard > 0 ? ard[nd.ard_off + d] : nd.lengthscale;
    GPK_CHECK_ARG(l > 0.0, "%s: lengthscales must be positive", who);
    k.l2[d] = l * l;
  }
  GPK_CHECK_ARG(k.var > 0.0, "%s: the kernel variance must be positive", who);
  return 0;
}

// ---- per-point factors ---------------------------------------------------------------------------------------
// mua [N, nd]: mu on the active dims; a1, b2 [N, nd]: 1/(l^2 + S), 1/(l^2 + 2S); cc [N, 2]: the two exponent shifts
// 1/2 sum log(1 + S/l^2), 1/2 sum log(1 + 2S/l^2)
__global__ void psi_prep_kernel(const PsiK k, const double* __restrict__ mu, const double* __restrict__ S, int64_t N,
                                int64_t Q, double* __restrict__ mua, double* __restrict__ a1, double* __restrict__ b2,
                                double* __restrict__ cc) {
  const int64_t n = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (n >= N) return;
  double c1 = 0.0, c2 = 0.0;
  for (int d = 0; d < k.nd; ++d) {
    const double s = S[n * Q + k.col[d]];
    mua[n * k.nd + d] = mu[n * Q + k.col[d]];
    a1[n * k.nd + d] = 1.0 / (k.l2[d] + s);
    b2[n * k.nd + d] = 1.0 / (k.l2[d] + 2.0 * s);
    c1 += log1p(s / k.l2[d]);
    c2 += log1p(2.0 * s / k.l2[d]);
  }
  cc[2 * n] = 0.5 * c1;
  cc[2 * n + 1] = 0.5 * c2;
}

__device__ __forceinline__ void exp_neg4(const double (&u)[4], const double* __restrict__ tab, double (&e)[4]) {
  stationary_value4<GPK_K_RBF>(u, 1.0, 0.0, true, tab, e);  // exp(-u), u >= 0 (the table holds 2^(j/64) unscaled)
}

__device__ __forceinline__ void load_tab(double* s_tab, const double* __restrict__ tab) {
  if (threadIdx.x < 64) s_tab[threadIdx.x] = tab[threadIdx.x];
}

// ---- psi1 ----------------------------------------------------------------------------------------------------
// P1[n * sn + m * sm] = psi1[n, m]; thread: one m (blockIdx.y), four consecutive points
__global__ void __launch_bounds__(128) psi1_kernel(const PsiK k, const double* __restrict__ mua,
                                                   const double* __restrict__ a1, const double* __restrict__ cc,
                                                   int64_t N, const double* __restrict__ Z, int64_t ldz,
                                                   double* __restrict__ P1, int64_t sn, int64_t sm,
                                                   const double* __restrict__ tab) {
  __shared__ double s_tab[64], zs[PS_MAXD];
  load_tab(s_tab, tab);
  const int64_t m = blockIdx.y;
  if (threadIdx.x < k.nd) zs[threadIdx.x] = Z[m * ldz + k.col[threadIdx.x]];
  __syncthreads();
  const int64_t n0 = 4 * ((int64_t)blockIdx.x * blockDim.x + threadIdx.x);
  if (n0 >= N) return;
  double u[4], e[4];
#pragma unroll
  for (int t = 0; t < 4; ++t) {
    const int64_t n = n0 + t < N ? n0 + t : N - 1;
    double acc = 0.0;
    for (int d = 0; d < k.nd; ++d) {
      const double df = mua[n * k.nd + d] - zs[d];
      acc = fma(df * df, a1[n * k.nd + d], acc);
    }
    u[t] = fma(0.5, acc, cc[2 * n]);
  }
  exp_neg4(u, s_tab, e);
#pragma unroll
  for (int t = 0; t < 4; ++t)
    if (n0 + t < N) P1[(n0 + t) * sn + m * sm] = k.var * e[t];
}

// Block sum of v over the CTA into *dst (atomic, one per CTA); red: blockDim.x / 32 doubles of shared memory.
__device__ __forceinline__ void block_add(double v, double* red, double* dst) {
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  const int warp = threadIdx.x >> 5, nw = blockDim.x >> 5;
  __syncthreads();
  if ((threadIdx.x & 31) == 0) red[warp] = v;
  __syncthreads();
  if (threadIdx.x == 0) {
    double s = 0.0;
    for (int w = 0; w < nw; ++w) s += red[w];
    atomicAdd(dst, s);
  }
}

// psi1 adjoint, point side: e = G1[n,m] psi1[n,m] (G1t[m * ldg + n] = dF/dpsi1[n,m]);
//   dmu_nd += -a sum_m e diff,  dS_nd += 1/2 a^2 sum_m e diff^2 - 1/2 a sum_m e,  diff = mu_nd - z_md, a = 1/(l^2 + S)
//   dl_d   += sum_n [l a^2 sum_m e diff^2 + S a sum_m e / l],  dsigma^2 += sum e / sigma^2   (gpar[0], gpar[1 + d])
template <int ND>
__global__ void __launch_bounds__(PS_PT) psi1_bwd_point_kernel(const PsiK k, const double* __restrict__ mua,
                                                               const double* __restrict__ a1,
                                                               const double* __restrict__ cc, const double* __restrict__ S,
                                                               int64_t N, int64_t Q, const double* __restrict__ Z,
                                                               int64_t ldz, int64_t M, const double* __restrict__ G1t,
                                                               int64_t ldg, double* __restrict__ dmu,
                                                               double* __restrict__ dS, double* __restrict__ gpar,
                                                               const double* __restrict__ tab) {
  __shared__ double s_tab[64], red[PS_PT / 32];
  load_tab(s_tab, tab);
  __syncthreads();
  const int64_t n = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const bool live = n < N;
  const int64_t nn = live ? n : N - 1;
  double mu[ND], a[ND], A1[ND], A2[ND], E = 0.0;
#pragma unroll
  for (int d = 0; d < ND; ++d) {
    mu[d] = d < k.nd ? mua[nn * k.nd + d] : 0.0;
    a[d] = d < k.nd ? a1[nn * k.nd + d] : 0.0;
    A1[d] = 0.0;
    A2[d] = 0.0;
  }
  const double c = cc[2 * nn];
  for (int64_t m0 = 0; m0 < M; m0 += 4) {
    double u[4], e[4];
#pragma unroll
    for (int t = 0; t < 4; ++t) {
      const int64_t m = m0 + t < M ? m0 + t : M - 1;
      double acc = 0.0;
#pragma unroll
      for (int d = 0; d < ND; ++d) {
        const double df = mu[d] - (d < k.nd ? Z[m * ldz + k.col[d]] : 0.0);
        acc = fma(df * df, a[d], acc);
      }
      u[t] = fma(0.5, acc, c);
    }
    exp_neg4(u, s_tab, e);
#pragma unroll
    for (int t = 0; t < 4; ++t) {
      if (m0 + t >= M) break;
      const int64_t m = m0 + t;
      const double w = G1t[m * ldg + nn] * k.var * e[t];
      E += w;
#pragma unroll
      for (int d = 0; d < ND; ++d) {
        const double df = mu[d] - (d < k.nd ? Z[m * ldz + k.col[d]] : 0.0);
        A1[d] = fma(w, df, A1[d]);
        A2[d] = fma(w * df, df, A2[d]);
      }
    }
  }
#pragma unroll
  for (int d = 0; d < ND; ++d) {
    if (d >= k.nd) break;  // uniform over the CTA (block_add synchronises)
    const double s = S[nn * Q + k.col[d]], l = sqrt(k.l2[d]);
    if (live) {
      dmu[nn * Q + k.col[d]] += -a[d] * A1[d];
      dS[nn * Q + k.col[d]] += 0.5 * a[d] * a[d] * A2[d] - 0.5 * a[d] * E;
    }
    block_add(live ? l * a[d] * a[d] * A2[d] + s * a[d] * E / l : 0.0, red, gpar + 1 + d);
  }
  block_add(live ? E / k.var : 0.0, red, gpar);
}

// psi1 adjoint, inducing side: dZ_md += sum_n e a diff (one CTA per m, its threads over the points)
template <int ND>
__global__ void __launch_bounds__(PS_PT) psi1_bwd_z_kernel(const PsiK k, const double* __restrict__ mua,
                                                           const double* __restrict__ a1, const double* __restrict__ cc,
                                                           int64_t N, int64_t Q, const double* __restrict__ Z,
                                                           int64_t ldz, const double* __restrict__ G1t, int64_t ldg,
                                                           double* __restrict__ dZ, const double* __restrict__ tab) {
  __shared__ double s_tab[64], zs[PS_MAXD], red[PS_PT / 32];
  load_tab(s_tab, tab);
  const int64_t m = blockIdx.x;
  if (threadIdx.x < k.nd) zs[threadIdx.x] = Z[m * ldz + k.col[threadIdx.x]];
  __syncthreads();
  double B[ND];
#pragma unroll
  for (int d = 0; d < ND; ++d) B[d] = 0.0;
  for (int64_t n0 = 4 * (int64_t)threadIdx.x; n0 < N; n0 += 4 * PS_PT) {
    double u[4], e[4];
#pragma unroll
    for (int t = 0; t < 4; ++t) {
      const int64_t n = n0 + t < N ? n0 + t : N - 1;
      double acc = 0.0;
      for (int d = 0; d < k.nd; ++d) {
        const double df = mua[n * k.nd + d] - zs[d];
        acc = fma(df * df, a1[n * k.nd + d], acc);
      }
      u[t] = fma(0.5, acc, cc[2 * n]);
    }
    exp_neg4(u, s_tab, e);
#pragma unroll
    for (int t = 0; t < 4; ++t) {
      if (n0 + t >= N) break;
      const int64_t n = n0 + t;
      const double w = G1t[m * ldg + n] * k.var * e[t];
#pragma unroll
      for (int d = 0; d < ND; ++d)
        if (d < k.nd) B[d] = fma(w * a1[n * k.nd + d], mua[n * k.nd + d] - zs[d], B[d]);
    }
  }
#pragma unroll
  for (int d = 0; d < ND; ++d)
    if (d < k.nd) block_add(B[d], red, dZ + m * Q + k.col[d]);
}

// ---- psi2 ----------------------------------------------------------------------------------------------------
__device__ __forceinline__ void pair_of(int64_t p, int64_t& i, int64_t& j) {  // p = i (i + 1) / 2 + j, j <= i
  i = (int64_t)((sqrt(8.0 * (double)p + 1.0) - 1.0) * 0.5);
  while (i * (i + 1) / 2 > p) --i;
  while ((i + 1) * (i + 2) / 2 <= p) ++i;
  j = p - i * (i + 1) / 2;
}

// Pair owner: thread holds PP pairs and walks the points [n_lo, n_hi) of its chunk (blockIdx.y), NN = 4 / PP points
// per step so that every exp_neg4 call carries four exponents.
//   forward (BWD false): part[chunk * npairs + p] = sum_n exp(-u2)     (sigma^4 applied by psi2_reduce_kernel)
//   adjoint (BWD true):  with e = w_p sigma^4 exp(-u2), w_p = G2[i,j] (twice off the diagonal), diff = mu - zbar:
//     dZ_i += -E (z_i - z_j) / (2 l^2) + sum_n e diff b,  dZ_j += E (z_i - z_j) / (2 l^2) + sum_n e diff b,
//     dl_d += E (z_id - z_jd)^2 / (2 l^3),  dsigma^2 += 2 E / sigma^2,   E = sum_n e, b = 1/(l^2 + 2S)
//   The adjoint accumulates the dims [D0, D0 + DA) only (dsigma^2 with D0 = 0): at ND = 32 two launches of 16 dims keep
//   zbar and the accumulators in registers, where one launch of 32 would not fit.
template <int ND, int PP, bool BWD, int D0 = 0, int DA = ND>
__global__ void __launch_bounds__(PS_T) psi2_pair_kernel(const PsiK k, const double* __restrict__ mua,
                                                         const double* __restrict__ b2, const double* __restrict__ cc,
                                                         int64_t N, int64_t nlen, int64_t Q,
                                                         const double* __restrict__ Z, int64_t ldz, int64_t npairs,
                                                         double* __restrict__ part, const double* __restrict__ G2,
                                                         int64_t ldg, double* __restrict__ dZ,
                                                         double* __restrict__ gpar, const double* __restrict__ tab) {
  constexpr int NN = 4 / PP;
  __shared__ double s_tab[64], smu[PS_NB][ND], sb[PS_NB][ND], sc[PS_NB], red[PS_T / 32];
  load_tab(s_tab, tab);
  const int64_t n_lo = (int64_t)blockIdx.y * nlen, n_hi = n_lo + nlen < N ? n_lo + nlen : N;
  int64_t pi[PP], pj[PP];
  double zb[PP][ND], ez[PP], acc[PP], w[PP];
  double bacc[BWD ? PP : 1][DA];
#pragma unroll
  for (int q = 0; q < PP; ++q) {
    const int64_t p = ((int64_t)blockIdx.x * PP + q) * PS_T + threadIdx.x;
    pair_of(p < npairs ? p : npairs - 1, pi[q], pj[q]);
    ez[q] = 0.0;
    acc[q] = 0.0;
#pragma unroll
    for (int d = 0; d < ND; ++d) {
      const double zi = d < k.nd ? Z[pi[q] * ldz + k.col[d]] : 0.0, zj = d < k.nd ? Z[pj[q] * ldz + k.col[d]] : 0.0;
      zb[q][d] = 0.5 * (zi + zj);
      if (d < k.nd) ez[q] = fma((zi - zj) * (zi - zj), 0.25 / k.l2[d], ez[q]);
    }
#pragma unroll
    for (int j = 0; j < DA; ++j) bacc[q][j] = 0.0;
    w[q] = BWD && p < npairs ? G2[pi[q] * ldg + pj[q]] * (pi[q] == pj[q] ? 1.0 : 2.0) * k.var * k.var : 0.0;
  }
  for (int64_t s0 = n_lo; s0 < n_hi; s0 += PS_NB) {
    const int cnt = (int)(n_hi - s0 < PS_NB ? n_hi - s0 : PS_NB);
    __syncthreads();
    for (int x = threadIdx.x; x < PS_NB * ND; x += PS_T) {
      const int r = x / ND, d = x % ND;
      const bool ok = r < cnt && d < k.nd;
      smu[r][d] = ok ? mua[(s0 + r) * k.nd + d] : 0.0;
      sb[r][d] = ok ? b2[(s0 + r) * k.nd + d] : 0.0;
    }
    if (threadIdx.x < PS_NB) sc[threadIdx.x] = (int)threadIdx.x < cnt ? cc[2 * (s0 + threadIdx.x) + 1] : 0.0;
    __syncthreads();
    for (int r0 = 0; r0 < cnt; r0 += NN) {
      double u[4], e[4];
#pragma unroll
      for (int q = 0; q < PP; ++q)
#pragma unroll
        for (int t = 0; t < NN; ++t) {
          const int r = r0 + t;
          double a = ez[q] + sc[r];
#pragma unroll
          for (int d = 0; d < ND; ++d) {
            const double df = smu[r][d] - zb[q][d];
            a = fma(df * df, sb[r][d], a);
          }
          u[q * NN + t] = a;
        }
      exp_neg4(u, s_tab, e);
#pragma unroll
      for (int q = 0; q < PP; ++q)
#pragma unroll
        for (int t = 0; t < NN; ++t) {
          const int r = r0 + t;
          if (r >= cnt) continue;
          if (!BWD) {
            acc[q] += e[q * NN + t];
          } else {
            const double ew = w[q] * e[q * NN + t];
            acc[q] += ew;
#pragma unroll
            for (int j = 0; j < DA; ++j)
              bacc[q][j] = fma(ew * sb[r][D0 + j], smu[r][D0 + j] - zb[q][D0 + j], bacc[q][j]);
          }
        }
    }
  }
  if (!BWD) {
#pragma unroll
    for (int q = 0; q < PP; ++q) {
      const int64_t p = ((int64_t)blockIdx.x * PP + q) * PS_T + threadIdx.x;
      if (p < npairs) part[(int64_t)blockIdx.y * npairs + p] = acc[q];
    }
    return;
  }
  double dl[DA], E = 0.0;
#pragma unroll
  for (int j = 0; j < DA; ++j) dl[j] = 0.0;
#pragma unroll
  for (int q = 0; q < PP; ++q) {
    const int64_t p = ((int64_t)blockIdx.x * PP + q) * PS_T + threadIdx.x;
    if (p >= npairs) continue;
    E += acc[q];
#pragma unroll
    for (int j = 0; j < DA; ++j) {
      const int d = D0 + j;
      if (d >= k.nd) continue;
      const double dz = Z[pi[q] * ldz + k.col[d]] - Z[pj[q] * ldz + k.col[d]];
      const double t = acc[q] * dz * (0.5 / k.l2[d]);
      atomicAdd(dZ + pi[q] * Q + k.col[d], bacc[q][j] - t);
      atomicAdd(dZ + pj[q] * Q + k.col[d], bacc[q][j] + t);
      dl[j] = fma(acc[q] * dz * dz, 0.5 / (k.l2[d] * sqrt(k.l2[d])), dl[j]);
    }
  }
#pragma unroll
  for (int j = 0; j < DA; ++j)
    if (D0 + j < k.nd) block_add(dl[j], red, gpar + 1 + D0 + j);
  if (D0 == 0) block_add(2.0 * E / k.var, red, gpar);
}

// Psi2 [M, ld] (full, symmetric) = sigma^4 sum over the chunks of part, in chunk order.
__global__ void psi2_reduce_kernel(const double* __restrict__ part, int64_t npairs, int nchunks, double var2,
                                   double* __restrict__ P2, int64_t ld) {
  const int64_t p = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= npairs) return;
  double s = 0.0;
  for (int c = 0; c < nchunks; ++c) s += part[(int64_t)c * npairs + p];
  int64_t i, j;
  pair_of(p, i, j);
  P2[i * ld + j] = var2 * s;
  P2[j * ld + i] = var2 * s;
}

// Point owner of the psi2 adjoint: thread holds one point and walks a chunk of pairs (blockIdx.y) staged as
// (zbar, the pair's exponent shift, its weight w_p sigma^4).  With e, diff, b as psi2_pair_kernel:
//   dmu_nd += -2 b sum_p e diff,  dS_nd += -b E + 2 b^2 sum_p e diff^2,
//   dl_d += 2 l b^2 sum_p e diff^2 + 2 S b E / l
// for the dims [D0, D0 + DA) (two launches of 16 at ND = 32, as psi2_pair_kernel).
template <int ND, int D0 = 0, int DA = ND>
__global__ void __launch_bounds__(PS_PT) psi2_point_kernel(const PsiK k, const double* __restrict__ mua,
                                                           const double* __restrict__ b2,
                                                           const double* __restrict__ cc, const double* __restrict__ S,
                                                           int64_t N, int64_t Q, const double* __restrict__ Z,
                                                           int64_t ldz, int64_t npairs, int64_t plen,
                                                           const double* __restrict__ G2, int64_t ldg,
                                                           double* __restrict__ dmu, double* __restrict__ dS,
                                                           double* __restrict__ gpar, const double* __restrict__ tab) {
  __shared__ double s_tab[64], szb[PS_PB][ND], sez[PS_PB], sw[PS_PB], red[PS_PT / 32];
  load_tab(s_tab, tab);
  const int64_t n = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const bool live = n < N;
  const int64_t nn = live ? n : N - 1;
  double mu[ND], b[ND], A1[DA], A2[DA], E = 0.0;
#pragma unroll
  for (int d = 0; d < ND; ++d) {
    mu[d] = d < k.nd ? mua[nn * k.nd + d] : 0.0;
    b[d] = d < k.nd ? b2[nn * k.nd + d] : 0.0;
  }
#pragma unroll
  for (int j = 0; j < DA; ++j) {
    A1[j] = 0.0;
    A2[j] = 0.0;
  }
  const double c = cc[2 * nn + 1];
  const int64_t p_lo = (int64_t)blockIdx.y * plen, p_hi = p_lo + plen < npairs ? p_lo + plen : npairs;
  for (int64_t s0 = p_lo; s0 < p_hi; s0 += PS_PB) {
    __syncthreads();
    for (int r = threadIdx.x; r < PS_PB; r += PS_PT) {
      const int64_t p = s0 + r;
      double ez = 0.0, w = 0.0;
      int64_t i = 0, j = 0;
      if (p < p_hi) {
        pair_of(p, i, j);
        w = G2[i * ldg + j] * (i == j ? 1.0 : 2.0) * k.var * k.var;
      }
      for (int d = 0; d < ND; ++d) {
        const double zi = d < k.nd ? Z[i * ldz + k.col[d]] : 0.0, zj = d < k.nd ? Z[j * ldz + k.col[d]] : 0.0;
        szb[r][d] = 0.5 * (zi + zj);
        if (d < k.nd) ez = fma((zi - zj) * (zi - zj), 0.25 / k.l2[d], ez);
      }
      sez[r] = ez;
      sw[r] = w;  // 0 past the chunk: the padded pairs add nothing
    }
    __syncthreads();
    for (int r0 = 0; r0 < PS_PB; r0 += 4) {
      double u[4], e[4];
#pragma unroll
      for (int t = 0; t < 4; ++t) {
        double a = sez[r0 + t] + c;
#pragma unroll
        for (int d = 0; d < ND; ++d) {
          const double df = mu[d] - szb[r0 + t][d];
          a = fma(df * df, b[d], a);
        }
        u[t] = a;
      }
      exp_neg4(u, s_tab, e);
#pragma unroll
      for (int t = 0; t < 4; ++t) {
        const double ew = sw[r0 + t] * e[t];
        E += ew;
#pragma unroll
        for (int j = 0; j < DA; ++j) {
          const double df = mu[D0 + j] - szb[r0 + t][D0 + j];
          A1[j] = fma(ew, df, A1[j]);
          A2[j] = fma(ew * df, df, A2[j]);
        }
      }
    }
  }
#pragma unroll
  for (int j = 0; j < DA; ++j) {
    const int d = D0 + j;
    if (d >= k.nd) break;  // uniform over the CTA (block_add synchronises)
    const double s = S[nn * Q + k.col[d]], l = sqrt(k.l2[d]);
    if (live) {
      atomicAdd(dmu + nn * Q + k.col[d], -2.0 * b[d] * A1[j]);
      atomicAdd(dS + nn * Q + k.col[d], -b[d] * E + 2.0 * b[d] * b[d] * A2[j]);
    }
    block_add(live ? 2.0 * l * b[d] * b[d] * A2[j] + 2.0 * s * b[d] * E / l : 0.0, red, gpar + 1 + d);
  }
}

// ---- host ----------------------------------------------------------------------------------------------------
struct PsiWs {
  double *mua, *a1, *b2, *cc, *part; size_t bytes;
};

static int psi2_chunks(int64_t N, int64_t tiles, int64_t* nlen) {
  // about 8 CTAs per SM of 132 over pair tiles x point chunks, at least PS_NB points per chunk
  int64_t ch = (1056 + tiles - 1) / tiles;
  const int64_t most = (N + PS_NB - 1) / PS_NB;
  ch = ch < 1 ? 1 : (ch > most ? most : ch);
  int64_t len = (N + ch - 1) / ch;
  len = (len + PS_NB - 1) / PS_NB * PS_NB;
  *nlen = len;
  return (int)((N + len - 1) / len);
}
static int pp_of(int nd) { return nd <= 8 ? 4 : (nd <= 16 ? 2 : 1); }
static int64_t npairs_of(int64_t M) { return M * (M + 1) / 2; }
static int64_t pair_tiles(int64_t M, int nd) { return (npairs_of(M) + (int64_t)PS_T * pp_of(nd) - 1) / ((int64_t)PS_T * pp_of(nd)); }

static PsiWs psi_layout(void* ws, int64_t N, int64_t M, int nd) {
  char* base = (char*)ws;
  size_t off = 0;
  auto take = [&](size_t bytes) -> double* {
    double* r = base ? (double*)(base + off) : nullptr;
    off += align_up(bytes, 256);
    return r;
  };
  PsiWs w;
  w.mua = take((size_t)N * nd * 8);
  w.a1 = take((size_t)N * nd * 8);
  w.b2 = take((size_t)N * nd * 8);
  w.cc = take((size_t)N * 2 * 8);
  int64_t nlen;
  const int nch = psi2_chunks(N, pair_tiles(M, nd), &nlen);
  w.part = take((size_t)nch * npairs_of(M) * 8);
  w.bytes = off;
  return w;
}

// Workspace of psi_forward / psi_backward for any number of active dims up to PS_MAXD.  The per-point arrays grow with
// nd but the chunk buffer of psi2 grows as nd shrinks (more pairs per thread: fewer pair tiles, more point chunks), so
// the size is the largest layout over the three kernel buckets; each bucket's layout is largest at its top nd.
size_t psi_ws_bytes(int64_t N, int64_t M) {
  size_t b = 0;
  for (int nd : {8, 16, PS_MAXD}) {
    const size_t x = psi_layout(nullptr, N, M, nd).bytes;
    b = x > b ? x : b;
  }
  return b;
}

static int psi_setup(const gpk_knode* nodes, int n_nodes, const int32_t* dims, const double* ard, const double* mu,
                     const double* S, int64_t N, int64_t Q, int64_t M, void* ws, PsiK& k, PsiWs& w,
                     const double** tab, const char* who, cudaStream_t st) {
  GPK_TRY(psi_kernel_of(nodes, n_nodes, dims, ard, Q, k, who));
  GPK_CHECK_ARG(M <= 65535, "%s: at most 65535 inducing points (M = %lld)", who, (long long)M);
  w = psi_layout(ws, N, M, k.nd);
  GPK_CHECK_ARG(w.bytes <= psi_ws_bytes(N, M), "%s: psi workspace layout of %zu bytes exceeds psi_ws_bytes (%zu)", who,
                w.bytes, psi_ws_bytes(N, M));
  GPK_TRY(exp2_table_device(tab));
  psi_prep_kernel<<<(unsigned)((N + 127) / 128), 128, 0, st>>>(k, mu, S, N, Q, w.mua, w.a1, w.b2, w.cc);
  GPK_LAUNCH_OK();
  return 0;
}

// psi1 into P1 (P1[n * sn + m * sm]) and psi2 into P2 [M, ldp2] (full); mu, S [N, Q] and Z [M, ldz] row-major.
int psi_forward(const gpk_knode* nodes, int n_nodes, const int32_t* dims, const double* ard, const double* mu,
                const double* S, int64_t N, int64_t Q, const double* Z, int64_t M, int64_t ldz, double* P1, int64_t sn,
                int64_t sm, double* P2, int64_t ldp2, void* ws, const char* who, cudaStream_t st) {
  PsiK k;
  PsiWs w;
  const double* tab = nullptr;
  GPK_TRY(psi_setup(nodes, n_nodes, dims, ard, mu, S, N, Q, M, ws, k, w, &tab, who, st));
  ProfScope ps(PROF_LEAF, st);
  const dim3 g1((unsigned)((N + 4 * 128 - 1) / (4 * 128)), (unsigned)M);
  psi1_kernel<<<g1, 128, 0, st>>>(k, w.mua, w.a1, w.cc, N, Z, ldz, P1, sn, sm, tab);
  GPK_LAUNCH_OK();
  const int64_t np = npairs_of(M), tiles = pair_tiles(M, k.nd);
  int64_t nlen;
  const int nch = psi2_chunks(N, tiles, &nlen);
  const dim3 g2((unsigned)tiles, (unsigned)nch);
#define GPK_P2F(ND, PP) \
  psi2_pair_kernel<ND, PP, false><<<g2, PS_T, 0, st>>>(k, w.mua, w.b2, w.cc, N, nlen, Q, Z, ldz, np, w.part, nullptr, \
                                                       0, nullptr, nullptr, tab)
  if (k.nd <= 8) GPK_P2F(8, 4);
  else if (k.nd <= 16) GPK_P2F(16, 2);
  else GPK_P2F(32, 1);
#undef GPK_P2F
  GPK_LAUNCH_OK();
  psi2_reduce_kernel<<<(unsigned)((np + 255) / 256), 256, 0, st>>>(w.part, np, nch, k.var * k.var, P2, ldp2);
  GPK_LAUNCH_OK();
  return 0;
}

// Launch geometry of psi_backward for N points, M inducing points and nd active dims (the one copy of its rules).
struct PsiBwdGeom {
  int nd_bucket, pp;                // kernel bucket ND (8, 16, 32) and pairs per thread of psi2_pair_kernel
  int64_t tiles, nch, nlen;         // psi2_pair_kernel: pair tiles x point chunks of nlen points
  int64_t gn, pch, plen;            // psi2_point_kernel (and psi1_bwd_point_kernel): point blocks x pair chunks of plen
  int launches;                     // launches of each psi2 kernel: 2 at ND = 32 (dims [0, 16) and [16, 32))
};

static PsiBwdGeom psi_bwd_geometry(int64_t N, int64_t M, int nd) {
  PsiBwdGeom g;
  g.nd_bucket = nd <= 8 ? 8 : (nd <= 16 ? 16 : 32);
  g.pp = pp_of(nd);
  g.tiles = pair_tiles(M, nd);
  g.nch = psi2_chunks(N, g.tiles, &g.nlen);
  g.gn = (N + PS_PT - 1) / PS_PT;
  // about 8 CTAs per SM over point blocks x pair chunks, at least PS_PB pairs per chunk
  const int64_t np = npairs_of(M);
  int64_t pch = (1056 + g.gn - 1) / g.gn;
  const int64_t most = (np + PS_PB - 1) / PS_PB;
  pch = pch < 1 ? 1 : (pch > most ? most : pch);
  g.plen = ((np + pch - 1) / pch + PS_PB - 1) / PS_PB * PS_PB;
  g.pch = (np + g.plen - 1) / g.plen;
  g.launches = g.nd_bucket == 32 ? 2 : 1;
  return g;
}

// Adjoints of psi1 and psi2 from G1t [M, ldg1] = (dF/dpsi1)^T and G2 [M, ldg2] = dF/dpsi2 (full, symmetric), ADDED into
// dmu, dS [N, Q], dZ [M, Q] and gpar [1 + nd] = {dF/dsigma^2, dF/dl_d per active dim}.  geom (optional): the geometry
// the launches used.
int psi_backward(const gpk_knode* nodes, int n_nodes, const int32_t* dims, const double* ard, const double* mu,
                 const double* S, int64_t N, int64_t Q, const double* Z, int64_t M, int64_t ldz, const double* G1t,
                 int64_t ldg1, const double* G2, int64_t ldg2, double* dmu, double* dS, double* dZ, double* gpar,
                 void* ws, const char* who, cudaStream_t st, PsiBwdGeom* geom) {
  PsiK k;
  PsiWs w;
  const double* tab = nullptr;
  GPK_TRY(psi_setup(nodes, n_nodes, dims, ard, mu, S, N, Q, M, ws, k, w, &tab, who, st));
  ProfScope ps(PROF_LEAF, st);
  const PsiBwdGeom g = psi_bwd_geometry(N, M, k.nd);
  if (geom) *geom = g;
  const unsigned gn = (unsigned)g.gn;
#define GPK_P1B(ND)                                                                                                 \
  psi1_bwd_point_kernel<ND><<<gn, PS_PT, 0, st>>>(k, w.mua, w.a1, w.cc, S, N, Q, Z, ldz, M, G1t, ldg1, dmu, dS, gpar, \
                                                  tab)
  if (g.nd_bucket == 8) GPK_P1B(8);
  else if (g.nd_bucket == 16) GPK_P1B(16);
  else GPK_P1B(32);
#undef GPK_P1B
  GPK_LAUNCH_OK();
#define GPK_P1Z(ND) psi1_bwd_z_kernel<ND><<<(unsigned)M, PS_PT, 0, st>>>(k, w.mua, w.a1, w.cc, N, Q, Z, ldz, G1t, ldg1, dZ, tab)
  if (g.nd_bucket == 8) GPK_P1Z(8);
  else if (g.nd_bucket == 16) GPK_P1Z(16);
  else GPK_P1Z(32);
#undef GPK_P1Z
  GPK_LAUNCH_OK();
  const int64_t np = npairs_of(M), nlen = g.nlen;
  const dim3 g2((unsigned)g.tiles, (unsigned)g.nch);
#define GPK_P2B(ND, PP, D0, DA)                                                                                     \
  psi2_pair_kernel<ND, PP, true, D0, DA><<<g2, PS_T, 0, st>>>(k, w.mua, w.b2, w.cc, N, nlen, Q, Z, ldz, np, nullptr, G2, \
                                                              ldg2, dZ, gpar, tab)
  if (g.nd_bucket == 8) GPK_P2B(8, 4, 0, 8);
  else if (g.nd_bucket == 16) GPK_P2B(16, 2, 0, 16);
  else {
    GPK_P2B(32, 1, 0, 16);
    GPK_LAUNCH_OK();
    GPK_P2B(32, 1, 16, 16);
  }
#undef GPK_P2B
  GPK_LAUNCH_OK();
  const int64_t plen = g.plen;
  const dim3 gp(gn, (unsigned)g.pch);
#define GPK_P2P(ND, D0, DA)                                                                                         \
  psi2_point_kernel<ND, D0, DA><<<gp, PS_PT, 0, st>>>(k, w.mua, w.b2, w.cc, S, N, Q, Z, ldz, np, plen, G2, ldg2, dmu, dS, \
                                                      gpar, tab)
  if (g.nd_bucket == 8) GPK_P2P(8, 0, 8);
  else if (g.nd_bucket == 16) GPK_P2P(16, 0, 16);
  else {
    GPK_P2P(32, 0, 16);
    GPK_LAUNCH_OK();
    GPK_P2P(32, 16, 16);
  }
#undef GPK_P2P
  GPK_LAUNCH_OK();
  return 0;
}

}  // namespace gpk
// gpk_debug_rbf_psi_grad: psi_backward alone, with the argument checks of gpk_rbf_psi; geom (host, may be NULL)
// receives {ND, PP, pair tiles, point chunks, nlen, point blocks, pair chunks, plen, psi2 launches}.
extern "C" int gpk_debug_rbf_psi_grad(const gpk_knode* nodes, int n_nodes, const int32_t* dims, const double* ard,
                                      const double* mu, const double* S, int64_t N, int64_t Q, const double* Z,
                                      int64_t M, int64_t ldz, const double* G1t, int64_t ldg1, const double* G2,
                                      int64_t ldg2, double* dmu, double* dS, double* dZ, double* gpar, void* ws,
                                      int64_t* geom, void* stream) {
  const cudaStream_t st = (cudaStream_t)stream;
  GPK_CHECK_ARG(N > 0 && Q > 0 && M > 0 && ldz >= Q && ldg1 >= N && ldg2 >= M, "debug_rbf_psi_grad: bad sizes");
  GPK_CHECK_ARG(mu && S && Z && G1t && G2 && dmu && dS && dZ && gpar && ws,
                "debug_rbf_psi_grad: a required pointer is NULL");
  PsiBwdGeom g;
  GPK_TRY(psi_backward(nodes, n_nodes, dims, ard, mu, S, N, Q, Z, M, ldz, G1t, ldg1, G2, ldg2, dmu, dS, dZ, gpar, ws,
                       "debug_rbf_psi_grad", st, &g));
  if (geom) {
    const int64_t v[9] = {g.nd_bucket, g.pp, g.tiles, g.nch, g.nlen, g.gn, g.pch, g.plen, g.launches};
    for (int i = 0; i < 9; ++i) geom[i] = v[i];
  }
  return 0;
}

// gpk_rbf_psi: psi0 (device scalar), psi1 [N, M] and psi2 [M, M] row-major.
extern "C" int gpk_rbf_psi(const gpk_knode* nodes, int n_nodes, const int32_t* dims, const double* ard,
                           const double* mu, const double* S, int64_t N, int64_t Q, const double* Z, int64_t M,
                           int64_t ldz, double* psi0, double* psi1, double* psi2, void* ws, void* stream) {
  const cudaStream_t st = (cudaStream_t)stream;
  GPK_CHECK_ARG(N > 0 && Q > 0 && M > 0 && ldz >= Q, "rbf_psi: bad sizes");
  GPK_CHECK_ARG(mu && S && Z && psi0 && psi1 && psi2 && ws, "rbf_psi: a required pointer is NULL");
  GPK_TRY(psi_forward(nodes, n_nodes, dims, ard, mu, S, N, Q, Z, M, ldz, psi1, M, 1, psi2, M, ws, "rbf_psi", st));
  return fill_impl(psi0, 1, 1, 1, (double)N * nodes[0].variance, GPK_F64, st);
}
namespace gpk {

// ---- the KL term of the bound and its gradient -----------------------------------------------------------------
// kl[i] = 1/2 log(p / S) - 1/2 + ((mu - m0)^2 + S) / (2 p) per element of [N, Q] (gplvm.py:195-204); with dmu / dS
// non-NULL also dmu -= (mu - m0) / p, dS -= 1/(2p) - 1/(2S)  (the bound is F = ... - KL)
__global__ void kl_diag_kernel(const double* __restrict__ mu, const double* __restrict__ S,
                               const double* __restrict__ m0, const double* __restrict__ p0, int64_t n,
                               double* __restrict__ kl, double* __restrict__ dmu, double* __restrict__ dS) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const double d = mu[i] - m0[i], s = S[i], p = p0[i];
  kl[i] = 0.5 * log(p / s) - 0.5 + (d * d + s) / (2.0 * p);
  if (dmu) {
    dmu[i] -= d / p;
    dS[i] -= 0.5 / p - 0.5 / s;
  }
}

int kl_diag(const double* mu, const double* S, const double* m0, const double* p0, int64_t n, double* kl, double* dmu,
            double* dS, cudaStream_t st) {
  kl_diag_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(mu, S, m0, p0, n, kl, dmu, dS);
  GPK_LAUNCH_OK();
  return 0;
}

}  // namespace gpk
