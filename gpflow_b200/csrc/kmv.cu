// kmv.cu — matrix-free kernel product out[N, P] = (K(X, X2) + c I) V[N2, P] for sm_90a, fp64.
//
// The conjugate-gradient bound (CGLB, gpflow/models/cglb.py:140-160) multiplies the exact K + s I into a vector once
// per CG step; at N = 2^17 that matrix would need 137 GB, so it is never formed.  A CTA owns a 64-row block of `out`,
// streams 64-column blocks of X2 and V through shared memory, evaluates the 64x64 tile in registers (4x4 micro-tile
// per thread) with the K-build's element formulas, and multiplies it into V straight from registers.
//   * Element formulas: the norm-expansion distance of kbuild.cu with its 1e-36 clip; for one stationary leaf the
//     folded scales and the table-driven stationary_value4 of fastexp.cuh (the K-build fast path), for any other
//     expression the generic leaf functions and postfix program (kleaf.cuh).
//   * Determinism: no atomics.  Each thread accumulates its 4 rows over the columns it owns in column order, the 16
//     threads of a row meet in a fixed xor butterfly, and when there are too few row blocks to fill the GPU the
//     column blocks split into a fixed number of contiguous chunks whose partial products a second pass sums in
//     chunk order.  The chunk count depends only on (N, N2), so two calls give the same bits on any GPU.
//   * Width of V: passes of PW = 8, 4 or 1 columns (acc[4][PW] in registers); a wider V takes further passes.
//   * Memory: the workspace holds the partial products only, O(N P) doubles; nothing of size N x N2 exists.
#include "fastexp.cuh"
#include "internal.cuh"
#include "kleaf.cuh"

namespace gpk {

int exp2_table_device(const double** tab);  // kbuild.cu

constexpr int KM_TILE = 64;      // row / column block edge
constexpr int KM_KC = 32;        // dims staged per chunk
constexpr int KM_TARGET = 264;   // CTAs the column split aims for (2 x 132 SMs); a constant, so the bits never vary

static int64_t kmv_nsplit(int64_t N, int64_t N2) {
  const int64_t nrb = (N + KM_TILE - 1) / KM_TILE, ncb = (N2 + KM_TILE - 1) / KM_TILE;
  if (nrb >= KM_TARGET || ncb <= 1) return 1;
  const int64_t want = (KM_TARGET + nrb - 1) / nrb;
  const int64_t per = (ncb + want - 1) / want;  // column blocks per chunk; every chunk is non-empty
  return (ncb + per - 1) / per;
}

size_t kmv_ws_bytes(int64_t N, int64_t N2, int64_t P) {
  const int64_t ns = kmv_nsplit(N, N2);
  return ns > 1 ? align_up((size_t)ns * N * P * sizeof(double), 256) : 256;
}

// FAST: one stationary leaf of type TYPE with c / lengthscale^2 folded into prog.w (as kbuild_fast_launch does).
template <bool FAST, int TYPE, int NG, int PW>
__global__ void __launch_bounds__(256)
kmv_kernel(const __grid_constant__ KProg prog, const double* __restrict__ X, int64_t N, int64_t ldx,
           const double* __restrict__ X2, int64_t N2, int64_t ldx2, const double* __restrict__ V, int64_t ldv, int pw,
           double diag_scalar, const double* __restrict__ tab, double* __restrict__ out, int64_t ldo,
           int64_t cb_per_split, const int32_t* __restrict__ skip) {
  if (skip && *skip) return;  // a converged CG loop: the product is not needed
  __shared__ __align__(16) double sA[KM_KC][KM_TILE];
  __shared__ __align__(16) double sB[KM_KC][KM_TILE];
  __shared__ double sNa[NG][KM_TILE], sNb[NG][KM_TILE];
  __shared__ double sV[KM_TILE][PW];
  __shared__ double s_tab[64];
  const int tid = threadIdx.x, tx = tid & 15, ty = tid >> 4;
  const int64_t row0 = (int64_t)blockIdx.x * KM_TILE;
  const int64_t ncb = (N2 + KM_TILE - 1) / KM_TILE;
  const int64_t cb0 = (int64_t)blockIdx.y * cb_per_split;
  const int64_t cb1 = min(ncb, cb0 + cb_per_split);
  const bool sym = prog.symmetric != 0;
  const double* Xb = sym ? X : X2;
  const int64_t ldb = sym ? ldx : ldx2;
  const double var = prog.l_var[0];
  const double var3 = var * (1.0 / 3.0);
  const bool var_ok = var >= 7.888609052210118e-31;  // 2^-100 (kbuild_fast_kernel)
  // the 2^(j/64) table in shared memory, pre-multiplied by the variance when the prefactor is constant
  if (FAST && tid < 64) s_tab[tid] = kf_const_pre<TYPE>() ? tab[tid] * var : tab[tid];

  double acc[4][PW];
#pragma unroll
  for (int r = 0; r < 4; ++r)
#pragma unroll
    for (int p = 0; p < PW; ++p) acc[r][p] = 0.0;

  for (int64_t cb = cb0; cb < cb1; ++cb) {
    const int64_t col0 = cb * KM_TILE;
    double dots[NG][4][4];
#pragma unroll
    for (int g = 0; g < NG; ++g)
#pragma unroll
      for (int r = 0; r < 4; ++r)
#pragma unroll
        for (int c = 0; c < 4; ++c) dots[g][r][c] = 0.0;
    __syncthreads();  // the previous block's readers of sNa / sNb / sV are done
    if (tid < KM_TILE) {
#pragma unroll
      for (int g = 0; g < NG; ++g) { sNa[g][tid] = 0.0; sNb[g][tid] = 0.0; }
    }
    for (int e = tid; e < KM_TILE * PW; e += 256) {
      const int c = e / PW, p = e % PW;
      const int64_t gc = col0 + c;
      sV[c][p] = (gc < N2 && p < pw) ? V[gc * ldv + p] : 0.0;
    }
#pragma unroll
    for (int g = 0; g < NG; ++g) {
      if (g >= prog.n_groups) break;
      const int nd = prog.g_ndims[g], off = prog.g_off[g];
      for (int d0 = 0; d0 < nd; d0 += KM_KC) {
        const int kc = min(KM_KC, nd - d0);
        __syncthreads();
        for (int e = tid; e < kc * KM_TILE; e += 256) {
          const int d = e % kc, r = e / kc;
          const int col = prog.dims[off + d0 + d];
          const int64_t gr = row0 + r, gc = col0 + r;
          const double a = gr < N ? X[gr * ldx + col] : 0.0;
          const double b = gc < N2 ? Xb[gc * ldb + col] : 0.0;
          const double wv = prog.w[off + d0 + d];
          sA[d][r] = a * wv;
          sB[d][r] = (FAST || prog.g_weighted[g] == 2) ? b * wv : b;
        }
        __syncthreads();
        // squared norms of the staged rows, in the K-build's summation order: the generic kernel's sequential fma
        // per chunk, or the fast path's 8-lane butterfly per 8 dims (zeros beyond the last dim), chunks in order
        if (tid < 2 * KM_TILE) {
          const int r = tid & (KM_TILE - 1);
          const double(*S)[KM_TILE] = tid < KM_TILE ? sA : sB;
          double* dst = tid < KM_TILE ? &sNa[g][r] : &sNb[g][r];
          if (FAST) {
            double q = *dst;
            for (int d8 = 0; d8 < kc; d8 += 8) {
              double sq[8];
#pragma unroll
              for (int j = 0; j < 8; ++j) { const double x = d8 + j < kc ? S[d8 + j][r] : 0.0; sq[j] = x * x; }
              const double t = ((sq[0] + sq[1]) + (sq[2] + sq[3])) + ((sq[4] + sq[5]) + (sq[6] + sq[7]));
              q = (d0 == 0 && d8 == 0) ? t : q + t;
            }
            *dst = q;
          } else {
            double a2 = 0.0;
            for (int d = 0; d < kc; ++d) { const double x = S[d][r]; a2 = fma(x, x, a2); }
            *dst += a2;
          }
        }
        for (int d = 0; d < kc; ++d) {
          double a[4], b[4];
#pragma unroll
          for (int r = 0; r < 4; ++r) a[r] = sA[d][ty * 4 + r];
#pragma unroll
          for (int c = 0; c < 4; ++c) b[c] = sB[d][tx * 4 + c];
#pragma unroll
          for (int r = 0; r < 4; ++r)
#pragma unroll
            for (int c = 0; c < 4; ++c) dots[g][r][c] = fma(a[r], b[c], dots[g][r][c]);
        }
      }
    }
    __syncthreads();

    double vals[16];
    if (FAST) {
#pragma unroll
      for (int r = 0; r < 4; ++r) {
        double r2[4], o[4];
        const double na = sNa[0][ty * 4 + r];
#pragma unroll
        for (int c = 0; c < 4; ++c) r2[c] = fma(-2.0, dots[0][r][c], na + sNb[0][tx * 4 + c]);
        stationary_value4<TYPE>(r2, var, var3, var_ok, s_tab, o);
#pragma unroll
        for (int c = 0; c < 4; ++c) vals[r * 4 + c] = o[c];
      }
      if (sym) {
#pragma unroll
        for (int r = 0; r < 4; ++r)
#pragma unroll
          for (int c = 0; c < 4; ++c)
            if (row0 + ty * 4 + r == col0 + tx * 4 + c) vals[r * 4 + c] += diag_scalar;
      }
    } else {
      // one rolled loop over the 16 elements (as kbuild_kernel: unrolling replicates the leaf code 16x)
#pragma unroll
      for (int r = 0; r < 4; ++r)
#pragma unroll
        for (int c = 0; c < 4; ++c) vals[r * 4 + c] = NG == 1 ? dots[0][r][c] : 0.0;
      const int n_ops = prog.n_ops;
#pragma unroll 1
      for (int e = 0; e < 16; ++e) {
        const int r = e >> 2, c = e & 3;
        const int64_t gi = row0 + ty * 4 + r, gj = col0 + tx * 4 + c;
        const bool on_diag = sym && gi == gj;
        double s0 = 0.0, s1 = 0.0, s2 = 0.0, s3 = 0.0;
        for (int o = 0; o < n_ops; ++o) {
          const int op = prog.ops[o];
          if (op < KB_MAXL) {
            const int g = prog.l_group[op];
            double dot = 0.0, na = 0.0, nb = 0.0;
            if (NG == 1) {
              dot = vals[e];
              if (g == 0) { na = sNa[0][ty * 4 + r]; nb = sNb[0][tx * 4 + c]; }
            } else {
#pragma unroll
              for (int gg = 0; gg < NG; ++gg)
                if (g == gg) {
                  double v = dots[gg][0][0];
#pragma unroll
                  for (int q = 1; q < 16; ++q)
                    if (e == q) v = dots[gg][q >> 2][q & 3];
                  dot = v;
                  na = sNa[gg][ty * 4 + r];
                  nb = sNb[gg][tx * 4 + c];
                }
            }
            const double v = leaf_value<double>(prog.l_type[op], dot, na, nb, prog.l_scale[op], prog.l_var[op],
                                                prog.l_alpha[op], on_diag);
            s3 = s2; s2 = s1; s1 = s0; s0 = v;
          } else {
            s0 = op == KB_OP_ADD ? s1 + s0 : s1 * s0;
            s1 = s2; s2 = s3;
          }
        }
        if (on_diag) s0 += diag_scalar;
        vals[e] = s0;
      }
    }
    // multiply the tile into V: columns beyond N2 carry V = 0, rows beyond N are never stored
#pragma unroll
    for (int r = 0; r < 4; ++r)
#pragma unroll
      for (int c = 0; c < 4; ++c) {
        const double k = vals[r * 4 + c];
#pragma unroll
        for (int p = 0; p < PW; ++p) acc[r][p] = fma(k, sV[tx * 4 + c][p], acc[r][p]);
      }
  }
  // the 16 threads of a row group meet in a fixed butterfly (every lane ends with the same bits)
#pragma unroll
  for (int r = 0; r < 4; ++r)
#pragma unroll
    for (int p = 0; p < PW; ++p)
#pragma unroll
      for (int o = 1; o < 16; o <<= 1) acc[r][p] += __shfl_xor_sync(0xffffffffu, acc[r][p], o);
  if (tx == 0) {
#pragma unroll
    for (int r = 0; r < 4; ++r) {
      const int64_t gi = row0 + ty * 4 + r;
      if (gi < N)
#pragma unroll
        for (int p = 0; p < PW; ++p)
          if (p < pw) out[(int64_t)blockIdx.y * N * ldo + gi * ldo + p] = acc[r][p];
    }
  }
}

// out[i, p] = sum over the chunks s, in chunk order, of part[s][i][p]
__global__ void kmv_combine_kernel(const double* __restrict__ part, int64_t ns, int64_t N, int64_t P,
                                   double* __restrict__ out, int64_t ldo, const int32_t* __restrict__ skip) {
  if (skip && *skip) return;
  const int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= N * P) return;
  const int64_t i = e / P, p = e % P;
  double s = part[e];
  for (int64_t c = 1; c < ns; ++c) s += part[c * N * P + e];
  out[i * ldo + p] = s;
}

template <bool FAST, int TYPE, int NG>
static void kmv_go(int pw_t, const KProg& p, const double* X, int64_t N, int64_t ldx, const double* X2, int64_t N2,
                   int64_t ldx2, const double* V, int64_t ldv, int pw, double diag, const double* tab, double* out,
                   int64_t ldo, int64_t ns, int64_t per, const int32_t* skip, cudaStream_t st) {
  const dim3 grid((unsigned)((N + KM_TILE - 1) / KM_TILE), (unsigned)ns);
#define GPK_KMV_GO(PW_)                                                                                          \
  kmv_kernel<FAST, TYPE, NG, PW_><<<grid, 256, 0, st>>>(p, X, N, ldx, X2, N2, ldx2, V, ldv, pw, diag, tab, out, ldo, \
                                                        per, skip)
  if (pw_t == 8) GPK_KMV_GO(8);
  else if (pw_t == 4) GPK_KMV_GO(4);
  else GPK_KMV_GO(1);
#undef GPK_KMV_GO
}

int kmv_impl(const gpk_knode* nodes, int n_nodes, const int32_t* dims, const double* ard, const double* X, int64_t N,
             int64_t ldx, const double* X2, int64_t N2, int64_t ldx2, int64_t D, const double* V, int64_t P,
             int64_t ldv, double diag_scalar, double* out, int64_t ldo, void* ws, const int32_t* skip, cudaStream_t st) {
  GPK_CHECK_ARG(X && V && out, "kmv: null X, V or out");
  const bool sym = X2 == nullptr;
  if (sym) { N2 = N; ldx2 = ldx; }
  GPK_CHECK_ARG(N >= 0 && N2 >= 0 && P >= 0 && ldx >= D && ldx2 >= D && ldv >= P && ldo >= P, "kmv: bad shape/stride");
  GPK_CHECK_ARG(sym || diag_scalar == 0.0, "kmv: the diagonal term needs the symmetric form (X2 == NULL)");
  GPK_CHECK_ARG(N < ((int64_t)1 << 31) * KM_TILE, "kmv: N = %lld exceeds the row-block grid", (long long)N);
  if (N == 0 || P == 0) return 0;
  GPK_CHECK_ARG(N2 > 0 || !skip, "kmv: empty X2 inside a CG loop");
  if (N2 == 0) return fill_impl(out, N, P, ldo, 0.0, GPK_F64, st);
  KProg p;
  GPK_TRY(compile_kprog(nodes, n_nodes, dims, ard, D, p));
  p.symmetric = sym ? 1 : 0;
  const int64_t ns = kmv_nsplit(N, N2);
  GPK_CHECK_ARG(ns == 1 || ws, "kmv: N = %lld needs the workspace of gpk_kmv_ws", (long long)N);
  const int64_t ncb = (N2 + KM_TILE - 1) / KM_TILE, per = (ncb + ns - 1) / ns;
  const double* tab = nullptr;
  const bool fast = p.n_leaves == 1 && p.n_ops == 1 && p.n_groups == 1 &&
                    (p.l_type[0] == GPK_K_RBF || p.l_type[0] == GPK_K_MATERN12 || p.l_type[0] == GPK_K_MATERN32 ||
                     p.l_type[0] == GPK_K_MATERN52 || p.l_type[0] == GPK_K_EXPONENTIAL);
  if (fast) GPK_TRY(exp2_table_device(&tab));
  ProfScope ps(PROF_KBUILD, st);
  for (int64_t p0 = 0; p0 < P; ) {
    const int64_t rem = P - p0;
    const int pw_t = rem >= 5 ? 8 : rem >= 2 ? 4 : 1;
    const int pw = (int)(rem < pw_t ? rem : pw_t);
    double* dst = ns > 1 ? (double*)ws + p0 : out + p0;
    const int64_t ldd = ns > 1 ? P : ldo;
    if (fast) {
      // fold c / lengthscale^2 into the per-dimension weights, as kbuild_fast_launch does
#define GPK_KMV_FAST(TY)                                                                                         \
  do {                                                                                                          \
    KProg q = p;                                                                                                \
    const double f = sqrt(q.l_scale[0] * kf_fold<TY>());                                                        \
    for (int d = 0; d < q.g_ndims[0]; ++d) q.w[d] *= f;                                                         \
    q.l_scale[0] = 1.0;                                                                                         \
    kmv_go<true, TY, 1>(pw_t, q, X, N, ldx, X2, N2, ldx2, V + p0, ldv, pw, diag_scalar, tab, dst, ldd, ns, per, skip, st); \
  } while (0)
      switch (p.l_type[0]) {
        case GPK_K_RBF: GPK_KMV_FAST(GPK_K_RBF); break;
        case GPK_K_MATERN12: GPK_KMV_FAST(GPK_K_MATERN12); break;
        case GPK_K_MATERN32: GPK_KMV_FAST(GPK_K_MATERN32); break;
        case GPK_K_MATERN52: GPK_KMV_FAST(GPK_K_MATERN52); break;
        default: GPK_KMV_FAST(GPK_K_EXPONENTIAL); break;
      }
#undef GPK_KMV_FAST
    } else {
#define GPK_KMV_GEN(NG_) \
  kmv_go<false, 0, NG_>(pw_t, p, X, N, ldx, X2, N2, ldx2, V + p0, ldv, pw, diag_scalar, tab, dst, ldd, ns, per, skip, st)
      switch (p.n_groups) {
        case 0:
        case 1: GPK_KMV_GEN(1); break;
        case 2: GPK_KMV_GEN(2); break;
        case 3: GPK_KMV_GEN(3); break;
        default: GPK_KMV_GEN(4); break;
      }
#undef GPK_KMV_GEN
    }
    GPK_LAUNCH_OK();
    p0 += pw;
  }
  if (ns > 1) {
    kmv_combine_kernel<<<(unsigned)((N * P + 255) / 256), 256, 0, st>>>((const double*)ws, ns, N, P, out, ldo, skip);
    GPK_LAUNCH_OK();
  }
  return 0;
}

}  // namespace gpk
