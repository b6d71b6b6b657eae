// vgp_oa.cu — VGPOpperArchambeau (gpflow/models/vgp.py:266-376): value and gradient of the ELBO in one call, for
// every likelihood gpk_lik describes.  q(f_p) = N(K alpha_p + m(X), (K^-1 + Lambda_p^2)^-1), Lambda_p = diag(lambda_p).
// Per latent p, with A_p = I + Lambda_p K Lambda_p = L L^T and B_p = A_p^-1:
//   fmean = K alpha + m(X),  fvar_j = (1 - B_jj) / lambda_j^2
//   KL    = 1/2 sum_p (log det A_p + tr B_p - N + alpha_p^T K alpha_p)
// and from the likelihood's adjoints R = dVE/dfmean, W = dVE/dfvar, D_p = diag(W_p / lambda_p^2):
//   Abar_p      = B (D_p + 1/2 I) B - 1/2 B                            (dF/dA_p)
//   dF/dK       = sum_p [sym(R_p alpha_p^T) - 1/2 alpha_p alpha_p^T + Lambda_p Abar_p Lambda_p]
//   dF/dalpha   = K (R - alpha)
//   dF/dlambda_j = -2 W_j (1 - B_jj) / lambda_j^3 + 2 [(W_j / lambda_j^2 + 1/2) B_jj - 1/2 - (Abar_p)_jj] / lambda_j
// The last term is 2 (K Lambda Abar)_jj rewritten through A Abar = (D + 1/2 I) B - 1/2 I, so it needs diagonals only.
//
// The likelihood couples the latents of a row (MultiClass, heteroskedastic), so R and W need fvar of every latent
// before any Abar_p: a first pass factors every A_p for fvar and the KL, a second pass refactors each A_p for its
// weighted product.  The second pass runs the latents in reverse, so the last latent's inverse from the first pass is
// reused: P factorisations and inverses in the first pass, P - 1 in the second, P weighted products.  The workspace
// holds four N x N matrices whatever P is.
#include "internal.cuh"

using namespace gpk;

namespace gpk {

// ---- A_p = I + Lambda_p K Lambda_p, lower triangle, into the factorisation buffer ----------------------------------
__global__ void oa_form_kernel(const double* __restrict__ K, int64_t ldk, const double* __restrict__ lam, int64_t P,
                               int64_t p, int64_t N, double* __restrict__ A, int64_t lda) {
  const int64_t j = (int64_t)blockIdx.x * 32 + threadIdx.x, i = (int64_t)blockIdx.y * 8 + threadIdx.y;
  if (i >= N || j > i) return;
  const double v = lam[i * P + p] * lam[j * P + p] * K[i * ldk + j];
  A[i * lda + j] = i == j ? 1.0 + v : v;
}

template <int NT>
__device__ __forceinline__ double block_sum(double v, double* red) {
  v = warp_sum(v);
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  if (lane == 0) red[warp] = v;
  __syncthreads();
  double s = 0.0;
  if (threadIdx.x == 0)
    for (int w = 0; w < NT / 32; ++w) s += red[w];
  __syncthreads();
  return s;
}

// First pass, per latent (one CTA, fixed summation order): fvar[p] from diag(B), and into scal
// [1] += tr B, [2] += alpha_p^T K alpha_p, [4] = the first failed factorisation as p N + pivot (0: none).
__global__ void __launch_bounds__(256)
oa_stats_kernel(const double* __restrict__ B, int64_t ldb, int64_t N, int64_t P, int64_t p,
                const double* __restrict__ lam, const double* __restrict__ alpha, const double* __restrict__ Kalpha,
                const int32_t* __restrict__ info, double* __restrict__ fvar, double* __restrict__ scal) {
  __shared__ double red[8];
  double tr = 0.0, ak = 0.0;
  for (int64_t j = threadIdx.x; j < N; j += 256) {
    const double b = B[j * ldb + j], l = lam[j * P + p];
    fvar[p * N + j] = (1.0 - b) / (l * l);
    tr += b;
    ak += alpha[j * P + p] * Kalpha[j * P + p];
  }
  tr = block_sum<256>(tr, red);
  ak = block_sum<256>(ak, red);
  if (threadIdx.x == 0) {
    scal[1] += tr;
    scal[2] += ak;
    if (scal[4] == 0.0 && info[0] != 0) scal[4] = (double)p * (double)N + (double)info[0];
  }
}

// scal: [0] log det, [1] tr, [2] alpha^T K alpha (all latents), [3] variational expectations, [4] info
__global__ void oa_finalize_kernel(double* out, const double* scal, double N, double P) {
  const double kl = 0.5 * (scal[0] + scal[1] - N * P + scal[2]);  // vgp.py:361-366
  out[0] = scal[3] - kl;                                           // vgp.py:369
  out[1] = scal[3];
  out[2] = kl;
  out[3] = scal[4];
}

// wv[j] = W_j / lambda_j^2 + 1/2, the diagonal weight of the product
__global__ void oa_weight_kernel(const double* __restrict__ Wt, const double* __restrict__ lam, int64_t N, int64_t P,
                                 int64_t p, double* __restrict__ wv) {
  const int64_t j = (int64_t)blockIdx.x * 256 + threadIdx.x;
  if (j >= N) return;
  const double l = lam[j * P + p];
  wv[j] = Wt[p * N + j] / (l * l) + 0.5;
}

// ---- Abar_p = B (D + 1/2 I) B - 1/2 B on the fp64 tensor cores (mma.sync.m16n8k16) ------------------------------------
// C_ij = sum_k B_ik w_k B_jk over the tiles on and below the diagonal: both operands are row blocks of the (mirrored,
// symmetric) B with k contiguous, and the weight w = diag(D) + 1/2 scales the second operand as it is staged.  w is
// negative wherever W_j < -lambda_j^2 / 2 (log-concave likelihoods have W < 0), so the product cannot be split into
// two square-root-scaled operands of one SYRK.  The tile is 64 x 64 with four warps of 32 x 32 and k steps of 16,
// one m16n8k16 per (16-row, 8-column) block: the generic fp64 GEMM (gemm.cu) stages its operands through fixed
// loaders with m8n8k4-shaped fragments and has no hook for a per-k weight or this epilogue.  The epilogue reads
// B_ij and adds Lambda Abar Lambda into the lower triangle of G and writes diag(Abar).
constexpr int OT = 64;        // CTA tile edge
constexpr int OK = 16;        // k step
constexpr int OS = OK + 4;    // shared row stride (doubles): the fragment reads of a half-warp hit 16 distinct banks
constexpr int OTHREADS = 128;

__global__ void __launch_bounds__(OTHREADS, 2)
oa_wprod_kernel(const double* __restrict__ B, int64_t ldb, const double* __restrict__ wv,
                const double* __restrict__ lam, int64_t P, int64_t p, int64_t N, double* __restrict__ G, int64_t ldg,
                double* __restrict__ dA) {
  // the tile pair (ti >= tj) of this CTA, from the triangular index
  const int64_t t = blockIdx.x;
  int64_t ti = (int64_t)((sqrt(8.0 * (double)t + 1.0) - 1.0) * 0.5);
  while (ti * (ti + 1) / 2 > t) --ti;
  while ((ti + 1) * (ti + 2) / 2 <= t) ++ti;
  const int64_t tj = t - ti * (ti + 1) / 2;
  const int64_t m0 = ti * OT, n0 = tj * OT;
  __shared__ __align__(16) double sA[OT * OS];
  __shared__ __align__(16) double sB[OT * OS];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int wm = (warp >> 1) * 32, wn = (warp & 1) * 32;
  const int g = lane >> 2, q = lane & 3;

  double acc[2][4][4];
#pragma unroll
  for (int a = 0; a < 2; ++a)
#pragma unroll
    for (int b = 0; b < 4; ++b)
#pragma unroll
      for (int e = 0; e < 4; ++e) acc[a][b][e] = 0.0;

  constexpr int PER = OT * OK / OTHREADS;  // 8 elements of each operand per thread and k step
  double ra[PER], rb[PER];
  auto load = [&](int64_t k0) {
#pragma unroll
    for (int i = 0; i < PER; ++i) {
      const int e = tid + i * OTHREADS, r = e / OK, kk = e % OK;
      const int64_t k = k0 + kk;
      const bool kin = k < N;
      ra[i] = (kin && m0 + r < N) ? B[(m0 + r) * ldb + k] : 0.0;
      rb[i] = (kin && n0 + r < N) ? B[(n0 + r) * ldb + k] * wv[k] : 0.0;
    }
  };
  load(0);
  for (int64_t k0 = 0; k0 < N; k0 += OK) {
    __syncthreads();
#pragma unroll
    for (int i = 0; i < PER; ++i) {
      const int e = tid + i * OTHREADS, r = e / OK, kk = e % OK;
      sA[r * OS + kk] = ra[i];
      sB[r * OS + kk] = rb[i];
    }
    __syncthreads();
    if (k0 + OK < N) load(k0 + OK);  // the next step's global loads run under this step's MMAs
    double bf[4][4];
#pragma unroll
    for (int nj = 0; nj < 4; ++nj)
#pragma unroll
      for (int i = 0; i < 4; ++i) bf[nj][i] = sB[(wn + 8 * nj + g) * OS + q + 4 * i];
#pragma unroll
    for (int mi = 0; mi < 2; ++mi) {
      double af[8];
#pragma unroll
      for (int i = 0; i < 8; ++i) af[i] = sA[(wm + 16 * mi + g + 8 * (i & 1)) * OS + q + 4 * (i >> 1)];
#pragma unroll
      for (int nj = 0; nj < 4; ++nj) dmma16816(acc[mi][nj], af, bf[nj]);
    }
  }

#pragma unroll
  for (int mi = 0; mi < 2; ++mi)
#pragma unroll
    for (int nj = 0; nj < 4; ++nj)
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const int64_t row = m0 + wm + 16 * mi + g + 8 * (e >> 1), col = n0 + wn + 8 * nj + 2 * q + (e & 1);
        if (row >= N || col > row) continue;
        const double abar = acc[mi][nj][e] - 0.5 * B[row * ldb + col];
        G[row * ldg + col] += lam[row * P + p] * lam[col * P + p] * abar;
        if (row == col) dA[row] = abar;
      }
}

// dq_lambda[:, p] from W_p, diag(B_p) and diag(Abar_p)
__global__ void oa_dlambda_kernel(const double* __restrict__ B, int64_t ldb, const double* __restrict__ Wt,
                                  const double* __restrict__ lam, const double* __restrict__ dA, int64_t N, int64_t P,
                                  int64_t p, double* __restrict__ dq_lambda) {
  const int64_t j = (int64_t)blockIdx.x * 256 + threadIdx.x;
  if (j >= N) return;
  const double l = lam[j * P + p], W = Wt[p * N + j], b = B[j * ldb + j];
  dq_lambda[j * P + p] = -2.0 * W * (1.0 - b) / (l * l * l) + 2.0 * ((W / (l * l) + 0.5) * b - 0.5 - dA[j]) / l;
}

struct OaWs {
  double *K, *A, *B, *G, *tmp, *fmu, *fvar, *R, *Wt, *U, *wv, *dA, *scal; void* dinv; int32_t* info; int64_t ldn;
  size_t dm_off, bytes;
};
static OaWs oa_layout(void* ws, int64_t N, int64_t P) {
  Arena a(ws);
  OaWs w;
  w.ldn = pad_ld(N);
  const size_t nn = (size_t)N * w.ldn * sizeof(double), np = (size_t)N * P * sizeof(double);
  const int64_t h = N / 2 + NB;
  w.K = (double*)a.take(nn);
  w.A = (double*)a.take(nn);
  w.B = (double*)a.take(nn);
  w.G = (double*)a.take(nn);
  w.tmp = (double*)a.take((size_t)h * h * sizeof(double));  // potri_lower's scratch
  w.dinv = a.take(potrf_ws_bytes(N, N, GPK_F64));
  w.info = (int32_t*)a.take(256);
  w.scal = (double*)a.take(256);
  w.fmu = (double*)a.take(np);   // K alpha [N][P]
  w.fvar = (double*)a.take(np);  // [P][N]
  w.dm_off = a.off;
  w.R = (double*)a.take(np);     // [N][P]
  w.Wt = (double*)a.take(np);    // [P][N]
  w.U = (double*)a.take(np);     // [N][P]
  w.wv = (double*)a.take((size_t)N * sizeof(double));
  w.dA = (double*)a.take((size_t)N * sizeof(double));
  w.bytes = a.off;
  return w;
}

}  // namespace gpk
extern "C" size_t gpk_vgp_oa_elbo_grad_ws(int64_t N, int64_t P, int) { return oa_layout(nullptr, N, P).bytes; }
extern "C" size_t gpk_vgp_oa_elbo_grad_dm(int64_t N, int64_t P, int) { return oa_layout(nullptr, N, P).dm_off; }
namespace gpk {

// Factor A_p (from w.K) and invert it: B_p (lower) in w.B, L^-1 in w.A; with logdet, log det A_p added to scal[0].
static int oa_factor(const OaWs& w, const double* lam, int64_t N, int64_t P, int64_t p, bool logdet, cudaStream_t st) {
  {
    ProfScope ps(PROF_MISC, st);
    oa_form_kernel<<<dim3((unsigned)((N + 31) / 32), (unsigned)((N + 7) / 8)), dim3(32, 8), 0, st>>>(
        w.K, w.ldn, lam, P, p, N, w.A, w.ldn);
    GPK_LAUNCH_OK();
  }
  GPK_TRY(potrf_any(w.A, N, N, w.ldn, GPK_F64, w.info, w.dinv, st));
  if (logdet) GPK_TRY(reduce_impl(2, w.A, N, w.ldn + 1, 2.0, 1, w.scal + 0, GPK_F64, st));  // 2 sum log diag L
  return potri_lower(w.A, N, w.ldn, (const double*)w.dinv, w.B, w.ldn, w.tmp, st);
}

}  // namespace gpk

extern "C" int gpk_vgp_oa_elbo_grad(const gpk_knode* nodes, int n_nodes, const int32_t* dims, const double* ard,
                                    const void* X, int64_t N, int64_t ldx, int64_t D, const void* Y, const void* mX,
                                    int64_t P, const double* q_alpha, const double* q_lambda, const gpk_lik* lik,
                                    int dtype, double* out, int n_out, double* dq_alpha, double* dq_lambda, void* ws,
                                    void* stream) {
  const cudaStream_t st = (cudaStream_t)stream;
  GPK_DTYPE_OK("vgp_oa_elbo_grad");
  GPK_CHECK_ARG(dtype == GPK_F64, "vgp_oa_elbo_grad: the device backward computes in float64 (dtype %d)", dtype);
  GPK_CHECK_ARG(N > 0 && P > 0 && D > 0 && ws && out && X && Y && q_alpha && q_lambda,
                "vgp_oa_elbo_grad: bad arguments");
  GPK_CHECK_ARG(dq_alpha && dq_lambda, "vgp_oa_elbo_grad: dq_alpha [N, P] and dq_lambda [N, P] are required");
  GPK_TRY(lik_check(lik, P, "vgp_oa_elbo_grad"));
  const int slots = grad_expr_slots(nodes, n_nodes, dims, ard, D, "vgp_oa_elbo_grad");
  if (slots < 0) return slots;
  GPK_CHECK_ARG(n_out >= 5 + slots, "vgp_oa_elbo_grad: n_out = %d, the expression needs %d outputs", n_out, 5 + slots);
  const OaWs w = oa_layout(ws, N, P);
  GPK_CHECK_ARG(D <= w.ldn, "vgp_oa_elbo_grad: X has %lld columns, the workspace's scratch holds %lld for N = %lld",
                (long long)D, (long long)w.ldn, (long long)N);
  const int64_t ldn = w.ldn;
  const double* mx = (const double*)mX;
  GPK_CUDA_OK(cudaMemsetAsync(out, 0, (size_t)n_out * sizeof(double), st));
  GPK_CUDA_OK(cudaMemsetAsync(w.scal, 0, 8 * sizeof(double), st));
  GPK_CUDA_OK(cudaMemsetAsync(w.G, 0, (size_t)N * ldn * sizeof(double), st));
  // ---- forward (vgp.py:349-369); K carries no jitter ----
  GPK_TRY(kbuild_impl(nodes, n_nodes, dims, ard, X, N, ldx, nullptr, N, ldx, D, w.K, ldn, GPK_F64, GPK_FULL, 0.0,
                      nullptr, st));
  GPK_TRY(gemm_any(0, 0, N, P, N, 1.0, w.K, ldn, q_alpha, P, 0.0, w.fmu, P, GPK_F64, 0, st));  // K alpha
  for (int64_t p = 0; p < P; ++p) {
    GPK_TRY(oa_factor(w, q_lambda, N, P, p, true, st));
    ProfScope ps(PROF_MISC, st);
    oa_stats_kernel<<<1, 256, 0, st>>>(w.B, ldn, N, P, p, q_lambda, q_alpha, w.fmu, w.info, w.fvar, w.scal);
    GPK_LAUNCH_OK();
  }
  GPK_TRY(lik_varexp_impl(lik, w.fmu, w.fvar, Y, mX, N, P, lik_ldy(lik, P), P, 1, N, 1.0, 1, w.scal + 3, GPK_F64,
                          st));
  oa_finalize_kernel<<<1, 1, 0, st>>>(out, w.scal, (double)N, (double)P);
  GPK_LAUNCH_OK();
  // ---- backward ----
  GPK_TRY(lik_grad_impl(lik, w.fmu, w.fvar, (const double*)Y, lik_ldy(lik, P), mx, N, P, 1.0, w.R, w.Wt, out + 4,
                        st));
  const unsigned gN = (unsigned)((N + 255) / 256);
  const int64_t nt = (N + OT - 1) / OT;
  for (int64_t p = P - 1; p >= 0; --p) {
    if (p != P - 1) GPK_TRY(oa_factor(w, q_lambda, N, P, p, false, st));  // the last latent's B is still in w.B
    GPK_TRY(svgp_bracket(SB_MIRROR, nullptr, w.B, N, ldn, nullptr, nullptr, nullptr, 0.0, 0.0, st));
    {
      ProfScope ps(PROF_MISC, st);
      oa_weight_kernel<<<gN, 256, 0, st>>>(w.Wt, q_lambda, N, P, p, w.wv);
      GPK_LAUNCH_OK();
    }
    {
      ProfScope ps(PROF_GEMM, st, (double)(nt * (nt + 1) / 2) * OT * OT * (double)(nt * OT));
      oa_wprod_kernel<<<(unsigned)(nt * (nt + 1) / 2), OTHREADS, 0, st>>>(w.B, ldn, w.wv, q_lambda, P, p, N, w.G, ldn,
                                                                          w.dA);
      GPK_LAUNCH_OK();
    }
    ProfScope ps(PROF_MISC, st);
    oa_dlambda_kernel<<<gN, 256, 0, st>>>(w.B, ldn, w.Wt, q_lambda, w.dA, N, P, p, dq_lambda);
    GPK_LAUNCH_OK();
  }
  // dF/dK += sym(U alpha^T), U = R - alpha / 2 (the mean and the KL's quadratic term); then mirror to the full square
  GPK_TRY(axpby_impl(N, P, 1.0, w.R, P, 0.0, w.U, P, GPK_F64, st));
  GPK_TRY(axpby_impl(N, P, -0.5, q_alpha, P, 1.0, w.U, P, GPK_F64, st));
  GPK_TRY(gemm_any(0, 1, N, N, P, 0.5, w.U, P, q_alpha, P, 1.0, w.G, ldn, GPK_F64, GPK_GEMM_LOWER_ONLY, st));
  GPK_TRY(gemm_any(0, 1, N, N, P, 0.5, q_alpha, P, w.U, P, 1.0, w.G, ldn, GPK_F64, GPK_GEMM_LOWER_ONLY, st));
  GPK_TRY(svgp_bracket(SB_MIRROR, nullptr, w.G, N, ldn, nullptr, nullptr, nullptr, 0.0, 0.0, st));
  // dF/dalpha = K (R - alpha)
  GPK_TRY(axpby_impl(N, P, -0.5, q_alpha, P, 1.0, w.U, P, GPK_F64, st));
  GPK_TRY(gemm_any(0, 0, N, P, N, 1.0, w.K, ldn, w.U, P, 0.0, dq_alpha, P, GPK_F64, 0, st));
  // the kernel parameters: dF/dK over the square K(X, X); w.A is dead and takes the discarded input derivative
  return square_grad_launch(nodes, n_nodes, dims, ard, (const double*)X, N, ldx, D, w.G, ldn, out + 4, w.A,
                            "vgp_oa_elbo_grad", st);
}
