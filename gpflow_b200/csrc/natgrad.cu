// natgrad.cu — one natural-gradient step on q(u) = N(q_mu, q_sqrt q_sqrt^T) per latent GP, for the XiNat and
// XiSqrtMeanVar transforms of gpflow/optimizers/natgrad.py:280-367 (the conversions of :429-502 written out so that
// neither Sig^-1, S^-1 nor a second Cholesky is ever formed; include/gpk.h gives the algebra).
//
// Per latent p, with S = tril(q_sqrt[p]), gS = dF/dS, gm = dF/dq_mu[:, p] and T = S^T gS (lower triangle):
//   XiNat:          JBJ = J (I - 2 gamma D H D) J = C C^T  (built from T in one pass, D = diag(sign diag S)),
//                   X = J (S D)^T  (the same pass), Y = C^-1 X, S' = (J Y)^T  (written forward, zeros above),
//                   m' = m + gamma S' S'^T gm;
//   XiSqrtMeanVar:  S' = S + gamma S Phi(T)  (Phi(T) = 2 Phi(H) by svgp_bracket SB_PHI),  m' = m + gamma S S^T gm.
#include <math.h>

#include "internal.cuh"

using namespace gpk;

namespace gpk {

static inline int64_t natgrad_ld(int64_t M) { return (M + 3) / 4 * 4; }

struct NatgradWs {
  double *T, *A, *B, *t;  // T [M, ld]; XiNat: A = JBJ, B = X / Y; XiSqrtMeanVar: A = Phi(T), B = S Phi(T); t [M]
  void* pws;              // XiNat: gpk_potrf's workspace for JBJ (its block inverses at the head)
  size_t bytes;
};

static NatgradWs natgrad_layout(void* ws, int64_t M, int xi) {
  const size_t mm = align_up((size_t)M * natgrad_ld(M) * sizeof(double), 256);
  char* b = (char*)ws;
  NatgradWs w;
  size_t off = 0;
  auto take = [&](size_t n) { void* r = b ? b + off : nullptr; off += align_up(n, 256); return r; };
  w.T = (double*)take(mm);
  w.A = (double*)take(mm);
  w.B = (double*)take(mm);
  w.t = (double*)take((size_t)M * sizeof(double));
  w.pws = xi == GPK_XI_NAT ? take(potrf_ws_bytes(M, M, GPK_F64)) : nullptr;
  w.bytes = off;
  return w;
}

__device__ __forceinline__ double diag_sign(const double* __restrict__ S, int64_t M, int64_t k) {
  return S[k * M + k] < 0.0 ? -1.0 : 1.0;
}

// One pass over the M x M grid (a, b), i = M-1-a, j = M-1-b, d = sign(diag S):
//   JBJ[a,b] = delta_ab - gamma d_i d_j T[j,i]  for a >= b (then i <= j: T's lower triangle), 0 above;
//   X[a,b]   = d_i S[b, i]  for b >= i, 0 otherwise (S's strict upper part is never read).
// The reads run along i, the reversed output row, so 32 x 32 tiles (block 32 x 8) stage them through shared memory
// with lanes along i, and the writes go out with lanes along b, as natgrad_out_kernel does for the write-back.
__global__ void __launch_bounds__(256)
natgrad_jbj_kernel(const double* __restrict__ T, const double* __restrict__ S, int64_t M, int64_t ld, double gamma,
                   double* __restrict__ JBJ, double* __restrict__ X) {
  __shared__ double tT[32][33], tS[32][33], da[32], db[32];
  const int64_t a0 = (int64_t)blockIdx.y * 32, b0 = (int64_t)blockIdx.x * 32;
  const int tx = threadIdx.x, ty = threadIdx.y;
  if (ty == 0) {
    da[tx] = a0 + tx < M ? diag_sign(S, M, M - 1 - (a0 + tx)) : 1.0;
    db[tx] = b0 + tx < M ? diag_sign(S, M, M - 1 - (b0 + tx)) : 1.0;
  }
  for (int k = ty; k < 32; k += 8) {  // tile[b - b0][a - a0], lanes along a (i contiguous)
    const int64_t a = a0 + tx, b = b0 + k;
    if (a >= M || b >= M) continue;
    const int64_t i = M - 1 - a, j = M - 1 - b;
    tT[k][tx] = a >= b ? T[j * ld + i] : 0.0;
    tS[k][tx] = b >= i ? S[b * M + i] : 0.0;
  }
  __syncthreads();
  for (int k = ty; k < 32; k += 8) {  // lanes along b
    const int64_t a = a0 + k, b = b0 + tx;
    if (a >= M || b >= M) continue;
    const double t = tT[tx][k];
    double v = 0.0;
    if (a == b) v = fma(-gamma, t, 1.0);
    else if (a > b) v = -gamma * da[k] * db[tx] * t;
    JBJ[a * ld + b] = v;
    X[a * ld + b] = da[k] * tS[tx][k];
  }
}

// q_sqrt_out [M, M] (ld M), written in full, zeros above the diagonal, in 32 x 32 tiles (block 32 x 8):
//   XiNat:          out[r,c] = Y[M-1-c, r]  (the reversal and the transpose through shared memory);
//   XiSqrtMeanVar:  out[r,c] = S[r,c] + gamma W[r,c].
__global__ void __launch_bounds__(256)
natgrad_out_kernel(int xi, const double* __restrict__ Y, const double* __restrict__ S, const double* __restrict__ W,
                   int64_t M, int64_t ld, double gamma, double* __restrict__ out) {
  __shared__ double tile[32][33];
  const int64_t r0 = (int64_t)blockIdx.y * 32, c0 = (int64_t)blockIdx.x * 32;
  const int tx = threadIdx.x, ty = threadIdx.y;
  const bool above = c0 > r0 + 31;  // the whole tile lies above the diagonal
  if (xi == GPK_XI_NAT && !above) {
    for (int k = ty; k < 32; k += 8) {
      const int64_t c = c0 + k, r = r0 + tx;
      tile[k][tx] = (c < M && r < M) ? Y[(M - 1 - c) * ld + r] : 0.0;
    }
    __syncthreads();
  }
  for (int k = ty; k < 32; k += 8) {
    const int64_t r = r0 + k, c = c0 + tx;
    if (r >= M || c >= M) continue;
    double v = 0.0;
    if (c <= r) v = xi == GPK_XI_NAT ? tile[tx][k] : fma(gamma, W[r * ld + c], S[r * M + c]);
    out[r * M + c] = v;
  }
}

// info[p] = -(i + 1) for the first i with q_sqrt[p][i, i] == 0, unless the factorisation already reported a pivot.
__global__ void __launch_bounds__(256)
natgrad_diag_check_kernel(const double* __restrict__ q_sqrt, int64_t M, int32_t* info) {
  __shared__ int first;
  const double* S = q_sqrt + (size_t)blockIdx.x * M * M;
  if (threadIdx.x == 0) first = INT32_MAX;
  __syncthreads();
  for (int64_t i = threadIdx.x; i < M; i += blockDim.x)
    if (S[i * M + i] == 0.0) atomicMin(&first, (int)i);
  __syncthreads();
  if (threadIdx.x == 0 && first != INT32_MAX && info[blockIdx.x] == 0) info[blockIdx.x] = -(first + 1);
}

// B = I - 2 gamma D H D is I minus a step: its conditioning has no bound the host knows (it diverges as the step
// approaches the largest one q admits).  An infinite hint states that: pick_slices gives it the 7 digit planes that serve
// every conditioning (the same count as the unknown hint 0), never the 6 of a hint <= 1e4.
constexpr double NATGRAD_COND_HINT = HUGE_VAL;

}  // namespace gpk

extern "C" size_t gpk_natgrad_step_ws(int64_t M, int64_t, int xi, int) {
  return M > 0 ? natgrad_layout(nullptr, M, xi).bytes : 0;
}

extern "C" int gpk_natgrad_step(int xi, int64_t M, int64_t P, const void* q_mu, const void* q_sqrt, const double* dq_mu,
                                const double* dq_sqrt, double gamma, int dtype, void* q_mu_out, void* q_sqrt_out,
                                int32_t* info, void* ws, void* stream) {
  const cudaStream_t st = (cudaStream_t)stream;
  GPK_CHECK_ARG(dtype == GPK_F64, "natgrad_step: the natural-gradient step computes in float64 (dtype %d)", dtype);
  GPK_CHECK_ARG(xi == GPK_XI_NAT || xi == GPK_XI_SQRT_MEAN_VAR, "natgrad_step: bad xi transform %d", xi);
  GPK_CHECK_ARG(M > 0 && P > 0 && q_mu && q_sqrt && dq_mu && dq_sqrt && q_mu_out && q_sqrt_out && info && ws,
                "natgrad_step: bad arguments");
  GPK_CHECK_ARG(gamma > 0.0 && isfinite(gamma), "natgrad_step: gamma must be positive and finite (%g)", gamma);
  GPK_CHECK_ARG(q_mu_out != q_mu && q_sqrt_out != q_sqrt, "natgrad_step: the step is out of place");
  const NatgradWs w = natgrad_layout(ws, M, xi);
  const int64_t ld = natgrad_ld(M);
  const size_t sq = (size_t)M * M;
  GPK_CUDA_OK(cudaMemsetAsync(info, 0, (size_t)P * sizeof(int32_t), st));
  GPK_CUDA_OK(cudaMemcpyAsync(q_mu_out, q_mu, (size_t)M * P * sizeof(double), cudaMemcpyDeviceToDevice, st));
  const dim3 tg((unsigned)((M + 31) / 32), (unsigned)((M + 31) / 32)), tb(32, 8);
  for (int64_t p = 0; p < P; ++p) {
    const double* S = (const double*)q_sqrt + p * sq;
    double* Sout = (double*)q_sqrt_out + p * sq;
    // T = S^T gS, lower triangle
    GPK_TRY(gemm_any(1, 0, M, M, M, 1.0, S, M, dq_sqrt + p * sq, M, 0.0, w.T, ld, GPK_F64,
                     GPK_GEMM_A_LOWER | GPK_GEMM_LOWER_ONLY, st));
    const double* Snew;
    if (xi == GPK_XI_NAT) {
      natgrad_jbj_kernel<<<tg, tb, 0, st>>>(w.T, S, M, ld, gamma, w.A, w.B);
      GPK_LAUNCH_OK();
      GPK_TRY(potrf_any(w.A, M, M, ld, GPK_F64, info + p, w.pws, st, true, NATGRAD_COND_HINT));
      GPK_TRY(trsm_any(0, w.A, M, ld, w.B, M, ld, GPK_F64, w.pws, st));
      natgrad_out_kernel<<<tg, tb, 0, st>>>(xi, w.B, nullptr, nullptr, M, ld, gamma, Sout);
      GPK_LAUNCH_OK();
      Snew = Sout;
    } else {
      GPK_TRY(svgp_bracket(SB_PHI, w.T, w.A, M, ld, nullptr, nullptr, nullptr, 0.0, 0.0, st));
      GPK_TRY(gemm_any(0, 0, M, M, M, 1.0, S, M, w.A, ld, 0.0, w.B, ld, GPK_F64,
                       GPK_GEMM_A_LOWER | GPK_GEMM_LOWER_ONLY, st));
      natgrad_out_kernel<<<tg, tb, 0, st>>>(xi, nullptr, S, w.B, M, ld, gamma, Sout);
      GPK_LAUNCH_OK();
      Snew = S;
    }
    // m' = m + gamma Snew Snew^T gm
    GPK_TRY(gemm_any(1, 0, M, 1, M, 1.0, Snew, M, dq_mu + p, P, 0.0, w.t, 1, GPK_F64, GPK_GEMM_A_LOWER, st));
    GPK_TRY(gemm_any(0, 0, M, 1, M, gamma, Snew, M, w.t, 1, 1.0, (double*)q_mu_out + p, P, GPK_F64, GPK_GEMM_A_LOWER,
                     st));
  }
  natgrad_diag_check_kernel<<<(unsigned)P, 256, 0, st>>>((const double*)q_sqrt, M, info);
  GPK_LAUNCH_OK();
  return 0;
}
