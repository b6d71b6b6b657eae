// capi.cu — the extern "C" surface declared in include/gpk.h (argument checks + dtype dispatch).
#include <stdarg.h>

#include <atomic>
#include <vector>

#include "internal.cuh"

namespace gpk {

static thread_local char g_err[512] = "";

void set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}

static std::atomic<long long> g_launches{0};
void count_launch() { g_launches.fetch_add(1, std::memory_order_relaxed); }

struct ProfRec { cudaEvent_t a, b; int cls; double work; };
static std::vector<ProfRec> g_recs;
static bool g_prof = false;

ProfScope::ProfScope(int cls, cudaStream_t s, double work) : idx(-1), st(s) {
  if (!g_prof) return;
  ProfRec r;
  r.cls = cls;
  r.work = work;
  if (cudaEventCreate(&r.a) != cudaSuccess || cudaEventCreate(&r.b) != cudaSuccess) return;
  cudaEventRecord(r.a, s);
  g_recs.push_back(r);
  idx = (int)g_recs.size() - 1;
}
ProfScope::~ProfScope() {
  if (idx >= 0) cudaEventRecord(g_recs[idx].b, st);
}

int gemm_any(int ta, int tb, int64_t m, int64_t n, int64_t k, double alpha, const void* A, int64_t lda, const void* B,
             int64_t ldb, double beta, void* C, int64_t ldc, int dtype, int flags, cudaStream_t st) {
  if (dtype == GPK_F64)
    return gemm_t<double>(ta, tb, m, n, k, alpha, (const double*)A, lda, (const double*)B, ldb, beta, (double*)C, ldc,
                          flags, st);
  return gemm_t<float>(ta, tb, m, n, k, (float)alpha, (const float*)A, lda, (const float*)B, ldb, (float)beta,
                       (float*)C, ldc, flags, st);
}

int potrf_any(void* A, int64_t n, int64_t rows, int64_t lda, int dtype, int32_t* info, void* ws, cudaStream_t st,
              bool need_dinv, double cond_hint) {
  const size_t tcb = potrf_tc_ws_bytes(n, rows, dtype);
  void* tcws = tcb ? (char*)ws + align_up(dinv_bytes(n, dtype), 256) + 256 : nullptr;
  if (dtype == GPK_F64)
    return potrf_t<double>((double*)A, n, rows, lda, info, (double*)ws, tcws, tcb, st, need_dinv, cond_hint);
  return potrf_t<float>((float*)A, n, rows, lda, info, (float*)ws, tcws, tcb, st, need_dinv);
}

int trsm_any(int trans, const void* L, int64_t n, int64_t ldl, void* B, int64_t nrhs, int64_t ldb, int dtype,
             const void* dinv, cudaStream_t st) {
  if (dtype == GPK_F64)
    return trsm_t<double>(trans, (const double*)L, n, ldl, (double*)B, nrhs, ldb, (const double*)dinv, st);
  return trsm_t<float>(trans, (const float*)L, n, ldl, (float*)B, nrhs, ldb, (const float*)dinv, st);
}

int trtri_diag_any(const void* L, int64_t n, int64_t ldl, void* dinv, int dtype, cudaStream_t st) {
  if (dtype == GPK_F64) return trtri_diag_t<double>((const double*)L, n, ldl, (double*)dinv, st);
  return trtri_diag_t<float>((const float*)L, n, ldl, (float*)dinv, st);
}

int leaf_debug(double* A, int64_t lda, int n, double* dinv, long long* dbg, int slim, cudaStream_t st);
int tc_debug_syrk(const double* A, int64_t lda, int64_t r0, int64_t k0, int64_t K, double* C, int64_t ldc, int64_t m,
                  int64_t n, int lower, int S, int cluster, double* rowscale_out, int* head_flag, cudaStream_t st);
int peak_probe(double* out_host, cudaStream_t st);
int debug_dmma16816(const double* A, const double* B, const double* C, double* D, int nwarps, cudaStream_t st);
int lookahead_warm(cudaStream_t st);
int tf32_reserve(size_t bytes, cudaStream_t st);
template <typename T>
int potrf_batched_small_t(T* A, int64_t n, int64_t lda, int64_t stride, int batch, int32_t* info, T* dinv, cudaStream_t st);
int kaux_impl(const gpk_kaux_desc* d, const void* X, int64_t N, int64_t ldx, const void* X2, int64_t N2, int64_t ldx2,
              void* K, int64_t ldk, int dtype, cudaStream_t st);
int kaux_diag_impl(const gpk_kaux_desc* d, const void* X, int64_t N, int64_t ldx, void* out, int dtype, cudaStream_t st);
int cp_weights_impl(const void* X, int64_t N, int64_t ldx, int dim, int has_lo, double loc_lo, double steep_lo,
                    int has_hi, double loc_hi, double steep_hi, void* out, int dtype, cudaStream_t st);
int hadamard_impl(int64_t m, int64_t n, const void* X, int64_t ldx, void* Y, int64_t ldy, int dtype, cudaStream_t st);
int clamp_min_impl(void* A, int64_t m, int64_t n, int64_t lda, double lower, int square, int dtype, cudaStream_t st);
int potrf_last_slices();
size_t gpr_lml_ws(int64_t N, int64_t P, int dtype);
int gpr_lml(const gpk_knode*, int, const int32_t*, const double*, const void*, int64_t, int64_t, int64_t, const void*,
            int64_t, double, const void*, int, double*, void*, cudaStream_t);
size_t gpr_lml_grad_ws(int64_t N, int64_t P, int dtype);
size_t gpr_lml_grad_alpha(int64_t N, int64_t P, int dtype);
int gpr_lml_grad_expr(const gpk_knode*, int, const int32_t*, const double*, const void*, int64_t, int64_t, int64_t,
                      const void*, int64_t, double, int, double*, int, void*, cudaStream_t);
size_t sgpr_elbo_ws(int64_t N, int64_t M, int64_t P, int dtype);
int sgpr_elbo(const gpk_knode*, int, const int32_t*, const double*, const void*, int64_t, int64_t, int64_t, const void*,
              int64_t, const void*, int64_t, int64_t, double, double, int, double*, void*, void*, void*, void*,
              cudaStream_t);
size_t sgpr_elbo_grad_ws(int64_t N, int64_t M, int64_t P, int dtype);
size_t sgpr_elbo_grad_dm(int64_t N, int64_t M, int64_t P, int dtype);
int sgpr_elbo_grad(const gpk_knode*, int, const int32_t*, const double*, const void*, int64_t, int64_t, int64_t,
                   const void*, int64_t, const void*, int64_t, int64_t, double, double, int, double*, int, double*,
                   void*, cudaStream_t);
size_t cglb_elbo_ws(int64_t N, int64_t M, int64_t P);
size_t cglb_elbo_grad_ws(int64_t N, int64_t M, int64_t P);
size_t cglb_elbo_grad_dm(int64_t N, int64_t M, int64_t P);
int cglb_elbo_grad(const gpk_knode*, int, const int32_t*, const double*, const double*, int64_t, int64_t, int64_t,
                   const double*, int64_t, const double*, int64_t, int64_t, double, double, double*, int, double, int,
                   int, double*, int, double*, double*, void*, cudaStream_t);
int cglb_elbo(const gpk_knode*, int, const int32_t*, const double*, const double*, int64_t, int64_t, int64_t,
              const double*, int64_t, const double*, int64_t, int64_t, double, double, double*, int, double, int, int,
              double*, void*, cudaStream_t);
int rbf_psi(const gpk_knode*, int, const int32_t*, const double*, const double*, const double*, int64_t, int64_t,
            const double*, int64_t, int64_t, double*, double*, double*, void*, cudaStream_t);
int rbf_psi_grad_debug(const gpk_knode*, int, const int32_t*, const double*, const double*, const double*, int64_t,
                       int64_t, const double*, int64_t, int64_t, const double*, int64_t, const double*, int64_t,
                       double*, double*, double*, double*, void*, int64_t*, cudaStream_t);
size_t bgplvm_elbo_ws(int64_t N, int64_t Q, int64_t M, int64_t P);
int bgplvm_elbo(const gpk_knode*, int, const int32_t*, const double*, const double*, const double*, int64_t, int64_t,
                const double*, int64_t, const double*, int64_t, int64_t, const double*, const double*, double, double,
                double*, void*, cudaStream_t);
size_t bgplvm_elbo_grad_ws(int64_t N, int64_t Q, int64_t M, int64_t P);
int bgplvm_elbo_grad(const gpk_knode*, int, const int32_t*, const double*, const double*, const double*, int64_t,
                     int64_t, const double*, int64_t, const double*, int64_t, int64_t, const double*, const double*,
                     double, double, double*, int, double*, double*, double*, void*, cudaStream_t);
size_t svgp_elbo_ws(int64_t B, int64_t M, int64_t P, int dtype);
int svgp_elbo(const gpk_knode*, int, const int32_t*, const double*, const void*, int64_t, int64_t, int64_t, const void*,
              const void*, int64_t, const void*, int64_t, int64_t, const void*, const void*, int, int, const gpk_lik*,
              double, double, int, int, int, double*, void*, cudaStream_t, int stage = 0, int64_t c0 = 0,
              int64_t c1 = 0);
size_t svgp_elbo_A(int64_t B, int64_t M, int64_t P, int dtype, int64_t* ld);
void svgp_elbo_fmu_fvar(int64_t B, int64_t M, int64_t P, int dtype, int64_t* fmu, int64_t* fvar);
size_t svgp_elbo_grad_ws(int64_t B, int64_t M, int64_t P, const gpk_lik* lik, int dtype);
size_t svgp_elbo_grad_dm(int64_t B, int64_t M, int64_t P, int dtype);
int svgp_elbo_grad(const gpk_knode*, int, const int32_t*, const double*, const void*, int64_t, int64_t, int64_t,
                   const void*, const void*, int64_t, const void*, int64_t, int64_t, const void*, const void*, int, int,
                   const gpk_lik*, double, double, int, double*, int, double*, double*, double*, void*, cudaStream_t);
size_t svgp_mo_elbo_grad_ws(int64_t B, int64_t M, int64_t L, int64_t P);
size_t svgp_mo_elbo_grad_dm(int64_t B, int64_t M, int64_t L, int64_t P);
int svgp_mo_elbo_grad(const gpk_kexpr*, int, const void*, int64_t, int64_t, int64_t, const void*, const void*, int64_t,
                      const void* const*, int, int64_t, int64_t, int64_t, const void*, const void*, int, int,
                      const void*, const gpk_lik*, double, double, int, double*, int, double* const*, double*, double*,
                      double*, void*, cudaStream_t);
size_t vgp_elbo_grad_ws(int64_t N, int64_t P, int dtype);
size_t vgp_elbo_grad_dm(int64_t N, int64_t P, int dtype);
int vgp_elbo_grad(const gpk_knode*, int, const int32_t*, const double*, const void*, int64_t, int64_t, int64_t,
                  const void*, int64_t, const void*, const void*, double, double, int, double*, int, double*, double*,
                  void*, cudaStream_t);
size_t vgp_oa_elbo_grad_ws(int64_t N, int64_t P);
size_t vgp_oa_elbo_grad_dm(int64_t N, int64_t P);
int vgp_oa_elbo_grad(const gpk_knode*, int, const int32_t*, const double*, const void*, int64_t, int64_t, int64_t,
                     const void*, const void*, int64_t, const double*, const double*, const gpk_lik*, int, double*, int,
                     double*, double*, void*, cudaStream_t);
size_t natgrad_step_ws(int64_t M, int xi);
int natgrad_step(int xi, int64_t M, int64_t P, const double* q_mu, const double* q_sqrt, const double* dq_mu,
                 const double* dq_sqrt, double gamma, double* q_mu_out, double* q_sqrt_out, int32_t* info, void* ws,
                 cudaStream_t st);
int adam_step(const gpk_adam_seg* segs, int n_segs, double lr_t, double beta_1, double beta_2, double epsilon,
              double sign, cudaStream_t st);

}  // namespace gpk

using namespace gpk;

#define GPK_DTYPE_OK(name) GPK_CHECK_ARG(dtype == GPK_F32 || dtype == GPK_F64, name ": bad dtype %d", dtype)

extern "C" {

int gpk_version(void) { return GPK_VERSION; }

int64_t gpk_launch_count(void) { return (int64_t)g_launches.load(); }
void gpk_launch_count_reset(void) { g_launches.store(0); }

int gpk_debug_leaf(void* A, int64_t lda, int n, void* dinv, void* dbg, int slim, void* stream) {
  return leaf_debug((double*)A, lda, n, (double*)dinv, (long long*)dbg, slim, (cudaStream_t)stream);
}

int gpk_debug_syrk_i8(const void* A, int64_t lda, int64_t r0, int64_t k0, int64_t K, void* C, int64_t ldc, int64_t m,
                      int64_t n, int lower, int S, int cluster, void* rowscale_out, void* head_flag, void* stream) {
  return tc_debug_syrk((const double*)A, lda, r0, k0, K, (double*)C, ldc, m, n, lower, S, cluster, (double*)rowscale_out,
                       (int*)head_flag, (cudaStream_t)stream);
}

size_t gpk_debug_inverse_chain_ws(int op, int64_t n) {
  // potri_lower's scratch: the [n1, n2] product of the top split, n1, n2 <= n / 2 + 128
  return op == GPK_CHAIN_POTRI && n > 0 ? (size_t)(n / 2 + 128) * (size_t)(n / 2 + 128) * sizeof(double) : 0;
}

int gpk_debug_inverse_chain(int op, double* L, int64_t n, int64_t ld, const double* dinv, double* T, double* out,
                            int64_t ldo, void* ws, void* stream) {
  GPK_CHECK_ARG(L && out && n >= 0 && ld >= n && ldo >= n, "debug_inverse_chain: bad arguments");
  if (n == 0) return 0;
  const cudaStream_t st = (cudaStream_t)stream;
  switch (op) {
    case GPK_CHAIN_POTRI:
      GPK_CHECK_ARG(dinv && ws, "debug_inverse_chain: POTRI needs dinv and ws");
      return potri_lower(L, n, ld, dinv, out, ldo, (double*)ws, st);
    case GPK_CHAIN_LAUUM:
      return lauum_lower(L, n, ld, out, ldo, st);
    case GPK_CHAIN_CHOL_ADJOINT:
      GPK_CHECK_ARG(dinv && T && ldo == ld, "debug_inverse_chain: CHOL_ADJOINT needs dinv, T and ldo == ld");
      return chol_adjoint(L, dinv, n, ld, T, out, st);
    default:
      GPK_CHECK_ARG(false, "debug_inverse_chain: bad op %d", op);
  }
  return 0;
}

int gpk_debug_gemm_tf32_batched(int transa, int transb, int64_t m, int64_t n, int64_t k, float alpha, const float* A,
                                int64_t lda, const float* B, int64_t ldb, float beta, float* C, int64_t ldc, int flags,
                                int batch, int64_t a_batch_stride, int64_t c_batch_stride, void* stream) {
  GPK_CHECK_ARG(A && B && C && m > 0 && n > 0 && k > 0 && batch >= 1, "debug_gemm_tf32_batched: bad arguments");
  return gemm_tf32(transa, transb, m, n, k, alpha, A, lda, B, ldb, beta, C, ldc, flags, (cudaStream_t)stream, batch,
                   a_batch_stride, c_batch_stride);
}

int gpk_debug_rbf_psi_grad(const gpk_knode* nodes, int n_nodes, const int32_t* dims, const double* ard,
                           const double* mu, const double* S, int64_t N, int64_t Q, const double* Z, int64_t M,
                           int64_t ldz, const double* G1t, int64_t ldg1, const double* G2, int64_t ldg2, double* dmu,
                           double* dS, double* dZ, double* gpar, void* ws, int64_t* geom, void* stream) {
  return rbf_psi_grad_debug(nodes, n_nodes, dims, ard, mu, S, N, Q, Z, M, ldz, G1t, ldg1, G2, ldg2, dmu, dS, dZ, gpar,
                            ws, geom, (cudaStream_t)stream);
}

int gpk_debug_trace(void* buf, void* pos, unsigned int capacity) {
  TraceBuf tb{(unsigned long long*)buf, (unsigned int*)pos, buf ? capacity : 0u};
  GPK_TRY(trace_set_potrf(tb));
  GPK_TRY(trace_set_tc(tb));
  return 0;
}

int gpk_prof_enable(int on) {
  for (auto& r : g_recs) { cudaEventDestroy(r.a); cudaEventDestroy(r.b); }
  g_recs.clear();
  g_prof = on != 0;
  return 0;
}

int gpk_peak_probe(double* out_host, void* stream) {
  GPK_CHECK_ARG(out_host, "peak_probe: bad arguments");
  return peak_probe(out_host, (cudaStream_t)stream);
}

int gpk_debug_dmma16816(const double* A, const double* B, const double* C, double* D, int nwarps, void* stream) {
  GPK_CHECK_ARG(A && B && C && D && nwarps > 0, "debug_dmma16816: bad arguments");
  return debug_dmma16816(A, B, C, D, nwarps, (cudaStream_t)stream);
}

int gpk_prof_read(double* ms, int64_t* launches, int n) { return gpk_prof_read2(ms, launches, nullptr, n); }

int gpk_potrf_last_slices(void) { return potrf_last_slices(); }

int gpk_warm(size_t tf32_scratch_bytes, void* stream) {
  GPK_TRY(lookahead_warm((cudaStream_t)stream));
  if (tf32_scratch_bytes) GPK_TRY(tf32_reserve(tf32_scratch_bytes, (cudaStream_t)stream));
  return 0;
}

int gpk_kaux(const gpk_kaux_desc* desc, const void* X, int64_t N, int64_t ldx, const void* X2, int64_t N2, int64_t ldx2, void* K,
             int64_t ldk, int dtype, void* stream) {
  GPK_DTYPE_OK("kaux");
  return kaux_impl(desc, X, N, ldx, X2, N2, ldx2, K, ldk, dtype, (cudaStream_t)stream);
}
int gpk_kaux_diag(const gpk_kaux_desc* desc, const void* X, int64_t N, int64_t ldx, void* out, int dtype, void* stream) {
  GPK_DTYPE_OK("kaux_diag");
  return kaux_diag_impl(desc, X, N, ldx, out, dtype, (cudaStream_t)stream);
}
int gpk_changepoint_weights(const void* X, int64_t N, int64_t ldx, int dim, int has_lo, double loc_lo, double steep_lo,
                            int has_hi, double loc_hi, double steep_hi, void* out, int dtype, void* stream) {
  GPK_DTYPE_OK("changepoint_weights");
  return cp_weights_impl(X, N, ldx, dim, has_lo, loc_lo, steep_lo, has_hi, loc_hi, steep_hi, out, dtype,
                         (cudaStream_t)stream);
}
int gpk_clamp_min(void* A, int64_t m, int64_t n, int64_t lda, double lower, int square, int dtype, void* stream) {
  GPK_DTYPE_OK("clamp_min");
  return clamp_min_impl(A, m, n, lda, lower, square, dtype, (cudaStream_t)stream);
}
int gpk_hadamard(int64_t m, int64_t n, const void* X, int64_t ldx, void* Y, int64_t ldy, int dtype, void* stream) {
  GPK_DTYPE_OK("hadamard");
  return hadamard_impl(m, n, X, ldx, Y, ldy, dtype, (cudaStream_t)stream);
}

int gpk_prof_read2(double* ms, int64_t* launches, double* work, int n) {
  GPK_CHECK_ARG(ms && launches && n > 0, "prof_read: bad arguments");
  for (int i = 0; i < n; ++i) { ms[i] = 0.0; launches[i] = 0; if (work) work[i] = 0.0; }
  GPK_CUDA_OK(cudaDeviceSynchronize());
  for (auto& r : g_recs) {
    float t = 0.f;
    if (cudaEventElapsedTime(&t, r.a, r.b) == cudaSuccess && r.cls < n) {
      ms[r.cls] += t;
      launches[r.cls] += 1;
      if (work) work[r.cls] += r.work;
    }
    cudaEventDestroy(r.a);
    cudaEventDestroy(r.b);
  }
  g_recs.clear();
  return 0;
}
const char* gpk_last_error(void) { return g_err; }

int gpk_kbuild(const gpk_knode* nodes, int n_nodes, const int32_t* dims, const double* ard, const void* X, int64_t N,
               int64_t ldx, const void* X2, int64_t N2, int64_t ldx2, int64_t D, void* K, int64_t ldk, int dtype,
               int uplo, double diag_scalar, const void* diag_vec, void* stream) {
  return kbuild_impl(nodes, n_nodes, dims, ard, X, N, ldx, X2, N2, ldx2, D, K, ldk, dtype, uplo, diag_scalar, diag_vec,
                     (cudaStream_t)stream);
}

int gpk_kdiag(const gpk_knode* nodes, int n_nodes, const int32_t* dims, const double* ard, const void* X, int64_t N,
              int64_t ldx, int64_t D, void* out, int dtype, void* stream) {
  return kdiag_impl(nodes, n_nodes, dims, ard, X, N, ldx, D, out, dtype, (cudaStream_t)stream);
}

size_t gpk_potrf_ws(int64_t n, int64_t rows, int dtype) { return potrf_ws_bytes(n, rows < n ? n : rows, dtype); }

int gpk_potrf(void* A, int64_t n, int64_t rows, int64_t lda, int dtype, int32_t* info, void* ws, void* stream) {
  GPK_DTYPE_OK("potrf");
  GPK_CHECK_ARG(A && ws && n >= 0 && rows >= n && lda >= n, "potrf: bad arguments (n=%lld rows=%lld lda=%lld)",
                (long long)n, (long long)rows, (long long)lda);
  return potrf_any(A, n, rows, lda, dtype, info, ws, (cudaStream_t)stream);
}

size_t gpk_potrf_batched_ws(int64_t n, int batch, int dtype) {
  if (n <= NB) return (size_t)(batch > 0 ? batch : 1) * NB * NB * dtype_size(dtype);  // one inverse slot per matrix
  return potrf_ws_bytes(n, n, dtype);
}

int gpk_potrf_batched(void* A, int64_t n, int64_t lda, int64_t stride, int batch, int dtype, int32_t* info, void* ws,
                      void* stream) {
  GPK_DTYPE_OK("potrf_batched");
  GPK_CHECK_ARG(A && ws && n >= 0 && lda >= n && batch >= 0, "potrf_batched: bad arguments");
  if (n <= NB) {  // the whole batch in ONE launch: grid over the matrices
    if (dtype == GPK_F64)
      return potrf_batched_small_t<double>((double*)A, n, lda, stride, batch, info, (double*)ws, (cudaStream_t)stream);
    return potrf_batched_small_t<float>((float*)A, n, lda, stride, batch, info, (float*)ws, (cudaStream_t)stream);
  }
  // larger matrices: each factorisation already fills the GPU; they run back to back on the stream and share the workspace
  for (int b = 0; b < batch; ++b)
    GPK_TRY(potrf_any((char*)A + (size_t)b * stride * dtype_size(dtype), n, n, lda, dtype, info ? info + b : nullptr,
                      ws, (cudaStream_t)stream));
  return 0;
}

size_t gpk_trsm_ws(int64_t n, int dtype) { return dinv_bytes(n, dtype); }

int gpk_trsm(int trans, const void* L, int64_t n, int64_t ldl, void* B, int64_t nrhs, int64_t ldb, int dtype,
             const void* dinv, void* ws, void* stream) {
  GPK_DTYPE_OK("trsm");
  GPK_CHECK_ARG(L && B && n >= 0 && nrhs >= 0 && ldl >= n && ldb >= nrhs, "trsm: bad arguments");
  GPK_CHECK_ARG(dinv || ws, "trsm: need either cached diagonal-block inverses or a workspace");
  if (!dinv) {
    GPK_TRY(trtri_diag_any(L, n, ldl, ws, dtype, (cudaStream_t)stream));
    dinv = ws;
  }
  return trsm_any(trans, L, n, ldl, B, nrhs, ldb, dtype, dinv, (cudaStream_t)stream);
}

int gpk_gemm(int transa, int transb, int64_t m, int64_t n, int64_t k, double alpha, const void* A, int64_t lda,
             const void* B, int64_t ldb, double beta, void* C, int64_t ldc, int dtype, int flags, void* stream) {
  GPK_DTYPE_OK("gemm");
  GPK_CHECK_ARG(A && B && C && m >= 0 && n >= 0 && k >= 0, "gemm: bad arguments");
  GPK_CHECK_ARG(lda >= (transa ? m : k) && ldb >= (transb ? k : n) && ((flags & GPK_GEMM_COLSUMSQ) || ldc >= n),
                "gemm: leading dimension too small");
  // In place, each element of the aliased operand must be read only by the CTA that overwrites it, and before it does.
  // C == B untransposed with ldb == ldc: a CTA reads B's columns [n0, n0 + BN), which only it stores, so one tile must
  // span m.  C == A likewise by rows, so one tile must span n.  The widest tile edge is 128; no tile spans both.
  const bool in_place_ok = C == A ? C != B && !transa && lda == ldc && n <= 128
                                  : C != B || (!transb && ldb == ldc && m <= 128);
  GPK_CHECK_ARG(in_place_ok,
                "gemm: in place needs C == B with transb = 0, ldb == ldc, m <= 128 or C == A with transa = 0, "
                "lda == ldc, n <= 128 (m=%lld n=%lld)", (long long)m, (long long)n);
  return gemm_any(transa, transb, m, n, k, alpha, A, lda, B, ldb, beta, C, ldc, dtype, flags, (cudaStream_t)stream);
}

int gpk_colsumsq(const void* A, int64_t m, int64_t n, int64_t lda, double scale, int accumulate, void* out, int dtype,
                 void* stream) {
  GPK_DTYPE_OK("colsumsq");
  return colsumsq_impl(A, m, n, lda, scale, accumulate, out, dtype, (cudaStream_t)stream);
}

int gpk_reduce(int f, const void* x, int64_t n, int64_t inc, double scale, int accumulate, double* out, int dtype,
               void* stream) {
  GPK_DTYPE_OK("reduce");
  return reduce_impl(f, x, n, inc, scale, accumulate, out, dtype, (cudaStream_t)stream);
}

int gpk_tril_sumsq(const void* A, int64_t n, int64_t lda, int64_t stride, int batch, double scale, int accumulate,
                   double* out, int dtype, void* stream) {
  GPK_DTYPE_OK("tril_sumsq");
  return tril_sumsq_impl(A, n, lda, stride, batch, scale, accumulate, out, dtype, (cudaStream_t)stream);
}

int gpk_axpby(int64_t m, int64_t n, double a, const void* X, int64_t ldx, double b, void* Y, int64_t ldy, int dtype,
              void* stream) {
  GPK_DTYPE_OK("axpby");
  return axpby_impl(m, n, a, X, ldx, b, Y, ldy, dtype, (cudaStream_t)stream);
}

int gpk_scale_cols(void* A, int64_t m, int64_t n, int64_t lda, const void* s, int invert, int dtype, void* stream) {
  GPK_DTYPE_OK("scale_cols");
  return scale_impl(A, m, n, lda, s, 0, invert, dtype, (cudaStream_t)stream);
}

int gpk_scale_rows(void* A, int64_t m, int64_t n, int64_t lda, const void* s, int invert, int dtype, void* stream) {
  GPK_DTYPE_OK("scale_rows");
  return scale_impl(A, m, n, lda, s, 1, invert, dtype, (cudaStream_t)stream);
}

int gpk_add_diag(void* A, int64_t n, int64_t lda, double scalar, const void* vec, int dtype, void* stream) {
  GPK_DTYPE_OK("add_diag");
  return add_diag_impl(A, n, lda, scalar, vec, dtype, (cudaStream_t)stream);
}

int gpk_fill(void* A, int64_t m, int64_t n, int64_t lda, double value, int dtype, void* stream) {
  GPK_DTYPE_OK("fill");
  return fill_impl(A, m, n, lda, value, dtype, (cudaStream_t)stream);
}

int gpk_tril(void* A, int64_t n, int64_t lda, int64_t stride, int batch, int dtype, void* stream) {
  GPK_DTYPE_OK("tril");
  return tril_impl(A, n, lda, stride, batch, dtype, (cudaStream_t)stream);
}

int gpk_transpose(const void* A, int64_t m, int64_t n, int64_t lda, void* B, int64_t ldb, int dtype, void* stream) {
  GPK_DTYPE_OK("transpose");
  return transpose_impl(A, m, n, lda, B, ldb, dtype, (cudaStream_t)stream);
}

// gpflow/likelihoods/base.py:344-400 and the closed forms of scalar_discrete.py / scalar_continuous.py
int gpk_lik_varexp_sum(const gpk_lik* lik, const void* Fmu, const void* Fvar, const void* Y, int64_t B, int64_t P,
                       double scale, int accumulate, double* out, int dtype, void* stream) {
  GPK_DTYPE_OK("lik_varexp_sum");
  return lik_varexp_impl(lik, Fmu, Fvar, Y, nullptr, B, P, lik_ldy(lik, P), P, P, 1, scale, accumulate, out, dtype,
                         (cudaStream_t)stream);
}

int gpk_lik_varexp_grad(const gpk_lik* lik, const double* Fmu, const double* Fvar, const double* Y, int64_t B,
                        int64_t P, double scale, double* R, double* Wt, double* dpar, void* stream) {
  GPK_CHECK_ARG(Fmu && Fvar && Y && R && Wt && dpar, "lik_varexp_grad: null argument");
  if (B <= 0) return lik_check(lik, P, "lik_varexp_grad");
  return lik_grad_impl(lik, Fmu, Fvar, Y, lik_ldy(lik, P), nullptr, B, P, scale, R, Wt, dpar, (cudaStream_t)stream);
}

int gpk_lik_predict_mean_and_var(const gpk_lik* lik, const void* Fmu, const void* Fvar, int64_t N, int64_t P,
                                 void* mean, void* var, int dtype, void* stream) {
  GPK_DTYPE_OK("lik_predict_mean_and_var");
  return lik_predict_mv_impl(lik, Fmu, Fvar, N, P, mean, var, dtype, (cudaStream_t)stream);
}

int gpk_lik_predict_log_density(const gpk_lik* lik, const void* Fmu, const void* Fvar, const void* Y, int64_t N,
                                int64_t P, void* out, int dtype, void* stream) {
  GPK_DTYPE_OK("lik_predict_log_density");
  return lik_predict_ld_impl(lik, Fmu, Fvar, Y, N, P, out, dtype, (cudaStream_t)stream);
}

size_t gpk_gpr_lml_ws(int64_t N, int64_t P, int dtype) { return gpr_lml_ws(N, P, dtype); }

int gpk_gpr_lml(const gpk_knode* nodes, int n_nodes, const int32_t* dims, const double* ard, const void* X, int64_t N,
                int64_t ldx, int64_t D, const void* Yc, int64_t P, double noise_variance, const void* noise_vec,
                int dtype, double* out, void* ws, void* stream) {
  GPK_DTYPE_OK("gpr_lml");
  return gpr_lml(nodes, n_nodes, dims, ard, X, N, ldx, D, Yc, P, noise_variance, noise_vec, dtype, out, ws,
                 (cudaStream_t)stream);
}

size_t gpk_sgpr_elbo_ws(int64_t N, int64_t M, int64_t P, int dtype) { return sgpr_elbo_ws(N, M, P, dtype); }

int gpk_sgpr_elbo(const gpk_knode* nodes, int n_nodes, const int32_t* dims, const double* ard, const void* X, int64_t N,
                  int64_t ldx, int64_t D, const void* Yc, int64_t P, const void* Z, int64_t M, int64_t ldz,
                  double noise_variance, double jitter, int dtype, double* out, void* cache_L, void* cache_LB,
                  void* cache_c, void* ws, void* stream) {
  GPK_DTYPE_OK("sgpr_elbo");
  return sgpr_elbo(nodes, n_nodes, dims, ard, X, N, ldx, D, Yc, P, Z, M, ldz, noise_variance, jitter, dtype, out,
                   cache_L, cache_LB, cache_c, ws, (cudaStream_t)stream);
}

size_t gpk_svgp_elbo_ws(int64_t B, int64_t M, int64_t P, int dtype) { return svgp_elbo_ws(B, M, P, dtype); }

int gpk_svgp_elbo(const gpk_knode* nodes, int n_nodes, const int32_t* dims, const double* ard, const void* Xb, int64_t B,
                  int64_t ldx, int64_t D, const void* Y, const void* mX, int64_t P, const void* Z, int64_t M,
                  int64_t ldz, const void* q_mu, const void* q_sqrt, int q_diag, int whiten, const gpk_lik* lik,
                  double num_data_scale, double jitter, int p_begin, int p_end, int dtype, double* out, void* ws,
                  void* stream) {
  GPK_DTYPE_OK("svgp_elbo");
  return svgp_elbo(nodes, n_nodes, dims, ard, Xb, B, ldx, D, Y, mX, P, Z, M, ldz, q_mu, q_sqrt, q_diag, whiten, lik,
                   num_data_scale, jitter, p_begin, p_end, dtype, out, ws, (cudaStream_t)stream);
}

size_t gpk_gpr_lml_grad_ws(int64_t N, int64_t P, int dtype) { return gpr_lml_grad_ws(N, P, dtype); }

size_t gpk_gpr_lml_grad_alpha(int64_t N, int64_t P, int dtype) { return gpr_lml_grad_alpha(N, P, dtype); }

int gpk_gpr_lml_grad_slots(const gpk_knode* nodes, int n_nodes, const int32_t* dims, const double* ard, int64_t D) {
  return grad_expr_slots(nodes, n_nodes, dims, ard, D, "gpr_lml_grad_slots");
}

int gpk_gpr_lml_grad_expr(const gpk_knode* nodes, int n_nodes, const int32_t* dims, const double* ard, const void* X,
                          int64_t N, int64_t ldx, int64_t D, const void* Yc, int64_t P, double noise_variance, int dtype,
                          double* out, int n_out, void* ws, void* stream) {
  GPK_DTYPE_OK("gpr_lml_grad_expr");
  return gpr_lml_grad_expr(nodes, n_nodes, dims, ard, X, N, ldx, D, Yc, P, noise_variance, dtype, out, n_out, ws,
                           (cudaStream_t)stream);
}

size_t gpk_sgpr_elbo_grad_ws(int64_t N, int64_t M, int64_t P, int dtype) { return sgpr_elbo_grad_ws(N, M, P, dtype); }

size_t gpk_sgpr_elbo_grad_dm(int64_t N, int64_t M, int64_t P, int dtype) { return sgpr_elbo_grad_dm(N, M, P, dtype); }

int gpk_sgpr_elbo_grad(const gpk_knode* nodes, int n_nodes, const int32_t* dims, const double* ard, const void* X,
                       int64_t N, int64_t ldx, int64_t D, const void* Yc, int64_t P, const void* Z, int64_t M,
                       int64_t ldz, double noise_variance, double jitter, int dtype, double* out, int n_out, double* dZ,
                       void* ws, void* stream) {
  GPK_DTYPE_OK("sgpr_elbo_grad");
  return sgpr_elbo_grad(nodes, n_nodes, dims, ard, X, N, ldx, D, Yc, P, Z, M, ldz, noise_variance, jitter, dtype, out,
                        n_out, dZ, ws, (cudaStream_t)stream);
}

size_t gpk_kmv_ws(int64_t N, int64_t N2, int64_t P) { return kmv_ws_bytes(N, N2, P); }

// replaces the product v @ K of gpflow/models/cglb.py:143, 384, 390 without forming K
int gpk_kmv(const gpk_knode* nodes, int n_nodes, const int32_t* dims, const double* ard, const double* X, int64_t N,
            int64_t ldx, const double* X2, int64_t N2, int64_t ldx2, int64_t D, const double* V, int64_t P, int64_t ldv,
            double diag_scalar, double* out, int64_t ldo, void* ws, void* stream) {
  return kmv_impl(nodes, n_nodes, dims, ard, X, N, ldx, X2, N2, ldx2, D, V, P, ldv, diag_scalar, out, ldo, ws, nullptr,
                  (cudaStream_t)stream);
}

size_t gpk_cglb_elbo_ws(int64_t N, int64_t M, int64_t P) { return cglb_elbo_ws(N, M, P); }

// replaces gpflow/models/cglb.py:83-160 (the bound, with the CG loop of cglb.py:343-420)
int gpk_cglb_elbo(const gpk_knode* nodes, int n_nodes, const int32_t* dims, const double* ard, const double* X,
                  int64_t N, int64_t ldx, int64_t D, const double* Yc, int64_t P, const double* Z, int64_t M,
                  int64_t ldz, double noise_variance, double jitter, double* v, int run_cg, double cg_tolerance,
                  int max_cg_iters, int restart_cg_iters, double* out, void* ws, void* stream) {
  return cglb_elbo(nodes, n_nodes, dims, ard, X, N, ldx, D, Yc, P, Z, M, ldz, noise_variance, jitter, v, run_cg,
                   cg_tolerance, max_cg_iters, restart_cg_iters, out, ws, (cudaStream_t)stream);
}

size_t gpk_cglb_elbo_grad_ws(int64_t N, int64_t M, int64_t P) { return cglb_elbo_grad_ws(N, M, P); }
size_t gpk_cglb_elbo_grad_dm(int64_t N, int64_t M, int64_t P) { return cglb_elbo_grad_dm(N, M, P); }

// replaces TensorFlow autodiff through gpflow/models/cglb.py:83-160 (v held fixed when CG chose it)
int gpk_cglb_elbo_grad(const gpk_knode* nodes, int n_nodes, const int32_t* dims, const double* ard, const double* X,
                       int64_t N, int64_t ldx, int64_t D, const double* Yc, int64_t P, const double* Z, int64_t M,
                       int64_t ldz, double noise_variance, double jitter, double* v, int run_cg, double cg_tolerance,
                       int max_cg_iters, int restart_cg_iters, double* out, int n_out, double* dZ, double* dv,
                       void* ws, void* stream) {
  return cglb_elbo_grad(nodes, n_nodes, dims, ard, X, N, ldx, D, Yc, P, Z, M, ldz, noise_variance, jitter, v, run_cg,
                        cg_tolerance, max_cg_iters, restart_cg_iters, out, n_out, dZ, dv, ws, (cudaStream_t)stream);
}

size_t gpk_rbf_psi_ws(int64_t N, int64_t M) { return psi_ws_bytes(N, M); }

// replaces the RBF expectations of gpflow/expectations/squared_exponentials.py:49-96, 207-292 (psi2 summed over n)
int gpk_rbf_psi(const gpk_knode* nodes, int n_nodes, const int32_t* dims, const double* ard, const double* mu,
                const double* S, int64_t N, int64_t Q, const double* Z, int64_t M, int64_t ldz, double* psi0,
                double* psi1, double* psi2, void* ws, void* stream) {
  return rbf_psi(nodes, n_nodes, dims, ard, mu, S, N, Q, Z, M, ldz, psi0, psi1, psi2, ws, (cudaStream_t)stream);
}

size_t gpk_bgplvm_elbo_ws(int64_t N, int64_t Q, int64_t M, int64_t P) { return bgplvm_elbo_ws(N, Q, M, P); }

int gpk_bgplvm_elbo(const gpk_knode* nodes, int n_nodes, const int32_t* dims, const double* ard, const double* mu,
                    const double* S, int64_t N, int64_t Q, const double* Y, int64_t P, const double* Z, int64_t M,
                    int64_t ldz, const double* prior_mean, const double* prior_var, double noise_variance,
                    double jitter, double* out, void* ws, void* stream) {
  return bgplvm_elbo(nodes, n_nodes, dims, ard, mu, S, N, Q, Y, P, Z, M, ldz, prior_mean, prior_var, noise_variance,
                     jitter, out, ws, (cudaStream_t)stream);
}

size_t gpk_bgplvm_elbo_grad_ws(int64_t N, int64_t Q, int64_t M, int64_t P) { return bgplvm_elbo_grad_ws(N, Q, M, P); }

// replaces TensorFlow autodiff through gplvm.py:162-216 and the psi statistics
int gpk_bgplvm_elbo_grad(const gpk_knode* nodes, int n_nodes, const int32_t* dims, const double* ard,
                         const double* mu, const double* S, int64_t N, int64_t Q, const double* Y, int64_t P,
                         const double* Z, int64_t M, int64_t ldz, const double* prior_mean, const double* prior_var,
                         double noise_variance, double jitter, double* out, int n_out, double* dmu, double* dS,
                         double* dZ, void* ws, void* stream) {
  return bgplvm_elbo_grad(nodes, n_nodes, dims, ard, mu, S, N, Q, Y, P, Z, M, ldz, prior_mean, prior_var,
                          noise_variance, jitter, out, n_out, dmu, dS, dZ, ws, (cudaStream_t)stream);
}

size_t gpk_svgp_elbo_grad_ws(int64_t B, int64_t M, int64_t P, const gpk_lik* lik, int dtype) {
  return svgp_elbo_grad_ws(B, M, P, lik, dtype);
}

size_t gpk_svgp_elbo_grad_dm(int64_t B, int64_t M, int64_t P, int dtype) { return svgp_elbo_grad_dm(B, M, P, dtype); }

// replaces TensorFlow autodiff through svgp.py:166-181 (conditionals/util.py:84-169, kullback_leiblers.py:59-165; the
// quadrature of likelihoods/base.py:361-376 and scalar_discrete.py:67-78 for the non-Gaussian likelihoods)
int gpk_svgp_elbo_grad(const gpk_knode* nodes, int n_nodes, const int32_t* dims, const double* ard, const void* Xb,
                       int64_t B, int64_t ldx, int64_t D, const void* Y, const void* mX, int64_t P, const void* Z,
                       int64_t M, int64_t ldz, const void* q_mu, const void* q_sqrt, int q_diag, int whiten,
                       const gpk_lik* lik, double num_data_scale, double jitter, int dtype, double* out, int n_out,
                       double* dZ, double* dq_mu, double* dq_sqrt, void* ws, void* stream) {
  GPK_DTYPE_OK("svgp_elbo_grad");
  return svgp_elbo_grad(nodes, n_nodes, dims, ard, Xb, B, ldx, D, Y, mX, P, Z, M, ldz, q_mu, q_sqrt, q_diag, whiten, lik,
                        num_data_scale, jitter, dtype, out, n_out, dZ, dq_mu, dq_sqrt, ws, (cudaStream_t)stream);
}

size_t gpk_svgp_mo_elbo_grad_ws(int64_t B, int64_t M, int64_t L, int64_t P, const gpk_lik* lik, int dtype) {
  (void)lik;
  (void)dtype;
  return svgp_mo_elbo_grad_ws(B, M, L, P);
}

size_t gpk_svgp_mo_elbo_grad_dm(int64_t B, int64_t M, int64_t L, int64_t P, int dtype) {
  (void)dtype;
  return svgp_mo_elbo_grad_dm(B, M, L, P);
}

// replaces TensorFlow autodiff through svgp.py:166-181 for a multi-output kernel (conditionals/multioutput/
// conditionals.py:45-152,261-311 with the mixing of conditionals/util.py:518-563)
int gpk_svgp_mo_elbo_grad(const gpk_kexpr* kernels, int n_kernels, const void* Xb, int64_t B, int64_t ldx, int64_t D,
                          const void* Y, const void* mX, int64_t P, const void* const* Z, int n_z, int64_t M,
                          int64_t ldz, int64_t L, const void* q_mu, const void* q_sqrt, int q_diag, int whiten,
                          const void* W, const gpk_lik* lik, double num_data_scale, double jitter, int dtype,
                          double* out, int n_out, double* const* dZ, double* dq_mu, double* dq_sqrt, double* dW,
                          void* ws, void* stream) {
  GPK_DTYPE_OK("svgp_mo_elbo_grad");
  return svgp_mo_elbo_grad(kernels, n_kernels, Xb, B, ldx, D, Y, mX, P, Z, n_z, M, ldz, L, q_mu, q_sqrt, q_diag, whiten,
                           W, lik, num_data_scale, jitter, dtype, out, n_out, dZ, dq_mu, dq_sqrt, dW, ws,
                           (cudaStream_t)stream);
}

size_t gpk_vgp_elbo_grad_ws(int64_t N, int64_t P, int dtype) { return vgp_elbo_grad_ws(N, P, dtype); }

size_t gpk_vgp_elbo_grad_dm(int64_t N, int64_t P, int dtype) { return vgp_elbo_grad_dm(N, P, dtype); }

// replaces TensorFlow autodiff through vgp.py:111-143 (kullback_leiblers.py:59-165, scalar_continuous.py:139-148)
int gpk_vgp_elbo_grad(const gpk_knode* nodes, int n_nodes, const int32_t* dims, const double* ard, const void* X,
                      int64_t N, int64_t ldx, int64_t D, const void* Yc, int64_t P, const void* q_mu,
                      const void* q_sqrt, double noise_variance, double jitter, int dtype, double* out, int n_out,
                      double* dq_mu, double* dq_sqrt, void* ws, void* stream) {
  GPK_DTYPE_OK("vgp_elbo_grad");
  return vgp_elbo_grad(nodes, n_nodes, dims, ard, X, N, ldx, D, Yc, P, q_mu, q_sqrt, noise_variance, jitter, dtype, out,
                       n_out, dq_mu, dq_sqrt, ws, (cudaStream_t)stream);
}

size_t gpk_vgp_oa_elbo_grad_ws(int64_t N, int64_t P, int dtype) {
  (void)dtype;
  return vgp_oa_elbo_grad_ws(N, P);
}

size_t gpk_vgp_oa_elbo_grad_dm(int64_t N, int64_t P, int dtype) {
  (void)dtype;
  return vgp_oa_elbo_grad_dm(N, P);
}

// replaces TensorFlow autodiff through vgp.py:325-376 (the likelihood's variational expectations as in
// gpk_svgp_elbo_grad)
int gpk_vgp_oa_elbo_grad(const gpk_knode* nodes, int n_nodes, const int32_t* dims, const double* ard, const void* X,
                         int64_t N, int64_t ldx, int64_t D, const void* Y, const void* mX, int64_t P,
                         const double* q_alpha, const double* q_lambda, const gpk_lik* lik, int dtype, double* out,
                         int n_out, double* dq_alpha, double* dq_lambda, void* ws, void* stream) {
  GPK_DTYPE_OK("vgp_oa_elbo_grad");
  return vgp_oa_elbo_grad(nodes, n_nodes, dims, ard, X, N, ldx, D, Y, mX, P, q_alpha, q_lambda, lik, dtype, out, n_out,
                          dq_alpha, dq_lambda, ws, (cudaStream_t)stream);
}

size_t gpk_natgrad_step_ws(int64_t M, int64_t P, int xi, int dtype) {
  (void)P;
  (void)dtype;
  return M > 0 ? natgrad_step_ws(M, xi) : 0;
}

// replaces NaturalGradient._natgrad_apply_gradients (gpflow/optimizers/natgrad.py:280-367) with the conversions of
// natgrad.py:429-502 for the XiNat and XiSqrtMeanVar transforms
int gpk_natgrad_step(int xi, int64_t M, int64_t P, const void* q_mu, const void* q_sqrt, const double* dq_mu,
                     const double* dq_sqrt, double gamma, int dtype, void* q_mu_out, void* q_sqrt_out, int32_t* info,
                     void* ws, void* stream) {
  GPK_CHECK_ARG(dtype == GPK_F64, "natgrad_step: the natural-gradient step computes in float64 (dtype %d)", dtype);
  GPK_CHECK_ARG(xi == GPK_XI_NAT || xi == GPK_XI_SQRT_MEAN_VAR, "natgrad_step: bad xi transform %d", xi);
  GPK_CHECK_ARG(M > 0 && P > 0 && q_mu && q_sqrt && dq_mu && dq_sqrt && q_mu_out && q_sqrt_out && info && ws,
                "natgrad_step: bad arguments");
  GPK_CHECK_ARG(gamma > 0.0 && isfinite(gamma), "natgrad_step: gamma must be positive and finite (%g)", gamma);
  GPK_CHECK_ARG(q_mu_out != q_mu && q_sqrt_out != q_sqrt, "natgrad_step: the step is out of place");
  return natgrad_step(xi, M, P, (const double*)q_mu, (const double*)q_sqrt, dq_mu, dq_sqrt, gamma, (double*)q_mu_out,
                      (double*)q_sqrt_out, info, ws, (cudaStream_t)stream);
}

// replaces tf_keras.optimizers.Adam.apply_gradients on the unconstrained variables (gpflow/utilities/misc.py:76-109)
int gpk_adam_step(const gpk_adam_seg* segs, int n_segs, double lr_t, double beta_1, double beta_2, double epsilon,
                  double sign, int dtype, void* stream) {
  GPK_CHECK_ARG(dtype == GPK_F64, "adam_step: the Adam step computes in float64 (dtype %d)", dtype);
  GPK_CHECK_ARG(segs && n_segs >= 1 && n_segs <= GPK_ADAM_MAX_SEGS, "adam_step: n_segs %d outside [1, %d]", n_segs,
                GPK_ADAM_MAX_SEGS);
  GPK_CHECK_ARG(sign == 1.0 || sign == -1.0, "adam_step: sign must be +1 or -1 (%g)", sign);
  for (int s = 0; s < n_segs; ++s) {
    const gpk_adam_seg& g = segs[s];
    GPK_CHECK_ARG(g.n >= 0, "adam_step: segment %d has a negative length", s);
    GPK_CHECK_ARG(g.n == 0 || (g.value && g.grad && g.m && g.v), "adam_step: segment %d has a null pointer", s);
    GPK_CHECK_ARG(g.transform == GPK_ADAM_IDENTITY || g.transform == GPK_ADAM_SOFTPLUS || g.transform == GPK_ADAM_EXP,
                  "adam_step: segment %d has an unknown transform %d", s, g.transform);
    GPK_CHECK_ARG((((uintptr_t)g.value | (uintptr_t)g.grad | (uintptr_t)g.m | (uintptr_t)g.v) & 7) == 0,
                  "adam_step: segment %d has a pointer that is not 8-byte aligned", s);
  }
  return adam_step(segs, n_segs, lr_t, beta_1, beta_2, epsilon, sign, (cudaStream_t)stream);
}

size_t gpk_svgp_elbo_A(int64_t B, int64_t M, int64_t P, int dtype, int64_t* ld) { return svgp_elbo_A(B, M, P, dtype, ld); }

int gpk_svgp_elbo_fmu_fvar(int64_t B, int64_t M, int64_t P, int dtype, int64_t* fmu, int64_t* fvar) {
  GPK_DTYPE_OK("svgp_elbo_fmu_fvar");
  GPK_CHECK_ARG(B > 0 && M > 0 && P > 0 && fmu && fvar, "svgp_elbo_fmu_fvar: bad arguments");
  svgp_elbo_fmu_fvar(B, M, P, dtype, fmu, fvar);
  return 0;
}

int gpk_svgp_elbo_staged(const gpk_knode* nodes, int n_nodes, const int32_t* dims, const double* ard, const void* Xb,
                         int64_t B, int64_t ldx, int64_t D, const void* Y, const void* mX, int64_t P, const void* Z,
                         int64_t M, int64_t ldz, const void* q_mu, const void* q_sqrt, int q_diag, int whiten,
                         const gpk_lik* lik, double num_data_scale, double jitter, int p_begin, int p_end, int stage,
                         int64_t col_begin, int64_t col_end, int dtype, double* out, void* ws, void* stream) {
  GPK_DTYPE_OK("svgp_elbo_staged");
  return svgp_elbo(nodes, n_nodes, dims, ard, Xb, B, ldx, D, Y, mX, P, Z, M, ldz, q_mu, q_sqrt, q_diag, whiten, lik,
                   num_data_scale, jitter, p_begin, p_end, dtype, out, ws, (cudaStream_t)stream, stage, col_begin,
                   col_end);
}

}  // extern "C"
