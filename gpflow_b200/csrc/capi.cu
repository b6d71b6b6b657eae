// capi.cu — the library's error, launch-count and profiler state, the dtype-erased dispatch of the typed templates,
// and the extern "C" argument checks of the primitives (include/gpk.h) whose implementations other code also calls.
// Every other entry point is defined in the file that implements it.
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

int lookahead_warm(cudaStream_t st);
int tf32_reserve(size_t bytes, cudaStream_t st);
template <typename T>
int potrf_batched_small_t(T* A, int64_t n, int64_t lda, int64_t stride, int batch, int32_t* info, T* dinv, cudaStream_t st);

}  // namespace gpk

using namespace gpk;

extern "C" {

int gpk_version(void) { return GPK_VERSION; }

int64_t gpk_launch_count(void) { return (int64_t)g_launches.load(); }
void gpk_launch_count_reset(void) { g_launches.store(0); }

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

int gpk_prof_read(double* ms, int64_t* launches, int n) { return gpk_prof_read2(ms, launches, nullptr, n); }

int gpk_warm(size_t tf32_scratch_bytes, void* stream) {
  GPK_TRY(lookahead_warm((cudaStream_t)stream));
  if (tf32_scratch_bytes) GPK_TRY(tf32_reserve(tf32_scratch_bytes, (cudaStream_t)stream));
  return 0;
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

int gpk_gpr_lml_grad_slots(const gpk_knode* nodes, int n_nodes, const int32_t* dims, const double* ard, int64_t D) {
  return grad_expr_slots(nodes, n_nodes, dims, ard, D, "gpr_lml_grad_slots");
}

size_t gpk_kmv_ws(int64_t N, int64_t N2, int64_t P) { return kmv_ws_bytes(N, N2, P); }

// replaces the product v @ K of gpflow/models/cglb.py:143, 384, 390 without forming K
int gpk_kmv(const gpk_knode* nodes, int n_nodes, const int32_t* dims, const double* ard, const double* X, int64_t N,
            int64_t ldx, const double* X2, int64_t N2, int64_t ldx2, int64_t D, const double* V, int64_t P, int64_t ldv,
            double diag_scalar, double* out, int64_t ldo, void* ws, void* stream) {
  return kmv_impl(nodes, n_nodes, dims, ard, X, N, ldx, X2, N2, ldx2, D, V, P, ldv, diag_scalar, out, ldo, ws, nullptr,
                  (cudaStream_t)stream);
}

size_t gpk_rbf_psi_ws(int64_t N, int64_t M) { return psi_ws_bytes(N, M); }

}  // extern "C"
