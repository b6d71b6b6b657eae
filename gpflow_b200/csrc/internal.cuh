// internal.cuh — untyped implementation entry points shared across translation units.  Each extern "C" entry point of
// gpk.h is defined in the file that implements it; capi.cu holds the argument checks of the primitives whose *_impl
// other code also calls, the error state and the profiler.
#pragma once
#include "common.cuh"

#define GPK_DTYPE_OK(name) GPK_CHECK_ARG(dtype == GPK_F32 || dtype == GPK_F64, name ": bad dtype %d", dtype)

namespace gpk {

constexpr double LOG2PI = 1.8378770664093454835606594728112;

// Workspace carving for the one-call objectives: consecutive 256-byte aligned pieces of a caller-provided block
// (base NULL: only the size is counted).
struct Arena {
  char* base;
  size_t off;
  explicit Arena(void* p) : base((char*)p), off(0) {}
  void* take(size_t bytes) {
    void* r = base ? base + off : nullptr;
    off += align_up(bytes, 256);
    return r;
  }
};

static inline int64_t pad_ld(int64_t n) { return (n + 3) / 4 * 4; }

int kbuild_impl(const gpk_knode* nodes, int n_nodes, const int32_t* dims, const double* ard, const void* X,
                int64_t N, int64_t ldx, const void* X2, int64_t N2, int64_t ldx2, int64_t D, void* K, int64_t ldk,
                int dtype, int uplo, double diag_scalar, const void* diag_vec, cudaStream_t st);
int kdiag_impl(const gpk_knode* nodes, int n_nodes, const int32_t* dims, const double* ard, const void* X,
               int64_t N, int64_t ldx, int64_t D, void* out, int dtype, cudaStream_t st);

int colsumsq_impl(const void* A, int64_t m, int64_t n, int64_t lda, double scale, int accumulate, void* out, int dtype,
                  cudaStream_t st, const void* w = nullptr, int64_t winc = 0);
int reduce_impl(int f, const void* x, int64_t n, int64_t inc, double scale, int accumulate, double* out, int dtype,
                cudaStream_t st);
int reduce_wsq_impl(const void* w, const void* x, int64_t n, int64_t inc, double scale, double* out, int dtype,
                    cudaStream_t st);
int tril_sumsq_impl(const void* A, int64_t n, int64_t lda, int64_t stride, int batch, double scale, int accumulate,
                    double* out, int dtype, cudaStream_t st);
// lik.cu: the scalar likelihoods of gpk_lik (gpk.h)
int lik_check(const gpk_lik* lik, int64_t P, const char* who);
// the row stride of Y: P targets per row, or one label (MULTICLASS) or target (HETEROSKEDASTIC) per row
inline int64_t lik_ldy(const gpk_lik* lik, int64_t P) {
  return lik && (lik->type == GPK_LIK_MULTICLASS || lik->type == GPK_LIK_HETEROSKEDASTIC) ? 1 : P;
}
// Y[b * ldy + p]; mX[b * ldmx + p] (NULL: zero mean) is added to Fmu
int lik_varexp_impl(const gpk_lik* lik, const void* Fmu, const void* Fvar, const void* Y, const void* mX, int64_t B,
                    int64_t P, int64_t ldy, int64_t ldmx, int64_t var_sb, int64_t var_sp, double scale, int accumulate,
                    double* out, int dtype, cudaStream_t st);
int lik_grad_impl(const gpk_lik* lik, const double* fmu, const double* fvar, const double* Y, int64_t ldy,
                  const double* mX, int64_t B, int64_t P, double c, double* R, double* Wt, double* gpar,
                  cudaStream_t st);
int lik_predict_mv_impl(const gpk_lik* lik, const void* Fmu, const void* Fvar, int64_t N, int64_t P, void* mean,
                        void* var, int dtype, cudaStream_t st);
int lik_predict_ld_impl(const gpk_lik* lik, const void* Fmu, const void* Fvar, const void* Y, int64_t N, int64_t P,
                        void* out, int dtype, cudaStream_t st);
int axpby_impl(int64_t m, int64_t n, double a, const void* X, int64_t ldx, double b, void* Y, int64_t ldy, int dtype,
               cudaStream_t st);
int scale_impl(void* A, int64_t m, int64_t n, int64_t lda, const void* s, int by_row, int invert, int dtype,
               cudaStream_t st);
int add_diag_impl(void* A, int64_t n, int64_t lda, double scalar, const void* vec, int dtype, cudaStream_t st);
int fill_impl(void* A, int64_t m, int64_t n, int64_t lda, double v, int dtype, cudaStream_t st);
int tril_impl(void* A, int64_t n, int64_t lda, int64_t stride, int batch, int dtype, cudaStream_t st);
int transpose_impl(const void* A, int64_t m, int64_t n, int64_t lda, void* B, int64_t ldb, int dtype, cudaStream_t st);

// dtype-erased wrappers over the typed templates
int gemm_any(int ta, int tb, int64_t m, int64_t n, int64_t k, double alpha, const void* A, int64_t lda, const void* B,
             int64_t ldb, double beta, void* C, int64_t ldc, int dtype, int flags, cudaStream_t st);
// ws = [dinv blocks | int8 tensor-core digit planes]; sized by potrf_ws_bytes(n, rows, dtype)
// need_dinv = false: the caller never runs trsm on this factor.  cond_hint: an upper bound of max_i A_ii / lambda_min(A)
// when the caller knows one (e.g. (kernel variance + noise) / noise), 0 = unknown; selects the number of digit planes /
// the engine of the fp64 trailing updates (potrf.cu::pick_slices).
int potrf_any(void* A, int64_t n, int64_t rows, int64_t lda, int dtype, int32_t* info, void* ws, cudaStream_t st,
              bool need_dinv = true, double cond_hint = 0.0);
inline size_t potrf_ws_bytes(int64_t n, int64_t rows, int dtype);
int trsm_any(int trans, const void* L, int64_t n, int64_t ldl, void* B, int64_t nrhs, int64_t ldb, int dtype,
             const void* dinv, cudaStream_t st);
int trtri_diag_any(const void* L, int64_t n, int64_t ldl, void* dinv, int dtype, cudaStream_t st);

// fused.cu: the fp64 M x M brackets of the device gradients, elementwise (i, j), T and G [M, ld]:
//   SB_MIRROR      G[i,j] <- G[j,i] above the diagonal (in place: a lower triangle made symmetric)
//   SB_PHI         G <- Phi(T), the strict lower triangle of T plus half its diagonal, zeros above (reads T's lower part)
//   SB_SYMNEG      G <- -sym(T)
//   SB_UNWHITENED  G <- -sym(T) + wP AAt + sym(V) / 2 - P/2 Kinv   (AAt, V, Kinv full)
enum { SB_MIRROR = 0, SB_PHI = 1, SB_SYMNEG = 2, SB_UNWHITENED = 3 };
int svgp_bracket(int mode, const void* T, void* G, int64_t M, int64_t ld, const void* AAt, const void* V,
                 const void* Kinv, double wP, double P, cudaStream_t st);
int chol_adjoint(const void* L, const void* dinv, int64_t n, int64_t ld, void* T, void* G, cudaStream_t st);

// grad.cu: the expression reductions of the device gradients, and the inverses of a Cholesky factor
int grad_expr_slots(const gpk_knode* nodes, int n_nodes, const int32_t* dims, const double* ard, int64_t D,
                    const char* who);
int gpr_grad_launch(const gpk_knode* nodes, int n_nodes, const int32_t* dims, const double* ard, const double* X,
                    int64_t N, int64_t ldx, int64_t D, const double* alpha, int P, const double* Kinv, int64_t ldk,
                    double* gout, cudaStream_t st);
int gpr_lowrank_grad_launch(const gpk_knode* nodes, int n_nodes, const int32_t* dims, const double* ard,
                            const double* X, int64_t N, int64_t ldx, int64_t D, const double* Vt, const double* Zt,
                            int P, double* gout, cudaStream_t st);
int inducing_grad_launch(const gpk_knode* nodes, int n_nodes, const int32_t* dims, const double* ard, const double* X,
                         int64_t N, int64_t ldx, int64_t D, const double* Z, int64_t M, int64_t ldz, const double* Guf,
                         int64_t ldgf, const double* Guu, int64_t ldgu, double kdiag_weight, const double* kdiag_vec,
                         double* gout, double* dZ, const char* who, cudaStream_t st);
int square_grad_launch(const gpk_knode* nodes, int n_nodes, const int32_t* dims, const double* ard, const double* X,
                       int64_t N, int64_t ldx, int64_t D, const double* G, int64_t ldg, double* gout,
                       double* dz_scratch, const char* who, cudaStream_t st);
int potri_lower(double* L, int64_t n, int64_t ldl, const double* dinv, double* Kinv, int64_t ldk, double* tmp,
                cudaStream_t st);
int lauum_lower(const double* A, int64_t n, int64_t lda, double* C, int64_t ldc, cudaStream_t st);

// psi.cu: the RBF psi statistics of the Bayesian GPLVM and the KL of q(X)
struct PsiBwdGeom;  // launch geometry of psi_backward (psi.cu)
size_t psi_ws_bytes(int64_t N, int64_t M);
int psi_forward(const gpk_knode* nodes, int n_nodes, const int32_t* dims, const double* ard, const double* mu,
                const double* S, int64_t N, int64_t Q, const double* Z, int64_t M, int64_t ldz, double* P1, int64_t sn,
                int64_t sm, double* P2, int64_t ldp2, void* ws, const char* who, cudaStream_t st);
int psi_backward(const gpk_knode* nodes, int n_nodes, const int32_t* dims, const double* ard, const double* mu,
                 const double* S, int64_t N, int64_t Q, const double* Z, int64_t M, int64_t ldz, const double* G1t,
                 int64_t ldg1, const double* G2, int64_t ldg2, double* dmu, double* dS, double* dZ, double* gpar,
                 void* ws, const char* who, cudaStream_t st, PsiBwdGeom* geom = nullptr);
int kl_diag(const double* mu, const double* S, const double* m0, const double* p0, int64_t n, double* kl, double* dmu,
            double* dS, cudaStream_t st);

// kmv.cu: the matrix-free product (K(X, X2) + diag_scalar I) V
size_t kmv_ws_bytes(int64_t N, int64_t N2, int64_t P);
int kmv_impl(const gpk_knode* nodes, int n_nodes, const int32_t* dims, const double* ard, const double* X, int64_t N,
             int64_t ldx, const double* X2, int64_t N2, int64_t ldx2, int64_t D, const double* V, int64_t P,
             int64_t ldv, double diag_scalar, double* out, int64_t ldo, void* ws, const int32_t* skip, cudaStream_t st);

inline size_t dinv_bytes(int64_t n, int dtype) { return (size_t)((n + NB - 1) / NB) * NB * NB * dtype_size(dtype); }
inline size_t potrf_ws_bytes(int64_t n, int64_t rows, int dtype) {
  return align_up(dinv_bytes(n, dtype), 256) + 256 /* look-ahead counter */ + potrf_tc_ws_bytes(n, rows, dtype);
}

}  // namespace gpk
