// kprog.cuh — the flattened kernel expression shared by the fused K-build (kbuild.cu) and the expression-driven
// gradient reduction (grad.cu).  compile_kprog (kbuild.cu) is the one flattener of a gpk_knode array.
#pragma once
#include "common.cuh"

namespace gpk {

constexpr int KB_MAXG = 4;      // gram groups (distinct (active_dims, weights) sets)
constexpr int KB_MAXL = 12;     // leaves
constexpr int KB_MAXDIMS = 256; // total active dims over groups
constexpr int KB_MAXOPS = 32;
constexpr int KB_OP_ADD = 0xFE, KB_OP_MUL = 0xFF;

// Leaves are numbered in node-array order.  ops: postfix program, entries < KB_MAXL push a leaf, KB_OP_ADD / KB_OP_MUL
// pop two and push the result (at most 4 entries deep).  Group g owns dims[g_off[g] .. g_off[g] + g_ndims[g]) and the
// weights w[] of the same range; g_weighted: 0 unweighted, 1 weights on the A side only (ARD Linear / Polynomial
// variances), 2 on both sides (1 / ARD lengthscales).
struct KProg {
  int n_groups, n_leaves, n_ops, symmetric;
  int g_ndims[KB_MAXG], g_off[KB_MAXG], g_weighted[KB_MAXG];
  int l_type[KB_MAXL], l_group[KB_MAXL];
  // l_scale: 1 / lengthscale^2 (scalar-lengthscale stationary), the offset (Polynomial), else 1.  l_var: the variance
  // (1 when ARD Linear / Polynomial variances ride in w).  l_alpha: RQ alpha / Polynomial degree.
  double l_scale[KB_MAXL], l_var[KB_MAXL], l_alpha[KB_MAXL];
  double l_len[KB_MAXL];  // the scalar lengthscale as given (stationary leaves without ARD), else 0
  unsigned char ops[KB_MAXOPS];
  short dims[KB_MAXDIMS];
  double w[KB_MAXDIMS];
};
static_assert(sizeof(KProg) < 4000, "KProg must fit the kernel parameter space");

int compile_kprog(const gpk_knode* nodes, int n_nodes, const int32_t* dims, const double* ard, int64_t D, KProg& p);

__host__ __device__ inline bool kprog_stationary(int type) {
  return type == GPK_K_RBF || type == GPK_K_MATERN12 || type == GPK_K_MATERN32 || type == GPK_K_MATERN52 ||
         type == GPK_K_RQ || type == GPK_K_EXPONENTIAL;
}

}  // namespace gpk
