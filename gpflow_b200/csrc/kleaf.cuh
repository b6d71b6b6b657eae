// kleaf.cuh — the generic per-element leaf functions of the fused K-build (kbuild.cu), shared with the matrix-free
// kernel product (kmv.cu) so that both evaluate every element by the same formulas.
#pragma once
#include "kprog.cuh"

namespace gpk {

template <typename T>
struct KMath;
template <>
struct KMath<double> {
  static __device__ __forceinline__ double exp_(double x) { return exp(x); }
  static __device__ __forceinline__ double sqrt_(double x) { return sqrt(x); }
  static __device__ __forceinline__ double pow_(double x, double y) { return pow(x, y); }
};
template <>
struct KMath<float> {
  static __device__ __forceinline__ float exp_(float x) { return expf(x); }
  static __device__ __forceinline__ float sqrt_(float x) { return sqrtf(x); }
  static __device__ __forceinline__ float pow_(float x, float y) { return powf(x, y); }
};

// value of one leaf given the (weighted) gram term `dot` and the row / column norms
template <typename T>
__device__ __forceinline__ T leaf_value(int type, T dot, T na, T nb, T scale, T var, T alpha, bool on_diag) {
  using M = KMath<T>;
  if (type == GPK_K_LINEAR) return var * dot;
  if (type == GPK_K_POLYNOMIAL) return M::pow_(var * dot + scale, alpha);  // linears.py:108 (offset rides in `scale`)
  if (type == GPK_K_CONSTANT) return var;
  if (type == GPK_K_WHITE) return on_diag ? var : T(0);
  T r2 = scale * (na + nb - T(2) * dot);  // ops.py:113-122 — may be slightly negative
  if (type == GPK_K_RBF) return var * M::exp_(T(-0.5) * r2);                 // stationaries.py:210
  if (type == GPK_K_RQ) return var * M::pow_(T(1) + T(0.5) * r2 / alpha, -alpha);  // :238
  T r = M::sqrt_(fmax(r2, T(1e-36)));                                         // :114
  if (type == GPK_K_MATERN52) {                                               // :311-313
    const T s5 = T(2.23606797749978969641);
    return var * (T(1) + s5 * r + T(5.0 / 3.0) * r * r) * M::exp_(-s5 * r);
  }
  if (type == GPK_K_MATERN32) {                                               // :290-292
    const T s3 = T(1.73205080756887729353);
    return var * (T(1) + s3 * r) * M::exp_(-s3 * r);
  }
  if (type == GPK_K_MATERN12) return var * M::exp_(-r);                       // :270-271
  return var * M::exp_(T(-0.5) * r);                                          // Exponential :250-251
}

}  // namespace gpk
