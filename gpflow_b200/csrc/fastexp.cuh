// fastexp.cuh — the table-driven fp64 exp (and MUFU-seeded sqrt) of the K-build fast path, shared by the
// stationary leaves of kbuild.cu and the RBF psi statistics of psi.cu.  The 2^(j/64) table lives in kbuild.cu
// (c_exp2_tab, exp2_table_device); callers stage it in shared memory.
#pragma once
#include "kprog.cuh"

namespace gpk {

// The fast path works on x = c * r2 (c folded into the per-dimension weights on the host together with the
// 1/lengthscale^2 scale): RBF c = 1/2 (k = v exp(-x)), Matern12 c = 1 (u = sqrt x, k = v exp(-u)),
// Exponential c = 1/4, Matern32 c = 3 (k = v (1 + u) exp(-u)), Matern52 c = 5 (k = v (1 + u + x/3) exp(-u)).
// The reference's clip of r2 at 1e-36 (stationaries.py:130-136) becomes a clip of x at c * 1e-36.
template <int TYPE> __host__ __device__ constexpr double kf_fold() {
  return TYPE == GPK_K_RBF ? 0.5 : TYPE == GPK_K_MATERN32 ? 3.0 : TYPE == GPK_K_MATERN52 ? 5.0
       : TYPE == GPK_K_EXPONENTIAL ? 0.25 : 1.0;
}
template <int TYPE> __host__ __device__ constexpr bool kf_const_pre() {  // prefactor is just the variance
  return TYPE == GPK_K_RBF || TYPE == GPK_K_MATERN12 || TYPE == GPK_K_EXPONENTIAL;
}

__device__ __forceinline__ float rsqrt_approx(float x) {
  float y;
  asm("rsqrt.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}

// Four fp64 elements at a time, stage by stage: every arithmetic step is issued for the four independent
// elements back to back, so the dependent chains (sqrt: 6, exp: 11 fp64 ops) overlap instead of each
// waiting out the fp64 latency alone.  fp64-pipe budget per element (Matern52): 2 (x) + 6 (sqrt) + 2 (pre)
// + 11 (exp) = 21 besides the D-term dot product; clamps, range checks and the 2^n scaling are integer ops.
//   tab: 2^(j/64) in SHARED memory (lanes hit different entries), pre-multiplied by the variance when the
//   prefactor is constant.  var_ok: variance >= 2^-100, so adding n to the exponent field cannot underflow
//   while n >= -900 (the slow path handles the rest: it scales by 2^n in two exact steps and returns 0 only for
//   u > 1416, where even var (1 + u + x/3) exp(-u) < var exp(-708)).
template <int TYPE>
__device__ __forceinline__ void stationary_value4(const double (&xin)[4], double var, double var3, bool var_ok,
                                                  const double* __restrict__ tab, double (&out)[4]) {
  double u[4], pre[4];
  if (TYPE == GPK_K_RBF) {
#pragma unroll
    for (int q = 0; q < 4; ++q) u[q] = __double2hiint(xin[q]) < 0 ? 0.0 : xin[q];  // max(x, 0) on the integer pipe
  } else {
    constexpr double clampv = kf_fold<TYPE>() * 1e-36;
    double x[4], g[4], h[4], r[4], d[4];
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      // x < clamp (or negative) by a signed compare of the high words: equal high words differ by < 2^-20 relative
      const int hi_c = (int)((unsigned long long)__double_as_longlong(clampv) >> 32);
      x[q] = __double2hiint(xin[q]) < hi_c ? clampv : xin[q];
    }
    // y0 ~ x^-1/2 to 2^-22 (MUFU); g = x y0 ~ sqrt x, h = y0/2; one coupled Newton step on g (2^-43), then a
    // Heron correction with the unrefined h: relative error 1.5 e0^3 ~ 2^-64 before rounding
#pragma unroll
    for (int q = 0; q < 4; ++q) h[q] = (double)rsqrt_approx((float)x[q]);
#pragma unroll
    for (int q = 0; q < 4; ++q) g[q] = x[q] * h[q];
#pragma unroll
    for (int q = 0; q < 4; ++q) h[q] = 0.5 * h[q];
#pragma unroll
    for (int q = 0; q < 4; ++q) r[q] = fma(-g[q], h[q], 0.5);
#pragma unroll
    for (int q = 0; q < 4; ++q) g[q] = fma(g[q], r[q], g[q]);
#pragma unroll
    for (int q = 0; q < 4; ++q) d[q] = fma(-g[q], g[q], x[q]);
#pragma unroll
    for (int q = 0; q < 4; ++q) u[q] = fma(h[q], d[q], g[q]);
    if (TYPE == GPK_K_MATERN52) {
#pragma unroll
      for (int q = 0; q < 4; ++q) pre[q] = fma(var3, x[q], fma(var, u[q], var));
    } else if (TYPE == GPK_K_MATERN32) {
#pragma unroll
      for (int q = 0; q < 4; ++q) pre[q] = fma(var, u[q], var);
    }
  }
  // exp(-u), u >= 0
  double sh[4], kd[4], rr[4], p[4];
  int k[4];
#pragma unroll
  for (int q = 0; q < 4; ++q) sh[q] = fma(u[q], -92.33248261689366, 6755399441055744.0);  // round(-u 64/ln2) in the low bits
#pragma unroll
  for (int q = 0; q < 4; ++q) { kd[q] = sh[q] - 6755399441055744.0; k[q] = __double2loint(sh[q]); }
#pragma unroll
  for (int q = 0; q < 4; ++q) rr[q] = fma(kd[q], -0.01083042468962958, -u[q]);   // ln2/64 hi (kd * hi exact)
#pragma unroll
  for (int q = 0; q < 4; ++q) rr[q] = fma(kd[q], -6.619564634077006e-12, rr[q]);  // ln2/64 lo
#pragma unroll
  for (int q = 0; q < 4; ++q) p[q] = fma(rr[q], 8.3333333333333332e-03, 4.1666666666666664e-02);
#pragma unroll
  for (int q = 0; q < 4; ++q) p[q] = fma(p[q], rr[q], 1.6666666666666666e-01);
#pragma unroll
  for (int q = 0; q < 4; ++q) p[q] = fma(p[q], rr[q], 0.5);
#pragma unroll
  for (int q = 0; q < 4; ++q) p[q] = fma(p[q], rr[q], 1.0);
#pragma unroll
  for (int q = 0; q < 4; ++q) p[q] = fma(p[q], rr[q], 1.0);
  double w[4];
#pragma unroll
  for (int q = 0; q < 4; ++q) {
    const double t = tab[k[q] & 63];
    w[q] = (kf_const_pre<TYPE>() ? t : pre[q] * t) * p[q];
  }
  const int kmin = min(min(k[0], k[1]), min(k[2], k[3]));
  if (var_ok && kmin >= -57600) {  // 2^n by an integer add on the exponent field (n >= -900, w >= 2^-101)
#pragma unroll
    for (int q = 0; q < 4; ++q)
      out[q] = __hiloint2double(__double2hiint(w[q]) + ((k[q] >> 6) << 20), __double2loint(w[q]));
  } else {  // 2^n in two halves (each >= -1022 while u <= 1416): the Matern prefactor and a large variance keep
            // w 2^n representable well past exp's own underflow at u = 708
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      const int n = k[q] >> 6, n1 = n >> 1;
      const double two_n1 = __longlong_as_double((long long)(max(n1, -1022) + 1023) << 52);
      const double two_n2 = __longlong_as_double((long long)(max(n - n1, -1022) + 1023) << 52);
      out[q] = u[q] > 1416.0 ? 0.0 : (w[q] * two_n1) * two_n2;
    }
  }
}

}  // namespace gpk
