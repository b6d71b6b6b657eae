// adam.cu — one Adam step on every device-resident parameter of a model in ONE launch (the "multi-tensor" form of
// tf_keras.optimizers.Adam.update_step applied to the UNCONSTRAINED variable of each Parameter; include/gpk.h gives the
// formulas).  A segment is one parameter: its constrained value (updated in place), the gradient of the objective
// w.r.t. that value, and the two moment buffers.
//
// Memory bound: 56 B per element (value, grad, m, v read; value, m, v written).  The segments are cut into chunks of
// two elements (16 B); a prefix table over the segments maps a global chunk index to (segment, chunk), so one
// grid-stride loop covers all segments and a small segment costs its own chunks, not a wave of CTAs.  A chunk whose four
// addresses are 16-byte aligned moves as double2; a segment whose four pointers are all 8 bytes past a 16-byte boundary
// peels one leading element (`head`) so that its body is aligned; the last odd element, the peeled one, and the segments
// whose pointers are misaligned differently from each other go element by element.
#include <math.h>

#include "internal.cuh"

using namespace gpk;

namespace gpk {

struct AdamSeg {
  double *value, *m, *v;
  const double* grad;
  int64_t n;
  double lower;
  int transform, head, vec;
};

struct AdamTable {
  AdamSeg seg[GPK_ADAM_MAX_SEGS];
  int64_t first[GPK_ADAM_MAX_SEGS + 1];  // first[s]: the global index of segment s's first chunk
  int n_segs;
};

struct AdamHyper {
  double lr_t, beta_1, beta_2, epsilon, sign;
};

// np.logaddexp(0, x), the branch NumPy takes (base.py::Softplus.forward)
__device__ __forceinline__ double softplus_forward(double x) { return x > 0.0 ? x + log1p(exp(-x)) : log1p(exp(x)); }

template <int TRANSFORM>
__device__ __forceinline__ void adam_element(double& value, double g, double& m, double& v, double lower,
                                             const AdamHyper& h) {
  double u, du;  // the unconstrained variable and d value / d u there
  if (TRANSFORM == GPK_ADAM_SOFTPLUS) {
    const double y = value - lower;
    u = y + log(-expm1(-y));
    du = 1.0 / (1.0 + exp(-u));
  } else if (TRANSFORM == GPK_ADAM_EXP) {
    u = log(value - lower);
    du = exp(u);
  } else {
    u = value;
    du = 1.0;
  }
  const double gu = h.sign * g * du;
  m += (1.0 - h.beta_1) * (gu - m);
  v += (1.0 - h.beta_2) * (gu * gu - v);
  u -= h.lr_t * m / (sqrt(v) + h.epsilon);
  if (TRANSFORM == GPK_ADAM_SOFTPLUS) value = softplus_forward(u) + lower;
  else if (TRANSFORM == GPK_ADAM_EXP) value = exp(u) + lower;
  else value = u;
}

template <int TRANSFORM>
__device__ __forceinline__ void adam_chunk(const AdamSeg& s, int64_t c, const AdamHyper& h) {
  const int64_t e0 = 2 * c - s.head;  // the chunk covers the elements [e0, e0 + 2) that lie in [0, n)
  if (s.vec && e0 >= 0 && e0 + 2 <= s.n) {
    double2 x = *reinterpret_cast<const double2*>(s.value + e0);
    const double2 g = *reinterpret_cast<const double2*>(s.grad + e0);
    double2 m = *reinterpret_cast<const double2*>(s.m + e0);
    double2 v = *reinterpret_cast<const double2*>(s.v + e0);
    adam_element<TRANSFORM>(x.x, g.x, m.x, v.x, s.lower, h);
    adam_element<TRANSFORM>(x.y, g.y, m.y, v.y, s.lower, h);
    *reinterpret_cast<double2*>(s.value + e0) = x;
    *reinterpret_cast<double2*>(s.m + e0) = m;
    *reinterpret_cast<double2*>(s.v + e0) = v;
    return;
  }
  for (int64_t e = e0 < 0 ? 0 : e0; e < e0 + 2 && e < s.n; ++e) {
    double x = s.value[e], m = s.m[e], v = s.v[e];
    adam_element<TRANSFORM>(x, s.grad[e], m, v, s.lower, h);
    s.value[e] = x;
    s.m[e] = m;
    s.v[e] = v;
  }
}

__global__ void __launch_bounds__(256)
adam_step_kernel(const __grid_constant__ AdamTable tab, const __grid_constant__ AdamHyper h) {
  const int64_t total = tab.first[tab.n_segs], stride = (int64_t)gridDim.x * blockDim.x;
  int s = 0;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += stride) {
    while (i >= tab.first[s + 1]) ++s;  // i only grows: the search resumes where it stopped
    const AdamSeg& seg = tab.seg[s];
    const int64_t c = i - tab.first[s];
    if (seg.transform == GPK_ADAM_IDENTITY) adam_chunk<GPK_ADAM_IDENTITY>(seg, c, h);
    else if (seg.transform == GPK_ADAM_SOFTPLUS) adam_chunk<GPK_ADAM_SOFTPLUS>(seg, c, h);
    else adam_chunk<GPK_ADAM_EXP>(seg, c, h);
  }
}

}  // namespace gpk

extern "C" int gpk_adam_step(const gpk_adam_seg* segs, int n_segs, double lr_t, double beta_1, double beta_2,
                             double epsilon, double sign, int dtype, void* stream) {
  const cudaStream_t st = (cudaStream_t)stream;
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
  AdamTable tab;
  tab.n_segs = n_segs;
  tab.first[0] = 0;
  for (int s = 0; s < n_segs; ++s) {
    const gpk_adam_seg& in = segs[s];
    AdamSeg& o = tab.seg[s];
    o.value = (double*)in.value;
    o.grad = in.grad;
    o.m = in.m;
    o.v = in.v;
    o.n = in.n;
    o.lower = in.lower;
    o.transform = in.transform;
    const uintptr_t a = (uintptr_t)in.value & 15, b = (uintptr_t)in.grad & 15, c = (uintptr_t)in.m & 15,
                    d = (uintptr_t)in.v & 15;
    o.vec = a == b && a == c && a == d && (a == 0 || a == 8);
    o.head = o.vec && a == 8;
    tab.first[s + 1] = tab.first[s] + (in.n + o.head + 1) / 2;
  }
  for (int s = n_segs; s < GPK_ADAM_MAX_SEGS; ++s) {
    tab.seg[s] = AdamSeg{};
    tab.first[s + 1] = tab.first[n_segs];
  }
  const int64_t total = tab.first[n_segs];
  if (total == 0) return 0;
  int dev = 0, sms = 0;
  GPK_CUDA_OK(cudaGetDevice(&dev));
  GPK_CUDA_OK(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
  const int64_t want = (total + 255) / 256, cap = (int64_t)sms * 4;  // 61 registers: 4 CTAs of 256 threads per SM
  const AdamHyper h{lr_t, beta_1, beta_2, epsilon, sign};
  adam_step_kernel<<<(unsigned)(want < cap ? want : cap), 256, 0, st>>>(tab, h);
  GPK_LAUNCH_OK();
  return 0;
}
