// reduce.cu — warp-shuffle reductions and the small elementwise steps of the GP hot path.
// Reductions accumulate in fp64 whatever the storage dtype (SURVEY 2.2 R1, V1):
//   colsumsq  : conditionals/util.py:133,164   reduce: logdensities.py:152-154, sgpr.py:233-243,267-268,
//   tril_sumsq: kullback_leiblers.py:120,134   kullback_leiblers.py:124,130,159
#include "common.cuh"

namespace gpk {

template <typename T>
__global__ void colsumsq_kernel(const T* __restrict__ A, int64_t m, int64_t n, int64_t lda, double scale,
                                T* __restrict__ out, int64_t rows_per_block, const T* __restrict__ w, int64_t winc) {
  // block: 32 columns x 8 row-lanes; grid.x over column groups, grid.y over row chunks
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
  const int64_t j = (int64_t)blockIdx.x * 32 + tx;
  const int64_t r0 = (int64_t)blockIdx.y * rows_per_block;
  const int64_t r1 = min(m, r0 + rows_per_block);
  double s = 0.0;
  if (j < n)
    for (int64_t i = r0 + ty; i < r1; i += 8) {
      double v = (double)A[i * lda + j];
      if (w) v *= (double)w[i * winc];  // row weights: q_sqrt diagonal case, conditionals/util.py:149
      s += v * v;
    }
  __shared__ double sh[8][33];
  sh[ty][tx] = s;
  __syncthreads();
  if (ty == 0 && j < n) {
    double t = 0.0;
#pragma unroll
    for (int q = 0; q < 8; ++q) t += sh[q][tx];
    atomicAdd(&out[j], (T)(scale * t));
  }
}

template <typename T>
__global__ void reduce_kernel(int f, const T* __restrict__ x, int64_t n, int64_t inc, double scale, double* out) {
  double s = 0.0;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const double v = (double)x[i * inc];
    s += f == 0 ? v : f == 1 ? v * v : f == 2 ? log(v) : log(v * v);
  }
  s = warp_sum(s);
  __shared__ double sh[32];
  if ((threadIdx.x & 31) == 0) sh[threadIdx.x >> 5] = s;
  __syncthreads();
  if (threadIdx.x < 32) {
    s = threadIdx.x < (blockDim.x >> 5) ? sh[threadIdx.x] : 0.0;
    s = warp_sum(s);
    if (threadIdx.x == 0) atomicAdd(out, scale * s);
  }
}

template <typename T>
__global__ void reduce_wsq_kernel(const T* __restrict__ w, const T* __restrict__ x, int64_t n, int64_t inc, double scale,
                                  double* out) {
  double s = 0.0;  // sum_i w[i] * x[i*inc]^2   (kullback_leiblers.py:136-145 diagonal fast path)
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const double v = (double)x[i * inc];
    s += (double)w[i] * v * v;
  }
  s = warp_sum(s);
  __shared__ double sh[32];
  if ((threadIdx.x & 31) == 0) sh[threadIdx.x >> 5] = s;
  __syncthreads();
  if (threadIdx.x < 32) {
    s = threadIdx.x < (blockDim.x >> 5) ? sh[threadIdx.x] : 0.0;
    s = warp_sum(s);
    if (threadIdx.x == 0) atomicAdd(out, scale * s);
  }
}

template <typename T>
__global__ void tril_sumsq_kernel(const T* __restrict__ A, int64_t n, int64_t lda, int64_t stride, double scale,
                                  double* out) {
  // grid.x over rows, grid.y over batch; each block sums one row's lower part
  const T* row = A + (int64_t)blockIdx.y * stride + (int64_t)blockIdx.x * lda;
  double s = 0.0;
  for (int64_t j = threadIdx.x; j <= blockIdx.x; j += blockDim.x) {
    const double v = (double)row[j];
    s += v * v;
  }
  s = warp_sum(s);
  __shared__ double sh[32];
  if ((threadIdx.x & 31) == 0) sh[threadIdx.x >> 5] = s;
  __syncthreads();
  if (threadIdx.x < 32) {
    s = threadIdx.x < (blockDim.x >> 5) ? sh[threadIdx.x] : 0.0;
    s = warp_sum(s);
    if (threadIdx.x == 0 && s != 0.0) atomicAdd(out, scale * s);
  }
}

// ---- elementwise -------------------------------------------------------------------------------
template <typename T>
__global__ void axpby_kernel(int64_t m, int64_t n, T a, const T* __restrict__ X, int64_t ldx, T b, T* __restrict__ Y,
                             int64_t ldy) {
  const int64_t tot = m * n;
  for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e < tot; e += (int64_t)gridDim.x * blockDim.x) {
    const int64_t i = e / n, j = e % n;
    const T x = a != T(0) ? a * X[i * ldx + j] : T(0);
    Y[i * ldy + j] = b != T(0) ? x + b * Y[i * ldy + j] : x;
  }
}

template <typename T>
__global__ void scale_kernel(T* __restrict__ A, int64_t m, int64_t n, int64_t lda, const T* __restrict__ s, int by_row,
                             int invert) {
  const int64_t tot = m * n;
  for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e < tot; e += (int64_t)gridDim.x * blockDim.x) {
    const int64_t i = e / n, j = e % n;
    const T f = s[by_row ? i : j];
    A[i * lda + j] = invert ? A[i * lda + j] / f : A[i * lda + j] * f;
  }
}

template <typename T>
__global__ void add_diag_kernel(T* __restrict__ A, int64_t n, int64_t lda, T scalar, const T* __restrict__ vec) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) A[i * lda + i] += scalar + (vec ? vec[i] : T(0));
}

template <typename T>
__global__ void fill_kernel(T* __restrict__ A, int64_t m, int64_t n, int64_t lda, T v) {
  const int64_t tot = m * n;
  for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e < tot; e += (int64_t)gridDim.x * blockDim.x)
    A[(e / n) * lda + e % n] = v;
}

template <typename T>
__global__ void tril_kernel(T* __restrict__ A, int64_t n, int64_t lda, int64_t stride) {
  T* M = A + (int64_t)blockIdx.y * stride;
  const int64_t tot = n * n;
  for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e < tot; e += (int64_t)gridDim.x * blockDim.x) {
    const int64_t i = e / n, j = e % n;
    if (j > i) M[i * lda + j] = T(0);
  }
}

template <typename T>
__global__ void transpose_kernel(const T* __restrict__ A, int64_t m, int64_t n, int64_t lda, T* __restrict__ B,
                                 int64_t ldb) {
  __shared__ T tile[32][33];
  const int64_t j0 = (int64_t)blockIdx.x * 32, i0 = (int64_t)blockIdx.y * 32;
  for (int r = threadIdx.y; r < 32; r += 8) {
    const int64_t i = i0 + r, j = j0 + threadIdx.x;
    tile[r][threadIdx.x] = (i < m && j < n) ? A[i * lda + j] : T(0);
  }
  __syncthreads();
  for (int r = threadIdx.y; r < 32; r += 8) {
    const int64_t j = j0 + r, i = i0 + threadIdx.x;
    if (i < m && j < n) B[j * ldb + i] = tile[threadIdx.x][r];
  }
}

static int reduce_num_sms() {  // of the CURRENT device
  int dev = 0, n = 0;
  cudaGetDevice(&dev);
  cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev);
  return n > 0 ? n : 132;
}

static unsigned grid_for(int64_t total, int threads = 256) {
  int64_t b = (total + threads - 1) / threads;
  if (b < 1) b = 1;
  const int64_t cap = (int64_t)reduce_num_sms() * 16;
  if (b > cap) b = cap;
  return (unsigned)b;
}

#define GPK_DISPATCH(dtype, CALL_F32, CALL_F64) \
  do {                                          \
    if ((dtype) == GPK_F64) { CALL_F64; } else { CALL_F32; } \
  } while (0)

int colsumsq_impl(const void* A, int64_t m, int64_t n, int64_t lda, double scale, int accumulate, void* out, int dtype,
                  cudaStream_t st, const void* w, int64_t winc) {
  if (n <= 0) return 0;
  if (!accumulate) GPK_CUDA_OK(cudaMemsetAsync(out, 0, n * dtype_size(dtype), st));
  if (m <= 0) return 0;
  const int64_t cgroups = (n + 31) / 32;
  int64_t rchunks = ((int64_t)reduce_num_sms() * 8 + cgroups - 1) / cgroups;
  if (rchunks < 1) rchunks = 1;
  int64_t rpb = (m + rchunks - 1) / rchunks;
  rpb = (rpb + 7) / 8 * 8;
  rchunks = (m + rpb - 1) / rpb;
  dim3 grid((unsigned)cgroups, (unsigned)rchunks);
  GPK_DISPATCH(dtype,
               (colsumsq_kernel<float><<<grid, 256, 0, st>>>((const float*)A, m, n, lda, scale, (float*)out, rpb, (const float*)w, winc)),
               (colsumsq_kernel<double><<<grid, 256, 0, st>>>((const double*)A, m, n, lda, scale, (double*)out, rpb, (const double*)w, winc)));
  GPK_LAUNCH_OK();
  return 0;
}

int reduce_impl(int f, const void* x, int64_t n, int64_t inc, double scale, int accumulate, double* out, int dtype,
                cudaStream_t st) {
  GPK_CHECK_ARG(f >= 0 && f <= 3, "reduce: bad function id %d", f);
  if (!accumulate) GPK_CUDA_OK(cudaMemsetAsync(out, 0, sizeof(double), st));
  if (n <= 0) return 0;
  const unsigned g = grid_for(n);
  GPK_DISPATCH(dtype, (reduce_kernel<float><<<g, 256, 0, st>>>(f, (const float*)x, n, inc, scale, out)),
               (reduce_kernel<double><<<g, 256, 0, st>>>(f, (const double*)x, n, inc, scale, out)));
  GPK_LAUNCH_OK();
  return 0;
}

int reduce_wsq_impl(const void* w, const void* x, int64_t n, int64_t inc, double scale, double* out, int dtype,
                    cudaStream_t st) {
  if (n <= 0) return 0;
  const unsigned g = grid_for(n);
  GPK_DISPATCH(dtype, (reduce_wsq_kernel<float><<<g, 256, 0, st>>>((const float*)w, (const float*)x, n, inc, scale, out)),
               (reduce_wsq_kernel<double><<<g, 256, 0, st>>>((const double*)w, (const double*)x, n, inc, scale, out)));
  GPK_LAUNCH_OK();
  return 0;
}

int tril_sumsq_impl(const void* A, int64_t n, int64_t lda, int64_t stride, int batch, double scale, int accumulate,
                    double* out, int dtype, cudaStream_t st) {
  if (!accumulate) GPK_CUDA_OK(cudaMemsetAsync(out, 0, sizeof(double), st));
  if (n <= 0 || batch <= 0) return 0;
  dim3 grid((unsigned)n, (unsigned)batch);
  GPK_DISPATCH(dtype, (tril_sumsq_kernel<float><<<grid, 256, 0, st>>>((const float*)A, n, lda, stride, scale, out)),
               (tril_sumsq_kernel<double><<<grid, 256, 0, st>>>((const double*)A, n, lda, stride, scale, out)));
  GPK_LAUNCH_OK();
  return 0;
}

int axpby_impl(int64_t m, int64_t n, double a, const void* X, int64_t ldx, double b, void* Y, int64_t ldy, int dtype,
               cudaStream_t st) {
  if (m * n <= 0) return 0;
  const unsigned g = grid_for(m * n);
  GPK_DISPATCH(dtype, (axpby_kernel<float><<<g, 256, 0, st>>>(m, n, (float)a, (const float*)X, ldx, (float)b, (float*)Y, ldy)),
               (axpby_kernel<double><<<g, 256, 0, st>>>(m, n, a, (const double*)X, ldx, b, (double*)Y, ldy)));
  GPK_LAUNCH_OK();
  return 0;
}

int scale_impl(void* A, int64_t m, int64_t n, int64_t lda, const void* s, int by_row, int invert, int dtype,
               cudaStream_t st) {
  if (m * n <= 0) return 0;
  const unsigned g = grid_for(m * n);
  GPK_DISPATCH(dtype, (scale_kernel<float><<<g, 256, 0, st>>>((float*)A, m, n, lda, (const float*)s, by_row, invert)),
               (scale_kernel<double><<<g, 256, 0, st>>>((double*)A, m, n, lda, (const double*)s, by_row, invert)));
  GPK_LAUNCH_OK();
  return 0;
}

int add_diag_impl(void* A, int64_t n, int64_t lda, double scalar, const void* vec, int dtype, cudaStream_t st) {
  if (n <= 0) return 0;
  const unsigned g = (unsigned)((n + 255) / 256);
  GPK_DISPATCH(dtype, (add_diag_kernel<float><<<g, 256, 0, st>>>((float*)A, n, lda, (float)scalar, (const float*)vec)),
               (add_diag_kernel<double><<<g, 256, 0, st>>>((double*)A, n, lda, scalar, (const double*)vec)));
  GPK_LAUNCH_OK();
  return 0;
}

int fill_impl(void* A, int64_t m, int64_t n, int64_t lda, double v, int dtype, cudaStream_t st) {
  if (m * n <= 0) return 0;
  const unsigned g = grid_for(m * n);
  GPK_DISPATCH(dtype, (fill_kernel<float><<<g, 256, 0, st>>>((float*)A, m, n, lda, (float)v)),
               (fill_kernel<double><<<g, 256, 0, st>>>((double*)A, m, n, lda, v)));
  GPK_LAUNCH_OK();
  return 0;
}

int tril_impl(void* A, int64_t n, int64_t lda, int64_t stride, int batch, int dtype, cudaStream_t st) {
  if (n <= 0 || batch <= 0) return 0;
  dim3 grid(grid_for(n * n), (unsigned)batch);
  GPK_DISPATCH(dtype, (tril_kernel<float><<<grid, 256, 0, st>>>((float*)A, n, lda, stride)),
               (tril_kernel<double><<<grid, 256, 0, st>>>((double*)A, n, lda, stride)));
  GPK_LAUNCH_OK();
  return 0;
}

int transpose_impl(const void* A, int64_t m, int64_t n, int64_t lda, void* B, int64_t ldb, int dtype, cudaStream_t st) {
  if (m * n <= 0) return 0;
  dim3 grid((unsigned)((n + 31) / 32), (unsigned)((m + 31) / 32)), block(32, 8);
  GPK_DISPATCH(dtype, (transpose_kernel<float><<<grid, block, 0, st>>>((const float*)A, m, n, lda, (float*)B, ldb)),
               (transpose_kernel<double><<<grid, block, 0, st>>>((const double*)A, m, n, lda, (double*)B, ldb)));
  GPK_LAUNCH_OK();
  return 0;
}

}  // namespace gpk
