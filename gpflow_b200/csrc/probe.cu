// probe.cu — in-run pipe peaks for the roofline denominators of the fp64 path (bench.py prints them next to every
// fraction): the wgmma m64n32k32 .s8 issue peak that bounds syrk_i8_kernel and the mma.sync.m16n8k16.f64 (DMMA) peak that
// bounds the panel / small-K kernels, next to the peak of the Ampere shape m8n8k4 (half of it on sm_90).  Operands are resident (shared memory / registers): these are pipe peaks, not
// kernel targets.
#include "tc_common.cuh"

using namespace gpk;

namespace gpk {

// two warpgroups per SM each issue `rounds` x 8 MMAs of 64 x 32 x 32 (int8, both operands in shared memory), the shape
// syrk_i8_kernel issues
__global__ void __launch_bounds__(256, 1) probe_i8_kernel(int rounds, int* sink) {
  extern __shared__ __align__(1024) uint8_t probe_smem[];
  for (int i = threadIdx.x; i < 64 * 1024 / 4; i += blockDim.x) reinterpret_cast<uint32_t*>(probe_smem)[i] = 0x01010101u;
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");  // generic-proxy stores before the MMAs read them
  __syncthreads();
  const uint32_t sa = smem_u32(probe_smem) + (threadIdx.x >> 7) * 8192;
  uint32_t acc[4 * 16];
#pragma unroll
  for (int i = 0; i < 64; ++i) acc[i] = 0u;
  for (int r = 0; r < rounds; ++r) {
    wg_fence();
#pragma unroll
    for (int i = 0; i < 8; ++i)
      WgmmaS8<32>::mma(acc + 16 * (i & 3), wg_desc(sa + (i & 1) * 2048, 128, 256), wg_desc(sa + 32768 + (i & 3) * 1024, 128, 256), 1u);
    wg_commit();
    wg_wait<1>();
  }
  wg_wait<0>();
  wg_keep(acc, 64);
  uint32_t x = 0;
#pragma unroll
  for (int i = 0; i < 64; ++i) x += acc[i];
  if (x == 0x12345u) sink[0] = (int)x;  // keeps the MMAs alive
}

__global__ void __launch_bounds__(256) probe_dmma884_kernel(double* out, int iters) {
  double c[8][2], a = 1.0 + threadIdx.x * 1e-9, b = 1e-3;
  for (int i = 0; i < 8; ++i) c[i][0] = c[i][1] = i;
  for (int it = 0; it < iters; ++it)
#pragma unroll
    for (int i = 0; i < 8; ++i)
      asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0,%1}, {%2}, {%3}, {%0,%1};\n"
                   : "+d"(c[i][0]), "+d"(c[i][1])
                   : "d"(a), "d"(b));
  double s = 0;
  for (int i = 0; i < 8; ++i) s += c[i][0] + c[i][1];
  if (s == 123.456) out[0] = s;  // keeps the loop alive
}

// the same instruction-level parallelism (8 independent accumulators, operands in registers) in the shape the kernels issue
__global__ void __launch_bounds__(256) probe_dmma16816_kernel(double* out, int iters) {
  double c[8][4], a[8], b[4];
  for (int i = 0; i < 8; ++i) a[i] = 1.0 + (threadIdx.x + i) * 1e-9;
  for (int i = 0; i < 4; ++i) b[i] = 1e-3 * (i + 1);
  for (int i = 0; i < 8; ++i) c[i][0] = c[i][1] = c[i][2] = c[i][3] = i;
  for (int it = 0; it < iters; ++it)
#pragma unroll
    for (int i = 0; i < 8; ++i) dmma16816(c[i], a, b);
  double s = 0;
  for (int i = 0; i < 8; ++i) s += c[i][0] + c[i][1] + c[i][2] + c[i][3];
  if (s == 123.456) out[0] = s;  // keeps the loop alive
}

// one dmma16816 per warp: D[w] = A[w] B[w] + C[w] with A [16][16], B [16][8] (k x n), C, D [16][8], all row-major; the lanes load
// their fragments by the map documented at dmma16816, so a wrong map shows up as misplaced elements
__global__ void debug_dmma16816_kernel(const double* A, const double* B, const double* C, double* D) {
  const int lane = threadIdx.x, g = lane >> 2, q = lane & 3;
  const double* a = A + blockIdx.x * 256;
  const double* b = B + blockIdx.x * 128;
  double af[8], bf[4], cf[4];
  for (int i = 0; i < 8; ++i) af[i] = a[(g + 8 * (i & 1)) * 16 + q + 4 * (i >> 1)];
  for (int i = 0; i < 4; ++i) bf[i] = b[(q + 4 * i) * 8 + g];
  for (int i = 0; i < 4; ++i) cf[i] = C[blockIdx.x * 128 + (g + 8 * (i >> 1)) * 8 + 2 * q + (i & 1)];
  dmma16816(cf, af, bf);
  for (int i = 0; i < 4; ++i) D[blockIdx.x * 128 + (g + 8 * (i >> 1)) * 8 + 2 * q + (i & 1)] = cf[i];
}

}  // namespace gpk

extern "C" int gpk_debug_dmma16816(const double* A, const double* B, const double* C, double* D, int nwarps,
                                   void* stream) {
  const cudaStream_t st = (cudaStream_t)stream;
  GPK_CHECK_ARG(A && B && C && D && nwarps > 0, "debug_dmma16816: bad arguments");
  debug_dmma16816_kernel<<<nwarps, 32, 0, st>>>(A, B, C, D);
  GPK_LAUNCH_OK();
  return 0;
}

// out[0] = wgmma .s8 (m64n32k32) peak, T(int8 op)/s (2 ops per MAC);  out[1] = DMMA fp64 peak of m16n8k16 (the shape the
// kernels issue), TFLOP/s;  out[2] = SM count;  out[3] = DMMA fp64 peak of m8n8k4, TFLOP/s
extern "C" int gpk_peak_probe(double* out_host, void* stream) {
  const cudaStream_t st = (cudaStream_t)stream;
  GPK_CHECK_ARG(out_host, "peak_probe: bad arguments");
  int dev = 0, sms = 0;
  GPK_CUDA_OK(cudaGetDevice(&dev));
  GPK_CUDA_OK(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
  cudaEvent_t e0, e1;
  GPK_CUDA_OK(cudaEventCreate(&e0));
  GPK_CUDA_OK(cudaEventCreate(&e1));
  float ms = 0.f;
  double* dummy = nullptr;
  GPK_CUDA_OK(cudaMalloc(&dummy, 8));
  GPK_CUDA_OK(cudaFuncSetAttribute(probe_i8_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 64 * 1024));
  const int rounds = 20000;
  probe_i8_kernel<<<sms, 256, 64 * 1024, st>>>(200, (int*)dummy);
  GPK_CUDA_OK(cudaEventRecord(e0, st));
  probe_i8_kernel<<<sms, 256, 64 * 1024, st>>>(rounds, (int*)dummy);
  GPK_CUDA_OK(cudaEventRecord(e1, st));
  GPK_CUDA_OK(cudaEventSynchronize(e1));
  GPK_CUDA_OK(cudaEventElapsedTime(&ms, e0, e1));
  out_host[0] = 2.0 * 64.0 * 32.0 * 32.0 * 8.0 * 2.0 * rounds * sms / (ms * 1e-3) / 1e12;
  const int iters = 20000;  // (per launch: 8 MMAs per iteration, 8 warps per CTA, 4 CTAs per SM)
  probe_dmma884_kernel<<<sms * 4, 256, 0, st>>>(dummy, 200);
  GPK_CUDA_OK(cudaEventRecord(e0, st));
  probe_dmma884_kernel<<<sms * 4, 256, 0, st>>>(dummy, iters);
  GPK_CUDA_OK(cudaEventRecord(e1, st));
  GPK_CUDA_OK(cudaEventSynchronize(e1));
  GPK_CUDA_OK(cudaEventElapsedTime(&ms, e0, e1));
  out_host[3] = 2.0 * 8.0 * 8.0 * 4.0 * 8.0 * iters * 8.0 * 4.0 * sms / (ms * 1e-3) / 1e12;
  const int iters16 = iters / 4;  // (8x the MACs per MMA at twice the rate: a quarter of the iterations for the same time)
  probe_dmma16816_kernel<<<sms * 4, 256, 0, st>>>(dummy, 50);
  GPK_CUDA_OK(cudaEventRecord(e0, st));
  probe_dmma16816_kernel<<<sms * 4, 256, 0, st>>>(dummy, iters16);
  GPK_CUDA_OK(cudaEventRecord(e1, st));
  GPK_CUDA_OK(cudaEventSynchronize(e1));
  GPK_CUDA_OK(cudaEventElapsedTime(&ms, e0, e1));
  out_host[1] = 2.0 * 16.0 * 8.0 * 16.0 * 8.0 * iters16 * 8.0 * 4.0 * sms / (ms * 1e-3) / 1e12;
  out_host[2] = sms;
  cudaFree(dummy);
  cudaEventDestroy(e0);
  cudaEventDestroy(e1);
  return 0;
}
