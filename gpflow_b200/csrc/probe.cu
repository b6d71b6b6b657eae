// probe.cu — in-run pipe peaks for the roofline denominators of the fp64 path (bench.py prints them next to every
// fraction): the wgmma m64n32k32 .s8 issue peak that bounds syrk_i8_kernel and the mma.sync.m8n8k4.f64 (DMMA) peak that
// bounds the panel / small-K kernels.  Operands are resident (shared memory / registers): these are pipe peaks, not
// kernel targets.
#include "tc_common.cuh"

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

__global__ void __launch_bounds__(256) probe_dmma_kernel(double* out, int iters) {
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

// out[0] = wgmma .s8 (m64n32k32) peak, T(int8 op)/s (2 ops per MAC);  out[1] = DMMA fp64 peak, TFLOP/s;  out[2] = SM count
int peak_probe(double* out_host, cudaStream_t st) {
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
  const int iters = 20000;
  probe_dmma_kernel<<<sms * 4, 256, 0, st>>>(dummy, 200);
  GPK_CUDA_OK(cudaEventRecord(e0, st));
  probe_dmma_kernel<<<sms * 4, 256, 0, st>>>(dummy, iters);
  GPK_CUDA_OK(cudaEventRecord(e1, st));
  GPK_CUDA_OK(cudaEventSynchronize(e1));
  GPK_CUDA_OK(cudaEventElapsedTime(&ms, e0, e1));
  out_host[1] = 2.0 * 8.0 * 8.0 * 4.0 * 8.0 * iters * 8.0 * 4.0 * sms / (ms * 1e-3) / 1e12;
  out_host[2] = sms;
  cudaFree(dummy);
  cudaEventDestroy(e0);
  cudaEventDestroy(e1);
  return 0;
}

}  // namespace gpk
