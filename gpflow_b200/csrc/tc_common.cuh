// tc_common.cuh — PTX wrappers shared by the warpgroup-MMA kernels (mbarrier, 1-D TMA bulk copy and reduction, cluster
// multicast, wgmma fences / commit / wait, shared-memory matrix descriptors).  sm_90a.
#pragma once
#include "common.cuh"
#include "wgmma_ops.cuh"

namespace gpk {

// ------------------------------------------------------------------------------------------------
// PTX wrappers
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count));
}
__device__ __forceinline__ void mbar_expect_tx(uint32_t bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint32_t bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}
// arrive on the mbarrier at the same shared-memory offset in CTA `rank` of the cluster (the own CTA included).  Used to
// release a pipeline stage: the caller has only READ the stage, and its reads are complete (wgmma.wait_group), so no
// release at cluster scope is needed -- `.release.cluster` costs a GPU-scope MEMBAR per arrive.
__device__ __forceinline__ void mbar_arrive_cluster(uint32_t bar, uint32_t rank) {
  asm volatile(
      "{\n\t.reg .b32 ra;\n\t"
      "mapa.shared::cluster.u32 ra, %0, %1;\n\t"
      "mbarrier.arrive.shared::cluster.b64 _, [ra];\n\t}"
      ::"r"(bar), "r"(rank)
      : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint32_t bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
      "selp.u32 %0, 1, 0, p;\n\t}"
      : "=r"(ok)
      : "r"(bar), "r"(parity)
      : "memory");
  return ok != 0;
}
// bounded wait: a protocol bug must abort the kernel, never hang the GPU
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity, int* err, int code) {
  for (uint32_t it = 0; !mbar_try_wait(bar, parity); ++it) {
    if (it > (1u << 26)) {
      if (err) atomicExch(err, code);
      __trap();
    }
  }
}
// the same wait with cluster scope (the stage's consumers may sit in a peer CTA of the cluster)
__device__ __forceinline__ bool mbar_try_wait_cluster(uint32_t bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "mbarrier.try_wait.parity.acquire.cluster.shared::cta.b64 p, [%1], %2;\n\t"
      "selp.u32 %0, 1, 0, p;\n\t}"
      : "=r"(ok)
      : "r"(bar), "r"(parity)
      : "memory");
  return ok != 0;
}
__device__ __forceinline__ void mbar_wait_cluster(uint32_t bar, uint32_t parity, int* err, int code) {
  for (uint32_t it = 0; !mbar_try_wait_cluster(bar, parity); ++it) {
    if (it > (1u << 26)) {
      if (err) atomicExch(err, code);
      __trap();
    }
  }
}
__device__ __forceinline__ void bulk_g2s(uint32_t dst, const void* src, uint32_t bytes, uint32_t bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
               ::"r"(dst), "l"(src), "r"(bytes), "r"(bar)
               : "memory");
}
// ---- bulk reduction shared -> global (async proxy, bulk async-groups of the issuing thread) ------------------------------
// the thread's generic-proxy shared-memory stores before its following bulk operations that read them
__device__ __forceinline__ void fence_proxy_async_shared() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
// completed bulk writes to global (async proxy) before the thread's following generic-proxy accesses (a release)
__device__ __forceinline__ void fence_proxy_async_global() { asm volatile("fence.proxy.async.global;" ::: "memory"); }
// dst[i] += src[i] for `bytes` / 8 doubles, each element rounded once (dst, src 16-byte aligned, bytes % 16 == 0)
__device__ __forceinline__ void bulk_reduce_add_f64(double* dst, uint32_t src, uint32_t bytes) {
  asm volatile("cp.reduce.async.bulk.global.shared::cta.bulk_group.add.f64 [%0], [%1], %2;" ::"l"(dst), "r"(src), "r"(bytes)
               : "memory");
}
__device__ __forceinline__ void bulk_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
// all but the newest N bulk groups of this thread have finished reading their shared-memory sources
template <int N>
__device__ __forceinline__ void bulk_wait_read() { asm volatile("cp.async.bulk.wait_group.read %0;" ::"n"(N) : "memory"); }
// all but the newest N bulk groups of this thread are complete (their global writes performed)
template <int N>
__device__ __forceinline__ void bulk_wait() { asm volatile("cp.async.bulk.wait_group %0;" ::"n"(N) : "memory"); }

// one lane of a converged warp issues (the rest of the warp keeps executing the same uniform control flow)
__device__ __forceinline__ bool elect_one() {
  uint32_t pred = 0;
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "elect.sync _|p, 0xffffffff;\n\t"
      "selp.u32 %0, 1, 0, p;\n\t}"
      : "=r"(pred));
  return pred != 0;
}

// ---- warpgroup MMA ordering ------------------------------------------------------------------------------
__device__ __forceinline__ void wg_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wg_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wg_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
// keeps the accumulator registers live across the asynchronous MMAs (the compiler must not move their uses above the wait)
template <typename T>
__device__ __forceinline__ void wg_keep(T* r, int n);
template <>
__device__ __forceinline__ void wg_keep<uint32_t>(uint32_t* r, int n) {
  for (int i = 0; i < n; ++i) asm volatile("" : "+r"(r[i])::"memory");
}
template <>
__device__ __forceinline__ void wg_keep<float>(float* r, int n) {
  for (int i = 0; i < n; ++i) asm volatile("" : "+f"(r[i])::"memory");
}

// four 8 x 8 b16 matrices (8 rows x 16 bytes) from shared memory; lanes 8 j .. 8 j + 7 give the row addresses of matrix j,
// register j receives matrix j (lane l: row l / 4, bytes 4 (l % 4) .. + 3)
__device__ __forceinline__ void ldsm_x4(uint32_t (&r)[4], uint32_t saddr) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0, %1, %2, %3}, [%4];"
               : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3])
               : "r"(saddr)
               : "memory");
}

// shared-memory matrix descriptor (sm_90): K-major, no swizzle; lbo = byte distance of the two 16-byte k chunks of a core
// matrix row pair, sbo = byte distance of consecutive groups of 8 rows
__device__ __forceinline__ uint64_t wg_desc(uint32_t saddr, uint32_t lbo, uint32_t sbo) {
  return (uint64_t)((saddr & 0x3FFFFu) >> 4) | ((uint64_t)(lbo >> 4) << 16) | ((uint64_t)(sbo >> 4) << 32);
}

// ---- thread-block cluster helpers (operand multicast) -------------------------------------------------
__device__ __forceinline__ uint32_t cluster_ctarank() {
  uint32_t r;
  asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r));
  return r;
}
__device__ __forceinline__ void cluster_sync_all() {
  asm volatile("barrier.cluster.arrive.release.aligned;" ::: "memory");
  asm volatile("barrier.cluster.wait.acquire.aligned;" ::: "memory");
}
// 1-D bulk copy replicated into the same shared-memory offset of every CTA in `mask`; each destination
// CTA's mbarrier (same offset) receives the complete_tx
__device__ __forceinline__ void bulk_g2s_mc(uint32_t dst, const void* src, uint32_t bytes, uint32_t bar, uint16_t mask) {
  asm volatile(
      "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes.multicast::cluster [%0], [%1], %2, [%3], %4;"
      ::"r"(dst), "l"(src), "r"(bytes), "r"(bar), "h"(mask)
      : "memory");
}

}  // namespace gpk
