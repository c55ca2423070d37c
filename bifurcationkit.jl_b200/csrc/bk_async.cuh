// bk_async.cuh -- PTX wrappers for the asynchronous copy engine (TMA bulk copies, SASS UBLKCP) and mbarriers, shared by the
// Krylov kernels (bk_krylov_tma.cuh) and the transform kernels (bk_fft_fast.cuh).  sm_90a.
#pragma once
#include "bk_common.cuh"

#ifdef __CUDACC__
__device__ __forceinline__ unsigned bk2_smem(const void* p) { return (unsigned)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(unsigned long long* b, unsigned cnt) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bk2_smem(b)), "r"(cnt) : "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(unsigned long long* b, unsigned bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bk2_smem(b)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(unsigned long long* b) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bk2_smem(b)) : "memory");
}
__device__ __forceinline__ void mbar_wait(unsigned long long* b, unsigned parity) {
  asm volatile(
      "{\n"
      ".reg .pred p;\n"
      "BK2_WAIT_%=:\n"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
      "@p bra BK2_DONE_%=;\n"
      "bra BK2_WAIT_%=;\n"
      "BK2_DONE_%=:\n"
      "}\n" ::"r"(bk2_smem(b)),
      "r"(parity)
      : "memory");
}
// TMA bulk copy global -> shared, completion counted in bytes on the mbarrier
__device__ __forceinline__ void bulk_g2s(void* dst, const void* src, unsigned bytes, unsigned long long* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(bk2_smem(dst)),
               "l"(src), "r"(bytes), "r"(bk2_smem(bar))
               : "memory");
}
// L2 eviction priorities for the cache-hint form of bulk_g2s: evict_first for data read once, evict_last for data the next
// kernel reads again
__device__ __forceinline__ unsigned long long l2_evict_first() {
  unsigned long long p;
  asm volatile("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(p));
  return p;
}
__device__ __forceinline__ unsigned long long l2_evict_last() {
  unsigned long long p;
  asm volatile("createpolicy.fractional.L2::evict_last.b64 %0, 1.0;" : "=l"(p));
  return p;
}
__device__ __forceinline__ void bulk_g2s(void* dst, const void* src, unsigned bytes, unsigned long long* bar,
                                         unsigned long long policy) {
  asm volatile(
      "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes.L2::cache_hint [%0], [%1], %2, [%3], %4;" ::"r"(
          bk2_smem(dst)),
      "l"(src), "r"(bytes), "r"(bk2_smem(bar)), "l"(policy)
      : "memory");
}
// TMA bulk copy shared -> global (bulk async-group completion); the source must stay valid until bulk_store_wait_read()
__device__ __forceinline__ void bulk_s2g(void* dst, const void* src, unsigned bytes) {
  asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;" ::"l"(dst), "r"(bk2_smem(src)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void bulk_store_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
__device__ __forceinline__ void bulk_store_wait_read() { asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory"); }
// waits until the bulk stores of this thread's groups are COMPLETE (written), not only until their source has been read
__device__ __forceinline__ void bulk_store_wait_all() { asm volatile("cp.async.bulk.wait_group 0;" ::: "memory"); }
__device__ __forceinline__ void bulk_prefetch_l2(const void* src, unsigned bytes) {
  asm volatile("cp.async.bulk.prefetch.L2.global [%0], %1;" ::"l"(src), "r"(bytes) : "memory");
}
__device__ __forceinline__ void fence_proxy_async_smem() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
// Executed by every consumer lane between its last ld.shared of a ring stage and the warp's arrive on the stage's
// `empty` barrier.  The refill of the stage is a TMA (async-proxy) write; without a cross-proxy fence the arrive can
// become visible while the warp's last ld.shared are still in flight (ptxas schedules the dependent DFMAs *after*
// SYNCS.ARRIVE), and the refill then overwrites rows that have not been read yet.  Seen as a handful of wrong tiles per
// launch with E = 8 and several waves of CTAs (tools/k2check); mbarrier release/acquire alone does not order the proxies.
#ifndef BK2_NO_WAR_FENCE
__device__ __forceinline__ void consumer_release_fence() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
#else
__device__ __forceinline__ void consumer_release_fence() {}
#endif
__device__ __forceinline__ void fence_mbar_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }

#endif
