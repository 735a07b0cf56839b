// PTX helpers shared by the tensor-core kernels (mbarrier, bulk copy / TMA, cluster / DSMEM).
#pragma once
#include <cuda_fp16.h>
#include <stdint.h>
#include <stdio.h>

namespace fsn {
namespace ptx {

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ uint32_t cluster_ctarank() {
  uint32_t r;
  asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r));
  return r;
}
// shared::cta address -> shared::cluster address of the same offset in CTA `rank`
__device__ __forceinline__ uint32_t mapa(uint32_t addr, uint32_t rank) {
  uint32_t r;
  asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(r) : "r"(addr), "r"(rank));
  return r;
}
__device__ __forceinline__ void cluster_sync_all() {
  asm volatile("barrier.cluster.arrive.release.aligned;\n\tbarrier.cluster.wait.acquire.aligned;" ::: "memory");
}
__device__ __forceinline__ bool elect_one() {
  uint32_t pred;
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "elect.sync _|p, 0xffffffff;\n\t"
      "selp.b32 %0, 1, 0, p;\n\t}"
      : "=r"(pred));
  return pred != 0;
}

// ---- mbarrier
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
// arrive on the barrier at the same offset in CTA `rank` of the cluster (own rank allowed)
__device__ __forceinline__ void mbar_arrive_cluster(uint64_t* bar, uint32_t rank) {
  asm volatile("mbarrier.arrive.release.cluster.shared::cluster.b64 _, [%0];" ::"r"(mapa(smem_u32(bar), rank))
               : "memory");
}
// same without release semantics: for pure "event" signals that publish no data of the arriving thread
// (a release at cluster scope is a fence and costs ~1000 cycles of issue time)
__device__ __forceinline__ void mbar_arrive_cluster_relaxed(uint64_t* bar, uint32_t rank) {
  asm volatile("mbarrier.arrive.relaxed.cluster.shared::cluster.b64 _, [%0];" ::"r"(mapa(smem_u32(bar), rank))
               : "memory");
}
// one cluster-scope release fence, to be followed by any number of relaxed arrives (release pattern with a
// single fence instead of one per arrive)
__device__ __forceinline__ void fence_release_cluster() { asm volatile("fence.acq_rel.cluster;" ::: "memory"); }
__device__ __forceinline__ bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "mbarrier.try_wait.parity.acquire.cluster.shared::cta.b64 p, [%1], %2;\n\t"
      "selp.b32 %0, 1, 0, p;\n\t}"
      : "=r"(ok)
      : "r"(smem_u32(bar)), "r"(parity)
      : "memory");
  return ok != 0;
}
__device__ __forceinline__ bool mbar_test_wait(uint64_t* bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "mbarrier.test_wait.parity.acquire.cluster.shared::cta.b64 p, [%1], %2;\n\t"
      "selp.b32 %0, 1, 0, p;\n\t}"
      : "=r"(ok)
      : "r"(smem_u32(bar)), "r"(parity)
      : "memory");
  return ok != 0;
}
// spin with a watchdog: a protocol bug traps (launch error) instead of hanging the GPU.  No printf here: any call in a
// kernel makes ptxas serialise all of its wgmma instructions
template <bool RELAXED>
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  uint32_t spins = 0;
  while (!mbar_try_wait(bar, parity)) {
    if (RELAXED) __nanosleep(64);
    if (++spins > (RELAXED ? (1u << 24) : (1u << 27))) asm volatile("trap;");
  }
}

// same without the back-off variants, for the threads that issue wgmma
__device__ __forceinline__ void mbar_wait_mma(uint64_t* bar, uint32_t parity) {
  uint32_t spins = 0;
  while (!mbar_try_wait(bar, parity))
    if (++spins > (1u << 27)) asm volatile("trap;");
}

// ---- CTA-scope hand-offs.  A wait with .acquire.cluster makes every successful wait invalidate L1 (CCTL.IVALL) and
// an arrive with .release.cluster fences at GPU scope (MEMBAR.ALL.GPU, ~1000 issue cycles) - neither is needed where
// the data behind the barrier is written by this CTA, or by the TMA engine (async proxy, complete_tx)
__device__ __forceinline__ bool mbar_try_wait_cta(uint64_t* bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "mbarrier.try_wait.parity.acquire.cta.shared::cta.b64 p, [%1], %2;\n\t"
      "selp.b32 %0, 1, 0, p;\n\t}"
      : "=r"(ok)
      : "r"(smem_u32(bar)), "r"(parity)
      : "memory");
  return ok != 0;
}
// spin with a watchdog (trap, see mbar_wait); SLEEP = back off between polls, for waits off the critical path
template <bool SLEEP>
__device__ __forceinline__ void mbar_wait_cta(uint64_t* bar, uint32_t parity) {
  uint32_t spins = 0;
  while (!mbar_try_wait_cta(bar, parity)) {
    if (SLEEP) __nanosleep(64);
    if (++spins > (SLEEP ? (1u << 24) : (1u << 27))) asm volatile("trap;");
  }
}
// the wait of mbar_wait_cta<false> for a whole warp at once, with the poll loop inside one asm block: the warp leaves
// the loop together (vote.all), so the compiler sees no divergent region to reconverge and can keep a warp-uniform
// barrier address and parity in uniform registers.  Same watchdog (trap after 2^27 polls)
__device__ __forceinline__ void mbar_wait_cta_warp(uint32_t bar, uint32_t parity) {
  asm volatile(
      "{\n\t.reg .pred p;\n\t.reg .b32 n;\n\t"
      "mov.b32 n, 0;\n"
      "WAIT:\n\t"
      "mbarrier.try_wait.parity.acquire.cta.shared::cta.b64 p, [%0], %1;\n\t"
      "vote.sync.all.pred p, p, 0xffffffff;\n\t"
      "@p bra.uni DONE;\n\t"
      "add.u32 n, n, 1;\n\t"
      "setp.gt.u32 p, n, 134217728;\n\t"
      "@p trap;\n\t"
      "bra.uni WAIT;\n"
      "DONE:\n\t}"
      ::"r"(bar), "r"(parity)
      : "memory");
}
// arrive by one elected lane of the warp if `pred` (warp-uniform): a predicated instruction, no divergent region
__device__ __forceinline__ void mbar_arrive_elect_if(uint32_t bar, uint32_t pred) {
  asm volatile(
      "{\n\t.reg .pred e, p;\n\t"
      "elect.sync _|e, 0xffffffff;\n\t"
      "setp.ne.and.b32 p, %1, 0, e;\n\t"
      "@p mbarrier.arrive.shared::cta.b64 _, [%0];\n\t}"
      ::"r"(bar), "r"(pred)
      : "memory");
}
// same on the barrier at the same offset in CTA `rank` of the cluster (default .release.cta: an event signal)
__device__ __forceinline__ void mbar_arrive_remote_elect_if(uint32_t bar, uint32_t rank, uint32_t pred) {
  asm volatile(
      "{\n\t.reg .pred e, p;\n\t.reg .b32 r;\n\t"
      "elect.sync _|e, 0xffffffff;\n\t"
      "setp.ne.and.b32 p, %2, 0, e;\n\t"
      "@p mapa.shared::cluster.u32 r, %0, %1;\n\t"
      "@p mbarrier.arrive.shared::cluster.b64 _, [r];\n\t}"
      ::"r"(bar), "r"(rank), "r"(pred)
      : "memory");
}
// generic-proxy writes to this CTA's shared memory -> later async-proxy reads (wgmma operands).  fence.proxy.async
// without a state space also covers global memory and costs a GPU-scope MEMBAR
__device__ __forceinline__ void fence_proxy_async_smem() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
// arrive on the barrier at the same offset in CTA `rank` of the cluster with the default .release.cta semantics: orders
// nothing beyond the arriving thread's own CTA, so it publishes no generic-proxy data to the peer - an event signal
__device__ __forceinline__ void mbar_arrive_remote(uint64_t* bar, uint32_t rank) {
  asm volatile("mbarrier.arrive.shared::cluster.b64 _, [%0];" ::"r"(mapa(smem_u32(bar), rank)) : "memory");
}
// same, also announcing `bytes` of asynchronous writes (complete_tx) that the current phase must wait for
__device__ __forceinline__ void mbar_arrive_expect_tx_remote(uint64_t* bar, uint32_t rank, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cluster.b64 _, [%0], %1;" ::"r"(mapa(smem_u32(bar), rank)), "r"(bytes)
               : "memory");
}
// bulk copy (async proxy) of `bytes` of this CTA's shared memory to the same offset in CTA `rank`, completing on the
// barrier at the same offset in that CTA.  The source must have been published to the async proxy
// (fence.proxy.async.shared::cta by its writers, then a barrier that orders them before this thread)
__device__ __forceinline__ void bulk_s2s_remote(const void* src, uint32_t bytes, uint64_t* bar, uint32_t rank) {
  const uint32_t s = smem_u32(src);
  asm volatile("cp.async.bulk.shared::cluster.shared::cta.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
                   mapa(s, rank)),
               "r"(s), "r"(bytes), "r"(mapa(smem_u32(bar), rank))
               : "memory");
}
// generic store to the same offset in CTA `rank` (publish with a .release.cluster arrive)
__device__ __forceinline__ void st_remote_f32(float* p, uint32_t rank, float v) {
  asm volatile("st.shared::cluster.f32 [%0], %1;" ::"r"(mapa(smem_u32(p), rank)), "f"(v) : "memory");
}
// named barrier of `count` threads (id 0 is __syncthreads)
__device__ __forceinline__ void named_sync(uint32_t id, uint32_t count) {
  asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(count) : "memory");
}

// ---- TMA engine (non-tensor bulk copy) and proxy fence
__device__ __forceinline__ void bulk_g2s(void* dst, const void* src, uint32_t bytes, uint64_t* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
                   smem_u32(dst)),
               "l"(src), "r"(bytes), "r"(smem_u32(bar))
               : "memory");
}
// same, multicast to the CTAs of `mask` in the cluster (same offset, each CTA's barrier at the same offset)
__device__ __forceinline__ void bulk_g2s_mc(void* dst, const void* src, uint32_t bytes, uint64_t* bar, uint16_t mask) {
  asm volatile(
      "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes.multicast::cluster [%0], [%1], %2, [%3], %4;" ::"r"(
          smem_u32(dst)),
      "l"(src), "r"(bytes), "r"(smem_u32(bar)), "h"(mask)
      : "memory");
}
// TMA tiled 2-D load (tensor map in kernel parameter space): box at element coordinates (c0 = inner, c1 = row)
__device__ __forceinline__ void tma_load_2d(void* dst, const void* tmap, int c0, int c1, uint64_t* bar) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3}], [%4];" ::"r"(
          smem_u32(dst)),
      "l"(tmap), "r"(c0), "r"(c1), "r"(smem_u32(bar))
      : "memory");
}
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async;" ::: "memory"); }
// bulk copy (async proxy) of `bytes` of this CTA's shared memory to global memory, in this thread's current bulk group.
// The source must have been published to the async proxy like that of bulk_s2s_remote
__device__ __forceinline__ void bulk_s2g(void* dst, const void* src, uint32_t bytes) {
  asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;" ::"l"(dst), "r"(smem_u32(src)), "r"(bytes)
               : "memory");
}
__device__ __forceinline__ void bulk_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
// every bulk group of this thread has finished reading its shared-memory source (the source may be overwritten)
__device__ __forceinline__ void bulk_wait_read_all() { asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory"); }
// every bulk group of this thread has completed its writes
__device__ __forceinline__ void bulk_wait_all() { asm volatile("cp.async.bulk.wait_group 0;" ::: "memory"); }

__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
// byte offset of element (row, k) in a K-major 128B-swizzled block of 64 k (rows of 128 B)
__host__ __device__ __forceinline__ int swz128_off(int row, int k) {
  return (row >> 3) * 1024 + (row & 7) * 128 + ((((k >> 3) ^ (row & 7)) & 7) << 4) + (k & 7) * 2;
}
// byte offset of element (row, k<32) in a K-major 64B-swizzled sub-tile (rows of 64 B, Swizzle<2,4,3>)
__host__ __device__ __forceinline__ int swz64_off(int row, int k) {
  return (row >> 3) * 512 + (row & 7) * 64 + ((((k >> 3) ^ ((row >> 1) & 3)) & 3) << 4) + (k & 7) * 2;
}

__device__ __forceinline__ float fast_sigmoid(float x) { return __fdividef(1.0f, 1.0f + __expf(-x)); }
__device__ __forceinline__ float fast_tanh(float x) { return 1.0f - __fdividef(2.0f, 1.0f + __expf(2.0f * x)); }

}  // namespace ptx
}  // namespace fsn
