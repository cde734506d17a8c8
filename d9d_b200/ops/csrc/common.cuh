// d9d_b200 — shared device-side primitives for sm_90a (H100).
//
// Everything in here is hand-written inline PTX for the Hopper execution
// model: mbarrier pipelines, TMA (cp.async.bulk.tensor, multicast within a
// cluster), register-resident wgmma accumulators (wgmma.cuh).  No CUTLASS / CuTe
// dependency.
#pragma once

#include <cuda.h>
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>

#include "wgmma.cuh"

#ifndef D9D_WATCHDOG
#define D9D_WATCHDOG 1  // bounded mbarrier spins: a protocol bug traps instead of hanging the GPU
#endif

namespace d9d {

// ----------------------------------------------------------------------------------------------
// misc
// ----------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}

__device__ __forceinline__ uint32_t lane_id() { return threadIdx.x & 31; }

__device__ __forceinline__ bool elect_one() {
  uint32_t pred = 0;
  asm volatile(
      "{\n\t"
      ".reg .pred P;\n\t"
      "elect.sync _|P, 0xffffffff;\n\t"
      "selp.b32 %0, 1, 0, P;\n\t"
      "}\n"
      : "=r"(pred));
  return pred != 0;
}

template <typename T>
__device__ __forceinline__ T warp_sum(T v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

template <typename T>
__device__ __forceinline__ T warp_max(T v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = max(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

// ----------------------------------------------------------------------------------------------
// mbarrier
// ----------------------------------------------------------------------------------------------
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;\n" ::"r"(smem_u32(bar)), "r"(count));
}

__device__ __forceinline__ void fence_barrier_init() {
  asm volatile("fence.mbarrier_init.release.cluster;\n" ::: "memory");
}

__device__ __forceinline__ void fence_proxy_async_all() { asm volatile("fence.proxy.async;\n" ::: "memory"); }

__device__ __forceinline__ void fence_proxy_async_smem() {
  asm volatile("fence.proxy.async.shared::cta;\n" ::: "memory");
}

__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];\n" ::"r"(smem_u32(bar)) : "memory");
}

__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;\n" ::"r"(smem_u32(bar)), "r"(bytes)
               : "memory");
}

// bar: shared-window address of the mbarrier
__device__ __forceinline__ bool mbar_try_wait(uint32_t bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n\t"
      ".reg .pred P;\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 P, [%1], %2;\n\t"
      "selp.b32 %0, 1, 0, P;\n\t"
      "}\n"
      : "=r"(ok)
      : "r"(bar), "r"(parity)
      : "memory");
  return ok != 0;
}

__device__ __forceinline__ bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
  return mbar_try_wait(smem_u32(bar), parity);
}

__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
#if D9D_WATCHDOG
  uint32_t spins = 0;
  while (!mbar_try_wait(bar, parity)) {
    if (++spins > (1u << 24)) {  // try_wait sleeps in HW; this is many seconds of wall-clock
      printf("d9d watchdog: mbarrier wait timed out (block %d thread %d parity %u)\n", blockIdx.x, threadIdx.x,
             parity);
      __trap();
    }
  }
#else
  while (!mbar_try_wait(bar, parity)) {
  }
#endif
}

// Same wait for kernels that issue wgmma: any function call (printf) in such a kernel makes ptxas serialise every
// wgmma of it, so the watchdog only traps.
__device__ __forceinline__ void mbar_wait_wg(uint64_t* bar, uint32_t parity) {
#if D9D_WATCHDOG
  uint32_t spins = 0;
  while (!mbar_try_wait(bar, parity)) {
    if (++spins > (1u << 24)) __trap();
  }
#else
  while (!mbar_try_wait(bar, parity)) {
  }
#endif
}

// Same wait for warps that raised their register budget with setmaxnreg.inc: a trap anywhere in such a region makes ptxas
// allocate all of it under the launch bound's cap (168 registers at 384 threads), with spills and serialised wgmma.  A
// timeout sets `stuck` and every later wait returns at once; the caller traps after the region ends.
__device__ __forceinline__ void mbar_wait_flag(uint32_t bar, uint32_t parity, bool& stuck) {
#if D9D_WATCHDOG
  uint32_t spins = 0;
  while (!stuck && !mbar_try_wait(bar, parity)) {
    if (++spins > (1u << 24)) stuck = true;
  }
#else
  while (!mbar_try_wait(bar, parity)) {
  }
#endif
}

__device__ __forceinline__ void mbar_wait_flag(uint64_t* bar, uint32_t parity, bool& stuck) {
  mbar_wait_flag(smem_u32(bar), parity, stuck);
}

// ----------------------------------------------------------------------------------------------
// TMA
// ----------------------------------------------------------------------------------------------
__device__ __forceinline__ void tma_prefetch_desc(const void* desc) {
  asm volatile("prefetch.tensormap [%0];\n" ::"l"(reinterpret_cast<uint64_t>(desc)) : "memory");
}

__device__ __forceinline__ void tma_load_2d(void* smem_dst, const void* desc, uint64_t* bar, int c0, int c1) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];\n"
      ::"r"(smem_u32(smem_dst)),
      "l"(reinterpret_cast<uint64_t>(desc)), "r"(smem_u32(bar)), "r"(c0), "r"(c1)
      : "memory");
}

__device__ __forceinline__ void tma_load_3d(void* smem_dst, const void* desc, uint64_t* bar, int c0, int c1, int c2) {
  asm volatile(
      "cp.async.bulk.tensor.3d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5}], "
      "[%2];\n" ::"r"(smem_u32(smem_dst)),
      "l"(reinterpret_cast<uint64_t>(desc)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2)
      : "memory");
}

__device__ __forceinline__ void tma_load_4d(void* smem_dst, const void* desc, uint64_t* bar, int c0, int c1, int c2, int c3) {
  asm volatile(
      "cp.async.bulk.tensor.4d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6}], "
      "[%2];\n" ::"r"(smem_u32(smem_dst)),
      "l"(reinterpret_cast<uint64_t>(desc)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
      : "memory");
}

__device__ __forceinline__ void tma_store_2d(const void* desc, const void* smem_src, int c0, int c1) {
  asm volatile("cp.async.bulk.tensor.2d.global.shared::cta.tile.bulk_group [%0, {%2, %3}], [%1];\n" ::"l"(
                   reinterpret_cast<uint64_t>(desc)),
               "r"(smem_u32(smem_src)), "r"(c0), "r"(c1)
               : "memory");
}

__device__ __forceinline__ void tma_store_3d(const void* desc, const void* smem_src, int c0, int c1, int c2) {
  asm volatile("cp.async.bulk.tensor.3d.global.shared::cta.tile.bulk_group [%0, {%2, %3, %4}], [%1];\n" ::"l"(
                   reinterpret_cast<uint64_t>(desc)),
               "r"(smem_u32(smem_src)), "r"(c0), "r"(c1), "r"(c2)
               : "memory");
}

// global[tile] += smem[tile]; the addition is performed by the memory system (L2), element type from the tensor map
__device__ __forceinline__ void tma_reduce_add_3d(const void* desc, const void* smem_src, int c0, int c1, int c2) {
  asm volatile("cp.reduce.async.bulk.tensor.3d.global.shared::cta.add.tile.bulk_group [%0, {%2, %3, %4}], [%1];\n" ::"l"(
                   reinterpret_cast<uint64_t>(desc)),
               "r"(smem_u32(smem_src)), "r"(c0), "r"(c1), "r"(c2)
               : "memory");
}

__device__ __forceinline__ void tma_store_commit() { asm volatile("cp.async.bulk.commit_group;\n" ::: "memory"); }
template <int N>
__device__ __forceinline__ void tma_store_wait_read() {
  asm volatile("cp.async.bulk.wait_group.read %0;\n" ::"n"(N) : "memory");
}
template <int N>
__device__ __forceinline__ void tma_store_wait() {
  asm volatile("cp.async.bulk.wait_group %0;\n" ::"n"(N) : "memory");
}

template <int N>
__device__ __forceinline__ void setmaxnreg_inc() { asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;\n" ::"n"(N)); }
template <int N>
__device__ __forceinline__ void setmaxnreg_dec() { asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;\n" ::"n"(N)); }

// named barrier over `threads` threads (a multiple of 32) of the CTA
__device__ __forceinline__ void named_barrier_sync(int id, int threads) {
  asm volatile("bar.sync %0, %1;\n" ::"r"(id), "r"(threads) : "memory");
}

// arrive on a named barrier without waiting for it (the threads that bar.sync it wait for these arrivals)
__device__ __forceinline__ void named_barrier_arrive(int id, int threads) {
  asm volatile("bar.arrive %0, %1;\n" ::"r"(id), "r"(threads) : "memory");
}

// two floats from an 8-byte aligned shared-memory address (a 32-bit shared-window address, as smem_u32 returns)
__device__ __forceinline__ float2 lds_f32x2(uint32_t addr) {
  float2 v;
  asm volatile("ld.shared.v2.f32 {%0, %1}, [%2];\n" : "=f"(v.x), "=f"(v.y) : "r"(addr) : "memory");
  return v;
}

// ----------------------------------------------------------------------------------------------
// numeric helpers
// ----------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t pack_bf16x2(float lo, float hi) {
  __nv_bfloat162 v = __floats2bfloat162_rn(lo, hi);
  return *reinterpret_cast<uint32_t*>(&v);
}

__device__ __forceinline__ float2 unpack_bf16x2(uint32_t v) {
  __nv_bfloat162 b = *reinterpret_cast<__nv_bfloat162*>(&v);
  return __bfloat1622float2(b);
}

// Counter-based RNG (Philox-4x32-10).  Stateless: value depends only on (seed, offset) so results are
// independent of launch geometry — required for reproducible stochastic rounding.
__device__ __forceinline__ uint4 philox4x32(uint64_t seed, uint64_t offset) {
  uint32_t k0 = static_cast<uint32_t>(seed), k1 = static_cast<uint32_t>(seed >> 32);
  uint32_t c0 = static_cast<uint32_t>(offset), c1 = static_cast<uint32_t>(offset >> 32), c2 = 0, c3 = 0;
#pragma unroll
  for (int i = 0; i < 10; ++i) {
    uint32_t hi0 = __umulhi(0xD2511F53u, c0), lo0 = 0xD2511F53u * c0;
    uint32_t hi1 = __umulhi(0xCD9E8D57u, c2), lo1 = 0xCD9E8D57u * c2;
    uint32_t n0 = hi1 ^ c1 ^ k0, n1 = lo1, n2 = hi0 ^ c3 ^ k1, n3 = lo0;
    c0 = n0; c1 = n1; c2 = n2; c3 = n3;
    k0 += 0x9E3779B9u; k1 += 0xBB67AE85u;
  }
  return make_uint4(c0, c1, c2, c3);
}

// Stochastic rounding fp32 -> bf16: add 16 random bits below the kept mantissa, truncate.
// E[round(x)] == x.  Inf passes through; a NaN whose payload lies only in the dropped low 16 bits gets the bf16 quiet
// bit, so that it stays a NaN instead of becoming an inf.
__device__ __forceinline__ uint16_t sr_bf16_bits(float x, uint32_t rnd16) {
  uint32_t b = __float_as_uint(x);
  if ((b & 0x7F800000u) == 0x7F800000u) return static_cast<uint16_t>((b >> 16) | ((b & 0xFFFFu) ? 0x40u : 0u));
  b += (rnd16 & 0xFFFFu);
  return static_cast<uint16_t>(b >> 16);
}

}  // namespace d9d

// ----------------------------------------------------------------------------------------------
// bulk copies
// ----------------------------------------------------------------------------------------------
namespace d9d {

// 1-D bulk copy global -> shared, completion counted on an mbarrier (bytes: multiple of 16, both addresses 16-byte aligned)
__device__ __forceinline__ void bulk_load_1d(void* smem_dst, const void* gmem_src, uint32_t bytes, uint64_t* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];\n" ::"r"(
                   smem_u32(smem_dst)),
               "l"(reinterpret_cast<uint64_t>(gmem_src)), "r"(bytes), "r"(smem_u32(bar))
               : "memory");
}

}  // namespace d9d

// ----------------------------------------------------------------------------------------------
// Clusters: CTAs of one cluster share operand tiles through TMA multicast and release each other's stages through
// remote mbarrier arrivals.
// ----------------------------------------------------------------------------------------------
namespace d9d {

__device__ __forceinline__ uint32_t cluster_ctarank() {
  uint32_t r;
  asm volatile("mov.u32 %0, %%cluster_ctarank;\n" : "=r"(r));
  return r;
}

__device__ __forceinline__ void cluster_sync_all() {
  asm volatile("barrier.cluster.arrive.release.aligned;\n" ::: "memory");
  asm volatile("barrier.cluster.wait.acquire.aligned;\n" ::: "memory");
}

// TMA load whose box lands at the same shared-memory offset in every CTA of `cta_mask`, completing on the mbarrier at
// the same offset in each of them
__device__ __forceinline__ void tma_load_3d_multicast(void* smem_dst, const void* desc, uint64_t* bar, uint16_t cta_mask, int c0,
                                                      int c1, int c2) {
  asm volatile(
      "cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes.multicast::cluster [%0], [%1, {%4, %5, %6}], "
      "[%2], %3;\n" ::"r"(smem_u32(smem_dst)),
      "l"(reinterpret_cast<uint64_t>(desc)), "r"(smem_u32(bar)), "h"(cta_mask), "r"(c0), "r"(c1), "r"(c2)
      : "memory");
}

// arrive on the mbarrier at this shared-window address in CTA `cta` of the cluster.  The arrival has the default
// .release.cta semantics: it frees a stage whose only readers were this CTA's wgmma (complete once wgmma.wait_group
// returns) for the next TMA write.  A .release.cluster arrival compiles to MEMBAR.ALL.GPU in front of the arrive (ptxas,
// sm_90a), which stalled the consumer warp that issues the next k-block's wgmma, twice per k-block.
__device__ __forceinline__ void mbar_arrive_cluster(uint32_t bar, uint32_t cta) {
  asm volatile(
      "{\n\t"
      ".reg .b32 remote;\n\t"
      "mapa.shared::cluster.u32 remote, %0, %1;\n\t"
      "mbarrier.arrive.shared::cluster.b64 _, [remote];\n\t"
      "}\n" ::"r"(bar),
      "r"(cta)
      : "memory");
}

}  // namespace d9d
