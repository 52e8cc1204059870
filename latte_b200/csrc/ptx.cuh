// Inline-PTX wrappers for sm_90a: mbarrier, TMA (cp.async.bulk.tensor), thread-block clusters, wgmma.
// Hand-written for this project; encodings follow the PTX ISA chapters on asynchronous warpgroup MMA (matrix
// descriptor format) and the tensor copy instructions.
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <cuda_fp16.h>
#include <cuda_bf16.h>
#include <cstdint>
#include <cstdio>

namespace b200 {

#ifndef B200_HANG_CYCLES
#define B200_HANG_CYCLES (4000000000ll)  // ~2 s at 2 GHz: a stuck pipeline traps instead of hanging the GPU
#endif

__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}
__device__ __forceinline__ uint32_t lane_id() { return threadIdx.x & 31; }

// ----------------------------------------------------------------------------- programmatic dependent launch (PDL)
// A kernel launched with the programmatic-stream-serialization attribute may start while its predecessor is still
// draining; everything before pdl_wait() (barrier init, descriptor prefetch) overlaps the
// predecessor's tail.  pdl_wait() returns once the predecessor grid has completed and its writes are visible.
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
__device__ __forceinline__ void pdl_launch_dependents() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }

// ----------------------------------------------------------------------------- mbarrier
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void fence_mbar_init() {
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
      "selp.u32 %0, 1, 0, p;\n\t}"
      : "=r"(ok)
      : "r"(smem_u32(bar)), "r"(parity)
      : "memory");
  return ok != 0;
}
// non-blocking probe of a phase (try_wait may suspend the thread for a hardware-defined interval; test_wait never does)
__device__ __forceinline__ bool mbar_test_wait(uint64_t* bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "mbarrier.test_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
      "selp.u32 %0, 1, 0, p;\n\t}"
      : "=r"(ok)
      : "r"(smem_u32(bar)), "r"(parity)
      : "memory");
  return ok != 0;
}
// The fast path is one try_wait (which itself suspends the thread for a hardware-defined interval); the slow path polls
// without touching the clock except every 1024th iteration, so a spinning role warp costs the SM few issue slots.  A wait
// that makes no progress for ~B200_HANG_CYCLES traps instead of hanging the GPU.  No printf here: these waits sit between
// wgmma issue and wgmma.wait_group, and a function call there makes ptxas serialize every wgmma of the kernel.
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  if (mbar_try_wait(bar, parity)) return;
  uint32_t it = 0;
  long long t0 = 0;
  while (!mbar_try_wait(bar, parity)) {
    if ((++it & 1023u) == 0) {
      const long long now = clock64();
      if (t0 == 0) t0 = now;
      else if (now - t0 > B200_HANG_CYCLES) {
        __trap();
      }
    }
  }
}

// acquire at CLUSTER scope: for barriers that a thread of the peer CTA arrives on with a generic-proxy remote arrive
__device__ __forceinline__ bool mbar_try_wait_cluster(uint64_t* bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "mbarrier.try_wait.parity.acquire.cluster.shared::cta.b64 p, [%1], %2;\n\t"
      "selp.u32 %0, 1, 0, p;\n\t}"
      : "=r"(ok)
      : "r"(smem_u32(bar)), "r"(parity)
      : "memory");
  return ok != 0;
}
__device__ __forceinline__ void mbar_wait_cluster(uint64_t* bar, uint32_t parity) {
  if (mbar_try_wait_cluster(bar, parity)) return;
  long long t0 = clock64();
  while (!mbar_try_wait_cluster(bar, parity)) {
    if (clock64() - t0 > B200_HANG_CYCLES) {
      __trap();
    }
  }
}

// ----------------------------------------------------------------------------- per-warpgroup register budget
// A warp-specialized kernel compiled for R registers per thread moves registers from its producer warpgroup (dec) to its
// consumer warpgroups (inc) through the CTA's pool; inc blocks until the pool holds enough, so the budgets must balance
// against R.  Every warp of the warpgroup executes the same instruction; N is a multiple of 8 in [24, 256].
template <uint32_t N>
__device__ __forceinline__ void setmaxnreg_dec() { asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(N)); }
template <uint32_t N>
__device__ __forceinline__ void setmaxnreg_inc() { asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(N)); }

// ----------------------------------------------------------------------------- proxies / fences
__device__ __forceinline__ void fence_proxy_async_smem() {  // generic-proxy smem writes -> visible to async proxy (wgmma/TMA)
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}
// orders this thread's global-memory accesses through the generic proxy with those through the async proxy (TMA stores
// and reductions), in both directions
__device__ __forceinline__ void fence_proxy_async_global() { asm volatile("fence.proxy.async.global;" ::: "memory"); }

// ----------------------------------------------------------------------------- TMA loads (tile mode, mbarrier completion)
__device__ __forceinline__ void tma_prefetch_desc(const CUtensorMap* m) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(m)) : "memory");
}
__device__ __forceinline__ void tma_load_2d(void* dst, const CUtensorMap* m, uint64_t* bar, int c0, int c1) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
      ::"r"(smem_u32(dst)), "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1)
      : "memory");
}
__device__ __forceinline__ void tma_load_3d(void* dst, const CUtensorMap* m, uint64_t* bar, int c0, int c1, int c2) {
  asm volatile(
      "cp.async.bulk.tensor.3d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5}], [%2];"
      ::"r"(smem_u32(dst)), "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2)
      : "memory");
}
__device__ __forceinline__ void tma_load_4d(void* dst, const CUtensorMap* m, uint64_t* bar, int c0, int c1, int c2,
                                            int c3) {
  asm volatile(
      "cp.async.bulk.tensor.4d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6}], [%2];"
      ::"r"(smem_u32(dst)), "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
      : "memory");
}

// multicast: the box lands at the same smem offset (and signals the mbarrier at the same offset) in every CTA of `mask`
__device__ __forceinline__ void tma_load_2d_mcast(void* dst, const CUtensorMap* m, uint64_t* bar, int c0, int c1,
                                                  uint16_t mask) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.tile.mbarrier::complete_tx::bytes.multicast::cluster"
      " [%0], [%1, {%3, %4}], [%2], %5;"
      ::"r"(smem_u32(dst)), "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "h"(mask)
      : "memory");
}

// ----------------------------------------------------------------------------- thread-block clusters
// shared::cluster address of `p` (a pointer into this CTA's smem) as seen in CTA `rank` of the cluster
__device__ __forceinline__ uint32_t mapa_u32(const void* p, uint32_t rank) {
  uint32_t r;
  asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(r) : "r"(smem_u32(p)), "r"(rank));
  return r;
}
// Remote arrive with the DEFAULT (.release.cta) semantics: it only has to order this thread's own prior observation of
// "my TMA bytes have landed"; a .release.cluster here costs a cluster-scope fence (~1.5k cycles) per call (measured).
__device__ __forceinline__ void mbar_arrive_cluster(uint32_t bar_cluster_addr) {
  asm volatile("mbarrier.arrive.shared::cluster.b64 _, [%0];" ::"r"(bar_cluster_addr) : "memory");
}
__device__ __forceinline__ uint32_t cluster_ctarank() {
  uint32_t r;
  asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r));
  return r;
}
__device__ __forceinline__ void cluster_sync_all() {  // every thread of every CTA in the cluster
  asm volatile("barrier.cluster.arrive.release.aligned;\n\tbarrier.cluster.wait.acquire.aligned;" ::: "memory");
}

// ----------------------------------------------------------------------------- TMA store (smem -> global, bulk-group completion)
__device__ __forceinline__ void tma_store_2d(const CUtensorMap* m, const void* src, int c0, int c1) {
  asm volatile("cp.async.bulk.tensor.2d.global.shared::cta.bulk_group [%0, {%2, %3}], [%1];"
               ::"l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(src)), "r"(c0), "r"(c1)
               : "memory");
}
__device__ __forceinline__ void tma_store_3d(const CUtensorMap* m, const void* src, int c0, int c1, int c2) {
  asm volatile("cp.async.bulk.tensor.3d.global.shared::cta.bulk_group [%0, {%2, %3, %4}], [%1];"
               ::"l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(src)), "r"(c0), "r"(c1), "r"(c2)
               : "memory");
}
__device__ __forceinline__ void tma_store_4d(const CUtensorMap* m, const void* src, int c0, int c1, int c2, int c3) {
  asm volatile("cp.async.bulk.tensor.4d.global.shared::cta.bulk_group [%0, {%2, %3, %4, %5}], [%1];"
               ::"l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(src)), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
               : "memory");
}
// smem tile ADDED into global memory (element type from the tensor map: fp32): x += delta without ever loading x
__device__ __forceinline__ void tma_reduce_add_2d(const CUtensorMap* m, const void* src, int c0, int c1) {
  asm volatile("cp.reduce.async.bulk.tensor.2d.global.shared::cta.add.tile.bulk_group [%0, {%2, %3}], [%1];"
               ::"l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(src)), "r"(c0), "r"(c1)
               : "memory");
}
// 8-byte shared-memory store through a shared-window address (a generic pointer would give a generic ST)
__device__ __forceinline__ void st_shared_f2(uint32_t saddr, float a, float b) {
  asm volatile("st.shared.v2.f32 [%0], {%1, %2};" ::"r"(saddr), "f"(a), "f"(b) : "memory");
}
// 4-byte shared-memory store through a shared-window address
__device__ __forceinline__ void st_shared_u32(uint32_t saddr, uint32_t v) {
  asm volatile("st.shared.u32 [%0], %1;" ::"r"(saddr), "r"(v) : "memory");
}
// four 8x8 16-bit matrices to shared memory: register i of lane (4g + q) holds row g, columns 2q, 2q + 1 of matrix i (the
// wgmma / mma accumulator fragment once packed); lane l gives the address of row l % 8 of matrix l / 8 (16 bytes)
__device__ __forceinline__ void stmatrix_x4(uint32_t saddr, uint32_t r0, uint32_t r1, uint32_t r2, uint32_t r3) {
  asm volatile("stmatrix.sync.aligned.m8n8.x4.shared.b16 [%0], {%1, %2, %3, %4};"
               ::"r"(saddr), "r"(r0), "r"(r1), "r"(r2), "r"(r3) : "memory");
}
__device__ __forceinline__ void tma_store_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void tma_store_wait_read() {  // <= N committed groups may still be READING shared memory
  asm volatile("cp.async.bulk.wait_group.read %0;" ::"n"(N) : "memory");
}
template <int N>
__device__ __forceinline__ void tma_store_wait_all() {   // <= N committed groups may still be in flight at all
  asm volatile("cp.async.bulk.wait_group %0;" ::"n"(N) : "memory");
}

// ----------------------------------------------------------------------------- wgmma (warpgroup MMA)
// Shared-memory matrix descriptor (64-bit), sm_90 format:
//   [0,14)  start address >> 4      [16,30) leading byte offset >> 4     [32,46) stride byte offset >> 4
//   [49,52) base offset = 0         [62,64) layout type
// K-major swizzled operands: SBO = distance between 8-row groups, LBO unused.  MN-major: LBO = distance between the
// swizzle-wide column blocks of the MN dimension, SBO = distance between 8-row groups of the K dimension.
enum : uint32_t { GMMA_LAYOUT_NONE = 0, GMMA_LAYOUT_SW128 = 1, GMMA_LAYOUT_SW64 = 2, GMMA_LAYOUT_SW32 = 3 };

__device__ __forceinline__ uint64_t gmma_desc(uint32_t saddr, uint32_t lbo_bytes, uint32_t sbo_bytes, uint32_t layout) {
  uint64_t d = 0;
  d |= static_cast<uint64_t>((saddr >> 4) & 0x3FFF);
  d |= static_cast<uint64_t>((lbo_bytes >> 4) & 0x3FFF) << 16;
  d |= static_cast<uint64_t>((sbo_bytes >> 4) & 0x3FFF) << 32;
  d |= static_cast<uint64_t>(layout) << 62;
  return d;
}
// Advance the start-address field by `bytes` (must keep the swizzle phase: multiples of 32 B inside a 128B-swizzle row for
// K-major operands, multiples of the 8-row group for the strided dimension).
__device__ __forceinline__ uint64_t gmma_desc_advance(uint64_t desc, uint32_t bytes) {
  return desc + static_cast<uint64_t>(bytes >> 4);
}
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
// keeps the compiler from moving accumulator reads / writes across an in-flight wgmma
template <int N>
__device__ __forceinline__ void reg_fence(float (&d)[N]) {
#pragma unroll
  for (int i = 0; i < N; ++i) asm volatile("" : "+f"(d[i])::"memory");
}

// ----------------------------------------------------------------------------- 16-bit packing
template <bool BF16>
__device__ __forceinline__ uint32_t pack2(float a, float b) {
  if constexpr (BF16) {
    __nv_bfloat162 v = __floats2bfloat162_rn(a, b);
    return *reinterpret_cast<uint32_t*>(&v);
  } else {
    __half2 v = __floats2half2_rn(a, b);
    return *reinterpret_cast<uint32_t*>(&v);
  }
}
template <bool BF16>
__device__ __forceinline__ float2 unpack2(uint32_t u) {
  if constexpr (BF16) {
    return __bfloat1622float2(*reinterpret_cast<__nv_bfloat162*>(&u));
  } else {
    return __half22float2(*reinterpret_cast<__half2*>(&u));
  }
}

// ----------------------------------------------------------------------------- e4m3 packing
// four fp32 values -> four e4m3 bytes, a in the lowest: round to nearest even, saturating to +-448 (cvt puts its first
// source operand in the upper byte of each pair)
__device__ __forceinline__ uint32_t pack_e4m3x4(float a, float b, float c, float d) {
  uint16_t lo, hi;
  asm("cvt.rn.satfinite.e4m3x2.f32 %0, %1, %2;" : "=h"(lo) : "f"(b), "f"(a));
  asm("cvt.rn.satfinite.e4m3x2.f32 %0, %1, %2;" : "=h"(hi) : "f"(d), "f"(c));
  return static_cast<uint32_t>(lo) | (static_cast<uint32_t>(hi) << 16);
}
// the per-row scale of an e4m3 operand: amax / 448 (448 = the largest finite e4m3), 1 for an all-zero row
__device__ __forceinline__ float e4m3_scale(float amax) { return amax > 0.f ? __fdiv_rn(amax, 448.0f) : 1.0f; }

}  // namespace b200
