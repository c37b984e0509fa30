// Thin inline-PTX layer for sm_90a: mbarrier, TMA (cp.async.bulk.tensor), programmatic
// dependent launch, cross-GPU memory ordering.  The warpgroup MMA lives in wgmma.cuh.
//
// Everything in this file is a direct statement of the PTX ISA; there is no
// reference-code counterpart (the reference, iammcy/BFLC-demo, ships no GPU
// code at all -- see SURVEY.md section 2.7).
#pragma once
#include <cstdint>
#include <cuda.h>
#include <cuda_runtime.h>

namespace bflc {
namespace ptx {

// ----------------------------------------------------------------------------
// misc
// ----------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}

__device__ __forceinline__ bool elect_one() {
  uint32_t pred = 0;
  asm volatile(
      "{\n\t.reg .pred P;\n\t"
      "elect.sync _|P, 0xffffffff;\n\t"
      "selp.u32 %0, 1, 0, P;\n\t}\n"
      : "=r"(pred));
  return pred != 0;
}

#ifndef BFLC_SPIN_LIMIT
// Every wait loop is bounded: a protocol bug traps instead of hanging the GPU
// box.
#define BFLC_SPIN_LIMIT (1ull << 31)
#endif

// ----------------------------------------------------------------------------
// programmatic dependent launch (PDL)
// ----------------------------------------------------------------------------
__device__ __forceinline__ void pdl_launch_dependents() {
  asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
}
__device__ __forceinline__ void pdl_wait() {
  asm volatile("griddepcontrol.wait;" ::: "memory");
}

// ----------------------------------------------------------------------------
// mbarrier
// ----------------------------------------------------------------------------
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void fence_mbar_init() {
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)),
               "r"(bytes)
               : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n\t.reg .pred P;\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 P, [%1], %2;\n\t"
      "selp.u32 %0, 1, 0, P;\n\t}\n"
      : "=r"(ok)
      : "r"(smem_u32(bar)), "r"(parity)
      : "memory");
  return ok != 0;
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  unsigned long long spins = 0;
  while (!mbar_try_wait(bar, parity)) {
    if (++spins > BFLC_SPIN_LIMIT) __trap();
  }
}

// ----------------------------------------------------------------------------
// thread-block clusters: cluster barrier, remote mbarrier arrive, distributed shared memory
// ----------------------------------------------------------------------------
__device__ __forceinline__ void cluster_sync() {
  asm volatile("barrier.cluster.arrive.release.aligned;\n\tbarrier.cluster.wait.acquire.aligned;" ::: "memory");
}
// the same shared-memory offset in cluster CTA `rank`
__device__ __forceinline__ uint32_t mapa(uint32_t smem_addr, uint32_t rank) {
  uint32_t r;
  asm("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(r) : "r"(smem_addr), "r"(rank));
  return r;
}
// arrive on the mbarrier at the same smem offset in cluster CTA `rank`
__device__ __forceinline__ void mbar_arrive_cluster(uint64_t* bar, uint32_t rank) {
  asm volatile("mbarrier.arrive.release.cluster.shared::cluster.b64 _, [%0];" ::"r"(mapa(smem_u32(bar), rank))
               : "memory");
}
// wait for a phase that other CTAs of the cluster complete: acquire at cluster scope, so their
// writes released by mbar_arrive_cluster are visible afterwards
__device__ __forceinline__ void mbar_wait_cluster(uint64_t* bar, uint32_t parity) {
  unsigned long long spins = 0;
  while (true) {
    uint32_t ok;
    asm volatile(
        "{\n\t.reg .pred P;\n\t"
        "mbarrier.try_wait.parity.acquire.cluster.shared::cta.b64 P, [%1], %2;\n\t"
        "selp.u32 %0, 1, 0, P;\n\t}\n"
        : "=r"(ok)
        : "r"(smem_u32(bar)), "r"(parity)
        : "memory");
    if (ok) break;
    if (++spins > BFLC_SPIN_LIMIT) __trap();
  }
}
// The same, with the default (CTA-scope) release: enough to tell a peer that this CTA is done
// READING something the peer may now overwrite, and without the GPU-scope memory barrier that a
// cluster-scope release costs per arrive.
__device__ __forceinline__ void mbar_arrive_remote(uint64_t* bar, uint32_t rank) {
  asm volatile("mbarrier.arrive.shared::cluster.b64 _, [%0];" ::"r"(mapa(smem_u32(bar), rank)) : "memory");
}
// Bulk copy (TMA engine) of `bytes` from this CTA's shared memory to a cluster CTA's (dst, bar:
// shared::cluster addresses from mapa), completing the bytes as transactions on that CTA's
// mbarrier `bar`.  The source must be fenced for the async proxy (fence_proxy_async_smem).
__device__ __forceinline__ void bulk_s2cluster(uint32_t dst, const void* src, uint32_t bytes, uint32_t bar) {
  asm volatile("cp.async.bulk.shared::cluster.shared::cta.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
               ::"r"(dst), "r"(smem_u32(src)), "r"(bytes), "r"(bar)
               : "memory");
}

// ----------------------------------------------------------------------------
// proxy fences around TMA and wgmma
// ----------------------------------------------------------------------------
// generic-proxy writes -> visible to the async proxy (TMA / wgmma smem reads)
__device__ __forceinline__ void fence_proxy_async_smem() {
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}
__device__ __forceinline__ void fence_proxy_async_all() {
  asm volatile("fence.proxy.async;" ::: "memory");
}

// ----------------------------------------------------------------------------
// TMA
// ----------------------------------------------------------------------------
__device__ __forceinline__ void tma_prefetch_desc(const void* tmap) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(tmap)) : "memory");
}

// 3-D tiled load: coordinates are (c0 = innermost element, c1 = row, c2 = batch)
__device__ __forceinline__ void tma_load_3d(void* smem_dst, const void* tmap, uint64_t* bar,
                                            int32_t c0, int32_t c1, int32_t c2) {
  asm volatile(
      "cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes "
      "[%0], [%1, {%3, %4, %5}], [%2];"
      :
      : "r"(smem_u32(smem_dst)), "l"(reinterpret_cast<uint64_t>(tmap)), "r"(smem_u32(bar)),
        "r"(c0), "r"(c1), "r"(c2)
      : "memory");
}

// 1-D bulk copy global -> shared (bytes and both addresses multiples of 16)
__device__ __forceinline__ void bulk_load(void* smem_dst, const void* gsrc, uint32_t bytes, uint64_t* bar) {
  asm volatile(
      "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
      :
      : "r"(smem_u32(smem_dst)), "l"(reinterpret_cast<uint64_t>(gsrc)), "r"(bytes), "r"(smem_u32(bar))
      : "memory");
}

// 4-D tiled load (NHWC activation boxes for the implicit-GEMM convolution): coordinates are
// (c0 = channel, c1 = w, c2 = h, c3 = image); out-of-range coordinates are zero-filled, which
// is the convolution's padding.
__device__ __forceinline__ void tma_load_4d(void* smem_dst, const void* tmap, uint64_t* bar,
                                            int32_t c0, int32_t c1, int32_t c2, int32_t c3) {
  asm volatile(
      "cp.async.bulk.tensor.4d.shared::cluster.global.mbarrier::complete_tx::bytes "
      "[%0], [%1, {%3, %4, %5, %6}], [%2];"
      :
      : "r"(smem_u32(smem_dst)), "l"(reinterpret_cast<uint64_t>(tmap)), "r"(smem_u32(bar)),
        "r"(c0), "r"(c1), "r"(c2), "r"(c3)
      : "memory");
}

// ----------------------------------------------------------------------------
// cross-GPU (system scope) ordering for peer-mapped memory
// ----------------------------------------------------------------------------
__device__ __forceinline__ void st_release_sys(uint32_t* p, uint32_t v) {
  asm volatile("st.release.sys.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ uint32_t ld_acquire_sys(const uint32_t* p) {
  uint32_t v;
  asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ uint32_t ld_relaxed_sys(const uint32_t* p) {
  uint32_t v;
  asm volatile("ld.relaxed.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ uint32_t atom_add_sys(uint32_t* p, uint32_t v) {
  uint32_t old;
  asm volatile("atom.add.acq_rel.sys.global.u32 %0, [%1], %2;" : "=r"(old) : "l"(p), "r"(v)
               : "memory");
  return old;
}
// Wait until *p >= want (epoch-tagged flags only ever grow, so no reset race).
__device__ __forceinline__ void wait_flag_ge(const uint32_t* p, uint32_t want) {
  unsigned long long spins = 0;
  while (static_cast<int32_t>(ld_acquire_sys(p) - want) < 0) {
    if (++spins > BFLC_SPIN_LIMIT) __trap();
    __nanosleep(20);
  }
}
// 16-byte streaming load of peer-mapped (or peer-written) memory.  The data is rewritten by
// other GPUs every second round, so the non-coherent path (ld.global.nc) is not defined for
// it: a relaxed system-scope load is always served from the point of coherence and never from a
// stale L1 line; L1::no_allocate because every address is read exactly once.
__device__ __forceinline__ float4 ld_peer_f4(const float4* p) {
  float4 v;
  asm volatile("ld.relaxed.sys.global.L1::no_allocate.v4.f32 {%0, %1, %2, %3}, [%4];"
               : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w)
               : "l"(p)
               : "memory");
  return v;
}
__device__ __forceinline__ float4 ld_f4_relaxed(const float4* p) {
  float4 v;
  asm volatile("ld.global.v4.f32 {%0, %1, %2, %3}, [%4];"
               : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w)
               : "l"(p)
               : "memory");
  return v;
}
// 16-byte vector reduction (sm_90+): one L2 atomic transaction for four floats
__device__ __forceinline__ void red_add_f32x4(float* p, float a, float b, float c, float d) {
  asm volatile("red.global.add.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(p), "f"(a), "f"(b), "f"(c),
               "f"(d)
               : "memory");
}
// NVLS multicast: one store lands in every replica bound to the multicast object
__device__ __forceinline__ void multimem_st_f4(float4* mc_ptr, float4 v) {
  asm volatile("multimem.st.relaxed.sys.global.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(mc_ptr),
               "f"(v.x), "f"(v.y), "f"(v.z), "f"(v.w)
               : "memory");
}
__device__ __forceinline__ float4 multimem_ld_reduce_add_f4(const float4* mc_ptr) {
  float4 v;
  asm volatile("multimem.ld_reduce.relaxed.sys.global.add.v4.f32 {%0, %1, %2, %3}, [%4];"
               : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w)
               : "l"(mc_ptr)
               : "memory");
  return v;
}

}  // namespace ptx
}  // namespace bflc
