// Thin inline-PTX wrappers for the sm_90a features used by the tensor-core kernels:
// mbarrier, TMA (cp.async.bulk.tensor), warpgroup MMA (wgmma.mma_async from shared-memory descriptors), proxy fences,
// thread-block clusters.  Encodings follow the PTX ISA 8.x (matrix descriptor format of the
// asynchronous warpgroup-level matrix instructions).
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <stdint.h>

namespace tfgnn {
namespace ptx {

__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}

// ---- mbarrier ------------------------------------------------------------------------------
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void fence_barrier_init() {
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes)
               : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  const uint32_t addr = smem_u32(bar);
  uint32_t done;
  do {
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
        "selp.u32 %0, 1, 0, p;\n\t}"
        : "=r"(done)
        : "r"(addr), "r"(parity)
        : "memory");
  } while (!done);
}
// Same, with `ns` nanoseconds of nanosleep between probes (ns == 0: plain spin): waiting roles otherwise take issue slots
// from the gather warps on the same schedulers.
__device__ __forceinline__ void mbar_wait_backoff(uint64_t* bar, uint32_t parity, uint32_t ns) {
  const uint32_t addr = smem_u32(bar);
  for (;;) {
    uint32_t done;
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
        "selp.u32 %0, 1, 0, p;\n\t}"
        : "=r"(done)
        : "r"(addr), "r"(parity)
        : "memory");
    if (done) break;
    if (ns) asm volatile("nanosleep.u32 %0;" ::"r"(ns));
  }
}

// ---- proxy fences ----------------------------------------------------------------------------
// generic-proxy smem writes -> visible to the async proxy (TMA / wgmma operand reads)
__device__ __forceinline__ void fence_proxy_async_smem() {
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}

// ---- TMA -------------------------------------------------------------------------------------
__device__ __forceinline__ void prefetch_tensormap(const CUtensorMap* m) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(m)) : "memory");
}
// 2-D tile load: coordinates (c0 = innermost/contiguous dim, c1 = row).  Completes on `bar` (tx bytes).
__device__ __forceinline__ void tma_load_2d(void* smem_dst, const CUtensorMap* map, uint64_t* bar, int c0, int c1) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
      ::"r"(smem_u32(smem_dst)), "l"(reinterpret_cast<uint64_t>(map)), "r"(smem_u32(bar)), "r"(c0), "r"(c1)
      : "memory");
}

// Prefetch a 2-D tile into L2 (no shared-memory destination, no barrier): issued a whole tile ahead by the GEMM's producer so
// that the later cp.async.bulk.tensor finds its lines in L2 instead of paying a loaded-HBM round trip inside the pipeline.
__device__ __forceinline__ void tma_prefetch_2d(const CUtensorMap* map, int c0, int c1) {
  asm volatile("cp.async.bulk.prefetch.tensor.2d.L2.global.tile [%0, {%1, %2}];" ::"l"(reinterpret_cast<uint64_t>(map)),
               "r"(c0), "r"(c1)
               : "memory");
}

// 2-D tile load with an L2 cache-policy operand (createpolicy).
__device__ __forceinline__ void tma_load_2d_hint(void* smem_dst, const CUtensorMap* map, uint64_t* bar, int c0,
                                                 int c1, uint64_t policy) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes.L2::cache_hint"
      " [%0], [%1, {%3, %4}], [%2], %5;"
      ::"r"(smem_u32(smem_dst)), "l"(reinterpret_cast<uint64_t>(map)), "r"(smem_u32(bar)), "r"(c0), "r"(c1),
        "l"(policy)
      : "memory");
}

// The same tile written to the same shared-memory offset in every CTA of the cluster named in cta_mask; each destination
// CTA's mbarrier at the offset of `bar` receives the complete_tx of its copy.
__device__ __forceinline__ void tma_load_2d_multicast_hint(void* smem_dst, const CUtensorMap* map, uint64_t* bar, int c0,
                                                           int c1, uint16_t cta_mask, uint64_t policy) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes.multicast::cluster.L2::cache_hint"
      " [%0], [%1, {%3, %4}], [%2], %5, %6;"
      ::"r"(smem_u32(smem_dst)), "l"(reinterpret_cast<uint64_t>(map)), "r"(smem_u32(bar)), "r"(c0), "r"(c1),
        "h"(cta_mask), "l"(policy)
      : "memory");
}

// ---- register reallocation between warpgroups (every warp of the warpgroup executes it) ----
template <uint32_t REGS>
__device__ __forceinline__ void setmaxnreg_inc() { asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(REGS)); }
template <uint32_t REGS>
__device__ __forceinline__ void setmaxnreg_dec() { asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(REGS)); }

// ---- L2 eviction policies (keep the producer/consumer ring, stream everything else) ----
__device__ __forceinline__ uint64_t policy_evict_first() {
  uint64_t p;
  asm volatile("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(p));
  return p;
}
__device__ __forceinline__ uint64_t policy_evict_last() {
  uint64_t p;
  asm volatile("createpolicy.fractional.L2::evict_last.b64 %0, 1.0;" : "=l"(p));
  return p;
}
// Drop a 128 B line from L2 WITHOUT writing it back (producer/consumer scratch that is dead after the read).
__device__ __forceinline__ void discard_l2_128(const void* ptr) {
  asm volatile("discard.global.L2 [%0], 128;" ::"l"(ptr) : "memory");
}
// LDGSTS, L1 bypass.
__device__ __forceinline__ void cp_async16(uint32_t smem_addr, const void* gptr) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(smem_addr), "l"(gptr) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
__device__ __forceinline__ void sts_f4(uint32_t saddr, float4 v) {
  asm volatile("st.shared.v4.f32 [%0], {%1,%2,%3,%4};" ::"r"(saddr), "f"(v.x), "f"(v.y), "f"(v.z), "f"(v.w) : "memory");
}
__device__ __forceinline__ void sts_u4(uint32_t saddr, uint4 v) {
  asm volatile("st.shared.v4.b32 [%0], {%1,%2,%3,%4};" ::"r"(saddr), "r"(v.x), "r"(v.y), "r"(v.z), "r"(v.w) : "memory");
}
__device__ __forceinline__ float4 lds_f4(uint32_t saddr) {
  float4 v;
  asm volatile("ld.shared.v4.f32 {%0,%1,%2,%3}, [%4];" : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "r"(saddr) : "memory");
  return v;
}
__device__ __forceinline__ void st_f4_hint(float* ptr, float4 v, uint64_t policy) {
  asm volatile("st.global.L2::cache_hint.v4.f32 [%0], {%1, %2, %3, %4}, %5;" ::"l"(ptr), "f"(v.x), "f"(v.y),
               "f"(v.z), "f"(v.w), "l"(policy)
               : "memory");
}

// ---- warpgroup MMA (wgmma) ------------------------------------------------------------------------
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
// Keeps the compiler from moving accesses of an accumulator register across a wgmma wait.
__device__ __forceinline__ void reg_fence(float& x) { asm volatile("" : "+f"(x)::"memory"); }
// Barrier over the 128 threads of one warpgroup (id 1..15; 0 is __syncthreads).
__device__ __forceinline__ void warpgroup_sync(int id) { asm volatile("bar.sync %0, 128;" ::"r"(id) : "memory"); }

// Shared-memory matrix descriptor of a K-major tile with 128-byte (ROW_BYTES = 128: 32 tf32 per row, 8-row groups 1024 B
// apart) or 64-byte swizzle (ROW_BYTES = 64, groups 512 B apart): start[0,14) LBO[16,30) SBO[32,46) layout[62,64)
// (1 = SWIZZLE_128B, 2 = SWIZZLE_64B); tile base aligned to the 8-row group.  A step of 8 tf32 (or 16 bf16) along K inside
// the swizzle row adds 32 B to the start address.
template <int ROW_BYTES>
__device__ __forceinline__ uint64_t gmma_desc_k(uint32_t smem_addr) {
  uint64_t d = 0;
  d |= (uint64_t)((smem_addr >> 4) & 0x3FFF);
  d |= (uint64_t)1 << 16;                                    // LBO (unused for swizzled K-major)
  d |= (uint64_t)((8 * ROW_BYTES) >> 4) << 32;               // SBO
  d |= (uint64_t)(ROW_BYTES == 128 ? 1 : 2) << 62;
  return d;
}

// ---- thread-block clusters ---------------------------------------------------------------------
__device__ __forceinline__ uint32_t cluster_ctarank() {
  uint32_t r;
  asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r));
  return r;
}
__device__ __forceinline__ void cluster_sync_all() {   // every thread of every CTA in the cluster
  asm volatile("barrier.cluster.arrive.release.aligned;\n\tbarrier.cluster.wait.acquire.aligned;" ::: "memory");
}
// shared::cluster address of `local` (a shared::cta address of this CTA) in CTA `rank` of the cluster
__device__ __forceinline__ uint32_t mapa_shared(uint32_t local, uint32_t rank) {
  uint32_t r;
  asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(r) : "r"(local), "r"(rank));
  return r;
}
__device__ __forceinline__ void mbar_arrive_cluster(uint32_t cluster_addr) {   // arrive on another CTA's mbarrier
  asm volatile("mbarrier.arrive.shared::cluster.b64 _, [%0];" ::"r"(cluster_addr) : "memory");
}
// Cluster-scope release / acquire: the arriving thread's earlier writes (shared OR global) become visible to a thread of
// ANOTHER CTA of the cluster that observes the phase with mbar_wait_cluster (split-tile mode of the fused kernel).
__device__ __forceinline__ void mbar_arrive_cluster_release(uint32_t cluster_addr) {
  asm volatile("mbarrier.arrive.release.cluster.shared::cluster.b64 _, [%0];" ::"r"(cluster_addr) : "memory");
}
__device__ __forceinline__ void mbar_wait_cluster(uint64_t* bar, uint32_t parity) {
  const uint32_t addr = smem_u32(bar);
  uint32_t done;
  do {
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "mbarrier.try_wait.parity.acquire.cluster.shared::cta.b64 p, [%1], %2;\n\t"
        "selp.u32 %0, 1, 0, p;\n\t}"
        : "=r"(done)
        : "r"(addr), "r"(parity)
        : "memory");
  } while (!done);
}
// ---- bf16-pair correction operands ----------------------------------------------------------------------------
// 3xTF32 needs A_hi B_hi + (A_lo B_hi + A_hi B_lo).  The two small products only need ~8 bits each, so they run as ONE
// kind::f16 (bf16) MMA over a K-interleaved operand: the 32-bit word at the position of fp32 element k holds the bf16
// pair (A: bf16(a_k) | bf16(a_k - tf32(a_k)),  B: bf16(b_k - tf32(b_k)) | bf16(b_k)), low half first.  A row of 32 fp32
// words is then a row of 64 bf16 K-elements in the SAME bytes, swizzle and descriptors as the fp32 tile, and
//   sum_j A'_j B'_j = sum_k a_k lo(b_k) + lo(a_k) b_k.
// Tensor work per K block: 4 tf32 + 4 bf16 instructions instead of 12 tf32 (-33 %); the splitter writes one tile, not two.
__device__ __forceinline__ uint32_t pack_bf16x2(float upper, float lower) {
  uint32_t d;
  asm("cvt.rn.bf16x2.f32 %0, %1, %2;" : "=r"(d) : "f"(upper), "f"(lower));
  return d;
}
// tf32 split of an fp32 value: hi keeps sign/exponent/10 mantissa bits (exact truncation, so the
// tensor core sees the same bits whether it truncates or rounds), lo = x - hi (exact in fp32).
__host__ __device__ __forceinline__ float tf32_hi(float x) {
#ifdef __CUDA_ARCH__
  return __uint_as_float(__float_as_uint(x) & 0xFFFFE000u);
#else
  union { float f; uint32_t u; } c; c.f = x; c.u &= 0xFFFFE000u; return c.f;
#endif
}

}  // namespace ptx
}  // namespace tfgnn
