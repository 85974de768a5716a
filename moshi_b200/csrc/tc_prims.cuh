// sm_90a primitives shared by the tensor-core kernels (gemm_sk.cu, gemm_ns.cu, dep_fused.cu, mimi_tc.cu): mbarriers, bulk /
// tensor TMA copies, warpgroup MMA (wgmma) fences and fragment coordinates, shared-memory matrix descriptors, programmatic
// dependent launch.
#pragma once

#include <cuda.h>
#include <stdint.h>

#include "wgmma_ops.cuh"

namespace b200 {
namespace tcp {

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
__device__ __forceinline__ uint64_t global_timer_ns() {
  uint64_t t;
  asm volatile("mov.u64 %0, %globaltimer;" : "=l"(t));
  return t;
}
// Bounded wait: a pipeline bug must surface as a launch failure, never as a hung GPU.  The bound is wall-clock (10 s on
// %globaltimer, sampled every 4096 polls), not a poll count: under programmatic dependent launch the consumer warps poll while
// the producer warp sits in griddepcontrol.wait for the whole predecessor kernel, and a profiler, a debugger or a
// time-sliced neighbour can stretch that by orders of magnitude without anything being wrong.
constexpr uint64_t WAIT_LIMIT_NS = 10ull * 1000ull * 1000ull * 1000ull;
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
  uint32_t done, spins = 0;
  uint64_t t0 = 0;
  do {
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
        "selp.u32 %0, 1, 0, p;\n\t}"
        : "=r"(done) : "r"(bar), "r"(parity) : "memory");
    if (!done && (++spins & 4095u) == 0u) {
      const uint64_t now = global_timer_ns();
      if (t0 == 0) t0 = now;
      else if (now - t0 > WAIT_LIMIT_NS) __trap();
    }
  } while (!done);
}
__device__ __forceinline__ void bulk_load(uint32_t dst, const void* src, uint32_t bytes, uint32_t bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
               ::"r"(dst), "l"(src), "r"(bytes), "r"(bar) : "memory");
}
__device__ __forceinline__ void tma_load_2d(uint32_t dst, const CUtensorMap* map, uint32_t bar, int c0, int c1) {
  asm volatile("cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
               ::"r"(dst), "l"(map), "r"(bar), "r"(c0), "r"(c1) : "memory");
}
__device__ __forceinline__ void tma_load_3d(uint32_t dst, const CUtensorMap* map, uint32_t bar, int c0, int c1, int c2) {
  asm volatile("cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5}], [%2];"
               ::"r"(dst), "l"(map), "r"(bar), "r"(c0), "r"(c1), "r"(c2) : "memory");
}
// Warpgroup MMA (wgmma): the four warps of a warpgroup issue together; `wg_fence` orders register / shared-memory writes
// before the MMAs that read them, `wg_commit` closes a group of issued MMAs, `wg_wait<n>` waits until at most n groups are
// still in flight (their accumulator registers and the shared-memory operands they read are then free).
__device__ __forceinline__ void wg_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wg_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wg_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
// keeps the compiler from moving accesses of an accumulator across the asynchronous MMAs that own it
template <int R>
__device__ __forceinline__ void wg_hold(uint32_t (&d)[R]) {
#pragma unroll
  for (int i = 0; i < R; ++i) asm volatile("" : "+r"(d[i])::"memory");
}
// (row, column) of accumulator element i of an m64nN fragment, for thread t (0..127) of its warpgroup
__device__ __forceinline__ int frag_row(int t, int i) { return 16 * (t >> 5) + ((t & 31) >> 2) + 8 * ((i >> 1) & 1); }
__device__ __forceinline__ int frag_col(int t, int i) { return 8 * (i >> 2) + 2 * (t & 3) + (i & 1); }
// named barrier over `count` threads (ids 1..15; 0 is __syncthreads)
__device__ __forceinline__ void named_bar(int id, int count) { asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(count) : "memory"); }
// Programmatic dependent launch: `pdl_wait` blocks until the preceding kernel in the stream has completed and its
// writes are visible; `pdl_trigger` lets the following kernel start its own prologue (and weight prefetch) early.
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
__device__ __forceinline__ void pdl_trigger() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }

// K-major SWIZZLE_128B shared-memory matrix descriptor (sm_90): start address >> 4 (bits 0-13), leading byte offset 1 (unused
// for swizzled K-major), stride byte offset 1024 B >> 4 (8 rows x 128 B, bits 32-45), layout type 1 = SWIZZLE_128B (bits 62-63).
// Tiles are 1024-byte aligned, so the base offset (bits 49-51) is 0; a K step inside the 128-byte row adds its byte offset.
__device__ __forceinline__ uint64_t make_desc(uint32_t smem_addr) {
  uint64_t d = (uint64_t)((smem_addr & 0x3FFFFu) >> 4);
  d |= (uint64_t)1 << 16;
  d |= (uint64_t)(1024 >> 4) << 32;
  d |= (uint64_t)1 << 62;
  return d;
}

// distributed shared memory of a thread block cluster: the address of `local_smem_addr` in rank `rank`'s shared memory, a
// two-word store there, and a barrier over every thread of the cluster (release / acquire)
__device__ __forceinline__ uint32_t map_to_rank(uint32_t local_smem_addr, uint32_t rank) {
  uint32_t r;
  asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(r) : "r"(local_smem_addr), "r"(rank));
  return r;
}
__device__ __forceinline__ void st_cluster_v2(uint32_t addr, uint32_t a, uint32_t b) {
  asm volatile("st.shared::cluster.v2.b32 [%0], {%1, %2};" ::"r"(addr), "r"(a), "r"(b) : "memory");
}
__device__ __forceinline__ void cluster_sync_all() {
  asm volatile("barrier.cluster.arrive.release.aligned;" ::: "memory");
  asm volatile("barrier.cluster.wait.acquire.aligned;" ::: "memory");
}
__device__ __forceinline__ float bf16_round(float v) { return __bfloat162float(__float2bfloat16_rn(v)); }

}  // namespace tcp
}  // namespace b200
