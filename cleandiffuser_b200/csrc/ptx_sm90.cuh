// Thin inline-PTX wrappers for the Hopper (sm_90a) async machinery: mbarrier, TMA (cp.async.bulk.tensor), programmatic
// dependent launch and the wgmma shared-memory matrix descriptor (the MMA instructions themselves: wgmma_sm90.cuh).
// Bit layouts follow the PTX ISA "asynchronous warpgroup level matrix" descriptor table.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "wgmma_sm90.cuh"

namespace cds {
namespace ptx {

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ bool elect_one() {
  uint32_t pred;
  asm volatile(
      "{\n\t.reg .pred p;\n\telect.sync _|p, 0xffffffff;\n\tselp.u32 %0, 1, 0, p;\n\t}\n"
      : "=r"(pred));
  return pred != 0;
}

// ---------------------------------------------------------------- mbarrier
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void fence_barrier_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  asm volatile(
      "{\n\t.reg .pred p;\n"
      "WAIT_%=:\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n\t"
      "@p bra DONE_%=;\n\t"
      "bra WAIT_%=;\n"
      "DONE_%=:\n\t}\n" ::"r"(smem_u32(bar)),
      "r"(parity)
      : "memory");
}

// ---------------------------------------------------------------- TMA (tile mode, mbarrier completion)
__device__ __forceinline__ void prefetch_tensormap(const void* tmap) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(tmap) : "memory");
}
__device__ __forceinline__ void tma_load_2d(void* smem_dst, const void* tmap, uint64_t* bar, int c0, int c1) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];" ::"r"(
          smem_u32(smem_dst)),
      "l"(tmap), "r"(smem_u32(bar)), "r"(c0), "r"(c1)
      : "memory");
}
__device__ __forceinline__ void tma_load_3d(void* smem_dst, const void* tmap, uint64_t* bar, int c0, int c1, int c2) {
  asm volatile(
      "cp.async.bulk.tensor.3d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5}], [%2];" ::
          "r"(smem_u32(smem_dst)),
      "l"(tmap), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2)
      : "memory");
}

// TMA store (tile mode, bulk-group completion): shared -> global box at the given coordinates; out-of-bound parts of the box
// are clipped by the TMA unit.  The shared-memory source must have been written with the tensor map's swizzle and made
// visible to the async proxy (fence_proxy_async) before the issue.
// pull a box into L2 without a destination (no completion mechanism: a hint)
__device__ __forceinline__ void tma_prefetch_2d(const void* tmap, int c0, int c1) {
  asm volatile("cp.async.bulk.prefetch.tensor.2d.L2.global.tile [%0, {%1, %2}];" ::"l"(tmap), "r"(c0), "r"(c1) : "memory");
}
__device__ __forceinline__ void tma_store_2d(const void* tmap, const void* smem_src, int c0, int c1) {
  asm volatile("cp.async.bulk.tensor.2d.global.shared::cta.tile.bulk_group [%0, {%2, %3}], [%1];" ::"l"(tmap), "r"(smem_u32(smem_src)),
               "r"(c0), "r"(c1)
               : "memory");
}
__device__ __forceinline__ void tma_store_3d(const void* tmap, const void* smem_src, int c0, int c1, int c2) {
  asm volatile("cp.async.bulk.tensor.3d.global.shared::cta.tile.bulk_group [%0, {%2, %3, %4}], [%1];" ::"l"(tmap),
               "r"(smem_u32(smem_src)), "r"(c0), "r"(c1), "r"(c2)
               : "memory");
}
__device__ __forceinline__ void tma_store_4d(const void* tmap, const void* smem_src, int c0, int c1, int c2, int c3) {
  asm volatile("cp.async.bulk.tensor.4d.global.shared::cta.tile.bulk_group [%0, {%2, %3, %4, %5}], [%1];" ::"l"(tmap),
               "r"(smem_u32(smem_src)), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
               : "memory");
}
__device__ __forceinline__ void bulk_commit_group() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
// wait until at most N of this thread's bulk groups still READ their shared-memory source (the source may then be reused)
template <int N>
__device__ __forceinline__ void bulk_wait_group_read() { asm volatile("cp.async.bulk.wait_group.read %0;" ::"n"(N) : "memory"); }
// ... until at most N bulk groups are still in flight at all (writes complete)
template <int N>
__device__ __forceinline__ void bulk_wait_group() { asm volatile("cp.async.bulk.wait_group %0;" ::"n"(N) : "memory"); }

// programmatic dependent launch: wait = block until the grids this one depends on have completed and their memory is visible
// (returns at once when the launch carried no programmatic dependency); launch_dependents = this CTA no longer holds back the
// launch of the next grid in the stream
__device__ __forceinline__ void grid_dep_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
__device__ __forceinline__ void grid_dep_launch_dependents() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }

// named barrier among a subset of the CTA's warps (id 1..15; 0 is __syncthreads)
__device__ __forceinline__ void named_bar_sync(uint32_t id, uint32_t n_threads) {
  asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(n_threads) : "memory");
}

// ---------------------------------------------------------------- descriptors
// K-major operand tile in shared memory, rows of `row_bytes` (64 or 128) written by TMA with the matching swizzle:
// 8-row swizzle atoms of 8*row_bytes, atoms stacked densely along M/N (SBO = 8*row_bytes).
//   bits  0-13 start address >> 4        bits 16-29 leading byte offset >> 4 (unused for swizzled K-major: 1)
//   bits 32-45 stride byte offset >> 4   bits 62-63 layout: 1 = SWIZZLE_128B, 2 = SWIZZLE_64B
// Advancing 32 bytes along K inside the swizzle span = +2 in the start-address field.
template <int kRowBytes>
__device__ __forceinline__ uint64_t make_kmajor_desc(uint32_t smem_addr) {
  static_assert(kRowBytes == 128 || kRowBytes == 64, "row must be one swizzle span");
  constexpr uint64_t layout = kRowBytes == 128 ? 1 : 2;
  constexpr uint64_t sbo = (8 * kRowBytes) >> 4;
  return (uint64_t)((smem_addr & 0x3FFFF) >> 4) | ((uint64_t)1 << 16) | (sbo << 32) | (layout << 62);
}

// W consecutive fp32 accumulator columns of one row of a shared-memory accumulator tile (16-byte aligned)
template <int W>
__device__ __forceinline__ void acc_ld(const float* row, float (&v)[W]) {
  static_assert(W % 4 == 0, "whole float4s");
#pragma unroll
  for (int k = 0; k < W / 4; ++k) {
    const float4 f = reinterpret_cast<const float4*>(row)[k];
    v[4 * k] = f.x; v[4 * k + 1] = f.y; v[4 * k + 2] = f.z; v[4 * k + 3] = f.w;
  }
}

// one warpgroup's 64 x N wgmma accumulator (fragment layout: wgmma_sm90.cuh) -> rows [0, 64) of a row-major shared-memory tile
// of `pitch` floats per row, columns [0, N) (the caller offsets `tile` to the warpgroup's first row and column)
template <int N>
__device__ __forceinline__ void acc_store(float* tile, int pitch, const float (&d)[N / 2], int wg_thread) {
  const int r = 16 * (wg_thread >> 5) + ((wg_thread & 31) >> 2);
  const int c = 2 * (wg_thread & 3);
#pragma unroll
  for (int j = 0; j < N / 8; ++j) {
    *reinterpret_cast<float2*>(tile + r * pitch + 8 * j + c) = make_float2(d[4 * j], d[4 * j + 1]);
    *reinterpret_cast<float2*>(tile + (r + 8) * pitch + 8 * j + c) = make_float2(d[4 * j + 2], d[4 * j + 3]);
  }
}

}  // namespace ptx
}  // namespace cds
