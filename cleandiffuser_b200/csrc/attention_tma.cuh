// Persistent, TMA-fed attention for the TF32 tensor-core programs (q/k/v: fp32 storage rounded to TF32, head_dim 32, L <= 128).
//
// With one CTA per (trajectory, head) the time goes into exposed global-load latency (each CTA first pulls 38 KB of strided
// q/k/v rows, then computes, 3-4 CTAs per SM).  Here
//   * every CTA is persistent (2 per SM) and walks the (trajectory, head) work list with stride gridDim.x;
//   * warp 7 is the producer: per work item three TMA boxes {32 channels, L rows} of the (B, L, 3C) q|k|v tensor land in a
//     2-stage shared-memory ring (128-byte rows, SWIZZLE_128B), completion on a "full" mbarrier, slots handed back through an
//     "empty" mbarrier -- the loads of item i+1 (and i+2) overlap the arithmetic of item i;
//   * warps 0..6 each own one 16-query tile (L <= 112: exactly one tile per warp and item): S = Q K^T and O = P V on
//     mma.sync.m16n8k8 (tf32 operands, fp32 accumulation) with every fragment read straight from the swizzled tiles -- the XOR
//     swizzle makes all of them bank-conflict free, V needs no transposed copy;
//   * the normalised 16 x 32 output tile goes through a per-warp 2 KB staging tile and ONE cp.async.bulk.tensor store (full
//     128-byte lines; rows >= L are clipped by the TMA unit).
// The S accumulator layout of m16n8k8 (row = lane/4 (+8), columns 2c, 2c+1 with c = lane%4) becomes the A operand of P V by
// RENAMING the summation index: MMA k-slot c stands for key 2c, slot c+4 for key 2c+1 of the 8-key tile, and the V fragment is
// fetched with the same renaming (V rows 2c and 2c+1) -- no shuffles.
// Reference: nn.MultiheadAttention inside DiTBlock, cleandiffuser/nn_diffusion/dit.py:10-36.
// Algorithmic HBM bytes per (trajectory, head): 4*L*32*3 (q, k, v) + 4*L*32 (out).
#pragma once
#include "attention.cuh"
#include "conv_tc.cuh"

namespace cds {

constexpr int kAttnTmaStages = 2;
constexpr int kAttnTmaConsumers = 7;                 // compute warps; warp 7 produces
constexpr int kAttnTmaThreads = 32 * (kAttnTmaConsumers + 1);

struct AttnTmaLaunch {
  bool ok = false;
  CUtensorMap tm_qkv, tm_out;
  int n_work = 0, smem_bytes = 0;
};

__device__ __forceinline__ void mma_tf32_1688(float (&d)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
  asm volatile("mma.sync.aligned.m16n8k8.row.col.f32.tf32.tf32.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
               : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
               : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}
__device__ __forceinline__ uint32_t to_tf32(float x) { uint32_t u; asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(u) : "f"(x)); return u; }
__device__ __forceinline__ float attn_ex2(float x) {            // 2^x, flush-to-zero, no range fix-up (x <= 0 here)
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}
__device__ __forceinline__ float attn_lds(const uint8_t* p) { return *reinterpret_cast<const float*>(p); }
// polite mbarrier wait for the single producer lane: try_wait with a suspend-time hint instead of a tight spin (the spin of
// the first version took a fifth of the issue slots of the scheduler it shared with two compute warps)
__device__ __forceinline__ void attn_mbar_wait_relaxed(uint64_t* bar, uint32_t parity) {
  asm volatile(
      "{\n\t.reg .pred p;\n"
      "WAIT_%=:\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1, %2;\n\t"
      "@p bra DONE_%=;\n\t"
      "bra WAIT_%=;\n"
      "DONE_%=:\n\t}\n" ::"r"(ptx::smem_u32(bar)), "r"(parity), "r"(20000u)
      : "memory");
}

// Addressing.  A tile is rows of 128 bytes under SWIZZLE_128B: element (row, channel f) sits at byte
//   row * 128 + (((f >> 2) ^ (row & 7)) << 4) + (f & 3) * 4.
// With a 1024-byte aligned tile and rows written as (8 * tile + r), the 16-byte chunk index only enters through an XOR on address
// bits 4..6, so every fragment address is  base + (lane_constant ^ (chunk << 4)) + 1024 * tile : eight per-lane registers per
// operand, everything else is an immediate.  NT = number of 8-key score tiles = ceil(L / 8), a template parameter.
template <int NT>
__global__ void __launch_bounds__(kAttnTmaThreads, 2)
attention_tma_tf32_hd32_kernel(const cds_attn_op p, const __grid_constant__ CUtensorMap tm_qkv,
                               const __grid_constant__ CUtensorMap tm_out, int n_work) {
  constexpr int HD = 32;
  extern __shared__ uint8_t attn_smem_raw[];
  __shared__ __align__(8) uint64_t full_bar[kAttnTmaStages], empty_bar[kAttnTmaStages];
  const int L = p.L;
  const int LP = (L + 15) & ~15;                     // rows per tile: whole 16-query tiles (pad rows stay zero)
  const int tile_b = LP * 128;                       // bytes per q / k / v tile
  const uint32_t base_u = (ptx::smem_u32(attn_smem_raw) + 1023u) & ~1023u;
  uint8_t* sm = attn_smem_raw + (base_u - ptx::smem_u32(attn_smem_raw));
  uint8_t* s_out = sm + kAttnTmaStages * 3 * tile_b; // [consumer warp][16 rows x 128 B]
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;

  if (threadIdx.x == 0) {
    for (int s = 0; s < kAttnTmaStages; ++s) { ptx::mbar_init(&full_bar[s], 1); ptx::mbar_init(&empty_bar[s], kAttnTmaConsumers); }
    ptx::fence_barrier_init();
    ptx::prefetch_tensormap(&tm_qkv);
    ptx::prefetch_tensormap(&tm_out);
  }
  // rows [L, LP) of every tile are never written by TMA (the box has L rows): zero them once.  (P is 0 for those keys, but
  // 0 * stale NaN would still poison the P V product.)
  {
    const int pad_f = (LP - L) * 32;
    for (int idx = threadIdx.x; idx < kAttnTmaStages * 3 * pad_f; idx += blockDim.x) {
      const int t = idx / pad_f, r = idx - t * pad_f;
      reinterpret_cast<float*>(sm + (size_t)t * tile_b)[L * 32 + r] = 0.f;
    }
  }
  ptx::fence_proxy_async();
  __syncthreads();

  if (warp == kAttnTmaConsumers) {                   // ------------------------------------------------ producer
    if (lane == 0) {
      int it = 0;
      for (int w = blockIdx.x; w < n_work; w += gridDim.x, ++it) {
        const int s = it % kAttnTmaStages;
        const uint32_t ph = (uint32_t)(it / kAttnTmaStages) & 1u;
        attn_mbar_wait_relaxed(&empty_bar[s], ph ^ 1u);
        const int b = w / p.heads, h = w - b * p.heads;
        uint8_t* dst = sm + (size_t)s * 3 * tile_b;
        ptx::mbar_expect_tx(&full_bar[s], (uint32_t)(3 * L * 128));
        ptx::tma_load_3d(dst, &tm_qkv, &full_bar[s], h * HD, 0, b);
        ptx::tma_load_3d(dst + tile_b, &tm_qkv, &full_bar[s], p.C + h * HD, 0, b);
        ptx::tma_load_3d(dst + 2 * tile_b, &tm_qkv, &full_bar[s], 2 * p.C + h * HD, 0, b);
      }
    }
    return;
  }

  // ---------------------------------------------------------------------------------------------------- consumers
  const int gr = lane >> 2, c = lane & 3;            // fragment row (0..7), k-slot / column-pair index (0..3)
  const float scale_log2e = rsqrtf((float)HD) * 1.4426950408889634f;
  // per-lane constants of the three fragment patterns (see "Addressing")
  const uint32_t lane_k = (uint32_t)(gr * 128 + (gr << 4) + c * 4);                     // K / Q: row gr (+ 8 * tile), word c
  const uint32_t lane_v0 = (uint32_t)((2 * c) * 128 + ((((gr >> 2) ^ (2 * c)) & 7) << 4) + (gr & 3) * 4);          // V row 2c, dim gr (+ 8 dn)
  const uint32_t lane_v1 = (uint32_t)((2 * c + 1) * 128 + ((((gr >> 2) ^ (2 * c + 1)) & 7) << 4) + (gr & 3) * 4);  // V row 2c + 1
  uint8_t* my_out = s_out + warp * 2048;
  const uint32_t out_lo = (uint32_t)(gr * 128 + (c & 1) * 8);                            // staging row gr (and gr + 8), words 2 (c & 1)..
  const int od = p.out_dtype;
  int it = 0;
  for (int w = blockIdx.x; w < n_work; w += gridDim.x, ++it) {
    const int s = it % kAttnTmaStages;
    const uint32_t ph = (uint32_t)(it / kAttnTmaStages) & 1u;
    const int b = w / p.heads, h = w - b * p.heads;
    const uint8_t* Qs = sm + (size_t)s * 3 * tile_b;
    const uint8_t* Ks = Qs + tile_b;
    const uint8_t* Vs = Ks + tile_b;
    const uint8_t* kx[8];
#pragma unroll
    for (int ch = 0; ch < 8; ++ch) kx[ch] = Ks + (lane_k ^ (uint32_t)(ch << 4));
    ptx::mbar_wait(&full_bar[s], ph);
    for (int qt = warp; qt * 16 < L; qt += kAttnTmaConsumers) {
      const uint8_t* qrow = Qs + qt * 2048;
      uint32_t aq[4][4];
#pragma unroll
      for (int ks = 0; ks < 4; ++ks) {
        const uint32_t o0 = lane_k ^ (uint32_t)((2 * ks) << 4), o1 = lane_k ^ (uint32_t)((2 * ks + 1) << 4);
        aq[ks][0] = __float_as_uint(attn_lds(qrow + o0));
        aq[ks][1] = __float_as_uint(attn_lds(qrow + o0 + 1024));
        aq[ks][2] = __float_as_uint(attn_lds(qrow + o1));
        aq[ks][3] = __float_as_uint(attn_lds(qrow + o1 + 1024));
      }
      float sc[NT][4];
#pragma unroll
      for (int nt = 0; nt < NT; ++nt) {
        sc[nt][0] = sc[nt][1] = sc[nt][2] = sc[nt][3] = 0.f;
#pragma unroll
        for (int ks = 0; ks < 4; ++ks)
          mma_tf32_1688(sc[nt], aq[ks], __float_as_uint(attn_lds(kx[2 * ks] + nt * 1024)), __float_as_uint(attn_lds(kx[2 * ks + 1] + nt * 1024)));
      }
      {                                              // keys >= L exist only in the last score tile
        const int j = (NT - 1) * 8 + 2 * c;
        if (j >= L) sc[NT - 1][0] = sc[NT - 1][2] = -INFINITY;
        if (j + 1 >= L) sc[NT - 1][1] = sc[NT - 1][3] = -INFINITY;
      }
      float m0 = -INFINITY, m1 = -INFINITY;
#pragma unroll
      for (int nt = 0; nt < NT; ++nt) {
        m0 = fmaxf(m0, fmaxf(sc[nt][0], sc[nt][1]));
        m1 = fmaxf(m1, fmaxf(sc[nt][2], sc[nt][3]));
      }
      m0 = fmaxf(m0, __shfl_xor_sync(0xffffffffu, m0, 1)); m0 = fmaxf(m0, __shfl_xor_sync(0xffffffffu, m0, 2));
      m1 = fmaxf(m1, __shfl_xor_sync(0xffffffffu, m1, 1)); m1 = fmaxf(m1, __shfl_xor_sync(0xffffffffu, m1, 2));
      float d0 = 0.f, d1 = 0.f;
      const float f0 = m0 * scale_log2e, f1 = m1 * scale_log2e;
#pragma unroll
      for (int nt = 0; nt < NT; ++nt) {
        sc[nt][0] = attn_ex2(fmaf(sc[nt][0], scale_log2e, -f0)); sc[nt][1] = attn_ex2(fmaf(sc[nt][1], scale_log2e, -f0));
        sc[nt][2] = attn_ex2(fmaf(sc[nt][2], scale_log2e, -f1)); sc[nt][3] = attn_ex2(fmaf(sc[nt][3], scale_log2e, -f1));
        d0 += sc[nt][0] + sc[nt][1];
        d1 += sc[nt][2] + sc[nt][3];
      }
      d0 += __shfl_xor_sync(0xffffffffu, d0, 1); d0 += __shfl_xor_sync(0xffffffffu, d0, 2);
      d1 += __shfl_xor_sync(0xffffffffu, d1, 1); d1 += __shfl_xor_sync(0xffffffffu, d1, 2);
      float o[HD / 8][4];
#pragma unroll
      for (int dn = 0; dn < HD / 8; ++dn) o[dn][0] = o[dn][1] = o[dn][2] = o[dn][3] = 0.f;
      const uint8_t* vx0[4];
      const uint8_t* vx1[4];
#pragma unroll
      for (int dn = 0; dn < 4; ++dn) { vx0[dn] = Vs + (lane_v0 ^ (uint32_t)(dn << 5)); vx1[dn] = Vs + (lane_v1 ^ (uint32_t)(dn << 5)); }
#pragma unroll
      for (int nt = 0; nt < NT; ++nt) {
        // A k-slot c <-> key 2c, slot c+4 <-> key 2c+1 of this tile: (a0, a1, a2, a3) = (P[r0][2c], P[r1][2c], P[r0][2c+1], P[r1][2c+1])
        uint32_t ap[4] = {to_tf32(sc[nt][0]), to_tf32(sc[nt][2]), to_tf32(sc[nt][1]), to_tf32(sc[nt][3])};
#pragma unroll
        for (int dn = 0; dn < HD / 8; ++dn)
          mma_tf32_1688(o[dn], ap, __float_as_uint(attn_lds(vx0[dn] + nt * 1024)), __float_as_uint(attn_lds(vx1[dn] + nt * 1024)));
      }
      const float i0 = 1.f / d0, i1 = 1.f / d1;
      // stage the 16 x 32 tile (swizzled like the store's tensor map) and hand it to the TMA unit
      if (lane == 0) ptx::bulk_wait_group_read<0>();            // the previous store of this warp has read its staging tile
      __syncwarp();
#pragma unroll
      for (int dn = 0; dn < HD / 8; ++dn) {
        const uint32_t off = out_lo + (uint32_t)((((2 * dn + (c >> 1)) ^ gr) & 7) << 4);
        *reinterpret_cast<float2*>(my_out + off) = make_float2(f32_for_store(o[dn][0] * i0, od), f32_for_store(o[dn][1] * i0, od));
        *reinterpret_cast<float2*>(my_out + off + 1024) = make_float2(f32_for_store(o[dn][2] * i1, od), f32_for_store(o[dn][3] * i1, od));
      }
      ptx::fence_proxy_async();
      __syncwarp();
      if (lane == 0) {
        ptx::tma_store_3d(&tm_out, my_out, h * HD, qt * 16, b);
        ptx::bulk_commit_group();
      }
    }
    __syncwarp();
    if (lane == 0) ptx::mbar_arrive(&empty_bar[s]);
  }
  if (lane == 0) ptx::bulk_wait_group<0>();
}

inline int attention_tma_smem_bytes(int L) {
  const int LP = (L + 15) & ~15;
  return kAttnTmaStages * 3 * LP * 128 + kAttnTmaConsumers * 2048 + 1024;
}

inline bool attention_tma_prepare(const cds_attn_op& a, AttnTmaLaunch* out) {
  AttnTmaLaunch& l = *out;
  l.ok = false;
  {
    uint64_t dims[3] = {(uint64_t)3 * a.C, (uint64_t)a.L, (uint64_t)a.batch};
    uint64_t str[2] = {(uint64_t)3 * a.C, (uint64_t)a.L * 3 * a.C};
    uint32_t box[3] = {32, (uint32_t)a.L, 1};
    if (!encode_act_map(&l.tm_qkv, a.qkv, 3, dims, str, box, 64, true)) return false;
  }
  {
    uint64_t dims[3] = {(uint64_t)a.C, (uint64_t)a.L, (uint64_t)a.batch};
    uint64_t str[2] = {(uint64_t)a.C, (uint64_t)a.L * a.C};
    uint32_t box[3] = {32, 16, 1};
    if (!encode_act_map(&l.tm_out, a.out, 3, dims, str, box, 64, true)) return false;
  }
  l.n_work = a.batch * a.heads;
  l.smem_bytes = attention_tma_smem_bytes(a.L);
  l.ok = true;
  return true;
}

typedef void (*AttnTmaKernel)(const cds_attn_op, const CUtensorMap, const CUtensorMap, int);
inline AttnTmaKernel attention_tma_kernel(int nt) {
  switch (nt) {
#define CDS_ATTN_NT(N) case N: return attention_tma_tf32_hd32_kernel<N>;
    CDS_ATTN_NT(1) CDS_ATTN_NT(2) CDS_ATTN_NT(3) CDS_ATTN_NT(4) CDS_ATTN_NT(5) CDS_ATTN_NT(6) CDS_ATTN_NT(7) CDS_ATTN_NT(8)
    CDS_ATTN_NT(9) CDS_ATTN_NT(10) CDS_ATTN_NT(11) CDS_ATTN_NT(12) CDS_ATTN_NT(13) CDS_ATTN_NT(14) CDS_ATTN_NT(15) CDS_ATTN_NT(16)
#undef CDS_ATTN_NT
    default: return nullptr;
  }
}

// (per device, before the first launch / graph capture: the kernels need more than 48 KB of dynamic shared memory)
inline cudaError_t attention_tma_preload_all() {
  for (int nt = 1; nt <= kAttnMaxL / 8; ++nt) {
    cudaError_t e = cudaFuncSetAttribute(reinterpret_cast<const void*>(attention_tma_kernel(nt)), cudaFuncAttributeMaxDynamicSharedMemorySize, 112 * 1024);
    if (e != cudaSuccess) return e;
  }
  return cudaSuccess;
}

inline cudaError_t attention_tma_launch(const cds_attn_op& a, const AttnTmaLaunch& l, int nt, int sm_count, cudaStream_t st) {
  static bool set = false;
  if (!set) {
    cudaError_t e = attention_tma_preload_all();
    if (e != cudaSuccess) return e;
    set = true;
  }
  AttnTmaKernel k = attention_tma_kernel(nt);
  if (!k) return cudaErrorInvalidValue;
  int grid = 2 * (sm_count > 0 ? sm_count : 148);
  if (grid > l.n_work) grid = l.n_work;
  k<<<grid, kAttnTmaThreads, l.smem_bytes, st>>>(a, l.tm_qkv, l.tm_out, l.n_work);
  return cudaGetLastError();
}

}  // namespace cds
