// CDS_OP_ATTN, fp32 CUDA-core path: softmax(Q K^T / sqrt(hd)) V for one (trajectory, head) per CTA.
// K and V of the head (L x hd each, L <= 128) are staged once in shared memory; each thread owns one query
// row and runs an online softmax over the keys, so the L x L score matrix never exists in memory.
// Algorithmic HBM bytes per (trajectory, head): 4*L*hd*4 (q, k, v read; out written).
#pragma once
#include <cuda_bf16.h>

#include "common.cuh"

namespace cds {

template <int HD>
__global__ void __launch_bounds__(128) attention_f32_kernel(const cds_attn_op p) {
  extern __shared__ __align__(16) float smem[];
  float* Ks = smem;                 // [L][HD]
  float* Vs = smem + p.L * HD;      // [L][HD]
  const int b = blockIdx.x / p.heads, h = blockIdx.x - b * p.heads;
  const int ld = 3 * p.C;
  const float* base = reinterpret_cast<const float*>(p.qkv) + (int64_t)b * p.L * ld + h * HD;
  for (int idx = threadIdx.x; idx < p.L * HD; idx += blockDim.x) {
    int j = idx / HD, d = idx - j * HD;
    Ks[idx] = base[(int64_t)j * ld + p.C + d];
    Vs[idx] = base[(int64_t)j * ld + 2 * p.C + d];
  }
  __syncthreads();
  const float scale = rsqrtf((float)HD);
  for (int i = threadIdx.x; i < p.L; i += blockDim.x) {
    float q[HD], o[HD];
#pragma unroll
    for (int d = 0; d < HD; ++d) { q[d] = base[(int64_t)i * ld + d] * scale; o[d] = 0.f; }
    float mx = -INFINITY, den = 0.f;
    for (int j = 0; j < p.L; ++j) {
      float s = 0.f;
#pragma unroll
      for (int d = 0; d < HD; ++d) s = fmaf(q[d], Ks[j * HD + d], s);
      float nm = fmaxf(mx, s);
      float corr = expf(mx - nm), w = expf(s - nm);
      den = den * corr + w;
#pragma unroll
      for (int d = 0; d < HD; ++d) o[d] = fmaf(o[d], corr, w * Vs[j * HD + d]);
      mx = nm;
    }
    float inv = 1.f / den;
    const int64_t o_off = ((int64_t)b * p.L + i) * p.C + h * HD;
    if (p.out_dtype == CDS_BF16) {
      __nv_bfloat16* dst = reinterpret_cast<__nv_bfloat16*>(p.out) + o_off;
#pragma unroll
      for (int d = 0; d < HD; ++d) dst[d] = __float2bfloat16_rn(o[d] * inv);
    } else {
      float* dst = reinterpret_cast<float*>(p.out) + o_off;
#pragma unroll
      for (int d = 0; d < HD; ++d) dst[d] = f32_for_store(o[d] * inv, p.out_dtype);
    }
  }
}

// ---------------------------------------------------------------------------------------------------------------------
// Tensor-core path (bf16 q/k/v, head_dim 32, L <= 128): one CTA per (trajectory, head), 4 warps, each warp owns 16-query tiles.
// S = Q K^T and O = P V run on mma.sync.m16n8k16 (bf16 operands, fp32 accumulate); the softmax stays in registers: the
// accumulator layout of S (row = lane/4 (+8), column pair = (lane%4)*2) IS the A-operand layout of the P V product, two
// adjacent 8-key tiles forming one 16-key K step (the FlashAttention-2 register trick).  K lives in shared memory row-major
// (rows padded to 80 B: conflict-free fragment loads), V transposed (dim-major) so that a B fragment is one 32-bit load.
// Algorithmic HBM bytes per (trajectory, head): 2*L*32*3 (q, k, v) + L*32*2 (out).
__device__ __forceinline__ void mma_bf16_16816(float (&d)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
  asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
               : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
               : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}
__device__ __forceinline__ uint32_t pack_bf16x2(float lo, float hi) {
  __nv_bfloat162 v = __floats2bfloat162_rn(lo, hi);
  return *reinterpret_cast<uint32_t*>(&v);
}

constexpr int kAttnMaxL = 128;
constexpr int kAttnKPitch = 40;                      // bf16 per K row in shared memory (32 + 8 pad)
constexpr int kAttnVPitch = kAttnMaxL + 8;           // bf16 per V^T row (keys, padded)

__global__ void __launch_bounds__(128) attention_mma_hd32_kernel(const cds_attn_op p) {
  constexpr int HD = 32;
  __shared__ __align__(16) __nv_bfloat16 Ks[kAttnMaxL * kAttnKPitch];
  __shared__ __align__(16) __nv_bfloat16 Vt[HD * kAttnVPitch];
  const int b = blockIdx.x / p.heads, h = blockIdx.x - b * p.heads;
  const int L = p.L, ld = 3 * p.C;
  const int LP = (L + 15) & ~15;                     // keys padded to whole 16-key MMA steps (zeros, masked below)
  const __nv_bfloat16* base = reinterpret_cast<const __nv_bfloat16*>(p.qkv) + (int64_t)b * L * ld + h * HD;
  // ---- stage K (row-major) and V (transposed); rows >= L are zero
  for (int idx = threadIdx.x; idx < LP * 4; idx += blockDim.x) {
    const int j = idx >> 2, c8 = (idx & 3) * 8;      // key row, first of 8 channels
    uint4 kq = make_uint4(0, 0, 0, 0), vq = kq;
    if (j < L) {
      kq = *reinterpret_cast<const uint4*>(base + (int64_t)j * ld + p.C + c8);
      vq = *reinterpret_cast<const uint4*>(base + (int64_t)j * ld + 2 * p.C + c8);
    }
    *reinterpret_cast<uint4*>(&Ks[j * kAttnKPitch + c8]) = kq;
    const __nv_bfloat16* vv = reinterpret_cast<const __nv_bfloat16*>(&vq);
#pragma unroll
    for (int e = 0; e < 8; ++e) Vt[(c8 + e) * kAttnVPitch + j] = vv[e];
  }
  __syncthreads();

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int gr = lane >> 2, gc = (lane & 3) * 2;      // fragment row (0..7) and column pair (0, 2, 4, 6)
  const float scale_log2e = rsqrtf((float)HD) * 1.4426950408889634f;
  constexpr int NT_MAX = kAttnMaxL / 8;               // 8-key score tiles
  const int NT = LP / 8;
  for (int qt = warp; qt * 16 < L; qt += 4) {
    const int r0 = qt * 16 + gr, r1 = r0 + 8;         // this thread's two query rows
    // ---- Q fragments (2 K steps over head_dim 32), straight from global memory
    uint32_t aq[2][4];
#pragma unroll
    for (int ks = 0; ks < 2; ++ks) {
      const int c = ks * 16 + gc;
      aq[ks][0] = r0 < L ? *reinterpret_cast<const uint32_t*>(base + (int64_t)r0 * ld + c) : 0u;
      aq[ks][1] = r1 < L ? *reinterpret_cast<const uint32_t*>(base + (int64_t)r1 * ld + c) : 0u;
      aq[ks][2] = r0 < L ? *reinterpret_cast<const uint32_t*>(base + (int64_t)r0 * ld + c + 8) : 0u;
      aq[ks][3] = r1 < L ? *reinterpret_cast<const uint32_t*>(base + (int64_t)r1 * ld + c + 8) : 0u;
    }
    // ---- S = Q K^T
    float s[NT_MAX][4];
#pragma unroll
    for (int nt = 0; nt < NT_MAX; ++nt) {
      s[nt][0] = s[nt][1] = s[nt][2] = s[nt][3] = 0.f;
      if (nt < NT) {
#pragma unroll
        for (int ks = 0; ks < 2; ++ks) {
          const __nv_bfloat16* kp = &Ks[(nt * 8 + gr) * kAttnKPitch + ks * 16 + gc];
          mma_bf16_16816(s[nt], aq[ks], *reinterpret_cast<const uint32_t*>(kp), *reinterpret_cast<const uint32_t*>(kp + 8));
        }
      }
    }
    // ---- softmax over the keys (rows r0: s[.][0..1], r1: s[.][2..3]); exp2 with the scale folded in
    float m0 = -INFINITY, m1 = -INFINITY;
#pragma unroll
    for (int nt = 0; nt < NT_MAX; ++nt) {
      if (nt < NT) {
        const int j = nt * 8 + gc;
        if (j >= L) s[nt][0] = s[nt][2] = -INFINITY;
        if (j + 1 >= L) s[nt][1] = s[nt][3] = -INFINITY;
        m0 = fmaxf(m0, fmaxf(s[nt][0], s[nt][1]));
        m1 = fmaxf(m1, fmaxf(s[nt][2], s[nt][3]));
      }
    }
    m0 = fmaxf(m0, __shfl_xor_sync(0xffffffffu, m0, 1)); m0 = fmaxf(m0, __shfl_xor_sync(0xffffffffu, m0, 2));
    m1 = fmaxf(m1, __shfl_xor_sync(0xffffffffu, m1, 1)); m1 = fmaxf(m1, __shfl_xor_sync(0xffffffffu, m1, 2));
    float d0 = 0.f, d1 = 0.f;
    const float o0 = m0 * scale_log2e, o1 = m1 * scale_log2e;
#pragma unroll
    for (int nt = 0; nt < NT_MAX; ++nt) {
      if (nt < NT) {
        s[nt][0] = exp2f(fmaf(s[nt][0], scale_log2e, -o0)); s[nt][1] = exp2f(fmaf(s[nt][1], scale_log2e, -o0));
        s[nt][2] = exp2f(fmaf(s[nt][2], scale_log2e, -o1)); s[nt][3] = exp2f(fmaf(s[nt][3], scale_log2e, -o1));
        d0 += s[nt][0] + s[nt][1];
        d1 += s[nt][2] + s[nt][3];
      }
    }
    d0 += __shfl_xor_sync(0xffffffffu, d0, 1); d0 += __shfl_xor_sync(0xffffffffu, d0, 2);
    d1 += __shfl_xor_sync(0xffffffffu, d1, 1); d1 += __shfl_xor_sync(0xffffffffu, d1, 2);
    // ---- O = P V
    float o[HD / 8][4];
#pragma unroll
    for (int dn = 0; dn < HD / 8; ++dn) o[dn][0] = o[dn][1] = o[dn][2] = o[dn][3] = 0.f;
#pragma unroll
    for (int kk = 0; kk < NT_MAX / 2; ++kk) {
      if (kk * 16 < LP) {
        uint32_t ap[4];
        ap[0] = pack_bf16x2(s[2 * kk][0], s[2 * kk][1]);
        ap[1] = pack_bf16x2(s[2 * kk][2], s[2 * kk][3]);
        ap[2] = pack_bf16x2(s[2 * kk + 1][0], s[2 * kk + 1][1]);
        ap[3] = pack_bf16x2(s[2 * kk + 1][2], s[2 * kk + 1][3]);
#pragma unroll
        for (int dn = 0; dn < HD / 8; ++dn) {
          const __nv_bfloat16* vp = &Vt[(dn * 8 + gr) * kAttnVPitch + kk * 16 + gc];
          mma_bf16_16816(o[dn], ap, *reinterpret_cast<const uint32_t*>(vp), *reinterpret_cast<const uint32_t*>(vp + 8));
        }
      }
    }
    // ---- normalise and store (row r0: o[.][0..1], row r1: o[.][2..3]; columns dn*8 + gc, +1)
    const float i0 = 1.f / d0, i1 = 1.f / d1;
#pragma unroll
    for (int dn = 0; dn < HD / 8; ++dn) {
      const int col = h * HD + dn * 8 + gc;
      if (p.out_dtype == CDS_BF16) {
        __nv_bfloat16* out = reinterpret_cast<__nv_bfloat16*>(p.out);
        if (r0 < L) *reinterpret_cast<uint32_t*>(out + ((int64_t)b * L + r0) * p.C + col) = pack_bf16x2(o[dn][0] * i0, o[dn][1] * i0);
        if (r1 < L) *reinterpret_cast<uint32_t*>(out + ((int64_t)b * L + r1) * p.C + col) = pack_bf16x2(o[dn][2] * i1, o[dn][3] * i1);
      } else {
        float* out = reinterpret_cast<float*>(p.out);
        const int od = p.out_dtype;
        if (r0 < L) { float* d = out + ((int64_t)b * L + r0) * p.C + col; d[0] = f32_for_store(o[dn][0] * i0, od); d[1] = f32_for_store(o[dn][1] * i0, od); }
        if (r1 < L) { float* d = out + ((int64_t)b * L + r1) * p.C + col; d[0] = f32_for_store(o[dn][2] * i1, od); d[1] = f32_for_store(o[dn][3] * i1, od); }
      }
    }
  }
}

// family (CDS_ATTN_F32 / _BF16_MMA) and, for the fp32 kernel, HD: as attn_pick (cds_api.cu) chose them
inline cudaError_t attention_launch(const cds_attn_op& p, int family, int hd, cudaStream_t st) {
  if (family == CDS_ATTN_BF16_MMA) {
    attention_mma_hd32_kernel<<<dim3(p.batch * p.heads), 128, 0, st>>>(p);
    return cudaGetLastError();
  }
  if (family != CDS_ATTN_F32) return cudaErrorInvalidValue;
  size_t smem = sizeof(float) * 2 * (size_t)p.L * hd;
  dim3 grid(p.batch * p.heads);
#define CDS_ATTN_CASE(HD)                                                                                   \
  case HD: {                                                                                                 \
    static bool set = false;                                                                                 \
    if (!set) { cudaFuncSetAttribute(attention_f32_kernel<HD>, cudaFuncAttributeMaxDynamicSharedMemorySize, \
                                     200 * 1024); set = true; }                                              \
    attention_f32_kernel<HD><<<grid, 128, smem, st>>>(p);                                                  \
    break; }
  switch (hd) {
    CDS_ATTN_CASE(16)
    CDS_ATTN_CASE(32)
    CDS_ATTN_CASE(64)
    default: return cudaErrorInvalidValue;
  }
#undef CDS_ATTN_CASE
  return cudaGetLastError();
}

}  // namespace cds
