// CDS_OP_MHA: masked multi-head attention with separate q and k|v sources, fp32 on CUDA cores.
// One warp per query row (b, h, i); lane l owns head channels l, l + 32, ... (HPL = head_dim / 32 of them), so every load of a
// q / k / v row is one coalesced 32-element access.  Each visible key costs one warp reduction for its score, then an online
// softmax update of the lane's HPL output channels: the Lq x Lk score matrix never exists.  K and V come from L1 / L2: the
// Lq query rows of one (trajectory, head) are consecutive warps, and at the sequence lengths served here (Lk <= 64, 10 or 11
// in ChiTransformer) attention is a small fraction of a layer's work -- tensor cores would not pay for their staging.
#pragma once
#include <cuda_bf16.h>

#include "common.cuh"

namespace cds {

constexpr int kMhaMaxL = 64;
constexpr int kMhaMaxHPL = 8;        // head_dim <= 256
constexpr int kMhaWarps = 4;         // query rows per CTA

template <bool BF16>
__device__ __forceinline__ float mha_load(const void* base, int64_t idx) {
  if (BF16) return __bfloat162float(reinterpret_cast<const __nv_bfloat16*>(base)[idx]);
  return reinterpret_cast<const float*>(base)[idx];
}

template <int HPL, bool BF16>
__global__ void __launch_bounds__(32 * kMhaWarps) mha_f32_kernel(const cds_mha_op p, const int* __restrict__ iter_ptr) {
  constexpr int HD = 32 * HPL;
  const int lane = threadIdx.x & 31;
  const int64_t row = (int64_t)blockIdx.x * kMhaWarps + (threadIdx.x >> 5);      // (b, h, i), i fastest
  if (row >= (int64_t)p.batch * p.heads * p.Lq) return;
  const int i = (int)(row % p.Lq);
  const int h = (int)((row / p.Lq) % p.heads);
  const int b = (int)(row / ((int64_t)p.Lq * p.heads));
  const int c0 = h * HD + lane;                                                  // this lane's first channel in [0, C)

  const float scale = rsqrtf((float)HD);
  float q[HPL], o[HPL];
  const int64_t q_off = (int64_t)b * p.q_bstride + (int64_t)i * p.q_lstride + c0;
#pragma unroll
  for (int e = 0; e < HPL; ++e) { q[e] = mha_load<BF16>(p.q, q_off + 32 * e); o[e] = 0.f; }

  const int64_t step_off = p.kv_step ? (int64_t)(*iter_ptr) * p.kv_step_stride + c0 : 0;
  const int64_t samp_off = (int64_t)b * p.kv_sample_bstride + c0;
  const int n_vis = p.masked ? max(0, min(p.Lk, i + p.diag + 1)) : p.Lk;
  float mx = -INFINITY, den = 0.f;
  for (int j = 0; j < n_vis; ++j) {
    float k[HPL], v[HPL];
#pragma unroll
    for (int e = 0; e < HPL; ++e) { k[e] = 0.f; v[e] = 0.f; }
    if (p.kv_step) {
      const int64_t off = step_off + (int64_t)j * p.kv_step_lstride;
#pragma unroll
      for (int e = 0; e < HPL; ++e) {
        k[e] += mha_load<BF16>(p.kv_step, off + 32 * e);
        v[e] += mha_load<BF16>(p.kv_step, off + p.C + 32 * e);
      }
    }
    if (p.kv_sample) {
      const int64_t off = samp_off + (int64_t)j * p.kv_sample_lstride;
#pragma unroll
      for (int e = 0; e < HPL; ++e) {
        k[e] += mha_load<BF16>(p.kv_sample, off + 32 * e);
        v[e] += mha_load<BF16>(p.kv_sample, off + p.C + 32 * e);
      }
    }
    float s = 0.f;
#pragma unroll
    for (int e = 0; e < HPL; ++e) s = fmaf(q[e], k[e], s);
    s = warp_sum(s) * scale;
    const float nm = fmaxf(mx, s);
    const float corr = expf(mx - nm), w = expf(s - nm);
    den = den * corr + w;
#pragma unroll
    for (int e = 0; e < HPL; ++e) o[e] = fmaf(o[e], corr, w * v[e]);
    mx = nm;
  }
  // no visible key (den = 0): the row is defined as zeros
  const float inv = den > 0.f ? 1.f / den : 0.f;
  const int64_t o_off = (int64_t)b * p.out_bstride + (int64_t)i * p.out_lstride + c0;
  if (p.out_dtype == CDS_BF16) {
    __nv_bfloat16* dst = reinterpret_cast<__nv_bfloat16*>(p.out) + o_off;
#pragma unroll
    for (int e = 0; e < HPL; ++e) dst[32 * e] = __float2bfloat16_rn(o[e] * inv);
  } else {
    float* dst = reinterpret_cast<float*>(p.out) + o_off;
#pragma unroll
    for (int e = 0; e < HPL; ++e) dst[32 * e] = f32_for_store(o[e] * inv, p.out_dtype);
  }
}

template <int HPL>
inline cudaError_t mha_launch_hpl(const cds_mha_op& p, const int* iter_ptr, cudaStream_t st) {
  const int64_t rows = (int64_t)p.batch * p.heads * p.Lq;
  const unsigned grid = (unsigned)((rows + kMhaWarps - 1) / kMhaWarps);
  if (p.in_dtype == CDS_BF16) mha_f32_kernel<HPL, true><<<grid, 32 * kMhaWarps, 0, st>>>(p, iter_ptr);
  else mha_f32_kernel<HPL, false><<<grid, 32 * kMhaWarps, 0, st>>>(p, iter_ptr);
  return cudaGetLastError();
}

// `hpl` = head_dim / 32 as chosen by mha_pick (cds_api.cu)
inline cudaError_t mha_launch(const cds_mha_op& p, int hpl, const int* iter_ptr, cudaStream_t st) {
  switch (hpl) {
    case 1: return mha_launch_hpl<1>(p, iter_ptr, st);
    case 2: return mha_launch_hpl<2>(p, iter_ptr, st);
    case 3: return mha_launch_hpl<3>(p, iter_ptr, st);
    case 4: return mha_launch_hpl<4>(p, iter_ptr, st);
    case 5: return mha_launch_hpl<5>(p, iter_ptr, st);
    case 6: return mha_launch_hpl<6>(p, iter_ptr, st);
    case 7: return mha_launch_hpl<7>(p, iter_ptr, st);
    case 8: return mha_launch_hpl<8>(p, iter_ptr, st);
  }
  return cudaErrorInvalidValue;
}

template <int HPL>
inline cudaError_t mha_preload_hpl() {
  cudaFuncAttributes a;
  cudaError_t e = cudaFuncGetAttributes(&a, mha_f32_kernel<HPL, false>);
  return e != cudaSuccess ? e : cudaFuncGetAttributes(&a, mha_f32_kernel<HPL, true>);
}

inline cudaError_t mha_preload_all() {
  cudaError_t e;
  if ((e = mha_preload_hpl<1>()) != cudaSuccess) return e;
  if ((e = mha_preload_hpl<2>()) != cudaSuccess) return e;
  if ((e = mha_preload_hpl<3>()) != cudaSuccess) return e;
  if ((e = mha_preload_hpl<4>()) != cudaSuccess) return e;
  if ((e = mha_preload_hpl<5>()) != cudaSuccess) return e;
  if ((e = mha_preload_hpl<6>()) != cudaSuccess) return e;
  if ((e = mha_preload_hpl<7>()) != cudaSuccess) return e;
  return mha_preload_hpl<8>();
}

}  // namespace cds
