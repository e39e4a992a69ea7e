// The input gradient of a transformer classifier (HalfDiT1d under classifier guidance): the backward modes of
//   CDS_OP_ATTN   (dout != NULL)  per (trajectory, head), the softmax recomputed from q and k
//   CDS_OP_LNMOD  (dout != NULL)  + a residual gradient, + a gated copy for the next data-gradient GEMM
//   CDS_OP_STASH  (grad != NULL)  act_out = grad * act'(src), elementwise (the GELU-tanh of DiT's MLP, whose GEMMs run on the
//                                 token-stream kernels)
// Every output element is one thread's (or one warp's fixed-butterfly) sum in a fixed order: no atomics, bitwise reproducible.
#pragma once
#include "common.cuh"
#include "elementwise.cuh"
#include "grad.cuh"

namespace cds {

constexpr int kAttnBwdMaxL = 128;
constexpr int kAttnBwdThreads = 256;

// shared memory of one CTA: q (pre-scaled), k, v, dO as [L][HD + 1] (the odd row stride keeps a warp reading 32 different rows
// conflict-free) and P / dS as [L][L + 1]
inline size_t attn_bwd_smem_bytes(int L, int hd) {
  return sizeof(float) * ((size_t)4 * L * (hd + 1) + (size_t)L * (L + 1));
}

template <int HD>
static __global__ void __launch_bounds__(kAttnBwdThreads) attn_bwd_kernel(const cds_attn_op p) {
  extern __shared__ float sm[];
  constexpr int HP = HD + 1;
  constexpr int JT = kAttnBwdMaxL / 32;                      // keys per lane in the row phases
  const int L = p.L, C = p.C, LP = L + 1;
  const int h = blockIdx.x % p.heads;
  const int64_t b = blockIdx.x / p.heads;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, nwarps = kAttnBwdThreads / 32;
  float* qs = sm;
  float* ks = qs + L * HP;
  float* vs = ks + L * HP;
  float* dos = vs + L * HP;
  float* P = dos + L * HP;
  const float scale = rsqrtf((float)HD);
  const float* src = reinterpret_cast<const float*>(p.qkv) + b * (int64_t)L * 3 * C + h * HD;
  const float* gsrc = p.dout + b * (int64_t)L * C + h * HD;
  for (int i = tid; i < L * HD; i += kAttnBwdThreads) {
    const int l = i / HD, c = i - l * HD;
    const float* row = src + (int64_t)l * 3 * C + c;
    qs[l * HP + c] = row[0] * scale;
    ks[l * HP + c] = row[C];
    vs[l * HP + c] = row[2 * C];
    dos[l * HP + c] = gsrc[(int64_t)l * C + c];
  }
  __syncthreads();

  // P = softmax(qs k^T), one warp per query row
  for (int i = warp; i < L; i += nwarps) {
    float s[JT];
    float mx = -INFINITY;
#pragma unroll
    for (int t = 0; t < JT; ++t) {
      const int j = lane + 32 * t;
      s[t] = -INFINITY;
      if (j < L) {
        float a = 0.f;
#pragma unroll
        for (int c = 0; c < HD; ++c) a = fmaf(qs[i * HP + c], ks[j * HP + c], a);
        s[t] = a;
        mx = fmaxf(mx, a);
      }
    }
    mx = warp_max(mx);
    float sum = 0.f;
#pragma unroll
    for (int t = 0; t < JT; ++t) {
      s[t] = (lane + 32 * t < L) ? expf(s[t] - mx) : 0.f;
      sum += s[t];
    }
    const float inv = 1.f / warp_sum(sum);
#pragma unroll
    for (int t = 0; t < JT; ++t)
      if (lane + 32 * t < L) P[i * LP + lane + 32 * t] = s[t] * inv;
  }
  __syncthreads();

  float* dst = reinterpret_cast<float*>(p.out) + b * (int64_t)L * 3 * C + h * HD;
  // dV = P^T dO
  for (int e = tid; e < L * HD; e += kAttnBwdThreads) {
    const int j = e / HD, c = e - j * HD;
    float a = 0.f;
    for (int i = 0; i < L; ++i) a = fmaf(P[i * LP + j], dos[i * HP + c], a);
    dst[(int64_t)j * 3 * C + 2 * C + c] = f32_for_store(a, p.out_dtype);
  }
  __syncthreads();

  // dS = P * (dP - rowsum(P * dP)), dP = dO v^T, in place of P (one warp per query row)
  for (int i = warp; i < L; i += nwarps) {
    float dp[JT];
    float d = 0.f;
#pragma unroll
    for (int t = 0; t < JT; ++t) {
      const int j = lane + 32 * t;
      dp[t] = 0.f;
      if (j < L) {
        float a = 0.f;
#pragma unroll
        for (int c = 0; c < HD; ++c) a = fmaf(dos[i * HP + c], vs[j * HP + c], a);
        dp[t] = a;
        d = fmaf(P[i * LP + j], a, d);
      }
    }
    d = warp_sum(d);
#pragma unroll
    for (int t = 0; t < JT; ++t) {
      const int j = lane + 32 * t;
      if (j < L) P[i * LP + j] = P[i * LP + j] * (dp[t] - d);
    }
  }
  __syncthreads();

  // dQ = dS k / sqrt(hd),  dK = dS^T qs  (qs already carries the 1 / sqrt(hd))
  for (int e = tid; e < L * HD; e += kAttnBwdThreads) {
    const int l = e / HD, c = e - l * HD;
    float aq = 0.f, ak = 0.f;
    for (int j = 0; j < L; ++j) {
      aq = fmaf(P[l * LP + j], ks[j * HP + c], aq);
      ak = fmaf(P[j * LP + l], qs[j * HP + c], ak);
    }
    dst[(int64_t)l * 3 * C + c] = f32_for_store(aq * scale, p.out_dtype);
    dst[(int64_t)l * 3 * C + C + c] = f32_for_store(ak, p.out_dtype);
  }
}

inline cudaError_t attn_bwd_launch(const cds_attn_op& p, cudaStream_t st) {
  const int hd = p.C / p.heads;
  const size_t smem = attn_bwd_smem_bytes(p.L, hd);
  const dim3 grid((unsigned)((int64_t)p.batch * p.heads));
  if (hd == 16) attn_bwd_kernel<16><<<grid, kAttnBwdThreads, smem, st>>>(p);
  else if (hd == 32) attn_bwd_kernel<32><<<grid, kAttnBwdThreads, smem, st>>>(p);
  else attn_bwd_kernel<64><<<grid, kAttnBwdThreads, smem, st>>>(p);
  return cudaGetLastError();
}

// every instantiation may use the shared memory of the longest sequence it serves
inline cudaError_t attn_bwd_preload_all() {
  cudaError_t e;
  if ((e = cudaFuncSetAttribute(attn_bwd_kernel<16>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                (int)attn_bwd_smem_bytes(kAttnBwdMaxL, 16))) != cudaSuccess) return e;
  if ((e = cudaFuncSetAttribute(attn_bwd_kernel<32>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                (int)attn_bwd_smem_bytes(kAttnBwdMaxL, 32))) != cudaSuccess) return e;
  return cudaFuncSetAttribute(attn_bwd_kernel<64>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                              (int)attn_bwd_smem_bytes(kAttnBwdMaxL, 64));
}

// one warp per token row; the statistics as ln_modulate_kernel computes them on its scalar path (lane-strided sums, xor
// butterfly, two passes)
static __global__ void __launch_bounds__(256) lnmod_bwd_kernel(const cds_lnmod_op p) {
  const int warps_per_block = blockDim.x >> 5;
  const int lane = threadIdx.x & 31;
  const int64_t n_rows = (int64_t)p.batch * p.L;
  const float inv_c = 1.f / (float)p.C;
  for (int64_t r = (int64_t)blockIdx.x * warps_per_block + (threadIdx.x >> 5); r < n_rows;
       r += (int64_t)gridDim.x * warps_per_block) {
    const int b = (int)(r / p.L), l = (int)(r - (int64_t)b * p.L);
    const float* x = p.in + r * p.C;
    const float* sc = p.scale + (int64_t)b * p.mod_bstride;
    const float* go = p.dout + (int64_t)b * p.dout_bstride + (int64_t)l * p.dout_lstride;
    float s = 0.f;
    for (int c = lane; c < p.C; c += 32) s += x[c];
    const float mean = warp_sum(s) * inv_c;
    float q = 0.f;
    for (int c = lane; c < p.C; c += 32) { const float d = x[c] - mean; q = fmaf(d, d, q); }
    const float rstd = rsqrtf(warp_sum(q) * inv_c + p.eps);
    float a = 0.f, ax = 0.f;
    for (int c = lane; c < p.C; c += 32) {
      const float dy = go[c] * (1.f + sc[c]);
      a += dy;
      ax = fmaf(dy, (x[c] - mean) * rstd, ax);
    }
    const float ma = warp_sum(a) * inv_c, max_ = warp_sum(ax) * inv_c;
    const float* gate = p.gated ? p.gate + (int64_t)b * p.gate_bstride : nullptr;
    for (int c = lane; c < p.C; c += 32) {
      const float dy = go[c] * (1.f + sc[c]);
      const float xhat = (x[c] - mean) * rstd;
      float v = rstd * ((dy - ma) - xhat * max_);
      if (p.res) v += p.res[r * p.C + c];
      reinterpret_cast<float*>(p.out)[r * p.C + c] = f32_for_store(v, p.out_dtype);
      if (gate) p.gated[r * p.C + c] = f32_for_store(gate[c] * v, p.gated_dtype);
    }
  }
}

inline int lnmod_bwd_grid(const cds_lnmod_op& p, int sm_count) {
  const int64_t blocks = ((int64_t)p.batch * p.L + 7) / 8, cap = (int64_t)sm_count * 8;
  return (int)(blocks < cap ? blocks : cap);
}

static __global__ void __launch_bounds__(256) act_bwd_kernel(const cds_stash_op p) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < p.n; i += (int64_t)gridDim.x * blockDim.x)
    p.act_out[i] = p.grad[i] * act_grad(p.act, p.src[i]);
}

}  // namespace cds
