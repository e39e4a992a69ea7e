// Elementwise operators of the reverse loop: solver update (CDS_OP_UPDATE), consistency-model
// pre-scale (CDS_OP_PREP) and LayerNorm+modulate (CDS_OP_LNMOD).  All HBM-bound streaming kernels:
// algorithmic bytes per element are listed with each kernel.
#pragma once
#include <cuda_bf16.h>

#include "common.cuh"

namespace cds {

// IEEE fp32 ops that the compiler may not contract into FMAs: the update mirrors the reference's tensor
// expression operation by operation (diffusionsde.py:539-592), so results agree to fp32 rounding of
// identical operations rather than to "some tolerance".
__device__ __forceinline__ float mul_(float a, float b) { return __fmul_rn(a, b); }
__device__ __forceinline__ float add_(float a, float b) { return __fadd_rn(a, b); }
__device__ __forceinline__ float sub_(float a, float b) { return __fsub_rn(a, b); }
__device__ __forceinline__ float div_(float a, float b) { return __fdiv_rn(a, b); }

// per-iteration scalars of the update (one row of the coefficient table)
struct UpdRow {
  float alpha, sigma, k0, k1, k2, k3, k4, xw, dw;
  float gs;                    // this iteration's guidance scale (0 without a guidance operand)
  int kind;
  const float* noise;          // this iteration's noise slot or NULL
};
__device__ __forceinline__ UpdRow load_upd_row(const cds_update_op& p, int iter) {
  const float* row = p.coef + (int64_t)iter * CDS_ROW_FLOATS;
  UpdRow r;
  r.alpha = row[CDS_ROW_ALPHA]; r.sigma = row[CDS_ROW_SIGMA];
  r.k0 = row[CDS_ROW_K0]; r.k1 = row[CDS_ROW_K1]; r.k2 = row[CDS_ROW_K2]; r.k3 = row[CDS_ROW_K3]; r.k4 = row[CDS_ROW_K4];
  r.xw = row[CDS_ROW_XW]; r.dw = row[CDS_ROW_DW];
  r.kind = (int)row[CDS_ROW_KIND];
  r.gs = p.guide ? p.guide_s[iter] : 0.f;
  const int slot = (int)row[CDS_ROW_NOISE] - 1;
  const int64_t slot_stride = p.noise_slot_stride > 0 ? p.noise_slot_stride : (int64_t)p.batch * p.row;
  r.noise = slot >= 0 ? p.noise + (int64_t)slot * slot_stride : nullptr;
  return r;
}

// One element of the reverse-process update as a pure function of its operands: e = index inside the trajectory, x = x_t,
// pr = the network prediction (after the CFG combine), z = this iteration's noise draw (ignored without a slot), prior = the
// conditioning value under the mask, hist = previous x0 estimate of the 2M solvers; *xhat_out receives the new estimate;
// g = the classifier's input gradient (EDM kinds with a guidance operand).
__device__ __forceinline__ float solver_update_value(const cds_update_op& p, const UpdRow& r, int e, float x, float pr, float z,
                                                     float prior, float hist, float* xhat_out, float aux_in = 0.f,
                                                     float* aux_out = nullptr, float g = 0.f) {
  const float alpha = r.alpha, sigma = r.sigma;
  float out;
  if (r.kind == CDS_UPD_EDM || r.kind == CDS_UPD_EDM_HEUN) {
    // D = c_skip*x + c_out*net ; clip ; Euler / Heun step of the probability-flow ODE (newedm.py:142-148, :411-431)
    float d_theta = add_(mul_(r.k0, x), mul_(r.k1, pr));
    if (p.guide) d_theta = add_(d_theta, mul_(r.gs, g));       // classifier guidance (newedm.py:231), before the clip
    if (p.final_clip) {
      if (p.x_min) d_theta = fmaxf(d_theta, p.x_min[e]);
      if (p.x_max) d_theta = fminf(d_theta, p.x_max[e]);
    }
    const float slope = r.xw != 0.f ? sub_(mul_(r.xw, x), mul_(r.dw, d_theta)) : div_(sub_(x, d_theta), sigma);
    if (r.kind == CDS_UPD_EDM) {
      out = sub_(x, mul_(slope, r.k2));
      if (xhat_out) *xhat_out = x;
      if (aux_out) *aux_out = slope;
    } else {
      out = sub_(hist, mul_(div_(add_(aux_in, slope), 2.f), r.k2));
    }
  } else if (r.kind == CDS_UPD_CM) {
    // f = c_skip*x + c_out*net ; clip (consistency_model.py:257-261)
    out = add_(mul_(r.k0, x), mul_(r.k1, pr));
    if (p.final_clip) {
      if (p.x_min) out = fmaxf(out, p.x_min[e]);
      if (p.x_max) out = fminf(out, p.x_max[e]);
    }
  } else {
    // clip_prediction (diffusionsde.py:208-223)
    if (p.predict_noise) {
      if (p.x_max) pr = fmaxf(pr, div_(sub_(x, mul_(alpha, p.x_max[e])), sigma));
      if (p.x_min) pr = fminf(pr, div_(sub_(x, mul_(alpha, p.x_min[e])), sigma));
    } else {
      if (p.x_min) pr = fmaxf(pr, p.x_min[e]);
      if (p.x_max) pr = fminf(pr, p.x_max[e]);
    }
    float eps, xhat;
    if (p.predict_noise) { eps = pr; xhat = div_(sub_(x, mul_(sigma, pr)), alpha); }
    else { xhat = pr; eps = div_(sub_(x, mul_(alpha, pr)), sigma); }

    if (r.kind == CDS_UPD_DDPM) {
      out = add_(mul_(r.k0, sub_(x, mul_(sigma, eps))), mul_(r.k1, eps));
      if (r.noise) out = add_(out, mul_(r.k2, z));
    } else if (r.kind == CDS_UPD_DDIM) {
      out = add_(mul_(r.k0, div_(sub_(x, mul_(sigma, eps)), alpha)), mul_(r.k1, eps));
    } else {
      float target;
      if (r.kind == CDS_UPD_EPS) target = eps;
      else if (r.kind == CDS_UPD_X2M) target = sub_(mul_(r.k3, xhat), mul_(r.k4, hist));
      else target = xhat;
      out = sub_(mul_(r.k0, x), mul_(r.k1, target));
      if (r.noise) out = add_(out, mul_(r.k2, z));
      if (xhat_out) *xhat_out = xhat;
    }
  }
  if (p.mask) { const float m = p.mask[e]; out = add_(mul_(out, 1.f - m), mul_(prior, m)); }
  return out;
}

// ... applied to element i of x in place: i = flat index into x (batch*row), e = i % row, cast_off = element offset in x_cast
// (ignored when x_cast is NULL).  Reads x (+noise, prior, xhat_prev), writes x (+xhat_prev, +the bf16 channel-padded copy).
__device__ __forceinline__ void solver_update_element(const cds_update_op& p, const UpdRow& r, int64_t i, int e, int64_t cast_off,
                                                      float pr) {
  float xhat = 0.f, aux = 0.f;
  const bool heun2 = r.kind == CDS_UPD_EDM_HEUN;
  const float out = solver_update_value(p, r, e, p.x[i], pr, r.noise ? r.noise[i] : 0.f, p.mask ? p.prior[i] : 0.f,
                                        (p.xhat_prev && (r.kind == CDS_UPD_X2M || heun2)) ? p.xhat_prev[i] : 0.f, &xhat,
                                        (p.aux && heun2) ? p.aux[i] : 0.f, &aux, p.guide ? p.guide[i] : 0.f);
  if (r.kind == CDS_UPD_EDM) {
    if (r.k4 != 0.f && p.xhat_prev && p.aux) { p.xhat_prev[i] = xhat; p.aux[i] = aux; }      // predictor of a Heun step
  } else if (p.xhat_prev && !heun2 && r.kind != CDS_UPD_CM && r.kind != CDS_UPD_DDPM && r.kind != CDS_UPD_DDIM) {
    p.xhat_prev[i] = xhat;
  }
  p.x[i] = out;
  if (p.x_cast) {
    if (p.x_cast_dtype == CDS_BF16) reinterpret_cast<__nv_bfloat16*>(p.x_cast)[cast_off] = __float2bfloat16_rn(out);
    else reinterpret_cast<float*>(p.x_cast)[cast_off] = f32_for_store(out, p.x_cast_dtype);
  }
}

// the last block of a grid to finish bumps the iteration counter ([0] = counter, [1] = blocks finished): saves the
// one-thread advance kernel at the end of every iteration.  Every block has read the counter before it signals.
__device__ __forceinline__ void advance_iteration_when_last(int* advance, int iter) {
  __syncthreads();
  if (threadIdx.x == 0) {
    __threadfence();
    if (atomicAdd(&advance[1], 1) == (int)gridDim.x - 1) { advance[1] = 0; advance[0] = iter + 1; }
  }
}

// reads x, pred (+pred_uncond, noise, prior, xhat_prev), writes x (+xhat_prev): 12..28 B / element
// One thread = 4 consecutive elements (float4 traffic on x / pred / noise / prior) when the row length allows it and there is
// no guidance operand (guided EDM programs take the scalar path).
static __global__ void __launch_bounds__(256) solver_update_kernel(const cds_update_op p, const int* iter_ptr, int* advance) {
  const int iter = *iter_ptr;
  const UpdRow r = load_upd_row(p, iter);
  const int64_t total = (int64_t)p.batch * p.row;
  const bool small = total < (int64_t)0x7fffffff;            // 32-bit index arithmetic (64-bit divisions are ~20x dearer)
  const bool vec4 = small && (p.row % 4 == 0) && !p.pred_uncond && !p.xhat_prev && !p.guide &&
                    (((uintptr_t)p.x | (uintptr_t)p.pred | (uintptr_t)p.prior | (uintptr_t)r.noise) % 16 == 0);
  if (vec4) {
    const unsigned n4 = (unsigned)(total / 4);
    for (unsigned g = blockIdx.x * blockDim.x + threadIdx.x; g < n4; g += gridDim.x * blockDim.x) {
      const unsigned i0 = 4u * g;
      const int e0 = (int)(i0 % (unsigned)p.row);
      const float4 xv = reinterpret_cast<const float4*>(p.x)[g];
      const float4 pv = reinterpret_cast<const float4*>(p.pred)[g];
      float4 zv = make_float4(0.f, 0.f, 0.f, 0.f), qv = zv;
      if (r.noise) zv = reinterpret_cast<const float4*>(r.noise)[g];
      if (p.mask) qv = reinterpret_cast<const float4*>(p.prior)[g];
      const float xs[4] = {xv.x, xv.y, xv.z, xv.w}, ps[4] = {pv.x, pv.y, pv.z, pv.w};
      const float zs[4] = {zv.x, zv.y, zv.z, zv.w}, qs[4] = {qv.x, qv.y, qv.z, qv.w};
      float os[4];
#pragma unroll
      for (int k = 0; k < 4; ++k) os[k] = solver_update_value(p, r, e0 + k, xs[k], ps[k], zs[k], qs[k], 0.f, nullptr);
      reinterpret_cast<float4*>(p.x)[g] = make_float4(os[0], os[1], os[2], os[3]);
      if (p.x_cast) {
        unsigned rr = i0 / (unsigned)p.cast_C_in, c = i0 - rr * (unsigned)p.cast_C_in;
        const bool cast_bf16 = p.x_cast_dtype == CDS_BF16;
#pragma unroll
        for (int k = 0; k < 4; ++k) {
          const int64_t o = (int64_t)rr * p.cast_C_out + c;
          if (cast_bf16) reinterpret_cast<__nv_bfloat16*>(p.x_cast)[o] = __float2bfloat16_rn(os[k]);
          else reinterpret_cast<float*>(p.x_cast)[o] = f32_for_store(os[k], p.x_cast_dtype);
          if (++c == (unsigned)p.cast_C_in) { c = 0; ++rr; }
        }
      }
    }
  } else {
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
      float pr = p.pred[i];
      if (p.pred_uncond) pr = add_(mul_(p.w_cfg, pr), mul_(p.w_uncond, p.pred_uncond[i]));
      int e;
      int64_t cast_off = 0;
      if (small) {
        const unsigned iu = (unsigned)i;
        e = (int)(iu % (unsigned)p.row);
        if (p.x_cast) { const unsigned rr = iu / (unsigned)p.cast_C_in; cast_off = (int64_t)rr * p.cast_C_out + (iu - rr * (unsigned)p.cast_C_in); }
      } else {
        e = (int)(i % p.row);
        if (p.x_cast) { const int64_t rr = i / p.cast_C_in; cast_off = rr * p.cast_C_out + (i - rr * p.cast_C_in); }
      }
      solver_update_element(p, r, i, e, cast_off, pr);
    }
  }
  if (advance) advance_iteration_when_last(advance, iter);
}

// x += K2*z (re-noise, only when the row has a noise slot); xin = K3*x.   8..16 B / element
static __global__ void __launch_bounds__(256) cm_prep_kernel(const cds_prep_op p, const int* __restrict__ iter_ptr) {
  const int iter = *iter_ptr;
  const float* row = p.coef + (int64_t)iter * CDS_ROW_FLOATS;
  const float k2 = row[CDS_ROW_K2], k3 = row[CDS_ROW_K3];
  const int slot = (int)row[CDS_ROW_NOISE] - 1;
  const int64_t total = (int64_t)p.batch * p.row;
  const float* noise = slot >= 0 ? p.noise + (int64_t)slot * total : nullptr;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    float x = p.x[i];
    if (noise) { x = add_(x, mul_(k2, noise[i])); p.x[i] = x; }
    p.xin[i] = mul_(k3, x);
  }
}

// one warp per token row: LayerNorm (biased variance, no affine) then x*(1+scale)+shift.  8 B / element (6 with bf16 out).
// Rows of up to 128*kLnVec channels with C % 4 == 0 (DiT1d: 320) are held in registers as float4s: ONE pass over global memory
// with 16-byte loads / stores (two-pass variance on the registers), two rows in flight per warp iteration; other shapes take
// the scalar path.
constexpr int kLnRegs = 16;
constexpr int kLnVec = 4;               // float4s per lane: rows of up to 512 channels
__device__ __forceinline__ void ln_store4(const cds_lnmod_op& p, int64_t off, float4 v) {
  if (p.out_dtype == CDS_BF16) {
    __nv_bfloat162 a = __floats2bfloat162_rn(v.x, v.y), b = __floats2bfloat162_rn(v.z, v.w);
    uint2 u; u.x = *reinterpret_cast<uint32_t*>(&a); u.y = *reinterpret_cast<uint32_t*>(&b);
    *reinterpret_cast<uint2*>(reinterpret_cast<__nv_bfloat16*>(p.out) + off) = u;
  } else {
    if (p.out_dtype == CDS_TF32) v = make_float4(round_tf32(v.x), round_tf32(v.y), round_tf32(v.z), round_tf32(v.w));
    *reinterpret_cast<float4*>(reinterpret_cast<float*>(p.out) + off) = v;
  }
}
// LPR lanes per row (32: one row per warp; 16: two rows per warp, each on a half-warp -- DiT1d's 320 channels are exactly
// 16 lanes x 5 float4s, so no lane idles and twice as many rows are in flight), K float4s per lane
template <int LPR, int K>
__device__ __forceinline__ void ln_rows_vec(const cds_lnmod_op& p, int64_t n_rows, float inv_c) {
  constexpr int RPW = 32 / LPR;                               // rows per warp
  const int lane = threadIdx.x & 31, sub = lane / LPR, li = lane % LPR;
  const int n4 = p.C >> 2;                                    // float4s per row
  const int64_t warp0 = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5), nwarps = (int64_t)gridDim.x * (blockDim.x >> 5);
  for (int64_t r0 = warp0 * RPW; r0 < n_rows; r0 += nwarps * RPW) {
    const int64_t r = r0 + sub;
    const bool live = r < n_rows;
    const int64_t rr = live ? r : n_rows - 1;                 // (idle half-warps shadow the last row: uniform shuffles, no store)
    const float4* src = reinterpret_cast<const float4*>(p.in + rr * p.C);
    const int b = (int)(rr / p.L);
    const float4* sh = reinterpret_cast<const float4*>(p.shift + (int64_t)b * p.mod_bstride);
    const float4* sc = reinterpret_cast<const float4*>(p.scale + (int64_t)b * p.mod_bstride);
    float4 x[K];
    float s = 0.f;
#pragma unroll
    for (int k = 0; k < K; ++k) {
      const int c4 = li + LPR * k;
      x[k] = c4 < n4 ? __ldg(src + c4) : make_float4(0.f, 0.f, 0.f, 0.f);
      s += (x[k].x + x[k].y) + (x[k].z + x[k].w);
    }
#pragma unroll
    for (int o = LPR / 2; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    const float mean = s * inv_c;
    float q = 0.f;
#pragma unroll
    for (int k = 0; k < K; ++k) {
      if (li + LPR * k < n4) {
        const float d0 = x[k].x - mean, d1 = x[k].y - mean, d2 = x[k].z - mean, d3 = x[k].w - mean;
        q = fmaf(d0, d0, q); q = fmaf(d1, d1, q); q = fmaf(d2, d2, q); q = fmaf(d3, d3, q);
      }
    }
#pragma unroll
    for (int o = LPR / 2; o > 0; o >>= 1) q += __shfl_xor_sync(0xffffffffu, q, o);
    const float rstd = rsqrtf(q * inv_c + p.eps);
#pragma unroll
    for (int k = 0; k < K; ++k) {
      const int c4 = li + LPR * k;
      if (c4 < n4 && live) {
        const float4 a = __ldg(sc + c4), d = __ldg(sh + c4);
        float4 o;
        o.x = fmaf((x[k].x - mean) * rstd, 1.f + a.x, d.x); o.y = fmaf((x[k].y - mean) * rstd, 1.f + a.y, d.y);
        o.z = fmaf((x[k].z - mean) * rstd, 1.f + a.z, d.z); o.w = fmaf((x[k].w - mean) * rstd, 1.f + a.w, d.w);
        ln_store4(p, r * p.C + 4 * c4, o);
      }
    }
  }
}

static __global__ void __launch_bounds__(256) ln_modulate_kernel(const cds_lnmod_op p) {
  const int warps_per_block = blockDim.x >> 5;
  const int lane = threadIdx.x & 31;
  const int64_t n_rows = (int64_t)p.batch * p.L;
  const float inv_c = 1.f / (float)p.C;
  const bool vec = (p.C % 4 == 0) && p.C <= 128 * kLnVec && ((uintptr_t)p.in % 16 == 0) && ((uintptr_t)p.out % 16 == 0) &&
                   ((uintptr_t)p.shift % 16 == 0) && ((uintptr_t)p.scale % 16 == 0) && (p.mod_bstride % 4 == 0);
  if (vec) {
    const int n4 = p.C >> 2;
    if (n4 <= 16 * 3) ln_rows_vec<16, 3>(p, n_rows, inv_c);
    else if (n4 <= 16 * 6 && n4 % 16 == 0) ln_rows_vec<16, 6>(p, n_rows, inv_c);
    else ln_rows_vec<32, kLnVec>(p, n_rows, inv_c);
    return;
  }
  const bool in_regs = p.C <= 32 * kLnRegs;
  for (int64_t r = (int64_t)blockIdx.x * warps_per_block + (threadIdx.x >> 5); r < n_rows;
       r += (int64_t)gridDim.x * warps_per_block) {
    const float* src = p.in + r * p.C;
    const int b = (int)(r / p.L);
    const float* sh = p.shift + (int64_t)b * p.mod_bstride;
    const float* sc = p.scale + (int64_t)b * p.mod_bstride;
    float x[kLnRegs];
    float s = 0.f;
    if (in_regs) {
#pragma unroll
      for (int k = 0; k < kLnRegs; ++k) { const int c = lane + 32 * k; x[k] = c < p.C ? src[c] : 0.f; s += x[k]; }
    } else {
      for (int c = lane; c < p.C; c += 32) s += src[c];
    }
    const float mean = warp_sum(s) * inv_c;
    float q = 0.f;
    if (in_regs) {
#pragma unroll
      for (int k = 0; k < kLnRegs; ++k) { const float d = (lane + 32 * k < p.C) ? x[k] - mean : 0.f; q = fmaf(d, d, q); }
    } else {
      for (int c = lane; c < p.C; c += 32) { float d = src[c] - mean; q = fmaf(d, d, q); }
    }
    const float rstd = rsqrtf(warp_sum(q) * inv_c + p.eps);
    auto value = [&](int c, float xv) { return fmaf((xv - mean) * rstd, 1.f + sc[c], sh[c]); };
    if (p.out_dtype == CDS_BF16) {
      __nv_bfloat16* dst = reinterpret_cast<__nv_bfloat16*>(p.out) + r * p.C;
      if (in_regs) {
#pragma unroll
        for (int k = 0; k < kLnRegs; ++k) { const int c = lane + 32 * k; if (c < p.C) dst[c] = __float2bfloat16_rn(value(c, x[k])); }
      } else {
        for (int c = lane; c < p.C; c += 32) dst[c] = __float2bfloat16_rn(value(c, src[c]));
      }
    } else {
      float* dst = reinterpret_cast<float*>(p.out) + r * p.C;
      if (in_regs) {
#pragma unroll
        for (int k = 0; k < kLnRegs; ++k) { const int c = lane + 32 * k; if (c < p.C) dst[c] = f32_for_store(value(c, x[k]), p.out_dtype); }
      } else {
        for (int c = lane; c < p.C; c += 32) dst[c] = f32_for_store(value(c, src[c]), p.out_dtype);
      }
    }
  }
}

// fp32 (rows, C_in) -> bf16 or fp32 (rows, C_out) zero padded; one thread per output pair.  4*C_in + (2|4)*C_out B / row
static __global__ void __launch_bounds__(256) cast_pad_kernel(const cds_cast_op p) {
  const int64_t rows = (int64_t)p.batch * p.L;
  const int pairs = p.C_out >> 1;
  const int64_t total = rows * pairs;
  const bool bf16 = p.out_dtype == CDS_BF16;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t r = i / pairs;
    const int c = (int)(i - r * pairs) * 2;
    const float a = c < p.C_in ? p.in[r * p.C_in + c] : 0.f;
    const float b = c + 1 < p.C_in ? p.in[r * p.C_in + c + 1] : 0.f;
    if (bf16) reinterpret_cast<__nv_bfloat162*>(p.out)[i] = __floats2bfloat162_rn(a, b);
    else reinterpret_cast<float2*>(p.out)[i] = make_float2(f32_for_store(a, p.out_dtype), f32_for_store(b, p.out_dtype));
  }
}

static __global__ void set_iter_kernel(int* iter_ptr, int value) { *iter_ptr = value; }
static __global__ void advance_iter_kernel(int* iter_ptr) { *iter_ptr += 1; }

}  // namespace cds
