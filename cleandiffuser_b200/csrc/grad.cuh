// Backward operators of a differentiable reverse loop (sample(requires_grad=True) over DQLMlp):
//   CDS_OP_STASH       per-iteration copy of a forward operand (+ the Mish of a pre-activation), 8..12 B / element
//   CDS_OP_UPDATE_BWD  backward of the solver update + clip_prediction + fix_mask (kinds DDPM, DDIM, EPS, X) and of the
//                      consistency model's combine + clip + fix_mask (kind CM), 24..36 B / element
//   CDS_OP_PREP        backward mode: gx += c_in * d xin (the consistency model's input scaling), 12 B / element
//   CDS_OP_DGRAD       dH = dZ W with the Mish or SiLU derivative of the stashed pre-activation fused into the epilogue
//   CDS_OP_WGRAD       dW += Z^T H, db += sum_rows dZ, accumulated over the iterations
// The two GEMM-shaped operators run on fp32 CUDA cores with 32 x 32 output tiles staged through shared memory: every output
// element is one thread's sum in a fixed order (no split-K, no atomics), so a backward run is bitwise reproducible.
#pragma once
#include "common.cuh"
#include "elementwise.cuh"

namespace cds {

// d/dx mish(x), ATen's formula (aten/src/ATen/native/cuda/ActivationMishKernel.cu): tanh(softplus(x)) + x sigmoid(x) (1 - tanh^2)
__device__ __forceinline__ float mish_grad(float x) {
  const float sig = 1.f / (1.f + expf(-x));
  const float tsp = tanhf(log1pf(expf(x)));
  return tsp + x * sig * (1.f - tsp * tsp);
}

// d/dx silu(x), ATen's formula (aten/src/ATen/native/cuda/ActivationSiluKernel.cu, silu_backward): sig (1 + x (1 - sig))
__device__ __forceinline__ float silu_grad(float x) {
  const float sig = 1.f / (1.f + expf(-x));
  return sig * (1.f + x * (1.f - sig));
}

// d/dx relu(x), ATen's threshold_backward: 1 where x > 0, else 0 (0 at x == 0)
__device__ __forceinline__ float relu_grad(float x) { return x > 0.f ? 1.f : 0.f; }

// d/dx gelu_tanh(x), ATen's formula (aten/src/ATen/native/cuda/ActivationGeluKernel.cu, GeluBackwardCUDAKernelImpl with
// approximate = "tanh"): 0.5 (1 + tanh(u)) + 0.5 x (1 - tanh(u)^2) sqrt(2/pi) (1 + 3 kappa x^2),  u = sqrt(2/pi) (x + kappa x^3)
__device__ __forceinline__ float gelu_tanh_grad(float x) {
  const float kBeta = 0.7978845608028654f, kKappa = 0.044715f;
  const float x_sq = x * x;
  const float inner = kBeta * (x + kKappa * x_sq * x);
  const float t = tanhf(inner);
  const float left = 0.5f * x, right = 1.f + t;
  const float left_derivative = 0.5f * right;
  const float right_derivative = left * (1.f - t * t) * (kBeta * (1.f + 3.f * kKappa * x_sq));
  return left_derivative + right_derivative;
}

// the derivative of the activations CDS_OP_DGRAD and CDS_OP_STASH's backward mode accept (cds_api.cu rejects every other act before a launch)
__device__ __forceinline__ float act_grad(int act, float x) {
  switch (act) {
    case CDS_ACT_SILU: return silu_grad(x);
    case CDS_ACT_RELU: return relu_grad(x);
    case CDS_ACT_GELU_TANH: return gelu_tanh_grad(x);
    case CDS_ACT_MISH:
    default: return mish_grad(x);
  }
}

static __global__ void __launch_bounds__(256) stash_kernel(const cds_stash_op p, const int* __restrict__ iter_ptr) {
  const int iter = *iter_ptr;
  float* dst = p.dst ? p.dst + (int64_t)iter * p.dst_iter_stride : nullptr;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < p.n; i += (int64_t)gridDim.x * blockDim.x) {
    const float v = p.src[i];
    if (dst) dst[i] = v;
    if (p.act_out) p.act_out[i] = apply_act(p.act, v);
  }
}

// One element of the update's backward.  Mirrors solver_update_value (elementwise.cuh) for kinds DDPM / DDIM / EPS / X / CM
// in reverse, op by op, with torch.clip's tensor-bound gradient rule for clip_prediction and for CM's final clip.  A kind
// without a backward here (X2M, EDM, EDM_HEUN) writes NaN to both outputs: the host never builds such a program, and a
// gradient of the wrong formula must not pass for a correct one.
static __global__ void __launch_bounds__(256) update_bwd_kernel(const cds_update_bwd_op p, const int* __restrict__ iter_ptr) {
  const int iter = *iter_ptr;
  const float* row = p.coef + (int64_t)iter * p.coef_iter_stride;
  const float alpha = row[CDS_ROW_ALPHA], sigma = row[CDS_ROW_SIGMA], k0 = row[CDS_ROW_K0], k1 = row[CDS_ROW_K1];
  const int kind = (int)row[CDS_ROW_KIND];
  const bool known = kind == CDS_UPD_DDPM || kind == CDS_UPD_DDIM || kind == CDS_UPD_EPS || kind == CDS_UPD_X || kind == CDS_UPD_CM;
  const float* xs = p.x + (int64_t)iter * p.x_iter_stride;
  const float* ps = p.pred + (int64_t)iter * p.pred_iter_stride;
  const int64_t total = (int64_t)p.batch * p.row;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int e = (int)(i % p.row);
    const float x = xs[i], pr = ps[i];
    float g = p.gx[i];
    if (p.mask) g = mul_(g, 1.f - p.mask[e]);
    if (!known) {
      p.gpred[i] = p.gx[i] = __int_as_float(0x7fc00000);
      continue;
    }
    if (kind == CDS_UPD_CM) {
      // f = c_skip*x + c_out*pred with the forward's fp32 ops, then clip(f, x_min, x_max): the gradient passes where f lies
      // inside the bounds or equals one (torch.clip's rule; none passes when x_min > x_max), and goes to neither operand elsewhere
      const float f = add_(mul_(k0, x), mul_(k1, pr));
      bool pass = true;
      if (p.x_min && p.x_max) pass = f >= p.x_min[e] && f <= p.x_max[e];
      else if (p.x_min) pass = f >= p.x_min[e];
      else if (p.x_max) pass = f <= p.x_max[e];
      const float gf = pass ? g : 0.f;
      p.gpred[i] = mul_(k1, gf);
      p.gx[i] = mul_(k0, gf);
      continue;
    }
    // d of the update with respect to x (direct), eps and xhat
    float dx = 0.f, deps = 0.f, dxhat = 0.f;
    if (kind == CDS_UPD_DDPM) {
      const float a = mul_(k0, g);                            // d (x - sigma*eps)
      dx = a;
      deps = add_(mul_(k1, g), -mul_(a, sigma));
    } else if (kind == CDS_UPD_DDIM) {
      const float a = div_(mul_(k0, g), alpha);               // d (x - sigma*eps)
      dx = a;
      deps = add_(mul_(k1, g), -mul_(a, sigma));
    } else if (kind == CDS_UPD_EPS) {
      dx = mul_(k0, g);
      deps = -mul_(k1, g);
    } else {                                                   // CDS_UPD_X
      dx = mul_(k0, g);
      dxhat = -mul_(k1, g);
    }
    // eps <-> x0 conversion
    float dpc;
    if (p.predict_noise) {                                     // xhat = (x - sigma*pc)/alpha
      const float q = div_(dxhat, alpha);
      dx = add_(dx, q);
      dpc = add_(deps, -mul_(q, sigma));
    } else {                                                   // eps = (x - alpha*pc)/sigma
      const float q = div_(deps, sigma);
      dx = add_(dx, q);
      dpc = add_(dxhat, -mul_(q, alpha));
    }
    // clip_prediction: pc = clip(pr, lo, hi)
    const bool has_lo = p.predict_noise ? p.x_max != nullptr : p.x_min != nullptr;
    const bool has_hi = p.predict_noise ? p.x_min != nullptr : p.x_max != nullptr;
    float lo = 0.f, hi = 0.f;
    if (p.predict_noise) {
      if (has_lo) lo = div_(sub_(x, mul_(alpha, p.x_max[e])), sigma);
      if (has_hi) hi = div_(sub_(x, mul_(alpha, p.x_min[e])), sigma);
    } else {
      if (has_lo) lo = p.x_min[e];
      if (has_hi) hi = p.x_max[e];
    }
    float gp = dpc, glo = 0.f, ghi = 0.f;
    if (has_lo && has_hi) {
      gp = (pr >= lo && pr <= hi) ? dpc : 0.f;
      glo = (pr < lo && lo < hi) ? dpc : 0.f;
      ghi = (pr > hi || hi < lo) ? dpc : 0.f;
    } else if (has_lo) {
      gp = pr >= lo ? dpc : 0.f;
      glo = pr < lo ? dpc : 0.f;
    } else if (has_hi) {
      gp = pr <= hi ? dpc : 0.f;
      ghi = pr > hi ? dpc : 0.f;
    }
    if (p.predict_noise) {                                     // the bounds (x - alpha*lim)/sigma depend on x_t
      if (has_lo) dx = add_(dx, div_(glo, sigma));
      if (has_hi) dx = add_(dx, div_(ghi, sigma));
    }
    p.gpred[i] = gp;
    p.gx[i] = dx;
  }
}

// Backward mode of CDS_OP_PREP (gxin != NULL): gx += K3 * gxin, with gx in the descriptor's x.  xin = K3*x is the network's
// input, so its gradient gxin reaches x scaled by K3; the re-noise x += K2*z is additive and passes gx through unchanged.
// 12 B / element.
static __global__ void __launch_bounds__(256) prep_bwd_kernel(const cds_prep_op p, const int* __restrict__ iter_ptr) {
  const int iter = *iter_ptr;
  const float k3 = p.coef[(int64_t)iter * p.coef_iter_stride + CDS_ROW_K3];
  const int64_t total = (int64_t)p.batch * p.row;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x)
    p.x[i] = add_(p.x[i], mul_(k3, p.gxin[i]));
}

constexpr int kGradTile = 32;

// out(r, k) [+]= (sum_n dz(r, n) W(n, k)) * act'(z(r, k)).  CTA = 32 rows x 32 columns, thread = 1 row x 4 columns.
static __global__ void __launch_bounds__(256) dgrad_kernel(const cds_dgrad_op p, const int* __restrict__ iter_ptr) {
  __shared__ float sdz[kGradTile][kGradTile + 1];
  __shared__ float sw[kGradTile][kGradTile + 4];
  const int iter = *iter_ptr;
  const int r0 = blockIdx.x * kGradTile, c0 = blockIdx.y * kGradTile;
  const int tid = threadIdx.x, lr = tid >> 3, lc = (tid & 7) * 4;
  float acc[4] = {0.f, 0.f, 0.f, 0.f};
  for (int n0 = 0; n0 < p.N; n0 += kGradTile) {
    for (int j = tid; j < kGradTile * kGradTile; j += 256) {
      const int a = j / kGradTile, b = j % kGradTile;
      const int r = r0 + a, n = n0 + b;
      sdz[a][b] = (r < p.rows && n < p.N) ? p.dz[(int64_t)r * p.ldz + n] : 0.f;
      const int nn = n0 + a, k = c0 + b;
      sw[a][b] = (nn < p.N && k < p.K) ? p.w[(int64_t)nn * p.ldw + k] : 0.f;
    }
    __syncthreads();
#pragma unroll 8
    for (int n = 0; n < kGradTile; ++n) {
      const float a = sdz[lr][n];
#pragma unroll
      for (int j = 0; j < 4; ++j) acc[j] = fmaf(a, sw[n][lc + j], acc[j]);
    }
    __syncthreads();
  }
  const int r = r0 + lr;
  if (r >= p.rows) return;
  const float* z = p.z ? p.z + (int64_t)iter * p.z_iter_stride : nullptr;
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    const int k = c0 + lc + j;
    if (k >= p.K) continue;
    float v = acc[j];
    if (p.act != CDS_ACT_NONE) v = mul_(v, act_grad(p.act, z[(int64_t)r * p.K + k]));
    float* o = p.out + (int64_t)r * p.ldo + k;
    *o = p.accumulate ? add_(*o, v) : v;
    if (p.out_sum) { float* s = p.out_sum + (int64_t)r * p.K + k; *s = add_(*s, v); }
  }
}

// dw(n, k) [+]= sum_r dz(r, n) act(h(r, k)); column k = K is the bias (h = 1).  CTA = 32 x 32 outputs, thread = 1 x 4,
// rows reduced in order in chunks of 32.
static __global__ void __launch_bounds__(256) wgrad_kernel(const cds_wgrad_op p, const int* __restrict__ iter_ptr) {
  __shared__ float sdz[kGradTile][kGradTile + 1];
  __shared__ float sh[kGradTile][kGradTile + 4];
  const int iter = *iter_ptr;
  const int n0 = blockIdx.x * kGradTile, c0 = blockIdx.y * kGradTile;
  const int tid = threadIdx.x, ln = tid >> 3, lc = (tid & 7) * 4;
  const float* h = p.h + (int64_t)iter * p.h_iter_stride;
  const bool bias = p.db != nullptr;
  float acc[4] = {0.f, 0.f, 0.f, 0.f};
  for (int rb = 0; rb < p.rows; rb += kGradTile) {
    for (int j = tid; j < kGradTile * kGradTile; j += 256) {
      const int a = j / kGradTile, b = j % kGradTile;           // a = row inside the chunk
      const int r = rb + a, n = n0 + b, k = c0 + b;
      sdz[a][b] = (r < p.rows && n < p.N) ? p.dz[(int64_t)r * p.ldz + n] : 0.f;
      float hv = 0.f;
      if (r < p.rows) {
        if (k < p.K) hv = apply_act(p.act, h[(int64_t)r * p.ldh + k]);
        else if (k == p.K && bias) hv = 1.f;
      }
      sh[a][b] = hv;
    }
    __syncthreads();
#pragma unroll 8
    for (int rr = 0; rr < kGradTile; ++rr) {
      const float a = sdz[rr][ln];
#pragma unroll
      for (int j = 0; j < 4; ++j) acc[j] = fmaf(a, sh[rr][lc + j], acc[j]);
    }
    __syncthreads();
  }
  const int n = n0 + ln;
  if (n >= p.N) return;
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    const int k = c0 + lc + j;
    float* o = nullptr;
    if (k < p.K) o = p.dw + (int64_t)n * p.lddw + k;
    else if (k == p.K && bias) o = p.db + (int64_t)iter * p.db_iter_stride + n;
    if (o) *o = p.accumulate ? add_(*o, acc[j]) : acc[j];
  }
}

inline dim3 dgrad_grid(const cds_dgrad_op& p) {
  return dim3((p.rows + kGradTile - 1) / kGradTile, (p.K + kGradTile - 1) / kGradTile);
}
inline dim3 wgrad_grid(const cds_wgrad_op& p) {
  const int cols = p.K + (p.db ? 1 : 0);
  return dim3((p.N + kGradTile - 1) / kGradTile, (cols + kGradTile - 1) / kGradTile);
}

}  // namespace cds
