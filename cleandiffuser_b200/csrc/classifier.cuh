// Classifier guidance inside the replayed loop (CumRewClassifier over HalfJannerUNet1d):
//   CDS_OP_GN      act(GroupNorm(h) gamma + beta) [+ vec] [+ res] over a kept pre-norm input h, 8..16 B / element
//   CDS_OP_GN_BWD  its backward with respect to h (statistics recomputed from h), 12 B / element
//   CDS_OP_GUIDE   pred += s[iter] * g, 12 B / element
// and, for QGPOClassifier (an Mlp of Linear + SiLU under an energy head 10 tanh(z / 10)):
//   CDS_OP_HEAD_GRAD  z = act(h) . w + b per row and the seed d logp / d z of the backward, 4 B / element of h
// One warp owns one (trajectory, group): a group holds at most a few hundred elements at the classifier's shapes (L x C/groups
// <= 64 x 32), too few to split, and a warp-local reduction keeps every sum in one fixed order with no atomics -- two runs are
// bitwise equal and CDS_OP_GN_BWD recomputes exactly the mean and rstd CDS_OP_GN used.
#pragma once
#include "common.cuh"
#include "elementwise.cuh"
#include "grad.cuh"

namespace cds {

struct GnGeom {
  int L, cpg, n;        // positions, channels per group, elements per group
};

// element e of group (b, g) -> offset of (l, c) in a (batch, L, C) view with the given strides
__device__ __forceinline__ int64_t gn_at(int64_t bstride, int lstride, int b, int l, int c) {
  return (int64_t)b * bstride + (int64_t)l * lstride + c;
}

// mean and rstd of one (b, group) over a warp: lane-strided partial sums, then the xor butterfly
__device__ __forceinline__ void gn_stats(const float* __restrict__ h, int64_t bstride, int lstride, int b, int c0, const GnGeom& g,
                                         float eps, float* mean, float* rstd) {
  const int lane = threadIdx.x & 31;
  float s = 0.f;
  for (int e = lane; e < g.n; e += 32) s += h[gn_at(bstride, lstride, b, e / g.cpg, c0 + e % g.cpg)];
  const float m = warp_sum(s) / (float)g.n;
  float q = 0.f;
  for (int e = lane; e < g.n; e += 32) {
    const float d = h[gn_at(bstride, lstride, b, e / g.cpg, c0 + e % g.cpg)] - m;
    q = fmaf(d, d, q);
  }
  const float var = warp_sum(q) / (float)g.n;
  *mean = m;
  *rstd = 1.f / sqrtf(var + eps);
}

static __global__ void __launch_bounds__(256) gn_kernel(const cds_gn_op p, const int* __restrict__ iter_ptr) {
  const int warp = (int)((blockIdx.x * blockDim.x + threadIdx.x) >> 5), lane = threadIdx.x & 31;
  if (warp >= p.batch * p.groups) return;
  const int b = warp / p.groups, c0 = (warp % p.groups) * (p.C / p.groups);
  const GnGeom g{p.L, p.C / p.groups, p.L * (p.C / p.groups)};
  float mean, rstd;
  gn_stats(p.h, p.h_bstride, p.h_lstride, b, c0, g, p.eps, &mean, &rstd);
  const VecRef v = resolve(p.vec, *iter_ptr);
  for (int e = lane; e < g.n; e += 32) {
    const int l = e / g.cpg, c = c0 + e % g.cpg;
    const float xhat = (p.h[gn_at(p.h_bstride, p.h_lstride, b, l, c)] - mean) * rstd;
    float y = apply_act(p.act, fmaf(xhat, p.gamma[c], p.beta[c]));
    if (v.present()) y += v.at(b, c);
    if (p.res) y += p.res[gn_at(p.res_bstride, p.res_lstride, b, l, c)];
    p.out[gn_at(p.out_bstride, p.out_lstride, b, l, c)] = f32_for_store(y, p.out_dtype);
  }
}

static __global__ void __launch_bounds__(256) gn_bwd_kernel(const cds_gn_bwd_op p) {
  const int warp = (int)((blockIdx.x * blockDim.x + threadIdx.x) >> 5), lane = threadIdx.x & 31;
  if (warp >= p.batch * p.groups) return;
  const int b = warp / p.groups, c0 = (warp % p.groups) * (p.C / p.groups);
  const GnGeom g{p.L, p.C / p.groups, p.L * (p.C / p.groups)};
  float mean, rstd;
  gn_stats(p.h, p.h_bstride, p.h_lstride, b, c0, g, p.eps, &mean, &rstd);
  // dxhat and the two group means of the backward (dxhat is recomputed in the write pass rather than kept)
  auto dxhat_at = [&](int l, int c, float* xhat_out) {
    const float xhat = (p.h[gn_at(p.h_bstride, p.h_lstride, b, l, c)] - mean) * rstd;
    float d = p.gamma[c] * p.dout[gn_at(p.dout_bstride, p.dout_lstride, b, l, c)];
    if (p.act == CDS_ACT_MISH) d *= mish_grad(fmaf(xhat, p.gamma[c], p.beta[c]));
    *xhat_out = xhat;
    return d;
  };
  float s1 = 0.f, s2 = 0.f;
  for (int e = lane; e < g.n; e += 32) {
    float xhat;
    const float d = dxhat_at(e / g.cpg, c0 + e % g.cpg, &xhat);
    s1 += d;
    s2 = fmaf(d, xhat, s2);
  }
  const float m1 = warp_sum(s1) / (float)g.n, m2 = warp_sum(s2) / (float)g.n;
  for (int e = lane; e < g.n; e += 32) {
    const int l = e / g.cpg, c = c0 + e % g.cpg;
    float xhat;
    const float d = dxhat_at(l, c, &xhat);
    p.dh[gn_at(p.dh_bstride, p.dh_lstride, b, l, c)] = f32_for_store(rstd * (d - m1 - xhat * m2), p.dh_dtype);
  }
}

static __global__ void __launch_bounds__(256) guide_kernel(const cds_guide_op p, const int* __restrict__ iter_ptr) {
  const float s = p.s[*iter_ptr];
  const int64_t row = (int64_t)p.L * p.C, total = (int64_t)p.batch * row;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t b = i / row;
    const int r = (int)(i - b * row), l = r / p.C, c = r - l * p.C;
    p.pred[i] = add_(p.pred[i], mul_(s, p.g[b * p.g_bstride + (int64_t)l * p.g_lstride + c]));
  }
}

// One warp per row: the out_dim-1 Linear is a K-long dot product (K = 256 at QGPO's shapes), too short for a GEMM tile and
// one launch instead of a conv plus an elementwise tanh.  Lane l sums elements l, l + 32, ... in order, then warp_sum's fixed
// xor butterfly: the same bits on every run.  The seed follows autograd's order for logp = scale * tanh(z / scale):
// mul's backward (1 * scale), tanh_backward (g * (1 - y * y)), then div's backward (/ scale).
static __global__ void __launch_bounds__(256) head_grad_kernel(const cds_head_grad_op p) {
  const int r = (int)((blockIdx.x * blockDim.x + threadIdx.x) >> 5), lane = threadIdx.x & 31;
  if (r >= p.rows) return;
  const float* h = p.h + (int64_t)r * p.ldh;
  float s = 0.f;
  for (int k = lane; k < p.K; k += 32) s = fmaf(apply_act(p.act, h[k]), p.w[k], s);
  const float z = add_(warp_sum(s), p.b[0]);
  const float y = tanhf(div_(z, p.scale));
  if (lane == 0) p.seed[r] = div_(mul_(mul_(1.f, p.scale), sub_(1.f, mul_(y, y))), p.scale);
}

inline int gn_grid(int batch, int groups) { return (int)(((int64_t)batch * groups + 7) / 8); }

inline int head_grad_grid(int rows) { return (rows + 7) / 8; }

}  // namespace cds
