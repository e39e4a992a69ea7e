// CDS_OP_CONV, tensor-core path for SHORT sequences ("position-sliced" kernel): stride-1 Conv1d + GroupNorm + Mish
// (+ additive time row / identity residual / 1x1 shortcut conv) at a resolution of P = 4 positions -- the bottom of the
// UNets, where two thirds of JannerUNet1d's FLOPs live.
//
// conv_tc_kernel makes a 128-row tile out of 128/L whole trajectories and re-fetches the activation tile once per tap;
// at L = 4 that is 32 trajectories per weight slab and 5 x the activation bytes.  Here the GEMM rows are TRAJECTORIES:
//
//   D_l'[128 trajectories x N] (fp32)  +=  A_l[128 x KC] * W_(l - l' + pad)[N x KC]^T      |l - l'| <= pad
//
// * A_l = the activations of input position l: ONE TMA box {KC channels, 1 position, 128 trajectories} of the channels-last
//   tensor; every activation byte enters the SM once, the conv's zero padding is simply the absence of the (l, l') pairs
//   that fall outside [0, P) (14 MMAs instead of 20 for P = 4, taps = 5).
// * W_j = TMA box {KC, N} of the [tap][C_out][C_in] weight, fetched once per channel chunk and used by up to P MMAs:
//   4 x the trajectories per weight byte of conv_tc_kernel.
// * two consumer warpgroups (warps 0-7): warpgroup g holds the P accumulators D_l' of trajectories [64 g, 64 g + 64) in
//   registers (wgmma, N columns each; the shortcut conv's P accumulators next to them).  The CTA has one tile, so once the
//   MMAs are done the operand ring is idle and the accumulators are written over it as a 128-row fp32 tile.
// * epilogue (the same 8 warps): thread = one trajectory x NH = N/2 columns (ONE GroupNorm group) x all P positions, so the
//   GroupNorm statistics over (P positions x C_out/8 channels) are plain in-thread sums: no shuffles.  Two passes over the
//   tile (statistics, then normalise + Mish + store).
// * CTA tile = 128 trajectories x N = C_out/4 columns (2 GroupNorm groups: one per epilogue column slice); grid =
//   ceil(batch/128) x 4 CTAs (128 CTAs at batch 4096), one tile per CTA, 4-stage smem ring over the channel chunks, warp 8
//   is the TMA producer.
//
// Algorithmic HBM bytes per launch: 2*(batch*P*C_in + batch*P*C_out) (+ shortcut input), weights once through L2.
#pragma once
#include "conv_tc.cuh"

namespace cds {

struct ConvPsParams {
  CUtensorMap tm_a, tm_b, tm_a2, tm_b2;
  CUtensorMap tm_out;             // output as a TMA-store target: box {16 channels, 1 position, 32 trajectories} (one epilogue warp's
  int out_tma;                    // lanes x 16 columns), staged in shared memory; valid when out_tma != 0
  int batch, C_out, taps, pad;
  int kchunks, kchunks2;          // channel chunks of the main conv / of the shortcut conv
  int n_tiles;                    // column tiles per trajectory tile (C_out / N)
  int in_batch_mod, res_batch_mod;
  cds_vec bias, shift;
  const float* gn_gamma; const float* gn_beta; float gn_eps;
  const void* res; int64_t res_bstride; int res_lstride;
  const float* res_bias;
  void* out; int64_t out_bstride; int out_lstride;
  long long* trace;
};

constexpr int kPsEpiWarps = 8;                        // two consumer warpgroups: MMA, then epilogue
constexpr int kPsEpiThreads = kPsEpiWarps * 32;
constexpr int kPsThreads = kPsEpiThreads + 32;        // + warp 8: TMA producer
constexpr int kPsWarpTma = kPsEpiWarps;

template <int KC, int N, int P, bool HAS_RES>
struct ConvPsCfg {
  static constexpr int kTapsMax = 5;
  static constexpr int kRowBytes = KC * 2;
  static constexpr int kATile = 128 * kRowBytes;
  static constexpr int kBTile = N * kRowBytes;
  static constexpr int kStageBytes = P * kATile + kTapsMax * kBTile;
  static constexpr int kStages = KC == 64 ? 2 : 4;     // ~200 KB of operands in flight either way; finer chunks pipeline better
  static constexpr int kSmemBytes = kStages * kStageBytes + 1024;
  // after the main loop: 16 KB of output staging (8 warps x 2 KB) and the accumulator tile, both over the idle ring
  static constexpr int kAccCols = P * N * (HAS_RES ? 2 : 1);
  static constexpr int kAccPitch = kAccCols + 4;       // padded against bank conflicts of the row-per-thread reads
  static constexpr int kStagingBytes = kPsEpiWarps * 2048;
  static_assert(kStagingBytes + 128 * kAccPitch * 4 <= kStages * kStageBytes, "accumulator tile must fit over the ring");
  static_assert(kSmemBytes <= 227 * 1024, "stage ring does not fit");
};

// TF32: fp32 activations / weights read as TF32; KC stays the row width in bf16-equivalents (row bytes / 2), see conv_tc.cuh
template <int KC, int N, int P, bool HAS_RES, bool TF32>
__global__ void __launch_bounds__(kPsThreads, 1)
conv_ps_kernel(const __grid_constant__ ConvPsParams p, const int* __restrict__ iter_ptr) {
  using Cfg = ConvPsCfg<KC, N, P, HAS_RES>;
  constexpr int kStages = Cfg::kStages;
  constexpr int KE = TF32 ? KC / 2 : KC;            // channels per chunk
  constexpr int kActDtype = TF32 ? CDS_TF32 : CDS_BF16;      // output: fp32 storage rounded to TF32 / bf16
  extern __shared__ uint8_t smem_raw[];
  __shared__ __align__(8) uint64_t full_bar[kStages];
  __shared__ __align__(8) uint64_t empty_bar[kStages];
  // per-column constants: 0 bias  1 GN gamma  2 GN beta  3 additive time row  4 shortcut bias
  __shared__ __align__(16) float s_col[5][N];

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const uint32_t smem_base = (ptx::smem_u32(smem_raw) + 1023u) & ~1023u;
  uint8_t* smem_al = smem_raw + (smem_base - ptx::smem_u32(smem_raw));
  float* const acc = reinterpret_cast<float*>(smem_al + Cfg::kStagingBytes);    // valid after the main loop
  if (threadIdx.x == 0) { CDS_TRACE(0, gtimer()); CDS_TRACE(1, clock64()); }

  const int tile_b = blockIdx.x / p.n_tiles;          // trajectory tile
  const int n_off = (blockIdx.x % p.n_tiles) * N;     // first output channel of this CTA
  const int b0 = tile_b * 128;
  const int n_main = p.kchunks;
  const int n_chunks = n_main + (HAS_RES ? p.kchunks2 : 0);
  const uint32_t main_bytes = (uint32_t)(P * Cfg::kATile + p.taps * Cfg::kBTile);
  const uint32_t res_bytes = (uint32_t)(P * Cfg::kATile + Cfg::kBTile);

  if (threadIdx.x == 0) {
    // a stage is free again when every consumer warp is done with it (one arrival per warp)
    for (int s = 0; s < kStages; ++s) { ptx::mbar_init(&full_bar[s], 1); ptx::mbar_init(&empty_bar[s], kPsEpiWarps); }
    ptx::fence_barrier_init();
  }
  if (warp == kPsWarpTma && lane == 0) {
    ptx::prefetch_tensormap(&p.tm_a);
    ptx::prefetch_tensormap(&p.tm_b);
    if (HAS_RES) { ptx::prefetch_tensormap(&p.tm_a2); ptx::prefetch_tensormap(&p.tm_b2); }
    if (p.out_tma) ptx::prefetch_tensormap(&p.tm_out);
  }
  __syncthreads();
  if (threadIdx.x == 0) { CDS_TRACE(2, clock64()); ptx::grid_dep_launch_dependents(); }

  if (warp == kPsWarpTma) {
    // ===================================== TMA producer =====================================
    if (ptx::elect_one()) {
      auto load_w = [&](int c, int s) {               // weight tiles of chunk c into stage s
        uint8_t* sb = smem_al + s * Cfg::kStageBytes + P * Cfg::kATile;
        if (!HAS_RES || c < n_main) {
          for (int j = 0; j < p.taps; ++j)
            ptx::tma_load_2d(sb + (p.taps - 1 - j) * Cfg::kBTile, &p.tm_b, &full_bar[s], c * KE, j * p.C_out + n_off);   // slot = taps-1-j
        } else {
          ptx::tma_load_2d(sb, &p.tm_b2, &full_bar[s], (c - n_main) * KE, n_off);
        }
      };
      // weights do not depend on the previous kernel: arm the first ring fill and fetch them before the dependency wait
      const int pre = n_chunks < kStages ? n_chunks : kStages;
      for (int c = 0; c < pre; ++c) {
        ptx::mbar_expect_tx(&full_bar[c], (!HAS_RES || c < n_main) ? main_bytes : res_bytes);
        load_w(c, c);
      }
      ptx::grid_dep_wait();
      const int a_b0 = p.in_batch_mod > 0 ? b0 % p.in_batch_mod : b0;
      const int r_b0 = p.res_batch_mod > 0 ? b0 % p.res_batch_mod : b0;
      for (int c = 0; c < n_chunks; ++c) {
        const int s = c % kStages;
        const bool is_main = !HAS_RES || c < n_main;
        if (c >= pre) {
          ptx::mbar_wait(&empty_bar[s], ((c / kStages) & 1) ^ 1);
          ptx::mbar_expect_tx(&full_bar[s], is_main ? main_bytes : res_bytes);
          load_w(c, s);
        }
        uint8_t* sa = smem_al + s * Cfg::kStageBytes;
        for (int l = 0; l < P; ++l) {
          const void* tm = is_main ? (const void*)&p.tm_a : (const void*)&p.tm_a2;
          const int ck = is_main ? c * KE : (c - n_main) * KE, bb = is_main ? a_b0 : r_b0;
          ptx::tma_load_3d(sa + l * Cfg::kATile, tm, &full_bar[s], ck, l, bb);
        }
      }
      CDS_TRACE(8, clock64());
    }
  } else {
    // ===================================== consumers (warps 0..7) =====================================
    ptx::grid_dep_wait();
    const int iter = iter_ptr ? *iter_ptr : 0;
    {
      const float* bstep = p.bias.step ? p.bias.step + (int64_t)iter * p.bias.step_stride : nullptr;
      const float* hstep = p.shift.step ? p.shift.step + (int64_t)iter * p.shift.step_stride : nullptr;
      for (int n = threadIdx.x; n < N; n += kPsEpiThreads) {
        const int c = n_off + n;
        s_col[0][n] = bstep ? __ldg(bstep + c) : 0.f;
        s_col[1][n] = __ldg(p.gn_gamma + c);
        s_col[2][n] = __ldg(p.gn_beta + c);
        s_col[3][n] = hstep ? __ldg(hstep + c) : 0.f;
        s_col[4][n] = (HAS_RES && p.res_bias) ? __ldg(p.res_bias + c) : 0.f;
      }
    }
    // ---- MMA: warpgroup g accumulates trajectories [64 g, 64 g + 64); D[l'] in registers, shortcut D2[l] next to them
    {
      const int g = warp >> 2;
      float d[P][N / 2];
      float d2[HAS_RES ? P : 1][N / 2];
#pragma unroll
      for (int l = 0; l < P; ++l)
#pragma unroll
        for (int i = 0; i < N / 2; ++i) { d[l][i] = 0.f; d2[HAS_RES ? l : 0][i] = 0.f; }
      for (int c = 0; c < n_chunks; ++c) {
        const int s = c % kStages;
        ptx::mbar_wait(&full_bar[s], (c / kStages) & 1);
        if (c == 0 && threadIdx.x == 0) CDS_TRACE(9, clock64());
        const uint32_t sa = smem_base + s * Cfg::kStageBytes + (uint32_t)(g * 64 * Cfg::kRowBytes);
        const uint32_t sb = smem_base + s * Cfg::kStageBytes + P * Cfg::kATile;
        ptx::wgmma_fence();
        if (!HAS_RES || c < n_main) {
          // input position l feeds output position l' through tap j = l - l' + pad, whose W tile sits in slot taps-1-j
#pragma unroll
          for (int l = 0; l < P; ++l) {
            const uint64_t da = ptx::make_kmajor_desc<Cfg::kRowBytes>(sa + l * Cfg::kATile);
#pragma unroll
            for (int lp = 0; lp < P; ++lp) {
              const int j = l - lp + p.pad;
              if (j < 0 || j >= p.taps) continue;
              const uint64_t db = ptx::make_kmajor_desc<Cfg::kRowBytes>(sb + (p.taps - 1 - j) * Cfg::kBTile);
#pragma unroll
              for (int k = 0; k < KC / 16; ++k) ptx::Wgmma<N, TF32>::mma(d[lp], da + (uint64_t)(2 * k), db + (uint64_t)(2 * k), 1u);
            }
          }
        } else if constexpr (HAS_RES) {
          const uint64_t db = ptx::make_kmajor_desc<Cfg::kRowBytes>(sb);
#pragma unroll
          for (int l = 0; l < P; ++l) {
            const uint64_t da = ptx::make_kmajor_desc<Cfg::kRowBytes>(sa + l * Cfg::kATile);
#pragma unroll
            for (int k = 0; k < KC / 16; ++k) ptx::Wgmma<N, TF32>::mma(d2[l], da + (uint64_t)(2 * k), db + (uint64_t)(2 * k), 1u);
          }
        }
        ptx::wgmma_commit();
        ptx::wgmma_wait<1>();                         // the previous chunk's MMAs are complete: its stage is free
        if (c > 0) { __syncwarp(); if (lane == 0) ptx::mbar_arrive(&empty_bar[(c - 1) % kStages]); }
      }
      ptx::wgmma_wait<0>();
      __syncwarp();
      if (lane == 0) ptx::mbar_arrive(&empty_bar[(n_chunks - 1) % kStages]);
      ptx::named_bar_sync(1, kPsEpiThreads);          // every consumer is done with the ring (and s_col is staged)
      float* const tile = acc + 64 * g * Cfg::kAccPitch;
#pragma unroll
      for (int l = 0; l < P; ++l) {
        ptx::acc_store<N>(tile + l * N, Cfg::kAccPitch, d[l], threadIdx.x & 127);
        if constexpr (HAS_RES) ptx::acc_store<N>(tile + P * N + l * N, Cfg::kAccPitch, d2[l], threadIdx.x & 127);
      }
      ptx::named_bar_sync(1, kPsEpiThreads);          // the accumulator tile is complete
    }
    // ===================================== epilogue =====================================
    // thread = one trajectory (accumulator row) x NH = N/2 columns (ONE GroupNorm group) x all P positions
    constexpr int NH = N / 2;
    static_assert(NH == 16 || NH == 32, "one GroupNorm group of 16 or 32 channels per epilogue column slice");
    const int q = warp & 3, half = warp >> 2;
    const int b = b0 + 32 * q + lane;
    const bool valid = b < p.batch;
    const int col0 = half * NH;                       // CTA-tile column of this thread's slice
    const float* const a_row = acc + (32 * q + lane) * Cfg::kAccPitch;
    const int rb = p.res_batch_mod > 0 ? b % p.res_batch_mod : b;
    if (threadIdx.x == 0) CDS_TRACE(10, clock64());

    // ---- pass 1: GroupNorm statistics of (accumulator + bias) over P positions x NH channels, all in this thread
    float s1 = 0.f, s2 = 0.f;
#pragma unroll
    for (int lp = 0; lp < P; ++lp) {
#pragma unroll
      for (int h = 0; h < NH / 16; ++h) {
        float v[16];
        ptx::acc_ld<16>(a_row + lp * N + col0 + 16 * h, v);
#pragma unroll
        for (int k = 0; k < 4; ++k) {
          const float4 bb = reinterpret_cast<const float4*>(&s_col[0][col0 + 16 * h])[k];
          const float x0 = v[4 * k] + bb.x, x1 = v[4 * k + 1] + bb.y, x2 = v[4 * k + 2] + bb.z, x3 = v[4 * k + 3] + bb.w;
          s1 += (x0 + x1) + (x2 + x3);
          s2 = fmaf(x0, x0, s2); s2 = fmaf(x1, x1, s2); s2 = fmaf(x2, x2, s2); s2 = fmaf(x3, x3, s2);
        }
      }
    }
    const float inv_cnt = 1.f / (float)(P * NH);
    const float mean = s1 * inv_cnt;
    const float ga = rsqrt_ftz(fmaxf(fmaf(s2, inv_cnt, -mean * mean), 0.f) + p.gn_eps);
    const float gc = -mean * ga;

    // ---- pass 2: normalise, affine, Mish, additive terms, store; 16-column chunks
    const bool add_res = p.res != nullptr;
    constexpr int kChunks = P * (NH / 16);
#pragma unroll 1
    for (int ci = 0; ci < kChunks; ++ci) {
      const int lp = ci / (NH / 16), h = ci % (NH / 16);
      const int n0 = col0 + 16 * h;                   // CTA-tile column
      float v[16];
      ptx::acc_ld<16>(a_row + lp * N + n0, v);
      float addv[16];
      const float4* sh4 = reinterpret_cast<const float4*>(&s_col[3][n0]);
#pragma unroll
      for (int k = 0; k < 4; ++k) { const float4 s = sh4[k]; addv[4 * k] = s.x; addv[4 * k + 1] = s.y; addv[4 * k + 2] = s.z; addv[4 * k + 3] = s.w; }
      if (add_res) {
        float resv[16];
#pragma unroll
        for (int j = 0; j < 16; ++j) resv[j] = 0.f;
        if (valid) load_row<16>(p.res, (int64_t)rb * p.res_bstride + (int64_t)lp * p.res_lstride + n_off + n0, kActDtype, resv);
#pragma unroll
        for (int j = 0; j < 16; ++j) addv[j] += resv[j];
      }
      if constexpr (HAS_RES) {
        float r2[16];
        ptx::acc_ld<16>(a_row + P * N + lp * N + n0, r2);
        const float4* rb4 = reinterpret_cast<const float4*>(&s_col[4][n0]);
#pragma unroll
        for (int k = 0; k < 4; ++k) {
          const float4 s = rb4[k];
          addv[4 * k] += r2[4 * k] + s.x; addv[4 * k + 1] += r2[4 * k + 1] + s.y;
          addv[4 * k + 2] += r2[4 * k + 2] + s.z; addv[4 * k + 3] += r2[4 * k + 3] + s.w;
        }
      }
      const float4* b4 = reinterpret_cast<const float4*>(&s_col[0][n0]);
      const float4* ga4 = reinterpret_cast<const float4*>(&s_col[1][n0]);
      const float4* be4 = reinterpret_cast<const float4*>(&s_col[2][n0]);
      float o[16];
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        const float4 bb = b4[k], gm = ga4[k], be = be4[k];
        o[4 * k + 0] = mish_fma(fmaf(fmaf(v[4 * k + 0] + bb.x, ga, gc), gm.x, be.x), addv[4 * k + 0]);
        o[4 * k + 1] = mish_fma(fmaf(fmaf(v[4 * k + 1] + bb.y, ga, gc), gm.y, be.y), addv[4 * k + 1]);
        o[4 * k + 2] = mish_fma(fmaf(fmaf(v[4 * k + 2] + bb.z, ga, gc), gm.z, be.z), addv[4 * k + 2]);
        o[4 * k + 3] = mish_fma(fmaf(fmaf(v[4 * k + 3] + bb.w, ga, gc), gm.w, be.w), addv[4 * k + 3]);
      }
      if (p.out_tma) {
        // 32 trajectories (lanes) x 16 columns of position lp through shared memory and ONE bulk store: a warp-level st.global
        // would touch 32 cache lines per instruction.  The first 16 KB of the idle ring serve as 2 KB of staging rows per warp
        // in the swizzle of tm_out.
        uint8_t* const stg = smem_al + warp * 2048;
        if (lane == 0) ptx::bulk_wait_group_read<0>();
        __syncwarp();
        if constexpr (TF32) {
          uint8_t* const sr = stg + lane * 64;
#pragma unroll
          for (int k = 0; k < 4; ++k)
            *reinterpret_cast<float4*>(sr + ((k ^ ((lane >> 1) & 3)) << 4)) =
                make_float4(round_tf32(o[4 * k]), round_tf32(o[4 * k + 1]), round_tf32(o[4 * k + 2]), round_tf32(o[4 * k + 3]));
        } else {
          uint8_t* const sr = stg + lane * 32;
          const int sw = (lane >> 2) & 1;
          uint32_t w[8];
#pragma unroll
          for (int k = 0; k < 8; ++k) { __nv_bfloat162 h2 = __floats2bfloat162_rn(o[2 * k], o[2 * k + 1]); w[k] = *reinterpret_cast<uint32_t*>(&h2); }
          *reinterpret_cast<uint4*>(sr + ((0 ^ sw) << 4)) = make_uint4(w[0], w[1], w[2], w[3]);
          *reinterpret_cast<uint4*>(sr + ((1 ^ sw) << 4)) = make_uint4(w[4], w[5], w[6], w[7]);
        }
        ptx::fence_proxy_async();
        __syncwarp();
        if (lane == 0) {
          ptx::tma_store_3d(&p.tm_out, stg, n_off + n0, lp, b0 + 32 * q);
          ptx::bulk_commit_group();
        }
      } else if (valid) {
        store_row<16>(p.out, (int64_t)b * p.out_bstride + (int64_t)lp * p.out_lstride + n_off + n0, kActDtype, o);
      }
    }
    if (lane == 0) ptx::bulk_wait_group<0>();        // the bulk stores are complete before the CTA retires
    if (threadIdx.x == 0) { CDS_TRACE(11, clock64()); CDS_TRACE(5, 1LL); }
  }

  __syncthreads();
  if (threadIdx.x == 0) { CDS_TRACE(3, clock64()); CDS_TRACE(4, gtimer()); }
}

// ------------------------------------------------------------------------------------------------ host side
constexpr int kPsPositions = 4;
constexpr int kPsKC = 32;            // channel chunk: 32 (SWIZZLE_64B tiles, 4-stage ring) pipelines better than 64 (2 stages)

// CTA tile width: a quarter of the layer (two GroupNorm groups); 0 = the kernel is not instantiated for this layer
inline int conv_ps_width(const cds_conv_op& c) {
  if (c.C_out == 256) return 64;
  if (c.C_out == 128) return 32;
  return 0;
}

// Can the position-sliced kernel serve this op?  (a subset of conv_tc_eligible: same layouts, same weight packing)
inline bool conv_ps_eligible(const cds_conv_op& c) {
  if (!conv_tc_eligible(c)) return false;
  if (c.L_in != kPsPositions || c.L_out != kPsPositions || c.stride != 1 || c.phases != 1) return false;
  if (c.taps < 1 || c.taps > 5 || (c.taps & 1) == 0 || c.pad != c.taps / 2) return false;
  if (c.groups != 8 || c.act != CDS_ACT_MISH || conv_ps_width(c) == 0) return false;
  if (c.res_w && conv_ps_width(c) > 32) return false;    // 2 x 4 x 64 accumulator columns do not fit over the ring: conv_tc
  if (c.C_in % 64 != 0 || (c.res_w && c.res_C % 64 != 0)) return false;
  if (c.bias.sample || c.scale.step || c.scale.sample || c.shift.sample) return false;
  if (conv_is_tf32(c)) { if (c.out_dtype != CDS_TF32 || (c.res && c.res_dtype == CDS_BF16)) return false; }
  else if (c.out_dtype != CDS_BF16 || (c.res && c.res_dtype != CDS_BF16)) return false;
  if (c.in_batch_mod > 0 && c.in_batch_mod % 128 != 0) return false;
  if (c.res_batch_mod > 0 && c.res_batch_mod % 128 != 0) return false;
  const char* env = getenv("CDS_PS");
  if (env && env[0] == '0') return false;
  return true;
}

struct ConvPsLaunch {
  ConvPsParams prm;
  bool tf32 = false;
  int n = 0;
  bool has_res = false;
  dim3 grid;
};

inline bool conv_ps_prepare(const cds_conv_op& c, ConvPsLaunch* out) {
  ConvPsLaunch& L = *out;
  memset(&L.prm, 0, sizeof(L.prm));
  ConvPsParams& p = L.prm;
  constexpr int kc = kPsKC;
  const bool tf32 = conv_is_tf32(c);
  const int ke = tf32 ? kc / 2 : kc;
  L.tf32 = tf32;
  L.n = conv_ps_width(c);
  L.has_res = c.res_w != nullptr;
  const uint64_t in_b = c.in_batch_mod > 0 ? (uint64_t)c.in_batch_mod : (uint64_t)c.batch;
  {
    uint64_t dims[3] = {(uint64_t)c.C_in, (uint64_t)c.L_in, in_b};
    uint64_t str[2] = {(uint64_t)c.in_lstride, (uint64_t)c.in_bstride};
    uint32_t box[3] = {(uint32_t)ke, 1u, 128u};
    if (!encode_act_map(&p.tm_a, c.in, 3, dims, str, box, kc, tf32)) return false;
  }
  {
    uint64_t dims[2] = {(uint64_t)c.C_in, (uint64_t)c.taps * c.C_out};
    uint64_t str[1] = {(uint64_t)c.C_in};
    uint32_t box[2] = {(uint32_t)ke, (uint32_t)L.n};
    if (!encode_act_map(&p.tm_b, c.w, 2, dims, str, box, kc, tf32)) return false;
  }
  if (L.has_res) {
    const uint64_t r_b = c.res_batch_mod > 0 ? (uint64_t)c.res_batch_mod : (uint64_t)c.batch;
    uint64_t dims[3] = {(uint64_t)c.res_C, (uint64_t)c.L_out, r_b};
    uint64_t str[2] = {(uint64_t)c.res_in_lstride, (uint64_t)c.res_in_bstride};
    uint32_t box[3] = {(uint32_t)ke, 1u, 128u};
    if (!encode_act_map(&p.tm_a2, c.res_in, 3, dims, str, box, kc, tf32)) return false;
    uint64_t d2[2] = {(uint64_t)c.res_C, (uint64_t)c.C_out};
    uint64_t s2[1] = {(uint64_t)c.res_C};
    uint32_t b2[2] = {(uint32_t)ke, (uint32_t)L.n};
    if (!encode_act_map(&p.tm_b2, c.res_w, 2, d2, s2, b2, kc, tf32)) return false;
  }
  p.batch = c.batch; p.C_out = c.C_out; p.taps = c.taps; p.pad = c.pad;
  p.kchunks = c.C_in / ke; p.kchunks2 = L.has_res ? c.res_C / ke : 0;
  p.n_tiles = c.C_out / L.n;
  p.in_batch_mod = c.in_batch_mod; p.res_batch_mod = c.res_batch_mod;
  p.bias = c.bias; p.shift = c.shift;
  p.gn_gamma = c.gn_gamma; p.gn_beta = c.gn_beta; p.gn_eps = c.gn_eps;
  p.res = c.res; p.res_bstride = c.res_bstride; p.res_lstride = c.res_lstride; p.res_bias = c.res_bias;
  p.out = c.out; p.out_bstride = c.out_bstride; p.out_lstride = c.out_lstride;
  {
    const int oes = tf32 ? 4 : 2;
    p.out_tma = 0;
    PFN_encodeTiled enc = get_encode_tiled();
    const bool ok = ((uintptr_t)c.out % 16) == 0 && ((int64_t)c.out_lstride * oes) % 16 == 0 && ((int64_t)c.out_bstride * oes) % 16 == 0 &&
                    !getenv("CDS_NO_TMA_STORE");
    cuuint64_t gdim[3] = {(cuuint64_t)c.C_out, (cuuint64_t)c.L_out, (cuuint64_t)c.batch};
    cuuint64_t gstr[2] = {(cuuint64_t)c.out_lstride * oes, (cuuint64_t)c.out_bstride * oes};
    cuuint32_t bx[3] = {16u, 1u, 32u};
    cuuint32_t es[3] = {1u, 1u, 1u};
    if (ok && enc && enc(&p.tm_out, tf32 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT32 : CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 3, c.out, gdim, gstr, bx, es,
                         CU_TENSOR_MAP_INTERLEAVE_NONE, tf32 ? CU_TENSOR_MAP_SWIZZLE_64B : CU_TENSOR_MAP_SWIZZLE_32B,
                         CU_TENSOR_MAP_L2_PROMOTION_NONE, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS)
      p.out_tma = 1;
  }
  L.grid = dim3((unsigned)(((c.batch + 127) / 128) * p.n_tiles));
  return true;
}

template <int N, bool HAS_RES, bool TF32>
cudaError_t conv_ps_launch_t(const ConvPsLaunch& L, const int* iter_ptr, cudaStream_t st) {
  using Cfg = ConvPsCfg<kPsKC, N, kPsPositions, HAS_RES>;
  static bool attr = false;
  static bool pdl = true;
  if (!attr) {
    cudaError_t e = cudaFuncSetAttribute(conv_ps_kernel<kPsKC, N, kPsPositions, HAS_RES, TF32>,
                                         cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg::kSmemBytes);
    if (e != cudaSuccess) return e;
    if (getenv("CDS_DEBUG"))
      fprintf(stderr, "[cds] conv_ps<%d,%d,%d,%d,%s>: smem %d B\n", kPsKC, N, kPsPositions, (int)HAS_RES,
              TF32 ? "tf32" : "bf16", Cfg::kSmemBytes);
    const char* pdl_env = getenv("CDS_PDL");
    pdl = !(pdl_env && pdl_env[0] == '0');
    attr = true;
  }
  ConvPsParams prm = L.prm;
  prm.trace = conv_tc_trace_hook((int)L.grid.x);
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = L.grid; cfg.blockDim = dim3(kPsThreads); cfg.dynamicSmemBytes = Cfg::kSmemBytes; cfg.stream = st;
  cudaLaunchAttribute at[1];
  int na = 0;
  if (pdl) { at[na].id = cudaLaunchAttributeProgrammaticStreamSerialization; at[na].val.programmaticStreamSerializationAllowed = 1; ++na; }
  cfg.attrs = at; cfg.numAttrs = na;
  return cudaLaunchKernelEx(&cfg, conv_ps_kernel<kPsKC, N, kPsPositions, HAS_RES, TF32>, prm, iter_ptr);
}
template <int N, bool HAS_RES, bool TF32>
cudaError_t conv_ps_preload_t() {
  cudaFuncAttributes a;
  return cudaFuncGetAttributes(&a, conv_ps_kernel<kPsKC, N, kPsPositions, HAS_RES, TF32>);
}

// X(N, HAS_RES, TF32) over every instantiation
#define CDS_PS_VARIANTS(X)                                                                   \
  X(32, false, false) X(32, true, false) X(64, false, false)                                \
  X(32, false, true) X(32, true, true) X(64, false, true)

#ifndef CDS_PS_INSTANTIATE
#define CDS_PS_EXTERN(N_, R_, T_)                                                                                 \
  extern template cudaError_t conv_ps_launch_t<N_, R_, T_>(const ConvPsLaunch&, const int*, cudaStream_t);        \
  extern template cudaError_t conv_ps_preload_t<N_, R_, T_>();
CDS_PS_VARIANTS(CDS_PS_EXTERN)
#undef CDS_PS_EXTERN

inline cudaError_t conv_ps_launch(const ConvPsLaunch& L, const int* iter_ptr, cudaStream_t st) {
#define CDS_PS_CASE(N_, R_, T_) if (L.n == N_ && L.has_res == R_ && L.tf32 == T_) return conv_ps_launch_t<N_, R_, T_>(L, iter_ptr, st);
  CDS_PS_VARIANTS(CDS_PS_CASE)
#undef CDS_PS_CASE
  return cudaErrorInvalidValue;
}
inline cudaError_t conv_ps_preload_all() {
  cudaError_t e;
#define CDS_PS_PRE(N_, R_, T_) if ((e = conv_ps_preload_t<N_, R_, T_>()) != cudaSuccess) return e;
  CDS_PS_VARIANTS(CDS_PS_PRE)
#undef CDS_PS_PRE
  return cudaSuccess;
}
#endif

}  // namespace cds
