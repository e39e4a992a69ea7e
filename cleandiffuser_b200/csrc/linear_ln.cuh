// Fused  Linear -> gate * (.) + residual -> LayerNorm + adaLN modulate  for DiT1d's token stream (TF32 tensor-core programs).
//
//   X[r, :] = (A[r, :] W^T + bias) * gate[traj(r), :] + R[r, :]                   (dit.py:33-36: x + gate * f(...))
//        or = (A[r, :] W^T + bias) + T[r mod L, :]                                (dit.py:118: x_proj(x) + pos_emb, T a (L, C) table)
//   Y[r, :] = LayerNorm(X[r, :]) * (1 + scale[traj(r), :]) + shift[traj(r), :]    (dit.py:30-31 of the NEXT block / final layer)
//
// It replaces, at plan-finalize time, a CDS_OP_CONV in its "gated" form directly followed by the CDS_OP_LNMOD that reads its
// output (cds_api.cu: fuse_linear_ln) -- the ABI and the lowering do not know about it.  Why a kernel of its own:
//   * LayerNorm needs the whole row, so one CTA owns all C = 2 * NH output columns of its 128 rows: two consumer warpgroups
//     (rows [0, 64) / [64, 128)) issue two wgmma (N = NH) per 32-byte K step into register accumulators for the column halves
//     [0, NH) and [NH, 2 NH); the activation chunk is staged ONCE for both halves (the generic kernel's 160-wide column tiles
//     re-fetch it per tile), which is what the L2-feed-bound TF32 main loop cares about;
//   * the separate LayerNorm launch (read X, write Y: 8 bytes per element of HBM traffic, ~230 us per call at cfg4's size)
//     disappears: X never leaves the SM between the two.
// Once a tile's MMAs have read their operands, the accumulators are written as a 128 x C fp32 tile over the operand ring (the
// ring is idle then: the producer is held back by the tile's last ring stages, which are handed back only after pass 1).
// Epilogue, the same 8 warps (accumulator row quarter q = warp & 3, column half hh = warp >> 2), two passes over the thread's
// NH columns; the ring is released after the FIRST one, so the producer fetches the next tile's operands during the second:
//   1. x = (acc + bias) * gate + residual.  The residual arrives by TMA, 16 columns x 32 rows per warp and request, one request
//      ahead (a thread walking its own 1280-byte-pitch row with ld.global costs 13 us per tile: scripts/micro/store_patterns.cu
//      v5 is the store-side twin of that pattern); x is computed IN PLACE in that buffer and bulk-stored from it to X; row moments
//      about a pivot (the row's first x: no cancellation), the two halves' (mean, M2) combine exactly in shared memory
//   2. the x chunks come back by TMA from the X just written (L2 hits; each request waits for the completion of that chunk's
//      store): y = (x - mean) * rstd * (1 + scale) + shift, in place, bulk-stored to Y (rounded to TF32 when Y feeds a Linear)
// Algorithmic HBM bytes per row: 4 K (A) + 4 C (R) + 4 C (X) + 4 C (Y);  flops per row: 2 K C.
#pragma once
#include "conv_tc.cuh"

namespace cds {

constexpr int kLlThreads = 288;                      // warps 0-7 MMA (two warpgroups) + epilogue, warp 8 TMA producer
constexpr int kLlEpiThreads = 256;
constexpr int kLlAhead = 4;                          // steps between the request of a per-trajectory vector chunk and its use

struct LinLnParams {
  CUtensorMap tm_a, tm_b, tm_x, tm_y, tm_r, tm_rp, tm_xl;   // tm_xl: X as a load source (pass 2 re-reads what pass 1 stored)   // tm_rp: the residual again, box {NH, 32}, for L2 prefetches
  int rows, K, C, L;                                 // L = tokens per trajectory
  const float* bias; int64_t bias_step_stride;       // bias row of iteration i = bias + i * stride
  const float* gate; int64_t gate_stride;            // per trajectory; nullptr: no gate (table form)
  int table_period;                                  // > 0: the residual is a (period, C) TABLE indexed by row % period (x_proj + pos_emb)
  int a_row_mod;                                     // > 0: the activation rows repeat with this period (CFG branches share x_t)
  const float* res; int64_t res_stride;              // (rows, C), elements
  const float* shift; const float* scale; int64_t mod_stride;
  float eps;
  int x_dtype, y_dtype;
  int num_tiles;
};

struct LinLnLaunch {
  bool ok = false;
  LinLnParams prm;
  int nh = 0, smem_bytes = 0;
};

template <int NH>
struct LinLnCfg {
  static constexpr int kStages = NH <= 160 ? 3 : 2;
  static constexpr int kStageA = 128 * 128;                           // 128 rows x 32 fp32
  static constexpr int kStageB = 2 * NH * 128;                        // 2 NH weight rows x 32 fp32
  static constexpr int kStage = kStageA + kStageB;
  static constexpr int kStaging = 8 * 3 * 2048;                       // per epilogue warp: three buffers of 32 rows x 16 fp32
  static constexpr int kSmemBytes = kStages * kStage + kStaging + 1024;
  static constexpr int kAccPitch = 2 * NH + 4;                        // accumulator tile row (floats), padded against bank conflicts
  static_assert(kStages * kStage >= 128 * kAccPitch * 4, "the accumulator tile must fit over the operand ring");
  static_assert(NH % 16 == 0 && NH >= 16 && NH <= 256, "column half");
  static_assert((NH * 128) % 1024 == 0, "the second weight half must start on a swizzle atom");
};

template <int NH>
__global__ void __launch_bounds__(kLlThreads, 1) linear_ln_kernel(const __grid_constant__ LinLnParams p, const int* __restrict__ iter_ptr) {
  using Cfg = LinLnCfg<NH>;
  constexpr int C = 2 * NH;
  extern __shared__ uint8_t ll_smem_raw[];
  __shared__ __align__(8) uint64_t full_bar[Cfg::kStages], empty_bar[Cfg::kStages];
  __shared__ __align__(16) float s_bias[C];
  __shared__ float s_red[2][2][2][128];            // [tile parity][mean | M2][column half][row]
  __shared__ __align__(8) uint64_t res_bar[8][3];
  const uint32_t base_u = (ptx::smem_u32(ll_smem_raw) + 1023u) & ~1023u;
  uint8_t* sm = ll_smem_raw + (base_u - ptx::smem_u32(ll_smem_raw));
  uint8_t* s_stage = sm + Cfg::kStages * Cfg::kStage;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int n_k = p.K >> 5;                            // 32-channel chunks

  if (threadIdx.x == 0) {
    // a stage is free again when every consumer warp is done with it (one arrival per warp)
    for (int s = 0; s < Cfg::kStages; ++s) { ptx::mbar_init(&full_bar[s], 1); ptx::mbar_init(&empty_bar[s], kLlEpiThreads / 32); }
    for (int w = 0; w < 8; ++w) for (int j = 0; j < 3; ++j) ptx::mbar_init(&res_bar[w][j], 1);
    ptx::fence_barrier_init();
    ptx::prefetch_tensormap(&p.tm_a); ptx::prefetch_tensormap(&p.tm_b);
    ptx::prefetch_tensormap(&p.tm_x); ptx::prefetch_tensormap(&p.tm_y); ptx::prefetch_tensormap(&p.tm_r); ptx::prefetch_tensormap(&p.tm_xl);
  }
  __syncthreads();
  float* const acc = reinterpret_cast<float*>(sm);     // accumulator tile over the operand ring: 128 rows x kAccPitch floats
  ptx::grid_dep_wait();                                // (no-op unless launched with a programmatic dependency)

  if (warp == 8) {                                     // ------------------------------------------------ producer
    if (lane == 0) {
      uint32_t n = 0;
      for (int tile = blockIdx.x; tile < p.num_tiles; tile += gridDim.x) {
        for (int kc = 0; kc < n_k; ++kc, ++n) {
          const int s = n % Cfg::kStages;
          ptx::mbar_wait(&empty_bar[s], ((n / Cfg::kStages) & 1u) ^ 1u);
          uint8_t* a = sm + s * Cfg::kStage;
          ptx::mbar_expect_tx(&full_bar[s], (uint32_t)Cfg::kStage);
          ptx::tma_load_2d(a, &p.tm_a, &full_bar[s], kc * 32, p.a_row_mod > 0 ? (tile * 128) % p.a_row_mod : tile * 128);
          ptx::tma_load_2d(a + Cfg::kStageA, &p.tm_b, &full_bar[s], kc * 32, 0);
          ptx::tma_load_2d(a + Cfg::kStageA + NH * 128, &p.tm_b, &full_bar[s], kc * 32, NH);
        }
      }
    }
  } else {                                             // ------------------------------------------------ epilogue (warps 0..7)
    const int q = warp & 3, hh = warp >> 2;
    const int m = 32 * q + lane;
    // ---- MMA of one tile: warpgroup hh accumulates rows [64 hh, 64 hh + 64) x all C columns in registers, then acc <- them
    uint32_t n = 0;                                    // k-blocks consumed so far (ring position)
    uint32_t n_tile0 = 0;                              // ... at the start of the current tile
    auto mma_tile = [&]() {
      float d0[NH / 2], d1[NH / 2];
#pragma unroll
      for (int i = 0; i < NH / 2; ++i) { d0[i] = 0.f; d1[i] = 0.f; }
      n_tile0 = n;
      for (int kc = 0; kc < n_k; ++kc, ++n) {
        const int s = n % Cfg::kStages;
        ptx::mbar_wait(&full_bar[s], (n / Cfg::kStages) & 1u);
        const uint32_t a = base_u + (uint32_t)(s * Cfg::kStage);
        const uint64_t da = ptx::make_kmajor_desc<128>(a + (uint32_t)(hh * 64 * 128));
        const uint64_t db0 = ptx::make_kmajor_desc<128>(a + Cfg::kStageA);
        const uint64_t db1 = ptx::make_kmajor_desc<128>(a + Cfg::kStageA + NH * 128);
        ptx::wgmma_fence();
#pragma unroll
        for (int k = 0; k < 4; ++k) {
          ptx::Wgmma<NH, true>::mma(d0, da + (uint64_t)(2 * k), db0 + (uint64_t)(2 * k), 1u);
          ptx::Wgmma<NH, true>::mma(d1, da + (uint64_t)(2 * k), db1 + (uint64_t)(2 * k), 1u);
        }
        ptx::wgmma_commit();
        ptx::wgmma_wait<1>();
        // the previous k-block's stage goes back to the producer, unless it is one of the tile's last kStages k-blocks: those
        // stages are where the accumulator tile goes (handed back after pass 1)
        if (kc >= 1 && kc - 1 < n_k - Cfg::kStages) { __syncwarp(); if (lane == 0) ptx::mbar_arrive(&empty_bar[(n - 1) % Cfg::kStages]); }
      }
      ptx::wgmma_wait<0>();
      ptx::named_bar_sync(2, kLlEpiThreads);           // both warpgroups' MMAs have read the ring
      ptx::acc_store<NH>(acc + 64 * hh * Cfg::kAccPitch, Cfg::kAccPitch, d0, threadIdx.x & 127);
      ptx::acc_store<NH>(acc + 64 * hh * Cfg::kAccPitch + NH, Cfg::kAccPitch, d1, threadIdx.x & 127);
      ptx::named_bar_sync(2, kLlEpiThreads);           // the accumulator tile is complete
    };
    // after pass 1 of every warp: the withheld stages (the accumulator tile) go back to the producer
    auto release_ring = [&]() {
      ptx::fence_proxy_async();                        // generic writes of the tile before the TMA unit refills the ring
      __syncwarp();
      if (lane == 0)
        for (int j = n_k - Cfg::kStages; j < n_k; ++j) ptx::mbar_arrive(&empty_bar[(n_tile0 + (uint32_t)j) % Cfg::kStages]);
    };
    for (int i = threadIdx.x; i < C; i += kLlEpiThreads) s_bias[i] = p.bias[(int64_t)(*iter_ptr) * p.bias_step_stride + i];
    ptx::named_bar_sync(1, kLlEpiThreads);
    // three rotating 2 KB buffers per warp (32 rows x 16 fp32, SWIZZLE_64B).  Use number u works in buffer u % 3: a 16-column
    // chunk is TMA-LOADED into it (pass 1: the residual, pass 2: the x just stored; chunks 0..2 up front, then two uses ahead),
    // the result is computed in place and TMA-stored from it (pass 1: X, pass 2: Y).  A buffer is reloaded only after the
    // store issued from it has read it.
    uint8_t* const stg = s_stage + warp * 6144;
    const int sw = (lane >> 1) & 3;
    const uint32_t lane_off = (uint32_t)lane * 64u;
    const float* const a_row = acc + m * Cfg::kAccPitch + hh * NH;
    const float inv_c = 1.f / (float)C;
    uint64_t* const rbar = &res_bar[warp][0];
    uint32_t t = 0, u = 0, par = 0;                    // tiles done, buffer uses, phase bit of each buffer's load barrier
    for (int tile = blockIdx.x; tile < p.num_tiles; tile += gridDim.x, ++t) {
      mma_tile();
      const int64_t grow = (int64_t)tile * 128 + m;
      const int row0 = tile * 128 + 32 * q;
      // Per-trajectory vectors (gate in pass 1; scale, shift in pass 2).  A warp's 32 rows touch at most two trajectories (L >= 32):
      // lanes 0-15 fetch 16 consecutive elements of the first one's vector, lanes 16-31 of the second one's -- ONE coalesced load
      // per vector and step, issued kLlAhead steps before its use and handed out by shuffles.  (A thread loading its own copy made
      // every 16-column step wait for an L2 / HBM round trip: ncu put 11 % of all stall samples on the first use of `scale`.)
      const int64_t last_traj = ((int64_t)p.rows - 1) / p.L;
      const int64_t traj_a = min((int64_t)row0 / p.L, last_traj);
      const int64_t traj = min(grow / p.L, last_traj);
      const int sel = traj != traj_a ? 16 : 0;          // which half of the warp holds this row's values
      const int64_t traj_ld = (lane < 16) ? traj_a : min(traj_a + 1, last_traj);
      const bool gated = p.gate != nullptr;
      const bool table = p.table_period > 0;
      const float* gate_ld = gated ? p.gate + traj_ld * p.gate_stride + hh * NH + (lane & 15) : p.scale;   // (never read when !gated)
      const float* scp_ld = p.scale + traj_ld * p.mod_stride + hh * NH + (lane & 15);
      const float* shp_ld = p.shift + traj_ld * p.mod_stride + hh * NH + (lane & 15);
      float gq[kLlAhead], aq[kLlAhead], dq[kLlAhead];
#pragma unroll
      for (int j = 0; j < kLlAhead; ++j) aq[j] = dq[j] = 0.f;
#pragma unroll
      for (int j = 0; j < kLlAhead; ++j) gq[j] = (gated && j < NH / 16) ? __ldg(gate_ld + 16 * j) : 1.f;
      // table form: this thread's table row (row % period), two 16-column chunks ahead in registers (the table is small and hot
      // in L2; a thread walks its own row, so the requests are issued early rather than wide)
      const float* trow = table ? p.res + (int64_t)((grow < p.rows ? grow : 0) % p.table_period) * p.res_stride + hh * NH : p.res;
      float4 rq[2][4];
#pragma unroll
      for (int j = 0; j < 2; ++j)
#pragma unroll
        for (int k = 0; k < 4; ++k) rq[j][k] = table ? __ldg(reinterpret_cast<const float4*>(trow + 16 * j) + k) : make_float4(0.f, 0.f, 0.f, 0.f);
      if (lane == 0 && !table) {                       // residual chunks 0..2: in flight while the main loop runs
        ptx::bulk_wait_group_read<0>();
#pragma unroll
        for (int j = 0; j < 3; ++j) {
          if (j < NH / 16) {
            const uint32_t bj = (u + j) % 3;
            ptx::mbar_expect_tx(&rbar[bj], 2048u);
            ptx::tma_load_2d(stg + bj * 2048, &p.tm_r, &rbar[bj], hh * NH + 16 * j, row0);
          }
        }
        // ... and the next tile's residual rows of this warp are pulled into L2 (they were written several launches ago)
        const int nt = tile + (int)gridDim.x;
        if (nt < p.num_tiles) ptx::tma_prefetch_2d(&p.tm_rp, hh * NH, nt * 128 + 32 * q);   // (residual form only: see the guard above)
      }
      // ---- pass 1: x = (acc + bias) * gate + residual -> X; shifted row moments
      float sh0 = 0.f, sd = 0.f, sdd = 0.f;            // pivot (the row's first x of this half), sum (x - pivot), sum (x - pivot)^2
#pragma unroll 1
      for (int ch = 0; ch < NH / 16; ++ch, ++u) {
        const uint32_t b = u % 3;
        uint8_t* const buf = stg + b * 2048;
        const float gcur = gq[0];
#pragma unroll
        for (int j = 0; j + 1 < kLlAhead; ++j) gq[j] = gq[j + 1];
        gq[kLlAhead - 1] = (gated && ch + kLlAhead < NH / 16) ? __ldg(gate_ld + 16 * (ch + kLlAhead)) : 1.f;
#pragma unroll
        for (int j = 0; j + 1 < kLlAhead; ++j) { aq[j] = aq[j + 1]; dq[j] = dq[j + 1]; }
        if (ch + kLlAhead >= NH / 16) {                // pass 2's first kLlAhead chunks are requested by pass 1's last steps
          const int j2 = ch + kLlAhead - NH / 16;
          aq[kLlAhead - 1] = __ldg(scp_ld + 16 * j2); dq[kLlAhead - 1] = __ldg(shp_ld + 16 * j2);
        }
        float v[16];
        ptx::acc_ld<16>(a_row + 16 * ch, v);
        float4 rt[4];
        if (table) {
#pragma unroll
          for (int k = 0; k < 4; ++k) { rt[k] = rq[0][k]; rq[0][k] = rq[1][k]; }
          if (ch + 2 < NH / 16) {
#pragma unroll
            for (int k = 0; k < 4; ++k) rq[1][k] = __ldg(reinterpret_cast<const float4*>(trow + 16 * (ch + 2)) + k);
          }
          if (lane == 0) ptx::bulk_wait_group_read<2>();        // the store issued from this buffer three uses ago has read it
          __syncwarp();
        } else {
          ptx::mbar_wait(&rbar[b], (par >> b) & 1u);
          par ^= 1u << b;
        }
        const float4* b4 = reinterpret_cast<const float4*>(&s_bias[hh * NH + 16 * ch]);
#pragma unroll
        for (int k = 0; k < 4; ++k) {
          const float4 bb = b4[k];
          const float4 r = table ? rt[k] : *reinterpret_cast<const float4*>(buf + lane_off + ((k ^ sw) << 4));
          v[4 * k] = fmaf(v[4 * k] + bb.x, __shfl_sync(0xffffffffu, gcur, sel + 4 * k), r.x);
          v[4 * k + 1] = fmaf(v[4 * k + 1] + bb.y, __shfl_sync(0xffffffffu, gcur, sel + 4 * k + 1), r.y);
          v[4 * k + 2] = fmaf(v[4 * k + 2] + bb.z, __shfl_sync(0xffffffffu, gcur, sel + 4 * k + 2), r.z);
          v[4 * k + 3] = fmaf(v[4 * k + 3] + bb.w, __shfl_sync(0xffffffffu, gcur, sel + 4 * k + 3), r.w);
        }
        if (ch == 0) sh0 = v[0];
#pragma unroll
        for (int j = 0; j < 16; ++j) { const float d = v[j] - sh0; sd += d; sdd = fmaf(d, d, sdd); }
#pragma unroll
        for (int k = 0; k < 4; ++k) {                  // x over the residual it came from (same thread, same bytes)
          float4 o4;
          if (p.x_dtype == CDS_TF32) o4 = make_float4(round_tf32(v[4 * k]), round_tf32(v[4 * k + 1]), round_tf32(v[4 * k + 2]), round_tf32(v[4 * k + 3]));
          else o4 = make_float4(v[4 * k], v[4 * k + 1], v[4 * k + 2], v[4 * k + 3]);
          *reinterpret_cast<float4*>(buf + lane_off + ((k ^ sw) << 4)) = o4;
        }
        if (!table && ch >= 1 && ch + 2 < NH / 16 && lane == 0) {
          // the buffer of the previous step is free once its X store has read it (issued a whole step ago): residual chunk
          // ch + 2 goes there, two steps ahead of its use
          const uint32_t bp = (u + 2) % 3;
          ptx::bulk_wait_group_read<0>();
          ptx::mbar_expect_tx(&rbar[bp], 2048u);
          ptx::tma_load_2d(stg + bp * 2048, &p.tm_r, &rbar[bp], hh * NH + 16 * (ch + 2), row0);
        }
        ptx::fence_proxy_async();
        __syncwarp();
        if (lane == 0) {
          ptx::tma_store_2d(&p.tm_x, buf, hh * NH + 16 * ch, row0);
          ptx::bulk_commit_group();
        }
      }
      // this half's (mean, M2) from the shifted moments; the two halves combine exactly (Chan et al.): M2 = M2a + M2b + d^2 n / 2
      {
        const float mh = sd * (1.f / (float)NH);
        s_red[t & 1][0][hh][m] = sh0 + mh;
        s_red[t & 1][1][hh][m] = fmaf(-sd, mh, sdd);
      }
      // X chunks 0..2 come back (from L2) into the three buffers: their stores must have COMPLETED (written), every store must
      // have read its buffer.  Committed groups of this thread at this point: ..., X(0) .. X(NCH-1).
      if (lane == 0) {
        ptx::bulk_wait_group_read<0>();
        ptx::bulk_wait_group<NH / 16 - 3>();
#pragma unroll
        for (int j = 0; j < 3; ++j) {
          const uint32_t bj = (u + j) % 3;
          ptx::mbar_expect_tx(&rbar[bj], 2048u);
          ptx::tma_load_2d(stg + bj * 2048, &p.tm_xl, &rbar[bj], hh * NH + 16 * j, row0);
        }
      }
      ptx::named_bar_sync(1, kLlEpiThreads);
      release_ring();                                  // every warp has read its accumulator rows
      const float ma = s_red[t & 1][0][0][m], mb = s_red[t & 1][0][1][m];
      const float mean = 0.5f * (ma + mb);
      const float m2 = s_red[t & 1][1][0][m] + s_red[t & 1][1][1][m] + (mb - ma) * (mb - ma) * (0.5f * (float)NH);
      const float rstd = rsqrtf(fmaxf(m2, 0.f) * inv_c + p.eps);
      // (s_red is double-buffered by tile parity: a warp may be a whole pass ahead of another one, never two tiles)
      // ---- pass 2: x (re-read from X, 16 columns x 32 rows per request, two steps ahead) -> normalise, modulate in place -> Y
#pragma unroll 1
      for (int ch = 0; ch < NH / 16; ++ch, ++u) {
        const uint32_t b = u % 3;
        uint8_t* const buf = stg + b * 2048;
        const float acur = aq[0], dcur = dq[0];
#pragma unroll
        for (int j = 0; j + 1 < kLlAhead; ++j) { aq[j] = aq[j + 1]; dq[j] = dq[j + 1]; }
        if (ch + kLlAhead < NH / 16) { aq[kLlAhead - 1] = __ldg(scp_ld + 16 * (ch + kLlAhead)); dq[kLlAhead - 1] = __ldg(shp_ld + 16 * (ch + kLlAhead)); }
        ptx::mbar_wait(&rbar[b], (par >> b) & 1u);
        par ^= 1u << b;
#pragma unroll
        for (int k = 0; k < 4; ++k) {
          const float4 x = *reinterpret_cast<const float4*>(buf + lane_off + ((k ^ sw) << 4));
          float4 o4;
          o4.x = fmaf((x.x - mean) * rstd, 1.f + __shfl_sync(0xffffffffu, acur, sel + 4 * k), __shfl_sync(0xffffffffu, dcur, sel + 4 * k));
          o4.y = fmaf((x.y - mean) * rstd, 1.f + __shfl_sync(0xffffffffu, acur, sel + 4 * k + 1), __shfl_sync(0xffffffffu, dcur, sel + 4 * k + 1));
          o4.z = fmaf((x.z - mean) * rstd, 1.f + __shfl_sync(0xffffffffu, acur, sel + 4 * k + 2), __shfl_sync(0xffffffffu, dcur, sel + 4 * k + 2));
          o4.w = fmaf((x.w - mean) * rstd, 1.f + __shfl_sync(0xffffffffu, acur, sel + 4 * k + 3), __shfl_sync(0xffffffffu, dcur, sel + 4 * k + 3));
          if (p.y_dtype == CDS_TF32) o4 = make_float4(round_tf32(o4.x), round_tf32(o4.y), round_tf32(o4.z), round_tf32(o4.w));
          *reinterpret_cast<float4*>(buf + lane_off + ((k ^ sw) << 4)) = o4;
        }
        if (ch >= 1 && ch + 2 < NH / 16 && lane == 0) {
          // X chunk ch + 2 into the previous step's buffer: that step's Y store has read it; the X store of chunk ch + 2 is complete
          // when at most (NCH - 1 - (ch + 2)) + ch = NCH - 3 younger groups are pending
          const uint32_t bp = (u + 2) % 3;
          ptx::bulk_wait_group_read<0>();
          ptx::bulk_wait_group<NH / 16 - 3>();
          ptx::mbar_expect_tx(&rbar[bp], 2048u);
          ptx::tma_load_2d(stg + bp * 2048, &p.tm_xl, &rbar[bp], hh * NH + 16 * (ch + 2), row0);
        }
        ptx::fence_proxy_async();
        __syncwarp();
        if (lane == 0) {
          ptx::tma_store_2d(&p.tm_y, buf, hh * NH + 16 * ch, row0);
          ptx::bulk_commit_group();
        }
      }
    }
    if (lane == 0) ptx::bulk_wait_group<0>();
  }
  ptx::grid_dep_launch_dependents();
  __syncthreads();
}

// ------------------------------------------------------------------------------------------------ host side
// Can the pair (conv, lnmod) run as one linear_ln launch?  conv: TF32 tensor-core Linear over flattened tokens in its gated form
// out = (acc + bias) * gate(trajectory) + res; lnmod: reads exactly that output, one row per token.
inline int linear_ln_pick_nh(int c_out) {
  // C = 256 only: each warpgroup holds 64 rows x C fp32 accumulators in registers, and a 9-warp CTA gets at most 168
  // registers per thread -- wider rows spill and run slower than the two-launch form, which serves them
  switch (c_out) { case 256: return 128; default: return 0; }
}
inline bool linear_ln_eligible(const cds_conv_op& c, const cds_lnmod_op& l) {
  { const char* e = getenv("CDS_FUSE_LN"); if (e && e[0] == '0') return false; }      // (read at every finalize: tests toggle it)
  if (c.math != CDS_MATH_TF32_TC || linear_ln_pick_nh(c.C_out) == 0) return false;
  if (c.taps != 1 || c.stride != 1 || c.pad != 0 || c.phases != 1 || c.L_in != 1 || c.L_out != 1) return false;
  if (c.C_in % 32 != 0 || c.C_in < 32 * 3 || c.groups != 0 || c.act != CDS_ACT_NONE) return false;   // (>= kStages k-blocks)
  if (c.in_batch_mod < 0 || c.in_batch_mod % 128 != 0) return false;        // (CFG branches sharing x_t: whole 128-row tiles repeat)
  if (c.in_dtype == CDS_BF16 || c.out_dtype == CDS_BF16 || c.res_dtype == CDS_BF16) return false;
  if (c.in_bstride != c.C_in || c.out_bstride != c.C_out) return false;                       // dense rows
  if (!c.bias.step || c.bias.sample) return false;
  if (c.scale.step || c.shift.step || c.shift.sample) return false;
  if (!c.res || c.res_w || c.res_bstride % 4 != 0) return false;
  // two forms: gated + dense residual (out-projection, second MLP Linear) / no gate + periodic table (x_proj + pos_emb)
  const bool gated_form = c.scale.sample && c.res_batch_mod == 0;
  const bool table_form = !c.scale.sample && c.res_batch_mod > 0 && c.res_batch_mod == c.sample_row_div;
  if (!gated_form && !table_form) return false;
  if (c.sample_row_div < 32) return false;             // (a warp's 32 rows then span at most two trajectories)
  if (gated_form && (c.scale.sample_stride % 4 != 0 || ((uintptr_t)c.scale.sample % 16))) return false;
  if (((uintptr_t)c.res % 16) || ((uintptr_t)c.bias.step % 4)) return false;
  if (((uintptr_t)c.in % 16) || ((uintptr_t)c.w % 16) || ((uintptr_t)c.out % 16)) return false;
  // the LayerNorm that follows
  if (l.in != c.out || l.C != c.C_out || (int64_t)l.batch * l.L != (int64_t)c.batch || l.L != c.sample_row_div) return false;
  if (l.out_dtype == CDS_BF16 || !l.out || ((uintptr_t)l.out % 16)) return false;
  if (l.mod_bstride % 4 != 0 || ((uintptr_t)l.shift % 16) || ((uintptr_t)l.scale % 16)) return false;
  return true;
}

inline bool linear_ln_encode_2d(CUtensorMap* m, const void* base, uint64_t inner, uint64_t outer, uint64_t row_stride_bytes, uint32_t box_inner,
                                uint32_t box_outer, CUtensorMapSwizzle sw) {
  PFN_encodeTiled enc = get_encode_tiled();
  if (!enc) return false;
  cuuint64_t gdim[2] = {inner, outer};
  cuuint64_t gstr[1] = {row_stride_bytes};
  cuuint32_t bx[2] = {box_inner, box_outer};
  cuuint32_t es[2] = {1u, 1u};
  return enc(m, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2, const_cast<void*>(base), gdim, gstr, bx, es, CU_TENSOR_MAP_INTERLEAVE_NONE, sw,
             CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
}

inline bool linear_ln_prepare(const cds_conv_op& c, const cds_lnmod_op& l, LinLnLaunch* out) {
  LinLnLaunch& L = *out;
  L.ok = false;
  LinLnParams& p = L.prm;
  memset(&p, 0, sizeof(p));
  L.nh = linear_ln_pick_nh(c.C_out);
  p.rows = c.batch; p.K = c.C_in; p.C = c.C_out; p.L = c.sample_row_div;
  p.bias = c.bias.step; p.bias_step_stride = c.bias.step_stride;
  p.gate = c.scale.sample; p.gate_stride = c.scale.sample_stride;
  p.table_period = c.res_batch_mod; p.a_row_mod = c.in_batch_mod;
  p.res = reinterpret_cast<const float*>(c.res); p.res_stride = c.res_bstride;
  p.shift = l.shift; p.scale = l.scale; p.mod_stride = l.mod_bstride;
  p.eps = l.eps; p.x_dtype = c.out_dtype; p.y_dtype = l.out_dtype;
  p.num_tiles = (c.batch + 127) / 128;
  const uint64_t a_rows = c.in_batch_mod > 0 ? (uint64_t)c.in_batch_mod : (uint64_t)c.batch;
  const uint64_t r_rows = c.res_batch_mod > 0 ? (uint64_t)c.res_batch_mod : (uint64_t)c.batch;      // (table form: the maps are not used)
  if (!linear_ln_encode_2d(&p.tm_a, c.in, (uint64_t)c.C_in, a_rows, (uint64_t)c.C_in * 4, 32, 128, CU_TENSOR_MAP_SWIZZLE_128B)) return false;
  if (!linear_ln_encode_2d(&p.tm_b, c.w, (uint64_t)c.C_in, (uint64_t)c.C_out, (uint64_t)c.C_in * 4, 32, (uint32_t)L.nh, CU_TENSOR_MAP_SWIZZLE_128B)) return false;
  if (!linear_ln_encode_2d(&p.tm_x, c.out, (uint64_t)c.C_out, (uint64_t)c.batch, (uint64_t)c.C_out * 4, 16, 32, CU_TENSOR_MAP_SWIZZLE_64B)) return false;
  if (!linear_ln_encode_2d(&p.tm_r, c.res, (uint64_t)c.C_out, r_rows, (uint64_t)c.res_bstride * 4, 16, 32, CU_TENSOR_MAP_SWIZZLE_64B)) return false;
  if (!linear_ln_encode_2d(&p.tm_rp, c.res, (uint64_t)c.C_out, r_rows, (uint64_t)c.res_bstride * 4, (uint32_t)L.nh, 32, CU_TENSOR_MAP_SWIZZLE_NONE)) return false;
  p.tm_xl = p.tm_x;
  if (!linear_ln_encode_2d(&p.tm_y, l.out, (uint64_t)c.C_out, (uint64_t)c.batch, (uint64_t)c.C_out * 4, 16, 32, CU_TENSOR_MAP_SWIZZLE_64B)) return false;
  L.ok = true;
  return true;
}

typedef void (*LinLnKernel)(const LinLnParams, const int*);
inline LinLnKernel linear_ln_kernel_for(int nh, int* smem) {
  switch (nh) {
#define CDS_LL(N) case N: *smem = LinLnCfg<N>::kSmemBytes; return linear_ln_kernel<N>;
    CDS_LL(128)
#undef CDS_LL
    default: return nullptr;
  }
}
inline cudaError_t linear_ln_preload_all() {
  for (int nh : {128}) {
    int smem = 0;
    LinLnKernel k = linear_ln_kernel_for(nh, &smem);
    cudaError_t e = cudaFuncSetAttribute(reinterpret_cast<const void*>(k), cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
    if (e != cudaSuccess) return e;
  }
  return cudaSuccess;
}
inline cudaError_t linear_ln_launch(const LinLnLaunch& L, const int* iter_ptr, int sm_count, cudaStream_t st) {
  int smem = 0;
  LinLnKernel k = linear_ln_kernel_for(L.nh, &smem);
  if (!k) return cudaErrorInvalidValue;
  int grid = sm_count > 0 ? sm_count : 132;
  if (grid > L.prm.num_tiles) grid = L.prm.num_tiles;
  k<<<grid, kLlThreads, smem, st>>>(L.prm, iter_ptr);
  return cudaGetLastError();
}

}  // namespace cds
