// libcds: C ABI (include/cds.h) over the sm_90a kernels.  Plans, validation, CUDA-graph replay.
#include <cuda_runtime.h>

#include <cstdarg>
#include <cstdio>
#include <cstring>
#include <string>
#include <vector>

#include "cds.h"
#include "attention.cuh"
#include "conv_simt.cuh"
#include "conv_tc.cuh"
#include "conv_ps.cuh"
#include "attention_tma.cuh"
#include "elementwise.cuh"
#include "mha.cuh"

namespace {

thread_local std::string g_err;

int fail(int code, const char* fmt, ...) {
  char buf[512];
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(buf, sizeof buf, fmt, ap);
  va_end(ap);
  g_err = buf;
  return code;
}

#define CDS_CUDA(call)                                                                                  \
  do {                                                                                                  \
    cudaError_t e__ = (call);                                                                           \
    if (e__ != cudaSuccess) return fail(CDS_ERR_CUDA, "%s failed: %s", #call, cudaGetErrorString(e__)); \
  } while (0)

// Makes `device` current for the lifetime of the guard and restores the caller's device afterwards: a plan may live on a
// GPU that is not the calling thread's current one (multi-GPU processes), and PyTorch's notion of "current device" must not
// change under the caller.
struct DeviceGuard {
  int prev = -1;
  cudaError_t err = cudaSuccess;
  explicit DeviceGuard(int device) {
    err = cudaGetDevice(&prev);
    if (err == cudaSuccess && prev != device) err = cudaSetDevice(device);
    else if (err == cudaSuccess) prev = -1;          // nothing to restore
  }
  ~DeviceGuard() { if (prev >= 0) cudaSetDevice(prev); }
};
#define CDS_ON_DEVICE(dev)                                                                                       \
  DeviceGuard guard__(dev);                                                                                      \
  if (guard__.err != cudaSuccess) return fail(CDS_ERR_CUDA, "cudaSetDevice(%d) failed: %s", (int)(dev), cudaGetErrorString(guard__.err))

struct Step {            // one validated operator + its kernel choice
  cds_op op;
  int conv_bn = 0;
  bool tc = false;       // tensor-core conv: tensor maps + launch geometry prepared at append time
  cds::ConvTcLaunch tcl;
  int branch = 0;        // (op.flags >> 8) & 0xff
  bool ps = false;       // ... served by the position-sliced kernel (short sequences, conv_ps.cuh)
  cds::ConvPsLaunch psl;
  int attn_family = 0, attn_param = 0;   // attention: attn_pick's kernel family and template parameter
  int mha_hpl = 0;       // CDS_OP_MHA: head_dim / 32 (mha_pick)
  cds::AttnTmaLaunch attl;   // TF32 attention: tensor maps of the persistent TMA-fed kernel (attention_tma.cuh)
};

int elementwise_grid(int64_t total, int sm_count) {
  int64_t blocks = (total + 255) / 256;
  int64_t cap = (int64_t)sm_count * 8;     // grid sized in multiples of the SM count; grid-stride loop inside
  return (int)(blocks < cap ? (blocks > 0 ? blocks : 1) : cap);
}

// The kernel family of a conv op (CDS_CONV_SIMT / _TC / _PS) and, for conv_simt, its tile width: every check of validate()
// except the null-pointer ones, so that cds_conv_choice answers for descriptors whose buffers do not exist yet.
int conv_pick(const cds_conv_op& c, int* family, int* bn) {
  if (c.batch <= 0 || c.L_in <= 0 || c.L_out <= 0 || c.C_in <= 0 || c.C_out <= 0 || c.taps <= 0 ||
      c.stride <= 0 || c.phases <= 0)
    return fail(CDS_ERR_INVALID, "conv: non-positive geometry");
  if (c.groups > 8) return fail(CDS_ERR_UNSUPPORTED, "conv: more than 8 GroupNorm groups");
  if (c.res_w && c.res_C <= 0) return fail(CDS_ERR_INVALID, "conv: shortcut conv without input");
  if (c.res_w && (c.stride != 1 || c.phases != 1)) return fail(CDS_ERR_INVALID, "conv: shortcut conv needs stride 1");
  *bn = 0;
  if (c.math == CDS_MATH_BF16_TC || c.math == CDS_MATH_TF32_TC) {
    if (!cds::conv_tc_eligible(c))
      return fail(CDS_ERR_INVALID, "conv: op is not eligible for the tensor-core kernel (ask cds_conv_tc_supported)");
    *family = cds::conv_ps_eligible(c) ? CDS_CONV_PS : CDS_CONV_TC;
    return CDS_OK;
  }
  if (c.math != CDS_MATH_FP32) return fail(CDS_ERR_UNSUPPORTED, "conv: math mode %d unknown", c.math);
  if (c.sample_row_div > 1) return fail(CDS_ERR_UNSUPPORTED, "conv: sample_row_div needs the tensor-core kernel");
  *bn = cds::conv_simt_pick_bn(c);
  if (*bn == 0)
    return fail(CDS_ERR_UNSUPPORTED, "conv: GroupNorm tile does not fit (L_out=%d C_out=%d groups=%d)", c.L_out,
                c.C_out, c.groups);
  *family = CDS_CONV_SIMT;
  return CDS_OK;
}

// The kernel family of an attention op (CDS_ATTN_*) and its template parameter (HD of the fp32 kernel, NT = ceil(L / 8) of the
// TMA kernel, else 0): every check of validate() except the null-pointer ones.  Reads the alignment of qkv and out, never the
// memory, so that cds_attn_choice answers for descriptors whose buffers do not exist yet.
int attn_pick(const cds_attn_op& a, int* family, int* param) {
  if (a.batch <= 0 || a.L <= 0 || a.heads <= 0 || a.C % a.heads != 0) return fail(CDS_ERR_INVALID, "attn: bad arguments");
  const int hd = a.C / a.heads;
  if (hd != 16 && hd != 32 && hd != 64) return fail(CDS_ERR_UNSUPPORTED, "attn: head_dim %d", hd);
  if ((size_t)a.L * hd * 8 > 200 * 1024) return fail(CDS_ERR_UNSUPPORTED, "attn: L=%d too long", a.L);
  const uintptr_t qkv = (uintptr_t)a.qkv, out = (uintptr_t)a.out;
  *param = 0;
  if (a.qkv_dtype == CDS_BF16) {
    if (hd != 32 || a.L > cds::kAttnMaxL || a.C % 8 != 0 || qkv % 16 != 0)
      return fail(CDS_ERR_UNSUPPORTED, "attn: bf16 q/k/v needs head_dim 32, L <= %d, 16-byte aligned rows", cds::kAttnMaxL);
    *family = CDS_ATTN_BF16_MMA;
    return CDS_OK;
  }
  // fp32 storage rounded to TF32 (TF32 tensor-core programs): mma.sync tf32 when the shape allows -- fed by TMA when out is
  // 16-byte aligned as well --, else the fp32 kernel
  const bool tf32_mma = a.qkv_dtype == CDS_TF32 && hd == 32 && a.L <= cds::kAttnMaxL && a.C % 4 == 0 && qkv % 16 == 0 &&
                        a.out_dtype != CDS_BF16 && out % 8 == 0;
  if (tf32_mma && out % 16 == 0 && cds::attention_tma_enabled()) {
    *family = CDS_ATTN_TF32_TMA;
    *param = (a.L + 7) / 8;
  } else if (tf32_mma) {
    *family = CDS_ATTN_TF32_MMA;
  } else {
    *family = CDS_ATTN_F32;
    *param = hd;
  }
  return CDS_OK;
}

bool is_act_dtype(int d) { return d == CDS_F32 || d == CDS_TF32 || d == CDS_BF16; }

// The instantiation of mha_f32_kernel for a CDS_OP_MHA op: every check of validate() except the null-pointer ones, so that
// cds_mha_choice answers for descriptors whose buffers do not exist yet.
int mha_pick(const cds_mha_op& m, int* hpl) {
  if (m.batch <= 0 || m.Lq <= 0 || m.Lk <= 0 || m.heads <= 0 || m.C <= 0 || m.C % m.heads != 0)
    return fail(CDS_ERR_INVALID, "mha: bad arguments");
  if (!is_act_dtype(m.in_dtype) || !is_act_dtype(m.out_dtype)) return fail(CDS_ERR_INVALID, "mha: unknown dtype");
  const int hd = m.C / m.heads;
  if (hd % 32 != 0 || hd > 32 * cds::kMhaMaxHPL) return fail(CDS_ERR_UNSUPPORTED, "mha: head_dim %d", hd);
  if (m.Lq > cds::kMhaMaxL || m.Lk > cds::kMhaMaxL)
    return fail(CDS_ERR_UNSUPPORTED, "mha: Lq=%d Lk=%d (at most %d)", m.Lq, m.Lk, cds::kMhaMaxL);
  *hpl = hd / 32;
  return CDS_OK;
}

int validate(const cds_op& op, Step* out) {
  out->op = op;
  out->branch = (op.flags & CDS_OPF_BRANCH_MASK) >> CDS_OPF_BRANCH_SHIFT;
  switch (op.kind) {
    case CDS_OP_CONV: {
      const cds_conv_op& c = op.u.conv;
      if (!c.in || !c.w || !c.out) return fail(CDS_ERR_INVALID, "conv: null in/w/out");
      if (c.groups > 0 && (!c.gn_gamma || !c.gn_beta)) return fail(CDS_ERR_INVALID, "conv: GroupNorm without affine");
      if (c.res_w && !c.res_in) return fail(CDS_ERR_INVALID, "conv: shortcut conv without input");
      int family = 0;
      int rc = conv_pick(c, &family, &out->conv_bn);
      if (rc != CDS_OK) return rc;
      if (family == CDS_CONV_PS) {
        if (!cds::conv_ps_prepare(c, &out->psl))
          return fail(CDS_ERR_CUDA, "conv: cuTensorMapEncodeTiled failed (position-sliced, C_in=%d C_out=%d)", c.C_in, c.C_out);
        out->tc = out->ps = true;
      } else if (family == CDS_CONV_TC) {
        if (!cds::conv_tc_prepare(c, &out->tcl))
          return fail(CDS_ERR_CUDA, "conv: cuTensorMapEncodeTiled failed (C_in=%d L=%d C_out=%d)", c.C_in, c.L_in, c.C_out);
        out->tc = true;
      }
      return CDS_OK;
    }
    case CDS_OP_UPDATE: {
      const cds_update_op& u = op.u.update;
      if (u.batch <= 0 || u.row <= 0 || !u.x || !u.pred || !u.coef) return fail(CDS_ERR_INVALID, "update: bad arguments");
      if (u.mask && !u.prior) return fail(CDS_ERR_INVALID, "update: mask without prior");
      if (u.aux && !u.xhat_prev) return fail(CDS_ERR_INVALID, "update: aux history without xhat_prev");
      if (u.x_cast && (u.cast_C_in <= 0 || u.cast_C_out < u.cast_C_in || u.row % u.cast_C_in != 0))
        return fail(CDS_ERR_INVALID, "update: bad x_cast geometry");
      return CDS_OK;
    }
    case CDS_OP_LNMOD: {
      const cds_lnmod_op& l = op.u.lnmod;
      if (l.batch <= 0 || l.L <= 0 || l.C <= 0 || !l.in || !l.out || !l.shift || !l.scale)
        return fail(CDS_ERR_INVALID, "lnmod: bad arguments");
      return CDS_OK;
    }
    case CDS_OP_ATTN: {
      const cds_attn_op& a = op.u.attn;
      if (!a.qkv || !a.out) return fail(CDS_ERR_INVALID, "attn: bad arguments");
      int rc = attn_pick(a, &out->attn_family, &out->attn_param);
      if (rc != CDS_OK) return rc;
      if (out->attn_family == CDS_ATTN_TF32_TMA && !cds::attention_tma_prepare(a, &out->attl))
        return fail(CDS_ERR_CUDA, "attn: cuTensorMapEncodeTiled failed (L=%d C=%d)", a.L, a.C);
      return CDS_OK;
    }
    case CDS_OP_MHA: {
      const cds_mha_op& m = op.u.mha;
      if (!m.q || (!m.kv_step && !m.kv_sample) || !m.out) return fail(CDS_ERR_INVALID, "mha: null q, k|v or out");
      return mha_pick(m, &out->mha_hpl);
    }
    case CDS_OP_PREP: {
      const cds_prep_op& p = op.u.prep;
      if (p.batch <= 0 || p.row <= 0 || !p.x || !p.xin || !p.coef) return fail(CDS_ERR_INVALID, "prep: bad arguments");
      return CDS_OK;
    }
    case CDS_OP_CAST: {
      const cds_cast_op& k = op.u.cast;
      if (k.batch <= 0 || k.L <= 0 || k.C_in <= 0 || k.C_out < k.C_in || (k.C_out & 1) || !k.in || !k.out ||
          (k.out_dtype != CDS_F32 && k.out_dtype != CDS_BF16 && k.out_dtype != CDS_TF32))
        return fail(CDS_ERR_INVALID, "cast: bad arguments");
      return CDS_OK;
    }
    default:
      return fail(CDS_ERR_INVALID, "unknown operator kind %d", op.kind);
  }
}

int launch(const Step& s, const int* iter_ptr, int sm_count, cudaStream_t st, int* advance = nullptr) {
  switch (s.op.kind) {
    case CDS_OP_CONV:
      if (s.ps) CDS_CUDA(cds::conv_ps_launch(s.psl, iter_ptr, st));
      else if (s.tc) CDS_CUDA(cds::conv_tc_launch(s.tcl, iter_ptr, st));
      else CDS_CUDA(cds::conv_simt_launch(s.op.u.conv, s.conv_bn, iter_ptr, st));
      return CDS_OK;
    case CDS_OP_UPDATE: {
      const cds_update_op& u = s.op.u.update;
      cds::solver_update_kernel<<<elementwise_grid((int64_t)u.batch * u.row, sm_count), 256, 0, st>>>(u, iter_ptr, advance);
      CDS_CUDA(cudaGetLastError());
      return CDS_OK;
    }
    case CDS_OP_PREP: {
      const cds_prep_op& p = s.op.u.prep;
      cds::cm_prep_kernel<<<elementwise_grid((int64_t)p.batch * p.row, sm_count), 256, 0, st>>>(p, iter_ptr);
      CDS_CUDA(cudaGetLastError());
      return CDS_OK;
    }
    case CDS_OP_LNMOD: {
      const cds_lnmod_op& l = s.op.u.lnmod;
      int64_t rows = (int64_t)l.batch * l.L;
      int64_t blocks = (rows + 7) / 8;
      int64_t cap = (int64_t)sm_count * 8;
      cds::ln_modulate_kernel<<<(int)(blocks < cap ? blocks : cap), 256, 0, st>>>(l);
      CDS_CUDA(cudaGetLastError());
      return CDS_OK;
    }
    case CDS_OP_ATTN:
      if (s.attn_family == CDS_ATTN_TF32_TMA) CDS_CUDA(cds::attention_tma_launch(s.op.u.attn, s.attl, s.attn_param, sm_count, st));
      else CDS_CUDA(cds::attention_launch(s.op.u.attn, s.attn_family, s.attn_param, st));
      return CDS_OK;
    case CDS_OP_MHA:
      CDS_CUDA(cds::mha_launch(s.op.u.mha, s.mha_hpl, iter_ptr, st));
      return CDS_OK;
    case CDS_OP_CAST: {
      const cds_cast_op& k = s.op.u.cast;
      cds::cast_pad_kernel<<<elementwise_grid((int64_t)k.batch * k.L * (k.C_out / 2), sm_count), 256, 0, st>>>(k);
      CDS_CUDA(cudaGetLastError());
      return CDS_OK;
    }
  }
  return fail(CDS_ERR_INVALID, "unknown operator kind");
}

// Touch every kernel once so that lazy module loading never happens inside a stream capture.
int preload_kernels() {
  cudaFuncAttributes a;
  CDS_CUDA(cudaFuncGetAttributes(&a, cds::conv_gemm_f32_kernel<32>));
  CDS_CUDA(cudaFuncGetAttributes(&a, cds::conv_gemm_f32_kernel<64>));
  CDS_CUDA(cudaFuncGetAttributes(&a, cds::conv_gemm_f32_kernel<128>));
  CDS_CUDA(cds::conv_tc_preload_all());
  CDS_CUDA(cds::conv_ps_preload_all());
  CDS_CUDA(cudaFuncGetAttributes(&a, cds::attention_f32_kernel<16>));
  CDS_CUDA(cudaFuncGetAttributes(&a, cds::attention_f32_kernel<32>));
  CDS_CUDA(cudaFuncGetAttributes(&a, cds::attention_f32_kernel<64>));
  CDS_CUDA(cudaFuncGetAttributes(&a, cds::attention_mma_hd32_kernel));
  CDS_CUDA(cudaFuncGetAttributes(&a, cds::attention_mma_tf32_hd32_kernel));
  CDS_CUDA(cds::attention_tma_preload_all());
  CDS_CUDA(cds::mha_preload_all());
  CDS_CUDA(cudaFuncGetAttributes(&a, cds::solver_update_kernel));
  CDS_CUDA(cudaFuncGetAttributes(&a, cds::cm_prep_kernel));
  CDS_CUDA(cudaFuncGetAttributes(&a, cds::cast_pad_kernel));
  CDS_CUDA(cudaFuncGetAttributes(&a, cds::ln_modulate_kernel));
  CDS_CUDA(cudaFuncGetAttributes(&a, cds::set_iter_kernel));
  CDS_CUDA(cudaFuncGetAttributes(&a, cds::advance_iter_kernel));
  return CDS_OK;
}

}  // namespace

// ---- debug timeline of one tensor-core conv launch (cds_debug_trace)
namespace cds {
static long long* g_trace_buf = nullptr;
static int64_t g_trace_cap = 0;       // entries
static int g_trace_target = -1, g_trace_count = 0, g_trace_grid = 0;
long long* conv_tc_trace_hook(int grid) {
  if (!g_trace_buf) return nullptr;
  const int ord = g_trace_count++;
  if (ord != g_trace_target || (int64_t)grid * kTraceSlots > g_trace_cap) return nullptr;
  g_trace_grid = grid;
  return g_trace_buf;
}
}  // namespace cds

// CDS_OP_MHA was added without a layout change: the union keeps its size
static_assert(sizeof(cds_mha_op) <= sizeof(cds_conv_op), "cds_mha_op must not grow the cds_op union");

struct cds_plan {
  int device = 0;
  int sm_count = 0;
  int n_iters = 0;
  bool finalized = false;
  std::vector<Step> steps;
  int* d_iter = nullptr;
  cudaStream_t cap_stream = nullptr;
  cudaGraph_t graph = nullptr;
  cudaGraphExec_t exec = nullptr;
  // the same program unrolled `multi` times in ONE graph (CDS_GRAPH_ITERS, default 10): fewer graph launches per run
  int multi = 0;
  // parallel branches (cds_op.flags bits 8..15): branch b > 0 is enqueued on side[b-1], forked from / joined to the caller's
  // stream with events once per iteration
  int n_branches = 1;
  std::vector<cudaStream_t> side;
  cudaEvent_t ev_fork = nullptr;
  std::vector<cudaEvent_t> ev_join;
  cudaGraph_t graph_multi = nullptr;
  cudaGraphExec_t exec_multi = nullptr;
};

extern "C" {

int cds_version(void) { return CDS_ABI_VERSION; }
int cds_op_size(void) { return (int)sizeof(cds_op); }
const char* cds_last_error(void) { return g_err.c_str(); }

int cds_conv_tc_supported(const cds_conv_op* op) {
  if (!op) return 0;
  cds_conv_op c = *op;
  if (c.math != CDS_MATH_TF32_TC) c.math = CDS_MATH_BF16_TC;
  return cds::conv_tc_eligible(c) ? 1 : 0;
}

int cds_conv_choice(const cds_conv_op* op, int32_t info[8]) {
  if (!op || !info) return fail(CDS_ERR_INVALID, "conv_choice: null argument");
  const cds_conv_op& c = *op;
  int family = 0, bn = 0;
  int rc = conv_pick(c, &family, &bn);
  if (rc != CDS_OK) return rc;
  for (int i = 0; i < 8; ++i) info[i] = 0;
  info[0] = family;
  if (family == CDS_CONV_TC) {
    const cds::ConvTcShape s = cds::conv_tc_shape(c);
    info[1] = s.kc; info[2] = s.n; info[3] = s.split; info[4] = s.col_tiles;
  } else if (family == CDS_CONV_PS) {
    info[1] = cds::kPsKC; info[2] = cds::conv_ps_width(c); info[3] = 1; info[4] = 1;
  } else {
    info[2] = bn;
    return CDS_OK;
  }
  info[5] = c.res_w ? 1 : 0;
  info[6] = cds::conv_is_tf32(c) ? 1 : 0;
  return CDS_OK;
}

int cds_attn_choice(const cds_attn_op* op, int32_t info[4]) {
  if (!op || !info) return fail(CDS_ERR_INVALID, "attn_choice: null argument");
  int family = 0, param = 0;
  int rc = attn_pick(*op, &family, &param);
  if (rc != CDS_OK) return rc;
  const int hd = op->C / op->heads;
  info[0] = family;
  info[1] = param;
  info[2] = hd;
  info[3] = family == CDS_ATTN_F32 ? (int)(sizeof(float) * 2 * (size_t)op->L * hd)
          : family == CDS_ATTN_TF32_TMA ? cds::attention_tma_smem_bytes(op->L) : 0;
  return CDS_OK;
}

int cds_mha_choice(const cds_mha_op* op, int32_t info[2]) {
  if (!op || !info) return fail(CDS_ERR_INVALID, "mha_choice: null argument");
  int hpl = 0;
  int rc = mha_pick(*op, &hpl);
  if (rc != CDS_OK) return rc;
  info[0] = hpl;
  info[1] = op->in_dtype == CDS_BF16 ? 1 : 0;
  return CDS_OK;
}

int cds_device_sm_count(int device) {
  int n = 0;
  if (cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, device) != cudaSuccess) return -1;
  return n;
}

int cds_plan_create(int device, cds_plan** out) {
  if (!out) return fail(CDS_ERR_INVALID, "plan_create: null out");
  int n_dev = 0;
  CDS_CUDA(cudaGetDeviceCount(&n_dev));
  if (device < 0 || device >= n_dev) return fail(CDS_ERR_INVALID, "plan_create: device %d of %d", device, n_dev);
  cds_plan* p = new cds_plan();
  p->device = device;
  p->sm_count = cds_device_sm_count(device);
  *out = p;
  return CDS_OK;
}

int cds_plan_destroy(cds_plan* p) {
  if (!p) return CDS_OK;
  DeviceGuard guard(p->device);
  if (p->exec) cudaGraphExecDestroy(p->exec);
  if (p->graph) cudaGraphDestroy(p->graph);
  if (p->exec_multi) cudaGraphExecDestroy(p->exec_multi);
  if (p->graph_multi) cudaGraphDestroy(p->graph_multi);
  if (p->cap_stream) cudaStreamDestroy(p->cap_stream);
  for (cudaStream_t s : p->side) cudaStreamDestroy(s);
  if (p->ev_fork) cudaEventDestroy(p->ev_fork);
  for (cudaEvent_t e : p->ev_join) cudaEventDestroy(e);
  if (p->d_iter) cudaFree(p->d_iter);
  delete p;
  return CDS_OK;
}

int cds_plan_append(cds_plan* p, const cds_op* ops, int32_t n_ops) {
  if (!p || (!ops && n_ops > 0)) return fail(CDS_ERR_INVALID, "plan_append: null argument");
  if (p->finalized) return fail(CDS_ERR_STATE, "plan_append after finalize");
  for (int i = 0; i < n_ops; ++i) {
    Step s;
    int rc = validate(ops[i], &s);
    if (rc != CDS_OK) {
      std::string inner = g_err;
      return fail(rc, "op %d: %s", (int)p->steps.size(), inner.c_str());
    }
    p->steps.push_back(s);
  }
  return CDS_OK;
}

int cds_plan_finalize(cds_plan* p, int32_t n_iters) {
  if (!p) return fail(CDS_ERR_INVALID, "plan_finalize: null plan");
  if (p->finalized) return fail(CDS_ERR_STATE, "plan already finalized");
  if (n_iters <= 0 || p->steps.empty()) return fail(CDS_ERR_INVALID, "plan_finalize: empty program");
  CDS_ON_DEVICE(p->device);
  { int rc = preload_kernels(); if (rc != CDS_OK) return rc; }
  CDS_CUDA(cudaMalloc(&p->d_iter, 2 * sizeof(int)));      // [0] iteration counter, [1] finished-block count of the update
  CDS_CUDA(cudaMemset(p->d_iter, 0, 2 * sizeof(int)));
  CDS_CUDA(cudaStreamCreateWithFlags(&p->cap_stream, cudaStreamNonBlocking));
  p->n_iters = n_iters;
  for (const Step& s : p->steps) if (s.branch + 1 > p->n_branches) p->n_branches = s.branch + 1;
  if (p->n_branches > 1) {
    CDS_CUDA(cudaEventCreateWithFlags(&p->ev_fork, cudaEventDisableTiming));
    for (int b = 1; b < p->n_branches; ++b) {
      cudaStream_t s; cudaEvent_t e;
      CDS_CUDA(cudaStreamCreateWithFlags(&s, cudaStreamNonBlocking));
      CDS_CUDA(cudaEventCreateWithFlags(&e, cudaEventDisableTiming));
      p->side.push_back(s); p->ev_join.push_back(e);
    }
    // the branches share the machine: one CTA per SM and kernel, so that kernels of different branches co-reside
    for (Step& s : p->steps) if (s.tc && !s.ps) s.tcl.max_ctas_per_sm = 1;
  }
  p->finalized = true;
  return CDS_OK;
}

// the iteration counter is advanced by the program's last operator when that is a solver update (fused), else by a
// one-thread kernel
static bool advance_fused(const cds_plan* p) {
  if (p->n_branches > 1) return false;             // several updates per iteration: a one-thread kernel advances after the join
  for (int i = (int)p->steps.size() - 1; i >= 0; --i)
    if (!(p->steps[i].op.flags & CDS_OPF_ONCE)) return p->steps[i].op.kind == CDS_OP_UPDATE;
  return false;
}

static int enqueue_once(cds_plan* p, cudaStream_t st) {
  for (const Step& s : p->steps) {
    if (!(s.op.flags & CDS_OPF_ONCE)) continue;
    int rc = launch(s, p->d_iter, p->sm_count, st);
    if (rc != CDS_OK) return rc;
  }
  return CDS_OK;
}

static int enqueue_iteration(cds_plan* p, cudaStream_t st) {
  const bool fused = advance_fused(p);
  if (p->n_branches == 1) {
    int last = -1;
    for (int i = 0; i < (int)p->steps.size(); ++i) if (!(p->steps[i].op.flags & CDS_OPF_ONCE)) last = i;
    for (int i = 0; i < (int)p->steps.size(); ++i) {
      const Step& s = p->steps[i];
      if (s.op.flags & CDS_OPF_ONCE) continue;
      int rc = launch(s, p->d_iter, p->sm_count, st, (fused && i == last) ? p->d_iter : nullptr);
      if (rc != CDS_OK) return rc;
    }
  } else {
    // fork: every side stream waits for the caller's stream; launch the branches round-robin (so that direct launches
    // interleave like the graph branches do); join: the caller's stream waits for every side stream
    CDS_CUDA(cudaEventRecord(p->ev_fork, st));
    for (cudaStream_t s : p->side) CDS_CUDA(cudaStreamWaitEvent(s, p->ev_fork, 0));
    std::vector<std::vector<int>> per(p->n_branches);
    for (int i = 0; i < (int)p->steps.size(); ++i) {
      const Step& s = p->steps[i];
      if (!(s.op.flags & CDS_OPF_ONCE)) per[s.branch].push_back(i);
    }
    for (size_t k = 0;; ++k) {
      bool any = false;
      for (int b = 0; b < p->n_branches; ++b) {
        if (k >= per[b].size()) continue;
        any = true;
        int rc = launch(p->steps[per[b][k]], p->d_iter, p->sm_count, b == 0 ? st : p->side[b - 1], nullptr);
        if (rc != CDS_OK) return rc;
      }
      if (!any) break;
    }
    for (int b = 1; b < p->n_branches; ++b) {
      CDS_CUDA(cudaEventRecord(p->ev_join[b - 1], p->side[b - 1]));
      CDS_CUDA(cudaStreamWaitEvent(st, p->ev_join[b - 1], 0));
    }
  }
  if (!fused) {
    cds::advance_iter_kernel<<<1, 1, 0, st>>>(p->d_iter);
    CDS_CUDA(cudaGetLastError());
  }
  return CDS_OK;
}

int cds_plan_run(cds_plan* p, int32_t first, int32_t count, void* stream, int32_t use_graph) {
  if (!p || !p->finalized) return fail(CDS_ERR_STATE, "plan_run before finalize");
  if (first < 0 || count < 0 || first + count > p->n_iters)
    return fail(CDS_ERR_INVALID, "plan_run: iterations [%d, %d) outside [0, %d)", first, first + count, p->n_iters);
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  CDS_ON_DEVICE(p->device);
  if (use_graph && !p->exec) {
    // capture on a private stream (the caller's may be the legacy default stream, which cannot capture);
    // capture itself never executes anything.
    CDS_CUDA(cudaStreamBeginCapture(p->cap_stream, cudaStreamCaptureModeThreadLocal));
    int rc = enqueue_iteration(p, p->cap_stream);
    cudaError_t e = cudaStreamEndCapture(p->cap_stream, &p->graph);
    if (rc != CDS_OK) return rc;
    if (e != cudaSuccess) return fail(CDS_ERR_CUDA, "graph capture failed: %s", cudaGetErrorString(e));
    CDS_CUDA(cudaGraphInstantiate(&p->exec, p->graph, 0));
    const char* gi = getenv("CDS_GRAPH_ITERS");
    p->multi = gi ? atoi(gi) : 10;
    if (p->multi > 1 && p->multi <= p->n_iters) {
      CDS_CUDA(cudaStreamBeginCapture(p->cap_stream, cudaStreamCaptureModeThreadLocal));
      int rc2 = CDS_OK;
      for (int k = 0; k < p->multi && rc2 == CDS_OK; ++k) rc2 = enqueue_iteration(p, p->cap_stream);
      cudaError_t e2 = cudaStreamEndCapture(p->cap_stream, &p->graph_multi);
      if (rc2 != CDS_OK) return rc2;
      if (e2 != cudaSuccess) return fail(CDS_ERR_CUDA, "graph capture (x%d) failed: %s", p->multi, cudaGetErrorString(e2));
      CDS_CUDA(cudaGraphInstantiate(&p->exec_multi, p->graph_multi, 0));
    } else {
      p->multi = 0;
    }
  }
  cds::set_iter_kernel<<<1, 1, 0, st>>>(p->d_iter, first);
  CDS_CUDA(cudaGetLastError());
  { int rc = enqueue_once(p, st); if (rc != CDS_OK) return rc; }
  for (int i = 0; i < count; ++i) {
    if (use_graph && p->exec_multi && count - i >= p->multi) {
      CDS_CUDA(cudaGraphLaunch(p->exec_multi, st));
      i += p->multi - 1;
    } else if (use_graph) {
      CDS_CUDA(cudaGraphLaunch(p->exec, st));
    } else {
      int rc = enqueue_iteration(p, st);
      if (rc != CDS_OK) return rc;
    }
  }
  return CDS_OK;
}

int cds_plan_run_range(cds_plan* p, int32_t iter, int32_t op_first, int32_t op_count, void* stream) {
  if (!p || !p->finalized) return fail(CDS_ERR_STATE, "plan_run_range before finalize");
  if (iter < 0 || iter >= p->n_iters) return fail(CDS_ERR_INVALID, "plan_run_range: iteration %d outside [0, %d)", iter, p->n_iters);
  if (op_first < 0 || op_count < 0 || op_first + op_count > (int)p->steps.size())
    return fail(CDS_ERR_INVALID, "plan_run_range: operators [%d, %d) outside [0, %d)", op_first, op_first + op_count, (int)p->steps.size());
  if (p->n_branches > 1) return fail(CDS_ERR_UNSUPPORTED, "plan_run_range: programs with parallel branches run whole iterations only");
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  CDS_ON_DEVICE(p->device);
  cds::set_iter_kernel<<<1, 1, 0, st>>>(p->d_iter, iter);
  CDS_CUDA(cudaGetLastError());
  for (int i = op_first; i < op_first + op_count; ++i) {
    const Step& s = p->steps[i];
    if (s.op.flags & CDS_OPF_ONCE) continue;
    int rc = launch(s, p->d_iter, p->sm_count, st);
    if (rc != CDS_OK) return rc;
  }
  return CDS_OK;
}

int cds_plan_profile(cds_plan* p, int32_t iter, void* stream, float* ms_per_op, int32_t n_ops) {
  if (!p || !p->finalized) return fail(CDS_ERR_STATE, "plan_profile before finalize");
  if (!ms_per_op || n_ops != (int)p->steps.size()) return fail(CDS_ERR_INVALID, "plan_profile: n_ops != %d", (int)p->steps.size());
  if (iter < 0 || iter >= p->n_iters) return fail(CDS_ERR_INVALID, "plan_profile: bad iteration");
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  CDS_ON_DEVICE(p->device);
  std::vector<cudaEvent_t> ev(2 * n_ops);
  for (auto& e : ev) CDS_CUDA(cudaEventCreate(&e));
  cds::set_iter_kernel<<<1, 1, 0, st>>>(p->d_iter, iter);
  for (int pass = 0; pass < 2; ++pass) {           // pass 0: the CDS_OPF_ONCE operators, pass 1: the iteration program
    for (int i = 0; i < n_ops; ++i) {
      const bool once = (p->steps[i].op.flags & CDS_OPF_ONCE) != 0;
      if (once != (pass == 0)) continue;
      CDS_CUDA(cudaEventRecord(ev[2 * i], st));
      int rc = launch(p->steps[i], p->d_iter, p->sm_count, st);
      if (rc != CDS_OK) return rc;
      CDS_CUDA(cudaEventRecord(ev[2 * i + 1], st));
    }
  }
  CDS_CUDA(cudaStreamSynchronize(st));
  for (int i = 0; i < n_ops; ++i) CDS_CUDA(cudaEventElapsedTime(&ms_per_op[i], ev[2 * i], ev[2 * i + 1]));
  for (auto& e : ev) cudaEventDestroy(e);
  return CDS_OK;
}

int cds_plan_launches_per_iter(const cds_plan* p) {
  if (!p) return 0;
  int n = advance_fused(p) ? 0 : 1;
  for (const Step& s : p->steps) if (!(s.op.flags & CDS_OPF_ONCE)) ++n;
  return n;
}

int cds_debug_trace(void* device_buffer, int64_t capacity_entries, int32_t target_launch) {
  cds::g_trace_buf = reinterpret_cast<long long*>(device_buffer);
  cds::g_trace_cap = capacity_entries;
  cds::g_trace_target = target_launch;
  cds::g_trace_count = 0;
  int g = cds::g_trace_grid;
  cds::g_trace_grid = 0;
  return g;
}

int cds_run_op(int device, const cds_op* op, int32_t iter, void* stream) {
  if (!op) return fail(CDS_ERR_INVALID, "run_op: null op");
  CDS_ON_DEVICE(device);
  Step s;
  int rc = validate(*op, &s);
  if (rc != CDS_OK) return rc;
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  int* d_iter = nullptr;
  CDS_CUDA(cudaMallocAsync(&d_iter, sizeof(int), st));
  cds::set_iter_kernel<<<1, 1, 0, st>>>(d_iter, iter);
  rc = launch(s, d_iter, cds_device_sm_count(device), st);
  cudaFreeAsync(d_iter, st);
  return rc;
}

}  // extern "C"
