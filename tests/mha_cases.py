"""TEST INFRASTRUCTURE: the operator-level case table of CDS_OP_MHA, the buffers of each case, and the error bound.

Every case is run with q / k / v in each of ``IN_DTYPES`` and names the head_dim it reaches; over the table and the input
dtypes every instantiation mha_f32_kernel<HPL = head_dim / 32, BF16> (HPL 1..8, fp32 or bf16 loads) is reached, which
tests/test_chitransformer_cpu.py checks through ``cabi.mha_choice``.  tests/test_chitransformer_gpu.py runs every case
through ``cds_run_op`` against the fp64 reference of tests/mha_ref.py.

Buffers are laid out the way the ChiTransformer lowering uses the operator, with odd strides: q is a column slice of a wider
activation (``Q_OFF`` channels in, rows of 3C + 1), the per-trajectory k|v rows are a column slice of rows of 2C + 3, the
per-iteration k|v table has ``N_ITERS`` iterations (the case reads iteration ``ITER``), and the output is a column slice of
NaN-filled rows of C + 2.
"""
import math
import zlib

import torch

import mha_ref
import opref
from cleandiffuser_b200.engine import cabi

TORCH_DT = {cabi.F32: torch.float32, cabi.TF32: torch.float32, cabi.BF16: torch.bfloat16}
IN_DTYPES = (cabi.F32, cabi.TF32, cabi.BF16)
OUTS = (cabi.F32, cabi.TF32, cabi.BF16)
F64 = torch.float64
R_OUT = {cabi.F32: 0.0, cabi.TF32: 2.0 ** -10, cabi.BF16: 2.0 ** -8}
MODES = ("n0.5", "n3", "q0", "v100")
N_ITERS, ITER = 3, 2
Q_OFF, KV_OFF, OUT_OFF = 1, 3, 1


def case(name, B, Lq, Lk, heads, hd, diag, kv):
    """diag: key j visible to query i iff j <= i + diag (None: no mask); kv: which parts hold k|v ("sample", "step", "both")"""
    return dict(name=name, B=B, Lq=Lq, Lk=Lk, heads=heads, hd=hd, diag=diag, kv=kv)


CASES = [
    # ChiTransformer's two attentions at the pipeline head_dims (64: pusht / robomimic, 192: kitchen) and the edge shape
    case("chi_self_hd64", 5, 10, 10, 4, 64, 0, "sample"),
    case("chi_cross_hd64", 5, 10, 3, 4, 64, 1, "both"),
    case("chi_self_hd192", 3, 10, 10, 4, 192, 0, "sample"),
    case("chi_cross_hd192", 3, 10, 3, 4, 192, 1, "both"),
    case("edge_self_hd32", 4, 16, 16, 2, 32, 0, "sample"),
    case("edge_cross_hd32", 4, 16, 2, 2, 32, 1, "both"),
    # the remaining head_dims, no mask, step-only k|v, the largest sequences, rows without a visible key (diag < 0)
    case("hd96_unmasked", 3, 7, 13, 3, 96, None, "sample"),
    case("hd128_step_only", 3, 5, 9, 2, 128, None, "step"),
    case("hd160_L64", 2, 64, 64, 1, 160, 0, "sample"),
    case("hd224_no_visible_rows", 2, 33, 17, 2, 224, -3, "both"),
    case("hd256_L1", 2, 1, 1, 1, 256, None, "sample"),
    case("hd256_L64", 2, 64, 40, 2, 256, 5, "both"),
    # many CTAs, the last one partly idle (701 * 3 * 10 query rows = 2 mod 4 warps)
    case("chi_cross_big", 701, 10, 3, 3, 64, 1, "both"),
]
CASES = {c["name"]: c for c in CASES}
# refused with CDS_ERR_UNSUPPORTED (-3) / CDS_ERR_INVALID (-1): (B, Lq, Lk, heads, hd), code
REFUSED = [((2, 10, 10, 4, 16), -3), ((2, 10, 10, 4, 48), -3), ((2, 10, 10, 1, 288), -3), ((2, 65, 10, 2, 32), -3),
           ((2, 10, 65, 2, 32), -3), ((0, 10, 10, 2, 32), -1), ((2, 0, 10, 2, 32), -1), ((2, 10, 10, 0, 32), -1)]


def descriptor(c, in_dtype, out_dtype, ptrs=None, B=None):
    """ptrs: (q, kv_step, kv_sample, out) addresses of the first element; None: made-up addresses (cds_mha_choice)"""
    C = c["heads"] * c["hd"]
    op = cabi.Op()
    op.kind = cabi.OP_MHA
    m = op.u.mha
    m.batch, m.Lq, m.Lk, m.C, m.heads = B or c["B"], c["Lq"], c["Lk"], C, c["heads"]
    m.masked, m.diag = (0, 0) if c["diag"] is None else (1, c["diag"])
    q, step, samp, out = ptrs or (1 << 20, 1 << 21, 1 << 22, 1 << 23)
    m.q, m.q_bstride, m.q_lstride = q, c["Lq"] * (3 * C + 1), 3 * C + 1
    if c["kv"] in ("step", "both"):
        m.kv_step, m.kv_step_stride, m.kv_step_lstride = step, c["Lk"] * (2 * C + 1), 2 * C + 1
    if c["kv"] in ("sample", "both"):
        m.kv_sample, m.kv_sample_bstride, m.kv_sample_lstride = samp, c["Lk"] * (2 * C + 3), 2 * C + 3
    m.out, m.out_bstride, m.out_lstride = out, c["Lq"] * (C + 2), C + 2
    m.in_dtype, m.out_dtype = in_dtype, out_dtype
    return op


def make(c, mode, in_dtype, device):
    """The case's input buffers as stored (bf16, or fp32 holding TF32 values for CDS_TF32), the padding filled with NaN so that
    a read outside the operands shows: dict with qbuf, stepbuf, sampbuf (None when absent) and the dense views q
    (B, Lq, C) and kv = step[ITER] + sample (B, Lk, 2C) in fp64, as the reference reads them.
      n0.5 / n3   N(0, sigma); at sigma = 3 the logits span tens of units and most P underflow
      q0          q = 0: every output row is the mean of its visible v
      v100        v = 100 + small noise: the terms of the bound relative to sum P|v| dominate"""
    B, Lq, Lk, C = c["B"], c["Lq"], c["Lk"], c["heads"] * c["hd"]
    g = torch.Generator().manual_seed(zlib.crc32(f"{c['name']}/{mode}/{in_dtype}".encode()))
    sigma = 3.0 if mode == "n3" else 0.5
    dt = TORCH_DT[in_dtype]

    def stored(x):
        return opref.tf32_round(x) if in_dtype == cabi.TF32 else x.to(dt).to(torch.float32)

    def kv_rows(*lead):
        k, v = sigma * torch.randn(*lead, Lk, C, generator=g), sigma * torch.randn(*lead, Lk, C, generator=g)
        if mode == "v100":
            v = 100 + 0.1 * v
        return stored(torch.cat([k, v], -1))

    q = stored(torch.zeros(B, Lq, C) if mode == "q0" else sigma * torch.randn(B, Lq, C, generator=g))
    qbuf = torch.full((B, Lq, 3 * C + 1), float("nan"))
    qbuf[..., Q_OFF:Q_OFF + C] = q
    kv = torch.zeros(B, Lk, 2 * C, dtype=F64)
    stepbuf = sampbuf = None
    if c["kv"] in ("step", "both"):
        step = kv_rows(N_ITERS)
        stepbuf = torch.full((N_ITERS, Lk, 2 * C + 1), float("nan"))
        stepbuf[..., :2 * C] = step
        kv += step[ITER].to(F64)
    if c["kv"] in ("sample", "both"):
        samp = kv_rows(B)
        if c["kv"] == "both" and mode == "v100":     # the sum of the two parts is the 100 + noise
            samp[..., C:] -= 100
        sampbuf = torch.full((B, Lk, 2 * C + 3), float("nan"))
        sampbuf[..., KV_OFF:KV_OFF + 2 * C] = samp
        kv += samp.to(F64)
    to = lambda t: None if t is None else t.to(dt).to(device)      # noqa: E731
    return dict(qbuf=to(qbuf), stepbuf=to(stepbuf), sampbuf=to(sampbuf), q=q.to(F64).to(device), kv=kv.to(device))


def reference(c, inp):
    return mha_ref.mha(inp["q"], inp["kv"], c["heads"], c["diag"])


def bound(c, q, kv, ref, out_dtype, kv_sum=None):
    """|y - ref| <= S * (2 e_logit + e_acc + e_kv) + r_out |ref| per element, S = sum_j P_j |v_j| over the visible keys:
      e_logit   relative error of each P from its exponent: 2^-22 (1 + 2 max|s|) for the rounding of s * scale, of s - max and
                for expf, plus (hd + 4) 2^-24 max sum_d |q_d k_d| / sqrt(hd) for the fp32 dot product (a lane's fma chain and
                the 5-level warp tree) and rsqrtf.  Relative errors d_j of P move the output by sum_j p_j d_j (v_j - o), at
                most 2 max d S: hence the factor 2
      e_acc     the online softmax over Lk keys: both running sums rescaled at every key, the reciprocal and the scaling:
                (4 Lk + 8) 2^-24
      e_kv      the fp32 sum step + sample of k and v when both parts are present: 2^-24 on v, and on every logit through k
      r_out     rounding of the stored output (TF32 / bf16)
    A query row without a visible key has bound 0: the kernel must store exact zeros."""
    B, Lq, C = q.shape
    heads, hd, Lk = c["heads"], c["hd"], kv.shape[1]
    qh = q.to(F64).reshape(B, Lq, heads, hd).transpose(1, 2)
    k, v = (t.to(F64).reshape(B, Lk, heads, hd).transpose(1, 2) for t in kv.split(C, dim=-1))
    s = qh @ k.transpose(-1, -2) / math.sqrt(hd)
    g = (qh.abs() @ k.abs().transpose(-1, -2)) / math.sqrt(hd)
    if c["diag"] is not None:
        vis = torch.arange(Lk, device=q.device)[None, :] <= torch.arange(Lq, device=q.device)[:, None] + c["diag"]
        s = s.masked_fill(~vis, float("-inf"))
        g = g.masked_fill(~vis, 0.0)
    p = torch.nan_to_num(torch.softmax(s, dim=-1), nan=0.0)
    S = p @ v.abs()
    a_max = s.nan_to_num(neginf=0.0).abs().amax(-1, keepdim=True)
    both = c["kv"] == "both" if kv_sum is None else kv_sum
    e_logit = 2.0 ** -22 * (1 + 2 * a_max) + (hd + 4 + (1 if both else 0)) * 2.0 ** -24 * g.amax(-1, keepdim=True)
    rel = 2 * e_logit + (4 * Lk + 8) * 2.0 ** -24 + (2.0 ** -24 if both else 0.0)
    per = (S * rel).transpose(1, 2).reshape(B, Lq, C)
    return per + R_OUT[out_dtype] * ref.abs()


def check(c, y, q, kv, ref, out_dtype):
    """(ok, largest error / bound, message) for a kernel output y (fp32 values) against the fp64 reference"""
    b = bound(c, q, kv, ref, out_dtype)
    err = (y.to(F64) - ref).abs()
    ratio = torch.where(b > 0, err / b.clamp_min(1e-300), torch.where(err > 0, torch.inf, 0.0))
    frac = ratio.max().item() if err.numel() else 0.0
    finite = bool(torch.isfinite(y).all())
    ok = finite and bool((err <= b).all())
    i = int(ratio.flatten().argmax())
    return ok, frac, f"{c['name']}: max err / bound = {frac:.3g} at flat index {i} (err {err.flatten()[i].item():.3g}, " \
                     f"bound {b.flatten()[i].item():.3g}), finite={finite}"
