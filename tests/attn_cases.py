"""TEST INFRASTRUCTURE: the operator-level case table of CDS_OP_ATTN, the inputs of each case, and the error bound of its
kernel.

Every case names the kernel instantiation it must reach (``want``, in the form ``choice_key`` gives ``cabi.attn_choice``):
("f32", HD), ("bf16_mma", 0) or ("tma", NT).  tests/test_attn_dispatch_cpu.py checks on the CPU that
each case reaches it, that the table covers every instantiation, and that ``check`` accepts the fp64 reference and rejects
typical kernel faults; tests/test_attention_gpu.py runs every case through ``cds_run_op`` against tests/opref.py.

``out_off`` places the output that many floats into its buffer: at 2 floats (8 bytes) TF32 q/k/v with head_dim 32 and
L <= 128 run on the fp32 kernel, since the persistent TMA kernel needs a 16-byte aligned output (the "_out8" cases).
"""
import math
import zlib

import torch

import opref
from cleandiffuser_b200.engine import cabi

TORCH_DT = {cabi.F32: torch.float32, cabi.TF32: torch.float32, cabi.BF16: torch.bfloat16}
F64 = torch.float64
LOG2E = 1.0 / math.log(2.0)
# P is rounded to the MMA operand type before P V: unit roundoff of bf16 (8 significant bits) and of TF32 (cvt.rna, 11)
U_P = {"f32": 0.0, "bf16_mma": 2.0 ** -8, "tma": 2.0 ** -11}
# relative rounding of the stored output, as in tests/test_conv_kernels_gpu.py
R_OUT = {cabi.F32: 0.0, cabi.TF32: 2.0 ** -10, cabi.BF16: 2.0 ** -8}
# value patterns every case runs with (see ``make``)
MODES = ("n0.5", "n3", "q0", "v100", "lastmax")
SMS = 132                                   # H100 SXM; the TMA kernel's grid is 2 CTAs per SM (the GPU test checks the
                                            # device's own SM count against the regime each TMA case was sized for)
MAX_L = {16: 1600, 32: 800, 64: 400}        # L * hd * 8 bytes of K and V <= 200 KB


def key(family, param=0):
    return (family, param)


def choice_key(ch):
    return key(ch["family"], ch["param"])


def case(name, want, B, L, heads, hd=32, qkv_dtype=cabi.TF32, outs=(cabi.F32, cabi.TF32), out_off=0):
    return dict(name=name, want=want, B=B, L=L, heads=heads, hd=hd, qkv_dtype=qkv_dtype, outs=tuple(outs), out_off=out_off)


ALL_OUTS = (cabi.F32, cabi.TF32, cabi.BF16)
CASES = []
# ---- persistent TMA kernel: every NT = ceil(L / 8) and every L mod 16; L in 113..128 gives warp 0 two query tiles.  Most
# cases have fewer (trajectory, head) items than the 2 x 132 CTA grid; the "_ring" ones at least 3x as many, so that every
# CTA walks its 2-stage ring round more than once and the phase bit wraps.
for L in (1, 10, 19, 28, 37, 46, 55, 64, 65, 74, 83, 92, 101, 110, *range(113, 129)):
    CASES.append(case(f"tma_L{L}", key("tma", (L + 7) // 8), B=3, L=L, heads=2 + L % 3))
for L in (1, 64, 113, 128):
    CASES.append(case(f"tma_L{L}_ring", key("tma", (L + 7) // 8), B=3 * 2 * SMS // 8 + 1, L=L, heads=8))
# ---- TF32 q/k/v in the TMA kernel's shapes with the output 8- but not 16-byte aligned: the fp32 kernel serves them.  Seven
# shapes of their own, and the shape of every TMA case above (the "_out8" twins)
for L in (1, 7, 16, 33, 100, 113, 128):
    CASES.append(case(f"f32_hd32_L{L}_tf32_out8", key("f32", 32), B=3, L=L, heads=3, out_off=2))
for c in [c for c in CASES if c["want"][0] == "tma"]:
    CASES.append(dict(c, name=f"f32_{c['name']}_out8", want=key("f32", 32), out_off=2))
# ---- bf16 mma.sync (every bf16 DiT program)
for L in (1, 15, 16, 17, 100, 127, 128):
    CASES.append(case(f"bf16mma_L{L}", key("bf16_mma"), B=3, L=L, heads=1 + L % 4, qkv_dtype=cabi.BF16, outs=ALL_OUTS))
# ---- fp32 kernel: head_dim 16 / 32 / 64, L up to the largest accepted (K and V above 48 KB of shared memory from
# L * hd > 6144 on), q/k/v fp32 or TF32-rounded.  With TF32 q/k/v, head_dim 32, L <= 128 and a 16-byte aligned output
# only a bf16 output reaches it.
for hd in (16, 32, 64):
    for L in (1, 100, 129, 300, MAX_L[hd]):
        for qd in (cabi.F32, cabi.TF32):
            outs = (cabi.BF16,) if (qd == cabi.TF32 and hd == 32 and L <= 128) else ALL_OUTS
            CASES.append(case(f"f32_hd{hd}_L{L}_{'tf32' if qd == cabi.TF32 else 'f32'}", key("f32", hd), B=2, L=L,
                              heads=3 if L < 400 else 2, hd=hd, qkv_dtype=qd, outs=outs))
CASES = {c["name"]: c for c in CASES}


def descriptor(c, qkv_ptr, out_ptr, out_dtype, B=None):
    op = cabi.Op()
    op.kind = cabi.OP_ATTN
    a = op.u.attn
    a.batch, a.L, a.C, a.heads = B or c["B"], c["L"], c["heads"] * c["hd"], c["heads"]
    a.qkv, a.out, a.out_dtype, a.qkv_dtype = qkv_ptr, out_ptr, out_dtype, c["qkv_dtype"]
    return op


def fake_descriptor(c, out_dtype=None):
    """descriptor with made-up, suitably aligned addresses: only alignment matters to cds_attn_choice"""
    return descriptor(c, 1 << 20, (1 << 21) + 4 * c["out_off"], c["outs"][0] if out_dtype is None else out_dtype)


def make(c, mode, device, B=None):
    """q | k | v of case ``c`` as stored (bf16 tensor, or fp32 holding TF32 values for a CDS_TF32 operand):
      n0.5 / n3   N(0, sigma); at sigma = 3 the logits span tens of units and most P underflow
      q0          q = 0: every output row is exactly the mean of v
      v100        v = 100 + small noise: the terms of the bound relative to sum P|v| dominate
      lastmax     q > 0 and the last key (in the ragged last tile) larger than every other: it holds each row's maximum"""
    B = B or c["B"]
    L, C = c["L"], c["heads"] * c["hd"]
    g = torch.Generator().manual_seed(zlib.crc32(f"{c['name']}/{mode}".encode()))
    sigma = 3.0 if mode == "n3" else 0.5
    q, k, v = (sigma * torch.randn(B, L, C, generator=g) for _ in range(3))
    if mode == "q0":
        q.zero_()
    elif mode == "v100":
        v = 100 + 0.1 * v
    elif mode == "lastmax":
        q = q.abs()
        k[:, -1] = 2.0
    qkv = torch.cat([q, k, v], dim=-1)
    if c["qkv_dtype"] == cabi.BF16:
        qkv = qkv.to(torch.bfloat16)
    elif c["qkv_dtype"] == cabi.TF32:
        qkv = opref.tf32_round(qkv)
    return qkv.to(device)


def _heads(qkv, heads):
    B, L, C3 = qkv.shape
    C = C3 // 3
    return (t.to(F64).reshape(B, L, heads, C // heads).transpose(1, 2) for t in qkv.split(C, dim=-1))


def bound(c, qkv, ref, out_dtype):
    """|y - ref| <= S * (u_P + 2 e_logit + e_acc) + r_out |ref| per element, S = sum_j P_j |v_j| (P normalised):
      u_P       rounding of P to the MMA operand type before P V (numerator only: the row sum adds the unrounded P)
      e_logit   relative error of each P from its exponent, in log2 units (exp2 of an error e is a relative error
                e ln 2 <= e): 2^-22 (1 + 2 max|s log2 e|) for the fp32 rounding of the scaled logit and of max * scale
                inside fmaf(s, scale log2e, -max scale log2e) and for ex2.approx, plus (hd + 2) 2^-24 max sum_d |q_d k_d| /
                sqrt(hd) log2e for the fp32 dot product q.k.  Relative errors d_j of P move the output by
                sum_j p_j d_j (v_j - o), at most 2 max d S: hence the factor 2
      e_acc     fp32 accumulation over L keys of the numerator and of the row sum, the reciprocal and the scaling:
                (2 L + 8) 2^-24; the fp32 kernel's online softmax rescales both sums at every key (one more rounding each,
                and the expf of the correction factor): (4 L + 8) 2^-24
      r_out     rounding of the stored output (TF32 / bf16)"""
    fam = c["want"][0]
    q, k, v = _heads(qkv, c["heads"])
    hd = c["hd"]
    s = q @ k.transpose(-1, -2) / math.sqrt(hd)
    p = torch.softmax(s, dim=-1)
    S = p @ v.abs()                                                                 # (B, heads, L, hd)
    a_max = s.abs().amax(-1, keepdim=True) * LOG2E
    g_max = (q.abs() @ k.abs().transpose(-1, -2)).amax(-1, keepdim=True) / math.sqrt(hd) * LOG2E
    e_logit = 2.0 ** -22 * (1 + 2 * a_max) + (hd + 2) * 2.0 ** -24 * g_max
    e_acc = ((4 if fam == "f32" else 2) * c["L"] + 8) * 2.0 ** -24
    rel = U_P[fam] + 2 * e_logit + e_acc
    B, L = qkv.shape[:2]
    per = (S * rel).transpose(1, 2).reshape(B, L, -1)
    return per + R_OUT[out_dtype] * ref.abs()


def check(c, y, qkv, ref, out_dtype):
    """(ok, largest error / bound, message) for a kernel output y (fp32 values) against the fp64 reference"""
    b = bound(c, qkv, ref, out_dtype)
    err = (y.to(F64) - ref).abs()
    frac = (err / b).max().item() if err.numel() else 0.0
    finite = bool(torch.isfinite(y).all())
    ok = finite and bool((err <= b).all())
    i = int((err / b).flatten().argmax())
    return ok, frac, f"{c['name']}: max err / bound = {frac:.3g} at flat index {i} (err {err.flatten()[i].item():.3g}, " \
                     f"bound {b.flatten()[i].item():.3g}), finite={finite}"
