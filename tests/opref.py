"""TEST INFRASTRUCTURE: the operator semantics of include/cds.h as plain torch fp64 code, on any device.

One reference for two users: tests/emulator.py loads the operands of a lowered program from raw memory and calls these
functions (CPU lowering tests), and the operator-level GPU tests run them on the H100 next to the kernels.

Operands are read the way the hardware reads them -- fp32 as is (CDS_MATH_FP32), the low 13 mantissa bits dropped
(wgmma .tf32, CDS_MATH_TF32_TC), bf16 values (CDS_MATH_BF16_TC) -- and everything after that is exact fp64 arithmetic:
products, sums, the two-pass GroupNorm / LayerNorm statistics, the activations and the epilogue.  The result is returned
in fp64; ``store`` applies the rounding of an output dtype.

Canonical layouts: activations (rows, L, C); conv weights w[tap][ci][n] with n < C_out * phases; per-channel vectors are
either (C,) (the same for every row) or (owners, C) indexed by row // sample_row_div.  A tensor with fewer rows than the
op's batch is read at row b % len(tensor): that is in_batch_mod / res_batch_mod (and a residual of one row is a
broadcast).  Never imported by the product.
"""
import math

import torch

from cleandiffuser_b200.engine import cabi

F64 = torch.float64


def tf32_trunc(x):
    """what wgmma .tf32 sees of an fp32 operand: the low 13 mantissa bits are ignored"""
    bits = x.to(torch.float32).contiguous().view(torch.int32)
    return (bits & ~0x1FFF).view(torch.float32)


def tf32_round(x):
    """fp32 -> nearest TF32 (ties away from zero, cvt.rna.tf32.f32): what a producer stores into a CDS_TF32 tensor"""
    bits = x.to(torch.float32).contiguous().view(torch.int32)
    return ((bits + 0x1000) & ~0x1FFF).view(torch.float32)


def operand(x, math_mode):
    """fp64 copy of a GEMM operand as the kernel family of ``math_mode`` reads it"""
    if math_mode == cabi.MATH_TF32_TC:
        return tf32_trunc(x).to(F64)
    if math_mode == cabi.MATH_BF16_TC:
        return x.to(torch.bfloat16).to(F64)
    return x.to(F64)


def store(y, dtype):
    """the value a kernel stores for the exact result ``y``, as fp32 (bf16 values widened)"""
    y32 = y.to(torch.float32)
    if dtype == cabi.TF32:
        return tf32_round(y32)
    if dtype == cabi.BF16:
        return y32.to(torch.bfloat16).to(torch.float32)
    return y32


def mish(x):
    return x * torch.tanh(torch.nn.functional.softplus(x))


def act(kind, x):
    if kind == cabi.ACT_MISH:
        return mish(x)
    if kind == cabi.ACT_SILU:
        return x * torch.sigmoid(x)
    if kind == cabi.ACT_GELU_TANH:
        return 0.5 * x * (1 + torch.tanh(math.sqrt(2 / math.pi) * (x + 0.044715 * x ** 3)))
    if kind == cabi.ACT_MISH_SILU:
        m = mish(x)
        return m * torch.sigmoid(m)
    if kind == cabi.ACT_LEAKY_RELU:
        return torch.where(x > 0, x, 0.01 * x)
    if kind == cabi.ACT_GELU_ERF:
        return 0.5 * x * (1 + torch.special.erf(x / math.sqrt(2)))
    assert kind == cabi.ACT_NONE, kind
    return x


def _rows(t, b):
    """rows b of t, read at b % len(t)"""
    return t[b % t.shape[0]]


def _vec(v, b, div):
    """per-row values of a (C,) or (owners, C) vector for the row indices b: shape (len(b), 1, C)"""
    if v is None:
        return None
    v = v.to(F64)
    return v[None, None] if v.dim() == 1 else v[b // div][:, None]


def conv(x, w, *, batch, L_out, taps=1, stride=1, pad=0, phases=1, math_mode=cabi.MATH_FP32, bias=None, groups=0,
         gamma=None, beta=None, eps=1e-5, act_kind=cabi.ACT_NONE, scale=None, shift=None, res=None, res_in=None,
         res_w=None, res_bias=None, sample_row_div=1, chunk_rows=1 << 16):
    """CDS_OP_CONV in fp64: (batch, L_out * phases, C_out).

    x (rows, L_in, C_in) and res_in (rows, L_out, res_C) are GEMM operands (read per ``math_mode``); w (taps, C_in, N) and
    res_w (res_C, C_out) likewise.  res (rows, L_out, C_out), bias / scale / shift / gamma / beta / res_bias are epilogue
    inputs, read exactly.  Computed in batch chunks of about ``chunk_rows`` output rows."""
    L_in = x.shape[1]
    N = w.shape[2]
    C_out = N // phases
    chan = torch.arange(N, device=x.device) % C_out
    wk = operand(w, math_mode)
    rw = operand(res_w, math_mode) if res_w is not None else None
    div = max(1, int(sample_row_div))
    step = max(1, chunk_rows // max(1, L_out))
    out = torch.empty(batch, L_out * phases, C_out, dtype=F64, device=x.device)
    pos = torch.arange(L_out, device=x.device) * stride - pad
    for b0 in range(0, batch, step):
        b = torch.arange(b0, min(batch, b0 + step), device=x.device)
        xb = operand(_rows(x, b), math_mode)
        y = torch.zeros(len(b), L_out, N, dtype=F64, device=x.device)
        for tap in range(taps):
            p = pos + tap
            ok = (p >= 0) & (p < L_in)
            if ok.any():
                y[:, ok] += xb[:, p[ok]] @ wk[tap]
        bv = _vec(bias, b, div)
        if bv is not None:
            y = y + bv[..., chan]
        if groups > 0:
            assert phases == 1
            g = y.reshape(len(b), L_out, groups, C_out // groups)
            mean = g.mean(dim=(1, 3), keepdim=True)
            var = ((g - mean) ** 2).mean(dim=(1, 3), keepdim=True)
            y = ((g - mean) / torch.sqrt(var + eps)).reshape(len(b), L_out, C_out)
            y = y * gamma.to(F64) + beta.to(F64)
        y = act(act_kind, y)
        sv, hv = _vec(scale, b, div), _vec(shift, b, div)
        if sv is not None:
            y = y * sv[..., chan]
        if hv is not None:
            y = y + hv[..., chan]
        if res is not None:
            y = y + _rows(res, b).to(F64)
        if rw is not None:
            y = y + operand(_rows(res_in, b), math_mode) @ rw
            if res_bias is not None:
                y = y + res_bias.to(F64)[chan]
        out[b0:b0 + len(b)] = y.reshape(len(b), L_out, phases, C_out).reshape(len(b), L_out * phases, C_out)
    return out


def attn(qkv, heads, qkv_dtype=cabi.F32):
    """CDS_OP_ATTN in fp64: softmax(q k^T / sqrt(hd)) v per (trajectory, head), (batch, L, C).  qkv (batch, L, 3C) with
    [q | k | v] column blocks, read as stored: bf16 values, or fp32 as is (a CDS_TF32 tensor already holds TF32 values)."""
    B, L, C3 = qkv.shape
    C = C3 // 3
    hd = C // heads
    if qkv_dtype == cabi.BF16:
        qkv = qkv.to(torch.bfloat16)
    q, k, v = (t.to(F64).reshape(B, L, heads, hd).transpose(1, 2) for t in qkv.split(C, dim=-1))   # (B, heads, L, hd)
    p = torch.softmax(q @ k.transpose(-1, -2) / math.sqrt(hd), dim=-1)
    return (p @ v).transpose(1, 2).reshape(B, L, C)


def lnmod(x, shift, scale, eps, *, L=1):
    """CDS_OP_LNMOD in fp64: LayerNorm(x) (two-pass statistics, no affine) * (1 + scale) + shift.  x (rows, C) or (batch, L, C);
    shift / scale (batch, C), one vector per trajectory = per L rows of a (rows, C) x."""
    x = x.to(F64)
    mean = x.mean(-1, keepdim=True)
    var = ((x - mean) ** 2).mean(-1, keepdim=True)
    n = (x - mean) / torch.sqrt(var + eps)
    if x.dim() == 2:
        own = torch.arange(x.shape[0], device=x.device) // L
        return n * (1 + scale.to(F64)[own]) + shift.to(F64)[own]
    return n * (1 + scale.to(F64)[:, None]) + shift.to(F64)[:, None]
