"""TEST INFRASTRUCTURE: a numpy interpreter of the libcds operator program (include/cds.h semantics).

It lets the CPU test-suite execute the *lowered* program (``engine/lower.py`` output, with CPU tensors behind
the raw pointers) and compare it with the reference goldens, so that lowering bugs (wrong strides, offsets,
table columns, phase packing ...) are caught here without a GPU; the kernels themselves are then checked
against the same goldens on the H100.  Never imported by the product.
"""
import ctypes

import numpy as np
import torch

import opref
from cleandiffuser_b200.engine import cabi


def _arr(ptr, shape, strides):
    """float32 view of raw memory; strides in floats."""
    if not ptr:
        return None
    extent = 1 + sum((s - 1) * abs(st) for s, st in zip(shape, strides))
    flat = np.ctypeslib.as_array((ctypes.c_float * extent).from_address(ptr))
    return np.lib.stride_tricks.as_strided(flat, shape=shape, strides=[4 * s for s in strides])


def _bf16_to_f32(u16):
    return (u16.astype(np.uint32) << 16).view(np.float32)


def _f32_to_bf16(x):
    import torch
    return torch.from_numpy(np.ascontiguousarray(x, dtype=np.float32)).to(torch.bfloat16).view(torch.int16).numpy().view(np.uint16)


def _rn_tf32(x):
    """fp32 -> nearest TF32 (ties away from zero): what producers store into a CDS_TF32 tensor"""
    u = np.ascontiguousarray(x, dtype=np.float32).view(np.uint32)
    return ((u + np.uint32(0x1000)) & np.uint32(0xFFFFE000)).view(np.float32)


def _load(ptr, shape, strides, dtype):
    """float32 COPY of an fp32 / bf16 activation view (strides in elements)."""
    if dtype in (cabi.F32, cabi.TF32):
        return np.array(_arr(ptr, shape, strides))
    extent = 1 + sum((s - 1) * abs(st) for s, st in zip(shape, strides))
    flat = np.ctypeslib.as_array((ctypes.c_uint16 * extent).from_address(ptr))
    return _bf16_to_f32(np.lib.stride_tricks.as_strided(flat, shape=shape, strides=[2 * s for s in strides]))


def _store(ptr, shape, strides, dtype, values):
    if dtype in (cabi.F32, cabi.TF32):
        _arr(ptr, shape, strides)[...] = _rn_tf32(values) if dtype == cabi.TF32 else values
        return
    extent = 1 + sum((s - 1) * abs(st) for s, st in zip(shape, strides))
    flat = np.ctypeslib.as_array((ctypes.c_uint16 * extent).from_address(ptr))
    np.lib.stride_tricks.as_strided(flat, shape=shape, strides=[2 * s for s in strides])[...] = _f32_to_bf16(values)


def _vec(v, it, rows, n, row_div=1):
    out = np.zeros((rows, n), dtype=np.float32)
    present = False
    if v.step:
        out += _arr(v.step + 4 * it * v.step_stride, (n,), (1,))[None]
        present = True
    if v.sample:
        owners = (rows + row_div - 1) // row_div                   # one vector per `row_div` rows (flattened token rows)
        out += _arr(v.sample, (owners, n), (v.sample_stride, 1))[np.arange(rows) // row_div]
        present = True
    return out if present else None


def _t(a):
    return None if a is None else torch.from_numpy(np.ascontiguousarray(a))


def run_conv(c, it):
    """CDS_OP_CONV: load the operands of the descriptor and evaluate tests/opref.py's fp64 reference"""
    B, N = c.batch, c.C_out * c.phases
    bmod = c.in_batch_mod if c.in_batch_mod > 0 else B
    xin = _load(c.in_, (bmod, c.L_in, c.C_in), (c.in_bstride, c.in_lstride, 1), c.in_dtype)
    tc = c.math in cabi.TC_MODES
    wdt = cabi.F32 if c.math == cabi.MATH_TF32_TC else cabi.BF16
    if tc:      # bf16 / fp32 [taps][C_out*phases][C_in]
        assert c.in_dtype == wdt or (wdt == cabi.F32 and c.in_dtype == cabi.TF32)
        w = _load(c.w, (c.taps, N, c.C_in), (N * c.C_in, c.C_in, 1), wdt).transpose(0, 2, 1)
    else:
        w = _arr(c.w, (c.taps, c.C_in, N), (c.C_in * N, N, 1))
    div = c.sample_row_div if c.sample_row_div > 1 else 1
    kw = dict(bias=_vec(c.bias, it, B, c.C_out, div), scale=_vec(c.scale, it, B, c.C_out, div),
              shift=_vec(c.shift, it, B, c.C_out, div))
    kw = {k: _t(v) for k, v in kw.items()}
    if c.groups > 0:
        kw.update(groups=c.groups, gamma=_t(_arr(c.gn_gamma, (c.C_out,), (1,))), beta=_t(_arr(c.gn_beta, (c.C_out,), (1,))),
                  eps=c.gn_eps)
    rmod = c.res_batch_mod if c.res_batch_mod > 0 else B
    if c.res:
        kw["res"] = _t(_load(c.res, (rmod if c.res_bstride else 1, c.L_out, c.C_out), (c.res_bstride, c.res_lstride, 1),
                             c.res_dtype))
    if c.res_w:
        kw["res_in"] = _t(_load(c.res_in, (rmod, c.L_out, c.res_C), (c.res_in_bstride, c.res_in_lstride, 1), c.res_in_dtype))
        kw["res_w"] = _t(_load(c.res_w, (c.C_out, c.res_C), (c.res_C, 1), wdt).T if tc else _arr(c.res_w, (c.res_C, N), (N, 1)))
        if c.res_bias:
            kw["res_bias"] = _t(_arr(c.res_bias, (c.C_out,), (1,)))
    y = opref.conv(_t(xin), _t(w), batch=B, L_out=c.L_out, taps=c.taps, stride=c.stride, pad=c.pad, phases=c.phases,
                   math_mode=c.math, act_kind=c.act, **kw)
    _store(c.out, (B, c.L_out * c.phases, c.C_out), (c.out_bstride, c.out_lstride, 1), c.out_dtype,
           y.to(torch.float32).numpy())


def run_lnmod(m):
    x = _arr(m.in_, (m.batch, m.L, m.C), (m.L * m.C, m.C, 1))
    sh = _arr(m.shift, (m.batch, m.C), (m.mod_bstride, 1))
    sc = _arr(m.scale, (m.batch, m.C), (m.mod_bstride, 1))
    y = opref.lnmod(_t(x), _t(sh), _t(sc), m.eps)
    _store(m.out, (m.batch, m.L, m.C), (m.L * m.C, m.C, 1), m.out_dtype, y.to(torch.float32).numpy())


def run_attn(a):
    """CDS_OP_ATTN: load q|k|v (bf16 values widened exactly) and evaluate tests/opref.py's fp64 reference"""
    qkv = _load(a.qkv, (a.batch, a.L, 3 * a.C), (a.L * 3 * a.C, 3 * a.C, 1), a.qkv_dtype)
    o = opref.attn(_t(qkv), a.heads, a.qkv_dtype)
    _store(a.out, (a.batch, a.L, a.C), (a.L * a.C, a.C, 1), a.out_dtype, o.to(torch.float32).numpy())


def run_cast(k):
    x = _arr(k.in_, (k.batch, k.L, k.C_in), (k.L * k.C_in, k.C_in, 1))
    y = np.zeros((k.batch, k.L, k.C_out), dtype=np.float32)
    y[..., :k.C_in] = x
    _store(k.out, (k.batch, k.L, k.C_out), (k.L * k.C_out, k.C_out, 1), k.out_dtype, y)


def _row(coef, it):
    return _arr(coef + 4 * it * cabi.ROW_FLOATS, (cabi.ROW_FLOATS,), (1,))


def run_prep(p, it):
    row = _row(p.coef, it)
    n = p.batch * p.row
    x = _arr(p.x, (n,), (1,))
    slot = int(row[8]) - 1
    if slot >= 0:
        x[...] = x + row[4] * _arr(p.noise + 4 * slot * n, (n,), (1,))
    _arr(p.xin, (n,), (1,))[...] = row[5] * x


def run_update(u, it):
    f = np.float32
    row = _row(u.coef, it)
    alpha, sigma, k0, k1, k2, k3, k4 = (f(row[i]) for i in range(7))
    kind, slot = int(row[7]), int(row[8]) - 1
    n = u.batch * u.row
    x = _arr(u.x, (u.batch, u.row), (u.row, 1))
    pr = _arr(u.pred, (u.batch, u.row), (u.row, 1)).copy()
    if u.pred_uncond:
        pr = f(u.w_cfg) * pr + f(u.w_uncond) * _arr(u.pred_uncond, (u.batch, u.row), (u.row, 1))
    xmin = _arr(u.x_min, (u.row,), (1,)) if u.x_min else None
    xmax = _arr(u.x_max, (u.row,), (1,)) if u.x_max else None
    slot_stride = u.noise_slot_stride if u.noise_slot_stride > 0 else n
    z = _arr(u.noise + 4 * slot * slot_stride, (u.batch, u.row), (u.row, 1)) if slot >= 0 else None
    if kind in (6, 7):                      # CDS_UPD_EDM / CDS_UPD_EDM_HEUN
        d_theta = k0 * x + k1 * pr
        if u.final_clip:
            if xmin is not None:
                d_theta = np.maximum(d_theta, xmin)
            if xmax is not None:
                d_theta = np.minimum(d_theta, xmax)
        slope = (f(row[10]) * x - f(row[11]) * d_theta) if row[10] != 0 else (x - d_theta) / sigma
        if kind == 6:
            out = x - slope * k2
            if k4 != 0 and u.xhat_prev and u.aux:
                _arr(u.xhat_prev, (u.batch, u.row), (u.row, 1))[...] = x
                _arr(u.aux, (u.batch, u.row), (u.row, 1))[...] = slope
        else:                               # (absent history buffers read as 0, as in the kernel)
            hist = _arr(u.xhat_prev, (u.batch, u.row), (u.row, 1)) if u.xhat_prev else f(0)
            aux = _arr(u.aux, (u.batch, u.row), (u.row, 1)) if u.aux else f(0)
            out = hist - (aux + slope) / f(2) * k2
    elif kind == 5:
        out = k0 * x + k1 * pr
        if u.final_clip:
            if xmin is not None:
                out = np.maximum(out, xmin)
            if xmax is not None:
                out = np.minimum(out, xmax)
    else:
        if u.predict_noise:
            if xmax is not None:
                pr = np.maximum(pr, (x - alpha * xmax) / sigma)
            if xmin is not None:
                pr = np.minimum(pr, (x - alpha * xmin) / sigma)
            eps, xhat = pr, (x - sigma * pr) / alpha
        else:
            if xmin is not None:
                pr = np.maximum(pr, xmin)
            if xmax is not None:
                pr = np.minimum(pr, xmax)
            xhat, eps = pr, (x - alpha * pr) / sigma
        if kind == 0:
            out = k0 * (x - sigma * eps) + k1 * eps
            if z is not None:
                out = out + k2 * z
        elif kind == 1:
            out = k0 * ((x - sigma * eps) / alpha) + k1 * eps
        else:
            hist = _arr(u.xhat_prev, (u.batch, u.row), (u.row, 1)) if u.xhat_prev else None
            target = eps if kind == 2 else (k3 * xhat - k4 * (hist if hist is not None else f(0)) if kind == 4 else xhat)
            out = k0 * x - k1 * target
            if z is not None:
                out = out + k2 * z
            if hist is not None:
                hist[...] = xhat
    if u.mask:
        m = _arr(u.mask, (u.row,), (1,))
        out = out * (f(1) - m) + _arr(u.prior, (u.batch, u.row), (u.row, 1)) * m
    x[...] = out.astype(np.float32)
    if u.x_cast:                     # bf16 channel-padded copy of the new x_t (pad channels untouched)
        rows = n // u.cast_C_in
        y = _load(u.x_cast, (rows, u.cast_C_out), (u.cast_C_out, 1), u.x_cast_dtype)
        y[:, :u.cast_C_in] = x.reshape(rows, u.cast_C_in)
        _store(u.x_cast, (rows, u.cast_C_out), (u.cast_C_out, 1), u.x_cast_dtype, y)


def run_program(ops, n_iters, first=0):
    with np.errstate(over="ignore", invalid="ignore", divide="ignore"):
        for op in ops:                       # CDS_OPF_ONCE operators: once per run, before the first iteration
            if op.flags & cabi.OPF_ONCE:
                assert op.kind == cabi.OP_CAST, op.kind
                run_cast(op.u.cast)
        for it in range(first, first + n_iters):
            for op in ops:
                if op.flags & cabi.OPF_ONCE:
                    continue
                if op.kind == cabi.OP_CONV:
                    run_conv(op.u.conv, it)
                elif op.kind == cabi.OP_UPDATE:
                    run_update(op.u.update, it)
                elif op.kind == cabi.OP_LNMOD:
                    run_lnmod(op.u.lnmod)
                elif op.kind == cabi.OP_ATTN:
                    run_attn(op.u.attn)
                elif op.kind == cabi.OP_PREP:
                    run_prep(op.u.prep, it)
                elif op.kind == cabi.OP_CAST:
                    run_cast(op.u.cast)
                else:
                    raise ValueError(op.kind)


class Handle:
    """Stand-in for ``cabi.Plan`` that executes the program on this interpreter (tests patch ``runtime._make_handle``)."""

    def __init__(self, ops, n_iters):
        self.ops, self.n_iters = list(ops), n_iters

    def run(self, first, count, stream, use_graph=True):
        run_program(self.ops, count, first)

    def run_range(self, it, op_first, op_count, stream):
        """cds_plan_run_range: operators [op_first, op_first + op_count) of iteration ``it`` (CDS_OPF_ONCE ones skipped)"""
        keep = [op for op in self.ops[op_first:op_first + op_count] if not (op.flags & cabi.OPF_ONCE)]
        run_program(keep, 1, it)

    def launches_per_iter(self):
        return len(self.ops)

    def close(self):
        pass
