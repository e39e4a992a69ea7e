"""TEST INFRASTRUCTURE: a numpy interpreter of the libcds operator program (include/cds.h semantics).

It lets the CPU test-suite execute the *lowered* program (``engine/lower.py`` output, with CPU tensors behind
the raw pointers) and compare it with the reference goldens, so that lowering bugs (wrong strides, offsets,
table columns, phase packing ...) are caught here without a GPU; the kernels themselves are then checked
against the same goldens on the H100.  Never imported by the product.

``OPS`` runs every operator kind; the fp64 semantics live in tests/opref.py (forward operators), tests/mha_ref.py,
tests/grad_ref.py (backward operators of a differentiable loop) and tests/cg_ref.py (classifier operators), and this module
is the one decoder of a descriptor's operands: every ``*_operands`` / ``run_*`` function takes ``(descriptor, iteration,
mem)``, with a memory backend ``mem`` -- ``RawHost`` (raw host addresses, no bounds check) or ``Owned`` (views of the
tensors that own the memory, on the host or the device, with every operand's extent checked against its owner).
tests/program_audit.py uses the same ``*_operands`` functions on the device state of a real plan.
"""
import bisect
import ctypes

import numpy as np
import torch

import cg_ref
import grad_ref
import mha_ref
import opref
from cleandiffuser_b200.engine import cabi

_TORCH_DT = {cabi.F32: torch.float32, cabi.TF32: torch.float32, cabi.BF16: torch.bfloat16}


def _span(shape, strides):
    """elements from the first element of a view to one past its last (strides >= 0)"""
    assert all(st >= 0 for st in strides), strides
    return 1 + sum((s - 1) * st for s, st in zip(shape, strides)) if all(s > 0 for s in shape) else 0


class RawHost:
    """Memory backend: host memory at raw addresses, read through ctypes with no bounds check (descriptors built by hand
    over CPU tensors, e.g. the operator cases of tests/test_elementwise_gpu.py)."""

    def view(self, ptr, shape, strides, dtype):
        n = max(1, _span(shape, strides))
        if dtype == cabi.BF16:
            flat = torch.from_numpy(np.ctypeslib.as_array((ctypes.c_int16 * n).from_address(ptr))).view(torch.bfloat16)
        else:
            flat = torch.from_numpy(np.ctypeslib.as_array((ctypes.c_float * n).from_address(ptr)))
        return flat.as_strided(shape, strides)


class Owned:
    """Memory backend: memory owned by known tensors, on any device.  Every operand must lie inside one owner -- its full
    extent, shape x strides x element size -- and is an ``as_strided`` view of that owner; an operand that reaches past
    its owner (or lies in no owner) raises.  ``host=True`` reads and writes host copies of the owners instead, taken at
    the first access to each, so that the numpy operators below can run on a device program's state without touching
    the device (``copies`` maps an owner's index to its copy)."""

    def __init__(self, owners, host=False):
        def span(t):
            return t.data_ptr(), t.data_ptr() + t.numel() * t.element_size()
        ts = sorted((t for t in owners if isinstance(t, torch.Tensor) and t.numel() > 0),
                    key=lambda t: (span(t)[0], -span(t)[1]))
        self.owners = []
        for t in ts:                          # a tensor inside another one (a view of it) is owned by the larger one
            if self.owners and span(t)[0] < span(self.owners[-1])[1]:
                assert span(t)[1] <= span(self.owners[-1])[1], \
                    f"owners overlap: {tuple(t.shape)} {t.dtype} at {t.data_ptr():#x} and {tuple(self.owners[-1].shape)}"
                continue
            self.owners.append(t)
        self.starts = [t.data_ptr() for t in self.owners]
        self.host, self.copies = host, {}

    def owner(self, ptr, nbytes):
        """index of the owner that holds bytes [ptr, ptr + nbytes)"""
        k = bisect.bisect_right(self.starts, ptr) - 1
        if k < 0:
            raise AssertionError(f"operand at {ptr:#x} ({nbytes} bytes) lies below every owning tensor")
        t = self.owners[k]
        end = t.data_ptr() + t.numel() * t.element_size()
        if ptr + nbytes > end:
            raise AssertionError(f"operand at {ptr:#x} ({nbytes} bytes) reaches {ptr + nbytes - end} bytes past its owner "
                                 f"{tuple(t.shape)} {t.dtype} at {t.data_ptr():#x}")
        return k

    def view(self, ptr, shape, strides, dtype):
        es = 2 if dtype == cabi.BF16 else 4
        k = self.owner(ptr, es * _span(shape, strides))
        t = self.owners[k]
        if self.host:
            if k not in self.copies:
                self.copies[k] = t.detach().to("cpu", copy=True)
            t = self.copies[k]
        assert t.is_contiguous()
        flat = t.detach().reshape(-1).view(_TORCH_DT[dtype])
        off, rem = divmod(ptr - self.starts[k], es)
        assert rem == 0, "misaligned operand"
        return flat.as_strided(shape, strides, flat.storage_offset() + off)


HOST = RawHost()


def view(mem, ptr, shape, strides, dtype):
    """torch view (fp32 or bf16, as stored) of the operand at ``ptr`` in memory backend ``mem``; strides in elements"""
    if not ptr:
        return None
    return mem.view(ptr, tuple(int(s) for s in shape), tuple(int(s) for s in strides), dtype)


def _arr(ptr, shape, strides, mem=HOST):
    """float32 numpy view of host memory; strides in floats."""
    v = view(mem, ptr, shape, strides, cabi.F32)
    return None if v is None else v.numpy()


def _bf16_to_f32(u16):
    return (u16.astype(np.uint32) << 16).view(np.float32)


def _f32_to_bf16(x):
    return torch.from_numpy(np.ascontiguousarray(x, dtype=np.float32)).to(torch.bfloat16).view(torch.int16).numpy().view(np.uint16)


def _rn_tf32(x):
    """fp32 -> nearest TF32 (ties away from zero): what producers store into a CDS_TF32 tensor"""
    u = np.ascontiguousarray(x, dtype=np.float32).view(np.uint32)
    return ((u + np.uint32(0x1000)) & np.uint32(0xFFFFE000)).view(np.float32)


def _load(ptr, shape, strides, dtype, mem=HOST):
    """float32 numpy COPY of an fp32 / bf16 activation view in host memory (strides in elements)."""
    return np.array(view(mem, ptr, shape, strides, dtype).float())


def _store(ptr, shape, strides, dtype, values, mem=HOST):
    """write ``values`` (torch or numpy, any float type) with the rounding of ``dtype``"""
    dst = view(mem, ptr, shape, strides, dtype)
    v = values if isinstance(values, torch.Tensor) else torch.from_numpy(np.ascontiguousarray(values, dtype=np.float32))
    dst.copy_(opref.store(v.to(dst.device), dtype).to(dst.dtype))


def vec(v, it, rows, n, row_div=1, mem=HOST):
    """cds_vec as tests/opref.py takes it: None, the (n,) step row, or the (owners, n) fp32 sum step + sample with one row per
    ``row_div`` rows (flattened token rows)"""
    out = None
    if v.step:
        out = view(mem, v.step + 4 * it * v.step_stride, (n,), (1,), cabi.F32)
    if v.sample:
        owners = (rows + row_div - 1) // row_div
        s = view(mem, v.sample, (owners, n), (v.sample_stride, 1), cabi.F32)
        out = s if out is None else s + out[None]
    return out


def conv_operands(c, it, mem=HOST):
    """(x, w, keyword arguments of opref.conv, output view) of a CDS_OP_CONV descriptor.  x, res and res_in are views in
    their stored dtype: opref reads them the way the kernel family of ``c.math`` does."""
    B, N = c.batch, c.C_out * c.phases
    bmod = c.in_batch_mod if c.in_batch_mod > 0 else B
    x = view(mem, c.in_, (bmod, c.L_in, c.C_in), (c.in_bstride, c.in_lstride, 1), c.in_dtype)
    tc = c.math in cabi.TC_MODES
    wdt = cabi.F32 if c.math == cabi.MATH_TF32_TC else cabi.BF16
    if tc:      # bf16 / fp32 [taps][C_out*phases][C_in]
        assert c.in_dtype == wdt or (wdt == cabi.F32 and c.in_dtype == cabi.TF32)
        w = view(mem, c.w, (c.taps, N, c.C_in), (N * c.C_in, c.C_in, 1), wdt).permute(0, 2, 1)
    else:
        w = view(mem, c.w, (c.taps, c.C_in, N), (c.C_in * N, N, 1), cabi.F32)
    div = c.sample_row_div if c.sample_row_div > 1 else 1
    kw = dict(batch=B, L_out=c.L_out, taps=c.taps, stride=c.stride, pad=c.pad, phases=c.phases, math_mode=c.math,
              act_kind=c.act, sample_row_div=div, bias=vec(c.bias, it, B, c.C_out, div, mem),
              scale=vec(c.scale, it, B, c.C_out, div, mem), shift=vec(c.shift, it, B, c.C_out, div, mem))
    if c.groups > 0:
        kw.update(groups=c.groups, gamma=view(mem, c.gn_gamma, (c.C_out,), (1,), cabi.F32),
                  beta=view(mem, c.gn_beta, (c.C_out,), (1,), cabi.F32), eps=c.gn_eps)
    rmod = c.res_batch_mod if c.res_batch_mod > 0 else B
    if c.res:
        kw["res"] = view(mem, c.res, (rmod if c.res_bstride else 1, c.L_out, c.C_out), (c.res_bstride, c.res_lstride, 1),
                         c.res_dtype)
    if c.res_w:
        kw["res_in"] = view(mem, c.res_in, (rmod, c.L_out, c.res_C), (c.res_in_bstride, c.res_in_lstride, 1), c.res_in_dtype)
        kw["res_w"] = view(mem, c.res_w, (c.C_out, c.res_C), (c.res_C, 1), wdt).T if tc else \
            view(mem, c.res_w, (c.res_C, N), (N, 1), cabi.F32)
        if c.res_bias:
            kw["res_bias"] = view(mem, c.res_bias, (c.C_out,), (1,), cabi.F32)
    out = view(mem, c.out, (B, c.L_out * c.phases, c.C_out), (c.out_bstride, c.out_lstride, 1), c.out_dtype)
    return x, w, kw, out


def run_conv(c, it, mem=HOST):
    """CDS_OP_CONV: the operands of the descriptor through tests/opref.py's fp64 reference, stored with the output's rounding"""
    x, w, kw, out = conv_operands(c, it, mem)
    y = opref.conv(x, w, **kw)
    out.copy_(opref.store(y, c.out_dtype).to(out.dtype))


def lnmod_operands(m, it, mem=HOST):
    """(x, shift, scale, output view) of a CDS_OP_LNMOD descriptor"""
    x = view(mem, m.in_, (m.batch, m.L, m.C), (m.L * m.C, m.C, 1), cabi.F32)
    sh = view(mem, m.shift, (m.batch, m.C), (m.mod_bstride, 1), cabi.F32)
    sc = view(mem, m.scale, (m.batch, m.C), (m.mod_bstride, 1), cabi.F32)
    return x, sh, sc, view(mem, m.out, (m.batch, m.L, m.C), (m.L * m.C, m.C, 1), m.out_dtype)


def run_lnmod(m, it, mem=HOST):
    x, sh, sc, out = lnmod_operands(m, it, mem)
    out.copy_(opref.store(opref.lnmod(x, sh, sc, m.eps), m.out_dtype).to(out.dtype))


def attn_operands(a, it, mem=HOST):
    """(q|k|v view as stored, output view) of a CDS_OP_ATTN descriptor"""
    qkv = view(mem, a.qkv, (a.batch, a.L, 3 * a.C), (a.L * 3 * a.C, 3 * a.C, 1), a.qkv_dtype)
    return qkv, view(mem, a.out, (a.batch, a.L, a.C), (a.L * a.C, a.C, 1), a.out_dtype)


def run_attn(a, it, mem=HOST):
    """CDS_OP_ATTN: q|k|v (bf16 values widened exactly) through tests/opref.py's fp64 reference"""
    qkv, out = attn_operands(a, it, mem)
    out.copy_(opref.store(opref.attn(qkv, a.heads, a.qkv_dtype), a.out_dtype).to(out.dtype))


def mha_operands(m, it, mem=HOST):
    """(q view as stored, k|v as the fp32 sum step + sample (the kernel's adds of the widened parts), output view, whether both
    k|v parts are present) of a CDS_OP_MHA descriptor"""
    esize = 2 if m.in_dtype == cabi.BF16 else 4
    q = view(mem, m.q, (m.batch, m.Lq, m.C), (m.q_bstride, m.q_lstride, 1), m.in_dtype)
    kv = None
    if m.kv_step:
        kv = view(mem, m.kv_step + esize * it * m.kv_step_stride, (m.Lk, 2 * m.C), (m.kv_step_lstride, 1),
                  m.in_dtype).float()[None].expand(m.batch, m.Lk, 2 * m.C)
    if m.kv_sample:
        s = view(mem, m.kv_sample, (m.batch, m.Lk, 2 * m.C), (m.kv_sample_bstride, m.kv_sample_lstride, 1),
                 m.in_dtype).float()
        kv = s if kv is None else s + kv
    out = view(mem, m.out, (m.batch, m.Lq, m.C), (m.out_bstride, m.out_lstride, 1), m.out_dtype)
    return q, kv, out, bool(m.kv_step and m.kv_sample)


def run_mha(m, it, mem=HOST):
    """CDS_OP_MHA: q and the k|v sum through tests/mha_ref.py"""
    q, kv, out, _ = mha_operands(m, it, mem)
    out.copy_(opref.store(mha_ref.mha(q, kv, m.heads, m.diag if m.masked else None), m.out_dtype).to(out.dtype))


def run_cast(k, it, mem=HOST):
    x = view(mem, k.in_, (k.batch, k.L, k.C_in), (k.L * k.C_in, k.C_in, 1), cabi.F32)
    y = torch.zeros((k.batch, k.L, k.C_out), dtype=torch.float32, device=x.device)
    y[..., :k.C_in] = x
    _store(k.out, (k.batch, k.L, k.C_out), (k.L * k.C_out, k.C_out, 1), k.out_dtype, y, mem)


def _row(coef, it, mem=HOST):
    return _arr(coef + 4 * it * cabi.ROW_FLOATS, (cabi.ROW_FLOATS,), (1,), mem)


def run_prep(p, it, mem=HOST):
    row = _row(p.coef, it, mem)
    n = p.batch * p.row
    x = _arr(p.x, (n,), (1,), mem)
    slot = int(row[8]) - 1
    if slot >= 0:
        x[...] = x + row[4] * _arr(p.noise + 4 * slot * n, (n,), (1,), mem)
    _arr(p.xin, (n,), (1,), mem)[...] = row[5] * x


def run_update(u, it, mem=HOST):
    f = np.float32
    row = _row(u.coef, it, mem)
    alpha, sigma, k0, k1, k2, k3, k4 = (f(row[i]) for i in range(7))
    kind, slot = int(row[7]), int(row[8]) - 1
    n = u.batch * u.row
    x = _arr(u.x, (u.batch, u.row), (u.row, 1), mem)
    pr = _arr(u.pred, (u.batch, u.row), (u.row, 1), mem).copy()
    if u.pred_uncond:
        pr = f(u.w_cfg) * pr + f(u.w_uncond) * _arr(u.pred_uncond, (u.batch, u.row), (u.row, 1), mem)
    xmin = _arr(u.x_min, (u.row,), (1,), mem) if u.x_min else None
    xmax = _arr(u.x_max, (u.row,), (1,), mem) if u.x_max else None
    slot_stride = u.noise_slot_stride if u.noise_slot_stride > 0 else n
    z = _arr(u.noise + 4 * slot * slot_stride, (u.batch, u.row), (u.row, 1), mem) if slot >= 0 else None
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
                _arr(u.xhat_prev, (u.batch, u.row), (u.row, 1), mem)[...] = x
                _arr(u.aux, (u.batch, u.row), (u.row, 1), mem)[...] = slope
        else:                               # (absent history buffers read as 0, as in the kernel)
            hist = _arr(u.xhat_prev, (u.batch, u.row), (u.row, 1), mem) if u.xhat_prev else f(0)
            aux = _arr(u.aux, (u.batch, u.row), (u.row, 1), mem) if u.aux else f(0)
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
            hist = _arr(u.xhat_prev, (u.batch, u.row), (u.row, 1), mem) if u.xhat_prev else None
            target = eps if kind == 2 else (k3 * xhat - k4 * (hist if hist is not None else f(0)) if kind == 4 else xhat)
            out = k0 * x - k1 * target
            if z is not None:
                out = out + k2 * z
            if hist is not None:
                hist[...] = xhat
    if u.mask:
        m = _arr(u.mask, (u.row,), (1,), mem)
        out = out * (f(1) - m) + _arr(u.prior, (u.batch, u.row), (u.row, 1), mem) * m
    x[...] = out.astype(np.float32)
    if u.x_cast:                     # bf16 channel-padded copy of the new x_t (pad channels untouched)
        rows = n // u.cast_C_in
        _store(u.x_cast, (rows, u.cast_C_in), (u.cast_C_out, 1), u.x_cast_dtype, x.reshape(rows, u.cast_C_in), mem)


# ---------------------------------------------------------------- backward operators (tests/grad_ref.py)
# Their operands are float32 numpy views (grad_ref's semantics are numpy code); _f32 stores an fp64 result
def _f32(v):
    return np.asarray(v, np.float64).astype(np.float32)


def stash_operands(s, it, mem=HOST):
    """(src, slot of iteration ``it`` or None, activation output or None) of a CDS_OP_STASH descriptor"""
    src = _arr(s.src, (s.n,), (1,), mem)
    slot = _arr(s.dst + 4 * it * s.dst_iter_stride, (s.n,), (1,), mem) if s.dst else None
    return src, slot, _arr(s.act_out, (s.n,), (1,), mem)


def run_stash(s, it, mem=HOST):
    src, slot, act_out = stash_operands(s, it, mem)
    if slot is not None:
        slot[...] = src
    if act_out is not None:
        act_out[...] = _f32(grad_ref.act(s.act, src))


def update_bwd_operands(u, it, mem=HOST):
    """(gx (read, then written), x, pred, keyword arguments of grad_ref.update_bwd, gpred view) of a CDS_OP_UPDATE_BWD
    descriptor"""
    shape, st = (u.batch, u.row), (u.row, 1)
    row = _arr(u.coef + 4 * it * u.coef_iter_stride, (cabi.ROW_FLOATS,), (1,), mem).astype(np.float64)
    kw = dict(alpha=row[0], sigma=row[1], k0=row[2], k1=row[3], kind=int(row[7]), predict_noise=bool(u.predict_noise),
              **{k: _arr(getattr(u, k), (u.row,), (1,), mem) for k in ("mask", "x_min", "x_max")})
    x = _arr(u.x + 4 * it * u.x_iter_stride, shape, st, mem)
    pr = _arr(u.pred + 4 * it * u.pred_iter_stride, shape, st, mem)
    return _arr(u.gx, shape, st, mem), x, pr, kw, _arr(u.gpred, shape, st, mem)


def run_update_bwd(u, it, mem=HOST):
    gx, x, pr, kw, gpred = update_bwd_operands(u, it, mem)
    gp, dx = grad_ref.update_bwd(gx, x, pr, **kw)
    gpred[...] = _f32(gp)
    gx[...] = _f32(dx)


def dgrad_operands(d, it, mem=HOST):
    """(dz, W, stashed pre-activation z of iteration ``it`` or None, output view, out_sum view or None) of a CDS_OP_DGRAD
    descriptor"""
    dz = _arr(d.dz, (d.rows, d.N), (d.ldz, 1), mem)
    w = _arr(d.w, (d.N, d.K), (d.ldw, 1), mem)
    z = _arr(d.z + 4 * it * d.z_iter_stride, (d.rows, d.K), (d.K, 1), mem) if d.z else None
    return dz, w, z, _arr(d.out, (d.rows, d.K), (d.ldo, 1), mem), _arr(d.out_sum, (d.rows, d.K), (d.K, 1), mem)


def run_dgrad(d, it, mem=HOST):
    dz, w, z, out, out_sum = dgrad_operands(d, it, mem)
    y = grad_ref.dgrad(dz, w, z, d.act)
    out[...] = _f32(out.astype(np.float64) + y) if d.accumulate else _f32(y)
    if out_sum is not None:
        out_sum[...] = _f32(out_sum.astype(np.float64) + y)


def wgrad_operands(g, it, mem=HOST):
    """(dz, h of iteration ``it``, dw view, bias-gradient row of iteration ``it`` or None) of a CDS_OP_WGRAD descriptor"""
    dz = _arr(g.dz, (g.rows, g.N), (g.ldz, 1), mem)
    h = _arr(g.h + 4 * it * g.h_iter_stride, (g.rows, g.K), (g.ldh, 1), mem)
    db = _arr(g.db + 4 * it * g.db_iter_stride, (g.N,), (1,), mem) if g.db else None
    return dz, h, _arr(g.dw, (g.N, g.K), (g.lddw, 1), mem), db


def run_wgrad(g, it, mem=HOST):
    dz, h, dw, db = wgrad_operands(g, it, mem)
    gw, gb = grad_ref.wgrad(dz, h, g.act)
    dw[...] = _f32(dw.astype(np.float64) + gw) if g.accumulate else _f32(gw)
    if db is not None:
        db[...] = _f32(db.astype(np.float64) + gb) if g.accumulate else _f32(gb)


# ---------------------------------------------------------------- classifier operators (tests/cg_ref.py)
def gn_operands(g, it, mem=HOST):
    """(h, gamma, beta, vec or None, res or None, output view) of a CDS_OP_GN descriptor"""
    act = (g.batch, g.L, g.C)
    h = view(mem, g.h, act, (g.h_bstride, g.h_lstride, 1), cabi.F32)
    gamma, beta = view(mem, g.gamma, (g.C,), (1,), cabi.F32), view(mem, g.beta, (g.C,), (1,), cabi.F32)
    res = view(mem, g.res, act, (g.res_bstride, g.res_lstride, 1), cabi.F32)
    out = view(mem, g.out, act, (g.out_bstride, g.out_lstride, 1), cabi.F32)
    return h, gamma, beta, vec(g.vec, it, g.batch, g.C, 1, mem), res, out


def run_gn(g, it, mem=HOST):
    h, gamma, beta, v, res, out = gn_operands(g, it, mem)
    out.copy_(opref.store(cg_ref.gn(h, gamma, beta, g.groups, g.eps, g.act, v, res), g.out_dtype))


def gn_bwd_operands(g, it, mem=HOST):
    """(h, gamma, beta, dout, dh view) of a CDS_OP_GN_BWD descriptor"""
    act = (g.batch, g.L, g.C)
    h = view(mem, g.h, act, (g.h_bstride, g.h_lstride, 1), cabi.F32)
    gamma, beta = view(mem, g.gamma, (g.C,), (1,), cabi.F32), view(mem, g.beta, (g.C,), (1,), cabi.F32)
    dout = view(mem, g.dout, act, (g.dout_bstride, g.dout_lstride, 1), cabi.F32)
    return h, gamma, beta, dout, view(mem, g.dh, act, (g.dh_bstride, g.dh_lstride, 1), cabi.F32)


def run_gn_bwd(g, it, mem=HOST):
    h, gamma, beta, dout, dh = gn_bwd_operands(g, it, mem)
    dh.copy_(opref.store(cg_ref.gn_bwd(h, gamma, beta, dout, g.groups, g.eps, g.act), g.dh_dtype))


def guide_operands(q, it, mem=HOST):
    """(guidance scale of iteration ``it``, pred view (read and written), gradient) of a CDS_OP_GUIDE descriptor"""
    s = view(mem, q.s + 4 * it, (1,), (1,), cabi.F32)[0]
    pred = view(mem, q.pred, (q.batch, q.L, q.C), (q.L * q.C, q.C, 1), cabi.F32)
    return s, pred, view(mem, q.g, (q.batch, q.L, q.C), (q.g_bstride, q.g_lstride, 1), cabi.F32)


def run_guide(q, it, mem=HOST):
    """fp32 multiply, then fp32 add: the kernel's exact arithmetic"""
    s, pred, g = guide_operands(q, it, mem)
    pred.copy_(pred + s * g)


def head_grad_operands(q, it, mem=HOST):
    """(h, w, b, seed view) of a CDS_OP_HEAD_GRAD descriptor, float32 numpy"""
    h = _arr(q.h, (q.rows, q.K), (q.ldh, 1), mem)
    return h, _arr(q.w, (q.K,), (1,), mem), _arr(q.b, (1,), (1,), mem), _arr(q.seed, (q.rows,), (1,), mem)


def run_head_grad(q, it, mem=HOST):
    h, w, b, seed = head_grad_operands(q, it, mem)
    seed[...] = _f32(cg_ref.head_grad(h, w, b, q.scale, q.act)[1])


# ---------------------------------------------------------------- programs
# every operator kind: (its field of the cds_op union, its runner)
OPS = {cabi.OP_CONV: ("conv", run_conv), cabi.OP_UPDATE: ("update", run_update), cabi.OP_LNMOD: ("lnmod", run_lnmod),
       cabi.OP_ATTN: ("attn", run_attn), cabi.OP_PREP: ("prep", run_prep), cabi.OP_CAST: ("cast", run_cast),
       cabi.OP_MHA: ("mha", run_mha), cabi.OP_STASH: ("stash", run_stash), cabi.OP_UPDATE_BWD: ("update_bwd", run_update_bwd),
       cabi.OP_DGRAD: ("dgrad", run_dgrad), cabi.OP_WGRAD: ("wgrad", run_wgrad), cabi.OP_GN: ("gn", run_gn),
       cabi.OP_GN_BWD: ("gn_bwd", run_gn_bwd), cabi.OP_GUIDE: ("guide", run_guide),
       cabi.OP_HEAD_GRAD: ("head_grad", run_head_grad)}


def run_program(ops, n_iters, first=0, mem=HOST):
    with np.errstate(over="ignore", invalid="ignore", divide="ignore"):
        for op in ops:                       # CDS_OPF_ONCE operators: once per run, before the first iteration
            if op.flags & cabi.OPF_ONCE:
                assert op.kind == cabi.OP_CAST, op.kind
                run_cast(op.u.cast, first, mem)
        for it in range(first, first + n_iters):
            for op in ops:
                if not op.flags & cabi.OPF_ONCE:
                    field, run = OPS[op.kind]
                    run(getattr(op.u, field), it, mem)


class Handle:
    """Stand-in for ``cabi.Plan`` that executes the program on this interpreter (tests patch ``runtime._make_handle``).
    ``owners``: the tensors the descriptors point into; every operand is then bounds-checked against its owner (``Owned``)."""

    def __init__(self, ops, n_iters, owners=None):
        self.ops, self.n_iters = list(ops), n_iters
        self.mem = HOST if owners is None else Owned(owners)

    def run(self, first, count, stream, use_graph=True):
        run_program(self.ops, count, first, self.mem)

    def run_range(self, it, op_first, op_count, stream):
        """cds_plan_run_range: operators [op_first, op_first + op_count) of iteration ``it`` (CDS_OPF_ONCE ones skipped)"""
        keep = [op for op in self.ops[op_first:op_first + op_count] if not (op.flags & cabi.OPF_ONCE)]
        run_program(keep, 1, it, self.mem)

    def launches_per_iter(self):
        return len(self.ops)

    def close(self):
        pass


def record_owners(monkeypatch):
    """Record every ``Program`` the lowering creates and every network it lowers, for the rest of a test; returns a function
    giving the tensors they own (kept buffers, packed weight copies, parameters and buffers): the ``owners`` of a Handle."""
    from cleandiffuser_b200.engine import lower, runtime
    progs, nets = [], []
    init, lower_denoiser = lower.Program.__init__, runtime.lower_denoiser

    def recording_init(self, *a, **k):
        init(self, *a, **k)
        progs.append(self)

    def recording_lower(p, net, *a, **k):
        nets.append(net)
        return lower_denoiser(p, net, *a, **k)
    monkeypatch.setattr(lower.Program, "__init__", recording_init)
    monkeypatch.setattr(runtime, "lower_denoiser", recording_lower)
    return lambda: [t for p in progs for t in p.keep if isinstance(t, torch.Tensor)] + \
        [t for n in nets for t in (*n.parameters(), *n.buffers())]


def emulate(monkeypatch):
    """For the rest of a test, the engine runs its programs on this interpreter: every device is usable, and each plan's
    handle is a ``Handle`` over the tensors the lowering records (``record_owners``), so every operand is bounds-checked"""
    from cleandiffuser_b200.engine import runtime
    monkeypatch.setattr(runtime, "_device_ok", lambda device: True)
    owners = record_owners(monkeypatch)
    monkeypatch.setattr(runtime, "_make_handle", lambda device, ops, n: Handle(ops, n, owners()))
