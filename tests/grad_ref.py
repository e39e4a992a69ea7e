"""TEST INFRASTRUCTURE: numpy semantics of the backward operators of a differentiable reverse loop (include/cds.h:
CDS_OP_STASH, CDS_OP_UPDATE_BWD, CDS_OP_DGRAD, CDS_OP_WGRAD), in fp64 with fp32 stores, like tests/opref.py does for the
forward operators.  ``run_program`` / ``Handle`` extend tests/emulator.py's interpreter with them (every other operator kind
is run by the emulator itself); the GPU parity tests compare the kernels against the same functions."""
import numpy as np

import emulator
from cleandiffuser_b200.engine import cabi


def mish(x):
    x = np.asarray(x, np.float64)
    return x * np.tanh(np.where(x > 20, x, np.log1p(np.exp(np.minimum(x, 20)))))


def mish_grad(x):
    """d/dx mish(x) (ATen: tanh(softplus(x)) + x sigmoid(x) (1 - tanh(softplus(x))^2))"""
    x = np.asarray(x, np.float64)
    tsp = np.tanh(np.logaddexp(0.0, x))
    sig = 1.0 / (1.0 + np.exp(-x))
    return tsp + x * sig * (1.0 - tsp * tsp)


def act(kind, x):
    return mish(x) if kind == cabi.ACT_MISH else np.asarray(x, np.float64)


def update_bwd(g, x, pr, *, alpha, sigma, k0, k1, kind, predict_noise, mask=None, x_min=None, x_max=None):
    """Backward of CDS_OP_UPDATE kinds DDPM / DDIM / EPS / X: (d pred, direct d x_n) from d x_{n+1} = g.  All arrays (batch, row)
    or broadcastable (row,) rows; torch.clip's gradient rule for tensor bounds (equal to a bound = not clipped)."""
    # the clip decisions are taken in the operands' own precision (an fp32 kernel compares fp32 bounds), the rest in fp64
    x_in, pr_in = np.asarray(x), np.asarray(pr)
    ft = x_in.dtype.type
    if predict_noise:
        lo = None if x_max is None else (x_in - ft(alpha) * np.asarray(x_max, x_in.dtype)) / ft(sigma)
        hi = None if x_min is None else (x_in - ft(alpha) * np.asarray(x_min, x_in.dtype)) / ft(sigma)
    else:
        lo = None if x_min is None else np.asarray(x_min, x_in.dtype)
        hi = None if x_max is None else np.asarray(x_max, x_in.dtype)
    g, x, pr = (np.asarray(v, np.float64) for v in (g, x, pr))
    if mask is not None:
        g = g * (1.0 - mask)
    dx, deps, dxhat = np.zeros_like(g), np.zeros_like(g), np.zeros_like(g)
    if kind == 0:          # DDPM   out = k0 (x - sigma eps) + k1 eps
        dx, deps = k0 * g, k1 * g - sigma * k0 * g
    elif kind == 1:        # DDIM   out = k0 (x - sigma eps) / alpha + k1 eps
        a = k0 * g / alpha
        dx, deps = a, k1 * g - sigma * a
    elif kind == 2:        # EPS    out = k0 x - k1 eps
        dx, deps = k0 * g, -k1 * g
    elif kind == 3:        # X      out = k0 x - k1 xhat
        dx, dxhat = k0 * g, -k1 * g
    else:
        raise ValueError(kind)
    if predict_noise:      # xhat = (x - sigma pc) / alpha
        dx = dx + dxhat / alpha
        dpc = deps - sigma * dxhat / alpha
    else:                  # eps = (x - alpha pc) / sigma
        dx = dx + deps / sigma
        dpc = dxhat - alpha * deps / sigma
    pr = pr_in
    zero = np.zeros_like(dpc)
    if lo is not None and hi is not None:
        gp = np.where((pr >= lo) & (pr <= hi), dpc, zero)
        glo = np.where((pr < lo) & (lo < hi), dpc, zero)
        ghi = np.where((pr > hi) | (hi < lo), dpc, zero)
    elif lo is not None:
        gp, glo, ghi = np.where(pr >= lo, dpc, zero), np.where(pr < lo, dpc, zero), zero
    elif hi is not None:
        gp, glo, ghi = np.where(pr <= hi, dpc, zero), zero, np.where(pr > hi, dpc, zero)
    else:
        gp, glo, ghi = dpc, zero, zero
    if predict_noise:
        dx = dx + glo / sigma + ghi / sigma
    return gp, dx


def dgrad(dz, w, z=None, act_kind=cabi.ACT_NONE):
    """(dz W) * act'(z) in fp64"""
    y = np.asarray(dz, np.float64) @ np.asarray(w, np.float64)
    if act_kind == cabi.ACT_MISH:
        y = y * mish_grad(z)
    return y


def wgrad(dz, h, act_kind=cabi.ACT_NONE):
    """(dz^T act(h), sum_rows dz) in fp64"""
    dz = np.asarray(dz, np.float64)
    return dz.T @ act(act_kind, h), dz.sum(0)


# ---------------------------------------------------------------- descriptor interpreters (memory backends of tests/emulator.py)
def _f32(v):
    return np.asarray(v, np.float64).astype(np.float32)


def run_stash(s, it, arr):
    src = arr(s.src, (s.n,), (1,))
    arr(s.dst + 4 * it * s.dst_iter_stride, (s.n,), (1,))[...] = src
    if s.act_out:
        arr(s.act_out, (s.n,), (1,))[...] = _f32(act(s.act, src))


def run_update_bwd(u, it, arr):
    row = arr(u.coef + 4 * it * u.coef_iter_stride, (cabi.ROW_FLOATS,), (1,)).astype(np.float64)
    shape, st = (u.batch, u.row), (u.row, 1)
    gx = arr(u.gx, shape, st)
    x = arr(u.x + 4 * it * u.x_iter_stride, shape, st)
    pr = arr(u.pred + 4 * it * u.pred_iter_stride, shape, st)
    vec = lambda p: None if not p else arr(p, (u.row,), (1,))          # noqa: E731
    gp, dx = update_bwd(gx, x, pr, alpha=row[0], sigma=row[1], k0=row[2], k1=row[3], kind=int(row[7]),
                        predict_noise=bool(u.predict_noise), mask=vec(u.mask), x_min=vec(u.x_min), x_max=vec(u.x_max))
    arr(u.gpred, shape, st)[...] = _f32(gp)
    gx[...] = _f32(dx)


def run_dgrad(d, it, arr):
    dz = arr(d.dz, (d.rows, d.N), (d.ldz, 1))
    w = arr(d.w, (d.N, d.K), (d.ldw, 1))
    z = arr(d.z + 4 * it * d.z_iter_stride, (d.rows, d.K), (d.K, 1)) if d.z else None
    y = dgrad(dz, w, z, d.act)
    out = arr(d.out, (d.rows, d.K), (d.ldo, 1))
    out[...] = _f32(out.astype(np.float64) + y) if d.accumulate else _f32(y)
    if d.out_sum:
        s = arr(d.out_sum, (d.rows, d.K), (d.K, 1))
        s[...] = _f32(s.astype(np.float64) + y)


def run_wgrad(g, it, arr):
    dz = arr(g.dz, (g.rows, g.N), (g.ldz, 1))
    h = arr(g.h + 4 * it * g.h_iter_stride, (g.rows, g.K), (g.ldh, 1))
    dw, db = wgrad(dz, h, g.act)
    out = arr(g.dw, (g.N, g.K), (g.lddw, 1))
    out[...] = _f32(out.astype(np.float64) + dw) if g.accumulate else _f32(dw)
    if g.db:
        b = arr(g.db + 4 * it * g.db_iter_stride, (g.N,), (1,))
        b[...] = _f32(b.astype(np.float64) + db) if g.accumulate else _f32(db)


# ---------------------------------------------------------------- programs with backward operators
_GRAD_OPS = {cabi.OP_STASH: (run_stash, "stash"), cabi.OP_UPDATE_BWD: (run_update_bwd, "update_bwd"),
             cabi.OP_DGRAD: (run_dgrad, "dgrad"), cabi.OP_WGRAD: (run_wgrad, "wgrad")}


def run_program(ops, n_iters, first=0, mem=emulator.HOST):
    """tests/emulator.py's run_program for programs that also hold backward operators: those run here, every other operator
    through the emulator (one operator at a time, so that program order is kept)."""
    arr = lambda ptr, shape, strides: emulator._arr(ptr, shape, strides, mem)       # noqa: E731
    with np.errstate(over="ignore", invalid="ignore", divide="ignore"):
        emulator.run_program([op for op in ops if op.flags & cabi.OPF_ONCE], 0, first, mem)   # CDS_OPF_ONCE operators
        for it in range(first, first + n_iters):
            for op in ops:
                if op.flags & cabi.OPF_ONCE:
                    continue
                if op.kind in _GRAD_OPS:
                    fn, field = _GRAD_OPS[op.kind]
                    fn(getattr(op.u, field), it, arr)
                else:
                    emulator.run_program([op], 1, it, mem)


class Handle(emulator.Handle):
    """emulator.Handle whose interpreter also runs the backward operators"""

    def run(self, first, count, stream, use_graph=True):
        run_program(self.ops, count, first, self.mem)

    def run_range(self, it, op_first, op_count, stream):
        keep = [op for op in self.ops[op_first:op_first + op_count] if not (op.flags & cabi.OPF_ONCE)]
        run_program(keep, 1, it, self.mem)
