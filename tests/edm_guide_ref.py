"""TEST INFRASTRUCTURE: semantics of CDS_OP_UPDATE's guidance operand (include/cds.h: ``guide`` / ``guide_s``, kinds
CDS_UPD_EDM / CDS_UPD_EDM_HEUN): D <- D + guide_s[iter] * guide between the c_skip / c_out combine and the clip, fp32 multiply
then fp32 add.  ``register(monkeypatch)`` teaches it to the interpreter (tests/emulator.py) for the duration of one test, the
way tests/few_step_grad_ref.py adds its operators; tests/program_audit.py checks UPDATE bit for bit through the interpreter, so
the audit follows, and its instantiation name tells the guided update apart.  The guided EDM kinds are restated here in full, in
the kernel's fp32 order, because the term enters between two operations of the interpreter's own EDM branch."""
import numpy as np

from cleandiffuser_b200.diffusion import solvers as S
from cleandiffuser_b200.engine import cabi


def guide_operands(u, it, mem):
    """(guidance scale of iteration ``it``, gradient (batch, row)) of an update descriptor with a guidance operand"""
    import emulator
    s = emulator._arr(u.guide_s + 4 * it, (1,), (1,), mem)[0]
    return np.float32(s), emulator._arr(u.guide, (u.batch, u.row), (u.row, 1), mem)


def run_guided_edm_update(u, it, mem):
    """kinds EDM / EDM_HEUN with the guidance term, as solver_update_value computes them (csrc/elementwise.cuh)"""
    import emulator
    f = np.float32
    row = emulator._row(u.coef, it, mem)
    sigma, k0, k1, k2, k4 = f(row[S.R_SIGMA]), f(row[S.R_K0]), f(row[S.R_K1]), f(row[S.R_K2]), f(row[S.R_K4])
    kind = int(row[S.R_KIND])
    shape, st = (u.batch, u.row), (u.row, 1)
    x = emulator._arr(u.x, shape, st, mem)
    pr = emulator._arr(u.pred, shape, st, mem).copy()
    s, g = guide_operands(u, it, mem)
    d = (k0 * x + k1 * pr).astype(f)
    d = (d + (s * g).astype(f)).astype(f)
    if u.final_clip:
        if u.x_min:
            d = np.maximum(d, emulator._arr(u.x_min, (u.row,), (1,), mem))
        if u.x_max:
            d = np.minimum(d, emulator._arr(u.x_max, (u.row,), (1,), mem))
    xw, dw = f(row[S.R_XW]), f(row[S.R_DW])
    slope = (xw * x - dw * d) if xw != 0 else (x - d) / sigma
    if kind == S.UPD_EDM:
        out = x - slope * k2
        if k4 != 0 and u.xhat_prev and u.aux:
            emulator._arr(u.xhat_prev, shape, st, mem)[...] = x
            emulator._arr(u.aux, shape, st, mem)[...] = slope
    else:
        hist = emulator._arr(u.xhat_prev, shape, st, mem) if u.xhat_prev else f(0)
        aux = emulator._arr(u.aux, shape, st, mem) if u.aux else f(0)
        out = hist - (aux + slope) / f(2) * k2
    if u.mask:
        m = emulator._arr(u.mask, (u.row,), (1,), mem)
        out = out * (f(1) - m) + emulator._arr(u.prior, shape, st, mem) * m
    x[...] = out.astype(f)
    if u.x_cast:
        rows = u.batch * u.row // u.cast_C_in
        emulator._store(u.x_cast, (rows, u.cast_C_in), (u.cast_C_out, 1), u.x_cast_dtype, x.reshape(rows, u.cast_C_in), mem)


def is_guided_edm(u, it, mem):
    import emulator
    return bool(u.guide) and int(emulator._row(u.coef, it, mem)[S.R_KIND]) in (S.UPD_EDM, S.UPD_EDM_HEUN)


def register(monkeypatch):
    """the guidance operand of CDS_OP_UPDATE in the interpreter and the program audit, until the test ends"""
    import emulator
    import program_audit as pa
    field, run_update = emulator.OPS[cabi.OP_UPDATE]

    def run(u, it, mem=emulator.HOST):
        if is_guided_edm(u, it, mem):
            run_guided_edm_update(u, it, mem)
        else:
            run_update(u, it, mem)
    monkeypatch.setitem(emulator.OPS, cabi.OP_UPDATE, (field, run))
    instantiation = pa.instantiation
    monkeypatch.setattr(pa, "instantiation", lambda op: "update + guide" if op.kind == cabi.OP_UPDATE and op.u.update.guide
                        else instantiation(op))
