"""TEST INFRASTRUCTURE: fp64 semantics and error bounds of what ``sample(requires_grad=True)`` with the consistency model adds
to the backward operators (include/cds.h, csrc/grad.cuh): CDS_OP_UPDATE_BWD's kind CM and CDS_OP_PREP's backward mode
(gxin != NULL).  ``register(monkeypatch)`` teaches them to the shared operator references for the duration of one test, the
way tests/relu_ref.py and tests/dit_grad_ref.py add theirs:
  - tests/emulator.py: the interpreter's UPDATE_BWD runner takes kind CM, its PREP runner the backward mode;
  - tests/program_audit.py: declared_outputs and instantiation of PREP's backward mode, and the Auditor's UPDATE_BWD reference
    (PREP's backward mode is checked bit for bit, like the forward PREP, through the patched interpreter).
Rectified flow adds nothing here: its Euler step is the EPS update, whose backward tests/grad_ref.py already describes."""
import numpy as np

import grad_ref
from cleandiffuser_b200.diffusion import solvers as S
from cleandiffuser_b200.engine import cabi

U32 = 2.0 ** -24


def cm_update_bwd(g, x, pr, *, k0, k1, mask=None, x_min=None, x_max=None):
    """Backward of the CM update out = clip(k0 x + k1 pred, x_min, x_max) (then fix_mask) -> (d pred, direct d x).  The clip
    decision is taken on f recomputed in the operands' own precision (the kernel's fp32 ops), with torch.clip's rule for tensor
    bounds: an f equal to a bound passes, none passes where x_min > x_max; the rest in fp64."""
    x_in, pr_in = np.asarray(x), np.asarray(pr)
    ft = x_in.dtype.type
    f = ft(k0) * x_in + ft(k1) * pr_in
    keep = np.ones(f.shape, bool)
    if x_min is not None:
        keep &= f >= np.asarray(x_min, x_in.dtype)
    if x_max is not None:
        keep &= f <= np.asarray(x_max, x_in.dtype)
    g = np.asarray(g, np.float64)
    if mask is not None:
        g = g * (1.0 - np.asarray(mask, np.float64))
    gf = np.where(keep, g, 0.0)
    return k1 * gf, k0 * gf


def update_bwd(g, x, pr, *, alpha, sigma, k0, k1, kind, predict_noise, mask=None, x_min=None, x_max=None):
    """tests/grad_ref.update_bwd with kind CM added"""
    if kind == S.UPD_CM:
        return cm_update_bwd(g, x, pr, k0=k0, k1=k1, mask=mask, x_min=x_min, x_max=x_max)
    return grad_ref.update_bwd(g, x, pr, alpha=alpha, sigma=sigma, k0=k0, k1=k1, kind=kind, predict_noise=predict_noise,
                               mask=mask, x_min=x_min, x_max=x_max)


def cm_update_bwd_bound(g, k0, k1):
    """kind CM: the mask's product and one product with k0 or k1, each within u: 4 u |g| (|k0| + |k1|)"""
    return 4 * U32 * np.abs(np.asarray(g, np.float64)) * (abs(k0) + abs(k1))


def update_bwd_bound(g, alpha, sigma, k0, k1, kind):
    if kind == S.UPD_CM:
        return cm_update_bwd_bound(g, k0, k1)
    return grad_ref.update_bwd_bound(g, alpha, sigma, k0, k1)


def prep_bwd(gx, gxin, k3):
    """PREP's backward mode in the kernel's arithmetic: fp32 product, then fp32 sum (exact, so the audit compares bits)"""
    gx, gxin = np.asarray(gx, np.float32), np.asarray(gxin, np.float32)
    return gx + np.float32(k3) * gxin


def is_prep_bwd(op):
    return op.kind == cabi.OP_PREP and bool(op.u.prep.gxin)


def prep_bwd_operands(p, it, mem):
    """(K3 of iteration ``it``, gx view (read and written), gxin) of a CDS_OP_PREP descriptor in backward mode"""
    import emulator
    n = p.batch * p.row
    row = emulator._arr(p.coef + 4 * it * p.coef_iter_stride, (cabi.ROW_FLOATS,), (1,), mem)
    return row[S.R_K3], emulator._arr(p.x, (n,), (1,), mem), emulator._arr(p.gxin, (n,), (1,), mem)


def run_prep_bwd(p, it, mem):
    k3, gx, gxin = prep_bwd_operands(p, it, mem)
    gx[...] = prep_bwd(gx, gxin, k3)


def run_update_bwd(u, it, mem):
    import emulator
    gx, x, pr, kw, gpred = emulator.update_bwd_operands(u, it, mem)
    gp, dx = update_bwd(gx, x, pr, **kw)
    gpred[...] = emulator._f32(gp)
    gx[...] = emulator._f32(dx)


def _audit_update_bwd(auditor, op, it):
    import emulator
    import program_audit as pa
    gx, x, pr, kw, _ = emulator.update_bwd_operands(op.u.update_bwd, it, auditor._host())
    gp, dx = update_bwd(gx, x, pr, **kw)
    bound = update_bwd_bound(gx, kw["alpha"], kw["sigma"], kw["k0"], kw["k1"], kw["kind"])
    return auditor._bounded(pa.declared_outputs(op, it), [(dx, bound), (gp, bound)])


def register(monkeypatch):
    """kind CM of CDS_OP_UPDATE_BWD and the backward mode of CDS_OP_PREP in the interpreter and the program audit, until the
    test ends"""
    import emulator
    import program_audit as pa
    field, run_prep = emulator.OPS[cabi.OP_PREP]
    monkeypatch.setitem(emulator.OPS, cabi.OP_PREP,
                        (field, lambda p, it, mem=emulator.HOST: run_prep_bwd(p, it, mem) if p.gxin else run_prep(p, it, mem)))
    monkeypatch.setitem(emulator.OPS, cabi.OP_UPDATE_BWD,
                        ("update_bwd", lambda u, it, mem=emulator.HOST: run_update_bwd(u, it, mem)))
    monkeypatch.setitem(pa.Auditor.REFERENCE, cabi.OP_UPDATE_BWD, _audit_update_bwd)
    declared, instantiation = pa.declared_outputs, pa.instantiation

    def declared_outputs(op, it):
        if is_prep_bwd(op):
            p = op.u.prep
            return [(p.x, (p.batch * p.row,), (1,), cabi.F32)]
        return declared(op, it)
    monkeypatch.setattr(pa, "declared_outputs", declared_outputs)
    monkeypatch.setattr(pa, "instantiation", lambda op: "prep bwd" if is_prep_bwd(op) else instantiation(op))
