"""TEST INFRASTRUCTURE: tests/program_audit.py's operator-by-operator audit extended to the operators QGPO's classifier
guidance adds: CDS_OP_HEAD_GRAD, CDS_OP_DGRAD with SiLU, and CDS_OP_STASH with SiLU or without a slot.  Those are checked
under tests/qgpo_ref.py's derived bounds; every other operator exactly as program_audit checks it.  ``Auditor`` and
``written_owners`` take the place of program_audit's for programs that hold QGPO's operators.  Never imported by the product.
"""
import numpy as np
import torch

import emulator
import grad_ref
import program_audit as pa
import qgpo_ref
from cleandiffuser_b200.engine import cabi

KIND_NAME = dict(pa.KIND_NAME)
KIND_NAME[cabi.OP_HEAD_GRAD] = "head_grad"


def declared_outputs(op, it):
    """pa.declared_outputs, plus HEAD_GRAD's seed and the activation output of a STASH without a slot"""
    if op.kind == cabi.OP_HEAD_GRAD:
        q = op.u.head_grad
        return [(q.seed, (q.rows,), (1,), cabi.F32)]
    if op.kind == cabi.OP_STASH and not op.u.stash.dst:
        s = op.u.stash
        return [(s.act_out, (s.n,), (1,), cabi.F32)]
    return pa.declared_outputs(op, it)


def instantiation(op):
    """pa.instantiation, with names for the SiLU variants and HEAD_GRAD"""
    if op.kind == cabi.OP_STASH and op.u.stash.act == cabi.ACT_SILU:
        return "stash silu" + ("" if op.u.stash.dst else " (no slot)")
    if op.kind == cabi.OP_DGRAD and op.u.dgrad.act == cabi.ACT_SILU:
        d = op.u.dgrad
        return f"dgrad silu{' +=' if d.accumulate else ''}{' +out_sum' if d.out_sum else ''}"
    if op.kind == cabi.OP_HEAD_GRAD:
        return f"head_grad{' silu' if op.u.head_grad.act == cabi.ACT_SILU else ''}"
    return pa.instantiation(op)


def written_owners(mem, ops, its):
    """pa.written_owners over this module's declared outputs"""
    idx = set()
    for it in its:
        for op in ops:
            for ptr, shape, strides, dt in declared_outputs(op, it):
                idx.add(mem.owner(ptr, (2 if dt == cabi.BF16 else 4) * emulator._span(shape, strides)))
    return sorted(idx)


class Auditor(pa.Auditor):
    """pa.Auditor that also knows QGPO's operators (see the module docstring)"""

    def _sums(self, ops, it):
        outs = [o for op in ops for o in declared_outputs(op, it)]
        if not outs:
            return []
        owners = [self.mem.owner(o[0], (2 if o[3] == cabi.BF16 else 4) * emulator._span(o[1], o[2])) for o in outs]
        sums = [int(pa._bits(emulator.view(self.mem, *o)).sum(dtype=torch.int64)) for o in outs]
        return list(zip(owners, sums))

    def _qgpo(self, op, it):
        """STASH / DGRAD with SiLU and HEAD_GRAD under qgpo_ref.silu_bound / dgrad_bound / head_grad_bound"""
        arr = self._host_arr()
        outs = declared_outputs(op, it)
        if op.kind == cabi.OP_HEAD_GRAD:
            q = op.u.head_grad
            h, w, b = arr(q.h, (q.rows, q.K), (q.ldh, 1)), arr(q.w, (q.K,), (1,)), arr(q.b, (1,), (1,))
            _, seed = qgpo_ref.head_grad(h, w, b, q.scale, q.act)
            return self._bounded(outs, [(seed, qgpo_ref.head_grad_bound(h, w, b, q.scale, q.act))])
        if op.kind == cabi.OP_STASH:
            s = op.u.stash
            src = arr(s.src, (s.n,), (1,)).copy()
            refs = []
            if s.dst:                          # the slot copy, bit for bit (zero bound)
                refs.append((src.astype(np.float64), 0.0))
            if s.act_out:
                refs.append((qgpo_ref.silu(src), qgpo_ref.silu_bound(src)) if s.act == cabi.ACT_SILU else
                            (grad_ref.act(s.act, src), grad_ref.mish_bound(src.astype(np.float64))))
            return self._bounded(outs, refs)
        d = op.u.dgrad
        dz, w = arr(d.dz, (d.rows, d.N), (d.ldz, 1)), arr(d.w, (d.N, d.K), (d.ldw, 1))
        z = arr(d.z + 4 * it * d.z_iter_stride, (d.rows, d.K), (d.K, 1))
        y = qgpo_ref.dgrad(dz, w, z, d.act)
        before = arr(d.out, (d.rows, d.K), (d.ldo, 1)).astype(np.float64) if d.accumulate else None
        refs = [(y if before is None else before + y, qgpo_ref.dgrad_bound(dz, w, z, d.act, before))]
        if d.out_sum:
            s0 = arr(d.out_sum, (d.rows, d.K), (d.K, 1)).astype(np.float64)
            refs.append((s0 + y, qgpo_ref.dgrad_bound(dz, w, z, d.act, s0)))
        return self._bounded(outs, refs)

    def reference(self, op, it):
        if qgpo_ref._ours(op) is not None:
            return self._qgpo(op, it)
        return super().reference(op, it)

    def audit_once(self, first):
        """pa.Auditor.audit_once with this module's instantiation names"""
        once = [op for op in self.ops if op.flags & cabi.OPF_ONCE]
        if not once:
            return
        checks = [self.reference(op, first) for op in once]
        before, sums = self._fingerprints(), self._sums(once, first)
        self.handle.run(first, 0, self.stream, False)
        self.sync()
        for op, chk in zip(once, checks):
            for frac, label in chk():
                self._record(instantiation(op), frac, f"once op: {label}")
        self._stray_writes(before, once, first, sums, "once ops")

    def audit_iteration(self, it):
        """pa.Auditor.audit_iteration with this module's operator and instantiation names"""
        fp = self._fingerprints()
        for i, op in enumerate(self.ops):
            if op.flags & cabi.OPF_ONCE:
                continue
            where = f"it {it} op {i} ({KIND_NAME[op.kind]})"
            check = self.reference(op, it)
            sums = self._sums([op], it)
            self._launch(it, i, 1)
            for frac, label in check():
                self._record(instantiation(op), frac, f"{where} {label}")
            fp = self._stray_writes(fp, [op], it, sums, where)
