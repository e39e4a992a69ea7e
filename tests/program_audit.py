"""TEST INFRASTRUCTURE: audit of a lowered sampler program at its real size, operator by operator and iteration by iteration.

The operands of every descriptor are decoded by tests/emulator.py (``Owned`` memory: views of the tensors that own them,
every operand's extent checked against its owner), on the device for a real plan or on the host for the interpreter's
``Handle``, so the kernels are judged against the same reading of include/cds.h as the CPU lowering tests.

``Auditor.audit_iteration`` runs each operator of one iteration alone (``run_range(it, i, 1)``) from the current state and
checks:
  - its output against tests/opref.py in fp64, computed from the same state before the launch, under the derived bound of
    the operator's kernel family: conv_cases.check (+ gn_offset_atol for GroupNorm on tensor cores), attn_cases.bound,
    mha_cases.bound, the LNMOD bound of tests/test_elementwise_gpu.py; UPDATE / PREP / CAST bit for bit against the
    interpreter run on host copies of their operands;
  - that nothing outside its declared outputs changed: every other owner keeps its fingerprint, and inside the owner of an
    output view the elements outside the view keep theirs;
  - every adjacent CONV -> LNMOD pair once more as ``run_range(it, i, 2)`` from the same inputs (one linear_ln launch when
    the plan fused the pair): X against fp64, Y against the LayerNorm of the X the kernel stored.
The largest error as a fraction of the bound is recorded per (program, kernel instantiation).
Never imported by the product.
"""
import math

import torch

import attn_cases
import conv_cases
import emulator
import mha_cases
import mha_ref
import opref
from cleandiffuser_b200.engine import cabi

F64 = torch.float64
LN_ATOL = 1e-4                                  # the LNMOD bound of tests/test_elementwise_gpu.py: ATOL s + r_out |ref|
R_OUT = {cabi.F32: 0.0, cabi.TF32: 2.0 ** -10, cabi.BF16: 2.0 ** -8}
CHUNK = 1 << 24                                 # output elements per fp64 reference chunk (128 MB)
PARK = 1 << 30                                  # fp64 references kept across a launch wait in host memory above this size
DT_NAME = {cabi.F32: "f32", cabi.TF32: "tf32", cabi.BF16: "bf16"}
KIND_NAME = {cabi.OP_CONV: "conv", cabi.OP_UPDATE: "update", cabi.OP_LNMOD: "lnmod", cabi.OP_ATTN: "attn",
             cabi.OP_PREP: "prep", cabi.OP_CAST: "cast", cabi.OP_MHA: "mha"}


def plan_owners(plan):
    """the tensors a SamplerPlan's descriptors may point into: every kept buffer and packed weight copy of the root program
    (which holds the branch programs' as well), and the network's parameters and buffers"""
    keep = [t for t in plan.program.keep if isinstance(t, torch.Tensor)]
    return keep + list(plan.net.parameters()) + list(plan.net.buffers())


def declared_outputs(op):
    """(ptr, shape, strides, dtype) of every view operator ``op`` may write"""
    k = op.kind
    if k == cabi.OP_CONV:
        c = op.u.conv
        return [(c.out, (c.batch, c.L_out * c.phases, c.C_out), (c.out_bstride, c.out_lstride, 1), c.out_dtype)]
    if k == cabi.OP_LNMOD:
        m = op.u.lnmod
        return [(m.out, (m.batch, m.L, m.C), (m.L * m.C, m.C, 1), m.out_dtype)]
    if k == cabi.OP_ATTN:
        a = op.u.attn
        return [(a.out, (a.batch, a.L, a.C), (a.L * a.C, a.C, 1), a.out_dtype)]
    if k == cabi.OP_MHA:
        m = op.u.mha
        return [(m.out, (m.batch, m.Lq, m.C), (m.out_bstride, m.out_lstride, 1), m.out_dtype)]
    if k == cabi.OP_CAST:
        c = op.u.cast
        return [(c.out, (c.batch, c.L, c.C_out), (c.L * c.C_out, c.C_out, 1), c.out_dtype)]
    if k == cabi.OP_PREP:
        p = op.u.prep
        n = p.batch * p.row
        return [(p.x, (n,), (1,), cabi.F32), (p.xin, (n,), (1,), cabi.F32)]
    assert k == cabi.OP_UPDATE, k
    u = op.u.update
    outs = [(u.x, (u.batch, u.row), (u.row, 1), cabi.F32)]
    outs += [(p, (u.batch, u.row), (u.row, 1), cabi.F32) for p in (u.xhat_prev, u.aux) if p]
    if u.x_cast:
        outs.append((u.x_cast, (u.batch * u.row // u.cast_C_in, u.cast_C_in), (u.cast_C_out, 1), u.x_cast_dtype))
    return outs


def instantiation(op):
    """name of the kernel instantiation that runs ``op`` (cabi.conv_choice / attn_choice / mha_choice)"""
    if op.kind == cabi.OP_CONV:
        ch = cabi.conv_choice(op.u.conv)
        key = conv_cases.choice_key(ch)
        return f"conv {key[0]}" + "".join(f" {v}" for v in key[1:]) + f" -> {DT_NAME[op.u.conv.out_dtype]}"
    if op.kind == cabi.OP_ATTN:
        ch = cabi.attn_choice(op.u.attn)
        return f"attn {ch['family']} {ch['param']} -> {DT_NAME[op.u.attn.out_dtype]}"
    if op.kind == cabi.OP_MHA:
        ch = cabi.mha_choice(op.u.mha)
        return f"mha hpl {ch['hpl']}{' bf16' if ch['bf16'] else ''} -> {DT_NAME[op.u.mha.out_dtype]}"
    if op.kind == cabi.OP_LNMOD:
        return f"lnmod -> {DT_NAME[op.u.lnmod.out_dtype]}"
    if op.kind == cabi.OP_CAST:
        return f"cast {'once ' if op.flags & cabi.OPF_ONCE else ''}-> {DT_NAME[op.u.cast.out_dtype]}"
    if op.kind == cabi.OP_UPDATE and op.u.update.x_cast:
        return f"update + x_cast -> {DT_NAME[op.u.update.x_cast_dtype]}"
    return KIND_NAME[op.kind]


def is_pair(ops, i):
    """operators i, i + 1 are an adjacent CONV -> LNMOD pair of the iteration program"""
    return (i + 1 < len(ops) and ops[i].kind == cabi.OP_CONV and ops[i + 1].kind == cabi.OP_LNMOD
            and not (ops[i].flags | ops[i + 1].flags) & cabi.OPF_ONCE)


def _bits(t):
    flat = t.detach().reshape(-1)
    return flat.view({1: torch.int8, 2: torch.int16, 4: torch.int32, 8: torch.int64}[flat.element_size()])


def same_bits(a, b):
    """bitwise equality (same shape and dtype)"""
    return bool(torch.equal(_bits(a.contiguous()), _bits(b.contiguous())))


def _rows(t, b0, b1):
    """rows [b0, b1) of an operand the op reads at row b % len(t) (in_batch_mod / res_batch_mod / a broadcast row)"""
    if t is None or t.shape[0] >= b1:
        return None if t is None else t[b0:b1]
    return t[torch.arange(b0, b1, device=t.device) % t.shape[0]]


def _chunks(B, per_row, align=1):
    step = max(align, CHUNK // max(1, per_row) // align * align)
    return [(b0, min(B, b0 + step)) for b0 in range(0, B, step)]


def _park(t, host):
    return t.cpu() if host and torch.is_tensor(t) else t


def _frac(err, bound, finite):
    ratio = torch.where(bound > 0, err / bound.clamp_min(1e-300), torch.where(err > 0, math.inf, 0.0))
    return float(ratio.max()) if finite else math.inf


class Auditor:
    """Audits the operator program ``ops`` run by ``handle`` (a cabi.Plan, or an emulator / mha_ref Handle over the same
    descriptors).  ``owners``: the tensors the descriptors point into (plan_owners); ``sync``: waits for the handle's work."""

    def __init__(self, name, ops, handle, owners, stream=0, sync=lambda: None):
        self.name, self.ops, self.handle, self.stream, self.sync = name, list(ops), handle, stream, sync
        self.mem = emulator.Owned(owners)
        self.worst = {}                       # instantiation -> (largest fraction of the bound, where)
        self.pairs = 0                        # CONV -> LNMOD pairs run as one range
        self.failures = []

    # ---- bookkeeping ---------------------------------------------------------------------------------------------------
    def _record(self, inst, frac, where):
        if frac > self.worst.get(inst, (-1.0, ""))[0]:
            self.worst[inst] = (frac, where)
        if not frac <= 1.0:
            self.failures.append(f"{self.name} {where} [{inst}]: {frac:.3g} of the bound")

    def _views(self, op):
        return [emulator.view(self.mem, *o) for o in declared_outputs(op)]

    def _fingerprints(self):
        """per owner, the sum of its bit patterns: any single changed element changes it"""
        return torch.stack([_bits(t).sum(dtype=torch.int64) for t in self.mem.owners]).tolist()

    def _sums(self, ops):
        """(owner index, sum of the bit patterns) of every declared output view of ``ops``"""
        outs = [o for op in ops for o in declared_outputs(op)]
        if not outs:
            return []
        owners = [self.mem.owner(o[0], (2 if o[3] == cabi.BF16 else 4) * emulator._span(o[1], o[2])) for o in outs]
        sums = torch.stack([_bits(emulator.view(self.mem, *o)).sum(dtype=torch.int64) for o in outs]).tolist()
        return list(zip(owners, sums))

    def _stray_writes(self, before, ops, sums_before, where):
        """every owner but the outputs' keeps its fingerprint; inside an output's owner, only the view changed: the owner's
        fingerprint minus its views' sums is the same before and after (the sums are exact int64 arithmetic)"""
        after, sums_after = self._fingerprints(), self._sums(ops)
        outside_before, outside_after = list(before), list(after)
        for (k, sb), (_, sa) in zip(sums_before, sums_after):
            outside_before[k] -= sb
            outside_after[k] -= sa
        for k, (a, b) in enumerate(zip(outside_before, outside_after)):
            if a != b:
                t = self.mem.owners[k]
                self.failures.append(f"{self.name} {where}: a write outside the declared outputs, in the owner "
                                     f"{tuple(t.shape)} {t.dtype}")
        return after

    # ---- references (computed from the state before the launch); each returns check() -> [(frac, label)] --------------
    def _conv(self, c, it, lazy=True):
        """``lazy``: the fp64 reference is computed chunk by chunk after the launch (a first pass before it only sums |ref| for
        the bound's scale s) -- possible when the launch cannot change the conv's operands, i.e. no operand shares a tensor
        with the output; otherwise every chunk is computed before the launch and kept (in host memory when large)."""
        x, w, kw, out = emulator.conv_operands(c, it, self.mem)
        B, div = c.batch, kw["sample_row_div"]
        gn = c.groups > 0 and c.math in cabi.TC_MODES
        inputs = [t for t in (x, kw.get("res"), kw.get("res_in")) if t is not None]
        lazy = lazy and all(t.untyped_storage().data_ptr() != out.untyped_storage().data_ptr() for t in inputs)

        def chunk(b0, b1):
            k = dict(kw, batch=b1 - b0)
            for n in ("bias", "scale", "shift"):
                if k[n] is not None and k[n].dim() == 2:
                    k[n] = k[n][b0 // div:(b1 + div - 1) // div]
            for n in ("res", "res_in"):
                if n in k:
                    k[n] = _rows(k[n], b0, b1)
            xc = _rows(x, b0, b1)
            ref = opref.conv(xc, w, **k)
            extra = 0.0
            if gn:
                pre = opref.conv(xc, w, batch=b1 - b0, L_out=c.L_out, taps=c.taps, stride=c.stride, pad=c.pad,
                                 math_mode=c.math, bias=k["bias"], sample_row_div=div)
                extra = conv_cases.gn_offset_atol(pre, c.groups, kw["gamma"])
            return ref, extra

        parts, total = [], 0.0
        park = 8 * B * c.L_out * c.phases * c.C_out > PARK
        for b0, b1 in _chunks(B, c.L_out * c.phases * c.C_out, div):
            ref, extra = chunk(b0, b1)
            total += float(ref.abs().sum())
            parts.append((b0, b1, None if lazy else _park(ref, park), None if lazy else _park(extra, park)))
        s = max(1.0, total / max(1, B * c.L_out * c.phases * c.C_out))

        def check():
            res = []
            for b0, b1, ref, extra in parts:
                if lazy:
                    ref, extra = chunk(b0, b1)
                extra = extra.to(out.device) if torch.is_tensor(extra) else extra
                ok, frac, msg = conv_cases.check({"out_dtype": c.out_dtype}, out[b0:b1].float(), ref.to(out.device), extra,
                                                 s=s)
                res.append((frac if ok or frac > 1 else math.inf, f"rows {b0}..{b1}: {msg}"))
            return res
        return check

    def _lnmod(self, m, x_state=None):
        x, sh, sc, out = emulator.lnmod_operands(m, self.mem)
        parts, total = [], 0.0
        park = 8 * m.batch * m.L * m.C > PARK
        for b0, b1 in _chunks(m.batch, m.L * m.C):
            ref = opref.lnmod(x[b0:b1], sh[b0:b1], sc[b0:b1], m.eps)
            total += float(ref.abs().sum())
            parts.append((b0, b1, _park(ref, park)))
        s = max(1.0, total / max(1, m.batch * m.L * m.C))

        def check():
            res = []
            for b0, b1, ref in parts:
                y, ref = out[b0:b1].float(), ref.to(out.device)
                err = (y.to(F64) - ref).abs()
                frac = _frac(err, LN_ATOL * s + R_OUT[m.out_dtype] * ref.abs(), bool(torch.isfinite(y).all()))
                if m.out_dtype == cabi.TF32 and int((y.contiguous().view(torch.int32) & 0x1FFF).abs().max()) != 0:
                    frac = math.inf
                res.append((frac, f"rows {b0}..{b1}"))
            return res
        return check

    def _attn(self, a):
        qkv, out = emulator.attn_operands(a, self.mem)
        ch = cabi.attn_choice(a)
        case = dict(want=(ch["family"], ch["param"]), heads=a.heads, hd=a.C // a.heads, L=a.L)
        parts, park = [], 16 * a.batch * a.L * a.C > PARK
        for b0, b1 in _chunks(a.batch, a.heads * a.L * max(a.L, a.C // a.heads)):
            ref = opref.attn(qkv[b0:b1], a.heads, a.qkv_dtype)
            parts.append((b0, b1, _park(ref, park), _park(attn_cases.bound(case, qkv[b0:b1], ref, a.out_dtype), park)))

        def check():
            res = []
            for b0, b1, ref, bound in parts:
                y = out[b0:b1].float()
                err = (y.to(F64) - ref.to(y.device)).abs()
                res.append((_frac(err, bound.to(y.device), bool(torch.isfinite(y).all())), f"rows {b0}..{b1}"))
            return res
        return check

    def _mha(self, m, it):
        q, kv, out, both = mha_ref.mha_operands(m, it, self.mem)
        diag = m.diag if m.masked else None
        case = dict(heads=m.heads, hd=m.C // m.heads, diag=diag, kv="both" if both else "one")
        parts, park = [], 16 * m.batch * m.Lq * m.C > PARK
        for b0, b1 in _chunks(m.batch, m.heads * m.Lq * max(m.Lk, m.C // m.heads)):
            ref = mha_ref.mha(q[b0:b1], kv[b0:b1], m.heads, diag)
            bound = mha_cases.bound(case, q[b0:b1], kv[b0:b1], ref, m.out_dtype, kv_sum=both)
            parts.append((b0, b1, _park(ref, park), _park(bound, park)))

        def check():
            res = []
            for b0, b1, ref, bound in parts:
                y = out[b0:b1].float()
                err = (y.to(F64) - ref.to(y.device)).abs()
                res.append((_frac(err, bound.to(y.device), bool(torch.isfinite(y).all())), f"rows {b0}..{b1}"))
            return res
        return check

    def _exact(self, op, it):
        """UPDATE / PREP / CAST: the interpreter on host copies of the operands; the kernel must give the same bits"""
        host = emulator.Owned(self.mem.owners, host=True)
        if op.kind == cabi.OP_UPDATE:
            emulator.run_update(op.u.update, it, host)
        elif op.kind == cabi.OP_PREP:
            emulator.run_prep(op.u.prep, it, host)
        else:
            emulator.run_cast(op.u.cast, host)
        outs = declared_outputs(op)
        want = [emulator.view(host, *o) for o in outs]

        def check():
            got = [emulator.view(self.mem, *o) for o in outs]
            return [(0.0 if same_bits(g.cpu(), w) else math.inf, f"output {j} bit for bit")
                    for j, (g, w) in enumerate(zip(got, want))]
        return check

    def reference(self, op, it, lazy=True):
        if op.kind == cabi.OP_CONV:
            return self._conv(op.u.conv, it, lazy)
        if op.kind == cabi.OP_LNMOD:
            return self._lnmod(op.u.lnmod)
        if op.kind == cabi.OP_ATTN:
            return self._attn(op.u.attn)
        if op.kind == cabi.OP_MHA:
            return self._mha(op.u.mha, it)
        return self._exact(op, it)

    # ---- the audit -------------------------------------------------------------------------------------------------------
    def _launch(self, it, i, n):
        self.handle.run_range(it, i, n, self.stream)
        self.sync()

    def audit_once(self, first):
        """the CDS_OPF_ONCE operators, through run(first, 0)"""
        once = [op for op in self.ops if op.flags & cabi.OPF_ONCE]
        if not once:
            return
        checks = [self.reference(op, first) for op in once]
        before, sums = self._fingerprints(), self._sums(once)
        self.handle.run(first, 0, self.stream, False)
        self.sync()
        for op, chk in zip(once, checks):
            for frac, label in chk():
                self._record(instantiation(op), frac, f"once op: {label}")
        self._stray_writes(before, once, sums, "once ops")

    def audit_iteration(self, it):
        """every operator of iteration ``it`` alone, then every CONV -> LNMOD pair as one range; leaves the state of the
        iteration's end"""
        ops = self.ops
        fp = self._fingerprints()
        pair_in = None                                 # (conv index, saved outputs of both, conv check) of an open pair
        for i, op in enumerate(ops):
            if op.flags & cabi.OPF_ONCE:
                continue
            where = f"it {it} op {i} ({KIND_NAME[op.kind]})"
            if is_pair(ops, i):
                pair_in = (i, [v.clone() for o in (op, ops[i + 1]) for v in self._views(o)], None)
            check = self.reference(op, it, lazy=not is_pair(ops, i))     # a pair's conv check is used again after the pair
            sums = self._sums([op])
            self._launch(it, i, 1)
            for frac, label in check():
                self._record(instantiation(op), frac, f"{where} {label}")
            fp = self._stray_writes(fp, [op], sums, where)
            if pair_in is not None and pair_in[0] == i:
                pair_in = (i, pair_in[1], check)
            elif pair_in is not None and pair_in[0] == i - 1:
                fp = self._pair(it, i - 1, pair_in, fp)
                pair_in = None

    def _pair(self, it, i, pair_in, fp):
        """operators i, i + 1 once more as one range from the inputs they had: X against the fp64 reference of the conv
        (computed before operator i ran), Y against the LayerNorm of the X the kernel stored"""
        ops = self.ops
        _, saved, conv_check = pair_in
        views = [v for o in (ops[i], ops[i + 1]) for v in self._views(o)]
        for v, s in zip(views, saved):
            v.copy_(s)
        before, sums = self._fingerprints(), self._sums([ops[i], ops[i + 1]])
        self._launch(it, i, 2)
        self.pairs += 1
        where = f"it {it} ops {i},{i + 1} (conv -> lnmod as one range)"
        for frac, label in conv_check():
            self._record(instantiation(ops[i]) + " [pair]", frac, f"{where} X {label}")
        for frac, label in self._lnmod(ops[i + 1].u.lnmod)():
            self._record(instantiation(ops[i + 1]) + " [pair]", frac, f"{where} Y {label}")
        return self._stray_writes(before, [ops[i], ops[i + 1]], sums, where)


# ---- whole iterations -------------------------------------------------------------------------------------------------
def written_owners(mem, ops):
    """indices of the owners some operator of ``ops`` writes"""
    idx = set()
    for op in ops:
        for ptr, shape, strides, dt in declared_outputs(op):
            idx.add(mem.owner(ptr, (2 if dt == cabi.BF16 else 4) * emulator._span(shape, strides)))
    return sorted(idx)


def run_op_by_op(handle, ops, first, count, stream, sync, pairs):
    """iterations [first, first + count) one operator at a time with a synchronisation after each (the CDS_OPF_ONCE operators
    first, as cds_plan_run does); ``pairs``: adjacent CONV -> LNMOD pairs run as one range (one launch where the plan fused
    them)"""
    if any(op.flags & cabi.OPF_ONCE for op in ops):
        handle.run(first, 0, stream, False)
        sync()
    for it in range(first, first + count):
        i = 0
        while i < len(ops):
            if ops[i].flags & cabi.OPF_ONCE:
                i += 1
                continue
            n = 2 if pairs and is_pair(ops, i) else 1
            handle.run_range(it, i, n, stream)
            sync()
            i += n


def fused_pairs(handle, ops):
    """number of CONV -> LNMOD pairs the plan runs as one launch, from launches_per_iter(): one launch per operator of the
    iteration program, one fewer per fused pair, and one more for the iteration-counter advance unless the last operator,
    a solver update of a single-branch program, advances it itself"""
    body = [op for op in ops if not op.flags & cabi.OPF_ONCE]
    branches = 1 + max((op.flags & 0xFF00) >> cabi.OPF_BRANCH_SHIFT for op in ops)
    advance = 0 if (branches == 1 and body and body[-1].kind == cabi.OP_UPDATE) else 1
    return len(body) + advance - handle.launches_per_iter()


def report_lines(worst):
    """table rows: program, instantiation, largest fraction of the bound, where"""
    lines = [f"{'program':<14} {'kernel instantiation':<48} {'worst':>7}  where"]
    for (prog, inst), (frac, where) in sorted(worst.items()):
        lines.append(f"{prog:<14} {inst:<48} {frac:>7.3f}  {where}")
    return lines
