"""TEST INFRASTRUCTURE: audit of a lowered sampler program at its real size, operator by operator and iteration by iteration.

The operands of every descriptor are decoded by tests/emulator.py (``Owned`` memory: views of the tensors that own them,
every operand's extent checked against its owner), on the device for a real plan or on the host for the interpreter's
``Handle``, so the kernels are judged against the same reading of include/cds.h as the CPU lowering tests.

``Auditor.audit_iteration`` runs each operator of one iteration alone (``run_range(it, i, 1)``) from the current state and
checks:
  - its output against tests/opref.py in fp64, computed from the same state before the launch, under the derived bound of
    the operator's kernel family: conv_cases.check (+ gn_offset_atol for GroupNorm on tensor cores), attn_cases.bound,
    mha_cases.bound, the LNMOD bound of tests/test_elementwise_gpu.py; UPDATE / PREP / CAST / GUIDE and STASH's slot
    copy bit for bit against the interpreter run on host copies of their operands; GN / GN_BWD / HEAD_GRAD under
    cg_ref.gn_bound / gn_bwd_bound / head_grad_bound, STASH's Mish or SiLU under grad_ref.ACT_BOUND, UPDATE_BWD / DGRAD /
    WGRAD under grad_ref.update_bwd_bound / dgrad_bound / wgrad_bound (accumulating outputs as before + contribution), the
    bounds the operator tests apply;
  - that nothing outside its declared outputs changed: every other owner keeps its fingerprint, and inside the owner of an
    output view the elements outside the view keep theirs.
The largest error as a fraction of the bound is recorded per (program, kernel instantiation).
Never imported by the product.
"""
import math

import numpy as np
import torch

import attn_cases
import cg_ref
import conv_cases
import emulator
import grad_ref
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
             cabi.OP_PREP: "prep", cabi.OP_CAST: "cast", cabi.OP_MHA: "mha", cabi.OP_STASH: "stash",
             cabi.OP_UPDATE_BWD: "update_bwd", cabi.OP_DGRAD: "dgrad", cabi.OP_WGRAD: "wgrad", cabi.OP_GN: "gn",
             cabi.OP_GN_BWD: "gn_bwd", cabi.OP_GUIDE: "guide", cabi.OP_HEAD_GRAD: "head_grad"}


def plan_owners(plan):
    """the tensors a SamplerPlan's descriptors may point into: every kept buffer and packed weight copy of the root program
    (which holds the branch programs' as well) and of a GradSamplerPlan's backward program, and the parameters and buffers
    of the network and of a lowered classifier"""
    progs = [plan.program] + ([plan.back] if getattr(plan, "back", None) is not None else [])
    keep = [t for p in progs for t in p.keep if isinstance(t, torch.Tensor)]
    nets = [plan.net] + ([plan.classifier.model_ema] if getattr(plan, "classifier", None) is not None else [])
    return keep + [t for n in nets for t in (*n.parameters(), *n.buffers())]


def declared_outputs(op, it):
    """(ptr, shape, strides, dtype) of every view operator ``op`` may write at iteration ``it`` (a stash slot and WGRAD's
    bias row move with the iteration)"""
    k = op.kind
    if k == cabi.OP_STASH:
        s = op.u.stash
        outs = [(s.dst + 4 * it * s.dst_iter_stride, (s.n,), (1,), cabi.F32)] if s.dst else []
        return outs + ([(s.act_out, (s.n,), (1,), cabi.F32)] if s.act_out else [])
    if k == cabi.OP_UPDATE_BWD:
        u = op.u.update_bwd
        return [(p, (u.batch, u.row), (u.row, 1), cabi.F32) for p in (u.gx, u.gpred)]
    if k == cabi.OP_DGRAD:
        d = op.u.dgrad
        outs = [(d.out, (d.rows, d.K), (d.ldo, 1), cabi.F32)]
        return outs + ([(d.out_sum, (d.rows, d.K), (d.K, 1), cabi.F32)] if d.out_sum else [])
    if k == cabi.OP_WGRAD:
        g = op.u.wgrad
        outs = [(g.dw, (g.N, g.K), (g.lddw, 1), cabi.F32)]
        return outs + ([(g.db + 4 * it * g.db_iter_stride, (g.N,), (1,), cabi.F32)] if g.db else [])
    if k == cabi.OP_GN:
        g = op.u.gn
        return [(g.out, (g.batch, g.L, g.C), (g.out_bstride, g.out_lstride, 1), g.out_dtype)]
    if k == cabi.OP_GN_BWD:
        g = op.u.gn_bwd
        return [(g.dh, (g.batch, g.L, g.C), (g.dh_bstride, g.dh_lstride, 1), g.dh_dtype)]
    if k == cabi.OP_GUIDE:
        q = op.u.guide
        return [(q.pred, (q.batch, q.L, q.C), (q.L * q.C, q.C, 1), cabi.F32)]
    if k == cabi.OP_HEAD_GRAD:
        q = op.u.head_grad
        return [(q.seed, (q.rows,), (1,), cabi.F32)]
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
    if op.kind == cabi.OP_GN:
        g = op.u.gn
        return f"gn{' +vec' if g.vec.step or g.vec.sample else ''}{' +res' if g.res else ''} -> {DT_NAME[g.out_dtype]}"
    if op.kind == cabi.OP_GN_BWD:
        return f"gn_bwd -> {DT_NAME[op.u.gn_bwd.dh_dtype]}"
    if op.kind == cabi.OP_STASH:
        s = op.u.stash
        if s.act == cabi.ACT_SILU:
            return "stash silu" + ("" if s.dst else " (no slot)")
        return "stash +act" if s.act_out else "stash"
    if op.kind == cabi.OP_UPDATE_BWD:
        u = op.u.update_bwd
        return f"update_bwd {'eps' if u.predict_noise else 'x0'}{' clip' if u.x_min or u.x_max else ''}" \
            f"{' mask' if u.mask else ''}"
    if op.kind == cabi.OP_DGRAD:
        d = op.u.dgrad
        act = {cabi.ACT_MISH: " mish", cabi.ACT_SILU: " silu"}.get(d.act, "")
        return f"dgrad{act}{' +=' if d.accumulate else ''}{' +out_sum' if d.out_sum else ''}"
    if op.kind == cabi.OP_WGRAD:
        g = op.u.wgrad
        return f"wgrad{' mish' if g.act == cabi.ACT_MISH else ''}{' +bias' if g.db else ''}"
    if op.kind == cabi.OP_HEAD_GRAD:
        return f"head_grad{' silu' if op.u.head_grad.act == cabi.ACT_SILU else ''}"
    return KIND_NAME[op.kind]


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
    """Audits the operator program ``ops`` run by ``handle`` (a cabi.Plan, or an emulator.Handle over the same descriptors).
    ``owners``: the tensors the descriptors point into (plan_owners); ``sync``: waits for the handle's work."""

    def __init__(self, name, ops, handle, owners, stream=0, sync=lambda: None):
        self.name, self.ops, self.handle, self.stream, self.sync = name, list(ops), handle, stream, sync
        self.mem = emulator.Owned(owners)
        self.worst = {}                       # instantiation -> (largest fraction of the bound, where)
        self.failures = []

    # ---- bookkeeping ---------------------------------------------------------------------------------------------------
    def _record(self, inst, frac, where):
        if frac > self.worst.get(inst, (-1.0, ""))[0]:
            self.worst[inst] = (frac, where)
        if not frac <= 1.0:
            self.failures.append(f"{self.name} {where} [{inst}]: {frac:.3g} of the bound")

    def _views(self, op, it):
        return [emulator.view(self.mem, *o) for o in declared_outputs(op, it)]

    def _fingerprints(self):
        """per owner, the sum of its bit patterns: any single changed element changes it"""
        return torch.stack([_bits(t).sum(dtype=torch.int64) for t in self.mem.owners]).tolist()

    def _sums(self, ops, it):
        """(owner index, sum of the bit patterns) of every declared output view of ``ops`` at iteration ``it``"""
        outs = [o for op in ops for o in declared_outputs(op, it)]
        if not outs:
            return []
        owners = [self.mem.owner(o[0], (2 if o[3] == cabi.BF16 else 4) * emulator._span(o[1], o[2])) for o in outs]
        sums = torch.stack([_bits(emulator.view(self.mem, *o)).sum(dtype=torch.int64) for o in outs]).tolist()
        return list(zip(owners, sums))

    def _stray_writes(self, before, ops, it, sums_before, where):
        """every owner but the outputs' keeps its fingerprint; inside an output's owner, only the view changed: the owner's
        fingerprint minus its views' sums is the same before and after (the sums are exact int64 arithmetic)"""
        after, sums_after = self._fingerprints(), self._sums(ops, it)
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
    def _conv(self, op, it):
        """The fp64 reference is computed chunk by chunk after the launch (a first pass before it only sums |ref| for the
        bound's scale s) when the launch cannot change the conv's operands, i.e. no operand shares a tensor with the output;
        otherwise every chunk is computed before the launch and kept (in host memory when large)."""
        c = op.u.conv
        x, w, kw, out = emulator.conv_operands(c, it, self.mem)
        B, div = c.batch, kw["sample_row_div"]
        gn = c.groups > 0 and c.math in cabi.TC_MODES
        inputs = [t for t in (x, kw.get("res"), kw.get("res_in")) if t is not None]
        lazy = all(t.untyped_storage().data_ptr() != out.untyped_storage().data_ptr() for t in inputs)

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

    def _lnmod(self, op, it):
        m = op.u.lnmod
        x, sh, sc, out = emulator.lnmod_operands(m, it, self.mem)
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

    def _attn(self, op, it):
        a = op.u.attn
        qkv, out = emulator.attn_operands(a, it, self.mem)
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

    def _mha(self, op, it):
        m = op.u.mha
        q, kv, out, both = emulator.mha_operands(m, it, self.mem)
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

    def _host(self):
        """host copies of the owners, taken at the first access to each"""
        return emulator.Owned(self.mem.owners, host=True)

    def _exact(self, op, it):
        """UPDATE / PREP / CAST / GUIDE: the interpreter on host copies of the operands; the kernel must give the same bits
        (GUIDE: emulator.run_guide is the kernel's fp32 multiply, then fp32 add)"""
        host = self._host()
        emulator.run_program([op], 1, it, host)
        outs = declared_outputs(op, it)
        want = [emulator.view(host, *o) for o in outs]

        def check():
            got = [emulator.view(self.mem, *o) for o in outs]
            return [(0.0 if same_bits(g.cpu(), w) else math.inf, f"output {j} bit for bit")
                    for j, (g, w) in enumerate(zip(got, want))]
        return check

    # ---- classifier operators (cg_ref) and the backward operators of a differentiable loop (grad_ref) ------------------
    def _bounded(self, outs, refs):
        """check() of the declared outputs ``outs`` against [(fp64 reference, bound)] (torch on any device, or numpy); a TF32
        output must also have the low 13 bits of every element clear"""
        def check():
            res = []
            for j, (o, (ref, bound)) in enumerate(zip(outs, refs)):
                ref = torch.as_tensor(ref, dtype=F64)
                y = emulator.view(self.mem, *o).float().to(ref.device)
                err = (y.to(F64) - ref).abs()
                frac = _frac(err, torch.as_tensor(bound, dtype=F64, device=ref.device).expand_as(err),
                             bool(torch.isfinite(y).all()))
                if o[3] == cabi.TF32 and int((y.contiguous().view(torch.int32) & 0x1FFF).abs().max()) != 0:
                    frac = math.inf
                res.append((frac, f"output {j}"))
            return res
        return check

    def _gn(self, op, it):
        g = op.u.gn
        h, gamma, beta, vec, res, _ = emulator.gn_operands(g, it, self.mem)
        ref = cg_ref.gn(h, gamma, beta, g.groups, g.eps, g.act, vec, res)
        bound = cg_ref.gn_bound(h, gamma, beta, g.groups, g.eps, ref, g.act, vec, res, g.out_dtype)
        return self._bounded(declared_outputs(op, it), [(ref, bound)])

    def _gn_bwd(self, op, it):
        g = op.u.gn_bwd
        h, gamma, beta, dout, _ = emulator.gn_bwd_operands(g, it, self.mem)
        ref = cg_ref.gn_bwd(h, gamma, beta, dout, g.groups, g.eps, g.act)
        bound = cg_ref.gn_bwd_bound(h, gamma, beta, dout, g.groups, g.eps, ref, g.act, g.dh_dtype)
        return self._bounded(declared_outputs(op, it), [(ref, bound)])

    def _head_grad(self, op, it):
        q = op.u.head_grad
        h, w, b, _ = emulator.head_grad_operands(q, it, self._host())
        _, seed = cg_ref.head_grad(h, w, b, q.scale, q.act)
        return self._bounded(declared_outputs(op, it), [(seed, cg_ref.head_grad_bound(h, w, b, q.scale, q.act))])

    def _stash(self, op, it):
        """the slot copy bit for bit; the Mish or SiLU of the pre-activation under grad_ref.ACT_BOUND"""
        s = op.u.stash
        src, _, _ = emulator.stash_operands(s, it, self._host())
        outs = declared_outputs(op, it)
        refs = [(grad_ref.act(s.act, src), grad_ref.ACT_BOUND[s.act](src.astype(np.float64)))] if s.act_out else []
        bounded = self._bounded(outs[-1:], refs)

        def check():
            res = []
            if s.dst:
                got = emulator.view(self.mem, *outs[0]).cpu()
                res.append((0.0 if same_bits(got, torch.from_numpy(src)) else math.inf, "slot bit for bit"))
            return res + bounded()
        return check

    def _update_bwd(self, op, it):
        gx, x, pr, kw, _ = emulator.update_bwd_operands(op.u.update_bwd, it, self._host())
        gp, dx = grad_ref.update_bwd(gx, x, pr, **kw)
        bound = grad_ref.update_bwd_bound(gx, kw["alpha"], kw["sigma"], kw["k0"], kw["k1"])
        return self._bounded(declared_outputs(op, it), [(dx, bound), (gp, bound)])

    def _dgrad(self, op, it):
        d = op.u.dgrad
        dz, w, z, out, out_sum = emulator.dgrad_operands(d, it, self._host())
        y = grad_ref.dgrad(dz, w, z, d.act)
        before = out.astype(np.float64) if d.accumulate else None
        refs = [(y if before is None else before + y, grad_ref.dgrad_bound(dz, w, z, d.act, before))]
        if out_sum is not None:
            s0 = out_sum.astype(np.float64)
            refs.append((s0 + y, grad_ref.dgrad_bound(dz, w, z, d.act, s0)))
        return self._bounded(declared_outputs(op, it), refs)

    def _wgrad(self, op, it):
        g = op.u.wgrad
        dz, h, dw, db = emulator.wgrad_operands(g, it, self._host())
        gw, gb = grad_ref.wgrad(dz, h, g.act)
        w0 = dw.astype(np.float64) if g.accumulate else None
        b0 = db.astype(np.float64) if db is not None and g.accumulate else None
        bw, bb = grad_ref.wgrad_bound(dz, h, g.act, w0, b0)
        refs = [(gw if w0 is None else w0 + gw, bw)] + ([(gb if b0 is None else b0 + gb, bb)] if g.db else [])
        return self._bounded(declared_outputs(op, it), refs)

    # the reference check of every operator kind
    REFERENCE = {cabi.OP_CONV: _conv, cabi.OP_UPDATE: _exact, cabi.OP_LNMOD: _lnmod, cabi.OP_ATTN: _attn,
                 cabi.OP_PREP: _exact, cabi.OP_CAST: _exact, cabi.OP_MHA: _mha, cabi.OP_STASH: _stash,
                 cabi.OP_UPDATE_BWD: _update_bwd, cabi.OP_DGRAD: _dgrad, cabi.OP_WGRAD: _wgrad, cabi.OP_GN: _gn,
                 cabi.OP_GN_BWD: _gn_bwd, cabi.OP_GUIDE: _exact, cabi.OP_HEAD_GRAD: _head_grad}

    def reference(self, op, it):
        """check() -> [(fraction of the bound, label)] of ``op`` at iteration ``it``, from the state before its launch"""
        return self.REFERENCE[op.kind](self, op, it)

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
        before, sums = self._fingerprints(), self._sums(once, first)
        self.handle.run(first, 0, self.stream, False)
        self.sync()
        for op, chk in zip(once, checks):
            for frac, label in chk():
                self._record(instantiation(op), frac, f"once op: {label}")
        self._stray_writes(before, once, first, sums, "once ops")

    def audit_iteration(self, it):
        """every operator of iteration ``it`` alone; leaves the state of the iteration's end"""
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


# ---- whole iterations -------------------------------------------------------------------------------------------------
def written_owners(mem, ops, its):
    """indices of the owners some operator of ``ops`` writes in an iteration of ``its``"""
    idx = set()
    for it in its:
        for op in ops:
            for ptr, shape, strides, dt in declared_outputs(op, it):
                idx.add(mem.owner(ptr, (2 if dt == cabi.BF16 else 4) * emulator._span(shape, strides)))
    return sorted(idx)


def run_op_by_op(handle, ops, first, count, stream, sync):
    """iterations [first, first + count) one operator at a time with a synchronisation after each (the CDS_OPF_ONCE operators
    first, as cds_plan_run does)"""
    if any(op.flags & cabi.OPF_ONCE for op in ops):
        handle.run(first, 0, stream, False)
        sync()
    for it in range(first, first + count):
        for i, op in enumerate(ops):
            if op.flags & cabi.OPF_ONCE:
                continue
            handle.run_range(it, i, 1, stream)
            sync()


def launches_per_iter(ops):
    """the launches of one iteration of ``ops``: one per operator of the iteration program, and one more for the
    iteration-counter advance unless the last operator, a solver update of a single-branch program, advances it itself"""
    body = [op for op in ops if not op.flags & cabi.OPF_ONCE]
    branches = 1 + max((op.flags & 0xFF00) >> cabi.OPF_BRANCH_SHIFT for op in ops)
    advance = 0 if (branches == 1 and body and body[-1].kind == cabi.OP_UPDATE) else 1
    return len(body) + advance


def report_lines(worst):
    """table rows: program, instantiation, largest fraction of the bound, where"""
    lines = [f"{'program':<14} {'kernel instantiation':<48} {'worst':>7}  where"]
    for (prog, inst), (frac, where) in sorted(worst.items()):
        lines.append(f"{prog:<14} {inst:<48} {frac:>7.3f}  {where}")
    return lines


# ---- differentiable plans ---------------------------------------------------------------------------------------------
def seed_backward(plan, seed):
    """the state GradSamplerPlan.backward starts from: a seeded d x0 in ``gx`` and the accumulators zeroed"""
    g = plan.grad
    with torch.no_grad():
        for t in g.accumulators:
            t.zero_()
        gen = torch.Generator().manual_seed(seed)
        g.gx.copy_(torch.randn(g.gx.shape, generator=gen))


def audit_grad_plan(name, plan, fwd, back, stream=0, sync=lambda: None, seed=3):
    """(forward auditor, backward auditor) of a GradSamplerPlan: every operator of every iteration of the forward program
    from the current x_t (run by ``fwd``), then of every iteration of the backward program (run by ``back``) from
    seed_backward.  Every iteration: backward iteration m reads the stash slots of forward iteration n_iters - 1 - m, and
    only the middle one of an odd count reads its own."""
    owners = plan_owners(plan)
    fa = Auditor(f"{name} fwd", plan.program.ops, fwd, owners, stream, sync)
    fa.audit_once(0)
    for it in range(plan.n_iters):
        fa.audit_iteration(it)
    seed_backward(plan, seed)
    sync()
    ba = Auditor(f"{name} bwd", plan.back.ops, back, owners, stream, sync)
    for it in range(plan.n_iters):
        ba.audit_iteration(it)
    return fa, ba
