"""TEST INFRASTRUCTURE: fp64 semantics and error bounds of the operators of HalfDiT1d's input gradient, the backward modes of
CDS_OP_ATTN (dout != NULL), CDS_OP_LNMOD (dout != NULL) and CDS_OP_STASH (grad != NULL) (include/cds.h, csrc/dit_grad.cuh).
``register(monkeypatch)`` teaches the shared operator references these modes for the duration of one test, the way
tests/relu_ref.py adds ReLU:
  - tests/emulator.py: the interpreter's runners of the three kinds run the backward mode when it is set;
  - tests/program_audit.py: declared_outputs, instantiation and the Auditor's references of the three kinds;
  - tests/grad_ref.py: CDS_ACT_GELU_TANH in ACT_BOUND / ACT_GRAD (the forward activation CDS_OP_STASH applies to DiT's MLP
    hidden layer, and the derivative of the backward mode).

Bounds.  Every output is compared per element as |got - ref| <= tol (|ref| + s), s = the RMS of the reference over the
operator's whole output (a scale for the cancellation inside the sums, which a purely relative bound would not allow).
  - fp32 outputs: tol = ATTN_TOL / LN_TOL / ACT_TOL below, derived from the longest fp32 sum of the kernel (n terms give at most
    n u of the sum of |terms|, u = 2^-24) and a factor 4 for the transcendental functions;
  - CDS_TF32 outputs add the store's rounding, 2^-11 |ref| (round to nearest on a 10-bit mantissa)."""
import math

import numpy as np
import torch

import grad_ref
import opref
from cleandiffuser_b200.engine import cabi

F64 = torch.float64
U32 = 2.0 ** -24
# CDS_OP_ATTN, backward mode: the softmax (hd-term dots, expf, an L-term sum), then dV / dP sums of L and hd terms, dS's row sum of L
# terms, and dQ / dK sums of L terms over products of dS: at most ~(hd + 3 L) u per chain, 4 x (64 + 3 * 128) u = 1.1e-4
ATTN_TOL = 4 * (64 + 3 * 128) * U32
# CDS_OP_LNMOD, backward mode: two C-term sums for the statistics and two for mean(dy) and mean(dy xhat) (C <= 1024 lanes-strided, 32
# partial sums of C / 32 terms then a 5-level butterfly: (C / 32 + 5) u each), times 4 for rsqrtf and the products
LN_TOL = 4 * (1024 // 32 + 5) * 4 * U32
# CDS_OP_STASH, backward mode: one product with act'(z), whose own fp32 error grad_ref bounds (GELU-tanh: tanhf within 2 ulp, a handful of
# products: 16 u (1 + |z|) absolute)
ACT_TOL = 4 * U32


def gelu_tanh_grad(z):
    """d/dz gelu_tanh(z) in fp64"""
    z = np.asarray(z, np.float64)
    k = math.sqrt(2 / math.pi)
    t = np.tanh(k * (z + 0.044715 * z ** 3))
    return 0.5 * (1 + t) + 0.5 * z * (1 - t * t) * k * (1 + 3 * 0.044715 * z * z)


def gelu_tanh_bound(z):
    """fp32 gelu_tanh(z) = 0.5 z (1 + tanhf(u)): tanhf within 2 ulp, the cubic and the products a rounding each"""
    z = np.asarray(z, np.float64)
    return 16 * U32 * (np.abs(z) + np.abs(z) ** 3 * 0.05) + grad_ref.TINY


def gelu_tanh_grad_bound(z):
    z = np.asarray(z, np.float64)
    return 16 * U32 * (1 + np.abs(z) + np.abs(z) ** 3 * 0.15)


def is_backward(op):
    """is ``op`` one of the backward modes this module describes"""
    return (op.kind == cabi.OP_ATTN and bool(op.u.attn.dout)) or (op.kind == cabi.OP_LNMOD and bool(op.u.lnmod.dout)) or \
        (op.kind == cabi.OP_STASH and bool(op.u.stash.grad))


def attn_bwd_operands(a, mem):
    """(q|k|v, d out, d q|k|v view) of a CDS_OP_ATTN descriptor in backward mode"""
    import emulator
    qkv = emulator.view(mem, a.qkv, (a.batch, a.L, 3 * a.C), (a.L * 3 * a.C, 3 * a.C, 1), cabi.F32)
    dout = emulator.view(mem, a.dout, (a.batch, a.L, a.C), (a.L * a.C, a.C, 1), cabi.F32)
    return qkv, dout, emulator.view(mem, a.out, (a.batch, a.L, 3 * a.C), (a.L * 3 * a.C, 3 * a.C, 1), cabi.F32)


def lnmod_bwd_operands(m, mem):
    """(x, scale, dout, res or None, gate or None, dx view, gated view or None) of a CDS_OP_LNMOD descriptor in backward mode"""
    import emulator
    act, dense = (m.batch, m.L, m.C), (m.L * m.C, m.C, 1)
    x = emulator.view(mem, m.in_, act, dense, cabi.F32)
    sc = emulator.view(mem, m.scale, (m.batch, m.C), (m.mod_bstride, 1), cabi.F32)
    dout = emulator.view(mem, m.dout, act, (m.dout_bstride, m.dout_lstride, 1), cabi.F32)
    res = emulator.view(mem, m.res, act, dense, cabi.F32)
    gate = emulator.view(mem, m.gate, (m.batch, m.C), (m.gate_bstride, 1), cabi.F32) if m.gated else None
    return x, sc, dout, res, gate, emulator.view(mem, m.out, act, dense, cabi.F32), emulator.view(mem, m.gated, act, dense,
                                                                                                   cabi.F32)


def act_bwd_operands(t, mem):
    """(z, dh, dz view) of a CDS_OP_STASH descriptor in backward mode"""
    import emulator
    return tuple(emulator.view(mem, ptr, (t.n,), (1,), cabi.F32) for ptr in (t.src, t.grad, t.act_out))


def run_attn_bwd(a, it, mem):
    qkv, dout, dqkv = attn_bwd_operands(a, mem)
    dqkv.copy_(opref.store(attn_bwd(qkv, dout, a.heads), a.out_dtype))


def run_lnmod_bwd(m, it, mem):
    x, sc, dout, res, gate, dx, gated = lnmod_bwd_operands(m, mem)
    d, g = lnmod_bwd(x, sc, dout, m.eps, res, gate)
    if gated is not None:
        gated.copy_(opref.store(g, m.gated_dtype))
    dx.copy_(opref.store(d, m.out_dtype))


def run_act_bwd(t, it, mem):
    z, dh, dz = act_bwd_operands(t, mem)
    dz.copy_(act_bwd(z, dh, t.act).to(torch.float32))


def backward_outputs(op):
    """program_audit.declared_outputs of a backward-mode descriptor"""
    if op.kind == cabi.OP_ATTN:
        a = op.u.attn
        return [(a.out, (a.batch, a.L, 3 * a.C), (a.L * 3 * a.C, 3 * a.C, 1), a.out_dtype)]
    if op.kind == cabi.OP_LNMOD:
        m = op.u.lnmod
        act, dense = (m.batch, m.L, m.C), (m.L * m.C, m.C, 1)
        return [(m.out, act, dense, m.out_dtype)] + ([(m.gated, act, dense, m.gated_dtype)] if m.gated else [])
    t = op.u.stash
    return [(t.act_out, (t.n,), (1,), cabi.F32)]


def backward_instantiation(op):
    """program_audit.instantiation of a backward-mode descriptor"""
    names = {cabi.F32: "f32", cabi.TF32: "tf32"}
    if op.kind == cabi.OP_ATTN:
        a = op.u.attn
        return f"attn_bwd hd {a.C // a.heads} -> {names[a.out_dtype]}"
    if op.kind == cabi.OP_LNMOD:
        m = op.u.lnmod
        return f"lnmod_bwd{' +res' if m.res else ''}{' +gated' if m.gated else ''}{' bcast' if m.dout_lstride == 0 else ''}"
    return f"stash grad {op.u.stash.act}"


def _audit_reference(auditor, op, it):
    """the Auditor's reference check of a backward-mode descriptor, from the state before its launch"""
    outs = backward_outputs(op)
    if op.kind == cabi.OP_ATTN:
        a = op.u.attn
        qkv, dout, _ = attn_bwd_operands(a, auditor.mem)
        ref = attn_bwd(qkv, dout, a.heads)
        return auditor._bounded(outs, [(ref, bound(ref, ATTN_TOL, a.out_dtype))])
    if op.kind == cabi.OP_LNMOD:
        m = op.u.lnmod
        x, sc, dout, res, gate, _, _ = lnmod_bwd_operands(m, auditor.mem)
        dx, g = lnmod_bwd(x, sc, dout, m.eps, res, gate)
        refs = [(dx, bound(dx, LN_TOL, m.out_dtype))] + ([(g, bound(g, LN_TOL, m.gated_dtype))] if g is not None else [])
        return auditor._bounded(outs, refs)
    t = op.u.stash
    z, dh, _ = act_bwd_operands(t, auditor.mem)
    ref = act_bwd(z, dh, t.act)
    return auditor._bounded(outs, [(ref, act_bwd_bound(z, dh, ref, t.act, cabi.F32))])


def register(monkeypatch):
    """the backward modes of CDS_OP_ATTN / LNMOD / STASH in the interpreter and the program audit, and CDS_ACT_GELU_TANH in
    grad_ref.ACT_BOUND / ACT_GRAD, until the test ends"""
    import emulator
    import program_audit as pa
    monkeypatch.setitem(grad_ref.ACT_BOUND, cabi.ACT_GELU_TANH, gelu_tanh_bound)
    monkeypatch.setitem(grad_ref.ACT_GRAD, cabi.ACT_GELU_TANH, (gelu_tanh_grad, gelu_tanh_grad_bound))
    for kind, mode, run_bwd in ((cabi.OP_ATTN, "dout", run_attn_bwd), (cabi.OP_LNMOD, "dout", run_lnmod_bwd),
                                (cabi.OP_STASH, "grad", run_act_bwd)):
        field, run = emulator.OPS[kind]

        def either(d, it, mem=emulator.HOST, run=run, run_bwd=run_bwd, mode=mode):
            return run_bwd(d, it, mem) if getattr(d, mode) else run(d, it, mem)
        monkeypatch.setitem(emulator.OPS, kind, (field, either))
        ref = pa.Auditor.REFERENCE[kind]
        monkeypatch.setitem(pa.Auditor.REFERENCE, kind,
                            lambda self, op, it, ref=ref: _audit_reference(self, op, it) if is_backward(op) else ref(self, op, it))
    declared, instantiation = pa.declared_outputs, pa.instantiation
    monkeypatch.setattr(pa, "declared_outputs", lambda op, it: backward_outputs(op) if is_backward(op) else declared(op, it))
    monkeypatch.setattr(pa, "instantiation",
                        lambda op: backward_instantiation(op) if is_backward(op) else instantiation(op))


@torch.enable_grad()
def attn_bwd(qkv, dout, heads):
    """d q|k|v of softmax(q k^T / sqrt(hd)) v per (trajectory, head) given d out: fp64 autograd.  qkv (B, L, 3C), dout (B, L, C)"""
    B, L, C3 = qkv.shape
    C = C3 // 3
    hd = C // heads
    x = qkv.to(F64).detach().clone().requires_grad_(True)
    q, k, v = (t.reshape(B, L, heads, hd).transpose(1, 2) for t in x.split(C, -1))
    p = torch.softmax(q @ k.transpose(-1, -2) / math.sqrt(hd), -1)
    out = (p @ v).transpose(1, 2).reshape(B, L, C)
    return torch.autograd.grad(out, x, dout.to(F64))[0]


@torch.enable_grad()
def lnmod_bwd(x, scale, dout, eps, res=None, gate=None):
    """(dx, gated or None): d x of LayerNorm(x) (no affine) * (1 + scale) given dout, + res; gate * dx.  x (B, L, C), scale / gate
    (B, C), dout broadcastable to x"""
    xx = x.to(F64).detach().clone().requires_grad_(True)
    mean = xx.mean(-1, keepdim=True)
    var = ((xx - mean) ** 2).mean(-1, keepdim=True)
    y = (xx - mean) / torch.sqrt(var + eps) * (1 + scale.to(F64)[:, None])
    dx = torch.autograd.grad(y, xx, dout.to(F64).expand_as(y))[0]
    if res is not None:
        dx = dx + res.to(F64)
    return dx, (None if gate is None else gate.to(F64)[:, None] * dx)


@torch.enable_grad()
def act_bwd(z, dh, act):
    """dh * act'(z) in fp64"""
    zz = z.to(F64).detach().clone().requires_grad_(True)
    return torch.autograd.grad(opref.act(act, zz), zz, dh.to(F64))[0]


def bound(ref, tol, dtype):
    """tol (|ref| + s) with s = the RMS of ref, plus a CDS_TF32 store's rounding"""
    s = float(ref.pow(2).mean().sqrt()) if ref.numel() else 0.0
    return tol * (ref.abs() + s) + (2.0 ** -11 * ref.abs() if dtype == cabi.TF32 else 0.0)


def act_bwd_bound(z, dh, ref, act, dtype):
    g = grad_ref.ACT_GRAD[act][1] if act in grad_ref.ACT_GRAD else gelu_tanh_grad_bound
    extra = torch.as_tensor(g(z.double().cpu().numpy()), device=ref.device) * dh.to(F64).abs()
    return bound(ref, ACT_TOL, dtype) + extra


# ---- the HalfDiT1d objects of tests/golden/half_dit.npz (make_golden_half_dit.py) on this package's classes
def make_classifier(kw, seed, device="cpu"):
    """this package's CumRewClassifier over a HalfDiT1d of constructor arguments ``kw`` (a ``horizon`` entry is ignored) with
    the golden generator's synthetic weights, model_ema in eval mode"""
    import make_golden_half_dit as mg
    from cleandiffuser_b200.classifier import CumRewClassifier
    from cleandiffuser_b200.nn_classifier import HalfDiT1d
    clf = CumRewClassifier(mg.make_net(HalfDiT1d, kw, seed), device=device)
    clf.model_ema.eval()
    return clf


def make_sample_agent(name, device="cpu", classifier=None):
    """(agent, prior, sample() keyword arguments) of golden sample case ``name``"""
    import make_golden_half_dit as mg
    from cleandiffuser_b200.diffusion import ContinuousDiffusionSDE, DiscreteDiffusionSDE
    from cleandiffuser_b200.nn_diffusion import DiT1d, JannerUNet1d
    clf = classifier if classifier is not None else make_classifier(mg.CLF, 32, device)
    agent = mg.make_agent(name, clf, DiscreteDiffusionSDE, ContinuousDiffusionSDE, JannerUNet1d, DiT1d, device)
    prior, _ = mg.sample_inputs()
    return agent, prior.to(device), mg.sample_kwargs(name)


@torch.enable_grad()
def input_gradient_fp64(clf, x, t):
    """d sum(logp) / d x of clf.model_ema in fp64 autograd, the time embedding evaluated in fp32 by the module's own map_noise
    (as the program's filler does; a Fourier embedding holds a Linear of its own)"""
    import copy
    import cg_ref
    net = copy.deepcopy(clf.model_ema).double()
    net.map_noise = cg_ref.Fp64Time(copy.deepcopy(clf.model_ema.map_noise))
    net.pos_emb_cache = None
    xx = x.detach().double().clone().requires_grad_(True)
    return torch.autograd.grad(net(xx, t).sum(), xx)[0]
