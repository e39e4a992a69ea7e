"""TEST INFRASTRUCTURE: torch fp64 semantics of the classifier-guidance operators (include/cds.h: CDS_OP_GN, CDS_OP_GN_BWD,
CDS_OP_GUIDE), with the stores of their output dtypes.  ``run_program`` / ``Handle`` extend tests/grad_ref.py's interpreter
(which extends tests/emulator.py's) with them; the GPU parity tests compare the kernels against the same functions."""
import torch

import emulator
import grad_ref
import opref
from cleandiffuser_b200.engine import cabi

F64 = torch.float64


def _stats(h, groups, eps):
    B, L, C = h.shape
    g = h.to(F64).reshape(B, L, groups, C // groups)
    mean = g.mean(dim=(1, 3), keepdim=True)
    var = ((g - mean) ** 2).mean(dim=(1, 3), keepdim=True)
    return g, mean, 1.0 / torch.sqrt(var + eps)


def gn(h, gamma, beta, groups, eps, act=cabi.ACT_MISH, vec=None, res=None):
    """CDS_OP_GN in fp64: act(GroupNorm(h) gamma + beta) [+ vec (B, C) or (C,)] [+ res (B, L, C)]"""
    B, L, C = h.shape
    g, mean, rstd = _stats(h, groups, eps)
    y = opref.act(act, ((g - mean) * rstd).reshape(B, L, C) * gamma.to(F64) + beta.to(F64))
    if vec is not None:
        v = vec.to(F64)
        y = y + (v[None, None] if v.dim() == 1 else v[:, None])
    if res is not None:
        y = y + res.to(F64)
    return y


def gn_bwd(h, gamma, beta, dout, groups, eps, act=cabi.ACT_MISH):
    """CDS_OP_GN_BWD in fp64: d h of act(GroupNorm(h) gamma + beta) given dout"""
    B, L, C = h.shape
    g, mean, rstd = _stats(h, groups, eps)
    xhat = ((g - mean) * rstd).reshape(B, L, C)
    d = gamma.to(F64) * dout.to(F64)
    if act == cabi.ACT_MISH:
        d = d * torch.from_numpy(grad_ref.mish_grad((xhat * gamma.to(F64) + beta.to(F64)).cpu().numpy())).to(d.device)
    dg = d.reshape(B, L, groups, C // groups)
    xg = xhat.reshape(B, L, groups, C // groups)
    m1 = dg.mean(dim=(1, 3), keepdim=True)
    m2 = (dg * xg).mean(dim=(1, 3), keepdim=True)
    return (rstd * (dg - m1 - xg * m2)).reshape(B, L, C)


# ---------------------------------------------------------------- descriptor interpreters (memory backends of tests/emulator.py)
def run_gn(g, it, mem):
    v = emulator.view
    h = v(mem, g.h, (g.batch, g.L, g.C), (g.h_bstride, g.h_lstride, 1), cabi.F32)
    vec = emulator.vec(g.vec, it, g.batch, g.C, 1, mem)
    res = v(mem, g.res, (g.batch, g.L, g.C), (g.res_bstride, g.res_lstride, 1), cabi.F32) if g.res else None
    y = gn(h, v(mem, g.gamma, (g.C,), (1,), cabi.F32), v(mem, g.beta, (g.C,), (1,), cabi.F32), g.groups, g.eps, g.act, vec, res)
    out = v(mem, g.out, (g.batch, g.L, g.C), (g.out_bstride, g.out_lstride, 1), cabi.F32)
    out.copy_(opref.store(y, g.out_dtype))


def run_gn_bwd(g, it, mem):
    v = emulator.view
    h = v(mem, g.h, (g.batch, g.L, g.C), (g.h_bstride, g.h_lstride, 1), cabi.F32)
    dout = v(mem, g.dout, (g.batch, g.L, g.C), (g.dout_bstride, g.dout_lstride, 1), cabi.F32)
    y = gn_bwd(h, v(mem, g.gamma, (g.C,), (1,), cabi.F32), v(mem, g.beta, (g.C,), (1,), cabi.F32), dout, g.groups, g.eps, g.act)
    out = v(mem, g.dh, (g.batch, g.L, g.C), (g.dh_bstride, g.dh_lstride, 1), cabi.F32)
    out.copy_(opref.store(y, g.dh_dtype))


def run_guide(q, it, mem):
    """fp32 multiply, then fp32 add: the kernel's exact arithmetic"""
    v = emulator.view
    s = v(mem, q.s + 4 * it, (1,), (1,), cabi.F32)[0]
    pred = v(mem, q.pred, (q.batch, q.L, q.C), (q.L * q.C, q.C, 1), cabi.F32)
    g = v(mem, q.g, (q.batch, q.L, q.C), (q.g_bstride, q.g_lstride, 1), cabi.F32)
    pred.copy_(pred + s * g)


_CG_OPS = {cabi.OP_GN: (run_gn, "gn"), cabi.OP_GN_BWD: (run_gn_bwd, "gn_bwd"), cabi.OP_GUIDE: (run_guide, "guide")}


def run_program(ops, n_iters, first=0, mem=emulator.HOST):
    """tests/grad_ref.py's run_program for programs that also hold the classifier-guidance operators"""
    emulator.run_program([op for op in ops if op.flags & cabi.OPF_ONCE], 0, first, mem)
    for it in range(first, first + n_iters):
        for op in ops:
            if op.flags & cabi.OPF_ONCE:
                continue
            if op.kind in _CG_OPS:
                fn, field = _CG_OPS[op.kind]
                fn(getattr(op.u, field), it, mem)
            else:
                grad_ref.run_program([op], 1, it, mem)


class Handle(emulator.Handle):
    """emulator.Handle whose interpreter also runs the backward and classifier-guidance operators"""

    def run(self, first, count, stream, use_graph=True):
        run_program(self.ops, count, first, self.mem)

    def run_range(self, it, op_first, op_count, stream):
        keep = [op for op in self.ops[op_first:op_first + op_count] if not (op.flags & cabi.OPF_ONCE)]
        run_program(keep, 1, it, self.mem)


# ---------------------------------------------------------------- the objects of tests/golden/classifier.npz
def golden():
    import os
    import numpy as np
    return np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "classifier.npz"), allow_pickle=False)


def make_classifier(kw, seed, device="cpu"):
    """this package's CumRewClassifier over HalfJannerUNet1d with the golden generator's synthetic weights"""
    from cleandiffuser_b200.classifier import CumRewClassifier
    from cleandiffuser_b200.nn_classifier import HalfJannerUNet1d
    from cleandiffuser_b200.testing import synth_state_dict
    net = HalfJannerUNet1d(**kw)
    net.load_state_dict(synth_state_dict(net.state_dict(), seed))
    return CumRewClassifier(net, device=device)


def make_sample_agent(name, device="cpu", classifier=None):
    """(agent, prior, sample() keyword arguments) of golden sample case ``name`` (make_golden_classifier.py)"""
    import make_golden_classifier as mg
    from cleandiffuser_b200.diffusion import ContinuousDiffusionSDE, DiscreteDiffusionSDE
    from cleandiffuser_b200.nn_diffusion import JannerUNet1d
    spec = mg.SAMPLES[name]
    clf = classifier if classifier is not None else make_classifier(dict(horizon=mg.H, in_dim=mg.D, dim_mult=(1, 2)), 32, device)
    prior, mask = mg.sample_inputs()
    common = dict(fix_mask=mask, predict_noise=spec["predict_noise"], device=device, classifier=clf)
    if spec["kind"] == "discrete":
        agent, sched = DiscreteDiffusionSDE(mg.make_denoiser(JannerUNet1d), diffusion_steps=mg.T, **common), "uniform"
    else:
        agent, sched = ContinuousDiffusionSDE(mg.make_denoiser(JannerUNet1d), **common), "uniform_continuous"
    kw = dict(solver=spec["solver"], n_samples=mg.BATCH, sample_steps=mg.STEPS, sample_step_schedule=sched, use_ema=True,
              temperature=0.8, w_cg=mg.W_CG)
    return agent, prior.to(device), kw


def tape_of(g, name):
    return [g[f"sample/{name}/z{j}"] for j in range(int(g[f"sample/{name}/n_draws"]))]


class Fp64Time(torch.nn.Module):
    """the timestep embedding computes in fp32 whatever the weights: its output widened for an fp64 copy of a network"""

    def __init__(self, m):
        super().__init__()
        self.m = m

    def forward(self, t):
        return self.m(t).double()


def input_gradient_fp64(clf, x, t):
    """d sum(logp) / d x of clf.model_ema in fp64 autograd"""
    import copy
    net = copy.deepcopy(clf.model_ema).double()
    net.map_noise = Fp64Time(net.map_noise)
    xx = x.detach().double().clone().requires_grad_(True)
    lp = net(xx, t)
    return torch.autograd.grad(lp.sum(), xx)[0]


def lowered_gradient(clf, x, t_all, it, math, device, handle=None):
    """the input gradient as the lowered program computes it at iteration ``it`` (time t_all[it] for every row): through
    ``handle(ops, n_iters, owners)`` (default: this module's interpreter) -> (rows, H, in_dim) fp32"""
    from cleandiffuser_b200.engine.lower import Program, View, lower_half_janner_grad
    B, Hh, Dd = x.shape
    p = Program(torch.device(device), B, len(t_all), math)
    xb = p.buf(B, Hh, Dd)
    xb.copy_(x)
    g = lower_half_janner_grad(p, clf, View(xb, Hh, Dd))

    class Ctx:
        pass
    ctx = Ctx()
    ctx.t_all, ctx.cond_rows = t_all.to(device), None
    with torch.no_grad():
        for fn in p.per_call:
            fn(ctx)
    h = (handle or (lambda ops, n, owners: Handle(ops, n, owners)))(p.ops, len(t_all), list(p.keep))
    h.run(it, 1, 0 if device == "cpu" else torch.cuda.current_stream().cuda_stream, False)
    return g.t.view(B, Hh, -1)[..., :Dd].clone(), p
