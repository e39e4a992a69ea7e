"""TEST INFRASTRUCTURE: fp64 semantics and error bounds of what QGPO's classifier guidance adds to the operators (include/cds.h):
CDS_OP_DGRAD and CDS_OP_STASH with act = CDS_ACT_SILU (STASH also without a slot), and CDS_OP_HEAD_GRAD.  ``run_program`` /
``Handle`` extend tests/cg_ref.py's interpreter with them, the way cg_ref extends tests/grad_ref.py's; the GPU operator tests
and the program audit compare the kernels against the same functions.  Plus the objects of tests/golden/qgpo.npz."""
import os

import numpy as np
import torch

import cg_ref
import emulator
import grad_ref
from cleandiffuser_b200.engine import cabi

U32 = grad_ref.U32
TINY = 1e-35          # silu(z) for z < -88, where the fp32 1 + expf(-z) overflows and the kernel returns -0


def silu(x):
    x = np.asarray(x, np.float64)
    return x / (1.0 + np.exp(-x))


def silu_grad(x):
    """d/dx silu(x) (ATen's silu_backward: sig (1 + x (1 - sig)))"""
    x = np.asarray(x, np.float64)
    sig = 1.0 / (1.0 + np.exp(-x))
    return sig * (1.0 + x * (1.0 - sig))


def silu_bound(z):
    """fp32 silu(z) = z / (1 + expf(-z)): expf within 2 ulp (4 u), the add and the division u each: 6 u relative, 8 u allowed;
    TINY covers the overflow of 1 + expf(-z) below z = -88"""
    return 8 * U32 * np.abs(silu(z)) + TINY


def silu_grad_bound(z):
    """fp32 silu'(z): sig carries 6 u relative (as in silu_bound), so 1 - sig an absolute 7 u (sig <= 1), z (1 - sig) 7 u |z| plus
    its rounding, 1 + that and the product with sig a rounding each: (12 + 12 |z|) u covers them with the margin of 2x on the
    roundings that the other bounds of the audit keep"""
    return (12 + 12 * np.abs(np.asarray(z, np.float64))) * U32


def dgrad(dz, w, z=None, act_kind=cabi.ACT_NONE):
    """(dz W) * act'(z) in fp64 for act NONE / MISH / SILU"""
    if act_kind != cabi.ACT_SILU:
        return grad_ref.dgrad(dz, w, z, act_kind)
    return (np.asarray(dz, np.float64) @ np.asarray(w, np.float64)) * silu_grad(z)


def dgrad_bound(dz, w, z=None, act_kind=cabi.ACT_NONE, before=None):
    """grad_ref.dgrad_bound with the SiLU derivative: the fma chain over N gives (N + 4) u |dz||W| |silu'(z)|, the fp32 silu'
    adds |dz W| silu_grad_bound(z)"""
    if act_kind != cabi.ACT_SILU:
        return grad_ref.dgrad_bound(dz, w, z, act_kind, before)
    dz, w, z = np.asarray(dz, np.float64), np.asarray(w, np.float64), np.asarray(z, np.float64)
    dzw, sg = dz @ w, silu_grad(z)
    bound = np.abs(dzw) * silu_grad_bound(z) + (dz.shape[1] + 4) * U32 * ((np.abs(dz) @ np.abs(w)) * np.abs(sg))
    if before is not None:
        bound = bound + 2 * U32 * (np.abs(np.asarray(before, np.float64)) + np.abs(dzw * sg))
    return bound


def head_grad(h, w, b, scale, act_kind=cabi.ACT_SILU):
    """CDS_OP_HEAD_GRAD in fp64 -> (z (rows,), seed (rows,)): z = act(h) . w + b, seed = d scale tanh(z / scale) / d z"""
    a = silu(h) if act_kind == cabi.ACT_SILU else np.asarray(h, np.float64)
    z = a @ np.asarray(w, np.float64).reshape(-1) + float(np.asarray(b).reshape(-1)[0])
    y = np.tanh(z / scale)
    return z, 1.0 - y * y


def head_grad_bound(h, w, b, scale, act_kind=cabi.ACT_SILU):
    """Per-row bound on |CDS_OP_HEAD_GRAD seed - head_grad(...)|.  z: each lane sums ceil(K/32) fma terms in order, then a
    5-level butterfly and the bias add, so (ceil(K/32) + 6) u sum|act(h) w| + u |b|, plus the fp32 SiLU's silu_bound(h) |w|.
    seed(z) = 1 - tanh(z/scale)^2 has |d seed / d z| <= 0.77 / scale (max of 2 y (1 - y^2)).  The evaluation: z / scale and
    tanhf (2 ulp) put 4 u |y| on y, 1 - y*y then carries 2 |y| 4 u |y| + 2 u and the product and quotient with scale 2 u: 12 u
    absolute covers it."""
    h = np.asarray(h, np.float64)
    w = np.abs(np.asarray(w, np.float64).reshape(-1))
    a = silu(h) if act_kind == cabi.ACT_SILU else h
    K = h.shape[1]
    e_z = (-(-K // 32) + 6) * U32 * (np.abs(a) @ w) + U32 * abs(float(np.asarray(b).reshape(-1)[0]))
    if act_kind == cabi.ACT_SILU:
        e_z = e_z + silu_bound(h) @ w
    return 0.77 / abs(scale) * e_z + 12 * U32


# ---------------------------------------------------------------- descriptor interpreters (memory backends of tests/emulator.py)
def run_stash(s, it, arr):
    """CDS_OP_STASH with SiLU or without a slot; the rest is grad_ref.run_stash"""
    src = arr(s.src, (s.n,), (1,))
    if s.dst:
        arr(s.dst + 4 * it * s.dst_iter_stride, (s.n,), (1,))[...] = src
    if s.act_out:
        y = silu(src) if s.act == cabi.ACT_SILU else grad_ref.act(s.act, src)
        arr(s.act_out, (s.n,), (1,))[...] = np.asarray(y, np.float64).astype(np.float32)


def run_dgrad(d, it, arr):
    dz = arr(d.dz, (d.rows, d.N), (d.ldz, 1))
    w = arr(d.w, (d.N, d.K), (d.ldw, 1))
    z = arr(d.z + 4 * it * d.z_iter_stride, (d.rows, d.K), (d.K, 1)) if d.z else None
    y = dgrad(dz, w, z, d.act)
    out = arr(d.out, (d.rows, d.K), (d.ldo, 1))
    out[...] = (out.astype(np.float64) + y if d.accumulate else y).astype(np.float32)
    if d.out_sum:
        s = arr(d.out_sum, (d.rows, d.K), (d.K, 1))
        s[...] = (s.astype(np.float64) + y).astype(np.float32)


def run_head_grad(q, it, arr):
    h = arr(q.h, (q.rows, q.K), (q.ldh, 1))
    _, seed = head_grad(h, arr(q.w, (q.K,), (1,)), arr(q.b, (1,), (1,)), q.scale, q.act)
    arr(q.seed, (q.rows,), (1,))[...] = seed.astype(np.float32)


def _ours(op):
    """the operators this module interprets; every other one goes to cg_ref.run_program"""
    if op.kind == cabi.OP_HEAD_GRAD:
        return run_head_grad, "head_grad"
    if op.kind == cabi.OP_DGRAD and op.u.dgrad.act == cabi.ACT_SILU:
        return run_dgrad, "dgrad"
    if op.kind == cabi.OP_STASH and (op.u.stash.act == cabi.ACT_SILU or not op.u.stash.dst):
        return run_stash, "stash"
    return None


def run_program(ops, n_iters, first=0, mem=emulator.HOST):
    """tests/cg_ref.py's run_program for programs that also hold QGPO's operators"""
    arr = lambda ptr, shape, strides: emulator._arr(ptr, shape, strides, mem)       # noqa: E731
    emulator.run_program([op for op in ops if op.flags & cabi.OPF_ONCE], 0, first, mem)
    with np.errstate(over="ignore", invalid="ignore", divide="ignore"):
        for it in range(first, first + n_iters):
            for op in ops:
                if op.flags & cabi.OPF_ONCE:
                    continue
                mine = _ours(op)
                if mine is not None:
                    mine[0](getattr(op.u, mine[1]), it, arr)
                else:
                    cg_ref.run_program([op], 1, it, mem)


class Handle(emulator.Handle):
    """emulator.Handle whose interpreter also runs the backward, classifier-guidance and QGPO operators"""

    def run(self, first, count, stream, use_graph=True):
        run_program(self.ops, count, first, self.mem)

    def run_range(self, it, op_first, op_count, stream):
        keep = [op for op in self.ops[op_first:op_first + op_count] if not (op.flags & cabi.OPF_ONCE)]
        run_program(keep, 1, it, self.mem)


# ---------------------------------------------------------------- the objects of tests/golden/qgpo.npz
# QGPO's classifier at the D4RL MuJoCo shapes (obs_dim, act_dim)
PIPELINES = {"hopper": dict(obs_dim=11, act_dim=3), "walker": dict(obs_dim=17, act_dim=6),
             "halfcheetah": dict(obs_dim=17, act_dim=6)}


def golden():
    return np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "qgpo.npz"), allow_pickle=False)


def make_classifier(kw, seed, device="cpu"):
    """this package's QGPOClassifier over QGPONNClassifier with the golden generator's synthetic weights"""
    import make_golden_qgpo as mg
    from cleandiffuser_b200.classifier import QGPOClassifier
    from cleandiffuser_b200.nn_classifier import QGPONNClassifier
    return mg.make_classifier(QGPONNClassifier, QGPOClassifier, kw, seed, device)


def make_sample_agent(name, device="cpu", classifier=None):
    """(agent, prior, sample() keyword arguments) of golden sample case ``name`` (make_golden_qgpo.py)"""
    import make_golden_qgpo as mg
    from cleandiffuser_b200.diffusion import ContinuousDiffusionSDE
    from cleandiffuser_b200.nn_condition import MLPCondition
    from cleandiffuser_b200.nn_diffusion import SfBCUNet
    clf = classifier if classifier is not None else make_classifier(dict(obs_dim=mg.OBS, act_dim=mg.ACT), 32, device)
    agent = mg.make_actor(ContinuousDiffusionSDE, SfBCUNet, MLPCondition, mg.SAMPLES[name]["predict_noise"], clf, device)
    prior, obs = mg.sample_inputs()
    return agent, prior.to(device), mg.sample_kwargs(name, obs.to(device))


def tape_of(g, name):
    return [g[f"sample/{name}/z{j}"] for j in range(int(g[f"sample/{name}/n_draws"]))]


def input_gradient_fp64(clf, x, t, obs):
    """d sum(logp) / d x of clf.model_ema in fp64 autograd (the Fourier features computed in fp32, as the engine's filler does)"""
    import copy
    net = copy.deepcopy(clf.model_ema).double()
    net.map_noise = cg_ref.Fp64Time(clf.model_ema.map_noise)
    xx = x.detach().double().clone().requires_grad_(True)
    lp = net(xx, t, obs.double())
    return torch.autograd.grad(lp.sum(), xx)[0]


def lowered_gradient(clf, x, t_all, obs, it, math, device, handle=None):
    """the input gradient as the lowered program computes it at iteration ``it`` (time t_all[it] for every row, condition obs):
    through ``handle(ops, n_iters, owners)`` (default: this module's interpreter) -> ((rows, act_dim) fp32, program)"""
    from cleandiffuser_b200.engine.lower import Program, View, lower_classifier_grad
    B, A = x.shape
    p = Program(torch.device(device), B, len(t_all), math)
    xb = p.buf(B, A)
    xb.copy_(x)
    g = lower_classifier_grad(p, clf, View(xb, 1, A))

    class Ctx:
        pass
    ctx = Ctx()
    ctx.t_all, ctx.cond_rows, ctx.cond_cg = t_all.to(device), None, obs.to(device)
    with torch.no_grad():
        for fn in p.per_call:
            fn(ctx)
    h = (handle or (lambda ops, n, owners: Handle(ops, n, owners)))(p.ops, len(t_all), list(p.keep))
    h.run(it, 1, 0 if device == "cpu" else torch.cuda.current_stream().cuda_stream, False)
    return g.t.view(B, A).clone(), p
