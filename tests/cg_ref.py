"""TEST INFRASTRUCTURE: fp64 semantics of the classifier operators (include/cds.h: CDS_OP_GN, CDS_OP_GN_BWD, CDS_OP_GUIDE,
CDS_OP_HEAD_GRAD, csrc/classifier.cuh) and the error bounds of their kernels.  tests/emulator.py runs them on a program's
descriptors; the GPU parity tests and tests/program_audit.py compare the kernels against the same functions.  Plus the
classifiers of tests/golden/classifier.npz and the lowered input gradient of either classifier."""
import numpy as np
import torch

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


def head_grad(h, w, b, scale, act_kind=cabi.ACT_SILU):
    """CDS_OP_HEAD_GRAD in fp64 (numpy) -> (z (rows,), seed (rows,)): z = act(h) . w + b, seed = d scale tanh(z/scale) / dz"""
    z = grad_ref.act(act_kind, h) @ np.asarray(w, np.float64).reshape(-1) + float(np.asarray(b).reshape(-1)[0])
    y = np.tanh(z / scale)
    return z, 1.0 - y * y


# ---------------------------------------------------------------- error bounds of csrc/classifier.cuh (u = 2^-24)
U32 = grad_ref.U32
# A TF32 store rounds to nearest: at most half a TF32 unit, 2^-11 |ref|.  The bound allows a whole unit, R_TF32 |ref|, as it
# does for the audit's other TF32 outputs (conv, LNMOD), so that a correctly rounded value of the exact result takes at most
# half of it.  That leaves room for a store that truncates instead of rounding; the rounding mode itself is pinned elsewhere:
# GN / GN_BWD store through f32_for_store (csrc/common.cuh), whose TF32 rounding every audited `update + x_cast -> tf32`
# compares bit for bit with opref.tf32_round, and the TF32 outputs here must have their low 13 bits clear.
R_TF32 = 2.0 ** -10
MISH_LIP, MISH_GRAD_LIP = 1.1, 1.0          # max Mish' = 1.089, max |Mish''| = 0.644


def _gmean(t, groups):
    """per-element (B, L, C) view of the (trajectory, group) mean of t"""
    B, L, C = t.shape
    return t.reshape(B, L, groups, C // groups).mean(dim=(1, 3), keepdim=True).expand(B, L, groups, C // groups).reshape(B, L, C)


def _xhat_error(h, groups, eps):
    """(xhat, rstd, k, e_x) in fp64.  One warp owns the n = L C / groups elements of a (trajectory, group): each lane sums
    about ceil(n/32) of them in order, then a 5-level butterfly, so k = ceil(n/32) + 5 is the summation depth.
      mean m:  |m - mean| <= (k + 1) u mean|h|  (k adds and the division by n)
      rstd:    the centred squares are positive, so their sum has relative error <= k u; each d = h - m rounds once (2 u on
               d^2); m enters the variance only to second order (sum (h - mean) = 0); with / n, + eps, sqrtf and 1 / x the
               relative error of rstd is at most (k/2 + 4) u
      xhat = (h - m) rstd:  e_x = rstd (k + 1) u mean|h| + (k/2 + 6) u |xhat|  (the subtraction and the product add 2 u)"""
    B, L, C = h.shape
    g, mean, rstd = _stats(h, groups, eps)
    k = -(-(L * C // groups) // 32) + 5
    xhat = ((g - mean) * rstd).reshape(B, L, C)
    rstd = rstd.expand(B, L, groups, C // groups).reshape(B, L, C)
    e_x = rstd * (k + 1) * U32 * _gmean(h.to(F64).abs(), groups) + (k / 2 + 6) * U32 * xhat.abs()
    return xhat, rstd, k, e_x


def _store_term(ref, dtype):
    return R_TF32 * ref.abs() if dtype == cabi.TF32 else 0.0


def gn_bound(h, gamma, beta, groups, eps, ref, act=cabi.ACT_MISH, vec=None, res=None, out_dtype=cabi.F32):
    """Per-element bound on |CDS_OP_GN - gn(...)| (gn_kernel; ``ref`` = gn(...) in fp64).  From the xhat error e_x of
    ``_xhat_error``:
      z = fmaf(xhat, gamma, beta):  e_z = |gamma| e_x + u |z|
      y = Mish(z):  MISH_LIP e_z (Mish is 1.1-Lipschitz) + grad_ref.mish_bound(z) (the fp32 evaluation)
      + vec, + res:  one rounding per add, 2 u (|y| + |vec|) and 2 u (|y| + |vec| + |res|): twice the rounding, so that
                     a store's rounding of the exact result is at most half of its term, as for R_TF32
      TF32 store:  R_TF32 |ref|"""
    xhat, _, _, e_x = _xhat_error(h, groups, eps)
    ga = gamma.to(F64)
    z = xhat * ga + beta.to(F64)
    e = ga.abs() * e_x + U32 * z.abs()
    if act == cabi.ACT_MISH:
        e = MISH_LIP * e + grad_ref.mish_bound(z)
    mag = opref.act(act, z).abs()
    if vec is not None:
        v = vec.to(F64).abs()
        mag = mag + (v[None, None] if v.dim() == 1 else v[:, None])
        e = e + 2 * U32 * mag
    if res is not None:
        mag = mag + res.to(F64).abs()
        e = e + 2 * U32 * mag
    return e + _store_term(ref, out_dtype)


def gn_bwd_bound(h, gamma, beta, dout, groups, eps, ref, act=cabi.ACT_MISH, dh_dtype=cabi.F32):
    """Per-element bound on |CDS_OP_GN_BWD - gn_bwd(...)| (gn_bwd_kernel; ``ref`` = gn_bwd(...) in fp64).  dh = rstd (d - m1 -
    xhat m2) cancels, so the bound is relative to rstd (|d| + mean|d| + |xhat| mean|d xhat|), not to dh.  From e_x of
    ``_xhat_error`` and e_z = |gamma| e_x + u |z|:
      d = gamma dout Mish'(z):  e_d = |gamma dout| (grad_ref.mish_grad_bound(z) + MISH_GRAD_LIP e_z) + 2 u |d|
      m1 = mean d:              e_m1 = (k + 1) u mean|d| + mean e_d
      m2 = mean d xhat (fmaf):  e_m2 = (k + 1) u mean|d xhat| + mean(e_d |xhat| + |d| e_x)
      dh:  rstd (e_d + e_m1 + |xhat| e_m2 + |m2| e_x + 3 u (|d| + |m1| + |xhat m2|)) + (k/2 + 5) u |dh| (rstd's relative
           error and the final product), + R_TF32 |ref| for a TF32 store"""
    xhat, rstd, k, e_x = _xhat_error(h, groups, eps)
    ga = gamma.to(F64)
    z = xhat * ga + beta.to(F64)
    d = gd = ga * dout.to(F64)
    e_d = 0.0
    if act == cabi.ACT_MISH:
        d = gd * torch.from_numpy(grad_ref.mish_grad(z.cpu().numpy())).to(gd.device)
        e_d = gd.abs() * (grad_ref.mish_grad_bound(z) + MISH_GRAD_LIP * (ga.abs() * e_x + U32 * z.abs()))
    e_d = e_d + 2 * U32 * d.abs()
    m1, m2 = _gmean(d, groups), _gmean(d * xhat, groups)
    e_m1 = (k + 1) * U32 * _gmean(d.abs(), groups) + _gmean(e_d, groups)
    e_m2 = (k + 1) * U32 * _gmean((d * xhat).abs(), groups) + _gmean(e_d * xhat.abs() + d.abs() * e_x, groups)
    e = rstd * (e_d + e_m1 + xhat.abs() * e_m2 + m2.abs() * e_x + 3 * U32 * (d.abs() + m1.abs() + (xhat * m2).abs()))
    return e + (k / 2 + 5) * U32 * ref.abs() + _store_term(ref, dh_dtype)


def head_grad_bound(h, w, b, scale, act_kind=cabi.ACT_SILU):
    """Per-row bound on |CDS_OP_HEAD_GRAD seed - head_grad(...)|.  z: each lane sums ceil(K/32) fma terms in order, then a
    5-level butterfly and the bias add, so (ceil(K/32) + 6) u sum|act(h) w| + u |b|, plus the fp32 SiLU's silu_bound(h) |w|.
    seed(z) = 1 - tanh(z/scale)^2 has |d seed / d z| <= 0.77 / scale (max of 2 y (1 - y^2)).  The evaluation: z / scale and
    tanhf (2 ulp) put 4 u |y| on y, 1 - y*y then carries 2 |y| 4 u |y| + 2 u and the product and quotient with scale 2 u: 12 u
    absolute covers it."""
    h = np.asarray(h, np.float64)
    w = np.abs(np.asarray(w, np.float64).reshape(-1))
    K = h.shape[1]
    e_z = (-(-K // 32) + 6) * U32 * (np.abs(grad_ref.act(act_kind, h)) @ w) + U32 * abs(float(np.asarray(b).reshape(-1)[0]))
    if act_kind == cabi.ACT_SILU:
        e_z = e_z + grad_ref.silu_bound(h) @ w
    return 0.77 / abs(scale) * e_z + 12 * U32


# the classifiers of the reference's guided pipelines (diffuser / adaptdiffuser / veteran on D4RL): HalfJannerUNet1d keyword
# arguments, and the observation part of x (the rest is the action)
PIPELINES = {"hopper": dict(horizon=32, in_dim=14), "walker": dict(horizon=32, in_dim=23),
             "halfcheetah": dict(horizon=4, in_dim=23, dim_mult=(1, 4, 2)), "antmaze": dict(horizon=64, in_dim=37),
             "kitchen": dict(horizon=32, in_dim=69)}
OBS_DIM = {"hopper": 11, "walker": 17, "halfcheetah": 17, "antmaze": 29, "kitchen": 60}


# ---------------------------------------------------------------- the objects of tests/golden/classifier.npz
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


def lowered_gradient(clf, x, t_all, it, math, device, cond=None, handle=None):
    """the input gradient of either lowered classifier (HalfJannerUNet1d: x (rows, H, in_dim); QGPO: x (rows, act_dim)) as
    the program computes it at iteration ``it`` (time t_all[it] for every row, classifier condition ``cond``): through
    ``handle(ops, n_iters, owners)`` (default: tests/emulator.py's Handle) -> (fp32 gradient shaped like x, program)"""
    import emulator
    from cleandiffuser_b200.engine.lower import Program, View, lower_classifier_grad
    from cleandiffuser_b200.engine.runtime import _Ctx
    B, H, D = x.shape if x.dim() == 3 else (x.shape[0], 1, x.shape[1])
    p = Program(torch.device(device), B, len(t_all), math)
    xb = p.buf(*x.shape)
    xb.copy_(x)
    g = lower_classifier_grad(p, clf, View(xb, H, D))
    ctx = _Ctx(t_all.to(device), None, None if cond is None else cond.to(device))
    with torch.no_grad():
        for fn in p.per_call:
            fn(ctx)
    (handle or emulator.Handle)(p.ops, len(t_all), list(p.keep)).run(
        it, 1, 0 if device == "cpu" else torch.cuda.current_stream().cuda_stream, False)
    return g.t.view(B, H, -1)[..., :D].reshape(x.shape).clone(), p
