"""TEST INFRASTRUCTURE: numpy semantics of the backward operators of a differentiable reverse loop (include/cds.h:
CDS_OP_STASH, CDS_OP_UPDATE_BWD, CDS_OP_DGRAD, CDS_OP_WGRAD, csrc/grad.cuh) for every activation they accept (NONE, MISH,
SILU), in fp64 with fp32 stores, like tests/opref.py does for the forward operators, and the error bounds of their kernels.
tests/emulator.py runs them on a program's descriptors; the GPU parity tests and tests/program_audit.py compare the kernels
against the same functions."""
import numpy as np
import torch

import opref
from cleandiffuser_b200.engine import cabi


def act(kind, x):
    """tests/opref.py's activation ``kind`` of a numpy array, in fp64"""
    return opref.act(kind, torch.from_numpy(np.array(x, np.float64))).numpy()


def mish_grad(x):
    """d/dx mish(x) (ATen: tanh(softplus(x)) + x sigmoid(x) (1 - tanh(softplus(x))^2))"""
    x = np.asarray(x, np.float64)
    tsp = np.tanh(np.logaddexp(0.0, x))
    sig = 1.0 / (1.0 + np.exp(-x))
    return tsp + x * sig * (1.0 - tsp * tsp)


def silu_grad(x):
    """d/dx silu(x) (ATen's silu_backward: sig (1 + x (1 - sig)))"""
    x = np.asarray(x, np.float64)
    sig = 1.0 / (1.0 + np.exp(-x))
    return sig * (1.0 + x * (1.0 - sig))


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
    if act_kind != cabi.ACT_NONE:
        y = y * ACT_GRAD[act_kind][0](z)
    return y


def wgrad(dz, h, act_kind=cabi.ACT_NONE):
    """(dz^T act(h), sum_rows dz) in fp64"""
    dz = np.asarray(dz, np.float64)
    return dz.T @ act(act_kind, h), dz.sum(0)


# ---------------------------------------------------------------- error bounds of the fp32 kernels (csrc/grad.cuh), u = 2^-24
# Each takes fp64 numpy arrays (or torch tensors where it only uses abs and arithmetic) and returns the per-element bound on
# |kernel - fp64 reference|.  The operator tests (tests/test_grad_sampling_gpu.py) and the program audit
# (tests/program_audit.py) both apply them.
U32 = 2.0 ** -24
TINY = 1e-35          # silu(z) for z < -88, where the fp32 1 + expf(-z) overflows and the kernel returns -0
# fp32 underflow: Mish(z) below z = -87 (expf(z) leaves the normal range; |Mish(z)| <= 103 e^-87 < TINY, and the kernel's
# value may be 0), and any product or sum that falls below the normal range 2^-126, keeps only an absolute accuracy.  A
# relative bound of such a result underflows in fp64 too (|Mish(-700)| ~ 1e-302), so a correctly computed fp32 -0 would
# exceed it; these absolute terms are ~1e-35 and leave every normal-range bound as it was.
NORMAL_MIN = 2.0 ** -126


def mish_bound(z):
    """fp32 Mish(z) = z tanh(log1pf(expf(z))): expf, log1pf and tanhf are within 2 ulp (4 u relative) each; the relative error
    of e^z passes at most once through log1p (log1p(y) >= y / (1 + y)) and through tanh ((1 - t^2) s / t <= 1), so with the
    product Mish's relative error is at most 11 u, and |Mish(z)| <= |z|: 12 u (1 + |z|) also covers the softplus threshold at
    z = 20 and values near 0."""
    return 12 * U32 * (1 + abs(z))


def mish_grad_bound(z):
    """fp32 Mish'(z): tanh(softplus(z)) and 1 - tanh^2 carry absolute errors of a few u, scaled by |z| through z sigmoid(z)"""
    return (8 + 8 * abs(z)) * U32


def silu_bound(z):
    """fp32 silu(z) = z / (1 + expf(-z)): expf within 2 ulp (4 u), the add and the division u each: 6 u relative, 8 u allowed;
    TINY covers the overflow of 1 + expf(-z) below z = -88"""
    return 8 * U32 * np.abs(act(cabi.ACT_SILU, z)) + TINY


def silu_grad_bound(z):
    """fp32 silu'(z): sig carries 6 u relative (as in silu_bound), so 1 - sig an absolute 7 u (sig <= 1), z (1 - sig) 7 u |z| plus
    its rounding, 1 + that and the product with sig a rounding each: (12 + 12 |z|) u covers them with the margin of 2x on the
    roundings that the other bounds of the audit keep"""
    return (12 + 12 * np.abs(np.asarray(z, np.float64))) * U32


# the activations the backward kernels fuse: their fp32 evaluation's bound, and their derivative with its fp32 bound
ACT_BOUND = {cabi.ACT_MISH: mish_bound, cabi.ACT_SILU: silu_bound}
ACT_GRAD = {cabi.ACT_MISH: (mish_grad, mish_grad_bound), cabi.ACT_SILU: (silu_grad, silu_grad_bound)}


def update_bwd_bound(g, alpha, sigma, k0, k1):
    """CDS_OP_UPDATE_BWD: a handful of fp32 operations per element, each within u of its exact result, on terms of size at
    most |g| (|k0| + |k1|) (1 + 1/alpha + 1/sigma)^2; 16 u of that (the clip decisions are exact: grad_ref.update_bwd takes
    them in fp32 like the kernel)"""
    return 16 * U32 * np.abs(np.asarray(g, np.float64)) * (abs(k0) + abs(k1)) * (1 + 1 / alpha + 1 / sigma) ** 2


def dgrad_bound(dz, w, z=None, act_kind=cabi.ACT_NONE, before=None):
    """CDS_OP_DGRAD, out [+]= (dz W) act'(z): each output is one thread's fma chain over N, so the dot-product bound
    (N + 4) u |dz||W|, times |act'(z)| when the derivative is fused; the fp32 act' adds |dz W| times its bound (ACT_GRAD).
    An accumulating store (``before``: the output before the launch, for accumulate = 1 and for out_sum) adds
    2 u (|before| + |y|)."""
    dz, w = np.asarray(dz, np.float64), np.asarray(w, np.float64)
    dzw = dz @ w
    mag, y = np.abs(dz) @ np.abs(w), dzw
    bound = 0.0
    if act_kind != cabi.ACT_NONE:
        grad, grad_bound = ACT_GRAD[act_kind]
        z = np.asarray(z, np.float64)
        g = grad(z)
        mag, y = mag * np.abs(g), dzw * g
        bound = np.abs(dzw) * grad_bound(z)
    bound = bound + (dz.shape[1] + 4) * (U32 * mag + NORMAL_MIN)
    if before is not None:
        bound = bound + 2 * U32 * (np.abs(np.asarray(before, np.float64)) + np.abs(y))
    return bound


def wgrad_bound(dz, h, act_kind=cabi.ACT_NONE, dw_before=None, db_before=None):
    """CDS_OP_WGRAD -> (bound of dw (N, K), bound of db (N,)): each output sums the rows in order in one thread, so
    (rows + 8) u |dz|^T |act(h)| (the fp32 activation's relative error included) and (rows + 2) u sum_rows |dz| for the bias
    column; an accumulating store adds 2 u (|before| + |contribution|).  Underflow: a Mish of a pre-activation far below
    zero is exact only to TINY, and each of the rows + 8 roundings to NORMAL_MIN, absolutely."""
    dz = np.asarray(dz, np.float64)
    rows, adz = dz.shape[0], np.abs(dz)
    gw, gb = wgrad(dz, h, act_kind)
    bw = (rows + 8) * (U32 * (adz.T @ np.abs(act(act_kind, h))) + NORMAL_MIN)
    if act_kind == cabi.ACT_MISH:
        bw = bw + TINY * adz.sum(0)[:, None]
    bb = (rows + 2) * U32 * adz.sum(0)
    if dw_before is not None:
        bw = bw + 2 * U32 * (np.abs(np.asarray(dw_before, np.float64)) + np.abs(gw))
    if db_before is not None:
        bb = bb + 2 * U32 * (np.abs(np.asarray(db_before, np.float64)) + np.abs(gb))
    return bw, bb


# ---------------------------------------------------------------- differentiable calls audited operator by operator
# (tests/test_program_audit_cpu.py, tests/test_program_audit_gpu.py), 5 steps each
GRAD_CASES = {
    # Diffusion-QL's call: discrete eps-prediction clipped to [-1, 1]
    "dql-eps": dict(net=dict(obs_dim=17, act_dim=6, emb_dim=16), kind="discrete", predict_noise=True, solver="ddpm"),
    # continuous x0-prediction with a fix_mask
    "dql-x0": dict(net=dict(obs_dim=11, act_dim=3), kind="continuous", predict_noise=False, solver="sde_dpmsolver++_1"),
}


def grad_agent(case, device):
    """(agent, sample() keyword arguments without the prior and the condition) of a GRAD_CASES case"""
    from cleandiffuser_b200.diffusion import ContinuousDiffusionSDE, DiscreteDiffusionSDE
    from cleandiffuser_b200.nn_condition import IdentityCondition
    from cleandiffuser_b200.nn_diffusion import DQLMlp
    from cleandiffuser_b200.testing import load_synth
    import torch
    spec = GRAD_CASES[case]
    net = load_synth(DQLMlp(**spec["net"]), seed=1)
    a = spec["net"]["act_dim"]
    kw = dict(predict_noise=spec["predict_noise"], device=device)
    if spec["kind"] == "discrete":
        kw.update(x_max=torch.full((1, a), 1.0), x_min=torch.full((1, a), -1.0))
        agent = DiscreteDiffusionSDE(net, IdentityCondition(dropout=0.0), diffusion_steps=5, **kw)
    else:
        mask = torch.zeros(a)
        mask[0] = 1.
        agent = ContinuousDiffusionSDE(net, IdentityCondition(dropout=0.0), fix_mask=mask, **kw)
    return agent, dict(solver=spec["solver"], sample_steps=5, use_ema=False, w_cfg=1.0, requires_grad=True)
