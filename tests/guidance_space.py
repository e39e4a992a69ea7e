"""TEST INFRASTRUCTURE: the constructor space of the programs that compute gradients, as a deterministic case table:
classifier guidance inside the replayed loop (``lower.guidable`` -> ``lower_half_janner_grad``, ``lower_mlp_classifier_grad``,
``lower_qgpo_grad``) and ``sample(requires_grad=True)`` over DQLMlp (``lower.DQLGrad``, ``runtime.GradSamplerPlan``).

Constructor values decide which operator shapes the gradient programs reach: HalfJannerUNet1d's ``kernel_size`` becomes the
taps of ``w_conv_dgrad`` (flipped taps, zero-padded input channels), ``dim_mult`` and the horizon decide where the
two-phase Downsample gradient runs and where L reaches 1 (the centre-tap-only gradient), ``out_dim`` the width of the
``ones`` seed, ``model_dim`` x ``dim_mult`` the GroupNorm group sizes; the MLP widths the DGRAD / WGRAD tile edges; the
DQLMlp call the UPDATE_BWD clip and mask branches.  Each family's axes are crossed all-pairs (backbone_space.all_pairs),
plus one explicit case per reason the lowering or the runtime declines.

A classifier case is plain data: ``{"name", "family": "half_janner" | "mlp" | "qgpo", "head": "cumrew" | "mse" | "qgpo",
"ctor": constructor kwargs, "x": x_t shape without the batch, "cond": "batch" (a (batch, width) classifier condition) |
"none" | "wide" (one column too many) | "one_row" (a single row), "train", "mutate": a key of MUTATIONS or None,
"runs": the host module can evaluate the case, "want"}``.  ``want`` is

- ``"graph"``: ``guidable`` accepts the case and the lowered input gradient serves it;
- ``"refused"``: lowered, but the library refuses an operator (CdsError -3), so the GPU falls back to the callback;
- any other string: the exact reason ``guidable`` gives, and the guided call keeps the host callback.

A grad case (``family`` "dql") holds the DQLMlp constructor, the agent ("discrete" / "continuous"), the solver,
``predict_noise``, the bounds ("none" / "min" / "max" / "both"), the mask ("none" / "cols"), the steps, and ``want``:
``"graph"`` or the exact ``try_sample_grad`` decline.  A request case (``family`` "request") is a guided or differentiable
call the runtime declines whatever the classifier: its ``want`` is the exact reason.

The outcomes follow the modules' shapes and the lowering's documented structure, independently of engine/lower.py."""
import copy

import torch
import torch.nn as nn

from backbone_space import EMB_TYPES, all_pairs
from cleandiffuser_b200.classifier import CumRewClassifier, MSEClassifier, QGPOClassifier
from cleandiffuser_b200.nn_classifier import HalfJannerUNet1d, MLPNNClassifier, QGPONNClassifier
from cleandiffuser_b200.testing import synth_state_dict

ACTS = {"ReLU": nn.ReLU, "SiLU": nn.SiLU, "Mish": nn.Mish, "Tanh": nn.Tanh}
TRAIN = "classifier model_ema in train mode"


# ---- mutations: module edits no constructor makes --------------------------------------------------------------------
def _mixed_acts(net):
    net.mlp.mlp[1][1] = nn.SiLU()                       # the other stages keep their ReLU


def _stage_extra(net):
    net.mlp.mlp[0].append(nn.Identity())               # Linear -> act -> Identity


def _not_mlp(net):
    net.mlp = nn.Identity()


def _widths_break(net):
    lin = net.mlp.mlp[1][0]
    net.mlp.mlp[1][0] = nn.Linear(lin.in_features + 1, lin.out_features)


def _qgpo_mish(net):
    net.mlp.mlp[0][1] = nn.Mish()


def _qgpo_obs_width(net):
    net.obs_proj = nn.Linear(net.obs_proj.in_features, net.obs_proj.out_features + 1)


def _qgpo_no_time(net):
    lin = net.mlp.mlp[0][0]
    net.mlp.mlp[0][0] = nn.Linear(2 * net.act_proj.out_features, lin.out_features)


MUTATIONS = {"mixed_acts": _mixed_acts, "stage_extra": _stage_extra, "not_mlp": _not_mlp, "widths_break": _widths_break,
             "qgpo_mish": _qgpo_mish, "qgpo_obs_width": _qgpo_obs_width, "qgpo_no_time": _qgpo_no_time}


def _clf(family, head, ctor, x, cond="none", train=False, mutate=None, runs=True, want="graph"):
    return dict(family=family, head=head, ctor=ctor, x=tuple(x), cond=cond, train=train, mutate=mutate, runs=runs, want=want)


# ---- HalfJannerUNet1d under CumRewClassifier ---------------------------------------------------------------------------
def _half_janner():
    axes = dict(horizon=[1, 2, 4, 8, 32, 64, 256], dim_mult=[[1], [1, 2], [1, 4], [1, 2, 2], [1, 2, 2, 2], [1, 4, 2]],
                kernel_size=[3, 5, 7], model_dim=[16, 32, 64], emb_dim=[16, 32, 64], emb=EMB_TYPES, out_dim=[1, 3],
                in_dim=[3, 14, 16, 23, 37, 69])
    out = []
    for r in all_pairs(axes):
        ctor = dict(horizon=r["horizon"], in_dim=r["in_dim"], out_dim=r["out_dim"], kernel_size=r["kernel_size"],
                    model_dim=r["model_dim"], emb_dim=r["emb_dim"], dim_mult=r["dim_mult"], timestep_emb_type=r["emb"])
        out.append(_clf("half_janner", "cumrew", ctor, (r["horizon"], r["in_dim"])))
    base = dict(horizon=16, in_dim=6, kernel_size=5, model_dim=16, emb_dim=16, dim_mult=[1, 2])
    out += [_clf("half_janner", "cumrew", dict(base, horizon=1, dim_mult=[1, 2, 2, 2], kernel_size=7), (1, 6)),  # L = 1 early
            _clf("half_janner", "cumrew", dict(base, horizon=256, model_dim=64, dim_mult=[1]), (256, 6)),   # groups of 2048
            _clf("half_janner", "cumrew", base, (16, 6), train=True, want=TRAIN),
            _clf("half_janner", "cumrew", dict(base, horizon=12), (12, 6), runs=False, want="classifier horizon must be 2^n"),
            _clf("half_janner", "cumrew", dict(base, norm_type="layernorm"), (16, 6),
                 want="classifier norm_type other than groupnorm"),
            _clf("half_janner", "cumrew", base, (16, 7), runs=False, want="classifier in_dim does not match x"),
            _clf("half_janner", "cumrew", base, (32, 6), runs=False,
                 want="classifier final_block does not match its feature map"),
            _clf("half_janner", "mse", base, (16, 6), cond="batch", runs=False,
                 want="classifier network HalfJannerUNet1d (MLPNNClassifier only)")]
    return out


# ---- MLPNNClassifier under MSEClassifier and CumRewClassifier ----------------------------------------------------------
def _mlp():
    axes = dict(head=["mse", "cumrew"], hidden=[[1], [7], [33, 100], [256], [100, 7, 33], [1024], [7, 256, 1, 33]],
                x_dim=[1, 9, 23, 60], out_dim=[1, 7, 60], temperature=[0.3, 1.0, 4.0], act=["ReLU", "SiLU", "Mish"],
                emb_dim=[16, 32, 64], emb=EMB_TYPES)
    out = []
    for r in all_pairs(axes):
        od = r["out_dim"] if r["head"] == "mse" else 1
        ctor = dict(x_dim=r["x_dim"], out_dim=od, emb_dim=r["emb_dim"], hidden_dims=r["hidden"], act=r["act"],
                    timestep_emb_type=r["emb"], temperature=r["temperature"])
        out.append(_clf("mlp", r["head"], ctor, (r["x_dim"],), cond="batch" if r["head"] == "mse" else "none"))
    base = dict(x_dim=5, out_dim=3, emb_dim=16, hidden_dims=[32, 32], act="ReLU", temperature=1.0)
    mse = lambda **k: _clf("mlp", "mse", dict(base, **k.pop("ctor", {})), (5,), **dict(dict(cond="batch"), **k))  # noqa
    out += [mse(mutate="mixed_acts", want="classifier hidden activations differ (ReLU, SiLU)"),
            mse(ctor=dict(act="Tanh"), want="classifier activation Tanh (ReLU, SiLU or Mish only)"),
            mse(ctor=dict(out_act="Tanh"), want="classifier out_activation Tanh (Identity only)"),
            mse(ctor=dict(hidden_dims=[]), want="classifier mlp has no hidden layer"),
            mse(mutate="stage_extra", want="classifier mlp hidden stages are not Linear + activation"),
            mse(mutate="not_mlp", runs=False, want="classifier mlp is not an Mlp"),
            mse(mutate="widths_break", runs=False, want="classifier mlp widths do not chain"),
            _clf("mlp", "mse", base, (6,), cond="batch", runs=False, want="classifier x_dim does not match x"),
            _clf("mlp", "cumrew", base, (5,), want="classifier out_dim 3 (1 only under CumRewClassifier)"),
            mse(cond="none", runs=False, want="no classifier condition (condition_cg=None)"),
            mse(cond="wide", runs=False, want="classifier condition is not (batch, out_dim)"),
            mse(train=True, want=TRAIN)]
    return out


# ---- QGPOClassifier over QGPONNClassifier ------------------------------------------------------------------------------
def _qgpo():
    axes = dict(obs=[1, 3, 11, 17, 40], act=[1, 2, 6, 9], hidden=[[7], [64, 64], [256, 256, 256], [33, 100], [1024]],
                emb_dim=[16, 32, 64], emb=EMB_TYPES)
    out = []
    for r in all_pairs(axes):
        ctor = dict(obs_dim=r["obs"], act_dim=r["act"], emb_dim=r["emb_dim"], hidden_dims=r["hidden"],
                    timestep_emb_type=r["emb"])
        out.append(_clf("qgpo", "qgpo", ctor, (r["act"],), cond="batch"))
    base = dict(obs_dim=5, act_dim=3, emb_dim=16, hidden_dims=[32, 32])
    q = lambda **k: _clf("qgpo", "qgpo", base, (3,), **dict(dict(cond="batch"), **k))         # noqa: E731
    out += [q(train=True, want=TRAIN),
            q(mutate="qgpo_obs_width", runs=False, want="classifier obs_proj / act_proj are not Linears of one width"),
            q(mutate="qgpo_mish", want="classifier mlp is not Linear + SiLU layers under an out_dim-1 Linear"),
            q(mutate="qgpo_no_time", runs=False, want="classifier mlp input has no time-embedding columns"),
            _clf("qgpo", "qgpo", base, (4,), cond="batch", runs=False, want="classifier act_proj does not match x"),
            q(cond="none", runs=False, want="no classifier condition (condition_cg=None)"),
            q(cond="wide", runs=False, want="classifier condition does not match obs_proj")]
    return out


def _named(cases, prefix):
    return {f"{prefix}-{i:02d}": dict(c, name=f"{prefix}-{i:02d}") for i, c in enumerate(cases)}


CLASSIFIERS = {**_named(_half_janner(), "hj"), **_named(_mlp(), "mlp"), **_named(_qgpo(), "qgpo")}


def cond_width(case):
    """the width of the case's classifier condition (MSE: out_dim, QGPO: obs_dim)"""
    return case["ctor"].get("out_dim", 1) if case["head"] == "mse" else case["ctor"].get("obs_dim", 0)


def build_classifier(case, seed=0, device="cpu"):
    """the case's classifier with synthetic weights, the mutation applied, model_ema in the case's mode"""
    kw = dict(case["ctor"])
    if case["family"] == "half_janner":
        net = HalfJannerUNet1d(**kw)
    elif case["family"] == "mlp":
        act, out_act, temp = ACTS[kw.pop("act")](), kw.pop("out_act", None), kw.pop("temperature")
        net = MLPNNClassifier(activation=act, out_activation=ACTS[out_act]() if out_act else nn.Identity(), **kw)
    else:
        net = QGPONNClassifier(**kw)
    net.load_state_dict(synth_state_dict(net.state_dict(), seed))
    if case["head"] == "mse":
        clf = MSEClassifier(net, temperature=case["ctor"]["temperature"] if case["family"] == "mlp" else 1.0, device=device)
    elif case["head"] == "qgpo":
        clf = QGPOClassifier(net, device=device)
    else:
        clf = CumRewClassifier(net, device=device)
    if case["mutate"]:
        MUTATIONS[case["mutate"]](clf.model_ema)
        clf.model_ema.to(device)
    clf.model_ema.train(case["train"])
    return clf


def classifier_inputs(case, batch, seed=1, device="cpu"):
    """(x in [-1, 1], the classifier condition or None) for ``batch`` trajectories"""
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(batch, *case["x"], generator=g).clamp(-1, 1)
    w = cond_width(case)
    c = {"none": None, "batch": (batch, w), "wide": (batch, w + 1), "one_row": (1, w)}[case["cond"]]
    c = None if c is None else torch.randn(*c, generator=g)
    return x.to(device), None if c is None else c.to(device)


def input_gradient_fp64(clf, case, x, t, c):
    """d sum(logp) / d x of the case's classifier in fp64 autograd: this package's module, the time embedding evaluated in
    fp32 as the engine's table filler does"""
    import cg_ref
    net = copy.deepcopy(clf.model_ema).double()
    net.map_noise = cg_ref.Fp64Time(clf.model_ema.map_noise)
    xx = x.detach().double().clone().requires_grad_(True)
    if case["head"] == "qgpo":
        lp = net(xx, t, c.double())
    else:
        lp = net(xx, t)
        if case["head"] == "mse":
            lp = -clf.temperature * ((lp - c.double()) ** 2).mean(-1, keepdim=True)
    return torch.autograd.grad(lp.sum(), xx)[0]


# per-element tolerance of a whole input or parameter gradient: |got - ref| <= TOL (|ref| + s), s the RMS of the whole
# reference tensor.  s is the gradient's scale: a trajectory whose own gradient is small (a saturated tanh head, where the
# seed 1 - y^2 cancels; Mish far in its negative tail) keeps the absolute error of the operators that produce it, which is
# relative to that scale, not to the trajectory's.  fp32 sums in another order than fp64 autograd (the operators are held to
# their dot-product bounds one by one in the program audit); TF32 rounds every GEMM operand to a 10-bit mantissa, and under
# ReLU a pre-activation within that error of 0 can switch a unit's whole term.  The GroupNorms of a short HalfJannerUNet1d
# normalise groups of a few elements and amplify that rounding: horizon 2 with 7 taps reaches 8e-2 on the interpreter.
TOL = {"fp32": 2e-4, "tf32": 1e-1}


def per_element_frac(got, ref, math, tol=TOL):
    """largest |got - ref| / (tol (|ref| + s)) and the flat index where it occurs"""
    got, ref = got.double().cpu().reshape(-1), ref.double().cpu().reshape(-1)
    s = float(ref.pow(2).mean().sqrt()) or 1e-30
    err = (got - ref).abs()
    frac = torch.where(torch.isfinite(err), err / (tol[math] * (ref.abs() + s)), torch.full_like(err, float("inf")))
    i = int(frac.argmax())
    return float(frac[i]), i


# ---- DQLMlp under sample(requires_grad=True) -------------------------------------------------------------------------
def _dql():
    axes = dict(obs=[1, 4, 9], act=[1, 2, 5, 9], emb_dim=[16, 32, 64], emb=EMB_TYPES, agent=["discrete", "continuous"],
                solver=["ddpm", "ddim", "ode_dpmsolver_1", "sde_dpmsolver++_1"], predict_noise=[True, False],
                bounds=["none", "min", "max", "both"], mask=["none", "cols"], steps=[1, 2, 5])
    out = []
    for r in all_pairs(axes):
        mask = r["mask"] if r["act"] > 1 else "none"            # a mask over every column leaves nothing to sample
        out.append(dict(family="dql", ctor=dict(obs_dim=r["obs"], act_dim=r["act"], emb_dim=r["emb_dim"],
                                                timestep_emb_type=r["emb"]),
                        agent=r["agent"], solver=r["solver"], predict_noise=r["predict_noise"], bounds=r["bounds"],
                        mask=mask, steps=r["steps"], w_cfg=1.0, math=None, want="graph"))
    base = dict(family="dql", ctor=dict(obs_dim=4, act_dim=3, emb_dim=16), agent="discrete", solver="ddpm",
                predict_noise=True, bounds="both", mask="none", steps=3, w_cfg=1.0, math=None)
    out += [dict(base, solver="ode_dpmsolver++_2M", want="requires_grad=True with the multistep solver ode_dpmsolver++_2M (history)"),
            dict(base, solver="sde_dpmsolver++_2M", want="requires_grad=True with the multistep solver sde_dpmsolver++_2M (history)"),
            dict(base, w_cfg=1.5, want="requires_grad=True with two-branch classifier-free guidance"),
            dict(base, guided=True, want="requires_grad=True with classifier guidance"),
            dict(base, math="bf16", want="requires_grad=True with CDS_MATH=bf16 (fp32 and tf32 only)")]
    return out


GRADS = _named(_dql(), "dql")


def bounds(case):
    """(x_min, x_max) of a grad case: per element, non-uniform, the last element with min > max where both are set"""
    a = case["ctor"]["act_dim"]
    lo = -0.6 - 0.3 * torch.arange(a, dtype=torch.float32) / max(a - 1, 1)
    hi = 0.5 + 0.4 * torch.cos(torch.arange(a, dtype=torch.float32))
    if case["bounds"] == "both":
        lo[-1], hi[-1] = 0.3, -0.2                       # min > max: torch.clip's max bound wins
    x_min = lo[None] if case["bounds"] in ("min", "both") else None
    x_max = hi[None] if case["bounds"] in ("max", "both") else None
    return x_min, x_max


def fix_mask(case):
    """a non-uniform multi-column mask (every other column from the first fixed) or None"""
    if case["mask"] == "none":
        return None
    m = torch.zeros(case["ctor"]["act_dim"])
    m[::2] = 1.0
    m[-1] = 0.0
    return m


# ---- guided and differentiable requests the runtime declines whatever the classifier ---------------------------------
REQUESTS = {"cfg-and-guidance": "classifier guidance together with two-branch classifier-free guidance",
            "bf16": "CDS_MATH=bf16",
            "condition-rows": "classifier condition rows != batch",
            "branches": "more than one sub-batch chain (CDS_BRANCHES)"}      # the GPU test: CDS_BRANCHES=2
