"""TEST INFRASTRUCTURE: the constructor space of the nine backbones ``lower_denoiser`` lowers, as a deterministic case table.

Constructor values decide which kernel and which instantiation every operator reaches: ``kernel_size`` becomes the conv
taps, ``model_dim`` x ``dim_mult`` the channel widths (tensor-core widths or conv_simt), the horizon L (conv_tc needs
L <= 32, conv_simt's GroupNorm tile holds 128 / L whole trajectories), DiT1d's head_dim and L the attention kernel,
``in_dim`` / ``act_dim`` the x_t cast widths, the condition and ``cond_predict_scale`` the FiLM columns.  Each backbone's
axes are crossed all-pairs (every pair of values of two axes appears in some case) rather than as a full product, plus
explicit cases for every reason the lowering declines.

A case is plain data: ``{"name", "kind", "ctor": constructor kwargs, "x": x_t shape without the batch, "cond": the
condition's shape without the batch or None, "t": "int" (discrete time) | "float", "train": module in train mode,
"mutate": a key of MUTATIONS or None, "want": outcome}``.  ``want`` is

- ``"served"``: the lowered program runs on the device;
- ``"refused"``: the lowering succeeds but the library refuses an operator (CdsError -3, e.g. a GroupNorm layer conv_simt
  cannot tile), so on the GPU ``sample()`` takes the PyTorch loop; the interpreter does not ask, so on the CPU it runs;
- ``"unsupported: <text>"``: ``lower_denoiser`` raises ``Unsupported`` with ``<text>`` in its message.

The outcome is derived here from the modules' and the kernels' documented limits, independently of engine/lower.py."""
import copy
import itertools

import numpy as np
import torch
import torch.nn as nn

from mlp_programs import _Widened
from cleandiffuser_b200.diffusion import ContinuousDiffusionSDE, DiscreteDiffusionSDE
from cleandiffuser_b200.engine import cabi
from cleandiffuser_b200.nn_condition import IdentityCondition
from cleandiffuser_b200.nn_diffusion import (ChiTransformer, ChiUNet1d, DiT1d, DQLMlp, DVInvMlp, IDQLMlp, JannerUNet1d,
                                             PearceMlp, SfBCUNet)
from cleandiffuser_b200.testing import synth_state_dict

CLASSES = {c.__name__: c for c in (JannerUNet1d, ChiUNet1d, DiT1d, ChiTransformer, DQLMlp, DVInvMlp, IDQLMlp, SfBCUNet,
                                   PearceMlp)}
SEQUENCE_KINDS = ("JannerUNet1d", "ChiUNet1d", "DiT1d", "ChiTransformer")       # x_t (horizon, channels); the MLPs: (act_dim,)
EMB_TYPES = ["positional", "fourier", "untrainable_fourier", "untrainable_positional"]


def all_pairs(axes):
    """deterministic all-pairs covering array over ``axes`` (name -> list of values): greedy, one case at a time, each case
    seeded with the first pair still uncovered and completed axis by axis with the value that covers most new pairs"""
    k = len(axes)
    sizes = [len(v) for v in axes.values()]
    todo = {(a, i, b, j) for a, b in itertools.combinations(range(k), 2) for i in range(sizes[a]) for j in range(sizes[b])}
    rows = []
    while todo:
        a, i, b, j = min(todo)
        row = {a: i, b: j}
        for n in range(k):
            if n not in row:
                gain = lambda v: sum(((m, row[m], n, v) if m < n else (n, v, m, row[m])) in todo for m in row)
                row[n] = max(range(sizes[n]), key=lambda v: (gain(v), -v))
        todo -= {(m, row[m], n, row[n]) for m, n in itertools.combinations(range(k), 2)}
        rows.append({name: vals[row[n]] for n, (name, vals) in enumerate(axes.items())})
    return rows


# ---- kernel limits the outcome follows (csrc/cds_api.cu conv_pick, attn_pick, mha_pick; csrc/conv_simt.cuh) -------------
def _gn_groups(c):
    """GroupNorm1d(c, 8, 4): groups = min(8, c // 4)"""
    return min(8, c // 4)


def gn_servable(c, L):
    """can a GroupNorm layer of c channels at length L run (conv_tc at L <= 32 with 8 groups of a tensor-core width, else
    conv_simt: a column tile of 32, 64 or 128 holds whole groups, a row tile of 128 whole trajectories)"""
    cpg = c // _gn_groups(c)
    return any(bn % cpg == 0 for bn in (32, 64, 128)) and L <= 128 and 128 % L == 0


def _unet(kind, ctor, L, has_cond):
    mult = list(np.cumprod(ctor["dim_mult"]))
    n = len(mult)
    if kind == "JannerUNet1d":
        if ctor.get("attention"):
            return "unsupported: attention=True"
        if ctor.get("norm_type", "groupnorm") != "groupnorm":
            return "unsupported: norm_type other than groupnorm"
    elif not has_cond:
        return "unsupported: ChiUNet1d needs a condition"
    if L & (L - 1):
        return "unsupported: horizon must be 2^n"
    if L >> (n - 1) < 1:
        return "unsupported: horizon too short"
    if mult[0] != 1:                     # the last stage gives model_dim * dim_mult[0] channels, final_conv takes model_dim
        return "unsupported: final_conv takes"
    md = ctor["model_dim"]
    if not all(gn_servable(md * m, L >> s) for s, m in enumerate(mult)):
        return "refused"
    return "served"


def expected(case):
    kind, ctor, x, cond = case["kind"], case["ctor"], case["x"], case["cond"]
    if len(x) != (2 if kind in SEQUENCE_KINDS else 1):
        return f"unsupported: backbone {kind} with x_shape"
    if kind in ("JannerUNet1d", "ChiUNet1d"):
        return _unet(kind, ctor, x[0], cond is not None)
    if kind == "DiT1d":
        return "unsupported: attention dropout in train mode" if case["train"] and ctor.get("dropout", 0) else "served"
    if kind == "ChiTransformer":
        if ctor.get("n_cond_layers", 0):
            return "unsupported: n_cond_layers > 0"
        if case["train"]:
            return "unsupported: in train mode (dropout)"
        if case["mutate"] == "post_norm_decoder":
            return "unsupported: decoder other than norm_first"
        if x[0] != ctor["Ta"]:
            return "unsupported: horizon != Ta"
        hd = ctor["d_model"] // ctor["nhead"]
        return "served" if hd % 32 == 0 and ctor["Ta"] <= 64 and 1 + ctor["To"] <= 64 else "refused"
    if kind == "DVInvMlp" and cond is None:
        return "unsupported: DVInvMlp needs a condition"
    if kind == "IDQLMlp":
        if case["train"]:
            return "unsupported: IDQLMlp in train mode"
        if case["mutate"] == "ln_without_affine":
            return "unsupported: LayerNorm without affine"
    if kind == "PearceMlp":
        if case["mutate"] == "tanh_gelu":
            return "unsupported: PearceMlp FCBlock other than"
        return "served" if gn_servable(ctor["hidden_dim"], 1) else "refused"
    return "served"


# ---- mutations: module edits no constructor makes, for the lowering's structural checks -------------------------------
def _no_upsample(net):
    net.ups[0][3] = nn.Identity()


def _ln_without_affine(net):
    blk = net.ln_resnet[0]
    blk.net[1] = nn.LayerNorm(blk.net[1].normalized_shape, elementwise_affine=False)


def _tanh_gelu(net):
    net.fcs[1].model[2] = nn.GELU(approximate="tanh")


def _post_norm_decoder(net):
    for layer in net.decoder.layers:
        layer.norm_first = False


MUTATIONS = {"no_upsample": _no_upsample, "ln_without_affine": _ln_without_affine, "tanh_gelu": _tanh_gelu,
             "post_norm_decoder": _post_norm_decoder}


def _case(kind, ctor, x, cond, t, train=False, mutate=None, want=None):
    c = dict(kind=kind, ctor=ctor, x=tuple(x), cond=None if cond is None else tuple(cond), t=t, train=train, mutate=mutate)
    c["want"] = want or expected(c)
    return c


# ---- the nine backbones ---------------------------------------------------------------------------------------------
def _janner():
    axes = dict(kernel_size=[3, 5, 7], dim_mult=[[1], [1, 2], [1, 4], [1, 2, 2], [1, 2, 2, 2], [1, 4, 2]],
                model_dim=[8, 16, 24, 32], horizon=[4, 8, 32, 64, 128, 256], in_dim=[3, 14, 16, 32, 37],
                cond=[False, True], emb=EMB_TYPES, t=["int", "float"])
    out = []
    for r in all_pairs(axes):
        ctor = dict(in_dim=r["in_dim"], model_dim=r["model_dim"], emb_dim=16, kernel_size=r["kernel_size"],
                    dim_mult=r["dim_mult"], timestep_emb_type=r["emb"])
        out.append(_case("JannerUNet1d", ctor, (r["horizon"], r["in_dim"]), (16,) if r["cond"] else None, r["t"]))
    base = dict(in_dim=6, model_dim=16, emb_dim=16, kernel_size=5, dim_mult=[1, 2])
    out += [_case("JannerUNet1d", dict(base, dim_mult=[2]), (8, 6), None, "int"),             # single stage, 32 channels
            _case("JannerUNet1d", dict(base, dim_mult=[4]), (16, 6), (16,), "float"),
            _case("JannerUNet1d", dict(base, dim_mult=[2, 2]), (16, 6), None, "int"),
            _case("JannerUNet1d", dict(base, dim_mult=[1]), (16, 6), None, "int"),              # single stage, 16 channels
            _case("JannerUNet1d", dict(base, attention=True), (16, 6), None, "int"),
            _case("JannerUNet1d", dict(base, norm_type="layernorm"), (16, 6), None, "int"),
            _case("JannerUNet1d", base, (12, 6), None, "int"),
            _case("JannerUNet1d", dict(base, dim_mult=[1, 2, 2, 2]), (4, 6), None, "int"),
            _case("JannerUNet1d", base, (16, 6), None, "int", mutate="no_upsample", want="unsupported: up stage without"),
            _case("JannerUNet1d", dict(base, model_dim=48, dim_mult=[1, 2]), (16, 6), None, "int"),
            _case("JannerUNet1d", dict(base, model_dim=32, dim_mult=[1, 3]), (16, 6), (16,), "int")]
    return out


def _chi():
    axes = dict(kernel_size=[3, 5, 7], dim_mult=[[1], [1, 2], [1, 2, 2], [1, 2, 2, 2], [1, 4]], model_dim=[8, 16, 32],
                horizon=[4, 8, 16, 32, 64, 128], act_dim=[2, 7, 16, 33], scale=[True, False], To=[1, 2], emb=EMB_TYPES,
                t=["int", "float"])
    out = []
    for r in all_pairs(axes):
        ctor = dict(act_dim=r["act_dim"], obs_dim=5, To=r["To"], model_dim=r["model_dim"], emb_dim=16,
                    kernel_size=r["kernel_size"], cond_predict_scale=r["scale"], dim_mult=r["dim_mult"],
                    timestep_emb_type=r["emb"])
        out.append(_case("ChiUNet1d", ctor, (r["horizon"], r["act_dim"]), (r["To"], 5), r["t"]))
    base = dict(act_dim=4, obs_dim=5, To=2, model_dim=16, emb_dim=16, kernel_size=5, dim_mult=[1, 2])
    out += [_case("ChiUNet1d", base, (8, 4), None, "int"),
            _case("ChiUNet1d", dict(base, obs_as_global_cond=False), (8, 4), (2, 5), "int",
                  want="unsupported: obs_as_global_cond=False"),
            _case("ChiUNet1d", base, (12, 4), (2, 5), "int"),
            _case("ChiUNet1d", dict(base, dim_mult=[2]), (8, 4), (2, 5), "int"),
            _case("ChiUNet1d", dict(base, dim_mult=[1, 2, 2, 2]), (4, 4), (2, 5), "float"),
            _case("ChiUNet1d", base, (256, 4), (2, 5), "int"),
            _case("ChiUNet1d", dict(base, model_dim=24, dim_mult=[1, 2]), (16, 4), (2, 5), "float")]
    return out


def _dit():
    axes = dict(width=[(64, 4), (96, 3), (128, 2), (256, 8), (192, 3)], horizon=[7, 16, 100, 128, 130, 200],
                in_dim=[3, 16, 29, 32, 40], depth=[1, 2], cond=[False, True], emb=EMB_TYPES, t=["int", "float"])
    out = []
    for r in all_pairs(axes):
        d, h = r["width"]
        ctor = dict(in_dim=r["in_dim"], emb_dim=32, d_model=d, n_heads=h, depth=r["depth"], timestep_emb_type=r["emb"])
        out.append(_case("DiT1d", ctor, (r["horizon"], r["in_dim"]), (32,) if r["cond"] else None, r["t"]))
    out += [_case("DiT1d", dict(in_dim=5, emb_dim=32, d_model=64, n_heads=2, depth=1, dropout=0.1), (16, 5), None, "int",
                  train=True),
            _case("DiT1d", dict(in_dim=5, emb_dim=32, d_model=64, n_heads=2, depth=1), (5,), None, "int")]
    return out


def _chitransformer():
    axes = dict(width=[(64, 2), (128, 4), (128, 2), (192, 3), (256, 4)], Ta=[1, 4, 8, 10, 16, 33], To=[1, 2, 3, 8],
                act_dim=[2, 7, 16], obs_dim=[5, 20], layers=[1, 2], cond=[True, False], emb=EMB_TYPES, t=["int", "float"])
    out = []
    for r in all_pairs(axes):
        d, h = r["width"]
        ctor = dict(act_dim=r["act_dim"], obs_dim=r["obs_dim"], Ta=r["Ta"], To=r["To"], d_model=d, nhead=h,
                    num_layers=r["layers"], timestep_emb_type=r["emb"])
        out.append(_case("ChiTransformer", ctor, (r["Ta"], r["act_dim"]), (r["To"], r["obs_dim"]) if r["cond"] else None,
                         r["t"]))
    base = dict(act_dim=3, obs_dim=5, Ta=8, To=2, d_model=64, nhead=2, num_layers=1)
    out += [_case("ChiTransformer", dict(base, n_cond_layers=1), (8, 3), (2, 5), "int"),
            _case("ChiTransformer", base, (8, 3), (2, 5), "int", train=True),
            _case("ChiTransformer", base, (8, 3), (2, 5), "int", mutate="post_norm_decoder"),
            _case("ChiTransformer", base, (4, 3), (2, 5), "int"),
            _case("ChiTransformer", dict(base, nhead=4), (8, 3), (2, 5), "float"),              # head_dim 16
            _case("ChiTransformer", dict(base, Ta=65), (65, 3), (2, 5), "int")]
    return out


def _mlps():
    out = []
    axes = dict(obs=[3, 17, 32], act=[1, 6, 16, 33], emb=[16, 32, 64], cond=[True, False], etype=EMB_TYPES,
                t=["int", "float"])
    for r in all_pairs(axes):
        ctor = dict(obs_dim=r["obs"], act_dim=r["act"], emb_dim=r["emb"], timestep_emb_type=r["etype"])
        out.append(_case("DQLMlp", ctor, (r["act"],), (r["obs"],) if r["cond"] else None, r["t"]))
    axes = dict(obs=[3, 17, 32], act=[1, 6, 33], hidden=[48, 96, 192, 256], emb=[16, 32], etype=EMB_TYPES, t=["int", "float"])
    for r in all_pairs(axes):
        ctor = dict(obs_dim=r["obs"], act_dim=r["act"], emb_dim=r["emb"], hidden_dim=r["hidden"], timestep_emb_type=r["etype"])
        out.append(_case("DVInvMlp", ctor, (r["act"],), (2 * r["obs"],), r["t"]))
    # (act_dim 1 of IDQLMlp: with synthetic weights its one output cancels to ~1 % of its terms, and the TF32 rounding of the
    # weights alone moves it by 3e-3 -- a conditioning outlier of the whole-network bound, not a lowering check)
    axes = dict(obs=[3, 17], act=[2, 6, 16, 33], hidden=[48, 64, 96, 192, 256], blocks=[1, 2, 3, 5], cond=[True, False],
                etype=EMB_TYPES, t=["int", "float"])
    for r in all_pairs(axes):
        ctor = dict(obs_dim=r["obs"], act_dim=r["act"], emb_dim=32, hidden_dim=r["hidden"], n_blocks=r["blocks"],
                    timestep_emb_type=r["etype"])
        out.append(_case("IDQLMlp", ctor, (r["act"],), (r["obs"],) if r["cond"] else None, r["t"]))
    axes = dict(act=[1, 6, 16, 33], hidden=[(64,), (128, 64), (96, 48, 24), (256, 128, 64, 32), (48, 96)], emb=[32, 64],
                cond=[True, False], etype=EMB_TYPES, t=["int", "float"])
    for r in all_pairs(axes):
        ctor = dict(act_dim=r["act"], emb_dim=r["emb"], hidden_dims=r["hidden"], timestep_emb_type=r["etype"])
        out.append(_case("SfBCUNet", ctor, (r["act"],), (r["emb"],) if r["cond"] else None, r["t"]))
    axes = dict(act=[2, 7, 9, 33], To=[1, 2, 3], hidden=[32, 64, 128, 256], emb=[16, 32, 64], cond=[True, False],
                etype=EMB_TYPES, t=["int", "float"])
    for r in all_pairs(axes):
        ctor = dict(act_dim=r["act"], To=r["To"], emb_dim=r["emb"], hidden_dim=r["hidden"], timestep_emb_type=r["etype"])
        out.append(_case("PearceMlp", ctor, (r["act"],), (r["To"], r["emb"]) if r["cond"] else None, r["t"]))
    out += [_case("DVInvMlp", dict(obs_dim=5, act_dim=3, emb_dim=16, hidden_dim=64), (3,), None, "int"),
            _case("IDQLMlp", dict(obs_dim=5, act_dim=3, emb_dim=16, hidden_dim=64, n_blocks=2), (3,), (5,), "int", train=True),
            _case("IDQLMlp", dict(obs_dim=5, act_dim=3, emb_dim=16, hidden_dim=64, n_blocks=2), (3,), (5,), "int",
                  mutate="ln_without_affine"),
            _case("PearceMlp", dict(act_dim=3, To=1, emb_dim=16, hidden_dim=64), (3,), None, "int", mutate="tanh_gelu"),
            _case("PearceMlp", dict(act_dim=3, To=1, emb_dim=16, hidden_dim=96), (3,), (1, 16), "float"),
            _case("SfBCUNet", dict(act_dim=3, emb_dim=32, hidden_dims=(64, 32)), (4, 3), None, "int"),
            _case("DQLMlp", dict(obs_dim=5, act_dim=3, emb_dim=16), (4, 3), (5,), "int")]
    return out


def _named(cases):
    out, seen = {}, {}
    for c in cases:
        k = c["kind"]
        seen[k] = seen.get(k, 0) + 1
        out[f"{k}-{seen[k]:02d}"] = dict(c, name=f"{k}-{seen[k]:02d}")
    return out


CASES = _named(_janner() + _chi() + _dit() + _chitransformer() + _mlps())


def build(case, seed=0):
    """the case's module on the CPU, synthetic weights (ChiTransformer keeps its attention masks), eval or train mode"""
    net = CLASSES[case["kind"]](**case["ctor"])
    sd = synth_state_dict(net.state_dict(), seed)
    for k in ("mask", "memory_mask"):
        if k in sd:
            sd[k] = net.state_dict()[k].clone()
    net.load_state_dict(sd)
    if case["mutate"]:
        MUTATIONS[case["mutate"]](net)
    return net.train(case["train"])


def inputs(case, batch, seed=1, device="cpu"):
    """(x, t: one time of the case's kind, condition or None) for ``batch`` trajectories"""
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(batch, *case["x"], generator=g)
    t = torch.tensor([417]) if case["t"] == "int" else torch.tensor([0.37])
    cond = None if case["cond"] is None else torch.randn(batch, *case["cond"], generator=g)
    return x.to(device), t.to(device), None if cond is None else cond.to(device)


def reference(net, case, x, t, cond):
    """the module in float64 on ``x`` at the batch-constant time ``t``.  The time embedding is evaluated as the module
    evaluates it (in float32; integer time with int64 phases), then widened: the lowering fills its per-call tables with
    the module's own ``map_noise`` by design, and a fourier embedding's float32 phases (frequencies ~16) alone move
    PearceMlp's output, whose first layer reads the embedding raw, by ~1e-5"""
    net64 = copy.deepcopy(net).double()
    B = x.shape[0]
    net64.map_noise = _Widened(net.map_noise)
    tt = t.expand(B)
    if cond is None and case["kind"] == "ChiTransformer":        # its own stand-in for a missing condition is float32
        cond = torch.zeros(B, net.To, net.obs_dim, device=x.device)
    with torch.no_grad():
        return net64(x.double(), tt, None if cond is None else cond.double())


def rel_err(y, ref):
    """normwise relative error"""
    y, ref = y.to(torch.float64).reshape(ref.shape[0], -1), ref.reshape(ref.shape[0], -1)
    return float((y - ref.to(y.device)).norm() / ref.norm())


def library_outcome(ops):
    """"refused" when the library refuses some operator of ``ops`` (CdsError -3, what sends sample() to the PyTorch loop
    on the GPU), else "served" (the host-side choice queries of libcds, no device needed)"""
    choice = {cabi.OP_CONV: ("conv", cabi.conv_choice), cabi.OP_ATTN: ("attn", cabi.attn_choice),
              cabi.OP_MHA: ("mha", cabi.mha_choice)}
    for op in ops:
        if op.kind in choice:
            field, ask = choice[op.kind]
            try:
                ask(getattr(op.u, field))
            except cabi.CdsError as e:
                if e.code != -3:
                    raise
                return "refused"
    return "served"


def agent(case, net, device, steps):
    """a DDPM-solver agent over ``net`` (discrete or continuous time as the case's ``t``); ``net`` itself is sampled
    (use_ema=False), in the mode the case asks for"""
    cls = DiscreteDiffusionSDE if case["t"] == "int" else ContinuousDiffusionSDE
    kw = dict(diffusion_steps=steps) if case["t"] == "int" else {}
    a = cls(net, IdentityCondition(dropout=0.0), device=device, **kw)
    a.model.train(case["train"])
    return a


def sample(a, case, batch, steps, device, seed=3):
    """x0 of one seeded sample() of ``batch`` trajectories"""
    g = torch.Generator().manual_seed(seed)
    cond = None if case["cond"] is None else torch.randn(batch, *case["cond"], generator=g).to(device)
    torch.manual_seed(seed)
    if device != "cpu":
        torch.cuda.manual_seed(seed)
    x0, _ = a.sample(torch.zeros(batch, *case["x"], device=device), "ddpm", n_samples=batch, sample_steps=steps,
                     condition_cfg=cond, w_cfg=1.0 if cond is not None else 0.0, use_ema=False)
    return x0
