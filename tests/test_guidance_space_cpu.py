"""The constructor space of the gradient programs (tests/guidance_space.py) on the interpreter (tests/emulator.py): every
classifier ``guidable`` accepts gives its input gradient within the per-element bound of fp64 autograd of this package's
module in fp32 and TF32, and the library's host-side queries serve exactly the cases labelled "graph"; every
``sample(requires_grad=True)`` over DQLMlp gives every parameter and condition gradient within the per-element bound of
fp64 autograd of the PyTorch reverse loop.  Every declined case gives exactly its labelled reason, keeps the host callback
or the PyTorch loop, and gives that path's result; every reason the lowering and the runtime can give is reached."""
import copy
import inspect
import re

import pytest
import torch

import backbone_space as bs
import cg_ref
import emulator
import guidance_space as gs
import relu_ref
from cleandiffuser_b200.diffusion import ContinuousDiffusionSDE, DiscreteDiffusionSDE
from cleandiffuser_b200.engine import cabi, lower, runtime
from cleandiffuser_b200.nn_condition import IdentityCondition
from cleandiffuser_b200.nn_diffusion import DiT1d, DQLMlp
from cleandiffuser_b200.testing import NoiseTape, ToyClassifier, load_synth

BATCH = 5                            # no multiple of any tile
MATHS = {"fp32": cabi.MATH_FP32, "tf32": cabi.MATH_TF32_TC}
T_ALL = torch.tensor([417, 3])       # the gradient is taken at iteration 1
LOWERED = [n for n, c in gs.CLASSIFIERS.items() if c["want"] in ("graph", "refused")]
DECLINED = [n for n, c in gs.CLASSIFIERS.items() if c["want"] not in ("graph", "refused")]
GRAD_SERVED = [n for n, c in gs.GRADS.items() if c["want"] == "graph"]
GRAD_DECLINED = [n for n, c in gs.GRADS.items() if c["want"] != "graph"]


@pytest.fixture(autouse=True)
def _relu(monkeypatch):
    relu_ref.register(monkeypatch)     # CDS_ACT_RELU in the shared operator references (tests/relu_ref.py)


@pytest.mark.parametrize("math", list(MATHS))
@pytest.mark.parametrize("name", LOWERED)
def test_lowered_input_gradient_matches_fp64_autograd(name, math):
    case = gs.CLASSIFIERS[name]
    clf = gs.build_classifier(case)
    x, c = gs.classifier_inputs(case, BATCH)
    assert lower.guidable(clf, case["x"], c) is None
    got, p = cg_ref.lowered_gradient(clf, x, T_ALL, 1, MATHS[math], "cpu", cond=c)
    want = gs.input_gradient_fp64(clf, case, x, T_ALL[1].expand(BATCH), c)
    frac, where = gs.per_element_frac(got, want, math)
    assert frac <= 1.0, (name, case["ctor"], frac, where)
    outcome = bs.library_outcome(p.ops)
    assert {"served": "graph"}.get(outcome, outcome) == case["want"], (name, case["ctor"])


# ---- guided sample() around a classifier ---------------------------------------------------------------------------
def guided_agent(case, clf, device="cpu"):
    """a small denoiser the engine serves at the case's x shape (DiT1d over (horizon, channels): any horizon; DQLMlp over
    (x_dim,)), guided by ``clf`` -> (agent, denoiser condition or None)"""
    x = case["x"]
    if len(x) == 2:
        net = load_synth(DiT1d(in_dim=x[1], emb_dim=32, d_model=64, n_heads=2, depth=1), seed=4)
        return DiscreteDiffusionSDE(net, classifier=clf, diffusion_steps=10, device=device), None
    net = load_synth(DQLMlp(obs_dim=3, act_dim=x[0], emb_dim=16), seed=4)
    return DiscreteDiffusionSDE(net, IdentityCondition(dropout=0.0), classifier=clf, diffusion_steps=10, device=device), 3


def guided_sample(agent, obs_dim, batch, cond_cg, tape, device="cpu", w_cfg=1.0, x_shape=None):
    g = torch.Generator().manual_seed(9)
    cond = None if obs_dim is None else torch.randn(batch, obs_dim, generator=g).to(device)
    with tape.active():
        x0, _ = agent.sample(torch.zeros(batch, *x_shape, device=device), "ddpm", n_samples=batch, sample_steps=2,
                             use_ema=False, condition_cfg=cond, w_cfg=w_cfg if cond is not None else 0.0,
                             condition_cg=cond_cg, w_cg=0.3)
    return x0


@pytest.mark.parametrize("name", DECLINED)
def test_declined_classifier_gives_its_reason_and_keeps_the_callback(name, monkeypatch):
    case = gs.CLASSIFIERS[name]
    clf = gs.build_classifier(case)
    x, c = gs.classifier_inputs(case, BATCH)
    assert lower.guidable(clf, case["x"], c) == case["want"]
    if not case["runs"]:                  # the host module cannot evaluate it: the reason is all there is to check
        return
    emulator.emulate(monkeypatch)
    monkeypatch.setenv("CDS_MATH", "fp32")
    monkeypatch.setenv("CDS_BACKEND", "cuda")
    agent, obs = guided_agent(case, clf)
    called = []
    inner = clf.gradients
    monkeypatch.setattr(clf, "gradients", lambda *a, **k: called.append(1) or inner(*a, **k))
    calls, tape = runtime.STATS["engine_calls"], NoiseTape()
    got = guided_sample(agent, obs, BATCH, c, tape, x_shape=case["x"])
    assert runtime.STATS["engine_calls"] == calls + 1
    assert runtime.STATS["guidance_path"] == "callback" and runtime.STATS["guidance_reason"] == case["want"]
    assert called
    monkeypatch.setenv("CDS_BACKEND", "torch")
    want = guided_sample(agent, obs, BATCH, c, NoiseTape(tape.draws), x_shape=case["x"])
    torch.testing.assert_close(got, want, rtol=1e-4, atol=1e-4)


def _request_agent():
    case = gs.CLASSIFIERS[next(n for n, c in gs.CLASSIFIERS.items() if c["family"] == "mlp" and c["head"] == "mse"
                               and c["want"] == "graph")]
    return case, gs.build_classifier(case)


@pytest.mark.parametrize("request_", [r for r in gs.REQUESTS if r != "branches"])
def test_declined_guided_request_gives_its_reason(request_, monkeypatch):
    emulator.emulate(monkeypatch)
    monkeypatch.setenv("CDS_MATH", "bf16" if request_ == "bf16" else "fp32")
    monkeypatch.setenv("CDS_BACKEND", "auto")
    case, clf = _request_agent()
    batch = 8
    _, c = gs.classifier_inputs(case, batch)
    if request_ == "condition-rows":
        c = c[:1]
    agent, obs = guided_agent(case, clf)
    calls, falls, tape = runtime.STATS["engine_calls"], runtime.STATS["fallbacks"], NoiseTape()
    got = guided_sample(agent, obs, batch, c, tape, w_cfg=1.5 if request_ == "cfg-and-guidance" else 1.0, x_shape=case["x"])
    want_reason = gs.REQUESTS[request_]
    if request_ == "cfg-and-guidance":         # the whole call takes the PyTorch loop
        assert runtime.STATS["engine_calls"] == calls and runtime.STATS["fallbacks"] == falls + 1
        assert runtime.STATS["last_fallback_reason"] == want_reason
    else:
        assert runtime.STATS["engine_calls"] == calls + 1
        assert runtime.STATS["guidance_path"] == "callback" and runtime.STATS["guidance_reason"] == want_reason
    monkeypatch.setenv("CDS_BACKEND", "torch")
    want = guided_sample(agent, obs, batch, c, NoiseTape(tape.draws), w_cfg=1.5 if request_ == "cfg-and-guidance" else 1.0,
                         x_shape=case["x"])
    if request_ == "bf16":                     # a bf16 denoiser program is far from the fp32 PyTorch loop whatever the guidance
        assert torch.isfinite(got).all()
    else:
        torch.testing.assert_close(got, want, rtol=1e-4, atol=1e-4)


# ---- sample(requires_grad=True) over DQLMlp --------------------------------------------------------------------------
class _Fp64Time(torch.nn.Module):
    def __init__(self, m):
        super().__init__()
        self.m = m

    def forward(self, t):
        return self.m(t).double()


def grad_agent(case, net, dtype=torch.float32, device="cpu", classifier=None):
    x_min, x_max = gs.bounds(case)
    mask = gs.fix_mask(case)
    kw = dict(predict_noise=case["predict_noise"], device=device, classifier=classifier,
              x_min=None if x_min is None else x_min.to(dtype), x_max=None if x_max is None else x_max.to(dtype),
              fix_mask=None if mask is None else mask.to(dtype))
    if case["agent"] == "discrete":
        return DiscreteDiffusionSDE(net, IdentityCondition(dropout=0.0), diffusion_steps=20, **kw)
    return ContinuousDiffusionSDE(net, IdentityCondition(dropout=0.0), **kw)


def grad_inputs(case, batch, seed=7):
    g = torch.Generator().manual_seed(seed)
    a, o = case["ctor"]["act_dim"], case["ctor"]["obs_dim"]
    return torch.randn(batch, a, generator=g), torch.randn(batch, o, generator=g), torch.randn(batch, a, generator=g)


def actor_grads(agent, prior, cond, weight, tape, case):
    """sample(requires_grad=True) -> backward of sum(x0 * weight) -> (x0, {parameter name or 'cond': gradient})"""
    model = agent.model
    model.zero_grad()
    cond = cond.clone().requires_grad_(True)
    kw = dict(condition_cg=None, w_cg=0.2) if case.get("guided") else {}
    with tape.active():
        x0, _ = agent.sample(prior, solver=case["solver"], n_samples=prior.shape[0], sample_steps=case["steps"],
                             use_ema=False, condition_cfg=cond, w_cfg=case["w_cfg"], requires_grad=True, temperature=0.8,
                             **kw)
    (x0 * weight).sum().backward()
    out = {n: p.grad.detach().double().clone() for n, p in model.named_parameters() if p.grad is not None}
    out["cond"] = cond.grad.detach().double().clone()
    return x0.detach().double(), out


def reference_grads(case, net, prior, cond, weight, draws):
    """fp64 autograd of the PyTorch reverse loop: same weights, same draws"""
    net64 = copy.deepcopy(net).double()
    net64.map_noise = _Fp64Time(copy.deepcopy(net.map_noise))   # the embedding computes in fp32 whatever the weights
    agent64 = grad_agent(case, net64, torch.float64)
    x0, grads = actor_grads(agent64, prior.double(), cond.double(), weight.double(), NoiseTape(draws), case)
    return x0, {k.replace("map_noise.m.", "map_noise."): v for k, v in grads.items()}


def check_grad_case(name, math, device, batch, monkeypatch, tol=gs.TOL):
    """the engine's x0 and gradients against fp64 autograd of the PyTorch loop, the loop's draws seeded -> ({gradient name:
    fraction of the bound}, the agent whose plan served the call)"""
    case = gs.GRADS[name]
    monkeypatch.setenv("CDS_MATH", math)
    monkeypatch.setenv("CDS_BACKEND", "cuda")
    net = load_synth(DQLMlp(**case["ctor"]), seed=2).to(device)
    agent = grad_agent(case, net, device=device)
    prior, cond, weight = (t.to(device) for t in grad_inputs(case, batch))
    calls, tape = runtime.STATS["engine_calls"], NoiseTape()
    torch.manual_seed(13)
    x0, got = actor_grads(agent, prior, cond, weight, tape, case)
    assert runtime.STATS["engine_calls"] == calls + 1, "the engine did not serve the call"
    monkeypatch.setenv("CDS_BACKEND", "torch")
    x0_ref, want = reference_grads(case, copy.deepcopy(net).cpu(), prior.cpu(), cond.cpu(), weight.cpu(), tape.draws)
    monkeypatch.setenv("CDS_BACKEND", "cuda")
    assert set(got) == set(want), (sorted(got), sorted(want))
    fracs = {"x0": gs.per_element_frac(x0, x0_ref, math, tol)[0]}
    for k in want:
        fracs[k] = gs.per_element_frac(got[k], want[k], math, tol)[0]
    return fracs, agent


@pytest.mark.parametrize("math", list(MATHS))
@pytest.mark.parametrize("name", GRAD_SERVED)
def test_grad_sampling_matches_fp64_autograd(name, math, monkeypatch):
    emulator.emulate(monkeypatch)
    fracs, _ = check_grad_case(name, math, "cpu", 6, monkeypatch)
    worst = max(fracs, key=fracs.get)
    assert fracs[worst] <= 1.0, (name, gs.GRADS[name], worst, fracs[worst])


@pytest.mark.parametrize("name", GRAD_DECLINED)
def test_declined_grad_request_takes_the_pytorch_loop(name, monkeypatch):
    emulator.emulate(monkeypatch)
    check_grad_decline(name, "cpu", 4, monkeypatch)


def check_grad_decline(name, device, batch, monkeypatch):
    """the declined request takes the PyTorch loop with exactly its reason, no engine call, and gives that loop's x0 and
    gradients bit for bit"""
    case = gs.GRADS[name]
    monkeypatch.setenv("CDS_MATH", case["math"] or "fp32")
    monkeypatch.setenv("CDS_BACKEND", "auto")
    net = load_synth(DQLMlp(**case["ctor"]), seed=2).to(device)
    clf = ToyClassifier((case["ctor"]["act_dim"],), device=device) if case.get("guided") else None
    agent = grad_agent(case, net, device=device, classifier=clf)
    prior, cond, weight = (t.to(device) for t in grad_inputs(case, batch))
    calls, falls, tape = runtime.STATS["engine_calls"], runtime.STATS["fallbacks"], NoiseTape()
    x0, got = actor_grads(agent, prior, cond, weight, tape, case)
    assert runtime.STATS["engine_calls"] == calls and runtime.STATS["fallbacks"] == falls + 1
    assert runtime.STATS["last_fallback_reason"] == case["want"]
    monkeypatch.setenv("CDS_BACKEND", "torch")
    x1, want = actor_grads(agent, prior, cond, weight, NoiseTape(tape.draws), case)
    assert torch.equal(x0, x1) and all(torch.equal(got[k], want[k]) for k in want)


# ---- every reason is reached ----------------------------------------------------------------------------------------
def _reason_prefixes(src):
    """the literal text of every reason string ``src`` returns (an f-string up to its first field)"""
    return {m.group(1) for m in re.finditer(r'return f?"([^"{]*)', src)}


def test_every_decline_reason_is_reached():
    """every ``return "..."`` reason of guidable's helpers and try_sample_grad's declines, and the guidance reasons of
    try_sample, is the labelled outcome of some case (whose reason the tests above check exactly)"""
    wants = {c["want"] for c in gs.CLASSIFIERS.values()}
    for fn in (lower._half_janner_reason, lower._qgpo_reason, lower._mlp_classifier_layers, lower._mlp_classifier_reason):
        prefixes = _reason_prefixes(inspect.getsource(fn))
        assert prefixes, fn
        missing = {p for p in prefixes if not any(w.startswith(p) for w in wants)}
        assert not missing, (fn.__name__, sorted(missing))
    grad_wants = {c["want"] for c in gs.GRADS.values()}
    src = inspect.getsource(runtime.try_sample_grad)
    decline = src[src.index("def decline"):src.index("screened =")]
    prefixes = _reason_prefixes(decline) - {"requires_grad=True: backbone "}          # backbones other than DQLMlp: tests/test_grad_sampling_cpu.py
    assert {p for p in prefixes if not any(w.startswith(p) for w in grad_wants)} == set()
    src = inspect.getsource(runtime.try_sample)
    cg = {m.group(1) for m in re.finditer(r'cg_reason = "([^"]*)"', src)} | \
        {m.group(1) for m in re.finditer(r'return "(classifier guidance[^"]*)"', src)}
    assert cg - {"no classifier"} == set(gs.REQUESTS.values())
    assert runtime._n_branches(8, 4, False) == 1          # "branches": the chain count the request below asks for
    with pytest.MonkeyPatch.context() as m:
        m.setenv("CDS_BRANCHES", "2")
        m.setenv("CDS_BRANCH_MIN_BATCH", "1")
        assert runtime._n_branches(8, 4, False) == 2


def test_the_table_reaches_the_new_axes():
    """the values the case table exists for"""
    graph = [c for c in gs.CLASSIFIERS.values() if c["want"] == "graph"]
    hj = [c for c in graph if c["family"] == "half_janner"]
    assert {c["ctor"]["kernel_size"] for c in hj} == {3, 5, 7}
    assert {c["x"][0] for c in hj} >= {1, 2, 4, 8, 32, 64, 256}
    assert {len(c["ctor"]["dim_mult"]) for c in hj} == {1, 2, 3, 4}
    assert {c["ctor"].get("out_dim", 1) for c in hj} == {1, 3} and {c["ctor"]["model_dim"] for c in hj} == {16, 32, 64}
    assert {c["ctor"].get("timestep_emb_type") for c in hj} - {None} == set(bs.EMB_TYPES)
    # L reaches 1 before the mid blocks: horizon <= 2^(stages - 1)
    assert any(c["x"][0] <= 2 ** (len(c["ctor"]["dim_mult"]) - 1) for c in hj)
    mlp = [c for c in graph if c["family"] == "mlp"]
    assert {len(c["ctor"]["hidden_dims"]) for c in mlp} == {1, 2, 3, 4}
    assert {w for c in mlp for w in c["ctor"]["hidden_dims"]} >= {1, 7, 33, 100, 256, 1024}
    assert {c["ctor"]["act"] for c in mlp} == {"ReLU", "SiLU", "Mish"} and {c["head"] for c in mlp} == {"mse", "cumrew"}
    assert {c["ctor"]["out_dim"] for c in mlp if c["head"] == "mse"} == {1, 7, 60}
    dql = [c for c in gs.GRADS.values() if c["want"] == "graph"]
    assert {c["bounds"] for c in dql} == {"none", "min", "max", "both"} and {c["mask"] for c in dql} == {"none", "cols"}
    assert {c["solver"] for c in dql} == {"ddpm", "ddim", "ode_dpmsolver_1", "sde_dpmsolver++_1"}
    assert {c["agent"] for c in dql} == {"discrete", "continuous"} and {c["predict_noise"] for c in dql} == {True, False}


def test_the_lowered_programs_reach_the_new_forms():
    """the operator forms the table exists for, read from the lowered programs themselves (the kernel each one selects,
    from libcds's host-side queries): conv data gradients at 5 and 7 taps, the two-phase Downsample gradient, the L = 1
    centre-tap gradient, DGRAD with ReLU, SiLU and Mish, GN and GN_BWD over groups of more than 1,000 elements, and WGRAD
    with its bias column in the DQLMlp backward"""
    import program_audit as pa
    forms = set()
    for name in LOWERED:
        case = gs.CLASSIFIERS[name]
        clf = gs.build_classifier(case)
        x, _ = gs.classifier_inputs(case, BATCH)
        B, H, D = x.shape if x.dim() == 3 else (x.shape[0], 1, x.shape[1])
        for math in MATHS.values():
            p = lower.Program(torch.device("cpu"), B, 2, math)
            lower.lower_classifier_grad(p, clf, lower.View(p.buf(*x.shape), H, D))
            for op in p.ops:
                f = pa.instantiation(op)
                if op.kind == cabi.OP_CONV:
                    c = op.u.conv
                    f += f" taps {c.taps} s{c.stride} ph{c.phases} L_in {c.L_in}"
                elif op.kind in (cabi.OP_GN, cabi.OP_GN_BWD):
                    g = op.u.gn if op.kind == cabi.OP_GN else op.u.gn_bwd
                    f += " group > 1000" if g.L * g.C // g.groups > 1000 else ""
                forms.add(f)
    convs = [f for f in forms if f.startswith("conv")]
    for taps in (5, 7):
        assert any(f" taps {taps} s1 ph1" in f for f in convs), (taps, sorted(convs))
    assert any(" taps 3 s1 ph2" in f for f in convs), sorted(convs)
    assert any(" taps 1 " in f and f.endswith(" L_in 1") for f in convs), sorted(convs)
    for act in ("relu", "silu", "mish"):
        assert any(f.startswith(f"dgrad {act}") for f in forms), (act, sorted(forms))
    for kind in ("gn ", "gn_bwd "):
        assert any(f.startswith(kind) and f.endswith("group > 1000") for f in forms), sorted(forms)
    p, bp = lower.Program(torch.device("cpu"), BATCH, 3), lower.Program(torch.device("cpu"), BATCH, 3)
    lower.DQLGrad(p, bp, load_synth(DQLMlp(obs_dim=4, act_dim=3)), lower.View(p.buf(BATCH, 3), 1, 3))
    assert "wgrad mish +bias" in {pa.instantiation(op) for op in bp.ops}
