"""``sample(requires_grad=True)`` with ContinuousConsistencyModel and Discrete / ContinuousRectifiedFlow over DQLMlp, lowered to
the forward + backward operator programs and executed by the numpy interpreter (tests/emulator.py, taught CDS_OP_UPDATE_BWD's
kind CM and CDS_OP_PREP's backward mode by tests/few_step_grad_ref.py): x0 and every parameter and condition gradient must
match fp64 autograd of the PyTorch loop under the same noise tape.  Also: the CM clip rule against torch.clip, the decline
reasons, the unchanged requires_grad=False programs, the programs' shapes and plan keys, re-packing after an optimiser step
and a stale backward."""
import copy

import numpy as np
import pytest
import torch

import emulator
import few_step_grad_ref
from cleandiffuser_b200.diffusion import ContinuousConsistencyModel, ContinuousRectifiedFlow, DiscreteRectifiedFlow
from cleandiffuser_b200.diffusion import solvers as S
from cleandiffuser_b200.engine import cabi, runtime
from cleandiffuser_b200.nn_condition import IdentityCondition
from cleandiffuser_b200.nn_diffusion import DQLMlp, IDQLMlp
from cleandiffuser_b200.testing import NoiseTape, load_synth


@pytest.fixture(autouse=True)
def _emulate(monkeypatch):
    emulator.emulate(monkeypatch)      # every operand is bounds-checked against its owner
    few_step_grad_ref.register(monkeypatch)
    monkeypatch.setenv("CDS_BACKEND", "cuda")       # any fallback to the PyTorch loop is a failure here
    monkeypatch.setenv("CDS_MATH", "fp32")


NET = dict(obs_dim=4, act_dim=3, emb_dim=16)
# per-element bounds; the last column has x_min > x_max (torch.clip then returns x_max and passes no gradient)
BOUNDS = {"none": (None, None), "min": ([-0.2, -0.1, 0.0], None), "max": (None, [0.2, 0.1, 0.05]),
          "both": ([-0.2, -0.1, 0.1], [0.25, 0.15, -0.1])}


def make_agent(family, net, *, bounds="none", mask=False, dtype=torch.float32):
    a = NET["act_dim"]
    lo, hi = BOUNDS[bounds]
    kw = dict(device="cpu")
    if lo is not None:
        kw["x_min"] = torch.tensor([lo], dtype=dtype)
    if hi is not None:
        kw["x_max"] = torch.tensor([hi], dtype=dtype)
    if mask:
        m = torch.zeros(a, dtype=dtype)
        m[0] = 1.
        kw["fix_mask"] = m
    if family == "cm":
        return ContinuousConsistencyModel(net, IdentityCondition(dropout=0.0), **kw)
    if family == "rf_discrete":
        return DiscreteRectifiedFlow(net, IdentityCondition(dropout=0.0), diffusion_steps=20, **kw)
    return ContinuousRectifiedFlow(net, IdentityCondition(dropout=0.0), **kw)


class _Fp64(torch.nn.Module):
    def __init__(self, m):
        super().__init__()
        self.m = m

    def forward(self, t):
        return self.m(t).double()


def actor_grads(agent, prior, cond, weight, tape, **kw):
    """sample(requires_grad=True) -> backward of sum(x0 * weight) -> (x0, {name: grad}) (parameters of the trained model, and
    'cond' when the call reads the condition)"""
    agent.model.zero_grad()
    cond = None if cond is None else cond.clone().requires_grad_(True)
    with tape.active():
        x0, _ = agent.sample(prior, n_samples=prior.shape[0], use_ema=False, condition_cfg=cond, requires_grad=True, **kw)
    (x0 * weight).sum().backward()
    out = {n: p.grad.detach().double().clone() for n, p in agent.model.named_parameters() if p.grad is not None}
    if cond is not None and cond.grad is not None:
        out["cond"] = cond.grad.detach().double().clone()
    return x0.detach().double(), out


def check_grads(monkeypatch, family, *, bounds="none", mask=False, cond=True, batch=16, seed=2, **kw):
    net = load_synth(DQLMlp(**NET), seed=seed)
    agent = make_agent(family, net, bounds=bounds, mask=mask)
    g = torch.Generator().manual_seed(7)
    a = NET["act_dim"]
    prior = torch.randn(batch, a, generator=g)
    c = torch.randn(batch, NET["obs_dim"], generator=g) if cond else None
    weight = torch.randn(batch, a, generator=g)
    before = runtime.STATS["engine_calls"]
    tape = NoiseTape()
    x0, got = actor_grads(agent, prior, c, weight, tape, **kw)
    assert runtime.STATS["engine_calls"] == before + 1, "the engine did not serve the call"
    plan = next(iter(agent._engine_plans.values()))
    assert isinstance(plan, runtime.GradSamplerPlan)

    # fp64 autograd of the PyTorch loop, same weights, same draws
    monkeypatch.setenv("CDS_BACKEND", "torch")
    net64 = copy.deepcopy(net).double()
    net64.map_noise = _Fp64(net64.map_noise)         # the timestep embedding computes in fp32 whatever the weights
    agent64 = make_agent(family, net64, bounds=bounds, mask=mask, dtype=torch.float64)
    x0_ref, want = actor_grads(agent64, prior.double(), None if c is None else c.double(), weight.double(),
                               NoiseTape(tape.draws), **kw)
    monkeypatch.setenv("CDS_BACKEND", "cuda")
    assert (x0 - x0_ref).abs().max() < 1e-4, (x0 - x0_ref).abs().max()
    assert set(got) == set(want), (sorted(got), sorted(want))
    for name in want:
        err = (got[name] - want[name]).abs().max().item()
        scale = want[name].abs().max().item()
        assert err <= 1e-4 * scale + 1e-6, (name, err, scale)
    return x0_ref, want


# ---------------------------------------------------------------------------------------------------- consistency model
@pytest.mark.parametrize("steps", [1, 2, 3])
@pytest.mark.parametrize("bounds", ["none", "min", "max", "both"])
def test_cm_grads(steps, bounds, monkeypatch):
    check_grads(monkeypatch, "cm", bounds=bounds, sample_steps=steps)


@pytest.mark.parametrize("cond", [True, False])
def test_cm_grads_mask_dx(cond, monkeypatch):
    """fix_mask, two Diffusion-X repeats of the last level, clipping on both sides, with and without a condition"""
    check_grads(monkeypatch, "cm", bounds="both", mask=True, cond=cond, sample_steps=2, diffusion_x_sampling_steps=2)


def test_cm_clip_is_exercised(monkeypatch):
    """the bounds of BOUNDS clip some elements of the consistency model's f and leave others inside: without the clip the
    same call gives another x0, and some gradient entries are cut"""
    x_clip, g_clip = check_grads(monkeypatch, "cm", bounds="both", sample_steps=2)
    x_free, g_free = check_grads(monkeypatch, "cm", bounds="none", sample_steps=2)
    lo, hi = (torch.tensor(b, dtype=torch.float64) for b in BOUNDS["both"])
    inside = (x_clip > lo) & (x_clip < hi)
    assert 0 < int(inside.sum()) < inside.numel()
    assert (g_clip["cond"] - g_free["cond"]).abs().max() > 1e-3


# ------------------------------------------------------------------------------------------------------- rectified flow
@pytest.mark.parametrize("family", ["rf_discrete", "rf_continuous"])
@pytest.mark.parametrize("w_cfg", [0.0, 1.0])
def test_rf_grads(family, w_cfg, monkeypatch):
    """w_cfg = 0 evaluates the unconditional network (the condition gets no gradient, on both paths)"""
    check_grads(monkeypatch, family, bounds="both", w_cfg=w_cfg, sample_steps=5)


@pytest.mark.parametrize("family", ["rf_discrete", "rf_continuous"])
def test_rf_grads_mask_dx_final_clip(family, monkeypatch):
    """fix_mask, Diffusion-X repeats of the last step, and the final clip (a PyTorch op after the loop)"""
    check_grads(monkeypatch, family, bounds="both", mask=True, w_cfg=1.0, sample_steps=3, diffusion_x_sampling_steps=2)


# ------------------------------------------------------------------------------------------------- the CM clip rule
def test_cm_clip_gradient_rule_matches_torch():
    """cm_update_bwd = autograd of clip(k0 x + k1 pred, x_min, x_max) * (1 - mask) for tensor bounds, ties included (an f equal
    to a bound passes its gradient) and x_min > x_max in one column (none passes)"""
    g = torch.Generator().manual_seed(3)
    k0, k1 = 0.25, 0.5
    for which in ("both", "min", "max"):
        x_min = None if which == "max" else torch.tensor([-0.5, -0.3, 0.4, -0.6], dtype=torch.float64)
        x_max = None if which == "min" else torch.tensor([0.5, 0.3, -0.2, 0.6], dtype=torch.float64)
        x = torch.randn(64, 4, generator=g, dtype=torch.float64)
        pred = torch.randn(64, 4, generator=g, dtype=torch.float64) * 2
        x[:16] = 0.0                                    # f = k1 pred exactly: ties with a bound
        if x_min is not None:
            pred[:8] = x_min / k1
        if x_max is not None:
            pred[8:16] = x_max / k1
        mask = torch.tensor([0.0, 1.0, 0.0, 0.0], dtype=torch.float64)
        xr, pr = x.clone().requires_grad_(True), pred.clone().requires_grad_(True)
        out = (k0 * xr + k1 * pr).clip(x_min, x_max) * (1 - mask)
        w = torch.randn(64, 4, generator=g, dtype=torch.float64)
        (out * w).sum().backward()
        gp, dx = few_step_grad_ref.cm_update_bwd(w.numpy(), x.numpy(), pred.numpy(), k0=k0, k1=k1, mask=mask.numpy(),
                                                 x_min=None if x_min is None else x_min.numpy(),
                                                 x_max=None if x_max is None else x_max.numpy())
        np.testing.assert_allclose(gp, pr.grad.numpy(), rtol=1e-12, atol=1e-12, err_msg=which)
        np.testing.assert_allclose(dx, xr.grad.numpy(), rtol=1e-12, atol=1e-12, err_msg=which)
        ties = slice(0, 8) if x_min is not None else slice(8, 16)
        assert (np.abs(gp[ties][:, [0, 3]]) > 0).all(), "a tie with a bound must pass its gradient"


# ----------------------------------------------------------------------------------------------------------- declines
def _fallback_reason(monkeypatch, agent, prior, **kw):
    monkeypatch.setenv("CDS_BACKEND", "auto")          # fall back quietly: the PyTorch loop serves the call
    before = runtime.STATS["engine_calls"]
    x0, _ = agent.sample(prior, n_samples=prior.shape[0], use_ema=False, requires_grad=True, **kw)
    assert runtime.STATS["engine_calls"] == before and x0.requires_grad
    monkeypatch.setenv("CDS_BACKEND", "cuda")
    with pytest.raises(RuntimeError, match="CDS_BACKEND=cuda"):
        agent.sample(prior, n_samples=prior.shape[0], use_ema=False, requires_grad=True, **kw)
    return runtime.STATS["last_fallback_reason"]


def test_decline_reasons(monkeypatch):
    prior, cond = torch.zeros(4, 3), torch.randn(4, 4)
    idql = load_synth(IDQLMlp(obs_dim=4, act_dim=3, emb_dim=16, hidden_dim=32, n_blocks=1))
    for family in ("cm", "rf_discrete", "rf_continuous"):
        assert _fallback_reason(monkeypatch, make_agent(family, idql), prior, sample_steps=2, condition_cfg=cond) == \
            "requires_grad=True: backbone IDQLMlp has no differentiable engine program (DQLMlp only)"
    net = load_synth(DQLMlp(**NET), seed=2)
    for family in ("rf_discrete", "rf_continuous"):
        assert _fallback_reason(monkeypatch, make_agent(family, net), prior, sample_steps=2, condition_cfg=cond, w_cfg=1.5) == \
            "requires_grad=True with two-branch classifier-free guidance"
    monkeypatch.setenv("CDS_MATH", "bf16")
    for family in ("cm", "rf_continuous"):
        assert _fallback_reason(monkeypatch, make_agent(family, net), prior, sample_steps=2, condition_cfg=cond) == \
            "requires_grad=True with CDS_MATH=bf16 (fp32 and tf32 only)"


def test_update_kind_without_backward_is_declined(monkeypatch):
    """a coefficient table with a kind CDS_OP_UPDATE_BWD does not differentiate (EDM, X2M) keeps the PyTorch loop: the program
    is never built, so no row can take another kind's formula"""
    agent = make_agent("rf_continuous", load_synth(DQLMlp(**NET), seed=2))
    rows = torch.zeros((2, S.ROW))
    rows[:, S.R_KIND] = torch.tensor([float(S.UPD_EPS), float(S.UPD_EDM)])
    xt = torch.randn(4, 3)
    kw = dict(model=agent.model, xt=xt, prior=xt, solver="custom", sample_steps=2, order=[2, 1], step_values=None, alphas=None,
              sigmas=None, hs=None, stds=None, cond_emb=None, w_cfg=0.0, n_samples=4, table=(rows, 0, torch.zeros(2)),
              clip_in_loop=False, predict_noise=True)
    monkeypatch.setenv("CDS_BACKEND", "auto")
    assert runtime.try_sample_grad(agent, **kw) is None
    assert runtime.STATS["last_fallback_reason"] == "requires_grad=True: update kind [6] has no backward operator"
    assert not agent._engine_plans
    monkeypatch.setenv("CDS_BACKEND", "cuda")
    with pytest.raises(RuntimeError, match="update kind"):
        runtime.try_sample_grad(agent, **kw)


def test_preserve_history_takes_the_pytorch_loop():
    net = load_synth(DQLMlp(**NET), seed=2)
    before = runtime.STATS["engine_calls"]
    x0, log = make_agent("cm", net).sample(torch.zeros(4, 3), n_samples=4, sample_steps=2, use_ema=False,
                                           condition_cfg=torch.randn(4, 4), requires_grad=True, preserve_history=True)
    assert runtime.STATS["engine_calls"] == before and x0.requires_grad and log["sample_history"] is not None


# ------------------------------------------------------------------------------------------------------ program shapes
def test_no_grad_programs_unchanged():
    """requires_grad=False keeps its programs: the consistency model's PREP, four fused Linear(+Mish) operators and the update
    with its final clip; rectified flow's four operators and the unclipped EPS update"""
    net = load_synth(DQLMlp(**NET), seed=2)
    for family, want in (("cm", [cabi.OP_PREP] + [cabi.OP_CONV] * 4 + [cabi.OP_UPDATE]),
                         ("rf_continuous", [cabi.OP_CONV] * 4 + [cabi.OP_UPDATE])):
        agent = make_agent(family, net, bounds="both", mask=True)
        with torch.no_grad():
            agent.sample(torch.zeros(4, 3), n_samples=4, sample_steps=3, use_ema=False, condition_cfg=torch.randn(4, 4),
                         w_cfg=1.0)
        (plan,) = agent._engine_plans.values()
        assert type(plan) is runtime.SamplerPlan
        ops = plan.program.ops
        assert [op.kind for op in ops] == want, family
        convs = [op.u.conv for op in ops if op.kind == cabi.OP_CONV]
        assert [c.act for c in convs] == [cabi.ACT_MISH] * 3 + [cabi.ACT_NONE]
        assert convs[0].in_ == (plan.xin.data_ptr() if family == "cm" else plan.x.data_ptr())
        u = ops[-1].u.update
        assert (u.final_clip, bool(u.x_min), bool(u.x_max)) == ((1, True, True) if family == "cm" else (0, False, False))
        assert not any(op.kind == cabi.OP_STASH for op in ops)


def test_grad_program_shapes_and_plan_key():
    net = load_synth(DQLMlp(**NET), seed=2)
    agent = make_agent("cm", net, bounds="both")
    x0, _ = agent.sample(torch.zeros(4, 3), n_samples=4, sample_steps=3, use_ema=False, condition_cfg=torch.randn(4, 4),
                         requires_grad=True)
    (plan,) = agent._engine_plans.values()
    S_, C_ = cabi.OP_STASH, cabi.OP_CONV
    assert [op.kind for op in plan.program.ops] == [cabi.OP_PREP, S_, S_, C_, S_, C_, S_, C_, S_, C_, S_, cabi.OP_UPDATE]
    assert [op.kind for op in plan.back.ops] == [cabi.OP_UPDATE_BWD] + [cabi.OP_WGRAD, cabi.OP_DGRAD] * 4 + [cabi.OP_PREP]
    assert plan.program.ops[-1].u.update.final_clip == 1
    first_conv = plan.program.ops[3].u.conv
    assert first_conv.in_ == plan.xin.data_ptr()
    last_dgrad = plan.back.ops[-2].u.dgrad
    assert last_dgrad.out == plan.grad.gxin.data_ptr() and last_dgrad.accumulate == 0
    prep_bwd = plan.back.ops[-1].u.prep
    assert (prep_bwd.x, prep_bwd.gxin, prep_bwd.coef_iter_stride) == (plan.grad.gx.data_ptr(), plan.grad.gxin.data_ptr(),
                                                                      -cabi.ROW_FLOATS)
    # an SDE-shaped request of the same shapes on the same agent (EPS rows, same iterations and draws) gets its own plan
    tab = agent._engine_tables[next(iter(agent._engine_tables))]
    rows = tab.rows.clone()
    rows[:, S.R_KIND] = float(S.UPD_EPS)
    rows[:, S.R_ALPHA] = rows[:, S.R_SIGMA] = 1.0
    xt = torch.randn(4, 3)
    with NoiseTape().active():
        runtime.try_sample_grad(agent, model=agent.model, xt=xt, prior=xt, solver="consistency", sample_steps=3, order=[2, 1],
                                step_values=None, alphas=None, sigmas=None, hs=None, stds=None, cond_emb=torch.randn(4, 4),
                                w_cfg=1.0, n_samples=4, table=(rows, tab.n_slots, tab.t.cpu()), predict_noise=True)
    assert len(agent._engine_plans) == 2
    sde = [p for p in agent._engine_plans.values() if p is not plan][0]
    assert sde.program.ops[0].kind == cabi.OP_STASH and sde.back.ops[-1].kind == cabi.OP_DGRAD


@pytest.mark.parametrize("family", ["cm", "rf_discrete"])
def test_weights_version_follows_optimizer_step(family, monkeypatch):
    """An optimiser step changes the weights in place; the next call must re-pack them (a stale copy would be silent)."""
    net = load_synth(DQLMlp(**NET), seed=2)
    agent = make_agent(family, net, bounds="both")
    opt = torch.optim.Adam(agent.model.parameters(), lr=1e-2)
    prior, cond = torch.zeros(8, 3), torch.randn(8, 4)
    kw = dict(n_samples=8, sample_steps=2, use_ema=False, w_cfg=1.0, condition_cfg=cond, requires_grad=True)
    v0 = runtime._weights_version(net)
    tape = NoiseTape()
    with tape.active():
        x0, _ = agent.sample(prior, **kw)
    (x0 * torch.randn(8, 3)).sum().backward()
    opt.step()
    assert runtime._weights_version(net) != v0
    with NoiseTape(tape.draws).active():
        x1, _ = agent.sample(prior, **kw)
    monkeypatch.setenv("CDS_BACKEND", "torch")
    with NoiseTape(tape.draws).active():
        x1_ref, _ = agent.sample(prior, **kw)
    assert (x1 - x1_ref).abs().max() < 1e-5 and (x1 - x0).abs().max() > 1e-3


@pytest.mark.parametrize("family", ["cm", "rf_continuous"])
def test_second_sample_before_backward_is_an_error(family):
    agent = make_agent(family, load_synth(DQLMlp(**NET), seed=2))
    kw = dict(n_samples=4, sample_steps=2, use_ema=False, w_cfg=1.0, condition_cfg=torch.randn(4, 4), requires_grad=True)
    x0, _ = agent.sample(torch.zeros(4, 3), **kw)
    x1, _ = agent.sample(torch.zeros(4, 3), **kw)
    x1.sum().backward()                                       # the latest call's backward is served
    with pytest.raises(RuntimeError, match="overwritten"):
        x0.sum().backward()
