"""``sample(requires_grad=True)`` over DQLMlp, lowered to the forward + backward operator programs and executed by the numpy
interpreter (tests/emulator.py, extended by tests/grad_ref.py) on CPU tensors: the parameter and condition gradients must match fp64
autograd of the PyTorch reverse loop under the same noise tape.  Also: the fallbacks, the unchanged requires_grad=False
program, and the gradient rule of clip_prediction against torch.clip's."""
import copy

import numpy as np
import pytest
import torch

import emulator
import grad_ref
from cleandiffuser_b200.diffusion import ContinuousDiffusionSDE, DiscreteDiffusionSDE
from cleandiffuser_b200.engine import cabi, runtime
from cleandiffuser_b200.nn_condition import IdentityCondition
from cleandiffuser_b200.nn_diffusion import DQLMlp, IDQLMlp
from cleandiffuser_b200.testing import NoiseTape, ToyClassifier, load_synth


@pytest.fixture(autouse=True)
def _emulate(monkeypatch):
    monkeypatch.setattr(runtime, "_device_ok", lambda device: True)
    owners = emulator.record_owners(monkeypatch)      # every operand is bounds-checked against its owner
    monkeypatch.setattr(runtime, "_make_handle", lambda device, ops, n: grad_ref.Handle(ops, n, owners()))
    monkeypatch.setenv("CDS_BACKEND", "cuda")       # any fallback to the PyTorch loop is a failure here
    monkeypatch.setenv("CDS_MATH", "fp32")


NETS = {"dql_tiny": dict(obs_dim=4, act_dim=3, emb_dim=16),       # tests/golden/cases.py SAMPLER_NETS["dql_tiny"]
        "dql_hopper": dict(obs_dim=11, act_dim=3, emb_dim=16)}    # Diffusion-QL's D4RL hopper shapes (hidden 256)


def make_agent(net, kind, *, predict_noise, clip, mask, dtype=torch.float32):
    a = net.mid_layer[0].in_features - net.obs_dim - net.time_mlp[2].out_features
    kw = dict(predict_noise=predict_noise, device="cpu")
    if clip:
        kw.update(x_max=torch.full((1, a), 1.0, dtype=dtype), x_min=torch.full((1, a), -1.0, dtype=dtype))
    if mask:
        m = torch.zeros(a, dtype=dtype)
        m[0] = 1.
        kw["fix_mask"] = m
    if kind == "discrete":
        return DiscreteDiffusionSDE(net, IdentityCondition(dropout=0.0), diffusion_steps=20, **kw)
    return ContinuousDiffusionSDE(net, IdentityCondition(dropout=0.0), **kw)


class _Fp64(torch.nn.Module):
    def __init__(self, m):
        super().__init__()
        self.m = m

    def forward(self, t):
        return self.m(t).double()


def actor_grads(agent, prior, cond, weight, tape, **kw):
    """sample(requires_grad=True) -> backward of sum(x0 * weight) -> {name: grad} (parameters of the trained model + 'cond')"""
    model = agent.model
    model.zero_grad()
    cond = cond.clone().requires_grad_(True)
    with tape.active():
        x0, _ = agent.sample(prior, n_samples=prior.shape[0], use_ema=False, condition_cfg=cond, requires_grad=True, **kw)
    (x0 * weight).sum().backward()
    out = {n: p.grad.detach().double().clone() for n, p in model.named_parameters() if p.grad is not None}
    out["cond"] = cond.grad.detach().double().clone()
    return x0.detach().double(), out


def check_grads(net_kw, kind, solver, predict_noise, clip, mask, dx, batch=16, steps=4, monkeypatch=None):
    net = load_synth(DQLMlp(**net_kw), seed=2)
    agent = make_agent(net, kind, predict_noise=predict_noise, clip=clip, mask=mask)
    g = torch.Generator().manual_seed(7)
    a = net_kw["act_dim"]
    prior = torch.randn(batch, a, generator=g)
    cond = torch.randn(batch, net_kw["obs_dim"], generator=g)
    weight = torch.randn(batch, a, generator=g)
    kw = dict(solver=solver, sample_steps=steps, w_cfg=1.0, diffusion_x_sampling_steps=dx,
              temperature=0.8)
    before = runtime.STATS["engine_calls"]
    tape = NoiseTape()
    x0, got = actor_grads(agent, prior, cond, weight, tape, **kw)
    assert runtime.STATS["engine_calls"] == before + 1, "the engine did not serve the call"

    # fp64 autograd of the PyTorch loop, same weights, same draws
    monkeypatch.setenv("CDS_BACKEND", "torch")
    net64 = copy.deepcopy(net).double()
    net64.map_noise = _Fp64(net64.map_noise)         # the timestep embedding computes in fp32 whatever the weights
    agent64 = make_agent(net64, kind, predict_noise=predict_noise, clip=clip, mask=mask, dtype=torch.float64)
    x0_ref, want = actor_grads(agent64, prior.double(), cond.double(), weight.double(), NoiseTape(tape.draws), **kw)
    monkeypatch.setenv("CDS_BACKEND", "cuda")
    assert (x0 - x0_ref).abs().max() < 1e-4, (x0 - x0_ref).abs().max()
    assert set(got) == set(want), (sorted(got), sorted(want))
    for name in want:
        err = (got[name] - want[name]).abs().max().item()
        scale = want[name].abs().max().item()
        assert err <= 1e-4 * scale + 1e-6, (name, err, scale)


SOLVERS = ["ddpm", "ddim", "ode_dpmsolver_1", "sde_dpmsolver++_1"]


@pytest.mark.parametrize("solver", SOLVERS)
@pytest.mark.parametrize("predict_noise", [True, False])
@pytest.mark.parametrize("clip", [True, False])
def test_grads_discrete(solver, predict_noise, clip, monkeypatch):
    check_grads(NETS["dql_tiny"], "discrete", solver, predict_noise, clip, mask=False, dx=0, monkeypatch=monkeypatch)


@pytest.mark.parametrize("solver", SOLVERS)
@pytest.mark.parametrize("predict_noise", [True, False])
def test_grads_continuous_mask_dx(solver, predict_noise, monkeypatch):
    """continuous time, fix_mask, Diffusion-X repeats of the last step, clipping on"""
    check_grads(NETS["dql_tiny"], "continuous", solver, predict_noise, True, mask=True, dx=2, monkeypatch=monkeypatch)


@pytest.mark.parametrize("solver", ["ddpm", "sde_dpmsolver++_1"])
def test_grads_dql_shaped(solver, monkeypatch):
    """Diffusion-QL's own call shape: DDPM, 5 steps, predict_noise, clip to [-1, 1], w_cfg = 1"""
    check_grads(NETS["dql_hopper"], "discrete", solver, True, True, mask=False, dx=0, batch=32, steps=5,
                monkeypatch=monkeypatch)


def test_clip_gradient_rule_matches_torch():
    """update_bwd's clip_prediction gradient = torch.clip's for tensor bounds, ties included (an element equal to a bound
    is not clipped: its gradient goes to the prediction; a clipped one's to the bound and, for eps-prediction, to x_t / sigma)"""
    g = torch.Generator().manual_seed(3)
    for predict_noise in (True, False):
        for which in ("both", "min", "max"):
            x = torch.randn(64, 4, generator=g, dtype=torch.float64)
            alpha, sigma = 0.8, 0.6
            x_min = None if which == "max" else torch.full((4,), -0.5, dtype=torch.float64)
            x_max = None if which == "min" else torch.full((4,), 0.5, dtype=torch.float64)
            if predict_noise:
                lo = None if x_max is None else (x - alpha * x_max) / sigma
                hi = None if x_min is None else (x - alpha * x_min) / sigma
            else:
                lo, hi = x_min, x_max
            pred = torch.randn(64, 4, generator=g, dtype=torch.float64) * 2
            full = lambda b: torch.broadcast_to(b, (64, 4))                # noqa: E731
            pred[:8] = full(lo if lo is not None else hi)[:8]              # ties with a bound
            pred[8:16] = full(hi if hi is not None else lo)[8:16]
            xr, pr = x.clone().requires_grad_(True), pred.clone().requires_grad_(True)
            if predict_noise:
                lo_t = None if x_max is None else (xr - alpha * x_max) / sigma
                hi_t = None if x_min is None else (xr - alpha * x_min) / sigma
            else:
                lo_t, hi_t = x_min, x_max
            pc = pr.clip(lo_t, hi_t)
            out = 0.9 * xr - 0.3 * pc                                        # CDS_UPD_EPS / X shaped: k0 x - k1 target
            if not predict_noise:
                out = 0.9 * xr - 0.3 * ((xr - alpha * pc) / sigma)
            w = torch.randn(64, 4, generator=g, dtype=torch.float64)
            (out * w).sum().backward()
            gp, dx = grad_ref.update_bwd(w.numpy(), x.numpy(), pred.numpy(), alpha=alpha, sigma=sigma, k0=0.9, k1=0.3, kind=2,
                                         predict_noise=predict_noise,
                                         x_min=None if x_min is None else x_min.numpy(),
                                         x_max=None if x_max is None else x_max.numpy())
            np.testing.assert_allclose(gp, pr.grad.numpy(), rtol=1e-12, atol=1e-12, err_msg=f"{predict_noise} {which}")
            np.testing.assert_allclose(dx, xr.grad.numpy(), rtol=1e-12, atol=1e-12, err_msg=f"{predict_noise} {which}")


# ------------------------------------------------------------------------------------------------------------- fallbacks
def _fallback_reason(monkeypatch, agent, prior, **kw):
    monkeypatch.setenv("CDS_BACKEND", "auto")          # fall back quietly: the PyTorch loop serves the call
    before = runtime.STATS["engine_calls"]
    x0, _ = agent.sample(prior, n_samples=prior.shape[0], use_ema=False, requires_grad=True, **kw)
    assert runtime.STATS["engine_calls"] == before and x0.requires_grad
    return runtime.STATS["last_fallback_reason"]


def test_fallbacks(monkeypatch):
    net = load_synth(DQLMlp(obs_dim=4, act_dim=3, emb_dim=16), seed=2)
    agent = make_agent(net, "discrete", predict_noise=True, clip=True, mask=False)
    prior, cond = torch.zeros(4, 3), torch.randn(4, 4)
    kw = dict(sample_steps=3, condition_cfg=cond)
    assert "history" in _fallback_reason(monkeypatch, agent, prior, solver="ode_dpmsolver++_2M", w_cfg=1.0, **kw)
    assert "two-branch" in _fallback_reason(monkeypatch, agent, prior, solver="ddpm", w_cfg=1.5, **kw)
    monkeypatch.setenv("CDS_MATH", "bf16")
    assert "bf16" in _fallback_reason(monkeypatch, agent, prior, solver="ddpm", w_cfg=1.0, **kw)
    monkeypatch.setenv("CDS_MATH", "fp32")
    guided = DiscreteDiffusionSDE(net, IdentityCondition(dropout=0.0), classifier=ToyClassifier((3,)), diffusion_steps=20,
                                  device="cpu")
    assert "classifier guidance" in _fallback_reason(monkeypatch, guided, prior, solver="ddpm", w_cfg=1.0, w_cg=0.5,
                                                     condition_cg=None, **kw)
    idql = DiscreteDiffusionSDE(load_synth(IDQLMlp(obs_dim=4, act_dim=3, emb_dim=16, hidden_dim=32, n_blocks=1)),
                                IdentityCondition(dropout=0.0), diffusion_steps=20, device="cpu")
    assert "IDQLMlp" in _fallback_reason(monkeypatch, idql, prior, solver="ddpm", w_cfg=1.0, **kw)
    from cleandiffuser_b200.diffusion import ContinuousEDM
    edm = ContinuousEDM(net, IdentityCondition(dropout=0.0), device="cpu")
    assert "ContinuousEDM" in _fallback_reason(monkeypatch, edm, prior, solver="euler", w_cfg=1.0, **kw)


def test_fallback_raises_under_cuda_backend():
    net = load_synth(DQLMlp(obs_dim=4, act_dim=3, emb_dim=16), seed=2)
    agent = make_agent(net, "discrete", predict_noise=True, clip=False, mask=False)
    with pytest.raises(RuntimeError, match="history"):
        agent.sample(torch.zeros(4, 3), solver="sde_dpmsolver++_2M", n_samples=4, sample_steps=3, use_ema=False,
                     condition_cfg=torch.randn(4, 4), w_cfg=1.0, requires_grad=True)


# ------------------------------------------------------------------------------------------------------ program shapes
def test_no_grad_program_unchanged():
    """requires_grad=False over DQLMlp keeps its program: four fused Linear(+Mish) operators and the update, no stash"""
    net = load_synth(DQLMlp(obs_dim=4, act_dim=3, emb_dim=16), seed=2)
    agent = make_agent(net, "discrete", predict_noise=True, clip=True, mask=False)
    with torch.no_grad():
        agent.sample(torch.zeros(4, 3), solver="ddpm", n_samples=4, sample_steps=3, use_ema=False,
                     condition_cfg=torch.randn(4, 4), w_cfg=1.0)
    (plan,) = agent._engine_plans.values()
    ops = plan.program.ops
    assert [op.kind for op in ops] == [cabi.OP_CONV] * 4 + [cabi.OP_UPDATE]
    assert [op.u.conv.act for op in ops[:4]] == [cabi.ACT_MISH] * 3 + [cabi.ACT_NONE]


def test_grad_program_shapes_and_plan_key():
    net = load_synth(DQLMlp(obs_dim=4, act_dim=3, emb_dim=16), seed=2)
    agent = make_agent(net, "discrete", predict_noise=True, clip=True, mask=False)
    kw = dict(solver="ddpm", n_samples=4, sample_steps=3, use_ema=False, w_cfg=1.0)
    with torch.no_grad():
        agent.sample(torch.zeros(4, 3), condition_cfg=torch.randn(4, 4), **kw)
    x0, _ = agent.sample(torch.zeros(4, 3), condition_cfg=torch.randn(4, 4), requires_grad=True, **kw)
    assert len(agent._engine_plans) == 2                      # the grad flag is part of the plan key
    plan = [p for p in agent._engine_plans.values() if isinstance(p, runtime.GradSamplerPlan)][0]
    fwd = [op.kind for op in plan.program.ops]
    bwd = [op.kind for op in plan.back.ops]
    S_, C_ = cabi.OP_STASH, cabi.OP_CONV
    assert fwd == [S_, C_, S_, C_, S_, C_, S_, C_, S_, cabi.OP_UPDATE]
    assert bwd == [cabi.OP_UPDATE_BWD] + [cabi.OP_WGRAD, cabi.OP_DGRAD] * 4


def test_weights_version_follows_optimizer_step(monkeypatch):
    """An optimiser step changes the weights in place; the next call must re-pack them (a stale copy would be silent)."""
    net = load_synth(DQLMlp(obs_dim=4, act_dim=3, emb_dim=16), seed=2)
    agent = make_agent(net, "discrete", predict_noise=True, clip=True, mask=False)
    opt = torch.optim.Adam(agent.model.parameters(), lr=1e-2)
    prior, cond = torch.zeros(8, 3), torch.randn(8, 4)
    kw = dict(solver="ddpm", n_samples=8, sample_steps=3, use_ema=False, w_cfg=1.0, condition_cfg=cond, requires_grad=True)
    v0 = runtime._weights_version(net)
    tape = NoiseTape()
    with tape.active():
        x0, _ = agent.sample(prior, **kw)
    x0.square().sum().backward()
    opt.step()
    assert runtime._weights_version(net) != v0
    with NoiseTape(tape.draws).active():
        x1, _ = agent.sample(prior, **kw)
    monkeypatch.setenv("CDS_BACKEND", "torch")
    with NoiseTape(tape.draws).active():
        x1_ref, _ = agent.sample(prior, **kw)
    assert (x1 - x1_ref).abs().max() < 1e-5 and (x1 - x0).abs().max() > 1e-3


def test_second_sample_before_backward_is_an_error():
    net = load_synth(DQLMlp(obs_dim=4, act_dim=3, emb_dim=16), seed=2)
    agent = make_agent(net, "discrete", predict_noise=True, clip=True, mask=False)
    kw = dict(solver="ddpm", n_samples=4, sample_steps=3, use_ema=False, w_cfg=1.0, condition_cfg=torch.randn(4, 4),
              requires_grad=True)
    x0, _ = agent.sample(torch.zeros(4, 3), **kw)
    x1, _ = agent.sample(torch.zeros(4, 3), **kw)
    x1.sum().backward()                                       # the latest call's backward is served
    with pytest.raises(RuntimeError, match="overwritten"):
        x0.sum().backward()
