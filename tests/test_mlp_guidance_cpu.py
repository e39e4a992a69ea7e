"""Classifier guidance with MLPNNClassifier inside the replayed loop, on CPU: this package's MSEClassifier, CumRewClassifier and
MLPNNClassifier against goldens written by the reference (tests/golden/make_golden_mlp_classifier.py -> mlp_classifier.npz),
the lowered input-gradient program on the numpy interpreter (tests/emulator.py) against fp64 autograd for every hidden
activation and both heads, and guided sample() calls shaped like the reference's classifier-guidance tutorial through the
lowered program with classifier.gradients never called.  The calls the lowering does not serve keep the host callback."""
import os

import numpy as np
import pytest
import torch

import cg_ref
import emulator
import make_golden_mlp_classifier as mg
import mlp_cg_ref
import program_audit as pa
import relu_ref
from common import load_golden, tape_of
from cleandiffuser_b200.engine import cabi, runtime
from cleandiffuser_b200.testing import NoiseTape

G = load_golden("mlp_classifier")
MATHS = {"fp32": cabi.MATH_FP32, "tf32": cabi.MATH_TF32_TC}
HEADS = {"mse": "mse_relu", "cumrew": "cumrew_relu"}          # the golden net case whose shape each head is tested at
TF32_REL = {"ReLU": 5e-2, "SiLU": 1e-2, "Mish": 1e-2}        # relative bound of a TF32 input gradient per hidden activation


@pytest.fixture(autouse=True)
def relu_semantics(monkeypatch):
    relu_ref.register(monkeypatch)     # CDS_ACT_RELU in the shared operator references for this test (tests/relu_ref.py)


@pytest.fixture
def emulated(monkeypatch):
    emulator.emulate(monkeypatch)      # every operand is bounds-checked against its owner
    monkeypatch.setenv("CDS_BACKEND", "cuda")            # a fallback to the PyTorch loop raises


def _net_case(name):
    x, t, c = (torch.from_numpy(G[f"net/{name}/{k}"]) for k in ("x", "t", "c"))
    return x, t, (c if mg.NETS[name]["head"] == "mse" else None)


@pytest.mark.parametrize("name", list(mg.NETS))
def test_modules_match_reference(name):
    clf = mlp_cg_ref.make_classifier(name, 31)
    x, t, c = _net_case(name)
    logp, grad = clf.gradients(x.clone(), t, c)
    np.testing.assert_allclose(logp.numpy(), G[f"net/{name}/logp"], rtol=1e-5, atol=1e-6)
    np.testing.assert_allclose(grad.numpy(), G[f"net/{name}/grad"], rtol=1e-4, atol=1e-6)
    assert not clf.model_ema.training


def test_state_dict_layout_is_the_reference_one():
    from cleandiffuser_b200.nn_classifier import MLPNNClassifier
    net = MLPNNClassifier(9, 60, 32, [256, 128], timestep_emb_type="untrainable_fourier")
    shapes = {k: tuple(v.shape) for k, v in net.state_dict().items()}
    assert shapes == {"map_noise.freqs": (16,), "mlp.mlp.0.0.weight": (256, 41), "mlp.mlp.0.0.bias": (256,),
                      "mlp.mlp.1.0.weight": (128, 256), "mlp.mlp.1.0.bias": (128,),
                      "mlp.mlp.2.weight": (60, 128), "mlp.mlp.2.bias": (60,)}
    assert type(net.mlp.mlp[0][1]).__name__ == "ReLU" and net.mlp.mlp[0][1] is net.mlp.mlp[1][1]


def test_mse_classifier_loss_and_logp_are_the_reference_ones():
    from cleandiffuser_b200.classifier import MSEClassifier
    clf = mlp_cg_ref.make_classifier("tutorial_mse_silu", 31)
    assert isinstance(clf, MSEClassifier) and clf.temperature == 1.0
    x, t, c = _net_case("tutorial_mse_silu")
    with torch.no_grad():
        y = clf.model(x, t)
        assert torch.equal(clf.loss(x, t, c), torch.nn.functional.mse_loss(y, c))
        clf.temperature = 0.25
        assert torch.allclose(clf.logp(x, t, c), -0.25 * ((clf.model_ema(x, t) - c) ** 2).mean(-1, keepdim=True))


@pytest.mark.parametrize("math", list(MATHS))
@pytest.mark.parametrize("act", mlp_cg_ref.ACTS)
@pytest.mark.parametrize("head", list(HEADS))
def test_lowered_input_gradient_matches_fp64_autograd(head, act, math):
    name = HEADS[head]
    clf = mlp_cg_ref.make_classifier(name, 31, act=act)
    clf.temperature = 0.7 if head == "mse" else None
    x, t, c = _net_case(name)
    # the engine evaluates one time per iteration: iteration k of a table holding every row's time
    for k in range(len(t)):
        got, _ = cg_ref.lowered_gradient(clf, x, t, k, MATHS[math], "cpu", cond=c)
        want = mlp_cg_ref.input_gradient_fp64(clf, x, t[k].expand(len(t)), c)
        rel = float((got.double() - want).norm() / want.norm())
        # fp32: summation order only (the interpreter's GEMMs are fp64 with fp32 stores).  TF32: the interpreter reads the
        # operands of the tensor-core Linears as TF32 where the kernels would.  Under ReLU a pre-activation within the TF32
        # error of 0 can change sign, which switches its unit's whole term of the gradient on or off: measured up to 1.4e-2
        # here (2.5e-4 with SiLU or Mish at the same shape)
        assert rel < (1e-6 if math == "fp32" else TF32_REL[act]), (k, rel)


def test_lowered_relu_gradient_is_zero_where_the_pre_activation_is_zero():
    """a hidden unit whose pre-activation is exactly 0 passes no gradient (ATen's threshold_backward), on every row"""
    clf = mlp_cg_ref.make_classifier("cumrew_relu", 31)
    x, t, _ = _net_case("cumrew_relu")
    lin1 = clf.model_ema.mlp.mlp[0][0]
    with torch.no_grad():
        lin1.weight[:7] = 0.0                   # units 0..6 of the first layer: z = 0 whatever x and t
        lin1.bias[:7] = 0.0
        lin1.weight[7:, :x.shape[1]] = 0.0      # every other unit ignores x: only units 0..6 could carry a gradient
    got, _ = cg_ref.lowered_gradient(clf, x, t, 0, cabi.MATH_FP32, "cpu")
    assert torch.equal(got, torch.zeros_like(got))
    assert torch.equal(mlp_cg_ref.input_gradient_fp64(clf, x, t[0].expand(len(t))), torch.zeros_like(got, dtype=torch.float64))


def _sample(agent, prior, kw, name):
    tape = NoiseTape(tape_of(G, f"sample/{name}"))
    with tape.active():
        x0, log = agent.sample(prior, **kw)
    assert tape.pos == len(tape.draws)
    return x0, log


def _refuse(*a, **k):
    raise AssertionError("classifier.gradients called: guidance left the program")


@pytest.mark.parametrize("math", list(MATHS))
@pytest.mark.parametrize("name", list(mg.SAMPLES))
def test_guided_sample_runs_in_the_lowered_program(emulated, name, math, monkeypatch):
    monkeypatch.setenv("CDS_MATH", math)
    agent, prior, kw = mlp_cg_ref.make_sample_agent(name)
    monkeypatch.setattr(agent.classifier, "gradients", _refuse)
    calls = runtime.STATS["engine_calls"]
    x0, log = _sample(agent, prior, kw, name)
    assert runtime.STATS["engine_calls"] == calls + 1 and runtime.STATS["guidance_path"] == "graph"
    err = np.abs(x0.numpy() - G[f"sample/{name}/x0"])
    # fp32: summation order through 5 steps.  TF32: the denoisers' and classifiers' 256-wide Linears read 10-bit mantissas
    assert err.max() < (3e-4 if math == "fp32" else 3e-2), float(err.max())
    # log_p: the classifier's PyTorch logp of x0 after the loop
    np.testing.assert_allclose(log["log_p"].numpy(), G[f"sample/{name}/log_p"], rtol=1e-3,
                               atol=1e-3 if math == "fp32" else 2e-2)


@pytest.mark.parametrize("name", list(mg.SAMPLES))
def test_guidance_moves_the_golden_samples(emulated, name, monkeypatch):
    """the goldens show the guidance: the same call with w_cg = 0 ends elsewhere"""
    monkeypatch.setenv("CDS_MATH", "fp32")
    agent, prior, kw = mlp_cg_ref.make_sample_agent(name)
    kw["w_cg"] = 0.0
    x0, _ = _sample(agent, prior, kw, name)
    assert np.abs(x0.numpy() - G[f"sample/{name}/x0"]).max() > 1e-3


class _Wrapped:
    """a classifier the lowering does not recognise (same behaviour as the one it wraps)"""

    def __init__(self, clf):
        self.clf = clf

    def logp(self, x, noise, c=None):
        return self.clf.logp(x, noise, c)

    def gradients(self, x, noise, c=None):
        return self.clf.gradients(x, noise, c)


def _swap_module(clf, index, module):
    """replace entry ``index`` of model_ema's Mlp stages: a hidden stage's activation (int) or the output activation (-1)"""
    seq = clf.model_ema.mlp.mlp
    if index == -1:
        seq[-1] = module
    else:
        for s in list(seq)[:-2]:
            s[1] = module


DECLINES = {"unrecognised": "classifier _Wrapped", "gelu": "classifier activation GELU (ReLU, SiLU or Mish only)",
            "tanh_out": "classifier out_activation Tanh (Identity only)", "train_mode": "train mode", "bf16": "bf16",
            "branches": "CDS_BRANCHES"}


@pytest.mark.parametrize("case", list(DECLINES))
def test_other_guided_calls_keep_the_callback(emulated, case, monkeypatch):
    name = "tutorial"
    monkeypatch.setenv("CDS_MATH", "bf16" if case == "bf16" else "fp32")
    agent, prior, kw = mlp_cg_ref.make_sample_agent(name)
    if case == "unrecognised":
        agent.classifier = _Wrapped(agent.classifier)
    if case == "gelu":
        _swap_module(agent.classifier, 0, torch.nn.GELU())
    if case == "tanh_out":
        _swap_module(agent.classifier, -1, torch.nn.Tanh())
    if case == "train_mode":
        agent.classifier.model_ema.train()
    if case == "branches":
        # the callback needs a single-branch program too: the call then falls back to the PyTorch loop
        monkeypatch.setenv("CDS_BRANCHES", "2")
        monkeypatch.setenv("CDS_BRANCH_MIN_BATCH", "8")
        monkeypatch.setenv("CDS_BACKEND", "auto")
    x0, log = _sample(agent, prior, kw, name)
    assert runtime.STATS["guidance_path"] == "callback", runtime.STATS["guidance_path"]
    reason = runtime.STATS["guidance_reason"]
    assert reason and DECLINES[case] in reason, reason
    if case in ("bf16", "gelu", "tanh_out"):     # another classifier, or a bf16 program of the denoiser: no golden
        assert torch.isfinite(x0).all()
    else:
        err = np.abs(x0.numpy() - G[f"sample/{name}/x0"])
        assert err.max() < 3e-4, float(err.max())


def test_cumrew_over_another_network_keeps_its_reason():
    from cleandiffuser_b200.classifier import CumRewClassifier
    from cleandiffuser_b200.engine import lower
    clf = CumRewClassifier(torch.nn.Linear(3, 1))
    assert lower.guidable(clf, (3,)) == "classifier network Linear (HalfJannerUNet1d or MLPNNClassifier only)"


def test_no_classifier_condition_raises_like_the_reference(emulated):
    """MSEClassifier with condition_cg=None keeps the callback, whose logp fails on ``pred_y - None`` exactly as the
    reference's does"""
    agent, prior, kw = mlp_cg_ref.make_sample_agent("tutorial")
    kw["condition_cg"] = None
    with pytest.raises(TypeError):
        _sample(agent, prior, kw, "tutorial")
    assert runtime.STATS["guidance_path"] == "callback"
    assert "condition_cg=None" in runtime.STATS["guidance_reason"]


def test_the_tutorial_call_runs_in_the_graph(emulated, monkeypatch):
    """the reference tutorial's guided inference, written as the tutorial writes it (tutorials/3_classifier_guidance.py with
    use_customized_classifier = False), batch 50; swapping in GELU or the tutorial's own classifier class keeps the callback"""
    import torch.nn as nn
    from cleandiffuser_b200.classifier import BaseClassifier, MSEClassifier
    from cleandiffuser_b200.diffusion import DiscreteDiffusionSDE
    from cleandiffuser_b200.nn_classifier import MLPNNClassifier
    from cleandiffuser_b200.nn_diffusion import PearceMlp
    from cleandiffuser_b200.testing import load_synth
    monkeypatch.setenv("CDS_MATH", "fp32")
    device, obs_dim, act_dim = "cpu", 60, 9
    nn_diffusion = load_synth(PearceMlp(act_dim, To=0, emb_dim=64, hidden_dim=256, timestep_emb_type="positional"), 1)
    nn_classifier = load_synth(MLPNNClassifier(x_dim=act_dim, out_dim=obs_dim, emb_dim=32, hidden_dims=[256, ],
                                               activation=nn.SiLU(), timestep_emb_type="positional"), 2)
    classifier = MSEClassifier(nn_classifier, temperature=1.0, device=device)
    actor = DiscreteDiffusionSDE(nn_diffusion, classifier=classifier, predict_noise=False, optim_params={"lr": 3e-4},
                                 x_max=+1. * torch.ones((1, act_dim)), x_min=-1. * torch.ones((1, act_dim)),
                                 diffusion_steps=5, ema_rate=0.9999, device=device)
    actor.eval()
    classifier.eval()
    obs = torch.randn(50, obs_dim, generator=torch.Generator().manual_seed(0))
    prior = torch.zeros((50, act_dim), device=device)

    def call():
        with NoiseTape().active():
            return actor.sample(prior, solver="ddpm", n_samples=50, sample_steps=5, temperature=0.5, w_cg=0.1,
                                condition_cg=torch.tensor(obs.numpy(), device=device, dtype=torch.float32))
    act, log = call()
    assert runtime.STATS["guidance_path"] == "graph", runtime.STATS["guidance_reason"]
    assert act.shape == (50, act_dim) and log["log_p"].shape == (50, 1)

    class MyObsClassifier(BaseClassifier):          # the tutorial's hand-written classifier
        def loss(self, x, noise, y):
            return nn.functional.mse_loss(self.model(x, noise, y), y)

        def logp(self, x, noise, c):
            return -((self.model_ema(x, noise) - c) ** 2).mean(-1, keepdim=True)
    actor.classifier = MyObsClassifier(nn_classifier, device=device)
    call()
    assert runtime.STATS["guidance_path"] == "callback" and "MyObsClassifier" in runtime.STATS["guidance_reason"]
    actor.classifier = classifier
    _swap_module(classifier, 0, nn.GELU())
    call()
    assert runtime.STATS["guidance_path"] == "callback" and "GELU" in runtime.STATS["guidance_reason"]


@pytest.mark.parametrize("name,ops", [
    ("tutorial", "C S C D D"),          # z_1, h_1 = silu(z_1), r = W_o h_1 + (b_o - c); dz_1 (SiLU'), dx
    ("dql_cumrew", "C S C D D D"),      # z_1, h_1 = relu(z_1), z_2; dz_2 = W_o relu'(z_2) (seed 1), dz_1, dx
])
def test_lowered_program_operators(name, ops):
    """the classifier's operators sit between the denoiser and CDS_OP_GUIDE, right before the update"""
    from cleandiffuser_b200.engine.runtime import SamplerPlan
    agent, prior, kw = mlp_cg_ref.make_sample_agent(name)
    net = mg.NETS[mg.SAMPLES[name]["net"]]
    plan = SamplerPlan(torch.device("cpu"), agent.model_ema["diffusion"], 16, (net["x_dim"],), 3, 2,
                       cfg_mode=1 if mg.SAMPLES[name]["kind"] == "continuous" else 0,
                       predict_noise=mg.SAMPLES[name]["predict_noise"], has_mask=False, has_min=True, has_max=True,
                       keep_history=False, math=cabi.MATH_FP32, classifier=agent.classifier)
    code = {cabi.OP_CONV: "C", cabi.OP_STASH: "S", cabi.OP_DGRAD: "D"}
    n = len(ops.split())
    tail = plan.program.ops[-n - 2:]
    assert " ".join(code.get(op.kind, "?") for op in tail[:-2]) == ops
    assert [op.kind for op in tail[-2:]] == [cabi.OP_GUIDE, cabi.OP_UPDATE]
    act = cabi.ACT_SILU if net["act"] == "SiLU" else cabi.ACT_RELU
    dgrads = [op.u.dgrad for op in tail if op.kind == cabi.OP_DGRAD]
    assert [d.act for d in dgrads] == [act] * (len(dgrads) - 1) + [cabi.ACT_NONE]
    assert all(op.u.stash.act == act and not op.u.stash.dst for op in tail if op.kind == cabi.OP_STASH)


def _retrain(clf, seed):
    g = torch.Generator().manual_seed(seed)
    x_dim, out_dim = clf.model.mlp.mlp[0][0].in_features - 32, clf.model.mlp.mlp[-2].out_features
    x, t, y = torch.randn(8, x_dim, generator=g), torch.randint(0, mg.T, (8,), generator=g), torch.randn(8, out_dim, generator=g)
    for _ in range(3):
        clf.update(x, t, y)


def _visible_ema(clf):
    """a visible change of model_ema through ema_update (the default rate moves it by 0.5 % per step)"""
    with torch.no_grad():
        for p in clf.model.parameters():
            p.data.mul_(-1.0)
    rate, clf.ema_rate = clf.ema_rate, 0.0
    clf.ema_update()
    clf.ema_rate = rate


@pytest.mark.parametrize("how", ["update", "ema_update", "load", "temperature"])
def test_plan_repacks_after_classifier_changes(emulated, how, monkeypatch, tmp_path):
    monkeypatch.setenv("CDS_MATH", "fp32")
    name = "dql_eps"
    agent, prior, kw = mlp_cg_ref.make_sample_agent(name)
    clf = agent.classifier
    first, _ = _sample(agent, prior, kw, name)
    epoch = clf.weights_epoch
    if how == "update":
        _retrain(clf, 3)
        _visible_ema(clf)
    elif how == "ema_update":
        _visible_ema(clf)
    elif how == "load":
        other = mlp_cg_ref.make_classifier(mg.SAMPLES[name]["net"], 33)
        path = os.path.join(tmp_path, "clf.pt")
        other.save(path)
        clf.load(path)
    else:
        clf.temperature = 8.0                     # a plain attribute: no epoch, read by every call
    assert clf.weights_epoch > epoch or how == "temperature"
    x0, _ = _sample(agent, prior, kw, name)
    assert runtime.STATS["guidance_path"] == "graph"
    monkeypatch.setenv("CDS_BACKEND", "torch")
    want, _ = _sample(agent, prior, kw, name)
    assert (x0 - want).abs().max() < 3e-4
    assert (want - first).abs().max() > 1e-3, "the classifier change did not move x0: the test shows nothing"


@pytest.mark.parametrize("math", list(MATHS))
@pytest.mark.parametrize("name", ["tutorial", "dql_eps"])
def test_program_audit_of_the_guided_iteration_on_the_interpreter(emulated, name, math, monkeypatch):
    """tests/program_audit.py drives the interpreter over the guided program: every operator of every iteration within its
    bound and nothing written outside its declared outputs (the same audit runs on the H100)"""
    monkeypatch.setenv("CDS_MATH", math)
    agent, prior, kw = mlp_cg_ref.make_sample_agent(name)
    _sample(agent, prior, kw, name)
    plan = next(iter(agent._engine_plans.values()))
    aud = pa.Auditor(f"mlp-{name}-{math}", plan.program.ops, plan.handle, pa.plan_owners(plan))
    aud.audit_once(0)
    for it in range(plan.n_iters):
        aud.audit_iteration(it)
    assert not aud.failures, "\n".join(aud.failures[:20])
    act = "silu" if name == "tutorial" else "relu"
    assert {f"dgrad {act}", f"stash {act} (no slot)", "dgrad", "guide"} <= set(aud.worst)
