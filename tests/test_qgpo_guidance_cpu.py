"""QGPO's classifier guidance inside the replayed loop, on CPU: this package's QGPOClassifier / QGPONNClassifier against goldens
written by the reference (tests/golden/make_golden_qgpo.py -> qgpo.npz), the lowered input-gradient program on the numpy
interpreter (tests/qgpo_ref.py over tests/cg_ref.py) against fp64 autograd, and QGPO-shaped guided sample() through the
lowered program with classifier.gradients never called.  The other guided calls keep the host callback."""
import os

import numpy as np
import pytest
import torch

import emulator
import make_golden_qgpo as mg
import qgpo_ref
from cleandiffuser_b200.engine import cabi, runtime
from cleandiffuser_b200.testing import NoiseTape

G = qgpo_ref.golden()
MATHS = {"fp32": cabi.MATH_FP32, "tf32": cabi.MATH_TF32_TC}


@pytest.fixture
def emulated(monkeypatch):
    monkeypatch.setattr(runtime, "_device_ok", lambda device: True)
    owners = emulator.record_owners(monkeypatch)      # every operand is bounds-checked against its owner
    monkeypatch.setattr(runtime, "_make_handle", lambda device, ops, n: qgpo_ref.Handle(ops, n, owners()))
    monkeypatch.setenv("CDS_BACKEND", "cuda")            # a fallback to the PyTorch loop raises


def _net_case(name):
    return (torch.from_numpy(G[f"net/{name}/{k}"]) for k in ("x", "t", "obs"))


@pytest.mark.parametrize("name", list(mg.NETS))
def test_modules_match_reference(name):
    clf = qgpo_ref.make_classifier(mg.NETS[name], 31)
    x, t, obs = _net_case(name)
    logp, grad = clf.gradients(x.clone(), t, obs)
    np.testing.assert_allclose(logp.numpy(), G[f"net/{name}/logp"], rtol=1e-5, atol=1e-6)
    np.testing.assert_allclose(grad.numpy(), G[f"net/{name}/grad"], rtol=1e-4, atol=1e-6)
    assert not clf.model_ema.training


def test_state_dict_layout_is_the_reference_one():
    from cleandiffuser_b200.nn_classifier import QGPONNClassifier
    net = QGPONNClassifier(11, 3, 64, [256, 256, 256], "untrainable_fourier")
    shapes = {k: tuple(v.shape) for k, v in net.state_dict().items()}
    assert shapes == {"map_noise.freqs": (32,), "obs_proj.weight": (64, 11), "obs_proj.bias": (64,),
                      "act_proj.weight": (64, 3), "act_proj.bias": (64,),
                      "mlp.mlp.0.0.weight": (256, 192), "mlp.mlp.0.0.bias": (256,), "mlp.mlp.1.0.weight": (256, 256),
                      "mlp.mlp.1.0.bias": (256,), "mlp.mlp.2.0.weight": (256, 256), "mlp.mlp.2.0.bias": (256,),
                      "mlp.mlp.3.weight": (1, 256), "mlp.mlp.3.bias": (1,)}


@pytest.mark.parametrize("math", list(MATHS))
@pytest.mark.parametrize("name", list(mg.NETS))
def test_lowered_input_gradient_matches_fp64_autograd(name, math):
    clf = qgpo_ref.make_classifier(mg.NETS[name], 31)
    x, t, obs = _net_case(name)
    # the engine evaluates one time per iteration: iteration k of a table holding every row's time
    for k in range(len(t)):
        got, _ = qgpo_ref.lowered_gradient(clf, x, t, obs, k, MATHS[math], "cpu")
        want = qgpo_ref.input_gradient_fp64(clf, x, t[k].expand(len(t)), obs)
        rel = float((got.double() - want).norm() / want.norm())
        # fp32: summation order only (the interpreter's GEMMs are fp64 with fp32 stores).  TF32: the interpreter reads the
        # act_proj and first-layer operands of the tensor-core programs as TF32 where the kernels would
        assert rel < (1e-6 if math == "fp32" else 1e-2), (k, rel)


def _sample(agent, prior, kw, name):
    tape = NoiseTape(qgpo_ref.tape_of(G, name))
    with tape.active():
        x0, log = agent.sample(prior, **kw)
    assert tape.pos == len(tape.draws)
    return x0, log


@pytest.mark.parametrize("math", list(MATHS))
@pytest.mark.parametrize("name", list(mg.SAMPLES))
def test_guided_sample_runs_in_the_lowered_program(emulated, name, math, monkeypatch):
    monkeypatch.setenv("CDS_MATH", math)
    agent, prior, kw = qgpo_ref.make_sample_agent(name)

    def refuse(*a, **k):
        raise AssertionError("classifier.gradients called: guidance left the program")
    monkeypatch.setattr(agent.classifier, "gradients", refuse)
    calls = runtime.STATS["engine_calls"]
    x0, log = _sample(agent, prior, kw, name)
    assert runtime.STATS["engine_calls"] == calls + 1 and runtime.STATS["guidance_path"] == "graph"
    err = np.abs(x0.numpy() - G[f"sample/{name}/x0"])
    # fp32: summation order through 5 steps.  TF32: SfBCUNet's 64..256-wide Linears read 10-bit mantissas
    assert err.max() < (3e-4 if math == "fp32" else 3e-2), float(err.max())
    # log_p: the classifier's PyTorch logp of x0 after the loop
    np.testing.assert_allclose(log["log_p"].numpy(), G[f"sample/{name}/log_p"], rtol=1e-3,
                               atol=1e-3 if math == "fp32" else 2e-2)


class _Wrapped:
    """a classifier the lowering does not recognise (same behaviour as the one it wraps)"""

    def __init__(self, clf):
        self.clf = clf

    def logp(self, x, noise, c=None):
        return self.clf.logp(x, noise, c)

    def gradients(self, x, noise, c=None):
        return self.clf.gradients(x, noise, c)


@pytest.mark.parametrize("case", ["unrecognised", "bf16", "train_mode", "branches"])
def test_other_guided_calls_keep_the_callback(emulated, case, monkeypatch):
    name = "ddpm_eps"
    monkeypatch.setenv("CDS_MATH", "bf16" if case == "bf16" else "fp32")
    agent, prior, kw = qgpo_ref.make_sample_agent(name)
    if case == "unrecognised":
        agent.classifier = _Wrapped(agent.classifier)
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
    assert reason and {"unrecognised": "classifier _Wrapped", "bf16": "bf16", "train_mode": "train mode",
                       "branches": "CDS_BRANCHES"}[case] in reason, reason
    if case == "bf16":            # (a bf16 program of the denoiser is far from fp32 whatever the guidance)
        assert torch.isfinite(x0).all()
    else:
        err = np.abs(x0.numpy() - G[f"sample/{name}/x0"])
        assert err.max() < 3e-4, float(err.max())


def test_no_classifier_condition_raises_like_the_reference(emulated):
    """condition_cg=None keeps the callback, whose QGPONNClassifier forward fails in obs_proj exactly as the reference's does"""
    agent, prior, kw = qgpo_ref.make_sample_agent("ddpm_eps")
    kw["condition_cg"] = None
    with pytest.raises(TypeError):
        _sample(agent, prior, kw, "ddpm_eps")
    assert runtime.STATS["guidance_path"] == "callback"
    assert "condition_cg=None" in runtime.STATS["guidance_reason"]


def test_lowered_program_operators():
    """act_proj, the three hidden Linears with SiLU stashes between them, the head, three SiLU data gradients, the two
    factor data gradients back to x, then CDS_OP_GUIDE right before the update"""
    from cleandiffuser_b200.engine.runtime import SamplerPlan
    agent, prior, kw = qgpo_ref.make_sample_agent("ddpm_eps")
    plan = SamplerPlan(torch.device("cpu"), agent.model_ema["diffusion"], 16, (mg.ACT,), 3, 2, cfg_mode=1, predict_noise=True,
                       has_mask=False, has_min=True, has_max=True, keep_history=False, math=cabi.MATH_FP32,
                       classifier=agent.classifier)
    kinds = [op.kind for op in plan.program.ops]
    C, S, D = cabi.OP_CONV, cabi.OP_STASH, cabi.OP_DGRAD
    assert kinds[-14:] == [C, C, S, C, S, C, cabi.OP_HEAD_GRAD, D, D, D, D, D, cabi.OP_GUIDE, cabi.OP_UPDATE]
    acts = [op.u.dgrad.act for op in plan.program.ops if op.kind == D]
    assert acts == [cabi.ACT_SILU] * 3 + [cabi.ACT_NONE] * 2
    assert all(op.u.stash.act == cabi.ACT_SILU and not op.u.stash.dst for op in plan.program.ops if op.kind == S)


def _retrain(clf, seed):
    g = torch.Generator().manual_seed(seed)
    x, t = torch.randn(8, 4, mg.ACT, generator=g), torch.rand(8, generator=g)
    y = {"soft_label": torch.softmax(torch.randn(8, 4, 1, generator=g), 1), "obs": torch.randn(8, mg.OBS, generator=g)}
    for _ in range(3):
        clf.update(x, t, y)
    with torch.no_grad():                 # a visible change of model_ema (the EMA moves it by 0.5 % per step)
        for p, q in zip(clf.model.parameters(), clf.model_ema.parameters()):
            q.data.copy_(p.data)


@pytest.mark.parametrize("how", ["update", "load"])
def test_plan_repacks_after_classifier_update_and_load(emulated, how, monkeypatch, tmp_path):
    monkeypatch.setenv("CDS_MATH", "fp32")
    name = "ddpm_eps"
    agent, prior, kw = qgpo_ref.make_sample_agent(name)
    first, _ = _sample(agent, prior, kw, name)
    if how == "update":
        _retrain(agent.classifier, 3)              # clf.update() directly, as QGPO trains, never agent.update_classifier
    else:
        other = qgpo_ref.make_classifier(dict(obs_dim=mg.OBS, act_dim=mg.ACT), 33)
        path = os.path.join(tmp_path, "clf.pt")
        other.save(path)
        epoch = agent.classifier.weights_epoch
        agent.classifier.load(path)
        assert agent.classifier.weights_epoch == epoch + 1
    x0, _ = _sample(agent, prior, kw, name)
    assert runtime.STATS["guidance_path"] == "graph"
    monkeypatch.setenv("CDS_BACKEND", "torch")
    want, _ = _sample(agent, prior, kw, name)
    assert (x0 - want).abs().max() < 3e-4
    assert (want - first).abs().max() > 1e-3, "the classifier change did not move x0: the test shows nothing"


@pytest.mark.parametrize("math", list(MATHS))
def test_program_audit_of_the_qgpo_iteration_on_the_interpreter(emulated, math, monkeypatch):
    """tests/qgpo_audit.py (tests/program_audit.py's audit with QGPO's operators) drives the interpreter over the guided program: every operator of every iteration within its
    bound and nothing written outside its declared outputs (the same audit runs on the H100)"""
    import program_audit as pa
    import qgpo_audit
    monkeypatch.setenv("CDS_MATH", math)
    agent, prior, kw = qgpo_ref.make_sample_agent("ddpm_eps")
    _sample(agent, prior, kw, "ddpm_eps")
    plan = next(iter(agent._engine_plans.values()))
    aud = qgpo_audit.Auditor(f"qgpo-{math}", plan.program.ops, plan.handle, pa.plan_owners(plan))
    aud.audit_once(0)
    for it in range(plan.n_iters):
        aud.audit_iteration(it)
    assert not aud.failures, "\n".join(aud.failures[:20])
    assert {"head_grad silu", "dgrad silu", "stash silu (no slot)"} <= set(aud.worst)
