"""Classifier guidance inside the replayed loop, on CPU: this package's CumRewClassifier / HalfJannerUNet1d against goldens
written by the reference (tests/golden/make_golden_classifier.py -> classifier.npz), the lowered input-gradient program on the
numpy interpreter (tests/emulator.py) against fp64 autograd, and guided sample()
through the lowered program with classifier.gradients never called.  The other guided calls keep the host callback."""
import numpy as np
import pytest
import torch

import cg_ref
import emulator
import make_golden_classifier as mg
from common import load_golden, tape_of
from cleandiffuser_b200.engine import cabi, runtime
from cleandiffuser_b200.testing import NoiseTape

G = load_golden("classifier")
MATHS = {"fp32": cabi.MATH_FP32, "tf32": cabi.MATH_TF32_TC}


@pytest.fixture
def emulated(monkeypatch):
    emulator.emulate(monkeypatch)      # every operand is bounds-checked against its owner
    monkeypatch.setenv("CDS_BACKEND", "cuda")            # a fallback to the PyTorch loop raises


@pytest.mark.parametrize("name", list(mg.NETS))
@pytest.mark.parametrize("tkind", ["long", "float"])
def test_modules_match_reference(name, tkind):
    clf = cg_ref.make_classifier(mg.NETS[name], 31)
    x, t = torch.from_numpy(G[f"net/{name}/x"]), torch.from_numpy(G[f"net/{name}/t_{tkind}"])
    logp, grad = clf.gradients(x.clone(), t, None)
    np.testing.assert_allclose(logp.numpy(), G[f"net/{name}/logp_{tkind}"], rtol=1e-5, atol=1e-6)
    np.testing.assert_allclose(grad.numpy(), G[f"net/{name}/grad_{tkind}"], rtol=1e-4, atol=1e-6)
    assert not clf.model_ema.training


@pytest.mark.parametrize("math", list(MATHS))
@pytest.mark.parametrize("name", list(mg.NETS))
@pytest.mark.parametrize("tkind", ["long", "float"])
def test_lowered_input_gradient_matches_fp64_autograd(name, tkind, math):
    clf = cg_ref.make_classifier(mg.NETS[name], 31)
    x, t = torch.from_numpy(G[f"net/{name}/x"]), torch.from_numpy(G[f"net/{name}/t_{tkind}"])
    # the engine evaluates one time per iteration: iteration k of a table holding every row's time
    for k in range(len(t)):
        got, _ = cg_ref.lowered_gradient(clf, x, t, k, MATHS[math], "cpu")
        want = cg_ref.input_gradient_fp64(clf, x, t[k].expand(len(t)))
        rel = float((got.double() - want).norm() / want.norm())
        assert rel < (1e-6 if math == "fp32" else 1e-2), rel


def _sample(agent, prior, kw, name):
    tape = NoiseTape(tape_of(G, f"sample/{name}"))
    with tape.active():
        x0, log = agent.sample(prior, **kw)
    assert tape.pos == len(tape.draws)
    return x0, log


@pytest.mark.parametrize("math", list(MATHS))
@pytest.mark.parametrize("name", list(mg.SAMPLES))
def test_guided_sample_runs_in_the_lowered_program(emulated, name, math, monkeypatch):
    monkeypatch.setenv("CDS_MATH", math)
    agent, prior, kw = cg_ref.make_sample_agent(name)

    def refuse(*a, **k):
        raise AssertionError("classifier.gradients called: guidance left the program")
    monkeypatch.setattr(agent.classifier, "gradients", refuse)
    calls = runtime.STATS["engine_calls"]
    x0, log = _sample(agent, prior, kw, name)
    assert runtime.STATS["engine_calls"] == calls + 1 and runtime.STATS["guidance_path"] == "graph"
    if math == "fp32":
        err = np.abs(x0.numpy() - G[f"sample/{name}/x0"])
        assert err.max() < 3e-4, float(err.max())
        np.testing.assert_allclose(log["log_p"].numpy(), G[f"sample/{name}/log_p"], rtol=1e-3, atol=1e-3)
    else:
        # the TF32 denoiser of this 16-channel toy net alone is 0.25 max / 0.048 mean off the fp32 golden (w_cg = 0), so the
        # classifier's part is measured against the same TF32 program with the fp32 PyTorch guidance term of the host callback:
        # the TF32 input gradient (1e-2 of its norm, test above) moves x0 by a fraction of the denoiser's own TF32 error
        monkeypatch.undo()
        agent.classifier = _Wrapped(cg_ref.make_sample_agent(name)[0].classifier)
        with monkeypatch.context() as m:
            m.setattr(runtime, "_device_ok", lambda device: True)
            m.setattr(runtime, "_make_handle", lambda device, ops, n: emulator.Handle(ops, n))
            m.setenv("CDS_BACKEND", "cuda")
            m.setenv("CDS_MATH", math)
            ref, _ = _sample(agent, prior, kw, name)
        assert runtime.STATS["guidance_path"] == "callback"
        err = (x0 - ref).abs()
        assert err.max() < 0.2 and err.mean() < 0.015, (float(err.max()), float(err.mean()))


class _Wrapped:
    """a classifier the lowering does not recognise (same behaviour as the one it wraps)"""

    def __init__(self, clf):
        self.clf = clf

    def logp(self, x, noise, c=None):
        return self.clf.logp(x, noise, c)

    def gradients(self, x, noise, c=None):
        return self.clf.gradients(x, noise, c)


@pytest.mark.parametrize("case", ["unrecognised", "bf16", "train_mode"])
def test_other_guided_calls_keep_the_callback(emulated, case, monkeypatch):
    name = "discrete_ddpm_eps"
    monkeypatch.setenv("CDS_MATH", "bf16" if case == "bf16" else "fp32")
    agent, prior, kw = cg_ref.make_sample_agent(name)
    if case == "unrecognised":
        agent.classifier = _Wrapped(agent.classifier)
    if case == "train_mode":
        agent.classifier.model_ema.train()
    x0, log = _sample(agent, prior, kw, name)
    assert runtime.STATS["guidance_path"] == "callback", runtime.STATS["guidance_path"]
    assert runtime.STATS["guidance_reason"]
    if case == "bf16":            # (a bf16 program of this 16-channel toy denoiser is far from fp32 whatever the guidance)
        assert torch.isfinite(x0).all()
    else:
        err = np.abs(x0.numpy() - G[f"sample/{name}/x0"])
        assert err.max() < 3e-4, float(err.max())


def test_lowered_program_operators():
    """the classifier sits between the denoiser and the update: GN / GN_BWD pairs, then CDS_OP_GUIDE right before the update"""
    from cleandiffuser_b200.engine.runtime import SamplerPlan
    agent, prior, kw = cg_ref.make_sample_agent("discrete_ddpm_eps")
    plan = SamplerPlan(torch.device("cpu"), agent.model_ema["diffusion"], 4, (mg.H, mg.D), 3, 2, cfg_mode=0, predict_noise=True,
                       has_mask=True, has_min=False, has_max=False, keep_history=False, math=cabi.MATH_FP32,
                       classifier=agent.classifier)
    kinds = [op.kind for op in plan.program.ops]
    assert kinds[-2:] == [cabi.OP_GUIDE, cabi.OP_UPDATE]
    assert kinds.count(cabi.OP_GN) == kinds.count(cabi.OP_GN_BWD) == 2 * 6       # 6 ResidualBlocks, 2 GroupNorms each
    assert kinds.count(cabi.OP_DGRAD) == 2


def test_weights_repacked_after_update_classifier(emulated, monkeypatch):
    monkeypatch.setenv("CDS_MATH", "fp32")
    name = "discrete_ddpm_eps"
    agent, prior, kw = cg_ref.make_sample_agent(name)
    _sample(agent, prior, kw, name)
    g = torch.Generator().manual_seed(3)
    for _ in range(2):
        agent.update_classifier(torch.randn(mg.BATCH, mg.H, mg.D, generator=g), torch.randn(mg.BATCH, 1, generator=g))
    x0, _ = _sample(agent, prior, kw, name)
    assert runtime.STATS["guidance_path"] == "graph"
    monkeypatch.setenv("CDS_BACKEND", "torch")
    want, _ = _sample(agent, prior, kw, name)
    assert (x0 - want).abs().max() < 3e-4
