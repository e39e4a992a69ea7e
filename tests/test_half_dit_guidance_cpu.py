"""Classifier guidance with HalfDiT1d inside the replayed loop, on CPU: this package's HalfDiT1d against goldens written by the
reference (tests/golden/make_golden_half_dit.py -> half_dit.npz), the lowered input-gradient program on the numpy interpreter
(tests/emulator.py) against fp64 autograd, guided sample() calls through the lowered program with classifier.gradients never
called, the calls the lowering declines, repacking, a program audit and a constructor-space sweep."""
import os

import numpy as np
import pytest
import torch

import cg_ref
import dit_grad_ref as dr
import emulator
import make_golden_half_dit as mg
import program_audit as pa
from common import load_golden, tape_of
from guidance_space import all_pairs
from cleandiffuser_b200.engine import cabi, lower, runtime
from cleandiffuser_b200.testing import NoiseTape

G = load_golden("half_dit")
MATHS = {"fp32": cabi.MATH_FP32, "tf32": cabi.MATH_TF32_TC}
# relative L2 bound of the lowered input gradient against fp64 autograd.  fp32: the interpreter's operators are fp64 with fp32
# stores, so only the stores' rounding (2^-24 relative) accumulates, through at most a few dozen operators: measured <= 5e-7.
# TF32: the interpreter reads the operands of the tensor-core token GEMMs with 10-bit mantissas (2^-11 relative each), and a
# gradient passes through six such GEMMs per block, each summing over d_model to 4 d_model terms: measured <= 2e-3
REL = {"fp32": 1e-5, "tf32": 1e-2}


@pytest.fixture(autouse=True)
def gelu_semantics(monkeypatch):
    dr.register(monkeypatch)           # CDS_ACT_GELU_TANH in the shared activation tables (CDS_OP_STASH of DiT's MLP)


@pytest.fixture
def emulated(monkeypatch):
    emulator.emulate(monkeypatch)      # every operand is bounds-checked against its owner
    monkeypatch.setenv("CDS_BACKEND", "cuda")            # a fallback to the PyTorch loop raises


def _net_case(name):
    return torch.from_numpy(G[f"net/{name}/x"]), torch.from_numpy(G[f"net/{name}/t"])


def _rel(got, want):
    return float((got.double() - want).norm() / want.norm())


@pytest.mark.parametrize("name", list(mg.NETS))
def test_module_matches_reference(name):
    clf = dr.make_classifier(mg.NETS[name], 31)
    x, t = _net_case(name)
    logp, grad = clf.gradients(x.clone(), t, None)
    np.testing.assert_allclose(logp.numpy(), G[f"net/{name}/logp"], rtol=1e-5, atol=1e-6)
    np.testing.assert_allclose(grad.numpy(), G[f"net/{name}/grad"], rtol=1e-4, atol=1e-6)


def test_constructor_and_state_dict_layout_are_the_reference_ones():
    from cleandiffuser_b200.nn_classifier import HalfDiT1d
    net = HalfDiT1d(10, 1, 64)
    assert (net.d_model, len(net.blocks), net.blocks[0].attn.num_heads) == (384, 12, 6)
    shapes = {k: tuple(v.shape) for k, v in net.state_dict().items()}
    assert shapes["final_layer.linear.weight"] == (192, 384) and shapes["final_layer.adaLN_modulation.1.weight"] == (768, 384)
    assert [shapes[f"proj.{i}.weight"] for i in (0, 2, 3, 5)] == [(192,), (96, 192), (96,), (1, 96)]
    assert not any(k.startswith("proj.1") or k.startswith("proj.4") for k in shapes)
    for m in (net.final_layer.linear, net.final_layer.adaLN_modulation[-1]):
        assert not m.weight.any() and not m.bias.any()
    assert net(torch.randn(2, 5, 10), torch.tensor([1, 2])).shape == (2, 1)


@pytest.mark.parametrize("math", list(MATHS))
@pytest.mark.parametrize("name", list(mg.NETS))
def test_lowered_input_gradient_matches_fp64_autograd(name, math):
    clf = dr.make_classifier(mg.NETS[name], 31)
    x, t = _net_case(name)
    for k in range(len(t)):            # the engine evaluates one time per iteration: iteration k of the table
        got, _ = cg_ref.lowered_gradient(clf, x, t, k, MATHS[math], "cpu")
        want = dr.input_gradient_fp64(clf, x, t[k].expand(len(t)))
        assert _rel(got, want) < REL[math], (k, _rel(got, want))


def _sample(agent, prior, kw, name):
    tape = NoiseTape(tape_of(G, f"sample/{name}"))
    with tape.active():
        x0, log = agent.sample(prior.clone(), **kw)
    assert tape.pos == len(tape.draws)
    return x0, log


def _refuse(*a, **k):
    raise AssertionError("classifier.gradients called: guidance left the program")


@pytest.mark.parametrize("math", list(MATHS))
@pytest.mark.parametrize("name", list(mg.SAMPLES))
def test_guided_sample_runs_in_the_lowered_program(emulated, name, math, monkeypatch):
    monkeypatch.setenv("CDS_MATH", math)
    agent, prior, kw = dr.make_sample_agent(name)
    monkeypatch.setattr(agent.classifier, "gradients", _refuse)
    x0, log = _sample(agent, prior, kw, name)
    assert runtime.STATS["guidance_path"] == "graph", runtime.STATS["guidance_reason"]
    if math == "fp32":
        # summation order through 4 steps
        assert np.abs(x0.numpy() - G[f"sample/{name}/x0"]).max() < 3e-4
        np.testing.assert_allclose(log["log_p"].numpy(), G[f"sample/{name}/log_p"], rtol=1e-3, atol=1e-3)
        return
    # TF32: the denoiser's own TF32 error over these synthetic weights reaches 0.3 against the fp32 golden (the Janner UNet's
    # GroupNorms amplify it), so the graph path is held to the callback path of the same TF32 program: they differ by the
    # classifier gradient's TF32 error times w_cg sigma, carried by the loop: measured <= 3e-3 (1 + |x0|) (the Janner samples
    # reach |x0| ~ 100 over these weights)
    monkeypatch.setattr(runtime, "guidable", lambda *a, **k: "the callback, for comparison")
    agent, prior, kw = dr.make_sample_agent(name)
    want, _ = _sample(agent, prior, kw, name)
    assert runtime.STATS["guidance_path"] == "callback"
    assert ((x0 - want).abs() / (1 + want.abs())).max() < 1e-2, float(((x0 - want).abs() / (1 + want.abs())).max())


@pytest.mark.parametrize("name", list(mg.SAMPLES))
def test_guidance_moves_the_golden_samples(emulated, name, monkeypatch):
    monkeypatch.setenv("CDS_MATH", "fp32")
    agent, prior, kw = dr.make_sample_agent(name)
    kw["w_cg"] = 0.0
    x0, _ = _sample(agent, prior, kw, name)
    assert np.abs(x0.numpy() - G[f"sample/{name}/x0"]).max() > 1e-3


def _clf_with(**change):
    return dr.make_classifier(dict(mg.CLF, **change), 32)


DECLINES = {
    "train_mode": "classifier model_ema in train mode",
    "head_dim_8": "classifier head_dim 8 (16, 32 or 64 only)",
    "in_dim": "classifier in_dim does not match x",
    "proj": "classifier proj / final_layer without the reference's structure",
    "mse": "classifier network HalfDiT1d (MLPNNClassifier only)",
    "bf16": "bf16",
}


@pytest.mark.parametrize("case", list(DECLINES))
def test_other_guided_calls_keep_the_callback(emulated, case, monkeypatch):
    from cleandiffuser_b200.classifier import MSEClassifier
    name = "continuous_dit"
    monkeypatch.setenv("CDS_MATH", "bf16" if case == "bf16" else "fp32")
    clf = None
    if case == "head_dim_8":
        clf = _clf_with(n_heads=8)
    if case == "in_dim":
        clf = _clf_with(in_dim=mg.D + 1)
    agent, prior, kw = dr.make_sample_agent(name, classifier=clf)
    if case == "train_mode":
        agent.classifier.model_ema.train()
    if case == "proj":
        agent.classifier.model_ema.proj[1] = torch.nn.ReLU()
    if case == "mse":
        agent.classifier = MSEClassifier(agent.classifier.model, device="cpu")
        agent.classifier.model_ema.eval()
        kw["condition_cg"] = torch.zeros(mg.BATCH, 1)
    if case == "in_dim":
        with pytest.raises(RuntimeError):          # the reference's classifier cannot read x either
            _sample(agent, prior, kw, name)
    else:
        x0, _ = _sample(agent, prior, kw, name)
        assert torch.isfinite(x0).all()
        if case == "train_mode":                   # the same weights, dropout 0: the callback gives the golden
            assert np.abs(x0.numpy() - G[f"sample/{name}/x0"]).max() < 3e-4
    assert runtime.STATS["guidance_path"] == "callback", runtime.STATS["guidance_path"]
    assert DECLINES[case] in runtime.STATS["guidance_reason"], runtime.STATS["guidance_reason"]


def test_long_horizon_is_declined():
    clf = dr.make_classifier(mg.CLF, 32)
    assert lower.guidable(clf, (129, mg.D)) == "classifier horizon 129 (at most 128)"
    assert lower.guidable(clf, (128, mg.D)) is None


def test_existing_reasons_are_unchanged():
    from cleandiffuser_b200.classifier import CumRewClassifier
    assert lower.guidable(CumRewClassifier(torch.nn.Linear(3, 1)), (3,)) == \
        "classifier network Linear (HalfJannerUNet1d or MLPNNClassifier only)"


def _visible_ema(clf):
    with torch.no_grad():
        for p in clf.model.parameters():
            p.data.mul_(-1.0)
    rate, clf.ema_rate = clf.ema_rate, 0.0
    clf.ema_update()
    clf.ema_rate = rate


@pytest.mark.parametrize("how", ["update", "ema_update", "load"])
def test_plan_repacks_after_classifier_changes(emulated, how, monkeypatch, tmp_path):
    monkeypatch.setenv("CDS_MATH", "fp32")
    name = "continuous_dit"
    agent, prior, kw = dr.make_sample_agent(name)
    clf = agent.classifier
    first, _ = _sample(agent, prior, kw, name)
    epoch = clf.weights_epoch
    if how == "update":
        g = torch.Generator().manual_seed(3)
        x, t, r = torch.randn(4, mg.H, mg.D, generator=g), torch.rand(4, generator=g), torch.randn(4, 1, generator=g)
        clf.update(x, t, r)
        _visible_ema(clf)
    elif how == "ema_update":
        _visible_ema(clf)
    else:
        other = dr.make_classifier(mg.CLF, 33)
        path = os.path.join(tmp_path, "clf.pt")
        other.save(path)
        clf.load(path)
    assert clf.weights_epoch > epoch
    x0, _ = _sample(agent, prior, kw, name)
    assert runtime.STATS["guidance_path"] == "graph"
    monkeypatch.setenv("CDS_BACKEND", "torch")
    want, _ = _sample(agent, prior, kw, name)
    assert (x0 - want).abs().max() < 3e-4
    assert (want - first).abs().max() > 1e-3, "the classifier change did not move x0: the test shows nothing"


@pytest.mark.parametrize("math", list(MATHS))
def test_program_audit_of_the_guided_iteration_on_the_interpreter(emulated, math, monkeypatch):
    monkeypatch.setenv("CDS_MATH", math)
    name = "continuous_dit"
    agent, prior, kw = dr.make_sample_agent(name)
    _sample(agent, prior, kw, name)
    plan = next(iter(agent._engine_plans.values()))
    aud = pa.Auditor(f"half-dit-{math}", plan.program.ops, plan.handle, pa.plan_owners(plan))
    aud.audit_once(0)
    aud.audit_iteration(0)
    assert not aud.failures, "\n".join(aud.failures[:20])
    names = set(aud.worst)
    assert {"lnmod_bwd +res +gated", "lnmod_bwd +gated bcast", "lnmod_bwd", "guide"} <= names, names
    assert any(n.startswith("attn_bwd hd 32") for n in names) and any(n.startswith("stash grad") for n in names), names


# ---- constructor space: every axis of HalfDiT1d crossed all-pairs
AXES = {"hd": [16, 32, 64], "heads": [1, 2, 3], "depth": [1, 2], "horizon": [1, 3, 16, 33, 128],
        "emb": ["positional", "fourier", "untrainable_fourier", "untrainable_positional"], "out_dim": [1, 2, 5],
        "in_dim": [1, 7, 16]}
SPACE = all_pairs(AXES)


@pytest.mark.parametrize("case", SPACE, ids=[
    "-".join(f"{k}{v}" for k, v in c.items()) for c in SPACE])
def test_constructor_space_on_the_interpreter(case):
    kw = dict(in_dim=case["in_dim"], out_dim=case["out_dim"], emb_dim=16, d_model=case["hd"] * case["heads"],
              n_heads=case["heads"], depth=case["depth"], timestep_emb_type=case["emb"])
    clf = dr.make_classifier(kw, 7)
    x = torch.randn(2, case["horizon"], case["in_dim"], generator=torch.Generator().manual_seed(1))
    t = torch.tensor([2, 11])
    assert lower.guidable(clf, tuple(x.shape[1:])) is None
    got, _ = cg_ref.lowered_gradient(clf, x, t, 1, cabi.MATH_FP32, "cpu")
    want = dr.input_gradient_fp64(clf, x, t[1].expand(2))
    assert _rel(got, want) < REL["fp32"], _rel(got, want)
