"""Classifier guidance in ContinuousEDM and the legacy DDPM class, on CPU: the PyTorch loop against goldens written by the
reference (tests/golden/make_golden_edm_guided.py -> edm_guided.npz), and the engine's programs on the numpy interpreter
(tests/emulator.py, with the update's guidance operand from tests/edm_guide_ref.py): the lowered classifier gradient with
classifier.gradients never called, the host callback for a classifier the lowering does not recognise, the guidance scale and
classifier time columns against the reference's expressions bit for bit, unguided programs without the operand, and the
requests that keep the PyTorch loop with their reason."""
import numpy as np
import pytest
import torch

import edm_guide_ref
import emulator
import make_golden_edm_guided as mg
from common import load_golden, tape_of
from cleandiffuser_b200.engine import cabi, runtime
from cleandiffuser_b200.testing import NoiseTape

G = load_golden("edm_guided")


def package_classes():
    from cleandiffuser_b200.classifier import CumRewClassifier, MSEClassifier
    from cleandiffuser_b200.diffusion import ContinuousEDM
    from cleandiffuser_b200.diffusion.legacy import DDPM
    from cleandiffuser_b200.nn_classifier import HalfJannerUNet1d, MLPNNClassifier
    from cleandiffuser_b200.nn_condition import IdentityCondition
    from cleandiffuser_b200.nn_diffusion import DQLMlp, JannerUNet1d
    return dict(CumRewClassifier=CumRewClassifier, MSEClassifier=MSEClassifier, DDPM=DDPM, ContinuousEDM=ContinuousEDM,
                HalfJannerUNet1d=HalfJannerUNet1d, MLPNNClassifier=MLPNNClassifier, IdentityCondition=IdentityCondition,
                DQLMlp=DQLMlp, JannerUNet1d=JannerUNet1d)


CLS = package_classes()


@pytest.fixture
def emulated(monkeypatch):
    emulator.emulate(monkeypatch)      # every operand is bounds-checked against its owner
    edm_guide_ref.register(monkeypatch)
    monkeypatch.setenv("CDS_BACKEND", "cuda")            # a fallback to the PyTorch loop raises
    monkeypatch.setenv("CDS_MATH", "fp32")


def run_case(name, agent=None, **over):
    agent = agent if agent is not None else mg.make_agent(name, CLS)
    prior, c = (torch.from_numpy(G[f"sample/{name}/{k}"]) for k in ("prior", "c"))
    fn, kw = mg.sample_call(name, agent, prior, c)
    kw.update(over)
    tape = NoiseTape(tape_of(G, f"sample/{name}"))
    with tape.active():
        x0, log = fn(prior.clone(), **kw)
    assert tape.pos == len(tape.draws)
    return x0, log


def _refuse(*a, **k):
    raise AssertionError("classifier.gradients called: guidance left the program")


class _Wrapped:
    """a classifier the lowering does not recognise (same behaviour as the one it wraps)"""

    def __init__(self, clf):
        self.clf = clf

    def logp(self, x, noise, c=None):
        return self.clf.logp(x, noise, c)

    def gradients(self, x, noise, c=None):
        return self.clf.gradients(x, noise, c)


@pytest.mark.parametrize("name", list(mg.CASES))
def test_pytorch_loop_matches_reference(name, monkeypatch):
    monkeypatch.setenv("CDS_BACKEND", "torch")
    x0, log = run_case(name)
    np.testing.assert_allclose(x0.numpy(), G[f"sample/{name}/x0"], rtol=1e-5, atol=1e-5)
    np.testing.assert_allclose(log["log_p"].numpy(), G[f"sample/{name}/log_p"], rtol=1e-5, atol=1e-5)


@pytest.mark.parametrize("name", list(mg.CASES))
def test_guided_sample_runs_in_the_lowered_program(emulated, name):
    agent = mg.make_agent(name, CLS)
    agent.classifier.gradients = _refuse
    calls = runtime.STATS["engine_calls"]
    x0, log = run_case(name, agent)
    assert runtime.STATS["engine_calls"] == calls + 1
    assert runtime.STATS["guidance_path"] == "graph" and runtime.STATS["guidance_reason"] is None
    # fp32: summation order of the interpreter's fp64 GEMMs with fp32 stores, through every step
    np.testing.assert_allclose(x0.numpy(), G[f"sample/{name}/x0"], rtol=1e-4, atol=2e-4)
    np.testing.assert_allclose(log["log_p"].numpy(), G[f"sample/{name}/log_p"], rtol=1e-4, atol=2e-4)


@pytest.mark.parametrize("name", list(mg.CASES))
def test_other_classifiers_keep_the_callback(emulated, name):
    agent = mg.make_agent(name, CLS)
    agent.classifier = _Wrapped(agent.classifier)
    x0, log = run_case(name, agent)
    assert runtime.STATS["guidance_path"] == "callback"
    assert "classifier _Wrapped" in runtime.STATS["guidance_reason"]
    np.testing.assert_allclose(x0.numpy(), G[f"sample/{name}/x0"], rtol=1e-4, atol=2e-4)
    np.testing.assert_allclose(log["log_p"].numpy(), G[f"sample/{name}/log_p"], rtol=1e-4, atol=2e-4)


def test_guidance_moves_the_samples(emulated):
    """the goldens show the guidance: the same calls with w_cg = 0 end elsewhere"""
    for name in mg.CASES:
        x0, _ = run_case(name, w_cg=0.0)
        assert np.abs(x0.numpy() - G[f"sample/{name}/x0"]).max() > 1e-3, name


def _plans(agent):
    return list(agent._engine_plans.values())


@pytest.mark.parametrize("name", ["edm_heun_janner", "edm_euler_mlp"])
def test_edm_guidance_is_the_update_operand(emulated, name):
    """guided: the classifier reads the raw x_t and its gradient is the update's operand (no CDS_OP_GUIDE); unguided: the
    program of the parent, without the operand"""
    agent = mg.make_agent(name, CLS)
    run_case(name, agent, w_cg=0.0)
    (plain,) = _plans(agent)
    kinds = [op.kind for op in plain.program.ops]
    assert cabi.OP_GUIDE not in kinds and not any(op.u.update.guide for op in plain.program.ops if op.kind == cabi.OP_UPDATE)
    run_case(name, agent)
    guided = next(p for p in _plans(agent) if p is not plain)
    ops = guided.program.ops
    assert cabi.OP_GUIDE not in [op.kind for op in ops] and ops[-1].kind == cabi.OP_UPDATE
    u = ops[-1].u.update
    assert u.guide and u.guide_s == guided.cg_scale.data_ptr()
    # the classifier's operators read x_t itself, not CDS_OP_PREP's c_in x
    reads = {op.u.conv.in_ if op.kind == cabi.OP_CONV else op.u.cast.in_
             for op in ops[len(kinds) - 1:-1] if op.kind in (cabi.OP_CONV, cabi.OP_CAST)}
    assert guided.x.data_ptr() in reads and guided.xin.data_ptr() not in reads


@pytest.mark.parametrize("name", ["ddpm_sample_eps_janner", "ddpm_sample_x0_mlp"])
def test_legacy_guidance_is_guide_before_the_update(emulated, name):
    agent = mg.make_agent(name, CLS)
    run_case(name, agent)
    (plan,) = _plans(agent)
    kinds = [op.kind for op in plan.program.ops]
    assert kinds[-2:] == [cabi.OP_GUIDE, cabi.OP_UPDATE] and not plan.program.ops[-1].u.update.guide


def _reference_edm_columns(agent, solver, steps, w):
    """the reference's guidance scale and classifier time of every evaluation (newedm.py:229-233, :411-431), 0-d op by op"""
    from cleandiffuser_b200.diffusion.edm import karras_grid
    sig = karras_grid(steps, agent.sigma_min, agent.sigma_max, agent.rho)
    scale, time = [], []
    for i in range(steps, 0, -1):
        t = torch.full((mg.BATCH,), sig[i], dtype=torch.float32)
        scale.append(w * (sig[i] ** 2))
        time.append((t.log() / 4.)[0])
        if solver == "heun" and i > 1:
            scale.append(w * (sig[i - 1] ** 2))
            time.append(((t / sig[i] * sig[i - 1]).log() / 4.)[0])
    return torch.stack(scale), torch.stack(time)


def _reference_ddpm_scale(agent, w, extra):
    out = []
    for t in list(range(agent.diffusion_steps - 1, -1, -1)) + [0] * extra:
        ab = agent.bar_alpha[t]
        out.append(-(w * (1 - ab).sqrt()) if agent.predict_noise else w * (1 - ab) / ab.sqrt())
    return torch.stack(out)


@pytest.mark.parametrize("name", list(mg.CASES))
def test_scale_and_time_columns_are_the_reference_expressions(emulated, name, monkeypatch):
    seen = {}
    fill = runtime.SamplerPlan.fill_tables

    def recording(self, t_all, cond_emb, t_key=None, cond_cg=None, cg_t=None):
        seen["t"] = t_all if cg_t is None else cg_t
        return fill(self, t_all, cond_emb, t_key, cond_cg, cg_t)
    monkeypatch.setattr(runtime.SamplerPlan, "fill_tables", recording)
    agent = mg.make_agent(name, CLS)
    run_case(name, agent)
    (plan,) = _plans(agent)
    spec = mg.CASES[name]
    if spec["family"] == "edm":
        scale, time = _reference_edm_columns(agent, spec["solver"], spec["steps"], spec["w_cg"])
    else:
        extra = mg.EXTRA if spec["method"] == "sample_x" else 0
        scale = _reference_ddpm_scale(agent, spec["w_cg"], extra)
        time = torch.tensor(list(range(mg.T - 1, -1, -1)) + [0] * extra)
    assert torch.equal(plan.cg_scale, scale.float()), (plan.cg_scale, scale)
    assert seen["t"].dtype == time.dtype and torch.equal(seen["t"], time), (seen["t"], time)


@pytest.mark.parametrize("family", ["edm", "ddpm"])
def test_unguided_programs_are_unchanged(emulated, family):
    """w_cg = 0: no classifier operator, no guidance operand, guidance_path None"""
    name = "edm_heun_janner" if family == "edm" else "ddpm_sample_x_x0_janner"
    agent = mg.make_agent(name, CLS)
    x0, log = run_case(name, agent, w_cg=0.0)
    assert runtime.STATS["guidance_path"] is None and runtime.STATS["guidance_reason"] is None
    (plan,) = _plans(agent)
    assert plan.classifier is None and not hasattr(plan, "cg_scale")
    assert {op.kind for op in plan.program.ops} <= {cabi.OP_PREP, cabi.OP_CAST, cabi.OP_CONV, cabi.OP_UPDATE}
    assert not any(op.u.update.guide for op in plan.program.ops if op.kind == cabi.OP_UPDATE)


DECLINES = {"two_branch_cfg": ("classifier guidance together with two-branch classifier-free guidance", dict(w_cfg=0.5)),
            "preserve_history": ("classifier guidance with preserve_history=True", dict(preserve_history=True)),
            "requires_grad": ("classifier guidance with requires_grad=True", dict(requires_grad=True))}


@pytest.mark.parametrize("case", list(DECLINES))
@pytest.mark.parametrize("name", ["edm_euler_mlp", "ddpm_sample_x_eps_mlp"])
def test_declined_requests_keep_the_pytorch_loop(emulated, name, case, monkeypatch):
    reason, over = DECLINES[case]
    if case == "requires_grad":
        # requires_grad=True on these classes is a recorded fallback, as before (it raises under CDS_BACKEND=cuda)
        monkeypatch.setenv("CDS_BACKEND", "auto")
    calls = runtime.STATS["engine_calls"]
    x0, log = run_case(name, **over)
    assert runtime.STATS["engine_calls"] == calls
    assert runtime.STATS["guidance_path"] is None and runtime.STATS["guidance_reason"] == reason
    monkeypatch.setenv("CDS_BACKEND", "torch")
    want, want_log = run_case(name, **over)
    assert torch.equal(x0.detach(), want.detach()) and torch.equal(log["log_p"], want_log["log_p"])
