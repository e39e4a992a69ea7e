"""Classifier-guided sampling (SURVEY 8a row a7 / 8f-1): ``sample(w_cg != 0)`` with a classifier attached, against goldens
written by the unmodified reference with the same toy classifier (make_golden.py::gen_guided -> guided.npz).

On the engine the loop runs step by step through the single-step entry (cds_plan_run_range): denoiser operators -> PyTorch
adds ``w_cg * sigma [* sigma / alpha] * grad log p`` to the prediction in place -> update operator; the classifier's forward and
input gradient stay PyTorch autograd.  The pipeline this mirrors: pipelines/diffuser_d4rl_mujoco.py:136-141 (w_cg = 0.3)."""
import numpy as np
import pytest
import torch

import cases
import emulator
from common import product_condition, product_net, tape_of
from cleandiffuser_b200.diffusion import ContinuousDiffusionSDE, DiscreteDiffusionSDE
from cleandiffuser_b200.engine import runtime
from cleandiffuser_b200.testing import NoiseTape, ToyClassifier

NAMES = list(cases.guided_cases())


def build(spec, device="cpu"):
    ncase = cases.SAMPLER_NETS[spec["net"]]
    net, _ = product_net(ncase)
    inp = cases.sampler_inputs(spec)
    common = dict(nn_condition=product_condition(spec), fix_mask=inp["fix_mask"], x_max=inp["x_max"], x_min=inp["x_min"],
                  predict_noise=spec["predict_noise"], device=device, noise_schedule=spec.get("schedule", "cosine"),
                  classifier=ToyClassifier(ncase["x"], device=device))
    if spec["kind"] == "discrete":
        agent, sched = DiscreteDiffusionSDE(net, diffusion_steps=spec["T"], **common), "uniform"
    else:
        agent, sched = ContinuousDiffusionSDE(net, **common), "uniform_continuous"
    kw = dict(solver=spec["solver"], n_samples=cases.SAMPLER_BATCH, sample_steps=spec["steps"], sample_step_schedule=sched,
              use_ema=True, temperature=spec["temperature"], condition_cfg=inp["cond"], w_cfg=spec["w_cfg"], w_cg=spec["w_cg"])
    return agent, inp, kw


@pytest.mark.parametrize("name", NAMES)
def test_guided_torch_path_matches_reference(golden, name, monkeypatch):
    monkeypatch.setenv("CDS_BACKEND", "torch")
    agent, inp, kw = build(cases.guided_cases()[name])
    tape = NoiseTape(tape_of(golden["guided"], name))
    with tape.active():
        x0, log = agent.sample(inp["prior"], **kw)
    assert tape.pos == len(tape.draws)
    np.testing.assert_allclose(x0.detach().numpy(), golden["guided"][name + "/x0"], rtol=1e-5, atol=2e-4)
    np.testing.assert_allclose(log["log_p"].detach().numpy(), golden["guided"][name + "/log_p"], rtol=1e-4, atol=2e-4)


@pytest.mark.parametrize("math", ["fp32", "tf32"])
@pytest.mark.parametrize("name", NAMES)
def test_guided_sampling_on_the_lowered_engine_program(golden, name, math, monkeypatch):
    monkeypatch.setattr(runtime, "_device_ok", lambda device: True)
    owners = emulator.record_owners(monkeypatch)      # every operand is bounds-checked against its owner
    monkeypatch.setattr(runtime, "_make_handle", lambda device, ops, n: emulator.Handle(ops, n, owners()))
    monkeypatch.setenv("CDS_BACKEND", "cuda")            # a fallback to the PyTorch loop raises
    monkeypatch.setenv("CDS_MATH", math)
    agent, inp, kw = build(cases.guided_cases()[name])
    calls, fb = runtime.STATS["engine_calls"], runtime.STATS["fallbacks"]
    tape = NoiseTape(tape_of(golden["guided"], name))
    with tape.active():
        x0, log = agent.sample(inp["prior"], **kw)
    assert runtime.STATS["engine_calls"] == calls + 1 and runtime.STATS["fallbacks"] == fb
    assert tape.pos == len(tape.draws)
    err = np.abs(x0.detach().numpy() - golden["guided"][name + "/x0"])
    if math == "fp32":
        assert err.max() < 3e-4, float(err.max())
        np.testing.assert_allclose(log["log_p"].detach().numpy(), golden["guided"][name + "/log_p"], rtol=1e-3, atol=1e-3)
    else:
        # (toy 8-channel nets with clipping: an element may sit on the other side of a clip decision -> isolated outliers)
        assert err.max() < 0.15 and err.mean() < 3e-3, (float(err.max()), float(err.mean()))


@pytest.mark.gpu
@pytest.mark.parametrize("math", ["fp32", "tf32"])
@pytest.mark.parametrize("name", NAMES)
def test_guided_sampling_on_the_cuda_engine(golden, name, math, monkeypatch):
    monkeypatch.setenv("CDS_BACKEND", "cuda")
    monkeypatch.setenv("CDS_MATH", math)
    dev = "cuda:0"
    agent, inp, kw = build(cases.guided_cases()[name], device=dev)
    if kw.get("condition_cfg") is not None:
        kw["condition_cfg"] = kw["condition_cfg"].to(dev)
    calls, fb = runtime.STATS["engine_calls"], runtime.STATS["fallbacks"]
    tape = NoiseTape(tape_of(golden["guided"], name))
    with tape.active():
        x0, log = agent.sample(inp["prior"].to(dev), **kw)
    assert runtime.STATS["engine_calls"] == calls + 1 and runtime.STATS["fallbacks"] == fb
    err = np.abs(x0.detach().cpu().numpy() - golden["guided"][name + "/x0"])
    if math == "fp32":
        assert err.max() < 1e-3, float(err.max())
        np.testing.assert_allclose(log["log_p"].detach().cpu().numpy(), golden["guided"][name + "/log_p"], rtol=2e-3, atol=2e-3)
    else:
        # (toy 8-channel nets with clipping: an element may sit on the other side of a clip decision -> isolated outliers)
        assert err.max() < 0.15 and err.mean() < 3e-3, (float(err.max()), float(err.mean()))
