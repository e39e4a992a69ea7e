"""Rectified flow (SURVEY 8f rank 3): product PyTorch path and the engine program (Euler step = the update kernel with
K0 = 1, K1 = -dt) against goldens written by the unmodified reference (make_golden.py::gen_rf -> rf.npz)."""
import numpy as np
import pytest
import torch

import cases
import emulator
from common import product_condition, product_net, tape_of
from cleandiffuser_b200.diffusion import ContinuousRectifiedFlow, DiscreteRectifiedFlow
from cleandiffuser_b200.engine import runtime
from cleandiffuser_b200.testing import NoiseTape

NAMES = list(cases.rf_cases())


def build(spec, device="cpu"):
    net, _ = product_net(cases.SAMPLER_NETS[spec["net"]])
    inp = cases.sampler_inputs(spec)
    common = dict(nn_condition=product_condition(spec), fix_mask=inp["fix_mask"], x_max=inp["x_max"], x_min=inp["x_min"], device=device)
    if spec["kind"] == "discrete":
        agent, sched = DiscreteRectifiedFlow(net, diffusion_steps=spec["T"], **common), spec.get("step_schedule", "uniform")
    else:
        agent, sched = ContinuousRectifiedFlow(net, **common), spec.get("step_schedule", "uniform_continuous")
    kw = dict(n_samples=cases.SAMPLER_BATCH, sample_steps=spec["steps"], sample_step_schedule=sched, use_ema=True,
              temperature=spec["temperature"], condition_cfg=inp["cond"], w_cfg=spec["w_cfg"],
              diffusion_x_sampling_steps=spec.get("diffusion_x", 0))
    if inp["warm"] is not None:
        kw.update(warm_start_reference=inp["warm"], warm_start_forward_level=spec["warm"])
    return agent, inp, kw


@pytest.mark.parametrize("name", NAMES)
def test_rf_torch_path_matches_reference(golden, name, monkeypatch):
    monkeypatch.setenv("CDS_BACKEND", "torch")
    agent, inp, kw = build(cases.rf_cases()[name])
    tape = NoiseTape(tape_of(golden["rf"], name))
    with tape.active(), torch.no_grad():
        x0, _ = agent.sample(inp["prior"], **kw)
    assert tape.pos == len(tape.draws)
    np.testing.assert_allclose(x0.numpy(), golden["rf"][name + "/x0"], rtol=1e-5, atol=2e-4)


@pytest.mark.parametrize("math", ["fp32", "tf32"])
@pytest.mark.parametrize("name", NAMES)
def test_rf_lowered_program(golden, name, math, monkeypatch):
    monkeypatch.setattr(runtime, "_device_ok", lambda device: True)
    owners = emulator.record_owners(monkeypatch)      # every operand is bounds-checked against its owner
    monkeypatch.setattr(runtime, "_make_handle", lambda device, ops, n: emulator.Handle(ops, n, owners()))
    monkeypatch.setenv("CDS_BACKEND", "cuda")
    monkeypatch.setenv("CDS_MATH", math)
    agent, inp, kw = build(cases.rf_cases()[name])
    calls = runtime.STATS["engine_calls"]
    tape = NoiseTape(tape_of(golden["rf"], name))
    with tape.active(), torch.no_grad():
        x0, _ = agent.sample(inp["prior"], **kw)
    assert runtime.STATS["engine_calls"] == calls + 1 and tape.pos == len(tape.draws)
    err = np.abs(x0.numpy() - golden["rf"][name + "/x0"])
    if math == "fp32":
        assert err.max() < 3e-4, float(err.max())
    else:
        assert err.max() < 0.1 and err.mean() < 4e-3, (float(err.max()), float(err.mean()))


@pytest.mark.gpu
@pytest.mark.parametrize("math", ["fp32", "tf32"])
@pytest.mark.parametrize("name", NAMES)
def test_rf_on_the_cuda_engine(golden, name, math, monkeypatch):
    monkeypatch.setenv("CDS_BACKEND", "cuda")
    monkeypatch.setenv("CDS_MATH", math)
    dev = "cuda:0"
    agent, inp, kw = build(cases.rf_cases()[name], device=dev)
    for k in ("condition_cfg", "warm_start_reference"):
        if kw.get(k) is not None:
            kw[k] = kw[k].to(dev)
    calls = runtime.STATS["engine_calls"]
    tape = NoiseTape(tape_of(golden["rf"], name))
    with tape.active(), torch.no_grad():
        x0, _ = agent.sample(inp["prior"].to(dev), **kw)
    assert runtime.STATS["engine_calls"] == calls + 1
    err = np.abs(x0.cpu().numpy() - golden["rf"][name + "/x0"])
    if math == "fp32":
        assert err.max() < 1e-3, float(err.max())
    else:
        assert err.max() < 0.1 and err.mean() < 4e-3, (float(err.max()), float(err.mean()))
