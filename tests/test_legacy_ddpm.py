"""The legacy ``DDPM`` class (SURVEY 8f rank 2: every dp_* / dbc_* pipeline constructs it): oracle, PyTorch path and the
engine program (same update kernel, beta-schedule coefficient table) against goldens written by the unmodified reference
(make_golden.py::gen_legacy -> legacy.npz)."""
import numpy as np
import pytest
import torch

import cases
import emulator
import oracle.sampler as osamp
from common import oracle_cond_emb, oracle_net, product_condition, product_net, tape_of
from cleandiffuser_b200.diffusion import DDPM
from cleandiffuser_b200.engine import runtime
from cleandiffuser_b200.testing import NoiseTape

NAMES = list(cases.legacy_cases())


def build(spec, device="cpu"):
    net, sd = product_net(cases.SAMPLER_NETS[spec["net"]])
    inp = cases.sampler_inputs(spec)
    agent = DDPM(net, product_condition(spec), fix_mask=inp["fix_mask"], x_max=inp["x_max"], x_min=inp["x_min"],
                 predict_noise=spec["predict_noise"], diffusion_steps=spec["T"], beta_schedule=spec["beta_schedule"], device=device)
    kw = dict(n_samples=cases.SAMPLER_BATCH, sample_steps=spec["T"], use_ema=True, temperature=spec["temperature"],
              condition_cfg=inp["cond"], w_cfg=spec["w_cfg"])
    return agent, inp, kw, sd


def run(agent, spec, prior, kw):
    if spec["extra"]:
        return agent.sample_x(prior, extra_sample_steps=spec["extra"], **kw)
    return agent.sample(prior, **kw)


@pytest.mark.parametrize("name", NAMES)
def test_oracle_legacy_ddpm_matches_reference(golden, name):
    spec = cases.legacy_cases()[name]
    case = cases.SAMPLER_NETS[spec["net"]]
    agent, inp, _, sd = build(spec)
    with torch.no_grad():
        x = osamp.sample_legacy_ddpm(oracle_net(case, sd), inp["prior"], osamp.Tape(tape_of(golden["legacy"], name)), T=spec["T"],
                                     beta=agent.beta, predict_noise=spec["predict_noise"], temperature=spec["temperature"],
                                     fix_mask=inp["fix_mask"][None] if inp["fix_mask"] is not None else 0.,
                                     cond_emb=oracle_cond_emb(spec, inp["cond"]), w_cfg=spec["w_cfg"], x_min=inp["x_min"],
                                     x_max=inp["x_max"], extra_steps=spec["extra"])
    np.testing.assert_allclose(x.numpy(), golden["legacy"][name + "/x0"], rtol=1e-5, atol=2e-4)


@pytest.mark.parametrize("name", NAMES)
def test_legacy_ddpm_torch_path_matches_reference(golden, name, monkeypatch):
    monkeypatch.setenv("CDS_BACKEND", "torch")
    spec = cases.legacy_cases()[name]
    agent, inp, kw, _ = build(spec)
    tape = NoiseTape(tape_of(golden["legacy"], name))
    with tape.active(), torch.no_grad():
        x0, log = run(agent, spec, inp["prior"], kw)
    assert tape.pos == len(tape.draws)
    np.testing.assert_allclose(x0.numpy(), golden["legacy"][name + "/x0"], rtol=1e-5, atol=2e-4)


@pytest.mark.parametrize("math", ["fp32", "tf32"])
@pytest.mark.parametrize("name", NAMES)
def test_legacy_ddpm_lowered_program(golden, name, math, monkeypatch):
    monkeypatch.setattr(runtime, "_device_ok", lambda device: True)
    owners = emulator.record_owners(monkeypatch)      # every operand is bounds-checked against its owner
    monkeypatch.setattr(runtime, "_make_handle", lambda device, ops, n: emulator.Handle(ops, n, owners()))
    monkeypatch.setenv("CDS_BACKEND", "cuda")
    monkeypatch.setenv("CDS_MATH", math)
    spec = cases.legacy_cases()[name]
    agent, inp, kw, _ = build(spec)
    calls = runtime.STATS["engine_calls"]
    tape = NoiseTape(tape_of(golden["legacy"], name))
    with tape.active(), torch.no_grad():
        x0, _ = run(agent, spec, inp["prior"], kw)
    assert runtime.STATS["engine_calls"] == calls + 1 and tape.pos == len(tape.draws)
    plan = next(iter(agent._engine_plans.values()))
    assert plan.n_iters == spec["T"] + spec["extra"]
    err = np.abs(x0.numpy() - golden["legacy"][name + "/x0"])
    if math == "fp32":
        assert err.max() < 3e-4, float(err.max())
    else:
        assert err.max() < 0.15 and err.mean() < 4e-3, (float(err.max()), float(err.mean()))


@pytest.mark.gpu
@pytest.mark.parametrize("math", ["fp32", "tf32"])
@pytest.mark.parametrize("name", NAMES)
def test_legacy_ddpm_on_the_cuda_engine(golden, name, math, monkeypatch):
    monkeypatch.setenv("CDS_BACKEND", "cuda")
    monkeypatch.setenv("CDS_MATH", math)
    dev = "cuda:0"
    spec = cases.legacy_cases()[name]
    agent, inp, kw, _ = build(spec, device=dev)
    if kw.get("condition_cfg") is not None:
        kw["condition_cfg"] = kw["condition_cfg"].to(dev)
    calls = runtime.STATS["engine_calls"]
    tape = NoiseTape(tape_of(golden["legacy"], name))
    with tape.active(), torch.no_grad():
        x0, _ = run(agent, spec, inp["prior"].to(dev), kw)
    assert runtime.STATS["engine_calls"] == calls + 1
    err = np.abs(x0.cpu().numpy() - golden["legacy"][name + "/x0"])
    if math == "fp32":
        assert err.max() < 1e-3, float(err.max())
    else:
        assert err.max() < 0.15 and err.mean() < 4e-3, (float(err.max()), float(err.mean()))


# ---------------------------------------------------------------------------------------------------------------
# the legacy EDM class (edm.py) of the dbc_* pipelines: goldens from the reference (make_golden.py::gen_legacy_edm)
from cleandiffuser_b200.diffusion import EDM  # noqa: E402

EDM_NAMES = list(cases.legacy_edm_cases())


def build_edm(spec, device="cpu"):
    net, _ = product_net(cases.SAMPLER_NETS[spec["net"]])
    inp = cases.sampler_inputs(dict(spec, clip=False))
    agent = EDM(net, product_condition(spec), fix_mask=inp["fix_mask"], device=device)
    kw = dict(n_samples=cases.SAMPLER_BATCH, sample_steps=spec["steps"], use_ema=True, solver=spec["solver"],
              condition_cfg=inp["cond"], w_cfg=spec["w_cfg"])
    return agent, inp, kw


def run_edm(agent, spec, prior, kw):
    if spec["extra"]:
        return agent.sample_x(prior, extra_sample_steps=spec["extra"], **kw)
    return agent.sample(prior, **kw)


@pytest.mark.parametrize("name", EDM_NAMES)
def test_legacy_edm_torch_path_matches_reference(golden, name, monkeypatch):
    monkeypatch.setenv("CDS_BACKEND", "torch")
    spec = cases.legacy_edm_cases()[name]
    agent, inp, kw = build_edm(spec)
    tape = NoiseTape(tape_of(golden["legacy_edm"], name))
    with tape.active(), torch.no_grad():
        x0, _ = run_edm(agent, spec, inp["prior"], kw)
    assert tape.pos == len(tape.draws)
    np.testing.assert_allclose(x0.numpy(), golden["legacy_edm"][name + "/x0"], rtol=1e-5, atol=2e-4)


@pytest.mark.parametrize("math", ["fp32", "tf32"])
@pytest.mark.parametrize("name", EDM_NAMES)
def test_legacy_edm_lowered_program(golden, name, math, monkeypatch):
    monkeypatch.setattr(runtime, "_device_ok", lambda device: True)
    owners = emulator.record_owners(monkeypatch)      # every operand is bounds-checked against its owner
    monkeypatch.setattr(runtime, "_make_handle", lambda device, ops, n: emulator.Handle(ops, n, owners()))
    monkeypatch.setenv("CDS_BACKEND", "cuda")
    monkeypatch.setenv("CDS_MATH", math)
    spec = cases.legacy_edm_cases()[name]
    agent, inp, kw = build_edm(spec)
    calls = runtime.STATS["engine_calls"]
    tape = NoiseTape(tape_of(golden["legacy_edm"], name))
    with tape.active(), torch.no_grad():
        x0, _ = run_edm(agent, spec, inp["prior"], kw)
    assert runtime.STATS["engine_calls"] == calls + 1 and tape.pos == len(tape.draws)
    err = np.abs(x0.numpy() - golden["legacy_edm"][name + "/x0"])
    ref = max(1.0, float(np.abs(golden["legacy_edm"][name + "/x0"]).mean()))
    if math == "fp32":
        assert err.max() / ref < 5e-4, float(err.max())
    else:
        assert err.max() / ref < 0.1 and err.mean() / ref < 4e-3, (float(err.max()), float(err.mean()))


@pytest.mark.gpu
@pytest.mark.parametrize("math", ["fp32", "tf32"])
@pytest.mark.parametrize("name", EDM_NAMES)
def test_legacy_edm_on_the_cuda_engine(golden, name, math, monkeypatch):
    monkeypatch.setenv("CDS_BACKEND", "cuda")
    monkeypatch.setenv("CDS_MATH", math)
    dev = "cuda:0"
    spec = cases.legacy_edm_cases()[name]
    agent, inp, kw = build_edm(spec, device=dev)
    if kw.get("condition_cfg") is not None:
        kw["condition_cfg"] = kw["condition_cfg"].to(dev)
    calls = runtime.STATS["engine_calls"]
    tape = NoiseTape(tape_of(golden["legacy_edm"], name))
    with tape.active(), torch.no_grad():
        x0, _ = run_edm(agent, spec, inp["prior"].to(dev), kw)
    assert runtime.STATS["engine_calls"] == calls + 1
    err = np.abs(x0.cpu().numpy() - golden["legacy_edm"][name + "/x0"])
    ref = max(1.0, float(np.abs(golden["legacy_edm"][name + "/x0"]).mean()))
    if math == "fp32":
        assert err.max() / ref < 2e-3, float(err.max())
    else:
        assert err.max() / ref < 0.1 and err.mean() / ref < 4e-3, (float(err.max()), float(err.mean()))
