"""ContinuousEDM (SURVEY 8a row a12): oracle, product PyTorch path and the lowered engine program against goldens written by
the unmodified reference (tests/golden/make_golden.py::gen_edm -> edm.npz); the CUDA kernels follow under ``-m gpu``."""
import numpy as np
import pytest
import torch

import cases
import emulator
import oracle.sampler as osamp
from common import oracle_cond_emb, oracle_net, product_condition, product_net, tape_of
from cleandiffuser_b200.diffusion import ContinuousEDM
from cleandiffuser_b200.engine import runtime
from cleandiffuser_b200.testing import NoiseTape

NAMES = list(cases.edm_cases())


def build_edm(spec, device="cpu"):
    net, sd = product_net(cases.SAMPLER_NETS[spec["net"]])
    inp = cases.sampler_inputs(spec)
    agent = ContinuousEDM(net, product_condition(spec), fix_mask=inp["fix_mask"], x_max=inp["x_max"], x_min=inp["x_min"],
                          device=device)
    kw = dict(solver=spec["solver"], n_samples=cases.SAMPLER_BATCH, sample_steps=spec["steps"], use_ema=True,
              temperature=spec["temperature"], condition_cfg=inp["cond"], w_cfg=spec["w_cfg"],
              diffusion_x_sampling_steps=spec.get("diffusion_x", 0))
    if inp["warm"] is not None:
        kw.update(warm_start_reference=inp["warm"], warm_start_forward_level=spec["warm"])
    return agent, inp, kw, sd


@pytest.mark.parametrize("name", NAMES)
def test_oracle_edm_matches_reference(golden, name):
    spec = cases.edm_cases()[name]
    case = cases.SAMPLER_NETS[spec["net"]]
    _, sd = product_net(case)
    inp = cases.sampler_inputs(spec)
    with torch.no_grad():
        x = osamp.sample_edm(oracle_net(case, sd), inp["prior"], osamp.Tape(tape_of(golden["edm"], name)), steps=spec["steps"],
                             solver=spec["solver"], temperature=spec["temperature"],
                             fix_mask=inp["fix_mask"][None] if inp["fix_mask"] is not None else 0.,
                             cond_emb=oracle_cond_emb(spec, inp["cond"]), w_cfg=spec["w_cfg"], x_min=inp["x_min"],
                             x_max=inp["x_max"], diffusion_x=spec.get("diffusion_x", 0), warm_start=inp["warm"],
                             warm_level=spec.get("warm", 0.3))
    np.testing.assert_allclose(x.numpy(), golden["edm"][name + "/x0"], rtol=1e-5, atol=2e-4)


@pytest.mark.parametrize("name", NAMES)
def test_edm_torch_path_matches_reference(golden, name, monkeypatch):
    monkeypatch.setenv("CDS_BACKEND", "torch")
    agent, inp, kw, _ = build_edm(cases.edm_cases()[name])
    tape = NoiseTape(tape_of(golden["edm"], name))
    with tape.active(), torch.no_grad():
        x0, log = agent.sample(inp["prior"], **kw)
    assert tape.pos == len(tape.draws) and log["sample_history"] is None
    np.testing.assert_allclose(x0.numpy(), golden["edm"][name + "/x0"], rtol=1e-5, atol=2e-4)



@pytest.mark.parametrize("math", ["fp32", "tf32"])
@pytest.mark.parametrize("name", NAMES)
def test_lowered_edm_program(golden, name, math, monkeypatch):
    """The engine program of ContinuousEDM.sample (PREP -> denoiser -> CDS_UPD_EDM / _HEUN per network evaluation) on the
    numpy interpreter of the ABI."""
    monkeypatch.setattr(runtime, "_device_ok", lambda device: True)
    owners = emulator.record_owners(monkeypatch)      # every operand is bounds-checked against its owner
    monkeypatch.setattr(runtime, "_make_handle", lambda device, ops, n: emulator.Handle(ops, n, owners()))
    monkeypatch.setenv("CDS_BACKEND", "cuda")
    monkeypatch.setenv("CDS_MATH", math)
    spec = cases.edm_cases()[name]
    agent, inp, kw, _ = build_edm(spec)
    before = runtime.STATS["engine_calls"]
    tape = NoiseTape(tape_of(golden["edm"], name))
    with tape.active(), torch.no_grad():
        x0, _ = agent.sample(inp["prior"], **kw)
    assert runtime.STATS["engine_calls"] == before + 1
    plan = next(iter(agent._engine_plans.values()))
    order = [1] * spec.get("diffusion_x", 0) + list(range(1, spec["steps"] + 1))
    assert plan.n_iters == sum(2 if (spec["solver"] == "heun" and i > 1) else 1 for i in order)    # network evaluations
    err = np.abs(x0.numpy() - golden["edm"][name + "/x0"])
    if math == "fp32":
        assert err.max() < 3e-4, float(err.max())
    else:
        assert err.max() < (0.1 if spec["w_cfg"] not in (0.0, 1.0) else 2e-2) and err.mean() < 4e-3, (float(err.max()), float(err.mean()))


@pytest.mark.gpu
@pytest.mark.parametrize("math", ["fp32", "tf32"])
@pytest.mark.parametrize("name", NAMES)
def test_edm_on_the_cuda_engine(golden, name, math, monkeypatch):
    monkeypatch.setenv("CDS_BACKEND", "cuda")
    monkeypatch.setenv("CDS_MATH", math)
    dev = "cuda:0"
    spec = cases.edm_cases()[name]
    agent, inp, kw, _ = build_edm(spec, device=dev)
    for k in ("condition_cfg", "warm_start_reference"):
        if kw.get(k) is not None:
            kw[k] = kw[k].to(dev)
    before = runtime.STATS["engine_calls"]
    tape = NoiseTape(tape_of(golden["edm"], name))
    with tape.active(), torch.no_grad():
        x0, _ = agent.sample(inp["prior"].to(dev), **kw)
    assert runtime.STATS["engine_calls"] == before + 1
    err = np.abs(x0.cpu().numpy() - golden["edm"][name + "/x0"])
    if math == "fp32":
        assert err.max() < 1e-3, float(err.max())
    else:
        assert err.max() < (0.1 if spec["w_cfg"] not in (0.0, 1.0) else 2e-2) and err.mean() < 4e-3, (float(err.max()), float(err.mean()))


def test_consistency_distillation_from_an_edm_teacher():
    """ContinuousConsistencyModel.prepare_distillation / update(loss_type="distillation") with a ContinuousEDM teacher
    (consistency_model.py:200-239, :264-293; tutorials/sp_consistency_policy.py:216,290): the capability the EDM class unlocks."""
    from cleandiffuser_b200.diffusion import ContinuousConsistencyModel
    from cleandiffuser_b200.nn_condition import IdentityCondition
    case = cases.NETS["chi_cm_fourier"]
    net_t, _ = product_net(case)
    net_s, _ = product_net(case, seed=1)
    kw = dict(x_max=torch.ones(1, 8, 3), x_min=-torch.ones(1, 8, 3), device="cpu")
    edm = ContinuousEDM(net_t, IdentityCondition(dropout=0.0), **kw)
    log = edm.update(torch.randn(4, 8, 3) * 0.3, torch.randn(4, 2, 5))
    assert np.isfinite(log["loss"])
    cm = ContinuousConsistencyModel(net_s, IdentityCondition(dropout=0.0), **kw)
    cm.prepare_distillation(edm, distillation_N=6)
    for a, b in zip(cm.model.parameters(), edm.model.parameters()):
        assert torch.equal(a, b)                                   # student initialised from the teacher
    before = [p.clone() for p in cm.model.parameters()]
    log = cm.update(torch.randn(4, 8, 3) * 0.3, torch.randn(4, 2, 5), loss_type="distillation")
    assert np.isfinite(log["loss"]) and any(not torch.equal(a, b) for a, b in zip(before, cm.model.parameters()))
    x0, _ = cm.sample(torch.zeros(4, 8, 3), n_samples=4, sample_steps=2, condition_cfg=torch.randn(4, 2, 5), w_cfg=1.0)
    assert x0.shape == (4, 8, 3) and float(x0.abs().max()) <= 1.0
