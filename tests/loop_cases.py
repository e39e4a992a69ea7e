"""TEST INFRASTRUCTURE: one golden case of every sampler family, built the way its own tests build it, for the loop-driver
tests (tests/test_loop_drivers_cpu.py, tests/test_loop_drivers_gpu.py), and the tolerances those tests state.

``golden_case(family, device)`` -> ``(agent, prior, run, draws, want)``: ``run(prior)`` is the family's ``sample()`` call and
returns x0 (inside the caller's ``NoiseTape``), ``draws`` the case's recorded noise tape, ``want`` its golden x0."""
import numpy as np
import torch

import cases
import cg_ref
import qgpo_ref
import test_edm
import test_guided
import test_legacy_ddpm
import test_rectifiedflow
from common import load_golden, product_net, tape_of
from test_host_golden import build_agent
from cleandiffuser_b200.diffusion import ContinuousConsistencyModel
from cleandiffuser_b200.nn_condition import IdentityCondition

# family -> (golden file, case name)
GOLDEN = {"ddpm": ("samplers", "disc_dup_ddpm_x0"), "sde_2m": ("samplers", "disc_dx_sde_dpmsolverpp_2M_eps"),
          "cfg2": ("samplers", "disc_cfg2branch_ddpm"), "consistency": ("consistency", "cm3"),
          "edm_heun": ("edm", "edm_heun_mask_clip_dx"), "legacy": ("legacy", "ddpm_x_eps_extra"),
          "legacy_edm": ("legacy_edm", "ledm_heun_cfg2branch_x"), "rf": ("rf", "rf_disc_cond_clip_dx"),
          "cg_graph": ("classifier", "discrete_ddpm_eps"), "qgpo": ("qgpo", "ddpm_eps"),
          "cg_callback": ("guided", "cg_disc_ddpm_x0")}


def _frac_allclose(rtol, atol):
    return lambda got, want: float((np.abs(got - want) / (atol + rtol * np.abs(want))).max())


def _frac_max(tol):
    return lambda got, want: float(np.abs(got - want).max() / tol)


def _frac_rel_max(tol):
    return lambda got, want: float(np.abs(got - want).max() / max(1.0, float(np.abs(want).mean())) / tol)


# the fp32 tolerance each golden file's interpreter test and GPU test state, as ``fraction(got, want)`` (<= 1 passes)
INTERP_TOL = {"samplers": _frac_allclose(1e-4, 3e-4), "consistency": _frac_allclose(1e-4, 3e-4), "edm": _frac_max(3e-4),
              "legacy": _frac_max(3e-4), "legacy_edm": _frac_rel_max(5e-4), "rf": _frac_max(3e-4),
              "classifier": _frac_max(3e-4), "qgpo": _frac_max(3e-4), "guided": _frac_max(3e-4)}
GPU_TOL = {"samplers": _frac_allclose(1e-3, 1e-3), "consistency": _frac_allclose(1e-3, 1e-3), "edm": _frac_max(1e-3),
           "legacy": _frac_max(1e-3), "legacy_edm": _frac_rel_max(2e-3), "rf": _frac_max(1e-3),
           "classifier": _frac_max(1e-3), "qgpo": _frac_max(1e-3), "guided": _frac_max(1e-3)}


def _dev(kw, device, keys=("condition_cfg", "condition_cg", "warm_start_reference")):
    for k in keys:
        if kw.get(k) is not None:
            kw[k] = kw[k].to(device)
    return kw


def golden_case(family, device="cpu", golden=None):
    file, name = GOLDEN[family]
    g = golden[file] if golden is not None and file in golden else load_golden(file)
    key = f"sample/{name}" if file in ("classifier", "qgpo") else name
    draws, want = tape_of(g, key), g[key + "/x0"]
    if file == "samplers":
        agent, inp, kw = build_agent(cases.sampler_cases()[name], device=device)
        return agent, inp["prior"].to(device), lambda p: agent.sample(p, **_dev(kw, device))[0], draws, want
    if file == "consistency":
        net, _ = product_net(cases.NETS["chi_cm_fourier"])
        agent = ContinuousConsistencyModel(net, IdentityCondition(dropout=0.0), x_max=torch.ones(1, 8, 3),
                                           x_min=-torch.ones(1, 8, 3), device=device)
        cond = torch.as_tensor(g[f"{name}/cond"]).to(device)
        steps = int(name[2:])
        return agent, torch.zeros(4, 8, 3, device=device), \
            lambda p: agent.sample(p, n_samples=p.shape[0], sample_steps=steps, condition_cfg=cond, w_cfg=1.0)[0], draws, want
    if file == "edm":
        agent, inp, kw, _ = test_edm.build_edm(cases.edm_cases()[name], device=device)
        return agent, inp["prior"].to(device), lambda p: agent.sample(p, **_dev(kw, device))[0], draws, want
    if file == "legacy":
        spec = cases.legacy_cases()[name]
        agent, inp, kw, _ = test_legacy_ddpm.build(spec, device=device)
        return agent, inp["prior"].to(device), lambda p: test_legacy_ddpm.run(agent, spec, p, _dev(kw, device))[0], draws, want
    if file == "legacy_edm":
        spec = cases.legacy_edm_cases()[name]
        agent, inp, kw = test_legacy_ddpm.build_edm(spec, device=device)
        return agent, inp["prior"].to(device), lambda p: test_legacy_ddpm.run_edm(agent, spec, p, _dev(kw, device))[0], draws, want
    if file == "rf":
        agent, inp, kw = test_rectifiedflow.build(cases.rf_cases()[name], device=device)
        return agent, inp["prior"].to(device), lambda p: agent.sample(p, **_dev(kw, device))[0], draws, want
    if file in ("classifier", "qgpo"):
        agent, prior, kw = (cg_ref if file == "classifier" else qgpo_ref).make_sample_agent(name, device=device)
        return agent, prior, lambda p: agent.sample(p, **kw)[0].detach(), draws, want
    assert file == "guided"
    agent, inp, kw = test_guided.build(cases.guided_cases()[name], device=device)
    return agent, inp["prior"].to(device), lambda p: agent.sample(p, **_dev(kw, device))[0].detach(), draws, want


def tape_mb(slots, prior):
    """the CDS_NOISE_TAPE_MB that holds exactly ``slots`` draws of x_t shaped like ``prior`` (a power-of-two quotient: exact)"""
    return repr(slots * 4 * prior.numel() / 2 ** 20)
