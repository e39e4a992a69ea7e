"""Helpers shared by the parity tests: build product modules / oracle closures for a golden case."""
import os

import numpy as np
import torch

import cases
import oracle.nets as onets
from cleandiffuser_b200 import nn_condition as pcond
from cleandiffuser_b200 import nn_diffusion as pnn
from cleandiffuser_b200.testing import synth_state_dict


def product_net(case, seed=0):
    net = getattr(pnn, case["cls"])(**case["ctor"])
    sd = synth_state_dict(net.state_dict(), seed=seed)
    net.load_state_dict(sd)
    return net.eval(), sd


def oracle_net(case, sd):
    kw = dict(case["oracle"])
    fn = getattr(onets, kw.pop("fn"))
    return lambda x, t, cond=None: fn(sd, x, t, cond, **kw)


def product_condition(spec):
    if spec["cond"] == "mlp":
        nc = pcond.MLPCondition(1, 8, [8], torch.nn.SiLU(), dropout=0.25)
        nc.load_state_dict(synth_state_dict(nc.state_dict(), seed=3))
        return nc
    if spec["cond"] in ("obs", "emb"):
        return pcond.IdentityCondition(dropout=0.0)
    return None


def oracle_cond_emb(spec, cond):
    if cond is None:
        return None
    if spec["cond"] == "mlp":
        nc = pcond.MLPCondition(1, 8, [8], torch.nn.SiLU(), dropout=0.25)   # template for shapes only
        sd = synth_state_dict(nc.state_dict(), seed=3)
        return onets.mlp_condition(sd, cond, torch.nn.functional.silu, 1)
    return cond * 1.


def load_golden(name):
    """tests/golden/<name>.npz"""
    return np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", name + ".npz"), allow_pickle=False)


def tape_of(npz, name):
    n = int(npz[name + "/n_draws"])
    return [npz[f"{name}/z{j}"] for j in range(n)]


# ---------------------------------------------------------------- BASELINE configs (cleandiffuser_b200/workloads.py)
def workload_oracle(wl, prior, cond, draws):
    """The CPU oracle's result for the workload's computation on ``prior`` / ``cond`` (a slice of the batch) with the noise
    draws ``draws`` (list of arrays, already sliced).  Resolves the plain-data ``wl.oracle`` description."""
    import oracle.sampler as osamp
    spec = wl.oracle
    net_kw = dict(spec["net"])
    net_fn = getattr(onets, net_kw.pop("fn"))
    model = wl.agent.model_ema if hasattr(wl.agent, "model_ema") else wl.agent.model
    sd = {k: v.detach().cpu().clone() for k, v in model["diffusion"].state_dict().items()}
    fn = lambda x, t, c=None: net_fn(sd, x, t, c, **net_kw)   # noqa: E731
    cond_emb = None
    if cond is not None:
        cspec = spec.get("cond")
        if cspec is None:
            cond_emb = cond * 1.
        else:
            csd = {k: v.detach().cpu().clone() for k, v in model["condition"].state_dict().items()}
            act = {"silu": torch.nn.functional.silu}[cspec["act"]]
            cond_emb = getattr(onets, cspec["fn"])(csd, cond, act, cspec["n_hidden"])
    with torch.no_grad():
        return getattr(osamp, spec["sampler"])(fn, prior, osamp.Tape(draws), fix_mask=spec["fix_mask"], cond_emb=cond_emb,
                                               **spec["kwargs"])
