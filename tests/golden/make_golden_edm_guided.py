"""Generate tests/golden/edm_guided.npz by running the UNMODIFIED reference (CPU, fp32): classifier guidance in ContinuousEDM
(newedm.py:217-235) and in the legacy DDPM class (ddpm.py:117-165, ``sample`` and ``sample_x``).

    python tests/golden/make_golden_edm_guided.py [REFERENCE_CHECKOUT]
                                  # the reference must be importable as `cleandiffuser`: installed, or its checkout given

Contents (synthetic weights from ``cleandiffuser_b200.testing.synth_state_dict``, seeded inputs):
  sample/<case>/{prior, c, z<j>, n_draws, x0, log_p}   guided sample() / sample_x() calls, noise tape recorded

Two denoiser / classifier pairs: "janner" -- JannerUNet1d over (horizon 8, dim 6) trajectories guided by a CumRewClassifier over
HalfJannerUNet1d, the first step fixed by the mask; "mlp" -- DQLMlp over 6-dim actions with the observations as its condition,
guided by an MSEClassifier over MLPNNClassifier whose target is ``c``, the first action dimension fixed by the mask.  Both clip
to per-element bounds.  ContinuousEDM runs Euler and Heun; the legacy DDPM runs eps- and x0-prediction through ``sample`` and
``sample_x`` (Diffusion-X steps at t = 0, guided too).
"""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
if len(sys.argv) > 1:
    sys.path.insert(0, sys.argv[1])

from cleandiffuser_b200.testing import NoiseTape, synth_state_dict  # noqa: E402

H, D, A, OBS, BATCH, T, EXTRA = 8, 6, 6, 11, 6, 5, 2
CASES = {
    "edm_euler_janner": dict(family="edm", net="janner", solver="euler", steps=4, w_cg=0.3),
    "edm_heun_janner": dict(family="edm", net="janner", solver="heun", steps=3, w_cg=0.3),
    "edm_euler_mlp": dict(family="edm", net="mlp", solver="euler", steps=4, w_cg=0.5),
    "edm_heun_mlp": dict(family="edm", net="mlp", solver="heun", steps=3, w_cg=0.5),
    "ddpm_sample_eps_janner": dict(family="ddpm", net="janner", method="sample", predict_noise=True, w_cg=0.3),
    "ddpm_sample_x_x0_janner": dict(family="ddpm", net="janner", method="sample_x", predict_noise=False, w_cg=0.3),
    "ddpm_sample_x0_mlp": dict(family="ddpm", net="mlp", method="sample", predict_noise=False, w_cg=0.5),
    "ddpm_sample_x_eps_mlp": dict(family="ddpm", net="mlp", method="sample_x", predict_noise=True, w_cg=0.5),
}


def x_shape(net):
    return (H, D) if net == "janner" else (A,)


def sample_inputs(name):
    """(prior, c): the masked entries of the prior are seeded values; c is the MSE head's target and DQLMlp's condition"""
    net = CASES[name]["net"]
    g = torch.Generator().manual_seed(11)
    prior = torch.zeros(BATCH, *x_shape(net))
    if net == "janner":
        prior[:, 0] = torch.randn(BATCH, D, generator=g)
    else:
        prior[:, 0] = torch.randn(BATCH, generator=g)
    return prior, torch.randn(BATCH, OBS, generator=g)


def agent_parts(net):
    """(fix_mask, x_min, x_max) of a denoiser pair"""
    g = torch.Generator().manual_seed(7)
    shape = x_shape(net)
    mask = torch.zeros(shape)
    mask[0] = 1.                                     # the first step of a trajectory / the first action dimension
    x_max = 0.8 + 0.7 * torch.rand(shape, generator=g)
    return mask, -x_max.clone(), x_max


def make_classifier(net, cls, device="cpu"):
    """the case's classifier from the classes ``cls`` (a dict of the reference's or this package's classes)"""
    if net == "janner":
        m = cls["HalfJannerUNet1d"](H, D, out_dim=1, model_dim=16, emb_dim=16, dim_mult=[1, 2])
        m.load_state_dict(synth_state_dict(m.state_dict(), 32))
        return cls["CumRewClassifier"](m, device=device)
    m = cls["MLPNNClassifier"](A, OBS, 32, [64, 64], activation=torch.nn.SiLU())
    m.load_state_dict(synth_state_dict(m.state_dict(), 32))
    return cls["MSEClassifier"](m, temperature=1.0, device=device)


def make_agent(name, cls, classifier=None, device="cpu"):
    spec = CASES[name]
    net = spec["net"]
    mask, x_min, x_max = agent_parts(net)
    if net == "janner":
        den = cls["JannerUNet1d"](D, model_dim=16, emb_dim=16, dim_mult=[1, 2])
        cond = None
    else:
        den = cls["DQLMlp"](obs_dim=OBS, act_dim=A)
        cond = cls["IdentityCondition"](dropout=0.0)
    den.load_state_dict(synth_state_dict(den.state_dict(), 21))
    clf = classifier if classifier is not None else make_classifier(net, cls, device)
    common = dict(fix_mask=mask, classifier=clf, x_min=x_min, x_max=x_max, device=device)
    if spec["family"] == "edm":
        agent = cls["ContinuousEDM"](den, cond, **common)
    else:
        agent = cls["DDPM"](den, cond, diffusion_steps=T, predict_noise=spec["predict_noise"], **common)
    agent.eval()
    return agent


def sample_call(name, agent, prior, c):
    """(method, keyword arguments) of the case's guided call"""
    spec = CASES[name]
    kw = dict(n_samples=BATCH, w_cg=spec["w_cg"], temperature=0.8,
              condition_cg=torch.zeros(BATCH, 1, device=c.device) if spec["net"] == "janner" else c)
    if spec["net"] == "mlp":
        kw.update(condition_cfg=c, w_cfg=1.0)
    if spec["family"] == "edm":
        kw.update(solver=spec["solver"], sample_steps=spec["steps"])
        return agent.sample, kw
    kw.update(sample_steps=T)
    if spec["method"] == "sample_x":
        kw.update(extra_sample_steps=EXTRA)
    return getattr(agent, spec["method"]), kw


def reference_classes():
    from cleandiffuser.classifier import CumRewClassifier, MSEClassifier
    from cleandiffuser.diffusion.ddpm import DDPM
    from cleandiffuser.diffusion.newedm import ContinuousEDM
    from cleandiffuser.nn_classifier import HalfJannerUNet1d, MLPNNClassifier
    from cleandiffuser.nn_condition import IdentityCondition
    from cleandiffuser.nn_diffusion import DQLMlp, JannerUNet1d
    return dict(CumRewClassifier=CumRewClassifier, MSEClassifier=MSEClassifier, DDPM=DDPM, ContinuousEDM=ContinuousEDM,
                HalfJannerUNet1d=HalfJannerUNet1d, MLPNNClassifier=MLPNNClassifier, IdentityCondition=IdentityCondition,
                DQLMlp=DQLMlp, JannerUNet1d=JannerUNet1d)


def main():
    cls = reference_classes()
    out = {}
    for k, name in enumerate(CASES):
        torch.manual_seed(100 + k)                       # the loop's torch.randn_like draws (recorded on the noise tape)
        agent = make_agent(name, cls)
        prior, c = sample_inputs(name)
        fn, kw = sample_call(name, agent, prior, c)
        tape = NoiseTape()
        with tape.active():
            x0, log = fn(prior.clone(), **kw)
        out[f"sample/{name}/prior"], out[f"sample/{name}/c"] = prior.numpy(), c.numpy()
        out[f"sample/{name}/x0"], out[f"sample/{name}/log_p"] = x0.detach().numpy(), log["log_p"].detach().numpy()
        for j, z in enumerate(tape.draws):
            out[f"sample/{name}/z{j}"] = z.numpy()
        out[f"sample/{name}/n_draws"] = np.array(len(tape.draws))
    np.savez_compressed(os.path.join(HERE, "edm_guided.npz"), **out)
    print("edm_guided.npz", len(out))


if __name__ == "__main__":
    main()
