"""TEST INFRASTRUCTURE: the QGPO objects of tests/golden/qgpo.npz -- QGPOClassifier at the D4RL MuJoCo shapes, the guided
sample() cases -- and QGPONNClassifier's input gradient in fp64 autograd.  Its lowered gradient (cg_ref.lowered_gradient)
uses STASH and DGRAD with SiLU (tests/grad_ref.py) and HEAD_GRAD (tests/cg_ref.py)."""
import torch

import cg_ref


# ---------------------------------------------------------------- the objects of tests/golden/qgpo.npz
# QGPO's classifier at the D4RL MuJoCo shapes (obs_dim, act_dim)
PIPELINES = {"hopper": dict(obs_dim=11, act_dim=3), "walker": dict(obs_dim=17, act_dim=6),
             "halfcheetah": dict(obs_dim=17, act_dim=6)}


def make_classifier(kw, seed, device="cpu"):
    """this package's QGPOClassifier over QGPONNClassifier with the golden generator's synthetic weights"""
    import make_golden_qgpo as mg
    from cleandiffuser_b200.classifier import QGPOClassifier
    from cleandiffuser_b200.nn_classifier import QGPONNClassifier
    return mg.make_classifier(QGPONNClassifier, QGPOClassifier, kw, seed, device)


def make_sample_agent(name, device="cpu", classifier=None):
    """(agent, prior, sample() keyword arguments) of golden sample case ``name`` (make_golden_qgpo.py)"""
    import make_golden_qgpo as mg
    from cleandiffuser_b200.diffusion import ContinuousDiffusionSDE
    from cleandiffuser_b200.nn_condition import MLPCondition
    from cleandiffuser_b200.nn_diffusion import SfBCUNet
    clf = classifier if classifier is not None else make_classifier(dict(obs_dim=mg.OBS, act_dim=mg.ACT), 32, device)
    agent = mg.make_actor(ContinuousDiffusionSDE, SfBCUNet, MLPCondition, mg.SAMPLES[name]["predict_noise"], clf, device)
    prior, obs = mg.sample_inputs()
    return agent, prior.to(device), mg.sample_kwargs(name, obs.to(device))


def input_gradient_fp64(clf, x, t, obs):
    """d sum(logp) / d x of clf.model_ema in fp64 autograd (the Fourier features computed in fp32, as the engine's filler does)"""
    import copy
    net = copy.deepcopy(clf.model_ema).double()
    net.map_noise = cg_ref.Fp64Time(clf.model_ema.map_noise)
    xx = x.detach().double().clone().requires_grad_(True)
    lp = net(xx, t, obs.double())
    return torch.autograd.grad(lp.sum(), xx)[0]
