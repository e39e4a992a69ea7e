"""TEST INFRASTRUCTURE: the MLPNNClassifier objects of tests/golden/mlp_classifier.npz -- MSEClassifier and CumRewClassifier
heads, the guided sample() cases -- and the classifier's input gradient in fp64 autograd.  Its lowered gradient
(cg_ref.lowered_gradient) uses CONV, STASH and DGRAD with ReLU, SiLU or Mish (tests/grad_ref.py; ReLU from
tests/relu_ref.py)."""
import copy

import torch

import cg_ref

ACTS = ("ReLU", "SiLU", "Mish")


def make_classifier(name, seed, device="cpu", act=None):
    """this package's classifier of golden net case ``name`` (make_golden_mlp_classifier.py) with the golden generator's
    synthetic weights; ``act`` replaces the case's hidden activation (class name)"""
    import make_golden_mlp_classifier as mg
    from cleandiffuser_b200.classifier import CumRewClassifier, MSEClassifier
    from cleandiffuser_b200.nn_classifier import MLPNNClassifier
    return mg.make_classifier(MLPNNClassifier, MSEClassifier, CumRewClassifier, name, seed, device, act)


def make_sample_agent(name, device="cpu", classifier=None):
    """(agent, prior, sample() keyword arguments) of golden sample case ``name`` (make_golden_mlp_classifier.py)"""
    import make_golden_mlp_classifier as mg
    from cleandiffuser_b200.diffusion import ContinuousDiffusionSDE, DiscreteDiffusionSDE
    from cleandiffuser_b200.nn_condition import IdentityCondition
    from cleandiffuser_b200.nn_diffusion import DQLMlp, PearceMlp
    clf = classifier if classifier is not None else make_classifier(mg.SAMPLES[name]["net"], 32, device)
    agent = mg.make_actor(name, clf, DiscreteDiffusionSDE, ContinuousDiffusionSDE, PearceMlp, DQLMlp, IdentityCondition, device)
    prior, c = mg.sample_inputs(name)
    return agent, prior.to(device), mg.sample_kwargs(name, c.to(device))


def logp_fp64(clf, x, t, c):
    """clf's logp over an fp64 copy of model_ema (the time embedding computed in fp32, as the engine's filler does)"""
    net = copy.deepcopy(clf.model_ema).double()
    net.map_noise = cg_ref.Fp64Time(clf.model_ema.map_noise)
    y = net(x, t)
    if type(clf).__name__ == "MSEClassifier":
        return -clf.temperature * ((y - c.double()) ** 2).mean(-1, keepdim=True)
    return y


def input_gradient_fp64(clf, x, t, c=None):
    """d sum(logp) / d x in fp64 autograd"""
    xx = x.detach().double().clone().requires_grad_(True)
    return torch.autograd.grad(logp_fp64(clf, xx, t, c).sum(), xx)[0]
