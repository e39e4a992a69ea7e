"""Generate tests/golden/mlp_classifier.npz by running the UNMODIFIED reference (CPU, fp32): MSEClassifier and CumRewClassifier
over MLPNNClassifier.

    python tests/golden/make_golden_mlp_classifier.py [REFERENCE_CHECKOUT]
                                  # the reference must be importable as `cleandiffuser`: installed, or its checkout given

Contents (synthetic weights from ``cleandiffuser_b200.testing.synth_state_dict``, seeded inputs):
  net/<case>/{x, t, c, logp, grad}   logp and input gradient (clf.gradients) at discrete times
  sample/<case>/{prior, c, z<j>, n_draws, x0, log_p}   guided sample() calls, noise tape recorded
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

# The classifier-guidance tutorial's classifier (tutorials/3_classifier_guidance.py): MSEClassifier over
# MLPNNClassifier(x_dim=act_dim, out_dim=obs_dim, emb_dim=32, hidden_dims=[256], SiLU) at kitchen's shapes (act 9, obs 60);
# MLPNNClassifier's default ReLU with two hidden layers; and a CumRewClassifier over an out_dim-1 MLPNNClassifier.
# kw: MLPNNClassifier arguments (act: activation class name); head: "mse" (with temperature) or "cumrew"
NETS = {
    "tutorial_mse_silu": dict(x_dim=9, out_dim=60, emb_dim=32, hidden=[256], act="SiLU", head="mse", temperature=1.0),
    "mse_relu": dict(x_dim=9, out_dim=60, emb_dim=32, hidden=[256, 256], act="ReLU", head="mse", temperature=2.0),
    "cumrew_relu": dict(x_dim=6, out_dim=1, emb_dim=32, hidden=[256, 256], act="ReLU", head="cumrew"),
}
NET_BATCH = 8
T = 5                                  # the tutorial's diffusion_steps
# Guided sample() calls.  "tutorial": DiscreteDiffusionSDE over PearceMlp(act_dim, To=0, emb_dim=64, hidden_dim=256) with
# x0 prediction clipped to [-1, 1], 5 DDPM steps, temperature 0.5, w_cg 0.1, condition_cg = the observations.  "dql_eps":
# ContinuousDiffusionSDE over DQLMlp (eps prediction, the observations as condition_cfg too) guided by a ReLU
# MSEClassifier; "dql_cumrew": the same denoiser, x0 prediction with DDIM, guided by a ReLU CumRewClassifier.  Small batches
# keep the CPU interpreter quick.
BATCH = 16
SAMPLES = {
    "tutorial": dict(net="tutorial_mse_silu", kind="discrete", predict_noise=False, solver="ddpm", w_cg=0.1, temperature=0.5),
    "dql_eps": dict(net="mse_relu", kind="continuous", predict_noise=True, solver="ddpm", w_cg=0.5, temperature=1.0),
    "dql_cumrew": dict(net="cumrew_relu", kind="continuous", predict_noise=False, solver="ddim", w_cg=2.0, temperature=1.0),
}


def make_classifier(cls_net, cls_mse, cls_cumrew, name, seed, device="cpu", act=None):
    """the classifier of net case ``name``; ``act``: another hidden activation (torch.nn class name) at the same shape"""
    kw = NETS[name]
    net = cls_net(kw["x_dim"], kw["out_dim"], kw["emb_dim"], kw["hidden"], activation=getattr(torch.nn, act or kw["act"])())
    net.load_state_dict(synth_state_dict(net.state_dict(), seed))
    if kw["head"] == "mse":
        return cls_mse(net, temperature=kw["temperature"], device=device)
    return cls_cumrew(net, device=device)


def net_inputs(name):
    kw = NETS[name]
    g = torch.Generator().manual_seed(13)
    x = torch.randn(NET_BATCH, kw["x_dim"], generator=g).clamp(-1, 1)
    t = torch.randint(0, T, (NET_BATCH,), generator=g)
    c = torch.randn(NET_BATCH, kw["out_dim"], generator=g)
    return x, t, c


def sample_inputs(name):
    """(prior, observations c): an MSE head's target is c (out_dim wide); DQLMlp reads c[:, :11] as its condition"""
    kw = NETS[SAMPLES[name]["net"]]
    g = torch.Generator().manual_seed(11)
    return torch.zeros(BATCH, kw["x_dim"]), torch.randn(BATCH, max(kw["out_dim"], 11), generator=g)


def make_actor(name, classifier, cls_discrete, cls_continuous, cls_pearce, cls_dql, cls_identity, device="cpu"):
    spec, kw = SAMPLES[name], NETS[SAMPLES[name]["net"]]
    a = kw["x_dim"]
    clip = dict(x_max=torch.ones((1, a)), x_min=-torch.ones((1, a)))
    if spec["kind"] == "discrete":
        net = cls_pearce(a, To=0, emb_dim=64, hidden_dim=256, timestep_emb_type="positional")
        net.load_state_dict(synth_state_dict(net.state_dict(), 41))
        agent = cls_discrete(net, classifier=classifier, predict_noise=spec["predict_noise"], diffusion_steps=T, device=device,
                             **clip)
    else:
        net = cls_dql(obs_dim=11, act_dim=a)
        net.load_state_dict(synth_state_dict(net.state_dict(), 41))
        agent = cls_continuous(net, cls_identity(dropout=0.0), classifier=classifier, predict_noise=spec["predict_noise"],
                               device=device, **clip)
    agent.eval()
    return agent


def sample_kwargs(name, c):
    """sample() keyword arguments; ``c``: the case's sample_inputs condition"""
    spec, kw = SAMPLES[name], NETS[SAMPLES[name]["net"]]
    out = dict(solver=spec["solver"], n_samples=BATCH, sample_steps=T, temperature=spec["temperature"], w_cg=spec["w_cg"],
               condition_cg=c[:, :kw["out_dim"]] if kw["head"] == "mse" else None)
    if spec["kind"] == "continuous":
        out.update(sample_step_schedule="uniform_continuous", condition_cfg=c[:, :11], w_cfg=1.0)
    return out


def main():
    from cleandiffuser.classifier import CumRewClassifier, MSEClassifier
    from cleandiffuser.diffusion import ContinuousDiffusionSDE, DiscreteDiffusionSDE
    from cleandiffuser.nn_classifier import MLPNNClassifier
    from cleandiffuser.nn_condition import IdentityCondition
    from cleandiffuser.nn_diffusion import DQLMlp, PearceMlp
    out = {}
    for name in NETS:
        clf = make_classifier(MLPNNClassifier, MSEClassifier, CumRewClassifier, name, seed=31)
        x, t, c = net_inputs(name)
        logp, grad = clf.gradients(x.clone(), t, c if NETS[name]["head"] == "mse" else None)
        out[f"net/{name}/x"], out[f"net/{name}/t"], out[f"net/{name}/c"] = x.numpy(), t.numpy(), c.numpy()
        out[f"net/{name}/logp"], out[f"net/{name}/grad"] = logp.numpy(), grad.numpy()
    for k, name in enumerate(SAMPLES):
        torch.manual_seed(100 + k)                       # the loop's torch.randn_like draws (recorded on the noise tape)
        clf = make_classifier(MLPNNClassifier, MSEClassifier, CumRewClassifier, SAMPLES[name]["net"], seed=32)
        agent = make_actor(name, clf, DiscreteDiffusionSDE, ContinuousDiffusionSDE, PearceMlp, DQLMlp, IdentityCondition)
        prior, c = sample_inputs(name)
        tape = NoiseTape()
        with tape.active():
            x0, log = agent.sample(prior.clone(), **sample_kwargs(name, c))
        out[f"sample/{name}/prior"], out[f"sample/{name}/c"] = prior.numpy(), c.numpy()
        out[f"sample/{name}/x0"], out[f"sample/{name}/log_p"] = x0.detach().numpy(), log["log_p"].detach().numpy()
        for j, z in enumerate(tape.draws):
            out[f"sample/{name}/z{j}"] = z.numpy()
        out[f"sample/{name}/n_draws"] = np.array(len(tape.draws))
    np.savez_compressed(os.path.join(HERE, "mlp_classifier.npz"), **out)
    print("mlp_classifier.npz", len(out))


if __name__ == "__main__":
    main()
