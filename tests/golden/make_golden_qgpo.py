"""Generate tests/golden/qgpo.npz by running the UNMODIFIED reference (CPU, fp32): QGPOClassifier over QGPONNClassifier.

    python tests/golden/make_golden_qgpo.py [REFERENCE_CHECKOUT]
                                  # the reference must be importable as `cleandiffuser`: installed, or its checkout given

Contents (synthetic weights from ``cleandiffuser_b200.testing.synth_state_dict``, seeded inputs):
  net/<case>/{x, t, obs, logp, grad}   QGPONNClassifier logp and input gradient (clf.gradients) at continuous times
  sample/<case>/{prior, obs, z<j>, n_draws, x0, log_p}   guided sample() shaped like QGPO's inference call, noise tape recorded
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

# QGPO's classifier: QGPONNClassifier(obs_dim, act_dim, 64, [256, 256, 256], "untrainable_fourier") at the D4RL MuJoCo shapes
NETS = {"hopper": dict(obs_dim=11, act_dim=3), "halfcheetah": dict(obs_dim=17, act_dim=6)}
EMB, HIDDEN = 64, [256, 256, 256]
NET_BATCH = 8
# QGPO's sample(): ContinuousDiffusionSDE over SfBCUNet(act_dim) with MLPCondition(obs_dim, 64, [64], SiLU), clip to [-1, 1],
# "quad_continuous" steps, w_cfg = 1 with the observations as condition_cfg and condition_cg.  Small batches keep the CPU
# interpreter quick.
OBS, ACT, BATCH, STEPS = 11, 3, 16, 5
SAMPLES = {"ddpm_eps": dict(solver="ddpm", predict_noise=True, w_cg=0.7),
           "ddim_x0": dict(solver="ddim", predict_noise=False, w_cg=2.0)}


def make_classifier(cls_net, cls_clf, kw, seed, device="cpu"):
    net = cls_net(kw["obs_dim"], kw["act_dim"], EMB, HIDDEN, "untrainable_fourier")
    net.load_state_dict(synth_state_dict(net.state_dict(), seed))
    return cls_clf(net, device=device)


def net_inputs(kw):
    g = torch.Generator().manual_seed(13)
    x = torch.randn(NET_BATCH, kw["act_dim"], generator=g).clamp(-1, 1)
    t = torch.rand(NET_BATCH, generator=g)
    obs = torch.randn(NET_BATCH, kw["obs_dim"], generator=g)
    return x, t, obs


def sample_inputs():
    g = torch.Generator().manual_seed(11)
    return torch.zeros(BATCH, ACT), torch.randn(BATCH, OBS, generator=g)


def make_actor(cls_sde, cls_unet, cls_cond, predict_noise, classifier, device="cpu"):
    net = cls_unet(ACT)
    net.load_state_dict(synth_state_dict(net.state_dict(), 41))
    cond = cls_cond(OBS, 64, [64], torch.nn.SiLU())
    cond.load_state_dict(synth_state_dict(cond.state_dict(), 42))
    agent = cls_sde(net, cond, x_max=torch.ones(ACT), x_min=-torch.ones(ACT), predict_noise=predict_noise, device=device)
    agent.classifier = classifier
    agent.eval()
    return agent


def sample_kwargs(name, obs):
    spec = SAMPLES[name]
    return dict(solver=spec["solver"], n_samples=BATCH, sample_steps=STEPS, sample_step_schedule="quad_continuous",
                condition_cfg=obs, w_cfg=1.0, condition_cg=obs, w_cg=spec["w_cg"])


def main():
    from cleandiffuser.classifier import QGPOClassifier
    from cleandiffuser.diffusion import ContinuousDiffusionSDE
    from cleandiffuser.nn_classifier import QGPONNClassifier
    from cleandiffuser.nn_condition import MLPCondition
    from cleandiffuser.nn_diffusion import SfBCUNet
    out = {}
    for name, kw in NETS.items():
        clf = make_classifier(QGPONNClassifier, QGPOClassifier, kw, seed=31)
        x, t, obs = net_inputs(kw)
        logp, grad = clf.gradients(x.clone(), t, obs)
        out[f"net/{name}/x"], out[f"net/{name}/t"], out[f"net/{name}/obs"] = x.numpy(), t.numpy(), obs.numpy()
        out[f"net/{name}/logp"], out[f"net/{name}/grad"] = logp.numpy(), grad.numpy()
    prior, obs = sample_inputs()
    for k, (name, spec) in enumerate(SAMPLES.items()):
        torch.manual_seed(100 + k)                       # the loop's torch.randn_like draws (recorded on the noise tape)
        clf = make_classifier(QGPONNClassifier, QGPOClassifier, dict(obs_dim=OBS, act_dim=ACT), seed=32)
        agent = make_actor(ContinuousDiffusionSDE, SfBCUNet, MLPCondition, spec["predict_noise"], clf)
        tape = NoiseTape()
        with tape.active():
            x0, log = agent.sample(prior.clone(), **sample_kwargs(name, obs))
        out[f"sample/{name}/prior"], out[f"sample/{name}/obs"] = prior.numpy(), obs.numpy()
        out[f"sample/{name}/x0"], out[f"sample/{name}/log_p"] = x0.detach().numpy(), log["log_p"].detach().numpy()
        for j, z in enumerate(tape.draws):
            out[f"sample/{name}/z{j}"] = z.numpy()
        out[f"sample/{name}/n_draws"] = np.array(len(tape.draws))
    np.savez_compressed(os.path.join(HERE, "qgpo.npz"), **out)
    print("qgpo.npz", len(out))


if __name__ == "__main__":
    main()
