"""Generate tests/golden/classifier.npz by running the UNMODIFIED reference (CPU, fp32): CumRewClassifier over HalfJannerUNet1d.

    python tests/golden/make_golden_classifier.py [REFERENCE_CHECKOUT]
                                  # the reference must be importable as `cleandiffuser`: installed, or its checkout given

Contents (synthetic weights from ``cleandiffuser_b200.testing.synth_state_dict``, seeded inputs):
  net/<case>/{x, t_long, t_float, logp_long, grad_long, logp_float, grad_float}   HalfJannerUNet1d logp and input gradient
  sample/<case>/{prior, z<j>, n_draws, x0, log_p}   guided sample() with a JannerUNet1d denoiser, noise tape recorded
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

# the classifier shapes of the reference's pipelines that reach different code: hopper-like, and halfcheetah-like (length 1)
NETS = {"hopper": dict(horizon=32, in_dim=14, dim_mult=(1, 2, 2, 2)),
        "halfcheetah": dict(horizon=4, in_dim=23, dim_mult=(1, 4, 2))}
NET_BATCH = 4
# guided sample(): small shapes so that the CPU interpreter runs them quickly
H, D, BATCH, W_CG = 8, 6, 8, 0.3
SAMPLES = {"discrete_ddpm_eps": dict(kind="discrete", solver="ddpm", predict_noise=True),
           "discrete_ddpm_x0": dict(kind="discrete", solver="ddpm", predict_noise=False),
           "continuous_ddim_eps": dict(kind="continuous", solver="ddim", predict_noise=True),
           "continuous_ddim_x0": dict(kind="continuous", solver="ddim", predict_noise=False)}
STEPS, T = 5, 20


def make_classifier(cls_net, cls_clf, kw, seed):
    net = cls_net(**kw)
    net.load_state_dict(synth_state_dict(net.state_dict(), seed))
    return cls_clf(net)


def sample_inputs():
    g = torch.Generator().manual_seed(11)
    prior = torch.zeros(BATCH, H, D)
    prior[:, 0] = torch.randn(BATCH, D, generator=g)
    mask = torch.zeros(H, D)
    mask[0] = 1.
    return prior, mask


def make_denoiser(cls):
    net = cls(D, model_dim=16, emb_dim=16, dim_mult=[1, 2])
    net.load_state_dict(synth_state_dict(net.state_dict(), 21))
    return net


def main():
    from cleandiffuser.classifier import CumRewClassifier
    from cleandiffuser.diffusion import ContinuousDiffusionSDE, DiscreteDiffusionSDE
    from cleandiffuser.nn_classifier import HalfJannerUNet1d
    from cleandiffuser.nn_diffusion import JannerUNet1d
    out = {}
    for name, kw in NETS.items():
        clf = make_classifier(HalfJannerUNet1d, CumRewClassifier, kw, seed=31)
        g = torch.Generator().manual_seed(13)
        x = torch.randn(NET_BATCH, kw["horizon"], kw["in_dim"], generator=g)
        t_long = torch.randint(0, 1000, (NET_BATCH,), generator=g)
        t_float = torch.rand(NET_BATCH, generator=g)
        out[f"net/{name}/x"], out[f"net/{name}/t_long"], out[f"net/{name}/t_float"] = x.numpy(), t_long.numpy(), t_float.numpy()
        for tn, t in (("long", t_long), ("float", t_float)):
            logp, grad = clf.gradients(x.clone(), t, None)
            out[f"net/{name}/logp_{tn}"], out[f"net/{name}/grad_{tn}"] = logp.numpy(), grad.numpy()
    prior, mask = sample_inputs()
    for k, (name, spec) in enumerate(SAMPLES.items()):
        torch.manual_seed(100 + k)                       # the loop's torch.randn_like draws (recorded on the noise tape)
        clf = make_classifier(HalfJannerUNet1d, CumRewClassifier, dict(horizon=H, in_dim=D, dim_mult=(1, 2)), seed=32)
        common = dict(fix_mask=mask, predict_noise=spec["predict_noise"], device="cpu", classifier=clf)
        if spec["kind"] == "discrete":
            agent, sched = DiscreteDiffusionSDE(make_denoiser(JannerUNet1d), diffusion_steps=T, **common), "uniform"
        else:
            agent, sched = ContinuousDiffusionSDE(make_denoiser(JannerUNet1d), **common), "uniform_continuous"
        agent.model_ema.eval()
        tape = NoiseTape()
        with tape.active():
            x0, log = agent.sample(prior.clone(), solver=spec["solver"], n_samples=BATCH, sample_steps=STEPS,
                                   sample_step_schedule=sched, use_ema=True, temperature=0.8, w_cg=W_CG)
        out[f"sample/{name}/x0"], out[f"sample/{name}/log_p"] = x0.detach().numpy(), log["log_p"].detach().numpy()
        for j, z in enumerate(tape.draws):
            out[f"sample/{name}/z{j}"] = z.numpy()
        out[f"sample/{name}/n_draws"] = np.array(len(tape.draws))
    np.savez_compressed(os.path.join(HERE, "classifier.npz"), **out)
    print("classifier.npz", len(out))


if __name__ == "__main__":
    main()
