"""Generate tests/golden/half_dit.npz by running the UNMODIFIED reference (CPU, fp32): CumRewClassifier over HalfDiT1d.

    python tests/golden/make_golden_half_dit.py [REFERENCE_CHECKOUT]
                                  # the reference must be importable as `cleandiffuser`: installed, or its checkout given

Contents (synthetic weights from ``cleandiffuser_b200.testing.synth_state_dict``: HalfDiT1d zero-initialises its final layer
and every adaLN, which would make the gradient vanish; seeded inputs):
  net/<case>/{x, t, logp, grad}   logp and input gradient (clf.gradients) at discrete times
  sample/<case>/{prior, z<j>, n_draws, x0, log_p}   guided sample() calls, noise tape recorded
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

# head_dim 16 / 32 / 64, horizons 1 to 64 (no power of two needed), every timestep embedding, out_dim 1 and 3.  Small widths
# keep the CPU interpreter quick; the reference's default shape (d_model 384, 6 heads, depth 12) is timed by
# scripts/half_dit_cg_bench.py and tested on the H100.
NETS = {
    "hd16_h1": dict(in_dim=5, out_dim=1, emb_dim=16, d_model=32, n_heads=2, depth=1, timestep_emb_type="positional", horizon=1),
    "hd32_h4": dict(in_dim=6, out_dim=3, emb_dim=16, d_model=64, n_heads=2, depth=2, timestep_emb_type="fourier", horizon=4),
    "hd64_h10": dict(in_dim=3, out_dim=1, emb_dim=32, d_model=128, n_heads=2, depth=1,
                     timestep_emb_type="untrainable_fourier", horizon=10),
    "hd16_h32": dict(in_dim=11, out_dim=3, emb_dim=16, d_model=64, n_heads=4, depth=2, timestep_emb_type="positional",
                     horizon=32),
    "hd64_h64": dict(in_dim=4, out_dim=1, emb_dim=16, d_model=64, n_heads=1, depth=1, timestep_emb_type="untrainable_positional",
                     horizon=64),
}
NET_BATCH = 3
T = 20
# guided sample(): DiscreteDiffusionSDE over JannerUNet1d (eps prediction, DDPM) and ContinuousDiffusionSDE over DiT1d
# (x0 prediction, DDIM), both with the first step of every trajectory fixed by the mask, guided by a CumRewClassifier(HalfDiT1d)
H, D, BATCH, W_CG, STEPS = 8, 6, 6, 0.3, 4
CLF = dict(in_dim=D, out_dim=1, emb_dim=16, d_model=64, n_heads=2, depth=2, timestep_emb_type="positional")
SAMPLES = {"discrete_janner": dict(kind="discrete", solver="ddpm", predict_noise=True),
           "continuous_dit": dict(kind="continuous", solver="ddim", predict_noise=False)}


def make_net(cls, kw, seed):
    net = cls(**{k: v for k, v in kw.items() if k != "horizon"})
    net.load_state_dict(synth_state_dict(net.state_dict(), seed))
    return net.eval()


def net_inputs(name):
    kw = NETS[name]
    g = torch.Generator().manual_seed(13)
    x = torch.randn(NET_BATCH, kw["horizon"], kw["in_dim"], generator=g)
    t = torch.randint(0, T, (NET_BATCH,), generator=g)
    return x, t


def sample_inputs():
    g = torch.Generator().manual_seed(11)
    prior = torch.zeros(BATCH, H, D)
    prior[:, 0] = torch.randn(BATCH, D, generator=g)
    mask = torch.zeros(H, D)
    mask[0] = 1.
    return prior, mask


def make_agent(name, classifier, cls_discrete, cls_continuous, cls_janner, cls_dit, device="cpu"):
    spec = SAMPLES[name]
    _, mask = sample_inputs()
    common = dict(fix_mask=mask, predict_noise=spec["predict_noise"], device=device, classifier=classifier)
    if spec["kind"] == "discrete":
        net = cls_janner(D, model_dim=16, emb_dim=16, dim_mult=[1, 2])
        net.load_state_dict(synth_state_dict(net.state_dict(), 21))
        agent = cls_discrete(net, diffusion_steps=T, **common)
    else:
        net = cls_dit(D, emb_dim=16, d_model=32, n_heads=1, depth=1)
        net.load_state_dict(synth_state_dict(net.state_dict(), 21))
        agent = cls_continuous(net, **common)
    agent.model_ema.eval()
    return agent


def sample_kwargs(name):
    return dict(solver=SAMPLES[name]["solver"], n_samples=BATCH, sample_steps=STEPS, use_ema=True, temperature=0.8, w_cg=W_CG,
                sample_step_schedule="uniform" if SAMPLES[name]["kind"] == "discrete" else "uniform_continuous")


def main():
    from cleandiffuser.classifier import CumRewClassifier
    from cleandiffuser.diffusion import ContinuousDiffusionSDE, DiscreteDiffusionSDE
    from cleandiffuser.nn_classifier import HalfDiT1d
    from cleandiffuser.nn_diffusion import DiT1d, JannerUNet1d
    out = {}
    for name, kw in NETS.items():
        clf = CumRewClassifier(make_net(HalfDiT1d, kw, 31), device="cpu")
        x, t = net_inputs(name)
        logp, grad = clf.gradients(x.clone(), t, None)
        out[f"net/{name}/x"], out[f"net/{name}/t"] = x.numpy(), t.numpy()
        out[f"net/{name}/logp"], out[f"net/{name}/grad"] = logp.numpy(), grad.numpy()
    prior, _ = sample_inputs()
    for k, name in enumerate(SAMPLES):
        torch.manual_seed(100 + k)                       # the loop's torch.randn_like draws (recorded on the noise tape)
        clf = CumRewClassifier(make_net(HalfDiT1d, CLF, 32), device="cpu")
        agent = make_agent(name, clf, DiscreteDiffusionSDE, ContinuousDiffusionSDE, JannerUNet1d, DiT1d)
        tape = NoiseTape()
        with tape.active():
            x0, log = agent.sample(prior.clone(), **sample_kwargs(name))
        out[f"sample/{name}/prior"] = prior.numpy()
        out[f"sample/{name}/x0"], out[f"sample/{name}/log_p"] = x0.detach().numpy(), log["log_p"].detach().numpy()
        for j, z in enumerate(tape.draws):
            out[f"sample/{name}/z{j}"] = z.numpy()
        out[f"sample/{name}/n_draws"] = np.array(len(tape.draws))
    np.savez_compressed(os.path.join(HERE, "half_dit.npz"), **out)
    print("half_dit.npz", len(out))


if __name__ == "__main__":
    main()
