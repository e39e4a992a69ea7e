"""Generate tests/golden/chitransformer.npz by running the UNMODIFIED reference ChiTransformer (CPU, fp32).

    python tests/golden/make_golden_chitransformer.py     # needs /root/reference

The cases are chi_cases.py: forward outputs at the Diffusion Policy shapes and an edge shape (synthetic weights from
``cleandiffuser_b200.testing.synth_state_dict`` with the attention masks kept), and two sampling runs with their recorded
noise tapes.  Like make_golden.py, the reference is only ever read here, never at test time.
"""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
sys.path.insert(0, "/root/reference")

import chi_cases as cc  # noqa: E402
from cleandiffuser_b200.testing import NoiseTape, synth_state_dict  # noqa: E402

import cleandiffuser.nn_diffusion as ref_nn  # noqa: E402
import cleandiffuser.nn_condition as ref_cond  # noqa: E402
from cleandiffuser.diffusion import DiscreteDiffusionSDE  # noqa: E402
from cleandiffuser.diffusion.ddpm import DDPM  # noqa: E402


def gen_chitransformer():
    """ChiTransformer forward at the pipeline shapes and an edge shape, and two sampling runs (chi_cases.py)."""
    out = {}
    for name, ctor in cc.NETS.items():
        net = ref_nn.ChiTransformer(**ctor)
        sd = cc.weights(net.state_dict(), synth_state_dict)
        net.load_state_dict(sd)
        net.eval()
        x, t, cond = cc.net_inputs(ctor)
        with torch.no_grad():
            out[name + "/y"] = net(x, t, cond).numpy()
            out[name + "/y_uncond"] = net(x, t, None).numpy()
        out[name + "/keys"] = np.array(["%s|%s" % (k, ",".join(map(str, v.shape))) for k, v in sd.items()])
    prior, cond, x_max, x_min = cc.sampler_inputs()
    for name, spec in cc.SAMPLERS.items():
        net = ref_nn.ChiTransformer(**cc.SAMPLE_NET)
        net.load_state_dict(cc.weights(net.state_dict(), synth_state_dict))
        nc = ref_cond.IdentityCondition(dropout=0.0)
        if spec["kind"] == "legacy":
            agent = DDPM(net, nc, x_max=x_max, x_min=x_min, diffusion_steps=spec["T"], device="cpu")
            kw = dict(sample_steps=spec["T"])
        else:
            agent = DiscreteDiffusionSDE(net, nc, x_max=x_max, x_min=x_min, diffusion_steps=spec["T"], device="cpu")
            kw = dict(solver=spec["solver"], sample_steps=spec["steps"])
        agent.model_ema.eval()
        tape = NoiseTape()
        torch.manual_seed(0)                     # the draws the tape records: the file is reproducible
        with tape.active(), torch.no_grad():
            x0, _ = agent.sample(prior, n_samples=cc.SAMPLE_BATCH, use_ema=True, condition_cfg=cond, w_cfg=spec["w_cfg"], **kw)
        out[name + "/x0"] = x0.numpy()
        for j, z in enumerate(tape.draws):
            out[f"{name}/z{j}"] = z.numpy()
        out[name + "/n_draws"] = np.array(len(tape.draws))
    np.savez_compressed(os.path.join(HERE, "chitransformer.npz"), **out)
    print("chitransformer.npz", len(out))


if __name__ == "__main__":
    torch.set_num_threads(1)
    gen_chitransformer()
