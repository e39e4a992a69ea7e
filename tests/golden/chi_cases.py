"""ChiTransformer golden cases (pure data plus the weight recipe): the shapes Diffusion Policy's pipelines build, an edge
shape, and two sampling runs.  ``make_golden_chitransformer.py`` instantiates them with the reference class to write chitransformer.npz;
the tests instantiate the same cases with the product class and the engine."""
import torch

# name -> constructor kwargs (all pipelines: Ta = horizon = 10, To = 2)
NETS = {
    "pusht": dict(act_dim=2, obs_dim=256, Ta=10, To=2, d_model=256, nhead=4, num_layers=4),       # + robomimic image
    "robomimic": dict(act_dim=7, obs_dim=23, Ta=10, To=2, d_model=256, nhead=4, num_layers=8),    # low-dim obs (lift)
    "kitchen": dict(act_dim=9, obs_dim=60, Ta=10, To=2, d_model=768, nhead=4, num_layers=8),      # head_dim 192
    "edge": dict(act_dim=3, obs_dim=5, Ta=16, To=1, d_model=64, nhead=2, num_layers=2),           # head_dim 32
}
BATCH = 3

# sampling runs on a small model (CPU-fast): the dp_* pipeline pattern (legacy DDPM, identity condition, w_cfg = 1, clipped
# to [-1, 1]) and the SDE sampler with two-branch classifier-free guidance
SAMPLE_NET = dict(act_dim=2, obs_dim=5, Ta=10, To=2, d_model=64, nhead=2, num_layers=2)
SAMPLERS = {
    "ddpm_legacy": dict(kind="legacy", T=5, w_cfg=1.0),
    "sde_ddpm_cfg2": dict(kind="discrete", solver="ddpm", T=20, steps=5, w_cfg=1.5),
}
SAMPLE_BATCH = 4


def weights(template, synth, seed=0):
    """``synth`` (cleandiffuser_b200.testing.synth_state_dict) over the state-dict template, with the attention masks kept:
    they are parameters, but the network is only defined with the causal and memory masks it was built with."""
    sd = synth(template, seed=seed)
    for k in ("mask", "memory_mask"):
        sd[k] = template[k].clone()
    return sd


def net_inputs(ctor, batch=BATCH, seed=1):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn((batch, ctor["Ta"], ctor["act_dim"]), generator=g)
    t = torch.tensor([0, 7, 63][:batch], dtype=torch.long)
    cond = torch.randn((batch, ctor["To"], ctor["obs_dim"]), generator=g)
    return x, t, cond


def sampler_inputs(seed=2):
    g = torch.Generator().manual_seed(seed)
    Ta, To, obs = SAMPLE_NET["Ta"], SAMPLE_NET["To"], SAMPLE_NET["obs_dim"]
    prior = torch.zeros((SAMPLE_BATCH, Ta, SAMPLE_NET["act_dim"]))
    cond = torch.randn((SAMPLE_BATCH, To, obs), generator=g)
    x_max = torch.ones((1, Ta, SAMPLE_NET["act_dim"]))
    return prior, cond, x_max, -x_max
