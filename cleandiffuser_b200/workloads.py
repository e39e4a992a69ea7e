"""The BASELINE configurations (cfg2 .. cfg5: the headline of bench.py and its other_configs) as synthetic workloads (SURVEY 8d recipe: weights seed 0, inputs seed 1).

One place that says what "cfg2 .. cfg5" are, shared by ``bench.py`` (headline + ``other_configs``), the parity
tests at the configs' full sizes (``tests/test_baseline_configs_gpu.py``) and the profiling scripts, so that the
thing measured is the thing tested.  Every builder returns a ``Workload``:

    agent        the product diffusion object (PyTorch host surface; ``sample()`` dispatches to the CUDA engine)
    prior        (batch, *x_shape) CPU tensor handed to ``sample`` (zeros + the conditioning portion under the mask)
    kwargs       the ``sample()`` keyword arguments of the config (``n_samples`` = batch)
    oracle       plain-data description of the same computation for the CPU oracle (function names + keyword
                 arguments, NO import of ``oracle/`` here: only tests / bench's CPU legs resolve it)
    gflop        algorithmic GFLOP per trajectory for a full sample() (SURVEY 8d)
    hbm_mb       algorithmic HBM megabytes per trajectory for a full sample() (0: not derived), see the builder

Reference call sites these mirror: pipelines/diffuser_d4rl_mujoco.py:39-66,136-148 (cfg2),
pipelines/dp_pusht.py (cfg3), pipelines/dd_d4rl_mujoco.py (cfg4), pipelines/ (consistency) cfg5.
"""
from dataclasses import dataclass, field
from typing import Any, Dict, Optional

import torch

from .testing import load_synth


@dataclass
class Workload:
    name: str
    agent: Any
    prior: torch.Tensor
    kwargs: Dict[str, Any]
    oracle: Dict[str, Any]
    gflop: float
    cond: Optional[torch.Tensor] = None
    describe: str = ""
    hbm_mb: float = 0.0
    extra: Dict[str, Any] = field(default_factory=dict)

    def sample(self, device, prior=None, cond=None, **over):
        """One ``sample()`` call of the config; tensors are moved to ``device``."""
        kw = dict(self.kwargs)
        kw.update(over)
        prior = self.prior if prior is None else prior
        cond = self.cond if cond is None else cond
        if cond is not None:
            kw["condition_cfg"] = cond.to(device)
        kw["n_samples"] = prior.shape[0]
        return self.agent.sample(prior.to(device), **kw)


def cfg2(device, batch=4096, steps=100, seed=0):
    """JannerUNet1d Diffuser, H=32 d=14 (hopper), DDPM ``steps`` of ``steps`` diffusion steps, fix_mask on the first observation."""
    from .diffusion import DiscreteDiffusionSDE
    from .nn_diffusion import JannerUNet1d
    H, D, OBS = 32, 14, 11
    net = load_synth(JannerUNet1d(D, model_dim=32, emb_dim=32, kernel_size=5, dim_mult=[1, 2, 2, 2]), seed=seed)
    mask = torch.zeros(H, D)
    mask[0, :OBS] = 1.
    agent = DiscreteDiffusionSDE(net, None, fix_mask=mask, predict_noise=False, diffusion_steps=steps, device=device)
    g = torch.Generator().manual_seed(1)
    prior = torch.zeros(batch, H, D)
    prior[:, 0, :OBS] = torch.randn(batch, OBS, generator=g)
    return Workload(
        "cfg2", agent, prior, dict(solver="ddpm", sample_steps=steps, temperature=0.5),
        dict(net=dict(fn="janner_unet", emb_dim=32, kernel_size=5, n_stages=4), sampler="sample_discrete",
             kwargs=dict(T=steps, steps=steps, solver="ddpm", temperature=0.5, predict_noise=False), fix_mask=mask[None]),
        gflop=3.920 * steps / 100,
        describe=f"JannerUNet1d(14,32,[1,2,2,2],k5) H=32 d=14, DiscreteDiffusionSDE DDPM {steps} steps, batch {batch}")


def _chi_net(seed, **kw):
    from .nn_diffusion import ChiUNet1d
    return load_synth(ChiUNet1d(7, 20, 2, model_dim=256, emb_dim=256, kernel_size=5, dim_mult=[1, 2, 2], **kw), seed=seed)


def cfg3(device, batch=2048, steps=50, seed=0):
    """ChiUNet1d Diffusion Policy (68.9 M parameters), obs 20 x To 2, act 7, H=16, DDIM 50 of 1000 steps, w_cfg = 1."""
    from .diffusion import DiscreteDiffusionSDE
    from .nn_condition import IdentityCondition
    net = _chi_net(seed)
    x_max, x_min = torch.ones(1, 16, 7), -torch.ones(1, 16, 7)
    agent = DiscreteDiffusionSDE(net, IdentityCondition(dropout=0.0), predict_noise=True, diffusion_steps=1000,
                                 x_max=x_max, x_min=x_min, device=device)
    g = torch.Generator().manual_seed(1)
    cond = torch.randn(batch, 2, 20, generator=g)
    return Workload(
        "cfg3", agent, torch.zeros(batch, 16, 7), dict(solver="ddim", sample_steps=steps, w_cfg=1.0),
        dict(net=dict(fn="chi_unet", emb_dim=256, kernel_size=5, n_stages=3), sampler="sample_discrete",
             kwargs=dict(T=1000, steps=steps, solver="ddim", predict_noise=True, w_cfg=1.0, x_min=x_min, x_max=x_max),
             fix_mask=0.),
        gflop=29.85 * steps / 50, cond=cond,
        describe=f"ChiUNet1d(act 7, obs 20x2, model_dim 256, [1,2,2]) H=16, DiscreteDiffusionSDE DDIM {steps}/1000, w_cfg 1, batch {batch}")


def cfg4(device, batch=2048, steps=20, seed=0, w_cfg=6.0):
    """DiT1d Decision Diffuser, H=100 d=29 (walker2d), DPM-Solver++ 2M 20 steps, two CFG branches (w_cfg = 6)."""
    from .diffusion import ContinuousDiffusionSDE
    from .nn_condition import MLPCondition
    from .nn_diffusion import DiT1d
    net = load_synth(DiT1d(29, emb_dim=128, d_model=320, n_heads=10, depth=2, timestep_emb_type="fourier"), seed=seed)
    nc = load_synth(MLPCondition(1, 128, [128], torch.nn.SiLU(), dropout=0.25), seed=3)
    mask = torch.zeros(100, 29)
    mask[0] = 1.
    agent = ContinuousDiffusionSDE(net, nc, fix_mask=mask, predict_noise=True, noise_schedule="linear", device=device)
    agent.model.eval()
    agent.model_ema.eval()
    g = torch.Generator().manual_seed(1)
    prior = torch.zeros(batch, 100, 29)
    prior[:, 0] = torch.randn(batch, 29, generator=g)
    cond = torch.rand(batch, 1, generator=g)
    return Workload(
        "cfg4", agent, prior,
        dict(solver="ode_dpmsolver++_2M", sample_steps=steps, sample_step_schedule="uniform_continuous", temperature=0.5, w_cfg=w_cfg),
        dict(net=dict(fn="dit1d", emb_dim=128, d_model=320, n_heads=10, depth=2, emb_kind="fourier"),
             sampler="sample_continuous",
             kwargs=dict(steps=steps, solver="ode_dpmsolver++_2M", schedule="linear", temperature=0.5, predict_noise=True, w_cfg=w_cfg),
             fix_mask=mask[None], cond=dict(fn="mlp_condition", act="silu", n_hidden=1)),
        gflop=20.96 * steps / 20, cond=cond,
        # fp32 tensors every fused operator of the TF32 program reads / writes per token row and iteration: x_proj 4 (32 + 320),
        # LN+modulate 2 x 1280, per block QKV 1280 + 3840, attention 3840 + 1280, out-proj (+LN) 4 x 1280, fc1 1280 + 5120,
        # fc2 (+LN) 5120 + 3 x 1280, head 1280 + 116 = 66.8 KB; 100 tokens x 2 CFG branches per trajectory
        hbm_mb=66804 * 100 * 2 * steps / 1e6,
        describe=f"DiT1d(29, d320, 10 heads, depth 2) H=100 d=29, ContinuousDiffusionSDE DPM-Solver++2M {steps} steps, w_cfg {w_cfg} (2 branches), batch {batch}")


def cfg5(device, batch=8192, steps=1, seed=0):
    """Consistency-distilled ChiUNet1d, 1-step sample, act 7 H=16."""
    from .diffusion import ContinuousConsistencyModel
    from .nn_condition import IdentityCondition
    net = _chi_net(seed, timestep_emb_type="untrainable_fourier")
    x_max, x_min = torch.ones(1, 16, 7), -torch.ones(1, 16, 7)
    cm = ContinuousConsistencyModel(net, IdentityCondition(dropout=0.0), x_max=x_max, x_min=x_min, device=device)
    g = torch.Generator().manual_seed(1)
    cond = torch.randn(batch, 2, 20, generator=g)
    return Workload(
        "cfg5", cm, torch.zeros(batch, 16, 7), dict(sample_steps=steps, w_cfg=1.0),
        dict(net=dict(fn="chi_unet", emb_dim=256, kernel_size=5, n_stages=3, emb_kind="untrainable_fourier"),
             sampler="sample_consistency", kwargs=dict(steps=steps, x_min=x_min, x_max=x_max), fix_mask=0.),
        gflop=0.597 * steps, cond=cond,
        describe=f"ContinuousConsistencyModel over ChiUNet1d(model_dim 256), {steps}-step sample, H=16 act 7, batch {batch}")


BUILDERS = {"cfg2": cfg2, "cfg3": cfg3, "cfg4": cfg4, "cfg5": cfg5}
