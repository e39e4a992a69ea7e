"""``nn_classifier`` plugin surface: networks ``(x, noise[, condition]) -> log p(y | x, t) + const`` of shape (batch, out_dim).

``HalfJannerUNet1d`` is the down half of JannerUNet1d followed by a small MLP head, with the reference's constructor signature,
parameter names and shapes (cleandiffuser/nn_classifier/half_jannerunet.py), so its checkpoints load.  Under classifier guidance
(``CumRewClassifier``) the engine lowers its forward and input gradient into the replayed loop (``engine/lower.py``,
``lower_half_janner_grad``); everything else about it runs in PyTorch.  ``QGPONNClassifier`` (nn_classifier/mlp.py) is QGPO's
energy network; under ``QGPOClassifier`` guidance its input gradient is lowered the same way (``lower_qgpo_grad``).
``MLPNNClassifier`` (nn_classifier/mlp.py) is the general-purpose MLP over ``[x | map_noise(t)]``; under ``MSEClassifier``
guidance, or ``CumRewClassifier`` guidance with ``out_dim = 1``, its input gradient is lowered by
``lower_mlp_classifier_grad`` when its hidden activation is ReLU, SiLU or Mish and its output activation the identity.
``HalfDiT1d`` (the reference's nn_classifier/half_dit.py) is DiT1d with a FinalLayer1d to d_model / 2 channels, a mean over the horizon and a
LayerNorm + SiLU + Linear head; under ``CumRewClassifier`` guidance its input gradient is lowered by ``lower_half_dit_grad``.
"""
from typing import List, Optional, Tuple

import numpy as np
import torch
import torch.nn as nn

from ..nn_diffusion.base import BaseNNDiffusion
from ..nn_diffusion.dit1d import DiT1d, FinalLayer1d
from ..nn_diffusion.unets import Downsample1d, ResidualBlock
from ..utils import Mlp


class HalfJannerUNet1d(BaseNNDiffusion):
    """x (b, horizon, in_dim), noise (b,), condition (b, model_dim... added to the time embedding) | None -> (b, out_dim).

    Stages: two ResidualBlocks per resolution of ``dim_mult`` with a Downsample1d between resolutions, then two mid
    ResidualBlocks (kernel 5) halving the channels, each followed by a Downsample1d, then
    ``Linear(fc_dim + model_dim, fc_dim // 2) -> Mish -> Linear(fc_dim // 2, out_dim)`` over ``[flatten(x), emb]`` with the
    features flattened channel-major, ``fc_dim = mid_dim // 4 * max(final length, 1)``."""

    def __init__(self, horizon: int, in_dim: int, out_dim: int = 1, kernel_size: int = 3, model_dim: int = 32,
                 emb_dim: int = 32, dim_mult: Tuple[int] = (1, 2, 2, 2), timestep_emb_type: str = "positional",
                 norm_type: str = "groupnorm"):
        super().__init__(emb_dim, timestep_emb_type)
        dims = [in_dim] + [model_dim * m for m in np.cumprod(dim_mult)]
        pairs = list(zip(dims[:-1], dims[1:]))
        self.map_emb = nn.Sequential(nn.Linear(emb_dim, model_dim * 4), nn.Mish(), nn.Linear(model_dim * 4, model_dim))
        self.downs = nn.ModuleList([])
        self.ups = nn.ModuleList([])           # empty: kept so that the module tree reads like the reference's
        length = horizon
        for i, (cin, cout) in enumerate(pairs):
            last = i == len(pairs) - 1
            self.downs.append(nn.ModuleList([
                ResidualBlock(cin, cout, model_dim, kernel_size, norm_type),
                ResidualBlock(cout, cout, model_dim, kernel_size, norm_type),
                nn.Identity() if last else Downsample1d(cout)]))
            if not last:
                length //= 2
        mid = dims[-1]
        self.mid_block1 = nn.ModuleList([ResidualBlock(mid, mid // 2, model_dim, kernel_size=5, norm_type=norm_type),
                                         Downsample1d(mid // 2)])
        self.mid_block2 = nn.ModuleList([ResidualBlock(mid // 2, mid // 4, model_dim, kernel_size=5, norm_type=norm_type),
                                         Downsample1d(mid // 4)])
        length = length // 4
        fc_dim = mid // 4 * max(length, 1)
        self.final_block = nn.Sequential(nn.Linear(fc_dim + model_dim, fc_dim // 2), nn.Mish(), nn.Linear(fc_dim // 2, out_dim))

    def forward(self, x: torch.Tensor, noise: torch.Tensor, condition: Optional[torch.Tensor] = None):
        h = x.permute(0, 2, 1)
        emb = self.map_noise(noise)
        if condition is not None:
            emb = emb + condition
        emb = self.map_emb(emb)
        for res1, res2, down in self.downs:
            h = down(res2(res1(h, emb), emb))
        for block, down in (self.mid_block1, self.mid_block2):
            h = down(block(h, emb))
        return self.final_block(torch.cat([h.flatten(1), emb], dim=-1))


class MLPNNClassifier(BaseNNDiffusion):
    """x (b, x_dim), t (b,), y ignored -> (b, out_dim): ``Mlp([x | map_noise(t)])`` with ``activation`` after every hidden
    Linear (one module instance, as in the reference) and ``out_activation`` after the output Linear.  State-dict keys
    ``map_noise.*``, ``mlp.mlp.<i>.0.*`` (hidden Linears), ``mlp.mlp.<n>.*`` (output Linear)."""

    def __init__(self, x_dim: int, out_dim: int, emb_dim: int, hidden_dims: List[int], activation: nn.Module = nn.ReLU(),
                 out_activation: nn.Module = nn.Identity(), timestep_emb_type: str = "positional"):
        super().__init__(emb_dim, timestep_emb_type)
        self.mlp = Mlp(in_dim=x_dim + emb_dim, hidden_dims=hidden_dims, out_dim=out_dim, activation=activation,
                       out_activation=out_activation)

    def forward(self, x: torch.Tensor, t: torch.Tensor, y: Optional[torch.Tensor] = None):
        return self.mlp(torch.cat([x, self.map_noise(t)], dim=-1))


class QGPONNClassifier(BaseNNDiffusion):
    """x (b, act_dim) noisy actions, t (b,), y (b, obs_dim) observations -> energy (b, 1) in (-10, 10):
    ``10 tanh(mlp([obs_proj(y), act_proj(x), map_noise(t)]) / 10)`` with an Mlp of Linear + SiLU hidden layers."""

    def __init__(self, obs_dim: int, act_dim: int, emb_dim: int, hidden_dims: List[int],
                 timestep_emb_type: str = "positional"):
        super().__init__(emb_dim, timestep_emb_type)
        self.obs_proj = nn.Linear(obs_dim, emb_dim)
        self.act_proj = nn.Linear(act_dim, emb_dim)
        self.mlp = Mlp(in_dim=3 * emb_dim, hidden_dims=hidden_dims, out_dim=1, activation=nn.SiLU())

    def forward(self, x: torch.Tensor, t: torch.Tensor, y: torch.Tensor):
        y = self.obs_proj(y)
        x = self.act_proj(x)
        out = self.mlp(torch.cat([y, x, self.map_noise(t)], dim=-1))
        return torch.tanh(out / 10) * 10


class HalfDiT1d(DiT1d):
    """x (b, horizon, in_dim), noise (b,), condition (b, emb_dim) | None -> (b, out_dim): ``proj(mean_L(DiT1d(x)))`` where DiT1d's
    final layer maps to d_model // 2 channels (weights and adaLN zero-initialised, as in the reference) and
    ``proj = LayerNorm, SiLU, Linear(d_model // 2, d_model // 4), LayerNorm, SiLU, Linear(d_model // 4, out_dim)``.
    Constructor, defaults and state-dict keys are the reference's (cleandiffuser/nn_classifier/half_dit.py)."""

    def __init__(self, in_dim: int, out_dim: int, emb_dim: int, d_model: int = 384, n_heads: int = 6, depth: int = 12,
                 dropout: float = 0.0, timestep_emb_type: str = "positional"):
        super().__init__(in_dim, emb_dim, d_model, n_heads, depth, dropout, timestep_emb_type)
        self.final_layer = FinalLayer1d(d_model, d_model // 2)
        for lin in (self.final_layer.adaLN_modulation[-1], self.final_layer.linear):
            nn.init.constant_(lin.weight, 0)
            nn.init.constant_(lin.bias, 0)
        self.proj = nn.Sequential(
            nn.LayerNorm(d_model // 2), nn.SiLU(), nn.Linear(d_model // 2, d_model // 4),
            nn.LayerNorm(d_model // 4), nn.SiLU(), nn.Linear(d_model // 4, out_dim))

    def forward(self, x: torch.Tensor, noise: torch.Tensor, condition: Optional[torch.Tensor] = None):
        return self.proj(super().forward(x, noise, condition).mean(1))
