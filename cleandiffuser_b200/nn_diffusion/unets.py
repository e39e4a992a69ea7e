"""1-D temporal UNet denoisers: ``JannerUNet1d`` (Diffuser) and ``ChiUNet1d`` (Diffusion Policy).

PyTorch definitions of the two UNets with parameter names/shapes identical to
the reference so ``.pt`` checkpoints interchange:
  JannerUNet1d -> cleandiffuser/nn_diffusion/jannerunet.py:98-201
  ChiUNet1d    -> cleandiffuser/nn_diffusion/chiunet.py:48-192
These modules are the weight containers and the autograd (training /
``requires_grad=True``) path.  For sampling, ``engine/lower.py`` walks the same
module tree and emits the fused conv+GN+Mish(+FiLM/+residual) op list that the
sm_90a kernels execute.
"""
from typing import List, Optional

import numpy as np
import torch
import torch.nn as nn

from .base import BaseNNDiffusion
from ..utils import GroupNorm1d


def _conv_gn_mish(cin, cout, k, norm_type="groupnorm"):
    return nn.Sequential(nn.Conv1d(cin, cout, k, padding=k // 2), get_norm(cout, norm_type), nn.Mish())


class LayerNorm(nn.Module):
    """Channel LayerNorm on (b, C, L) used by the optional attention (jannerunet.py:39-49)."""

    def __init__(self, dim, eps=1e-5):
        super().__init__()
        self.eps = eps
        self.g = nn.Parameter(torch.ones(1, dim, 1))
        self.b = nn.Parameter(torch.zeros(1, dim, 1))

    def forward(self, x):
        mu = x.mean(dim=1, keepdim=True)
        var = x.var(dim=1, unbiased=False, keepdim=True)
        return (x - mu) / (var + self.eps).sqrt() * self.g + self.b


def get_norm(dim: int, norm_type: str = "groupnorm"):
    if norm_type == "groupnorm":
        return GroupNorm1d(dim, 8, 4)
    if norm_type == "layernorm":
        return LayerNorm(dim)
    return nn.Identity()


class Downsample1d(nn.Module):
    """Stride-2 k=3 conv: L -> L/2."""

    def __init__(self, dim):
        super().__init__()
        self.conv = nn.Conv1d(dim, dim, 3, 2, 1)

    def forward(self, x):
        return self.conv(x)


class Upsample1d(nn.Module):
    """Stride-2 k=4 transposed conv: L -> 2L."""

    def __init__(self, dim):
        super().__init__()
        self.conv = nn.ConvTranspose1d(dim, dim, 4, 2, 1)

    def forward(self, x):
        return self.conv(x)


class LinearAttention(nn.Module):
    """Linear attention block (off in every pipeline; PyTorch path only). jannerunet.py:72-95."""

    def __init__(self, dim, heads=4, dim_head=32):
        super().__init__()
        self.norm = LayerNorm(dim)
        self.scale = dim_head ** -0.5
        self.heads = heads
        inner = dim_head * heads
        self.to_qkv = nn.Conv1d(dim, inner * 3, 1, bias=False)
        self.to_out = nn.Conv1d(inner, dim, 1)

    def forward(self, x):
        x = self.norm(x)
        b, _, n = x.shape
        q, k, v = (t.reshape(b, self.heads, -1, n) for t in self.to_qkv(x).chunk(3, dim=1))
        q = q * self.scale
        k = k.softmax(dim=-1)
        ctx = torch.einsum('bhdn,bhen->bhde', k, v)
        out = torch.einsum('bhde,bhdn->bhen', ctx, q).reshape(b, -1, n)
        return self.to_out(out) + x


class ResidualBlock(nn.Module):
    """conv-GN-Mish (+ time bias) -> conv-GN-Mish, plus a 1x1/identity shortcut (jannerunet.py:52-69)."""

    def __init__(self, in_dim: int, out_dim: int, emb_dim: int, kernel_size: int = 3, norm_type: str = "groupnorm"):
        super().__init__()
        self.conv1 = _conv_gn_mish(in_dim, out_dim, kernel_size, norm_type)
        self.conv2 = _conv_gn_mish(out_dim, out_dim, kernel_size, norm_type)
        self.emb_mlp = nn.Sequential(nn.Mish(), nn.Linear(emb_dim, out_dim))
        self.residual_conv = nn.Conv1d(in_dim, out_dim, 1) if in_dim != out_dim else nn.Identity()

    def forward(self, x, emb):
        h = self.conv1(x) + self.emb_mlp(emb).unsqueeze(-1)
        return self.conv2(h) + self.residual_conv(x)


class ChiResidualBlock(nn.Module):
    """Like ``ResidualBlock`` but FiLM-conditioned: scale*h+bias (chiunet.py:13-45)."""

    def __init__(self, in_dim: int, out_dim: int, emb_dim: int, kernel_size: int = 3, cond_predict_scale: bool = False):
        super().__init__()
        self.conv1 = _conv_gn_mish(in_dim, out_dim, kernel_size)
        self.conv2 = _conv_gn_mish(out_dim, out_dim, kernel_size)
        self.cond_predict_scale = cond_predict_scale
        self.out_dim = out_dim
        self.cond_encoder = nn.Sequential(nn.Mish(), nn.Linear(emb_dim, 2 * out_dim if cond_predict_scale else out_dim))
        self.residual_conv = nn.Conv1d(in_dim, out_dim, 1) if in_dim != out_dim else nn.Identity()

    def forward(self, x, emb):
        h = self.conv1(x)
        film = self.cond_encoder(emb)
        if self.cond_predict_scale:
            film = film.reshape(film.shape[0], 2, self.out_dim, 1)
            h = film[:, 0, ...] * h + film[:, 1, ...]
        else:
            h = h + film.unsqueeze(-1)
        return self.conv2(h) + self.residual_conv(x)


def _stage_dims(first: int, model_dim: int, dim_mult):
    dims = [first] + [model_dim * m for m in np.cumprod(dim_mult)]
    return dims, list(zip(dims[:-1], dims[1:]))


class JannerUNet1d(BaseNNDiffusion):
    def __init__(self, in_dim: int, model_dim: int = 32, emb_dim: int = 32, kernel_size: int = 3,
                 dim_mult: List[int] = [1, 2, 2, 2], norm_type: str = "groupnorm", attention: bool = False,
                 timestep_emb_type: str = "positional", timestep_emb_params: Optional[dict] = None):
        super().__init__(emb_dim, timestep_emb_type, timestep_emb_params)
        dims, in_out = _stage_dims(in_dim, model_dim, dim_mult)
        n_res = len(in_out)

        self.map_emb = nn.Sequential(nn.Linear(emb_dim, model_dim * 4), nn.Mish(), nn.Linear(model_dim * 4, model_dim))

        def block(a, b):
            return ResidualBlock(a, b, model_dim, kernel_size, norm_type)

        def attn(d):
            return LinearAttention(d) if attention else nn.Identity()

        self.downs = nn.ModuleList([])
        self.ups = nn.ModuleList([])
        for i, (cin, cout) in enumerate(in_out):
            last = i >= n_res - 1
            self.downs.append(nn.ModuleList([
                block(cin, cout), block(cout, cout), attn(cout),
                nn.Identity() if last else Downsample1d(cout)]))

        mid = dims[-1]
        self.mid_block1 = block(mid, mid)
        self.mid_attn = attn(mid)
        self.mid_block2 = block(mid, mid)

        # NB (SURVEY 8a quirk 8): only n_res-1 up stages exist, so the `last` test never fires
        # and every up stage ends in an Upsample1d.
        for i, (cin, cout) in enumerate(reversed(in_out[1:])):
            last = i >= n_res - 1
            self.ups.append(nn.ModuleList([
                block(cout * 2, cin), block(cin, cin), attn(cin),
                nn.Identity() if last else Upsample1d(cin)]))

        self.final_conv = nn.Sequential(
            nn.Conv1d(model_dim, model_dim, 5, padding=2), get_norm(model_dim, norm_type), nn.Mish(),
            nn.Conv1d(model_dim, in_dim, 1))

    def forward(self, x: torch.Tensor, noise: torch.Tensor, condition: Optional[torch.Tensor] = None):
        """x (b, horizon, in_dim), noise (b,), condition (b, emb_dim)|None -> (b, horizon, in_dim)."""
        assert x.shape[1] & (x.shape[1] - 1) == 0, "Ta dimension must be 2^n"
        x = x.permute(0, 2, 1)

        emb = self.map_noise(noise)
        emb = emb + (condition if condition is not None else torch.zeros_like(emb))
        emb = self.map_emb(emb)

        skips = []
        for res1, res2, attn, down in self.downs:
            x = attn(res2(res1(x, emb), emb))
            skips.append(x)
            x = down(x)

        x = self.mid_block2(self.mid_attn(self.mid_block1(x, emb)), emb)

        for res1, res2, attn, up in self.ups:
            x = torch.cat([x, skips.pop()], dim=1)
            x = up(attn(res2(res1(x, emb), emb)))

        return self.final_conv(x).permute(0, 2, 1)


class ChiUNet1d(BaseNNDiffusion):
    def __init__(self, act_dim: int, obs_dim: int, To: int, model_dim: int = 256, emb_dim: int = 256,
                 kernel_size: int = 5, cond_predict_scale: bool = True, obs_as_global_cond: bool = True,
                 dim_mult: List[int] = [1, 2, 2], timestep_emb_type: str = "positional",
                 timestep_emb_params: Optional[dict] = None):
        super().__init__(emb_dim, timestep_emb_type, timestep_emb_params)
        self.obs_as_global_cond = obs_as_global_cond
        self.model_dim = model_dim
        self.emb_dim = emb_dim

        dims, in_out = _stage_dims(act_dim, model_dim, dim_mult)
        n_res = len(in_out)
        self.map_emb = nn.Sequential(nn.Linear(emb_dim, emb_dim * 4), nn.Mish(), nn.Linear(emb_dim * 4, emb_dim))

        film_dim = emb_dim * 2 if obs_as_global_cond else emb_dim   # cat[time, obs]

        def block(a, b):
            return ChiResidualBlock(a, b, film_dim, kernel_size, cond_predict_scale)

        if obs_as_global_cond:
            self.global_cond_encoder = nn.Linear(To * obs_dim, emb_dim)
            self.local_cond_encoder = None
        else:
            self.global_cond_encoder = None
            self.local_cond_encoder = nn.ModuleList([
                block(obs_dim, model_dim), block(obs_dim, model_dim), Downsample1d(model_dim)])

        self.downs = nn.ModuleList([])
        self.ups = nn.ModuleList([])
        for i, (cin, cout) in enumerate(in_out):
            last = i >= n_res - 1
            self.downs.append(nn.ModuleList([
                block(cin, cout), block(cout, cout), nn.Identity() if last else Downsample1d(cout)]))

        mid = dims[-1]
        self.mids = nn.ModuleList([block(mid, mid), block(mid, mid)])

        for i, (cin, cout) in enumerate(reversed(in_out[1:])):
            last = i >= n_res - 1
            self.ups.append(nn.ModuleList([
                block(cout * 2, cin), block(cin, cin), nn.Identity() if last else Upsample1d(cin)]))

        self.final_conv = nn.Sequential(
            nn.Conv1d(model_dim, model_dim, kernel_size, padding=kernel_size // 2),
            GroupNorm1d(model_dim, 8, 4), nn.Mish(), nn.Conv1d(model_dim, act_dim, 1))

    def forward(self, x: torch.Tensor, noise: torch.Tensor, condition: Optional[torch.Tensor] = None):
        """x (b, Ta, act_dim), noise (b,), condition (b, To, obs_dim) -> (b, Ta, act_dim)."""
        assert x.shape[1] & (x.shape[1] - 1) == 0, "Ta dimension must be 2^n"
        x = x.permute(0, 2, 1)
        emb = self.map_emb(self.map_noise(noise))

        local = None
        if self.obs_as_global_cond:
            # flatten(None) raises TypeError: this net cannot run unconditionally (tests/test_chi_unet.py:29-38)
            obs = self.global_cond_encoder(torch.flatten(condition, 1))
            emb = torch.cat([emb, obs], dim=-1)
        else:
            condition = condition.permute(0, 2, 1)
            assert x.shape[-1] == condition.shape[-1]
            enc1, enc2, enc_down = self.local_cond_encoder
            local = [enc1(condition, emb), enc_down(enc2(condition, emb))]

        skips = []
        for i, (res1, res2, down) in enumerate(self.downs):
            x = res1(x, emb)
            if i == 0 and local is not None:
                x = x + local[0]
            x = res2(x, emb)
            skips.append(x)
            x = down(x)

        for blk in self.mids:
            x = blk(x, emb)

        for i, (res1, res2, up) in enumerate(self.ups):
            x = res1(torch.cat((x, skips.pop()), dim=1), emb)
            if i == len(self.ups) - 1 and local is not None:
                x = x + local[1]
            x = up(res2(x, emb))

        return self.final_conv(x).permute(0, 2, 1)
