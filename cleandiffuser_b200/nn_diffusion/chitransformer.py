"""``ChiTransformer``: the transformer denoiser of Diffusion Policy.

Reference: cleandiffuser/nn_diffusion/chitransformer.py.  Same constructor signature, parameter names and shapes (including
the unused ``cond_encoder`` and the ``mask`` / ``memory_mask`` parameters) so that checkpoints load.

memory = encoder(cat[map_noise(t), obs_emb(condition)] + cond_pos_emb)            (b, 1 + To, d)
h      = act_emb(x) + pos_emb                                                      (b, Ta, d)
h      = TransformerDecoder(h, memory): per layer (norm_first) causal self-attention, cross-attention under the memory mask
         t >= s - 1, exact-GELU MLP
out    = head(ln_f(h))

The engine lowers it with the per-iteration part of the memory (token 0) and the per-trajectory part (tokens 1..To) hoisted
out of the loop as key / value tables (engine/lower.py, ``lower_chitransformer``).
"""
from typing import Optional

import torch
import torch.nn as nn

from .base import BaseNNDiffusion


def _additive_mask(visible: torch.Tensor) -> torch.Tensor:
    """bool visibility -> additive float mask: 0 where visible, -inf elsewhere"""
    return torch.zeros(visible.shape).masked_fill(~visible, float("-inf"))


def causal_mask(Ta: int) -> torch.Tensor:
    """query i sees keys j <= i"""
    i, j = torch.meshgrid(torch.arange(Ta), torch.arange(Ta), indexing="ij")
    return _additive_mask(j <= i)


def memory_mask(Ta: int, To: int) -> torch.Tensor:
    """action token t sees memory token s when t >= s - 1 (memory token 0 is the time token)"""
    t, s = torch.meshgrid(torch.arange(Ta), torch.arange(To + 1), indexing="ij")
    return _additive_mask(t >= s - 1)


class ChiTransformer(BaseNNDiffusion):
    def __init__(self, act_dim: int, obs_dim: int, Ta: int, To: int, d_model: int = 256, nhead: int = 4,
                 num_layers: int = 8, p_drop_emb: float = 0.0, p_drop_attn: float = 0.3, n_cond_layers: int = 0,
                 timestep_emb_type: str = "positional", timestep_emb_params: Optional[dict] = None):
        super().__init__(d_model, timestep_emb_type, timestep_emb_params)
        self.To, self.obs_dim = To, obs_dim
        self.T, self.T_cond = Ta, 1 + To

        self.act_emb = nn.Linear(act_dim, d_model)
        self.pos_emb = nn.Parameter(torch.zeros(1, Ta, d_model))
        self.obs_emb = nn.Linear(obs_dim, d_model)
        self.cond_pos_emb = nn.Parameter(torch.zeros(1, 1 + To, d_model))
        self.drop = nn.Dropout(p_drop_emb)
        # present in the reference's state dict but never called by its forward
        self.cond_encoder = nn.Sequential(nn.Linear(d_model, 4 * d_model), nn.Mish(), nn.Linear(4 * d_model, d_model))

        if n_cond_layers > 0:
            layer = nn.TransformerEncoderLayer(d_model, nhead, 4 * d_model, p_drop_attn, activation="gelu",
                                               batch_first=True, norm_first=True)
            self.encoder = nn.TransformerEncoder(layer, num_layers=n_cond_layers)
        else:
            self.encoder = nn.Sequential(nn.Linear(d_model, 4 * d_model), nn.Mish(), nn.Linear(4 * d_model, d_model))

        layer = nn.TransformerDecoderLayer(d_model, nhead, 4 * d_model, p_drop_attn, activation="gelu",
                                           batch_first=True, norm_first=True)
        self.decoder = nn.TransformerDecoder(layer, num_layers=num_layers)

        self.mask = nn.Parameter(causal_mask(Ta), requires_grad=False)
        self.memory_mask = nn.Parameter(memory_mask(Ta, To), requires_grad=False)

        self.ln_f = nn.LayerNorm(d_model)
        self.head = nn.Linear(d_model, act_dim)
        self._init_weights()

    def _init_weights(self):
        """N(0, 0.02) for Linear / attention projections and both position tables, zero biases, unit LayerNorms."""
        for m in self.modules():
            if isinstance(m, nn.Linear):
                nn.init.normal_(m.weight, mean=0.0, std=0.02)
                if m.bias is not None:
                    nn.init.zeros_(m.bias)
            elif isinstance(m, nn.MultiheadAttention):
                nn.init.normal_(m.in_proj_weight, mean=0.0, std=0.02)
                nn.init.zeros_(m.in_proj_bias)
            elif isinstance(m, nn.LayerNorm):
                nn.init.ones_(m.weight)
                nn.init.zeros_(m.bias)
        nn.init.normal_(self.pos_emb, mean=0.0, std=0.02)
        nn.init.normal_(self.cond_pos_emb, mean=0.0, std=0.02)

    def forward(self, x: torch.Tensor, noise: torch.Tensor, condition: Optional[torch.Tensor] = None):
        """x (b, Ta, act_dim), noise (b,), condition (b, To, obs_dim) | None (zeros) -> (b, Ta, act_dim)."""
        if condition is None:
            condition = torch.zeros((x.shape[0], self.To, self.obs_dim), device=x.device)
        tokens = torch.cat([self.map_noise(noise).unsqueeze(1), self.obs_emb(condition)], dim=1)
        memory = self.encoder(self.drop(tokens + self.cond_pos_emb[:, :tokens.shape[1]]))
        h = self.drop(self.act_emb(x) + self.pos_emb[:, :x.shape[1]])
        h = self.decoder(tgt=h, memory=memory, tgt_mask=self.mask, memory_mask=self.memory_mask)
        return self.head(self.ln_f(h))
