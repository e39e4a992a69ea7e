"""``DiffusionModel``: the object every pipeline constructs and drives.

Owns the user's plugins as a genuine ``nn.ModuleDict{"diffusion","condition"}`` plus a
deep-copied EMA twin, the AdamW optimiser, the optional classifier, and the broadcastable
``fix_mask`` / ``loss_weight``.  Pipelines reach into all of these (``actor.model["diffusion"](...)``,
``actor.optimizer.step()``, ``agent.model_ema.train()`` ...), so they are real attributes, not
proxies.  Checkpoints are ``{"model": state_dict, "model_ema": state_dict}``.

Reference: cleandiffuser/diffusion/basic.py:14-103.
"""
from copy import deepcopy
from typing import Optional, Union

import numpy as np
import torch
import torch.nn as nn

from ..nn_condition import BaseNNCondition, IdentityCondition
from ..nn_diffusion import BaseNNDiffusion
from ..utils import to_tensor


class DiffusionModel:
    def __init__(self,
                 nn_diffusion: BaseNNDiffusion,
                 nn_condition: Optional[BaseNNCondition] = None,
                 fix_mask: Union[list, np.ndarray, torch.Tensor] = None,
                 loss_weight: Union[list, np.ndarray, torch.Tensor] = None,
                 classifier=None,
                 grad_clip_norm: Optional[float] = None,
                 diffusion_steps: int = 1000,
                 ema_rate: float = 0.995,
                 optim_params: Optional[dict] = None,
                 device: Union[torch.device, str] = "cpu"):
        self.device = device
        self.grad_clip_norm = grad_clip_norm
        self.diffusion_steps = diffusion_steps
        self.ema_rate = ema_rate

        # No embedder given => the raw condition tensor is the embedding.
        nn_condition = IdentityCondition() if nn_condition is None else nn_condition

        self.model = nn.ModuleDict({
            "diffusion": nn_diffusion.to(self.device),
            "condition": nn_condition.to(self.device)})
        self.model_ema = deepcopy(self.model).requires_grad_(False)
        self.model.train()
        self.model_ema.eval()

        self.optimizer = torch.optim.AdamW(
            self.model.parameters(), **({"lr": 2e-4, "weight_decay": 1e-5} if optim_params is None else optim_params))
        self.classifier = classifier

        # (1, *x_shape) tensors, or the python scalars 0. / 1. when absent
        self.fix_mask = to_tensor(fix_mask, self.device)[None, ] if fix_mask is not None else 0.
        self.loss_weight = to_tensor(loss_weight, self.device)[None, ] if loss_weight is not None else 1.

        # sm_90a sampling plans, keyed by (which weights, shapes, option set); see engine/runtime.py.  The plans hold packed
        # copies of the weights: ``_weights_epoch`` is bumped by everything in this class that mutates parameters (optimiser
        # step, EMA update, checkpoint load) and is part of the version the plans compare before every run.
        self._engine_plans = {}
        self._weights_epoch = 0

    # ---- mode toggles -----------------------------------------------------
    def _classifier_net(self):
        return None if self.classifier is None else self.classifier.model

    def train(self):
        self.model.train()
        if self.classifier is not None:
            self._classifier_net().train()

    def eval(self):
        self.model.eval()
        if self.classifier is not None:
            self._classifier_net().eval()

    # ---- EMA / checkpoints ------------------------------------------------
    def ema_update(self):
        keep = self.ema_rate
        with torch.no_grad():
            for live, avg in zip(self.model.parameters(), self.model_ema.parameters()):
                # in-place on the parameter itself (not ``.data``): bumps its version counter, which the engine's packed-weight
                # cache also watches
                avg.mul_(keep).add_(live.detach(), alpha=1. - keep)
        self._weights_epoch += 1

    def save(self, path: str):
        torch.save({"model": self.model.state_dict(), "model_ema": self.model_ema.state_dict()}, path)

    def load(self, path: str):
        ckpt = torch.load(path, map_location=self.device)
        self.model.load_state_dict(ckpt["model"])
        self.model_ema.load_state_dict(ckpt["model_ema"])
        self._weights_epoch += 1
        self._engine_plans.clear()   # packed weights are stale

    # ---- to be provided by the concrete diffusion process ------------------
    def update(self, x0, condition=None, update_ema=True, **kwargs):
        raise NotImplementedError

    def sample(self, *args, **kwargs):
        raise NotImplementedError
