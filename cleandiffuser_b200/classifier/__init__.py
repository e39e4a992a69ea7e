"""Classifiers for classifier guidance: ``logp(x, noise, c)`` and its input gradient ``gradients(x, noise, c)``.

Same surface as the reference's (cleandiffuser/classifier/base.py, rew_classifiers.py, mse_classifier.py,
qgpo_classifier.py): ``model`` is trained, ``model_ema`` (an eval-mode copy updated by ``ema_update``) is what ``logp``
evaluates.  When one of these guides ``sample()``, the engine evaluates the input gradient inside the replayed loop and
``gradients`` is not called:
  - ``CumRewClassifier`` over ``HalfJannerUNet1d``, over ``HalfDiT1d``, or over ``MLPNNClassifier`` with ``out_dim = 1``;
  - ``MSEClassifier`` over ``MLPNNClassifier`` (ReLU, SiLU or Mish hidden layers, identity output), given ``condition_cg``;
  - ``QGPOClassifier`` over ``QGPONNClassifier``, given ``condition_cg``.
Any other classifier keeps a host callback between the denoiser and the update (``engine/lower.py``, ``guidable``).
"""
from copy import deepcopy
from typing import Dict, Optional

import torch
import torch.nn.functional as F


class BaseClassifier:
    def __init__(self, nn_classifier: torch.nn.Module, ema_rate: float = 0.995, grad_clip_norm: Optional[float] = None,
                 optim_params: Optional[dict] = None, device: str = "cpu"):
        if optim_params is None:
            optim_params = {"lr": 2e-4, "weight_decay": 1e-4}
        self.device = device
        self.ema_rate, self.grad_clip_norm = ema_rate, grad_clip_norm
        self.model = nn_classifier.to(device)
        self.model_ema = deepcopy(self.model).eval()
        self.optim = torch.optim.Adam(self.model.parameters(), **optim_params)
        # bumped by every write to model_ema that moves no autograd version counter (ema_update writes through .data, load
        # replaces the values): the engine folds it into the fingerprint of the weights it has packed copies of
        self.weights_epoch = 0

    def eval(self):
        self.model.eval()
        self.model_ema.eval()

    def train(self):
        self.model.train()

    def ema_update(self):
        """model_ema <- rate * model_ema + (1 - rate) * model, written through ``.data``"""
        with torch.no_grad():
            for p, p_ema in zip(self.model.parameters(), self.model_ema.parameters()):
                p_ema.data.mul_(self.ema_rate).add_(p.data, alpha=1. - self.ema_rate)
        self.weights_epoch += 1

    def loss(self, x: torch.Tensor, noise: torch.Tensor, y: torch.Tensor):
        raise NotImplementedError

    def update(self, x: torch.Tensor, noise: torch.Tensor, y: torch.Tensor, update_ema: bool = True):
        loss = self.loss(x, noise, y)
        self.optim.zero_grad()
        loss.backward()
        grad_norm = None
        if isinstance(self.grad_clip_norm, float):
            grad_norm = torch.nn.utils.clip_grad_norm_(self.model.parameters(), self.grad_clip_norm).item()
        self.optim.step()
        if update_ema:
            self.ema_update()
        return {"loss": loss.item(), "grad_norm": grad_norm}

    def logp(self, x: torch.Tensor, noise: torch.Tensor, c: torch.Tensor):
        """log p(c | x_t, noise) + const, (batch, 1)"""
        raise NotImplementedError

    def gradients(self, x: torch.Tensor, noise: torch.Tensor, c: torch.Tensor):
        """(logp, d sum(logp) / d x), both detached"""
        x.requires_grad_()
        logp = self.logp(x, noise, c)
        grad = torch.autograd.grad([logp.sum()], [x])[0]
        x.detach()
        return logp.detach(), grad.detach()

    def save(self, path):
        torch.save({"model": self.model.state_dict(), "model_ema": self.model_ema.state_dict()}, path)

    def load(self, path):
        ckpt = torch.load(path, map_location=self.device)
        self.model.load_state_dict(ckpt["model"])
        self.model_ema.load_state_dict(ckpt["model_ema"])
        self.weights_epoch += 1


class CumRewClassifier(BaseClassifier):
    """Regresses the cumulative reward R of a trajectory: ``loss = mean((model(x, noise) - R)^2)``, ``logp = model_ema(x, noise)``."""

    def __init__(self, nn_classifier: torch.nn.Module, device: str = "cpu", optim_params: Optional[dict] = None):
        super().__init__(nn_classifier, 0.995, None, optim_params, device)

    def loss(self, x, noise, R):
        return ((self.model(x, noise, None) - R) ** 2).mean()

    def update(self, x, noise, R):
        self.optim.zero_grad()
        loss = self.loss(x, noise, R)
        loss.backward()
        self.optim.step()
        self.ema_update()
        return {"loss": loss.item()}

    def logp(self, x, noise, c=None):
        return self.model_ema(x, noise)


class MSEClassifier(BaseClassifier):
    """Gaussian log-likelihood of a condition c under a regression network (mse_classifier.py):
    ``logp = -temperature * mean((model_ema(x, noise) - c)^2, -1)``, trained with ``mse_loss(model(x, noise), y)``.
    ``temperature`` is a plain attribute; a guided ``sample()`` reads it on every call."""

    def __init__(self, nn_classifier: torch.nn.Module, temperature: float = 1.0, ema_rate: float = 0.995,
                 grad_clip_norm: Optional[float] = None, optim_params: Optional[dict] = None, device: str = "cpu"):
        super().__init__(nn_classifier, ema_rate, grad_clip_norm, optim_params, device)
        self.temperature = temperature

    def loss(self, x: torch.Tensor, noise: torch.Tensor, y: torch.Tensor):
        return F.mse_loss(self.model(x, noise), y)

    def logp(self, x: torch.Tensor, noise: torch.Tensor, c: torch.Tensor):
        """x (batch, x_dim), noise (batch,), c (batch, out_dim) -> (batch, 1)"""
        pred_y = self.model_ema(x, noise)
        return -self.temperature * ((pred_y - c) ** 2).mean(-1, keepdim=True)


class QGPOClassifier(BaseClassifier):
    """QGPO's energy guidance f_phi (qgpo_classifier.py; https://arxiv.org/abs/2304.12824): ``logp = model_ema(x, t, obs)``,
    trained with the in-support contrastive energy prediction loss over K support actions per observation."""

    def loss(self, x: torch.Tensor, t: torch.Tensor, y: Dict[str, torch.Tensor]):
        """x (batch, K, act_dim) noisy support actions, t (batch,), y = {"soft_label": (batch, K, 1) softmax of Q values,
        "obs": (batch, obs_dim)} -> (loss, {f_max, f_mean, f_min})"""
        b, k = x.shape[:2]
        soft_label, obs = y["soft_label"], y["obs"]
        f = self.model(x, t.unsqueeze(1).repeat(1, k), obs.unsqueeze(1).repeat(1, k, 1))
        loss = -(soft_label * F.log_softmax(f, 1)).sum(1).mean()
        with torch.no_grad():
            f_max, f_mean, f_min = f.max(1)[0].mean().item(), f.mean().item(), f.min(1)[0].mean().item()
        return loss, {"f_max": f_max, "f_mean": f_mean, "f_min": f_min}

    def update(self, x: torch.Tensor, noise: torch.Tensor, y: Dict[str, torch.Tensor], update_ema: bool = True):
        loss, log = self.loss(x, noise, y)
        self.optim.zero_grad()
        loss.backward()
        grad_norm = None
        if isinstance(self.grad_clip_norm, float):
            grad_norm = torch.nn.utils.clip_grad_norm_(self.model.parameters(), self.grad_clip_norm).item()
        self.optim.step()
        if update_ema:
            self.ema_update()
        log.update({"loss": loss.item(), "grad_norm": grad_norm})
        return log

    def logp(self, x: torch.Tensor, t: torch.Tensor, c: torch.Tensor):
        """x (batch, act_dim), t (batch,), c (batch, obs_dim) observations -> energy (batch, 1)"""
        return self.model_ema(x, t, c)
