"""``ContinuousEDM``: Karras et al.'s preconditioned diffusion (sigma(t) = t, scale 1) with Euler / Heun ODE samplers.

Same constructor / ``D`` / ``add_noise`` / ``loss`` / ``update`` / ``update_classifier`` / ``sample`` surface as
cleandiffuser/diffusion/newedm.py (:15-121 ctor, :128-148 preconditioning, :152-215 training, :219-438 sampling).

``sample()`` dispatches like the SDE classes: on a CUDA device with a lowerable backbone and no per-step Python hook the
whole loop runs on the engine -- every network evaluation is one engine iteration of
``CDS_OP_PREP`` (c_in * x) -> denoiser -> ``CDS_OP_UPDATE`` kind ``CDS_UPD_EDM`` / ``CDS_UPD_EDM_HEUN`` (c_skip / c_out
combine, clip, Euler step or Heun corrector, fix_mask) -- otherwise the PyTorch loop below, the reference algorithm step for
step.  The EDM teacher of ``ContinuousConsistencyModel.prepare_distillation`` is an instance of this class.
"""
from typing import Optional, Union

import numpy as np
import torch
import torch.nn as nn

from .basic import DiffusionModel
from . import solvers as S
from ..utils import at_least_ndim


def karras_grid(sample_steps: int, sigma_min: float, sigma_top, rho: float, device=None):
    """sigma_0 = sigma_min ... sigma_S = sigma_top on the rho-warped grid (newedm.py:395-397), fp32 on ``device``."""
    ramp = torch.arange(sample_steps + 1, device=device) / sample_steps
    return (sigma_min ** (1 / rho) + ramp * (sigma_top ** (1 / rho) - sigma_min ** (1 / rho))) ** rho


class ContinuousEDM(DiffusionModel):
    def __init__(self, nn_diffusion, nn_condition=None, fix_mask=None, loss_weight=None, classifier=None,
                 grad_clip_norm: Optional[float] = None, ema_rate: float = 0.995, optim_params: Optional[dict] = None,
                 sigma_data: float = 0.5, sigma_min: float = 0.002, sigma_max: float = 80., rho: float = 7.,
                 P_mean: float = -1.2, P_std: float = 1.2,
                 x_max: Optional[torch.Tensor] = None, x_min: Optional[torch.Tensor] = None,
                 device: Union[torch.device, str] = "cpu"):
        super().__init__(nn_diffusion, nn_condition, fix_mask, loss_weight, classifier, grad_clip_norm,
                         0, ema_rate, optim_params, device)
        self.sigma_data, self.sigma_min, self.sigma_max = sigma_data, sigma_min, sigma_max
        self.rho, self.P_mean, self.P_std = rho, P_mean, P_std
        self.x_max = x_max.to(device) if isinstance(x_max, torch.Tensor) else x_max
        self.x_min = x_min.to(device) if isinstance(x_min, torch.Tensor) else x_min
        self.t_diffusion = [sigma_min, sigma_max]

    @property
    def supported_solvers(self):
        return ["euler", "heun"]

    @property
    def clip_pred(self):
        return (self.x_max is not None) or (self.x_min is not None)

    # ------------------------------------------------------------------ preconditioning (newedm.py:128-148)
    def c_skip(self, sigma):
        return self.sigma_data ** 2 / (self.sigma_data ** 2 + sigma ** 2)

    def c_out(self, sigma):
        return sigma * self.sigma_data / (self.sigma_data ** 2 + sigma ** 2).sqrt()

    def c_in(self, sigma):
        return 1 / (self.sigma_data ** 2 + sigma ** 2).sqrt()

    def c_noise(self, sigma):
        return 0.25 * sigma.log()

    def D(self, x, sigma, condition=None, model=None):
        """Denoiser D(x; sigma) = c_skip x + c_out F(c_in x, c_noise, condition)."""
        model = self.model if model is None else model
        nd = x.dim()
        skip, out, cin = (at_least_ndim(f(sigma), nd) for f in (self.c_skip, self.c_out, self.c_in))
        return skip * x + out * model["diffusion"](cin * x, self.c_noise(sigma), condition)

    # ------------------------------------------------------------------ training (stays PyTorch / autograd)
    def add_noise(self, x0, t=None, eps=None):
        if t is None:
            t = (torch.randn((x0.shape[0],), device=self.device) * self.P_std + self.P_mean).exp()
        eps = torch.randn_like(x0) if eps is None else eps
        xt = x0 + at_least_ndim(t, x0.dim()) * eps
        return (1. - self.fix_mask) * xt + self.fix_mask * x0, t, eps

    def loss(self, x0, condition=None):
        xt, t, _ = self.add_noise(x0)
        cond = self.model["condition"](condition) if condition is not None else None
        err = (self.D(xt, t, cond) - x0) ** 2
        weight = at_least_ndim((t ** 2 + self.sigma_data ** 2) / ((t * self.sigma_data) ** 2), x0.dim())
        return (err * self.loss_weight * (1 - self.fix_mask) * weight).mean()

    def update(self, x0, condition=None, update_ema=True, **kwargs):
        loss = self.loss(x0, condition)
        loss.backward()
        grad_norm = nn.utils.clip_grad_norm_(self.model.parameters(), self.grad_clip_norm) \
            if self.grad_clip_norm else None
        self.optimizer.step()
        self.optimizer.zero_grad()
        self._weights_epoch += 1
        if update_ema:
            self.ema_update()
        return {"loss": loss.item(), "grad_norm": grad_norm}

    def update_classifier(self, x0, condition):
        xt, t, _ = self.add_noise(x0)
        return self.classifier.update(xt, t.log() / 4., condition)

    # ------------------------------------------------------------------ guidance (newedm.py:219-283)
    def classifier_guidance(self, xt, t, sigma, model, condition=None, w: float = 1.0, pred=None):
        if pred is None:
            pred = self.D(xt, t, None, model)
        if self.classifier is None or w == 0.0 or condition is None:
            return pred, None
        log_p, grad = self.classifier.gradients(xt.clone(), t.log() / 4., condition)
        return pred + w * (at_least_ndim(sigma, pred.dim()) ** 2) * grad, log_p

    def classifier_free_guidance(self, xt, t, model, condition=None, w: float = 1.0, pred=None, pred_uncond=None,
                                 requires_grad: bool = False):
        """w == 0: unconditional only; w == 1: conditional only; else ONE evaluation of D on the doubled batch."""
        with torch.set_grad_enabled(requires_grad):
            if w != 0.0 and w != 1.0:
                if pred is None or pred_uncond is None:
                    b = xt.shape[0]
                    both = self.D(xt.repeat(*([2] + [1] * (xt.dim() - 1))), t.repeat(2),
                                  torch.cat([condition, torch.zeros_like(condition)], 0), model)
                    pred, pred_uncond = both[:b], both[b:]
            elif w == 0.0:
                pred, pred_uncond = 0., self.D(xt, t, None, model)
            else:
                pred, pred_uncond = self.D(xt, t, condition, model), 0.
        return w * pred + (1 - w) * pred_uncond

    def guided_sampling(self, xt, t, sigma, model, condition_cfg=None, w_cfg: float = 0.0, condition_cg=None,
                        w_cg: float = 0.0, requires_grad: bool = False):
        pred = self.classifier_free_guidance(xt, t, model, condition_cfg, w_cfg, None, None, requires_grad)
        return self.classifier_guidance(xt, t, sigma, model, condition_cg, w_cg, pred)

    # ------------------------------------------------------------------ sampling (newedm.py:286-438)
    def sample(self, prior: torch.Tensor, solver: str = "euler", n_samples: int = 1, sample_steps: int = 5,
               use_ema: bool = True, temperature: float = 1.0, condition_cfg=None, mask_cfg=None, w_cfg: float = 0.0,
               condition_cg=None, w_cg: float = 0.0, diffusion_x_sampling_steps: int = 0,
               warm_start_reference: Optional[torch.Tensor] = None, warm_start_forward_level: float = 0.3,
               requires_grad: bool = False, preserve_history: bool = False, **kwargs):
        assert solver in ["euler", "heun"], f"Solver {solver} is not supported. Use 'euler' or 'heun' instead."
        log = {"sample_history": np.empty((n_samples, sample_steps + 1, *prior.shape)) if preserve_history else None}
        model = self.model_ema if use_ema else self.model

        prior = prior.to(self.device)
        if isinstance(warm_start_reference, torch.Tensor) and warm_start_forward_level > 0.:
            top = self.sigma_min + (self.sigma_max - self.sigma_min) * warm_start_forward_level
            xt = warm_start_reference + top * torch.randn_like(warm_start_reference)
        else:
            top = self.sigma_max
            xt = torch.randn_like(prior) * self.sigma_max * temperature
        xt = xt * (1. - self.fix_mask) + prior * self.fix_mask
        if preserve_history:
            log["sample_history"][:, 0] = xt.cpu().numpy()
        with torch.set_grad_enabled(requires_grad):
            cvec = model["condition"](condition_cfg, mask_cfg) if condition_cfg is not None else None

        sigmas = karras_grid(sample_steps, self.sigma_min, top, self.rho, self.device)
        order = list(reversed([1] * diffusion_x_sampling_steps + list(range(1, sample_steps + 1))))

        guided = self.classifier is not None and w_cg != 0.0 and condition_cg is not None
        from ..engine import runtime
        done = False
        if requires_grad:
            runtime.grad_fallback(self)
        if not (requires_grad or preserve_history or guided) and runtime._device_ok(torch.device(self.device)):
            def table():
                # every network evaluation is one engine iteration: ``euler`` one per reverse step, ``heun`` a predictor and a
                # corrector for every step but the last
                sig = sigmas.detach().float().cpu()
                evals = []                      # (sigma of the evaluation, kind, dt, predictor flag)
                for i in order:
                    dt = sig[i] - sig[i - 1]
                    heun = solver == "heun" and i > 1
                    evals.append((sig[i], S.UPD_EDM, dt, 1.0 if heun else 0.0))
                    if heun:
                        # the corrector evaluates at t = t_i / sigma_i * sigma_{i-1} (newedm.py:421) = sigma_{i-1} exactly (x / x == 1)
                        evals.append((sig[i - 1], S.UPD_EDM_HEUN, dt, 0.0))
                return S.edm_table(evals, self.sigma_data)
            out = runtime.try_sample(self, model=model, xt=xt, prior=prior, solver=solver, sample_steps=sample_steps, order=order,
                                     step_values=None, alphas=None, sigmas=None, hs=None, stds=None, cond_emb=cvec, w_cfg=w_cfg,
                                     n_samples=n_samples, predict_noise=False, consistency=True, aux_history=solver == "heun",
                                     table=table, sched_id=(int(sample_steps), float(self.sigma_min), float(top), float(self.rho),
                                                            float(self.sigma_data)))
            if out is not None:
                xt, done = out, True

        def slope(x, t_vec, sigma):
            pred, _ = self.guided_sampling(x, t_vec, sigma, model, cvec, w_cfg, condition_cg, w_cg, requires_grad)
            if self.clip_pred:
                pred = pred.clip(self.x_min, self.x_max)
            return (x - pred) / at_least_ndim(sigma, x.dim())

        for i in ([] if done else order):
            t = torch.full((n_samples,), sigmas[i], dtype=torch.float32, device=self.device)
            d_cur = slope(xt, t, sigmas[i])
            dt = sigmas[i] - sigmas[i - 1]
            nxt = (xt - d_cur * dt) * (1. - self.fix_mask) + prior * self.fix_mask
            if solver == "heun" and i > 1:
                d_nxt = slope(nxt, t / sigmas[i] * sigmas[i - 1], sigmas[i - 1])
                nxt = (xt - (d_cur + d_nxt) / 2. * dt) * (1. - self.fix_mask) + prior * self.fix_mask
            xt = nxt
            if preserve_history:
                log["sample_history"][:, sample_steps - i + 1] = xt.cpu().numpy()

        if self.classifier is not None:
            with torch.no_grad():
                t = torch.ones((n_samples,), dtype=torch.long, device=self.device) * self.sigma_min
                log["log_p"] = self.classifier.logp(xt, t.log() / 4., condition_cg)
        if self.clip_pred:
            xt = xt.clip(self.x_min, self.x_max)
        return xt, log
