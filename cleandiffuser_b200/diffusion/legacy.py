"""The legacy ``DDPM`` and ``EDM`` classes that the ``dp_*`` / ``dbc_*`` pipelines construct.

``DDPM``: beta-schedule parameterisation.

Same constructor / ``add_noise`` / ``loss`` / ``update`` / ``update_classifier`` / ``predict_function`` / ``sample`` /
``sample_x`` surface as cleandiffuser/diffusion/ddpm.py (:17-72 ctor, :81-112 training, :117-165 prediction, :168-253
ancestral sampling, :256-378 Diffusion-X sampling with extra denoising steps at t = 0).  SURVEY section 8f rank 2.

On the engine the ancestral step is the SAME update kernel as the SDE classes' solvers with another coefficient table:
with a_t = alpha_t, ab_t = bar_alpha_t, b_t = beta_t,

    eps-prediction   x <- x / sqrt(a_t)  -  b_t / (sqrt(a_t) sqrt(1 - ab_t)) * eps                       (CDS_UPD_EPS)
    x0-prediction    x <- sqrt(a_t) (1 - ab_{t-1}) / (1 - ab_t) * x  +  b_t sqrt(ab_{t-1}) / (1 - ab_t) * x0   (CDS_UPD_X)
    t > 0            x <- x + sqrt(b_t (1 - ab_{t-1}) / (1 - ab_t)) * z

and the prediction is clipped with (alpha, sigma) = (sqrt(ab_t), sqrt(1 - ab_t)) exactly like BaseDiffusionSDE.clip_prediction.
The reference additionally multiplies the prediction by (1 - fix_mask) (eps) / re-imposes x under the mask (x0) before the
step; both only touch entries that the final ``x (1 - mask) + prior mask`` overwrites, so the engine skips them.

Classifier guidance (ddpm.py:144-149) is added to the raw prediction before the clip, as in the SDE classes: CDS_OP_GUIDE with
the per-iteration scale -(w_cg sqrt(1 - ab_t)) (eps) or w_cg (1 - ab_t) / sqrt(ab_t) (x0) when ``lower.guidable`` accepts the
classifier, else a host callback between the denoiser and the update.  ``log["log_p"]`` is the reference's: the log p of the
last guided evaluation, at the input of the final iteration.
"""
import warnings
from typing import Optional, Union

import numpy as np
import torch
import torch.nn as nn

from .basic import DiffusionModel
from . import solvers as S
from .edm import _guidance_decline
from ..utils import at_least_ndim, cosine_beta_schedule, linear_beta_schedule


class DDPM(DiffusionModel):
    def __init__(self, nn_diffusion, nn_condition=None, fix_mask=None, loss_weight=None, classifier=None,
                 grad_clip_norm: Optional[float] = None, diffusion_steps: int = 1000, ema_rate: float = 0.995,
                 optim_params: Optional[dict] = None, x_max: Optional[torch.Tensor] = None,
                 x_min: Optional[torch.Tensor] = None, predict_noise: bool = True, beta_schedule: str = "cosine",
                 beta_schedule_params: Optional[dict] = None, device: Union[torch.device, str] = "cpu"):
        super().__init__(nn_diffusion, nn_condition, fix_mask, loss_weight, classifier, grad_clip_norm,
                         diffusion_steps, ema_rate, optim_params, device)
        self.predict_noise = predict_noise
        params = dict(beta_schedule_params or {})
        params["T"] = self.diffusion_steps
        if beta_schedule == "linear":
            beta = linear_beta_schedule(**params)
        elif beta_schedule == "cosine":
            beta = cosine_beta_schedule(**params)
        else:
            raise ValueError(f"Unknown beta schedule: {beta_schedule}")
        self.beta = torch.tensor(beta, device=self.device, dtype=torch.float32)
        self.alpha = 1 - self.beta
        self.bar_alpha = torch.cumprod(self.alpha.clone(), 0)
        # (the reference keeps the bounds where the caller put them and fails on a CUDA model with CPU bounds; moved here)
        self.x_max = x_max.to(device) if isinstance(x_max, torch.Tensor) else x_max
        self.x_min = x_min.to(device) if isinstance(x_min, torch.Tensor) else x_min

    @property
    def clip_pred(self):
        return (self.x_max is not None) or (self.x_min is not None)

    # ------------------------------------------------------------------ training (PyTorch / autograd)
    def add_noise(self, x0, t=None, eps=None):
        t = torch.randint(self.diffusion_steps, (x0.shape[0],), device=self.device) if t is None else t
        eps = torch.randn_like(x0) if eps is None else eps
        ab = at_least_ndim(self.bar_alpha[t], x0.dim())
        xt = x0 * ab.sqrt() + eps * (1 - ab).sqrt()
        return xt * (1. - self.fix_mask) + x0 * self.fix_mask, t, eps

    def loss(self, x0, condition=None):
        xt, t, eps = self.add_noise(x0)
        cond = self.model["condition"](condition) if condition is not None else None
        target = eps if self.predict_noise else x0
        err = (self.model["diffusion"](xt, t, cond) - target) ** 2
        return (err * self.loss_weight * (1 - self.fix_mask)).mean()

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
        return self.classifier.update(xt, t, condition)

    # ------------------------------------------------------------------ one guided, clipped prediction (ddpm.py:117-165)
    def predict_function(self, x, t, bar_alpha, use_ema=False, requires_grad=False, condition_vec_cfg=None,
                         w_cfg: float = 0.0, condition_vec_cg=None, w_cg: float = 1.0):
        b = x.shape[0]
        net = (self.model_ema if use_ema else self.model)["diffusion"]
        with torch.set_grad_enabled(requires_grad):
            if w_cfg != 0.0 and w_cfg != 1.0:
                both = net(x.repeat(*([2] + [1] * (x.dim() - 1))), t.repeat(2),
                           torch.cat([condition_vec_cfg, torch.zeros_like(condition_vec_cfg)], 0))
                pred = w_cfg * both[:b] + (1. - w_cfg) * both[b:]
            elif w_cfg == 0.0:
                pred = net(x, t, None)
            else:
                pred = net(x, t, condition_vec_cfg)
        log_p = None
        if self.classifier is not None and w_cg != 0.0 and condition_vec_cg is not None:
            log_p, grad = self.classifier.gradients(x.clone(), t, condition_vec_cg)
            if self.predict_noise:
                pred = pred - w_cg * (1 - bar_alpha).sqrt() * grad
            else:
                pred = pred + w_cg * (1 - bar_alpha) / bar_alpha.sqrt() * grad
        if self.predict_noise:
            if self.clip_pred:
                hi = (x - bar_alpha.sqrt() * self.x_min) / (1 - bar_alpha).sqrt() if self.x_min is not None else None
                lo = (x - bar_alpha.sqrt() * self.x_max) / (1 - bar_alpha).sqrt() if self.x_max is not None else None
                pred = pred.clip(lo, hi)
            pred = pred * (1 - self.fix_mask)
        else:
            if self.clip_pred:
                pred = pred.clip(self.x_min, self.x_max)
            pred = pred * (1 - self.fix_mask) + x * self.fix_mask
        return pred, {"log_p": log_p}

    # ------------------------------------------------------------------ sampling
    def _step_scalars(self, t):
        ab = self.bar_alpha[t]
        ab_prev = self.bar_alpha[t - 1] if t > 0 else torch.tensor(1.0, device=self.device)
        return ab, ab_prev, self.alpha[t], self.beta[t]

    def _ancestral_step(self, xt, pred, t, noise: bool):
        ab, ab_prev, a, b = self._step_scalars(t)
        if self.predict_noise:
            xt = 1 / a.sqrt() * (xt - b / (1 - ab).sqrt() * pred)
        else:
            xt = 1 / (1 - ab) * (a.sqrt() * (1 - ab_prev) * xt + b * ab_prev.sqrt() * pred)
        if noise:
            xt = xt + (b * (1 - ab_prev) / (1 - ab)).sqrt() * torch.randn_like(xt)
        return xt

    def _engine_table(self, extra_steps: int):
        """Per-iteration coefficient rows (engine/solvers row layout) of the T ancestral steps + ``extra_steps`` at t = 0."""
        T = self.diffusion_steps
        ts = list(range(T - 1, -1, -1)) + [0] * extra_steps
        rows = torch.zeros((len(ts), S.ROW), dtype=torch.float32)
        slots = 0
        for n, t in enumerate(ts):
            ab, ab_prev, a, b = (z.detach().float().cpu() for z in self._step_scalars(t))
            rows[n, S.R_ALPHA], rows[n, S.R_SIGMA] = float(ab.sqrt()), float((1 - ab).sqrt())
            if self.predict_noise:
                rows[n, S.R_KIND] = float(S.UPD_EPS)
                rows[n, S.R_K0] = float(1 / a.sqrt())
                rows[n, S.R_K1] = float(1 / a.sqrt() * (b / (1 - ab).sqrt()))
            else:
                rows[n, S.R_KIND] = float(S.UPD_X)
                rows[n, S.R_K0] = float(1 / (1 - ab) * (a.sqrt() * (1 - ab_prev)))
                rows[n, S.R_K1] = float(-(1 / (1 - ab) * (b * ab_prev.sqrt())))
            if t != 0 and n < T:
                slots += 1
                rows[n, S.R_K2] = float((b * (1 - ab_prev) / (1 - ab)).sqrt())
                rows[n, S.R_NOISE] = float(slots)
            rows[n, S.R_T] = float(t)
        return rows, slots, torch.tensor(ts, dtype=torch.long)

    def _sample_impl(self, prior, n_samples, sample_steps, extra_sample_steps, use_ema, temperature, condition_cfg, mask_cfg,
                     w_cfg, condition_cg, w_cg, requires_grad, preserve_history):
        log = {"sample_history": np.empty((n_samples, sample_steps + 1, *prior.shape)) if preserve_history else None}
        model = self.model_ema if use_ema else self.model
        if sample_steps != self.diffusion_steps:
            warnings.warn("sample_steps != diffusion_steps, sample_steps will be set to diffusion_steps.")
            sample_steps = self.diffusion_steps
        xt = torch.randn_like(prior, device=self.device) * temperature
        xt = xt * (1. - self.fix_mask) + prior * self.fix_mask
        if preserve_history:
            log["sample_history"][:, 0] = xt.cpu().numpy()
        with torch.set_grad_enabled(requires_grad):
            cvec = model["condition"](condition_cfg, mask_cfg) if condition_cfg is not None else None

        guided = self.classifier is not None and w_cg != 0.0 and condition_cg is not None
        from ..engine import runtime
        if requires_grad:
            runtime.grad_fallback(self)
        declined = guided and _guidance_decline(requires_grad, preserve_history, w_cfg)
        if declined:
            runtime.guidance_declined(self, declined)
        if not (requires_grad or preserve_history or declined) and runtime._device_ok(torch.device(self.device)):
            rows, slots, t_all = self._engine_table(extra_sample_steps)
            cg, last = {}, {"log_p": None}
            if guided:
                t_dev = t_all.to(self.device)
                with torch.no_grad():                    # the reference's expressions (ddpm.py:144-149) on the device
                    ab = self.bar_alpha[t_dev]
                    scale = -(w_cg * (1 - ab).sqrt()) if self.predict_noise else w_cg * (1 - ab) / ab.sqrt()

                def guide(n, _, x_t, pred):
                    t_batch = t_dev[n].repeat(n_samples)
                    with torch.enable_grad():
                        _, grad = self.classifier.gradients(x_t.clone(), t_batch, condition_cg)
                    with torch.no_grad():
                        pred.copy_(pred + scale[n] * grad)

                def last_input(x):
                    # the reference returns the log p of its last guided evaluation, taken at the final iteration's input
                    with torch.no_grad():
                        last["log_p"] = self.classifier.logp(x, t_dev[-1].repeat(n_samples), condition_cg)
                cg = dict(guide=guide, classifier=self.classifier, w_cg=w_cg, cond_cg=condition_cg, cg_scale=scale,
                          last_input=last_input)
            out = runtime.try_sample(self, model=model, xt=xt, prior=prior.to(self.device), solver="legacy_ddpm",
                                     sample_steps=sample_steps, order=list(range(rows.shape[0])), step_values=None, alphas=None,
                                     sigmas=None, hs=None, stds=None, cond_emb=cvec, w_cfg=w_cfg, n_samples=n_samples,
                                     table=(rows, slots, t_all), **cg)
            if out is not None:
                return out, {**log, "log_p": last["log_p"]}

        extra = {"log_p": None}
        for t in range(self.diffusion_steps - 1, -1, -1):
            t_batch = torch.tensor(t, device=self.device, dtype=torch.long).repeat(n_samples)
            pred, extra = self.predict_function(xt, t_batch, self.bar_alpha[t], use_ema=use_ema, requires_grad=requires_grad,
                                                condition_vec_cfg=cvec, condition_vec_cg=condition_cg, w_cfg=w_cfg, w_cg=w_cg)
            xt = self._ancestral_step(xt, pred, t, noise=t != 0)
            xt = xt * (1. - self.fix_mask) + prior * self.fix_mask
            if preserve_history:
                log["sample_history"][:, 1] = xt.cpu().numpy()
        t_batch = torch.tensor(0, device=self.device, dtype=torch.long).repeat(n_samples)
        for _ in range(extra_sample_steps):
            pred, extra = self.predict_function(xt, t_batch, self.bar_alpha[0], use_ema=use_ema, requires_grad=requires_grad,
                                                condition_vec_cfg=cvec, condition_vec_cg=condition_cg, w_cfg=w_cfg, w_cg=w_cg)
            xt = self._ancestral_step(xt, pred, 0, noise=False)
            xt = xt * (1. - self.fix_mask) + prior * self.fix_mask
        log["log_p"] = extra["log_p"]
        if log["log_p"] is None and self.classifier is not None and condition_cg is not None:
            with torch.no_grad():
                log["log_p"] = self.classifier.logp(xt, t_batch, condition_cg)
        return xt, log

    def sample(self, prior: Optional[torch.Tensor] = None, n_samples: int = 1, sample_steps: int = None, use_ema: bool = True,
               temperature: float = 1.0, condition_cfg=None, mask_cfg=None, w_cfg: float = 0.0, condition_cg=None,
               w_cg: float = 0.0, requires_grad: bool = False, preserve_history: bool = False, **kwargs):
        """Ancestral sampling over all ``diffusion_steps`` steps (ddpm.py:168-253)."""
        return self._sample_impl(prior, n_samples, sample_steps, 0, use_ema, temperature, condition_cfg, mask_cfg, w_cfg,
                                 condition_cg, w_cg, requires_grad, preserve_history)

    def sample_x(self, prior: Optional[torch.Tensor] = None, n_samples: int = 1, sample_steps: int = None,
                 extra_sample_steps: int = 8, use_ema: bool = True, temperature: float = 1.0, condition_cfg=None, mask_cfg=None,
                 w_cfg: float = 0.0, condition_cg=None, w_cg: float = 0.0, requires_grad: bool = False,
                 preserve_history: bool = False, **kwargs):
        """Diffusion-X: ancestral sampling followed by ``extra_sample_steps`` noise-free denoising steps at t = 0
        (ddpm.py:256-378)."""
        return self._sample_impl(prior, n_samples, sample_steps, extra_sample_steps, use_ema, temperature, condition_cfg,
                                 mask_cfg, w_cfg, condition_cg, w_cg, requires_grad, preserve_history)


# ======================================================================================================================
class EDM(DiffusionModel):
    """The legacy ``EDM`` class of the ``dbc_*`` pipelines (cleandiffuser/diffusion/edm.py: ``EDMArchetecture`` :15-355 with the
    ``EDM`` parameterisation :358-428): Karras preconditioning, sigma(t) = t, scale 1, Euler / Heun over a DESCENDING sigma grid
    ``sigma_0 = sigma_max ... sigma_N = sigma_min``, no clipping, slope ``x_weight x - D_weight D`` with both weights ``1/sigma``.

    On the engine this is the ContinuousEDM program (``CDS_OP_PREP`` -> denoiser -> ``CDS_UPD_EDM`` / ``CDS_UPD_EDM_HEUN``) with
    the slope weights passed explicitly (``CDS_ROW_XW`` / ``CDS_ROW_DW``) so that the arithmetic is the reference's."""

    def __init__(self, nn_diffusion, nn_condition=None, fix_mask=None, loss_weight=None, classifier=None,
                 grad_clip_norm: Optional[float] = None, diffusion_steps: int = 1000, ema_rate: float = 0.995,
                 optim_params: Optional[dict] = None, sigma_data: float = 0.5, sigma_min: float = 0.002, sigma_max: float = 80.,
                 rho: float = 7., P_mean: float = -1.2, P_std: float = 1.2, device: Union[torch.device, str] = "cpu"):
        super().__init__(nn_diffusion, nn_condition, fix_mask, loss_weight, classifier, grad_clip_norm,
                         diffusion_steps, ema_rate, optim_params, device)
        self.sigma_data, self.sigma_min, self.sigma_max, self.rho = sigma_data, sigma_min, sigma_max, rho
        self.P_mean, self.P_std = P_mean, P_std
        self.sample_steps = None
        self.sigma_s = self.t_s = self.scale_s = self.dot_sigma_s = self.dot_scale_s = None
        self.x_weight_s = self.D_weight_s = None
        self.x_min = self.x_max = None                      # (no clipping in this class; the engine looks the attributes up)

    # ---- the EDM parameterisation (edm.py:400-428) ------------------------------------------------------------
    def set_sample_steps(self, N: int):
        self.sample_steps = N
        ramp = torch.arange(N + 1, device=self.device) / N
        self.sigma_s = (self.sigma_max ** (1 / self.rho) + ramp * (self.sigma_min ** (1 / self.rho) - self.sigma_max ** (1 / self.rho))) ** self.rho
        self.t_s = self.sigma_s
        self.scale_s = torch.ones_like(self.sigma_s)
        self.dot_sigma_s = torch.ones_like(self.sigma_s)
        self.dot_scale_s = torch.zeros_like(self.sigma_s)
        self.x_weight_s = (self.dot_sigma_s / self.sigma_s + self.dot_scale_s / self.scale_s)
        self.D_weight_s = self.dot_sigma_s / self.sigma_s * self.scale_s

    def c_skip(self, sigma):
        return self.sigma_data ** 2 / (self.sigma_data ** 2 + sigma ** 2)

    def c_out(self, sigma):
        return sigma * self.sigma_data / (self.sigma_data ** 2 + sigma ** 2).sqrt()

    def c_in(self, sigma):
        return 1 / (self.sigma_data ** 2 + sigma ** 2).sqrt()

    def c_noise(self, sigma):
        return 0.25 * sigma.log()

    def loss_weighting(self, sigma):
        return (self.sigma_data ** 2 + sigma ** 2) / ((sigma * self.sigma_data) ** 2)

    def sample_noise_distribution(self, N):
        return (torch.randn(N, device=self.device) * self.P_std + self.P_mean).exp()

    def sample_scale_distribution(self, N):
        return torch.ones(N, device=self.device)

    def D(self, x, sigma, condition=None, use_ema=False):
        net = (self.model_ema if use_ema else self.model)["diffusion"]
        c_noise = at_least_ndim(self.c_noise(sigma).squeeze(), 1)
        return self.c_skip(sigma) * x + self.c_out(sigma) * net(self.c_in(sigma) * x, c_noise, condition)

    # ---- training (edm.py:88-116) -----------------------------------------------------------------------------
    def loss(self, x0, condition=None):
        sigma = at_least_ndim(self.sample_noise_distribution(x0.shape[0]), x0.dim())
        eps = torch.randn_like(x0) * sigma * (1. - self.fix_mask)
        cond = self.model["condition"](condition) if condition is not None else None
        err = self.loss_weighting(sigma) * (self.D(x0 + eps, sigma, cond) - x0) ** 2
        return (err * self.loss_weight).mean()

    def update(self, x0, condition=None, **kwargs):
        self.optimizer.zero_grad()
        loss = self.loss(x0, condition)
        loss.backward()
        grad_norm = nn.utils.clip_grad_norm_(self.model.parameters(), self.grad_clip_norm) \
            if self.grad_clip_norm else None
        self.optimizer.step()
        self._weights_epoch += 1
        self.ema_update()
        return {"loss": loss.item(), "grad_norm": grad_norm}

    def update_classifier(self, x0, condition):
        sigma = at_least_ndim(self.sample_noise_distribution(x0.shape[0]), x0.dim())
        eps = torch.randn_like(x0) * sigma * (1. - self.fix_mask)
        return self.classifier.update(x0 + eps, at_least_ndim(self.c_noise(sigma).squeeze(), 1), condition)

    # ---- sampling (edm.py:118-355) ----------------------------------------------------------------------------
    def dot_x(self, x, i, use_ema=False, condition_vec_cfg=None, w_cfg: float = 0.0, condition_vec_cg=None, w_cg: float = 1.0):
        b = x.shape[0]
        sigma = at_least_ndim(self.sigma_s[i].repeat(b), x.dim())
        unscale = 1. / self.scale_s[i] * (1. - self.fix_mask) + self.fix_mask
        with torch.no_grad():
            if w_cfg != 0.0 and w_cfg != 1.0:
                rep = [2] + [1] * (x.dim() - 1)
                both = self.D((x * unscale).repeat(*rep), sigma.repeat(*rep),
                              torch.cat([condition_vec_cfg, torch.zeros_like(condition_vec_cfg)], 0), use_ema)
                D = w_cfg * both[:b] + (1. - w_cfg) * both[b:]
            elif w_cfg == 0.0:
                D = self.D(x * unscale, sigma, None, use_ema)
            else:
                D = self.D(x * unscale, sigma, condition_vec_cfg, use_ema)
        log_p = None
        if self.classifier is not None and w_cg != 0.0 and condition_vec_cg is not None:
            log_p, grad = self.classifier.gradients(x * unscale, at_least_ndim(self.c_noise(sigma).squeeze(), 1), condition_vec_cg)
            D = D + w_cg * self.scale_s[i] * (sigma ** 2) * grad
        slope = self.x_weight_s[i] * x - self.D_weight_s[i] * D
        return slope * (1. - self.fix_mask), {"log_p": log_p}

    def _reimpose(self, x, prior):
        return x if prior is None else x * (1. - self.fix_mask) + prior * self.fix_mask

    def _sample_impl(self, prior, n_samples, sample_steps, extra_sample_steps, use_ema, solver, condition_cfg, mask_cfg, w_cfg,
                     condition_cg, w_cg, preserve_history):
        if sample_steps != self.sample_steps:
            self.set_sample_steps(sample_steps)
        N = self.sample_steps
        model = self.model_ema if use_ema else self.model
        cvec = model["condition"](condition_cfg, mask_cfg) if condition_cfg is not None else None
        xt = torch.randn_like(prior, device=self.device) * self.sigma_s[0] * self.scale_s[0]
        xt = xt * (1. - self.fix_mask) + prior * self.fix_mask
        x_history = None
        if preserve_history:
            x_history = np.empty((n_samples, N + 1, *xt.shape))
            x_history[:, 0] = xt.cpu().numpy()

        heun_at = [solver == "heun" and i != N - 1 and bool(self.sigma_s[i + 1] > 0.005) for i in range(N)]
        guided = self.classifier is not None and w_cg != 0.0 and condition_cg is not None
        from ..engine import runtime
        if not (preserve_history or guided) and runtime._device_ok(torch.device(self.device)):
            sig, xw, dw = (z.detach().float().cpu() for z in (self.sigma_s, self.x_weight_s, self.D_weight_s))
            evals = []
            for i in list(range(N)) + [N - 1] * extra_sample_steps:
                dt = sig[i] - sig[i + 1]
                heun = heun_at[i]                    # (never at i = N-1, hence never in the extra steps, which repeat it)
                evals.append((sig[i], S.UPD_EDM, dt, 1.0 if heun else 0.0, xw[i], dw[i]))
                if heun:
                    evals.append((sig[i + 1], S.UPD_EDM_HEUN, dt, 0.0, xw[i + 1], dw[i + 1]))
            out = runtime.try_sample(self, model=model, xt=xt, prior=prior.to(self.device),
                                     solver="heun" if any(heun_at) else "euler", sample_steps=N, order=list(range(len(evals))),
                                     step_values=None, alphas=None, sigmas=None, hs=None, stds=None, cond_emb=cvec, w_cfg=w_cfg,
                                     n_samples=n_samples, table=S.edm_table(evals, self.sigma_data), clip_in_loop=False,
                                     predict_noise=False, consistency=True, aux_history=any(heun_at))
            if out is not None:
                return out, {"log_p": None, "sample_history": None}

        log = {"log_p": None}
        for i in range(N):
            d1, log = self.dot_x(xt, i, use_ema, cvec, w_cfg, condition_cg, w_cg)
            dt = self.t_s[i] - self.t_s[i + 1]
            nxt = self._reimpose(xt - d1 * dt, prior)
            if heun_at[i]:
                d2, log = self.dot_x(nxt, i + 1, use_ema, cvec, w_cfg, condition_cg, w_cg)
                nxt = self._reimpose(xt - (d1 + d2) / 2. * dt, prior)
            xt = nxt
            if preserve_history:
                x_history[:, i + 1] = xt.cpu().numpy()
        if extra_sample_steps > 0:
            dt = self.t_s[N - 1] - self.t_s[N]
            for _ in range(extra_sample_steps):
                d1, log = self.dot_x(xt, N - 1, use_ema, cvec, w_cfg, condition_cg, w_cg)
                xt = self._reimpose(xt - d1 * dt, prior)
        log["sample_history"] = x_history
        if log["log_p"] is None and self.classifier is not None and condition_cg is not None:
            with torch.no_grad():
                log["log_p"] = self.classifier.logp(xt, at_least_ndim(self.c_noise(self.sigma_s[-1]).squeeze(), 1), condition_cg)
        return xt, log

    def sample(self, prior: Optional[torch.Tensor] = None, n_samples: int = 1, sample_steps: int = 5, use_ema: bool = True,
               solver: str = "euler", condition_cfg=None, mask_cfg=None, w_cfg: float = 0.0, condition_cg=None, w_cg: float = 0.0,
               preserve_history: bool = False, **kwargs):
        return self._sample_impl(prior, n_samples, sample_steps, 0, use_ema, solver, condition_cfg, mask_cfg, w_cfg, condition_cg,
                                 w_cg, preserve_history)

    def sample_x(self, prior: Optional[torch.Tensor] = None, n_samples: int = 1, sample_steps: int = 5, extra_sample_steps: int = 8,
                 use_ema: bool = True, solver: str = "euler", condition_cfg=None, mask_cfg=None, w_cfg: float = 0.0,
                 condition_cg=None, w_cg: float = 0.0, preserve_history: bool = False, **kwargs):
        return self._sample_impl(prior, n_samples, sample_steps, extra_sample_steps, use_ema, solver, condition_cfg, mask_cfg,
                                 w_cfg, condition_cg, w_cg, preserve_history)
