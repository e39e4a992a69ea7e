"""``ContinuousConsistencyModel``: one/few-step sampler on the EDM (sigma) parameterisation.

Surface of cleandiffuser/diffusion/consistency_model.py:96-428.  ``sample()`` (the latency-floor
config: ONE denoiser evaluation per trajectory) goes through the CUDA engine when it can; the
training side (consistency training with the Nk curriculum, distillation from an EDM teacher) is an
autograd workload and stays PyTorch.

    f(x, s) = c_skip(s) x + c_out(s) net(c_in(s) x, 1/4 ln s, cond),   clipped to [x_min, x_max]
    c_skip = sd^2 / (sd^2 + (s - s_min)^2)
    c_out  = (s - s_min) sd / sqrt(sd^2 + s^2)
    c_in   = 1 / sqrt(sd^2 + s^2)
"""
import math
from typing import Callable, List, Optional, Union

import numpy as np
import torch
import torch.nn as nn

from .basic import DiffusionModel
from . import solvers as S
from ..utils import at_least_ndim


def _erf_as(x):
    """Abramowitz-Stegun 7.1.26 rational approximation (what the reference's curriculum uses)."""
    a = (0.254829592, -0.284496736, 1.421413741, -1.453152027, 1.061405429)
    sgn, x = np.sign(x), np.abs(x)
    t = 1.0 / (1.0 + 0.3275911 * x)
    poly = ((((a[4] * t + a[3]) * t) + a[2]) * t + a[1]) * t + a[0]
    return sgn * (1.0 - poly * t * np.exp(-x * x))


def karras_sigmas(n: int, sigma_min: float, sigma_max: float, rho: float, xp=np, **kw):
    """(s_min^(1/rho) + i/n (s_max^(1/rho) - s_min^(1/rho)))^rho for i = 0..n."""
    lo, hi = sigma_min ** (1 / rho), sigma_max ** (1 / rho)
    return (lo + xp.arange(n + 1, **kw) / n * (hi - lo)) ** rho


def pseudo_huber_loss(source: torch.Tensor, target: torch.Tensor, c: float = 0.0):
    return ((source - target) ** 2 + c ** 2).sqrt() - c


def compare_properties(obj1, obj2, properties: List[str]):
    """Names of attributes that differ between two diffusion objects (tensor / ndarray aware)."""
    bad = []
    for name in properties:
        a, b = getattr(obj1, name), getattr(obj2, name)
        if isinstance(a, torch.Tensor):
            same = torch.allclose(a, b)
        elif isinstance(a, np.ndarray):
            same = np.allclose(a, b)
        else:
            same = a == b
        if not same:
            bad.append(name)
    return bad


class CMCurriculumLogger:
    """Discretisation curriculum of improved consistency training: Nk doubles every K' updates."""

    def __init__(self, s0: int = 10, s1: int = 1280, curriculum_cycle: int = 100_000, sigma_min: float = 0.002,
                 sigma_max: float = 80., rho: float = 7., P_mean: float = -1.1, P_std: float = 2.0):
        self.Kprime = np.ceil(curriculum_cycle / (np.log2(np.ceil(s1 / s0)) + 1))
        self.Nk, self.s0, self.s1 = s0, s0, s1
        self.curriculum_cycle = curriculum_cycle
        self.sigma_min, self.sigma_max, self.rho = sigma_min, sigma_max, rho
        self.P_mean, self.P_std = P_mean, P_std
        self.ceil_k_div_Kprime, self.k = None, None
        self.update_k(0)

    def update_k(self, k):
        self.k = k
        stage = np.ceil(k / self.Kprime)
        if stage == self.ceil_k_div_Kprime:
            return
        self.ceil_k_div_Kprime = stage
        self.Nk = int(min(self.s0 * (2 ** stage), self.s1))
        self.sigmas = karras_sigmas(self.Nk, self.sigma_min, self.sigma_max, self.rho, dtype=np.float32)
        z = (np.log(self.sigmas) - self.P_mean) / (self.P_std * (2 ** 0.5))
        mass = _erf_as(z[1:]) - _erf_as(z[:-1])
        self.p_sigmas = mass / mass.sum()

    def incremental_update_k(self):
        self.update_k(self.k + 1)

    @property
    def curriculum_process(self):
        return (self.k % self.curriculum_cycle) / self.curriculum_cycle


class ContinuousConsistencyModel(DiffusionModel):
    def __init__(self, nn_diffusion, nn_condition=None, fix_mask=None, loss_weight=None, classifier=None,
                 grad_clip_norm: Optional[float] = None, ema_rate: float = 0.9999,
                 optim_params: Optional[dict] = None, s0: int = 10, s1: int = 1280, data_dim: int = None,
                 P_mean: float = -1.1, P_std: float = 2.0, sigma_min: float = 0.002, sigma_max: float = 80.,
                 sigma_data: float = 0.5, rho: float = 7.0, curriculum_cycle: int = 100_000,
                 x_max: Optional[torch.Tensor] = None, x_min: Optional[torch.Tensor] = None,
                 device: Union[torch.device, str] = "cpu"):
        super().__init__(nn_diffusion, nn_condition, fix_mask, loss_weight, classifier, grad_clip_norm,
                         0, ema_rate, optim_params, device)
        self.cur_logger = CMCurriculumLogger(s0, s1, curriculum_cycle, sigma_min, sigma_max, rho, P_mean, P_std)
        self.pseudo_huber_constant = 0.01 if data_dim is None else 0.00054 * np.sqrt(data_dim)
        self.rho = rho
        self.sigma_data, self.sigma_max, self.sigma_min = sigma_data, sigma_max, sigma_min
        self.x_max = x_max.to(device) if isinstance(x_max, torch.Tensor) else x_max
        self.x_min = x_min.to(device) if isinstance(x_min, torch.Tensor) else x_min
        self.edm = None
        self.distillation_sigmas, self.distillation_N = None, None

    @property
    def supported_solvers(self):
        return ["none"]

    @property
    def clip_pred(self):
        return (self.x_max is not None) or (self.x_min is not None)

    # ---- preconditioning (consistency_model.py:241-251) ---------------------------------
    def c_skip(self, sigma):
        return self.sigma_data ** 2 / (self.sigma_data ** 2 + (sigma - self.sigma_min) ** 2)

    def c_out(self, sigma):
        return (sigma - self.sigma_min) * self.sigma_data / (self.sigma_data ** 2 + sigma ** 2).sqrt()

    def c_in(self, sigma):
        return 1 / (self.sigma_data ** 2 + sigma ** 2).sqrt()

    def c_noise(self, sigma):
        return 0.25 * sigma.log()

    def f(self, x, t, condition=None, model=None):
        """The consistency function (consistency_model.py:253-262)."""
        model = self.model if model is None else model
        nd = x.dim()
        skip, out, cin = (at_least_ndim(c, nd) for c in (self.c_skip(t), self.c_out(t), self.c_in(t)))
        pred_x = skip * x + out * model["diffusion"](cin * x, self.c_noise(t), condition)
        return pred_x.clip(self.x_min, self.x_max) if self.clip_pred else pred_x

    # ---- training ------------------------------------------------------------------------
    def training_noise_schedule(self, N):
        sig = karras_sigmas(N, self.sigma_min, self.sigma_max, self.rho)
        return torch.tensor(sig, device=self.device, dtype=torch.float32)

    def prepare_distillation(self, edm, distillation_N: int = 18):
        must_match = ["sigma_data", "sigma_max", "sigma_min", "rho", "x_max", "x_min",
                      "fix_mask", "loss_weight", "device"]
        diff = compare_properties(self, edm, must_match)
        if len(diff) != 0:
            raise ValueError(f"Properties {diff} are different between the EDM and the Consistency Model.")
        self.edm = edm
        self.model.load_state_dict(edm.model.state_dict())
        self.model_ema.load_state_dict(edm.model_ema.state_dict())
        self._engine_plans.clear()
        self.distillation_N = distillation_N
        self.distillation_sigmas = self.training_noise_schedule(distillation_N)

    def distillation_loss(self, x0, condition=None):
        """One Euler step of the teacher's PF-ODE gives the target pair (consistency_model.py:264-293)."""
        assert self.edm is not None, "Please call `prepare_distillation` before distillation."
        idx = torch.randint(self.distillation_N, (x0.shape[0],), device=self.device)
        t_m, t_n = self.distillation_sigmas[idx + 1], self.distillation_sigmas[idx]
        x_m, t_m, _ = self.edm.add_noise(x0, t_m, None)
        with torch.no_grad():
            teacher = self.edm.model_ema
            cvec = teacher["condition"](condition) if condition is not None else None
            pred, _ = self.edm.guided_sampling(x_m, t_m, None, teacher, cvec, 1.0, None, 0.0, False)
            slope = (x_m - pred) / at_least_ndim(t_m, x_m.dim())
            x_n = x_m - slope * at_least_ndim(t_m - t_n, x_m.dim())
            x_n = x_n * (1. - self.fix_mask) + x0 * self.fix_mask
        cvec = self.model["condition"](condition) if condition is not None else None
        pred_m = self.f(x_m, t_m, cvec, self.model)
        with torch.no_grad():
            cvec_ema = self.model_ema["condition"](condition) if condition is not None else None
            pred_n = self.f(x_n, t_n, cvec_ema, self.model_ema)
        loss = (((pred_n - pred_m) ** 2) * (1 - self.fix_mask) * self.loss_weight
                * at_least_ndim((1 / (t_m - t_n)), pred_n.dim()))
        return loss.mean(), None

    def training_loss(self, x0, condition=None):
        """Improved consistency training, adjacent sigmas from the curriculum (consistency_model.py:295-320)."""
        idx = np.random.choice(self.cur_logger.Nk, size=x0.shape[0], p=self.cur_logger.p_sigmas)
        s_n = torch.tensor(self.cur_logger.sigmas[idx], device=self.device)
        s_m = torch.tensor(self.cur_logger.sigmas[idx + 1], device=self.device)
        eps = torch.randn_like(x0)
        x_n = x0 + at_least_ndim(s_n, x0.dim()) * eps
        x_m = x0 + at_least_ndim(s_m, x0.dim()) * eps
        condition = self.model["condition"](condition) if condition is not None else None
        pred_m = self.f(x_m, s_m, condition, self.model)
        with torch.no_grad():
            pred_n = self.f(x_n, s_n, condition.detach(), self.model)
        unweighted = pseudo_huber_loss(pred_m, pred_n, self.pseudo_huber_constant) * (1 - self.fix_mask) * self.loss_weight
        weight = at_least_ndim(1 / (s_m - s_n), x0.dim())
        return (unweighted * weight).mean(), unweighted.mean().item()

    def update(self, x0, condition=None, update_ema=True, loss_type="training", **kwargs):
        if loss_type == "training":
            loss, unweighted = self.training_loss(x0, condition)
        elif loss_type == "distillation":
            loss, unweighted = self.distillation_loss(x0, condition)
        else:
            raise ValueError(f"Unknown loss type: {loss_type}")
        loss.backward()
        grad_norm = nn.utils.clip_grad_norm_(self.model.parameters(), self.grad_clip_norm) \
            if self.grad_clip_norm else None
        self.optimizer.step()
        self.optimizer.zero_grad()
        self._weights_epoch += 1
        if update_ema:
            self.ema_update()
        if loss_type == "training":
            self.cur_logger.incremental_update_k()
        return {"loss": loss.item(), "grad_norm": grad_norm, "unweighted_loss": unweighted}

    # ---- sampling --------------------------------------------------------------------------
    def sample(self, prior: torch.Tensor, solver: str = "none", n_samples: int = 1, sample_steps: int = 5,
               sample_step_schedule: Union[str, Callable] = "uniform", use_ema: bool = True,
               temperature: float = 1.0, condition_cfg=None, mask_cfg=None, w_cfg: float = 0.0,
               condition_cg=None, w_cg: float = 0.0, diffusion_x_sampling_steps: int = 0,
               warm_start_reference: Optional[torch.Tensor] = None, warm_start_forward_level: float = 0.3,
               requires_grad: bool = False, preserve_history: bool = False, **kwargs):
        """x_T ~ N(0, (sigma_max T)^2) -> f(x_T, sigma_max) [-> re-noise to sigma_i -> f ...] (:366-428).
        ``w_cfg`` is ignored exactly like in the reference (the conditional branch is always used)."""
        assert w_cg == 0.0 and condition_cg is None, "Consistency Distillation does not support classifier guidance."
        log = {"sample_history": np.empty((n_samples, sample_steps + 1, *prior.shape)) if preserve_history else None}
        model = self.model_ema if use_ema else self.model

        prior = prior.to(self.device)
        xt = torch.randn_like(prior) * self.sigma_max * temperature
        xt = xt * (1. - self.fix_mask) + prior * self.fix_mask
        if preserve_history:
            log["sample_history"][:, 0] = xt.cpu().numpy()
        with torch.set_grad_enabled(requires_grad):
            cvec = model["condition"](condition_cfg, mask_cfg) if condition_cfg is not None else None

        sigmas = karras_sigmas(sample_steps, self.sigma_min, self.sigma_max, self.rho, xp=torch, device=self.device)
        order = list(reversed([1] * diffusion_x_sampling_steps + list(range(1, sample_steps))))

        from ..engine import runtime
        if requires_grad:
            runtime.grad_fallback(self)
        if not (requires_grad or preserve_history) and runtime._device_ok(torch.device(self.device)):
            out = runtime.try_sample(self, model=model, xt=xt, prior=prior, solver="consistency", sample_steps=sample_steps,
                                     order=order, step_values=None, alphas=None, sigmas=None, hs=None, stds=None, cond_emb=cvec,
                                     w_cfg=1.0 if cvec is not None else 0.0, n_samples=n_samples, predict_noise=False,
                                     consistency=True,
                                     table=lambda: S.consistency_table(sigmas, order, self.sigma_data, self.sigma_min),
                                     sched_id=(int(sample_steps), float(self.sigma_min), float(self.sigma_max), float(self.rho),
                                               int(diffusion_x_sampling_steps), float(self.sigma_data)))
            if out is not None:
                return out, log

        def denoise(x, sigma_value):
            t = torch.full((n_samples,), sigma_value, dtype=torch.float32, device=self.device)
            px = self.f(x, t, cvec, model)
            return px * (1. - self.fix_mask) + prior * self.fix_mask, t

        pred_x, _ = denoise(xt, sigmas[-1])
        for i in order:
            t = torch.full((n_samples,), sigmas[i], dtype=torch.float32, device=self.device)
            xt = pred_x + (at_least_ndim(t, xt.dim()) ** 2 - self.sigma_min ** 2).sqrt() * torch.randn_like(xt)
            pred_x, _ = denoise(xt, sigmas[i])
        return pred_x, log
