"""``DiscreteRectifiedFlow`` / ``ContinuousRectifiedFlow``: straight-path flow matching with an Euler sampler.

Same constructor / ``loss`` / ``update`` / ``sample`` surface as cleandiffuser/diffusion/rectifiedflow.py (:16-337 discrete,
:340-632 continuous).  SURVEY section 8f rank 3.  The network predicts the velocity x0 - x1; one reverse step is
``x <- x + (t_i - t_{i-1}) * v`` followed by the fix_mask re-imposition -- on the engine that is the SDE classes' update
kernel with the coefficient row (kind CDS_UPD_EPS, K0 = 1, K1 = -(t_i - t_{i-1})): bit-identical fp32 arithmetic, no clipping
inside the loop (the reference clips only the final sample).
"""
from typing import Callable, Optional, Union

import numpy as np
import torch
import torch.nn as nn

from .basic import DiffusionModel
from . import solvers as S
from ..utils import at_least_ndim, SUPPORTED_DISCRETIZATIONS, SUPPORTED_SAMPLING_STEP_SCHEDULE


class _RectifiedFlow(DiffusionModel):
    """What both time parameterisations share: training objective, velocity guidance, the Euler loop and its engine program."""

    @property
    def supported_solvers(self):
        return ["euler"]

    @property
    def clip_pred(self):
        return (self.x_max is not None) or (self.x_min is not None)

    # ---- training ---------------------------------------------------------------------------------------------
    def _sample_training_time(self, n):
        raise NotImplementedError

    def loss(self, x0, x1=None, condition=None):
        if x1 is None:
            x1 = torch.randn_like(x0)
        else:
            assert x0.shape == x1.shape, "x0 and x1 must have the same shape"
        t, t_c = self._sample_training_time(x0.shape[0])
        t_c = at_least_ndim(t_c, x0.dim())
        xt = t_c * x1 + (1 - t_c) * x0
        xt = xt * (1. - self.fix_mask) + x0 * self.fix_mask
        cond = self.model["condition"](condition) if condition is not None else None
        err = (self.model["diffusion"](xt, t, cond) - (x0 - x1)) ** 2
        return (err * self.loss_weight * (1 - self.fix_mask)).mean()

    def update(self, x0, condition=None, update_ema=True, x1=None, **kwargs):
        loss = self.loss(x0, x1, condition)
        loss.backward()
        grad_norm = nn.utils.clip_grad_norm_(self.model.parameters(), self.grad_clip_norm) \
            if self.grad_clip_norm else None
        self.optimizer.step()
        self.optimizer.zero_grad()
        self._weights_epoch += 1
        if update_ema:
            self.ema_update()
        return {"loss": loss.item(), "grad_norm": grad_norm}

    # ---- sampling ---------------------------------------------------------------------------------------------
    def _velocity(self, model, xt, t, cvec, w_cfg):
        net = model["diffusion"]
        if w_cfg != 0.0 and w_cfg != 1.0 and cvec is not None:
            both = net(xt.repeat(*([2] + [1] * (xt.dim() - 1))), t.repeat(2), torch.cat([cvec, torch.zeros_like(cvec)], 0))
            v_c, v_u = both.chunk(2, dim=0)
            return w_cfg * v_c + (1 - w_cfg) * v_u
        if w_cfg == 0.0 or cvec is None:
            return net(xt, t, None)
        return net(xt, t, cvec)

    def _euler_loop(self, *, xt, prior, model, cvec, w_cfg, n_samples, sample_steps, diffusion_x_sampling_steps, t_of, dt_of,
                    t_dtype, requires_grad, preserve_history, log):
        """``t_of(i)`` = the network's time input of loop index i, ``dt_of(i)`` = t_i - t_{i-1} (0-d tensors)."""
        order = list(reversed([1] * diffusion_x_sampling_steps + list(range(1, sample_steps + 1))))
        from ..engine import runtime
        if not preserve_history and runtime._device_ok(torch.device(self.device)):
            rows = torch.zeros((len(order), S.ROW), dtype=torch.float32)
            for n, i in enumerate(order):
                rows[n, S.R_KIND] = float(S.UPD_EPS)
                rows[n, S.R_ALPHA], rows[n, S.R_SIGMA] = 1.0, 1.0
                rows[n, S.R_K0] = 1.0
                rows[n, S.R_K1] = -float(dt_of(i))
            t_all = torch.stack([t_of(i).detach().cpu().to(t_dtype) for i in order])
            eff_w = w_cfg if cvec is not None else 0.0          # (the reference falls back to the unconditional branch)
            # requires_grad=True (flow policies' Q loss through the Euler steps): the differentiable program, whose backward
            # of this EPS-shaped step is CDS_OP_UPDATE_BWD's; the final clip stays a PyTorch op that autograd sees
            engine = runtime.try_sample_grad if requires_grad else runtime.try_sample
            out = engine(self, model=model, xt=xt, prior=prior, solver="rectified_flow_euler", sample_steps=sample_steps,
                         order=order, step_values=None, alphas=None, sigmas=None, hs=None, stds=None, cond_emb=cvec, w_cfg=eff_w,
                         n_samples=n_samples, table=(rows, 0, t_all), clip_in_loop=False, predict_noise=True)
            if out is not None:
                return out
        for i in order:
            t = torch.full((n_samples,), t_of(i), dtype=t_dtype, device=self.device)
            with torch.set_grad_enabled(requires_grad):
                vel = self._velocity(model, xt, t, cvec, w_cfg)
            xt = xt + dt_of(i) * vel
            xt = xt * (1. - self.fix_mask) + prior * self.fix_mask
            if preserve_history:
                log["sample_history"][:, sample_steps - i + 1] = xt.cpu().numpy()
        return xt


def _resolve_schedule(schedule, span, sample_steps):
    if isinstance(schedule, str):
        if schedule not in SUPPORTED_SAMPLING_STEP_SCHEDULE:
            raise ValueError(f"Sampling step schedule {schedule} is not supported.")
        return SUPPORTED_SAMPLING_STEP_SCHEDULE[schedule](span, sample_steps)
    if callable(schedule):
        return schedule(span, sample_steps)
    raise ValueError("sample_step_schedule must be a callable or a string")


class DiscreteRectifiedFlow(_RectifiedFlow):
    def __init__(self, nn_diffusion, nn_condition=None, fix_mask=None, loss_weight=None, classifier=None,
                 grad_clip_norm: Optional[float] = None, ema_rate: float = 0.995, optim_params: Optional[dict] = None,
                 diffusion_steps: int = 1000, discretization: Union[str, Callable] = "uniform",
                 x_max: Optional[torch.Tensor] = None, x_min: Optional[torch.Tensor] = None,
                 device: Union[torch.device, str] = "cpu"):
        super().__init__(nn_diffusion, nn_condition, fix_mask, loss_weight, classifier, grad_clip_norm,
                         diffusion_steps, ema_rate, optim_params, device)
        assert classifier is None, "Rectified Flow does not support classifier-guidance."
        self.x_max = x_max.to(device) if isinstance(x_max, torch.Tensor) else x_max
        self.x_min = x_min.to(device) if isinstance(x_min, torch.Tensor) else x_min
        if isinstance(discretization, str):
            fn = SUPPORTED_DISCRETIZATIONS.get(discretization, SUPPORTED_DISCRETIZATIONS["uniform"])
            self.t_diffusion = fn(diffusion_steps, 0.).to(device)
        elif callable(discretization):
            self.t_diffusion = discretization(diffusion_steps, 0.).to(device)
        else:
            raise ValueError("discretization must be a callable or a string")

    def _sample_training_time(self, n):
        t = torch.randint(self.diffusion_steps, (n,), device=self.device)
        return t, self.t_diffusion[t]

    def sample(self, prior: torch.Tensor, x1: torch.Tensor = None, n_samples: int = 1, sample_steps: int = 5,
               sample_step_schedule: Union[str, Callable] = "uniform", use_ema: bool = True, temperature: float = 1.0,
               condition_cfg=None, mask_cfg=None, w_cfg: float = 0.0, condition_cg=None, w_cg: float = 0.0,
               diffusion_x_sampling_steps: int = 0, warm_start_reference: Optional[torch.Tensor] = None,
               warm_start_forward_level: float = 0.3, requires_grad: bool = False, preserve_history: bool = False, **kwargs):
        assert w_cg == 0.0 and condition_cg is None, "Rectified Flow does not support classifier-guidance."
        prior = prior.to(self.device)
        if isinstance(warm_start_reference, torch.Tensor):
            grid_len = int(warm_start_forward_level * self.diffusion_steps)
            t_c = at_least_ndim(self.t_diffusion[grid_len], prior.dim())
            x1 = torch.randn_like(prior) * t_c + warm_start_reference * (1 - t_c)
        else:
            grid_len = self.diffusion_steps
            if x1 is None:
                x1 = torch.randn_like(prior) * temperature
            else:
                assert prior.shape == x1.shape, "prior and x1 must have the same shape"
        log = {"sample_history": np.empty((n_samples, sample_steps + 1, *prior.shape)) if preserve_history else None}
        model = self.model_ema if use_ema else self.model
        xt = x1.clone() * (1. - self.fix_mask) + prior * self.fix_mask
        if preserve_history:
            log["sample_history"][:, 0] = xt.cpu().numpy()
        with torch.set_grad_enabled(requires_grad):
            cvec = model["condition"](condition_cfg, mask_cfg) if condition_cfg is not None else None
        idx = _resolve_schedule(sample_step_schedule, grid_len, sample_steps)
        xt = self._euler_loop(xt=xt, prior=prior, model=model, cvec=cvec, w_cfg=w_cfg, n_samples=n_samples,
                              sample_steps=sample_steps, diffusion_x_sampling_steps=diffusion_x_sampling_steps,
                              t_of=lambda i: idx[i], dt_of=lambda i: self.t_diffusion[idx[i]] - self.t_diffusion[idx[i - 1]],
                              t_dtype=torch.long, requires_grad=requires_grad, preserve_history=preserve_history, log=log)
        if self.clip_pred:
            xt = xt.clip(self.x_min, self.x_max)
        return xt, log


class ContinuousRectifiedFlow(_RectifiedFlow):
    def __init__(self, nn_diffusion, nn_condition=None, fix_mask=None, loss_weight=None, classifier=None,
                 grad_clip_norm: Optional[float] = None, ema_rate: float = 0.995, optim_params: Optional[dict] = None,
                 x_max: Optional[torch.Tensor] = None, x_min: Optional[torch.Tensor] = None,
                 device: Union[torch.device, str] = "cpu"):
        super().__init__(nn_diffusion, nn_condition, fix_mask, loss_weight, classifier, grad_clip_norm,
                         0, ema_rate, optim_params, device)
        assert classifier is None, "Rectified Flow does not support classifier-guidance."
        self.x_max = x_max.to(device) if isinstance(x_max, torch.Tensor) else x_max
        self.x_min = x_min.to(device) if isinstance(x_min, torch.Tensor) else x_min

    def _sample_training_time(self, n):
        t = torch.rand((n,), device=self.device)
        return t, t

    def sample(self, prior: torch.Tensor, x1: torch.Tensor = None, n_samples: int = 1, sample_steps: int = 5,
               sample_step_schedule: Union[str, Callable] = "uniform_continuous", use_ema: bool = True,
               temperature: float = 1.0, condition_cfg=None, mask_cfg=None, w_cfg: float = 0.0, condition_cg=None,
               w_cg: float = 0.0, diffusion_x_sampling_steps: int = 0, warm_start_reference: Optional[torch.Tensor] = None,
               warm_start_forward_level: float = 0.3, requires_grad: bool = False, preserve_history: bool = False, **kwargs):
        assert w_cg == 0.0 and condition_cg is None, "Rectified Flow does not support classifier-guidance."
        prior = prior.to(self.device)
        warm = isinstance(warm_start_reference, torch.Tensor)
        if warm:
            t_c = torch.ones_like(prior) * warm_start_forward_level
            x1 = torch.randn_like(prior) * t_c + warm_start_reference * (1 - t_c)
        elif x1 is None:
            x1 = torch.randn_like(prior) * temperature
        else:
            assert prior.shape == x1.shape, "prior and x1 must have the same shape"
        log = {"sample_history": np.empty((n_samples, sample_steps + 1, *prior.shape)) if preserve_history else None}
        model = self.model_ema if use_ema else self.model
        xt = x1.clone() * (1. - self.fix_mask) + prior * self.fix_mask
        if preserve_history:
            log["sample_history"][:, 0] = xt.cpu().numpy()
        with torch.set_grad_enabled(requires_grad):
            cvec = model["condition"](condition_cfg, mask_cfg) if condition_cfg is not None else None
        final_t = warm_start_forward_level if (warm and warm_start_forward_level > 0.) else 1.
        ts = _resolve_schedule(sample_step_schedule, [0., final_t], sample_steps)
        xt = self._euler_loop(xt=xt, prior=prior, model=model, cvec=cvec, w_cfg=w_cfg, n_samples=n_samples,
                              sample_steps=sample_steps, diffusion_x_sampling_steps=diffusion_x_sampling_steps,
                              t_of=lambda i: ts[i], dt_of=lambda i: ts[i] - ts[i - 1], t_dtype=torch.float32,
                              requires_grad=requires_grad, preserve_history=preserve_history, log=log)
        if self.clip_pred:
            xt = xt.clip(self.x_min, self.x_max)
        return xt, log
