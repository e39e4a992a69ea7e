"""VP diffusion SDE samplers: ``DiscreteDiffusionSDE`` and ``ContinuousDiffusionSDE``.

Same constructor / ``sample()`` / ``update()`` / ``loss()`` / ``add_noise()`` surface as
cleandiffuser/diffusion/diffusionsde.py (:35-245 base, :247-606 discrete, :609-952 continuous).

``sample()`` is a dispatcher.  When the model lives on a CUDA device, the backbone is one the
engine can lower (JannerUNet1d / ChiUNet1d / DiT1d / DQLMlp) and no per-step Python hook is needed
(history capture), the whole reverse loop runs as one replayed CUDA-graph of hand-written sm_90a
kernels with x_t resident on the device (``engine/runtime.py``).  ``requires_grad=True`` (Diffusion-QL
back-propagates through the loop) runs on the engine for DQLMlp with the first-order solvers, a
forward and a backward program (``runtime.try_sample_grad``).  Everything else -- CPU tensors,
user-defined backbones, other ``requires_grad=True`` requests, ``preserve_history`` -- takes the
PyTorch loop below, which is step-for-step the reference algorithm and is pinned against the
reference's goldens on CPU (tests/test_host_golden.py).
"""
from typing import Callable, Dict, Optional, Union

import numpy as np
import torch
import torch.nn as nn

from .basic import DiffusionModel
from . import solvers as S
from .solvers import SUPPORTED_SOLVERS
from ..utils import (at_least_ndim, SUPPORTED_NOISE_SCHEDULES, SUPPORTED_DISCRETIZATIONS,
                     SUPPORTED_SAMPLING_STEP_SCHEDULE)


def epstheta_to_xtheta(x, alpha, sigma, eps_theta):
    return (x - sigma * eps_theta) / alpha


def xtheta_to_epstheta(x, alpha, sigma, x_theta):
    return (x - alpha * x_theta) / sigma


def _resolve_step_schedule(schedule, span, sample_steps):
    if isinstance(schedule, str):
        if schedule not in SUPPORTED_SAMPLING_STEP_SCHEDULE:
            raise ValueError(f"Sampling step schedule {schedule} is not supported.")
        return SUPPORTED_SAMPLING_STEP_SCHEDULE[schedule](span, sample_steps)
    if callable(schedule):
        return schedule(span, sample_steps)
    raise ValueError("sample_step_schedule must be a callable or a string")


class BaseDiffusionSDE(DiffusionModel):
    def __init__(self, nn_diffusion, nn_condition=None, fix_mask=None, loss_weight=None, classifier=None,
                 grad_clip_norm: Optional[float] = None, ema_rate: float = 0.995,
                 optim_params: Optional[dict] = None, epsilon: float = 1e-3,
                 noise_schedule: Union[str, Dict[str, Callable]] = "cosine",
                 noise_schedule_params: Optional[dict] = None,
                 x_max: Optional[torch.Tensor] = None, x_min: Optional[torch.Tensor] = None,
                 predict_noise: bool = True, device: Union[torch.device, str] = "cpu"):
        super().__init__(nn_diffusion, nn_condition, fix_mask, loss_weight, classifier, grad_clip_norm,
                         0, ema_rate, optim_params, device)
        self.predict_noise = predict_noise
        self.epsilon = epsilon
        self.x_max = x_max.to(device) if isinstance(x_max, torch.Tensor) else x_max
        self.x_min = x_min.to(device) if isinstance(x_min, torch.Tensor) else x_min

    @property
    def supported_solvers(self):
        return SUPPORTED_SOLVERS

    @property
    def clip_pred(self):
        return (self.x_max is not None) or (self.x_min is not None)

    # ------------------------------------------------------------------ training
    def add_noise(self, x0, t=None, eps=None):
        raise NotImplementedError

    def _forward_marginal(self, x0, alpha, sigma, eps):
        xt = at_least_ndim(alpha, x0.dim()) * x0 + at_least_ndim(sigma, x0.dim()) * eps
        return (1. - self.fix_mask) * xt + self.fix_mask * x0

    def loss(self, x0, condition=None, **kwargs):
        """Masked, weighted denoising MSE (diffusionsde.py:94-112).  Autograd path: stays PyTorch."""
        xt, t, eps = self.add_noise(x0)
        cond = self.model["condition"](condition) if condition is not None else None
        target = eps if self.predict_noise else x0
        err = (self.model["diffusion"](xt, t, cond) - target) ** 2
        err = err * self.loss_weight * (1 - self.fix_mask)
        wr = kwargs.get("weighted_regression_tensor", None)
        if wr is not None:
            err *= wr.unsqueeze(-1)
        return err.mean()

    def update(self, x0, condition=None, update_ema=True, **kwargs):
        """One optimiser step -> ``{"loss", "grad_norm"}`` (diffusionsde.py:114-141)."""
        loss = self.loss(x0, condition, **kwargs)
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
        out = self.classifier.update(xt, t, condition)
        self._weights_epoch += 1        # the EMA update writes through .data: no version counter moves
        return out

    # ------------------------------------------------------------------ guidance
    def classifier_free_guidance(self, xt, t, model, condition=None, w: float = 1.0,
                                 pred=None, pred_uncond=None, requires_grad: bool = False):
        """``w*pred_cond + (1-w)*pred_uncond`` with the reference's three regimes (diffusionsde.py:175-206):
        w==0 -> unconditional only (condition=None); w==1 -> conditional only; otherwise ONE forward on the
        doubled batch ``[x; x]`` with conditions ``[c; 0]``.  A missing branch is the python float 0."""
        net = model["diffusion"]
        with torch.set_grad_enabled(requires_grad):
            if w != 0.0 and w != 1.0:
                if pred is None or pred_uncond is None:
                    b = xt.shape[0]
                    both = net(xt.repeat(*([2] + [1] * (xt.dim() - 1))), t.repeat(2),
                               torch.cat([condition, torch.zeros_like(condition)], 0))
                    pred, pred_uncond = both[:b], both[b:]
            elif w == 0.0:
                pred, pred_uncond = 0., net(xt, t, None)
            else:
                pred, pred_uncond = net(xt, t, condition), 0.
        return w * pred + (1 - w) * pred_uncond

    def classifier_guidance(self, xt, t, alpha, sigma, model, condition=None, w: float = 1.0, pred=None):
        """eps -= w*sigma*grad  /  x0 += w*sigma^2/alpha*grad  (diffusionsde.py:153-173)."""
        if pred is None:
            pred = model["diffusion"](xt, t, None)
        if self.classifier is None or w == 0.0:
            return pred, None
        log_p, grad = self.classifier.gradients(xt.clone(), t, condition)
        if self.predict_noise:
            pred = pred - w * sigma * grad
        else:
            pred = pred + w * ((sigma ** 2) / alpha) * grad
        return pred, log_p

    def clip_prediction(self, pred, xt, alpha, sigma):
        """Keep the implied x0 inside [x_min, x_max] (diffusionsde.py:208-223)."""
        if not self.clip_pred:
            return pred
        if not self.predict_noise:
            return pred.clip(self.x_min, self.x_max)
        hi = (xt - alpha * self.x_min) / sigma if self.x_min is not None else None
        lo = (xt - alpha * self.x_max) / sigma if self.x_max is not None else None
        return pred.clip(lo, hi)

    def guided_sampling(self, xt, t, alpha, sigma, model, condition_cfg=None, w_cfg: float = 0.0,
                        condition_cg=None, w_cg: float = 0.0, requires_grad: bool = False):
        pred = self.classifier_free_guidance(xt, t, model, condition_cfg, w_cfg, None, None, requires_grad)
        return self.classifier_guidance(xt, t, alpha, sigma, model, condition_cg, w_cg, pred)

    # ------------------------------------------------------------------ sampling (shared)
    def _t_vector(self, n_samples, value):
        raise NotImplementedError

    def _final_logp_wanted(self, w_cg):
        raise NotImplementedError

    def _reverse_loop(self, *, xt, prior, model, solver, sample_steps, step_values, alphas, sigmas,
                      condition_vec_cfg, w_cfg, condition_vec_cg, w_cg, diffusion_x_sampling_steps,
                      requires_grad, preserve_history, n_samples, log, engine_ok, sched_id=None):
        hs, stds = S.schedule_tables(alphas, sigmas, sample_steps, self.device)
        order = S.loop_indices(sample_steps, diffusion_x_sampling_steps)

        if engine_ok and requires_grad:
            # differentiable loop on the engine (Diffusion-QL's actor loss): x0 comes back connected to autograd
            from ..engine import runtime
            out = runtime.try_sample_grad(self, model=model, xt=xt, prior=prior, solver=solver, sample_steps=sample_steps,
                                          order=order, step_values=step_values, alphas=alphas, sigmas=sigmas, hs=hs, stds=stds,
                                          cond_emb=condition_vec_cfg, w_cfg=w_cfg, n_samples=n_samples,
                                          guided=self.classifier is not None and w_cg != 0.0, sched_id=sched_id)
            if out is not None:
                return out
        elif engine_ok:
            from ..engine import runtime
            guide = None
            if self.classifier is not None and w_cg != 0.0:
                # classifier guidance on the engine.  A classifier lower.guidable accepts (CumRewClassifier over HalfJannerUNet1d,
                # HalfDiT1d or MLPNNClassifier, MSEClassifier over MLPNNClassifier, QGPOClassifier over QGPONNClassifier) is lowered into
                # the replayed program (runtime.try_sample); any other classifier runs step by step: the engine evaluates the denoiser, this
                # callback adds the guidance term to the prediction in place (same tensor expression as classifier_guidance
                # above), the engine applies the update.
                def guide(n, i, x_t, pred):
                    t = self._t_vector(n_samples, step_values[i])
                    with torch.enable_grad():
                        _, grad = self.classifier.gradients(x_t.clone(), t, condition_vec_cg)
                    with torch.no_grad():
                        if self.predict_noise:
                            pred.copy_(pred - w_cg * sigmas[i] * grad)
                        else:
                            pred.copy_(pred + w_cg * ((sigmas[i] ** 2) / alphas[i]) * grad)
            out = runtime.try_sample(self, model=model, xt=xt, prior=prior, solver=solver,
                                     sample_steps=sample_steps, order=order, step_values=step_values,
                                     alphas=alphas, sigmas=sigmas, hs=hs, stds=stds,
                                     cond_emb=condition_vec_cfg, w_cfg=w_cfg, n_samples=n_samples, guide=guide, sched_id=sched_id,
                                     classifier=self.classifier, w_cg=w_cg, cond_cg=condition_vec_cg)
            if out is not None:
                return out

        history = [] if S.solver_keeps_history(solver) else None
        for i in order:
            t = self._t_vector(n_samples, step_values[i])
            pred, _ = self.guided_sampling(xt, t, alphas[i], sigmas[i], model, condition_vec_cfg, w_cfg,
                                           condition_vec_cg, w_cg, requires_grad)
            pred = self.clip_prediction(pred, xt, alphas[i], sigmas[i])
            coeffs = S.step_coeffs(solver, i, sample_steps, alphas, sigmas, hs, stds)
            xt = S.apply_update(coeffs, xt, pred, self.predict_noise, torch.randn_like, history)
            xt = xt * (1. - self.fix_mask) + prior * self.fix_mask
            if preserve_history:
                log["sample_history"][:, sample_steps - i + 1] = xt.cpu().numpy()
        return xt

    def _engine_candidate(self, requires_grad, preserve_history, w_cg, warm_start_reference):
        """Cheap host-side screen; the detailed backbone/shape screen lives in engine/runtime.py."""
        if preserve_history:
            return False
        from ..engine import runtime
        return runtime._device_ok(torch.device(self.device))

    def _finish(self, xt, log, n_samples, condition_vec_cg, w_cg):
        if self.classifier is not None and self._final_logp_wanted(w_cg):
            with torch.no_grad():
                t0 = torch.zeros((n_samples,), dtype=torch.long, device=self.device)
                log["log_p"] = self.classifier.logp(xt, t0, condition_vec_cg)
        if self.clip_pred:
            xt = xt.clip(self.x_min, self.x_max)
        return xt, log

    def sample(self, *args, **kwargs):
        raise NotImplementedError


class DiscreteDiffusionSDE(BaseDiffusionSDE):
    """Discrete-time VP-SDE: the network is only defined on ``diffusion_steps`` grid points and is
    queried with int64 timestep indices (diffusionsde.py:247-606)."""

    def __init__(self, nn_diffusion, nn_condition=None, fix_mask=None, loss_weight=None, classifier=None,
                 grad_clip_norm: Optional[float] = None, ema_rate: float = 0.995,
                 optim_params: Optional[dict] = None, epsilon: float = 1e-3, diffusion_steps: int = 1000,
                 discretization: Union[str, Callable] = "uniform",
                 noise_schedule: Union[str, Dict[str, Callable]] = "cosine",
                 noise_schedule_params: Optional[dict] = None,
                 x_max: Optional[torch.Tensor] = None, x_min: Optional[torch.Tensor] = None,
                 predict_noise: bool = True, device: Union[torch.device, str] = "cpu"):
        super().__init__(nn_diffusion, nn_condition, fix_mask, loss_weight, classifier, grad_clip_norm, ema_rate,
                         optim_params, epsilon, noise_schedule, noise_schedule_params, x_max, x_min,
                         predict_noise, device)
        self.diffusion_steps = diffusion_steps
        if 1. / diffusion_steps < epsilon:
            raise ValueError("epsilon is too large for the number of diffusion steps")

        if isinstance(discretization, str):
            grid_fn = SUPPORTED_DISCRETIZATIONS.get(discretization, SUPPORTED_DISCRETIZATIONS["uniform"])
        elif callable(discretization):
            grid_fn = discretization
        else:
            raise ValueError("discretization must be a callable or a string")
        self.t_diffusion = grid_fn(diffusion_steps, epsilon).to(device)

        if isinstance(noise_schedule, str):
            if noise_schedule not in SUPPORTED_NOISE_SCHEDULES:
                raise ValueError(f"Noise schedule {noise_schedule} is not supported.")
            forward = SUPPORTED_NOISE_SCHEDULES[noise_schedule]["forward"]
        elif isinstance(noise_schedule, dict):
            forward = noise_schedule["forward"]
        else:
            raise ValueError("noise_schedule must be a callable or a string")
        self.alpha, self.sigma = forward(self.t_diffusion, **(noise_schedule_params or {}))
        self.logSNR = torch.log(self.alpha / self.sigma)

    def add_noise(self, x0, t=None, eps=None):
        """q(x_t | x_0) at random (or given) grid indices; masked entries keep x0 (:387-397)."""
        if t is None:
            t = torch.randint(self.diffusion_steps, (x0.shape[0],), device=self.device)
        if eps is None:
            eps = torch.randn_like(x0)
        return self._forward_marginal(x0, self.alpha[t], self.sigma[t], eps), t, eps

    def _t_vector(self, n_samples, value):
        return torch.full((n_samples,), value, dtype=torch.long, device=self.device)

    def _final_logp_wanted(self, w_cg):
        return True          # discrete: whenever a classifier is attached (:597)

    def sample(self, prior: torch.Tensor, solver: str = "ddpm", n_samples: int = 1, sample_steps: int = 5,
               sample_step_schedule: Union[str, Callable] = "uniform", use_ema: bool = True,
               temperature: float = 1.0, condition_cfg=None, mask_cfg=None, w_cfg: float = 0.0,
               condition_cg=None, w_cg: float = 0.0, diffusion_x_sampling_steps: int = 0,
               warm_start_reference: Optional[torch.Tensor] = None, warm_start_forward_level: float = 0.3,
               requires_grad: bool = False, preserve_history: bool = False, **kwargs):
        """Run the reverse process from noise (or a forward-noised warm start) -> ``(x0, log)``.

        ``prior`` is ``(n_samples, *x_shape)``; entries where ``fix_mask`` is 1 are re-imposed after every
        step.  Returns x0 on ``self.device`` and ``log`` with ``"sample_history"`` (None or float64 ndarray)
        and, when a classifier is attached, ``"log_p"``."""
        assert solver in SUPPORTED_SOLVERS, f"Solver {solver} is not supported."
        log = {"sample_history": np.empty((n_samples, sample_steps + 1, *prior.shape)) if preserve_history else None}
        model = self.model_ema if use_ema else self.model

        prior = prior.to(self.device)
        if isinstance(warm_start_reference, torch.Tensor):
            grid_len = int(warm_start_forward_level * self.diffusion_steps)
            xt = warm_start_reference * self.alpha[grid_len] + \
                self.sigma[grid_len] * torch.randn_like(warm_start_reference)
        else:
            grid_len = self.diffusion_steps
            xt = torch.randn_like(prior) * temperature
        xt = xt * (1. - self.fix_mask) + prior * self.fix_mask
        if preserve_history:
            log["sample_history"][:, 0] = xt.cpu().numpy()

        with torch.set_grad_enabled(requires_grad):
            cond_vec = model["condition"](condition_cfg, mask_cfg) if condition_cfg is not None else None

        idx = _resolve_step_schedule(sample_step_schedule, grid_len, sample_steps)
        xt = self._reverse_loop(
            xt=xt, prior=prior, model=model, solver=solver, sample_steps=sample_steps, step_values=idx,
            alphas=self.alpha[idx], sigmas=self.sigma[idx], condition_vec_cfg=cond_vec, w_cfg=w_cfg,
            condition_vec_cg=condition_cg, w_cg=w_cg, diffusion_x_sampling_steps=diffusion_x_sampling_steps,
            requires_grad=requires_grad, preserve_history=preserve_history, n_samples=n_samples, log=log,
            engine_ok=self._engine_candidate(requires_grad, preserve_history, w_cg, warm_start_reference),
            # what idx / alphas / sigmas are functions of (named step schedules only): lets the engine reuse its coefficient table
            # without reading the schedule back from the device
            sched_id=(("disc", sample_step_schedule, int(grid_len), self.alpha.data_ptr(), self.alpha._version,
                       self.sigma.data_ptr(), self.sigma._version) if isinstance(sample_step_schedule, str) else None))
        return self._finish(xt, log, n_samples, condition_cg, w_cg)


class ContinuousDiffusionSDE(BaseDiffusionSDE):
    """Continuous-time VP-SDE: the network takes float times in ``[epsilon, 1]`` and the schedule is
    evaluated analytically at the sampling points (diffusionsde.py:609-952)."""

    def __init__(self, nn_diffusion, nn_condition=None, fix_mask=None, loss_weight=None, classifier=None,
                 grad_clip_norm: Optional[float] = None, ema_rate: float = 0.995,
                 optim_params: Optional[dict] = None, epsilon: float = 1e-3,
                 noise_schedule: Union[str, Dict[str, Callable]] = "cosine",
                 noise_schedule_params: Optional[dict] = None,
                 x_max: Optional[torch.Tensor] = None, x_min: Optional[torch.Tensor] = None,
                 predict_noise: bool = True, device: Union[torch.device, str] = "cpu"):
        super().__init__(nn_diffusion, nn_condition, fix_mask, loss_weight, classifier, grad_clip_norm, ema_rate,
                         optim_params, epsilon, noise_schedule, noise_schedule_params, x_max, x_min,
                         predict_noise, device)
        self.t_diffusion = [epsilon, 0.9946] if noise_schedule == "cosine" else [epsilon, 1.]
        if isinstance(noise_schedule, str):
            if noise_schedule not in SUPPORTED_NOISE_SCHEDULES:
                raise ValueError(f"Noise schedule {noise_schedule} is not supported.")
            self.noise_schedule_funcs = SUPPORTED_NOISE_SCHEDULES[noise_schedule]
        elif isinstance(noise_schedule, dict):
            self.noise_schedule_funcs = noise_schedule
        else:
            raise ValueError("noise_schedule must be a callable or a string")
        self.noise_schedule_params = noise_schedule_params

    def _alpha_sigma(self, t):
        return self.noise_schedule_funcs["forward"](t, **(self.noise_schedule_params or {}))

    def add_noise(self, x0, t=None, eps=None):
        """q(x_t | x_0) at uniform random (or given) times (:725-739)."""
        if t is None:
            lo, hi = self.t_diffusion
            t = torch.rand((x0.shape[0],), device=self.device) * (hi - lo) + lo
        if eps is None:
            eps = torch.randn_like(x0)
        alpha, sigma = self._alpha_sigma(t)
        return self._forward_marginal(x0, alpha, sigma, eps), t, eps

    def _t_vector(self, n_samples, value):
        return torch.full((n_samples,), value, dtype=torch.float32, device=self.device)

    def _final_logp_wanted(self, w_cg):
        return w_cg != 0.    # continuous: only when classifier guidance was active (:943)

    def sample(self, prior: torch.Tensor, solver: str = "ddpm", n_samples: int = 1, sample_steps: int = 5,
               sample_step_schedule: Union[str, Callable] = "uniform_continuous", use_ema: bool = True,
               temperature: float = 1.0, condition_cfg=None, mask_cfg=None, w_cfg: float = 0.0,
               condition_cg=None, w_cg: float = 0.0, diffusion_x_sampling_steps: int = 0,
               warm_start_reference: Optional[torch.Tensor] = None, warm_start_forward_level: float = 0.3,
               requires_grad: bool = False, preserve_history: bool = False, **kwargs):
        """Continuous-time counterpart of ``DiscreteDiffusionSDE.sample`` (same arguments / returns)."""
        assert solver in SUPPORTED_SOLVERS, f"Solver {solver} is not supported."
        log = {"sample_history": np.empty((n_samples, sample_steps + 1, *prior.shape)) if preserve_history else None}
        model = self.model_ema if use_ema else self.model

        prior = prior.to(self.device)
        warm = isinstance(warm_start_reference, torch.Tensor) and warm_start_forward_level > 0.
        if warm:
            warm_start_forward_level = self.epsilon + warm_start_forward_level * (1. - self.epsilon)
            a_w, s_w = self._alpha_sigma(torch.ones((1,), device=self.device) * warm_start_forward_level)
            xt = warm_start_reference * a_w + s_w * torch.randn_like(warm_start_reference)
            span = [self.t_diffusion[0], warm_start_forward_level]
        else:
            xt = torch.randn_like(prior) * temperature
            span = self.t_diffusion
        xt = xt * (1. - self.fix_mask) + prior * self.fix_mask
        if preserve_history:
            log["sample_history"][:, 0] = xt.cpu().numpy()

        with torch.set_grad_enabled(requires_grad):
            cond_vec = model["condition"](condition_cfg, mask_cfg) if condition_cfg is not None else None

        times = _resolve_step_schedule(sample_step_schedule, span, sample_steps)
        alphas, sigmas = self._alpha_sigma(times)
        xt = self._reverse_loop(
            xt=xt, prior=prior, model=model, solver=solver, sample_steps=sample_steps, step_values=times,
            alphas=alphas, sigmas=sigmas, condition_vec_cfg=cond_vec, w_cfg=w_cfg,
            condition_vec_cg=condition_cg, w_cg=w_cg, diffusion_x_sampling_steps=diffusion_x_sampling_steps,
            requires_grad=requires_grad, preserve_history=preserve_history, n_samples=n_samples, log=log,
            engine_ok=self._engine_candidate(requires_grad, preserve_history, w_cg, warm_start_reference),
            sched_id=self._schedule_identity(sample_step_schedule, span))
        return self._finish(xt, log, n_samples, condition_cg, w_cg)

    def _schedule_identity(self, sample_step_schedule, span):
        """What (times, alphas, sigmas) are functions of, when that can be named: a named step schedule, the identity of the noise schedule's
        forward function and plain-number parameters.  None otherwise (the engine then reads the schedule back and keys its table on the values)."""
        params = self.noise_schedule_params or {}
        if not isinstance(sample_step_schedule, str) or not all(isinstance(v, (int, float)) for v in params.values()):
            return None
        return ("cont", sample_step_schedule, id(self.noise_schedule_funcs["forward"]), tuple(sorted(params.items())),
                tuple(float(v) for v in span))
