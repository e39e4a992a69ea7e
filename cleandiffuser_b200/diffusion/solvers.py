"""Reverse-process step tables shared by the PyTorch path and the CUDA engine.

The reference writes each solver as one long tensor expression inside the loop
(cleandiffuser/diffusion/diffusionsde.py:539-589, repeated at :885-935).  Every one of
those expressions is "scalars from the (alpha, sigma, h, std) tables" x "a few big
tensors", so we split them: this module evaluates the scalar sub-expressions once per
step, as 0-d fp32 tensors and in the reference's association order, and both back ends
then apply the same five update shapes elementwise:

  UPD_DDPM   x <- k0*(x - sigma_i*eps) + k1*eps                    [+ k2*z]
  UPD_DDIM   x <- k0*((x - sigma_i*eps)/alpha_i) + k1*eps
  UPD_EPS    x <- k0*x - k1*eps                                    [+ k2*z]
  UPD_X      x <- k0*x - k1*xhat                                   [+ k2*z]
  UPD_X2M    D = k3*xhat - k4*xhat_prev ;  x <- k0*x - k1*D        [+ k2*z]

with  eps/xhat  obtained from the (guided, clipped) network prediction by
``xhat = (x - sigma_i*eps)/alpha_i`` or ``eps = (x - alpha_i*xhat)/sigma_i`` (:21-32).
Because the scalar parts are computed exactly like the reference computes them, the
elementwise part differs from it only by fp32 rounding of identical operations.

The engine receives the rows as a ``[n_iters, ROW]`` fp32 table (layout below) and indexes
it with a device-side step counter, so the whole loop replays from one CUDA graph.
"""
from dataclasses import dataclass
from typing import List

import torch

SUPPORTED_SOLVERS = [
    "ddpm", "ddim",
    "ode_dpmsolver_1", "ode_dpmsolver++_1", "ode_dpmsolver++_2M",
    "sde_dpmsolver_1", "sde_dpmsolver++_1", "sde_dpmsolver++_2M", ]

# update shapes (must match enum cds_update_kind in include/cds.h)
UPD_DDPM, UPD_DDIM, UPD_EPS, UPD_X, UPD_X2M, UPD_CM, UPD_EDM, UPD_EDM_HEUN = 0, 1, 2, 3, 4, 5, 6, 7

# row layout of the per-iteration coefficient table (floats)
ROW = 12
(R_ALPHA, R_SIGMA, R_K0, R_K1, R_K2, R_K3, R_K4, R_KIND, R_NOISE, R_T, R_SPARE0, R_SPARE1) = range(ROW)
R_XW, R_DW = R_SPARE0, R_SPARE1          # EDM kinds: explicit slope weights (legacy EDM archetecture)


def solver_draws_noise(solver: str) -> bool:
    return solver == "ddpm" or solver.startswith("sde_")


def solver_keeps_history(solver: str) -> bool:
    return solver.endswith("_2M")


@dataclass
class StepCoeffs:
    """Scalars of one reverse iteration.  ``k*`` are 0-d fp32 tensors (or python floats)."""
    i: int
    kind: int
    alpha: torch.Tensor
    sigma: torch.Tensor
    k0: object = 0.
    k1: object = 0.
    k2: object = 0.
    k3: object = 0.
    k4: object = 0.
    noise: bool = False


def step_coeffs(solver: str, i: int, n_steps: int, alphas, sigmas, hs, stds) -> StepCoeffs:
    """Scalar coefficients of iteration ``i`` (``i`` runs n_steps..1), reference op order."""
    a_i, s_i, a_p, s_p, h = alphas[i], sigmas[i], alphas[i - 1], sigmas[i - 1], hs[i]
    c = StepCoeffs(i=i, kind=UPD_X, alpha=a_i, sigma=s_i)

    if solver == "ddpm":                                   # diffusionsde.py:543-548
        c.kind = UPD_DDPM
        c.k0 = a_p / a_i
        c.k1 = (s_p ** 2 - stds[i] ** 2 + 1e-8).sqrt()
        c.k2 = stds[i]
        c.noise = i > 1
    elif solver == "ddim":                                 # :550-551
        c.kind = UPD_DDIM
        c.k0, c.k1 = a_p, s_p
    elif solver == "ode_dpmsolver_1":                      # :553-554
        c.kind = UPD_EPS
        c.k0 = a_p / a_i
        c.k1 = s_p * torch.expm1(h)
    elif solver == "sde_dpmsolver_1":                      # :568-571
        c.kind = UPD_EPS
        c.k0 = a_p / a_i
        c.k1 = 2 * s_p * torch.expm1(h)
        c.k2 = s_p * torch.expm1(2 * h).sqrt()
        c.noise = True
    elif solver in ("ode_dpmsolver++_1", "ode_dpmsolver++_2M"):   # :556-566
        c.k0 = s_p / s_i
        c.k1 = a_p * torch.expm1(-h)
    elif solver in ("sde_dpmsolver++_1", "sde_dpmsolver++_2M"):   # :573-589
        c.k0 = (s_p / s_i) * (-h).exp()
        c.k1 = a_p * torch.expm1(-2 * h)
        c.k2 = s_p * (-torch.expm1(-2 * h)).sqrt()
        c.noise = True
    else:
        raise AssertionError(f"Solver {solver} is not supported.")

    if solver_keeps_history(solver) and i < n_steps:
        # multistep correction; r may be inf when h_i == 0 (duplicated schedule index): 0.5/inf = 0
        r = hs[i + 1] / h
        c.kind = UPD_X2M
        c.k3 = 1 + 0.5 / r
        c.k4 = 0.5 / r
    return c


def apply_update(c: StepCoeffs, xt, pred, predict_noise: bool, noise_fn, history: List[torch.Tensor]):
    """Elementwise part of one reverse step on PyTorch tensors (the engine mirrors this in CUDA)."""
    if predict_noise:
        eps = pred
        xhat = (xt - c.sigma * pred) / c.alpha
    else:
        xhat = pred
        eps = (xt - c.alpha * pred) / c.sigma

    if c.kind == UPD_DDPM:
        out = c.k0 * (xt - c.sigma * eps) + c.k1 * eps
        if c.noise:
            out += (c.k2 * noise_fn(out))
        return out
    if c.kind == UPD_DDIM:
        return c.k0 * ((xt - c.sigma * eps) / c.alpha) + c.k1 * eps
    if c.kind == UPD_EPS:
        out = c.k0 * xt - c.k1 * eps
    else:
        target = xhat
        if history is not None:
            history.append(xhat)
            if c.kind == UPD_X2M:
                target = c.k3 * history[-1] - c.k4 * history[-2]
        out = c.k0 * xt - c.k1 * target
    if c.noise:
        out = out + c.k2 * noise_fn(xt)
    return out


def loop_indices(sample_steps: int, diffusion_x_sampling_steps: int = 0) -> List[int]:
    """Iteration order S, S-1, ..., 1 followed by the Diffusion-X repeats of step 1 (:525)."""
    return list(reversed([1] * diffusion_x_sampling_steps + list(range(1, sample_steps + 1))))


def schedule_tables(alphas, sigmas, sample_steps: int, device):
    """(hs, stds) exactly as diffusionsde.py:516-520."""
    log_snr = torch.log(alphas / sigmas)
    hs = torch.zeros_like(log_snr)
    hs[1:] = log_snr[:-1] - log_snr[1:]          # hs[0] is meaningless and never read
    stds = torch.zeros((sample_steps + 1,), device=device)
    stds[1:] = sigmas[:-1] / sigmas[1:] * (1 - (alphas[1:] / alphas[:-1]) ** 2).sqrt()
    return hs, stds


def coeff_table(solver: str, order: List[int], n_steps: int, alphas, sigmas, hs, stds, t_values) -> torch.Tensor:
    """Pack the iterations of one ``sample()`` call into the engine's ``[len(order), ROW]`` fp32 table."""
    rows = torch.zeros((len(order), ROW), dtype=torch.float32)
    for n, i in enumerate(order):
        c = step_coeffs(solver, i, n_steps, alphas, sigmas, hs, stds)
        rows[n, R_ALPHA], rows[n, R_SIGMA] = float(c.alpha), float(c.sigma)
        for col, v in ((R_K0, c.k0), (R_K1, c.k1), (R_K2, c.k2), (R_K3, c.k3), (R_K4, c.k4)):
            rows[n, col] = float(v)
        rows[n, R_KIND] = float(c.kind)
        rows[n, R_NOISE] = 1.0 if c.noise else 0.0
        rows[n, R_T] = float(t_values[i])
    return rows


def consistency_table(sigmas, order: List[int], sigma_data, sigma_min):
    """ContinuousConsistencyModel.sample as engine rows -> ``(rows, n_slots, c_noise per iteration)``: iteration 0 evaluates f at
    sigma_max, iteration n > 0 re-noises to sigma_{order[n-1]} with the draw in noise slot n and evaluates f again
    (consistency_model.py:401-426).  The network sees c_noise = ln(sigma)/4 as its "time"."""
    sig = sigmas.detach().float().cpu()
    levels = [sig[-1]] + [sig[i] for i in order]
    sd, smin = sigma_data, sigma_min
    table = torch.zeros((len(levels), ROW), dtype=torch.float32)
    for n, s in enumerate(levels):                     # 0-d fp32 tensors, reference op order (:241-251, :423)
        table[n, R_K0] = float(sd ** 2 / (sd ** 2 + (s - smin) ** 2))                      # c_skip
        table[n, R_K1] = float((s - smin) * sd / (sd ** 2 + s ** 2).sqrt())               # c_out
        table[n, R_K3] = float(1 / (sd ** 2 + s ** 2).sqrt())                              # c_in
        table[n, R_KIND] = float(UPD_CM)
        if n > 0:
            table[n, R_K2] = float((s ** 2 - smin ** 2).sqrt())                            # re-noise scale
            table[n, R_NOISE] = float(n)
        table[n, R_T] = float(0.25 * s.log())                                               # c_noise
    return table, len(levels) - 1, table[:, R_T]


def edm_table(evals, sigma_data):
    """EDM network evaluations as engine rows -> ``(rows, 0 noise slots, c_noise per evaluation)``.  ``evals``: one
    ``(sigma of the evaluation, kind, dt, predictor flag[, x_weight, D_weight])`` per evaluation (UPD_EDM, or UPD_EDM_HEUN for a
    Heun corrector), 0-d fp32 tensors."""
    sd = sigma_data
    table = torch.zeros((len(evals), ROW), dtype=torch.float32)
    for n, ev in enumerate(evals):                         # 0-d fp32 tensors, reference op order (newedm.py:128-148)
        s, kind, dt, pred_flag = ev[:4]
        if len(ev) > 4:
            table[n, R_XW], table[n, R_DW] = float(ev[4]), float(ev[5])
        table[n, R_K0] = float(sd ** 2 / (sd ** 2 + s ** 2))                  # c_skip
        table[n, R_K1] = float(s * sd / (sd ** 2 + s ** 2).sqrt())            # c_out
        table[n, R_K3] = float(1 / (sd ** 2 + s ** 2).sqrt())                 # c_in
        table[n, R_K2] = float(dt)
        table[n, R_K4] = pred_flag
        table[n, R_SIGMA] = float(s)                                          # the slope divides by it
        table[n, R_KIND] = float(kind)
        table[n, R_T] = float(0.25 * s.log())                                 # c_noise
    return table, 0, table[:, R_T]
