"""CPU float64 ORACLE for the Karras-grid samplers (DPMSolverSampler / UniPCSampler with grid="karras").  TEST INFRASTRUCTURE ONLY.

Restatements of k-diffusion (Crowson, k_diffusion/sampling.py and external.py), which is not a dependency of this project:

  * get_sigmas_karras(n, sigma_min, sigma_max, rho = 7): (sigma_max^(1/rho) + ramp (sigma_min^(1/rho) - sigma_max^(1/rho)))^rho,
    ramp = linspace(0, 1, n), then a 0 appended;
  * DiscreteSchedule.sigma_to_t: the last discrete log sigma_k not above log sigma (capped at T - 2), and the linear weight in
    log sigma towards the next one, clamped to [0, 1];
  * sample_dpmpp_2m and sample_dpmpp_2m_sde (solver_type "midpoint") in their variance-exploding form: state x~ = x / alpha,
    noise level sigma, the model called at c_in x~ = x~ / sqrt(1 + sigma^2) (the VP state) and t = sigma_to_t(sigma), denoised =
    x~ - sigma eps.  A step to sigma = 0 is denoised itself, and the SDE draws no noise for it.  The step noise is a standard
    normal of the latent's shape drawn after the model pass (k-diffusion's default BrownianTreeNoiseSampler is replaced by the
    plain draws the product makes).

UniPC and the third-order DPM-Solver++ step run oracle/unipc_oracle.py and oracle/dpm_solver_oracle.py on the Karras (alpha, sigma)
points before sigma = 0, then the final step x_S = m_{S-1}.  All runs start from x_T as the VP state at sigma_max (as every sampler of
this project takes x_T; k-diffusion's sigma_max randn in VE form is 0.2 % smaller there), or for image-to-image from
alpha_0 init + sigma_vp,0 noise at the first point run.  The product expands each step into coefficient rows instead
(dpm_solver.grid_coefficients / grid_sde_coefficients, unipc.grid_coefficients); tests compare the two.
"""
from __future__ import annotations

import math
from typing import List, Optional

import torch

from oracle import dpm_solver_oracle as DO
from oracle import sampler_oracle as SO
from oracle import unipc_oracle as UPO


# ---- the schedule -----------------------------------------------------------------------------------------------------------
def discrete_sigmas(alphas_cumprod) -> torch.Tensor:
    ac = alphas_cumprod.double()
    return ((1 - ac) / ac) ** 0.5


def get_sigmas_karras(n: int, sigma_min: float, sigma_max: float, rho: float = 7.0) -> torch.Tensor:
    ramp = torch.linspace(0, 1, n, dtype=torch.float64)
    min_inv_rho = sigma_min ** (1 / rho)
    max_inv_rho = sigma_max ** (1 / rho)
    sigmas = (max_inv_rho + ramp * (min_inv_rho - max_inv_rho)) ** rho
    return torch.cat([sigmas, sigmas.new_zeros([1])])


def sigma_to_t(sigma: torch.Tensor, sigmas: torch.Tensor) -> torch.Tensor:
    log_sigmas = sigmas.log()
    log_sigma = sigma.double().log()
    dists = log_sigma - log_sigmas[:, None]
    low_idx = dists.ge(0).cumsum(dim=0).argmax(dim=0).clamp(max=log_sigmas.shape[0] - 2)
    high_idx = low_idx + 1
    low, high = log_sigmas[low_idx], log_sigmas[high_idx]
    w = ((low - log_sigma) / (low - high)).clamp(0, 1)
    return (1 - w) * low_idx + w * high_idx


def karras_schedule(S: int, sched=None):
    """(sigmas [S + 1] ending in 0, model times [S] of the evaluated points), float64."""
    sched = sched or SO.make_schedule()
    sig = discrete_sigmas(sched["alphas_cumprod"])
    sigmas = get_sigmas_karras(S, float(sig[0]), float(sig[-1]))
    return sigmas, sigma_to_t(sigmas[:-1], sig)


# ---- the VE-form samplers ---------------------------------------------------------------------------------------------------
def sample_dpmpp_2m(data_pred, x, sigmas):
    """k-diffusion's sample_dpmpp_2m.  data_pred(i, x~) -> (x~, denoised) at sigmas[i] (the blend may replace x~)."""
    t_fn = lambda s: -math.log(s)
    old_denoised = None
    for i in range(len(sigmas) - 1):
        x, denoised = data_pred(i, x)
        if sigmas[i + 1] == 0:
            x = denoised
        else:
            t, t_next = t_fn(sigmas[i]), t_fn(sigmas[i + 1])
            h = t_next - t
            if old_denoised is None:
                x = (sigmas[i + 1] / sigmas[i]) * x - math.expm1(-h) * denoised
            else:
                r = (t - t_fn(sigmas[i - 1])) / h
                denoised_d = (1 + 1 / (2 * r)) * denoised - (1 / (2 * r)) * old_denoised
                x = (sigmas[i + 1] / sigmas[i]) * x - math.expm1(-h) * denoised_d
        old_denoised = denoised
    return x


def sample_dpmpp_2m_sde(data_pred, x, sigmas, eta: float, draw):
    """k-diffusion's sample_dpmpp_2m_sde, solver_type "midpoint", s_noise = 1; draw(x) -> a standard normal like x."""
    old_denoised, h_last = None, None
    for i in range(len(sigmas) - 1):
        x, denoised = data_pred(i, x)
        if sigmas[i + 1] == 0:
            x = denoised
        else:
            t, s = -math.log(sigmas[i]), -math.log(sigmas[i + 1])
            h = s - t
            eta_h = eta * h
            x = sigmas[i + 1] / sigmas[i] * math.exp(-eta_h) * x + (-math.expm1(-h - eta_h)) * denoised
            if old_denoised is not None:
                r = h_last / h
                x = x + 0.5 * (-math.expm1(-h - eta_h)) * (1 / r) * (denoised - old_denoised)
            if eta:
                x = x + draw(x) * sigmas[i + 1] * math.sqrt(-math.expm1(-2 * eta_h))
            h_last = h
        old_denoised = denoised
    return x


# ---- the VP-form samplers (DPM-Solver++ of any order, UniPC) -------------------------------------------------------------------
def _orders(n: int, order: int) -> List[int]:
    out = DO.orders_for(n, order)
    out[-1] = 1
    return out


def dpm_vp(data_pred, x, alphas, sigmas, order: int):
    """DPM-Solver++ (dpm_solver_oracle.dpm_step) over the points before sigma = 0, then x_S = m_{S-1}."""
    n = len(alphas) - 1
    orders = _orders(n, order)
    ms: List[torch.Tensor] = []
    for i, k in enumerate(orders):
        x, m = data_pred(i, x)
        if i == n - 1:
            return m
        ms = [m] + ms[:2]
        idx = [i + 1] + [i - j for j in range(k)]
        x = DO.dpm_step(x, ms[:k], [alphas[j] for j in idx], [sigmas[j] for j in idx], k)
    return x


def unipc_vp(data_pred, x, alphas, sigmas, order: int):
    """unipc_oracle.solve over the first n points (the orders of the n-step run), then the last model pass and x_S = m_{S-1}."""
    n = len(alphas) - 1
    orders = _orders(n, order)
    if n > 1:
        x = UPO.solve(x, alphas[:n], sigmas[:n], order, data_pred, orders=orders[:n - 1])
    _, m = data_pred(n - 1, x)
    return m


# ---- the sampler ------------------------------------------------------------------------------------------------------------
@torch.no_grad()
def karras_sample(kind: str, eps_fn: SO.EpsFn, S: int, shape, sched=None, x_T=None, use_cfg=True, guidance_scale=7.5, order: int = 2,
                  eta: float = 0.0, alphas: Optional[List[float]] = None, on_alpha=None, mask=None, x0=None, init=None, noise=None,
                  strength: float = 1.0):
    """kind "dpm2m" (VE, k-diffusion's 2M), "dpm2msde" (VE, 2M SDE at eta), "dpm" (VP, DPM-Solver++ of `order`) or "unipc" (VP) on the
    S-step Karras grid; with init (image-to-image) the last n = min(S, int(strength S)) steps.  Generator draws: per step the blend's
    standard normal with a mask (x0 alpha + sigma_vp z), then for the SDE the step noise, none on the final step.  UNet in fp32
    (eps_fn), solver in float64."""
    sched = sched or SO.make_schedule()
    sigmas, ts = karras_schedule(S, sched)
    if init is not None:
        n = min(S, int(strength * S))
        sigmas, ts = sigmas[S - n:], ts[S - n:]
    sig = [float(v) for v in sigmas]
    al = [1.0 / math.sqrt(1.0 + s * s) for s in sig]
    sg = [s * a for s, a in zip(sig, al)]
    b = shape[0]
    if init is not None:
        x = al[0] * init.double() + sg[0] * noise.double()
    else:
        x = x_T.double()
    use_cfg = use_cfg and guidance_scale != 1

    def data_pred(i, xx):                                        # VP state in, (VP state, data prediction) out
        if alphas is not None and on_alpha is not None:
            on_alpha(alphas[i])
        if mask is not None:
            xx = (al[i] * x0.double() + sg[i] * torch.randn(tuple(x0.shape)).double()) * mask + (1.0 - mask) * xx
        t = torch.full((b,), float(ts[i]), dtype=torch.float64)
        e = SO._cfg_eps(eps_fn, xx.float(), t, use_cfg, guidance_scale).double()
        return xx, (xx - sg[i] * e) / al[i]

    def data_pred_ve(i, xt):
        xx, m = data_pred(i, xt * al[i])
        return xx / al[i], m

    if kind == "dpm2m":
        return sample_dpmpp_2m(data_pred_ve, x / al[0], sig).float()
    if kind == "dpm2msde":
        return sample_dpmpp_2m_sde(data_pred_ve, x / al[0], sig, eta, lambda xx: torch.randn(tuple(xx.shape)).double()).float()
    if kind == "dpm":
        return dpm_vp(data_pred, x, al, sg, order).float()
    if kind == "unipc":
        return unipc_vp(data_pred, x, al, sg, order).float()
    raise ValueError(kind)
