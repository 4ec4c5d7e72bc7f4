"""CPU float64 ORACLE for the DPM-Solver++ multistep sampler (ldm/models/diffusion/dpm_solver.py).  TEST INFRASTRUCTURE ONLY.

A restatement of Lu et al. 2022, "DPM-Solver++: Fast Solver for Guided Sampling of Diffusion Probabilistic Models", Algorithm 2
(multistep, data prediction) in the paper's D0 / D1 / D2 form, applied to tensors.  The product expands each step into four
coefficients instead (step_coefficients); tests compare the two, so neither is derived from the other.

Also the analytic test problem: data ~ N(mu, s^2) per element.  Then x_t ~ N(alpha mu, alpha^2 s^2 + sigma^2), the optimal noise
prediction is eps*(x) = sigma (x - alpha mu) / (alpha^2 s^2 + sigma^2), and the probability-flow ODE moves every point along
x(lambda) = alpha mu + sqrt(alpha^2 s^2 + sigma^2) z with its z-score z fixed by the start state.
"""
from __future__ import annotations

import math
from typing import List, Optional

import numpy as np
import torch

from oracle import sampler_oracle as SO


# ---- one step ---------------------------------------------------------------------------------------------------------------
def dpm_step(x, ms, alphas, sigmas, order: int):
    """x at the step's target from x at s0.  ms = [m0, m1, m2] (newest first, as many as the order needs): data predictions at
    s0, s1, s2.  alphas / sigmas = [a_t, a_s0, a_s1, a_s2] (likewise).  float64."""
    lam = [math.log(a / s) for a, s in zip(alphas, sigmas)]
    a_t, s_t, s_s0 = alphas[0], sigmas[0], sigmas[1]
    h = lam[0] - lam[1]
    phi_1 = math.expm1(-h)
    D0 = ms[0]
    if order == 1:
        return (s_t / s_s0) * x - a_t * phi_1 * D0
    r0 = (lam[1] - lam[2]) / h
    D1_0 = (ms[0] - ms[1]) / r0
    if order == 2:
        return (s_t / s_s0) * x - a_t * phi_1 * (D0 + 0.5 * D1_0)
    r1 = (lam[2] - lam[3]) / h
    D1_1 = (ms[1] - ms[2]) / r1
    D1 = D1_0 + r0 / (r0 + r1) * (D1_0 - D1_1)
    D2 = (D1_0 - D1_1) / (r0 + r1)
    phi_2 = phi_1 / h + 1.0
    phi_3 = phi_2 / h - 0.5
    return (s_t / s_s0) * x - a_t * phi_1 * D0 + a_t * phi_2 * D1 - a_t * phi_3 * D2


def orders_for(n: int, order: int) -> List[int]:
    """Order of each of n steps: warm-up min(order, i + 1); a run of fewer than 15 steps ends with order 1, after at most 2."""
    out = []
    for i in range(n):
        k = min(order, i + 1)
        if n < 15 and i == n - 1:
            k = 1
        elif n < 15 and i == n - 2:
            k = min(k, 2)
        out.append(k)
    return out


def solve(x, alphas, sigmas, order: int, data_pred):
    """The multistep loop over a grid of len(alphas) points; data_pred(i, x) -> (x, m): the data prediction m at point i, and x
    as the step starts from it (the inpainting blend replaces it).  float64 scalars."""
    n = len(alphas) - 1
    ms: List[torch.Tensor] = []
    for i, k in enumerate(orders_for(n, order)):
        x, m = data_pred(i, x)
        ms = [m] + ms[:2]
        idx = [i + 1] + [i - j for j in range(k)]
        x = dpm_step(x, ms[:k], [alphas[j] for j in idx], [sigmas[j] for j in idx], k)
    return x


# ---- the analytic problem ---------------------------------------------------------------------------------------------------
def gaussian_eps(x, alpha, sigma, mu, s):
    return sigma * (x - alpha * mu) / (alpha ** 2 * s ** 2 + sigma ** 2)


def gaussian_flow(x_start, alpha0, sigma0, alpha, sigma, mu, s):
    """The exact probability-flow solution at (alpha, sigma) through x_start at (alpha0, sigma0)."""
    z = (x_start - alpha0 * mu) / math.sqrt(alpha0 ** 2 * s ** 2 + sigma0 ** 2)
    return alpha * mu + math.sqrt(alpha ** 2 * s ** 2 + sigma ** 2) * z


def lambda_grid(lam0: float, lam1: float, n: int):
    """(alpha, sigma) of n + 1 lambda-uniform points, alpha^2 + sigma^2 = 1."""
    lam = np.linspace(lam0, lam1, n + 1)
    alpha = 1.0 / np.sqrt(1.0 + np.exp(-2.0 * lam))
    return alpha, alpha * np.exp(-lam)


# ---- the sampler ------------------------------------------------------------------------------------------------------------
@torch.no_grad()
def dpm_sample(eps_fn: SO.EpsFn, S: int, shape, sched=None, x_T=None, use_cfg=True, guidance_scale=7.5, order: int = 2,
               alphas: Optional[List[float]] = None, on_alpha=None, mask=None, x0=None):
    """DPMSolverSampler.sample on the DDIM uniform grid (sampler_oracle.ddim_timesteps), the last step to alphas_cumprod[0].
    Generator draws: randn(shape) when x_T is None, one q_sample noise per step with a mask.  The UNet runs in fp32 (eps_fn);
    the solver arithmetic in float64."""
    sched = sched or SO.make_schedule()
    ac = sched["alphas_cumprod"].double()
    time_range = np.flip(SO.ddim_timesteps(S))
    grid = [float(ac[int(t)]) for t in time_range] + [float(ac[0])]
    al = [math.sqrt(v) for v in grid]
    sg = [math.sqrt(1.0 - v) for v in grid]
    b = shape[0]
    x = (torch.randn(shape) if x_T is None else x_T).double()
    use_cfg = use_cfg and guidance_scale != 1

    def data_pred(i, xx):
        if alphas is not None and on_alpha is not None:
            on_alpha(alphas[i])
        ts = torch.full((b,), int(time_range[i]), dtype=torch.long)
        if mask is not None:
            xx = SO.q_sample(sched, x0, ts).double() * mask + (1.0 - mask) * xx
        e = SO._cfg_eps(eps_fn, xx.float(), ts, use_cfg, guidance_scale).double()
        return xx, (xx - sg[i] * e) / al[i]

    return solve(x, al, sg, order, data_pred).float()
