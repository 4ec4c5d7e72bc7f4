"""CPU float64 ORACLE for the DPM-Solver++ 2M SDE sampler (DPMSolverSampler with eta > 0).  TEST INFRASTRUCTURE ONLY.

A restatement of the midpoint 2M SDE step as k-diffusion's sample_dpmpp_2m_sde states it, in the variance-exploding form: the
state is x~ = x / alpha, the noise level sigma~ = sigma / alpha, and the step from sigma~_s to sigma~_t with h = log sigma~_s -
log sigma~_t (= lambda_t - lambda_s) is

    x~_t = (sigma~_t / sigma~_s) e^{-eta h} x~_s + (1 - e^{-(1 + eta) h}) m0
           + 1/2 (1 - e^{-(1 + eta) h}) (m0 - m1) / r                     (r = h_prev / h; not on a first-order step)
           + sigma~_t sqrt(1 - e^{-2 eta h}) z.

The product expands each step into five coefficients on the VP state x instead (dpm_solver.sde_coefficients); tests compare
the two, so neither is derived from the other.  The step orders are dpm_solver_oracle.orders_for's.
"""
from __future__ import annotations

import math
from typing import List, Optional

import numpy as np
import torch

from oracle import dpm_solver_oracle as DO
from oracle import sampler_oracle as SO


def sde_step_ve(xt, m0, m1, sig_s, sig_t, h_prev, eta: float, z):
    """x~ at sigma~_t from x~ at sigma~_s (VE form).  m1 None: first order.  z None: no noise term.  float64."""
    h = math.log(sig_s) - math.log(sig_t)
    eta_h = eta * h
    big_e = -math.expm1(-h - eta_h)
    x = (sig_t / sig_s) * math.exp(-eta_h) * xt + big_e * m0
    if m1 is not None:
        r = h_prev / h
        x = x + 0.5 * big_e * (1.0 / r) * (m0 - m1)
    if z is not None and eta > 0:
        x = x + z * sig_t * math.sqrt(-math.expm1(-2.0 * eta_h))
    return x


def solve(x, alphas, sigmas, order: int, eta: float, data_pred, draw):
    """The 2M SDE loop over the VP grid (alphas, sigmas) of len n + 1, on the VE state.  data_pred(i, x) -> (x, m) as in
    dpm_solver_oracle.solve (x the VP state); draw(x) -> z after each model pass.  Returns the VP state at the last point."""
    n = len(alphas) - 1
    sig = [s / a for a, s in zip(alphas, sigmas)]
    m_prev, h_prev = None, None
    for i, k in enumerate(DO.orders_for(n, order)):
        x, m = data_pred(i, x)
        z = draw(x)
        xt = sde_step_ve(x / alphas[i], m, m_prev if k >= 2 else None, sig[i], sig[i + 1], h_prev, eta, z)
        x = alphas[i + 1] * xt
        m_prev, h_prev = m, math.log(sig[i]) - math.log(sig[i + 1])
    return x


@torch.no_grad()
def sde_sample(eps_fn: SO.EpsFn, S: int, shape, sched=None, x_T=None, use_cfg=True, guidance_scale=7.5, order: int = 2,
               eta: float = 1.0, alphas: Optional[List[float]] = None, on_alpha=None, mask=None, x0=None, time_range=None):
    """DPMSolverSampler(order, eta).sample on the DDIM uniform grid (or the given time_range, e.g. an image-to-image truncation),
    the last step to alphas_cumprod[0].  Generator draws: randn(shape) when x_T is None; per step the q_sample noise with a mask,
    then one standard normal of the latent's shape (fp32, as randn_like(x) draws it).  UNet in fp32 (eps_fn), solver in float64."""
    sched = sched or SO.make_schedule()
    ac = sched["alphas_cumprod"].double()
    if time_range is None:
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

    return solve(x, al, sg, order, eta, data_pred, lambda xx: torch.randn(tuple(xx.shape)).double()).float()
