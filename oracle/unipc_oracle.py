"""CPU float64 ORACLE for the UniPC sampler (ldm/models/diffusion/unipc.py).  TEST INFRASTRUCTURE ONLY.

A restatement of Zhao et al. 2023, "UniPC: A Unified Predictor-Corrector Framework for Fast Sampling of Diffusion Models"
(appendix algorithms, data prediction, B(h) = expm1(-h)), in the paper's r_k / D_k / R / b form applied to tensors.  The product
expands each step into nine coefficients instead (step_coefficients); tests compare the two, so neither is derived from the
other.  The analytic test problem (Gaussian data, exact probability-flow solution) is oracle/dpm_solver_oracle.py's.
"""
from __future__ import annotations

import math
from typing import List, Optional

import numpy as np
import torch

from oracle import dpm_solver_oracle as DO
from oracle import sampler_oracle as SO


# ---- one step ---------------------------------------------------------------------------------------------------------------
def _r_b(lams, p):
    """(h, B, [r_1 .. r_p], R, b) of a step of order p; lams = [lambda_t, lambda_s, lambda_s1, ...] (newest history first)."""
    h = lams[0] - lams[1]
    hh = -h
    phi_1 = math.expm1(hh)
    B = math.expm1(hh)
    rks = [(lams[1 + k] - lams[1]) / h for k in range(1, p)] + [1.0]
    R = np.array([[r ** a for r in rks] for a in range(p)], dtype=np.float64)
    g = [phi_1 / hh - 1.0]                                      # g_1, g_2, ...
    for a in range(1, p):
        g.append(g[-1] / hh - 1.0 / math.factorial(a + 1))
    b = np.array([g[a] * math.factorial(a + 1) / B for a in range(p)])
    return h, B, phi_1, rks, R, b


def _D(ms, rks, p):
    """D_k = (m_{s_k} - m_s) / r_k, k = 1 .. p - 1; ms = [m_s, m_s1, ...]."""
    return [(ms[k] - ms[0]) / rks[k - 1] for k in range(1, p)]


def unip(x_s, ms, lams, alpha_t, sigma_t, sigma_s, p: int):
    """UniP-p: x at t from x at s.  ms = [m_s, m_s1, ..., m_s(p-1)] (newest first), lams = [lambda_t, lambda_s, lambda_s1, ...]."""
    h, B, phi_1, rks, R, b = _r_b(lams, p)
    out = (sigma_t / sigma_s) * x_s - alpha_t * phi_1 * ms[0]
    if p == 1:
        return out
    rho = [0.5] if p == 2 else list(np.linalg.solve(R[:p - 1, :p - 1], b[:p - 1]))
    return out - alpha_t * B * sum(r * d for r, d in zip(rho, _D(ms, rks, p)))


def unic(xc_s, m_t, ms, lams, alpha_t, sigma_t, sigma_s, p: int):
    """UniC-p: the corrected x at t from the corrected x at s, with m_t the data prediction evaluated at t."""
    h, B, phi_1, rks, R, b = _r_b(lams, p)
    rho = [0.5] if p == 1 else list(np.linalg.solve(R, b))
    corr = sum((r * d for r, d in zip(rho[:-1], _D(ms, rks, p))), torch.zeros_like(m_t)) + rho[-1] * (m_t - ms[0])
    return (sigma_t / sigma_s) * xc_s - alpha_t * phi_1 * ms[0] - alpha_t * B * corr


def orders_for(n: int, order: int) -> List[int]:
    """DPM-Solver++'s step orders (oracle/dpm_solver_oracle.py): warm-up min(order, i + 1), a run of fewer than 15 steps ends
    with order 1 after at most 2."""
    return DO.orders_for(n, order)


def solve(x, alphas, sigmas, order: int, data_pred, corrector: bool = True, orders: Optional[List[int]] = None):
    """The predictor-corrector loop over a grid of len(alphas) points.  data_pred(i, x) -> (x, m): the data prediction m at
    point i and x as the model saw it (the inpainting blend replaces it).  The corrected state carried from step to step is
    not blended; at i = 0 it is the (blended) x_0.  corrector=False drops UniC (xc_i = x_i), for measuring UniP alone."""
    n = len(alphas) - 1
    orders = orders or orders_for(n, order)
    lam = [math.log(a / s) for a, s in zip(alphas, sigmas)]
    ms: List[torch.Tensor] = []
    xc = None
    for i in range(n):
        x, m = data_pred(i, x)
        if i == 0 or not corrector:
            xc = x
        else:
            p = orders[i - 1]
            xc = unic(xc, m, ms[:p], [lam[i]] + [lam[i - 1 - k] for k in range(p)], alphas[i], sigmas[i], sigmas[i - 1], p)
        ms = [m] + ms[:3]
        p = orders[i]
        x = unip(xc, ms[:p], [lam[i + 1]] + [lam[i - k] for k in range(p)], alphas[i + 1], sigmas[i + 1], sigmas[i], p)
    return x


# ---- the sampler ------------------------------------------------------------------------------------------------------------
@torch.no_grad()
def unipc_sample(eps_fn: SO.EpsFn, S: int, shape, sched=None, x_T=None, use_cfg=True, guidance_scale=7.5, order: int = 2,
                 alphas: Optional[List[float]] = None, on_alpha=None, mask=None, x0=None):
    """UniPCSampler.sample on the DDIM uniform grid (sampler_oracle.ddim_timesteps), the last step to alphas_cumprod[0].
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
