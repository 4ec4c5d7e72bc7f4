"""The Karras noise schedule (Karras et al. 2022, "Elucidating the Design Space of Diffusion-Based Generative Models", eq. 5) on
the discrete SD-1.x schedule, for DPMSolverSampler(grid="karras") and UniPCSampler(grid="karras").  All arithmetic is float64.

    sigma_k  = sqrt((1 - abar_k) / abar_k)                      the VE noise level of DDPM step k (about 0.029 .. 14.6 for SD-1.x)
    grid     = (sigma_max^(1/rho) + i/(S-1) (sigma_min^(1/rho) - sigma_max^(1/rho)))^rho, i = 0 .. S-1, then 0;   rho = 7
    t(sigma) = linear interpolation in log sigma between the neighbouring sigma_k (k-diffusion's DiscreteSchedule.sigma_to_t):
               exactly k at sigma_k; the UNet's (fractional) timestep input
    VP form  : alpha = 1 / sqrt(1 + sigma^2), sigma_vp = sigma / sqrt(1 + sigma^2)

The update coefficients use (alpha, sigma_vp) of the grid sigma itself; the interpolated t only feeds the UNet.  The last point,
sigma = 0, is (alpha, sigma_vp) = (1, 0): the final step lands on the data prediction.
"""
import numpy as np

from ._sampling import SamplingGrid

RHO = 7.0


def discrete_sigmas(alphas_cumprod) -> np.ndarray:
    """float64 [T]: sigma_k of every DDPM step, increasing in k."""
    ac = np.asarray(alphas_cumprod.detach().cpu() if hasattr(alphas_cumprod, "detach") else alphas_cumprod, dtype=np.float64)
    return np.sqrt((1.0 - ac) / ac)


def karras_sigmas(alphas_cumprod, S: int) -> np.ndarray:
    """float64 [S + 1]: the S Karras sigmas from sigma_max = sigma_{T-1} down to sigma_min = sigma_0 (rho = 7), then 0."""
    if S < 1:
        raise ValueError(f"the Karras grid needs at least one step, got S={S!r}")
    sig = discrete_sigmas(alphas_cumprod)
    lo, hi = sig[0] ** (1.0 / RHO), sig[-1] ** (1.0 / RHO)
    ramp = np.linspace(0.0, 1.0, S) if S > 1 else np.zeros(1)
    return np.append((hi + ramp * (lo - hi)) ** RHO, 0.0)


def sigma_to_t(alphas_cumprod, sigma) -> np.ndarray:
    """float64 model time of sigma (array or scalar, within [sigma_0, sigma_{T-1}]): k + w between the neighbouring discrete
    steps k and k + 1, w linear in log sigma (clamped to [0, 1])."""
    log_sig = np.log(discrete_sigmas(alphas_cumprod))
    ls = np.log(np.asarray(sigma, dtype=np.float64))
    low = np.clip(np.searchsorted(log_sig, ls, side="right") - 1, 0, len(log_sig) - 2)
    w = np.clip((log_sig[low] - ls) / (log_sig[low] - log_sig[low + 1]), 0.0, 1.0)
    return (1.0 - w) * low + w * (low + 1)


def vp(sigma):
    """(alpha, sigma_vp) of VE noise levels sigma: alpha = 1 / sqrt(1 + sigma^2), sigma_vp = sigma alpha."""
    sigma = np.asarray(sigma, dtype=np.float64)
    alpha = 1.0 / np.sqrt(1.0 + sigma * sigma)
    return alpha, sigma * alpha


def karras_grid(alphas_cumprod, S: int) -> SamplingGrid:
    """The SamplingGrid of an S-step Karras run: model times t(sigma_i) of the S evaluated points, (alpha, sigma_vp) of all S + 1."""
    sig = karras_sigmas(alphas_cumprod, S)
    alpha, sigma_vp = vp(sig)
    return SamplingGrid(sigma_to_t(alphas_cumprod, sig[:-1]), alpha, sigma_vp)
