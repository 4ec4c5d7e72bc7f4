"""DDIMSampler with the reference's call surface (ldm/models/diffusion/ddim.py:9-134) plus `eta` in [0, 1].

eta = 0 is the deterministic step (glg_sampler_update).  eta > 0 is the reference's stochastic p_sample_ddim:
x_prev = sqrt(a_prev) pred_x0 + sqrt(1 - a_prev - sigma_t^2) e_t + sigma_t z with sigma_t = ddim_sigmas[index], one fused
kernel per step (glg_sde_update), z drawn by torch.randn_like(x) where the reference draws it.
"""
import math

import torch

from ._sampling import SamplerBase


def ddim_sde_coefficients(a_t, a_prev, sigma_t):
    """float64 (cx, k0, k1, ce, cz) of glg_sde_update for one DDIM step from abar = a_t to a_prev with noise scale sigma_t."""
    return (0.0, math.sqrt(a_prev), 0.0, math.sqrt(max(1.0 - a_prev - sigma_t * sigma_t, 0.0)), float(sigma_t))


class DDIMSampler(SamplerBase):
    @torch.no_grad()
    def sample(self, S, shape, input, uc=None, guidance_scale=1, mask=None, x0=None, *, init_latent=None, strength=1.0, noise=None,
               eta=0.0):
        """init_latent / strength / noise: image-to-image, started part-way down the grid (SamplerBase._begin).  eta in [0, 1]:
        the noise scale of each step (make_schedule's ddim_eta)."""
        self.make_schedule(ddim_num_steps=S, ddim_eta=eta)
        return self.ddim_sampling(shape, input, uc, guidance_scale, mask=mask, x0=x0, init_latent=init_latent, strength=strength,
                                  noise=noise)

    @torch.no_grad()
    def ddim_sampling(self, shape, input, uc, guidance_scale=1, mask=None, x0=None, init_latent=None, strength=1.0, noise=None):
        """Runs at the eta of the last make_schedule call.  Generator draws as the reference's: x_T (SamplerBase._begin), then per
        step the inpainting blend's q_sample noise (with a mask) and one randn_like(x) after the model pass."""
        b = shape[0]
        img, grid, alphas = self._begin(shape, input, init_latent, strength, noise)
        time_range = grid.times
        stochastic = self.ddim_eta > 0
        total = len(time_range)                                 # step i runs at ddim_timesteps[total - i - 1]
        for i, step in enumerate(time_range):
            self._apply_alpha(alphas, i)
            index = total - i - 1
            ts = torch.full((b,), int(step), device=self.device, dtype=torch.long)
            img = self._inpaint_blend(img, mask, x0, ts)
            input["x"], input["timesteps"] = img, ts
            e_c, e_u = self._eps_pair(input, uc, guidance_scale)
            if stochastic:
                img = self._sde_step(img, e_c, e_u, guidance_scale, index)
            else:
                img, _ = self._update(img, e_c, e_u, guidance_scale, [], (1.0, 0, 0, 0), index, False)
            input["x"] = img
        return img

    def _sde_step(self, x, e_c, e_u, guidance_scale, index):
        """The reference's stochastic x_prev: its sigma_t * randn_like(x) drawn here, where _update draws (and drops) it."""
        z = torch.randn_like(x)
        a_t = self._alphas_host[index]
        coefs = ddim_sde_coefficients(a_t, self._alphas_prev_host[index], self._sigmas_host[index])
        return self._sde_update(x, e_c, e_u, guidance_scale, None, z, math.sqrt(a_t), math.sqrt(1.0 - a_t), coefs, None)


# names this drop-in does not define resolve to the reference module of the same name when a reference checkout
# follows this repo on sys.path (gligen_b200/_overlay.py)
from gligen_b200._overlay import fallback as _fallback  # noqa: E402

__getattr__ = _fallback(__name__, __file__)
