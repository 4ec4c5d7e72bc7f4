"""DDIMSampler with the reference's call surface (ldm/models/diffusion/ddim.py:9-134), eta = 0."""
import torch

from ._sampling import SamplerBase


class DDIMSampler(SamplerBase):
    @torch.no_grad()
    def sample(self, S, shape, input, uc=None, guidance_scale=1, mask=None, x0=None, *, init_latent=None, strength=1.0, noise=None):
        """init_latent / strength / noise: image-to-image, started part-way down the grid (SamplerBase._begin)."""
        self.make_schedule(ddim_num_steps=S)
        return self.ddim_sampling(shape, input, uc, guidance_scale, mask=mask, x0=x0, init_latent=init_latent, strength=strength,
                                  noise=noise)

    @torch.no_grad()
    def ddim_sampling(self, shape, input, uc, guidance_scale=1, mask=None, x0=None, init_latent=None, strength=1.0, noise=None):
        b = shape[0]
        img, time_range, alphas = self._begin(shape, input, init_latent, strength, noise)
        total = len(time_range)                                 # step i runs at ddim_timesteps[total - i - 1]
        for i, step in enumerate(time_range):
            self._apply_alpha(alphas, i)
            index = total - i - 1
            ts = torch.full((b,), int(step), device=self.device, dtype=torch.long)
            img = self._inpaint_blend(img, mask, x0, ts)
            input["x"], input["timesteps"] = img, ts
            e_c, e_u = self._eps_pair(input, uc, guidance_scale)
            img, _ = self._update(img, e_c, e_u, guidance_scale, [], (1.0, 0, 0, 0), index, False)
            input["x"] = img
        return img


# names this drop-in does not define resolve to the reference module of the same name when a reference checkout
# follows this repo on sys.path (gligen_b200/_overlay.py)
from gligen_b200._overlay import fallback as _fallback  # noqa: E402

__getattr__ = _fallback(__name__, __file__)
