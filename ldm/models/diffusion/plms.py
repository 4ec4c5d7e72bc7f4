"""PLMSSampler with the reference's call surface (ldm/models/diffusion/plms.py:9-162):
PLMSSampler(diffusion, model, schedule, alpha_generator_func, set_alpha_scale).sample(S, shape, input, uc,
guidance_scale, mask, x0) -> x0 latent.  See _sampling.py for what is fused."""
import torch

from ._sampling import AB_COEFS, SamplerBase


class PLMSSampler(SamplerBase):
    @torch.no_grad()
    def sample(self, S, shape, input, uc=None, guidance_scale=1, mask=None, x0=None, *, init_latent=None, strength=1.0, noise=None):
        """init_latent / strength / noise: image-to-image, started part-way down the grid (SamplerBase._begin).  The first
        step is the pseudo improved Euler step, so a run of n steps takes n + 1 UNet passes."""
        self.make_schedule(ddim_num_steps=S)
        return self.plms_sampling(shape, input, uc, guidance_scale, mask=mask, x0=x0, init_latent=init_latent, strength=strength,
                                  noise=noise)

    @torch.no_grad()
    def plms_sampling(self, shape, input, uc=None, guidance_scale=1, mask=None, x0=None, init_latent=None, strength=1.0, noise=None):
        b = shape[0]
        img, time_range, alphas = self._begin(shape, input, init_latent, strength, noise)
        total = len(time_range)                                 # step i runs at ddim_timesteps[total - i - 1]
        history = []                                            # newest first: e_{t-1}, e_{t-2}, e_{t-3}
        for i, step in enumerate(time_range):
            self._apply_alpha(alphas, i)
            index = total - i - 1
            ts = torch.full((b,), int(step), device=self.device, dtype=torch.long)
            ts_next = torch.full((b,), int(time_range[min(i + 1, len(time_range) - 1)]), device=self.device, dtype=torch.long)
            img = self._inpaint_blend(img, mask, x0, ts)
            input["x"], input["timesteps"] = img, ts
            e_c, e_u = self._eps_pair(input, uc, guidance_scale)
            if not history:
                # pseudo improved Euler: evaluate again at the Euler point (plms.py:143-149)
                x_euler, e_t = self._update(img, e_c, e_u, guidance_scale, [], (1.0, 0, 0, 0), index, True)
                input["x"], input["timesteps"] = x_euler, ts_next
                n_c, n_u = self._eps_pair(input, uc, guidance_scale)
                img, _ = self._update(img, n_c, n_u, guidance_scale, [e_t], (0.5, 0.5, 0, 0), index, False)
            else:
                k = min(len(history), 3)
                img, e_t = self._update(img, e_c, e_u, guidance_scale, history[:k], AB_COEFS[k], index, True)
            input["x"] = img
            history = [e_t] + history[:2]
        return img


# names this drop-in does not define resolve to the reference module of the same name when a reference checkout
# follows this repo on sys.path (gligen_b200/_overlay.py)
from gligen_b200._overlay import fallback as _fallback  # noqa: E402

__getattr__ = _fallback(__name__, __file__)
