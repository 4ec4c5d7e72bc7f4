"""Shared machinery of the PLMS / DDIM samplers of this repo.

Same call surface and RNG consumption order as the reference samplers (ldm/models/diffusion/plms.py,
ddim.py); the per-step arithmetic (classifier-free-guidance mix, Adams-Bashforth combination, x_{t-1}
update; plms.py:121-158) is ONE fused fp32 kernel (glg_sampler_update) instead of ~10 eager launches, and
when the model is this repo's UNetModel the cond and uncond passes run as a single 2B batch.
"""
import numpy as np
import torch

from gligen_b200 import lib as _L
from ldm.modules.diffusionmodules.util import make_ddim_sampling_parameters, make_ddim_timesteps


class SamplerBase(object):
    def __init__(self, diffusion, model, schedule="linear", alpha_generator_func=None, set_alpha_scale=None):
        super().__init__()
        self.diffusion = diffusion
        self.model = model
        self.device = diffusion.betas.device
        self.ddpm_num_timesteps = diffusion.num_timesteps
        self.schedule = schedule
        self.alpha_generator_func = alpha_generator_func
        self.set_alpha_scale = set_alpha_scale

    def register_buffer(self, name, attr):
        if type(attr) == torch.Tensor:
            attr = attr.to(self.device)
        setattr(self, name, attr)

    def make_schedule(self, ddim_num_steps, ddim_discretize="uniform", ddim_eta=0., verbose=False):
        if ddim_eta != 0:
            raise ValueError("ddim_eta must be 0 (the fused update has no noise term)")
        self.ddim_timesteps = make_ddim_timesteps(ddim_discr_method=ddim_discretize, num_ddim_timesteps=ddim_num_steps,
                                                  num_ddpm_timesteps=self.ddpm_num_timesteps, verbose=verbose)
        ac = self.diffusion.alphas_cumprod
        assert ac.shape[0] == self.ddpm_num_timesteps, "alphas have to be defined for each timestep"
        f32 = lambda x: x.clone().detach().to(torch.float32).to(self.device)
        self.register_buffer("betas", f32(self.diffusion.betas))
        self.register_buffer("alphas_cumprod", f32(ac))
        self.register_buffer("alphas_cumprod_prev", f32(self.diffusion.alphas_cumprod_prev))
        acc = ac.cpu()
        self.register_buffer("sqrt_alphas_cumprod", f32(np.sqrt(acc)))
        self.register_buffer("sqrt_one_minus_alphas_cumprod", f32(np.sqrt(1. - acc)))
        sig, al, alp = make_ddim_sampling_parameters(alphacums=acc, ddim_timesteps=self.ddim_timesteps, eta=ddim_eta, verbose=verbose)
        self.register_buffer("ddim_sigmas", sig)
        self.register_buffer("ddim_alphas", al)
        self.register_buffer("ddim_alphas_prev", alp)
        self.register_buffer("ddim_sqrt_one_minus_alphas", np.sqrt(1. - al))
        # host copies for the per-step scalars: indexing the device buffers would block the host on the whole UNet
        # pass every step (float(tensor[i]) is a device-to-host sync)
        self._alphas_host = [float(v) for v in np.asarray(al, dtype=np.float64)]
        self._alphas_prev_host = [float(v) for v in np.asarray(alp, dtype=np.float64)]

    # ---- pieces shared by every loop -----------------------------------------------------------
    def _begin(self, shape, input, init_latent=None, strength=1.0, noise=None):
        """(start state, the time steps to run, the scheduled-sampling alphas | None).

        Without init_latent the run starts at x_T: input['x'], or randn(shape) drawn here when it is None, and covers the
        whole grid.  With init_latent (image-to-image) it starts part-way down the grid of L = len(np.flip(ddim_timesteps))
        steps: it runs the last n = min(L, int(strength * L)) of them, from t0 = time_range[L - n], at
        x = sqrt(abar_t0) init_latent + sqrt(1 - abar_t0) noise (diffusion.q_sample).  input['x'] is not read; noise is the
        caller's, or one randn(shape) drawn here, where the x_T draw would be.  n = 0 (strength 0, or strength * L < 1)
        draws nothing and returns init_latent in fp32 with an empty step list: the caller runs no UNet pass.  The
        scheduled-sampling alphas are alpha_generator_func(n), over the steps actually run."""
        if init_latent is None:
            if noise is not None or strength != 1.0:
                raise ValueError("strength and noise apply to image-to-image only: pass init_latent as well")
            img = input["x"]
            if img is None:
                img = torch.randn(shape, device=self.device)          # RNG draw #1 (plms.py:72)
                input["x"] = img
            time_range = np.flip(self.ddim_timesteps)
        else:
            if not 0.0 <= strength <= 1.0:
                raise ValueError(f"strength must lie in [0, 1], got {strength!r}")
            if tuple(init_latent.shape) != tuple(shape):
                raise ValueError(f"init_latent has shape {tuple(init_latent.shape)}, the sampler was asked for {tuple(shape)}")
            if noise is not None and tuple(noise.shape) != tuple(shape):
                raise ValueError(f"noise has shape {tuple(noise.shape)}, the sampler was asked for {tuple(shape)}")
            full = np.flip(self.ddim_timesteps)
            n = min(len(full), int(strength * len(full)))
            time_range = full[len(full) - n:]
            init_latent = init_latent.to(self.device, torch.float32)
            if n == 0:
                return init_latent, time_range, None
            if noise is None:
                noise = torch.randn(shape, device=self.device)        # where x_T would be drawn
            t0 = torch.full((shape[0],), int(time_range[0]), device=self.device, dtype=torch.long)
            img = self.diffusion.q_sample(init_latent, t0, noise=noise.to(self.device, torch.float32))
            input["x"] = img
        # a new sample() call: the engine's cache of timestep-invariant work (PositionNet tokens, text K/V, grounding
        # K/V) is only an intra-loop optimisation - never trust tensor identity across calls
        inv = getattr(self.model, "invalidate_static", None)
        if inv is not None:
            inv()
        alphas = self.alpha_generator_func(len(time_range)) if self.alpha_generator_func is not None else None
        return img, time_range, alphas

    def _apply_alpha(self, alphas, i):
        if alphas is not None:
            self.set_alpha_scale(self.model, alphas[i])
            if alphas[i] == 0:
                self.model.restore_first_conv_from_SD()

    def _eps_pair(self, input, uc, guidance_scale):
        """(eps_cond, eps_uncond | None) at input['x'], input['timesteps']."""
        use_cfg = uc is not None and guidance_scale != 1
        if use_cfg and hasattr(self.model, "forward_cfg") and "grounding_input" in input:
            return self.model.forward_cfg(input, uc)
        e_c = self.model(input)
        if not use_cfg:
            return e_c, None
        un = dict(x=input["x"], timesteps=input["timesteps"], context=uc,
                  inpainting_extra_input=input["inpainting_extra_input"], grounding_extra_input=input["grounding_extra_input"])
        return e_c, self.model(un)

    def _update(self, x, e_c, e_u, guidance_scale, olds, coefs, index, want_e):
        """Fused CFG + multistep + x_{t-1}.  Returns (x_prev, e | None).  The reference draws
        sigma_t * randn_like(x) here with sigma_t == 0: draw (and drop) it to keep the generator in step."""
        torch.randn_like(x)
        if x.device.type != "cuda":
            raise RuntimeError("gligen_b200 samplers run on CUDA tensors only (no CPU fallback)")
        x = x.contiguous().float()
        e_c = e_c.contiguous()
        x_prev = torch.empty_like(x)
        e_out = torch.empty_like(x) if want_e else None
        lib = _L.load()
        st = torch.cuda.current_stream(x.device).cuda_stream
        o = [t.data_ptr() for t in olds] + [None] * (3 - len(olds))
        _L.check(lib.glg_sampler_update(x.data_ptr(), e_c.data_ptr(), None if e_u is None else e_u.contiguous().data_ptr(),
                                        float(guidance_scale), o[0], o[1], o[2],
                                        float(coefs[0]), float(coefs[1]), float(coefs[2]), float(coefs[3]),
                                        self._alphas_host[index], self._alphas_prev_host[index],
                                        None if e_out is None else e_out.data_ptr(), x_prev.data_ptr(), x.numel(), st),
                  "glg_sampler_update")
        return x_prev, e_out

    def _inpaint_blend(self, img, mask, x0, ts):
        if mask is None:
            return img
        assert x0 is not None
        return self.diffusion.q_sample(x0, ts) * mask + (1. - mask) * img      # plms.py:96-100


AB_COEFS = {
    1: (3 / 2, -1 / 2, 0.0, 0.0),
    2: (23 / 12, -16 / 12, 5 / 12, 0.0),
    3: (55 / 24, -59 / 24, 37 / 24, -9 / 24),
}
