"""DPMSolverSampler: DPM-Solver++ multistep (Lu et al. 2022, "DPM-Solver++: Fast Solver for Guided Sampling of Diffusion
Probabilistic Models", Algorithm 2) with PLMSSampler's call surface plus `order` in {1, 2, 3}:

    DPMSolverSampler(diffusion, model, schedule, alpha_generator_func, set_alpha_scale, order=2).sample(S, shape, input, uc,
                     guidance_scale, mask, x0) -> x0 latent

It steps on the DDIM uniform grid of PLMS and DDIM (S = 30 gives 31 steps; the last step goes to alphas_cumprod[0]) with one UNet
pass per step (one 2B pass when CFG is on), so S = 20 costs 20 passes where PLMSSampler.sample(S=50) costs 51.  Scheduled
sampling, the first-conv swap and the inpainting blend are SamplerBase's.  Order 1 is DDIM with eta = 0.  The CFG mix, the data
prediction and the multistep update are one fp32 kernel per step (glg_dpm_update); the per-step scalars come from float64 host
tables, so the loop never waits on the device.
"""
import numpy as np
import torch

from gligen_b200 import lib as _L

from ._sampling import SamplerBase

# below this many steps the last step is first order and the one before at most second order (the final steps of a short run
# are the largest in lambda, where the higher-order terms lose accuracy)
LOWER_ORDER_FINAL_BELOW = 15


def step_orders(n, order):
    """The order of each of n steps: min(order, i + 1), lowered at the end of runs shorter than LOWER_ORDER_FINAL_BELOW."""
    orders = [min(order, i + 1) for i in range(n)]
    if n < LOWER_ORDER_FINAL_BELOW:
        orders[-1] = 1
        if n >= 2:
            orders[-2] = min(orders[-2], 2)
    return orders


def step_coefficients(alpha, sigma, orders):
    """float64 [n, 4]: (cx, k0, k1, k2) of x_next = cx x + k0 m0 + k1 m1 + k2 m2 for each step.  alpha, sigma: float64 [n + 1],
    point i the time step i evaluates the model at and point i + 1 its target; m_j the data prediction of step i - j."""
    alpha = np.asarray(alpha, dtype=np.float64)
    sigma = np.asarray(sigma, dtype=np.float64)
    lam = np.log(alpha) - np.log(sigma)
    out = np.zeros((len(orders), 4))
    for i, k in enumerate(orders):
        h = lam[i + 1] - lam[i]
        em = np.expm1(-h)
        a_t = alpha[i + 1]
        c = np.array([-a_t * em, 0.0, 0.0])                          # phi m0
        if k >= 2:
            r0 = (lam[i] - lam[i - 1]) / h
            d1_0 = np.array([1.0, -1.0, 0.0]) / r0
        if k == 2:
            c += c[0] / 2 * d1_0                                     # phi D1_0 / 2
        elif k == 3:
            r1 = (lam[i - 1] - lam[i - 2]) / h
            d1_1 = np.array([0.0, 1.0, -1.0]) / r1
            d1 = d1_0 + r0 / (r0 + r1) * (d1_0 - d1_1)
            d2 = (d1_0 - d1_1) / (r0 + r1)
            c += a_t * (em / h + 1.0) * d1 - a_t * ((em + h) / h ** 2 - 0.5) * d2
        out[i, 0] = sigma[i + 1] / sigma[i]
        out[i, 1:] = c
    return out


def grid_alpha_sigma(alphas_cumprod, time_range):
    """float64 (alpha, sigma) [n + 1] at the timesteps of time_range followed by alphas_cumprod[0] (DDIM's last alphas_prev)."""
    ac = np.asarray(alphas_cumprod.detach().cpu(), dtype=np.float64)
    grid = np.append(ac[np.asarray(time_range)], ac[0])
    return np.sqrt(grid), np.sqrt(1.0 - grid)


def dpm_solve(x, alpha, sigma, order, model_fn, update_fn):
    """The multistep loop over the n + 1 grid points of (alpha, sigma).  model_fn(i, x) -> (x, e_cond, e_uncond | None): the
    model at grid point i (it may replace x, as the inpainting blend does).  update_fn(x, e_cond, e_uncond, m1, m2, alpha_i,
    sigma_i, coefs, m0_out) -> x at point i + 1, writing this step's data prediction into m0_out.  The data predictions rotate
    through three buffers allocated once: step i writes buffer i % 3 and reads the two before it."""
    orders = step_orders(len(alpha) - 1, order)
    coefs = step_coefficients(alpha, sigma, orders)
    hist = [torch.empty_like(x) for _ in range(3)]
    for i, k in enumerate(orders):
        x, e_c, e_u = model_fn(i, x)
        m1 = hist[(i - 1) % 3] if k >= 2 else None
        m2 = hist[(i - 2) % 3] if k >= 3 else None
        x = update_fn(x, e_c, e_u, m1, m2, float(alpha[i]), float(sigma[i]), [float(c) for c in coefs[i]], hist[i % 3])
    return x


class DPMSolverSampler(SamplerBase):
    """Generator draws: randn(shape) for x_T when input['x'] is None, and one randn_like per step for the q_sample noise of the
    inpainting blend when a mask is given.  With init_latent, randn(shape) for the noise of the start state in place of x_T, none
    when the caller passes noise or no step runs.  Nothing else: unlike PLMSSampler and DDIMSampler there is no dropped sigma = 0 draw
    per step, so a run with the same seed consumes a different stream from theirs."""

    def __init__(self, diffusion, model, schedule="linear", alpha_generator_func=None, set_alpha_scale=None, order=2):
        if order not in (1, 2, 3):
            raise ValueError(f"DPM-Solver++ order must be 1, 2 or 3, got {order!r}")
        super().__init__(diffusion, model, schedule, alpha_generator_func, set_alpha_scale)
        self.order = order

    @torch.no_grad()
    def sample(self, S, shape, input, uc=None, guidance_scale=1, mask=None, x0=None, *, init_latent=None, strength=1.0, noise=None):
        """init_latent / strength / noise: image-to-image, started part-way down the grid (SamplerBase._begin).  The (alpha,
        sigma) grid is the truncated time steps plus alphas_cumprod[0]; step_orders lowers the orders at its start as usual."""
        self.make_schedule(ddim_num_steps=S)
        return self.dpm_sampling(shape, input, uc, guidance_scale, mask=mask, x0=x0, init_latent=init_latent, strength=strength,
                                 noise=noise)

    @torch.no_grad()
    def dpm_sampling(self, shape, input, uc=None, guidance_scale=1, mask=None, x0=None, init_latent=None, strength=1.0, noise=None):
        b = shape[0]
        img, time_range, alphas = self._begin(shape, input, init_latent, strength, noise)
        if len(time_range) == 0:                                # strength 0: init_latent as it is
            return img
        alpha, sigma = grid_alpha_sigma(self.diffusion.alphas_cumprod, time_range)

        def model_fn(i, x):
            self._apply_alpha(alphas, i)
            ts = torch.full((b,), int(time_range[i]), device=self.device, dtype=torch.long)
            x = self._inpaint_blend(x, mask, x0, ts)
            input["x"], input["timesteps"] = x, ts
            e_c, e_u = self._eps_pair(input, uc, guidance_scale)
            return x, e_c, e_u

        def update_fn(x, e_c, e_u, m1, m2, a, s, coefs, m0_out):
            x = self._dpm_update(x, e_c, e_u, guidance_scale, m1, m2, a, s, coefs, m0_out)
            input["x"] = x
            return x

        return dpm_solve(img.contiguous().float(), alpha, sigma, self.order, model_fn, update_fn)

    def _dpm_update(self, x, e_c, e_u, guidance_scale, m1, m2, alpha, sigma, coefs, m0_out):
        """Fused CFG mix + data prediction (into m0_out) + DPM-Solver++ update.  Returns x at the next grid point."""
        if x.device.type != "cuda":
            raise RuntimeError("gligen_b200 samplers run on CUDA tensors only (no CPU fallback)")
        x = x.contiguous().float()
        e_c = e_c.contiguous().float()
        e_u = None if e_u is None else e_u.contiguous().float()
        x_prev = torch.empty_like(x)
        lib = _L.load()
        st = torch.cuda.current_stream(x.device).cuda_stream
        _L.check(lib.glg_dpm_update(x.data_ptr(), e_c.data_ptr(), None if e_u is None else e_u.data_ptr(), float(guidance_scale),
                                    None if m1 is None else m1.data_ptr(), None if m2 is None else m2.data_ptr(),
                                    alpha, sigma, coefs[0], coefs[1], coefs[2], coefs[3], m0_out.data_ptr(), x_prev.data_ptr(),
                                    x.numel(), st),
                 "glg_dpm_update")
        return x_prev
