"""DPMSolverSampler: DPM-Solver++ multistep (Lu et al. 2022, "DPM-Solver++: Fast Solver for Guided Sampling of Diffusion
Probabilistic Models", Algorithm 2) with PLMSSampler's call surface plus `order` in {1, 2, 3}:

    DPMSolverSampler(diffusion, model, schedule, alpha_generator_func, set_alpha_scale, order=2).sample(S, shape, input, uc,
                     guidance_scale, mask, x0) -> x0 latent

It steps on the DDIM uniform grid of PLMS and DDIM (S = 30 gives 31 steps; the last step goes to alphas_cumprod[0]) with one UNet
pass per step (one 2B pass when CFG is on), so S = 20 costs 20 passes where PLMSSampler.sample(S=50) costs 51.  grid="karras" steps
on the Karras sigma grid instead (_karras.py): exactly S steps and S passes, the UNet evaluated at fractional timesteps, the final
step to sigma = 0 first order (x_S = m_{S-1}, k-diffusion's sample_dpmpp_2m / sample_dpmpp_2m_sde).  Scheduled
sampling, the first-conv swap and the inpainting blend are SamplerBase's.  Order 1 is DDIM with eta = 0.  The CFG mix, the data
prediction and the multistep update are one fp32 kernel per step (glg_dpm_update); the per-step scalars come from float64 host
tables, so the loop never waits on the device.
"""
import numpy as np
import torch

from gligen_b200 import lib as _L

from . import _karras
from ._sampling import SamplerBase, grid_alpha_sigma  # noqa: F401  (grid_alpha_sigma: re-exported for callers of this module)

GRIDS = ("ddim", "karras")

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


def grid_orders(sigma, order):
    """step_orders over the n steps of a grid of n + 1 points; a final step to sigma = 0 is first order whatever n (its target
    is the data prediction itself: x_S = m_{S-1})."""
    orders = step_orders(len(sigma) - 1, order)
    if sigma[-1] == 0.0:
        orders[-1] = 1
    return orders


def _to_zero(table, alpha, sigma, orders, final_row):
    """table(alpha, sigma, orders) with its last row replaced by final_row when the grid ends at sigma = 0 (lambda = +inf): the
    rows before it see only the finite points, and the final row is stated, not derived through infinite arithmetic."""
    if sigma[-1] > 0.0:
        return table(alpha, sigma, orders)
    out = np.zeros((len(orders), len(final_row)))
    out[:-1] = table(alpha[:-1], sigma[:-1], orders[:-1])
    out[-1] = final_row
    return out


def grid_coefficients(alpha, sigma, orders):
    """step_coefficients, with the final step to sigma = 0 (when the grid ends there) the row x_S = m_{S-1}: (0, 1, 0, 0)."""
    return _to_zero(step_coefficients, alpha, sigma, orders, (0.0, 1.0, 0.0, 0.0))


def grid_sde_coefficients(alpha, sigma, orders, eta):
    """sde_coefficients, with the final step to sigma = 0 (when the grid ends there) the noiseless row x_S = m_{S-1}:
    (0, 1, 0, 0, 0)."""
    return _to_zero(lambda a, s, o: sde_coefficients(a, s, o, eta), alpha, sigma, orders, (0.0, 1.0, 0.0, 0.0, 0.0))


def sde_coefficients(alpha, sigma, orders, eta):
    """float64 [n, 5]: (cx, k0, k1, ce, cz) of the DPM-Solver++ 2M SDE step (midpoint form) x_next = cx x + k0 m0 + k1 m1 + cz z,
    ce = 0, for each step of order 1 or 2; alpha, sigma as for step_coefficients.  With h = lambda_t - lambda_s, r = h_prev / h and
    E = -expm1(-(1 + eta) h): cx = (sigma_t / sigma_s) exp(-eta h), k0 = alpha_t E (1 + 1 / (2 r)), k1 = -alpha_t E / (2 r),
    cz = sigma_t sqrt(-expm1(-2 eta h)); order 1 drops the r terms.  eta = 0 gives step_coefficients' (cx, k0, k1)."""
    alpha = np.asarray(alpha, dtype=np.float64)
    sigma = np.asarray(sigma, dtype=np.float64)
    lam = np.log(alpha) - np.log(sigma)
    out = np.zeros((len(orders), 5))
    for i, k in enumerate(orders):
        if k not in (1, 2):
            raise ValueError(f"the SDE step has orders 1 and 2, got {k!r}")
        h = lam[i + 1] - lam[i]
        big_e = -np.expm1(-(1.0 + eta) * h)
        a_t, s_t = alpha[i + 1], sigma[i + 1]
        out[i, 0] = s_t / sigma[i] * np.exp(-eta * h)
        out[i, 1] = a_t * big_e
        if k == 2:
            r = (lam[i] - lam[i - 1]) / h
            out[i, 1] += a_t * big_e / (2.0 * r)
            out[i, 2] = -a_t * big_e / (2.0 * r)
        out[i, 4] = s_t * np.sqrt(-np.expm1(-2.0 * eta * h))
    return out


def sde_solve(x, alpha, sigma, order, eta, model_fn, update_fn, final_fn):
    """The 2M SDE loop over the n + 1 grid points of (alpha, sigma), orders from grid_orders.  model_fn as for dpm_solve;
    update_fn(x, e_cond, e_uncond, m1, alpha_i, sigma_i, coefs, m0_out) -> x at point i + 1 (it draws the step's noise).  A grid
    ending at sigma = 0 ends with the noiseless step x_S = m_{S-1}: final_fn(x, e_cond, e_uncond, alpha_i, sigma_i, coefs (cx, k0,
    k1, 0), m0_out) runs it and draws nothing.  The data predictions rotate through two buffers allocated once."""
    orders = grid_orders(sigma, order)
    coefs = grid_sde_coefficients(alpha, sigma, orders, eta)
    hist = [torch.empty_like(x) for _ in range(2)]
    for i, k in enumerate(orders):
        x, e_c, e_u = model_fn(i, x)
        m1 = hist[(i - 1) % 2] if k >= 2 else None
        c = [float(v) for v in coefs[i]]
        if sigma[i + 1] == 0.0:
            x = final_fn(x, e_c, e_u, float(alpha[i]), float(sigma[i]), c[:3] + [0.0], hist[i % 2])
        else:
            x = update_fn(x, e_c, e_u, m1, float(alpha[i]), float(sigma[i]), c, hist[i % 2])
    return x


def dpm_solve(x, alpha, sigma, order, model_fn, update_fn):
    """The multistep loop over the n + 1 grid points of (alpha, sigma).  model_fn(i, x) -> (x, e_cond, e_uncond | None): the
    model at grid point i (it may replace x, as the inpainting blend does).  update_fn(x, e_cond, e_uncond, m1, m2, alpha_i,
    sigma_i, coefs, m0_out) -> x at point i + 1, writing this step's data prediction into m0_out.  The data predictions rotate
    through three buffers allocated once: step i writes buffer i % 3 and reads the two before it."""
    orders = grid_orders(sigma, order)
    coefs = grid_coefficients(alpha, sigma, orders)
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
    per step, so a run with the same seed consumes a different stream from theirs.

    eta > 0 (orders 1 and 2) is DPM-Solver++ 2M SDE (sde_coefficients, one glg_sde_update per step): it also draws one
    randn_like(x) per step after the model pass, the last step included, after the blend's draw when there is a mask.

    grid="karras": the same draws, except that the last step (to sigma = 0) of an eta > 0 run draws no step noise: it is the
    noiseless x_S = m_{S-1} (one glg_dpm_update).  The blend's draw is x0 alpha + sigma randn_like(x0), one per step with a mask,
    as q_sample's.  The start state of image-to-image is alpha_0 init_latent + sigma_0 noise at the first point run."""

    def __init__(self, diffusion, model, schedule="linear", alpha_generator_func=None, set_alpha_scale=None, order=2, eta=0.0,
                 grid="ddim"):
        if order not in (1, 2, 3):
            raise ValueError(f"DPM-Solver++ order must be 1, 2 or 3, got {order!r}")
        if grid not in GRIDS:
            raise ValueError(f"grid must be one of {GRIDS}, got {grid!r}")
        if not 0.0 <= eta <= 1.0:
            raise ValueError(f"eta must lie in [0, 1], got {eta!r}")
        if eta > 0 and order == 3:
            raise ValueError("the SDE form (eta > 0) has orders 1 and 2 only")
        super().__init__(diffusion, model, schedule, alpha_generator_func, set_alpha_scale)
        self.order = order
        self.eta = float(eta)
        self.grid = grid
        self._grid = None                                       # the Karras SamplingGrid of the current sample() call

    @torch.no_grad()
    def sample(self, S, shape, input, uc=None, guidance_scale=1, mask=None, x0=None, *, init_latent=None, strength=1.0, noise=None):
        """init_latent / strength / noise: image-to-image, started part-way down the grid (SamplerBase._begin).  The (alpha,
        sigma) grid is the truncated time steps plus alphas_cumprod[0] (grid="ddim") or the last steps of the S-step Karras grid
        (grid="karras"); step_orders lowers the orders at its start as usual."""
        self.make_schedule(ddim_num_steps=S)
        self._grid = _karras.karras_grid(self.diffusion.alphas_cumprod, S) if self.grid == "karras" else None
        return self.dpm_sampling(shape, input, uc, guidance_scale, mask=mask, x0=x0, init_latent=init_latent, strength=strength,
                                 noise=noise)

    @torch.no_grad()
    def dpm_sampling(self, shape, input, uc=None, guidance_scale=1, mask=None, x0=None, init_latent=None, strength=1.0, noise=None):
        b = shape[0]
        img, grid, alphas = self._begin(shape, input, init_latent, strength, noise, self._grid)
        if len(grid.times) == 0:                                # strength 0: init_latent as it is
            return img
        alpha, sigma = grid.alpha, grid.sigma

        def model_fn(i, x):
            self._apply_alpha(alphas, i)
            x, ts = self._point(x, grid, i, b, mask, x0)
            input["x"], input["timesteps"] = x, ts
            e_c, e_u = self._eps_pair(input, uc, guidance_scale)
            return x, e_c, e_u

        def update_fn(x, e_c, e_u, m1, m2, a, s, coefs, m0_out):
            x = self._dpm_update(x, e_c, e_u, guidance_scale, m1, m2, a, s, coefs, m0_out)
            input["x"] = x
            return x

        if self.eta > 0:
            def sde_fn(x, e_c, e_u, m1, a, s, coefs, m0_out):
                z = torch.randn_like(x)
                x = self._sde_update(x, e_c, e_u, guidance_scale, m1, z, a, s, coefs, m0_out)
                input["x"] = x
                return x

            def final_fn(x, e_c, e_u, a, s, coefs, m0_out):
                return update_fn(x, e_c, e_u, None, None, a, s, coefs, m0_out)

            return sde_solve(img.contiguous().float(), alpha, sigma, self.order, self.eta, model_fn, sde_fn, final_fn)
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
