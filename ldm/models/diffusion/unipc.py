"""UniPCSampler: UniPC (Zhao et al. 2023, "UniPC: A Unified Predictor-Corrector Framework for Fast Sampling of Diffusion Models"),
data prediction with B(h) = expm1(-h) ("bh2"), with PLMSSampler's call surface plus `order` in {1, 2, 3}:

    UniPCSampler(diffusion, model, schedule, alpha_generator_func, set_alpha_scale, order=2).sample(S, shape, input, uc,
                 guidance_scale, mask, x0) -> x0 latent

It steps on DPMSolverSampler's grid (the DDIM uniform grid, the last step to alphas_cumprod[0]) with its step orders, one UNet
pass per step (one 2B pass when CFG is on): S = 10 costs 10 passes.  After each model evaluation the corrector UniC refines the
state the model was evaluated at with the data prediction just computed, which costs no pass and raises the order by one; then
the predictor UniP steps from the corrected state.  The last step is not corrected (that would need a pass at x_S).
grid="karras" steps on the Karras sigma grid (_karras.py), as DPMSolverSampler's: S steps and S passes, fractional timesteps, and a
final first-order step to sigma = 0, x_S = m_{S-1}; the predictor and corrector tables are unchanged on its lambda grid.  UniP of
order 2 is DPM-Solver++ 2M.  Scheduled sampling, the first-conv swap and the inpainting blend are SamplerBase's; the blend
replaces the point the model is evaluated at and reaches the corrected state only through that point's data prediction.  The
CFG mix, the data prediction, the corrector and the predictor are one fp32 kernel per step (glg_unipc_update); the per-step
scalars come from float64 host tables, so the loop never waits on the device.
"""
import math

import numpy as np
import torch

from gligen_b200 import lib as _L

from . import _karras
from ._sampling import SamplerBase
from .dpm_solver import GRIDS, grid_orders


def _bh2_rhos(lam_t, lam_s, lam_hist, corrector):
    """(h, B, r_1 .. r_{p-1}, rho) of one step from lambda_s to lambda_t with the earlier points lam_hist (newest first, p - 1 of
    them): rho_p (predictor, p - 1 weights of D_1 .. D_{p-1}) or rho_c (corrector, p weights: D_1 .. D_{p-1}, then m_t - m_s)."""
    p = len(lam_hist) + 1
    h = lam_t - lam_s
    hh = -h
    B = math.expm1(hh)
    rks = [(l - lam_s) / h for l in lam_hist] + [1.0]
    R = np.array([[r ** a for r in rks] for a in range(p)])
    b = np.empty(p)
    g, fact = B / hh - 1.0, 1.0
    for a in range(p):
        b[a] = g * fact / B
        fact *= a + 2
        g = g / hh - 1.0 / fact
    if corrector:
        rho = np.array([0.5]) if p == 1 else np.linalg.solve(R, b)
    else:
        rho = np.zeros(0) if p == 1 else np.array([0.5]) if p == 2 else np.linalg.solve(R[:-1, :-1], b[:-1])
    return h, B, rks, rho


def _expand(alpha, sigma, lam, s, t, p, corrector):
    """float64 (cx, k_t, k_s, k_{s-1}, k_{s-2}) of one step from point s to t = s + 1 of order p: the new state is cx x_s +
    k_t m_t + k_s m_s + k_{s-1} m_{s-1} + k_{s-2} m_{s-2} (k_t = 0 for the predictor)."""
    h, B, rks, rho = _bh2_rhos(lam[t], lam[s], [lam[s - k] for k in range(1, p)], corrector)
    a_t = alpha[t]
    out = np.zeros(5)
    out[0] = sigma[t] / sigma[s]
    out[2] = -a_t * B                                               # -alpha_t phi_1 m_s; phi_1 = B for bh2
    for k in range(1, p):                                           # -alpha_t B rho_k D_k, D_k = (m_{s-k} - m_s) / r_k
        w = a_t * B * rho[k - 1] / rks[k - 1]
        out[2 + k] -= w
        out[2] += w
    if corrector:                                                   # -alpha_t B rho_p (m_t - m_s)
        out[1] -= a_t * B * rho[p - 1]
        out[2] += a_t * B * rho[p - 1]
    return out


def step_coefficients(alpha, sigma, orders):
    """float64 [n, 9]: (cc, c0, c1, c2, c3, pc, p0, p1, p2) of step i,
        xc_i    = cc xc_{i-1} + c0 m_i + c1 m_{i-1} + c2 m_{i-2} + c3 m_{i-3}      (UniC of order orders[i - 1]; zero at i = 0)
        x_{i+1} = pc xc_i     + p0 m_i + p1 m_{i-1} + p2 m_{i-2}                   (UniP of order orders[i])
    alpha, sigma: float64 [n + 1], point i the time step i evaluates the model at; m_j the data prediction at point j."""
    alpha = np.asarray(alpha, dtype=np.float64)
    sigma = np.asarray(sigma, dtype=np.float64)
    lam = np.log(alpha) - np.log(sigma)
    out = np.zeros((len(orders), 9))
    for i, k in enumerate(orders):
        if i > 0:
            out[i, :5] = _expand(alpha, sigma, lam, i - 1, i, orders[i - 1], corrector=True)
        pred = _expand(alpha, sigma, lam, i, i + 1, k, corrector=False)
        out[i, 5] = pred[0]
        out[i, 6:] = pred[2:]
    return out


def grid_coefficients(alpha, sigma, orders):
    """step_coefficients; when the grid ends at sigma = 0 (lambda = +inf) the final row's predictor is stated as x_S = m_{S-1},
    (pc, p0, p1, p2) = (0, 1, 0, 0), and its corrector (of the state the final model pass saw) is the usual one."""
    if sigma[-1] > 0.0:
        return step_coefficients(alpha, sigma, orders)
    n = len(orders)
    a, s = np.asarray(alpha[:-1], dtype=np.float64), np.asarray(sigma[:-1], dtype=np.float64)
    out = np.zeros((n, 9))
    out[:-1] = step_coefficients(a, s, orders[:-1])
    if n > 1:
        out[-1, :5] = _expand(a, s, np.log(a) - np.log(s), n - 2, n - 1, orders[n - 2], corrector=True)
    out[-1, 5:] = (0.0, 1.0, 0.0, 0.0)
    return out


def history_depth(orders, i):
    """How many earlier data predictions step i reads: m_{i-1} .. m_{i-depth}."""
    return max(orders[i - 1] if i > 0 else 0, orders[i] - 1)


def unipc_solve(x, alpha, sigma, order, model_fn, update_fn):
    """The predictor-corrector loop over the n + 1 grid points of (alpha, sigma).  model_fn(i, x) -> (x, e_cond, e_uncond | None):
    the model at grid point i (it may replace x, as the inpainting blend does).  update_fn(x, xc_prev, e_cond, e_uncond, m1, m2,
    m3, alpha_i, sigma_i, coefs, m_out, xc_out) -> x at point i + 1, writing this step's data prediction into m_out and its
    corrected state into xc_out (xc_prev None at i = 0: xc_0 = x_0).  The data predictions rotate through four buffers and the
    corrected states through two, allocated once: step i writes m buffer i % 4 and xc buffer i % 2 and reads the ones before."""
    orders = grid_orders(sigma, order)
    coefs = grid_coefficients(alpha, sigma, orders)
    hist = [torch.empty_like(x) for _ in range(4)]
    xcs = [torch.empty_like(x) for _ in range(2)]
    xc = None
    for i in range(len(orders)):
        x, e_c, e_u = model_fn(i, x)
        depth = history_depth(orders, i)
        m1, m2, m3 = (hist[(i - j) % 4] if j <= depth else None for j in (1, 2, 3))
        x = update_fn(x, xc, e_c, e_u, m1, m2, m3, float(alpha[i]), float(sigma[i]), [float(c) for c in coefs[i]], hist[i % 4],
                      xcs[i % 2])
        xc = xcs[i % 2]
    return x


class UniPCSampler(SamplerBase):
    """Generator draws: randn(shape) for x_T when input['x'] is None, and one randn_like per step for the q_sample noise of the
    inpainting blend when a mask is given.  With init_latent, randn(shape) for the noise of the start state in place of x_T, none
    when the caller passes noise or no step runs.  Nothing else, as DPMSolverSampler.  grid="karras" draws the same; its blend
    draw is x0 alpha + sigma randn_like(x0), as q_sample's."""

    def __init__(self, diffusion, model, schedule="linear", alpha_generator_func=None, set_alpha_scale=None, order=2, grid="ddim"):
        if order not in (1, 2, 3):
            raise ValueError(f"UniPC order must be 1, 2 or 3, got {order!r}")
        if grid not in GRIDS:
            raise ValueError(f"grid must be one of {GRIDS}, got {grid!r}")
        super().__init__(diffusion, model, schedule, alpha_generator_func, set_alpha_scale)
        self.order = order
        self.grid = grid
        self._grid = None                                       # the Karras SamplingGrid of the current sample() call

    @torch.no_grad()
    def sample(self, S, shape, input, uc=None, guidance_scale=1, mask=None, x0=None, *, init_latent=None, strength=1.0, noise=None):
        """init_latent / strength / noise: image-to-image, started part-way down the grid (SamplerBase._begin).  The (alpha,
        sigma) grid is the truncated time steps plus alphas_cumprod[0] (grid="ddim") or the last steps of the S-step Karras grid
        (grid="karras"); step_orders lowers the orders at its start as usual."""
        self.make_schedule(ddim_num_steps=S)
        self._grid = _karras.karras_grid(self.diffusion.alphas_cumprod, S) if self.grid == "karras" else None
        return self.unipc_sampling(shape, input, uc, guidance_scale, mask=mask, x0=x0, init_latent=init_latent, strength=strength,
                                   noise=noise)

    @torch.no_grad()
    def unipc_sampling(self, shape, input, uc=None, guidance_scale=1, mask=None, x0=None, init_latent=None, strength=1.0, noise=None):
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

        def update_fn(x, xc, e_c, e_u, m1, m2, m3, a, s, coefs, m_out, xc_out):
            x = self._unipc_update(x, xc, e_c, e_u, guidance_scale, m1, m2, m3, a, s, coefs, m_out, xc_out)
            input["x"] = x
            return x

        return unipc_solve(img.contiguous().float(), alpha, sigma, self.order, model_fn, update_fn)

    def _unipc_update(self, x, xc, e_c, e_u, guidance_scale, m1, m2, m3, alpha, sigma, coefs, m_out, xc_out):
        """Fused CFG mix + data prediction (into m_out) + UniC (into xc_out) + UniP.  Returns x at the next grid point."""
        if x.device.type != "cuda":
            raise RuntimeError("gligen_b200 samplers run on CUDA tensors only (no CPU fallback)")
        x = x.contiguous().float()
        e_c = e_c.contiguous().float()
        e_u = None if e_u is None else e_u.contiguous().float()
        x_next = torch.empty_like(x)
        ptr = lambda t: None if t is None else t.data_ptr()
        lib = _L.load()
        st = torch.cuda.current_stream(x.device).cuda_stream
        _L.check(lib.glg_unipc_update(x.data_ptr(), ptr(xc), e_c.data_ptr(), ptr(e_u), float(guidance_scale), ptr(m1), ptr(m2), ptr(m3),
                                      alpha, sigma, *coefs, m_out.data_ptr(), xc_out.data_ptr(), x_next.data_ptr(), x.numel(), st),
                 "glg_unipc_update")
        return x_next
