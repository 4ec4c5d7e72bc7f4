"""CPU: sampling on the Karras sigma grid (DPMSolverSampler / UniPCSampler with grid="karras") and the UNet at fractional timesteps,
without a GPU.

* The grid (ldm/models/diffusion/_karras.py) against the float64 restatement of k-diffusion (oracle/karras_oracle.py).
* The coefficient rows: the non-final rows are the DDIM-grid expansions on the Karras (alpha, sigma); 2M and 2M SDE are k-diffusion's
  VE-form steps; the final step to sigma = 0 is exactly x_S = m_{S-1}.
* Convergence on Gaussian data to the exact probability flow (and, for the SDE, to the exact marginal) at sigma_min.
* The host logic on a stand-in model: S UNet passes, generator draws and their order, refusals, grid="ddim" unchanged.
* The engine's fp32-timestep plan and the samplers end to end on the torch-fp32 checker ops (tests/ref_ops.py), against the
  fixtures (tests/golden/karras_*.pt, oracle/gen_golden_karras.py).
"""
import math
import os
import sys
from functools import partial

import numpy as np
import pytest
import torch

from bounds_dpm import dpm_update_ref
from bounds_sde import sde_update_ref
from bounds_unipc import unipc_update_ref
from conftest import GOLD, rel_l2
from gligen_b200 import synth
from gligen_b200.engine import Engine
from gligen_b200.pipeline import alpha_generator, build_model, sampler_inputs, set_alpha_scale
from gligen_b200.spec import NAMED_CONFIGS, SAMPLING_GATED_CA, synthetic_state_dict
from ldm.models.diffusion import _karras as K
from ldm.models.diffusion import _sampling
from ldm.models.diffusion import dpm_solver as DS
from ldm.models.diffusion import unipc as UP
from oracle import dpm_solver_oracle as DO
from oracle import img2img_oracle as IO
from oracle import karras_oracle as KO
from oracle import sampler_oracle as SO
from ref_ops import RefOps

STEP_COUNTS = (1, 2, 3, 6, 10, 14, 15, 20, 25, 50)


def _ac():
    return SO.make_schedule()["alphas_cumprod"]


def _diffusion():
    from ldm.models.diffusion.ldm import LatentDiffusion
    return LatentDiffusion(linear_start=0.00085, linear_end=0.012, timesteps=1000)


# ---- the grid ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("S", STEP_COUNTS[1:])
def test_grid_ends_and_oracle(S):
    sig = K.discrete_sigmas(_ac())
    assert abs(sig[0] - 0.0292) < 1e-4 and abs(sig[-1] - 14.61) < 1e-2
    g = K.karras_sigmas(_ac(), S)
    assert len(g) == S + 1 and g[-1] == 0.0
    assert abs(g[0] - sig[-1]) <= 1e-12 and abs(g[S - 1] - sig[0]) <= 1e-12
    assert np.all(np.diff(g) < 0)
    ko_sig, ko_t = KO.karras_schedule(S)
    assert np.abs(g - ko_sig.numpy()).max() <= 1e-12
    grid = K.karras_grid(_ac(), S)
    assert np.abs(grid.times - ko_t.numpy()).max() <= 1e-12
    assert not grid.integer and len(grid.times) == S and len(grid.alpha) == S + 1
    assert np.abs(grid.alpha ** 2 + grid.sigma ** 2 - 1.0).max() <= 1e-15
    assert (grid.alpha[-1], grid.sigma[-1]) == (1.0, 0.0)
    assert abs(grid.times[0] - 999.0) <= 1e-9 and abs(grid.times[-1]) <= 1e-9


def test_sigma_to_t_is_exact_at_the_discrete_steps_and_monotone():
    sig = K.discrete_sigmas(_ac())
    t = K.sigma_to_t(_ac(), sig)
    assert np.abs(t - np.arange(1000)).max() <= 1e-9
    dense = np.exp(np.linspace(np.log(sig[0]), np.log(sig[-1]), 20001))
    td = K.sigma_to_t(_ac(), dense)
    assert np.all(np.diff(td) > 0) and td[0] >= 0.0 and td[-1] <= 999.0
    assert np.abs(td - KO.sigma_to_t(torch.tensor(dense), torch.tensor(sig)).numpy()).max() <= 1e-12


def test_vp_form():
    s = np.array([0.0, 0.03, 1.0, 14.6])
    a, sv = K.vp(s)
    assert np.abs(a ** 2 + sv ** 2 - 1).max() <= 1e-15
    assert np.allclose(sv / np.where(a > 0, a, 1), s, rtol=1e-15, atol=0)


# ---- coefficient rows -------------------------------------------------------------------------------------------------------
def _kgrid(S):
    g = K.karras_grid(_ac(), S)
    return g.alpha, g.sigma


@pytest.mark.parametrize("order", [1, 2, 3])
@pytest.mark.parametrize("S", STEP_COUNTS)
def test_dpm_rows(S, order):
    """Non-final rows: step_coefficients on the finite Karras points (the expansion of the DDIM-grid sampler), and each row applied to
    random state equals dpm_solver_oracle.dpm_step on the same points to 1e-12.  The final row is (0, 1, 0, 0)."""
    alpha, sigma = _kgrid(S)
    orders = DS.grid_orders(sigma, order)
    assert orders[-1] == 1 and orders[:-1] == DS.step_orders(S, order)[:-1]
    rows = DS.grid_coefficients(alpha, sigma, orders)
    assert tuple(rows[-1]) == (0.0, 1.0, 0.0, 0.0)
    g = torch.Generator().manual_seed(S * 10 + order)
    for i in range(S - 1):
        ref = DS.step_coefficients(alpha[:i + 2], sigma[:i + 2], orders[:i + 1])[i]
        assert np.abs(rows[i] - ref).max() <= 1e-12 * np.abs(ref).max()
        k = orders[i]
        x, m0, m1, m2 = (torch.randn(64, generator=g, dtype=torch.float64) for _ in range(4))
        got = rows[i, 0] * x + rows[i, 1] * m0 + rows[i, 2] * m1 + rows[i, 3] * m2
        idx = [i + 1] + [i - j for j in range(k)]
        want = DO.dpm_step(x, [m0, m1, m2][:k], [alpha[j] for j in idx], [sigma[j] for j in idx], k)
        scale = (np.abs(rows[i]) * 4).sum() * 4
        assert (got - want).abs().max().item() <= 1e-12 * scale, (S, order, i)


def _ms(n, seed):
    g = torch.Generator().manual_seed(seed)
    return [torch.randn(64, generator=g, dtype=torch.float64) for _ in range(n)]


def _product_loop(alpha, sigma, rows, orders, ms, x, eta=False, zs=None):
    """x after each step of the DPM rows (or SDE rows with eta) with data predictions ms[i] that do not depend on x."""
    xs = [x]
    for i, k in enumerate(orders):
        r = rows[i]
        m1 = ms[i - 1] if k >= 2 else 0
        if eta:
            x = r[0] * x + r[1] * ms[i] + r[2] * m1 + r[4] * zs[i]
        else:
            m2 = ms[i - 2] if k >= 3 else 0
            x = r[0] * x + r[1] * ms[i] + r[2] * m1 + r[3] * m2
        xs.append(x)
    return xs


@pytest.mark.parametrize("eta", [0.0, 0.5, 1.0])
@pytest.mark.parametrize("S", STEP_COUNTS)
def test_2m_rows_are_k_diffusion(S, eta):
    """2M (eta = 0) and 2M SDE (eta > 0) rows driven by the same data predictions and noise give k-diffusion's VE-form trajectory
    (times alpha) at every point to 1e-12; the SDE final row has cz = 0 and the oracle draws no noise for it."""
    alpha, sigma = _kgrid(S)
    orders = DS.grid_orders(sigma, 2)
    sig = list(K.karras_sigmas(_ac(), S))
    ms, zs = _ms(S, S), _ms(S, S + 1000)
    x0 = torch.randn(64, generator=torch.Generator().manual_seed(3), dtype=torch.float64)
    if eta:
        rows = DS.grid_sde_coefficients(alpha, sigma, orders, eta)
        assert tuple(rows[-1]) == (0.0, 1.0, 0.0, 0.0, 0.0)
    else:
        rows = DS.grid_coefficients(alpha, sigma, orders)
    got = _product_loop(alpha, sigma, rows, orders, ms, x0, eta > 0, zs)
    ve = []
    draws = []

    def data_pred(i, xt):
        ve.append(xt)
        return xt, ms[i]

    def draw(xt):
        draws.append(len(draws))
        return zs[len(draws) - 1]

    if eta:
        out = KO.sample_dpmpp_2m_sde(data_pred, x0 / alpha[0], sig, eta, draw)
        assert len(draws) == S - 1
    else:
        out = KO.sample_dpmpp_2m(data_pred, x0 / alpha[0], sig)
    ve.append(out)
    for i in range(S + 1):
        want = alpha[i] * ve[i]
        assert (got[i] - want).abs().max().item() <= 1e-12 * max(1.0, want.abs().max().item()), (S, eta, i)


@pytest.mark.parametrize("order", [1, 2, 3])
@pytest.mark.parametrize("S", STEP_COUNTS)
def test_unipc_rows(S, order):
    """Non-final rows: unipc.step_coefficients on the finite Karras points; the final predictor row is (0, 1, 0, 0); the loop on the
    rows reproduces oracle/karras_oracle.unipc_vp (the paper's r / D / R / b form) to 1e-12."""
    alpha, sigma = _kgrid(S)
    orders = DS.grid_orders(sigma, order)
    rows = UP.grid_coefficients(alpha, sigma, orders)
    assert tuple(rows[-1, 5:]) == (0.0, 1.0, 0.0, 0.0)
    for i in range(S - 1):
        ref = UP.step_coefficients(alpha[:i + 2], sigma[:i + 2], orders[:i + 1])[i]
        assert np.abs(rows[i] - ref).max() <= 1e-12 * np.abs(ref).max()
    ms = _ms(S, 7 * S + order)
    x = torch.randn(64, generator=torch.Generator().manual_seed(4), dtype=torch.float64)
    x_start = x
    hist, xc = [], None
    for i in range(S):
        r = rows[i]
        m = ms[i]
        h = [ms[i - j] if i - j >= 0 else 0 for j in (1, 2, 3)]
        xc = x if i == 0 else r[0] * xc + r[1] * m + r[2] * h[0] + r[3] * h[1] + r[4] * h[2]
        x = r[5] * xc + r[6] * m + r[7] * h[0] + r[8] * h[1]
        hist.append(m)
    want = KO.unipc_vp(lambda i, xx: (xx, ms[i]), x_start, list(alpha), list(sigma), order)
    assert torch.equal(x, ms[-1]) and torch.equal(want, ms[-1])
    # the intermediate states: the oracle run over the first S points
    if S > 1:
        got_prev = None
        xx, xcc = x_start, None
        for i in range(S - 1):
            r = rows[i]
            h = [ms[i - j] if i - j >= 0 else 0 for j in (1, 2, 3)]
            xcc = xx if i == 0 else r[0] * xcc + r[1] * ms[i] + r[2] * h[0] + r[3] * h[1] + r[4] * h[2]
            xx = r[5] * xcc + r[6] * ms[i] + r[7] * h[0] + r[8] * h[1]
            got_prev = xx
        from oracle import unipc_oracle as UPO
        want_prev = UPO.solve(x_start, list(alpha[:S]), list(sigma[:S]), order, lambda i, q: (q, ms[i]), orders=orders[:S - 1])
        assert (got_prev - want_prev).abs().max().item() <= 1e-12 * max(1.0, want_prev.abs().max().item()) * 10


# ---- convergence on Gaussian data -------------------------------------------------------------------------------------------
MU, SD = 0.5, 0.8
CONV_S = (25, 50, 100, 200)


def _gauss_m(x, a, s):
    return (x - s * DO.gaussian_eps(x, a, s, MU, SD)) / a


def _ode_to_sigma_min(kind, order, S):
    """(x at sigma_min, its exact flow value, x_S from the final row, the exact data prediction at x_{S-1})."""
    alpha, sigma = _kgrid(S)
    orders = DS.grid_orders(sigma, order)
    x0 = torch.linspace(-3, 3, 41, dtype=torch.float64) * math.sqrt(alpha[0] ** 2 * SD ** 2 + sigma[0] ** 2) + alpha[0] * MU
    x = x0
    ms = []
    if kind == "dpm":
        rows = DS.grid_coefficients(alpha, sigma, orders)
        for i in range(S):
            m = _gauss_m(x, alpha[i], sigma[i])
            ms.insert(0, m)
            if i == S - 1:
                x_min, m_min = x, m
            r = rows[i]
            k = orders[i]
            x = r[0] * x + r[1] * ms[0] + (r[2] * ms[1] if k >= 2 else 0) + (r[3] * ms[2] if k >= 3 else 0)
    else:
        rows = UP.grid_coefficients(alpha, sigma, orders)
        xc = None
        for i in range(S):
            m = _gauss_m(x, alpha[i], sigma[i])
            ms.insert(0, m)
            h = [ms[j] if j < len(ms) else 0 for j in (1, 2, 3)]
            r = rows[i]
            xc = x if i == 0 else r[0] * xc + r[1] * m + r[2] * h[0] + r[3] * h[1] + r[4] * h[2]
            if i == S - 1:
                x_min, m_min = x, m
            x = r[5] * xc + r[6] * m + r[7] * h[0] + r[8] * h[1]
    exact = DO.gaussian_flow(x0, alpha[0], sigma[0], alpha[S - 1], sigma[S - 1], MU, SD)
    return x_min, exact, x, m_min


# the least order of the error at sigma_min over the last two refinements of CONV_S (50 -> 100 -> 200), stated in DESIGN §2: measured
# 2.06 / 2.03 (2M), 1.85 / 1.94 (3M: its error is 4x below 2M's at every S, but it converges at second order on this grid),
# 3.06 / 3.03 (UniPC-2)
ODE_ORDERS = {("dpm", 2): 1.9, ("dpm", 3): 1.75, ("unipc", 2): 2.9}


@pytest.mark.parametrize("kind,order", list(ODE_ORDERS))
def test_ode_converges_to_the_flow_at_sigma_min(kind, order):
    errs = []
    for S in CONV_S:
        x_min, exact, x_S, m_min = _ode_to_sigma_min(kind, order, S)
        errs.append((x_min - exact).abs().max().item())
        # the final step lands exactly on the data prediction at sigma_min
        assert (x_S - m_min).abs().max().item() <= 1e-12 * m_min.abs().max().item()
    obs = [math.log(errs[j] / errs[j + 1]) / math.log(CONV_S[j + 1] / CONV_S[j]) for j in range(len(errs) - 1)]
    print(f"{kind}-{order} Karras: errors at sigma_min {errs}, orders {obs}")
    assert min(obs[-2:]) >= ODE_ORDERS[(kind, order)], obs
    assert errs[-1] < 1e-3


def _sde_moments(S, eta):
    """Mean and variance at sigma_min (final jump excluded) and after the final step, from the exact marginal at sigma_max; as
    test_sde_cpu's moment propagation: (x_i, m_{i-1}) stays jointly Gaussian under the affine exact data prediction."""
    alpha, sigma = _kgrid(S)
    orders = DS.grid_orders(sigma, 2)
    rows = DS.grid_sde_coefficients(alpha, sigma, orders, eta)
    mean = np.array([alpha[0] * MU, 0.0])
    cov = np.diag([alpha[0] ** 2 * SD ** 2 + sigma[0] ** 2, 0.0])
    at_min = None
    for i, (cx, k0, k1, ce, cz) in enumerate(rows):
        if i == S - 1:
            at_min = (mean[0], cov[0, 0])
        a, s = alpha[i], sigma[i]
        v = a * a * SD * SD + s * s
        A, B = a * SD * SD / v, MU * s * s / v
        M = np.array([[cx + k0 * A, k1], [A, 0.0]])
        mean = M @ mean + np.array([k0 * B, B])
        cov = M @ cov @ M.T + np.diag([cz * cz, 0.0])
    a, s = alpha[S - 1], sigma[S - 1]
    v = a * a * SD * SD + s * s
    A, B = a * SD * SD / v, MU * s * s / v
    final_exact = (A * at_min[0] + B, A * A * at_min[1])            # m(x_{S-1}) of the propagated law at sigma_min
    return at_min, (mean[0], cov[0, 0]), final_exact, (a * MU, v)


# weak order of the final variance at sigma_min, measured 2.07 / 2.03 at eta = 0.5 and 1 (S 50 -> 100 -> 200)
SDE_ORDERS = {0.5: 1.9, 1.0: 1.9}


@pytest.mark.parametrize("eta", list(SDE_ORDERS))
def test_sde_weak_convergence_at_sigma_min(eta):
    errs = []
    for S in CONV_S:
        (m, v), final, final_exact, (m_true, v_true) = _sde_moments(S, eta)
        assert abs(m - m_true) <= 1e-12
        assert abs(final[0] - final_exact[0]) <= 1e-12 and abs(final[1] - final_exact[1]) <= 1e-12
        errs.append(abs(v - v_true))
    obs = [math.log(errs[j] / errs[j + 1]) / math.log(CONV_S[j + 1] / CONV_S[j]) for j in range(len(errs) - 1)]
    print(f"2M SDE eta={eta} Karras: variance errors at sigma_min {errs}, orders {obs}")
    assert min(obs[-2:]) >= SDE_ORDERS[eta], obs
    assert errs[-1] < 1e-2


# ---- host logic on a stand-in model -----------------------------------------------------------------------------------------
def _dpm_update(self, x, e_c, e_u, guidance_scale, m1, m2, alpha, sigma, coefs, m0_out):
    m0, xp = dpm_update_ref(x.float(), e_c.float(), None if e_u is None else e_u.float(), guidance_scale, m1, m2, alpha, sigma, coefs)
    m0_out.copy_(m0)
    return xp


def _sde_update(self, x, e_c, e_u, guidance_scale, m1, z, alpha, sigma, coefs, m0_out):
    m0, xn = sde_update_ref(x.float(), e_c.float(), None if e_u is None else e_u.float(), guidance_scale, m1, z.float(), alpha, sigma,
                            coefs)
    if m0_out is not None:
        m0_out.copy_(m0)
    return xn


def _unipc_update(self, x, xc, e_c, e_u, guidance_scale, m1, m2, m3, alpha, sigma, coefs, m_out, xc_out):
    m0, xcn, xn = unipc_update_ref(x.float(), xc, e_c.float(), None if e_u is None else e_u.float(), guidance_scale, m1, m2, m3,
                                   alpha, sigma, coefs)
    m_out.copy_(m0)
    xc_out.copy_(xcn)
    return xn


@pytest.fixture
def ref_updates(monkeypatch):
    monkeypatch.setattr(DS.DPMSolverSampler, "_dpm_update", _dpm_update)
    monkeypatch.setattr(_sampling.SamplerBase, "_sde_update", _sde_update)
    monkeypatch.setattr(UP.UniPCSampler, "_unipc_update", _unipc_update)


class _Eps(torch.nn.Module):
    def __init__(self):
        super().__init__()
        self.calls = 0
        self.timesteps = []

    def forward(self, input):
        self.calls += 1
        self.timesteps.append(input["timesteps"])
        return 0.1 * input["x"]


SHAPE = (2, 4, 8, 8)
SAMPLERS = {"dpm2": dict(cls="dpm", order=2), "dpm3": dict(cls="dpm", order=3), "unipc2": dict(cls="unipc", order=2),
            "dpm2sde": dict(cls="dpm", order=2, eta=1.0)}


def _make(name, grid="karras", model=None):
    kw = dict(SAMPLERS[name])
    cls = kw.pop("cls")
    model = model or _Eps()
    if cls == "dpm":
        return DS.DPMSolverSampler(_diffusion(), model, grid=grid, **kw)
    return UP.UniPCSampler(_diffusion(), model, grid=grid, **kw)


@pytest.mark.parametrize("name", list(SAMPLERS))
@pytest.mark.parametrize("S", [1, 2, 6, 10, 14, 15, 16, 20, 25])
def test_s_passes(ref_updates, name, S):
    """grid="karras": exactly S UNet passes at every S, at fp32 timesteps t(sigma_i) from 999 down to 0."""
    s = _make(name)
    out = s.sample(S, SHAPE, dict(x=None))
    assert torch.isfinite(out).all()
    assert s.model.calls == S
    ts = torch.stack([t[0] for t in s.model.timesteps])
    assert all(t.dtype == torch.float32 for t in s.model.timesteps)
    want = torch.tensor(K.karras_grid(_ac(), S).times, dtype=torch.float32)
    assert torch.equal(ts, want)


@pytest.mark.parametrize("name", list(SAMPLERS))
@pytest.mark.parametrize("with_mask", [False, True])
@pytest.mark.parametrize("with_x", [False, True])
@pytest.mark.parametrize("with_init", [False, True])
def test_rng_draws(monkeypatch, ref_updates, name, with_mask, with_x, with_init):
    """randn(shape) first for x_T when input['x'] is None (with init_latent: for the start noise, input['x'] unread); then per step
    the blend's randn_like(x0) with a mask, and for the SDE the step noise after the model pass - none on the final step."""
    log = []
    randn, randn_like = torch.randn, torch.randn_like

    def wrap(name_, fn):
        def wrapped(*a, **k):
            log.append((name_, sys._getframe(1).f_code.co_name))
            return fn(*a, **k)
        return wrapped

    monkeypatch.setattr(torch, "randn", wrap("randn", randn))
    monkeypatch.setattr(torch, "randn_like", wrap("randn_like", randn_like))
    S, strength = 10, 0.5
    x = randn(SHAPE) if with_x else None
    mask = torch.ones(2, 1, 8, 8) if with_mask else None
    x0 = torch.zeros(SHAPE) if with_mask else None
    kw = dict(init_latent=randn(SHAPE), strength=strength) if with_init else {}
    sampler = _make(name)
    out = sampler.sample(S, SHAPE, dict(x=x), mask=mask, x0=x0, **kw)
    assert torch.isfinite(out).all()
    n = min(S, int(strength * S)) if with_init else S
    assert sampler.model.calls == n
    blend = [("randn_like", "_inpaint_blend")] if with_mask else []
    noisy = [("randn_like", "sde_fn")] if name == "dpm2sde" else []
    first = [] if (with_x and not with_init) else [("randn", "_begin")]
    assert log == first + (blend + noisy) * (n - 1) + blend, log


def test_refusals():
    for cls in (DS.DPMSolverSampler, UP.UniPCSampler):
        with pytest.raises(ValueError, match="grid"):
            cls(_diffusion(), _Eps(), grid="exponential")
        with pytest.raises(ValueError, match="grid"):
            cls(_diffusion(), _Eps(), grid="Karras")
        with pytest.raises(ValueError, match="order"):
            cls(_diffusion(), _Eps(), order=4, grid="karras")
    with pytest.raises(ValueError, match="orders 1 and 2"):
        DS.DPMSolverSampler(_diffusion(), _Eps(), order=3, eta=0.5, grid="karras")
    with pytest.raises(ValueError, match="strength"):
        _make("dpm2").sample(6, SHAPE, dict(x=None), init_latent=torch.zeros(SHAPE), strength=1.5)
    with pytest.raises(ValueError, match="init_latent"):
        _make("unipc2").sample(6, SHAPE, dict(x=None), strength=0.5)
    from ldm.models.diffusion.ddim import DDIMSampler
    from ldm.models.diffusion.plms import PLMSSampler
    for cls in (DDIMSampler, PLMSSampler):
        with pytest.raises(TypeError):
            cls(_diffusion(), _Eps(), grid="karras")


def test_strength_zero_runs_nothing(ref_updates):
    s = _make("dpm2")
    init = torch.randn(SHAPE)
    out = s.sample(6, SHAPE, dict(x=None), init_latent=init, strength=0.0)
    assert torch.equal(out, init) and s.model.calls == 0


def test_image_to_image_start_state(ref_updates, monkeypatch):
    """The start state of a truncated Karras run is alpha_0 init_latent + sigma_0 noise at the first point run."""
    seen = []
    s = _make("dpm2")
    orig = s.model.forward

    def fwd(input):
        seen.append(input["x"].clone())
        return orig(input)

    s.model.forward = fwd
    init, noise = torch.randn(SHAPE), torch.randn(SHAPE)
    s.sample(10, SHAPE, dict(x=None), init_latent=init, strength=0.5, noise=noise)
    g = K.karras_grid(_ac(), 10).last(5)
    assert torch.allclose(seen[0], float(g.alpha[0]) * init + float(g.sigma[0]) * noise, rtol=0, atol=1e-6)
    assert len(seen) == 5


# ---- the engine and the loops on the checker ops -----------------------------------------------------------------------------
def _engine(cfg):
    eng = Engine(cfg, RefOps())
    eng.load_state_dict(synthetic_state_dict(cfg, 0))
    return eng


def test_fp32_t_plan_matches_reference_at_fractional_t():
    gold = torch.load(os.path.join(GOLD, "karras_unet_tiny.pt"))
    assert gold["oracle_maxabs"] == 0.0
    cfg = NAMED_CONFIGS[gold["config"]]
    eng = _engine(cfg)
    inp = synth.make_inputs(cfg, gold["B"], gold["max_objs"], seed=gold["seed"])
    ts = gold["timesteps"]
    assert ts.dtype == torch.float32 and not torch.equal(ts, ts.round())
    for t in (ts, ts.double()):                                  # float64 runs as fp32, as the reference's timesteps.float()
        e_c = eng.forward(inp["x"], t, inp["context"], inp["grounding_input"])
        e_u = eng.forward(inp["x"], t, inp["uc"], None)
        c2, u2 = eng.forward_cfg(inp["x"], t, inp["context"], inp["uc"], inp["grounding_input"])
        for got, ref in ((e_c, gold["eps_cond"]), (e_u, gold["eps_null"]), (c2, gold["eps_cond"]), (u2, gold["eps_null"])):
            err = (got - ref).abs().max().item()
            assert err <= 5e-5, err
    # the truncating int64 plan would not: the fractional rows differ from their integer parts
    e_int = eng.forward(inp["x"], ts.long(), inp["context"], inp["grounding_input"])
    assert (e_int[1:] - gold["eps_cond"][1:]).abs().max() > 1e-3
    assert sorted(k[-1] == "f32_t" for k in eng.plans) == [False, True, True]


def test_fp32_t_plan_equals_int64_plan_at_integer_t():
    cfg = NAMED_CONFIGS["tiny"]
    eng = _engine(cfg)
    inp = synth.make_inputs(cfg, 2, 6, seed=2)
    ts = torch.tensor([981, 501])
    a = eng.forward_cfg(inp["x"], ts, inp["context"], inp["uc"], inp["grounding_input"])
    a = [t.clone() for t in a]
    b = eng.forward_cfg(inp["x"], ts.float(), inp["context"], inp["uc"], inp["grounding_input"])
    assert all(torch.equal(p, q) for p, q in zip(a, b))
    keys = list(eng.plans)
    assert len(keys) == 2 and keys[0] == (4, 6, 77) and keys[1] == (4, 6, 77, "f32_t")
    assert eng.plans[keys[0]].inp["t"].dtype == torch.int64 and eng.plans[keys[1]].inp["t"].dtype == torch.float32


def test_integer_grid_never_builds_the_fp32_plan(ref_updates, monkeypatch):
    built = []
    orig = Engine._build_plan

    def spy(self, *a, **k):
        built.append(k.get("fractional_t", a[5] if len(a) > 5 else False))
        return orig(self, *a, **k)

    monkeypatch.setattr(Engine, "_build_plan", spy)
    _cpu_engine(monkeypatch)
    gold = torch.load(os.path.join(GOLD, "karras_dpm2m_tiny.pt"))
    run_fixture(dict(gold, grid="ddim"))
    assert built == [False]


def _cpu_engine(monkeypatch):
    from ldm.modules.diffusionmodules.openaimodel import UNetModel

    def engine(self):
        if self._engine is None:
            self._engine = Engine(self.cfg, RefOps())
            self._engine_stale = True
        if self._engine_stale:
            self._engine.load_state_dict(self.state_dict())
            self._engine_stale = False
        return self._engine

    monkeypatch.setattr(UNetModel, "engine", engine)


@pytest.fixture
def cpu_backend(monkeypatch, ref_updates):
    _cpu_engine(monkeypatch)


def fixture_config(gold):
    return SAMPLING_GATED_CA if gold["config"] == "sampling_gated_ca" else NAMED_CONFIGS[gold["config"]]


def run_fixture(gold, device="cpu", grid=None):
    """The product sampler on the fixture's model, inputs, seed and arguments (generator seeded 1234, CPU draws)."""
    diffusion = _diffusion().to(device)
    cfg, model = build_model(fixture_config(gold), device)
    inp = synth.make_inputs(cfg, gold["B"], gold["max_objs"], seed=2)
    input, mask, x0 = sampler_inputs(cfg, model, {k: inp[k] for k in ("x", "context", "uc", "z0") if k in inp}, inp["batch"])
    gen = partial(alpha_generator, type=gold["alpha_type"])
    shape = tuple(inp["x"].shape)
    kw = {}
    if gold["strength"] < 1.0:
        init, noise = IO.init_and_noise(shape, gold["init_seed"])
        kw = dict(init_latent=init.to(device), strength=gold["strength"], noise=noise.to(device))
    grid = gold["grid"] if grid is None else grid
    common = dict(alpha_generator_func=gen, set_alpha_scale=set_alpha_scale, order=gold["order"])
    if grid is not None:
        common["grid"] = grid
    if gold["sampler"] == "unipc":
        sampler = UP.UniPCSampler(diffusion, model, **common)
    else:
        sampler = DS.DPMSolverSampler(diffusion, model, eta=gold["eta"], **common)
    cwd = os.getcwd()
    os.chdir(GOLD)                               # restore_first_conv_from_SD reads a CWD-relative file, like the reference
    try:
        torch.manual_seed(gold["noise_seed"])
        return sampler.sample(S=gold["S"], shape=shape, input=input, uc=inp["uc"], guidance_scale=gold["guidance"], mask=mask, x0=x0,
                              **kw)
    finally:
        os.chdir(cwd)


KARRAS_FIXTURES = ["karras_dpm2m_tiny.pt", "karras_dpm3m_tiny.pt", "karras_unipc2_tiny.pt", "karras_dpm2msde_tiny.pt",
                   "karras_dpm2m_tiny_inpaint.pt", "karras_dpm2m_sampling_gated_ca.pt", "karras_dpm2m_img2img_tiny.pt",
                   "karras_dpm2m_sd14_box_text.pt"]


@pytest.mark.parametrize("gold_file", [f for f in KARRAS_FIXTURES if "sd14" not in f])
def test_loops_match_fixtures(cpu_backend, gold_file):
    """2M and 2M SDE against k-diffusion's VE-form steps, 3M and UniPC-2 against the paper-form oracles, all over the fp32 UNet oracle
    at fractional timesteps; the inpainting blend, scheduled sampling with the first-conv swap and image-to-image included."""
    gold = torch.load(os.path.join(GOLD, gold_file))
    lat = run_fixture(gold)
    r = rel_l2(lat, gold["latent"])
    print(f"{gold_file}: rel-L2 {r:.3e}")
    assert r < 2e-5, r


@pytest.mark.parametrize("name", ["dpm2", "unipc2", "dpm2sde"])
def test_explicit_ddim_grid_is_the_default(cpu_backend, name):
    """grid="ddim" passed explicitly is the default run, bit for bit, through the checker-op engine."""
    gold = dict(torch.load(os.path.join(GOLD, "karras_dpm2m_tiny.pt")))
    gold.update(sampler=SAMPLERS[name]["cls"], order=SAMPLERS[name]["order"], eta=SAMPLERS[name].get("eta", 0.0))
    a = run_fixture(dict(gold, grid=None))
    b = run_fixture(dict(gold, grid="ddim"))
    assert torch.equal(a, b)
