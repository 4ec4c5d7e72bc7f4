"""CPU: the UniPC sampler (ldm/models/diffusion/unipc.py) without a GPU.

* Its float64 coefficient expansion against the paper's r_k / D_k / R / b form (oracle/unipc_oracle.py) on the DDIM grids, and
  its predictor rows against DPM-Solver++ (orders 1 and 2: DDIM and 2M).
* Its stepping loop on an analytic problem (Gaussian data, exact probability-flow solution): the local order of one corrected
  step and the global order on lambda-uniform grids, and the oracle's own measurement of both with and without the corrector.
* Its host logic end to end (schedule, history and corrected-state rotation, scheduled sampling, inpainting blend, RNG draws)
  through the drop-in UNetModel on the torch-fp32 checker ops (tests/ref_ops.py), with the update kernel replaced by its torch
  statement (tests/bounds_unipc.py) through test-only injection, against the oracle fixtures (tests/golden/unipc_*.pt).
* The float64 bound of the update kernel against the faithful fp32 statement and against realistic mistakes.
"""
import math
import os
from functools import partial

import numpy as np
import pytest
import torch

from bounds_unipc import unipc_update_check, unipc_update_ref
from conftest import GOLD, rel_l2
from gligen_b200 import synth
from gligen_b200.engine import Engine
from gligen_b200.pipeline import alpha_generator, build_model, sampler_inputs, set_alpha_scale
from ldm.models.diffusion import dpm_solver as DS
from ldm.models.diffusion import unipc as UP
from oracle import dpm_solver_oracle as DO
from oracle import sampler_oracle as SO
from oracle import unipc_oracle as UO
from ref_ops import RefOps

STEP_COUNTS = (5, 8, 10, 14, 15, 20, 30)


def ddim_grid(S):
    ac = SO.make_schedule()["alphas_cumprod"]
    return DS.grid_alpha_sigma(ac, np.flip(SO.ddim_timesteps(S)))


# ---- coefficients ------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("order", [1, 2, 3])
@pytest.mark.parametrize("S", STEP_COUNTS)
def test_coefficients_match_r_b_form(S, order):
    """Each step's nine coefficients applied to random float64 state equal the oracle's UniC then UniP to 1e-12."""
    alpha, sigma = ddim_grid(S)
    n = len(alpha) - 1
    orders = DS.step_orders(n, order)
    assert orders == UO.orders_for(n, order)
    lam = np.log(alpha) - np.log(sigma)
    coefs = UP.step_coefficients(alpha, sigma, orders)
    assert coefs.shape == (n, 9) and not coefs[0, :5].any()
    g = torch.Generator().manual_seed(S * 10 + order)
    for i, k in enumerate(orders):
        xcp, m0, m1, m2, m3 = (torch.randn(64, generator=g, dtype=torch.float64) for _ in range(5))
        cc, c0, c1, c2, c3, pc, p0, p1, p2 = coefs[i]
        depth = UP.history_depth(orders, i)
        assert all(c == 0.0 for c, j in ((c1, 1), (c2, 2), (c3, 3), (p1, 1), (p2, 2)) if j > depth)
        if i == 0:
            xc = ref_xc = xcp                    # xc_0 = x_0
            scale_c = 1.0
        else:
            p = orders[i - 1]
            assert all(c == 0.0 for c, j in ((c2, 2), (c3, 3)) if j > p)
            xc = cc * xcp + c0 * m0 + c1 * m1 + c2 * m2 + c3 * m3
            ref_xc = UO.unic(xcp, m0, [m1, m2, m3][:p], [lam[i]] + [lam[i - 1 - j] for j in range(p)], alpha[i], sigma[i],
                             sigma[i - 1], p)
            scale_c = sum(abs(c) * t.abs() for c, t in ((cc, xcp), (c0, m0), (c1, m1), (c2, m2), (c3, m3))).max().item()
        assert (xc - ref_xc).abs().max().item() <= 1e-12 * scale_c, (S, order, i, "corrector")
        xn = pc * xc + p0 * m0 + p1 * m1 + p2 * m2
        ref_xn = UO.unip(xc, [m0, m1, m2][:k], [lam[i + 1]] + [lam[i - j] for j in range(k)], alpha[i + 1], sigma[i + 1], sigma[i], k)
        scale_p = sum(abs(c) * t.abs() for c, t in ((pc, xc), (p0, m0), (p1, m1), (p2, m2))).max().item()
        assert (xn - ref_xn).abs().max().item() <= 1e-12 * scale_p, (S, order, i, "predictor")


@pytest.mark.parametrize("order", [1, 2])
@pytest.mark.parametrize("S", STEP_COUNTS)
def test_predictor_is_dpm_solver(S, order):
    """With the corrector dropped, UniP-1 is DDIM and UniP-2 (rho = 1/2) is DPM-Solver++ 2M: the predictor rows equal
    dpm_solver.step_coefficients to 1e-12."""
    alpha, sigma = ddim_grid(S)
    orders = DS.step_orders(len(alpha) - 1, order)
    got = UP.step_coefficients(alpha, sigma, orders)[:, 5:]
    ref = DS.step_coefficients(alpha, sigma, orders)
    assert np.abs(got - ref).max() <= 1e-12 * np.abs(ref).max(), np.abs(got - ref).max()


def test_refuses_bad_order():
    with pytest.raises(ValueError, match="order"):
        UP.UniPCSampler(None, None, order=4)
    with pytest.raises(ValueError, match="order"):
        UP.UniPCSampler(None, None, order=0)


# ---- the analytic problem ----------------------------------------------------------------------------------------------------
MU, SD = 0.5, 0.8


def _x0_pred(x, a, s):
    return (x - s * DO.gaussian_eps(x, a, s, MU, SD)) / a


def _f64_update(x, xc, e_c, e_u, m1, m2, m3, a, s, coefs, m_out, xc_out):
    m0, xcn, xn = unipc_update_ref(x, xc, e_c, e_u, 1.0, m1, m2, m3, a, s, coefs)
    m_out.copy_(m0)
    xc_out.copy_(xcn)
    return xn


@pytest.mark.parametrize("order", [1, 2, 3])
def test_local_order(order):
    """One corrected step from exact history on a lambda-uniform grid of spacing h, h/2, h/4: UniP-p from the exact x_s to
    x^_t, the model at x^_t, UniC-p from the exact x_s.  The error of the corrected state shrinks by ~2^(p + 2)."""
    z = torch.linspace(-2.5, 2.5, 11, dtype=torch.float64)
    errs = []
    for h in (0.2, 0.1, 0.05):
        lam = np.array([-h * (order - 1 - j) for j in range(order)] + [h, 2 * h])     # history ..., s = 0, t = h, one more
        alpha = 1.0 / np.sqrt(1.0 + np.exp(-2.0 * lam))
        sigma = alpha * np.exp(-lam)
        xs = [DO.gaussian_flow(MU + SD * z, 1.0, 0.0, alpha[j], sigma[j], MU, SD) for j in range(order + 1)]   # exact states
        coefs = UP.step_coefficients(alpha, sigma, list(range(1, order + 1)) + [1])
        s, t = order - 1, order
        hist = [_x0_pred(xs[s - j], alpha[s - j], sigma[s - j]) for j in range(order)] + [None] * (3 - order)
        e_s = DO.gaussian_eps(xs[s], alpha[s], sigma[s], MU, SD)
        _, _, x_hat = unipc_update_ref(xs[s], None, e_s, None, 1.0, hist[1], hist[2], None, alpha[s], sigma[s], coefs[s])
        e_t = DO.gaussian_eps(x_hat, alpha[t], sigma[t], MU, SD)
        m_t, xc, _ = unipc_update_ref(x_hat, xs[s], e_t, None, 1.0, *hist[:3], alpha[t], sigma[t], coefs[t])
        assert torch.allclose(m_t, _x0_pred(x_hat, alpha[t], sigma[t]), rtol=0, atol=1e-14)
        errs.append((xc - xs[t]).abs().max().item())
    ratios = [errs[0] / errs[1], errs[1] / errs[2]]
    print(f"order {order}: local errors {errs}, ratios {ratios} (expected ~{2 ** (order + 2)})")
    assert min(ratios) >= 0.8 * 2 ** (order + 2), (errs, ratios)


def _analytic(n, mu=MU, s=SD, lam0=-2.5):
    alpha, sigma = DO.lambda_grid(lam0, 3.0, n)
    z = torch.linspace(-2.5, 2.5, 11, dtype=torch.float64)
    x_T = DO.gaussian_flow(mu + s * z, 1.0, 0.0, alpha[0], sigma[0], mu, s)
    exact = DO.gaussian_flow(x_T, alpha[0], sigma[0], alpha[-1], sigma[-1], mu, s)
    return alpha, sigma, x_T, exact


def _product_solve(order, n):
    alpha, sigma, x_T, exact = _analytic(n)

    def model_fn(i, x):
        return x, DO.gaussian_eps(x, alpha[i], sigma[i], MU, SD), None

    return UP.unipc_solve(x_T, alpha, sigma, order, model_fn, _f64_update), exact


def _oracle_solve(order, n, corrector=True, mu=MU, s=SD, x_T=None, lam0=-2.5):
    alpha, sigma, xz, exact = _analytic(n, mu, s, lam0)
    if x_T is not None:
        xz = torch.tensor([x_T], dtype=torch.float64)
        exact = DO.gaussian_flow(xz, alpha[0], sigma[0], alpha[-1], sigma[-1], mu, s)

    def data_pred(i, x):
        return x, (x - sigma[i] * DO.gaussian_eps(x, alpha[i], sigma[i], mu, s)) / alpha[i]

    got = UO.solve(xz, list(alpha), list(sigma), order, data_pred, corrector=corrector, orders=[min(order, i + 1) for i in range(n)])
    return got, exact


def _observed(errs):
    return [math.log2(errs[k] / errs[k + 1]) for k in range(len(errs) - 1)]


# global order of the product's loop over n = 20, 40, 80, 160 (no lowered final orders at n >= 15).  Order 3's warm-up steps
# (UniP-1 + UniC-1, then UniP-2 + UniC-2) are locally O(h^3) and O(h^4) and would bound it at 3, but at lambda_0 = -2.5 their
# terms carry alpha ~ e^-2.5: the oracle measures 3.32, 3.76, 3.89 here (test_oracle_orders, DESIGN section 2).
MIN_GLOBAL_ORDER = {1: 1.8, 2: 2.7, 3: 3.2}


@pytest.mark.parametrize("order", [1, 2, 3])
def test_global_convergence(order):
    """The product's loop (unipc_solve: order warm-up, history and corrected-state rotation) over lambda-uniform grids, through
    the kernel's statement in float64; it agrees with the oracle's loop to rounding."""
    errs = []
    for n in (20, 40, 80, 160):
        got, exact = _product_solve(order, n)
        ref, _ = _oracle_solve(order, n)
        assert (got - ref).abs().max().item() <= 1e-11 * exact.abs().max().item(), (order, n)
        errs.append((got - exact).abs().max().item())
    observed = _observed(errs)
    print(f"order {order}: global errors {errs}, observed order {observed}")
    assert min(observed) >= MIN_GLOBAL_ORDER[order], (errs, observed)


# (order, corrector): the oracle's observed order per doubling of n = 10 ... 160 on x_T = 1.9, mu = 0.7, s = 1.3, last doubling
ORACLE_ORDERS = {(1, True): 2.0, (1, False): 1.0, (2, True): 3.0, (2, False): 2.0, (3, True): 3.85, (3, False): 2.0}


@pytest.mark.parametrize("order", [1, 2, 3])
@pytest.mark.parametrize("corrector", [True, False])
def test_oracle_orders(order, corrector):
    """The oracle alone: UniC raises the global order by one (UniP-p alone converges at min(p, 2), as DPM-Solver++ does: the
    first step is order 1 and locally O(h^2)).  Order 3 with the corrector measures 2.67 -> 3.85 here, and 3.0 once the warm-up
    steps sit at lambda_0 = 0."""
    errs = [(lambda r: (r[0] - r[1]).abs().max().item())(_oracle_solve(order, n, corrector, 0.7, 1.3, 1.9)) for n in (10, 20, 40, 80, 160)]
    observed = _observed(errs)
    print(f"order {order} corrector {corrector}: observed order {observed}")
    assert abs(observed[-1] - ORACLE_ORDERS[(order, corrector)]) <= 0.1, observed
    if order == 3 and corrector:
        errs = [(lambda r: (r[0] - r[1]).abs().max().item())(_oracle_solve(3, n, lam0=0.0)) for n in (80, 160, 320)]
        assert all(abs(o - 3.0) <= 0.1 for o in _observed(errs)), _observed(errs)


# ---- the loop through the checker-op engine ----------------------------------------------------------------------------------
def _fp32_update(self, x, xc, e_c, e_u, guidance_scale, m1, m2, m3, alpha, sigma, coefs, m_out, xc_out):
    m0, xcn, xn = unipc_update_ref(x.float(), xc, e_c.float(), None if e_u is None else e_u.float(), guidance_scale, m1, m2, m3,
                                   alpha, sigma, coefs)
    m_out.copy_(m0)
    xc_out.copy_(xcn)
    return xn


@pytest.fixture
def cpu_backend(monkeypatch):
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
    monkeypatch.setattr(UP.UniPCSampler, "_unipc_update", _fp32_update)


def _run(cfg_or_name, gold_like, order, S, alpha_type, guidance):
    from ldm.models.diffusion.ldm import LatentDiffusion
    diffusion = LatentDiffusion(linear_start=0.00085, linear_end=0.012, timesteps=1000)
    cfg, model = build_model(cfg_or_name, "cpu")
    inp = synth.make_inputs(cfg, gold_like["B"], gold_like["max_objs"], seed=2)
    input, mask, x0 = sampler_inputs(cfg, model, {k: inp[k] for k in ("x", "context", "uc", "z0") if k in inp}, inp["batch"])
    sampler = UP.UniPCSampler(diffusion, model, alpha_generator_func=partial(alpha_generator, type=alpha_type),
                              set_alpha_scale=set_alpha_scale, order=order)
    shape = tuple(inp["x"].shape)
    cwd = os.getcwd()
    os.chdir(GOLD)                               # restore_first_conv_from_SD reads a CWD-relative file, like the reference
    try:
        torch.manual_seed(1234)
        return sampler.sample(S=S, shape=shape, input=input, uc=inp["uc"], guidance_scale=guidance, mask=mask, x0=x0)
    finally:
        os.chdir(cwd)


UNIPC_FIXTURES = ["unipc_tiny_o2.pt", "unipc_tiny_o3.pt", "unipc_tiny_o2_s16.pt", "unipc_tiny_inpaint_o2.pt",
                  "unipc_sampling_gated_ca_o2.pt", "unipc_sd14_box_text_o2.pt"]


def fixture_config(gold):
    from gligen_b200.spec import NAMED_CONFIGS, SAMPLING_GATED_CA
    return SAMPLING_GATED_CA if gold["config"] == "sampling_gated_ca" else NAMED_CONFIGS[gold["config"]]


@pytest.mark.parametrize("gold_file", UNIPC_FIXTURES)
def test_loop_matches_oracle(cpu_backend, gold_file):
    """Orders 2 and 3 (S = 6: 7 steps with the lowered final orders; S = 16: 17 steps without), scheduled sampling with the
    first-conv swap and the inpainting blend, against the float64 oracle sampler over the fp32 UNet oracle.  Both run their
    UNet in fp32 with different operation orders: measured rel-L2 4.5e-6 to 7.1e-6."""
    gold = torch.load(os.path.join(GOLD, gold_file))
    lat = _run(fixture_config(gold), gold, gold["order"], gold["S"], gold["alpha_type"], gold["guidance"])
    r = rel_l2(lat, gold["latent"])
    print(f"{gold_file}: rel-L2 {r:.3e}")
    assert r < 2e-5, r


def test_fixtures_differ_from_dpm_solver():
    """The corrector changes the result: each UniPC-2 fixture is away from the DPM-Solver++ 2M fixture of the same model and
    inputs by far more than the loop tolerance above."""
    for name in ("tiny", "tiny_inpaint", "sampling_gated_ca", "sd14_box_text"):
        u = torch.load(os.path.join(GOLD, f"unipc_{name}_o2.pt"))["latent"]
        d = torch.load(os.path.join(GOLD, f"dpm_{name}_o2.pt"))["latent"]
        assert rel_l2(u, d) > 1e-3, name


class _Eps(torch.nn.Module):
    """A stand-in model: eps = 0.1 x, no grounding path."""

    def forward(self, input):
        return 0.1 * input["x"]


@pytest.mark.parametrize("with_mask", [False, True])
@pytest.mark.parametrize("with_x", [False, True])
def test_rng_draws(monkeypatch, with_mask, with_x):
    """x_T is drawn only when input['x'] is None; the inpainting blend draws one q_sample noise per step; nothing else."""
    from ldm.models.diffusion.ldm import LatentDiffusion
    diffusion = LatentDiffusion(linear_start=0.00085, linear_end=0.012, timesteps=1000)
    monkeypatch.setattr(UP.UniPCSampler, "_unipc_update", _fp32_update)
    calls = {"randn": 0, "randn_like": 0}
    randn, randn_like = torch.randn, torch.randn_like

    def count(name, fn):
        def wrapped(*a, **k):
            calls[name] += 1
            return fn(*a, **k)
        return wrapped

    monkeypatch.setattr(torch, "randn", count("randn", randn))
    monkeypatch.setattr(torch, "randn_like", count("randn_like", randn_like))
    sampler = UP.UniPCSampler(diffusion, _Eps(), order=2)
    shape = (2, 4, 8, 8)
    x = randn(shape) if with_x else None
    mask = torch.ones(2, 1, 8, 8) if with_mask else None
    x0 = torch.zeros(shape) if with_mask else None
    S = 10
    out = sampler.sample(S=S, shape=shape, input=dict(x=x), uc=None, guidance_scale=1, mask=mask, x0=x0)
    assert torch.isfinite(out).all()
    assert calls == {"randn": 0 if with_x else 1, "randn_like": len(SO.ddim_timesteps(S)) if with_mask else 0}, calls


@pytest.mark.parametrize("order", [2, 3])
def test_blend_reaches_corrector_only_through_data_prediction(order):
    """The inpainting blend replaces the point the model is evaluated at; the carried corrected state is the blended x only at
    i = 0.  The product's loop reproduces the oracle loop, which states that rule independently, to float64 rounding, and is
    far from the loop that would also blend each corrected state."""
    S = 8
    ac = SO.make_schedule()["alphas_cumprod"].double()
    time_range = np.flip(SO.ddim_timesteps(S))
    alpha, sigma = ddim_grid(S)
    lam = np.log(alpha) - np.log(sigma)
    g = torch.Generator().manual_seed(5)
    x_T, known = (torch.randn(64, generator=g, dtype=torch.float64) for _ in range(2))
    mask = (torch.rand(64, generator=g) > 0.5).double()
    noise = [torch.randn(64, generator=g, dtype=torch.float64) for _ in range(len(time_range))]

    def blend(i, x):
        a = float(ac[int(time_range[i])])
        return (math.sqrt(a) * known + math.sqrt(1 - a) * noise[i]) * mask + (1 - mask) * x

    def eps(x):
        return 0.3 * x - 0.1 * known

    def model_fn(i, x):
        x = blend(i, x)
        return x, eps(x), None

    def data_pred(i, x):
        x = blend(i, x)
        return x, (x - sigma[i] * eps(x)) / alpha[i]

    got = UP.unipc_solve(x_T, alpha, sigma, order, model_fn, _f64_update)
    ref = UO.solve(x_T, list(alpha), list(sigma), order, data_pred)
    assert (got - ref).abs().max().item() <= 1e-12 * ref.abs().max().item()

    orders, ms, x = DS.step_orders(len(alpha) - 1, order), [], x_T          # the other rule: blend every corrected state
    for i, k in enumerate(orders):
        x, m = data_pred(i, x)
        if i == 0:
            xc = x
        else:
            p = orders[i - 1]
            xc = blend(i, UO.unic(xc, m, ms[:p], [lam[i]] + [lam[i - 1 - j] for j in range(p)], alpha[i], sigma[i], sigma[i - 1], p))
        ms = [m] + ms[:3]
        x = UO.unip(xc, ms[:k], [lam[i + 1]] + [lam[i - j] for j in range(k)], alpha[i + 1], sigma[i + 1], sigma[i], k)
    assert (got - x).abs().max().item() > 1e-3 * ref.abs().max().item()


# ---- the kernel's bound ------------------------------------------------------------------------------------------------------
def _kernel_inputs(n=4096, seed=0):
    g = torch.Generator().manual_seed(seed)
    return [torch.randn(n, generator=g) for _ in range(7)]          # x, xc_prev, e_c, e_u, m1, m2, m3


def _step(S, order, step):
    alpha, sigma = ddim_grid(S)
    n = len(alpha) - 1
    i = step % n
    orders = DS.step_orders(n, order)
    return alpha[i], sigma[i], UP.step_coefficients(alpha, sigma, orders)[i], UP.history_depth(orders, i), i


def _fma_statement(x, xcp, ec, eu, g, m1, m2, m3, a, s, coefs):
    """The kernel's statement as nvcc contracts it: every a * b + c one rounding (exact in float64, then rounded to fp32)."""
    r = lambda t: t.float().double()
    f = lambda v: float(np.float32(v))
    c = [f(v) for v in coefs]
    x64, e = x.double(), ec.double()
    if eu is not None:
        e = r(f(g) * r(e - eu.double()) + eu.double())
    m0 = r(r(-f(s) * e + x64) / f(a))
    if xcp is None:
        xc = x64
    else:
        xc = r(c[0] * xcp.double())
        for k, m in zip(c[1:5], (m0, m1, m2, m3)):
            if m is not None:
                xc = r(k * m.double() + xc)
    xn = r(c[5] * xc)
    for k, m in zip(c[6:], (m0, m1, m2)):
        if m is not None:
            xn = r(k * m.double() + xn)
    return m0.float(), xc.float(), xn.float()


def _hist(ms, depth):
    return [m if j + 1 <= depth else None for j, m in enumerate(ms)]


@pytest.mark.parametrize("S,order,step", [(10, 1, 0), (10, 2, 1), (15, 3, 2), (20, 3, 10), (10, 2, -1), (20, 3, -1), (6, 3, 3)])
@pytest.mark.parametrize("cfg", [True, False])
def test_bound_accepts_fp32_statements(S, order, step, cfg):
    """The faithful fp32 statement, unfused (tests/bounds_unipc.unipc_update_ref) and FMA-contracted, passes."""
    x, xcp, ec, eu, m1, m2, m3 = _kernel_inputs(seed=S + step)
    a, s, coefs, depth, i = _step(S, order, step)
    eu = eu if cfg else None
    xcp = xcp if i > 0 else None
    h1, h2, h3 = _hist((m1, m2, m3), depth)
    for what, fn in (("unfused", unipc_update_ref), ("fma", _fma_statement)):
        m0, xc, xn = fn(x, xcp, ec, eu, 7.5, h1, h2, h3, a, s, coefs)
        rep = unipc_update_check(m0, xc, xn, x, xcp, ec, eu, 7.5, h1, h2, h3, a, s, coefs, what=what)
        assert rep.ok, rep


MUTANTS = ["swapped_c1_c2", "swapped_p0_p1", "dropped_m_i_in_unic", "xc_from_x", "history_rotated", "predictor_from_x"]


@pytest.mark.parametrize("mutant", MUTANTS)
def test_bound_rejects_mutants(mutant):
    S, order, step = 20, 3, 6
    x, xcp, ec, eu, m1, m2, m3 = _kernel_inputs(seed=7)
    a, s, coefs, depth, _ = _step(S, order, step)
    assert depth == 3
    bad = list(coefs)
    hist = [m1, m2, m3]
    if mutant == "swapped_c1_c2":
        bad[2], bad[3] = coefs[3], coefs[2]
    elif mutant == "swapped_p0_p1":
        bad[6], bad[7] = coefs[7], coefs[6]
    elif mutant == "dropped_m_i_in_unic":
        bad[1] = 0.0
    elif mutant == "history_rotated":
        hist = [m2, m3, m1]
    m0, xc, xn = unipc_update_ref(x, x if mutant == "xc_from_x" else xcp, ec, eu, 7.5, *hist, a, s, bad)
    if mutant == "predictor_from_x":
        _, _, xn = unipc_update_ref(x, None, ec, eu, 7.5, m1, m2, m3, a, s, coefs)
    rep = unipc_update_check(m0, xc, xn, x, xcp, ec, eu, 7.5, m1, m2, m3, a, s, coefs)
    print(rep)
    assert not rep.ok, f"{mutant} passed: {rep}"
