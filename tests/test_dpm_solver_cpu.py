"""CPU: the DPM-Solver++ sampler (ldm/models/diffusion/dpm_solver.py) without a GPU.

* Its float64 coefficient expansion against the paper's D0 / D1 / D2 form (oracle/dpm_solver_oracle.py) on the DDIM grids.
* Its stepping loop on an analytic problem (Gaussian data, exact probability-flow solution): the local order of each formula
  and the global order of orders 1 and 2 on lambda-uniform grids.
* Its host logic end to end (schedule, history, scheduled sampling, inpainting blend, RNG draws) through the drop-in UNetModel
  on the torch-fp32 checker ops (tests/ref_ops.py), with the update kernel replaced by its torch statement (tests/bounds_dpm.py)
  through test-only injection: order 1 against the reference DDIMSampler's latents, orders 2 and 3 against the oracle fixtures.
* The float64 bound of the update kernel against the faithful fp32 statement and against realistic mistakes.
"""
import math
import os
from functools import partial

import numpy as np
import pytest
import torch

from bounds import g_n
from bounds_dpm import dpm_update_bound, dpm_update_check, dpm_update_ref
from conftest import GOLD, rel_l2
from gligen_b200 import synth
from gligen_b200.engine import Engine
from gligen_b200.pipeline import alpha_generator, build_model, sampler_inputs, set_alpha_scale
from ldm.models.diffusion import dpm_solver as DS
from oracle import dpm_solver_oracle as DO
from oracle import sampler_oracle as SO
from ref_ops import RefOps

STEP_COUNTS = (4, 10, 14, 15, 20, 30, 50)


def ddim_grid(S):
    ac = SO.make_schedule()["alphas_cumprod"]
    return DS.grid_alpha_sigma(ac, np.flip(SO.ddim_timesteps(S)))


# ---- coefficients ------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("order", [1, 2, 3])
@pytest.mark.parametrize("S", STEP_COUNTS)
def test_coefficients_match_d_form(S, order):
    """Each step's (cx, k0, k1, k2) applied to random float64 state equals the oracle's D-form step to 1e-12."""
    alpha, sigma = ddim_grid(S)
    n = len(alpha) - 1
    assert n == len(SO.ddim_timesteps(S)) and (S != 30 or n == 31)
    ac = SO.make_schedule()["alphas_cumprod"].double()
    assert alpha[-1] == math.sqrt(float(ac[0])) and alpha[0] == math.sqrt(float(ac[int(SO.ddim_timesteps(S)[-1])]))
    orders = DS.step_orders(n, order)
    assert orders == DO.orders_for(n, order)
    if n < 15:
        assert orders[-1] == 1 and (n < 2 or orders[-2] <= 2)
    else:
        assert orders == [min(order, i + 1) for i in range(n)]
    coefs = DS.step_coefficients(alpha, sigma, orders)
    g = torch.Generator().manual_seed(S * 10 + order)
    for i, k in enumerate(orders):
        x, m0, m1, m2 = (torch.randn(64, generator=g, dtype=torch.float64) for _ in range(4))
        cx, k0, k1, k2 = coefs[i]
        got = cx * x + k0 * m0 + k1 * m1 + k2 * m2
        idx = [i + 1] + [i - j for j in range(k)]
        ref = DO.dpm_step(x, [m0, m1, m2][:k], [alpha[j] for j in idx], [sigma[j] for j in idx], k)
        scale = (abs(cx) * x.abs() + abs(k0) * m0.abs() + abs(k1) * m1.abs() + abs(k2) * m2.abs()).max().item()
        assert (got - ref).abs().max().item() <= 1e-12 * scale, (S, order, i, k)
        if k < 3:
            assert k2 == 0.0 and (k == 2 or k1 == 0.0)


def test_order_one_is_ddim():
    """Order 1 expands to DDIM with eta = 0: x_prev = sqrt(a_prev) (x - sqrt(1 - a_t) e) / sqrt(a_t) + sqrt(1 - a_prev) e."""
    alpha, sigma = ddim_grid(20)
    coefs = DS.step_coefficients(alpha, sigma, [1] * (len(alpha) - 1))
    x, e = 0.7, -1.3
    for i in range(len(alpha) - 1):
        m0 = (x - sigma[i] * e) / alpha[i]
        got = coefs[i, 0] * x + coefs[i, 1] * m0
        assert abs(got - (alpha[i + 1] * m0 + sigma[i + 1] * e)) <= 1e-12 * (abs(got) + abs(m0))


def test_refuses_bad_order():
    with pytest.raises(ValueError, match="order"):
        DS.DPMSolverSampler(None, None, order=4)


# ---- the analytic problem ----------------------------------------------------------------------------------------------------
MU, SD = 0.5, 0.8


def _x0_pred(x, a, s):
    return (x - s * DO.gaussian_eps(x, a, s, MU, SD)) / a


def _f64_update(x, e_c, e_u, m1, m2, a, s, coefs, m0_out):
    m0, xp = dpm_update_ref(x, e_c, e_u, 1.0, m1, m2, a, s, coefs)
    m0_out.copy_(m0)
    return xp


# local error exponent of each update.  3M is O(h^3) like 2M: along the solution m(lambda_s0 + u) = m0 + u m' + u^2/2 m'' + ...
# the exact step carries -alpha_t h^2 phi_3 m'' (= alpha_t h^3 / 6 m'' + O(h^4)), while the published update's D2 estimates
# h^2 m'' / 2, so it keeps half of that term.  The test pins the published formula's behaviour.
LOCAL_EXPONENT = {1: 2, 2: 3, 3: 3}


@pytest.mark.parametrize("order", [1, 2, 3])
def test_local_order(order):
    """One step from exact history on a lambda-uniform grid of spacing h, h/2, h/4: the error shrinks by ~2^LOCAL_EXPONENT."""
    z = torch.linspace(-2.5, 2.5, 11, dtype=torch.float64)
    errs = []
    for h in (0.2, 0.1, 0.05):
        lam = np.array([-h * (order - 1 - j) for j in range(order)] + [h])          # history ..., s1, s0 = 0, target h
        alpha = 1.0 / np.sqrt(1.0 + np.exp(-2.0 * lam))
        sigma = alpha * np.exp(-lam)
        xs = [DO.gaussian_flow(MU + SD * z, 1.0, 0.0, alpha[j], sigma[j], MU, SD) for j in range(order + 1)]   # exact states
        coefs = DS.step_coefficients(alpha, sigma, list(range(1, order + 1)))[-1]
        i = order - 1
        ms = [_x0_pred(xs[i - j], alpha[i - j], sigma[i - j]) for j in range(order)] + [None] * (3 - order)
        m0_out = torch.empty_like(z)
        e = DO.gaussian_eps(xs[i], alpha[i], sigma[i], MU, SD)
        got = _f64_update(xs[i], e, None, ms[1], ms[2], alpha[i], sigma[i], coefs, m0_out)
        assert torch.allclose(m0_out, ms[0], rtol=0, atol=1e-14)
        errs.append((got - xs[order]).abs().max().item())
    ratios = [errs[0] / errs[1], errs[1] / errs[2]]
    p = LOCAL_EXPONENT[order]
    print(f"order {order}: local errors {errs}, ratios {ratios} (expected ~{2 ** p})")
    assert min(ratios) >= 0.8 * 2 ** p, (errs, ratios)


def _global_error(order, n):
    alpha, sigma = DO.lambda_grid(-2.5, 3.0, n)
    z = torch.linspace(-2.5, 2.5, 11, dtype=torch.float64)
    x_T = DO.gaussian_flow(MU + SD * z, 1.0, 0.0, alpha[0], sigma[0], MU, SD)

    def model_fn(i, x):
        return x, DO.gaussian_eps(x, alpha[i], sigma[i], MU, SD), None

    got = DS.dpm_solve(x_T, alpha, sigma, order, model_fn, _f64_update)
    exact = DO.gaussian_flow(x_T, alpha[0], sigma[0], alpha[-1], sigma[-1], MU, SD)
    return (got - exact).abs().max().item()


@pytest.mark.parametrize("order,min_order", [(1, 0.9), (2, 1.8), (3, None)])
def test_global_convergence(order, min_order):
    """The product's loop (dpm_solve: order warm-up, history rotation) over lambda-uniform grids of 50, 100, 200 steps.  The
    observed order of 3M is reported, not checked: its update is locally O(h^3) (LOCAL_EXPONENT) and its start-up steps are
    lower order, so it converges at about 2."""
    errs = [_global_error(order, n) for n in (50, 100, 200)]
    observed = [math.log2(errs[0] / errs[1]), math.log2(errs[1] / errs[2])]
    print(f"order {order}: global errors {errs}, observed order {observed}")
    if min_order is not None:
        assert min(observed) >= min_order, (errs, observed)


# ---- the loop through the checker-op engine ----------------------------------------------------------------------------------
def _fp32_update(self, x, e_c, e_u, guidance_scale, m1, m2, alpha, sigma, coefs, m0_out):
    m0, xp = dpm_update_ref(x.float(), e_c.float(), None if e_u is None else e_u.float(), guidance_scale, m1, m2, alpha, sigma, coefs)
    m0_out.copy_(m0)
    return xp


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
    monkeypatch.setattr(DS.DPMSolverSampler, "_dpm_update", _fp32_update)


def _run(cfg_or_name, gold_like, order, S, alpha_type, guidance):
    from ldm.models.diffusion.ldm import LatentDiffusion
    diffusion = LatentDiffusion(linear_start=0.00085, linear_end=0.012, timesteps=1000)
    cfg, model = build_model(cfg_or_name, "cpu")
    inp = synth.make_inputs(cfg, gold_like["B"], gold_like["max_objs"], seed=2, n_valid=gold_like.get("n_valid"))
    input, mask, x0 = sampler_inputs(cfg, model, {k: inp[k] for k in ("x", "context", "uc", "z0") if k in inp}, inp["batch"])
    sampler = DS.DPMSolverSampler(diffusion, model, alpha_generator_func=partial(alpha_generator, type=alpha_type),
                                  set_alpha_scale=set_alpha_scale, order=order)
    shape = tuple(inp["x"].shape)
    cwd = os.getcwd()
    os.chdir(GOLD)                               # restore_first_conv_from_SD reads a CWD-relative file, like the reference
    try:
        torch.manual_seed(1234)
        return sampler.sample(S=S, shape=shape, input=input, uc=inp["uc"], guidance_scale=guidance, mask=mask, x0=x0)
    finally:
        os.chdir(cwd)


@pytest.mark.parametrize("name,gold_file", [("tiny", "tiny_B2_G6.pt"), ("tiny_text_image", "tiny_text_image_B2_G5.pt"),
                                            ("tiny_keypoint", "tiny_keypoint_B2_G34.pt")])
def test_order_one_matches_reference_ddim(cpu_backend, name, gold_file):
    """Order 1 is DDIM with eta = 0: it reproduces the reference DDIMSampler's latents (tests/golden, written by the real
    reference).  Without a mask the reference's extra sigma = 0 draws do not reach the result."""
    gold = torch.load(os.path.join(GOLD, gold_file))
    g = gold["ddim"]
    lat = _run(name, gold, 1, g["S"], g["alpha_type"], g["guidance"])
    r = rel_l2(lat, g["latent"])
    print(f"{name} order 1 vs reference DDIM S={g['S']}: rel-L2 {r:.3e}")
    assert r < 2e-4, r


DPM_FIXTURES = ["dpm_tiny_o2.pt", "dpm_tiny_o3.pt", "dpm_tiny_inpaint_o2.pt", "dpm_sampling_gated_ca_o2.pt"]


def fixture_config(gold):
    from gligen_b200.spec import NAMED_CONFIGS, SAMPLING_GATED_CA
    return SAMPLING_GATED_CA if gold["config"] == "sampling_gated_ca" else NAMED_CONFIGS[gold["config"]]


@pytest.mark.parametrize("gold_file", DPM_FIXTURES)
def test_orders_two_three_match_oracle(cpu_backend, gold_file):
    """Orders 2 and 3 (S = 6: 7 steps, the lowered final orders included), scheduled sampling with the first-conv swap and the
    inpainting blend, against the float64 oracle sampler over the fp32 UNet oracle."""
    gold = torch.load(os.path.join(GOLD, gold_file))
    lat = _run(fixture_config(gold), gold, gold["order"], gold["S"], gold["alpha_type"], gold["guidance"])
    r = rel_l2(lat, gold["latent"])
    print(f"{gold_file}: rel-L2 {r:.3e}")
    assert r < 2e-4, r


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
    monkeypatch.setattr(DS.DPMSolverSampler, "_dpm_update", _fp32_update)
    calls = {"randn": 0, "randn_like": 0}
    randn, randn_like = torch.randn, torch.randn_like

    def count(name, fn):
        def wrapped(*a, **k):
            calls[name] += 1
            return fn(*a, **k)
        return wrapped

    monkeypatch.setattr(torch, "randn", count("randn", randn))
    monkeypatch.setattr(torch, "randn_like", count("randn_like", randn_like))
    sampler = DS.DPMSolverSampler(diffusion, _Eps(), order=2)
    shape = (2, 4, 8, 8)
    x = randn(shape) if with_x else None
    mask = torch.ones(2, 1, 8, 8) if with_mask else None
    x0 = torch.zeros(shape) if with_mask else None
    S = 10
    out = sampler.sample(S=S, shape=shape, input=dict(x=x), uc=None, guidance_scale=1, mask=mask, x0=x0)
    assert torch.isfinite(out).all()
    assert calls == {"randn": 0 if with_x else 1, "randn_like": len(SO.ddim_timesteps(S)) if with_mask else 0}, calls


# ---- the kernel's bound ------------------------------------------------------------------------------------------------------
def _kernel_inputs(n=4096, seed=0):
    g = torch.Generator().manual_seed(seed)
    return [torch.randn(n, generator=g) for _ in range(5)]          # x, e_c, e_u, m1, m2


def _step_scalars(S, order, step):
    alpha, sigma = ddim_grid(S)
    n = len(alpha) - 1
    i = step % n
    coefs = DS.step_coefficients(alpha, sigma, DS.step_orders(n, order))[i]
    return alpha[i], sigma[i], coefs, DS.step_orders(n, order)[i]


def _fma_statement(x, ec, eu, g, m1, m2, a, s, coefs):
    """The kernel's statement as nvcc contracts it: every a * b + c one rounding (exact in float64, then rounded to fp32)."""
    r = lambda t: t.float().double()
    f = lambda v: float(np.float32(v))
    x64, e = x.double(), ec.double()
    if eu is not None:
        e = r(f(g) * r(e - eu.double()) + eu.double())
    m0 = r(r(-f(s) * e + x64) / f(a))
    xp = r(f(coefs[0]) * x64)
    for c, m in zip(coefs[1:], (m0, m1, m2)):
        if m is not None:
            xp = r(f(c) * m.double() + xp)
    return m0.float(), xp.float()


@pytest.mark.parametrize("S,order,step", [(20, 1, 0), (20, 2, 1), (25, 3, 2), (50, 3, 10), (20, 2, -1), (6, 3, 3)])
@pytest.mark.parametrize("cfg", [True, False])
def test_bound_accepts_fp32_statements(S, order, step, cfg):
    """The faithful fp32 statement, unfused (tests/bounds_dpm.dpm_update_ref) and FMA-contracted, passes."""
    x, ec, eu, m1, m2 = _kernel_inputs(seed=S + step)
    a, s, coefs, k = _step_scalars(S, order, step)
    eu = eu if cfg else None
    m1 = m1 if k >= 2 else None
    m2 = m2 if k >= 3 else None
    for what, fn in (("unfused", dpm_update_ref), ("fma", _fma_statement)):
        m0, xp = fn(x, ec, eu, 7.5, m1, m2, a, s, coefs)
        rep = dpm_update_check(m0, xp, x, ec, eu, 7.5, m1, m2, a, s, coefs, what=what)
        assert rep.ok, rep


MUTANTS = ["bf16_data_prediction", "sigma_s0_for_sigma_t", "swapped_k0_k1", "no_cfg_mix"]


@pytest.mark.parametrize("mutant", MUTANTS)
def test_bound_rejects_mutants(mutant):
    S, order, step = 20, 2, 5
    x, ec, eu, m1, m2 = _kernel_inputs(seed=7)
    alpha, sigma = ddim_grid(S)
    n = len(alpha) - 1
    coefs = DS.step_coefficients(alpha, sigma, DS.step_orders(n, order))[step]
    a, s = alpha[step], sigma[step]
    bad = list(coefs)
    g_eu = eu
    if mutant == "sigma_s0_for_sigma_t":
        bad[0] = sigma[step] / sigma[step]
    elif mutant == "swapped_k0_k1":
        bad[1], bad[2] = coefs[2], coefs[1]
    elif mutant == "no_cfg_mix":
        g_eu = None
    m0, xp = dpm_update_ref(x, ec, g_eu, 7.5, m1, None, a, s, bad)
    if mutant == "bf16_data_prediction":
        m0 = m0.bfloat16().float()
        xp = float(np.float32(coefs[0])) * x + float(np.float32(coefs[1])) * m0 + float(np.float32(coefs[2])) * m1.bfloat16().float()
    rep = dpm_update_check(m0, xp, x, ec, eu, 7.5, m1, None, a, s, coefs)
    print(rep)
    assert not rep.ok, f"{mutant} passed: {rep}"


def test_bound_carries_first_step_amplification():
    """The CFG error reaches the data prediction multiplied by sigma / alpha: ~11 at t = 951 (S = 20's first step) and 14.6 at
    t = 999.  A perturbation of e of that size passes through m0 at that factor, and the bound admits it."""
    ac = SO.make_schedule()["alphas_cumprod"].double()
    ratio = lambda t: math.sqrt((1 - float(ac[t])) / float(ac[t]))
    assert 10.5 < ratio(951) < 11.5 and abs(ratio(999) - 14.6) < 0.05
    assert SO.ddim_timesteps(20)[-1] == 951
    n = 4096
    x, ec, eu, _, _ = _kernel_inputs(n, seed=3)
    alpha, sigma = ddim_grid(20)
    coefs = DS.step_coefficients(alpha, sigma, DS.step_orders(len(alpha) - 1, 2))[0]
    a, s = alpha[0], sigma[0]
    _, dm0, _, _ = dpm_update_bound(x, ec, eu, 7.5, None, None, a, s, coefs)
    de = g_n(3) * (eu.double().abs() + 7.5 * (ec.double() - eu.double()).abs())
    assert torch.all(dm0 >= 0.999 * (s / a) * de)
    # a CFG mix off by one ulp-scale error per element, pushed through m0 exactly
    e = (eu.double() + 7.5 * (ec.double() - eu.double()))
    e_bad = e + 0.5 * de
    m0_bad = ((x.double() - float(np.float32(s)) * e_bad) / float(np.float32(a))).float()
    xp_bad = float(np.float32(coefs[0])) * x + float(np.float32(coefs[1])) * m0_bad
    assert dpm_update_check(m0_bad, xp_bad, x, ec, eu, 7.5, None, None, a, s, coefs).ok
