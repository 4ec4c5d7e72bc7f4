"""CPU: the stochastic samplers (DDIMSampler.sample(eta > 0), DPMSolverSampler(eta > 0): DPM-Solver++ 2M SDE) without a GPU.

* The float64 coefficient expansions: at eta = 0 they reduce to the deterministic DDIM step and to step_coefficients; at eta > 0
  they equal the reference's DDIM sigma_t form and the VE-form 2M SDE step of oracle/sde_oracle.py.
* Exact moment propagation on Gaussian data: the final mean and variance converge to the true marginal at alphas_cumprod[0] as S
  grows, at the orders stated in DESIGN §2.
* The host logic on a stand-in model: generator draws and their order, refusals, and that eta = 0 keeps the deterministic path.
* The samplers end to end through the drop-in UNetModel on the torch-fp32 checker ops (tests/ref_ops.py), with the update kernel
  replaced by its torch statement (tests/bounds_sde.py), against the fixtures (tests/golden/sde_*.pt, oracle/gen_golden_sde.py).
* The kernel's float64 bound against the faithful fp32 statement and against realistic mistakes.
"""
import math
import os
from functools import partial

import numpy as np
import pytest
import torch

from bounds_dpm import dpm_update_ref
from bounds_sde import sde_update_check, sde_update_ref
from conftest import GOLD, rel_l2
from gligen_b200 import synth
from gligen_b200.engine import Engine
from gligen_b200.pipeline import alpha_generator, build_model, sampler_inputs, set_alpha_scale
from ldm.models.diffusion import _sampling
from ldm.models.diffusion import dpm_solver as DS
from ldm.models.diffusion.ddim import DDIMSampler, ddim_sde_coefficients
from ldm.models.diffusion.plms import PLMSSampler
from oracle import img2img_oracle as IO
from oracle import sampler_oracle as SO
from oracle import sde_oracle as SDO
from ref_ops import RefOps

STEP_COUNTS = (4, 6, 10, 14, 15, 20, 25, 50)


def _diffusion():
    from ldm.models.diffusion.ldm import LatentDiffusion
    return LatentDiffusion(linear_start=0.00085, linear_end=0.012, timesteps=1000)


def ddim_grid(S):
    return DS.grid_alpha_sigma(SO.make_schedule()["alphas_cumprod"], np.flip(SO.ddim_timesteps(S)))


def _ddim_tables(S, eta):
    """float64 (a_t, a_prev, sigma_t) per DDIM index, as make_schedule computes them."""
    s = DDIMSampler(_diffusion(), None)
    s.make_schedule(S, ddim_eta=eta)
    return s._alphas_host, s._alphas_prev_host, s._sigmas_host


# ---- coefficients ------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("S", STEP_COUNTS)
def test_ddim_coefficients_reduce_at_eta_zero(S):
    """eta = 0: cx x + k0 m0 + ce e + cz z is glg_sampler_update's x_prev = sqrt(a_prev) m0 + sqrt(1 - a_prev) e, to 1e-12."""
    a, ap, sg = _ddim_tables(S, 0.0)
    assert max(sg) == 0.0
    g = torch.Generator().manual_seed(S)
    for i in range(len(a)):
        x, e, z = (torch.randn(64, generator=g, dtype=torch.float64) for _ in range(3))
        cx, k0, k1, ce, cz = ddim_sde_coefficients(a[i], ap[i], sg[i])
        assert cx == 0.0 and k1 == 0.0 and cz == 0.0
        m0 = (x - math.sqrt(1 - a[i]) * e) / math.sqrt(a[i])
        got = cx * x + k0 * m0 + ce * e + cz * z
        ref = math.sqrt(ap[i]) * m0 + math.sqrt(1 - ap[i]) * e
        assert (got - ref).abs().max().item() <= 1e-12 * (m0.abs() + e.abs()).max().item()


@pytest.mark.parametrize("eta", [0.5, 1.0])
@pytest.mark.parametrize("S", STEP_COUNTS)
def test_ddim_coefficients_are_the_references_step(S, eta):
    """eta > 0: sigma_t = eta sqrt((1 - a_prev) / (1 - a_t)) sqrt(1 - a_t / a_prev) (ddim.py make_ddim_sampling_parameters) and
    the step sqrt(a_prev) pred_x0 + sqrt(1 - a_prev - sigma_t^2) e + sigma_t z."""
    a, ap, sg = _ddim_tables(S, eta)
    ref_sig, ref_a, ref_ap = SO.ddim_parameters(SO.make_schedule()["alphas_cumprod"], SO.ddim_timesteps(S), eta)
    for i in range(len(a)):
        want = eta * math.sqrt((1 - ap[i]) / (1 - a[i]) * (1 - a[i] / ap[i]))
        # ddim_sigmas is make_ddim_sampling_parameters' (the reference's) evaluation on the fp32 alphas_cumprod
        assert abs(sg[i] - want) <= 1e-6 * want and abs(sg[i] - float(ref_sig[i])) <= 1e-6 * want
        cx, k0, k1, ce, cz = ddim_sde_coefficients(a[i], ap[i], sg[i])
        assert (cx, k1) == (0.0, 0.0) and k0 == math.sqrt(ap[i]) and cz == sg[i]
        assert abs(ce - math.sqrt(1 - ap[i] - sg[i] ** 2)) <= 1e-15
    if eta == 1.0:           # eta = 1 is the DDPM posterior variance: a_prev's noise split into ce^2 + cz^2
        for i in range(len(a)):
            _, _, _, ce, cz = ddim_sde_coefficients(a[i], ap[i], sg[i])
            assert abs(ce ** 2 + cz ** 2 - (1 - ap[i])) <= 1e-12


@pytest.mark.parametrize("order", [1, 2])
@pytest.mark.parametrize("S", STEP_COUNTS)
def test_sde_coefficients_reduce_to_step_coefficients(S, order):
    """eta = 0: (cx, k0, k1) equal step_coefficients' for orders 1 and 2, and ce = cz = 0, to 1e-12."""
    alpha, sigma = ddim_grid(S)
    orders = DS.step_orders(len(alpha) - 1, order)
    det = DS.step_coefficients(alpha, sigma, orders)
    sde = DS.sde_coefficients(alpha, sigma, orders, 0.0)
    assert np.all(sde[:, 3:] == 0.0) and np.all(det[:, 3] == 0.0)
    assert np.abs(sde[:, :3] - det[:, :3]).max() <= 1e-12 * np.abs(det[:, :3]).max()


@pytest.mark.parametrize("eta", [0.25, 0.5, 1.0])
@pytest.mark.parametrize("S", STEP_COUNTS)
def test_sde_coefficients_match_ve_form(S, eta):
    """Each step's (cx, k0, k1, cz) applied to random float64 state equals sde_oracle's VE-form step (times alpha_t) to 1e-12;
    the last step (to alphas_cumprod[0], sigma > 0) keeps its noise term."""
    alpha, sigma = ddim_grid(S)
    orders = DS.step_orders(len(alpha) - 1, 2)
    coefs = DS.sde_coefficients(alpha, sigma, orders, eta)
    sig = sigma / alpha
    g = torch.Generator().manual_seed(S)
    for i, k in enumerate(orders):
        x, m0, m1, z = (torch.randn(64, generator=g, dtype=torch.float64) for _ in range(4))
        cx, k0, k1, ce, cz = coefs[i]
        assert ce == 0.0 and cz > 0.0 and (k == 2 or k1 == 0.0)
        got = cx * x + k0 * m0 + k1 * m1 + cz * z
        h_prev = math.log(sig[i - 1]) - math.log(sig[i]) if i > 0 else None
        ref = alpha[i + 1] * SDO.sde_step_ve(x / alpha[i], m0, m1 if k == 2 else None, sig[i], sig[i + 1], h_prev, eta, z)
        scale = (abs(cx) * x.abs() + abs(k0) * m0.abs() + abs(k1) * m1.abs() + cz * z.abs()).max().item()
        assert (got - ref).abs().max().item() <= 1e-12 * scale, (S, eta, i, k)


# ---- exact moment propagation on Gaussian data ------------------------------------------------------------------------------
MU, SD = 0.5, 0.8


def _propagate(S, steps):
    """Mean and variance of the final state when x_0 ~ N(MU, SD^2), starting from the exact marginal at the first grid point.
    steps(S) -> (alpha [n + 1], sigma [n + 1], rows [n] of (cx, k0, k1, ce, cz)).  The exact data prediction
    m(x) = A x + B, A = alpha SD^2 / v, B = MU sigma^2 / v, v = alpha^2 SD^2 + sigma^2, is affine, so (x_i, m_{i-1}) stays jointly
    Gaussian: its mean and covariance go through each step in float64, with cz^2 added to the variance of x."""
    alpha, sigma, rows = steps(S)
    mean = np.array([alpha[0] * MU, 0.0])
    cov = np.diag([alpha[0] ** 2 * SD ** 2 + sigma[0] ** 2, 0.0])
    for i, (cx, k0, k1, ce, cz) in enumerate(rows):
        a, s = alpha[i], sigma[i]
        v = a * a * SD * SD + s * s
        A, B = a * SD * SD / v, MU * s * s / v
        # e = (x - a m) / s; x' = cx x + k0 m + k1 m_prev + ce e + cz z; m = A x + B
        cxx = cx + k0 * A + ce * (1.0 - a * A) / s
        cb = k0 * B - ce * a * B / s
        M = np.array([[cxx, k1], [A, 0.0]])
        mean = M @ mean + np.array([cb, B])
        cov = M @ cov @ M.T + np.diag([cz * cz, 0.0])
    return mean[0], cov[0, 0], alpha[-1] * MU, alpha[-1] ** 2 * SD ** 2 + sigma[-1] ** 2


def _ddim_steps(eta):
    def steps(S):
        a, ap, sg = _ddim_tables(S, eta)
        idx = list(range(len(a)))[::-1]                              # step i runs DDIM index n - i - 1
        alpha = [math.sqrt(a[j]) for j in idx] + [math.sqrt(ap[0])]
        sigma = [math.sqrt(1 - a[j]) for j in idx] + [math.sqrt(1 - ap[0])]
        return alpha, sigma, [ddim_sde_coefficients(a[j], ap[j], sg[j]) for j in idx]
    return steps


def _sde_steps(eta, order):
    def steps(S):
        alpha, sigma = ddim_grid(S)
        return alpha, sigma, DS.sde_coefficients(alpha, sigma, DS.step_orders(len(alpha) - 1, order), eta)
    return steps


MOMENT_S = (25, 50, 100, 200, 500)
# (sampler, eta, order): the least convergence order of the final variance error measured over the last two refinements of
# MOMENT_S (S = 100 -> 200 -> 500; orders over the step-count ratio), stated in DESIGN §2
MOMENT_ORDERS = {("ddim", 0.5, 1): 0.85, ("ddim", 1.0, 1): 0.8, ("sde", 0.5, 1): 0.85, ("sde", 1.0, 1): 0.8,
                 ("sde", 0.5, 2): 1.65, ("sde", 1.0, 2): 1.6}


@pytest.mark.parametrize("kind,eta,order", list(MOMENT_ORDERS))
def test_moments_converge_to_marginal(kind, eta, order):
    """The final mean is exact to rounding at every S (each step is exact when the data prediction is a constant); the final
    variance converges to the marginal's at the order of the step (1 for DDIM and order-1 SDE, 2 for 2M SDE)."""
    steps = _ddim_steps(eta) if kind == "ddim" else _sde_steps(eta, order)
    ev, ns = [], []
    for S in MOMENT_S:
        m, v, m_true, v_true = _propagate(S, steps)
        assert abs(m - m_true) <= 1e-12, (S, m, m_true)
        ev.append(abs(v - v_true))
        ns.append(len(SO.ddim_timesteps(S)))
    obs = [math.log(ev[j] / ev[j + 1]) / math.log(ns[j + 1] / ns[j]) for j in range(len(ev) - 1)]
    print(f"{kind} eta={eta} order={order}: variance errors {ev} (orders {obs})")
    assert min(obs[-2:]) >= MOMENT_ORDERS[(kind, eta, order)], obs
    assert ev[-1] < 1.2e-2


@pytest.mark.parametrize("S", STEP_COUNTS)
def test_ddim_eta_one_is_first_order_sde(S):
    """DDIM at eta = 1 and the order-1 SDE step at eta = 1 are the same step (the DDPM posterior): with e = (x - alpha m) / sigma
    substituted, their coefficients of x, m and z agree to the fp32 rounding of the DDIM sigmas (relative 1e-5)."""
    a, ap, sg = _ddim_tables(S, 1.0)
    alpha, sigma, rows = _ddim_steps(1.0)(S)
    sde = DS.sde_coefficients(alpha, sigma, [1] * len(rows), 1.0)
    for i, (cx, k0, k1, ce, cz) in enumerate(rows):
        as_sde = (cx + ce / sigma[i], k0 - ce * alpha[i] / sigma[i], k1, 0.0, cz)
        # the DDIM sigmas come from an fp32 evaluation (make_ddim_sampling_parameters); 1 - a_prev - sigma_t^2 cancels
        assert np.allclose(as_sde, sde[i], rtol=1e-5, atol=1e-12), (S, i, as_sde, sde[i])


# ---- host logic on a stand-in model ------------------------------------------------------------------------------------------
def _sde_update(self, x, e_c, e_u, guidance_scale, m1, z, alpha, sigma, coefs, m0_out):
    m0, xn = sde_update_ref(x.float(), e_c.float(), None if e_u is None else e_u.float(), guidance_scale, m1, z.float(), alpha, sigma,
                            coefs)
    if m0_out is not None:
        m0_out.copy_(m0)
    return xn


class _Eps(torch.nn.Module):
    def __init__(self):
        super().__init__()
        self.calls = 0

    def forward(self, input):
        self.calls += 1
        return 0.1 * input["x"]


SHAPE = (2, 4, 8, 8)


def _make(kind, eta, **kw):
    if kind == "ddim":
        return DDIMSampler(_diffusion(), _Eps(), **kw)
    return DS.DPMSolverSampler(_diffusion(), _Eps(), order=2, eta=eta, **kw)


def _sample(kind, sampler, eta, S, x, **kw):
    if kind == "ddim":
        return sampler.sample(S, SHAPE, dict(x=x), eta=eta, **kw)
    return sampler.sample(S, SHAPE, dict(x=x), **kw)


@pytest.mark.parametrize("kind", ["ddim", "dpm"])
@pytest.mark.parametrize("with_mask", [False, True])
@pytest.mark.parametrize("with_x", [False, True])
@pytest.mark.parametrize("with_init", [False, True])
def test_rng_draws(monkeypatch, kind, with_mask, with_x, with_init):
    """randn(shape) first for x_T when input['x'] is None (or, with init_latent, for the start noise; input['x'] is then not
    read); then per step the inpainting blend's q_sample noise with a mask, followed by the step noise z after the model pass,
    the last step included.  Nothing else."""
    monkeypatch.setattr(_sampling.SamplerBase, "_sde_update", _sde_update)
    log = []
    randn, randn_like = torch.randn, torch.randn_like
    import sys

    def wrap(name, fn):
        def wrapped(*a, **k):
            log.append((name, sys._getframe(1).f_code.co_name))
            return fn(*a, **k)
        return wrapped

    monkeypatch.setattr(torch, "randn", wrap("randn", randn))
    monkeypatch.setattr(torch, "randn_like", wrap("randn_like", randn_like))
    S, strength = 10, 0.5
    x = randn(SHAPE) if with_x else None
    mask = torch.ones(2, 1, 8, 8) if with_mask else None
    x0 = torch.zeros(SHAPE) if with_mask else None
    kw = dict(init_latent=randn(SHAPE), strength=strength) if with_init else {}
    sampler = _make(kind, 1.0)
    out = _sample(kind, sampler, 1.0, S, x, mask=mask, x0=x0, **kw)
    assert torch.isfinite(out).all()
    L = len(SO.ddim_timesteps(S))
    n = min(L, int(strength * L)) if with_init else L
    assert sampler.model.calls == n
    step = [("randn_like", "q_sample")] if with_mask else []
    step = step + [("randn_like", "_sde_step" if kind == "ddim" else "sde_fn")]
    first = [] if (with_x and not with_init) else [("randn", "_begin")]
    assert log == first + step * n, log


@pytest.mark.parametrize("kind", ["ddim", "dpm"])
def test_eta_zero_keeps_the_deterministic_path(monkeypatch, kind):
    """eta = 0 (default or explicit) never reaches glg_sde_update and gives the same latent, bit for bit."""
    def _sampler_update(self, x, e_c, e_u, guidance_scale, olds, coefs, index, want_e):
        torch.randn_like(x)
        x_prev = torch.empty_like(x)
        RefOps().sampler_update(x.float(), e_c.float(), None, 1.0, olds, [float(c) for c in coefs], self._alphas_host[index],
                                self._alphas_prev_host[index], None, x_prev)
        return x_prev, None

    def _dpm_update(self, x, e_c, e_u, guidance_scale, m1, m2, alpha, sigma, coefs, m0_out):
        m0, xp = dpm_update_ref(x.float(), e_c.float(), None, 1.0, m1, m2, alpha, sigma, coefs)
        m0_out.copy_(m0)
        return xp

    monkeypatch.setattr(_sampling.SamplerBase, "_update", _sampler_update)
    monkeypatch.setattr(DS.DPMSolverSampler, "_dpm_update", _dpm_update)

    def refuse(*a, **k):
        raise AssertionError("glg_sde_update reached at eta = 0")

    monkeypatch.setattr(_sampling.SamplerBase, "_sde_update", refuse)
    outs = []
    for explicit in (False, True):
        torch.manual_seed(5)
        if kind == "ddim":
            s = DDIMSampler(_diffusion(), _Eps())
            outs.append(s.sample(10, SHAPE, dict(x=None), eta=0.0) if explicit else s.sample(10, SHAPE, dict(x=None)))
        else:
            s = DS.DPMSolverSampler(_diffusion(), _Eps(), eta=0.0) if explicit else DS.DPMSolverSampler(_diffusion(), _Eps())
            outs.append(s.sample(10, SHAPE, dict(x=None)))
    assert torch.equal(outs[0], outs[1])


def test_refusals():
    with pytest.raises(ValueError, match="eta"):
        DDIMSampler(_diffusion(), _Eps()).sample(10, SHAPE, dict(x=None), eta=1.5)
    with pytest.raises(ValueError, match="eta"):
        DDIMSampler(_diffusion(), _Eps()).make_schedule(10, ddim_eta=-0.1)
    with pytest.raises(ValueError, match="PLMS"):
        PLMSSampler(_diffusion(), _Eps()).make_schedule(10, ddim_eta=0.5)
    with pytest.raises(ValueError, match="orders 1 and 2"):
        DS.DPMSolverSampler(_diffusion(), _Eps(), order=3, eta=0.5)
    with pytest.raises(ValueError, match="eta"):
        DS.DPMSolverSampler(_diffusion(), _Eps(), order=2, eta=2.0)
    DS.DPMSolverSampler(_diffusion(), _Eps(), order=3, eta=0.0)
    PLMSSampler(_diffusion(), _Eps()).make_schedule(10, ddim_eta=0.0)


# ---- the loops through the checker-op engine against the fixtures ------------------------------------------------------------
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
    monkeypatch.setattr(_sampling.SamplerBase, "_sde_update", _sde_update)


def fixture_config(gold):
    from gligen_b200.spec import NAMED_CONFIGS, SAMPLING_GATED_CA
    return SAMPLING_GATED_CA if gold["config"] == "sampling_gated_ca" else NAMED_CONFIGS[gold["config"]]


def run_fixture(gold, device="cpu"):
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
    if gold["sampler"] == "ddim":
        sampler = DDIMSampler(diffusion, model, alpha_generator_func=gen, set_alpha_scale=set_alpha_scale)
        kw["eta"] = gold["eta"]
    else:
        sampler = DS.DPMSolverSampler(diffusion, model, alpha_generator_func=gen, set_alpha_scale=set_alpha_scale, order=gold["order"],
                                      eta=gold["eta"])
    cwd = os.getcwd()
    os.chdir(GOLD)                               # restore_first_conv_from_SD reads a CWD-relative file, like the reference
    try:
        torch.manual_seed(gold["noise_seed"])
        return sampler.sample(S=gold["S"], shape=shape, input=input, uc=inp["uc"], guidance_scale=gold["guidance"], mask=mask, x0=x0,
                              **kw)
    finally:
        os.chdir(cwd)


SDE_FIXTURES = ["sde_ddim_eta05_tiny.pt", "sde_ddim_eta1_tiny.pt", "sde_ddim_eta1_tiny_inpaint.pt",
                "sde_ddim_eta1_sampling_gated_ca.pt", "sde_ddim_eta1_sd14_box_text.pt", "sde_ddim_eta1_img2img_tiny.pt",
                "sde_dpm2sde_tiny.pt", "sde_dpm2sde_tiny_inpaint.pt", "sde_dpm2sde_sampling_gated_ca.pt",
                "sde_dpm2sde_sd14_box_text.pt", "sde_dpm2sde_img2img_tiny.pt"]


@pytest.mark.parametrize("gold_file", [f for f in SDE_FIXTURES if "sd14" not in f])
def test_loops_match_fixtures(cpu_backend, gold_file):
    """DDIM-eta against the reference's own DDIMSampler, 2M SDE against the float64 VE-form oracle, both over the fp32 UNet oracle;
    scheduled sampling with the first-conv swap, the inpainting blend and image-to-image at strength 0.5 included."""
    gold = torch.load(os.path.join(GOLD, gold_file))
    lat = run_fixture(gold)
    r = rel_l2(lat, gold["latent"])
    print(f"{gold_file}: rel-L2 {r:.3e}")
    assert r < 2e-5, r


# ---- the kernel's bound ------------------------------------------------------------------------------------------------------
def _kernel_inputs(n=4096, seed=0):
    g = torch.Generator().manual_seed(seed)
    return [torch.randn(n, generator=g) for _ in range(5)]          # x, e_c, e_u, m1, z


def _fma_statement(x, ec, eu, g, m1, z, a, s, coefs):
    """The kernel's statement as nvcc contracts it: every a * b + c one rounding (exact in float64, then rounded to fp32)."""
    r = lambda t: t.float().double()
    f = lambda v: float(np.float32(v))
    x64, e = x.double(), ec.double()
    if eu is not None:
        e = r(f(g) * r(e - eu.double()) + eu.double())
    m0 = r(r(-f(s) * e + x64) / f(a))
    xn = r(f(coefs[0]) * x64)
    for c, m in zip(coefs[1:], (m0, m1, e, z)):
        if m is not None:
            xn = r(f(c) * m.double() + xn)
    return m0.float(), xn.float()


def _step(kind, S, step, eta):
    """(alpha, sigma, coefs, has m1) of one step of a schedule."""
    if kind == "ddim":
        a, ap, sg = _ddim_tables(S, eta)
        j = (len(a) - 1 - step) % len(a)
        return math.sqrt(a[j]), math.sqrt(1 - a[j]), ddim_sde_coefficients(a[j], ap[j], sg[j]), False
    alpha, sigma = ddim_grid(S)
    orders = DS.step_orders(len(alpha) - 1, 2)
    i = step % len(orders)
    return alpha[i], sigma[i], DS.sde_coefficients(alpha, sigma, orders, eta)[i], orders[i] == 2


@pytest.mark.parametrize("kind,S,step,eta", [("ddim", 20, 0, 1.0), ("ddim", 50, 10, 0.5), ("ddim", 25, -1, 1.0),
                                              ("sde", 20, 0, 1.0), ("sde", 20, 5, 0.5), ("sde", 25, -1, 1.0), ("sde", 50, 30, 1.0)])
@pytest.mark.parametrize("cfg", [True, False])
def test_bound_accepts_fp32_statements(kind, S, step, eta, cfg):
    x, ec, eu, m1, z = _kernel_inputs(seed=S + step)
    a, s, coefs, has_m1 = _step(kind, S, step, eta)
    eu = eu if cfg else None
    m1 = m1 if has_m1 else None
    for what, fn in (("unfused", sde_update_ref), ("fma", _fma_statement)):
        m0, xn = fn(x, ec, eu, 7.5, m1, z, a, s, coefs)
        rep = sde_update_check(m0, xn, x, ec, eu, 7.5, m1, z, a, s, coefs, what=what)
        assert rep.ok, rep


MUTANTS = ["no_noise", "noise_scaled_by_sigma_s", "no_direction_term", "bf16_noise", "no_cfg_mix", "swapped_k0_k1"]


@pytest.mark.parametrize("mutant", MUTANTS)
def test_bound_rejects_mutants(mutant):
    x, ec, eu, m1, z = _kernel_inputs(seed=7)
    kind = "ddim" if mutant in ("no_direction_term",) else "sde"
    a, s, coefs, has_m1 = _step(kind, 20, 5, 1.0)
    m1 = m1 if has_m1 else None
    bad = list(coefs)
    g_eu, g_z = eu, z
    if mutant == "no_noise":
        bad[4] = 0.0
    elif mutant == "noise_scaled_by_sigma_s":
        bad[4] = coefs[4] * s / float(ddim_grid(20)[1][6])
    elif mutant == "no_direction_term":
        bad[3] = 0.0
    elif mutant == "bf16_noise":
        g_z = z.bfloat16().float()
    elif mutant == "no_cfg_mix":
        g_eu = None
    elif mutant == "swapped_k0_k1":
        bad[1], bad[2] = coefs[2], coefs[1]
    m0, xn = sde_update_ref(x, ec, g_eu, 7.5, m1, g_z, a, s, bad)
    rep = sde_update_check(m0, xn, x, ec, eu, 7.5, m1, z, a, s, coefs)
    print(rep)
    assert not rep.ok, f"{mutant} passed: {rep}"
