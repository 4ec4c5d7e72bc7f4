"""CPU: image-to-image (init_latent / strength / noise on every sampler's sample()) and two-pass high-resolution sampling
(gligen_b200.pipeline.sample_hires) without a GPU.

* The host logic on a stand-in model: UNet passes per (S, strength), generator draws and their order, the scheduled-sampling
  length, the refusals, and that a call without init_latent runs as before.
* The truncated DPM-Solver++ / UniPC runs on the analytic Gaussian problem (oracle/dpm_solver_oracle.py) against the exact
  probability flow from t0.
* The samplers end to end through the drop-in UNetModel on the torch-fp32 checker ops (tests/ref_ops.py), with the update kernels
  replaced by their torch statements through test-only injection (the CPU loop backend below), against the fixtures
  (tests/golden/img2img_*.pt, oracle/gen_golden_img2img.py); and the oracle itself against the fixtures.
"""
import math
import os
import subprocess
import sys
from functools import partial

import numpy as np
import pytest
import torch

from bounds_dpm import dpm_update_ref
from bounds_unipc import unipc_update_ref
from conftest import GOLD, ROOT, rel_l2
from gligen_b200 import pipeline, synth
from gligen_b200.engine import Engine
from gligen_b200.pipeline import alpha_generator, build_model, sample_hires, sampler_inputs, set_alpha_scale
from ldm.models.diffusion import _sampling
from ldm.models.diffusion import dpm_solver as DS
from ldm.models.diffusion import unipc as UP
from ldm.models.diffusion.ddim import DDIMSampler
from ldm.models.diffusion.plms import PLMSSampler
from oracle import dpm_solver_oracle as DO
from oracle import img2img_oracle as IO
from ref_ops import RefOps

KINDS = ("plms", "ddim", "dpm", "unipc")


# ---- the CPU loop backend ----------------------------------------------------------------------------------------------------
def _sampler_update(self, x, e_c, e_u, guidance_scale, olds, coefs, index, want_e):
    torch.randn_like(x)                          # the product path's draw (sigma_t == 0 noise)
    x_prev = torch.empty_like(x)
    e_out = torch.empty_like(x) if want_e else None
    RefOps().sampler_update(x.float(), e_c.float(), None if e_u is None else e_u.float(), float(guidance_scale), olds,
                            [float(c) for c in coefs], float(self.ddim_alphas[index]), float(self.ddim_alphas_prev[index]), e_out,
                            x_prev)
    return x_prev, e_out


def _dpm_update(self, x, e_c, e_u, guidance_scale, m1, m2, alpha, sigma, coefs, m0_out):
    m0, xp = dpm_update_ref(x.float(), e_c.float(), None if e_u is None else e_u.float(), guidance_scale, m1, m2, alpha, sigma, coefs)
    m0_out.copy_(m0)
    return xp


def _unipc_update(self, x, xc, e_c, e_u, guidance_scale, m1, m2, m3, alpha, sigma, coefs, m_out, xc_out):
    m0, xcn, xn = unipc_update_ref(x.float(), xc, e_c.float(), None if e_u is None else e_u.float(), guidance_scale, m1, m2, m3,
                                   alpha, sigma, coefs)
    m_out.copy_(m0)
    xc_out.copy_(xcn)
    return xn


@pytest.fixture
def cpu_updates(monkeypatch):
    monkeypatch.setattr(_sampling.SamplerBase, "_update", _sampler_update)
    monkeypatch.setattr(DS.DPMSolverSampler, "_dpm_update", _dpm_update)
    monkeypatch.setattr(UP.UniPCSampler, "_unipc_update", _unipc_update)


@pytest.fixture
def cpu_backend(monkeypatch, cpu_updates):
    from ldm.modules.diffusionmodules.openaimodel import UNetModel

    def engine(self):
        if self._engine is None:
            self._engine = Engine(self.cfg, RefOps())
            self._engine_stale = True
        if self._engine_stale:
            self._engine.load_state_dict(self.state_dict())
            self._engine_stale = False
        return self._engine

    def upscale(z, H, W):                        # glg_resize_plane's statement (bicubic, A = -0.75, align_corners = False)
        return torch.nn.functional.interpolate(z.float(), size=(H, W), mode="bicubic", align_corners=False)

    monkeypatch.setattr(UNetModel, "engine", engine)
    monkeypatch.setattr(pipeline, "upscale_latent", upscale)


def _diffusion():
    from ldm.models.diffusion.ldm import LatentDiffusion
    return LatentDiffusion(linear_start=0.00085, linear_end=0.012, timesteps=1000)


def make_sampler(kind, diffusion, model, order=2, **kw):
    if kind == "plms":
        return PLMSSampler(diffusion, model, **kw)
    if kind == "ddim":
        return DDIMSampler(diffusion, model, **kw)
    return (DS.DPMSolverSampler if kind == "dpm" else UP.UniPCSampler)(diffusion, model, order=order, **kw)


# ---- host logic on a stand-in model ------------------------------------------------------------------------------------------
class _Eps(torch.nn.Module):
    """eps = 0.1 x; records the time step of every pass."""

    def __init__(self):
        super().__init__()
        self.calls = []

    def forward(self, input):
        self.calls.append(int(input["timesteps"][0]))
        return 0.1 * input["x"]


SHAPE = (2, 4, 8, 8)


def _steps_run(S, strength):
    L = len(IO.truncated_range(S, 1.0)[0])
    return min(L, int(strength * L)), L


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("S", [10, 15, 20, 50])
@pytest.mark.parametrize("strength", [0.0, 0.02, 0.3, 0.5, 0.75, 1.0])
def test_unet_passes(cpu_updates, kind, S, strength):
    """n = min(L, int(strength L)) steps from time_range[L - n]; PLMS takes n + 1 passes (its first step evaluates twice), the
    others n.  n = 0 runs no pass and returns init_latent in fp32."""
    model = _Eps()
    sampler = make_sampler(kind, _diffusion(), model)
    init = torch.randn(SHAPE, dtype=torch.float64)
    out = sampler.sample(S, SHAPE, dict(x=None), init_latent=init, strength=strength, noise=torch.randn(SHAPE))
    n, L = _steps_run(S, strength)
    full = list(np.flip(sampler.ddim_timesteps))
    assert n == len(IO.truncated_range(S, strength)[0])
    passes = n + 1 if kind == "plms" and n > 0 else n
    assert len(model.calls) == passes, (kind, S, strength, model.calls)
    if n == 0:
        assert out.dtype == torch.float32 and torch.equal(out, init.float())
        return
    if kind == "plms":
        assert model.calls[0] == full[L - n] and model.calls[2:] == full[L - n + 1:]
        assert model.calls[1] == full[min(L - n + 1, L - 1)]               # the pseudo improved Euler point
    else:
        assert model.calls == full[L - n:]


def _count_draws(monkeypatch):
    log = []
    randn, randn_like = torch.randn, torch.randn_like

    def wrap(name, fn):
        def wrapped(*a, **k):
            log.append(name)
            return fn(*a, **k)
        return wrapped

    monkeypatch.setattr(torch, "randn", wrap("randn", randn))
    monkeypatch.setattr(torch, "randn_like", wrap("randn_like", randn_like))
    return log, randn


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("with_noise", [False, True])
@pytest.mark.parametrize("with_mask", [False, True])
def test_rng_draws(cpu_updates, monkeypatch, kind, with_noise, with_mask):
    """Without noise, one randn(shape) first, where x_T would be drawn (input['x'] is not read); with it, none.  Then the loop's
    draws as in a full run: one q_sample noise per step with a mask, and for PLMS / DDIM one dropped sigma = 0 draw per update."""
    log, randn = _count_draws(monkeypatch)
    S, strength = 10, 0.5
    n, _ = _steps_run(S, strength)
    init = randn(SHAPE)
    noise = randn(SHAPE) if with_noise else None
    mask = torch.ones(2, 1, 8, 8) if with_mask else None
    x0 = torch.zeros(SHAPE) if with_mask else None
    sampler = make_sampler(kind, _diffusion(), _Eps())
    sampler.sample(S, SHAPE, dict(x=randn(SHAPE)), mask=mask, x0=x0, init_latent=init, strength=strength, noise=noise)
    updates = {"plms": n + 1, "ddim": n, "dpm": 0, "unipc": 0}[kind]
    per_step = ["randn_like"] if with_mask else []
    expected = ([] if with_noise else ["randn"])
    if kind == "plms":
        expected += per_step + ["randn_like"] * 2 + (per_step + ["randn_like"]) * (n - 1)
    elif kind == "ddim":
        expected += (per_step + ["randn_like"]) * n
    else:
        expected += per_step * n
    assert log == expected, (kind, log)
    assert log.count("randn_like") == updates + (n if with_mask else 0)


@pytest.mark.parametrize("kind", KINDS)
def test_strength_zero_draws_nothing(cpu_updates, monkeypatch, kind):
    log, randn = _count_draws(monkeypatch)
    init = randn(SHAPE).to(torch.bfloat16)
    model = _Eps()
    out = make_sampler(kind, _diffusion(), model).sample(10, SHAPE, dict(x=None), init_latent=init, strength=0.0)
    assert log == [] and model.calls == [] and out.dtype == torch.float32 and torch.equal(out, init.float())


@pytest.mark.parametrize("kind", KINDS)
def test_without_init_latent_runs_as_before(cpu_updates, monkeypatch, kind):
    """No init_latent: x_T drawn when input['x'] is None, every step of the grid, the alphas over the whole grid; passing the new
    keywords at their defaults changes nothing, bit for bit."""
    lengths = []

    def gen(n):
        lengths.append(n)
        return [1] * n

    outs, logs, calls = [], [], []
    for extra in ({}, dict(init_latent=None, strength=1.0, noise=None)):
        log, _ = _count_draws(monkeypatch)
        torch.manual_seed(3)
        model = _Eps()
        sampler = make_sampler(kind, _diffusion(), model, alpha_generator_func=gen, set_alpha_scale=lambda m, a: None)
        outs.append(sampler.sample(10, SHAPE, dict(x=None), **extra))
        logs.append(list(log))
        calls.append(model.calls)
        monkeypatch.undo()
        monkeypatch.setattr(_sampling.SamplerBase, "_update", _sampler_update)
        monkeypatch.setattr(DS.DPMSolverSampler, "_dpm_update", _dpm_update)
        monkeypatch.setattr(UP.UniPCSampler, "_unipc_update", _unipc_update)
    L = len(IO.truncated_range(10, 1.0)[0])
    assert torch.equal(outs[0], outs[1]) and logs[0] == logs[1] and calls[0] == calls[1]
    assert logs[0][0] == "randn" and lengths == [L, L]
    assert calls[0][0] == int(IO.truncated_range(10, 1.0)[0][0])


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("strength", [0.3, 0.7, 1.0])
def test_alpha_generator_gets_steps_run(cpu_updates, kind, strength):
    """Scheduled sampling runs over the steps actually run: alpha_generator_func(n), alphas[i] at step i (a strength <= 0.7 run
    with alpha_type [0.3, 0, 0.7] still starts grounded)."""
    got, seen = [], []
    gen = partial(alpha_generator, type=[0.3, 0, 0.7])

    def record(n):
        got.append(n)
        return gen(n)

    model = _Eps()
    model.restore_first_conv_from_SD = lambda: None
    sampler = make_sampler(kind, _diffusion(), model, alpha_generator_func=record, set_alpha_scale=lambda m, a: seen.append(a))
    sampler.sample(20, SHAPE, dict(x=None), init_latent=torch.zeros(SHAPE), strength=strength)
    n, _ = _steps_run(20, strength)
    assert got == [n] and seen == gen(n) and seen[0] == 1


def test_refusals(cpu_updates):
    sampler = make_sampler("dpm", _diffusion(), _Eps())
    init = torch.zeros(SHAPE)
    for kw in (dict(init_latent=init, strength=-0.1), dict(init_latent=init, strength=1.01), dict(init_latent=init, strength=float("nan")),
               dict(init_latent=torch.zeros(2, 4, 8, 16)), dict(init_latent=init, noise=torch.zeros(1, 4, 8, 8)),
               dict(strength=0.5), dict(noise=torch.zeros(SHAPE))):
        with pytest.raises(ValueError):
            sampler.sample(10, SHAPE, dict(x=None), **kw)


# ---- the truncated run on the analytic problem -------------------------------------------------------------------------------
MU, SD = 0.5, 0.8


class _GaussEps(torch.nn.Module):
    """The optimal noise prediction for data ~ N(MU, SD^2), in float64."""

    def __init__(self, ac):
        super().__init__()
        self.ac = ac

    def forward(self, input):
        a = float(self.ac[int(input["timesteps"][0])])
        return DO.gaussian_eps(input["x"].double(), math.sqrt(a), math.sqrt(1 - a), MU, SD)


def _f64_dpm(self, x, e_c, e_u, guidance_scale, m1, m2, alpha, sigma, coefs, m0_out):
    m0, xp = dpm_update_ref(x.double(), e_c.double(), None, 1.0, m1, m2, alpha, sigma, coefs)
    m0_out.copy_(m0)
    return xp


def _f64_unipc(self, x, xc, e_c, e_u, guidance_scale, m1, m2, m3, alpha, sigma, coefs, m_out, xc_out):
    m0, xcn, xn = unipc_update_ref(x.double(), xc, e_c.double(), None, 1.0, m1, m2, m3, alpha, sigma, coefs)
    m_out.copy_(m0)
    xc_out.copy_(xcn)
    return xn


@pytest.mark.parametrize("kind", ["dpm", "unipc"])
@pytest.mark.parametrize("strength", [0.4, 0.75])
def test_truncated_run_converges_to_exact_flow(monkeypatch, kind, strength):
    """From the start state at t0 the truncated run follows the probability flow to alphas_cumprod[0]: its error against the exact
    solution through that state falls as S grows (t0 moves with S; the exact solution is taken from each run's own t0)."""
    monkeypatch.setattr(DS.DPMSolverSampler, "_dpm_update", _f64_dpm)
    monkeypatch.setattr(UP.UniPCSampler, "_unipc_update", _f64_unipc)
    diffusion = _diffusion()
    ac = diffusion.alphas_cumprod.double()
    z = torch.linspace(-2.5, 2.5, 11, dtype=torch.float64)
    init = (MU + SD * z).reshape(1, 1, 1, 11)
    noise = torch.linspace(-1.5, 1.5, 11).reshape(1, 1, 1, 11)
    errs = []
    for S in (10, 20, 40, 80, 160):
        sampler = make_sampler(kind, diffusion, _GaussEps(ac))
        got = sampler.sample(S, (1, 1, 1, 11), dict(x=None), init_latent=init, strength=strength, noise=noise)
        t0 = int(IO.truncated_range(S, strength)[0][0])
        a0 = float(ac[t0])
        x_t0 = diffusion.q_sample(init.float(), torch.tensor([t0]), noise=noise).double()      # the fp32 start state the run used
        exact = DO.gaussian_flow(x_t0, math.sqrt(a0), math.sqrt(1 - a0), math.sqrt(float(ac[0])), math.sqrt(1 - float(ac[0])), MU, SD)
        errs.append((got.double() - exact).abs().max().item())
    print(f"{kind} strength {strength}: errors {errs}")
    assert all(errs[k] >= 2.0 * errs[k + 1] for k in range(len(errs) - 1)), errs
    assert errs[-1] < 0.03 * errs[0], errs


# ---- the samplers through the drop-in UNetModel against the fixtures -----------------------------------------------------------
def _cfg(name):
    from gligen_b200.spec import NAMED_CONFIGS
    return NAMED_CONFIGS[name]


def run_case(gold, device="cpu", hires=False):
    """The product's run of a fixture: (model, final latent)."""
    cfg, model = build_model(_cfg(gold["config"]), device)
    inp = synth.make_inputs(cfg, gold["B"], gold["max_objs"], seed=gold["seed"])
    to = lambda t: t.to(device)
    input, mask, x0 = sampler_inputs(cfg, model, {k: to(inp[k]) for k in ("x", "context", "uc", "z0") if k in inp},
                                     {k: to(v) for k, v in inp["batch"].items()})
    sampler = make_sampler(gold["sampler"], _diffusion().to(device), model, order=gold["order"] or 2,
                           alpha_generator_func=partial(alpha_generator, type=gold["alpha_type"]), set_alpha_scale=set_alpha_scale)
    shape = tuple(inp["x"].shape)
    cwd = os.getcwd()
    os.chdir(GOLD)                               # restore_first_conv_from_SD reads a CWD-relative file, like the reference
    try:
        torch.manual_seed(gold["noise_seed"])
        if hires:
            return model, sample_hires(sampler, gold["S"], shape, input, to(inp["uc"]), gold["guidance"], scale=gold["scale"],
                                       strength=gold["strength"])
        init, noise = IO.init_and_noise(shape, gold["init_seed"])
        return model, sampler.sample(gold["S"], shape, input, to(inp["uc"]), gold["guidance"], mask=mask, x0=x0,
                                     init_latent=to(init), strength=gold["strength"], noise=to(noise))
    finally:
        os.chdir(cwd)


TINY_FIXTURES = ["img2img_tiny_plms.pt", "img2img_tiny_ddim.pt", "img2img_tiny_dpm2.pt", "img2img_tiny_unipc2.pt",
                 "img2img_tiny_inpaint_dpm2.pt"]


@pytest.mark.parametrize("gold_file", TINY_FIXTURES)
def test_loop_matches_fixture(cpu_backend, gold_file):
    """Every sampler at strength 0.5 / 0.6 (and the inpainting blend with init_latent) through the checker ops, against the
    oracle.  Both run their UNet in fp32 with different operation orders."""
    gold = torch.load(os.path.join(GOLD, gold_file))
    _, lat = run_case(gold)
    r = rel_l2(lat, gold["latent"])
    print(f"{gold_file}: rel-L2 {r:.3e}")
    assert r < 2e-4, r


def test_hires_matches_fixture(cpu_backend, monkeypatch):
    """sample_hires on the tiny model, 16 x 16 -> 32 x 32: pass 1, bicubic upscale, pass 2 at strength 0.5 drawing its noise from
    the generator; against the oracle's composition from the pass-1 fixture."""
    gold = torch.load(os.path.join(GOLD, "img2img_hires_tiny_dpm2.pt"))
    pass1 = torch.load(os.path.join(GOLD, gold["pass1"]))
    _, lat = run_case(dict(gold, sampler="dpm"), hires=True)
    assert tuple(lat.shape) == (gold["B"], 4, 32, 32)
    r = rel_l2(lat, gold["latent"])
    print(f"hires: rel-L2 {r:.3e} (pass-1 fixture S={pass1['S']})")
    assert r < 2e-4, r


def test_hires_refusals(cpu_backend):
    cfg, model = build_model("tiny", "cpu", load_weights=False)
    sampler = make_sampler("dpm", _diffusion(), model)
    for kw in (dict(scale=1.3), dict(scale=0.25), dict(strength=1.5)):
        with pytest.raises(ValueError):
            sample_hires(sampler, 6, (1, 4, 16, 16), dict(x=None), None, 1.0, **kw)
    _, inpaint = build_model("tiny_inpaint", "cpu", load_weights=False)
    with pytest.raises(ValueError, match="inpainting"):
        sample_hires(make_sampler("dpm", _diffusion(), inpaint), 6, (1, 4, 16, 16), dict(x=None), None, 1.0)


def _oracle_case(gold_file):
    """The oracle's run of a fixture, as oracle/gen_golden_img2img.py made it."""
    from oracle import gen_golden_img2img as G
    gold = torch.load(os.path.join(GOLD, gold_file))
    cfg = _cfg(gold["config"])
    init, noise = IO.init_and_noise((gold["B"], 4, cfg.image_size, cfg.image_size), gold["init_seed"])
    return gold, G.oracle_latent(cfg, gold["sampler"], gold["order"], gold["S"], gold["strength"], gold["alpha_type"], init, noise,
                                 gold["B"], gold["max_objs"])


@pytest.mark.parametrize("gold_file", ["img2img_tiny_dpm2.pt", "img2img_tiny_unipc2.pt", "img2img_tiny_inpaint_dpm2.pt"])
def test_oracle_reproduces_fixture(gold_file):
    gold, lat = _oracle_case(gold_file)
    assert torch.equal(lat, gold["latent"]) or rel_l2(lat, gold["latent"]) < 1e-6


def _reference_available():
    from oracle import build_ref
    return os.path.isdir(build_ref.REF) or build_ref.available()


@pytest.mark.skipif(not _reference_available(), reason="needs the reference (oracle/build_ref.py archive or checkout)")
@pytest.mark.parametrize("gold_file", ["img2img_tiny_plms.pt", "img2img_tiny_ddim.pt"])
def test_reference_oracle_reproduces_fixture(gold_file):
    """PLMS / DDIM step through the reference's own p_sample_plms / p_sample_ddim, which must be imported in a process that has
    not imported this repo's ldm."""
    code = (f"import os, sys, torch; sys.path.insert(0, {ROOT!r})\n"
            "from oracle import ref_harness as RH; RH.mount()\n"
            "from gligen_b200.spec import NAMED_CONFIGS\n"
            "from oracle import gen_golden_img2img as G, img2img_oracle as IO\n"
            f"gold = torch.load({os.path.join(GOLD, gold_file)!r}); cfg = NAMED_CONFIGS[gold['config']]\n"
            "init, noise = IO.init_and_noise((gold['B'], 4, cfg.image_size, cfg.image_size), gold['init_seed'])\n"
            "lat = G.oracle_latent(cfg, gold['sampler'], gold['order'], gold['S'], gold['strength'], gold['alpha_type'], init, noise,"
            " gold['B'], gold['max_objs'])\n"
            "print(((lat - gold['latent']).norm() / gold['latent'].norm()).item())\n")
    out = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, timeout=900)
    assert out.returncode == 0, out.stderr[-3000:]
    assert float(out.stdout.strip().splitlines()[-1]) < 1e-6, out.stdout
