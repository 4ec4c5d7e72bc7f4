"""GPU: fractional timesteps through every layer (glg_timestep_embedding_f32, the engine's fp32-timestep plans, the drop-in UNetModel,
exported plans) and the Karras-grid samplers over the drop-in UNetModel against the fixtures (tests/golden/karras_*.pt,
oracle/gen_golden_karras.py).  Forward tolerance as tests/test_engine_gpu.py (rel-L2 <= 2.5e-2, max-abs <= 9 % of max|eps|), loop
tolerance rel-L2 <= 6e-2 and max-abs <= 10 % of max|latent| (bf16 UNet against the fp32 oracle), with the blend's and the SDE's
noise drawn from the CPU generator, as the fixtures draw it."""
import os
from functools import partial

import pytest
import torch

import bounds
from conftest import GOLD, assert_close
from gligen_b200 import synth
from gligen_b200.export import export_plan
from gligen_b200.pipeline import alpha_generator, build_model, sampler_inputs, set_alpha_scale, to_device
from gligen_b200.spec import NAMED_CONFIGS, SAMPLING_GATED_CA
from ldm.models.diffusion import dpm_solver as DS
from ldm.models.diffusion import unipc as UP
from native_plan import DEV, PlanCase
from oracle import sampler_oracle as SO

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ops():
    from gligen_b200.ops import CudaOps
    return CudaOps(DEV)


# ---- the kernel -------------------------------------------------------------------------------------------------------------
GUARD = 64


def _embed(ops, t, dim):
    """out written into the middle of a NaN-filled buffer; the guards must come back untouched."""
    B = t.numel()
    buf = torch.full((B * dim + 2 * GUARD,), float("nan"), device=DEV, dtype=torch.bfloat16)
    out = buf[GUARD:GUARD + B * dim].view(B, dim)
    ops.timestep_embedding(t, out)
    torch.cuda.synchronize()
    assert torch.isnan(buf[:GUARD].float()).all() and torch.isnan(buf[GUARD + B * dim:].float()).all(), "write outside out"
    return out


@pytest.mark.parametrize("dim", sorted({c.model_channels for c in NAMED_CONFIGS.values()} | {SAMPLING_GATED_CA.model_channels}))
@pytest.mark.parametrize("B", [1, 7, 64, 128])
def test_f32_kernel_within_bound(ops, dim, B):
    g = torch.Generator(device=DEV).manual_seed(dim * 1000 + B)
    t = torch.rand(B, generator=g, device=DEV) * 1000.0
    t[0] = 0.0
    out = _embed(ops, t, dim)
    rep = bounds.timestep_embedding_check(out, t, what=f"timestep_embedding_f32 dim={dim} B={B}")
    print(rep)
    assert rep.ok, str(rep)


@pytest.mark.parametrize("dim", [32, 64, 320])
def test_f32_kernel_equals_int64_kernel_at_integer_t(ops, dim):
    t = torch.arange(0, 1000, 7, device=DEV, dtype=torch.int64)
    a = _embed(ops, t, dim)
    b = _embed(ops, t.float(), dim)
    assert torch.equal(a, b)


# ---- the forward ------------------------------------------------------------------------------------------------------------
def _model_case(gold):
    cfg, model = build_model(gold["config"], DEV)
    inp = synth.make_inputs(cfg, gold["B"], gold["max_objs"], seed=gold["seed"])
    grounding = model.grounding_tokenizer_input.prepare(to_device(inp["batch"], DEV))
    return cfg, model, inp, grounding


@pytest.mark.parametrize("name", ["tiny", "sd14_box_text"])
def test_forward_at_fractional_t(name):
    gold = torch.load(os.path.join(GOLD, f"karras_unet_{name}.pt"))
    cfg, model, inp, grounding = _model_case(gold)
    x, ctx, uc = inp["x"].to(DEV), inp["context"].to(DEV), inp["uc"].to(DEV)
    ts = gold["timesteps"].to(DEV)
    d = dict(x=x, timesteps=ts, context=ctx, grounding_input=grounding, inpainting_extra_input=None)
    e_c = model(d).clone()
    e_u = model(dict(x=x, timesteps=ts, context=uc, inpainting_extra_input=None)).clone()
    c2, u2 = model.forward_cfg(d, uc)
    for got, ref, what in ((e_c, gold["eps_cond"], "forward cond"), (e_u, gold["eps_null"], "forward null"),
                           (c2, gold["eps_cond"], "forward_cfg cond"), (u2, gold["eps_null"], "forward_cfg uncond")):
        r, m = assert_close(got, ref, rel=2.5e-2, max_rel=9e-2, what=f"{name} {what}")
        print(f"{name} {what} t={gold['timesteps'].tolist()}: rel-L2 {r:.3e} max-rel {m:.3e}")


def test_float_integer_timesteps_equal_int64():
    gold = torch.load(os.path.join(GOLD, "karras_unet_tiny.pt"))
    cfg, model, inp, grounding = _model_case(gold)
    x, ctx, uc = inp["x"].to(DEV), inp["context"].to(DEV), inp["uc"].to(DEV)
    ti = torch.tensor([999, 500, 12, 0], device=DEV)
    outs = []
    for ts in (ti, ti.float(), ti.double()):
        d = dict(x=x, timesteps=ts, context=ctx, grounding_input=grounding, inpainting_extra_input=None)
        outs.append([model(d).clone()] + [e.clone() for e in model.forward_cfg(d, uc)])
    for o in outs[1:]:
        assert all(torch.equal(p, q) for p, q in zip(outs[0], o))


# ---- exported plans ---------------------------------------------------------------------------------------------------------
def test_fractional_t_plan_replays_python_engine(tmp_path):
    """An exported fractional_t plan (fp32 in:t): its static and per-step parts replay model.forward_cfg bit for bit; its per-step
    part captured in a CUDA graph and replayed after new in:x / fp32 in:t gives the Python engine's eps for them."""
    c = PlanCase("tiny", 2, 6, tmp_path)
    c.plan.close()
    c.path = os.path.join(str(tmp_path), "tiny_fractional_t.glgplan")
    export_plan(c.eng, 2 * c.B, c.batch["boxes"].shape[1], c.ctx.shape[1], c.path, fractional_t=True)
    c.ts = torch.tensor([500.37, 12.25], device=DEV)
    c.load()                                                      # glg_engine_load accepts it
    _, n = c.plan.buffer("in:t")
    assert n == 2 * c.B * 4
    c.set_scale(1.0)
    want = c.python(c.x, c.ts)
    c.run(static_part=True)
    c.run(static_part=False)
    eager = c.out()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        c.run(static_part=False)
    x2 = torch.randn(tuple(c.x.shape), generator=torch.Generator().manual_seed(11)).to(DEV)
    t2 = torch.tensor([999.0, 0.5], device=DEV)
    want2 = c.python(x2, t2)
    c.write_step(x2, t2)
    graph.replay()
    replay2 = c.out()
    torch.cuda.synchronize()
    assert torch.equal(eager, want), f"eager: max diff {(eager - want).abs().max().item():.3e}"
    assert not torch.equal(want2, want)
    assert torch.equal(replay2, want2), f"replay with new inputs: max diff {(replay2 - want2).abs().max().item():.3e}"
    del graph
    c.plan.close()


# ---- the loops --------------------------------------------------------------------------------------------------------------
class cpu_rng_noise:
    """The fixtures' blend and step noise come from the CPU generator: draw the same noise in the same order."""

    def __enter__(self):
        self.orig = torch.randn_like
        torch.randn_like = lambda x, **kw: torch.randn(x.shape, dtype=x.dtype).to(x.device)
        return self

    def __exit__(self, *a):
        torch.randn_like = self.orig


def _fixture_cfg(name):
    return SAMPLING_GATED_CA if name == "sampling_gated_ca" else NAMED_CONFIGS[name]


def _sample(gold, grid="karras"):
    from ldm.models.diffusion.ldm import LatentDiffusion
    from oracle import img2img_oracle as IO
    cfg, model = build_model(_fixture_cfg(gold["config"]), DEV)
    inp = synth.make_inputs(cfg, gold["B"], gold["max_objs"], seed=2)
    dinp = to_device({k: v for k, v in inp.items() if k in ("x", "context", "uc", "z0")}, DEV)
    input, mask, x0 = sampler_inputs(cfg, model, dinp, to_device(inp["batch"], DEV))
    diffusion = LatentDiffusion(linear_start=0.00085, linear_end=0.012, timesteps=1000).to(DEV)
    kw = dict(alpha_generator_func=partial(alpha_generator, type=gold["alpha_type"]), set_alpha_scale=set_alpha_scale,
              order=gold["order"], grid=grid)
    shape = tuple(dinp["x"].shape)
    call = {}
    if gold["strength"] < 1.0:
        init, noise = IO.init_and_noise(shape, gold["init_seed"])
        call = dict(init_latent=init.to(DEV), strength=gold["strength"], noise=noise.to(DEV))
    if gold["sampler"] == "unipc":
        sampler = UP.UniPCSampler(diffusion, model, **kw)
    else:
        sampler = DS.DPMSolverSampler(diffusion, model, eta=gold["eta"], **kw)
    calls = []
    orig = model.forward_cfg
    model.forward_cfg = lambda *a, **k: calls.append(1) or orig(*a, **k)
    cwd = os.getcwd()
    os.chdir(GOLD)                  # SD_input_conv_weight_bias.pth is read CWD-relative, like the reference
    try:
        torch.manual_seed(gold["noise_seed"])
        with cpu_rng_noise():
            lat = sampler.sample(S=gold["S"], shape=shape, input=input, uc=dinp["uc"], guidance_scale=gold["guidance"], mask=mask, x0=x0,
                                 **call)
    finally:
        os.chdir(cwd)
        del model.forward_cfg
    return cfg, model, lat, len(calls)


KARRAS_FIXTURES = ["karras_dpm2m_tiny.pt", "karras_dpm3m_tiny.pt", "karras_unipc2_tiny.pt", "karras_dpm2msde_tiny.pt",
                   "karras_dpm2m_tiny_inpaint.pt", "karras_dpm2m_sampling_gated_ca.pt", "karras_dpm2m_img2img_tiny.pt",
                   "karras_dpm2m_sd14_box_text.pt"]


@pytest.mark.parametrize("gold_file", KARRAS_FIXTURES)
def test_loop_matches_fixture(gold_file):
    gold = torch.load(os.path.join(GOLD, gold_file))
    cfg, model, lat, passes = _sample(gold)
    n = min(gold["S"], int(gold["strength"] * gold["S"]))
    assert passes == n
    if gold["alpha_type"][0] < 1 and not cfg.inpaint_mode:
        assert model.first_conv_type == "SD"
    assert any(k[-1] == "f32_t" for k in model.engine().plans)
    r, m = assert_close(lat, gold["latent"], rel=6e-2, max_rel=0.1, what=f"{gold_file} latent")
    print(f"{gold_file}: {gold['sampler']}-{gold['order']} eta={gold['eta']} S={gold['S']} strength={gold['strength']}: latent "
          f"rel-L2 {r:.3e} max-rel {m:.3e}")


def test_ddim_grid_builds_no_fp32_plan():
    """The integer-grid samplers never build (or allocate) the fp32-timestep plan."""
    gold = torch.load(os.path.join(GOLD, "karras_dpm2m_tiny.pt"))
    _, model, lat, passes = _sample(gold, grid="ddim")
    assert passes == len(SO.ddim_timesteps(gold["S"]))
    assert model.engine().plans and not any(k[-1] == "f32_t" for k in model.engine().plans)
    assert torch.isfinite(lat).all()
