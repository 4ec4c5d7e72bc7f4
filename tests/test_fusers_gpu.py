"""GPU: UNets built with the gatedCA and gatedSA2 fusers on the sm_90a kernels.

glg_grid_resample_gate against float64 within the bound of tests/fuser_checks.py (up, identity and down resampling, strided rows,
guard bands), whole forwards against the reference fixtures of oracle/gen_golden_fusers.py, the scale = 0 invariant, exported
plans replayed through glg_engine_*, and a float64 census of every kernel call of the SD-1.4-sized models."""
import os
from dataclasses import replace

import pytest
import torch

from conftest import GOLD, assert_close
from fuser_checks import resample_gate_check, stats_check
from gligen_b200 import synth
from gligen_b200.spec import NAMED_CONFIGS, TINY, synthetic_state_dict

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
SENTINEL = -12345.0


@pytest.fixture(scope="module")
def ops():
    from gligen_b200.ops import CudaOps
    return CudaOps(DEV)


def _run_kernel(ops, B, g, n, C, gate, ldx_pad=0, seed=0):
    """x rows inside a guarded, optionally strided buffer; stats_out inside a guarded one.  Returns (out rows, x0, grid, stats)."""
    gen = torch.Generator().manual_seed(seed)
    T = n * n
    grid = torch.randn(B, g * g, C, generator=gen).to(DEV)
    ld = C + ldx_pad
    buf = torch.full((B * T + 2, ld), SENTINEL, dtype=torch.bfloat16, device=DEV)
    x0 = (0.5 * torch.randn(B * T, C, generator=gen)).to(torch.bfloat16).to(DEV)
    buf[1:-1, :C] = x0
    x = buf[1:-1, :C].view(B, T, C)
    sbuf = torch.full((C // 32 + 1, B * T + 2, 2), SENTINEL, device=DEV)
    stats = sbuf[: C // 32, 1:-1]
    gt = torch.tensor([gate], device=DEV)
    ops.grid_resample_gate(grid, x, gt, stats, g, n)
    torch.cuda.synchronize()
    # guard bands: rows before / after, the padding columns, the spare slot and rows of the statistics
    assert (buf[0] == SENTINEL).all() and (buf[-1] == SENTINEL).all() and (buf[:, C:] == SENTINEL).all()
    assert (sbuf[-1] == SENTINEL).all() and (sbuf[:, 0] == SENTINEL).all() and (sbuf[:, -1] == SENTINEL).all()
    return x.reshape(B * T, C).clone(), x0, grid, stats.clone()


def _check(out, x0, grid, stats, B, g, n, C, gate):
    T = n * n
    for b in range(B):                                  # one image at a time keeps the float64 gather small
        rows = slice(b * T, (b + 1) * T)
        rep = resample_gate_check(out[rows].view(1, T, C), x0[rows].view(1, T, C), grid[b:b + 1], gate, g, n,
                                  what=f"grid_resample_gate B={B} g={g} n={n} C={C} gate={gate} b={b}")
        assert rep.ok, str(rep)
    rep = stats_check(stats, out)
    assert rep.ok, str(rep)


@pytest.mark.parametrize("g", [1, 2, 4, 8])
@pytest.mark.parametrize("n", [1, 2, 4, 8, 16, 32, 64, 128])
def test_grid_resample_gate_sizes(ops, g, n):
    """Every grid side against every visual side (upsample, identity, downsample), C = 64, two images."""
    out, x0, grid, stats = _run_kernel(ops, 2, g, n, 64, 0.8, seed=g * 1000 + n)
    _check(out, x0, grid, stats, 2, g, n, 64, 0.8)


@pytest.mark.parametrize("B,g,n,C", [(8, 8, 64, 320), (8, 8, 32, 640), (8, 8, 16, 1280), (8, 8, 8, 1280), (2, 4, 64, 320), (3, 4, 2, 640),
                                     (1, 8, 128, 64)])
@pytest.mark.parametrize("gate", [0.0, -0.6, 7.5])
def test_grid_resample_gate_model_shapes(ops, B, g, n, C, gate):
    """The SD-1.4 gatedSA2 shapes (8 x 8 tokens onto the 64 / 32 / 16 / 8 levels at 8 rows), the 16-token tiny model, gates 0,
    negative and large."""
    out, x0, grid, stats = _run_kernel(ops, B, g, n, C, gate, seed=B + g + n + C)
    if gate == 0.0:
        assert torch.equal(out, x0)
    _check(out, x0, grid, stats, B, g, n, C, gate)


def test_grid_resample_gate_strided_rows(ops):
    """x rows with a leading dimension larger than C (a channel slice of a wider buffer)."""
    out, x0, grid, stats = _run_kernel(ops, 2, 4, 16, 320, -1.7, ldx_pad=64, seed=5)
    _check(out, x0, grid, stats, 2, 4, 16, 320, -1.7)


def test_grid_resample_gate_refuses_bad_arguments(ops):
    from gligen_b200 import lib as L
    x = torch.zeros(16, 64, dtype=torch.bfloat16, device=DEV)
    grid = torch.zeros(1, 4, 64, device=DEV)
    st = torch.zeros(2, 16, 2, device=DEV)
    gate = torch.zeros(1, device=DEV)
    lib = L.load()
    args = [grid.data_ptr(), 4 * 64, x.data_ptr(), 64, gate.data_ptr(), st.data_ptr(), 16, 1, 2, 4, 64, None]
    assert lib.glg_grid_resample_gate(*args) == 0
    torch.cuda.synchronize()
    for i, v in ((0, None), (4, None), (5, None), (10, 48), (3, 32), (6, 8), (8, 0), (9, 0), (8, 20)):
        bad = list(args)
        bad[i] = v
        assert lib.glg_grid_resample_gate(*bad) != 0, (i, v)


# ---- whole forwards against the reference ----------------------------------------------------------------------------------
CASES = [("tiny_gated_ca", None), ("tiny_text_image_gated_ca", None), ("tiny_keypoint_gated_ca", None), ("tiny_hed_gated_sa2", None),
         ("tiny_gated_sa2_text", replace(TINY, fuser_type="gatedSA2")), ("sd14_box_text_gated_ca", None), ("sd14_hed_gated_sa2", None)]


def _model(cfg):
    from gligen_b200.pipeline import build_model
    return build_model(cfg, DEV)[1]


@pytest.mark.parametrize("name,cfg", CASES)
def test_forward_matches_reference(name, cfg):
    """eps of the drop-in UNetModel, single and CFG-batched passes, at fuser scale 1 and 0.5, against the reference."""
    from gligen_b200.pipeline import to_device
    gold = torch.load(os.path.join(GOLD, f"fuser_{name}.pt"))
    cfg = cfg or NAMED_CONFIGS[name]
    inp = synth.make_inputs(cfg, gold["B"], gold["max_objs"], seed=gold["seed"])
    model = _model(cfg)
    ts = gold["timesteps"].to(DEV)
    x, ctx, uc = inp["x"].to(DEV), inp["context"].to(DEV), inp["uc"].to(DEV)
    grounding = model.grounding_tokenizer_input.prepare(to_device(inp["batch"], DEV))
    ge = inp.get("grounding_extra_input")
    ge = None if ge is None else ge.to(DEV)
    for scale, f in gold["forward"].items():
        for fu in model._fusers:
            fu.scale = scale
        d = dict(x=x, timesteps=ts, context=ctx, grounding_input=grounding, grounding_extra_input=ge)
        e_c = model(d).clone()
        e_u = model(dict(x=x, timesteps=ts, context=uc, grounding_extra_input=ge)).clone()
        c2, u2 = model.forward_cfg(d, uc)
        for got, ref, what in ((e_c, f["eps_cond"], "cond"), (e_u, f["eps_null"], "null"), (c2, f["eps_cond"], "cfg cond"), (u2, f["eps_null"], "cfg null")):
            assert_close(got, ref, rel=2.5e-2, max_rel=0.09, what=f"{name} scale={scale} {what}")


@pytest.mark.parametrize("name", ["tiny_gated_ca", "tiny_hed_gated_sa2", "tiny_keypoint_gated_ca"])
def test_scale_zero_equals_gated_sa(name):
    """At scale 0 the fuser is skipped: a gatedCA / gatedSA2 model gives bit for bit the eps of the gatedSA model with the same
    non-fuser weights."""
    from gligen_b200.pipeline import to_device
    cfg = NAMED_CONFIGS[name]
    sa = replace(cfg, fuser_type="gatedSA")
    sd_sa = synthetic_state_dict(sa, 0)
    sd = {k: (v if ".fuser." in k else sd_sa[k]) for k, v in synthetic_state_dict(cfg, 0).items()}
    inp = synth.make_inputs(cfg, 2, 6, seed=3)
    outs = []
    for c, w in ((cfg, sd), (sa, sd_sa)):
        from gligen_b200.pipeline import build_model
        _, m = build_model(c, DEV, load_weights=False)
        m.load_state_dict(w)
        for fu in m._fusers:
            fu.scale = 0.0
        gr = m.grounding_tokenizer_input.prepare(to_device(inp["batch"], DEV))
        ge = inp.get("grounding_extra_input")
        e_c, e_u = m.forward_cfg(dict(x=inp["x"].to(DEV), timesteps=torch.tensor([981, 21], device=DEV), context=inp["context"].to(DEV),
                                      grounding_input=gr, grounding_extra_input=None if ge is None else ge.to(DEV)), inp["uc"].to(DEV))
        outs.append(torch.cat([e_c, e_u]).clone())
    assert torch.equal(outs[0], outs[1])


@pytest.mark.parametrize("name,max_objs,scales", [("tiny_gated_ca", 6, (1.0, 0.0)), ("tiny_hed_gated_sa2", 0, (1.0,))])
def test_exported_plan_matches_python_engine(name, max_objs, scales, tmp_path):
    """gatedCA and gatedSA2 plans replayed by the library alone (glg_engine_*), bit for bit (every fuser variant, its other scales
    and SD-sized models: tests/test_native_engine_variants_gpu.py)."""
    from native_plan import _case
    info = _case(name, 2, max_objs, tmp_path, scales=scales)
    assert info["ops"] > 300


# ---- scheduled sampling against the reference sampler ----------------------------------------------------------------------
@pytest.mark.parametrize("name", ["sampling_gated_ca", "sampling_hed_gated_sa2"])
def test_plms_scheduled_sampling_matches_reference(name):
    """PLMS S=4, alpha_type [0.3, 0, 0.7] (alphas [1, 0, 0, 0]), CFG 7.5, through this repo's PLMSSampler with the reference's
    set_alpha_scale, against the REFERENCE sampler's latent.  From step 2 on the gatedCA fusers are at scale 0 (skipped) while the
    gatedSA2 fusers stay at scale 1, and restore_first_conv_from_SD swaps in SD's first conv (the hed model: the 4-channel conv,
    engine-side zero weights on the downsampler planes)."""
    from functools import partial
    from gligen_b200.pipeline import alpha_generator, build_model, sampler_inputs, set_alpha_scale, to_device
    from gligen_b200.spec import SAMPLING_GATED_CA, SAMPLING_HED_GATED_SA2
    from ldm.models.diffusion.ldm import LatentDiffusion
    from ldm.models.diffusion.plms import PLMSSampler
    gp = torch.load(os.path.join(GOLD, f"fuser_plms_{name}.pt"))
    cfg = {"sampling_gated_ca": SAMPLING_GATED_CA, "sampling_hed_gated_sa2": SAMPLING_HED_GATED_SA2}[name]
    cfg, model = build_model(cfg, DEV)
    inp = synth.make_inputs(cfg, gp["B"], gp["max_objs"], seed=gp["seed"])
    dinp = to_device({k: v for k, v in inp.items() if k in ("x", "context", "uc")}, DEV)
    input, _, _ = sampler_inputs(cfg, model, dinp, to_device(inp["batch"], DEV))
    diffusion = LatentDiffusion(linear_start=0.00085, linear_end=0.012, timesteps=1000).to(DEV)
    sampler = PLMSSampler(diffusion, model, alpha_generator_func=partial(alpha_generator, type=gp["alpha_type"]), set_alpha_scale=set_alpha_scale)
    cwd = os.getcwd()
    os.chdir(GOLD)                  # SD_input_conv_weight_bias.pth is read CWD-relative, like the reference
    try:
        torch.manual_seed(gp["noise_seed"])
        shape = (gp["B"], cfg.in_channels, cfg.image_size, cfg.image_size)
        lat = sampler.sample(S=gp["S"], shape=shape, input=input, uc=dinp["uc"], guidance_scale=gp["guidance"])
    finally:
        os.chdir(cwd)
    assert model.first_conv_type == "SD"
    assert sorted({f.scale for f in model._fusers}) == gp["final_fuser_scales"]
    r = assert_close(lat, gp["latent"], rel=6e-2, max_rel=0.1, what=f"{name} PLMS S=4 latent")
    print(f"{name} PLMS S=4 alpha={gp['alpha_type']}: latent rel-L2 {r[0]:.3e} max-rel {r[1]:.3e}")


# ---- float64 census ----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", ["sd14_box_text_gated_ca", "sd14_hed_gated_sa2", "tiny_gated_ca", "tiny_text_image_gated_ca",
                                  "tiny_keypoint_gated_ca", "tiny_hed_gated_sa2"])
def test_census_fusers(name):
    """Every kernel call of one CFG forward (B = 2, 4 UNet rows) at the native size against float64, with the census checks of
    tests/test_op_census_gpu.py, glg_grid_resample_gate included."""
    from gligen_b200.engine import Engine
    from gligen_b200.ops import CudaOps
    from gligen_b200.spec import SPATIAL_MAP_KEY
    from test_op_census_gpu import CheckedOps, _summary

    cfg = NAMED_CONFIGS[name]
    ops = CheckedOps(CudaOps(DEV))
    eng = Engine(cfg, ops, use_graphs=False)
    eng.load_state_dict(synthetic_state_dict(cfg, 0))
    inp = synth.make_inputs(cfg, 2, seed=2)
    x, ctx, uc = (inp[k].to(DEV) for k in ("x", "context", "uc"))
    gr = {k: v.to(DEV) for k, v in inp["grounding_input"].items()}
    gextra = inp["batch"][SPATIAL_MAP_KEY[cfg.tokenizer]].to(DEV) if cfg.spatial else None
    eng.forward_cfg(x, torch.tensor([981, 501], device=DEV), ctx, uc, gr, None, gextra)
    torch.cuda.synchronize()
    if cfg.fuser_type == "gatedSA2":
        assert len(ops.records["grid_resample_gate"]) == len(eng.st_prefixes)
    _summary(f"{name} B=2 cfg", ops)
