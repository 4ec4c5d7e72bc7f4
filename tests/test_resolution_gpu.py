"""Any resolution and aspect ratio on the GPU.

The 3x3 convolution of glg_gemm (im2col-mode TMA, 128 consecutive output pixels per tile across row and image
boundaries) at widths that neither divide 128 nor are multiples of it, images smaller than a tile and tiles that
straddle images, under every schedule the library's test hooks can force, against float64 within the GEMM / conv bound
of tests/bounds.py; outputs written into a channel slice of a wider buffer leave every other column and every row past M
untouched."""
from functools import partial

import pytest
import torch

import bounds

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
BF = torch.bfloat16


@pytest.fixture(scope="module")
def ops():
    from gligen_b200.ops import CudaOps
    return CudaOps(DEV)


def gen(seed):
    return torch.Generator(device="cpu").manual_seed(seed)


class schedule:
    """Force one GEMM schedule through the library's test hooks for a block and always restore the defaults."""

    def __init__(self, ops, bn=0, pp=0, cta2=0, splitk=0):
        self.ops, self.v = ops, (bn, pp, cta2, splitk)

    def __enter__(self):
        L = self.ops.lib
        bn, pp, cta2, splitk = self.v
        L.glg_debug_force_bn(bn); L.glg_debug_gemm_pp(pp); L.glg_debug_gemm_cta2(cta2); L.glg_debug_splitk(splitk)

    def __exit__(self, *a):
        L = self.ops.lib
        L.glg_debug_force_bn(0); L.glg_debug_gemm_pp(0); L.glg_debug_gemm_cta2(0); L.glg_debug_splitk(0)


# name -> (force_bn, ping-pong mode, CTA-pair mode, split-K mode); "auto" is the heuristic
SCHEDULES = {
    "auto": (0, 0, 0, 0), "bn64": (64, 1, 1, 1), "bn64_pp": (64, 2, 1, 1), "bn128": (128, 1, 1, 1), "bn128_pp": (128, 2, 1, 1),
    "bn160": (160, 1, 1, 1), "bn256": (256, 1, 1, 1), "pair128": (128, 1, 2, 1), "pair256": (256, 1, 2, 1), "splitk": (0, 1, 1, 2),
}

WIDTHS = [3, 6, 7, 10, 12, 20, 24, 40, 48, 72, 80, 96, 160, 192, 320]


def conv_shapes():
    """(B, H, W, C) per width: one image smaller than a tile where W allows, one that makes tiles straddle rows and images,
    B cycling through 1..3 and C through 128 / 320 / 640 / 1280 (the largest channel counts on the smaller images)."""
    out = []
    cs = [128, 320, 640, 1280]
    for i, W in enumerate(WIDTHS):
        hs = sorted({max(1, 100 // W), 3 if W >= 160 else max(2, 700 // W)})
        for j, H in enumerate(hs):
            B = 1 + (i + j) % 3
            C = cs[(i + 2 * j) % 4]
            if B * H * W * C > 3_000_000:
                C = 128 if C != 320 else 320
            out.append((B, H, W, C))
    return out


CONV_SHAPES = conv_shapes()


@pytest.mark.parametrize("B,H,W,C", CONV_SHAPES, ids=[f"B{b}_{h}x{w}_C{c}" for b, h, w, c in CONV_SHAPES])
def test_conv3x3_any_width_bounded(ops, B, H, W, C):
    g = gen(B * 1000 + H * 10 + W + C)
    a = torch.randn(B, H * W, C, generator=g).to(DEV, BF)
    w = (torch.randn(9 * C, C, generator=g) * (9 * C) ** -0.5).to(DEV, BF)
    bias = torch.randn(C, generator=g).to(DEV)
    rowbias = torch.randn(B, C, generator=g).to(DEV)
    res = torch.randn(B, H * W, C, generator=g).to(DEV, BF)
    bad = []
    for name, (bn, pp, cta2, splitk) in SCHEDULES.items():
        if bn and C % bn:
            continue
        out = torch.zeros(B, H * W, C, device=DEV, dtype=BF)
        with schedule(ops, bn, pp, cta2, splitk):
            ops.gemm(a, w, out, bias=bias, rowbias=rowbias, rows_per_batch=H * W, residual=res, conv=(B, H, W))
            torch.cuda.synchronize()
        rep = bounds.gemm_check(out, a, w, bias=bias, rowbias=rowbias, rows_per_batch=H * W, residual=res, conv=(B, H, W),
                                splits=8, what=f"conv B{B} {H}x{W} C{C} {name}")
        if not rep.ok:
            bad.append(str(rep))
    assert not bad, "\n".join(bad)


@pytest.mark.parametrize("B,H,W,Cin,Cout,off", [(2, 12, 20, 320, 320, 640), (3, 5, 7, 128, 256, 64), (1, 24, 72, 640, 320, 320),
                                                 (2, 3, 96, 1280, 640, 1280)])
@pytest.mark.parametrize("sched", ["auto", "bn64_pp", "pair128", "splitk"])
def test_conv3x3_into_concat_slice(ops, B, H, W, Cin, Cout, off, sched):
    """Output into columns [off, off + Cout) of a [M + 64, Ctot] buffer (ldc > N), as the UNet writes skip connections into
    its concat buffers: the other columns and the 64 rows past M keep their sentinel."""
    bn, pp, cta2, splitk = SCHEDULES[sched]
    if bn and Cout % bn:
        pytest.skip("tile width does not divide N")
    g = gen(B + H + W + Cin + off)
    M = B * H * W
    ctot = off + Cout + 192
    a = torch.randn(B, H * W, Cin, generator=g).to(DEV, BF)
    w = (torch.randn(9 * Cout, Cin, generator=g) * (9 * Cin) ** -0.5).to(DEV, BF)
    bias = torch.randn(Cout, generator=g).to(DEV)
    sentinel = -1234.0
    big = torch.full((M + 64, ctot), sentinel, device=DEV, dtype=BF)
    out = big[:M].view(B, H * W, ctot)[:, :, off:off + Cout]
    with schedule(ops, bn, pp, cta2, splitk):
        ops.gemm(a, w, out, bias=bias, conv=(B, H, W))
        torch.cuda.synchronize()
    assert (big[M:] == sentinel).all(), "wrote rows past M"
    assert (big[:M, :off] == sentinel).all() and (big[:M, off + Cout:] == sentinel).all(), "wrote outside the channel slice"
    rep = bounds.gemm_check(out.contiguous(), a, w, bias=bias, conv=(B, H, W), splits=8, what=f"concat-slice conv {sched}")
    assert rep.ok, str(rep)


def test_conv3x3_refusals(ops):
    """Cin that is not a multiple of 64 and leading dimensions that are not multiples of 8 stay refused."""
    from gligen_b200.lib import GligenLibraryError
    a = torch.zeros(1, 6 * 10, 96, device=DEV, dtype=BF)
    with pytest.raises(GligenLibraryError, match="K must be"):
        ops.gemm(a, torch.zeros(9 * 64, 96, device=DEV, dtype=BF), torch.zeros(1, 60, 64, device=DEV, dtype=BF), conv=(1, 6, 10))
    big = torch.zeros(60, 132, device=DEV, dtype=BF)
    with pytest.raises(GligenLibraryError, match="leading dims"):
        ops.gemm(big[:, :64], torch.zeros(9 * 64, 64, device=DEV, dtype=BF), torch.zeros(1, 60, 64, device=DEV, dtype=BF), conv=(1, 6, 10))


# ---- whole forwards at non-square latents ----------------------------------------------------------------------------
# per-forward tolerance of tests/test_batch_gpu.py: bf16 against fp32, amplified through ~70 layers of a random UNet
REL, MAX_REL = 2.5e-2, 9e-2


def _latent(cfg, B, H, W, seed):
    g = torch.Generator().manual_seed(seed)
    return torch.randn(B, cfg.in_channels, H, W, generator=g), torch.randn(B, cfg.in_channels, H, W, generator=g) * 0.9


@pytest.mark.parametrize("name,H,W", [("sd14_box_text", 64, 96), ("sd14_box_text", 96, 64)])
def test_census_sd14_non_square(name, H, W):
    """Every GEMM / conv / attention / GroupNorm call of a 512 x 768 (768 x 512) box+text forward within its float64 bound."""
    from test_op_census_gpu import CheckedOps, _summary
    from gligen_b200 import synth
    from gligen_b200.engine import Engine
    from gligen_b200.ops import CudaOps
    from gligen_b200.spec import NAMED_CONFIGS, synthetic_state_dict
    cfg = NAMED_CONFIGS[name]
    ops = CheckedOps(CudaOps(DEV))
    eng = Engine(cfg, ops, use_graphs=False)
    eng.load_state_dict(synthetic_state_dict(cfg, 0))
    inp = synth.make_inputs(cfg, 1, 30, seed=2)
    x, _ = _latent(cfg, 1, H, W, seed=H + W)
    gr = {k: v.to(DEV) for k, v in inp["grounding_input"].items()}
    e = eng.forward(x.to(DEV), torch.tensor([501], device=DEV), inp["context"].to(DEV), gr)
    torch.cuda.synchronize()
    assert e.shape == (1, cfg.out_channels, H, W) and torch.isfinite(e).all()
    _summary(f"{name} {H}x{W}", ops)


def _fixture(name, H, W):
    """(cfg, fixture, synth inputs, extra input) of the reference fixture tests/golden/res_<name>_<H>x<W>.pt."""
    import os
    from conftest import GOLD
    from gligen_b200 import synth
    from gligen_b200.spec import NAMED_CONFIGS
    cfg = NAMED_CONFIGS[name]
    gold = torch.load(os.path.join(GOLD, f"res_{name}_{H}x{W}.pt"))
    inp = synth.make_inputs(cfg, gold["B"], gold["max_objs"], seed=2)
    extra = None if gold["mask"] is None else torch.cat([gold["z0"] * gold["mask"], gold["mask"]], 1)
    return cfg, gold, inp, extra


@pytest.mark.parametrize("name,H,W", [(n, h, w) for n in ("tiny", "tiny_text_image", "tiny_keypoint", "tiny_inpaint")
                                      for h, w in ((16, 24), (24, 16))] + [("sd14_box_text", 64, 96), ("sd14_box_text", 96, 64)])
def test_forward_non_square_matches_reference(name, H, W):
    """eps of the drop-in UNetModel (single and CFG-batched passes) against the reference at the same non-square latent."""
    from conftest import assert_close
    from gligen_b200.pipeline import build_model, to_device
    cfg, gold, inp, extra = _fixture(name, H, W)
    _, model = build_model(name, DEV)
    grounding = model.grounding_tokenizer_input.prepare(to_device(inp["batch"], DEV))
    x, ts, ctx, uc = gold["x"].to(DEV), gold["timesteps"].to(DEV), inp["context"].to(DEV), inp["uc"].to(DEV)
    extra = None if extra is None else extra.to(DEV)
    e_c = model(dict(x=x, timesteps=ts, context=ctx, grounding_input=grounding, inpainting_extra_input=extra)).clone()
    c2, u2 = model.forward_cfg(dict(x=x, timesteps=ts, context=ctx, grounding_input=grounding, inpainting_extra_input=extra), uc)
    torch.cuda.synchronize()
    for nm, got, ref in (("cond", e_c, gold["eps_cond"]), ("cfg.cond", c2, gold["eps_cond"]), ("cfg.null", u2, gold["eps_null"])):
        r, m = assert_close(got.cpu(), ref, rel=REL, max_rel=MAX_REL, what=f"{name} {H}x{W} {nm}")
        print(f"{name} {H}x{W} {nm}: rel_l2={r:.3e} max_rel={m:.3e}")


def test_plms_loop_sd14_64x96_matches_reference():
    """PLMSSampler.sample(S=4, shape=(1, 4, 64, 96)) through the drop-in UNetModel: CFG 7.5, scheduled sampling [0.5, 0, 0.5]
    with the SD first-conv swap, against the reference loop's final latent (short-loop tolerance of tests/test_engine_gpu.py)."""
    import os
    from conftest import GOLD, assert_close
    from ldm.models.diffusion.ldm import LatentDiffusion
    from ldm.models.diffusion.plms import PLMSSampler
    from gligen_b200.pipeline import alpha_generator, build_model, set_alpha_scale, to_device
    cfg, gold, inp, _ = _fixture("sd14_box_text", 64, 96)
    g = gold["plms"]
    _, model = build_model("sd14_box_text", DEV)
    grounding = model.grounding_tokenizer_input.prepare(to_device(inp["batch"], DEV))
    diffusion = LatentDiffusion(linear_start=0.00085, linear_end=0.012, timesteps=1000).to(DEV)
    sampler = PLMSSampler(diffusion, model, alpha_generator_func=partial(alpha_generator, type=g["alpha_type"]), set_alpha_scale=set_alpha_scale)
    input = dict(x=gold["x"].to(DEV), timesteps=None, context=inp["context"].to(DEV), grounding_input=grounding,
                 inpainting_extra_input=None, grounding_extra_input=None)
    cwd = os.getcwd()
    os.chdir(GOLD)                        # restore_first_conv_from_SD reads a CWD-relative file, like the reference
    try:
        torch.manual_seed(1234)
        lat = sampler.sample(S=g["S"], shape=tuple(gold["x"].shape), input=input, uc=inp["uc"].to(DEV), guidance_scale=g["guidance"])
    finally:
        os.chdir(cwd)
    r, m = assert_close(lat.cpu(), g["latent"], rel=6e-2, max_rel=0.1, what="sd14_box_text 64x96 plms S=4 latent")
    print(f"sd14_box_text 64x96 plms S=4: latent rel_l2={r:.3e} max_rel={m:.3e}")


def test_batch_rows_equal_single_sample_non_square():
    """Rows of a B = 3 pass at 64 x 96 against the same samples run alone (B = 1)."""
    from conftest import assert_close
    from gligen_b200 import synth
    from gligen_b200.pipeline import build_model, to_device
    cfg, model = build_model("sd14_box_text", DEV)
    inp = synth.make_inputs(cfg, 3, 30, seed=7)
    x, _ = _latent(cfg, 3, 64, 96, seed=3)
    x, ctx, uc = x.to(DEV), inp["context"].to(DEV), inp["uc"].to(DEV)
    batch = to_device(inp["batch"], DEV)
    gr = model.grounding_tokenizer_input.prepare(batch)
    ts = torch.tensor([981, 501, 21], device=DEV)
    e_c, e_u = (t.clone() for t in model.forward_cfg(dict(x=x, timesteps=ts, context=ctx, grounding_input=gr), uc))
    for i in range(3):
        gi = {k: v[i:i + 1] for k, v in gr.items()}
        s_c, s_u = model.forward_cfg(dict(x=x[i:i + 1], timesteps=ts[i:i + 1], context=ctx[i:i + 1], grounding_input=gi), uc[i:i + 1])
        assert_close(e_c[i:i + 1], s_c, rel=REL, max_rel=MAX_REL, what=f"row {i} cond")
        assert_close(e_u[i:i + 1], s_u, rel=REL, max_rel=MAX_REL, what=f"row {i} uncond")


def test_vae_sd14_non_square_census():
    """sd14_vae decode of a 64 x 96 latent (a 512 x 768 image) and encode of that image: every call within its float64 bound."""
    from test_op_census_gpu import CheckedOps, _summary
    from gligen_b200.ops import CudaOps
    from gligen_b200.spec import NAMED_VAE_CONFIGS, synthetic_vae_encoder_state_dict, synthetic_vae_state_dict
    from gligen_b200.vae import VAEDecoderEngine, VAEEncoderEngine
    cfg = NAMED_VAE_CONFIGS["sd14_vae"]
    ops = CheckedOps(CudaOps(DEV))
    dec = VAEDecoderEngine(cfg, ops)
    dec.load_state_dict(synthetic_vae_state_dict(cfg, 0))
    g = torch.Generator().manual_seed(4)
    img = dec.decode(torch.randn(1, 4, 64, 96, generator=g).to(DEV))
    assert img.shape == (1, 3, 512, 768)
    enc = VAEEncoderEngine(cfg, ops)
    enc.load_state_dict(synthetic_vae_encoder_state_dict(cfg, 1))
    mom = enc.encode_moments(torch.rand(1, 3, 768, 512, generator=g).to(DEV) * 2 - 1)
    assert mom.shape == (1, 8, 96, 64)
    torch.cuda.synchronize()
    _summary("sd14_vae 64x96 decode + 768x512 encode", ops)


def test_small_vae_non_square_matches_reference():
    """small_vae decode of a 32 x 48 latent and encode of a 192 x 128 image against the reference fixture."""
    import os
    from conftest import GOLD, assert_close
    from gligen_b200.ops import CudaOps
    from gligen_b200.spec import NAMED_VAE_CONFIGS, synthetic_vae_encoder_state_dict, synthetic_vae_state_dict
    from gligen_b200.vae import VAEDecoderEngine, VAEEncoderEngine
    cfg = NAMED_VAE_CONFIGS["small_vae"]
    gold = torch.load(os.path.join(GOLD, "res_small_vae_32x48.pt"))
    dec = VAEDecoderEngine(cfg, CudaOps(DEV))
    dec.load_state_dict(synthetic_vae_state_dict(cfg, 0))
    assert_close(dec.decode(gold["z"].to(DEV)).cpu(), gold["image"], rel=1e-2, max_rel=0.10, what="small_vae decode 32x48")
    enc = VAEEncoderEngine(cfg, CudaOps(DEV))
    enc.load_state_dict(synthetic_vae_encoder_state_dict(cfg, 1))
    assert_close(enc.encode_moments(gold["x"].to(DEV)).cpu(), gold["moments"], rel=1e-2, max_rel=0.10, what="small_vae encode 192x128")


def test_vae_sd14_non_square_matches_oracle():
    """sd14_vae decode of a 64 x 96 latent (a 512 x 768 image, rel-L2 <= 1e-2) and encode of a 768 x 512 image, end to end
    against oracle/vae_oracle.py on the CPU in fp32 (pinned to the reference at non-square sizes by the small_vae fixture)."""
    from conftest import assert_close
    from gligen_b200.ops import CudaOps
    from gligen_b200.spec import NAMED_VAE_CONFIGS, synthetic_vae_encoder_state_dict, synthetic_vae_state_dict
    from gligen_b200.vae import VAEDecoderEngine, VAEEncoderEngine
    from oracle import vae_oracle as VO
    cfg = NAMED_VAE_CONFIGS["sd14_vae"]
    g = torch.Generator().manual_seed(4)
    z = torch.randn(1, 4, 64, 96, generator=g) * cfg.scale_factor * 4.0
    sd = synthetic_vae_state_dict(cfg, 0)
    dec = VAEDecoderEngine(cfg, CudaOps(DEV))
    dec.load_state_dict(sd)
    img = dec.decode(z.to(DEV)).cpu()
    with torch.no_grad():
        ref = VO.vae_decode(cfg, sd, z)
    assert img.shape == ref.shape == (1, 3, 512, 768)
    r, m = assert_close(img, ref, rel=1e-2, max_rel=0.10, what="sd14_vae decode 512x768")
    print(f"sd14_vae decode 512x768: rel_l2={r:.3e} max_rel={m:.3e}")
    x = torch.rand(1, 3, 768, 512, generator=g) * 2 - 1
    sde = synthetic_vae_encoder_state_dict(cfg, 1)
    enc = VAEEncoderEngine(cfg, CudaOps(DEV))
    enc.load_state_dict(sde)
    mom = enc.encode_moments(x.to(DEV)).cpu()
    with torch.no_grad():
        refm = VO.vae_encode_moments(cfg, sde, x)
    assert mom.shape == refm.shape == (1, 8, 96, 64)
    # a white-noise image in [-1, 1]: measured rel-L2 1.1e-2 on an H100; the full-size VAE tolerance of tests/test_vae_gpu.py
    r, m = assert_close(mom, refm, rel=3e-2, max_rel=0.10, what="sd14_vae encode 768x512")
    print(f"sd14_vae encode 768x512: rel_l2={r:.3e} max_rel={m:.3e}")


def test_exported_non_square_plan_replays_bit_for_bit(tmp_path):
    import os
    from gligen_b200 import synth
    from gligen_b200.export import NativePlan, export_plan
    from gligen_b200.pipeline import build_model, to_device
    cfg, model = build_model("tiny", DEV)
    B, H, W = 2, 16, 24
    inp = synth.make_inputs(cfg, B, 6, seed=4)
    x, _ = _latent(cfg, B, H, W, seed=9)
    x, ctx, uc = x.to(DEV), inp["context"].to(DEV), inp["uc"].to(DEV)
    batch = to_device(inp["batch"], DEV)
    grounding = model.grounding_tokenizer_input.prepare(batch)
    ts = torch.tensor([981, 401], device=DEV)
    e_c, e_u = model.forward_cfg(dict(x=x, timesteps=ts, context=ctx, grounding_input=grounding), uc)
    want = torch.cat([e_c, e_u]).clone()
    eng = model.engine()
    path = os.path.join(str(tmp_path), "tiny_16x24.glgplan")
    export_plan(eng, 2 * B, batch["boxes"].shape[1], ctx.shape[1], path, H=H, W=W)
    plan = NativePlan(path)
    z = lambda t: torch.cat([t, torch.zeros_like(t)])
    plan.write("in:x", torch.cat([x, x])); plan.write("in:t", torch.cat([ts, ts])); plan.write("in:context", torch.cat([ctx, uc]))
    plan.write("in:coords", z(batch["boxes"])); plan.write("in:masks", z(batch["masks"]))
    plan.write("in:feat0", z(batch["text_embeddings"])); plan.write("in:fmask0", z(batch["masks"]))
    plan.write("W:gates", eng.W["gates"])
    plan.run(static_part=True, fuser_on=True)
    plan.run(static_part=False, fuser_on=True)
    got = plan.read("out", want.shape)
    torch.cuda.synchronize()
    plan.close()
    assert torch.equal(got, want), f"max diff {(got - want).abs().max().item():.3e}"
