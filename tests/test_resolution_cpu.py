"""Non-square latents on the CPU, against the REFERENCE fixtures tests/golden/res_*.pt (oracle/gen_golden_resolution.py: the
unmodified reference at 16 x 24 / 24 x 16 tiny latents, 64 x 96 / 96 x 64 SD-1.4 latents, PLMS S = 4 loops, a 32 x 48 small_vae
latent): the oracle restatement, the UNet engine's plan and the VAE engines executed with the torch-fp32 checker ops
(tests/ref_ops.py: H != W strides, concat slices, transposed shapes), the drop-in PLMSSampler at 16 x 24; and the sizes the
engines refuse."""
import os
from functools import partial

import pytest
import torch

from conftest import GOLD, rel_l2
from gligen_b200 import synth
from gligen_b200.engine import Engine
from gligen_b200.spec import NAMED_CONFIGS, NAMED_VAE_CONFIGS, synthetic_state_dict, synthetic_vae_encoder_state_dict, synthetic_vae_state_dict
from gligen_b200.vae import VAEDecoderEngine, VAEEncoderEngine
from oracle import unet_oracle as UO
from oracle import vae_oracle as VO
from ref_ops import RefOps
from test_sampler_host_cpu import cpu_backend  # noqa: F401  (fixture: the drop-in samplers on the checker ops)

TINY = [("tiny", 6), ("tiny_text_image", 5), ("tiny_keypoint", 34), ("tiny_inpaint", 6)]
SIZES = [(16, 24), (24, 16)]


def load_case(name, H, W):
    """(cfg, fixture, synth inputs, extra input) of tests/golden/res_<name>_<H>x<W>.pt."""
    cfg = NAMED_CONFIGS[name]
    gold = torch.load(os.path.join(GOLD, f"res_{name}_{H}x{W}.pt"))
    inp = synth.make_inputs(cfg, gold["B"], gold["max_objs"], seed=2)
    extra = None if gold["mask"] is None else torch.cat([gold["z0"] * gold["mask"], gold["mask"]], 1)
    return cfg, gold, inp, extra


def _close(got, ref, tol):
    return (got - ref).abs().max().item() <= tol * max(1.0, ref.abs().max().item())


@pytest.mark.parametrize("name,H,W", [(n, h, w) for n, _ in TINY for h, w in SIZES] + [("sd14_box_text", 64, 96), ("sd14_box_text", 96, 64)])
def test_oracle_matches_reference_fixture(name, H, W):
    cfg, gold, inp, extra = load_case(name, H, W)
    sd = synthetic_state_dict(cfg, 0)
    gr = inp["grounding_input"]
    assert _close(UO.unet_forward(cfg, sd, gold["x"], gold["timesteps"], inp["context"], gr, 1.0, extra), gold["eps_cond"], 2e-5)
    assert _close(UO.unet_forward(cfg, sd, gold["x"], gold["timesteps"], inp["uc"], UO.null_grounding(cfg, gr), 1.0, extra), gold["eps_null"], 2e-5)


@pytest.mark.parametrize("name", [n for n, _ in TINY])
@pytest.mark.parametrize("H,W", SIZES)
def test_engine_plan_non_square_matches_reference(name, H, W):
    cfg, gold, inp, extra = load_case(name, H, W)
    eng = Engine(cfg, RefOps())
    eng.load_state_dict(synthetic_state_dict(cfg, 0))
    x, ts = gold["x"], gold["timesteps"]
    e_c = eng.forward(x, ts, inp["context"], inp["grounding_input"], extra)
    c2, u2 = eng.forward_cfg(x, ts, inp["context"], inp["uc"], inp["grounding_input"], extra)
    assert e_c.shape == (2, cfg.out_channels, H, W)
    for got, ref in ((e_c, gold["eps_cond"]), (c2, gold["eps_cond"]), (u2, gold["eps_null"])):
        assert (got - ref).abs().max() < 5e-5
    # square and non-square plans live side by side
    sq = eng.forward(inp["x"], ts, inp["context"], inp["grounding_input"],
                     torch.cat([inp["z0"], torch.zeros(2, 1, cfg.image_size, cfg.image_size)], 1) if cfg.inpaint_mode else None)
    assert sq.shape[2:] == (cfg.image_size, cfg.image_size)
    assert sorted(k[:1] + k[3:] for k in eng.plans) == [(2,), (2, H, W), (4, H, W)]     # the square default keeps the short key


@pytest.mark.parametrize("name", ["tiny", "tiny_inpaint"])
def test_dropin_plms_non_square_matches_reference_latents(cpu_backend, name):  # noqa: F811
    """PLMSSampler.sample(S=4, shape=(2, 4, 16, 24)) through the drop-in UNetModel (CFG 7.5; tiny_inpaint: scheduled sampling
    and the per-step inpainting blend) against the reference loop's final latent."""
    import test_engine_gpu as teg
    from ldm.models.diffusion.ldm import LatentDiffusion
    from ldm.models.diffusion.plms import PLMSSampler
    cfg, gold, inp, extra = load_case(name, 16, 24)
    g = gold["plms"]
    _, model = teg.build_model(name)
    grounding = model.grounding_tokenizer_input.prepare(inp["batch"])
    diffusion = LatentDiffusion(linear_start=0.00085, linear_end=0.012, timesteps=1000)
    sampler = PLMSSampler(diffusion, model, alpha_generator_func=partial(teg.alpha_generator, type=g["alpha_type"]),
                          set_alpha_scale=teg.set_alpha_scale)
    input = dict(x=gold["x"].clone(), timesteps=None, context=inp["context"], grounding_input=grounding, inpainting_extra_input=extra,
                 grounding_extra_input=None)
    torch.manual_seed(1234)
    lat = sampler.sample(S=g["S"], shape=tuple(gold["x"].shape), input=input, uc=inp["uc"], guidance_scale=g["guidance"],
                         mask=gold["mask"], x0=gold["z0"])
    r = rel_l2(lat, g["latent"])
    assert r < 2e-4, f"{name} plms 16x24: latent rel_l2 {r:.3e}"


def test_engine_refuses_sides_the_downsamples_cannot_halve():
    cfg = NAMED_CONFIGS["tiny"]
    eng = Engine(cfg, RefOps())
    eng.load_state_dict(synthetic_state_dict(cfg, 0))
    inp = synth.make_inputs(cfg, 1, 4, seed=2)
    f = max(b.ds for b in eng.blocks)
    x = torch.zeros(1, cfg.in_channels, 16, 16 + f // 2)
    with pytest.raises(ValueError, match=f"16x{16 + f // 2}"):
        eng.forward(x, torch.tensor([10]), inp["context"], inp["grounding_input"])


def test_engine_refuses_downsampler_models_off_their_native_size():
    cfg = NAMED_CONFIGS["tiny_canny"]
    eng = Engine(cfg, RefOps())
    with pytest.raises(ValueError, match="grounding downsampler"):
        eng.check_latent_size(cfg.image_size, cfg.image_size + 8)
    eng.check_latent_size(cfg.image_size, cfg.image_size)


def test_vae_non_square_matches_reference():
    """small_vae decode of a 32 x 48 latent and encode of a 192 x 128 image: oracle and checker-op engines against the reference."""
    cfg = NAMED_VAE_CONFIGS["small_vae"]
    gold = torch.load(os.path.join(GOLD, "res_small_vae_32x48.pt"))
    sd, sde = synthetic_vae_state_dict(cfg, 0), synthetic_vae_encoder_state_dict(cfg, 1)
    assert _close(VO.vae_decode(cfg, sd, gold["z"]), gold["image"], 2e-5)
    assert _close(VO.vae_encode_moments(cfg, sde, gold["x"]), gold["moments"], 2e-5)
    dec = VAEDecoderEngine(cfg, RefOps("cpu", torch.float32))
    dec.load_state_dict(sd)
    img = dec.decode(gold["z"])
    assert img.shape == gold["image"].shape and rel_l2(img, gold["image"]) < 2e-5
    enc = VAEEncoderEngine(cfg, RefOps("cpu", torch.float32))
    enc.load_state_dict(sde)
    mom = enc.encode_moments(gold["x"])
    assert mom.shape == gold["moments"].shape and rel_l2(mom, gold["moments"]) < 2e-5


def test_vae_refuses_sizes_it_cannot_halve():
    cfg = NAMED_VAE_CONFIGS["tiny_vae64"]
    dec = VAEDecoderEngine(cfg, RefOps("cpu", torch.float32))
    dec.load_state_dict(synthetic_vae_state_dict(cfg, 0))
    with pytest.raises(ValueError, match="8x12"):
        dec.decode(torch.zeros(1, cfg.embed_dim, 8, 12))
    enc = VAEEncoderEngine(cfg, RefOps("cpu", torch.float32))
    enc.load_state_dict(synthetic_vae_encoder_state_dict(cfg, 1))
    with pytest.raises(ValueError, match="16x17"):
        enc.encode_moments(torch.zeros(1, 3, 16, 17))
