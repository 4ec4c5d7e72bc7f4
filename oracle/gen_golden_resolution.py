"""Pin the oracle against the REAL reference at non-square latents and write tests/golden/res_*.pt.   (authoring machine
only: it imports the unmodified reference from /root/reference, like oracle/gen_golden.py, whose helpers it uses)

    python oracle/gen_golden_resolution.py

Cases: the tiny UNet (text, text_image, keypoint, inpaint) at latents 16 x 24 and 24 x 16, B = 2; sd14_box_text B = 1,
G = 30 at 64 x 96 and 96 x 64 (one forward each); PLMS S = 4 loops with CFG at 16 x 24 (tiny, and tiny_inpaint with scheduled
sampling and the inpainting blend) and at 64 x 96 for sd14_box_text (scheduled sampling with the first-conv swap), final
latents only; small_vae decode of a 32 x 48 latent and encode of a 192 x 128 image.  Every reference output is compared
with the oracle restatement (oracle/unet_oracle.py, sampler_oracle.py, vae_oracle.py) to fp32 round-off before it is stored.
Grounding, context and uc come from gligen_b200.synth.make_inputs(seed=2); x (and the inpainting mask / z0) are stored.
"""
from __future__ import annotations

import os
import sys
import time
from functools import partial

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from oracle import gen_golden as GG  # noqa: E402  (mounts the reference `ldm` package)
from oracle import sampler_oracle as SO  # noqa: E402
from oracle import unet_oracle as UO  # noqa: E402
from gligen_b200 import synth  # noqa: E402
from gligen_b200.spec import NAMED_CONFIGS, NAMED_VAE_CONFIGS, synthetic_state_dict  # noqa: E402

GOLD = GG.GOLD


def latent_inputs(cfg, B, H, W):
    """x_T, and for inpainting a box mask and z0 (the mask is the caller's job at non-square sizes)."""
    g = torch.Generator().manual_seed(1000 * H + W)
    x = torch.randn(B, cfg.in_channels, H, W, generator=g)
    if not cfg.inpaint_mode:
        return x, None, None
    z0 = torch.randn(B, cfg.in_channels, H, W, generator=g) * 0.9
    mask = torch.zeros(B, 1, H, W)
    mask[:, :, H // 4: 3 * H // 4, W // 3:] = 1.0
    return x, mask, z0


@torch.no_grad()
def run_case(name, B, max_objs, H, W, plms_S=0, alpha_type=(1, 0, 0)):
    cfg = NAMED_CONFIGS[name]
    print(f"== {name} {H}x{W}: B={B} max_objs={max_objs}", flush=True)
    sd = synthetic_state_dict(cfg, seed=0)
    model = GG.ref_model(cfg)
    print("   ", model.load_state_dict(sd, strict=True))
    gin = GG.ref_grounding_input(cfg)
    model.grounding_tokenizer_input = gin
    inp = synth.make_inputs(cfg, B, max_objs, seed=2)
    grounding = gin.prepare(inp["batch"])
    x, mask, z0 = latent_inputs(cfg, B, H, W)
    extra = None if mask is None else torch.cat([z0 * mask, mask], dim=1)
    ts = torch.tensor([981, 501, 21, 1][:B], dtype=torch.long)
    GG.set_alpha_scale(model, 1.0)
    t0 = time.time()
    e_c = model(dict(x=x, timesteps=ts, context=inp["context"], grounding_input=grounding, inpainting_extra_input=extra,
                     grounding_extra_input=None))
    e_u = model(dict(x=x, timesteps=ts, context=inp["uc"], inpainting_extra_input=extra, grounding_extra_input=None))
    print(f"   ref forwards {time.time() - t0:.1f}s", flush=True)
    GG.check("eps_cond", UO.unet_forward(cfg, sd, x, ts, inp["context"], grounding, 1.0, extra), e_c, 2e-4)
    GG.check("eps_null", UO.unet_forward(cfg, sd, x, ts, inp["uc"], UO.null_grounding(cfg, grounding), 1.0, extra), e_u, 2e-4)
    out = {"cfg": name, "B": B, "max_objs": max_objs, "H": H, "W": W, "x": x, "mask": mask, "z0": z0, "timesteps": ts,
           "eps_cond": e_c.clone(), "eps_null": e_u.clone()}
    if plms_S:
        out["plms"] = plms_loop(cfg, sd, gin, inp, grounding, x, mask, z0, extra, plms_S, list(alpha_type))
    path = os.path.join(GOLD, f"res_{name}_{H}x{W}.pt")
    torch.save(out, path)
    print(f"   wrote {path} ({os.path.getsize(path) / 1024:.0f} KiB)", flush=True)


def plms_loop(cfg, sd, gin, inp, grounding, x, mask, z0, extra, S, atype):
    """Reference PLMSSampler.sample(S, shape=x.shape, CFG 7.5) and its oracle twin (gen_golden.run_config's recipe)."""
    from ldm.models.diffusion.ldm import LatentDiffusion
    from ldm.models.diffusion.plms import PLMSSampler
    diffusion = LatentDiffusion(linear_start=0.00085, linear_end=0.012, timesteps=1000)
    sd_conv = torch.load(os.path.join(GG.REF, "SD_input_conv_weight_bias.pth"))
    m = GG.ref_model(cfg)
    m.load_state_dict(sd, strict=True)
    m.grounding_tokenizer_input = gin
    sampler = PLMSSampler(diffusion, m, alpha_generator_func=partial(SO.alpha_generator, type=atype), set_alpha_scale=GG.set_alpha_scale)
    input = dict(x=x.clone(), timesteps=None, context=inp["context"], grounding_input=grounding, inpainting_extra_input=extra,
                 grounding_extra_input=None)
    cwd = os.getcwd()
    os.chdir(GG.REF)                                   # restore_first_conv_from_SD reads a CWD-relative file
    try:
        torch.manual_seed(1234)
        t0 = time.time()
        ref = sampler.sample(S=S, shape=tuple(x.shape), input=input, uc=inp["uc"], guidance_scale=7.5, mask=mask, x0=z0)
        print(f"   ref plms S={S} alpha={atype}: {time.time() - t0:.1f}s", flush=True)
    finally:
        os.chdir(cwd)
    state = {"scale": 1.0, "sd": dict(sd)}

    def on_alpha(a):
        state["scale"] = a
        if a == 0 and not cfg.inpaint_mode:            # openaimodel.py:400-413
            state["sd"]["input_blocks.0.0.weight"] = sd_conv["weight"]
            state["sd"]["input_blocks.0.0.bias"] = sd_conv["bias"]

    def eps_fn(xx, t, cond):
        gr = grounding if cond else UO.null_grounding(cfg, grounding)
        return UO.unet_forward(cfg, state["sd"], xx, t, inp["context"] if cond else inp["uc"], gr, state["scale"], extra)

    torch.manual_seed(1234)
    got = SO.plms_sample(eps_fn, S, tuple(x.shape), SO.make_schedule(), x_T=x.clone(), use_cfg=True, guidance_scale=7.5,
                         alphas=SO.alpha_generator(S, atype), on_alpha=on_alpha, mask=mask, x0=z0)
    GG.check(f"plms S={S}", got, ref, 5e-4)
    return {"S": S, "alpha_type": atype, "guidance": 7.5, "latent": ref.clone()}


@torch.no_grad()
def run_vae(name="small_vae", h=32, w=48):
    """Reference AutoencoderKL.decode of an h x w latent and encode of a (w * f) x (h * f) image (the transposed shape)."""
    from gligen_b200.spec import synthetic_vae_encoder_state_dict, synthetic_vae_state_dict
    from oracle import vae_oracle as VO
    from ldm.models.autoencoder import AutoencoderKL
    cfg = NAMED_VAE_CONFIGS[name]
    f = 1 << (len(cfg.ch_mult) - 1)
    dd = dict(double_z=True, z_channels=cfg.z_channels, resolution=cfg.image_size, in_channels=3, out_ch=cfg.out_ch, ch=cfg.ch,
              ch_mult=list(cfg.ch_mult), num_res_blocks=cfg.num_res_blocks, attn_resolutions=[], dropout=0.0)
    ref = AutoencoderKL(ddconfig=dd, embed_dim=cfg.embed_dim, scale_factor=cfg.scale_factor).eval()
    sd = dict(synthetic_vae_state_dict(cfg, 0))
    sd.update(synthetic_vae_encoder_state_dict(cfg, 1))
    ref.load_state_dict(sd, strict=True)
    g = torch.Generator().manual_seed(h * w)
    z = torch.randn(1, cfg.embed_dim, h, w, generator=g) * cfg.scale_factor * 4.0
    img = ref.decode(z)
    GG.check("vae decode", VO.vae_decode(cfg, sd, z), img, 1e-4)
    x = (torch.rand(1, 3, w * f, h * f, generator=g) * 2 - 1)
    mom = ref.quant_conv(ref.encoder(x))
    GG.check("vae encode moments", VO.vae_encode_moments(cfg, sd, x), mom, 1e-4)
    path = os.path.join(GOLD, f"res_{name}_{h}x{w}.pt")
    torch.save({"name": name, "z": z, "image": img, "x": x, "moments": mom}, path)
    print(f"   wrote {path} ({os.path.getsize(path) / 1024:.0f} KiB)", flush=True)


if __name__ == "__main__":
    torch.set_num_threads(os.cpu_count())
    run_vae()
    for name, G in (("tiny", 6), ("tiny_text_image", 5), ("tiny_keypoint", 34), ("tiny_inpaint", 6)):
        for H, W in ((16, 24), (24, 16)):
            S = 4 if (H, W) == (16, 24) and name in ("tiny", "tiny_inpaint") else 0
            run_case(name, 2, G, H, W, plms_S=S, alpha_type=(0.5, 0, 0.5) if name == "tiny_inpaint" else (1, 0, 0))
    run_case("sd14_box_text", 1, 30, 64, 96, plms_S=4, alpha_type=(0.5, 0, 0.5))
    run_case("sd14_box_text", 1, 30, 96, 64)
