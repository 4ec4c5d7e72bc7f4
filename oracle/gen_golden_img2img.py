"""Write tests/golden/img2img_*.pt: final latents of image-to-image runs (oracle/img2img_oracle.py) over the fp32 UNet oracle
(oracle/fuser_oracle.py), on the models, weights and inputs of the dpm_* fixtures (oracle/gen_golden_dpm.py).

    python oracle/gen_golden_img2img.py

PLMS / DDIM step through the reference's own per-step methods, so this needs the reference (/root/reference, or the archive
oracle/build_ref.py writes).  Weights are gligen_b200.spec.synthetic_state_dict(cfg, 0), inputs gligen_b200.synth.make_inputs(
seed=2), the start image and noise img2img_oracle.init_and_noise(shape, INIT_SEED), the generator seeded with 1234 before each
run (it feeds the per-step draws), CFG 7.5.  On an alpha = 0 step the fusers run at scale 0 and, except for inpainting models,
the first conv becomes SD's, as restore_first_conv_from_SD does.

The hires case is the two-pass composition of gligen_b200.pipeline.sample_hires: pass 1 is the dpm_tiny_o2 fixture (16 x 16),
upscaled x2 by float64 bicubic interpolation (align_corners = False), then DPM-Solver++ 2M at strength 0.5 on 32 x 32 from the
noise torch.randn(B, 4, 32, 32) drawn first after seeding 1234 (pass 2's only draw).
"""
from __future__ import annotations

import os
import sys
import time

import torch

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)
from gligen_b200.spec import NAMED_CONFIGS, synthetic_state_dict  # noqa: E402
from oracle import fuser_oracle as FO  # noqa: E402
from oracle import img2img_oracle as IO  # noqa: E402
from oracle import unet_oracle as UO  # noqa: E402
from oracle.gen_golden_dpm import GOLD, GUIDANCE, NOISE_SEED, SEED, case_inputs  # noqa: E402

INIT_SEED = 77

# (fixture name, config name, B, grounding objects, sampler, order, S, strength, alpha_type)
CASES = [("tiny_plms", "tiny", 2, 6, "plms", 0, 10, 0.6, [1, 0, 0]),
         ("tiny_ddim", "tiny", 2, 6, "ddim", 0, 10, 0.6, [1, 0, 0]),
         ("tiny_dpm2", "tiny", 2, 6, "dpm", 2, 10, 0.6, [1, 0, 0]),
         ("tiny_unipc2", "tiny", 2, 6, "unipc", 2, 10, 0.6, [1, 0, 0]),
         ("tiny_inpaint_dpm2", "tiny_inpaint", 2, 6, "dpm", 2, 10, 0.5, [0.5, 0, 0.5]),
         ("tiny_hed_unipc2", "tiny_hed", 2, 30, "unipc", 2, 6, 0.5, [1, 0, 0]),
         ("sd14_box_text_unipc2", "sd14_box_text", 1, 30, "unipc", 2, 10, 0.5, [0.3, 0, 0.7]),
         ("sd14_box_text_plms", "sd14_box_text", 1, 30, "plms", 0, 10, 0.5, [0.3, 0, 0.7])]
HIRES = ("hires_tiny_dpm2", "dpm_tiny_o2.pt", 2, 6, 0.5)          # (name, pass-1 fixture, scale, S, strength)


def model_fns(cfg, sd, inp, extra):
    """(eps_fn, on_alpha) of the fp32 UNet oracle with the scheduled-sampling state."""
    sd_conv = torch.load(os.path.join(GOLD, "SD_input_conv_weight_bias.pth"))
    grounding = inp["grounding_input"]
    gextra = inp.get("grounding_extra_input")
    state = {"scale": 1.0, "sd": dict(sd)}

    def on_alpha(a):
        state["scale"] = a
        if a == 0 and not cfg.inpaint_mode:
            state["sd"]["input_blocks.0.0.weight"] = sd_conv["weight"]
            state["sd"]["input_blocks.0.0.bias"] = sd_conv["bias"]

    def eps_fn(xx, t, cond):
        gr = grounding if cond else UO.null_grounding(cfg, grounding)
        return FO.unet_forward(cfg, state["sd"], xx, t, inp["context"] if cond else inp["uc"], gr, state["scale"], extra,
                               grounding_extra_input=gextra)

    return eps_fn, on_alpha


@torch.no_grad()
def oracle_latent(cfg, kind, order, S, strength, alpha_type, init, noise, B, max_objs):
    sd = synthetic_state_dict(cfg, 0)
    inp, extra, mask, z0 = case_inputs(cfg, B, max_objs)
    eps_fn, on_alpha = model_fns(cfg, sd, inp, extra)
    torch.manual_seed(NOISE_SEED)
    if kind in ("plms", "ddim"):
        return IO.ref_sample(kind, eps_fn, S, strength, init, noise, GUIDANCE, alpha_type, on_alpha, mask, z0)
    return IO.fast_sample(kind, eps_fn, S, strength, init, noise, guidance_scale=GUIDANCE, order=order, alpha_type=alpha_type,
                          on_alpha=on_alpha, mask=mask, x0=z0)


def run(name, config, B, max_objs, kind, order, S, strength, alpha_type):
    t0 = time.time()
    cfg = NAMED_CONFIGS[config]
    shape = (B, 4, cfg.image_size, cfg.image_size)
    init, noise = IO.init_and_noise(shape, INIT_SEED)
    lat = oracle_latent(cfg, kind, order, S, strength, alpha_type, init, noise, B, max_objs)
    _save(name, {"config": config, "B": B, "max_objs": max_objs, "seed": SEED, "sampler": kind, "order": order, "S": S,
                 "strength": strength, "alpha_type": alpha_type, "guidance": GUIDANCE, "noise_seed": NOISE_SEED,
                 "init_seed": INIT_SEED}, lat, t0)


def run_hires(name, pass1, scale, S, strength):
    t0 = time.time()
    gold = torch.load(os.path.join(GOLD, pass1))
    cfg = NAMED_CONFIGS[gold["config"]]
    B, n = gold["B"], cfg.image_size * scale
    up = torch.nn.functional.interpolate(gold["latent"].double(), size=(n, n), mode="bicubic", align_corners=False).float()
    torch.manual_seed(NOISE_SEED)
    noise = torch.randn(B, 4, n, n)
    lat = oracle_latent(cfg, "dpm", gold["order"], S, strength, gold["alpha_type"], up, noise, B, gold["max_objs"])
    _save(name, {"config": gold["config"], "pass1": pass1, "B": B, "max_objs": gold["max_objs"], "seed": SEED, "sampler": "dpm",
                 "order": gold["order"], "S": S, "scale": scale, "strength": strength, "alpha_type": gold["alpha_type"],
                 "guidance": GUIDANCE, "noise_seed": NOISE_SEED}, lat, t0)


def _save(name, meta, lat, t0):
    path = os.path.join(GOLD, f"img2img_{name}.pt")
    torch.save({**meta, "latent": lat.clone()}, path)
    print(f"{name}: latent std {lat.std():.3f} ({time.time() - t0:.1f} s); wrote {os.path.basename(path)}", flush=True)


if __name__ == "__main__":
    from oracle import ref_harness as RH
    RH.mount()                  # before anything imports ldm: PLMS / DDIM run the reference's own per-step methods
    torch.set_num_threads(os.cpu_count())
    only = os.environ.get("ONLY")
    for case in CASES:
        if only is None or case[0] in only.split(","):
            run(*case)
    if only is None or HIRES[0] in only.split(","):
        run_hires(*HIRES)
