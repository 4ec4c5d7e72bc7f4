"""Write tests/golden/karras_*.pt: the UNet at fractional timesteps, and final latents of Karras-grid sampling runs.

    python oracle/gen_golden_karras.py            # ONLY=unet_tiny,dpm2m_tiny,... for a subset

  * karras_unet_<config>.pt: the UNMODIFIED reference UNetModel (oracle/ref_harness.py) at the fractional timesteps
    t = [999.0, 500.37, 12.25, 0.5] (one per batch row), cond and null passes at fuser scale 1, after asserting that the fp32
    oracle (oracle/unet_oracle.py) agrees with it; the measured max-abs difference is stored as "oracle_maxabs".  This part needs
    the reference checkout that oracle/ref_harness.py mounts (or the archive oracle/build_ref.py writes).
  * karras_<sampler>_<case>.pt: S = 6 runs of oracle/karras_oracle.py over the fp32 UNet oracle (oracle/fuser_oracle.py), on the
    models, weights and inputs of the dpm_* fixtures (oracle/gen_golden_dpm.py): weights gligen_b200.spec.synthetic_state_dict(cfg,
    0), inputs gligen_b200.synth.make_inputs(seed=2), the CPU generator seeded with 1234 before each run (it feeds the blend's and the
    SDE's per-step draws), CFG 7.5.  The image-to-image case starts from img2img_oracle.init_and_noise(shape, 77) at strength 0.5.
"""
from __future__ import annotations

import os
import sys
import time

import torch

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)
from gligen_b200 import synth  # noqa: E402
from gligen_b200.spec import NAMED_CONFIGS, SAMPLING_GATED_CA, synthetic_state_dict  # noqa: E402
from oracle import img2img_oracle as IO  # noqa: E402
from oracle import karras_oracle as KO  # noqa: E402
from oracle import sampler_oracle as SO  # noqa: E402
from oracle import unet_oracle as UO  # noqa: E402
from oracle.gen_golden_dpm import GOLD, GUIDANCE, NOISE_SEED, SEED, case_inputs  # noqa: E402
from oracle.gen_golden_img2img import INIT_SEED, model_fns  # noqa: E402

S = 6
FRACTIONAL_T = [999.0, 500.37, 12.25, 0.5]

# (config name, grounding objects)
UNET_CASES = [("tiny", 6), ("sd14_box_text", 30)]

# (fixture name, config name, B, grounding objects, oracle kind, order, eta, strength, alpha_type)
CASES = [("dpm2m_tiny", "tiny", 2, 6, "dpm2m", 2, 0.0, 1.0, [1, 0, 0]),
         ("dpm3m_tiny", "tiny", 2, 6, "dpm", 3, 0.0, 1.0, [1, 0, 0]),
         ("unipc2_tiny", "tiny", 2, 6, "unipc", 2, 0.0, 1.0, [1, 0, 0]),
         ("dpm2msde_tiny", "tiny", 2, 6, "dpm2msde", 2, 1.0, 1.0, [1, 0, 0]),
         ("dpm2m_tiny_inpaint", "tiny_inpaint", 2, 6, "dpm2m", 2, 0.0, 1.0, [0.5, 0, 0.5]),
         ("dpm2m_sampling_gated_ca", "sampling_gated_ca", 2, 6, "dpm2m", 2, 0.0, 1.0, [0.3, 0, 0.7]),
         ("dpm2m_img2img_tiny", "tiny", 2, 6, "dpm2m", 2, 0.0, 0.5, [1, 0, 0]),
         ("dpm2m_sd14_box_text", "sd14_box_text", 1, 30, "dpm2m", 2, 0.0, 1.0, [0.3, 0, 0.7])]

# the product sampler each oracle kind stands for: (sampler, order)
PRODUCT = {"dpm2m": ("dpm", 2), "dpm": ("dpm", 3), "unipc": ("unipc", 2), "dpm2msde": ("dpm", 2)}


def config(name):
    return SAMPLING_GATED_CA if name == "sampling_gated_ca" else NAMED_CONFIGS[name]


@torch.no_grad()
def run_unet(config_name, max_objs):
    from oracle import ref_harness as RH
    t0 = time.time()
    cfg = NAMED_CONFIGS[config_name]
    sd = synthetic_state_dict(cfg, 0)
    model = RH.ref_model(cfg)
    model.load_state_dict(sd, strict=True)
    B = len(FRACTIONAL_T)
    inp = synth.make_inputs(cfg, B, max_objs, seed=SEED)
    ts = torch.tensor(FRACTIONAL_T, dtype=torch.float32)
    gin = RH.ref_grounding_input(cfg)
    model.grounding_tokenizer_input = gin
    RH.set_alpha_scale(model, 1.0)
    grounding = gin.prepare(inp["batch"])           # the null pass below reads the shape of this prepared input
    e_c = model(dict(x=inp["x"], timesteps=ts, context=inp["context"], grounding_input=grounding, inpainting_extra_input=None,
                     grounding_extra_input=None))
    e_u = model(dict(x=inp["x"], timesteps=ts, context=inp["uc"], inpainting_extra_input=None, grounding_extra_input=None))
    o_c = UO.unet_forward(cfg, sd, inp["x"], ts, inp["context"], inp["grounding_input"], 1.0)
    o_u = UO.unet_forward(cfg, sd, inp["x"], ts, inp["uc"], UO.null_grounding(cfg, inp["grounding_input"]), 1.0)
    err = max((o_c - e_c).abs().max().item(), (o_u - e_u).abs().max().item())
    assert err <= 2e-4 * max(1.0, e_c.abs().max().item()), err
    path = os.path.join(GOLD, f"karras_unet_{config_name}.pt")
    torch.save({"config": config_name, "B": B, "max_objs": max_objs, "seed": SEED, "timesteps": ts, "scale": 1.0,
                "eps_cond": e_c.clone(), "eps_null": e_u.clone(), "oracle_maxabs": err}, path)
    print(f"unet {config_name}: oracle vs reference max-abs {err:.3e}, eps std {e_c.std():.3f} ({time.time() - t0:.1f} s); "
          f"wrote {os.path.basename(path)}", flush=True)


@torch.no_grad()
def run(name, config_name, B, max_objs, kind, order, eta, strength, alpha_type):
    t0 = time.time()
    cfg = config(config_name)
    sd = synthetic_state_dict(cfg, 0)
    inp, extra, mask, z0 = case_inputs(cfg, B, max_objs)
    eps_fn, on_alpha = model_fns(cfg, sd, inp, extra)
    shape = tuple(inp["x"].shape)
    init = noise = None
    if strength < 1.0:
        init, noise = IO.init_and_noise(shape, INIT_SEED)
    n = min(S, int(strength * S))
    torch.manual_seed(NOISE_SEED)
    lat = KO.karras_sample(kind, eps_fn, S, shape, x_T=inp["x"].clone(), guidance_scale=GUIDANCE, order=order, eta=eta,
                           alphas=SO.alpha_generator(n, alpha_type), on_alpha=on_alpha, mask=mask, x0=z0, init=init, noise=noise,
                           strength=strength)
    sampler, order_ = PRODUCT[kind]
    path = os.path.join(GOLD, f"karras_{name}.pt")
    torch.save({"config": config_name, "B": B, "max_objs": max_objs, "seed": SEED, "sampler": sampler, "order": order_, "eta": eta,
                "grid": "karras", "S": S, "strength": strength, "alpha_type": alpha_type, "guidance": GUIDANCE,
                "noise_seed": NOISE_SEED, "init_seed": INIT_SEED if init is not None else None, "oracle": kind,
                "latent": lat.float().clone()}, path)
    print(f"{name}: latent std {lat.std():.3f} ({time.time() - t0:.1f} s); wrote {os.path.basename(path)}", flush=True)


if __name__ == "__main__":
    torch.set_num_threads(os.cpu_count())
    only = os.environ.get("ONLY")
    for cfg_name, objs in UNET_CASES:
        if only is None or f"unet_{cfg_name}" in only.split(","):
            run_unet(cfg_name, objs)
    for case in CASES:
        if only is None or case[0] in only.split(","):
            run(*case)
