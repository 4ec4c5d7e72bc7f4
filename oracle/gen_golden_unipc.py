"""Write tests/golden/unipc_*.pt: final latents of the float64 UniPC oracle (oracle/unipc_oracle.py) driving the fp32 UNet oracle
(oracle/fuser_oracle.py), on the models, weights and inputs of the dpm_* fixtures (oracle/gen_golden_dpm.py).

    python oracle/gen_golden_unipc.py

CPU only; it needs no reference checkout.  Weights are gligen_b200.spec.synthetic_state_dict(cfg, 0), inputs
gligen_b200.synth.make_inputs(seed=2), the generator seeded with 1234 before each run (it feeds the inpainting blend's q_sample
noise), CFG 7.5.  On an alpha = 0 step the fusers run at scale 0 and, except for inpainting models, the first conv becomes SD's
(tests/golden/SD_input_conv_weight_bias.pth), as restore_first_conv_from_SD does.  S = 6 (7 steps, the final orders lowered);
one tiny run at S = 16 (17 steps) covers a run whose final orders are not lowered.
"""
from __future__ import annotations

import os
import sys
import time

import torch

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)
from gligen_b200.spec import NAMED_CONFIGS, SAMPLING_GATED_CA, synthetic_state_dict  # noqa: E402
from oracle import fuser_oracle as FO  # noqa: E402
from oracle import sampler_oracle as SO  # noqa: E402
from oracle import unet_oracle as UO  # noqa: E402
from oracle import unipc_oracle as UPO  # noqa: E402
from oracle.gen_golden_dpm import GOLD, GUIDANCE, NOISE_SEED, SEED, case_inputs  # noqa: E402

# (fixture name, config name, config, B, grounding objects, alpha_type, order, S)
CASES = [("tiny_o2", "tiny", NAMED_CONFIGS["tiny"], 2, 6, [1, 0, 0], 2, 6),
         ("tiny_o3", "tiny", NAMED_CONFIGS["tiny"], 2, 6, [1, 0, 0], 3, 6),
         ("tiny_o2_s16", "tiny", NAMED_CONFIGS["tiny"], 2, 6, [1, 0, 0], 2, 16),
         ("tiny_inpaint_o2", "tiny_inpaint", NAMED_CONFIGS["tiny_inpaint"], 2, 6, [0.5, 0, 0.5], 2, 6),
         ("sampling_gated_ca_o2", "sampling_gated_ca", SAMPLING_GATED_CA, 2, 6, [0.3, 0, 0.7], 2, 6),
         ("sd14_box_text_o2", "sd14_box_text", NAMED_CONFIGS["sd14_box_text"], 1, 30, [0.3, 0, 0.7], 2, 6)]


@torch.no_grad()
def oracle_latent(cfg, sd, inp, extra, mask, z0, S, order, alpha_type, x=None):
    """The UniPC oracle sampler's final latent from x (default inp['x'])."""
    sd_conv = torch.load(os.path.join(GOLD, "SD_input_conv_weight_bias.pth"))
    grounding = inp["grounding_input"]
    state = {"scale": 1.0, "sd": dict(sd)}

    def on_alpha(a):
        state["scale"] = a
        if a == 0 and not cfg.inpaint_mode:
            state["sd"]["input_blocks.0.0.weight"] = sd_conv["weight"]
            state["sd"]["input_blocks.0.0.bias"] = sd_conv["bias"]

    def eps_fn(xx, t, cond):
        gr = grounding if cond else UO.null_grounding(cfg, grounding)
        return FO.unet_forward(cfg, state["sd"], xx, t, inp["context"] if cond else inp["uc"], gr, state["scale"], extra)

    x = inp["x"] if x is None else x
    torch.manual_seed(NOISE_SEED)
    return UPO.unipc_sample(eps_fn, S, tuple(x.shape), SO.make_schedule(), x_T=x.clone(), use_cfg=True, guidance_scale=GUIDANCE,
                            order=order, alphas=SO.alpha_generator(len(SO.ddim_timesteps(S)), alpha_type), on_alpha=on_alpha,
                            mask=mask, x0=z0)


def run(name, config, cfg, B, max_objs, alpha_type, order, S):
    t0 = time.time()
    sd = synthetic_state_dict(cfg, 0)
    inp, extra, mask, z0 = case_inputs(cfg, B, max_objs)
    lat = oracle_latent(cfg, sd, inp, extra, mask, z0, S, order, alpha_type)
    path = os.path.join(GOLD, f"unipc_{name}.pt")
    torch.save({"config": config, "B": B, "max_objs": max_objs, "seed": SEED, "S": S, "order": order, "alpha_type": alpha_type,
                "guidance": GUIDANCE, "noise_seed": NOISE_SEED, "latent": lat.clone()}, path)
    print(f"{name}: latent std {lat.std():.3f} ({time.time() - t0:.1f} s); wrote {os.path.basename(path)}", flush=True)


if __name__ == "__main__":
    torch.set_num_threads(os.cpu_count())
    only = os.environ.get("ONLY")
    for case in CASES:
        if only is None or case[0] in only.split(","):
            run(*case)
