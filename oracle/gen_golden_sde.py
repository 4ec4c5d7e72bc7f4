"""Write tests/golden/sde_*.pt: final latents of stochastic runs over the fp32 UNet oracle (oracle/fuser_oracle.py), on the models,
weights and inputs of the dpm_* fixtures (oracle/gen_golden_dpm.py).

    python oracle/gen_golden_sde.py

  * DDIM with eta > 0: the REFERENCE's own DDIMSampler (unmodified, mounted by oracle/ref_harness.py): make_schedule(S,
    ddim_eta=eta), then ddim_sampling(...) for a full run, or its p_sample_ddim over the truncated range for image-to-image
    (as oracle/img2img_oracle.ref_sample does).  The reference's sample() fixes eta = 0; these calls reach its stochastic path.
  * DPM-Solver++ 2M SDE: the float64 VE-form oracle (oracle/sde_oracle.py).

Weights are gligen_b200.spec.synthetic_state_dict(cfg, 0), inputs gligen_b200.synth.make_inputs(seed=2), the CPU generator seeded
with 1234 before each run (it feeds the per-step noise and the inpainting blend's q_sample noise), CFG 7.5.  The image-to-image
case starts from img2img_oracle.init_and_noise(shape, 77) at strength 0.5.
"""
from __future__ import annotations

import os
import sys
import time

import torch

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)
from gligen_b200.spec import NAMED_CONFIGS, SAMPLING_GATED_CA, synthetic_state_dict  # noqa: E402
from oracle import img2img_oracle as IO  # noqa: E402
from oracle import sampler_oracle as SO  # noqa: E402
from oracle import sde_oracle as SDO  # noqa: E402
from oracle.gen_golden_dpm import GOLD, GUIDANCE, NOISE_SEED, SEED, case_inputs  # noqa: E402
from oracle.gen_golden_img2img import INIT_SEED, model_fns  # noqa: E402

S = 6

# (fixture name, config name, B, grounding objects, sampler, eta, strength, alpha_type)
CASES = [("ddim_eta05_tiny", "tiny", 2, 6, "ddim", 0.5, 1.0, [1, 0, 0]),
         ("ddim_eta1_tiny", "tiny", 2, 6, "ddim", 1.0, 1.0, [1, 0, 0]),
         ("ddim_eta1_tiny_inpaint", "tiny_inpaint", 2, 6, "ddim", 1.0, 1.0, [0.5, 0, 0.5]),
         ("ddim_eta1_sampling_gated_ca", "sampling_gated_ca", 2, 6, "ddim", 1.0, 1.0, [0.3, 0, 0.7]),
         ("ddim_eta1_sd14_box_text", "sd14_box_text", 1, 30, "ddim", 1.0, 1.0, [0.3, 0, 0.7]),
         ("ddim_eta1_img2img_tiny", "tiny", 2, 6, "ddim", 1.0, 0.5, [1, 0, 0]),
         ("dpm2sde_tiny", "tiny", 2, 6, "dpm2sde", 1.0, 1.0, [1, 0, 0]),
         ("dpm2sde_tiny_inpaint", "tiny_inpaint", 2, 6, "dpm2sde", 1.0, 1.0, [0.5, 0, 0.5]),
         ("dpm2sde_sampling_gated_ca", "sampling_gated_ca", 2, 6, "dpm2sde", 1.0, 1.0, [0.3, 0, 0.7]),
         ("dpm2sde_sd14_box_text", "sd14_box_text", 1, 30, "dpm2sde", 1.0, 1.0, [0.3, 0, 0.7]),
         ("dpm2sde_img2img_tiny", "tiny", 2, 6, "dpm2sde", 1.0, 0.5, [1, 0, 0])]


def config(name):
    return SAMPLING_GATED_CA if name == "sampling_gated_ca" else NAMED_CONFIGS[name]


class _RefModel(IO._EpsModel):
    """The model the reference DDIMSampler drives: on_alpha (called through set_alpha_scale) already swaps the first conv."""

    def restore_first_conv_from_SD(self):
        pass


@torch.no_grad()
def ref_ddim(eps_fn, on_alpha, shape, x_T, eta, strength, alpha_type, mask, z0, init=None, noise=None):
    from oracle import ref_harness as RH
    RH.mount()
    from ldm.models.diffusion.ddim import DDIMSampler
    assert RH.is_reference_module(DDIMSampler)
    diffusion = RH.ref_diffusion("cpu")
    sampler = DDIMSampler(diffusion, _RefModel(eps_fn), alpha_generator_func=lambda n: SO.alpha_generator(n, alpha_type),
                          set_alpha_scale=lambda model, a: on_alpha(a))
    sampler.make_schedule(ddim_num_steps=S, ddim_eta=eta)
    input = dict(x=x_T, timesteps=None, context=None, grounding_input=True, inpainting_extra_input=None, grounding_extra_input=None)
    if init is None:
        return sampler.ddim_sampling(shape, input, uc=True, guidance_scale=GUIDANCE, mask=mask, x0=z0)
    time_range, L = IO.truncated_range(S, strength)
    n, b = len(time_range), shape[0]
    alphas = SO.alpha_generator(n, alpha_type)
    img = diffusion.q_sample(init.float(), torch.full((b,), int(time_range[0]), dtype=torch.long), noise=noise.float())
    for i, step in enumerate(time_range):
        on_alpha(alphas[i])
        ts = torch.full((b,), int(step), dtype=torch.long)
        if mask is not None:
            img = diffusion.q_sample(z0, ts) * mask + (1.0 - mask) * img
        input["x"], input["timesteps"] = img, ts
        img, _ = sampler.p_sample_ddim(input, index=n - i - 1, uc=True, guidance_scale=GUIDANCE)
    return img


@torch.no_grad()
def run(name, config_name, B, max_objs, kind, eta, strength, alpha_type):
    t0 = time.time()
    cfg = config(config_name)
    sd = synthetic_state_dict(cfg, 0)
    inp, extra, mask, z0 = case_inputs(cfg, B, max_objs)
    eps_fn, on_alpha = model_fns(cfg, sd, inp, extra)
    shape = tuple(inp["x"].shape)
    init = noise = None
    if strength < 1.0:
        init, noise = IO.init_and_noise(shape, INIT_SEED)
    torch.manual_seed(NOISE_SEED)
    if kind == "ddim":
        lat = ref_ddim(eps_fn, on_alpha, shape, inp["x"].clone(), eta, strength, alpha_type, mask, z0, init, noise)
    else:
        time_range, _ = IO.truncated_range(S, strength)
        x_T = inp["x"].clone()
        if init is not None:
            t0_ = torch.full((B,), int(time_range[0]), dtype=torch.long)
            x_T = SO.q_sample(SO.make_schedule(), init.float(), t0_, noise.float())
        lat = SDO.sde_sample(eps_fn, S, shape, x_T=x_T, guidance_scale=GUIDANCE, order=2, eta=eta,
                             alphas=SO.alpha_generator(len(time_range), alpha_type), on_alpha=on_alpha, mask=mask, x0=z0,
                             time_range=time_range)
    path = os.path.join(GOLD, f"sde_{name}.pt")
    torch.save({"config": config_name, "B": B, "max_objs": max_objs, "seed": SEED, "sampler": kind, "order": 2, "eta": eta, "S": S,
                "strength": strength, "alpha_type": alpha_type, "guidance": GUIDANCE, "noise_seed": NOISE_SEED,
                "init_seed": INIT_SEED if init is not None else None, "latent": lat.float().clone()}, path)
    print(f"{name}: latent std {lat.std():.3f} ({time.time() - t0:.1f} s); wrote {os.path.basename(path)}", flush=True)


if __name__ == "__main__":
    from oracle import ref_harness as RH
    RH.mount()                  # before anything imports ldm: DDIM runs the reference's own sampler
    torch.set_num_threads(os.cpu_count())
    only = os.environ.get("ONLY")
    for case in CASES:
        if only is None or case[0] in only.split(","):
            run(*case)
