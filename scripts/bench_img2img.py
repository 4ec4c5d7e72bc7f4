"""Images/s of image-to-image at strength 0.3 / 0.5 / 0.75 against full sampling, and of two-pass high-resolution sampling
(gligen_b200.pipeline.sample_hires, 512 -> 1024) against direct 1024 x 1024 sampling, on one GPU.

    python scripts/bench_img2img.py [--repeats 2] [--batch 4]

Workload: sd14_box_text (seeded synthetic weights), batch 4, 30 grounding objects, CFG 7.5, alpha_type [0.3, 0, 0.7].
* UniPC-2 S = 15, DPM-Solver++ 2M S = 20 and PLMS S = 50, each in full (from x_T, 64 x 64 latent) and from a seeded 64 x 64
  init_latent at strength 0.3, 0.5 and 0.75.  A run at strength s takes n = int(s L) of the grid's L steps, so the expected
  time is about n / L of the full run's (PLMS: (n + 1) / (L + 1)).
* sample_hires with UniPC-2, S = 15 at 64 x 64, then S = 15 at strength 0.5 on the 128 x 128 upscaled latent, against UniPC-2
  S = 15 sampled directly at 128 x 128.
Every arm once untimed (plans, graphs), then all arms alternately, `--repeats` times each: wall time between device
synchronisations.  Each run reloads the weights first (untimed), so each starts from the GLIGEN first conv.  The UNet passes per
image are counted.  The card's name and power limit are read and printed in the same process as the numbers.
"""
from __future__ import annotations

import argparse
import json
import os
import sys
import time
from functools import partial

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))
from bench_fusers import card  # noqa: E402

DEV = "cuda:0"
ALPHA_TYPE = [0.3, 0.0, 0.7]
SAMPLERS = [("UniPC-2 15", "unipc", 15), ("DPM-Solver++ 2M-20", "dpm", 20), ("PLMS-50", "plms", 50)]
STRENGTHS = [None, 0.3, 0.5, 0.75]              # None: full sampling from x_T


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=2)
    ap.add_argument("--batch", type=int, default=4)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_img2img.py measures on a CUDA device; none is available")
    from gligen_b200 import synth
    from gligen_b200.pipeline import alpha_generator, build_model, sample_hires, sampler_inputs, set_alpha_scale, to_device
    from ldm.models.diffusion.dpm_solver import DPMSolverSampler
    from ldm.models.diffusion.ldm import LatentDiffusion
    from ldm.models.diffusion.plms import PLMSSampler
    from ldm.models.diffusion.unipc import UniPCSampler

    print(card(), flush=True)
    cfg, model = build_model("sd14_box_text", DEV)
    weights = {k: v.detach().cpu().clone() for k, v in model.state_dict().items()}
    inp = synth.make_inputs(cfg, a.batch, 30, seed=2)
    dinp = to_device({k: v for k, v in inp.items() if k in ("x", "context", "uc")}, DEV)
    dbatch = to_device(inp["batch"], DEV)
    shape = tuple(dinp["x"].shape)
    big = shape[:2] + (shape[2] * 2, shape[3] * 2)
    init = (torch.randn(shape, generator=torch.Generator().manual_seed(77)) * 0.9).to(DEV)
    diffusion = LatentDiffusion(linear_start=0.00085, linear_end=0.012, timesteps=1000).to(DEV)
    passes = {"n": 0}
    forward_cfg = model.forward_cfg

    def counted(*args, **kw):
        passes["n"] += 1
        return forward_cfg(*args, **kw)

    model.forward_cfg = counted
    kw = dict(alpha_generator_func=partial(alpha_generator, type=ALPHA_TYPE), set_alpha_scale=set_alpha_scale)
    make = {"plms": lambda: PLMSSampler(diffusion, model, **kw), "dpm": lambda: DPMSolverSampler(diffusion, model, order=2, **kw),
            "unipc": lambda: UniPCSampler(diffusion, model, order=2, **kw)}

    def call(arm):
        kind, S, strength, mode = arm
        sampler = make[kind]()
        input, _, _ = sampler_inputs(cfg, model, dinp, dbatch)
        if mode == "hires":
            return sample_hires(sampler, S, shape, input, dinp["uc"], 7.5, scale=2, strength=0.5)
        if mode == "direct":
            input["x"] = None                                          # x_T drawn at the 128 x 128 size
            return sampler.sample(S, big, input, dinp["uc"], 7.5)
        if strength is None:
            return sampler.sample(S, shape, input, dinp["uc"], 7.5)
        return sampler.sample(S, shape, input, dinp["uc"], 7.5, init_latent=init, strength=strength)

    def run(arm):
        model.load_state_dict(weights)
        model.engine()                                  # re-pack the weights outside the timed window
        passes["n"] = 0
        torch.manual_seed(1234)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        lat = call(arm)
        torch.cuda.synchronize()
        return time.perf_counter() - t0, passes["n"], lat

    arms = {}
    for name, kind, S in SAMPLERS:
        for s in STRENGTHS:
            arms[f"{name} " + ("full" if s is None else f"strength {s}")] = (kind, S, s, "img2img")
    arms["hires 512->1024 UniPC-2 15+15 strength 0.5"] = ("unipc", 15, 0.5, "hires")
    arms["direct 1024 UniPC-2 15"] = ("unipc", 15, None, "direct")

    cwd = os.getcwd()
    os.chdir(os.path.join(ROOT, "tests", "golden"))     # restore_first_conv_from_SD reads SD_input_conv_weight_bias.pth CWD-relative
    try:
        npass, times = {}, {k: [] for k in arms}
        for name, arm in arms.items():                  # warm-up: every shape and schedule once
            _, npass[name], lat = run(arm)
            assert torch.isfinite(lat).all(), name
        for _ in range(a.repeats):
            for name, arm in arms.items():
                secs, n, _ = run(arm)
                times[name].append(secs)
                assert n == npass[name], (name, n, npass[name])
    finally:
        os.chdir(cwd)
    results = {}
    for name in arms:
        ips = [a.batch / t for t in times[name]]
        results[name] = dict(images_per_s=max(ips), images_per_s_runs=ips, unet_passes_per_image=npass[name])
    for sname, _, _ in SAMPLERS:
        full = results[f"{sname} full"]
        for s in STRENGTHS[1:]:
            r = results[f"{sname} strength {s}"]
            r["speedup_vs_full"] = r["images_per_s"] / full["images_per_s"]
            r["pass_ratio_vs_full"] = r["unet_passes_per_image"] / full["unet_passes_per_image"]
    h, d = results["hires 512->1024 UniPC-2 15+15 strength 0.5"], results["direct 1024 UniPC-2 15"]
    h["speedup_vs_direct"] = h["images_per_s"] / d["images_per_s"]
    for name, r in results.items():
        extra = "".join(f", {k} {r[k]:.2f}" for k in ("speedup_vs_full", "pass_ratio_vs_full", "speedup_vs_direct") if k in r)
        print(f"{name}: {', '.join(f'{v:.3f}' for v in r['images_per_s_runs'])} images/s (batch {a.batch}), "
              f"{r['unet_passes_per_image']} UNet passes{extra}", flush=True)
    print(json.dumps(dict(card=card(), batch=a.batch, alpha_type=ALPHA_TYPE, guidance=7.5, results=results)))


if __name__ == "__main__":
    main()
