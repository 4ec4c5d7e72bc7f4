"""Images/s of the stochastic samplers on one GPU against their deterministic forms at the same number of UNet passes: DDIM at
S = 50 with eta = 1 against eta = 0, and DPM-Solver++ 2M SDE (eta = 1) against 2M at S = 20 and 25.

    python scripts/bench_stochastic.py [--repeats 3] [--batch 4]

Workload: sd14_box_text (seeded synthetic weights), batch 4, 64 x 64 latent (512 x 512 images), 30 grounding objects, CFG 7.5,
alpha_type [0.3, 0, 0.7].
1. Every arm once untimed, then the arms alternately, `--repeats` times each: wall time of sample() between device
   synchronisations -> images/s, and the UNet passes per image (the paired arms must take the same number).
2. glg_sde_update alone, CUDA events around a CUDA graph of 200 launches at the batch's latent (4 x 4 x 64 x 64), with CFG and m1
   (a 2M SDE step): x, e_c, e_u, m1, z read and x0_out, x_next written, 28 B per element, against the HBM bound at 3.35 TB/s
   (H100 SXM data sheet).
The card's name and power limit are printed with the numbers.
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
from bench_samplers import _graph_time, _step20_grid  # noqa: E402

DEV = "cuda:0"
ALPHA_TYPE = [0.3, 0.0, 0.7]
# (name, sampler, S, eta); each stochastic arm follows its deterministic pair
RUNS = [("DDIM-50", "ddim", 50, 0.0), ("DDIM-50 eta=1", "ddim", 50, 1.0),
        ("DPM-Solver++ 2M-20", "dpm", 20, 0.0), ("DPM-Solver++ 2M SDE-20", "dpm", 20, 1.0),
        ("DPM-Solver++ 2M-25", "dpm", 25, 0.0), ("DPM-Solver++ 2M SDE-25", "dpm", 25, 1.0)]


def sde_update_kernel_time(batch):
    from gligen_b200.ops import CudaOps
    from ldm.models.diffusion import dpm_solver as DS
    ops = CudaOps(DEV)
    x, ec, eu, m1, z = (torch.randn(batch, 4, 64, 64, device=DEV) for _ in range(5))
    m0, xn = torch.empty_like(x), torch.empty_like(x)
    alpha, sigma = _step20_grid()
    coefs = DS.sde_coefficients(alpha, sigma, DS.step_orders(len(alpha) - 1, 2), 1.0)[5]
    return _graph_time("glg_sde_update", batch, lambda: ops.sde_update(x, ec, eu, 7.5, m1, z, alpha[5], sigma[5], coefs, m0, xn),
                       7 * x.numel() * 4)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--batch", type=int, default=4)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_stochastic.py measures on a CUDA device; none is available")
    from gligen_b200 import synth
    from gligen_b200.pipeline import alpha_generator, build_model, sampler_inputs, set_alpha_scale, to_device
    from ldm.models.diffusion.ddim import DDIMSampler
    from ldm.models.diffusion.dpm_solver import DPMSolverSampler
    from ldm.models.diffusion.ldm import LatentDiffusion

    print(card(), flush=True)
    cfg, model = build_model("sd14_box_text", DEV)
    weights = {k: v.detach().cpu().clone() for k, v in model.state_dict().items()}
    inp = synth.make_inputs(cfg, a.batch, 30, seed=2)
    dinp = to_device({k: v for k, v in inp.items() if k in ("x", "context", "uc")}, DEV)
    dbatch = to_device(inp["batch"], DEV)
    diffusion = LatentDiffusion(linear_start=0.00085, linear_end=0.012, timesteps=1000).to(DEV)
    passes = {"n": 0}
    forward_cfg = model.forward_cfg

    def counted(*args, **kw):
        passes["n"] += 1
        return forward_cfg(*args, **kw)

    model.forward_cfg = counted
    kw = dict(alpha_generator_func=partial(alpha_generator, type=ALPHA_TYPE), set_alpha_scale=set_alpha_scale)

    def run(kind, S, eta):
        model.load_state_dict(weights)
        model.engine()                                  # re-pack the weights outside the timed window
        call = {}
        if kind == "ddim":
            sampler = DDIMSampler(diffusion, model, **kw)
            call["eta"] = eta
        else:
            sampler = DPMSolverSampler(diffusion, model, order=2, eta=eta, **kw)
        input, _, _ = sampler_inputs(cfg, model, dinp, dbatch)
        passes["n"] = 0
        torch.manual_seed(1234)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        lat = sampler.sample(S=S, shape=tuple(dinp["x"].shape), input=input, uc=dinp["uc"], guidance_scale=7.5, **call)
        torch.cuda.synchronize()
        return time.perf_counter() - t0, passes["n"], lat

    cwd = os.getcwd()
    os.chdir(os.path.join(ROOT, "tests", "golden"))     # restore_first_conv_from_SD reads SD_input_conv_weight_bias.pth CWD-relative
    try:
        times, npass = {name: [] for name, *_ in RUNS}, {}
        for name, kind, S, eta in RUNS:                 # warm-up: every shape and schedule once
            _, npass[name], lat = run(kind, S, eta)
            if not torch.isfinite(lat).all():
                raise SystemExit(f"{name}: non-finite latent")
        for i in range(0, len(RUNS), 2):
            if npass[RUNS[i][0]] != npass[RUNS[i + 1][0]]:
                raise SystemExit(f"{RUNS[i][0]} and {RUNS[i + 1][0]} take different numbers of UNet passes")
        for _ in range(a.repeats):
            for name, kind, S, eta in RUNS:
                times[name].append(run(kind, S, eta)[0])
        results = {}
        for name, *_ in RUNS:
            ips = [a.batch / t for t in times[name]]
            results[name] = dict(images_per_s=max(ips), images_per_s_runs=ips, unet_passes_per_image=npass[name])
            print(f"{name}: {', '.join(f'{v:.3f}' for v in ips)} images/s (batch {a.batch}), {npass[name]} UNet passes per image",
                  flush=True)
        for i in range(0, len(RUNS), 2):
            det, sto = RUNS[i][0], RUNS[i + 1][0]
            results[sto]["ratio_to_deterministic"] = results[sto]["images_per_s"] / results[det]["images_per_s"]
    finally:
        os.chdir(cwd)
    kern = sde_update_kernel_time(a.batch)
    print(json.dumps(dict(card=card(), batch=a.batch, alpha_type=ALPHA_TYPE, guidance=7.5, samplers=results, sde_update=kern)))


if __name__ == "__main__":
    main()
