"""Images/s of the samplers on one GPU: PLMS-50 against DPM-Solver++ 2M at 20 and 25 steps, and UniPC-2 at 10 and 15 steps
against DPM-Solver++ 2M at 10 (the same number of passes); and on the Karras sigma grid (grid="karras"): 2M at 10 / 15 / 20 steps,
UniPC-2 at 10 / 15 and 2M SDE (eta = 1) at 20.

    python scripts/bench_samplers.py [--repeats 2] [--batch 4]

Workload: sd14_box_text (seeded synthetic weights), batch 4, 64 x 64 latent (512 x 512 images), 30 grounding objects, CFG 7.5,
alpha_type [0.3, 0, 0.7] (gligen_inference's default: the fusers are on for the first 30 % of the steps, then SD's first conv).
1. Every sampler once untimed, then the samplers alternately, `--repeats` times each: wall time of sample() between device
   synchronisations -> images/s, and the UNet passes per image (one CFG-batched pass evaluates cond and uncond).
2. glg_dpm_update alone, CUDA events around a CUDA graph of 200 launches at the batch's latent (4 x 4 x 64 x 64, CFG, order 2), against its HBM
   bound: x, e_c, e_u, m1 read and x0_out, x_prev written, over 3.35 TB/s (H100 SXM data sheet).  Likewise glg_unipc_update
   (order 3, a step that reads all three earlier data predictions): x, xc_prev, e_c, e_u, m1, m2, m3 read and m_out, xc_out,
   x_next written.  The UniPC rows must take exactly one UNet pass per image and step of the DDIM uniform grid (S of them, but
   16 at S = 15: the grid's spacing is 1000 // S); the Karras rows exactly S.  The script stops if one does not.
3. A diagnostic, not a quality measure: the rel-L2 distance of each sampler's final latent from a DPM-Solver++ 3M run at 250
   steps on the same seeded inputs, on the sampler's own grid.  The DDIM-grid run is not a converged solution (the grid's last
   step, t = 1 -> alphas_cumprod[0], has the same size at every S); the Karras one shrinks every step.  With synthetic weights the
   distance says how the solvers differ, not how the images look, and the SDE row's distance includes its own noise.
Every run reloads the weights first (untimed), so each starts from the GLIGEN first conv like a fresh model.  The card's name and
power limit are printed with the numbers.
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
from bench_fusers import HBM_BYTES_PER_S, card  # noqa: E402

DEV = "cuda:0"
ALPHA_TYPE = [0.3, 0.0, 0.7]
# (name, sampler, S, order, grid, eta); the Karras arms alternate with the DDIM-grid ones
RUNS = [("PLMS-50", "plms", 50, None, "ddim", 0.0), ("DPM-Solver++ 2M Karras-10", "dpm", 10, 2, "karras", 0.0),
        ("DPM-Solver++ 2M-20", "dpm", 20, 2, "ddim", 0.0), ("DPM-Solver++ 2M Karras-15", "dpm", 15, 2, "karras", 0.0),
        ("DPM-Solver++ 2M-25", "dpm", 25, 2, "ddim", 0.0), ("DPM-Solver++ 2M Karras-20", "dpm", 20, 2, "karras", 0.0),
        ("UniPC-2 10", "unipc", 10, 2, "ddim", 0.0), ("UniPC-2 Karras-10", "unipc", 10, 2, "karras", 0.0),
        ("UniPC-2 15", "unipc", 15, 2, "ddim", 0.0), ("UniPC-2 Karras-15", "unipc", 15, 2, "karras", 0.0),
        ("DPM-Solver++ 2M-10", "dpm", 10, 2, "ddim", 0.0), ("DPM-Solver++ 2M SDE Karras-20", "dpm", 20, 2, "karras", 1.0)]
REFERENCE_RUNS = {"ddim": ("DPM-Solver++ 3M-250", "dpm", 250, 3, "ddim", 0.0),
                  "karras": ("DPM-Solver++ 3M Karras-250", "dpm", 250, 3, "karras", 0.0)}


def _graph_time(name, batch, launch, nbytes, reps=200):
    """CUDA events around a CUDA graph of `reps` launch() calls -> us per launch, against the HBM bound of nbytes."""
    # the launches are captured in a CUDA graph: issued one by one from Python, the ctypes call takes longer than the kernel and
    # the events would time the host
    stream = torch.cuda.Stream()
    with torch.cuda.stream(stream):
        for _ in range(20):
            launch()
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph, stream=stream):
            for _ in range(reps):
                launch()
    graph.replay()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    graph.replay()
    e1.record()
    torch.cuda.synchronize()
    us = e0.elapsed_time(e1) * 1e3 / reps
    bound_us = nbytes / HBM_BYTES_PER_S * 1e6
    print(f"{name} {batch} x 4 x 64 x 64: {us:.2f} us, {nbytes / 1e6:.2f} MB -> {nbytes / us / 1e3:.0f} GB/s; "
          f"HBM bound {bound_us:.2f} us, {us / bound_us:.2f}x the bound", flush=True)
    return dict(us=us, bound_us=bound_us, mb=nbytes / 1e6)


def _step20_grid():
    from ldm.models.diffusion import dpm_solver as DS
    import numpy as np
    from oracle import sampler_oracle as SO
    return DS.grid_alpha_sigma(SO.make_schedule()["alphas_cumprod"], np.flip(SO.ddim_timesteps(20)))


def update_kernel_time(batch):
    from gligen_b200.ops import CudaOps
    from ldm.models.diffusion import dpm_solver as DS
    ops = CudaOps(DEV)
    x, ec, eu, m1 = (torch.randn(batch, 4, 64, 64, device=DEV) for _ in range(4))
    m0, xp = torch.empty_like(x), torch.empty_like(x)
    alpha, sigma = _step20_grid()
    coefs = DS.step_coefficients(alpha, sigma, DS.step_orders(len(alpha) - 1, 2))[5]
    return _graph_time("glg_dpm_update", batch, lambda: ops.dpm_update(x, ec, eu, 7.5, m1, None, alpha[5], sigma[5], coefs, m0, xp),
                       6 * x.numel() * 4)


def unipc_update_kernel_time(batch):
    from gligen_b200.ops import CudaOps
    from ldm.models.diffusion import dpm_solver as DS
    from ldm.models.diffusion import unipc as UP
    ops = CudaOps(DEV)
    x, xcp, ec, eu, m1, m2, m3 = (torch.randn(batch, 4, 64, 64, device=DEV) for _ in range(7))
    m0, xc, xn = torch.empty_like(x), torch.empty_like(x), torch.empty_like(x)
    alpha, sigma = _step20_grid()
    coefs = UP.step_coefficients(alpha, sigma, DS.step_orders(len(alpha) - 1, 3))[5]
    return _graph_time("glg_unipc_update", batch,
                       lambda: ops.unipc_update(x, xcp, ec, eu, 7.5, m1, m2, m3, alpha[5], sigma[5], coefs, m0, xc, xn),
                       10 * x.numel() * 4)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=2)
    ap.add_argument("--batch", type=int, default=4)
    ap.add_argument("--no-reference-run", action="store_true", help="skip the 3M-250 diagnostic")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_samplers.py measures on a CUDA device; none is available")
    from gligen_b200 import synth
    from gligen_b200.pipeline import alpha_generator, build_model, sampler_inputs, set_alpha_scale, to_device
    from ldm.models.diffusion.dpm_solver import DPMSolverSampler
    from ldm.models.diffusion.ldm import LatentDiffusion
    from ldm.models.diffusion.plms import PLMSSampler
    from ldm.models.diffusion.unipc import UniPCSampler
    from ldm.modules.diffusionmodules.util import make_ddim_timesteps

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

    def run(kind, S, order, grid, eta):
        model.load_state_dict(weights)
        model.engine()                                  # re-pack the weights outside the timed window
        if kind == "plms":
            sampler = PLMSSampler(diffusion, model, **kw)
        elif kind == "dpm":
            sampler = DPMSolverSampler(diffusion, model, order=order, eta=eta, grid=grid, **kw)
        else:
            sampler = UniPCSampler(diffusion, model, order=order, grid=grid, **kw)
        input, _, _ = sampler_inputs(cfg, model, dinp, dbatch)
        passes["n"] = 0
        torch.manual_seed(1234)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        lat = sampler.sample(S=S, shape=tuple(dinp["x"].shape), input=input, uc=dinp["uc"], guidance_scale=7.5)
        torch.cuda.synchronize()
        return time.perf_counter() - t0, passes["n"], lat

    cwd = os.getcwd()
    os.chdir(os.path.join(ROOT, "tests", "golden"))     # restore_first_conv_from_SD reads SD_input_conv_weight_bias.pth CWD-relative
    try:
        latents, times, npass = {}, {name: [] for name, *_ in RUNS}, {}
        for name, kind, S, order, grid, eta in RUNS:    # warm-up: every shape and schedule once
            _, npass[name], latents[name] = run(kind, S, order, grid, eta)
            steps = S if grid == "karras" else len(make_ddim_timesteps("uniform", S, 1000, verbose=False))
            if (kind == "unipc" or grid == "karras") and npass[name] != steps:
                raise SystemExit(f"{name}: {npass[name]} UNet passes per image, expected one per step of the grid ({steps})")
        for _ in range(a.repeats):
            for name, kind, S, order, grid, eta in RUNS:
                secs, n, lat = run(kind, S, order, grid, eta)
                times[name].append(secs)
                if n != npass[name] or not torch.equal(lat, latents[name]):
                    print(f"{name}: a repeat run differs from the first ({n} passes)", flush=True)
        results = {}
        for name, *_ in RUNS:
            ips = [a.batch / t for t in times[name]]
            results[name] = dict(images_per_s=max(ips), images_per_s_runs=ips, unet_passes_per_image=npass[name])
            print(f"{name}: {', '.join(f'{v:.3f}' for v in ips)} images/s (batch {a.batch}), {npass[name]} UNet passes per image",
                  flush=True)
        base = results["PLMS-50"]["images_per_s"]
        for name in results:
            results[name]["speedup_vs_plms50"] = results[name]["images_per_s"] / base
        if not a.no_reference_run:
            for grid, (name, *ref_run) in REFERENCE_RUNS.items():
                _, n, ref = run(*ref_run)
                for k, *_, g, _eta in RUNS:
                    if g != grid:
                        continue
                    results[k]["rel_l2_vs_3m250"] = ((latents[k] - ref).norm() / ref.norm()).item()
                    print(f"{k}: rel-L2 of the final latent from {name} = {results[k]['rel_l2_vs_3m250']:.3e} "
                          "(solver diagnostic on synthetic weights, not an image-quality measure)", flush=True)
    finally:
        os.chdir(cwd)
    kern = update_kernel_time(a.batch)
    ukern = unipc_update_kernel_time(a.batch)
    print(json.dumps(dict(card=card(), batch=a.batch, alpha_type=ALPHA_TYPE, guidance=7.5, samplers=results, dpm_update=kern,
                          unipc_update=ukern)))


if __name__ == "__main__":
    main()
