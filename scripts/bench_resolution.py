#!/usr/bin/env python
"""Throughput at other resolutions and aspect ratios: PLMS-50, CFG 7.5, SD-1.4 box+text with 30 grounding slots, batch 4,
at 512 x 512, 512 x 768, 768 x 512 and 768 x 768 -> images/s and megapixels/s; VAE decode ms/image at each size; and the
3x3-convolution TFLOP/s per UNet level from per-op CUDA-graph replay (as scripts/profile_unet_ops.py).  Prints the card
name and power limit of the run, then one JSON line per size.

    python scripts/bench_resolution.py [--runs 2] [--sizes 512x512,512x768,768x512,768x768]
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import time
from functools import partial

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from gligen_b200 import synth  # noqa: E402
from gligen_b200.spec import NAMED_CONFIGS, NAMED_VAE_CONFIGS, synthetic_vae_state_dict  # noqa: E402

DEV = "cuda:0"


def card():
    q = "name,power.limit,clocks.max.sm"
    r = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True, timeout=30)
    return dict(zip(q.split(","), [v.strip() for v in r.stdout.strip().splitlines()[0].split(",")]))


def conv_levels(eng, rows, N, n_ctx, H, W, reps=4):
    """{level: (FLOP, ms, calls)} of the plan's 3x3 convolutions (level = log2 of latent side / conv side), each op timed
    from its own CUDA graph."""
    ops = eng.ops
    P = eng._plan(rows, N, n_ctx, H=H, W=W)
    steps = [fn for _, fu, st, fn in P.steps if not st]
    inner, convs = ops.gemm, []

    def spy(a, w, out, **kw):
        cv = kw.get("conv")
        convs.append(None if cv is None else (cv, 2.0 * cv[0] * cv[1] * cv[2] * w.shape[0] * w.shape[1]))      # w: [9 N, K]
        return inner(a, w, out, **kw)

    ops.gemm = spy
    try:
        owner = []
        for fn in steps:                                    # eager pass: which step launched which conv
            n0 = len(convs)
            fn()
            owner.append(convs[n0:])
    finally:
        ops.gemm = inner
    torch.cuda.synchronize()
    lv = {}
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    for fn, cv in zip(steps, owner):
        if len(cv) != 1 or cv[0] is None:
            continue
        (_, ch, _), flop = cv[0]
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            for _ in range(reps):
                fn()
        g.replay()
        torch.cuda.synchronize()
        e0.record(); g.replay(); e1.record()
        torch.cuda.synchronize()
        ms = e0.elapsed_time(e1) / reps
        del g
        a = lv.setdefault((H // ch).bit_length() - 1, [0.0, 0.0, 0])
        a[0] += flop; a[1] += ms; a[2] += 1
    return lv


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=2)
    ap.add_argument("--batch", type=int, default=4)
    ap.add_argument("--sizes", default="512x512,512x768,768x512,768x768")
    args = ap.parse_args()
    from ldm.models.diffusion.ldm import LatentDiffusion
    from ldm.models.diffusion.plms import PLMSSampler
    from gligen_b200.ops import CudaOps
    from gligen_b200.pipeline import alpha_generator, build_model, sampler_inputs, set_alpha_scale
    from gligen_b200.vae import VAEDecoderEngine

    print(json.dumps({"card": card()}), flush=True)
    cfg, model = build_model(NAMED_CONFIGS["sd14_box_text"], DEV)
    diffusion = LatentDiffusion(linear_start=0.00085, linear_end=0.012, timesteps=1000).to(DEV)
    sampler = PLMSSampler(diffusion, model, alpha_generator_func=partial(alpha_generator, type=[1.0, 0.0, 0.0]), set_alpha_scale=set_alpha_scale)
    vcfg = NAMED_VAE_CONFIGS["sd14_vae"]
    vae = VAEDecoderEngine(vcfg, CudaOps(DEV))
    vae.load_state_dict(synthetic_vae_state_dict(vcfg, 0))
    B = args.batch
    inp = synth.make_inputs(cfg, B, 30, seed=100)
    t = {k: v.to(DEV) for k, v in inp.items() if isinstance(v, torch.Tensor)}
    bt = {k: v.to(DEV) for k, v in inp["batch"].items()}
    for size in args.sizes.split(","):
        ih, iw = (int(v) for v in size.split("x"))
        h, w = ih // 8, iw // 8
        shape = (B, cfg.in_channels, h, w)

        def sample():
            torch.manual_seed(1234)
            input, mask, x0 = sampler_inputs(cfg, model, t, bt)
            input["x"] = None                               # x_T drawn by the sampler at `shape`
            return sampler.sample(S=50, shape=shape, input=input, uc=t["uc"], guidance_scale=7.5, mask=mask, x0=x0)

        lat = sample()                                      # warm-up: plans, graphs, tensor maps
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for _ in range(args.runs):
            lat = sample()
        torch.cuda.synchronize()
        dt = (time.perf_counter() - t0) / args.runs
        z = lat[:1].contiguous()
        vae.decode(z)
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(3):
            vae.decode(z)
        e1.record()
        torch.cuda.synchronize()
        vae_ms = e0.elapsed_time(e1) / 3
        eng = model.engine()
        per = conv_levels(eng, 2 * B, 30, t["context"].shape[1], h, w)
        print(json.dumps({"size": f"{ih}x{iw}", "latent": [h, w], "batch": B, "images_per_s": round(B / dt, 3),
                          "megapixels_per_s": round(B * ih * iw / dt / 1e6, 3), "vae_decode_ms_per_image": round(vae_ms, 2),
                          "conv3x3_tflops_per_level": {f"L{k}": round(f / ms / 1e9, 1) for k, (f, ms, n) in sorted(per.items())},
                          "conv3x3_ms_per_level": {f"L{k}": round(ms, 3) for k, (f, ms, n) in sorted(per.items())}}), flush=True)


if __name__ == "__main__":
    main()
