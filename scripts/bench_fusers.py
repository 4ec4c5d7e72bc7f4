"""Cost of the gatedCA / gatedSA2 fusers on one GPU.

    python scripts/bench_fusers.py [--steps 2] [--warmup 1] [--no-e2e]

1. glg_grid_resample_gate alone, CUDA events over 200 launches, at the 8-row shapes of the SD-1.4 gatedSA2 model's levels 0-2
   (8 x 8 grounding tokens onto 64 x 64 / 32 x 32 / 16 x 16 pixels at 320 / 640 / 1280 channels), against its HBM bound: the
   bytes of x read and written plus the statistics, over 3.35 TB/s (H100 SXM data sheet).
2. PLMS-50, CFG 7.5, batch 4, 512 x 512 images/s of sd14_box_text with gatedSA vs gatedCA and of sd14_hed with gatedSA vs
   gatedSA2, each through bench.py in its own process.
The card's name and power limit are printed with the numbers.
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
HBM_BYTES_PER_S = 3.35e12


def card():
    name = torch.cuda.get_device_name(0)
    try:
        pl = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                            text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception as e:  # noqa: BLE001 - reported, not fatal
        pl = f"unknown ({e})"
    return f"{name}, power limit / max SM clock: {pl}"


def kernel_times(reps=200):
    from gligen_b200.ops import CudaOps
    ops = CudaOps("cuda:0")
    out = []
    for level, (n, C) in enumerate(((64, 320), (32, 640), (16, 1280))):
        B, g = 8, 8
        rows = B * n * n
        grid = torch.randn(B, g * g, C, device="cuda:0")
        x = torch.randn(B, n * n, C, device="cuda:0").to(torch.bfloat16)
        stats = torch.empty(C // 32, rows, 2, device="cuda:0")
        gate = torch.full((1,), 1e-3, device="cuda:0")
        for _ in range(20):
            ops.grid_resample_gate(grid, x, gate, stats, g, n)
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(reps):
            ops.grid_resample_gate(grid, x, gate, stats, g, n)
        e1.record()
        torch.cuda.synchronize()
        us = e0.elapsed_time(e1) * 1e3 / reps
        nbytes = 2 * rows * C * 2 + rows * (C // 32) * 8
        bound_us = nbytes / HBM_BYTES_PER_S * 1e6
        out.append(dict(level=level, n=n, C=C, rows=rows, us=us, mb=nbytes / 1e6, bound_us=bound_us, ratio=us / bound_us))
        print(f"grid_resample_gate level {level}: 8 x {n}x{n} x {C}: {us:.2f} us, {nbytes / 1e6:.1f} MB -> {nbytes / us / 1e3:.0f} GB/s; "
              f"HBM bound {bound_us:.2f} us, {us / bound_us:.2f}x the bound", flush=True)
    return out


def images_per_s(config, steps, warmup):
    cmd = [sys.executable, os.path.join(ROOT, "bench.py"), "--gpus", "1", "--config", config, "--batch", "4", "--plms-steps", "50",
           "--guidance", "7.5", "--steps", str(steps), "--warmup", str(warmup), "--no-cpu-baseline", "--no-kernel-pass"]
    res = subprocess.run(cmd, capture_output=True, text=True, cwd=ROOT)
    lines = [ln for ln in res.stdout.splitlines() if ln.startswith("{")]
    if res.returncode != 0 or not lines:
        print(f"{config}: bench.py failed (rc {res.returncode}):\n{res.stdout[-2000:]}\n{res.stderr[-3000:]}", flush=True)
        return None
    r = json.loads(lines[-1])
    print(f"{config}: {json.dumps(r)}", flush=True)
    return r


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=2)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--no-e2e", action="store_true")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_fusers: needs a CUDA device (nothing is measured without one)")
    print(card(), flush=True)
    kernel_times()
    if not a.no_e2e:
        for cfg in ("sd14_box_text", "sd14_box_text_gated_ca", "sd14_hed", "sd14_hed_gated_sa2"):
            images_per_s(cfg, a.steps, a.warmup)
    print(card(), flush=True)


if __name__ == "__main__":
    main()
