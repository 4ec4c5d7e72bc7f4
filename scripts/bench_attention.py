#!/usr/bin/env python
"""CUDA-event timings of glg_attention at every call shape of one UNet pass of the benchmark workload (SD-1.4 box+text,
batch 4, CFG -> 8 rows), one shape at a time, set against the two bounds of the long-key kernel.

    python scripts/bench_attention.py OUT_DIR [--rows 8] [--reps 20]

Shapes: per UNet level (0: 64 x 64 tokens, d 40; 1: 32 x 32, d 80; 2: 16 x 16, d 160; mid: 8 x 8, d 160; 8 heads)
self-attention (q, k, v strided views of one [rows, T, 3C] buffer), the fuser (queries are the T visual rows, keys
T + 30 grounding tokens) and cross-attention (77 text tokens); plus the CLIP ViT-L/14 image tower (16 heads, d 64, 257 x 257
tokens, 8 images).  Every shape is captured `reps` times into a CUDA graph, warmed up, and the replay timed with CUDA events.

Bounds, from shapes and per-clock data-sheet rates at the SM clock nvidia-smi reports right after the shape ran:
  SFU: one ex2 per score at 16 / clk / SM;
  MMA: 4 DPAD FLOP per score (QK^T and PV at the head dim padded to a multiple of 16) at 4096 dense bf16 FLOP / clk / SM.
Writes OUT_DIR/attention.txt and OUT_DIR/attention.json."""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

SFU_PER_CLK, MMA_FLOP_PER_CLK = 16, 4096          # per SM, sm_90
UNET_LEVELS = [("L0", 4096, 320), ("L1", 1024, 640), ("L2", 256, 1280), ("mid", 64, 1280)]   # (name, tokens, channels)
HEADS, N_GROUNDING, N_TEXT = 8, 30, 77


def shapes(rows):
    """(name, B, heads, d, Lq, Lk, kind): kind 'self' / 'fuser' / 'cross' selects how q, k, v are laid out."""
    out = []
    for lvl, T, C in UNET_LEVELS:
        d = C // HEADS
        out.append((f"{lvl} attn1", rows, HEADS, d, T, T, "self"))
        out.append((f"{lvl} fuser", rows, HEADS, d, T, T + N_GROUNDING, "fuser"))
        out.append((f"{lvl} attn2", rows, HEADS, d, T, N_TEXT, "cross"))
    out.append(("clip_vit_l14", 8, 16, 64, 257, 257, "self"))
    return out


def make_inputs(B, heads, d, Lq, Lk, kind, seed):
    """q, k, v views laid out as the engine passes them, from a seeded generator; out [B, Lq, heads d]."""
    g = torch.Generator(device="cpu").manual_seed(seed)
    C = heads * d
    if kind == "cross":
        q = torch.randn(B, Lq, C, generator=g)
        kv = torch.randn(B, Lk, 2 * C, generator=g)
        q, kv = q.cuda().bfloat16(), kv.cuda().bfloat16()
        return q, kv[:, :, :C], kv[:, :, C:]
    qkv = torch.randn(B, Lk, 3 * C, generator=g).cuda().bfloat16()   # fuser: [visual ; grounding] rows, queries are visual
    return qkv[:, :Lq, :C], qkv[:, :, C:2 * C], qkv[:, :, 2 * C:]


def card_info():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    r = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader,nounits"], capture_output=True, text=True, timeout=30)
    vals = [v.strip() for v in r.stdout.strip().splitlines()[0].split(",")]
    return dict(zip(q.split(","), vals))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("out_dir")
    ap.add_argument("--rows", type=int, default=8)
    ap.add_argument("--reps", type=int, default=20)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_attention.py needs a CUDA device")
    os.makedirs(a.out_dir, exist_ok=True)
    from gligen_b200.ops import CudaOps
    ops = CudaOps("cuda:0")
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    recs = []
    for i, (name, B, heads, d, Lq, Lk, kind) in enumerate(shapes(a.rows)):
        q, k, v = make_inputs(B, heads, d, Lq, Lk, kind, seed=i)
        out = torch.empty(B, Lq, heads * d, device="cuda", dtype=torch.bfloat16)
        ops.attention(q, k, v, out, heads, d)                    # first launch: module load, attributes
        torch.cuda.synchronize()
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            for _ in range(a.reps):
                ops.attention(q, k, v, out, heads, d)
        for _ in range(3):
            g.replay()
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        ms = []
        for _ in range(5):
            e0.record()
            g.replay()
            e1.record()
            torch.cuda.synchronize()
            ms.append(e0.elapsed_time(e1) / a.reps)
        info = card_info()
        del g
        ms_med = sorted(ms)[len(ms) // 2]
        clk = float(info["clocks.sm"]) * 1e6
        scores = B * heads * Lq * Lk
        dpad = (d + 15) // 16 * 16
        sfu_ms = scores / (SFU_PER_CLK * sms * clk) * 1e3
        mma_ms = 4.0 * dpad * scores / (MMA_FLOP_PER_CLK * sms * clk) * 1e3
        recs.append(dict(name=name, B=B, heads=heads, d=d, Lq=Lq, Lk=Lk, ms=ms_med, ms_min=min(ms), ms_max=max(ms),
                         scores_per_s=scores / (ms_med * 1e-3), sm_clock_mhz=clk / 1e6, sfu_bound_ms=sfu_ms,
                         mma_bound_ms=mma_ms, x_sfu=ms_med / sfu_ms, x_mma=ms_med / mma_ms))
    info = card_info()
    lines = [f"{'shape':14s} {'B':>2s} {'h':>2s} {'d':>3s} {'Lq':>5s} {'Lk':>5s} {'ms':>8s} {'Gscore/s':>9s} {'MHz':>5s} "
             f"{'SFU ms':>7s} {'x SFU':>6s} {'MMA ms':>7s} {'x MMA':>6s}"]
    for r in recs:
        lines.append(f"{r['name']:14s} {r['B']:2d} {r['heads']:2d} {r['d']:3d} {r['Lq']:5d} {r['Lk']:5d} {r['ms']:8.4f} "
                     f"{r['scores_per_s'] / 1e9:9.1f} {r['sm_clock_mhz']:5.0f} {r['sfu_bound_ms']:7.4f} {r['x_sfu']:6.2f} "
                     f"{r['mma_bound_ms']:7.4f} {r['x_mma']:6.2f}")
    lines.append(f"card: {info}, {sms} SMs")
    text = "\n".join(lines)
    print(text)
    with open(os.path.join(a.out_dir, "attention.txt"), "w") as f:
        f.write(text + "\n")
    with open(os.path.join(a.out_dir, "attention.json"), "w") as f:
        json.dump({"card": info, "sms": sms, "shapes": recs}, f, indent=1)


if __name__ == "__main__":
    main()
