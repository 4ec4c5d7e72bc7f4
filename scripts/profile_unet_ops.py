#!/usr/bin/env python
"""Per-op GPU time of one UNet pass of the benchmark workload (bench.py defaults: SD-1.4 box+text, batch 4, CFG -> 8 rows),
set against each op's roofline lower bound, with the GEMM tile the picker chose.

    python scripts/profile_unet_ops.py OUT_DIR [--config sd14_box_text] [--batch 4]

Writes OUT_DIR/profile.txt (one line per op, totals per kind and per category) and OUT_DIR/profile.json.  Op times come
from bench.kernel_pass: every op replayed from its own CUDA graph and timed with CUDA events.  Bound = max(FLOP / 989 TFLOP/s,
bytes / 3.35 TB/s): the H100 SXM data-sheet dense bf16 and HBM3 rates at 700 W, so on a power-capped card the bound is
optimistic.  Attention rows also get the SFU bound (one ex2 per score at 16 / clk / SM, at the SM clock nvidia-smi reports
after the pass), which is what limits small head dims, and are split by op (attn1 / fuser / attn2) and UNet level."""
from __future__ import annotations

import argparse
import json
import os
import re
import subprocess
import sys
from functools import partial

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import bench  # noqa: E402
from gligen_b200 import synth  # noqa: E402
from gligen_b200.spec import NAMED_CONFIGS, synthetic_state_dict  # noqa: E402

PEAK_FLOPS, PEAK_BYTES = 989e12, 3.35e12
SFU_PER_CLK = 16                                 # ex2 results / clk / SM
LEVEL_OF_C = {320: 0, 640: 1, 1280: 2}


def attention_category(name, heads, d):
    op = "attn1" if ".attn1." in name else "fuser" if ".fuser." in name else "attn2" if ".attn2." in name else "attention"
    return f"{op} L{LEVEL_OF_C.get(heads * d, '?')}"


def card_info():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        r = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True, timeout=30)
        return dict(zip(q.split(","), [v.strip() for v in r.stdout.strip().splitlines()[0].split(",")]))
    except Exception as e:                                                      # pragma: no cover
        return {"error": str(e)}


def category(name, kind, M, N, K, geglu):
    """ff1 / ff2 / qkv / C->C projections / skip / conv, with the UNet level from the channel count."""
    lvl = f"L{LEVEL_OF_C.get(N if N in LEVEL_OF_C else K, '?')}"
    if kind == "conv3x3":
        return "conv " + lvl
    if geglu:
        return "ff1 " + lvl
    if name.endswith(".ff.2"):
        return "ff2 " + lvl
    if re.search(r"\.qkv(\.objs\d+)?$", name):
        return "qkv " + lvl
    if name.endswith(".skip"):
        return "skip " + lvl
    if N == K:
        return "C->C " + lvl
    return "other gemm"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("out_dir")
    ap.add_argument("--config", default="sd14_box_text")
    ap.add_argument("--batch", type=int, default=4)
    ap.add_argument("--reps", type=int, default=8)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("profile_unet_ops.py needs a CUDA device")
    os.makedirs(a.out_dir, exist_ok=True)
    out_dir = os.path.abspath(a.out_dir)

    from ldm.models.diffusion.ldm import LatentDiffusion
    from ldm.models.diffusion.plms import PLMSSampler
    from gligen_b200.pipeline import alpha_generator, build_model, sampler_inputs, set_alpha_scale

    args = bench.parse(["--config", a.config, "--batch", str(a.batch)])
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    cfg = NAMED_CONFIGS[args.config]
    atype = [float(v) for v in args.alpha_type.split(",")]
    cfg, model = build_model(cfg, dev, load_weights=False)
    model.load_state_dict(synthetic_state_dict(cfg, seed=0))
    model.broadcast_packed_weights(src=0)
    diffusion = LatentDiffusion(linear_start=0.00085, linear_end=0.012, timesteps=1000).to(dev)
    sampler = PLMSSampler(diffusion, model, alpha_generator_func=partial(alpha_generator, type=atype), set_alpha_scale=set_alpha_scale)
    host = synth.make_inputs(cfg, a.batch, args.max_objs, seed=100)
    t = {k: v.to(dev) for k, v in host.items() if isinstance(v, torch.Tensor)}
    bt = {k: v.to(dev) for k, v in host["batch"].items()}
    torch.manual_seed(1234)
    inp, mask, x0 = sampler_inputs(cfg, model, t, bt)
    shape = (a.batch, cfg.in_channels, cfg.image_size, cfg.image_size)
    sampler.sample(S=4, shape=shape, input=inp, uc=t["uc"], guidance_scale=args.guidance, mask=mask, x0=x0)   # fills every buffer
    torch.cuda.synchronize()

    eng = model.engine()
    ops = eng.ops
    set_alpha_scale(model, 1.0 if atype[0] > 0 else 0.0)
    model._sync_scales(eng)
    # record the GEMM problem of every op in the order kernel_pass records its trace
    shapes, cur = [], {}
    orig_gemm, orig_note = ops.gemm, ops._note

    def gemm(x, w, out, **kw):
        M, No = out.numel() // out.shape[-1], out.shape[-1]
        geglu = bool(kw.get("geglu"))
        conv = kw.get("conv") is not None
        cur["s"] = (M, No * (2 if geglu else 1), x.shape[-1], 9 if conv else 1, geglu,
                    int(not geglu and kw.get("ln") is None and kw.get("stats_out") is None and out.dtype != torch.float32))
        return orig_gemm(x, w, out, **kw)

    orig_attention = ops.attention

    def attention(q, k, v, out, heads, d_head, causal=False):
        cur["s"] = (q.shape[0], heads, d_head, q.shape[1], k.shape[1])
        return orig_attention(q, k, v, out, heads, d_head, causal=causal)

    def note(kind, flops=0.0, nbytes=0.0):
        if ops.trace is not None:
            shapes.append(cur.pop("s", None))
        return orig_note(kind, flops, nbytes)

    ops.gemm, ops.attention, ops._note = gemm, attention, note
    N = bt["boxes"].shape[1]
    agg, per_op = bench.kernel_pass(model, N, t["uc"].shape[1], a.batch, reps=a.reps)
    ops.gemm, ops.attention, ops._note = orig_gemm, orig_attention, orig_note
    info = card_info()
    sms = torch.cuda.get_device_properties(dev).multi_processor_count
    sm_hz = float(info["clocks.sm"].split()[0]) * 1e6 if "clocks.sm" in info else 0.0

    lib = ops.lib
    import ctypes as C
    pick = (C.c_int32 * 3)()
    ws = ops.splitk_ws.numel() * 4
    has_pp = hasattr(lib, "glg_debug_pick_pingpong")         # libraries without the ping-pong schedule: pp = 0
    lines, rows = [], []
    cats = {}
    hdr = f"{'op':44s} {'kind':8s} {'M':>6s} {'N':>5s} {'K':>5s} tap {'BN':>3s} pair res spl pp {'ms':>8s} {'TFLOP/s':>8s} {'GB/s':>7s} {'bound ms':>8s} by  {'x bound':>7s}"
    lines.append(hdr)
    for (name, kind, fl, by, ms), sh in zip(per_op, shapes):
        bound_f, bound_b = fl / PEAK_FLOPS * 1e3, by / PEAK_BYTES * 1e3
        bound = max(bound_f, bound_b)
        by_what = "F" if bound_f >= bound_b else "B"
        rec = dict(name=name, kind=kind, flops=fl, bytes=by, ms=ms, bound_ms=bound, bound_by=by_what)
        tile = ""
        if kind in ("gemm", "conv3x3") and sh is not None:
            M, Nn, K, taps, geglu, can_split = sh
            lib.glg_debug_pick_tile(M, Nn, K, int(geglu), int(taps == 9), can_split, ws, pick)
            pp = lib.glg_debug_pick_pingpong(M, Nn, K, int(geglu), int(taps == 9), can_split, ws) if has_pp else 0
            rec.update(M=M, N=Nn, K=K, taps=taps, geglu=geglu, bn=pick[0], pair=pick[1] & 255, resident=pick[1] >> 8, splits=pick[2], pp=pp)
            cat = category(name, kind, M, Nn, K, geglu)
            tile = f"{M:6d} {Nn:5d} {K:5d} {taps:3d} {pick[0]:3d} {pick[1] & 255:4d} {pick[1] >> 8:3d} {pick[2]:3d} {pp:2d}"
        elif kind == "attention" and sh is not None:
            B, heads, d, Lq, Lk = sh
            sfu = B * heads * Lq * Lk / (SFU_PER_CLK * sms * sm_hz) * 1e3 if sm_hz else 0.0
            if sfu > bound:
                bound, by_what = sfu, "S"
            rec.update(B=B, heads=heads, d=d, Lq=Lq, Lk=Lk, sfu_bound_ms=sfu, bound_ms=bound, bound_by=by_what)
            cat = attention_category(name, heads, d)
            tile = f"B{B} h{heads} d{d} {Lq}x{Lk}".ljust(47)
        else:
            cat = kind
            tile = " " * 47
        rec["category"] = cat
        c = cats.setdefault(cat, [0.0, 0.0, 0.0, 0.0, 0])
        c[0] += fl; c[1] += by; c[2] += ms; c[3] += bound; c[4] += 1
        rows.append(rec)
        tf = fl / (ms * 1e-3) / 1e12 if ms > 0 else 0.0
        gb = by / (ms * 1e-3) / 1e9 if ms > 0 else 0.0
        lines.append(f"{name[:44]:44s} {kind[:8]:8s} {tile} {ms:8.4f} {tf:8.1f} {gb:7.0f} {bound:8.4f} {by_what:2s} {ms / bound if bound else 0:7.2f}")

    def total_lines(title, d):
        out = ["", title, f"{'':22s} {'n':>4s} {'ms':>8s} {'TFLOP':>7s} {'GB':>6s} {'TFLOP/s':>8s} {'bound ms':>8s} {'x bound':>7s}"]
        for k, (fl, by, ms, bound, n) in sorted(d.items(), key=lambda kv: -kv[1][2]):
            out.append(f"{k:22s} {n:4d} {ms:8.3f} {fl / 1e12:7.3f} {by / 1e9:6.2f} {fl / (ms * 1e-3) / 1e12 if ms else 0:8.1f} {bound:8.3f} {ms / bound if bound else 0:7.2f}")
        return out

    kinds = {}
    for r in rows:
        k = kinds.setdefault(r["kind"], [0.0, 0.0, 0.0, 0.0, 0])
        k[0] += r["flops"]; k[1] += r["bytes"]; k[2] += r["ms"]; k[3] += r["bound_ms"]; k[4] += 1
    lines += total_lines("per kind", kinds)
    lines += total_lines("per category", cats)
    total = sum(r["ms"] for r in rows)
    lines.append("")
    lines.append(f"sum of per-op GPU times of one {2 * a.batch}-row pass: {total:.3f} ms")
    lines.append(f"card: {info}")
    text = "\n".join(lines)
    print(text)
    with open(os.path.join(out_dir, "profile.txt"), "w") as f:
        f.write(text + "\n")
    with open(os.path.join(out_dir, "profile.json"), "w") as f:
        json.dump({"card": info, "ops": rows, "total_ms": total}, f, indent=1)


if __name__ == "__main__":
    main()
