#!/usr/bin/env python
"""Once-per-image front / back end rows on one GPU (CUDA events, after warm-up): CLIP text encoder, ConvNeXt grounding tokenizer +
grounding downsampler (the static part of a spatial model's plan), VAE decode.  Prints one JSON line per item.
    python scripts/bench_frontend.py [B]"""
import json, os, sys
import torch
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from gligen_b200 import synth
from gligen_b200.clip_text import SD14_CLIP_TEXT, ClipTextEngine, synthetic_clip_state_dict, synthetic_token_ids
from gligen_b200.engine import Engine
from gligen_b200.ops import CudaOps
from gligen_b200.spec import NAMED_CONFIGS, SPATIAL_MAP_KEY, synthetic_state_dict

dev = "cuda:0"
B = int(sys.argv[1]) if len(sys.argv) > 1 else 4
ops = CudaOps(dev)


def timed(fn, iters=10):
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record(); torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters


# CLIP text encoder: prompt + negative prompt of B images = 2B sequences
clip = ClipTextEngine(SD14_CLIP_TEXT, ops)
clip.load_state_dict(synthetic_clip_state_dict(SD14_CLIP_TEXT, 0))
ids = synthetic_token_ids(SD14_CLIP_TEXT, 2 * B, 1).to(dev)
n0 = ops.launch_count()
ms = timed(lambda: clip.forward(ids))
flops = 2 * B * 77 * 12 * (2 * 4 * 768 * 768 + 2 * 2 * 768 * 3072 + 4 * 77 * 768)
print(json.dumps({"item": "clip_text_encoder", "sequences": 2 * B, "ms": round(ms, 3), "tflops": round(flops / ms / 1e9, 1),
                  "launches_per_call": (ops.launch_count() - n0) // 13}), flush=True)

# spatial front end: static part of the plan (ConvNeXt tokenizer + downsampler + the usual text K/V, grounding K/V projections)
for name in ("sd14_hed", "sd14_sem"):
    cfg = NAMED_CONFIGS[name]
    eng = Engine(cfg, ops)
    eng.load_state_dict(synthetic_state_dict(cfg, 0))
    inp = synth.make_inputs(cfg, B, seed=3)
    key = SPATIAL_MAP_KEY[cfg.tokenizer]
    m = inp["batch"][key].to(dev)
    gr = {key: m, "mask": inp["batch"]["mask"].to(dev)}
    x, ctx, uc = inp["x"].to(dev), inp["context"].to(dev), inp["uc"].to(dev)
    ts = torch.full((B,), 500, device=dev)
    eng.forward_cfg(x, ts, ctx, uc, gr, None, m); eng.forward_cfg(x, ts, ctx, uc, gr, None, m)
    P = next(iter(eng.plans.values()))
    steps = [fn for n, fu, st, fn in P.steps if st and n.startswith(("cx.", "pn.", "ds."))]
    def front():
        for fn in steps:
            fn()
    ms = timed(front)
    def whole():
        eng.invalidate_static()
        eng.forward_cfg(x, ts, ctx, uc, gr, None, m)
    ms_all = timed(whole, iters=5)
    ms_step = timed(lambda: eng.forward_cfg(x, ts, ctx, uc, gr, None, m), iters=5)
    print(json.dumps({"item": f"{name} tokenizer+downsampler", "rows": 2 * B, "ms": round(ms, 3), "kernels": len(steps),
                      "forward_with_static_ms": round(ms_all, 3), "forward_per_step_ms": round(ms_step, 3)}), flush=True)
    del eng
    torch.cuda.empty_cache()
