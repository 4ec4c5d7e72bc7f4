#!/usr/bin/env python
"""Forced-tile sweep over the GEMM / conv shapes of the SD-1.4 GLIGEN forward (2B = 8): auto heuristic vs BN in {64,128,160,256},
each on the cooperative (co) and, where legal, the ping-pong (pp) consumer schedule.  Times in microseconds (CUDA events)."""
import os, sys
import torch
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from gligen_b200.ops import CudaOps
dev = "cuda:0"; ops = CudaOps(dev)
has_pp = hasattr(ops.lib, "glg_debug_gemm_pp")
def rnd(*shape, scale=1.0): return (torch.randn(*shape, device=dev) * scale).to(torch.bfloat16)
def timeit(fn, iters=20):
    for _ in range(3): fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters): fn()
    e1.record(); torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters * 1e3
Bt = 8
shapes = []
for (T, C) in ((4096, 320), (1024, 640), (256, 1280), (64, 1280)):
    M = Bt * T
    shapes += [("qkv", M, 3 * C, C, None), ("out/proj", M, C, C, None), ("ff1 geglu", M, 8 * C, C, "geglu"), ("ff2", M, C, 4 * C, None),
               ("kv ctx", Bt * 77, 2 * C, 768, None)]
for (H, Cin, Cout) in ((64, 320, 320), (64, 960, 320), (64, 640, 320), (32, 640, 640), (32, 1920, 640), (32, 1280, 640), (32, 960, 640), (16, 1280, 1280), (16, 2560, 1280), (16, 1920, 1280), (8, 1280, 1280), (8, 2560, 1280)):
    shapes.append(("conv", Bt * H * H, Cout, Cin, H))
for (H, Cin, Cout) in ((64, 960, 320), (32, 1920, 640), (16, 2560, 1280), (8, 2560, 1280)):
    shapes.append(("skip1x1", Bt * H * H, Cout, Cin, None))
for name, M, N, K, H in shapes:
    geglu = H == "geglu"
    conv = isinstance(H, int)
    a = rnd(Bt, H * H, K) if conv else rnd(M, K)
    w = rnd((9 if conv else 1) * N, K, scale=K ** -0.5)
    No = N // 2 if geglu else N
    o = torch.empty(Bt, H * H, N, device=dev, dtype=torch.bfloat16) if conv else torch.empty(M, No, device=dev, dtype=torch.bfloat16)
    bias = torch.randn(N, device=dev)
    kw = dict(bias=bias, conv=(Bt, H, H)) if conv else dict(bias=bias, geglu=geglu)
    res = {}
    for bn in (0, 64, 128, 160, 256):
        if bn and (N % bn or (geglu and bn != 256)): continue
        for pp in ((1, 2) if has_pp else (0,)):
            if has_pp: ops.lib.glg_debug_gemm_pp(pp)
            ops.lib.glg_debug_force_bn(bn)
            res[(bn, pp)] = timeit(lambda: ops.gemm(a, w, o, **kw))
    ops.lib.glg_debug_force_bn(0)
    if has_pp:
        ops.lib.glg_debug_gemm_pp(0)
        res[("auto", 0)] = timeit(lambda: ops.gemm(a, w, o, **kw))
    auto = res[("auto", 0)] if has_pp else res[(0, 0)]
    best = min(v for k, v in res.items() if k[0] not in (0, "auto"))
    tag = {0: "", 1: "co", 2: "pp"}
    print(f"{name:9s} M={M:6d} N={N:5d} K={K:5d}{' 3x3' if conv else '    '} auto {auto:7.1f} us | " +
          " ".join(f"bn{k[0]}{tag[k[1]]}={v:7.1f}" for k, v in res.items() if k[0] != "auto") + f" | auto/best {auto / best:.2f}", flush=True)
