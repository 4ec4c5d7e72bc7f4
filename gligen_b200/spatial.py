"""Spatial grounding modalities (hed / canny / depth / normal / sem; SURVEY 8f-4) on this repo's kernels.

Two timestep-invariant pieces sit in front of the denoiser for these models (openaimodel.py:293-297, 436-443):
  * the grounding tokenizer `PositionNet` = ConvNeXt-tiny over the conditioning map resampled to `resize_input`, one token per
    32 x 32 patch, mask / null-feature replacement, learned position embedding, 3-layer MLP
    ({hed,canny,depth,normal,sem}_grounding_net.py:38-63, convnext.py:38-110), and
  * the `GroundingDownsampler` whose output planes join the latent in front of the first conv
    ({hed,...}_grounding_downsampler.py).
Both are emitted here as STATIC steps of the engine's plan (run once per sample, cached across the sampling loop).
Layout: channels-last bf16 rows like the UNet; the 96-channel stage lives in 128-column rows whose last 32 columns are
zero (glg_gemm wants K, N % 64 == 0; zero weight rows / columns keep the padding exactly zero through the residual adds).
Every dense layer is a glg_gemm: the stem (4 x 4 / 4) and downsample (2 x 2 / 2) convolutions over patch rows (glg_patchify_*),
pwconv1 with the exact-GELU epilogue, pwconv2 with the layer scale gamma folded into its weights and the residual add in its
epilogue; depthwise 7 x 7 + LayerNorm is one kernel (glg_dwconv7_ln).
"""
from __future__ import annotations

from typing import Dict

import torch

from .ops import ACT_GELU, ACT_SILU, round_up
from .spec import CONVNEXT_TINY_DEPTHS as DEPTHS, CONVNEXT_TINY_DIMS as DIMS

_PN, _CX = "position_net", "position_net.convnext_tiny_backbone"


def _pad2(w: torch.Tensor, rows: int, cols: int) -> torch.Tensor:
    out = torch.zeros(rows, cols, dtype=w.dtype)
    out[: w.shape[0], : w.shape[1]] = w
    return out


def _pad1(v: torch.Tensor, n: int) -> torch.Tensor:
    out = torch.zeros(n, dtype=v.dtype)
    out[: v.shape[0]] = v
    return out


def pack(engine, sd: Dict[str, torch.Tensor]) -> None:
    """ConvNeXt / PositionNet MLP / downsampler weights into the engine's packed table (keys "cx.*", "pn.*", "ds.*")."""
    cfg, W, a, f = engine.cfg, engine.W, engine._a, engine._f
    cp = [round_up(c, 64) for c in DIMS]                  # 128, 192, 384, 768
    d = f"{_CX}.downsample_layers"
    w = sd[f"{d}.0.0.weight"].float()                     # [96, 3, 4, 4] -> [Cout, (ky, kx, c)]
    W["cx.stem.w"] = a(_pad2(w.permute(0, 2, 3, 1).reshape(DIMS[0], -1), cp[0], 64))
    W["cx.stem.b"] = f(_pad1(sd[f"{d}.0.0.bias"].float(), cp[0]))
    W["cx.stem.g"], W["cx.stem.beta"] = f(sd[f"{d}.0.1.weight"]), f(sd[f"{d}.0.1.bias"])
    for i in range(1, 4):
        W[f"cx.down{i}.g"], W[f"cx.down{i}.beta"] = f(sd[f"{d}.{i}.0.weight"]), f(sd[f"{d}.{i}.0.bias"])
        w = sd[f"{d}.{i}.1.weight"].float()               # [Cout, Cin, 2, 2] -> [Cout, (ky, kx, c)], dense over the real Cin
        W[f"cx.down{i}.w"] = a(_pad2(w.permute(0, 2, 3, 1).reshape(DIMS[i], -1), cp[i], 4 * DIMS[i - 1]))
        W[f"cx.down{i}.b"] = f(_pad1(sd[f"{d}.{i}.1.bias"].float(), cp[i]))
    for i in range(4):
        c, cpad = DIMS[i], cp[i]
        for j in range(DEPTHS[i]):
            b, k = f"{_CX}.stages.{i}.{j}", f"cx.s{i}.{j}"
            W[f"{k}.dw.w"] = f(sd[f"{b}.dwconv.weight"].float().reshape(c, 49).t())           # [49][C]
            W[f"{k}.dw.b"] = f(sd[f"{b}.dwconv.bias"])
            W[f"{k}.ln.g"], W[f"{k}.ln.b"] = f(sd[f"{b}.norm.weight"]), f(sd[f"{b}.norm.bias"])
            W[f"{k}.pw1.w"] = a(_pad2(sd[f"{b}.pwconv1.weight"].float(), 4 * c, cpad))
            W[f"{k}.pw1.b"] = f(sd[f"{b}.pwconv1.bias"])
            g = sd[f"{b}.gamma"].float()                   # layer scale folded: gamma * (W x + b)
            W[f"{k}.pw2.w"] = a(_pad2(g[:, None] * sd[f"{b}.pwconv2.weight"].float(), cpad, 4 * c))
            W[f"{k}.pw2.b"] = f(_pad1(g * sd[f"{b}.pwconv2.bias"].float(), cpad))
    if cfg.tokenizer == "sem":
        w = sd[f"{_PN}.in_conv.weight"].float()            # [3, in_dim, 3, 3] -> [(ci, ky, kx), Cout]
        W["cx.in_conv.w"] = f(w.permute(1, 2, 3, 0).reshape(-1, 3))
        W["cx.in_conv.b"] = f(sd[f"{_PN}.in_conv.bias"])
    W["pn.pos"] = f(sd[f"{_PN}.pos_embedding"].reshape(cfg.spatial_tokens, DIMS[-1]))
    W["pn.null"] = f(sd[f"{_PN}.null_feature"])
    for li in (0, 2, 4):
        W[f"pn.l{li}.w"], W[f"pn.l{li}.b"] = a(sd[f"{_PN}.linears.{li}.weight"]), f(sd[f"{_PN}.linears.{li}.bias"])
    if cfg.tokenizer != "hed":
        for li in (0, 2):
            w = sd[f"downsample_net.layers.{li}.weight"].float()      # [Cout, Cin, 4, 4] -> [(ci, ky, kx), Cout]
            W[f"ds.l{li}.w"] = f(w.permute(1, 2, 3, 0).reshape(-1, w.shape[0]))
            W[f"ds.l{li}.b"] = f(sd[f"downsample_net.layers.{li}.bias"])


def emit_tokenizer(engine, P, Bt: int, objs: torch.Tensor) -> None:
    """Static plan steps: P.inp["map"] fp32 [Bt, Cm, Hm, Wm], P.inp["gmask"] fp32 [Bt]  ->  objs bf16 [Bt * n, out_dim]."""
    cfg, ops, W = engine.cfg, engine.ops, engine.W
    R, n = cfg.tok_resize, cfg.spatial_tokens
    cp = [round_up(c, 64) for c in DIMS]
    side = [R // 4, R // 8, R // 16, R // 32]
    rows = [Bt * s * s for s in side]
    xa = engine._buf(max(r * c for r, c in zip(rows, cp)))
    xb = engine._buf(max(r * c for r, c in zip(rows, cp)))
    hid = engine._buf(max(r * 4 * c for r, c in zip(rows, DIMS)))
    col = engine._buf(max(rows[0] * 64, max(rows[i] * 4 * DIMS[i - 1] for i in range(1, 4))))

    def add(name, fn):
        P.add(name, fn, static=True)

    src = P.inp["map"]
    if cfg.tokenizer == "sem":         # nearest resize fused into the 3 x 3 in_conv (sem_grounding_net.py:44-45)
        rgb = engine._zeros(Bt, 3, R, R)
        add("cx.in_conv", lambda src=src: ops.conv2d_small(src, W["cx.in_conv.w"], W["cx.in_conv.b"], rgb, 3, 1, 1, False, virtual=(R, R)))
        src = rgb
    c0 = col[: rows[0] * 64].view(rows[0], 64)
    x0 = xa[: rows[0] * cp[0]].view(rows[0], cp[0])
    add("cx.stem.patches", lambda src=src: ops.patchify_nchw(src, c0, R, R, 4))
    add("cx.stem.conv", lambda: ops.gemm(c0, W["cx.stem.w"], x0, bias=W["cx.stem.b"]))
    add("cx.stem.ln", lambda: ops.layernorm_rows(x0, x0, W["cx.stem.g"], W["cx.stem.beta"], DIMS[0], 1e-6))
    x = x0
    for i in range(4):
        c, cpad, s = DIMS[i], cp[i], side[i]
        if i > 0:
            t = xb[: rows[i - 1] * cp[i - 1]].view(rows[i - 1], cp[i - 1])
            ci = col[: rows[i] * 4 * DIMS[i - 1]].view(rows[i], 4 * DIMS[i - 1])
            xn = xa[: rows[i] * cpad].view(rows[i], cpad)
            k = f"cx.down{i}"
            add(f"{k}.ln", lambda x=x, t=t, k=k, i=i: ops.layernorm_rows(x, t, W[f"{k}.g"], W[f"{k}.beta"], DIMS[i - 1], 1e-6))
            add(f"{k}.patches", lambda t=t, ci=ci, i=i: ops.patchify_nhwc(t, ci, side[i - 1], side[i - 1], DIMS[i - 1], 2))
            add(f"{k}.conv", lambda ci=ci, xn=xn, k=k: ops.gemm(ci, W[f"{k}.w"], xn, bias=W[f"{k}.b"]))
            x = xn
        t = xb[: rows[i] * cpad].view(rows[i], cpad)
        h = hid[: rows[i] * 4 * c].view(rows[i], 4 * c)
        for j in range(DEPTHS[i]):
            k = f"cx.s{i}.{j}"
            add(f"{k}.dwconv_ln", lambda x=x, t=t, k=k, s=s, c=c: ops.dwconv7_ln(x, t, W[f"{k}.dw.w"], W[f"{k}.dw.b"], W[f"{k}.ln.g"], W[f"{k}.ln.b"],
                                                                           Bt, s, s, c, 1e-6))
            add(f"{k}.pwconv1", lambda t=t, h=h, k=k: ops.gemm(t, W[f"{k}.pw1.w"], h, bias=W[f"{k}.pw1.b"], act=ACT_GELU))
            add(f"{k}.pwconv2", lambda x=x, h=h, k=k: ops.gemm(h, W[f"{k}.pw2.w"], x, bias=W[f"{k}.pw2.b"], residual=x))
    # tokens: mask / null replacement + position embedding, then the MLP (hed_grounding_net.py:47-59)
    D, HID = cfg.tok_out_dim, cfg.tok_hidden
    tok = xb[: Bt * n * DIMS[-1]].view(Bt * n, DIMS[-1])
    h1 = hid[: Bt * n * HID].view(Bt * n, HID)
    h2 = hid[Bt * n * HID: 2 * Bt * n * HID].view(Bt * n, HID)
    feat = x
    add("pn.tokens", lambda: ops.spatial_tokens(feat, P.inp["gmask"], W["pn.null"], W["pn.pos"], tok, n))
    add("pn.l0", lambda: ops.gemm(tok, W["pn.l0.w"], h1, bias=W["pn.l0.b"], act=ACT_SILU))
    add("pn.l2", lambda: ops.gemm(h1, W["pn.l2.w"], h2, bias=W["pn.l2.b"], act=ACT_SILU))
    add("pn.l4", lambda: ops.gemm(h2, W["pn.l4.w"], objs, bias=W["pn.l4.b"]))


def emit_downsampler(engine, P, Bt: int) -> torch.Tensor:
    """Static plan steps: P.inp["extra_map"] fp32 [Bt, Cm, Hm, Wm] -> fp32 planes [Bt, ds_out_dim, L, L] that conv_in reads next to
    the latent (openaimodel.py:441-443).  L = latent size (the reference hard-codes 64 for hed; the conv stacks give resize / 4)."""
    cfg, ops, W = engine.cfg, engine.ops, engine.W
    L, R, t = cfg.image_size, cfg.ds_resize, cfg.tokenizer
    out = engine._zeros(Bt, cfg.ds_out_dim, L, L)
    src = P.inp["extra_map"]

    def add(name, fn):
        P.add(name, fn, static=True)

    if t == "hed":
        add("ds.bicubic", lambda: ops.resize_plane(src, out, 1, "bicubic"))
        return out
    assert R // 4 == L, f"GroundingDownsampler(resize_input={R}) gives {R // 4} x {R // 4} planes, the latent is {L} x {L}"
    mid = W["ds.l0.w"].shape[1]
    c1 = engine._zeros(Bt, mid, R // 2, R // 2)
    if t == "sem":                     # nearest resize fused into the first conv
        add("ds.conv0", lambda: ops.conv2d_small(src, W["ds.l0.w"], W["ds.l0.b"], c1, 4, 2, 1, True, virtual=(R, R)))
    else:
        cin = 3 if t == "normal" else 1
        r1 = engine._zeros(Bt, cin, R, R)
        add("ds.bicubic", lambda: ops.resize_plane(src, r1, cin, "bicubic"))
        add("ds.conv0", lambda: ops.conv2d_small(r1, W["ds.l0.w"], W["ds.l0.b"], c1, 4, 2, 1, True))
    add("ds.conv2", lambda: ops.conv2d_small(c1, W["ds.l2.w"], W["ds.l2.b"], out, 4, 2, 1, False))
    return out
