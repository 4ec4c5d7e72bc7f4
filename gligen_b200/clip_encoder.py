"""The pre-LayerNorm transformer shared by the CLIP text and image towers (transformers CLIPEncoder), on this repo's kernels.

Each block: LayerNorm rows, the fused-QKV glg_gemm, the attention kernel (causal for the text tower, bidirectional for the image
tower), out-projection / fc2 GEMMs with the residual add in the epilogue, fc1 with the quick_gelu epilogue.  bf16 activations
and weights, fp32 accumulation / statistics.  The towers' embeddings and heads live in clip_text.py and clip_vision.py.
"""
from __future__ import annotations

from collections import OrderedDict
from math import prod
from typing import Dict

import torch

from .ops import ACT_QUICK_GELU, EngineBase


def layer_param_shapes(cfg, prefix: str) -> "OrderedDict[str, tuple]":
    """State-dict keys / shapes of `prefix` + `encoder.layers.{i}.*`, registration order (the order the seeded weights are drawn in)."""
    p: "OrderedDict[str, tuple]" = OrderedDict()
    C = cfg.width
    for i in range(cfg.layers):
        l = f"{prefix}encoder.layers.{i}"
        for n in ("k_proj", "v_proj", "q_proj", "out_proj"):
            p[f"{l}.self_attn.{n}.weight"], p[f"{l}.self_attn.{n}.bias"] = (C, C), (C,)
        p[f"{l}.layer_norm1.weight"], p[f"{l}.layer_norm1.bias"] = (C,), (C,)
        p[f"{l}.mlp.fc1.weight"], p[f"{l}.mlp.fc1.bias"] = (cfg.ffn, C), (cfg.ffn,)
        p[f"{l}.mlp.fc2.weight"], p[f"{l}.mlp.fc2.bias"] = (C, cfg.ffn), (C,)
        p[f"{l}.layer_norm2.weight"], p[f"{l}.layer_norm2.bias"] = (C,), (C,)
    return p


def synthetic_state_dict(shapes: "OrderedDict[str, tuple]", seed: int, massive: str) -> Dict[str, torch.Tensor]:
    """Seeded fp32 weights in the order of `shapes`: projections and convolutions ~ N(0, 1/fan_in), the embedding whose key ends
    with `massive` ~ N(0, 0.02) with every (width/4)-th channel scaled by 8 like the massive channels trained CLIP towers show,
    position embeddings ~ N(0, 0.01), norm scales 1 + 0.1 N, biases 0.05 N."""
    g = torch.Generator(device="cpu").manual_seed(seed)
    sd: Dict[str, torch.Tensor] = OrderedDict()
    for key, shape in shapes.items():
        if key.endswith(massive):
            t = torch.randn(shape, generator=g) * 0.02
            t[..., :: max(1, shape[-1] // 4)] *= 8.0
        elif key.endswith("position_embedding.weight"):
            t = torch.randn(shape, generator=g) * 0.01
        elif key.endswith(".bias"):
            t = torch.randn(shape, generator=g) * 0.05
        elif len(shape) == 1:
            t = 1.0 + 0.1 * torch.randn(shape, generator=g)
        else:
            t = torch.randn(shape, generator=g) * (prod(shape[1:]) ** -0.5)
        sd[key] = t
    return sd


class ClipEncoderEngine(EngineBase):
    """Base of ClipTextEngine and ClipVisionEngine: the packed weights `W`, the per-shape workspaces `_ws`, and the blocks."""

    def __init__(self, cfg, ops):
        super().__init__(ops)
        self.cfg = cfg
        self.W: Dict[str, torch.Tensor] = {}
        self._ws: Dict[int, Dict[str, torch.Tensor]] = {}
        self.loaded = False

    def _load_layers(self, sd: Dict[str, torch.Tensor], pre: str) -> None:
        """`pre` + `encoder.layers.{i}.*` -> W["{i}.ln1.g"], ..., with q | k | v fused into one weight and bias."""
        W = self.W
        for i in range(self.cfg.layers):
            l = f"{pre}encoder.layers.{i}"
            W[f"{i}.ln1.g"], W[f"{i}.ln1.b"] = self._f(sd[f"{l}.layer_norm1.weight"]), self._f(sd[f"{l}.layer_norm1.bias"])
            W[f"{i}.ln2.g"], W[f"{i}.ln2.b"] = self._f(sd[f"{l}.layer_norm2.weight"]), self._f(sd[f"{l}.layer_norm2.bias"])
            W[f"{i}.qkv.w"] = self._a(torch.cat([sd[f"{l}.self_attn.{n}_proj.weight"] for n in ("q", "k", "v")], dim=0))
            W[f"{i}.qkv.b"] = self._f(torch.cat([sd[f"{l}.self_attn.{n}_proj.bias"] for n in ("q", "k", "v")], dim=0))
            W[f"{i}.out.w"], W[f"{i}.out.b"] = self._a(sd[f"{l}.self_attn.out_proj.weight"]), self._f(sd[f"{l}.self_attn.out_proj.bias"])
            W[f"{i}.fc1.w"], W[f"{i}.fc1.b"] = self._a(sd[f"{l}.mlp.fc1.weight"]), self._f(sd[f"{l}.mlp.fc1.bias"])
            W[f"{i}.fc2.w"], W[f"{i}.fc2.b"] = self._a(sd[f"{l}.mlp.fc2.weight"]), self._f(sd[f"{l}.mlp.fc2.bias"])

    def _run_layers(self, ws: Dict[str, torch.Tensor], causal: bool) -> None:
        """The blocks over the residual stream ws["x"] [B*L, C], in place; workspace t [B*L, C], qkv [B, L, 3C], ao [B, L, C],
        h [B*L, ffn]."""
        c, ops, W = self.cfg, self.ops, self.W
        x, t, qkv, ao, h = ws["x"], ws["t"], ws["qkv"], ws["ao"], ws["h"]
        B, L, _ = qkv.shape
        C, d = c.width, c.width // c.heads
        for i in range(c.layers):
            ops.layernorm_rows(x, t, W[f"{i}.ln1.g"], W[f"{i}.ln1.b"], C, c.eps)
            ops.gemm(t, W[f"{i}.qkv.w"], qkv.view(B * L, 3 * C), bias=W[f"{i}.qkv.b"])
            ops.attention(qkv[:, :, :C], qkv[:, :, C: 2 * C], qkv[:, :, 2 * C:], ao, c.heads, d, causal=causal)
            ops.gemm(ao.view(B * L, C), W[f"{i}.out.w"], x, bias=W[f"{i}.out.b"], residual=x)
            ops.layernorm_rows(x, t, W[f"{i}.ln2.g"], W[f"{i}.ln2.b"], C, c.eps)
            ops.gemm(t, W[f"{i}.fc1.w"], h, bias=W[f"{i}.fc1.b"], act=ACT_QUICK_GELU)
            ops.gemm(h, W[f"{i}.fc2.w"], x, bias=W[f"{i}.fc2.b"], residual=x)
