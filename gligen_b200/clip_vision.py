"""The CLIP ViT-L/14 image tower behind `prepare_batch`'s image-grounded phrases, on this repo's kernels.

Reference call site: gligen_inference.py:101-117 - `CLIPModel.from_pretrained("openai/clip-vit-large-patch14")` (:151-153) run on
`CLIPProcessor` pixel values; the box+text+image PositionNet reads `image_embeds @ projection_matrix`, rescaled to norm 28.7.
The arithmetic lives in the third-party `transformers` package: CLIPVisionEmbeddings = Conv2d(3, C, 14, stride 14, no bias) over
the 224 x 224 image, a learned class token in front of the 256 patch tokens, learned position embeddings; `pre_layrnorm`; 24
pre-LayerNorm blocks (bidirectional self-attention with 16 heads of 64, MLP 1024 -> 4096 -> 1024 with quick_gelu);
pooler_output = post_layernorm(last_hidden_state[:, 0]); image_embeds = pooler_output @ visual_projection.weight^T (no bias).
Restated in tests/clip_vision_oracle.py and pinned against the installed transformers' CLIPVisionModelWithProjection.

Here: glg_patchify_nchw (14 x 14 stride-14 patches as GEMM rows) + glg_gemm against the repacked conv weight with fp32 out,
glg_clip_vision_embed (class token, position add and pre_layrnorm in one launch), the blocks as in ClipTextEngine (fused-QKV
GEMM, the wgmma attention kernel over 257 keys, residual / quick_gelu epilogues), glg_clip_image_head (post_layernorm of the
class token, visual projection and GLIGEN's reprojection in fp32).  bf16 activations and weights, fp32 accumulation /
statistics / head, fp32 outputs.
"""
from __future__ import annotations

from collections import OrderedDict
from dataclasses import dataclass
from typing import Dict, Optional, Tuple

import torch
import torch.nn.functional as F

ACT_QUICK_GELU = 3
CLIP_MEAN = (0.48145466, 0.4578275, 0.40821073)          # CLIPImageProcessor image_mean / image_std
CLIP_STD = (0.26862954, 0.26130258, 0.27577711)


@dataclass(frozen=True)
class ClipVisionConfig:
    image_size: int = 224
    patch: int = 14
    width: int = 1024
    layers: int = 24
    heads: int = 16
    ffn: int = 4096
    projection: int = 768
    eps: float = 1e-5

    @property
    def patches(self) -> int:
        return (self.image_size // self.patch) ** 2

    @property
    def tokens(self) -> int:
        return self.patches + 1

    @property
    def k_pad(self) -> int:
        """Patch-row length: 3 * patch^2 columns in (ky, kx, c) order, zero-padded to a multiple of 64 for glg_gemm."""
        return (3 * self.patch * self.patch + 63) // 64 * 64


SD14_CLIP_VISION = ClipVisionConfig()                                       # openai/clip-vit-large-patch14 vision tower
TINY_CLIP_VISION = ClipVisionConfig(width=128, layers=2, heads=2, ffn=512)   # same 257-token geometry and 768-d projection
NAMED_CLIP_VISION_CONFIGS = {"sd14_clip_vision": SD14_CLIP_VISION, "tiny_clip_vision": TINY_CLIP_VISION}


def clip_vision_param_shapes(cfg: ClipVisionConfig, prefix: str = "") -> "OrderedDict[str, tuple]":
    """State-dict keys / shapes of the image tower inside transformers' CLIPModel (also CLIPVisionModelWithProjection's keys)."""
    p: "OrderedDict[str, tuple]" = OrderedDict()
    v, C = f"{prefix}vision_model", cfg.width
    p[f"{v}.embeddings.class_embedding"] = (C,)
    p[f"{v}.embeddings.patch_embedding.weight"] = (C, 3, cfg.patch, cfg.patch)
    p[f"{v}.embeddings.position_embedding.weight"] = (cfg.tokens, C)
    p[f"{v}.pre_layrnorm.weight"], p[f"{v}.pre_layrnorm.bias"] = (C,), (C,)
    for i in range(cfg.layers):
        l = f"{v}.encoder.layers.{i}"
        for n in ("k_proj", "v_proj", "q_proj", "out_proj"):
            p[f"{l}.self_attn.{n}.weight"], p[f"{l}.self_attn.{n}.bias"] = (C, C), (C,)
        p[f"{l}.layer_norm1.weight"], p[f"{l}.layer_norm1.bias"] = (C,), (C,)
        p[f"{l}.mlp.fc1.weight"], p[f"{l}.mlp.fc1.bias"] = (cfg.ffn, C), (cfg.ffn,)
        p[f"{l}.mlp.fc2.weight"], p[f"{l}.mlp.fc2.bias"] = (C, cfg.ffn), (C,)
        p[f"{l}.layer_norm2.weight"], p[f"{l}.layer_norm2.bias"] = (C,), (C,)
    p[f"{v}.post_layernorm.weight"], p[f"{v}.post_layernorm.bias"] = (C,), (C,)
    p[f"{prefix}visual_projection.weight"] = (cfg.projection, C)
    return p


def synthetic_clip_vision_state_dict(cfg: ClipVisionConfig, seed: int = 0, prefix: str = "") -> Dict[str, torch.Tensor]:
    """Seeded fp32 weights, the scheme of clip_text.synthetic_clip_state_dict: projections and the patch convolution ~ N(0, 1/fan_in),
    class / position embeddings ~ N(0, 0.02) / N(0, 0.01), norm scales 1 + 0.1 N, biases 0.05 N; a few class-embedding channels
    are scaled up like the massive channels trained CLIP towers show."""
    g = torch.Generator(device="cpu").manual_seed(seed)
    sd: Dict[str, torch.Tensor] = OrderedDict()
    for key, shape in clip_vision_param_shapes(cfg, prefix).items():
        if key.endswith("class_embedding"):
            t = torch.randn(shape, generator=g) * 0.02
            t[:: max(1, cfg.width // 4)] *= 8.0
        elif key.endswith("position_embedding.weight"):
            t = torch.randn(shape, generator=g) * 0.01
        elif key.endswith(".bias"):
            t = torch.randn(shape, generator=g) * 0.05
        elif len(shape) == 1:
            t = 1.0 + 0.1 * torch.randn(shape, generator=g)
        else:
            fan_in = 1
            for s in shape[1:]:
                fan_in *= s
            t = torch.randn(shape, generator=g) * (fan_in ** -0.5)
        sd[key] = t
    return sd


def synthetic_pixel_values(N: int, seed: int = 0, size: int = 224) -> torch.Tensor:
    """[N, 3, size, size] fp32 the way CLIPProcessor delivers them: uniform [0, 1] RGB, normalised with CLIP's mean / std."""
    g = torch.Generator(device="cpu").manual_seed(seed)
    u = torch.rand(N, 3, size, size, generator=g)
    return (u - torch.tensor(CLIP_MEAN).view(1, 3, 1, 1)) / torch.tensor(CLIP_STD).view(1, 3, 1, 1)


def synthetic_projection_matrix(D: int = 768, seed: int = 0) -> torch.Tensor:
    """A seeded stand-in for GLIGEN's `projection_matrix` (fp32 [D, D], entries ~ N(0, 1/D)).  The released file is 2.4 MB and is
    read at run time from where the reference reads it; the reprojected feature is rescaled to a fixed norm, so the matrix's
    overall scale does not matter."""
    g = torch.Generator(device="cpu").manual_seed(seed)
    return torch.randn(D, D, generator=g) * D ** -0.5


class ClipVisionEngine:
    def __init__(self, cfg: ClipVisionConfig, ops):
        self.cfg, self.ops, self.dev = cfg, ops, ops.device
        self.adt = ops.act_dtype
        self.W: Dict[str, torch.Tensor] = {}
        self._ws: Dict[int, Dict[str, torch.Tensor]] = {}
        self.loaded = False

    def _a(self, t):
        return t.detach().to(device=self.dev, dtype=self.adt).contiguous()

    def _f(self, t):
        return t.detach().to(device=self.dev, dtype=torch.float32).contiguous()

    def load_state_dict(self, sd: Dict[str, torch.Tensor]) -> None:
        """Accepts the keys of CLIPModel (`vision_model.*`, `visual_projection.weight`; the text tower's `text_model.*`,
        `text_projection.weight` and `logit_scale` are ignored), of CLIPVisionModelWithProjection (the same two prefixes) or bare
        (`embeddings.*`, ..., `visual_projection.weight`); the `position_ids` buffer older transformers versions save is ignored."""
        key0 = next(k for k in sd if k.endswith("embeddings.class_embedding"))
        pre = key0[: -len("embeddings.class_embedding")]
        cfg, W, C, k = self.cfg, self.W, self.cfg.width, self.cfg.patch
        W.clear()
        W["cls"], W["pos"] = self._f(sd[pre + "embeddings.class_embedding"]), self._f(sd[pre + "embeddings.position_embedding.weight"])
        assert W["cls"].shape == (C,) and W["pos"].shape == (cfg.tokens, C)
        # Conv2d weight [C, 3, k, k] -> GEMM weight [C, (ky, kx, c)] (glg_patchify_nchw's column order), zero-padded to k_pad
        w = sd[pre + "embeddings.patch_embedding.weight"].detach().float().permute(0, 2, 3, 1).reshape(C, 3 * k * k)
        W["patch"] = self._a(F.pad(w, (0, cfg.k_pad - 3 * k * k)))
        W["pre.g"], W["pre.b"] = self._f(sd[pre + "pre_layrnorm.weight"]), self._f(sd[pre + "pre_layrnorm.bias"])
        for i in range(cfg.layers):
            l = f"{pre}encoder.layers.{i}"
            W[f"{i}.ln1.g"], W[f"{i}.ln1.b"] = self._f(sd[f"{l}.layer_norm1.weight"]), self._f(sd[f"{l}.layer_norm1.bias"])
            W[f"{i}.ln2.g"], W[f"{i}.ln2.b"] = self._f(sd[f"{l}.layer_norm2.weight"]), self._f(sd[f"{l}.layer_norm2.bias"])
            W[f"{i}.qkv.w"] = self._a(torch.cat([sd[f"{l}.self_attn.{n}_proj.weight"] for n in ("q", "k", "v")], dim=0))
            W[f"{i}.qkv.b"] = self._f(torch.cat([sd[f"{l}.self_attn.{n}_proj.bias"] for n in ("q", "k", "v")], dim=0))
            W[f"{i}.out.w"], W[f"{i}.out.b"] = self._a(sd[f"{l}.self_attn.out_proj.weight"]), self._f(sd[f"{l}.self_attn.out_proj.bias"])
            W[f"{i}.fc1.w"], W[f"{i}.fc1.b"] = self._a(sd[f"{l}.mlp.fc1.weight"]), self._f(sd[f"{l}.mlp.fc1.bias"])
            W[f"{i}.fc2.w"], W[f"{i}.fc2.b"] = self._a(sd[f"{l}.mlp.fc2.weight"]), self._f(sd[f"{l}.mlp.fc2.bias"])
        W["post.g"], W["post.b"] = self._f(sd[pre + "post_layernorm.weight"]), self._f(sd[pre + "post_layernorm.bias"])
        W["proj"] = self._f(sd[next(k for k in sd if k.endswith("visual_projection.weight"))])
        assert W["proj"].shape == (cfg.projection, C)
        self.loaded = True

    def _workspace(self, N: int) -> Dict[str, torch.Tensor]:
        if N not in self._ws:
            c, T, P = self.cfg, self.cfg.tokens, self.cfg.patches
            e = lambda *s, dt=None: torch.empty(*s, device=self.dev, dtype=dt or self.adt)
            f32 = torch.float32
            self._ws[N] = dict(px=e(N, 3, c.image_size, c.image_size, dt=f32), pt=e(N * P, c.k_pad), pe=e(N * P, c.width, dt=f32),
                               x=e(N * T, c.width), t=e(N * T, c.width), qkv=e(N, T, 3 * c.width), ao=e(N, T, c.width), h=e(N * T, c.ffn),
                               pooled=e(N, c.width, dt=f32), emb=e(N, c.projection, dt=f32), feat=e(N, c.projection, dt=f32))
        return self._ws[N]

    def _run(self, pixel_values: torch.Tensor, proj: Optional[torch.Tensor], target_norm: float) -> Dict[str, torch.Tensor]:
        assert self.loaded, "load_state_dict first"
        c, ops, W = self.cfg, self.ops, self.W
        N = pixel_values.shape[0]
        assert pixel_values.shape == (N, 3, c.image_size, c.image_size), pixel_values.shape
        ws = self._workspace(N)
        ws["px"].copy_(pixel_values)
        x, t, qkv, ao, h = ws["x"], ws["t"], ws["qkv"], ws["ao"], ws["h"]
        C, d, T = c.width, c.width // c.heads, c.tokens
        ops.patchify_nchw(ws["px"], ws["pt"], c.image_size, c.image_size, c.patch)
        ops.gemm(ws["pt"], W["patch"], ws["pe"])
        ops.clip_vision_embed(ws["pe"], W["cls"], W["pos"], W["pre.g"], W["pre.b"], x, c.patches, c.eps)
        for i in range(c.layers):
            ops.layernorm_rows(x, t, W[f"{i}.ln1.g"], W[f"{i}.ln1.b"], C, c.eps)
            ops.gemm(t, W[f"{i}.qkv.w"], qkv.view(N * T, 3 * C), bias=W[f"{i}.qkv.b"])
            ops.attention(qkv[:, :, :C], qkv[:, :, C: 2 * C], qkv[:, :, 2 * C:], ao, c.heads, d, causal=False)
            ops.gemm(ao.view(N * T, C), W[f"{i}.out.w"], x, bias=W[f"{i}.out.b"], residual=x)
            ops.layernorm_rows(x, t, W[f"{i}.ln2.g"], W[f"{i}.ln2.b"], C, c.eps)
            ops.gemm(t, W[f"{i}.fc1.w"], h, bias=W[f"{i}.fc1.b"], act=ACT_QUICK_GELU)
            ops.gemm(h, W[f"{i}.fc2.w"], x, bias=W[f"{i}.fc2.b"], residual=x)
        ops.clip_image_head(x.view(N, T, C), W["post.g"], W["post.b"], W["proj"], ws["pooled"], ws["emb"],
                            proj, None if proj is None else ws["feat"], target_norm, c.eps)
        return ws

    @torch.no_grad()
    def forward(self, pixel_values: torch.Tensor) -> Tuple[torch.Tensor, torch.Tensor, torch.Tensor]:
        """pixel_values fp32 [N, 3, 224, 224] -> (last_hidden_state fp32 [N, 257, C] (before post_layernorm, as transformers
        defines it), pooler_output fp32 [N, C], image_embeds fp32 [N, projection])."""
        ws = self._run(pixel_values, None, 0.0)
        N, T, C = pixel_values.shape[0], self.cfg.tokens, self.cfg.width
        # the bf16 residual stream read out as fp32 (result read-out, host glue)
        return ws["x"].view(N, T, C).to(torch.float32, copy=True), ws["pooled"].clone(), ws["emb"].clone()

    @torch.no_grad()
    def grounding_features(self, pixel_values: torch.Tensor, proj: torch.Tensor, target_norm: float = 28.7) -> torch.Tensor:
        """GLIGEN's 'after_reproject' image feature (gligen_inference.py:114-116): f = image_embeds @ proj rescaled to norm
        target_norm, computed from the fp32 image_embeds; proj fp32 [projection, projection] on this device -> fp32 [N, projection]."""
        return self._run(pixel_values, proj, target_norm)["feat"].clone()
