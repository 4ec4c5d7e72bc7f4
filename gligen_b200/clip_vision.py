"""The CLIP ViT-L/14 image tower behind `prepare_batch`'s image-grounded phrases, on this repo's kernels.

Reference call site: gligen_inference.py:101-117 - `CLIPModel.from_pretrained("openai/clip-vit-large-patch14")` (:151-153) run on
`CLIPProcessor` pixel values; the box+text+image PositionNet reads `image_embeds @ projection_matrix`, rescaled to norm 28.7.
The arithmetic lives in the third-party `transformers` package: CLIPVisionEmbeddings = Conv2d(3, C, 14, stride 14, no bias) over
the 224 x 224 image, a learned class token in front of the 256 patch tokens, learned position embeddings; `pre_layrnorm`; 24
pre-LayerNorm blocks (bidirectional self-attention with 16 heads of 64, MLP 1024 -> 4096 -> 1024 with quick_gelu);
pooler_output = post_layernorm(last_hidden_state[:, 0]); image_embeds = pooler_output @ visual_projection.weight^T (no bias).
Restated in tests/clip_vision_oracle.py and pinned against the installed transformers' CLIPVisionModelWithProjection.

Here: glg_patchify_nchw (14 x 14 stride-14 patches as GEMM rows) + glg_gemm against the repacked conv weight with fp32 out,
glg_clip_vision_embed (class token, position add and pre_layrnorm in one launch), the blocks of clip_encoder.py (the wgmma
attention kernel over 257 keys, no mask), glg_clip_image_head (post_layernorm of the class token, visual projection and
GLIGEN's reprojection in fp32).  bf16 activations and weights, fp32 accumulation / statistics / head, fp32 outputs.
"""
from __future__ import annotations

from collections import OrderedDict
from dataclasses import dataclass
from typing import Dict, Optional, Tuple

import torch
import torch.nn.functional as F

from .clip_encoder import ClipEncoderEngine, layer_param_shapes, synthetic_state_dict

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
    p.update(layer_param_shapes(cfg, f"{v}."))
    p[f"{v}.post_layernorm.weight"], p[f"{v}.post_layernorm.bias"] = (C,), (C,)
    p[f"{prefix}visual_projection.weight"] = (cfg.projection, C)
    return p


def synthetic_clip_vision_state_dict(cfg: ClipVisionConfig, seed: int = 0, prefix: str = "") -> Dict[str, torch.Tensor]:
    """Seeded fp32 weights, the scheme of clip_encoder.synthetic_state_dict (the patch convolution ~ N(0, 1/fan_in) too); the
    class embedding carries the scaled-up massive channels."""
    return synthetic_state_dict(clip_vision_param_shapes(cfg, prefix), seed, massive="class_embedding")


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


class ClipVisionEngine(ClipEncoderEngine):
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
        self._load_layers(sd, pre)
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
        ops.patchify_nchw(ws["px"], ws["pt"], c.image_size, c.image_size, c.patch)
        ops.gemm(ws["pt"], W["patch"], ws["pe"])
        ops.clip_vision_embed(ws["pe"], W["cls"], W["pos"], W["pre.g"], W["pre.b"], ws["x"], c.patches, c.eps)
        self._run_layers(ws, causal=False)
        ops.clip_image_head(ws["x"].view(N, c.tokens, c.width), W["post.g"], W["post.b"], W["proj"], ws["pooled"], ws["emb"],
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
