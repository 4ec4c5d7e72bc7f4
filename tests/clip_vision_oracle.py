"""CPU fp32 ORACLE for the image-grounding front end of gligen_inference.py.  TEST INFRASTRUCTURE ONLY.

The reference's `prepare_batch` (gligen_inference.py:146-187) creates `transformers.CLIPModel` and runs its image tower
(third party, pinned transformers==4.19.2 by env_docker/Dockerfile:3, not vendored) and text tower on each phrase / image.
This file restates, in plain torch:
  * clip_vision_forward - transformers/models/clip/modeling_clip.py CLIPVisionEmbeddings (patch conv without bias, class
    token, position embeddings), CLIPVisionTransformer (pre_layrnorm, the encoder with bidirectional attention and quick_gelu,
    post_layernorm of the class token = pooler_output) and CLIPVisionModelWithProjection's visual_projection (image_embeds);
  * gligen_image_feature - gligen_inference.py:91-98 `project` and :114-116 (reprojection, norm 28.7);
  * complete_mask, prepare_batch - gligen_inference.py:131-142, :146-187, phrase / image features supplied by callables, one item
    at a time.
Pinned by scripts/gen_golden_clip_vision.py against the INSTALLED transformers' CLIPVisionModelWithProjection on seeded weights
(tests/golden/clip_vision_*.pt)."""
from __future__ import annotations

from typing import Callable, Dict, Optional, Tuple

import torch
import torch.nn.functional as F


def clip_vision_forward(cfg, sd: Dict[str, torch.Tensor], pixel_values: torch.Tensor,
                        prefix: str = "vision_model.", proj_key: str = "visual_projection.weight") -> Tuple[torch.Tensor, torch.Tensor, torch.Tensor]:
    """-> (last_hidden_state [N, T, C] (encoder output, before post_layernorm), pooler_output [N, C], image_embeds [N, D])."""
    C, H = cfg.width, cfg.heads
    d = C // H
    N = pixel_values.shape[0]
    p = F.conv2d(pixel_values, sd[prefix + "embeddings.patch_embedding.weight"], stride=cfg.patch)       # [N, C, 16, 16]
    p = p.flatten(2).transpose(1, 2)
    cls = sd[prefix + "embeddings.class_embedding"].expand(N, 1, C)
    x = torch.cat([cls, p], dim=1) + sd[prefix + "embeddings.position_embedding.weight"][None]
    x = F.layer_norm(x, (C,), sd[prefix + "pre_layrnorm.weight"], sd[prefix + "pre_layrnorm.bias"], cfg.eps)
    T = x.shape[1]
    for i in range(cfg.layers):
        l = f"{prefix}encoder.layers.{i}"
        h = F.layer_norm(x, (C,), sd[f"{l}.layer_norm1.weight"], sd[f"{l}.layer_norm1.bias"], cfg.eps)
        q = F.linear(h, sd[f"{l}.self_attn.q_proj.weight"], sd[f"{l}.self_attn.q_proj.bias"]) * d ** -0.5
        k = F.linear(h, sd[f"{l}.self_attn.k_proj.weight"], sd[f"{l}.self_attn.k_proj.bias"])
        v = F.linear(h, sd[f"{l}.self_attn.v_proj.weight"], sd[f"{l}.self_attn.v_proj.bias"])
        q, k, v = (t.view(N, T, H, d).transpose(1, 2) for t in (q, k, v))
        a = torch.softmax(q @ k.transpose(-1, -2), dim=-1) @ v
        a = a.transpose(1, 2).reshape(N, T, C)
        x = x + F.linear(a, sd[f"{l}.self_attn.out_proj.weight"], sd[f"{l}.self_attn.out_proj.bias"])
        h = F.layer_norm(x, (C,), sd[f"{l}.layer_norm2.weight"], sd[f"{l}.layer_norm2.bias"], cfg.eps)
        h = F.linear(h, sd[f"{l}.mlp.fc1.weight"], sd[f"{l}.mlp.fc1.bias"])
        h = h * torch.sigmoid(1.702 * h)                                   # quick_gelu
        x = x + F.linear(h, sd[f"{l}.mlp.fc2.weight"], sd[f"{l}.mlp.fc2.bias"])
    pooled = F.layer_norm(x[:, 0], (C,), sd[prefix + "post_layernorm.weight"], sd[prefix + "post_layernorm.bias"], cfg.eps)
    return x, pooled, pooled @ sd[proj_key].t()


def gligen_image_feature(image_embeds: torch.Tensor, projection_matrix: torch.Tensor, target_norm: float = 28.7) -> torch.Tensor:
    """gligen_inference.py:114-116 for each row: `project(feature, projection_matrix.T)` (= feature @ projection_matrix, :91-98),
    then `feature / feature.norm() * 28.7`."""
    f = image_embeds @ projection_matrix.to(image_embeds.dtype)
    return f / f.norm(dim=-1, keepdim=True) * target_norm


def complete_mask(has_mask, max_objs):
    """gligen_inference.py:131-142."""
    mask = torch.ones(1, max_objs)
    if has_mask is None:
        return mask
    if type(has_mask) == int or type(has_mask) == float:
        return mask * has_mask
    for idx, value in enumerate(has_mask):
        mask[0, idx] = value
    return mask


def prepare_batch(meta, text_feature: Callable, image_feature: Callable, batch: int = 1, max_objs: int = 30,
                  text_dim: int = 768, image_dim: int = 768) -> Dict[str, torch.Tensor]:
    """gligen_inference.py:146-187 on the CPU.  text_feature(phrase) / image_feature(image) return a [1, dim] feature or None
    (get_clip_feature, :101-117, one item per call)."""
    phrases, images = meta.get("phrases"), meta.get("images")
    images = [None] * len(phrases) if images is None else images                     # :147-149
    phrases = [None] * len(images) if phrases is None else phrases
    boxes = torch.zeros(max_objs, 4)                                                  # :155-160
    masks = torch.zeros(max_objs)
    text_masks = torch.zeros(max_objs)
    image_masks = torch.zeros(max_objs)
    text_embeddings = torch.zeros(max_objs, text_dim)
    image_embeddings = torch.zeros(max_objs, image_dim)
    text_features, image_features = [], []
    for phrase, image in zip(phrases, images):                                        # :162-166
        text_features.append(None if phrase is None else text_feature(phrase))
        image_features.append(None if image is None else image_feature(image))
    for idx, (box, tf, imf) in enumerate(zip(meta["locations"], text_features, image_features)):    # :168-176
        boxes[idx] = torch.tensor(box)
        masks[idx] = 1
        if tf is not None:
            text_embeddings[idx] = tf
            text_masks[idx] = 1
        if imf is not None:
            image_embeddings[idx] = imf
            image_masks[idx] = 1
    return {                                                                          # :178-185
        "boxes": boxes.unsqueeze(0).repeat(batch, 1, 1),
        "masks": masks.unsqueeze(0).repeat(batch, 1),
        "text_masks": text_masks.unsqueeze(0).repeat(batch, 1) * complete_mask(meta.get("text_mask"), max_objs),
        "image_masks": image_masks.unsqueeze(0).repeat(batch, 1) * complete_mask(meta.get("image_mask"), max_objs),
        "text_embeddings": text_embeddings.unsqueeze(0).repeat(batch, 1, 1),
        "image_embeddings": image_embeddings.unsqueeze(0).repeat(batch, 1, 1),
    }
