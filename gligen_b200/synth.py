"""Seeded synthetic inputs of the shapes/value conventions the reference feeds the UNet.

There is no network for CLIP / VAE / checkpoints, so the benchmark and the parity tests use
random embeddings (SURVEY 8d).  Everything is drawn on the CPU from one torch.Generator so the
CPU oracle and the GPU engine see identical bits.

Value conventions: boxes xyxy in [0,1] (dataset/tsv_dataset.py:263); text/image embeddings are
zero where the object slot is unused (gligen_inference.py:155-176); keypoints xy in [0,1],
invalid -> (0,0) and mask = (mean != 0) (gligen_inference.py:199-218).
"""
from __future__ import annotations

from typing import Dict, Optional, Tuple, Union

import torch

from .spec import SPATIAL_MAP_KEY, UNetConfig


def make_grounding_batch(cfg: UNetConfig, B: int, max_objs: int, g: torch.Generator,
                         n_valid: Optional[int] = None, map_size: Optional[Tuple[int, int]] = None) -> Dict[str, torch.Tensor]:
    """The `batch` dict handed to GroundingNetInput.prepare (gligen_inference.py:411)."""
    if cfg.spatial:
        return make_spatial_batch(cfg, B, g, map_size)
    if cfg.tokenizer == "keypoint":
        n = cfg.max_persons * 17
        pts = torch.rand(B, n, 2, generator=g)
        drop = torch.rand(B, n, generator=g) < 0.35
        pts[drop] = 0.0
        masks = (pts.mean(dim=-1) != 0).float()
        return {"points": pts, "masks": masks}
    xy0 = torch.rand(B, max_objs, 2, generator=g) * 0.6
    wh = 0.1 + torch.rand(B, max_objs, 2, generator=g) * 0.3
    boxes = torch.cat([xy0, (xy0 + wh).clamp(max=1.0)], dim=-1)
    if n_valid is None:
        nv = torch.randint(1, max_objs + 1, (B,), generator=g)
    else:
        nv = torch.full((B,), n_valid)
    masks = (torch.arange(max_objs)[None, :] < nv[:, None]).float()
    boxes = boxes * masks[..., None]
    te = torch.randn(B, max_objs, cfg.tok_in_dim, generator=g) * masks[..., None]
    out = {"boxes": boxes, "masks": masks, "text_embeddings": te}
    if cfg.tokenizer == "text_image":
        ie = torch.randn(B, max_objs, cfg.tok_in_dim, generator=g)
        ie = 28.7 * ie / ie.norm(dim=-1, keepdim=True) * masks[..., None]
        out.update({"text_masks": masks.clone(), "image_masks": masks.clone(), "image_embeddings": ie})
    return out


def make_spatial_batch(cfg: UNetConfig, B: int, g: torch.Generator,
                       size: Optional[Union[int, Tuple[int, int]]] = None) -> Dict[str, torch.Tensor]:
    """A spatial conditioning map of `size` = side or (H, W), by default square at twice the tokenizer's input size (512 x 512
    for the shipped configs), the way the datasets deliver it: grey maps (hed / canny / depth) replicated to 3 channels in
    [0, 1], normals in [-1, 1], semantic maps one-hot over `sem_in_dim` classes in constant label blocks; `mask` = 1 (map
    present; the null input is a zero map with mask 0).  Square maps use 16-pixel blocks; non-square ones use 13-pixel
    blocks, which no resampling ratio of theirs lines up with, so an off-by-one source index changes the labels it reads."""
    size = size or 2 * cfg.tok_resize
    H, W = (size, size) if isinstance(size, int) else size
    key = SPATIAL_MAP_KEY[cfg.tokenizer]
    if cfg.tokenizer == "sem":
        blk = 16 if H == W else 13
        coarse = torch.randint(0, cfg.sem_in_dim, (B, -(-H // blk), -(-W // blk)), generator=g)
        labels = coarse.repeat_interleave(blk, 1).repeat_interleave(blk, 2)[:, :H, :W]
        m = torch.nn.functional.one_hot(labels, cfg.sem_in_dim).permute(0, 3, 1, 2).float().contiguous()
    elif cfg.tokenizer == "normal":
        m = torch.rand(B, 3, H, W, generator=g) * 2 - 1
    else:
        base = torch.rand(B, 1, H, W, generator=g)
        if cfg.tokenizer in ("hed", "canny"):
            base = (base > 0.8).float() * torch.rand(B, 1, H, W, generator=g)       # sparse edge responses
        m = base.repeat(1, 3, 1, 1).contiguous()
    return {key: m, "mask": torch.ones(B)}


def grounding_kwargs(cfg: UNetConfig, batch: Dict[str, torch.Tensor]) -> Dict[str, torch.Tensor]:
    """What GroundingNetInput.prepare returns (grounding_input/*_tokinzer_input.py)."""
    if cfg.spatial:
        return {SPATIAL_MAP_KEY[cfg.tokenizer]: batch[SPATIAL_MAP_KEY[cfg.tokenizer]], "mask": batch["mask"]}
    if cfg.tokenizer == "text":
        return {"boxes": batch["boxes"], "masks": batch["masks"], "positive_embeddings": batch["text_embeddings"]}
    if cfg.tokenizer == "text_image":
        return {k: batch[k] for k in ("boxes", "masks", "text_masks", "image_masks", "text_embeddings", "image_embeddings")}
    return {"points": batch["points"], "masks": batch["masks"]}


def make_inputs(cfg: UNetConfig, B: int, max_objs: int = 30, seed: int = 2, n_valid: Optional[int] = None,
                n_ctx: int = 77, map_size: Optional[Tuple[int, int]] = None) -> Dict[str, object]:
    """x_T, context, uc, grounding batch (+ inpainting tensors when cfg.inpaint_mode); `map_size` (H, W): the spatial map's."""
    g = torch.Generator(device="cpu").manual_seed(seed)
    hw = cfg.image_size
    out: Dict[str, object] = {
        "x": torch.randn(B, cfg.in_channels, hw, hw, generator=g),
        "context": torch.randn(B, n_ctx, cfg.context_dim, generator=g),
        "uc": torch.randn(B, n_ctx, cfg.context_dim, generator=g),
    }
    batch = make_grounding_batch(cfg, B, max_objs, g, n_valid, map_size)
    out["batch"] = batch
    out["grounding_input"] = grounding_kwargs(cfg, batch)
    if cfg.spatial:          # GroundingDSInput.prepare (grounding_input/*_grounding_downsampler_input.py:16): the same map
        out["grounding_extra_input"] = batch[SPATIAL_MAP_KEY[cfg.tokenizer]]
    if cfg.inpaint_mode:
        out["z0"] = torch.randn(B, cfg.in_channels, hw, hw, generator=g) * 0.9
    return out
