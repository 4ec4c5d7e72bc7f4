"""Host-side glue around the drop-in call surface, the way gligen_inference.py drives it:

  * `build_model(name)` = `instantiate_from_config(config['model']).to(device).eval()` + `load_state_dict` +
    `model.grounding_tokenizer_input = instantiate_from_config(config['grounding_tokenizer_input'])`
    (gligen_inference.py:70-86, 346-349) with the yaml `params` as plain dicts (configs/*.yaml);
  * `set_alpha_scale` (gligen_inference.py:24-28) and `alpha_generator` (:31-66) - restated because the script itself
    needs `clip` / `omegaconf` to import (absent offline);
  * `sampler_inputs(...)`: the `input` dict / mask / x0 of `run()` (:384-430) from synthetic embeddings;
  * `prepare_batch(meta, batch, max_objs, encoder)` (:146-187): the box + text + image grounding batch, CLIP features from
    gligen_b200.clip_grounding.ClipGroundingEncoder.

Shared by bench.py, __graft_entry__.smoke() and the GPU parity tests, so the benchmark never imports the test tree.
"""
from __future__ import annotations

import importlib
from typing import Dict, Optional

import numpy as np
import torch

from .spec import NAMED_CONFIGS, SPATIAL_MAP_KEY, SPATIAL_TOKENIZERS, UNetConfig, synthetic_state_dict

TOKENIZER = {
    "text": ("ldm.modules.diffusionmodules.text_grounding_net.PositionNet", lambda c: dict(in_dim=c.tok_in_dim, out_dim=c.tok_out_dim)),
    "text_image": ("ldm.modules.diffusionmodules.text_image_grounding_net.PositionNet", lambda c: dict(in_dim=c.tok_in_dim, out_dim=c.tok_out_dim)),
    "keypoint": ("ldm.modules.diffusionmodules.keypoint_grounding_net.PositionNet", lambda c: dict(max_persons_per_image=c.max_persons, out_dim=c.tok_out_dim)),
}
for _t in SPATIAL_TOKENIZERS:
    TOKENIZER[_t] = (f"ldm.modules.diffusionmodules.{_t}_grounding_net.PositionNet",
                     (lambda c: dict(resize_input=c.tok_resize, out_dim=c.tok_out_dim, in_dim=c.sem_in_dim)) if _t == "sem" else
                     (lambda c: dict(resize_input=c.tok_resize, out_dim=c.tok_out_dim)))
GROUNDING_INPUT = {"text": "grounding_input.text_grounding_tokinzer_input.GroundingNetInput",
                   "text_image": "grounding_input.text_image_grounding_tokinzer_input.GroundingNetInput",
                   "keypoint": "grounding_input.keypoint_grounding_tokinzer_input.GroundingNetInput"}


GROUNDING_INPUT.update({t: f"grounding_input.{t}_grounding_tokinzer_input.GroundingNetInput" for t in SPATIAL_TOKENIZERS})
GROUNDING_DS_INPUT = {t: f"grounding_input.{t}_grounding_downsampler_input.GroundingDSInput" for t in SPATIAL_TOKENIZERS}


def downsampler_config(cfg: UNetConfig) -> Optional[Dict]:
    """The `grounding_downsampler` entry of configs/cc3m_hed.yaml, cc3m_canny.yaml, cc3m_depth.yaml, diode_normal.yaml, ade_sem.yaml."""
    if not cfg.ds_out_dim:
        return None
    par = dict(out_dim=cfg.ds_out_dim)
    if cfg.tokenizer != "hed":
        par["resize_input"] = cfg.ds_resize
    if cfg.tokenizer == "sem":
        par["in_dim"] = cfg.sem_in_dim
    return dict(target=f"ldm.modules.diffusionmodules.{cfg.tokenizer}_grounding_downsampler.GroundingDownsampler", params=par)


def model_config(cfg: UNetConfig) -> Dict:
    """The `config['model']` entry a GLIGEN checkpoint carries (configs/*.yaml -> config_dict)."""
    tgt, par = TOKENIZER[cfg.tokenizer]
    extra = {} if not cfg.ds_out_dim else dict(grounding_downsampler=downsampler_config(cfg))
    return dict(target="ldm.modules.diffusionmodules.openaimodel.UNetModel", params=dict(**extra, **dict(
        image_size=cfg.image_size, in_channels=cfg.in_channels, out_channels=cfg.out_channels, model_channels=cfg.model_channels,
        attention_resolutions=list(cfg.attention_resolutions), num_res_blocks=cfg.num_res_blocks, channel_mult=list(cfg.channel_mult),
        num_heads=cfg.num_heads, transformer_depth=1, context_dim=cfg.context_dim, fuser_type=cfg.fuser_type, use_checkpoint=True,
        inpaint_mode=cfg.inpaint_mode, grounding_tokenizer=dict(target=tgt, params=par(cfg)))))


def build_model(name, device="cuda:0", load_weights: bool = True, seed: int = 0):
    """(cfg, model) for a named configuration (gligen_b200.spec.NAMED_CONFIGS), seeded synthetic weights."""
    from ldm.util import instantiate_from_config
    cfg = NAMED_CONFIGS[name] if isinstance(name, str) else name
    model = instantiate_from_config(model_config(cfg)).to(device).eval()
    if load_weights:
        model.load_state_dict(synthetic_state_dict(cfg, seed=seed))
    model.grounding_tokenizer_input = instantiate_from_config(dict(target=GROUNDING_INPUT[cfg.tokenizer]))
    return cfg, model


def set_alpha_scale(model, alpha_scale):
    """gligen_inference.py:24-28 (type identity on the classes exported by ldm.modules.attention)."""
    from ldm.modules.attention import GatedCrossAttentionDense, GatedSelfAttentionDense
    for module in model.modules():
        if type(module) == GatedCrossAttentionDense or type(module) == GatedSelfAttentionDense:
            module.scale = alpha_scale


def alpha_generator(length, type=None):
    """gligen_inference.py:31-66: [1]*stage0 + linear decay over stage1 + [0]*stage2."""
    if type is None:
        type = [1, 0, 0]
    assert len(type) == 3 and abs(type[0] + type[1] + type[2] - 1) < 1e-9
    s0, s1 = int(type[0] * length), int(type[1] * length)
    s2 = length - s0 - s1
    decay = list(np.arange(start=0, stop=1, step=1 / s1)[::-1]) if s1 != 0 else []
    alphas = [1] * s0 + decay + [0] * s2
    assert len(alphas) == length
    return alphas


def to_device(d, device):
    if d is None:
        return None
    if isinstance(d, dict):
        return {k: to_device(v, device) for k, v in d.items()}
    return d.to(device)


def sampler_inputs(cfg: UNetConfig, model, tensors: Dict[str, torch.Tensor], batch: Dict[str, torch.Tensor]):
    """(input dict, mask, x0) as gligen_inference.run() builds them (:400-430); `tensors` / `batch` already on the
    device (gligen_b200.synth.make_inputs layout: x, context, uc, [z0] and the grounding batch)."""
    grounding = model.grounding_tokenizer_input.prepare(batch)
    extra = mask = x0 = None
    if cfg.inpaint_mode:
        from inpaint_mask_func import draw_masks_from_boxes
        mask = draw_masks_from_boxes(batch["boxes"], cfg.image_size).to(tensors["x"].device)
        x0 = tensors["z0"]
        extra = torch.cat([x0 * mask, mask], dim=1)
    gextra = None
    if cfg.spatial and cfg.ds_out_dim:          # gligen_inference.py:414-416: grounding_downsampler_input.prepare(batch)
        from ldm.util import instantiate_from_config
        gextra = instantiate_from_config(dict(target=GROUNDING_DS_INPUT[cfg.tokenizer])).prepare(batch)
    input = dict(x=tensors["x"].clone(), timesteps=None, context=tensors["context"], grounding_input=grounding,
                 inpainting_extra_input=extra, grounding_extra_input=gextra)
    return input, mask, x0


def prepare_batch(meta, batch: int = 1, max_objs: int = 30, encoder=None) -> Dict[str, torch.Tensor]:
    """gligen_inference.py:146-187 with the features from `encoder` (a gligen_b200.clip_grounding.ClipGroundingEncoder): all
    phrases in one text forward, all images in one image forward.  meta: "locations" (xyxy boxes), "phrases" and / or "images" (None entries allowed), optional "text_mask" /
    "image_mask" (a number or a per-object list, complete_mask :131-142).  Returns boxes, masks, text_masks, image_masks,
    text_embeddings, image_embeddings repeated over `batch`, on the encoder's device."""
    if encoder is None:
        raise ValueError("prepare_batch needs a ClipGroundingEncoder (its weights come from a CLIPModel state dict)")
    phrases, images = meta.get("phrases"), meta.get("images")
    images = [None] * len(phrases) if images is None else images
    phrases = [None] * len(images) if phrases is None else phrases
    locations = meta["locations"]
    assert len(locations) <= max_objs
    dev = encoder.device
    boxes = torch.zeros(max_objs, 4)
    masks = torch.zeros(max_objs)
    text_masks = torch.zeros(max_objs)
    image_masks = torch.zeros(max_objs)
    text_embeddings = torch.zeros(max_objs, encoder.text_dim, device=dev)
    image_embeddings = torch.zeros(max_objs, encoder.image_dim, device=dev)
    n = min(len(locations), len(phrases), len(images))     # the reference zips locations with the features (:168)
    t_idx = [i for i in range(n) if phrases[i] is not None]
    i_idx = [i for i in range(n) if images[i] is not None]
    if t_idx:
        text_embeddings[t_idx] = encoder.text_features(encoder.phrase_ids([phrases[i] for i in t_idx]))
        text_masks[t_idx] = 1
    if i_idx:
        image_embeddings[i_idx] = encoder.image_features(encoder.pixel_values([images[i] for i in i_idx]))
        image_masks[i_idx] = 1
    for idx, box in enumerate(locations[:n]):
        boxes[idx] = torch.tensor(box)
        masks[idx] = 1

    def complete_mask(has_mask):
        mask = torch.ones(1, max_objs)
        if has_mask is None:
            return mask
        if isinstance(has_mask, (int, float)):
            return mask * has_mask
        for idx, value in enumerate(has_mask):
            mask[0, idx] = value
        return mask

    out = {"boxes": boxes.unsqueeze(0).repeat(batch, 1, 1),
           "masks": masks.unsqueeze(0).repeat(batch, 1),
           "text_masks": text_masks.unsqueeze(0).repeat(batch, 1) * complete_mask(meta.get("text_mask")),
           "image_masks": image_masks.unsqueeze(0).repeat(batch, 1) * complete_mask(meta.get("image_mask")),
           "text_embeddings": text_embeddings.unsqueeze(0).repeat(batch, 1, 1),
           "image_embeddings": image_embeddings.unsqueeze(0).repeat(batch, 1, 1)}
    return {k: v.to(dev) for k, v in out.items()}
