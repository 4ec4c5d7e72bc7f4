"""Grounding features of `prepare_batch` (gligen_inference.py:101-117) on this repo's CLIP towers.

The reference builds `CLIPModel.from_pretrained("openai/clip-vit-large-patch14")` inside every `prepare_batch` call (:151-153) and
runs it in fp32 on one phrase or one image at a time.  `ClipGroundingEncoder` builds the text tower (gligen_b200/clip_text.py) and
the image tower (gligen_b200/clip_vision.py) once, from ONE CLIPModel state dict, and encodes all phrases of a call in one
forward and all images in another:
  * text_features(input_ids)     -> text_model_output.pooler_output ('before', :119-127).  Phrases are padded to the longest
    one: under the causal mask the pooled EOT state does not depend on what follows it, so this equals the one-at-a-time result.
  * image_features(pixel_values) -> image_embeds @ projection_matrix rescaled to norm 28.7 ('after_reproject', :110-116).
Tokenisation (CLIPTokenizer) and image preprocessing (CLIPProcessor) stay the library's; they are loaded lazily and only for
string phrases / image paths.  Compute is CUDA only (no CPU fallback)."""
from __future__ import annotations

from typing import Dict, Sequence, Union

import torch

from .clip_text import SD14_CLIP_TEXT, ClipTextConfig, ClipTextEngine
from .clip_vision import SD14_CLIP_VISION, ClipVisionConfig, ClipVisionEngine

VERSION = "openai/clip-vit-large-patch14"


class ClipGroundingEncoder:
    def __init__(self, state_dict: Dict[str, torch.Tensor], projection_matrix: Union[str, torch.Tensor] = "projection_matrix",
                 device="cuda:0", text_config: ClipTextConfig = SD14_CLIP_TEXT, vision_config: ClipVisionConfig = SD14_CLIP_VISION,
                 target_norm: float = 28.7, version: str = VERSION, ops=None):
        """state_dict: a CLIPModel state dict (`text_model.*`, `vision_model.*`, `visual_projection.weight`; other keys are ignored).
        projection_matrix: the [768, 768] tensor, or a path for torch.load (default: the CWD-relative file the reference reads).
        ops: the operator backend (default: CudaOps on `device`)."""
        if ops is None:
            dev = torch.device(device)
            if dev.type != "cuda":
                raise RuntimeError("gligen_b200 ClipGroundingEncoder runs only on a CUDA device (sm_90a kernels)")
            from .ops import CudaOps
            ops = CudaOps(dev)
        self.ops, self.device, self.version, self.target_norm = ops, ops.device, version, float(target_norm)
        P = torch.load(projection_matrix, map_location="cpu") if isinstance(projection_matrix, str) else projection_matrix
        assert P.shape == (vision_config.projection, vision_config.projection), P.shape
        self.P = P.detach().to(device=self.device, dtype=torch.float32).contiguous()
        self.text = ClipTextEngine(text_config, ops)
        self.text.load_state_dict(state_dict)
        self.vision = ClipVisionEngine(vision_config, ops)
        self.vision.load_state_dict(state_dict)
        self.text_dim, self.image_dim = text_config.width, vision_config.projection
        self._tokenizer = self._processor = None

    def text_features(self, input_ids: torch.Tensor) -> torch.Tensor:
        """int64 [n, L] (EOT = the highest id of each row, padded after it) -> pooler_output fp32 [n, text width]."""
        return self.text.forward(input_ids.to(self.device))[1]

    def image_features(self, pixel_values: torch.Tensor) -> torch.Tensor:
        """fp32 [n, 3, 224, 224] -> the 'after_reproject' features fp32 [n, projection], each of norm target_norm."""
        return self.vision.grounding_features(pixel_values.to(self.device, torch.float32), self.P, self.target_norm)

    # ---- host-side inputs: the library's tokenizer / processor for strings and paths ----------------------------------------
    def phrase_ids(self, phrases: Sequence[Union[str, torch.Tensor]]) -> torch.Tensor:
        """Strings (CLIPTokenizer, as FrozenCLIPEmbedder) or int64 id tensors -> one [n, L] batch padded with each row's EOT."""
        rows = []
        for p in phrases:
            if isinstance(p, str):
                if self._tokenizer is None:
                    from transformers import CLIPTokenizer
                    self._tokenizer = CLIPTokenizer.from_pretrained(self.version)
                p = self._tokenizer(p, truncation=True, max_length=self.text.cfg.max_length, return_tensors="pt")["input_ids"]
            rows.append(p.reshape(-1).to(torch.int64).cpu())
        L = max(r.numel() for r in rows)
        ids = torch.stack([torch.cat([r, r.max().expand(L - r.numel())]) for r in rows])
        return ids

    def pixel_values(self, images: Sequence[Union[str, torch.Tensor]]) -> torch.Tensor:
        """Image paths (PIL + CLIPProcessor, as gligen_inference.py:107-108) or fp32 [3, 224, 224] / [1, 3, 224, 224] tensors."""
        out = []
        for im in images:
            if isinstance(im, str):
                if self._processor is None:
                    from transformers import CLIPProcessor
                    self._processor = CLIPProcessor.from_pretrained(self.version)
                from PIL import Image
                im = self._processor(images=[Image.open(im).convert("RGB")], return_tensors="pt")["pixel_values"]
            out.append(im.reshape(3, *im.shape[-2:]).to(torch.float32).cpu())
        return torch.stack(out)

