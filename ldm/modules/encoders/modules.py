"""`FrozenCLIPEmbedder` at the reference's import path (ldm/modules/encoders/modules.py:144-173; located by string through
`instantiate_from_config(config['text_encoder'])`, gligen_inference.py:77), with the CLIP text transformer on this repo's sm_90a
kernels (gligen_b200/clip_text.py).  Same surface: `FrozenCLIPEmbedder(version, device, max_length)`, `.to(device).eval()`,
`load_state_dict(saved_ckpt["text_encoder"])` with the `transformer.text_model.*` keys of transformers' CLIPTextModel,
`encode(text, return_pooler_output=False)` / `forward(...)` -> last_hidden_state [B, 77, 768] (, pooler_output).

The tokenizer is host-side string processing and stays the library's (`transformers.CLIPTokenizer`, loaded lazily so that
constructing the module needs no vocabulary files); `encode_tokens(input_ids)` is the same call on ready-made ids.
Weights are NOT fetched here: the reference's `CLIPTextModel.from_pretrained(version)` download is replaced by the checkpoint's
own `text_encoder` state dict, which gligen_inference.load_ckpt loads right after construction (:83) - until then the parameters
are zeros.  Compute is CUDA only (no CPU fallback).  Other names of the reference module (FrozenCLIPTextEmbedder, BERTEmbedder,
SpatialRescaler, ...) resolve to the reference when a checkout follows this repo on sys.path.
"""
import torch
import torch.nn as nn

from gligen_b200 import _overlay
from gligen_b200.clip_text import SD14_CLIP_TEXT, ClipTextConfig, ClipTextEngine, clip_text_param_shapes
from ldm.modules.attention import attach_params


class AbstractEncoder(nn.Module):
    def encode(self, *args, **kwargs):
        raise NotImplementedError


class FrozenCLIPEmbedder(AbstractEncoder):
    """Uses the CLIP transformer encoder for text (weights: transformers CLIPTextModel layout)."""

    def __init__(self, version="openai/clip-vit-large-patch14", device="cuda", max_length=77, text_config=None):
        """text_config (not in the reference): a ClipTextConfig, the name of one (gligen_b200.clip_text.NAMED_CLIP_CONFIGS) or a dict
        of its fields - for towers other than clip-vit-large-patch14's (tests use a small one)."""
        super().__init__()
        self.version, self.device, self.max_length = version, device, max_length
        if isinstance(text_config, str):
            from gligen_b200.clip_text import NAMED_CLIP_CONFIGS
            text_config = NAMED_CLIP_CONFIGS[text_config]
        elif isinstance(text_config, dict):
            text_config = ClipTextConfig(**text_config)
        self.cfg = text_config or SD14_CLIP_TEXT
        self._tokenizer = None
        attach_params(self, clip_text_param_shapes(self.cfg, "transformer."), "")
        self._engine, self._stale = None, True

    # ---- weights ----------------------------------------------------------------------------------------------------
    def freeze(self):
        return self.eval()

    def load_state_dict(self, state_dict, strict=True, **kw):
        sd = {k: v for k, v in state_dict.items() if not k.endswith("embeddings.position_ids")}     # buffer saved by transformers < 4.31
        out = super().load_state_dict(sd, strict=strict, **kw)
        self._stale = True
        return out

    def _apply(self, fn, *a, **kw):
        out = super()._apply(fn, *a, **kw)
        self._engine, self._stale = None, True
        return out

    def engine(self) -> ClipTextEngine:
        dev = self.transformer.text_model.final_layer_norm.weight.device
        if dev.type != "cuda":
            raise RuntimeError("gligen_b200 FrozenCLIPEmbedder runs only on a CUDA device (sm_90a kernels); call .to('cuda') first")
        if self._engine is None:
            from gligen_b200.ops import CudaOps
            self._engine = ClipTextEngine(self.cfg, CudaOps(dev))
            self._stale = True
        if self._stale:
            self._engine.load_state_dict(self.state_dict())
            self._stale = False
        return self._engine

    # ---- the reference's call surface ---------------------------------------------------------------------------------
    @property
    def tokenizer(self):
        if self._tokenizer is None:
            from transformers import CLIPTokenizer
            self._tokenizer = CLIPTokenizer.from_pretrained(self.version)
        return self._tokenizer

    @torch.no_grad()
    def encode_tokens(self, input_ids, return_pooler_output=False):
        dev = self.transformer.text_model.final_layer_norm.weight.device
        z, pooled = self.engine().forward(input_ids.to(dev))
        return (z, pooled) if return_pooler_output else z

    def forward(self, text, return_pooler_output=False):
        batch_encoding = self.tokenizer(text, truncation=True, max_length=self.max_length, return_length=True,
                                        return_overflowing_tokens=False, padding="max_length", return_tensors="pt")
        return self.encode_tokens(batch_encoding["input_ids"], return_pooler_output)

    def encode(self, text, return_pooler_output=False):
        return self(text, return_pooler_output)


# names this drop-in does not define resolve to the reference module of the same name when a reference checkout
# follows this repo on sys.path (gligen_b200/_overlay.py)
__getattr__ = _overlay.fallback(__name__, __file__)
