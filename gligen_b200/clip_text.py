"""The CLIP text encoder behind `FrozenCLIPEmbedder` (SURVEY 8f-3) on this repo's kernels.

Reference call site: ldm/modules/encoders/modules.py:144-173 - `CLIPTextModel.from_pretrained("openai/clip-vit-large-patch14")`
run on the tokenizer's ids; `gligen_inference.py:377-380` encodes the prompt and the negative / empty prompt once per image.
The arithmetic lives in the third-party `transformers` package (pinned 4.19.2 by env_docker/Dockerfile:3, absent from the
reference tree): CLIPTextTransformer = token + position embeddings, 12 pre-LayerNorm blocks (causal self-attention with
12 heads of 64, MLP 768 -> 3072 -> 768 with quick_gelu), final LayerNorm; pooler_output = the final hidden state at the
position of the highest token id (the EOT token).  Restated in oracle/clip_oracle.py and pinned against the installed
transformers' CLIPTextModel.

Here: one gather kernel for the embeddings, the blocks of clip_encoder.py with the short-key attention kernel's causal
mask, the final LayerNorm with fp32 output.  bf16 activations and weights, fp32 accumulation / statistics, fp32 output.
"""
from __future__ import annotations

from collections import OrderedDict
from dataclasses import dataclass
from typing import Dict, Tuple

import torch

from .clip_encoder import ClipEncoderEngine, layer_param_shapes, synthetic_state_dict


@dataclass(frozen=True)
class ClipTextConfig:
    vocab_size: int = 49408
    width: int = 768
    layers: int = 12
    heads: int = 12
    ffn: int = 3072
    max_length: int = 77
    eps: float = 1e-5


SD14_CLIP_TEXT = ClipTextConfig()                                           # openai/clip-vit-large-patch14 text tower
TINY_CLIP_TEXT = ClipTextConfig(vocab_size=1000, width=128, layers=2, heads=2, ffn=512, max_length=77)
NAMED_CLIP_CONFIGS = {"sd14_clip_text": SD14_CLIP_TEXT, "tiny_clip_text": TINY_CLIP_TEXT}


def clip_text_param_shapes(cfg: ClipTextConfig, prefix: str = "transformer.") -> "OrderedDict[str, tuple]":
    """State-dict keys / shapes of FrozenCLIPEmbedder (`transformer` = transformers.CLIPTextModel), registration order."""
    p: "OrderedDict[str, tuple]" = OrderedDict()
    t = f"{prefix}text_model"
    p[f"{t}.embeddings.token_embedding.weight"] = (cfg.vocab_size, cfg.width)
    p[f"{t}.embeddings.position_embedding.weight"] = (cfg.max_length, cfg.width)
    p.update(layer_param_shapes(cfg, f"{t}."))
    p[f"{t}.final_layer_norm.weight"], p[f"{t}.final_layer_norm.bias"] = (cfg.width,), (cfg.width,)
    return p


def synthetic_clip_state_dict(cfg: ClipTextConfig, seed: int = 0, prefix: str = "transformer.") -> Dict[str, torch.Tensor]:
    """Seeded fp32 weights, the scheme of clip_encoder.synthetic_state_dict (CLIP's init); the token embedding carries the
    scaled-up massive channels."""
    return synthetic_state_dict(clip_text_param_shapes(cfg, prefix), seed, massive="token_embedding.weight")


def synthetic_token_ids(cfg: ClipTextConfig, B: int, seed: int = 0) -> torch.Tensor:
    """[B, max_length] int64 the way CLIPTokenizer pads: BOS (vocab-2), n words, EOT (vocab-1 = the highest id), then EOT padding."""
    g = torch.Generator(device="cpu").manual_seed(seed)
    ids = torch.full((B, cfg.max_length), cfg.vocab_size - 1, dtype=torch.int64)
    ids[:, 0] = cfg.vocab_size - 2
    for b in range(B):
        n = int(torch.randint(0, cfg.max_length - 2, (1,), generator=g))        # n = 0: the empty (negative) prompt
        ids[b, 1: 1 + n] = torch.randint(0, cfg.vocab_size - 2, (n,), generator=g)
    return ids


class ClipTextEngine(ClipEncoderEngine):
    def load_state_dict(self, sd: Dict[str, torch.Tensor]) -> None:
        """Accepts the keys of FrozenCLIPEmbedder (`transformer.text_model.*`), of CLIPTextModel (`text_model.*`) or bare; the
        `position_ids` buffer older transformers versions save is ignored."""
        key0 = next(k for k in sd if k.endswith("embeddings.token_embedding.weight"))
        pre = key0[: -len("embeddings.token_embedding.weight")]
        cfg, W = self.cfg, self.W
        W.clear()
        W["tok"], W["pos"] = self._f(sd[pre + "embeddings.token_embedding.weight"]), self._f(sd[pre + "embeddings.position_embedding.weight"])
        assert W["tok"].shape == (cfg.vocab_size, cfg.width) and W["pos"].shape[1] == cfg.width
        self._load_layers(sd, pre)
        W["lnf.g"], W["lnf.b"] = self._f(sd[pre + "final_layer_norm.weight"]), self._f(sd[pre + "final_layer_norm.bias"])
        self.loaded = True

    def _workspace(self, B: int, L: int) -> Dict[str, torch.Tensor]:
        key = B * 1000 + L
        if key not in self._ws:
            c, M = self.cfg, B * L
            e = lambda *s, dt=None: torch.empty(*s, device=self.dev, dtype=dt or self.adt)
            self._ws[key] = dict(ids=torch.zeros(B, L, device=self.dev, dtype=torch.int64), x=e(M, c.width), t=e(M, c.width), qkv=e(B, L, 3 * c.width),
                                 ao=e(B, L, c.width), h=e(M, c.ffn), z=e(B, L, c.width, dt=torch.float32))
        return self._ws[key]

    @torch.no_grad()
    def forward(self, input_ids: torch.Tensor) -> Tuple[torch.Tensor, torch.Tensor]:
        """input_ids int64 [B, L <= max_length] -> (last_hidden_state fp32 [B, L, width], pooler_output fp32 [B, width])."""
        assert self.loaded, "load_state_dict first"
        c, ops, W = self.cfg, self.ops, self.W
        B, L = input_ids.shape
        assert L <= c.max_length and L <= 128
        ws = self._workspace(B, L)
        ws["ids"].copy_(input_ids)
        x, z = ws["x"], ws["z"]
        ops.embed_tokens(ws["ids"], W["tok"], W["pos"], x)
        self._run_layers(ws, causal=True)
        ops.layernorm_rows_f32(x, z.view(B * L, c.width), W["lnf.g"], W["lnf.b"], c.eps)
        out = z.clone()
        # pooler_output: the hidden state at the (first) position of the highest token id = the EOT token (result read-out, host glue)
        pooled = out[torch.arange(B, device=out.device), ws["ids"].argmax(dim=-1)]
        return out, pooled
