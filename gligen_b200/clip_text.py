"""The CLIP text encoder behind `FrozenCLIPEmbedder` (SURVEY 8f-3) on this repo's kernels.

Reference call site: ldm/modules/encoders/modules.py:144-173 - `CLIPTextModel.from_pretrained("openai/clip-vit-large-patch14")`
run on the tokenizer's ids; `gligen_inference.py:377-380` encodes the prompt and the negative / empty prompt once per image.
The arithmetic lives in the third-party `transformers` package (pinned 4.19.2 by env_docker/Dockerfile:3, absent from the
reference tree): CLIPTextTransformer = token + position embeddings, 12 pre-LayerNorm blocks (causal self-attention with
12 heads of 64, MLP 768 -> 3072 -> 768 with quick_gelu), final LayerNorm; pooler_output = the final hidden state at the
position of the highest token id (the EOT token).  Restated in oracle/clip_oracle.py and pinned against the installed
transformers' CLIPTextModel.

Here: one gather kernel for the embeddings, LayerNorm rows, fused-QKV glg_gemm, the short-key attention kernel with
its causal mask, out-projection / fc2 GEMMs with the residual add in the epilogue, fc1 with the quick_gelu epilogue.
bf16 activations and weights, fp32 accumulation / statistics, fp32 output.
"""
from __future__ import annotations

from collections import OrderedDict
from dataclasses import dataclass
from typing import Dict, Tuple

import torch

ACT_QUICK_GELU = 3


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
    for i in range(cfg.layers):
        l = f"{t}.encoder.layers.{i}"
        for n in ("k_proj", "v_proj", "q_proj", "out_proj"):
            p[f"{l}.self_attn.{n}.weight"], p[f"{l}.self_attn.{n}.bias"] = (cfg.width, cfg.width), (cfg.width,)
        p[f"{l}.layer_norm1.weight"], p[f"{l}.layer_norm1.bias"] = (cfg.width,), (cfg.width,)
        p[f"{l}.mlp.fc1.weight"], p[f"{l}.mlp.fc1.bias"] = (cfg.ffn, cfg.width), (cfg.ffn,)
        p[f"{l}.mlp.fc2.weight"], p[f"{l}.mlp.fc2.bias"] = (cfg.width, cfg.ffn), (cfg.width,)
        p[f"{l}.layer_norm2.weight"], p[f"{l}.layer_norm2.bias"] = (cfg.width,), (cfg.width,)
    p[f"{t}.final_layer_norm.weight"], p[f"{t}.final_layer_norm.bias"] = (cfg.width,), (cfg.width,)
    return p


def synthetic_clip_state_dict(cfg: ClipTextConfig, seed: int = 0, prefix: str = "transformer.") -> Dict[str, torch.Tensor]:
    """Seeded fp32 weights: projections ~ N(0, 1/fan_in), embeddings ~ N(0, 0.02) / N(0, 0.01) (CLIP's init), norm scales 1 + 0.1 N,
    biases 0.05 N; a few embedding channels are scaled up like the massive channels trained CLIP towers show."""
    g = torch.Generator(device="cpu").manual_seed(seed)
    sd: Dict[str, torch.Tensor] = OrderedDict()
    for key, shape in clip_text_param_shapes(cfg, prefix).items():
        if key.endswith("token_embedding.weight"):
            t = torch.randn(shape, generator=g) * 0.02
            t[:, :: max(1, cfg.width // 4)] *= 8.0
        elif key.endswith("position_embedding.weight"):
            t = torch.randn(shape, generator=g) * 0.01
        elif key.endswith(".bias"):
            t = torch.randn(shape, generator=g) * 0.05
        elif len(shape) == 1:
            t = 1.0 + 0.1 * torch.randn(shape, generator=g)
        else:
            t = torch.randn(shape, generator=g) * (shape[1] ** -0.5)
        sd[key] = t
    return sd


def synthetic_token_ids(cfg: ClipTextConfig, B: int, seed: int = 0) -> torch.Tensor:
    """[B, max_length] int64 the way CLIPTokenizer pads: BOS (vocab-2), n words, EOT (vocab-1 = the highest id), then EOT padding."""
    g = torch.Generator(device="cpu").manual_seed(seed)
    ids = torch.full((B, cfg.max_length), cfg.vocab_size - 1, dtype=torch.int64)
    ids[:, 0] = cfg.vocab_size - 2
    for b in range(B):
        n = int(torch.randint(0, cfg.max_length - 2, (1,), generator=g))        # n = 0: the empty (negative) prompt
        ids[b, 1: 1 + n] = torch.randint(0, cfg.vocab_size - 2, (n,), generator=g)
    return ids


class ClipTextEngine:
    def __init__(self, cfg: ClipTextConfig, ops):
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
        """Accepts the keys of FrozenCLIPEmbedder (`transformer.text_model.*`), of CLIPTextModel (`text_model.*`) or bare; the
        `position_ids` buffer older transformers versions save is ignored."""
        key0 = next(k for k in sd if k.endswith("embeddings.token_embedding.weight"))
        pre = key0[: -len("embeddings.token_embedding.weight")]
        cfg, W = self.cfg, self.W
        W.clear()
        W["tok"], W["pos"] = self._f(sd[pre + "embeddings.token_embedding.weight"]), self._f(sd[pre + "embeddings.position_embedding.weight"])
        assert W["tok"].shape == (cfg.vocab_size, cfg.width) and W["pos"].shape[1] == cfg.width
        for i in range(cfg.layers):
            l = f"{pre}encoder.layers.{i}"
            W[f"{i}.ln1.g"], W[f"{i}.ln1.b"] = self._f(sd[f"{l}.layer_norm1.weight"]), self._f(sd[f"{l}.layer_norm1.bias"])
            W[f"{i}.ln2.g"], W[f"{i}.ln2.b"] = self._f(sd[f"{l}.layer_norm2.weight"]), self._f(sd[f"{l}.layer_norm2.bias"])
            W[f"{i}.qkv.w"] = self._a(torch.cat([sd[f"{l}.self_attn.{n}_proj.weight"] for n in ("q", "k", "v")], dim=0))
            W[f"{i}.qkv.b"] = self._f(torch.cat([sd[f"{l}.self_attn.{n}_proj.bias"] for n in ("q", "k", "v")], dim=0))
            W[f"{i}.out.w"], W[f"{i}.out.b"] = self._a(sd[f"{l}.self_attn.out_proj.weight"]), self._f(sd[f"{l}.self_attn.out_proj.bias"])
            W[f"{i}.fc1.w"], W[f"{i}.fc1.b"] = self._a(sd[f"{l}.mlp.fc1.weight"]), self._f(sd[f"{l}.mlp.fc1.bias"])
            W[f"{i}.fc2.w"], W[f"{i}.fc2.b"] = self._a(sd[f"{l}.mlp.fc2.weight"]), self._f(sd[f"{l}.mlp.fc2.bias"])
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
        x, t, qkv, ao, h, z = ws["x"], ws["t"], ws["qkv"], ws["ao"], ws["h"], ws["z"]
        C, d = c.width, c.width // c.heads
        ops.embed_tokens(ws["ids"], W["tok"], W["pos"], x)
        for i in range(c.layers):
            ops.layernorm_rows(x, t, W[f"{i}.ln1.g"], W[f"{i}.ln1.b"], C, c.eps)
            ops.gemm(t, W[f"{i}.qkv.w"], qkv.view(B * L, 3 * C), bias=W[f"{i}.qkv.b"])
            ops.attention(qkv[:, :, :C], qkv[:, :, C: 2 * C], qkv[:, :, 2 * C:], ao, c.heads, d, causal=True)
            ops.gemm(ao.view(B * L, C), W[f"{i}.out.w"], x, bias=W[f"{i}.out.b"], residual=x)
            ops.layernorm_rows(x, t, W[f"{i}.ln2.g"], W[f"{i}.ln2.b"], C, c.eps)
            ops.gemm(t, W[f"{i}.fc1.w"], h, bias=W[f"{i}.fc1.b"], act=ACT_QUICK_GELU)
            ops.gemm(h, W[f"{i}.fc2.w"], x, bias=W[f"{i}.fc2.b"], residual=x)
        ops.layernorm_rows_f32(x, z.view(B * L, C), W["lnf.g"], W["lnf.b"], c.eps)
        out = z.clone()
        # pooler_output: the hidden state at the (first) position of the highest token id = the EOT token (result read-out, host glue)
        pooled = out[torch.arange(B, device=out.device), ws["ids"].argmax(dim=-1)]
        return out, pooled
