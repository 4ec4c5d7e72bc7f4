"""UNet configuration, block schedule and parameter inventory for the GLIGEN denoiser.

This module is pure host-side bookkeeping (no torch ops on the hot path).  It restates
*structure* only: which blocks exist, their channel counts, and the state-dict key of every
parameter, so that a reference checkpoint loads verbatim.

Reference: ldm/modules/diffusionmodules/openaimodel.py:238-397 (UNetModel.__init__),
ldm/modules/attention.py:303-376, ldm/modules/diffusionmodules/{text,text_image,keypoint}_grounding_net.py.
"""
from __future__ import annotations

from collections import OrderedDict
from dataclasses import dataclass, field, replace
from typing import Dict, List, Optional, Tuple

import torch


@dataclass(frozen=True)
class UNetConfig:
    image_size: int = 64
    in_channels: int = 4
    out_channels: int = 4
    model_channels: int = 320
    num_res_blocks: int = 2
    attention_resolutions: Tuple[int, ...] = (4, 2, 1)
    channel_mult: Tuple[int, ...] = (1, 2, 4, 4)
    num_heads: int = 8
    transformer_depth: int = 1
    context_dim: int = 768
    # "gatedSA" (every shipped config), "gatedCA" (cross-attention to the grounding tokens) or "gatedSA2" (self-attention whose
    # grounding rows are resampled onto the visual grid), reference attention.py:190-297
    fuser_type: str = "gatedSA"
    inpaint_mode: bool = False
    # grounding tokenizer: "text" | "text_image" | "keypoint" (discrete objects) or one of SPATIAL_TOKENIZERS
    # ("hed" | "canny" | "depth" | "normal" | "sem": a ConvNeXt-tiny over a spatial map, SURVEY 8f-4)
    tokenizer: str = "text"
    tok_in_dim: int = 768          # text / text_image: CLIP feature dim
    tok_out_dim: int = 768
    tok_hidden: int = 512          # hard-coded 512 in the reference PositionNets
    fourier_freqs: int = 8
    max_persons: int = 8           # keypoint only
    # spatial-map modalities (configs/cc3m_hed.yaml, cc3m_canny.yaml, cc3m_depth.yaml, diode_normal.yaml, ade_sem.yaml)
    tok_resize: int = 256          # PositionNet(resize_input=...): the map is resampled to this size; tokens = (resize / 32)^2
    sem_in_dim: int = 152          # sem only: one-hot classes (PositionNet / GroundingDownsampler in_dim)
    ds_out_dim: int = 0            # GroundingDownsampler.out_dim: extra first-conv channels (0 = no downsampler)
    ds_resize: int = 256           # GroundingDownsampler(resize_input=...) (hed: unused, bicubic straight to the latent size)

    @property
    def time_embed_dim(self) -> int:
        return self.model_channels * 4

    @property
    def first_conv_in(self) -> int:
        # openaimodel.py:293-304
        if self.inpaint_mode:
            return self.in_channels * 2 + 1 + self.ds_out_dim
        return self.in_channels + self.ds_out_dim

    @property
    def spatial(self) -> bool:
        return self.tokenizer in SPATIAL_TOKENIZERS

    @property
    def map_channels(self) -> int:
        """Channels of the spatial conditioning map as the dataset delivers it (grey maps are replicated to RGB)."""
        return self.sem_in_dim if self.tokenizer == "sem" else 3

    @property
    def spatial_tokens(self) -> int:
        return (self.tok_resize // 32) ** 2

    @property
    def position_dim(self) -> int:
        ncoord = 2 if self.tokenizer == "keypoint" else 4
        return self.fourier_freqs * 2 * ncoord

    @property
    def tok_feat_dim(self) -> int:
        """Width of the non-positional part fed to the PositionNet MLP."""
        return self.tok_out_dim if self.tokenizer == "keypoint" else self.tok_in_dim

    def tokens_per_sample(self, max_objs: int) -> int:
        if self.spatial:
            return self.spatial_tokens
        return 2 * max_objs if self.tokenizer == "text_image" else max_objs


SPATIAL_TOKENIZERS = ("hed", "canny", "depth", "normal", "sem")
#: kwarg name of the map in the tokenizer's forward / GroundingNetInput (grounding_input/*_grounding_tokinzer_input.py:19-26)
SPATIAL_MAP_KEY = {"hed": "hed_edge", "canny": "canny_edge", "depth": "depth", "normal": "normal", "sem": "sem"}
CONVNEXT_TINY_DEPTHS, CONVNEXT_TINY_DIMS = (3, 3, 9, 3), (96, 192, 384, 768)


SD14_BOX_TEXT = UNetConfig()
SD14_BOX_TEXT_IMAGE = replace(SD14_BOX_TEXT, tokenizer="text_image")
SD14_KEYPOINT = replace(SD14_BOX_TEXT, tokenizer="keypoint")
SD14_INPAINT_BOX_TEXT = replace(SD14_BOX_TEXT, inpaint_mode=True)
# Small structurally-identical model used by fast parity tests (every width still a multiple of 64
# so that the tensor-core tiles apply; latent 16x16 -> levels 16/8/4/2).
TINY = UNetConfig(image_size=16, model_channels=64, context_dim=128, tok_in_dim=128, tok_out_dim=128)
TINY_TEXT_IMAGE = replace(TINY, tokenizer="text_image")
TINY_KEYPOINT = replace(TINY, tokenizer="keypoint", max_persons=2)
TINY_INPAINT = replace(TINY, inpaint_mode=True)
# spatial-map modalities: the shipped configs (out_dim 768, resize 256 -> 64 tokens; hed adds 1 first-conv channel, the rest 8)
SD14_HED = replace(SD14_BOX_TEXT, tokenizer="hed", ds_out_dim=1)
SD14_CANNY = replace(SD14_BOX_TEXT, tokenizer="canny", ds_out_dim=8)
SD14_DEPTH = replace(SD14_BOX_TEXT, tokenizer="depth", ds_out_dim=8)
SD14_NORMAL = replace(SD14_BOX_TEXT, tokenizer="normal", ds_out_dim=8)
SD14_SEM = replace(SD14_BOX_TEXT, tokenizer="sem", ds_out_dim=8)
# tiny UNets behind the real ConvNeXt-tiny (the backbone has one size); 128-pixel tokenizer input -> 16 tokens
TINY_HED = replace(TINY, tokenizer="hed", ds_out_dim=1, tok_resize=128, image_size=64)     # hed: bicubic straight to 64 x 64 (hard-coded in the reference)
TINY_CANNY = replace(TINY, tokenizer="canny", ds_out_dim=8, tok_resize=128, ds_resize=64)
TINY_DEPTH = replace(TINY, tokenizer="depth", ds_out_dim=8, tok_resize=128, ds_resize=64)
TINY_NORMAL = replace(TINY, tokenizer="normal", ds_out_dim=8, tok_resize=128, ds_resize=64)
TINY_SEM = replace(TINY, tokenizer="sem", ds_out_dim=8, tok_resize=128, ds_resize=64, sem_in_dim=24)
# the other two fusers the reference builds (BasicTransformerBlock, attention.py:313-321).  gatedCA: any token count (keypoint with
# 8 persons = 136 tokens takes the long-key attention kernel); gatedSA2 needs a square token count: the spatial tokenizers' 16 / 64
SD14_BOX_TEXT_GATED_CA = replace(SD14_BOX_TEXT, fuser_type="gatedCA")
SD14_HED_GATED_SA2 = replace(SD14_HED, fuser_type="gatedSA2")
TINY_GATED_CA = replace(TINY, fuser_type="gatedCA")
TINY_TEXT_IMAGE_GATED_CA = replace(TINY_TEXT_IMAGE, fuser_type="gatedCA")
TINY_KEYPOINT_GATED_CA = replace(TINY_KEYPOINT, fuser_type="gatedCA", max_persons=8)
TINY_HED_GATED_SA2 = replace(TINY_HED, fuser_type="gatedSA2")
FUSER_TYPES = ("gatedSA", "gatedCA", "gatedSA2")
# small 320-channel models for scheduled-sampling loops: the reference's restore_first_conv_from_SD builds SD's 4 -> 320 first conv
# whatever the model (openaimodel.py:400-413), so a loop with alpha = 0 steps needs model_channels = 320.  Not in NAMED_CONFIGS.
SAMPLING_GATED_CA = replace(TINY_GATED_CA, model_channels=320, channel_mult=(1, 1), num_res_blocks=1, attention_resolutions=(1, 2))
SAMPLING_HED_GATED_SA2 = replace(TINY_HED_GATED_SA2, model_channels=320, channel_mult=(1, 1, 1), num_res_blocks=1, attention_resolutions=(2, 4))

NAMED_CONFIGS = {
    "sd14_box_text": SD14_BOX_TEXT,
    "sd14_box_text_image": SD14_BOX_TEXT_IMAGE,
    "sd14_keypoint": SD14_KEYPOINT,
    "sd14_inpaint_box_text": SD14_INPAINT_BOX_TEXT,
    "tiny": TINY,
    "tiny_text_image": TINY_TEXT_IMAGE,
    "tiny_keypoint": TINY_KEYPOINT,
    "tiny_inpaint": TINY_INPAINT,
    "sd14_hed": SD14_HED, "sd14_canny": SD14_CANNY, "sd14_depth": SD14_DEPTH, "sd14_normal": SD14_NORMAL, "sd14_sem": SD14_SEM,
    "tiny_hed": TINY_HED, "tiny_canny": TINY_CANNY, "tiny_depth": TINY_DEPTH, "tiny_normal": TINY_NORMAL, "tiny_sem": TINY_SEM,
    "sd14_box_text_gated_ca": SD14_BOX_TEXT_GATED_CA, "sd14_hed_gated_sa2": SD14_HED_GATED_SA2,
    "tiny_gated_ca": TINY_GATED_CA, "tiny_text_image_gated_ca": TINY_TEXT_IMAGE_GATED_CA, "tiny_keypoint_gated_ca": TINY_KEYPOINT_GATED_CA,
    "tiny_hed_gated_sa2": TINY_HED_GATED_SA2,
}


# ----------------------------------------------------------------------------------------------
# Block schedule
# ----------------------------------------------------------------------------------------------
@dataclass
class Layer:
    kind: str                 # "conv_in" | "res" | "st" | "down" | "up"
    prefix: str               # state-dict prefix, e.g. "input_blocks.1.0"
    cin: int = 0
    cout: int = 0
    heads: int = 0
    d_head: int = 0


@dataclass
class Block:
    where: str                # "in" | "mid" | "out"
    index: int
    layers: List[Layer] = field(default_factory=list)
    ds: int = 1               # downsample factor of the block's *input* resolution
    skip_ch: int = 0          # (output blocks) channels popped from the skip stack
    out_ch: int = 0
    out_ds: int = 1


def block_schedule(cfg: UNetConfig) -> List[Block]:
    """Enumerate input/middle/output blocks exactly as openaimodel.py:305-388 builds them."""
    mc = cfg.model_channels
    blocks: List[Block] = []
    b0 = Block("in", 0, [Layer("conv_in", "input_blocks.0.0", cfg.first_conv_in, mc)], ds=1, out_ch=mc, out_ds=1)
    blocks.append(b0)
    chans = [mc]
    ch, ds = mc, 1
    idx = 1
    for level, mult in enumerate(cfg.channel_mult):
        for _ in range(cfg.num_res_blocks):
            blk = Block("in", idx, ds=ds)
            blk.layers.append(Layer("res", f"input_blocks.{idx}.0", ch, mult * mc))
            ch = mult * mc
            if ds in cfg.attention_resolutions:
                blk.layers.append(Layer("st", f"input_blocks.{idx}.1", ch, ch, cfg.num_heads, ch // cfg.num_heads))
            blk.out_ch, blk.out_ds = ch, ds
            blocks.append(blk)
            chans.append(ch)
            idx += 1
        if level != len(cfg.channel_mult) - 1:
            blk = Block("in", idx, [Layer("down", f"input_blocks.{idx}.0", ch, ch)], ds=ds, out_ch=ch, out_ds=ds * 2)
            blocks.append(blk)
            chans.append(ch)
            ds *= 2
            idx += 1
    mid = Block("mid", 0, ds=ds, out_ch=ch, out_ds=ds)
    mid.layers = [
        Layer("res", "middle_block.0", ch, ch),
        Layer("st", "middle_block.1", ch, ch, cfg.num_heads, ch // cfg.num_heads),
        Layer("res", "middle_block.2", ch, ch),
    ]
    blocks.append(mid)
    oidx = 0
    for level, mult in list(enumerate(cfg.channel_mult))[::-1]:
        for i in range(cfg.num_res_blocks + 1):
            ich = chans.pop()
            blk = Block("out", oidx, ds=ds, skip_ch=ich)
            blk.layers.append(Layer("res", f"output_blocks.{oidx}.0", ch + ich, mc * mult))
            ch = mc * mult
            j = 1
            if ds in cfg.attention_resolutions:
                blk.layers.append(Layer("st", f"output_blocks.{oidx}.{j}", ch, ch, cfg.num_heads, ch // cfg.num_heads))
                j += 1
            out_ds = ds
            if level and i == cfg.num_res_blocks:
                blk.layers.append(Layer("up", f"output_blocks.{oidx}.{j}", ch, ch))
                out_ds = ds // 2
            blk.out_ch, blk.out_ds = ch, out_ds
            blocks.append(blk)
            ds = out_ds
            oidx += 1
    return blocks


# ----------------------------------------------------------------------------------------------
# Parameter inventory (state-dict keys and shapes)
# ----------------------------------------------------------------------------------------------
def _attn_params(p: "OrderedDict[str, tuple]", prefix: str, qdim: int, kdim: int) -> None:
    p[f"{prefix}.to_q.weight"] = (qdim, qdim)
    p[f"{prefix}.to_k.weight"] = (qdim, kdim)
    p[f"{prefix}.to_v.weight"] = (qdim, kdim)
    p[f"{prefix}.to_out.0.weight"] = (qdim, qdim)
    p[f"{prefix}.to_out.0.bias"] = (qdim,)


def _ff_params(p, prefix: str, dim: int) -> None:
    p[f"{prefix}.net.0.proj.weight"] = (dim * 8, dim)
    p[f"{prefix}.net.0.proj.bias"] = (dim * 8,)
    p[f"{prefix}.net.2.weight"] = (dim, dim * 4)
    p[f"{prefix}.net.2.bias"] = (dim,)


def _norm_params(p, prefix: str, dim: int) -> None:
    p[f"{prefix}.weight"] = (dim,)
    p[f"{prefix}.bias"] = (dim,)


def _mlp3(p, prefix: str, din: int, hidden: int, dout: int) -> None:
    for i, (a, b) in zip((0, 2, 4), ((din, hidden), (hidden, hidden), (hidden, dout))):
        p[f"{prefix}.{i}.weight"] = (b, a)
        p[f"{prefix}.{i}.bias"] = (b,)


def unet_param_shapes(cfg: UNetConfig) -> "OrderedDict[str, tuple]":
    """All parameters of UNetModel in registration order (matches reference state_dict() order)."""
    p: "OrderedDict[str, tuple]" = OrderedDict()
    mc, ted = cfg.model_channels, cfg.time_embed_dim
    p["time_embed.0.weight"] = (ted, mc)
    p["time_embed.0.bias"] = (ted,)
    p["time_embed.2.weight"] = (ted, ted)
    p["time_embed.2.bias"] = (ted,)

    def res(prefix, cin, cout):
        _norm_params(p, f"{prefix}.in_layers.0", cin)
        p[f"{prefix}.in_layers.2.weight"] = (cout, cin, 3, 3)
        p[f"{prefix}.in_layers.2.bias"] = (cout,)
        p[f"{prefix}.emb_layers.1.weight"] = (cout, ted)
        p[f"{prefix}.emb_layers.1.bias"] = (cout,)
        _norm_params(p, f"{prefix}.out_layers.0", cout)
        p[f"{prefix}.out_layers.3.weight"] = (cout, cout, 3, 3)
        p[f"{prefix}.out_layers.3.bias"] = (cout,)
        if cin != cout:
            p[f"{prefix}.skip_connection.weight"] = (cout, cin, 1, 1)
            p[f"{prefix}.skip_connection.bias"] = (cout,)

    def st(prefix, c):
        _norm_params(p, f"{prefix}.norm", c)
        p[f"{prefix}.proj_in.weight"] = (c, c, 1, 1)
        p[f"{prefix}.proj_in.bias"] = (c,)
        for d in range(cfg.transformer_depth):
            tb = f"{prefix}.transformer_blocks.{d}"
            _attn_params(p, f"{tb}.attn1", c, c)
            _ff_params(p, f"{tb}.ff", c)
            _attn_params(p, f"{tb}.attn2", c, cfg.context_dim)
            _norm_params(p, f"{tb}.norm1", c)
            _norm_params(p, f"{tb}.norm2", c)
            _norm_params(p, f"{tb}.norm3", c)
            fu = f"{tb}.fuser"
            p[f"{fu}.alpha_attn"] = ()
            p[f"{fu}.alpha_dense"] = ()
            if cfg.fuser_type == "gatedCA":          # GatedCrossAttentionDense: no linear, K / V project the tokens themselves
                _attn_params(p, f"{fu}.attn", c, cfg.context_dim)
            else:                                     # GatedSelfAttentionDense / GatedSelfAttentionDense2: the same parameters
                p[f"{fu}.linear.weight"] = (c, cfg.context_dim)
                p[f"{fu}.linear.bias"] = (c,)
                _attn_params(p, f"{fu}.attn", c, c)
            _ff_params(p, f"{fu}.ff", c)
            _norm_params(p, f"{fu}.norm1", c)
            _norm_params(p, f"{fu}.norm2", c)
        p[f"{prefix}.proj_out.weight"] = (c, c, 1, 1)
        p[f"{prefix}.proj_out.bias"] = (c,)

    for blk in block_schedule(cfg):
        for ly in blk.layers:
            if ly.kind == "conv_in":
                p[f"{ly.prefix}.weight"] = (ly.cout, ly.cin, 3, 3)
                p[f"{ly.prefix}.bias"] = (ly.cout,)
            elif ly.kind == "res":
                res(ly.prefix, ly.cin, ly.cout)
            elif ly.kind == "st":
                st(ly.prefix, ly.cin)
            elif ly.kind == "down":
                p[f"{ly.prefix}.op.weight"] = (ly.cout, ly.cin, 3, 3)
                p[f"{ly.prefix}.op.bias"] = (ly.cout,)
            elif ly.kind == "up":
                p[f"{ly.prefix}.conv.weight"] = (ly.cout, ly.cin, 3, 3)
                p[f"{ly.prefix}.conv.bias"] = (ly.cout,)
    _norm_params(p, "out.0", mc)
    p["out.2.weight"] = (cfg.out_channels, mc, 3, 3)
    p["out.2.bias"] = (cfg.out_channels,)

    pn = "position_net"
    din = cfg.tok_feat_dim + cfg.position_dim
    if cfg.tokenizer == "text":
        p[f"{pn}.null_positive_feature"] = (cfg.tok_in_dim,)
        p[f"{pn}.null_position_feature"] = (cfg.position_dim,)
        _mlp3(p, f"{pn}.linears", din, cfg.tok_hidden, cfg.tok_out_dim)
    elif cfg.tokenizer == "text_image":
        p[f"{pn}.null_text_feature"] = (cfg.tok_in_dim,)
        p[f"{pn}.null_image_feature"] = (cfg.tok_in_dim,)
        p[f"{pn}.null_position_feature"] = (cfg.position_dim,)
        _mlp3(p, f"{pn}.linears_text", din, cfg.tok_hidden, cfg.tok_out_dim)
        _mlp3(p, f"{pn}.linears_image", din, cfg.tok_hidden, cfg.tok_out_dim)
    elif cfg.tokenizer == "keypoint":
        p[f"{pn}.person_embeddings"] = (cfg.max_persons, cfg.tok_out_dim)
        p[f"{pn}.keypoint_embeddings"] = (17, cfg.tok_out_dim)
        p[f"{pn}.null_person_feature"] = (cfg.tok_out_dim,)
        p[f"{pn}.null_xy_feature"] = (cfg.position_dim,)
        _mlp3(p, f"{pn}.linears", din, cfg.tok_hidden, cfg.tok_out_dim)
    elif cfg.spatial:
        # hed_grounding_net.py:13-35 (canny / depth / normal identical; sem adds in_conv, sem_grounding_net.py:21)
        if cfg.tokenizer == "sem":
            p[f"{pn}.in_conv.weight"] = (3, cfg.sem_in_dim, 3, 3)
            p[f"{pn}.in_conv.bias"] = (3,)
        p.update(convnext_tiny_param_shapes(f"{pn}.convnext_tiny_backbone"))
        p[f"{pn}.pos_embedding"] = (1, cfg.spatial_tokens, CONVNEXT_TINY_DIMS[-1])
        _mlp3(p, f"{pn}.linears", CONVNEXT_TINY_DIMS[-1], cfg.tok_hidden, cfg.tok_out_dim)
        p[f"{pn}.null_feature"] = (CONVNEXT_TINY_DIMS[-1],)
    else:
        raise ValueError(f"unknown tokenizer {cfg.tokenizer!r}")
    p.update(downsampler_param_shapes(cfg))
    return p


def convnext_tiny_param_shapes(prefix: str) -> "OrderedDict[str, tuple]":
    """ConvNeXt-tiny without head (convnext.py:53-94, depths 3/3/9/3, dims 96/192/384/768), registration order."""
    p: "OrderedDict[str, tuple]" = OrderedDict()
    dims, depths = CONVNEXT_TINY_DIMS, CONVNEXT_TINY_DEPTHS
    d = f"{prefix}.downsample_layers"
    p[f"{d}.0.0.weight"], p[f"{d}.0.0.bias"] = (dims[0], 3, 4, 4), (dims[0],)
    p[f"{d}.0.1.weight"], p[f"{d}.0.1.bias"] = (dims[0],), (dims[0],)
    for i in range(3):
        p[f"{d}.{i + 1}.0.weight"], p[f"{d}.{i + 1}.0.bias"] = (dims[i],), (dims[i],)
        p[f"{d}.{i + 1}.1.weight"], p[f"{d}.{i + 1}.1.bias"] = (dims[i + 1], dims[i], 2, 2), (dims[i + 1],)
    for i in range(4):
        for j in range(depths[i]):
            b, c = f"{prefix}.stages.{i}.{j}", dims[i]
            p[f"{b}.gamma"] = (c,)
            p[f"{b}.dwconv.weight"], p[f"{b}.dwconv.bias"] = (c, 1, 7, 7), (c,)
            p[f"{b}.norm.weight"], p[f"{b}.norm.bias"] = (c,), (c,)
            p[f"{b}.pwconv1.weight"], p[f"{b}.pwconv1.bias"] = (4 * c, c), (4 * c,)
            p[f"{b}.pwconv2.weight"], p[f"{b}.pwconv2.bias"] = (c, 4 * c), (c,)
    return p


def downsampler_param_shapes(cfg: UNetConfig) -> "OrderedDict[str, tuple]":
    """GroundingDownsampler parameters (`downsample_net.*`): hed has none (bicubic only, hed_grounding_downsampler.py:9-21);
    canny / depth 1->4->out, normal 3->4->out, sem in_dim->16->out, all Conv2d(k=4, s=2, p=1)."""
    p: "OrderedDict[str, tuple]" = OrderedDict()
    if not cfg.spatial or cfg.tokenizer == "hed":
        return p
    cin, mid = {"canny": (1, 4), "depth": (1, 4), "normal": (3, 4), "sem": (cfg.sem_in_dim, 16)}[cfg.tokenizer]
    p["downsample_net.layers.0.weight"], p["downsample_net.layers.0.bias"] = (mid, cin, 4, 4), (mid,)
    p["downsample_net.layers.2.weight"], p["downsample_net.layers.2.bias"] = (cfg.ds_out_dim, mid, 4, 4), (cfg.ds_out_dim,)
    return p


def synthetic_state_dict(cfg: UNetConfig, seed: int = 0) -> Dict[str, torch.Tensor]:
    """Seeded fp32 CPU weights with NO all-zero tensors.

    The reference zero-initialises 253 tensors (zero_module on proj_out / out_layers.3 / out.2 and
    alpha_attn/alpha_dense, SURVEY 8c) which would make eps == 0 and hide every bug; here every
    tensor is drawn so that activations stay O(1): weights ~ N(0, 1/fan_in), norm scales ~ 1 + 0.1 N,
    biases ~ 0.05 N, alphas ~ U(-1, 1).  The draw order is the registration order, one generator,
    so the same bits are produced on every box with this torch build.
    """
    g = torch.Generator(device="cpu").manual_seed(seed)
    sd: Dict[str, torch.Tensor] = OrderedDict()
    for key, shape in unet_param_shapes(cfg).items():
        leaf = key.rsplit(".", 1)[-1]
        if leaf in ("alpha_attn", "alpha_dense"):
            t = torch.rand((), generator=g) * 2 - 1
        elif leaf == "bias" or key.startswith("position_net.null_"):
            t = torch.randn(shape, generator=g) * 0.05
        elif len(shape) == 1:                                   # norm scales
            t = 1.0 + 0.1 * torch.randn(shape, generator=g)
        elif key.endswith("_embeddings"):
            t = torch.randn(shape, generator=g)
        elif key.endswith("pos_embedding"):
            t = torch.randn(shape, generator=g) * 0.02            # hed_grounding_net.py:25 (BERT-style)
        elif leaf == "gamma":                                       # ConvNeXt layer scale (1e-6 at init, O(0.1-1) when trained)
            t = 0.5 + 0.1 * torch.randn(shape, generator=g)
        else:
            fan_in = 1
            for s in shape[1:]:
                fan_in *= s
            t = torch.randn(shape, generator=g) * (fan_in ** -0.5)
        sd[key] = t
    return sd


def flops_per_forward(cfg: UNetConfig, G: int, fuser_on: bool = True, latent: Optional[Tuple[int, int]] = None) -> float:
    """Algorithmic 2*MAC of one UNet forward for ONE sample (SURVEY 8d analytic generator); latent = (H, W), default square
    cfg.image_size."""
    ctx, ted = cfg.context_dim, cfg.time_embed_dim
    Hl, Wl = latent or (cfg.image_size, cfg.image_size)
    total = 0.0
    for blk in block_schedule(cfg):
        hw = (Hl // blk.ds) * (Wl // blk.ds)
        for ly in blk.layers:
            if ly.kind == "conv_in":
                total += 18.0 * hw * ly.cin * ly.cout
            elif ly.kind == "res":
                total += 18.0 * hw * ly.cin * ly.cout + 18.0 * hw * ly.cout ** 2 + 2.0 * ted * ly.cout
                if ly.cin != ly.cout:
                    total += 2.0 * hw * ly.cin * ly.cout
            elif ly.kind == "st":
                C, T = ly.cin, hw
                total += 4.0 * T * C * C                                   # proj in/out
                total += 8.0 * T * C * C + 4.0 * T * T * C                 # attn1
                if fuser_on and cfg.fuser_type == "gatedCA":          # q, K/V of the tokens, attention T x G, out, ff
                    total += 4.0 * T * C * C + 4.0 * G * ctx * C + 4.0 * T * G * C + 24.0 * T * C * C
                elif fuser_on and cfg.fuser_type == "gatedSA2":       # only the G grounding rows query and leave the attention
                    total += 2.0 * G * ctx * C + 6.0 * G * C * C + 4.0 * T * C * C + 4.0 * G * (T + G) * C + 2.0 * G * C * C + 24.0 * T * C * C
                elif fuser_on:
                    total += 2.0 * G * ctx * C + 8.0 * (T + G) * C * C + 4.0 * (T + G) ** 2 * C + 24.0 * T * C * C
                total += 4.0 * T * C * C + 4.0 * 77 * ctx * C + 4.0 * T * 77 * C   # attn2
                total += 24.0 * T * C * C                                  # ff
            elif ly.kind == "down":
                total += 18.0 * (hw // 4) * ly.cin * ly.cout
            elif ly.kind == "up":
                total += 18.0 * (hw * 4) * ly.cin * ly.cout
    total += 18.0 * Hl * Wl * cfg.model_channels * cfg.out_channels
    total += 2.0 * (cfg.model_channels * ted + ted * ted)
    if cfg.spatial:
        return total          # the ConvNeXt tokenizer runs once per sample, not per forward
    din = cfg.tok_feat_dim + cfg.position_dim
    n_mlp = 2 if cfg.tokenizer == "text_image" else 1
    gtok = G // n_mlp
    total += n_mlp * 2.0 * gtok * (din * cfg.tok_hidden + cfg.tok_hidden ** 2 + cfg.tok_hidden * cfg.tok_out_dim)
    return total


# ------------------------------------------------------------------------------------------------
# SURVEY 8(f) rank 1 (next row, not on the hot path yet): the VAE decoder that turns the sampled
# latent into pixels (reference ldm/models/autoencoder.py:40-44, ldm/modules/diffusionmodules/model.py:462-568).
# Only the specification (state-dict keys / shapes, synthetic weights) lives here; the oracle is oracle/vae_oracle.py.
# ------------------------------------------------------------------------------------------------
@dataclass(frozen=True)
class VAEDecoderConfig:
    name: str = "sd14_vae"
    ch: int = 128
    ch_mult: Tuple[int, ...] = (1, 2, 4, 4)
    num_res_blocks: int = 2
    z_channels: int = 4
    embed_dim: int = 4
    out_ch: int = 3
    in_channels: int = 3                  # encoder input (ddconfig.in_channels)
    latent_size: int = 64                 # decode(z) with z of shape [B, embed_dim, latent_size, latent_size]
    scale_factor: float = 0.18215         # AutoencoderKL(scale_factor=...), configs/*: decode divides by it

    @property
    def image_size(self) -> int:
        return self.latent_size * 2 ** (len(self.ch_mult) - 1)


NAMED_VAE_CONFIGS = {
    "sd14_vae": VAEDecoderConfig(),
    "tiny_vae": VAEDecoderConfig(name="tiny_vae", ch=32, ch_mult=(1, 2), num_res_blocks=1, latent_size=8),      # oracle only (32 channels)
    # channel counts that are multiples of 64 (tensor-core tiles): 8x8 -> 16x16, and a 64x64 -> 256x256 case whose last
    # level is wider than one 128-pixel tile
    "tiny_vae64": VAEDecoderConfig(name="tiny_vae64", ch=64, ch_mult=(1, 2), num_res_blocks=1, latent_size=8),
    "small_vae": VAEDecoderConfig(name="small_vae", ch=64, ch_mult=(1, 1, 2), num_res_blocks=1, latent_size=64),
}


def vae_decoder_param_shapes(cfg: VAEDecoderConfig) -> "OrderedDict[str, tuple]":
    """Keys / shapes of `post_quant_conv.*` and `decoder.*` in registration order (model.py:462-533)."""
    p: "OrderedDict[str, tuple]" = OrderedDict()

    def conv(prefix, cin, cout, k):
        p[prefix + ".weight"] = (cout, cin, k, k)
        p[prefix + ".bias"] = (cout,)

    def norm(prefix, c):
        p[prefix + ".weight"] = (c,)
        p[prefix + ".bias"] = (c,)

    def resblock(prefix, cin, cout):
        norm(prefix + ".norm1", cin)
        conv(prefix + ".conv1", cin, cout, 3)
        norm(prefix + ".norm2", cout)
        conv(prefix + ".conv2", cout, cout, 3)
        if cin != cout:
            conv(prefix + ".nin_shortcut", cin, cout, 1)

    conv("post_quant_conv", cfg.embed_dim, cfg.z_channels, 1)
    nres = len(cfg.ch_mult)
    block_in = cfg.ch * cfg.ch_mult[-1]
    conv("decoder.conv_in", cfg.z_channels, block_in, 3)
    resblock("decoder.mid.block_1", block_in, block_in)
    norm("decoder.mid.attn_1.norm", block_in)
    for nm in ("q", "k", "v", "proj_out"):
        conv(f"decoder.mid.attn_1.{nm}", block_in, block_in, 1)
    resblock("decoder.mid.block_2", block_in, block_in)
    # nn.ModuleList `up` is built from the last level down but inserted at the front: state-dict order is level 0 first
    per_level = {}
    for i_level in reversed(range(nres)):
        block_out = cfg.ch * cfg.ch_mult[i_level]
        entries = []
        for i_block in range(cfg.num_res_blocks + 1):
            entries.append((f"decoder.up.{i_level}.block.{i_block}", block_in, block_out))
            block_in = block_out
        per_level[i_level] = (entries, block_in)
    for i_level in range(nres):
        entries, c = per_level[i_level]
        for prefix, cin, cout in entries:
            resblock(prefix, cin, cout)
        if i_level != 0:
            conv(f"decoder.up.{i_level}.upsample.conv", c, c, 3)
    norm("decoder.norm_out", cfg.ch * cfg.ch_mult[0])
    conv("decoder.conv_out", cfg.ch * cfg.ch_mult[0], cfg.out_ch, 3)
    return p


def vae_encoder_param_shapes(cfg: VAEDecoderConfig) -> "OrderedDict[str, tuple]":
    """Keys / shapes of `encoder.*` and `quant_conv.*` (SURVEY 8f rank 3, the inpainting front end: model.py:368-432,
    autoencoder.py:24-38).  attn_resolutions is empty in every shipped config: the only attention is mid.attn_1."""
    p: "OrderedDict[str, tuple]" = OrderedDict()

    def conv(prefix, cin, cout, k):
        p[prefix + ".weight"] = (cout, cin, k, k)
        p[prefix + ".bias"] = (cout,)

    def norm(prefix, c):
        p[prefix + ".weight"] = (c,)
        p[prefix + ".bias"] = (c,)

    def resblock(prefix, cin, cout):
        norm(prefix + ".norm1", cin)
        conv(prefix + ".conv1", cin, cout, 3)
        norm(prefix + ".norm2", cout)
        conv(prefix + ".conv2", cout, cout, 3)
        if cin != cout:
            conv(prefix + ".nin_shortcut", cin, cout, 1)

    conv("encoder.conv_in", cfg.in_channels, cfg.ch, 3)
    in_mult = (1,) + tuple(cfg.ch_mult)
    block_in = cfg.ch
    for i_level in range(len(cfg.ch_mult)):
        block_in = cfg.ch * in_mult[i_level]
        block_out = cfg.ch * cfg.ch_mult[i_level]
        for i_block in range(cfg.num_res_blocks):
            resblock(f"encoder.down.{i_level}.block.{i_block}", block_in, block_out)
            block_in = block_out
        if i_level != len(cfg.ch_mult) - 1:
            conv(f"encoder.down.{i_level}.downsample.conv", block_in, block_in, 3)
    resblock("encoder.mid.block_1", block_in, block_in)
    norm("encoder.mid.attn_1.norm", block_in)
    for nm in ("q", "k", "v", "proj_out"):
        conv(f"encoder.mid.attn_1.{nm}", block_in, block_in, 1)
    resblock("encoder.mid.block_2", block_in, block_in)
    norm("encoder.norm_out", block_in)
    conv("encoder.conv_out", block_in, 2 * cfg.z_channels, 3)
    conv("quant_conv", 2 * cfg.z_channels, 2 * cfg.embed_dim, 1)
    return p


def _draw(shapes, seed):
    g = torch.Generator(device="cpu").manual_seed(seed)
    sd: Dict[str, torch.Tensor] = OrderedDict()
    for key, shape in shapes.items():
        if key.endswith(".bias"):
            t = torch.randn(shape, generator=g) * 0.05
        elif len(shape) == 1:
            t = 1.0 + 0.1 * torch.randn(shape, generator=g)
        else:
            fan_in = shape[1] * shape[2] * shape[3]
            t = torch.randn(shape, generator=g) * (fan_in ** -0.5)
        sd[key] = t
    return sd


def synthetic_vae_encoder_state_dict(cfg: VAEDecoderConfig, seed: int = 1) -> Dict[str, torch.Tensor]:
    """Seeded fp32 CPU weights for the encoder half (its own generator: the decoder fixtures do not move)."""
    return _draw(vae_encoder_param_shapes(cfg), seed)


def synthetic_vae_state_dict(cfg: VAEDecoderConfig, seed: int = 0) -> Dict[str, torch.Tensor]:
    """Seeded fp32 CPU weights for the decoder half (same drawing rules as synthetic_state_dict)."""
    g = torch.Generator(device="cpu").manual_seed(seed)
    sd: Dict[str, torch.Tensor] = OrderedDict()
    for key, shape in vae_decoder_param_shapes(cfg).items():
        if key.endswith(".bias"):
            t = torch.randn(shape, generator=g) * 0.05
        elif len(shape) == 1:
            t = 1.0 + 0.1 * torch.randn(shape, generator=g)
        else:
            fan_in = shape[1] * shape[2] * shape[3]
            t = torch.randn(shape, generator=g) * (fan_in ** -0.5)
        sd[key] = t
    return sd
