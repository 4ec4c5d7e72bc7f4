"""CPU fp32 ORACLE for UNets built with the gatedCA and gatedSA2 fusers.  TEST INFRASTRUCTURE ONLY.

oracle/unet_oracle.py restates the gatedSA model every shipped config uses; this file restates the two other fusers the reference's
BasicTransformerBlock builds (ldm/modules/attention.py:313-321) and a UNet forward that dispatches on cfg.fuser_type, reusing every
other piece of unet_oracle.py.  Pinned against the executed reference by oracle/gen_golden_fusers.py.
"""
from __future__ import annotations

import math
from typing import Dict, Optional

import torch
import torch.nn.functional as F

from gligen_b200.spec import UNetConfig, block_schedule
from oracle import unet_oracle as UO


def gated_cross_attention(sd, p, x, objs, heads, scale):
    """attention.py:190-212 GatedCrossAttentionDense.forward: cross-attention from LN1(x) to the raw grounding tokens (no linear,
    no norm on objs, no mask; to_k / to_v without bias), then the gated FF."""
    a = UO._cross_attn(sd, f"{p}.attn", UO._ln(sd, f"{p}.norm1", x), objs, heads)
    x = x + scale * torch.tanh(sd[f"{p}.alpha_attn"]) * a
    x = x + scale * torch.tanh(sd[f"{p}.alpha_dense"]) * UO._ff(sd, f"{p}.ff", UO._ln(sd, f"{p}.norm2", x))
    return x


def gated_self_attention2(sd, p, x, objs, heads, scale):
    """attention.py:269-297 GatedSelfAttentionDense2.forward: the self-attention of gatedSA, of which only the G grounding rows are
    kept; reshaped row-major to a sqrt(G) x sqrt(G) grid and resampled bicubically (A = -0.75, align_corners = False) onto the
    sqrt(T) x sqrt(T) visual grid, they are the gated residual."""
    B, T, C = x.shape
    G = objs.shape[1]
    sv, sg = math.sqrt(T), math.sqrt(G)
    assert int(sv) == sv, "Visual tokens must be square rootable"
    assert int(sg) == sg, "Grounding tokens must be square rootable"
    sv, sg = int(sv), int(sg)
    o = F.linear(objs, sd[f"{p}.linear.weight"], sd[f"{p}.linear.bias"])
    out = UO._self_attn(sd, f"{p}.attn", UO._ln(sd, f"{p}.norm1", torch.cat([x, o], dim=1)), heads)[:, T:, :]
    out = out.permute(0, 2, 1).reshape(B, -1, sg, sg)
    out = F.interpolate(out, (sv, sv), mode="bicubic")
    residual = out.reshape(B, -1, T).permute(0, 2, 1)
    x = x + scale * torch.tanh(sd[f"{p}.alpha_attn"]) * residual
    x = x + scale * torch.tanh(sd[f"{p}.alpha_dense"]) * UO._ff(sd, f"{p}.ff", UO._ln(sd, f"{p}.norm2", x))
    return x


FUSERS = {"gatedSA": UO.gated_self_attention, "gatedCA": gated_cross_attention, "gatedSA2": gated_self_attention2}


def transformer_block(fuser, sd, p, x, ctx, objs, heads, scale):
    """attention.py:333-338 BasicTransformerBlock._forward with the configured fuser."""
    x = UO._self_attn(sd, f"{p}.attn1", UO._ln(sd, f"{p}.norm1", x), heads) + x
    x = fuser(sd, f"{p}.fuser", x, objs, heads, scale)
    x = UO._cross_attn(sd, f"{p}.attn2", UO._ln(sd, f"{p}.norm2", x), ctx, heads) + x
    x = UO._ff(sd, f"{p}.ff", UO._ln(sd, f"{p}.norm3", x)) + x
    return x


def spatial_transformer(fuser, sd, p, x, ctx, objs, heads, scale):
    """attention.py:366-376, as unet_oracle.spatial_transformer."""
    B, C, H, W = x.shape
    h = F.group_norm(x, 32, sd[f"{p}.norm.weight"], sd[f"{p}.norm.bias"], 1e-6)
    h = F.conv2d(h, sd[f"{p}.proj_in.weight"], sd[f"{p}.proj_in.bias"])
    h = h.permute(0, 2, 3, 1).reshape(B, H * W, C)
    h = transformer_block(fuser, sd, f"{p}.transformer_blocks.0", h, ctx, objs, heads, scale)
    h = h.reshape(B, H, W, C).permute(0, 3, 1, 2)
    h = F.conv2d(h, sd[f"{p}.proj_out.weight"], sd[f"{p}.proj_out.bias"])
    return h + x


@torch.no_grad()
def unet_forward(cfg: UNetConfig, sd: Dict[str, torch.Tensor], x: torch.Tensor, timesteps: torch.Tensor, context: torch.Tensor,
                 grounding: Dict[str, torch.Tensor], scale: float = 1.0, inpainting_extra_input: Optional[torch.Tensor] = None,
                 grounding_extra_input: Optional[torch.Tensor] = None) -> torch.Tensor:
    """openaimodel.py:420-464 UNetModel.forward for any fuser type (unet_oracle.unet_forward without taps)."""
    fuser = FUSERS[cfg.fuser_type]
    objs = UO.position_net(cfg, sd, grounding)
    emb = UO.timestep_embedding(timesteps, cfg.model_channels)
    emb = F.linear(emb, sd["time_embed.0.weight"], sd["time_embed.0.bias"])
    emb = F.linear(F.silu(emb), sd["time_embed.2.weight"], sd["time_embed.2.bias"])
    h = x.float()
    if cfg.ds_out_dim and grounding_extra_input is not None:
        from oracle.spatial_oracle import grounding_downsampler
        h = torch.cat([h, grounding_downsampler(cfg, sd, grounding_extra_input, cfg.image_size)], dim=1)
    if cfg.inpaint_mode:
        h = torch.cat([h, inpainting_extra_input], dim=1)
    hs = []
    for blk in block_schedule(cfg):
        if blk.where == "out":
            h = torch.cat([h, hs.pop()], dim=1)
        for ly in blk.layers:
            if ly.kind == "conv_in":
                h = F.conv2d(h, sd[f"{ly.prefix}.weight"], sd[f"{ly.prefix}.bias"], padding=1)
            elif ly.kind == "res":
                h = UO.res_block(sd, ly.prefix, h, emb)
            elif ly.kind == "st":
                h = spatial_transformer(fuser, sd, ly.prefix, h, context, objs, ly.heads, scale)
            elif ly.kind == "down":
                h = F.conv2d(h, sd[f"{ly.prefix}.op.weight"], sd[f"{ly.prefix}.op.bias"], stride=2, padding=1)
            elif ly.kind == "up":
                h = F.interpolate(h, scale_factor=2, mode="nearest")
                h = F.conv2d(h, sd[f"{ly.prefix}.conv.weight"], sd[f"{ly.prefix}.conv.bias"], padding=1)
        if blk.where == "in":
            hs.append(h)
    h = F.silu(F.group_norm(h, 32, sd["out.0.weight"], sd["out.0.bias"], 1e-5))
    return F.conv2d(h, sd["out.2.weight"], sd["out.2.bias"], padding=1)
