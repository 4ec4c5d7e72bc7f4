"""CPU fp32 ORACLE for the GLIGEN per-timestep UNet forward.  TEST INFRASTRUCTURE ONLY.

This is a functional restatement (plain torch fp32 on the CPU, state-dict in / tensor out) of the
reference algorithm.  It is *not* part of the product: only tests/, __graft_entry__.smoke() and
bench.py's cpu_baseline / `--impl reference` legs may import it.  The product path
(gligen_b200.engine + libgligen_b200.so) never touches this file.

Parity pinning: the reference has no tests or golden vectors of its own (SURVEY 4, 8c), so this
restatement is pinned by EXECUTING the reference: oracle/gen_golden.py imports /root/reference,
loads the same seeded weights into the reference `UNetModel`, asserts agreement with this file to
fp32 round-off and writes tests/golden/*.pt, which travel to the GPU machine.

Every function cites the reference file:line it follows.
"""
from __future__ import annotations

import math
from typing import Dict, Optional

import torch
import torch.nn.functional as F

from gligen_b200.spec import UNetConfig, block_schedule


# --------------------------------------------------------------------------------------------
# small pieces
# --------------------------------------------------------------------------------------------
def timestep_embedding(t: torch.Tensor, dim: int, max_period: float = 10000.0) -> torch.Tensor:
    """ldm/modules/diffusionmodules/util.py:160-180 (repeat_only=False): [cos | sin]."""
    half = dim // 2
    freqs = torch.exp(-math.log(max_period) * torch.arange(half, dtype=torch.float32) / half)
    args = t[:, None].float() * freqs[None]
    return torch.cat([torch.cos(args), torch.sin(args)], dim=-1)


def fourier_embed(x: torch.Tensor, num_freqs: int = 8, temperature: float = 100.0) -> torch.Tensor:
    """util.py:12-26 FourierEmbedder: per frequency [sin(f x) | cos(f x)] concatenated on the last dim."""
    bands = temperature ** (torch.arange(num_freqs) / num_freqs)
    out = []
    for f in bands:
        out.append(torch.sin(f * x))
        out.append(torch.cos(f * x))
    return torch.cat(out, dim=-1)


def _mlp3(sd, prefix, x):
    x = F.silu(F.linear(x, sd[f"{prefix}.0.weight"], sd[f"{prefix}.0.bias"]))
    x = F.silu(F.linear(x, sd[f"{prefix}.2.weight"], sd[f"{prefix}.2.bias"]))
    return F.linear(x, sd[f"{prefix}.4.weight"], sd[f"{prefix}.4.bias"])


def position_net(cfg: UNetConfig, sd: Dict[str, torch.Tensor], g: Dict[str, torch.Tensor]) -> torch.Tensor:
    """PositionNet.forward of the three discrete tokenisers -> objs [B, G, out_dim].

    text:        text_grounding_net.py:30-47
    text_image:  text_image_grounding_net.py:41-65  (text tokens then image tokens, G = 2N)
    keypoint:    keypoint_grounding_net.py:34-58
    """
    pn = "position_net"
    if cfg.spatial:
        from oracle.spatial_oracle import position_net_spatial
        return position_net_spatial(cfg, sd, g)
    if cfg.tokenizer == "text":
        m = g["masks"].unsqueeze(-1)
        xyxy = fourier_embed(g["boxes"], cfg.fourier_freqs)
        emb = g["positive_embeddings"] * m + (1 - m) * sd[f"{pn}.null_positive_feature"].view(1, 1, -1)
        xyxy = xyxy * m + (1 - m) * sd[f"{pn}.null_position_feature"].view(1, 1, -1)
        return _mlp3(sd, f"{pn}.linears", torch.cat([emb, xyxy], dim=-1))
    if cfg.tokenizer == "text_image":
        m = g["masks"].unsqueeze(-1)
        tm = g["text_masks"].unsqueeze(-1)
        im = g["image_masks"].unsqueeze(-1)
        xyxy = fourier_embed(g["boxes"], cfg.fourier_freqs)
        te = g["text_embeddings"] * tm + (1 - tm) * sd[f"{pn}.null_text_feature"].view(1, 1, -1)
        ie = g["image_embeddings"] * im + (1 - im) * sd[f"{pn}.null_image_feature"].view(1, 1, -1)
        xyxy = xyxy * m + (1 - m) * sd[f"{pn}.null_position_feature"].view(1, 1, -1)
        ot = _mlp3(sd, f"{pn}.linears_text", torch.cat([te, xyxy], dim=-1))
        oi = _mlp3(sd, f"{pn}.linears_image", torch.cat([ie, xyxy], dim=-1))
        return torch.cat([ot, oi], dim=1)
    if cfg.tokenizer == "keypoint":
        m = g["masks"].unsqueeze(-1)
        N = g["points"].shape[0]
        P = cfg.max_persons
        pe = sd[f"{pn}.person_embeddings"].unsqueeze(1).repeat(1, 17, 1).reshape(P * 17, -1)
        ke = torch.cat([sd[f"{pn}.keypoint_embeddings"]] * P, dim=0)
        pe = (pe + ke).unsqueeze(0).repeat(N, 1, 1)
        xy = fourier_embed(g["points"], cfg.fourier_freqs)
        pe = pe * m + (1 - m) * sd[f"{pn}.null_person_feature"].view(1, 1, -1)
        xy = xy * m + (1 - m) * sd[f"{pn}.null_xy_feature"].view(1, 1, -1)
        return _mlp3(sd, f"{pn}.linears", torch.cat([pe, xy], dim=-1))
    raise ValueError(cfg.tokenizer)


def null_grounding(cfg: UNetConfig, like: Dict[str, torch.Tensor]) -> Dict[str, torch.Tensor]:
    """GroundingNetInput.get_null_input (grounding_input/*_tokinzer_input.py): zeros of the prepared shapes."""
    return {k: torch.zeros_like(v) for k, v in like.items()}


def _attention(q, k, v, heads):
    """attention.py:167-186 / 127-149: softmax(q k^T d^-1/2) v over `heads` heads, fp32, materialised."""
    B, N, HC = q.shape
    M = k.shape[1]
    C = HC // heads
    q = q.view(B, N, heads, C).permute(0, 2, 1, 3)
    k = k.view(B, M, heads, C).permute(0, 2, 1, 3)
    v = v.view(B, M, heads, C).permute(0, 2, 1, 3)
    sim = torch.einsum("bhic,bhjc->bhij", q, k) * (C ** -0.5)
    attn = sim.softmax(dim=-1)
    out = torch.einsum("bhij,bhjc->bhic", attn, v)
    return out.permute(0, 2, 1, 3).reshape(B, N, HC)


def _self_attn(sd, p, x, heads):
    q = F.linear(x, sd[f"{p}.to_q.weight"])
    k = F.linear(x, sd[f"{p}.to_k.weight"])
    v = F.linear(x, sd[f"{p}.to_v.weight"])
    return F.linear(_attention(q, k, v, heads), sd[f"{p}.to_out.0.weight"], sd[f"{p}.to_out.0.bias"])


def _cross_attn(sd, p, x, ctx, heads):
    q = F.linear(x, sd[f"{p}.to_q.weight"])
    k = F.linear(ctx, sd[f"{p}.to_k.weight"])
    v = F.linear(ctx, sd[f"{p}.to_v.weight"])
    return F.linear(_attention(q, k, v, heads), sd[f"{p}.to_out.0.weight"], sd[f"{p}.to_out.0.bias"])


def _ff(sd, p, x):
    """attention.py:37-64: GEGLU (exact erf GELU) then Linear."""
    h = F.linear(x, sd[f"{p}.net.0.proj.weight"], sd[f"{p}.net.0.proj.bias"])
    a, gate = h.chunk(2, dim=-1)
    return F.linear(a * F.gelu(gate), sd[f"{p}.net.2.weight"], sd[f"{p}.net.2.bias"])


def _ln(sd, p, x):
    return F.layer_norm(x, (x.shape[-1],), sd[f"{p}.weight"], sd[f"{p}.bias"], 1e-5)


def gated_self_attention(sd, p, x, objs, heads, scale):
    """attention.py:236-244 GatedSelfAttentionDense.forward."""
    T = x.shape[1]
    o = F.linear(objs, sd[f"{p}.linear.weight"], sd[f"{p}.linear.bias"])
    a = _self_attn(sd, f"{p}.attn", _ln(sd, f"{p}.norm1", torch.cat([x, o], dim=1)), heads)[:, :T]
    x = x + scale * torch.tanh(sd[f"{p}.alpha_attn"]) * a
    x = x + scale * torch.tanh(sd[f"{p}.alpha_dense"]) * _ff(sd, f"{p}.ff", _ln(sd, f"{p}.norm2", x))
    return x


def transformer_block(sd, p, x, ctx, objs, heads, scale):
    """attention.py:333-338 BasicTransformerBlock._forward."""
    x = _self_attn(sd, f"{p}.attn1", _ln(sd, f"{p}.norm1", x), heads) + x
    x = gated_self_attention(sd, f"{p}.fuser", x, objs, heads, scale)
    x = _cross_attn(sd, f"{p}.attn2", _ln(sd, f"{p}.norm2", x), ctx, heads) + x
    x = _ff(sd, f"{p}.ff", _ln(sd, f"{p}.norm3", x)) + x
    return x


def spatial_transformer(sd, p, x, ctx, objs, heads, scale):
    """attention.py:366-376: GroupNorm(32, eps=1e-6) -> 1x1 -> tokens -> block -> 1x1 -> + x_in."""
    B, C, H, W = x.shape
    h = F.group_norm(x, 32, sd[f"{p}.norm.weight"], sd[f"{p}.norm.bias"], 1e-6)
    h = F.conv2d(h, sd[f"{p}.proj_in.weight"], sd[f"{p}.proj_in.bias"])
    h = h.permute(0, 2, 3, 1).reshape(B, H * W, C)
    h = transformer_block(sd, f"{p}.transformer_blocks.0", h, ctx, objs, heads, scale)
    h = h.reshape(B, H, W, C).permute(0, 3, 1, 2)
    h = F.conv2d(h, sd[f"{p}.proj_out.weight"], sd[f"{p}.proj_out.bias"])
    return h + x


def res_block(sd, p, x, emb):
    """openaimodel.py:212-232 ResBlock._forward (use_scale_shift_norm=False, no up/down)."""
    h = F.silu(F.group_norm(x, 32, sd[f"{p}.in_layers.0.weight"], sd[f"{p}.in_layers.0.bias"], 1e-5))
    h = F.conv2d(h, sd[f"{p}.in_layers.2.weight"], sd[f"{p}.in_layers.2.bias"], padding=1)
    e = F.linear(F.silu(emb), sd[f"{p}.emb_layers.1.weight"], sd[f"{p}.emb_layers.1.bias"])
    h = h + e[:, :, None, None]
    h = F.silu(F.group_norm(h, 32, sd[f"{p}.out_layers.0.weight"], sd[f"{p}.out_layers.0.bias"], 1e-5))
    h = F.conv2d(h, sd[f"{p}.out_layers.3.weight"], sd[f"{p}.out_layers.3.bias"], padding=1)
    if f"{p}.skip_connection.weight" in sd:
        x = F.conv2d(x, sd[f"{p}.skip_connection.weight"], sd[f"{p}.skip_connection.bias"])
    return x + h


# --------------------------------------------------------------------------------------------
# the forward
# --------------------------------------------------------------------------------------------
@torch.no_grad()
def unet_forward(cfg: UNetConfig, sd: Dict[str, torch.Tensor], x: torch.Tensor, timesteps: torch.Tensor,
                 context: torch.Tensor, grounding: Dict[str, torch.Tensor], scale: float = 1.0,
                 inpainting_extra_input: Optional[torch.Tensor] = None,
                 taps: Optional[dict] = None, grounding_extra_input: Optional[torch.Tensor] = None) -> torch.Tensor:
    """openaimodel.py:420-464 UNetModel.forward.  `scale` is GatedSelfAttentionDense.scale
    (gligen_inference.py:24-28).  `taps`, if given, receives named intermediate activations."""
    objs = position_net(cfg, sd, grounding)
    emb = timestep_embedding(timesteps, cfg.model_channels)
    emb = F.linear(emb, sd["time_embed.0.weight"], sd["time_embed.0.bias"])
    emb = F.linear(F.silu(emb), sd["time_embed.2.weight"], sd["time_embed.2.bias"])
    h = x.float()
    if cfg.ds_out_dim and grounding_extra_input is not None:
        # openaimodel.py:441-443: downsample_net output joins the latent while first_conv_type == "GLIGEN"; pass
        # grounding_extra_input=None to state the "SD" first-conv case (after restore_first_conv_from_SD)
        from oracle.spatial_oracle import grounding_downsampler
        temp = grounding_downsampler(cfg, sd, grounding_extra_input, cfg.image_size)
        if taps is not None:
            taps["downsample_net"] = temp
        h = torch.cat([h, temp], dim=1)
    if cfg.inpaint_mode:
        h = torch.cat([h, inpainting_extra_input], dim=1)
    if taps is not None:
        taps["objs"] = objs
        taps["emb"] = emb
    hs = []
    for blk in block_schedule(cfg):
        if blk.where == "out":
            h = torch.cat([h, hs.pop()], dim=1)
        for ly in blk.layers:
            if ly.kind == "conv_in":
                h = F.conv2d(h, sd[f"{ly.prefix}.weight"], sd[f"{ly.prefix}.bias"], padding=1)
            elif ly.kind == "res":
                h = res_block(sd, ly.prefix, h, emb)
            elif ly.kind == "st":
                h = spatial_transformer(sd, ly.prefix, h, context, objs, ly.heads, scale)
            elif ly.kind == "down":
                h = F.conv2d(h, sd[f"{ly.prefix}.op.weight"], sd[f"{ly.prefix}.op.bias"], stride=2, padding=1)
            elif ly.kind == "up":
                h = F.interpolate(h, scale_factor=2, mode="nearest")
                h = F.conv2d(h, sd[f"{ly.prefix}.conv.weight"], sd[f"{ly.prefix}.conv.bias"], padding=1)
            if taps is not None:
                taps[ly.prefix] = h
        if blk.where == "in":
            hs.append(h)
    h = F.silu(F.group_norm(h, 32, sd["out.0.weight"], sd["out.0.bias"], 1e-5))
    return F.conv2d(h, sd["out.2.weight"], sd["out.2.bias"], padding=1)
