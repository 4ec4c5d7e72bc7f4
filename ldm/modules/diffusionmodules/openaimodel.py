"""Drop-in `UNetModel` at the reference's import path (ldm.modules.diffusionmodules.openaimodel.UNetModel,
located by string through instantiate_from_config; reference openaimodel.py:237-464).

Same constructor kwargs, same state_dict keys/shapes, same `forward(input: dict) -> eps` contract, same
externally visible attributes (`image_size`, `in_channels`, `inpaint_mode`, `grounding_tokenizer_input`,
`first_conv_type`, `restore_first_conv_from_SD`, fuser modules with `.scale`).  The arithmetic is NOT
PyTorch: forward() hands raw device pointers to libgligen_b200.so (hand-written sm_90a kernels) through
gligen_b200.engine.  There is no CPU / eager fallback: parameters must live on a CUDA device.
"""
import os
import re
from copy import deepcopy

import torch
import torch.nn as nn

from gligen_b200.spec import UNetConfig, unet_param_shapes
from ldm.modules.attention import (BasicTransformerBlock, CrossAttention, FeedForward, GatedSelfAttentionDense,
                                   ParamNode, SelfAttention, SpatialTransformer, attach_params)
from gligen_b200.spec import SPATIAL_TOKENIZERS
from ldm.modules.diffusionmodules.grounding_common import downsampler_config, tokenizer_config
from ldm.util import instantiate_from_config

_TOKENIZERS = {
    "ldm.modules.diffusionmodules.text_grounding_net.PositionNet": "text",
    "ldm.modules.diffusionmodules.text_image_grounding_net.PositionNet": "text_image",
    "ldm.modules.diffusionmodules.keypoint_grounding_net.PositionNet": "keypoint",
}
_TOKENIZERS.update({f"ldm.modules.diffusionmodules.{t}_grounding_net.PositionNet": t for t in SPATIAL_TOKENIZERS})
_DOWNSAMPLERS = {f"ldm.modules.diffusionmodules.{t}_grounding_downsampler.GroundingDownsampler": t for t in SPATIAL_TOKENIZERS}


class TimestepEmbedSequential(ParamNode):
    pass


class ResBlock(ParamNode):
    pass


class Downsample(ParamNode):
    pass


class Upsample(ParamNode):
    pass


def _node_class(path: str):
    """Container type for a module path (purely cosmetic except for the fuser, which set_alpha_scale finds by type)."""
    if re.fullmatch(r"(input_blocks|output_blocks)\.\d+|middle_block", path):
        return TimestepEmbedSequential
    if path.endswith(".fuser"):
        return GatedSelfAttentionDense
    if path.endswith((".attn1", ".fuser.attn")):
        return SelfAttention
    if path.endswith(".attn2"):
        return CrossAttention
    if path.endswith(".ff"):
        return FeedForward
    if re.search(r"transformer_blocks\.\d+$", path):
        return BasicTransformerBlock
    return ParamNode


class UNetModel(ParamNode):
    def __init__(self, image_size, in_channels, model_channels, out_channels, num_res_blocks, attention_resolutions,
                 dropout=0, channel_mult=(1, 2, 4, 8), conv_resample=True, dims=2, use_checkpoint=False, num_heads=8,
                 use_scale_shift_norm=False, transformer_depth=1, context_dim=None, fuser_type=None, inpaint_mode=False,
                 grounding_downsampler=None, grounding_tokenizer=None):
        super().__init__()
        assert fuser_type in ["gatedSA", "gatedSA2", "gatedCA"]
        unsupported = []
        if fuser_type != "gatedSA":
            unsupported.append(f"fuser_type={fuser_type} (every shipped config uses gatedSA)")
        target = (grounding_tokenizer or {}).get("target")
        ds_target = (grounding_downsampler or {}).get("target")
        if grounding_downsampler is not None and (ds_target not in _DOWNSAMPLERS or _DOWNSAMPLERS[ds_target] != _TOKENIZERS.get(target)):
            unsupported.append(f"grounding_downsampler target {ds_target!r} (must be the downsampler of the tokenizer's modality)")
        if grounding_downsampler is not None and inpaint_mode:
            unsupported.append("grounding_downsampler with inpaint_mode (the reference stops at a breakpoint() there, openaimodel.py:445-446)")
        if use_scale_shift_norm or transformer_depth != 1 or dims != 2 or not conv_resample or dropout:
            unsupported.append("use_scale_shift_norm / transformer_depth != 1 / dims != 2 / conv_resample=False / dropout")
        if target not in _TOKENIZERS:
            unsupported.append(f"grounding_tokenizer target {target!r}")
        if unsupported:
            raise NotImplementedError("gligen_b200 UNetModel: " + "; ".join(unsupported))

        self.image_size = image_size
        self.in_channels = in_channels
        self.model_channels = model_channels
        self.out_channels = out_channels
        self.num_res_blocks = num_res_blocks
        self.attention_resolutions = attention_resolutions
        self.dropout = dropout
        self.channel_mult = channel_mult
        self.conv_resample = conv_resample
        self.use_checkpoint = use_checkpoint
        self.num_heads = num_heads
        self.context_dim = context_dim
        self.fuser_type = fuser_type
        self.inpaint_mode = inpaint_mode
        self.grounding_tokenizer_input = None          # set externally (gligen_inference.py:349)
        self.downsample_net = None
        self.additional_channel_from_downsampler = 0
        self.first_conv_type = "SD"
        self.first_conv_restorable = not inpaint_mode

        base = UNetConfig(image_size=image_size, in_channels=in_channels, out_channels=out_channels,
                          model_channels=model_channels, num_res_blocks=num_res_blocks,
                          attention_resolutions=tuple(attention_resolutions), channel_mult=tuple(channel_mult),
                          num_heads=num_heads, transformer_depth=transformer_depth, context_dim=context_dim,
                          fuser_type=fuser_type, inpaint_mode=inpaint_mode)
        self.cfg = tokenizer_config(_TOKENIZERS[target], base, **grounding_tokenizer.get("params", {}))
        if grounding_downsampler is not None:           # openaimodel.py:293-297
            self.cfg = downsampler_config(_TOKENIZERS[target], self.cfg, **grounding_downsampler.get("params", {}))
            self.downsample_net = instantiate_from_config(grounding_downsampler)
            self.additional_channel_from_downsampler = self.downsample_net.out_dim
            self.first_conv_type = "GLIGEN"
        shapes = unet_param_shapes(self.cfg)
        body = {k: v for k, v in shapes.items() if not k.startswith(("position_net.", "downsample_net."))}
        attach_params(self, body, "", _node_class)
        self.position_net = instantiate_from_config(grounding_tokenizer)
        self._fusers = [m for m in self.modules() if type(m) == GatedSelfAttentionDense]
        self._engine = None
        self._engine_stale = True
        self._sd_conv_cache = None

    # ---- weights ---------------------------------------------------------------------------------
    def load_state_dict(self, state_dict, strict=True, **kw):
        conv, key = self.input_blocks[0][0], "input_blocks.0.0.weight"
        if key in state_dict and self.downsample_net is not None and conv.weight.shape[1] != state_dict[key].shape[1] \
                and state_dict[key].shape[1] == self.cfg.first_conv_in:
            # a spatial-map model whose first conv was swapped for SD's 4-channel one (restore_first_conv_from_SD) gets its
            # (4 + d)-channel GLIGEN conv back with the new weights
            conv.weight = nn.Parameter(torch.zeros_like(state_dict[key], device=conv.weight.device), requires_grad=False)
        out = super().load_state_dict(state_dict, strict=strict, **kw)
        self._engine_stale = True
        self._masters_valid = True
        self._forget_first_conv_swap()
        if self.downsample_net is not None:
            self.first_conv_type = "GLIGEN"
        return out

    def _forget_first_conv_swap(self):
        """New weights: the SD first conv is no longer what input_blocks[0][0] holds (the reference re-loads it on
        every alpha == 0 step, openaimodel.py:400-413, so it never goes stale there)."""
        self._sd_applied = False
        if hasattr(self, "GLIGEN_first_conv_state_dict"):
            del self.GLIGEN_first_conv_state_dict

    def invalidate_static(self):
        """Drop the engine's cache of timestep-invariant work (called by the samplers at the start of sample())."""
        if self._engine is not None:
            self._engine.invalidate_static()

    def _apply(self, fn, *a, **kw):
        out = super()._apply(fn, *a, **kw)              # .to(device) / .cuda(): re-pack on the next forward
        self._engine_stale = True
        self._engine = None
        self._sd_applied = False
        return out

    def engine(self):
        """The native engine bound to this module's parameters (built lazily on the parameters' device)."""
        dev = self.time_embed[0].weight.device
        if dev.type != "cuda":
            raise RuntimeError("gligen_b200 UNetModel runs only on a CUDA device (sm_90a kernels); "
                               "there is no CPU fallback - call .to('cuda') first")
        if self._engine is None:
            from gligen_b200.engine import Engine
            from gligen_b200.ops import CudaOps
            self._engine = Engine(self.cfg, CudaOps(dev))
            self._engine_stale = True
        if self._engine_stale:
            if not getattr(self, "_masters_valid", True):
                raise RuntimeError("this rank received only the packed weights (broadcast_packed_weights); its fp32 module "
                                   "parameters are not authoritative and cannot be re-packed - load a state dict first")
            self._engine.load_state_dict(self.state_dict())
            self._engine_stale = False
        return self._engine

    def broadcast_packed_weights(self, src=0):
        """Multi-GPU init (one process per GPU): rank `src` holds the checkpoint; every other rank receives the engine's
        packed bf16 arena in a few large NCCL broadcasts (half the bytes of the fp32 masters, no re-packing on the
        receivers).  The receivers' nn.Parameters keep their construction-time values and are marked non-authoritative.
        Returns the bytes sent (0 when torch.distributed is not initialised)."""
        import torch.distributed as dist
        if not (dist.is_available() and dist.is_initialized()) or dist.get_world_size() == 1:
            return 0
        eng = self.engine()                       # src: packs the real weights; others: packs placeholders (allocates slots)
        sent = eng.broadcast_packed(src)
        if dist.get_rank() != src:
            self._masters_valid = False
        return sent

    def restore_first_conv_from_SD(self):
        """reference openaimodel.py:400-413: swap input_blocks[0][0] for SD's 4->C conv, read from the
        CWD-relative file "SD_input_conv_weight_bias.pth"."""
        if not self.first_conv_restorable:
            print("First conv layer is not restorable and skipped this process, probably because this is an inpainting model?")
            return
        conv = self.input_blocks[0][0]
        path = "SD_input_conv_weight_bias.pth"
        stamp = (os.path.abspath(path), os.path.getmtime(path))
        if self._sd_conv_cache is None or self._sd_conv_cache[0] != stamp:
            sd = torch.load(path, map_location="cpu")
            self._sd_conv_cache = (stamp, sd["weight"].float(), sd["bias"].float())
            self._sd_applied = False
        if getattr(self, "_sd_applied", False) and self.first_conv_type == "SD" and hasattr(self, "GLIGEN_first_conv_state_dict"):
            return                                       # already swapped in: idempotent
        _, w, b = self._sd_conv_cache
        narrower = self.downsample_net is not None and w.shape[1] == self.in_channels and tuple(w.shape[:1] + w.shape[2:]) == tuple(
            conv.weight.shape[:1] + conv.weight.shape[2:])
        if tuple(w.shape) != tuple(conv.weight.shape) and not narrower:
            raise RuntimeError(f"{path}: weight {tuple(w.shape)} does not fit the first conv {tuple(conv.weight.shape)}")
        self.GLIGEN_first_conv_state_dict = deepcopy(conv.state_dict())
        with torch.no_grad():
            if narrower:
                # spatial modalities: the reference replaces the (4 + d)-channel conv by SD's 4-channel one and stops feeding the
                # downsampler planes (first_conv_type == "SD", openaimodel.py:407-411, 441); the engine keeps its plan and gets
                # zero weights on the extra channels (Engine.set_first_conv)
                dev = conv.weight.device
                conv.weight = nn.Parameter(w.to(dev), requires_grad=False)
                conv.bias = nn.Parameter(b.to(dev), requires_grad=False)
            else:
                conv.weight.copy_(w)
                conv.bias.copy_(b)
        if self._engine is not None and not self._engine_stale:
            self._engine.set_first_conv(conv.weight, conv.bias)
        self.first_conv_type = "SD"
        self._sd_applied = True

    # ---- forward -----------------------------------------------------------------------------------
    def _sync_scales(self, eng):
        scales = [float(m.scale) for m in self._fusers]
        if getattr(eng, "scales", None) != scales:
            eng.set_scale(scales)

    def _grounding(self, input):
        if "grounding_input" in input:
            return input["grounding_input"]
        return self.grounding_tokenizer_input.get_null_input()       # guidance null case (openaimodel.py:422-426)

    @torch.no_grad()
    def forward(self, input):
        eng = self.engine()
        self._sync_scales(eng)
        return eng.forward(input["x"], input["timesteps"], input["context"], self._grounding(input),
                           input.get("inpainting_extra_input") if self.inpaint_mode else None,
                           input.get("grounding_extra_input") if self.downsample_net is not None else None)

    @torch.no_grad()
    def forward_cfg(self, input, uc):
        """cond + uncond in one 2B-row pass (used by the samplers in this repo; same results as two calls)."""
        eng = self.engine()
        self._sync_scales(eng)
        return eng.forward_cfg(input["x"], input["timesteps"], input["context"], uc, input["grounding_input"],
                               input.get("inpainting_extra_input") if self.inpaint_mode else None,
                               input.get("grounding_extra_input") if self.downsample_net is not None else None)


# names this drop-in does not define resolve to the reference module of the same name when a reference checkout
# follows this repo on sys.path (gligen_b200/_overlay.py)
from gligen_b200._overlay import fallback as _fallback  # noqa: E402

__getattr__ = _fallback(__name__, __file__)
