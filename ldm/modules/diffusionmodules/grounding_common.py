"""Shared constructor logic of the PositionNet / GroundingDownsampler containers (parameters only)."""
from dataclasses import replace

from gligen_b200.spec import SPATIAL_TOKENIZERS, UNetConfig, downsampler_param_shapes, unet_param_shapes
from ldm.modules.attention import ParamNode, attach_params


def tokenizer_config(kind: str, base: UNetConfig = UNetConfig(), **params) -> UNetConfig:
    if kind in SPATIAL_TOKENIZERS:      # hed_grounding_net.py:13 PositionNet(resize_input=448, out_dim=768[, in_dim=152])
        return replace(base, tokenizer=kind, tok_resize=params.get("resize_input", 448), tok_out_dim=params.get("out_dim", 768),
                       sem_in_dim=params.get("in_dim", 152))
    if kind == "keypoint":
        return replace(base, tokenizer=kind, max_persons=params.get("max_persons_per_image", 8),
                       tok_out_dim=params.get("out_dim", 768), fourier_freqs=params.get("fourier_freqs", 8))
    return replace(base, tokenizer=kind, tok_in_dim=params.get("in_dim", 768), tok_out_dim=params.get("out_dim", 768),
                   fourier_freqs=params.get("fourier_freqs", 8))


def downsampler_config(kind: str, base: UNetConfig, **params) -> UNetConfig:
    """GroundingDownsampler(resize_input=256, out_dim=8[, in_dim=152]); hed: GroundingDownsampler(out_dim=1)."""
    cfg = replace(base, ds_out_dim=params.get("out_dim", 1 if kind == "hed" else 8), ds_resize=params.get("resize_input", 256))
    if kind == "sem" and "in_dim" in params:
        assert params["in_dim"] == cfg.sem_in_dim, "grounding tokenizer and downsampler disagree on in_dim"
    return cfg


def make_downsampler(kind: str):
    class _GroundingDownsampler(ParamNode):
        def __init__(self, **params):
            super().__init__()
            self.kind = kind
            self.params = dict(params)
            cfg = downsampler_config(kind, replace(UNetConfig(), tokenizer=kind, sem_in_dim=params.get("in_dim", 152)), **params)
            self.out_dim = cfg.ds_out_dim
            self.resize_input = cfg.ds_resize
            attach_params(self, downsampler_param_shapes(cfg), "downsample_net.")
    return _GroundingDownsampler


def make_position_net(kind: str):
    class _PositionNet(ParamNode):
        def __init__(self, **params):
            super().__init__()
            self.kind = kind
            self.params = dict(params)
            cfg = tokenizer_config(kind, **params)
            self.out_dim = cfg.tok_out_dim
            attach_params(self, unet_param_shapes(cfg), "position_net.")
    return _PositionNet
