"""`AutoencoderKL` at the reference's import path (ldm/models/autoencoder.py:17-44), with `decode` and `encode` on this
repo's sm_90a kernels (gligen_b200/vae.py).  What gligen_inference.py does with it: `instantiate_from_config(config['autoencoder'])
.to(device).eval()`, `load_state_dict(saved_ckpt["autoencoder"])` (:76-84), `autoencoder.decode(samples_fake)` (:441) and, for
inpainting only, `autoencoder.encode(...)` (:403).

Two shapes, decided at import time:
  * overlaid on a reference checkout (INTEGRATION.md 1): a subclass of the reference's own AutoencoderKL - state-dict
    keys and every other method are the reference's; `decode` / `encode` are replaced when the parameters live on a CUDA
    device (on the CPU they are the reference's own PyTorch code);
  * this repo alone: a parameter-only module with the reference's `encoder.*` / `decoder.*` / `quant_conv.*` /
    `post_quant_conv.*` names (a full checkpoint loads strictly); CUDA only.
`encode` returns what the reference returns: one sample of the diagonal Gaussian posterior times scale_factor, the noise
drawn with torch's global CPU generator and moved to the device (distributions.py:24-37), so the same seed gives the same z0.
"""
import torch
import torch.nn as nn

from gligen_b200 import _overlay
from gligen_b200.spec import VAEDecoderConfig, vae_decoder_param_shapes, vae_encoder_param_shapes
from ldm.modules.attention import attach_params

_ref = _overlay._shadowed_module(__name__, __file__)


class _CudaDecodeMixin:
    """decode(z) through gligen_b200.vae.VAEDecoderEngine (weights re-packed lazily after load_state_dict / .to())."""

    def _vae_cfg(self) -> VAEDecoderConfig:
        return self._glg_cfg

    def _vae_engine(self):
        dev = self.post_quant_conv_weight_device()
        if dev.type != "cuda":
            raise RuntimeError("gligen_b200 AutoencoderKL.decode runs only on a CUDA device (sm_90a kernels); call .to('cuda') first")
        if getattr(self, "_glg_engine", None) is None or self._glg_engine.dev != dev:
            from gligen_b200.ops import CudaOps
            from gligen_b200.vae import VAEDecoderEngine
            self._glg_engine = VAEDecoderEngine(self._vae_cfg(), CudaOps(dev))
            self._glg_stale = True
        if getattr(self, "_glg_stale", True):
            sd = {k: v for k, v in self.state_dict().items() if k.startswith(("decoder.", "post_quant_conv."))}
            self._glg_engine.load_state_dict(sd)
            self._glg_stale = False
        return self._glg_engine

    def load_state_dict(self, state_dict, strict=True, **kw):
        out = super().load_state_dict(state_dict, strict=strict, **kw)
        self._glg_stale = self._glg_enc_stale = True
        return out

    def _apply(self, fn, *a, **kw):
        out = super()._apply(fn, *a, **kw)
        self._glg_stale = self._glg_enc_stale = True
        self._glg_engine = self._glg_enc = None
        return out

    def _vae_enc_engine(self):
        dev = self.post_quant_conv_weight_device()
        if dev.type != "cuda":
            raise RuntimeError("gligen_b200 AutoencoderKL.encode runs only on a CUDA device (sm_90a kernels); call .to('cuda') first")
        if getattr(self, "_glg_enc", None) is None or self._glg_enc.dev != dev:
            from gligen_b200.ops import CudaOps
            from gligen_b200.vae import VAEEncoderEngine
            self._glg_enc = VAEEncoderEngine(self._vae_cfg(), CudaOps(dev))
            self._glg_enc_stale = True
        if getattr(self, "_glg_enc_stale", True):
            sd = {k: v for k, v in self.state_dict().items() if k.startswith(("encoder.", "quant_conv."))}
            self._glg_enc.load_state_dict(sd)
            self._glg_enc_stale = False
        return self._glg_enc

    @torch.no_grad()
    def decode(self, z):
        return self._vae_engine().decode(z)

    @torch.no_grad()
    def encode_moments(self, x):
        """quant_conv(encoder(x)): the posterior's (mean | logvar), fp32 [B, 2 * embed_dim, h, w]."""
        return self._vae_enc_engine().encode_moments(x)

    @torch.no_grad()
    def encode(self, x):
        mean, logvar = torch.chunk(self.encode_moments(x), 2, dim=1)
        std = torch.exp(0.5 * torch.clamp(logvar, -30.0, 20.0))
        return (mean + std * torch.randn(mean.shape).to(device=mean.device)) * self.scale_factor


def _cfg_from_ddconfig(ddconfig, embed_dim, scale_factor, latent_size=64) -> VAEDecoderConfig:
    return VAEDecoderConfig(name="from_ddconfig", ch=ddconfig["ch"], ch_mult=tuple(ddconfig["ch_mult"]), num_res_blocks=ddconfig["num_res_blocks"],
                            z_channels=ddconfig["z_channels"], embed_dim=embed_dim, out_ch=ddconfig["out_ch"],
                            in_channels=ddconfig.get("in_channels", 3), latent_size=latent_size,
                            scale_factor=scale_factor)


if _ref is not None:
    class AutoencoderKL(_CudaDecodeMixin, _ref.AutoencoderKL):
        def __init__(self, ddconfig, embed_dim, scale_factor=1):
            _ref.AutoencoderKL.__init__(self, ddconfig, embed_dim, scale_factor)
            self._glg_cfg = _cfg_from_ddconfig(ddconfig, embed_dim, scale_factor)
            self._glg_engine, self._glg_stale = None, True

        def post_quant_conv_weight_device(self):
            return self.post_quant_conv.weight.device

        @torch.no_grad()
        def decode(self, z):
            if self.post_quant_conv.weight.device.type != "cuda":
                return _ref.AutoencoderKL.decode(self, z)          # the reference's own PyTorch path (CPU)
            return self._vae_engine().decode(z)

        @torch.no_grad()
        def encode(self, x):
            if self.post_quant_conv.weight.device.type != "cuda":
                return _ref.AutoencoderKL.encode(self, x)
            return _CudaDecodeMixin.encode(self, x)
else:
    class AutoencoderKL(_CudaDecodeMixin, nn.Module):
        """Parameters under the reference's names (no reference checkout behind this repo); compute is CUDA only."""

        def __init__(self, ddconfig, embed_dim, scale_factor=1):
            nn.Module.__init__(self)
            assert ddconfig["double_z"]
            self.embed_dim, self.scale_factor = embed_dim, scale_factor
            self._glg_cfg = _cfg_from_ddconfig(ddconfig, embed_dim, scale_factor)
            shapes = dict(vae_encoder_param_shapes(self._glg_cfg))
            shapes.update(vae_decoder_param_shapes(self._glg_cfg))
            attach_params(self, shapes, "")
            self._glg_engine, self._glg_stale = None, True

        def post_quant_conv_weight_device(self):
            return self.post_quant_conv.weight.device

        def forward(self, *a, **kw):
            raise RuntimeError("call decode(z)")


# names this drop-in does not define resolve to the reference module of the same name when a reference checkout
# follows this repo on sys.path (gligen_b200/_overlay.py)
__getattr__ = _overlay.fallback(__name__, __file__)
