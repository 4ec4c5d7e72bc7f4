"""Module *types* of the transformer blocks, kept at the reference's import path.

In this engine these classes are parameter containers only: the arithmetic of
reference ldm/modules/attention.py (SelfAttention :154-186, CrossAttention :102-149,
GatedSelfAttentionDense :215-244, BasicTransformerBlock :303-338, SpatialTransformer :341-376) runs as
fused sm_90a kernels driven by gligen_b200.engine; the containers exist so that
  * state_dict() keys equal the reference's (checkpoints load verbatim), and
  * `set_alpha_scale` (gligen_inference.py:24-28), which walks model.modules() and tests
    `type(module) == GatedSelfAttentionDense`, finds the fusers and sets `.scale` on them.
"""
import torch
import torch.nn as nn


class ParamNode(nn.Module):
    """A named bag of parameters / child nodes; children with integer names are indexable like
    nn.ModuleList / nn.Sequential (`model.input_blocks[0][0]`)."""

    def __getitem__(self, idx):
        return self._modules[str(idx)]

    def __setitem__(self, idx, module):
        self._modules[str(idx)] = module

    def __len__(self):
        return len(self._modules)

    def forward(self, *args, **kwargs):
        raise RuntimeError(f"{type(self).__name__} is a parameter container; call UNetModel.forward(input) "
                           "(the whole denoiser runs inside the gligen_b200 engine)")


def attach_params(root: ParamNode, shapes, strip: str, node_cls=lambda path: ParamNode):
    """Create nested ParamNodes + zero-initialised fp32 parameters for every `strip`-prefixed key."""
    for key, shape in shapes.items():
        if not key.startswith(strip):
            continue
        parts = key[len(strip):].split(".")
        node = root
        for i, name in enumerate(parts[:-1]):
            if name not in node._modules:
                node.add_module(name, node_cls(".".join(parts[: i + 1]))())
            node = node._modules[name]
        node.register_parameter(parts[-1], nn.Parameter(torch.zeros(shape), requires_grad=False))


class LinearAttention(nn.Module):
    """Softmax-over-keys linear attention on feature maps (reference attention.py:80-99).  NOT on the denoiser's path
    (no UNet config uses it); it lives here, as ordinary PyTorch, only because the reference's VAE module
    `ldm/modules/diffusionmodules/model.py:9` imports this name from `ldm.modules.attention`, which this file replaces
    in an overlay.  Parameter names (`to_qkv`, `to_out`) follow the reference so checkpoints load."""

    def __init__(self, dim, heads=4, dim_head=32):
        super().__init__()
        self.heads = heads
        inner = heads * dim_head
        self.to_qkv = nn.Conv2d(dim, 3 * inner, kernel_size=1, bias=False)
        self.to_out = nn.Conv2d(inner, dim, kernel_size=1)

    def forward(self, x):
        b, _, h, w = x.shape
        q, k, v = self.to_qkv(x).view(b, 3, self.heads, -1, h * w).unbind(dim=1)      # each [b, heads, d, n]
        ctx = torch.matmul(k.softmax(dim=-1), v.transpose(-1, -2))                   # [b, heads, d, e]
        out = torch.matmul(ctx.transpose(-1, -2), q)                                 # [b, heads, e, n]
        return self.to_out(out.reshape(b, -1, h, w))


class SelfAttention(ParamNode):
    pass


class CrossAttention(ParamNode):
    pass


class FeedForward(ParamNode):
    pass


class GatedSelfAttentionDense(ParamNode):
    """Fuser of visual and grounding tokens.  `scale` multiplies tanh(alpha) of both gated residuals; the
    engine reads it at the next forward and skips the fuser entirely when it is 0."""

    def __init__(self):
        super().__init__()
        self.scale = 1


class GatedCrossAttentionDense(ParamNode):
    """Importable for `set_alpha_scale`; no shipped config selects fuser_type=gatedCA (not accelerated)."""

    def __init__(self):
        super().__init__()
        self.scale = 1


class GatedSelfAttentionDense2(ParamNode):
    """Importable name only; no shipped config selects fuser_type=gatedSA2 (not accelerated)."""

    def __init__(self):
        super().__init__()
        self.scale = 1


class BasicTransformerBlock(ParamNode):
    pass


class SpatialTransformer(ParamNode):
    pass


# names this drop-in does not define resolve to the reference module of the same name when a reference checkout
# follows this repo on sys.path (gligen_b200/_overlay.py)
from gligen_b200._overlay import fallback as _fallback  # noqa: E402

__getattr__ = _fallback(__name__, __file__)
