"""GPU: the CLIP text encoder (SURVEY 8f-3) through the C ABI against the library fixture (tests/golden/clip_text_*.pt), and the
kernels it adds: causal mask of the short-key attention kernel, token-embedding gather, fp32-output LayerNorm.
Tolerance: 12 bf16 pre-LN blocks -> rel-L2 <= 1.5e-2, max-abs <= 6 % of max|z| on last_hidden_state and pooler_output (the UNet
reads the context in bf16 anyway: `context.cast`)."""
import os

import pytest
import torch

from conftest import GOLD, assert_close
from ref_ops import RefOps

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


@pytest.fixture(scope="module")
def ops():
    from gligen_b200.ops import CudaOps
    return CudaOps(DEV)


@pytest.fixture(scope="module")
def ref():
    return RefOps(DEV, torch.float32)


def rnd(*shape, scale=1.0, seed=0, dtype=torch.bfloat16):
    g = torch.Generator(device="cpu").manual_seed(seed + sum(shape))
    return (torch.randn(*shape, generator=g) * scale).to(DEV).to(dtype)


@pytest.mark.parametrize("B,heads,d,L", [(2, 12, 64, 77), (3, 2, 64, 40), (1, 8, 40, 128), (2, 4, 80, 16), (1, 12, 64, 1)])
def test_causal_attention(ops, ref, B, heads, d, L):
    C = heads * d
    qkv = rnd(B, L, 3 * C)
    out, out_r = torch.zeros(B, L, C, device=DEV, dtype=torch.bfloat16), torch.zeros(B, L, C, device=DEV)
    ops.attention(qkv[:, :, :C], qkv[:, :, C:2 * C], qkv[:, :, 2 * C:], out, heads, d, causal=True)
    ref.attention(qkv[:, :, :C], qkv[:, :, C:2 * C], qkv[:, :, 2 * C:], out_r, heads, d, causal=True)
    assert_close(out, out_r, rel=1e-2, max_rel=5e-2, what=f"causal attention {L}x{L} d={d}")
    # row 0 sees only key 0: its output is V[0]
    assert_close(out[:, 0], qkv[:, 0, 2 * C:], rel=1e-2, max_rel=2e-2, what="row 0 == V[0]")


def test_causal_needs_short_keys(ops):
    from gligen_b200.lib import GligenLibraryError
    qkv = rnd(1, 256, 3 * 64)
    out = torch.zeros(1, 256, 64, device=DEV, dtype=torch.bfloat16)
    with pytest.raises(GligenLibraryError):
        ops.attention(qkv[:, :, :64], qkv[:, :, 64:128], qkv[:, :, 128:], out, 1, 64, causal=True)


def test_embed_tokens_and_f32_layernorm(ops, ref):
    V, C, B, L = 1000, 768, 3, 77
    table, pos = rnd(V, C, dtype=torch.float32), 0.01 * rnd(L, C, seed=1, dtype=torch.float32)
    ids = torch.randint(0, V, (B, L), device=DEV)
    x, x_r = torch.zeros(B * L, C, device=DEV, dtype=torch.bfloat16), torch.zeros(B * L, C, device=DEV)
    ops.embed_tokens(ids, table, pos, x)
    ref.embed_tokens(ids, table, pos, x_r)
    assert torch.equal(x, x_r.to(torch.bfloat16))
    g, b = 1 + 0.1 * rnd(C, seed=2, dtype=torch.float32), 0.1 * rnd(C, seed=3, dtype=torch.float32)
    y, y_r = torch.zeros(B * L, C, device=DEV), torch.zeros(B * L, C, device=DEV)
    ops.layernorm_rows_f32(x, y, g, b, 1e-5)
    ref.layernorm_rows_f32(x, y_r, g, b, 1e-5)
    assert (y - y_r).abs().max() <= 1e-4


@pytest.mark.parametrize("name", ["tiny_clip_text", "sd14_clip_text"])
def test_text_encoder_vs_library(name):
    from gligen_b200.clip_text import NAMED_CLIP_CONFIGS, synthetic_clip_state_dict
    from ldm.util import instantiate_from_config
    g = torch.load(os.path.join(GOLD, f"clip_text_{name}.pt"))
    cfg = NAMED_CLIP_CONFIGS[name]
    m = instantiate_from_config(dict(target="ldm.modules.encoders.modules.FrozenCLIPEmbedder", params=dict(text_config=name))).to(DEV).eval()
    m.load_state_dict(synthetic_clip_state_dict(cfg, 0))
    z, pooled = m.encode_tokens(g["input_ids"], return_pooler_output=True)
    torch.cuda.synchronize()
    r1 = assert_close(z, g["last_hidden_state"], rel=1.5e-2, max_rel=6e-2, what=f"{name} last_hidden_state")
    r2 = assert_close(pooled, g["pooler_output"], rel=1.5e-2, max_rel=6e-2, what=f"{name} pooler_output")
    z1 = m.encode_tokens(g["input_ids"][:1])                  # another batch size
    assert_close(z1, g["last_hidden_state"][:1], rel=1.5e-2, max_rel=6e-2, what=f"{name} B=1")
    print(f"{name}: last_hidden_state rel-L2 {r1[0]:.3e} max-rel {r1[1]:.3e}; pooler_output rel-L2 {r2[0]:.3e} max-rel {r2[1]:.3e}")
