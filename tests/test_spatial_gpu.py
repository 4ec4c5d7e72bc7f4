"""GPU: spatial grounding modalities (SURVEY 8f-4) through the C ABI.
  * every front-end kernel of csrc/frontend.cu (+ the GELU / quick-GELU GEMM epilogues) against its torch statement in tests/ref_ops.py;
  * grounding tokens (ConvNeXt-tiny tokenizer), downsampler planes and eps of the drop-in UNetModel against the fixtures written from the
    unmodified reference (tests/golden/spatial_*.pt): four tiny UNets behind the real ConvNeXt-tiny, and the full-size SD-1.4 hed and
    sem models.  Tolerance = the per-forward tolerance of the other tokenizers (DESIGN 2): rel-L2 <= 2.5e-2, max-abs <= 9 % of max|eps|;
    tokens after 18 bf16 ConvNeXt blocks: rel-L2 <= 2e-2.
  * a short PLMS loop with scheduled sampling on a spatial model: the SD first-conv swap happens mid-loop without re-planning."""
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


def rnd(*shape, scale=1.0, seed=0, dtype=torch.float32):
    g = torch.Generator(device="cpu").manual_seed(seed + sum(shape))
    return (torch.randn(*shape, generator=g) * scale).to(DEV).to(dtype)


@pytest.mark.parametrize("B,C,Hs,Hv,k,ldo", [(2, 3, 512, 256, 4, 64), (1, 3, 256, 256, 4, 64), (2, 3, 300, 128, 4, 64), (1, 5, 64, 64, 2, 24)])
def test_patchify_nchw(ops, ref, B, C, Hs, Hv, k, ldo):
    x = rnd(B, C, Hs, Hs + 16)
    rows = B * (Hv // k) * (Hv // k)
    out = torch.full((rows, ldo), 7.0, device=DEV, dtype=torch.bfloat16)
    out_r = torch.zeros(rows, ldo, device=DEV)
    ops.patchify_nchw(x, out, Hv, Hv, k)
    ref.patchify_nchw(x, out_r, Hv, Hv, k)
    assert torch.equal(out.float(), out_r.to(torch.bfloat16).float())          # a gather: bit-exact


@pytest.mark.parametrize("B,H,C,ld", [(2, 64, 96, 128), (1, 32, 192, 192), (3, 8, 384, 384)])
def test_patchify_nhwc(ops, ref, B, H, C, ld):
    x = rnd(B * H * H, ld, dtype=torch.bfloat16)
    out = torch.zeros(B * (H // 2) ** 2, 4 * C, device=DEV, dtype=torch.bfloat16)
    out_r = torch.zeros_like(out)
    ops.patchify_nhwc(x, out, H, H, C, 2)
    ref.patchify_nhwc(x, out_r, H, H, C, 2)
    assert torch.equal(out, out_r)


@pytest.mark.parametrize("rows,C,Cpad", [(4096, 96, 128), (1000, 192, 192), (37, 768, 768), (64, 384, 448)])
def test_layernorm_rows(ops, ref, rows, C, Cpad):
    x = (rnd(rows, Cpad, scale=1.5) + 0.7).to(torch.bfloat16)
    g, b = 1 + 0.1 * rnd(C, seed=1), 0.1 * rnd(C, seed=2)
    y = torch.full((rows, Cpad), 3.0, device=DEV, dtype=torch.bfloat16)
    y_r = torch.zeros(rows, Cpad, device=DEV)
    ops.layernorm_rows(x, y, g, b, C, 1e-6)
    ref.layernorm_rows(x, y_r, g, b, C, 1e-6)
    assert_close(y, y_r, what="layernorm_rows")
    assert float(y[:, C:].abs().sum()) == 0.0
    ops.layernorm_rows(x, x, g, b, C, 1e-6)                 # in place (the stem's LayerNorm)
    assert torch.equal(x, y)


@pytest.mark.parametrize("B,H,C,Cpad", [(2, 64, 96, 128), (1, 32, 192, 192), (2, 16, 384, 384), (3, 8, 768, 768), (1, 4, 768, 768)])
def test_dwconv7_ln(ops, ref, B, H, C, Cpad):
    x = rnd(B * H * H, Cpad, dtype=torch.bfloat16)
    w, bias = rnd(49, C, scale=1 / 7.0, seed=3), 0.1 * rnd(C, seed=4)
    g, b = 1 + 0.1 * rnd(C, seed=1), 0.1 * rnd(C, seed=2)
    y = torch.full((B * H * H, Cpad), 3.0, device=DEV, dtype=torch.bfloat16)
    y_r = torch.zeros(B * H * H, Cpad, device=DEV)
    ops.dwconv7_ln(x, y, w, bias, g, b, B, H, H, C, 1e-6)
    ref.dwconv7_ln(x, y_r, w, bias, g, b, B, H, H, C, 1e-6)
    assert_close(y, y_r, what="dwconv7_ln")
    assert float(y[:, C:].abs().sum()) == 0.0


def test_spatial_tokens(ops, ref):
    B, n, C = 3, 64, 768
    x = rnd(B * n, C, dtype=torch.bfloat16)
    mask = torch.tensor([1.0, 0.0, 1.0], device=DEV)
    null, pos = rnd(C, seed=1), 0.02 * rnd(n, C, seed=2)
    y, y_r = torch.zeros(B * n, C, device=DEV, dtype=torch.bfloat16), torch.zeros(B * n, C, device=DEV)
    ops.spatial_tokens(x, mask, null, pos, y, n)
    ref.spatial_tokens(x, mask, null, pos, y_r, n)
    assert_close(y, y_r, what="spatial_tokens")


@pytest.mark.parametrize("mode", ["nearest", "bicubic"])
@pytest.mark.parametrize("B,Cx,C,Hs,Ho", [(2, 3, 1, 512, 64), (2, 3, 1, 512, 256), (1, 3, 3, 512, 256), (2, 3, 3, 100, 256), (1, 2, 2, 64, 64)])
def test_resize_plane(ops, ref, mode, B, Cx, C, Hs, Ho):
    x = rnd(B, Cx, Hs, Hs)
    y, y_r = torch.zeros(B, C, Ho, Ho, device=DEV), torch.zeros(B, C, Ho, Ho, device=DEV)
    ops.resize_plane(x, y, C, mode)
    ref.resize_plane(x, y_r, C, mode)
    if mode == "nearest":
        assert torch.equal(y, y_r)
    else:
        assert (y - y_r).abs().max() <= 2e-5 * max(1.0, float(y_r.abs().max()))          # fp32, different summation order


@pytest.mark.parametrize("B,Cin,Cout,Hs,virtual,k,stride,pad,silu", [
    (2, 1, 4, 256, None, 4, 2, 1, True), (2, 4, 8, 128, None, 4, 2, 1, False), (1, 3, 4, 256, None, 4, 2, 1, True),
    (1, 152, 16, 512, (256, 256), 4, 2, 1, True), (2, 16, 8, 128, None, 4, 2, 1, False), (1, 152, 3, 512, (256, 256), 3, 1, 1, False),
    (2, 24, 3, 256, (128, 128), 3, 1, 1, False)])
def test_conv2d_small(ops, ref, B, Cin, Cout, Hs, virtual, k, stride, pad, silu):
    x = rnd(B, Cin, Hs, Hs)
    w, bias = rnd(Cin * k * k, Cout, scale=(Cin * k * k) ** -0.5, seed=1), 0.1 * rnd(Cout, seed=2)
    Hv = virtual[0] if virtual else Hs
    Ho = (Hv + 2 * pad - k) // stride + 1
    y, y_r = torch.zeros(B, Cout, Ho, Ho, device=DEV), torch.zeros(B, Cout, Ho, Ho, device=DEV)
    ops.conv2d_small(x, w, bias, y, k, stride, pad, silu, virtual=virtual)
    tf32 = torch.backends.cudnn.allow_tf32
    torch.backends.cudnn.allow_tf32 = False          # the checker must be fp32 (cuDNN convolutions default to TF32: 3e-4 off)
    try:
        ref.conv2d_small(x, w, bias, y_r, k, stride, pad, silu, virtual=virtual)
    finally:
        torch.backends.cudnn.allow_tf32 = tf32
    assert_close(y, y_r, rel=1e-5, max_rel=1e-4, what="conv2d_small")


@pytest.mark.parametrize("act", [2, 3])
@pytest.mark.parametrize("M,N,K", [(4096, 384, 128), (64, 3072, 768), (154, 3072, 768), (32, 512, 768)])
def test_gemm_gelu_epilogues(ops, ref, act, M, N, K):
    a, w = rnd(M, K, dtype=torch.bfloat16), rnd(N, K, scale=K ** -0.5, seed=1, dtype=torch.bfloat16)
    bias = 0.1 * rnd(N, seed=2)
    out, out_r = torch.zeros(M, N, device=DEV, dtype=torch.bfloat16), torch.zeros(M, N, device=DEV)
    ops.gemm(a, w, out, bias=bias, act=act)
    ref.gemm(a, w, out_r, bias=bias, act=act)
    assert_close(out, out_r, what=f"gemm act={act}")


# ---- the drop-in model against the reference fixtures ------------------------------------------------------------------------------
def _run(name, model=None):
    """The drop-in model (a fresh one, or `model`) on the inputs of fixture spatial_{name}.pt, against its eps."""
    from gligen_b200 import synth
    from gligen_b200.pipeline import build_model, sampler_inputs, to_device
    g = torch.load(os.path.join(GOLD, f"spatial_{name}.pt"))
    if model is None:
        cfg, model = build_model(g["config"], device=DEV)
    else:
        cfg = model.engine().cfg
    inp = synth.make_inputs(cfg, g["B"], seed=g["seed"], map_size=g.get("map_size"))
    ts = torch.tensor(g["timesteps"], device=DEV)
    dinp = to_device({k: v for k, v in inp.items() if k in ("x", "context", "uc")}, DEV)
    input, _, _ = sampler_inputs(cfg, model, dinp, to_device(inp["batch"], DEV))
    input["timesteps"] = ts
    e_c = model(input)
    null_in = dict(input, context=dinp["uc"])
    del null_in["grounding_input"]
    e_n = model(null_in)
    c2, n2 = model.forward_cfg(input, dinp["uc"])
    torch.cuda.synchronize()
    out = {}
    for got, key in ((e_c, "eps_cond"), (e_n, "eps_null"), (c2, "eps_cond"), (n2, "eps_null")):
        out[key] = assert_close(got, g[key], rel=2.5e-2, max_rel=9e-2, what=f"{name} {key}")
    print(f"{name}: eps rel-L2 / max-rel vs reference: cond {out['eps_cond'][0]:.3e} / {out['eps_cond'][1]:.3e}  null {out['eps_null'][0]:.3e} / {out['eps_null'][1]:.3e}")
    return cfg, model, g, inp


@pytest.mark.parametrize("name", ["tiny_hed", "tiny_canny", "tiny_depth", "tiny_normal", "tiny_sem",
                                  "tiny_hed_192x320", "tiny_normal_300x224", "tiny_sem_300x224"])
def test_forward_tiny_spatial(name):
    _run(name)


@pytest.mark.parametrize("square,other", [("tiny_hed", "tiny_hed_192x320"), ("tiny_sem", "tiny_sem_300x224")])
def test_map_size_change_replans(square, other):
    """One model fed a square map, then a non-square one, then the square one again: each result matches its own fixture,
    so no plan or static buffer sized for one map survives the change to the other."""
    _, model, _, _ = _run(square)
    _run(other, model)
    _run(square, model)


@pytest.mark.parametrize("name", ["sd14_hed", "sd14_sem"])
def test_forward_sd14_spatial(name):
    _run(name)


@pytest.mark.parametrize("name", ["tiny_depth", "sd14_hed", "sd14_sem"])
def test_tokens_and_planes(name):
    """The static front end alone: ConvNeXt tokens and downsampler planes against the reference's."""
    from gligen_b200 import synth
    from gligen_b200.engine import Engine
    from gligen_b200.ops import CudaOps
    from gligen_b200.spec import NAMED_CONFIGS, SPATIAL_MAP_KEY, synthetic_state_dict
    g = torch.load(os.path.join(GOLD, f"spatial_{name}.pt"))
    cfg = NAMED_CONFIGS[name]
    eng = Engine(cfg, CudaOps(DEV), use_graphs=False)
    eng.load_state_dict(synthetic_state_dict(cfg, 0))
    inp = synth.make_inputs(cfg, g["B"], seed=g["seed"])
    m = inp["batch"][SPATIAL_MAP_KEY[cfg.tokenizer]].to(DEV)
    gr = {SPATIAL_MAP_KEY[cfg.tokenizer]: m, "mask": inp["batch"]["mask"].to(DEV)}
    seen = {}
    orig_gemm, orig_conv_in = eng.ops.gemm, eng.ops.conv_in
    def gemm(a, w, out, **kw):
        orig_gemm(a, w, out, **kw)
        if w is eng.W["pn.l4.w"]:
            seen["objs"] = out.float().clone()
    def conv_in(x, extra, w, b, o):
        seen["ds"] = extra.clone()
        orig_conv_in(x, extra, w, b, o)
    eng.ops.gemm, eng.ops.conv_in = gemm, conv_in
    eng.forward(inp["x"].to(DEV), torch.tensor(g["timesteps"], device=DEV), inp["context"].to(DEV), gr, None, m)
    torch.cuda.synchronize()
    r = assert_close(seen["objs"].view(g["objs"].shape), g["objs"], rel=2e-2, max_rel=8e-2, what=f"{name} tokens")
    d = assert_close(seen["ds"], g["ds"], rel=1e-4, max_rel=1e-3, what=f"{name} downsampler planes")
    print(f"{name}: tokens rel-L2 {r[0]:.3e} max-rel {r[1]:.3e}; downsampler planes rel-L2 {d[0]:.3e}")


def test_plms_with_first_conv_swap_on_a_spatial_model():
    """PLMS S=4, alpha_type [0.5, 0, 0.5], CFG 5 on the full-size hed model against the REFERENCE sampler's latent: from step 2 on
    the sampler calls restore_first_conv_from_SD, which for a model with a grounding downsampler swaps in SD's 4-channel conv and
    drops the downsampler planes (engine: zero weights on those channels, no re-plan)."""
    from functools import partial
    from gligen_b200 import synth
    from gligen_b200.pipeline import alpha_generator, build_model, sampler_inputs, set_alpha_scale, to_device
    from ldm.models.diffusion.ldm import LatentDiffusion
    from ldm.models.diffusion.plms import PLMSSampler
    g = torch.load(os.path.join(GOLD, "spatial_sd14_hed.pt"))
    gp = g["plms"]
    cfg, model = build_model("sd14_hed", device=DEV)
    inp = synth.make_inputs(cfg, g["B"], seed=g["seed"])
    dinp = to_device({k: v for k, v in inp.items() if k in ("x", "context", "uc")}, DEV)
    input, _, _ = sampler_inputs(cfg, model, dinp, to_device(inp["batch"], DEV))
    diffusion = LatentDiffusion(linear_start=0.00085, linear_end=0.012, timesteps=1000).to(DEV)
    sampler = PLMSSampler(diffusion, model, alpha_generator_func=partial(alpha_generator, type=gp["alpha_type"]), set_alpha_scale=set_alpha_scale)
    cwd = os.getcwd()
    os.chdir(GOLD)                  # SD_input_conv_weight_bias.pth is read CWD-relative, like the reference
    try:
        torch.manual_seed(1234)
        shape = (g["B"], cfg.in_channels, cfg.image_size, cfg.image_size)
        lat = sampler.sample(S=gp["S"], shape=shape, input=input, uc=dinp["uc"], guidance_scale=gp["guidance"])
    finally:
        os.chdir(cwd)
    assert model.first_conv_type == "SD" and model.input_blocks[0][0].weight.shape[1] == 4
    assert len(model.engine().plans) == 1
    r = assert_close(lat, gp["latent"], rel=6e-2, max_rel=0.1, what="sd14_hed PLMS S=4 latent")
    print(f"sd14_hed PLMS S=4 alpha={gp['alpha_type']}: latent rel-L2 {r[0]:.3e} max-rel {r[1]:.3e}")
