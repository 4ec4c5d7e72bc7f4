"""GroupNorm, the row LayerNorms (plain, dwconv7_ln, CLIP vision embed / head), softmax_rows, the CUDA-core edge
convolutions, the embeddings and the sampler update against float64.

Bounded checks use the derived per-element bounds of tests/bounds.py on adversarial inputs: every (sample, group) or row
with its own mean (|mean| / std up to 100) and std (1e-3 .. 1e3), outliers at each GroupNorm path's pivot, constant
groups and groups with variance near eps.  Every GroupNorm kernel is reached on purpose; which one ran is read from the
profiler's kernel names and compared with the dispatch rule restated in bounds.gn_dispatch.  The edge convolutions are
checked exactly, on inputs whose every partial sum is representable in fp32, and the kernel variant each case reaches
is read from the profiler."""
import os
import subprocess
import sys

import pytest
import torch

import bounds
from gligen_b200.ops import gn_scratch_floats
from test_bounds_norm_cpu import exact_conv_out_inputs, gn_input, ln_input

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
BF = torch.bfloat16
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def ops():
    from gligen_b200.ops import CudaOps
    return CudaOps(DEV)


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _affine(C, seed):
    g = torch.Generator().manual_seed(seed)
    return (1 + 0.3 * torch.randn(C, generator=g)).to(DEV), (0.2 * torch.randn(C, generator=g)).to(DEV)


def _kernels_run(fn):
    """Names of the CUDA kernels `fn` launches."""
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    return [e.name for e in prof.events() if e.device_type.name == "CUDA"]


GN_KERNEL = {"reg5": "gn_reg_kernel<5>", "reg10": "gn_reg_kernel<10>", "reg20": "gn_reg_kernel<20>",
             "small": "gn_small_kernel", "fused": "gn_fused_kernel"}


def _strided(t, lead):
    """t [B, HW, C] copied into columns [lead, lead + C) of a wider buffer whose row stride stays a multiple of 8."""
    B, HW, C = t.shape
    big = torch.zeros(B, HW, C + -(-2 * lead // 8) * 8, device=DEV, dtype=t.dtype)
    big[:, :, lead:lead + C] = t
    return big[:, :, lead:lead + C]


def _gn_run(ops, x, y, gamma, beta, stats, G, eps, silu, path):
    ops.groupnorm(x, y, gamma, beta, stats, G, eps, silu)
    torch.cuda.synchronize()
    rep = bounds.groupnorm_check(y, x, gamma, beta, G, eps, silu, path, num_sms=_sms(),
                                 what=f"groupnorm x={tuple(x.shape)}/{x.stride()} silu={silu} eps={eps}")
    print(rep)
    return rep


# ---- every dispatch path, confirmed from the profiler ------------------------------------------------------------------
PATH_CASES = [  # B, HW, C, lead (x column offset; 2 = a 4-byte-aligned view), expected path
    (2, 64, 1280, 0, "reg5"),        # cpg 40: 640 units
    (2, 256, 1280, 0, "reg10"),      # 2560 units
    (2, 256, 2560, 0, "reg20"),      # cpg 80: 5120 units
    (2, 256, 1920, 8, "reg20"),      # cpg 60, strided rows
    (2, 256, 320, 0, "small"),       # cpg 10: cpg % 4 != 0
    (2, 64, 1280, 2, "small"),       # x 4-byte but not 8-byte aligned
    (2, 4096, 320, 0, "fused"),
    (1, 4096, 640, 8, "fused"),
]


@pytest.mark.parametrize("B,HW,C,lead,path", PATH_CASES)
@pytest.mark.parametrize("silu", [False, True])
def test_groupnorm_paths(ops, B, HW, C, lead, path, silu):
    G = 32
    x = _strided(gn_input(B, HW, C, G, 100 + HW + C).to(DEV), lead)
    assert bounds.gn_dispatch(B, HW, C, G, aligned8=x.data_ptr() % 8 == 0) == path
    gamma, beta = _affine(C, 1)
    y = _strided(torch.zeros(B, HW, C, device=DEV, dtype=BF), 8)
    stats = torch.zeros(gn_scratch_floats(B), device=DEV)
    names = _kernels_run(lambda: ops.groupnorm(x, y, gamma, beta, stats, G, 1e-6, silu))
    assert sum(GN_KERNEL[path] in n for n in names) == 1, names
    rep = _gn_run(ops, x, y, gamma, beta, stats, G, 1e-6, silu, path)
    assert rep.ok, str(rep)


# ---- real shapes -------------------------------------------------------------------------------------------------------
UNET_C = [320, 640, 960, 1280, 1920, 2560]
UNET_HW = [4096, 1024, 256, 64]


@pytest.mark.parametrize("C", UNET_C)
@pytest.mark.parametrize("HW", UNET_HW)
def test_groupnorm_unet_shapes(ops, C, HW):
    B, G = 2, 32
    x = gn_input(B, HW, C, G, HW + C).to(DEV)
    gamma, beta = _affine(C, 2)
    y = torch.zeros(B, HW, C, device=DEV, dtype=BF)
    stats = torch.zeros(gn_scratch_floats(B), device=DEV)
    rep = _gn_run(ops, x, y, gamma, beta, stats, G, 1e-5, True, bounds.gn_dispatch(B, HW, C, G))
    assert rep.ok, str(rep)


@pytest.mark.parametrize("B,HW,C", [(1, 4096, 320), (8, 1024, 640), (64, 256, 320), (64, 4096, 320), (8, 64, 2560),
                                    (64, 1000, 640)])                          # 1000 rows: a ragged last chunk
def test_groupnorm_batches(ops, B, HW, C):
    G = 32
    x = _strided(gn_input(B, HW, C, G, B + HW + C).to(DEV), 8)
    gamma, beta = _affine(C, 3)
    y = torch.zeros(B, HW, C, device=DEV, dtype=BF)
    stats = torch.zeros(gn_scratch_floats(B), device=DEV)
    rep = _gn_run(ops, x, y, gamma, beta, stats, G, 1e-5, False, bounds.gn_dispatch(B, HW, C, G))
    assert rep.ok, str(rep)
    assert int(stats[:128].view(torch.int32).abs().sum()) == 0


@pytest.mark.parametrize("HW,C", [(512 * 512, 128), (256 * 256, 256), (128 * 128, 512), (64 * 64, 512)])
def test_groupnorm_vae_shapes(ops, HW, C):
    """The VAE's GroupNorms (eps 1e-6): the longest reductions of the project, up to 512^2 rows x 128 channels."""
    B, G = 1, 32
    x = gn_input(B, HW, C, G, HW + C, ratio=30.0).to(DEV)
    gamma, beta = _affine(C, 4)
    y = torch.zeros(B, HW, C, device=DEV, dtype=BF)
    stats = torch.zeros(gn_scratch_floats(B), device=DEV)
    path = bounds.gn_dispatch(B, HW, C, G)
    assert path == "fused"
    rep = _gn_run(ops, x, y, gamma, beta, stats, G, 1e-6, True, path)
    assert rep.ok, str(rep)


def test_groupnorm_scratch_reuse(ops):
    """One stats buffer: input A, then a different input B of the same shape (partials left by A must not leak), then
    another input with a different B and HW.  Each against float64; the barrier counters re-arm themselves."""
    G, C = 32, 640
    gamma, beta = _affine(C, 5)
    stats = torch.zeros(gn_scratch_floats(8), device=DEV)
    for i, (B, HW, ratio) in enumerate([(8, 1024, 3.0), (8, 1024, 100.0), (3, 2000, 30.0)]):
        x = gn_input(B, HW, C, G, 200 + i, ratio=ratio).to(DEV)
        y = torch.zeros(B, HW, C, device=DEV, dtype=BF)
        rep = _gn_run(ops, x, y, gamma, beta, stats, G, 1e-5, i == 1, "fused")
        assert rep.ok, f"call {i}: {rep}"
        assert int(stats[:128].view(torch.int32).abs().sum()) == 0


_FORCED_FUSED = r"""
import os, sys
sys.path[:0] = [{root!r}, {tests!r}]
import torch
import bounds
from gligen_b200.ops import CudaOps, gn_scratch_floats
from test_bounds_norm_cpu import gn_input
ops = CudaOps("cuda:0")
sms = torch.cuda.get_device_properties(0).multi_processor_count
worst = 0.0
for B, HW, C in ((2, 256, 1280), (2, 64, 2560), (4, 256, 320), (1, 16, 640)):
    x = gn_input(B, HW, C, 32, HW + C).cuda()
    g = torch.Generator().manual_seed(C)
    gamma, beta = (1 + 0.3 * torch.randn(C, generator=g)).cuda(), (0.2 * torch.randn(C, generator=g)).cuda()
    y = torch.zeros(B, HW, C, device="cuda:0", dtype=torch.bfloat16)
    stats = torch.zeros(gn_scratch_floats(B), device="cuda:0")
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        ops.groupnorm(x, y, gamma, beta, stats, 32, 1e-6, True)
        torch.cuda.synchronize()
    names = [e.name for e in prof.events() if e.device_type.name == "CUDA"]
    assert sum("gn_fused_kernel" in n for n in names) == 1, names
    rep = bounds.groupnorm_check(y, x, gamma, beta, 32, 1e-6, True, "fused", num_sms=sms, what=f"forced fused {{(B, HW, C)}}")
    print(rep)
    assert rep.ok, str(rep)
print("forced-fused ok")
"""


def test_groupnorm_fused_forced_on_small_shapes():
    """GLG_GN_SMALL=0 sends H*W <= 256 through the barrier kernel too; the setting is read once per process, so the
    check runs in a short child process."""
    env = dict(os.environ, GLG_GN_SMALL="0")
    code = _FORCED_FUSED.format(root=ROOT, tests=os.path.join(ROOT, "tests"))
    r = subprocess.run([sys.executable, "-c", code], env=env, capture_output=True, text=True, timeout=600)
    print(r.stdout[-4000:], r.stderr[-4000:])
    assert r.returncode == 0 and "forced-fused ok" in r.stdout


# ---- LayerNorms --------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("C", [512, 520, 1280, 1288, 2048])              # the MAXV 2 / 5 / 8 edges of ln_kernel
def test_layernorm_maxv_edges(ops, C):
    B, rows = 3, 50
    x = ln_input(B * rows, C, C, 100.0).view(B, rows, C).to(DEV)
    gamma, beta = _affine(C, 6)
    big = torch.full((B, rows + 5, C), float("nan"), device=DEV, dtype=BF)
    y = big[:, 5:]                                                         # batch-strided output
    ops.layernorm(x, y, gamma, beta, 1e-5)
    torch.cuda.synchronize()
    rep = bounds.layernorm_check(y, x, gamma, beta, 1e-5, what=f"layernorm C={C}")
    print(rep)
    assert rep.ok, str(rep)
    assert torch.isnan(big[:, :5].float()).all(), "rows outside the batch-strided view must stay untouched"


@pytest.mark.parametrize("C,Cpad", [(768, 768), (768, 832), (1024, 1024), (1000, 1024), (320, 1024)])
def test_layernorm_rows(ops, C, Cpad):
    R = 333
    x = torch.zeros(R, Cpad, dtype=BF)
    x[:, :C] = ln_input(R, C, C + Cpad, 100.0)
    x = x.to(DEV)
    gamma, beta = _affine(C, 7)
    y = torch.full((R, Cpad), float("nan"), device=DEV, dtype=BF)
    ops.layernorm_rows(x, y, gamma, beta, C, 1e-6)
    torch.cuda.synchronize()
    rep = bounds.layernorm_check(y[:, :C], x[:, :C], gamma, beta, 1e-6, what=f"layernorm_rows C={C} Cpad={Cpad}")
    print(rep)
    assert rep.ok, str(rep)
    assert torch.equal(y[:, C:], torch.zeros_like(y[:, C:])), "padding columns must be zeroed"
    ops.layernorm_rows(x, x, gamma, beta, C, 1e-6)                         # in place
    torch.cuda.synchronize()
    assert torch.equal(x, y)


@pytest.mark.parametrize("C", [768, 1024])
def test_layernorm_rows_f32(ops, C):
    R = 154
    x = ln_input(R, C, C, 100.0).to(DEV)
    gamma, beta = _affine(C, 8)
    y = torch.full((R, C), float("nan"), device=DEV)
    ops.layernorm_rows_f32(x, y, gamma, beta, 1e-5)
    torch.cuda.synchronize()
    rep = bounds.layernorm_check(y, x, gamma, beta, 1e-5, what=f"layernorm_rows_f32 C={C}")
    print(rep)
    assert rep.ok, str(rep)


@pytest.mark.parametrize("B,H,W,C,Cpad", [(2, 16, 16, 96, 128), (1, 8, 8, 768, 768), (2, 3, 5, 192, 256)])
def test_dwconv7_ln(ops, B, H, W, C, Cpad):
    """Depthwise 7x7 + bias + LayerNorm (ConvNeXt tokenizer blocks) against float64: channels with their own offsets (rows
    then carry |mean| / std far from 0), the 3-pixel borders, and padding columns [C, Cpad) that come back as zeros."""
    g = torch.Generator().manual_seed(C + H)
    x = torch.randn(B * H * W, Cpad, generator=g) + 5 * torch.randn(1, Cpad, generator=g)
    x = x.to(DEV, BF)
    w = (0.1 * torch.randn(49, C, generator=g)).to(DEV)
    bias, (gamma, beta) = (torch.randn(C, generator=g)).to(DEV), _affine(C, 10)
    y = torch.full((B * H * W, Cpad), float("nan"), device=DEV, dtype=BF)
    ops.dwconv7_ln(x, y, w, bias, gamma, beta, B, H, W, C, 1e-6)
    torch.cuda.synchronize()
    assert torch.equal(y[:, C:], torch.zeros_like(y[:, C:]))
    rep = bounds.dwconv7_ln_check(y, x, w, bias, gamma, beta, B, H, W, C, 1e-6, what=f"dwconv7_ln C={C}")
    print(rep)
    assert rep.ok, str(rep)


@pytest.mark.parametrize("ratio", [0.0, 100.0])
def test_clip_vision_embed(ops, ratio):
    """ViT-L/14 input rows: N images x (256 patches + class token), C = 1024; patch rows with their own mean / std."""
    N, P, C = 2, 256, 1024
    g = torch.Generator().manual_seed(int(ratio) + 1)
    std = 10.0 ** (2 * torch.rand(N * P, 1, generator=g) - 1)
    patch = (std * (ratio * (2 * torch.rand(N * P, 1, generator=g) - 1) + torch.randn(N * P, C, generator=g))).to(DEV)
    cls, pos = torch.randn(C, generator=g).to(DEV), (0.1 * torch.randn(P + 1, C, generator=g)).to(DEV)
    gamma, beta = _affine(C, 11)
    x = torch.full((N * (P + 1), C), float("nan"), device=DEV, dtype=BF)
    ops.clip_vision_embed(patch, cls, pos, gamma, beta, x, P, 1e-5)
    torch.cuda.synchronize()
    rep = bounds.clip_vision_embed_check(x, patch, cls, pos, gamma, beta, P, 1e-5)
    print(rep)
    assert rep.ok, str(rep)


def test_clip_image_head(ops):
    """Pooled output (post-LayerNorm of each image's class token, fp32) and the visual projection, C = 1024, D = 768."""
    N, T_, C, D = 3, 257, 1024, 768
    g = torch.Generator().manual_seed(12)
    x = (torch.randn(N, T_, C, generator=g) * torch.tensor([0.1, 3.0, 30.0]).view(N, 1, 1) + 2.0).to(DEV, BF)
    gamma, beta = _affine(C, 13)
    w = (torch.randn(D, C, generator=g) * C ** -0.5).to(DEV)
    pooled, emb = torch.full((N, C), float("nan"), device=DEV), torch.full((N, D), float("nan"), device=DEV)
    ops.clip_image_head(x, gamma, beta, w, pooled, emb)
    torch.cuda.synchronize()
    rep = bounds.clip_image_head_check(pooled, emb, x, gamma, beta, w, 1e-5)
    print(rep)
    assert rep.ok, str(rep)


def test_timestep_embedding(ops):
    t = torch.tensor([0, 1, 21, 500, 981, 999], device=DEV)
    for dim in (320, 1280):
        out = torch.full((t.numel(), dim), float("nan"), device=DEV, dtype=BF)
        ops.timestep_embedding(t, out)
        torch.cuda.synchronize()
        rep = bounds.timestep_embedding_check(out, t, what=f"timestep_embedding dim={dim}")
        print(rep)
        assert rep.ok, str(rep)


@pytest.mark.parametrize("F_,nc,ldo,bc", [(768, 4, 832, False), (768, 2, 832, True), (1024, 4, 1088, False)])
def test_position_features(ops, F_, nc, ldo, bc):
    B, N = 3, 30
    g = torch.Generator().manual_seed(F_ + nc)
    feat = torch.randn(*((N, F_) if bc else (B, N, F_)), generator=g).to(DEV)
    fm = (torch.rand(B, N, generator=g) > 0.4).float().to(DEV)
    pm = (torch.rand(B, N, generator=g) > 0.4).float().to(DEV)
    coords = torch.rand(B, N, nc, generator=g).to(DEV)
    nf, npos = torch.randn(F_, generator=g).to(DEV), torch.randn(16 * nc, generator=g).to(DEV)
    out = torch.full((B * N, ldo), float("nan"), device=DEV, dtype=BF)
    ops.position_features(feat, fm, nf, coords, pm, npos, out, 8)
    torch.cuda.synchronize()
    rep = bounds.position_features_check(out, feat, fm, nf, coords, pm, npos, 8)
    print(rep)
    assert rep.ok, str(rep)


def test_sampler_update(ops):
    """DDIM (1 term) and PLMS (2 and 4 terms) updates at the latent shape, late and early in the schedule."""
    n = (4, 4, 64, 64)
    g = torch.Generator().manual_seed(14)
    xs, ec, eu, o1, o2, o3 = ((torch.randn(*n, generator=g) * s).to(DEV) for s in (30.0, 1, 1, 1, 1, 1))
    for (a_t, a_prev) in ((0.0047, 0.0052), (0.62, 0.9991)):
        for olds, coefs in (([], (1.0, 0, 0, 0)), ([o1], (1.5, -0.5, 0, 0)), ([o1, o2, o3], (55 / 24, -59 / 24, 37 / 24, -9 / 24))):
            e, xp = torch.zeros(n, device=DEV), torch.zeros(n, device=DEV)
            ops.sampler_update(xs, ec, eu, 7.5, olds, coefs, a_t, a_prev, e, xp)
            torch.cuda.synchronize()
            rep = bounds.sampler_update_check(e, xp, xs, ec, eu, 7.5, olds, coefs, a_t, a_prev,
                                              what=f"sampler_update terms={len(olds) + 1} a_t={a_t}")
            print(rep)
            assert rep.ok, str(rep)


# ---- softmax_rows ------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("cols", [4, 1020, 1024, 1028, 4096])
@pytest.mark.parametrize("std", [1.0, 8.0, 30.0])
def test_softmax_rows(ops, cols, std):
    R, lds = 40, cols + 12
    g = torch.Generator().manual_seed(cols + int(std))
    big = torch.randn(R, lds, generator=g) * std
    big[5, cols // 3] = 40.0 * std                                         # a single dominant column
    s = big.to(DEV)[:, :cols]
    pbig = torch.full((R, cols + 8), float("nan"), device=DEV, dtype=BF)
    p = pbig[:, :cols]
    ops.softmax_rows(s, p, 0.0625)
    torch.cuda.synchronize()
    rep = bounds.softmax_check(p, s, 0.0625, what=f"softmax_rows cols={cols} std={std}")
    print(rep)
    assert rep.ok, str(rep)
    assert torch.isnan(pbig[:, cols:].float()).all()


def test_softmax_rows_rejects_unaligned_output_rows(ops):
    """softmax_rows_kernel writes 4 bf16 probabilities as one 8-byte store: an output row stride of 2 mod 4 elements
    would put every other row's stores off 8-byte alignment.  glg_softmax_rows used to accept ldp % 2 == 0 and
    launch; it must refuse such a layout up front.  Should that host check ever be removed, this call launches the
    misaligned store and the resulting device error ends the rest of the session's GPU tests: run this file on its
    own to find it.  The output buffer is 8-byte aligned and only the row stride is wrong, so nothing else can fault."""
    s = torch.randn(4, 8, device=DEV)
    pbig = torch.zeros(4, 10, device=DEV, dtype=BF)
    with pytest.raises(RuntimeError, match="glg_softmax_rows"):
        ops.softmax_rows(s, pbig[:, :8], 1.0)
    torch.cuda.synchronize()


# ---- edge convolutions, exactly ----------------------------------------------------------------------------------------
def _conv_out_kernel(W, Cout):
    """glg_conv_out's choice (elementwise.cu), restated."""
    return f"conv_out_px8_kernel<{Cout}>" if W % 8 == 0 and Cout in (3, 4) else f"conv_out_kernel<{Cout}>"


CONV_OUT_CASES = [  # B, H, W, Cin, Cout, x row lead: W % 8 == 0 -> conv_out_px8_kernel (Cout 3 / 4), else conv_out_kernel
    (2, 64, 64, 320, 4, 0), (1, 3, 8, 320, 3, 8), (2, 1, 16, 128, 4, 0), (1, 2, 8, 320, 4, 16),
    (2, 5, 7, 320, 4, 0), (1, 3, 1, 320, 3, 8), (2, 1, 2, 256, 8, 0), (1, 2, 3, 128, 4, 8), (1, 9, 9, 320, 8, 0),
]


def test_conv_out_cases_reach_every_variant():
    """The profiler does not report conv_out's launches reliably, so the variant of each case comes from the restated
    dispatch: every kernel of glg_conv_out must be reached by CONV_OUT_CASES."""
    reached = {_conv_out_kernel(W, Cout) for _, _, W, _, Cout, _ in CONV_OUT_CASES}
    assert reached == {"conv_out_px8_kernel<3>", "conv_out_px8_kernel<4>", "conv_out_kernel<3>", "conv_out_kernel<4>",
                       "conv_out_kernel<8>"}, reached


@pytest.mark.parametrize("B,H,W,Cin,Cout,lead", CONV_OUT_CASES)
def test_conv_out_exact(ops, B, H, W, Cin, Cout, lead):
    x, w, bias = exact_conv_out_inputs(B, H, W, Cin, Cout, H * W + Cin + Cout)
    exact = torch.nn.functional.conv2d(x.double().reshape(B, H, W, Cin).permute(0, 3, 1, 2),
                                       w.double().view(3, 3, Cout, Cin).permute(2, 3, 0, 1), bias.double(), padding=1)
    xs = _strided(x.to(DEV), lead)
    out = torch.full((B, Cout, H, W), float("nan"), device=DEV)
    ops.conv_out(xs, w.to(DEV), bias.to(DEV), out, H, W)
    torch.cuda.synchronize()
    assert torch.equal(out.double().cpu(), exact), f"max |diff| {(out.double().cpu() - exact).abs().max().item()}"


def exact_conv_in_inputs(B, C0, C1, H, W, Cout, seed):
    g = torch.Generator().manual_seed(seed)
    x = torch.randint(-3, 4, (B, C0, H, W), generator=g).float()
    extra = torch.randint(-3, 4, (B, C1, H, W), generator=g).float() if C1 else None
    w = torch.randint(-1023, 1024, (9, C0 + C1, Cout), generator=g).float() * 2.0 ** -10
    bias = torch.randint(-4096, 4097, (Cout,), generator=g).float() * 2.0 ** -10
    return x, extra, w, bias


CONV_IN_CASES = [  # B, C0, C1, H, W, Cout, out row lead: W % 4 == 0 and a large grid -> conv_in_px4_kernel
    (2, 4, 0, 64, 64, 320, 0), (2, 4, 5, 64, 64, 320, 160), (4, 4, 0, 32, 128, 320, 0),
    (2, 4, 0, 5, 7, 320, 0), (1, 4, 5, 3, 1, 320, 16), (2, 9, 0, 1, 2, 64, 0), (1, 4, 0, 2, 3, 128, 8), (1, 4, 5, 8, 8, 64, 0),
]


PX4_EXPECTED = {(2, 4, 0, 64, 64, 320), (2, 4, 5, 64, 64, 320), (4, 4, 0, 32, 128, 320)}


@pytest.mark.parametrize("B,C0,C1,H,W,Cout,lead", CONV_IN_CASES)
def test_conv_in_exact(ops, B, C0, C1, H, W, Cout, lead):
    x, extra, w, bias = exact_conv_in_inputs(B, C0, C1, H, W, Cout, H * W + C0 + C1 + Cout)
    xin = x if extra is None else torch.cat([x, extra], 1)
    exact = torch.nn.functional.conv2d(xin.double(), w.double().view(3, 3, C0 + C1, Cout).permute(3, 2, 0, 1), bias.double(), padding=1)
    exact = exact.permute(0, 2, 3, 1).reshape(B, H * W, Cout)
    out = _strided(torch.full((B, H * W, Cout), float("nan"), device=DEV, dtype=BF), lead)
    names = _kernels_run(lambda: ops.conv_in(x.to(DEV), None if extra is None else extra.to(DEV), w.to(DEV), bias.to(DEV), out))
    px4 = W % 4 == 0 and 9 * (C0 + C1) * Cout * 4 <= 110 * 1024 and B * H * W * Cout // 8 >= 4 * 256 * 64
    assert sum(("conv_in_px4_kernel" if px4 else "conv_in_kernel(") in n for n in names) == 1, names
    assert px4 == ((B, C0, C1, H, W, Cout) in PX4_EXPECTED)
    want = exact.to(BF)                                                    # the exact sum, rounded once
    assert torch.equal(out.cpu(), want), f"{(out.cpu().double() != want.double()).sum().item()} elements differ"
