"""768 x 768 and 1024 x 1024 images, and the production forwards the op census had not run.

The engine samples any latent whose sides are multiples of 8.  At 768^2 and 1024^2 the kernels run at shapes no other
test reaches: self-attention over 9216 and 16384 tokens, fuser attention over T + 30 keys with a ragged last key tile,
softmax rows of 9216 and 16384 columns and a 16384 x 16384 fp32 score matrix in the VAE, GroupNorm reductions over up to
2^20 rows (more cross-CTA chunks), 3x3 convolutions over ~1 M pixels per image at widths up to 1024, and the data-movement
and edge kernels of 1024-pixel images.  Each census checks every kernel call of one forward against float64 within its
bound of tests/bounds.py and tests/bounds_resample.py (CheckedOps of tests/test_op_census_gpu.py, no CUDA graphs), with
the GEMM, softmax and attention checks evaluated in row chunks so that their float64 intermediates stay near
CHUNK_BYTES; each census prints its peak device memory.  The kernel tests run the same bounds, or exact constructions,
at the new edges."""
import json
import os

import pytest
import torch

import bounds
from test_bounds_norm_cpu import exact_conv_out_inputs, gn_input
from test_kernel_stress_gpu import ATTN_KERNELS, attention_inputs, onehot_attention, run_attention
from test_norm_edge_kernels_gpu import exact_conv_in_inputs
from test_op_census_gpu import CheckedOps, _summary
from test_resolution_gpu import SCHEDULES, schedule

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
BF = torch.bfloat16
CHUNK_BYTES = 2 ** 28                 # one float64 intermediate of a chunked check: 256 MiB


@pytest.fixture(scope="module")
def ops():
    from gligen_b200.ops import CudaOps
    return CudaOps(DEV)


def gen(seed):
    return torch.Generator(device="cpu").manual_seed(seed)


def _census(ops, title, forward):
    """Run forward(CheckedOps) and check every call; print the peak device memory of the forward and its checks."""
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    torch.cuda.reset_peak_memory_stats(DEV)
    checked = CheckedOps(ops, max_elems=CHUNK_BYTES)
    forward(checked)
    torch.cuda.synchronize()
    print(f"census {title}: peak memory {torch.cuda.max_memory_allocated(DEV) / 2 ** 30:.1f} GiB")
    _summary(title, checked)


# ---- censuses of whole forwards ----------------------------------------------------------------------------------------
def _unet_cfg_forward(name, B, latent=None):
    """One CFG forward (2B UNet rows) of a seeded SD-1.4-sized model, at its native latent or at latent (H, W)."""
    from gligen_b200 import synth
    from gligen_b200.engine import Engine
    from gligen_b200.spec import NAMED_CONFIGS, SPATIAL_MAP_KEY, synthetic_state_dict
    cfg = NAMED_CONFIGS[name]

    def forward(checked):
        eng = Engine(cfg, checked, use_graphs=False)
        eng.load_state_dict(synthetic_state_dict(cfg, 0))
        inp = synth.make_inputs(cfg, B, seed=2)
        x = inp["x"] if latent is None else torch.randn(B, cfg.in_channels, *latent, generator=gen(sum(latent)))
        gr = {k: v.to(DEV) for k, v in inp["grounding_input"].items()}
        gextra = inp["batch"][SPATIAL_MAP_KEY[cfg.tokenizer]].to(DEV) if cfg.spatial else None
        ts = torch.tensor([981, 501][:B], device=DEV)
        e_c, e_u = eng.forward_cfg(x.to(DEV), ts, inp["context"].to(DEV), inp["uc"].to(DEV), gr, None, gextra)
        torch.cuda.synchronize()
        assert e_c.shape == e_u.shape == (B, cfg.out_channels) + tuple(x.shape[2:])
        assert torch.isfinite(e_c).all() and torch.isfinite(e_u).all()
    return forward


@pytest.mark.parametrize("H,W", [(96, 96), (128, 128), (48, 128)], ids=["768x768", "1024x1024", "384x1024"])
def test_census_sd14_box_text_large(ops, H, W):
    """The box+text model at 768^2, 1024^2 and 384 x 1024 (bottom level 6 x 16), CFG at B = 1."""
    _census(ops, f"sd14_box_text cfg B=1 {H}x{W}", _unet_cfg_forward("sd14_box_text", 1, (H, W)))


@pytest.mark.parametrize("name,B", [("sd14_box_text_image", 2), ("sd14_hed", 1), ("sd14_sem", 1)])
def test_census_sd14_native(ops, name, B):
    """box+text+image (two grounding streams of 30 tokens: the fuser attends over T + 60 keys) and the SD-sized spatial
    models (grounding downsampler, ConvNeXt tokenizer, first-conv extra channels) at their native size."""
    _census(ops, f"{name} cfg B={B}", _unet_cfg_forward(name, B))


@pytest.mark.parametrize("h", [96, 128])
def test_census_vae_decode_large(ops, h):
    """sd14_vae decode of an h x h latent: the mid attention's T x T scores (T = 9216, 16384), softmax over T columns,
    the P.V GEMM with K = T, and the last levels at 768^2 / 1024^2."""
    from gligen_b200.spec import NAMED_VAE_CONFIGS, synthetic_vae_state_dict
    from gligen_b200.vae import VAEDecoderEngine
    cfg = NAMED_VAE_CONFIGS["sd14_vae"]

    def forward(checked):
        dec = VAEDecoderEngine(cfg, checked)
        dec.load_state_dict(synthetic_vae_state_dict(cfg, 0))
        img = dec.decode(torch.randn(1, 4, h, h, generator=gen(h)).to(DEV))
        assert img.shape == (1, 3, 8 * h, 8 * h) and torch.isfinite(img).all()
    _census(ops, f"sd14_vae decode {h}x{h}", forward)


@pytest.mark.parametrize("px", [768, 1024])
def test_census_vae_encode_large(ops, px):
    from gligen_b200.spec import NAMED_VAE_CONFIGS, synthetic_vae_encoder_state_dict
    from gligen_b200.vae import VAEEncoderEngine
    cfg = NAMED_VAE_CONFIGS["sd14_vae"]

    def forward(checked):
        enc = VAEEncoderEngine(cfg, checked)
        enc.load_state_dict(synthetic_vae_encoder_state_dict(cfg, 1))
        mom = enc.encode_moments(torch.rand(1, 3, px, px, generator=gen(px)).to(DEV) * 2 - 1)
        assert mom.shape == (1, 8, px // 8, px // 8) and torch.isfinite(mom).all()
    _census(ops, f"sd14_vae encode {px}x{px}", forward)


def test_census_clip_vision(ops):
    """The CLIP ViT-L/14 image tower at B = 2: 257 tokens (a ragged last query tile), quick-GELU epilogues, the patch
    GEMM, the embed and head LayerNorms."""
    from gligen_b200.clip_vision import NAMED_CLIP_VISION_CONFIGS, ClipVisionEngine, synthetic_clip_vision_state_dict, synthetic_pixel_values
    cfg = NAMED_CLIP_VISION_CONFIGS["sd14_clip_vision"]

    def forward(checked):
        eng = ClipVisionEngine(cfg, checked)
        eng.load_state_dict(synthetic_clip_vision_state_dict(cfg, 0))
        hidden, pooled, emb = eng.forward(synthetic_pixel_values(2, seed=3).to(DEV))
        assert hidden.shape == (2, cfg.tokens, cfg.width) and torch.isfinite(emb).all()
    _census(ops, "sd14_clip_vision B=2", forward)


# ---- softmax_rows over T columns ---------------------------------------------------------------------------------------
SOFTMAX_COLS = [4100, 6144, 8192, 9216, 16384]


@pytest.mark.parametrize("cols", SOFTMAX_COLS)
def test_softmax_rows_long(ops, cols):
    """Rows of std 1 / 8 / 30 and rows whose max sits in the last 4-column group, within the float64 bound; rows with
    one entry ahead by 3000 (every other exp2 underflows to 0) are one-hot, exactly."""
    R, scale = 48, 0.0625
    g = gen(cols)
    s = torch.randn(R, cols, generator=g) * torch.tensor([1.0, 8.0, 30.0]).repeat(R // 3)[:, None]
    for r in range(0, 12):                                    # the max in the last group, at each of its 4 lanes
        s[r, cols - 1 - r % 4] = s[r].max() + 2.0 + r
    hot = [0, 4095, 4096, cols // 2, cols - 4, cols - 1] * 2
    for r, j in zip(range(24, 36), hot):
        s[r, j] = s[r].max() + 3000.0
    sd = s.to(DEV)
    p = torch.full((R, cols), float("nan"), device=DEV, dtype=BF)
    ops.softmax_rows(sd, p, scale)
    torch.cuda.synchronize()
    rep = bounds.softmax_check(p, sd, scale, what=f"softmax_rows cols={cols}", max_elems=CHUNK_BYTES)
    print(rep)
    assert rep.ok, str(rep)
    want = torch.zeros(12, cols, dtype=BF)
    want[torch.arange(12), torch.tensor(hot)] = 1.0
    assert torch.equal(p[24:36].cpu(), want), "dominant-entry rows are not one-hot"


# ---- attention at T = 9216 / 16384 tokens ------------------------------------------------------------------------------
BOUNDED_KERNELS = ["auto", "mma_sync", "wgmma_fma2"]
LARGE_ATTN = [  # B, heads, d, Lq, Lk
    (1, 8, 40, 9216, 9216), (1, 8, 40, 16384, 16384),          # level-0 self-attention at 768^2 / 1024^2
    (1, 8, 80, 4096, 4096),                                     # level 1 at 1024^2
    (1, 8, 40, 9216, 9216 + 30), (1, 8, 40, 16384, 16384 + 30),  # the fuser: T visual + 30 grounding keys
]


@pytest.mark.parametrize("kind", ["std4", "argmax_last"])
@pytest.mark.parametrize("B,heads,d,Lq,Lk", LARGE_ATTN, ids=[f"d{d}_{lq}x{lk}" for _, _, d, lq, lk in LARGE_ATTN])
def test_attention_large_bounded(ops, kind, B, heads, d, Lq, Lk):
    q, k, v = attention_inputs(kind, B, heads, d, Lq, Lk, seed=Lk + d)
    bad = []
    for kernel in BOUNDED_KERNELS:
        out = run_attention(ops, q, k, v, heads, d, kernel)
        rep = bounds.attention_check(out, q, k, v, heads, d, poly=ATTN_KERNELS[kernel][1], max_elems=CHUNK_BYTES,
                                     what=f"attention {kind} d={d} {Lq}x{Lk} {kernel}")
        print(rep)
        if not rep.ok:
            bad.append(str(rep))
    assert not bad, "\n".join(bad)


@pytest.mark.parametrize("Lq,Lk", [(16384, 16384), (16384, 16384 + 30)])
def test_attention_large_dominant_key_exact(ops, Lq, Lk):
    """One key per query row ahead by >= 30 scaled logits: every kernel returns that key's V row bit for bit, including
    keys in the ragged last tile."""
    q, k, v, want = onehot_attention(1, 8, 40, Lq, Lk, False, seed=Lk)
    for kernel in (n for n in ATTN_KERNELS if n != "short_key"):
        out = run_attention(ops, q, k, v, 8, 40, kernel)
        bad = (out != want).any(-1)
        assert not bad.any(), f"{kernel} {Lq}x{Lk}: rows {bad.nonzero()[:8].tolist()} differ from V[pi(i)]"


# ---- GroupNorm over 2^18 .. 2^20 rows ----------------------------------------------------------------------------------
GN_LARGE = [(B, HW, C) for HW, C in ((768 * 768, 128), (1024 * 1024, 128), (512 * 512, 256)) for B in (1, 2)]

_GN_PROFILE = r"""
import json, os, sys
sys.path[:0] = [{root!r}, {tests!r}]
import torch
from torch.profiler import ProfilerActivity, profile
from gligen_b200.ops import CudaOps, gn_scratch_floats
from test_bounds_norm_cpu import gn_input
ops = CudaOps("cuda:0")
calls = []
for B, HW, C in {shapes!r}:
    x = gn_input(B, HW, C, 32, HW + C + B, ratio=30.0).cuda()
    gamma, beta = torch.ones(C, device="cuda:0"), torch.zeros(C, device="cuda:0")
    y = torch.zeros(B, HW, C, device="cuda:0", dtype=torch.bfloat16)
    calls.append((x, y, gamma, beta, torch.zeros(gn_scratch_floats(B), device="cuda:0")))
torch.cuda.synchronize()
with profile(activities=[ProfilerActivity.CUDA]) as prof:
    for x, y, gamma, beta, stats in calls:
        ops.groupnorm(x, y, gamma, beta, stats, 32, 1e-6, True)
    torch.cuda.synchronize()
prof.export_chrome_trace({trace!r})
with open({trace!r}) as f:
    ev = [e for e in json.load(f)["traceEvents"] if str(e.get("cat", "")).lower() == "kernel"]
print("GN_KERNELS " + json.dumps([[e["name"], e.get("args", {{}}).get("grid")] for e in sorted(ev, key=lambda e: e["ts"])]))
"""


@pytest.fixture(scope="module")
def gn_launches(tmp_path_factory):
    """(kernel name, grid) of each GN_LARGE shape's glg_groupnorm call, in order, from one profiled region of a short child
    process.  Profiling there keeps the profiler's state out of this test session: in-process sessions followed by
    trace exports have left every later profiled region of the session without kernel records."""
    import subprocess
    import sys
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    trace = str(tmp_path_factory.mktemp("gn_profile") / "trace.json")
    code = _GN_PROFILE.format(root=root, tests=os.path.join(root, "tests"), shapes=GN_LARGE, trace=trace)
    r = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, timeout=600)
    line = next((ln for ln in r.stdout.splitlines() if ln.startswith("GN_KERNELS ")), None)
    assert r.returncode == 0 and line, r.stdout[-2000:] + r.stderr[-4000:]
    launches = json.loads(line[len("GN_KERNELS "):])
    assert len(launches) == len(GN_LARGE), launches
    return dict(zip(GN_LARGE, launches))


@pytest.mark.parametrize("B,HW,C", GN_LARGE)
def test_groupnorm_large(ops, gn_launches, B, HW, C):
    """The VAE's GroupNorms at 768^2 / 1024^2 (and 512^2 x 256 channels): every (sample, group) with its own mean and
    std, against float64 per group.  The fused cross-CTA kernel runs (profiler), and its chunk count is printed."""
    from gligen_b200.ops import gn_scratch_floats
    G = 32
    name, grid = gn_launches[(B, HW, C)]
    assert "gn_fused_kernel" in name, name
    assert bounds.gn_dispatch(B, HW, C, G) == "fused"
    chunks = None if grid is None else grid[0]
    print(f"groupnorm B={B} HW={HW} C={C}: gn_fused_kernel grid {grid}, chunks {chunks}")
    if chunks is not None:
        assert grid[1] == B
        rpi = bounds.gn_fused_geometry(B, HW, C, G)[0]
        assert 1 <= chunks <= -(-HW // (4 * rpi))
    x = gn_input(B, HW, C, G, HW + C + B, ratio=30.0).to(DEV)
    g = gen(C + B)
    gamma, beta = (1 + 0.3 * torch.randn(C, generator=g)).to(DEV), (0.2 * torch.randn(C, generator=g)).to(DEV)
    y = torch.zeros(B, HW, C, device=DEV, dtype=BF)
    stats = torch.zeros(gn_scratch_floats(B), device=DEV)
    ops.groupnorm(x, y, gamma, beta, stats, G, 1e-6, True)
    torch.cuda.synchronize()
    sms = torch.cuda.get_device_properties(DEV).multi_processor_count
    torch.cuda.reset_peak_memory_stats(DEV)
    rep = bounds.groupnorm_check(y, x, gamma, beta, G, 1e-6, True, "fused", num_sms=sms,
                                 what=f"groupnorm B={B} HW={HW} C={C}")
    print(f"{rep}; peak memory {torch.cuda.max_memory_allocated(DEV) / 2 ** 30:.1f} GiB")
    assert rep.ok, str(rep)
    assert int(stats[:128].view(torch.int32).abs().sum()) == 0, "barrier counters not re-armed"


# ---- conv3x3 at widths up to 1024 --------------------------------------------------------------------------------------
CONV_LARGE = [  # B, H, W, C: a few rows at the VAE's last-level widths, widths that are not multiples of 128
    (1, 3, 384, 256), (2, 3, 768, 128), (1, 4, 1024, 128), (2, 3, 1000, 128), (1, 5, 1000, 256), (1, 3, 1016, 128),
]


@pytest.mark.parametrize("B,H,W,C", CONV_LARGE, ids=[f"B{b}_{h}x{w}_C{c}" for b, h, w, c in CONV_LARGE])
def test_conv3x3_wide_rows(ops, B, H, W, C):
    g = gen(B * 1000 + H * 10 + W + C)
    a = torch.randn(B, H * W, C, generator=g).to(DEV, BF)
    w = (torch.randn(9 * C, C, generator=g) * (9 * C) ** -0.5).to(DEV, BF)
    bias = torch.randn(C, generator=g).to(DEV)
    res = torch.randn(B, H * W, C, generator=g).to(DEV, BF)
    bad = []
    for name, (bn, pp, cta2, splitk) in SCHEDULES.items():
        if bn and C % bn:
            continue
        out = torch.zeros(B, H * W, C, device=DEV, dtype=BF)
        with schedule(ops, bn, pp, cta2, splitk):
            ops.gemm(a, w, out, bias=bias, residual=res, conv=(B, H, W))
            torch.cuda.synchronize()
        rep = bounds.gemm_check(out, a, w, bias=bias, residual=res, conv=(B, H, W), splits=8, max_elems=CHUNK_BYTES,
                                what=f"conv B{B} {H}x{W} C{C} {name}")
        if not rep.ok:
            bad.append(str(rep))
    assert not bad, "\n".join(bad)


def test_conv3x3_full_768_image(ops):
    """One whole 768 x 768 x 128 image (589824 output pixels, 4608 M tiles) under the default schedule."""
    H = W = 768
    C = 128
    g = gen(768)
    a = torch.randn(1, H * W, C, generator=g).to(DEV, BF)
    w = (torch.randn(9 * C, C, generator=g) * (9 * C) ** -0.5).to(DEV, BF)
    bias = torch.randn(C, generator=g).to(DEV)
    out = torch.zeros(1, H * W, C, device=DEV, dtype=BF)
    ops.gemm(a, w, out, bias=bias, conv=(1, H, W))
    torch.cuda.synchronize()
    rep = bounds.gemm_check(out, a, w, bias=bias, conv=(1, H, W), splits=8, max_elems=CHUNK_BYTES, what="conv 768x768 C128")
    print(rep)
    assert rep.ok, str(rep)


# ---- data movement and the edge convolutions of 1024-pixel images ------------------------------------------------------
@pytest.mark.parametrize("C", [128, 256])
def test_upsample2x_512_to_1024_exact(ops, C):
    from ref_ops import RefOps
    H = W = 512
    x = torch.randn(1, H * W, C, generator=gen(C)).to(DEV, BF)
    y = torch.full((1, 4 * H * W, C), float("nan"), device=DEV, dtype=BF)
    want = torch.empty_like(y)
    ops.upsample2x(x, y, H, W)
    RefOps(DEV).upsample2x(x, want, H, W)
    torch.cuda.synchronize()
    assert torch.equal(y, want)


@pytest.mark.parametrize("C", [128, 256])
@pytest.mark.parametrize("pad_lo", [0, 1])
def test_im2col_s2_1024_to_512_exact(ops, C, pad_lo):
    """The stride-2 gather of a 1024^2 image: pad_lo 0 (the VAE encoder's right / bottom padding) and 1 (the UNet's)."""
    from ref_ops import RefOps
    H = W = 1024
    x = torch.randn(1, H * W, C, generator=gen(C + pad_lo)).to(DEV, BF)
    col = torch.full(((H // 2) * (W // 2), 9 * C), float("nan"), device=DEV, dtype=BF)
    want = torch.empty_like(col)
    ops.im2col_s2(x, col, H, W, pad_lo=pad_lo)
    RefOps(DEV).im2col_s2(x, want, H, W, pad_lo=pad_lo)
    torch.cuda.synchronize()
    assert torch.equal(col, want)


def test_conv_in_1024_exact(ops):
    """The VAE encoder's first convolution (3 -> 128 channels) of a 1024^2 image, on inputs whose every partial sum is
    representable in fp32: the exact sum rounded once to bf16."""
    B, C0, H, W, Cout = 1, 3, 1024, 1024, 128
    x, _, w, bias = exact_conv_in_inputs(B, C0, 0, H, W, Cout, 1024)
    x, w, bias = x.to(DEV), w.to(DEV), bias.to(DEV)
    exact = torch.nn.functional.conv2d(x.double(), w.double().view(3, 3, C0, Cout).permute(3, 2, 0, 1), bias.double(), padding=1)
    want = exact.permute(0, 2, 3, 1).reshape(B, H * W, Cout).to(BF)
    out = torch.full((B, H * W, Cout), float("nan"), device=DEV, dtype=BF)
    ops.conv_in(x, None, w, bias, out)
    torch.cuda.synchronize()
    assert torch.equal(out, want), f"{(out.double() != want.double()).sum().item()} elements differ"


def test_conv_out_1024_exact(ops):
    """The VAE decoder's last convolution (128 -> 3 channels) to a 1024^2 image, exactly."""
    B, H, W, Cin, Cout = 1, 1024, 1024, 128, 3
    x, w, bias = exact_conv_out_inputs(B, H, W, Cin, Cout, 1025)
    x, w, bias = x.to(DEV), w.to(DEV), bias.to(DEV)
    exact = torch.nn.functional.conv2d(x.double().reshape(B, H, W, Cin).permute(0, 3, 1, 2),
                                       w.double().view(3, 3, Cout, Cin).permute(2, 3, 0, 1), bias.double(), padding=1)
    out = torch.full((B, Cout, H, W), float("nan"), device=DEV)
    ops.conv_out(x, w, bias, out, H, W)
    torch.cuda.synchronize()
    assert torch.equal(out.double(), exact), f"max |diff| {(out.double() - exact).abs().max().item()}"
