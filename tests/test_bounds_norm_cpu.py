"""The GroupNorm, LayerNorm, softmax_rows, edge-convolution, embedding and sampler bounds of tests/bounds.py have teeth: on the CPU, a torch
restatement of each kernel's arithmetic (op for op in fp32, in the kernel's summation order) passes its bound, and each
realistic mutant of that arithmetic fails it.

gn_reg_restated: gn_reg_kernel (norm.cu) - 256 threads, 4-element units idx = thread + 256 i, pivot x[row 0, first
channel], warp_sum butterflies, the 8 warp partials in order, t = fmaf((v - mean) rstd, gamma, beta).
gn_fused_restated: gn_fused_kernel - per-channel row-0 pivots, rpi row lanes per channel vector, the exact-algebra move
onto the group's first channel, per-CTA partials, the fixed-order reduce over chunks, t = fmaf(v, gamma rstd, beta -
mean gamma rstd).  ln_restated: ln_kernel / layernorm_rows_kernel.  softmax_restated: softmax_rows_kernel.
conv_out_restated, dwconv7_ln_restated, timestep_restated, sampler_restated: the kernels of the same names; the
clip_vision_embed restatement is its fp32 add followed by ln_restated."""
import math

import pytest
import torch

import bounds
from test_bounds_cpu import _fma32

F32, F64, BF = torch.float32, torch.float64, torch.bfloat16


def _warp_sum(v):
    """warp_sum (common.cuh) over the last dim of 32 lanes: xor butterfly 16, 8, 4, 2, 1; lane 0's value."""
    lane = torch.arange(32)
    for o in (16, 8, 4, 2, 1):
        v = v + v[..., lane ^ o]
    return v[..., 0]


def _rsqrt32(v):
    return torch.rsqrt(v.to(F64)).to(F32)


def _silu32(t):
    return t / (1 + torch.exp(-t))


# ---------------------------------------------------------------------------------------------------------------------
def gn_reg_restated(x, gamma, beta, G, eps, silu, mutant=None):
    B, HW, C = x.shape
    cpg = C // G
    N = HW * cpg
    xs = x.float().view(B, HW, G, cpg).permute(0, 2, 1, 3)                     # [B, G, HW, cpg]
    P = xs[:, :, 0, 0] if mutant != "raw" else torch.zeros(B, G)
    d = (xs - P[:, :, None, None]).reshape(B, G, -1, 4)
    n = -(-d.shape[2] // 256)
    d = torch.nn.functional.pad(d, (0, 0, 0, n * 256 - d.shape[2])).view(B, G, n, 256, 4)
    s = torch.zeros(B, G, 256)
    ss = torch.zeros(B, G, 256)
    for i in range(n):
        u = d[:, :, i]
        s = s + ((u[..., 0] + u[..., 1]) + (u[..., 2] + u[..., 3]))
        ss = _fma32(u[..., 0], u[..., 0], _fma32(u[..., 1], u[..., 1], _fma32(u[..., 2], u[..., 2], _fma32(u[..., 3], u[..., 3], ss))))
    ws, wss = _warp_sum(s.view(B, G, 8, 32)), _warp_sum(ss.view(B, G, 8, 32))
    ts, tss = torch.zeros(B, G), torch.zeros(B, G)
    for w in range(8):
        ts, tss = ts + ws[..., w], tss + wss[..., w]
    inv_n = torch.tensor(1.0 / N, dtype=F32)
    m1 = ts * inv_n
    var = (tss * inv_n - m1 * m1).clamp_min(0)
    if mutant == "unbiased":
        var = var * torch.tensor(N / (N - 1), dtype=F32)
    mean = P + m1
    rstd = _rsqrt32(var + (0.0 if mutant == "no_eps" else eps))
    ch = torch.arange(C)
    gi = ((ch + 1) // cpg).clamp_max(G - 1) if mutant == "group_shift" else ch // cpg
    v = x.float()
    z = (v - mean[:, None, gi]) * rstd[:, None, gi]
    if mutant == "silu_first":
        z = _silu32(z)
    t = _fma32(z, gamma[None, None].expand_as(z), beta[None, None].expand_as(z))
    if silu and mutant != "silu_first":
        t = _silu32(t)
    return t.to(BF)


def gn_fused_partials(x, G, rpi, chunks):
    """Steps 1-2 of gn_fused_kernel: per-CTA partials [B, chunks, G, 2] (fp32) and the per-channel pivots."""
    B, HW, C = x.shape
    cpg = C // G
    rpc = -(-HW // chunks)
    v = x.float()
    piv = v[:, 0]                                                              # [B, C]
    part = torch.zeros(B, chunks, G, 2)
    for k in range(chunks):
        r0, r1 = k * rpc, min(HW, (k + 1) * rpc)
        d = v[:, r0:r1] - piv[:, None]
        n_r = -(-(r1 - r0) // rpi)
        d = torch.nn.functional.pad(d, (0, 0, 0, n_r * rpi - (r1 - r0))).view(B, n_r, rpi, C)
        a, q = torch.zeros(B, rpi, C), torch.zeros(B, rpi, C)
        for i in range(n_r):
            a = a + d[:, i]
            q = _fma32(d[:, i], d[:, i], q)
        s1, s2 = torch.zeros(B, C), torch.zeros(B, C)
        for lane in range(rpi):
            s1, s2 = s1 + a[:, lane], s2 + q[:, lane]
        rows = torch.tensor(float(r1 - r0))
        s, ss = torch.zeros(B, G), torch.zeros(B, G)
        pv = piv.view(B, G, cpg)
        s1g, s2g = s1.view(B, G, cpg), s2.view(B, G, cpg)
        for c in range(cpg):
            dc = pv[..., c] - pv[..., 0]
            s = s + _fma32(rows.expand_as(dc), dc, s1g[..., c])
            ss = ss + _fma32(dc, _fma32(rows.expand_as(dc), dc, 2 * s1g[..., c]), s2g[..., c])
        part[:, k, :, 0], part[:, k, :, 1] = s, ss
    return part, piv


def gn_fused_restated(x, gamma, beta, G, eps, silu, rpi, chunks, mutant=None, prev=None):
    B, HW, C = x.shape
    cpg = C // G
    part, piv = gn_fused_partials(x, G, rpi, chunks)
    if mutant == "sample_shift":
        part = part.roll(-1, 0)                                                # sample b reads sample b + 1's partials
    if mutant == "stale":
        part[:, -1] = gn_fused_partials(prev, G, rpi, chunks)[0][:, -1]        # one CTA's partial left from the last call
    if mutant == "drop_ragged":
        part[:, -1] = 0                                                        # the ragged last chunk's rows never summed
    Q = (C // 8) * rpi // G
    ts, tss = torch.zeros(B, G), torch.zeros(B, G)
    for p in range(Q):
        s, ss = torch.zeros(B, G), torch.zeros(B, G)
        for k in range(p, chunks, Q):
            s, ss = s + part[:, k, :, 0], ss + part[:, k, :, 1]
        ts, tss = ts + s, tss + ss
    inv_n = torch.tensor(1.0, dtype=F32) / (torch.tensor(float(HW), dtype=F32) * torch.tensor(float(cpg), dtype=F32))
    m1 = ts * inv_n
    var = (tss * inv_n - m1 * m1).clamp_min(0)
    mean = piv.view(B, G, cpg)[..., 0] + m1
    rstd = _rsqrt32(var + eps)
    gi = torch.arange(C) // cpg
    ga = gamma[None] * rstd[:, gi]                                              # [B, C]
    sb = beta[None] - mean[:, gi] * ga
    v = x.float()
    t = _fma32(v, ga[:, None].expand_as(v), sb[:, None].expand_as(v))
    if silu:
        t = _silu32(t)
    return t.to(BF)


def gn_input(B, HW, C, G, seed, ratio=100.0, outlier=30.0):
    """Each (sample, group) its own std (1e-3 .. 1e3) and mean (|mean| / std up to `ratio`); an outlier of `outlier` std at
    the pivot position (row 0, first channel of the group); group 1 constant; group 2 with variance near 1e-6."""
    g = torch.Generator().manual_seed(seed)
    cpg = C // G
    std = 10.0 ** (6 * torch.rand(B, 1, G, 1, generator=g) - 3)
    mean = std * ratio * (2 * torch.rand(B, 1, G, 1, generator=g) - 1)
    x = (mean + std * torch.randn(B, HW, G, cpg, generator=g))
    x[:, 0, :, 0] += outlier * std[:, 0, :, 0]
    x[:, :, 1] = 0.75
    x[:, :, 2] = 0.01 + 1e-3 * torch.randn(B, HW, cpg, generator=g)
    return x.reshape(B, HW, C).to(BF)


def _affine(C, seed):
    g = torch.Generator().manual_seed(seed)
    return 1 + 0.3 * torch.randn(C, generator=g), 0.2 * torch.randn(C, generator=g)


REG = dict(B=2, HW=64, C=640, G=32)                   # cpg 20: 320 units -> gn_reg<5>


@pytest.mark.parametrize("silu", [False, True])
@pytest.mark.parametrize("outlier", [0.0, 30.0])
def test_gn_reg_faithful_passes(silu, outlier):
    B, HW, C, G = REG.values()
    assert bounds.gn_dispatch(B, HW, C, G) == "reg5"
    x = gn_input(B, HW, C, G, 1, outlier=outlier)
    gamma, beta = _affine(C, 2)
    rep = bounds.groupnorm_check(gn_reg_restated(x, gamma, beta, G, 1e-6, silu), x, gamma, beta, G, 1e-6, silu, "reg5")
    print(rep)
    assert rep.ok, str(rep)


@pytest.mark.parametrize("mutant,HW,ratio,silu", [
    ("group_shift", 64, 100.0, False),                # channel c normalised with group (c + 1) / cpg
    ("raw", 64, 100.0, False),                        # E[x^2] - E[x]^2 with no pivot
    ("unbiased", 4, 3.0, False),                      # N - 1: visible at the smallest groups (N = 80)
    ("no_eps", 64, 3.0, False),                       # group 2 has var ~ eps
    ("silu_first", 64, 3.0, True),
])
def test_gn_reg_mutants_rejected(mutant, HW, ratio, silu):
    B, _, C, G = REG.values()
    x = gn_input(B, HW, C, G, 3, ratio=ratio, outlier=0.0)
    gamma, beta = _affine(C, 4)
    path = bounds.gn_dispatch(B, HW, C, G)
    assert bounds.groupnorm_check(gn_reg_restated(x, gamma, beta, G, 1e-6, silu), x, gamma, beta, G, 1e-6, silu, path).ok
    rep = bounds.groupnorm_check(gn_reg_restated(x, gamma, beta, G, 1e-6, silu, mutant), x, gamma, beta, G, 1e-6, silu, path)
    print(rep)
    assert not rep.ok, str(rep)


FUSED = dict(B=3, HW=1000, C=128, G=32, rpi=16, chunks=6)      # 6 chunks of 167 rows, the last one 165


@pytest.mark.parametrize("outlier", [0.0, 30.0])
def test_gn_fused_faithful_passes(outlier):
    B, HW, C, G, rpi, chunks = FUSED.values()
    x = gn_input(B, HW, C, G, 5, outlier=outlier)
    gamma, beta = _affine(C, 6)
    assert bounds.gn_fused_geometry(B, HW, C, G, chunks=chunks)[0] == rpi
    out = gn_fused_restated(x, gamma, beta, G, 1e-6, True, rpi, chunks)
    rep = bounds.groupnorm_check(out, x, gamma, beta, G, 1e-6, True, "fused", chunks=chunks)
    print(rep)
    assert rep.ok, str(rep)


@pytest.mark.parametrize("mutant", ["sample_shift", "stale", "drop_ragged"])
def test_gn_fused_mutants_rejected(mutant):
    B, HW, C, G, rpi, chunks = FUSED.values()
    prev = gn_input(B, HW, C, G, 7, ratio=3.0, outlier=0.0)
    x = gn_input(B, HW, C, G, 8, ratio=3.0, outlier=0.0)
    gamma, beta = _affine(C, 9)
    good = gn_fused_restated(x, gamma, beta, G, 1e-6, False, rpi, chunks)
    assert bounds.groupnorm_check(good, x, gamma, beta, G, 1e-6, False, "fused", chunks=chunks).ok
    bad = gn_fused_restated(x, gamma, beta, G, 1e-6, False, rpi, chunks, mutant, prev)
    rep = bounds.groupnorm_check(bad, x, gamma, beta, G, 1e-6, False, "fused", chunks=chunks)
    print(rep)
    assert not rep.ok, str(rep)


# ---------------------------------------------------------------------------------------------------------------------
def ln_restated(x, gamma, beta, eps, mutant=None, f32_out=False):
    """ln_kernel / layernorm_rows_kernel: lane l holds the 8-column vectors l + 32 i; two-pass in registers."""
    R, C = x.shape
    nv = C // 8
    n_i = -(-nv // 32)
    v = torch.nn.functional.pad(x.float(), (0, n_i * 256 - C)).view(R, n_i, 32, 8)
    valid = torch.nn.functional.pad(torch.ones(C, dtype=torch.bool), (0, n_i * 256 - C)).view(n_i, 32, 8)
    if mutant == "mean_short":
        valid = valid.clone().view(-1)
        valid[C - 8:] = False
        valid = valid.view(n_i, 32, 8)
    s = torch.zeros(R, 32)
    for i in range(n_i):
        for j in range(8):
            s = torch.where(valid[i, :, j], s + v[:, i, :, j], s)
    cnt = C - 8 if mutant == "mean_short" else C
    mean = _warp_sum(s) / torch.tensor(float(cnt), dtype=F32)
    q = torch.zeros(R, 32)
    full = torch.nn.functional.pad(torch.ones(C, dtype=torch.bool), (0, n_i * 256 - C)).view(n_i, 32, 8)
    for i in range(n_i):
        for j in range(8):
            if mutant == "one_pass":
                q = torch.where(full[i, :, j], _fma32(v[:, i, :, j], v[:, i, :, j], q), q)
            else:
                d = v[:, i, :, j] - mean[:, None]
                q = torch.where(full[i, :, j], _fma32(d, d, q), q)
    var = _warp_sum(q) / torch.tensor(float(C), dtype=F32)
    if mutant == "one_pass":
        var = var - mean * mean
    rstd = _rsqrt32(var + eps)
    z = (x.float() - mean[:, None]) * rstd[:, None]
    if mutant == "round_z":
        z = z.to(BF).float()
    g, b = (gamma.roll(8), beta.roll(8)) if mutant == "affine_shift" else (gamma, beta)
    t = _fma32(z, g[None].expand_as(z), b[None].expand_as(z))
    return t if f32_out else t.to(BF)


def ln_input(R, C, seed, ratio):
    g = torch.Generator().manual_seed(seed)
    std = 10.0 ** (4 * torch.rand(R, 1, generator=g) - 2)
    mean = std * ratio * (2 * torch.rand(R, 1, generator=g) - 1)
    return (mean + std * torch.randn(R, C, generator=g)).to(BF)


@pytest.mark.parametrize("C", [320, 768, 1024, 1288])
@pytest.mark.parametrize("f32_out", [False, True])
def test_ln_faithful_passes(C, f32_out):
    x = ln_input(64, C, 10, 100.0)
    gamma, beta = _affine(C, 11)
    rep = bounds.layernorm_check(ln_restated(x, gamma, beta, 1e-5, f32_out=f32_out), x, gamma, beta, 1e-5)
    print(rep)
    assert rep.ok, str(rep)


@pytest.mark.parametrize("mutant,ratio", [("mean_short", 3.0), ("one_pass", 100.0), ("affine_shift", 3.0), ("round_z", 3.0)])
def test_ln_mutants_rejected(mutant, ratio):
    C = 768
    x = ln_input(64, C, 12, ratio)
    gamma, beta = _affine(C, 13)
    assert bounds.layernorm_check(ln_restated(x, gamma, beta, 1e-5), x, gamma, beta, 1e-5).ok
    rep = bounds.layernorm_check(ln_restated(x, gamma, beta, 1e-5, mutant), x, gamma, beta, 1e-5)
    print(rep)
    assert not rep.ok, str(rep)


# ---------------------------------------------------------------------------------------------------------------------
def softmax_restated(s, scale, mutant=None):
    """softmax_rows_kernel: thread t owns columns 4 t + 1024 k; exp2f(fmaf(v, c, -m c)); warp_sum; 8 warps in order."""
    R, cols = s.shape
    c = torch.tensor(scale, dtype=F32) * torch.tensor(1.4426950408889634, dtype=F32)
    m = (s[:, :4096] if mutant == "stop_4096" else s).amax(1, keepdim=True)
    ms = m * c
    e = torch.exp2(_fma32(s, c.expand_as(s), (-ms).expand_as(s)).to(F64)).to(F32)
    n_k = -(-cols // 1024)
    ep = torch.nn.functional.pad(e, (0, n_k * 1024 - cols)).view(R, n_k, 256, 4)
    acc = torch.zeros(R, 256)
    for k in range(n_k):
        if mutant == "skip_stride" and k == 1 or mutant == "stop_4096" and k >= 4:     # stop_4096: max and sum loops end at 4096
            continue
        u = ep[:, k]
        acc = acc + (((u[..., 0] + u[..., 1]) + u[..., 2]) + u[..., 3])
    ws = _warp_sum(acc.view(R, 8, 32))
    tot = torch.zeros(R)
    for w in range(8):
        tot = tot + ws[:, w]
    inv = torch.tensor(1.0, dtype=F32) / tot
    if mutant == "round_p":
        e = e.to(BF).float()
    return (e * inv[:, None]).to(BF)


@pytest.mark.parametrize("cols", [4, 1020, 1024, 1028, 4096])
@pytest.mark.parametrize("std", [1.0, 30.0])
def test_softmax_faithful_passes(cols, std):
    g = torch.Generator().manual_seed(cols)
    s = torch.randn(16, cols, generator=g) * std
    s[3, cols // 2] = 200.0                                                    # a single dominant column
    rep = bounds.softmax_check(softmax_restated(s, 0.125), s, 0.125)
    print(rep)
    assert rep.ok, str(rep)


@pytest.mark.parametrize("cols", [4100, 9216, 16384])
def test_softmax_faithful_passes_long_rows(cols):
    """The VAE mid attention's rows at 768^2 and 1024^2 images (T = 9216, 16384 columns) and one past a 4-column group
    of 4096; the max in the last 4-column group, and one dominant entry."""
    g = torch.Generator().manual_seed(cols)
    s = torch.randn(6, cols, generator=g) * 4
    s[1, cols - 1] = 60.0
    s[2, cols - 3] = 400.0
    rep = bounds.softmax_check(softmax_restated(s, 0.125), s, 0.125)
    print(rep)
    assert rep.ok, str(rep)


def test_softmax_stop_at_4096_rejected_on_long_rows():
    """A column loop that ends at 4096 (the longest rows tested before) on a 9216-column row: the probabilities of
    every column are normalised by the sum of the first 4096 only."""
    g = torch.Generator().manual_seed(22)
    s = torch.randn(8, 9216, generator=g)
    assert bounds.softmax_check(softmax_restated(s, 0.5), s, 0.5).ok
    rep = bounds.softmax_check(softmax_restated(s, 0.5, "stop_4096"), s, 0.5)
    print(rep)
    assert not rep.ok, str(rep)


@pytest.mark.parametrize("mutant", ["round_p", "skip_stride"])
def test_softmax_mutants_rejected(mutant):
    g = torch.Generator().manual_seed(21)
    s = torch.randn(64, 4096, generator=g)
    rep = bounds.softmax_check(softmax_restated(s, 0.5, mutant), s, 0.5)
    print(rep)
    assert not rep.ok, str(rep)


# ---------------------------------------------------------------------------------------------------------------------
def exact_conv_out_inputs(B, H, W, Cin, Cout, seed):
    """x in {-3 .. 3} (bf16), w = k 2^-10 with |k| <= 1023 (10 significant bits: a bf16 rounding changes most of them),
    bias a multiple of 2^-10: every partial sum is an integer multiple of 2^-10 below 2^14, exact in fp32."""
    g = torch.Generator().manual_seed(seed)
    x = torch.randint(-3, 4, (B, H * W, Cin), generator=g).to(BF)
    w = torch.randint(-1023, 1024, (9, Cout, Cin), generator=g).float() * 2.0 ** -10
    bias = torch.randint(-4096, 4097, (Cout,), generator=g).float() * 2.0 ** -10
    return x, w, bias


def conv_out_exact(x, w, bias, H, W):
    """The exact result (fp64, representable in fp32 for exact_conv_out_inputs)."""
    B, _, Cin = x.shape
    Cout = w.shape[1]
    xi = x.double().reshape(B, H, W, Cin).permute(0, 3, 1, 2)
    wk = w.double().view(3, 3, Cout, Cin).permute(2, 3, 0, 1)
    return torch.nn.functional.conv2d(xi, wk, bias.double(), padding=1)


def conv_out_restated(x, w, bias, H, W):
    """conv_out_kernel / conv_out_px8_kernel: lane l takes channels 8 l + 256 i; per tap and step acc += the 8 products
    summed left to right; warp_sum over the 32 lanes; + bias."""
    B, _, Cin = x.shape
    Cout = w.shape[1]
    n_i = -(-Cin // 256)
    xp = torch.nn.functional.pad(x.float().reshape(B, H, W, Cin), (0, n_i * 256 - Cin, 1, 1, 1, 1))   # zero border, zero channels
    wp = torch.nn.functional.pad(w.float(), (0, n_i * 256 - Cin))
    acc = torch.zeros(B, Cout, H, W, 32)
    for tap in range(9):
        xs = xp[:, tap // 3:tap // 3 + H, tap % 3:tap % 3 + W].reshape(B, H, W, n_i, 32, 8)
        ws = wp[tap].reshape(Cout, n_i, 32, 8)
        for i in range(n_i):
            prod = xs[:, None, :, :, i] * ws[None, :, None, None, i]                    # [B, Cout, H, W, 32, 8]
            t = prod[..., 0]
            for j in range(1, 8):
                t = t + prod[..., j]
            acc = acc + t
    return _warp_sum(acc) + bias.view(1, Cout, 1, 1)


def test_conv_out_exact_inputs_catch_bf16_weights():
    """On exact inputs, the fp32 result in the kernel's summation order equals the exact sum, and passes the bound; a
    kernel that rounded its weights to bf16 fails both the exact check and the bound (depth 8 + 9 ceil(Cin / 256) + 6)."""
    B, H, W, Cin, Cout = 2, 5, 7, 320, 4
    x, w, bias = exact_conv_out_inputs(B, H, W, Cin, Cout, 30)
    exact = conv_out_exact(x, w, bias, H, W)
    assert exact.abs().max() < 2 ** 14 and torch.equal(exact.float().double(), exact)
    faithful = conv_out_restated(x, w, bias, H, W)
    assert torch.equal(faithful.double(), exact)
    assert bounds.conv_check(faithful, x, w, bias, "out", H, W).ok
    mutant = conv_out_restated(x, w.to(BF).float(), bias, H, W)
    assert not torch.equal(mutant.double(), exact)
    assert not bounds.conv_check(mutant, x, w, bias, "out", H, W).ok


def test_conv_out_bound_passes_kernel_order_on_random_inputs():
    B, H, W, Cin, Cout = 1, 6, 8, 512, 4
    g = torch.Generator().manual_seed(31)
    x = torch.randn(B, H * W, Cin, generator=g).to(BF)
    w, bias = 0.05 * torch.randn(9, Cout, Cin, generator=g), torch.randn(Cout, generator=g)
    rep = bounds.conv_check(conv_out_restated(x, w, bias, H, W), x, w, bias, "out", H, W)
    print(rep)
    assert rep.ok, str(rep)


# ---------------------------------------------------------------------------------------------------------------------
def dwconv7_ln_restated(x, w, bias, gamma, beta, B, H, W, C, eps, mutant=None):
    """dwconv7_ln_kernel: acc = bias, then fmaf over taps ky, kx in order (zero taps outside the image are skipped); the
    row LayerNorm of the fp32 acc."""
    xv = torch.nn.functional.pad(x.float().reshape(B, H, W, -1)[..., :C], (0, 0, 3, 3, 3, 3))
    wt = w.view(7, 7, C).transpose(0, 1).reshape(49, C) if mutant == "taps_transposed" else w
    acc = bias.float().expand(B, H, W, C).clone()
    for ky in range(7):
        for kx in range(7):
            acc = _fma32(xv[:, ky:ky + H, kx:kx + W], wt[ky * 7 + kx].expand(B, H, W, C), acc)   # padding adds 0 * w: exact
    return ln_restated(acc.reshape(-1, C), gamma, beta, eps)


@pytest.mark.parametrize("mutant", [None, "taps_transposed"])
def test_dwconv7_ln_bound(mutant):
    B, H, W, C = 1, 9, 8, 96
    g = torch.Generator().manual_seed(40)
    x = (torch.randn(B * H * W, C, generator=g) + 5 * torch.randn(1, C, generator=g)).to(BF)
    w, bias = 0.1 * torch.randn(49, C, generator=g), torch.randn(C, generator=g)
    gamma, beta = _affine(C, 41)
    y = dwconv7_ln_restated(x, w, bias, gamma, beta, B, H, W, C, 1e-6, mutant)
    rep = bounds.dwconv7_ln_check(y, x, w, bias, gamma, beta, B, H, W, C, 1e-6)
    print(rep)
    assert rep.ok == (mutant is None), str(rep)


@pytest.mark.parametrize("mutant", [None, "pos_shift"])
def test_clip_vision_embed_bound(mutant):
    """clip_vision_embed_kernel: the fp32 add patch + pos, then the row LayerNorm; the mutant adds the next token's pos."""
    N, P, C = 2, 16, 256
    g = torch.Generator().manual_seed(42)
    patch = torch.randn(N * P, C, generator=g) * 3 + 50 * torch.randn(N * P, 1, generator=g)
    cls, pos = torch.randn(C, generator=g), torch.randn(P + 1, C, generator=g)
    gamma, beta = _affine(C, 43)
    rows = torch.cat([cls.view(1, 1, C).expand(N, 1, C), patch.view(N, P, C)], 1)
    pp = pos.roll(-1, 0) if mutant == "pos_shift" else pos
    v = (rows + pp[None]).reshape(-1, C)                                       # one fp32 rounding per element
    rep = bounds.clip_vision_embed_check(ln_restated(v, gamma, beta, 1e-5), patch, cls, pos, gamma, beta, P, 1e-5)
    print(rep)
    assert rep.ok == (mutant is None), str(rep)


def timestep_restated(t, dim, mutant=None):
    """timestep_embedding_kernel in fp32: freq = expf(-9.2103404f * k / half), arg = t freq, cos | sin."""
    half = dim // 2
    k = torch.arange(half, dtype=F32)
    den = torch.tensor(float(half - 1 if mutant == "half_minus_1" else half), dtype=F32)
    freq = torch.exp(torch.tensor(-9.210340371976184, dtype=F32) * k / den)
    arg = t.float()[:, None] * freq[None]
    return torch.cat([torch.cos(arg.double()).float(), torch.sin(arg.double()).float()], 1).to(BF)


@pytest.mark.parametrize("mutant", [None, "half_minus_1"])
def test_timestep_embedding_bound(mutant):
    t = torch.tensor([0, 1, 21, 500, 981, 999])
    rep = bounds.timestep_embedding_check(timestep_restated(t, 320, mutant), t)
    print(rep)
    assert rep.ok == (mutant is None), str(rep)


def sampler_restated(x, ec, eu, g, olds, coefs, a_t, a_prev, mutant=None):
    """sampler_update_kernel in fp32, with the host's fp32 scalars."""
    f = lambda v: torch.tensor(v, dtype=F32)
    c = [f(v) for v in coefs]
    s0, s1 = torch.sqrt(f(a_t)), torch.sqrt(1 - f(a_t))
    s2, s3 = torch.sqrt(f(a_prev)), torch.sqrt(1 - f(a_prev))
    e = eu + f(g) * (ec - eu)
    ep = c[0] * e
    ol = list(olds)
    if mutant == "olds_swapped":
        ol[0], ol[1] = ol[1], ol[0]
    for ci, o in zip(c[1:], ol):
        ep = ep + ci * o
    pred = (x - s1 * ep) / s0
    return e, s2 * pred + s3 * ep


@pytest.mark.parametrize("mutant", [None, "olds_swapped"])
def test_sampler_update_bound(mutant):
    g = torch.Generator().manual_seed(44)
    x, ec, eu, o1, o2, o3 = (torch.randn(4, 64, 64, generator=g) * s for s in (30.0, 1, 1, 1, 1, 1))
    coefs = (55 / 24, -59 / 24, 37 / 24, -9 / 24)
    e, xp = sampler_restated(x, ec, eu, 7.5, [o1, o2, o3], coefs, 0.0047, 0.0052, mutant)
    rep = bounds.sampler_update_check(e, xp, x, ec, eu, 7.5, [o1, o2, o3], coefs, 0.0047, 0.0052)
    print(rep)
    assert rep.ok == (mutant is None), str(rep)
