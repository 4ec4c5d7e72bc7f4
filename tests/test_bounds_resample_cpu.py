"""CPU: the resampling bounds of tests/bounds_resample.py (resize_plane nearest / bicubic, conv2d_small) against restatements of
csrc/frontend.cu in fp32, in the kernels' own order (the bicubic coordinate as the one FMA nvcc makes of it, the FMA
chains over the taps, the weight layout [(ci, ky, kx)][Cout]).  Every faithful restatement must pass its bound, and every
mutant - one plausible slip in the kernel - must fail it.  Shapes are non-square wherever that can matter: a kernel that
swapped the two axes' scales or strides passes every square test."""
from types import SimpleNamespace

import numpy as np
import pytest
import torch

import bounds_resample

f32 = np.float32


def _fma(a, b, c):
    """fp32 fma(a, b, c): the product of two fp32 values is exact in fp64, so one rounding of the fp64 sum (exact here)."""
    return (np.asarray(a, np.float64) * np.asarray(b, np.float64) + np.asarray(c, np.float64)).astype(f32)


def _src(v, scale, n_in, rnd=np.floor):
    """nearest_src: min(floor(v * scale), in - 1), the product in fp32."""
    return np.minimum(rnd(np.asarray(v).astype(f32) * scale).astype(np.int64), n_in - 1)


def _keys(t, A):
    c1 = lambda a: ((f32(A + 2) * a - f32(A + 3)) * a) * a + f32(1)
    c2 = lambda a: ((f32(A) * a - f32(5 * A)) * a + f32(8 * A)) * a - f32(4 * A)
    return [c2(t + f32(1)), c1(t), c1(f32(1) - t), c2(f32(2) - t)]


OK = SimpleNamespace(swap=False, trunc=False, A=-0.75, align=False, zero_pad=False, clamp_ws=False, round=False,
                     src_bounds=False, w_cout_major=False, silu_first=False, cin_short=False)


def _m(**kw):
    return SimpleNamespace(**{**vars(OK), **kw})


def resize_f32(x, C, Ho, Wo, mode, m=OK):
    """resize_plane_kernel restated: x fp32 [B, Cx, Hs, Ws] -> [B, C, Ho, Wo]."""
    B, Cx, Hs, Ws = x.shape
    sh, sw = f32(Hs) / f32(Ho), f32(Ws) / f32(Wo)
    if m.swap:
        sh, sw = sw, sh
    if mode == "nearest":
        rnd = np.round if m.round else np.floor
        return x[:, :C][:, :, _src(np.arange(Ho), sh, Hs, rnd)][:, :, :, _src(np.arange(Wo), sw, Ws, rnd)]

    def axis(n_in, n_out, s):
        o = np.arange(n_out, dtype=f32)
        if m.align:
            r = o * (f32(n_in - 1) / f32(n_out - 1)) if n_out > 1 else np.zeros(n_out, f32)
        else:
            r = _fma(o + f32(0.5), s, f32(-0.5))
        fl = (np.trunc if m.trunc else np.floor)(r).astype(f32)
        return fl.astype(np.int64), _keys((r - fl).astype(f32), m.A)

    iy, cy = axis(Hs, Ho, sh)
    ix, cx = axis(Ws, Wo, sw)
    flat = np.concatenate([x.reshape(-1), np.full(Ws + 1, 1e3, f32)])     # what a read past the last plane would see
    b_, c_ = np.arange(B)[:, None, None, None], np.arange(C)[None, :, None, None]
    acc = np.zeros((B, C, Ho, Wo), f32)
    for j in range(4):
        yy = iy - 1 + j
        yin = (yy >= 0) & (yy < Hs)
        yy = np.clip(yy, 0, Hs - 1)
        row = np.zeros((B, C, Ho, Wo), f32)
        for k in range(4):
            xx = ix - 1 + k
            xin = (xx >= 0) & (xx < Ws)
            xx = np.clip(xx, 0, Ws if m.clamp_ws else Ws - 1)
            v = flat[(b_ * Cx + c_) * Hs * Ws + yy[None, None, :, None] * Ws + xx[None, None, None, :]]
            if m.zero_pad:
                v = np.where(yin[:, None] & xin[None, :], v, f32(0))
            row = _fma(cx[k][None, None, None, :], v, row)
        acc = _fma(cy[j][None, None, :, None], row, acc)
    return acc


def conv2d_small_f32(x, w, bias, Cout, k, stride, pad, silu, virtual=None, m=OK):
    """conv2d_small_kernel restated: x fp32 [B, Cin, Hs, Ws], w fp32 [Cin * k * k, Cout] -> [B, Cout, Ho, Wo]."""
    B, Cin, Hs, Ws = x.shape
    Hv, Wv = virtual or (Hs, Ws)
    Ho, Wo = (Hv + 2 * pad - k) // stride + 1, (Wv + 2 * pad - k) // stride + 1
    wf = w.reshape(-1)
    acc = np.broadcast_to((np.zeros(Cout, f32) if m.silu_first else bias)[None, :, None, None], (B, Cout, Ho, Wo)).astype(f32)
    lim_h, lim_w = (Hs, Ws) if m.src_bounds else (Hv, Wv)
    for ky in range(k):
        vy = np.arange(Ho) * stride - pad + ky
        yin = (vy >= 0) & (vy < lim_h)
        sy = _src(np.maximum(vy, 0), f32(Hs) / f32(Hv), Hs)
        for kx in range(k):
            vx = np.arange(Wo) * stride - pad + kx
            xin = (vx >= 0) & (vx < lim_w)
            sx = _src(np.maximum(vx, 0), f32(Ws) / f32(Wv), Ws)
            valid = (yin[:, None] & xin[None, :])[None, None]
            v = x[:, :, sy][:, :, :, sx]                              # [B, Cin, Ho, Wo]
            for ci in range(Cin - 1 if m.cin_short else Cin):
                row = ci * k * k + ky * k + kx
                wj = wf[np.arange(Cout) * (Cin * k * k) + row] if m.w_cout_major else wf[row * Cout + np.arange(Cout)]
                acc = np.where(valid, _fma(v[:, ci:ci + 1], wj[None, :, None, None], acc), acc)
    if silu:
        acc = acc / (f32(1) + np.exp(-acc))
    if m.silu_first:
        acc = acc + bias[None, :, None, None]
    return acc.astype(f32)


def _rand(*shape, seed=0):
    return np.random.default_rng(seed + sum(shape)).standard_normal(shape, dtype=f32)


def _resize_report(x, C, Ho, Wo, mode, m=OK):
    got = torch.from_numpy(resize_f32(x, C, Ho, Wo, mode, m))
    return bounds_resample.resize_check(got, torch.from_numpy(x), mode)


def _conv_case(B, Cin, Cout, Hs, Ws, virtual, k, stride, pad, silu, seed=0):
    x = _rand(B, Cin, Hs, Ws, seed=seed)
    w = (_rand(Cin * k * k, Cout, seed=seed + 1) * (Cin * k * k) ** -0.5).astype(f32)
    b = (0.1 * _rand(Cout, seed=seed + 2)).astype(f32)
    return x, w, b


def _conv_report(x, w, b, Cout, k, stride, pad, silu, virtual, m=OK):
    got = torch.from_numpy(conv2d_small_f32(x, w, b, Cout, k, stride, pad, silu, virtual, m))
    return bounds_resample.conv2d_small_check(got, torch.from_numpy(x), torch.from_numpy(w), torch.from_numpy(b), k, stride, pad, silu, virtual)


# (B, Cx, C, Hs, Ws, Ho, Wo): non-square both ways, down / up / one axis each, 1- and 2-pixel sources, 1-pixel outputs,
# outputs that are not powers of two (inexact coordinates), channel subsets of wider maps
RESIZE_SHAPES = [(2, 3, 1, 48, 64, 32, 32), (1, 3, 3, 30, 22, 16, 16), (2, 3, 2, 20, 36, 48, 24), (1, 1, 1, 1, 7, 5, 9),
                 (1, 2, 1, 9, 2, 4, 6), (3, 3, 3, 13, 17, 1, 1), (1, 1, 1, 40, 30, 1, 7), (4, 3, 1, 37, 53, 25, 14),
                 (1, 3, 3, 24, 18, 100, 56), (1, 1, 1, 2, 1, 3, 2)]


@pytest.mark.parametrize("mode", ["nearest", "bicubic"])
@pytest.mark.parametrize("B,Cx,C,Hs,Ws,Ho,Wo", RESIZE_SHAPES)
def test_resize_restatement_within_bound(mode, B, Cx, C, Hs, Ws, Ho, Wo):
    rep = _resize_report(_rand(B, Cx, Hs, Ws), C, Ho, Wo, mode)
    assert rep.ok, str(rep)
    if mode == "nearest":
        assert rep.ratio == 0.0


CONV_SHAPES = [  # (B, Cin, Cout, Hs, Ws, virtual, k, stride, pad, silu): the downsamplers' 4/2/1 and the sem in_conv's 3/1/1
    (2, 1, 4, 21, 34, None, 4, 2, 1, True), (1, 4, 8, 17, 11, None, 4, 2, 1, False), (1, 6, 16, 30, 22, (19, 13), 4, 2, 1, True),
    (1, 5, 3, 14, 22, (29, 17), 3, 1, 1, False), (2, 3, 8, 9, 13, (8, 8), 4, 2, 1, True), (1, 2, 3, 1, 5, (3, 7), 3, 1, 1, True)]


@pytest.mark.parametrize("B,Cin,Cout,Hs,Ws,virtual,k,stride,pad,silu", CONV_SHAPES)
def test_conv2d_small_restatement_within_bound(B, Cin, Cout, Hs, Ws, virtual, k, stride, pad, silu):
    x, w, b = _conv_case(B, Cin, Cout, Hs, Ws, virtual, k, stride, pad, silu)
    rep = _conv_report(x, w, b, Cout, k, stride, pad, silu, virtual)
    assert rep.ok, str(rep)


def test_coordinate_forms_within_one_ulp():
    """The contracted coordinate fl(p - 0.5), p = s (o + 0.5), and torch's fl(fl(p) - 0.5) differ by at most the
    coordinate term's d = ulp(p) + ulp(r), over every output coordinate of every size pair up to 600 x 300 and of the
    phone-sized source 4032 x 3024 onto 1 .. 512 - the coordinate term's premise."""
    pairs = [(i, o) for i in range(1, 601) for o in range(1, 301)] + [(i, o) for i in (4032, 3024) for o in range(1, 513)]
    worst = 0.0
    for n_in, n_out in pairs:
        _, _, _, d = bounds_resample.bicubic_axis(n_in, n_out)
        s = f32(n_in) / f32(n_out)
        o = np.arange(n_out, dtype=f32) + f32(0.5)
        fused = _fma(o, s, f32(-0.5)).astype(np.float64)
        twice = ((o * s).astype(f32) - f32(0.5)).astype(np.float64)
        diff = np.abs(fused - twice)
        dd = d.numpy()
        assert np.all((diff == 0) | (dd > 0)), (n_in, n_out)
        worst = max(worst, float((diff / np.where(dd > 0, dd, 1.0)).max()))
    assert worst <= 1.0, worst


@pytest.mark.parametrize("n_in,n_out", [(512, 256), (256, 128), (256, 64), (512, 64), (128, 128), (64, 256), (3, 12)])
def test_coordinate_term_vanishes_where_exact(n_in, n_out):
    """Power-of-two ratios (every production resize) give fp32-exact coordinates: the coordinate term is zero there."""
    _, _, _, d = bounds_resample.bicubic_axis(n_in, n_out)
    assert float(d.abs().max()) == 0.0


def test_coordinate_term_present_where_inexact():
    _, _, _, d = bounds_resample.bicubic_axis(480, 100)
    assert float(d.max()) > 0.0


# ---- mutants: each one slip of the kernel, at a shape where it changes the result -----------------------------------------
RESIZE_MUTANTS = {
    "nearest, scales swapped": ("nearest", (1, 1, 1, 30, 48, 20, 20), _m(swap=True)),
    "nearest with round": ("nearest", (1, 1, 1, 30, 48, 20, 14), _m(round=True)),
    "bicubic, scales swapped": ("bicubic", (1, 1, 1, 30, 48, 20, 20), _m(swap=True)),
    "trunc for a negative coordinate": ("bicubic", (1, 1, 1, 12, 20, 30, 50), _m(trunc=True)),
    "A = -0.5": ("bicubic", (1, 1, 1, 30, 48, 20, 14), _m(A=-0.5)),
    "align_corners=True coordinate": ("bicubic", (1, 1, 1, 30, 48, 20, 14), _m(align=True)),
    "zero padding instead of clamped taps": ("bicubic", (1, 1, 1, 30, 48, 20, 14), _m(zero_pad=True)),
    "right-border clamp at Ws": ("bicubic", (1, 2, 1, 12, 20, 30, 50), _m(clamp_ws=True)),
}
CONV_CASE = (1, 5, 8, 14, 22, (29, 17), 3, 1, 1, True)
CONV_MUTANTS = {
    "conv2d_small padding on the source grid": (CONV_CASE, _m(src_bounds=True)),
    "conv2d_small weights read [Cout][Cin k k]": (CONV_CASE, _m(w_cout_major=True)),
    "conv2d_small SiLU before the bias": (CONV_CASE, _m(silu_first=True)),
    "conv2d_small Cin loop one short": (CONV_CASE, _m(cin_short=True)),
}


@pytest.mark.parametrize("name", list(RESIZE_MUTANTS))
def test_resize_mutant_fails_bound(name):
    mode, (B, Cx, C, Hs, Ws, Ho, Wo), m = RESIZE_MUTANTS[name]
    x = _rand(B, Cx, Hs, Ws, seed=7)
    assert _resize_report(x, C, Ho, Wo, mode).ok                  # the same case passes without the slip
    rep = _resize_report(x, C, Ho, Wo, mode, m)
    print(f"mutant '{name}': {rep}")
    assert not rep.ok, f"mutant '{name}' passes its bound: {rep}"


@pytest.mark.parametrize("name", list(CONV_MUTANTS))
def test_conv2d_small_mutant_fails_bound(name):
    (B, Cin, Cout, Hs, Ws, virtual, k, stride, pad, silu), m = CONV_MUTANTS[name]
    x, w, b = _conv_case(B, Cin, Cout, Hs, Ws, virtual, k, stride, pad, silu, seed=7)
    assert _conv_report(x, w, b, Cout, k, stride, pad, silu, virtual).ok
    rep = _conv_report(x, w, b, Cout, k, stride, pad, silu, virtual, m)
    print(f"mutant '{name}': {rep}")
    assert not rep.ok, f"mutant '{name}' passes its bound: {rep}"
