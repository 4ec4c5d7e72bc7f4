"""Rounding-level checks of the resampling kernels of the spatial modalities against a float64 statement of the same
operation, in the notation of tests/bounds.py (u, g(L), h(x), the summation lemma and the activation terms), from which
the shared pieces are imported.  Nothing here is fitted to measured errors.

Resampling of the spatial modalities (frontend.cu: resize_plane_kernel, conv2d_small_kernel, patchify_nchw_kernel)
---------------------------------------------------------------------------------------------------------------
Nearest (resize_plane mode 0, and the virtual grids of conv2d_small and patchify_nchw): the source index is
min(floor(dst * fp32(in / out)), in - 1) with the product rounded to fp32, F.interpolate's rule
(tests/test_resize_formula_cpu.py pins it against torch).  The gather moves values: resize_plane nearest is bit-exact,
and patchify_nchw is the gather plus one round-to-nearest-even to bf16 with the columns [k^2 C, ldo) zero, so it is
bit-exact too.

Bicubic (resize_plane mode 1; align_corners = False, Keys kernel W with A = -0.75, taps clamped to the border).  The
reference is the float64 sum_jk W(ty + 1 - j) W(tx + 1 - k) x[clamp(iy - 1 + j), clamp(ix - 1 + k)] with the integer index
and the fraction taken from the kernel's fp32 coordinate r = fl(s (o + 0.5) - 0.5), s = fp32(in / out): nvcc contracts
that statement into one FMA, so r is the exact real rounded once; t = r - floor(r) is then exact (Sterbenz).
  * Coefficients.  The kernel forms the arguments t + 1, 1 - t, 2 - t in fp32 (u |arg| each) and evaluates the cubic
    pieces by Horner: ((1.25 a - 2.25) a) a + 1 (5 roundings) and ((-0.75 a + 3.75) a - 6) a + 3 (6 roundings), any of
    them fused.  Horner's bound with <= 6 roundings is g(6) p~(a), p~ the polynomial with |coefficients|
    (1.25 a^3 + 2.25 a^2 + 1 and 0.75 a^3 + 3.75 a^2 + 6 a + 3); the argument's rounding moves the value by at most the
    piece's slope on its interval (1.35 on [0, 1], 0.75 on [1, 2]) times u |a|.  So |c~ - c| <= dc per tap.
  * Rows, then columns: r_j = fma chain over the 4 taps from 0 (each product through <= 4 roundings),
    |r~_j - r_j| <= sum_k dc_k |x_jk| + g(4) sum_k (|c_k| + dc_k) |x_jk| = er_j, |r~_j| <= (1 + g(4)) sum_k (|c_k| + dc_k) |x_jk|
    = R_j; the output is the same chain over j: sum_j |cy_j| er_j + sum_j dcy_j R_j + g(4) sum_j (|cy_j| + dcy_j) R_j.
  * Coordinate.  Compiled without the contraction, r would be fl(fl(p) - 0.5) with p = s (o + 0.5) (torch's
    statement, two roundings).  Its first rounding costs ulp(p) / 2, its second at most ulp(r) (the difference lands
    in r's binade or the one above), the FMA ulp(r) / 2, so the two forms differ by at most d = ulp(p) + ulp(r)
    (tests/test_bounds_resample_cpu.py checks this over every coordinate of many size pairs; near r = 0 the ulp(p)
    part dominates, so one ulp(r) alone would not do).  The interpolant sum_m W(r - m) x[clamp(m)] is Lipschitz in r
    with constant max|W'| = 1.35 (at |s| = 0.6; 0.75 on the outer piece) per tap, and a tap entering or leaving at an
    integer crossing carries W(2 - e) = A e^2 (1 - e), so a move of d in r changes the output by at most
    1.35 d sum|x| over the 16 taps + 0.75 d^2 max|x|.  Where p and p - 0.5 are both fp32 numbers the coordinate is
    exact, both forms return it, and d = 0: so at every power-of-two output size (s (2o + 1) / 2 has at most the bits of
    (2o + 1) in) the term vanishes.
conv2d_small: fp32 FMA chain from the bias over the output pixel's in-bounds taps of the virtual (nearest-resampled)
grid times Cin, n terms: g(n) (|b| + sum |w| |x|); with SiLU, the activation terms above (silu_f: __expf, __fdividef).

A zero bound (an output whose every tap is zero, as on the blank parts of an edge map) admits only an exact zero.
"""
from __future__ import annotations

import math

import torch

from bounds import U, Report, _silu_error, g_n

KEYS_A = -0.75
KEYS_SLOPE = 1.35                       # max |W'| of the Keys kernel at A = -0.75 (|s| = 0.6)


def nearest_index(n_out: int, n_in: int, device="cpu") -> torch.Tensor:
    """F.interpolate(mode="nearest") source indices: min(floor(dst * fp32(in / out)), in - 1), the product in fp32."""
    scale = torch.tensor(float(n_in), dtype=torch.float32) / torch.tensor(float(n_out), dtype=torch.float32)
    s = torch.floor(torch.arange(n_out, dtype=torch.float32, device=device) * scale.to(device)).long()
    return s.clamp_max(n_in - 1)


def _ulp32(r: torch.Tensor) -> torch.Tensor:
    return torch.exp2(torch.floor(torch.log2(r.abs().clamp_min(2.0 ** -126))) - 23)


def bicubic_axis(n_in: int, n_out: int, device="cpu"):
    """One axis of the bicubic resample: (clamped tap indices [n_out, 4], exact Keys weights at the kernel's fp32
    coordinate [n_out, 4], their fp32 evaluation error dc [n_out, 4], the coordinate move d [n_out])."""
    f64 = torch.float64
    s = float(torch.tensor(float(n_in), dtype=torch.float32) / torch.tensor(float(n_out), dtype=torch.float32))
    prod = (torch.arange(n_out, dtype=f64, device=device) + 0.5) * s               # exact in fp64 (<= 38 significant bits)
    exact = prod - 0.5
    r = exact.float().to(f64)                                                       # the FMA: one rounding
    fl = torch.floor(r)
    t = r - fl
    idx = (fl.long()[:, None] - 1 + torch.arange(4, device=device)[None]).clamp(0, n_in - 1)
    A = KEYS_A
    args = torch.stack([t + 1, t, 1 - t, 2 - t], 1)
    outer = torch.tensor([True, False, False, True], device=device)[None]
    w_in = ((A + 2) * args - (A + 3)) * args * args + 1
    w_out = ((A * args - 5 * A) * args + 8 * A) * args - 4 * A
    w = torch.where(outer, w_out, w_in)
    ptil = torch.where(outer, 0.75 * args ** 3 + 3.75 * args ** 2 + 6 * args + 3, 1.25 * args ** 3 + 2.25 * args ** 2 + 1)
    slope = torch.where(outer, torch.full_like(args, 0.75), torch.full_like(args, KEYS_SLOPE))
    dc = g_n(6) * ptil + slope * U * args.abs() * (1 + U)
    d = torch.where((r == exact) & (prod.float().to(f64) == prod), torch.zeros_like(r), _ulp32(prod) + _ulp32(r))
    return idx, w, dc, d


def _exact_check(got, ref, what) -> Report:
    """Bit-exact: ratio 0 when every element matches, inf otherwise (worst = the first mismatch)."""
    g64 = got.to(torch.float64).reshape(ref.shape)
    bad = (g64 != ref) & ~(torch.isnan(g64) & torch.isnan(ref))
    if not bool(bad.any()):
        return Report(what, 0.0)
    i = int(torch.nonzero(bad.reshape(-1))[0])
    idx = [int(v) for v in torch.unravel_index(torch.tensor(i), tuple(ref.shape))]
    return Report(what, math.inf, 0.0, f"({int(bad.sum())} mismatches, first at index {idx}: got {g64.reshape(-1)[i].item():.9g} "
                                       f"ref {ref.reshape(-1)[i].item():.9g})")


def _fp32_check(got, ref, err, what) -> Report:
    """|got - ref| <= err + u (|ref| + err) per element (the fp32 store rounds once); an exact element passes a zero bound."""
    g64 = got.to(torch.float64).reshape(ref.shape)
    diff = (g64 - ref).abs()
    bound = err + U * (ref.abs() + err)
    r = torch.where(diff == 0, torch.zeros_like(diff), diff / bound)
    i = int(torch.argmax(r))
    idx = [int(v) for v in torch.unravel_index(torch.tensor(i), tuple(ref.shape))]
    return Report(what, r.reshape(-1)[i].item(), 0.0,
                  f"(worst at index {idx}: got {g64.reshape(-1)[i].item():.6g} ref {ref.reshape(-1)[i].item():.6g})")


def resize_check(got, x, mode, what="resize_plane") -> Report:
    """glg_resize_plane: x fp32 [B, Cx, Hs, Ws] (channels [0, C) read), got fp32 [B, C, Ho, Wo]; mode "nearest" | "bicubic"."""
    f64 = torch.float64
    B, C, Ho, Wo = got.shape
    Hs, Ws = x.shape[2:]
    dev = got.device
    xv = x[:, :C].to(f64)
    if mode == "nearest":
        ref = xv[:, :, nearest_index(Ho, Hs, dev)][:, :, :, nearest_index(Wo, Ws, dev)]
        return _exact_check(got, ref, what)
    iy, cy, dcy, dy = bicubic_axis(Hs, Ho, dev)
    ix, cx, dcx, dx = bicubic_axis(Ws, Wo, dev)
    g4 = g_n(4)
    ref = torch.empty(B, C, Ho, Wo, dtype=f64, device=dev)
    err = torch.empty_like(ref)
    for b in range(B):                                        # one image at a time keeps the [C, Ho, 4, Wo, 4] gather small
        tap = xv[b][:, iy][:, :, :, ix]                       # [C, Ho, 4, Wo, 4]
        a = tap.abs()
        rows = (tap * cx[None, None, None]).sum(-1)           # [C, Ho, 4, Wo]
        er = (a * dcx[None, None, None]).sum(-1) + g4 * (a * (cx.abs() + dcx)[None, None, None]).sum(-1)
        R = (1 + g4) * (a * (cx.abs() + dcx)[None, None, None]).sum(-1)
        cyv, dcyv = cy[None, :, :, None], dcy[None, :, :, None]
        ref[b] = (rows * cyv).sum(2)
        e = (cyv.abs() * er).sum(2) + (dcyv * R).sum(2) + g4 * ((cyv.abs() + dcyv) * R).sum(2)
        d = dy[None, :, None] + dx[None, None, :]
        xmax = a.amax(dim=(1, 2, 3, 4))[:, None, None]
        err[b] = e + KEYS_SLOPE * d * a.sum((2, 4)) + 0.75 * d * d * xmax
    return _fp32_check(got, ref, err, what)


def conv2d_small_check(got, x, w, bias, k, stride, pad, silu, virtual=None, what="conv2d_small") -> Report:
    """glg_conv2d_small: x fp32 [B, Cin, Hs, Ws] resampled (nearest) onto `virtual` = (Hv, Wv) (None: no resampling),
    w fp32 [Cin * k * k, Cout] ((ci, ky, kx) rows), got fp32 [B, Cout, Ho, Wo]: g(n) (|b| + sum |w| |x|), n = in-bounds taps x Cin."""
    f64 = torch.float64
    F = torch.nn.functional
    B, Cin, Hs, Ws = x.shape
    Cout = got.shape[1]
    Hv, Wv = virtual or (Hs, Ws)
    dev = got.device
    xv = x.to(f64)[:, :, nearest_index(Hv, Hs, dev)][:, :, :, nearest_index(Wv, Ws, dev)]
    wk = w.to(f64).reshape(Cin, k, k, Cout).permute(3, 0, 1, 2)
    b64 = bias.to(f64)
    ref = F.conv2d(xv, wk, b64, stride=stride, padding=pad)
    S = F.conv2d(xv.abs(), wk.abs(), b64.abs(), stride=stride, padding=pad)
    n = Cin * F.conv2d(torch.ones(1, 1, Hv, Wv, dtype=f64, device=dev), torch.ones(1, 1, k, k, dtype=f64, device=dev), stride=stride, padding=pad)
    err = g_n(n) * S
    if silu:
        err, ref = _silu_error(ref, err)
    return _fp32_check(got, ref, err, what)
