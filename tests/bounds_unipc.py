"""The UniPC update kernel (elementwise.cu: unipc_update_kernel, glg_unipc_update) stated in torch, and its rounding-level check
against float64, in the notation of tests/bounds.py (u, g(L)), from which the shared pieces are imported.  Nothing here is
fitted to measured errors.

The reference is the float64 evaluation of the kernel's formula with the fp32 scalars it receives (guidance, alpha, sigma and
the nine coefficients: the host rounds its float64 values once).  Per element, any order of FMA contraction:
  * e = u + g (e_c - u) and m0 = (x - sigma e) / alpha exactly as for glg_dpm_update (tests/bounds_dpm.py): |de| <= g(3) (|u| +
    |g| |e_c - u|), dn = g(2) (|x| + |sigma e|) + sigma |de|, |dm0| <= dn / alpha + u (|m0| + dn / alpha).
  * xc = cc xc_prev + c0 m0 + c1 m1 + c2 m2 + c3 m3: a chain of <= 5 products, |dxc| <= |c0| dm0 + g(5) (|cc xc_prev| +
    |c0| (|m0| + dm0) + |c1 m1| + |c2 m2| + |c3 m3|) (xc_prev, m1, m2, m3 are inputs, exact).  Without xc_prev xc = x exactly.
  * x_next = pc xc + p0 m0 + p1 m1 + p2 m2 is computed from the fp32 xc the kernel stores, so it is checked against the stored
    xc_out: |dx| <= |p0| dm0 + g(4) (|pc xc_out| + |p0| (|m0| + dm0) + |p1 m1| + |p2 m2|).  That pins the two outputs to each
    other, not only each to float64.
m_out, xc_out and x_next are checked with these bounds (tests/bounds.py _plain_check: elementwise).
"""
from __future__ import annotations

import numpy as np
import torch

from bounds import U, Report, _plain_check, g_n


def _f32(v) -> float:
    return float(np.float32(v))


def unipc_update_ref(x, xc_prev, e_cond, e_uncond, guidance, m1, m2, m3, alpha, sigma, coefs):
    """(m0, xc, x_next) of glg_unipc_update in the dtype of x: fp32 tensors give the kernel's statement with fp32 scalars,
    float64 tensors the float64 solver step.  xc_prev, e_uncond, m1, m2, m3 may be None."""
    cast = _f32 if x.dtype == torch.float32 else float
    g, a, s = cast(guidance), cast(alpha), cast(sigma)
    cc, c0, c1, c2, c3, pc, p0, p1, p2 = (cast(c) for c in coefs)
    e = e_cond if e_uncond is None else e_uncond + g * (e_cond - e_uncond)
    m0 = (x - s * e) / a
    if xc_prev is None:
        xc = x.clone()
    else:
        xc = cc * xc_prev + c0 * m0
        for c, m in ((c1, m1), (c2, m2), (c3, m3)):
            if m is not None:
                xc = xc + c * m
    xn = pc * xc + p0 * m0
    for c, m in ((p1, m1), (p2, m2)):
        if m is not None:
            xn = xn + c * m
    return m0, xc, xn


def unipc_update_bound(xc_out, x, xc_prev, e_cond, e_uncond, guidance, m1, m2, m3, alpha, sigma, coefs):
    """float64 (m0, dm0, xc, dxc, x_next, dx_next): the exact values with the kernel's fp32 scalars and their error bounds;
    x_next from the kernel's stored xc_out."""
    f64 = torch.float64
    g, a, s = _f32(guidance), _f32(alpha), _f32(sigma)
    cc, c0, c1, c2, c3, pc, p0, p1, p2 = (_f32(c) for c in coefs)
    ec = e_cond.to(f64)
    if e_uncond is not None:
        eu = e_uncond.to(f64)
        e = eu + g * (ec - eu)
        de = g_n(3) * (eu.abs() + abs(g) * (ec - eu).abs())
    else:
        e, de = ec, torch.zeros_like(ec)
    xv = x.to(f64)
    m0 = (xv - s * e) / a
    dn = g_n(2) * (xv.abs() + (s * e).abs()) + s * de
    dm0 = dn / a + U * (m0.abs() + dn / a)
    if xc_prev is None:
        xc, dxc = xv.clone(), torch.zeros_like(xv)
    else:
        xp = xc_prev.to(f64)
        xc = cc * xp + c0 * m0
        mag = (cc * xp).abs() + abs(c0) * (m0.abs() + dm0)
        for c, m in ((c1, m1), (c2, m2), (c3, m3)):
            if m is not None:
                xc = xc + c * m.to(f64)
                mag = mag + (c * m.to(f64)).abs()
        dxc = abs(c0) * dm0 + g_n(5) * mag
    xs = xc_out.to(f64).reshape(xv.shape)
    xn = pc * xs + p0 * m0
    mag = (pc * xs).abs() + abs(p0) * (m0.abs() + dm0)
    for c, m in ((p1, m1), (p2, m2)):
        if m is not None:
            xn = xn + c * m.to(f64)
            mag = mag + (c * m.to(f64)).abs()
    dxn = abs(p0) * dm0 + g_n(4) * mag
    return m0, dm0, xc, dxc, xn, dxn


def unipc_update_check(m_out, xc_out, x_next, x, xc_prev, e_cond, e_uncond, guidance, m1, m2, m3, alpha, sigma, coefs,
                       what="unipc_update") -> Report:
    """The worst of the m_out, xc_out and x_next reports against unipc_update_bound."""
    m0, dm0, xc, dxc, xn, dxn = unipc_update_bound(xc_out, x, xc_prev, e_cond, e_uncond, guidance, m1, m2, m3, alpha, sigma, coefs)
    reps = [_plain_check(m_out.reshape(m0.shape), m0, dm0, what + " m_out"),
            _plain_check(xc_out.reshape(xc.shape), xc, dxc, what + " xc_out"),
            _plain_check(x_next.reshape(xn.shape), xn, dxn, what + " x_next")]
    return max(reps, key=lambda r: r.ratio)
