"""The DPM-Solver++ update kernel (elementwise.cu: dpm_update_kernel, glg_dpm_update) stated in torch, and its rounding-level
check against float64, in the notation of tests/bounds.py (u, g(L)), from which the shared pieces are imported.  Nothing here
is fitted to measured errors.

The reference is the float64 evaluation of the kernel's formula with the fp32 scalars it receives (guidance, alpha, sigma,
cx, k0, k1, k2: the host rounds its float64 values once).  Per element, any order of FMA contraction:
  * e = u + g (e_c - u): two roundings, |de| <= g(3) (|u| + |g| |e_c - u|); without CFG e = e_c exactly.
  * m0 = (x - sigma e) / alpha, an IEEE division: |dm0| <= dn / alpha + u (|m0| + dn / alpha) with
    dn = g(2) (|x| + |sigma e|) + sigma |de|.  The CFG error reaches m0 multiplied by sigma / alpha, the noise-to-signal ratio
    of the evaluated timestep: 11 at t = 951 (the first step of S = 20) and 14.6 at t = 999 in SD's schedule.  That factor is
    the bound's, not slack: it is what the data prediction does to any error in e.
  * x_prev = cx x + k0 m0 + k1 m1 + k2 m2: a chain of <= 4 products, |dx| <= |k0| dm0 + g(4) (|cx x| + |k0 m0| + |k1 m1| + |k2 m2|)
    (m1, m2 are inputs, exact).
x0_out is checked against m0 and x_prev against x_prev with these bounds (tests/bounds.py _plain_check: elementwise and rel-L2).
"""
from __future__ import annotations

import numpy as np
import torch

from bounds import U, Report, _plain_check, g_n


def _f32(v) -> float:
    return float(np.float32(v))


def dpm_update_ref(x, e_cond, e_uncond, guidance, m1, m2, alpha, sigma, coefs):
    """(m0, x_prev) of glg_dpm_update in the dtype of x: fp32 tensors give the kernel's statement with fp32 scalars, float64
    tensors the float64 solver step.  m1, m2 may be None."""
    cast = _f32 if x.dtype == torch.float32 else float
    g, a, s = cast(guidance), cast(alpha), cast(sigma)
    cx, k0, k1, k2 = (cast(c) for c in coefs)
    e = e_cond if e_uncond is None else e_uncond + g * (e_cond - e_uncond)
    m0 = (x - s * e) / a
    xp = cx * x + k0 * m0
    if m1 is not None:
        xp = xp + k1 * m1
    if m2 is not None:
        xp = xp + k2 * m2
    return m0, xp


def dpm_update_bound(x, e_cond, e_uncond, guidance, m1, m2, alpha, sigma, coefs):
    """float64 (m0, dm0, x_prev, dx_prev): the exact values with the kernel's fp32 scalars and their error bounds."""
    f64 = torch.float64
    g, a, s = _f32(guidance), _f32(alpha), _f32(sigma)
    cx, k0, k1, k2 = (_f32(c) for c in coefs)
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
    xp = cx * xv + k0 * m0
    mag = (cx * xv).abs() + (k0 * m0).abs()
    for k, m in ((k1, m1), (k2, m2)):
        if m is not None:
            xp = xp + k * m.to(f64)
            mag = mag + (k * m.to(f64)).abs()
    dxp = abs(k0) * dm0 + g_n(4) * mag
    return m0, dm0, xp, dxp


def dpm_update_check(x0_out, x_prev, x, e_cond, e_uncond, guidance, m1, m2, alpha, sigma, coefs, what="dpm_update") -> Report:
    """The worse of the x0_out and x_prev reports against dpm_update_bound."""
    m0, dm0, xp, dxp = dpm_update_bound(x, e_cond, e_uncond, guidance, m1, m2, alpha, sigma, coefs)
    rep = _plain_check(x_prev.reshape(xp.shape), xp, dxp, what + " x_prev")
    r2 = _plain_check(x0_out.reshape(m0.shape), m0, dm0, what + " x0_out")
    return r2 if r2.ratio > rep.ratio else rep
