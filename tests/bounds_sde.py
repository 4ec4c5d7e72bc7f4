"""The stochastic update kernel (elementwise.cu: sde_update_kernel, glg_sde_update) stated in torch, and its rounding-level check
against float64, in the notation of tests/bounds.py (u, g(L)).  Nothing here is fitted to measured errors.

The reference is the float64 evaluation of the kernel's formula with the fp32 scalars it receives (guidance, alpha, sigma, cx,
k0, k1, ce, cz: the host rounds its float64 values once).  Per element, any order of FMA contraction:
  * e = u + g (e_c - u) and m0 = (x - sigma e) / alpha exactly as for glg_dpm_update (tests/bounds_dpm.py): |de| <= g(3) (|u| +
    |g| |e_c - u|), |dm0| <= dn / alpha + u (|m0| + dn / alpha) with dn = g(2) (|x| + |sigma e|) + sigma |de|.
  * x_next = cx x + k0 m0 + k1 m1 + ce e + cz z: a chain of <= 5 products, |dx| <= |k0| dm0 + |ce| de + g(5) (|cx x| + |k0 m0| +
    |k1 m1| + |ce e| + |cz z|) (m1, z are inputs, exact).
x0_out is checked against m0 and x_next against x_next with these bounds (tests/bounds.py _plain_check: elementwise and rel-L2).
"""
from __future__ import annotations

import torch

from bounds import U, Report, _plain_check, g_n
from bounds_dpm import _f32


def sde_update_ref(x, e_cond, e_uncond, guidance, m1, z, alpha, sigma, coefs):
    """(m0, x_next) of glg_sde_update in the dtype of x: fp32 tensors give the kernel's statement with fp32 scalars, float64
    tensors the float64 step.  m1 may be None; coefs = (cx, k0, k1, ce, cz)."""
    cast = _f32 if x.dtype == torch.float32 else float
    g, a, s = cast(guidance), cast(alpha), cast(sigma)
    cx, k0, k1, ce, cz = (cast(c) for c in coefs)
    e = e_cond if e_uncond is None else e_uncond + g * (e_cond - e_uncond)
    m0 = (x - s * e) / a
    xn = cx * x + k0 * m0
    if m1 is not None:
        xn = xn + k1 * m1
    xn = xn + ce * e + cz * z
    return m0, xn


def sde_update_bound(x, e_cond, e_uncond, guidance, m1, z, alpha, sigma, coefs):
    """float64 (m0, dm0, x_next, dx_next): the exact values with the kernel's fp32 scalars and their error bounds."""
    f64 = torch.float64
    g, a, s = _f32(guidance), _f32(alpha), _f32(sigma)
    cx, k0, k1, ce, cz = (_f32(c) for c in coefs)
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
    zv = z.to(f64)
    xn = cx * xv + k0 * m0 + ce * e + cz * zv
    mag = (cx * xv).abs() + (k0 * m0).abs() + (ce * e).abs() + (cz * zv).abs()
    if m1 is not None:
        xn = xn + k1 * m1.to(f64)
        mag = mag + (k1 * m1.to(f64)).abs()
    dxn = abs(k0) * dm0 + abs(ce) * de + g_n(5) * mag
    return m0, dm0, xn, dxn


def sde_update_check(x0_out, x_next, x, e_cond, e_uncond, guidance, m1, z, alpha, sigma, coefs, what="sde_update") -> Report:
    """The worse of the x0_out (when given) and x_next reports against sde_update_bound."""
    m0, dm0, xn, dxn = sde_update_bound(x, e_cond, e_uncond, guidance, m1, z, alpha, sigma, coefs)
    rep = _plain_check(x_next.reshape(xn.shape), xn, dxn, what + " x_next")
    if x0_out is None:
        return rep
    r2 = _plain_check(x0_out.reshape(m0.shape), m0, dm0, what + " x0_out")
    return r2 if r2.ratio > rep.ratio else rep
