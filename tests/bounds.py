"""Rounding-level checks of the GEMM and attention kernels against a float64 statement of the same operation.

Each check bounds |got - ref64| per element by what the kernel's arithmetic can cost, derived below from the kernel
source (gligen_b200/csrc/gemm_tc.cu, attention.cu, common.cuh).  Nothing here is fitted to measured errors.

Notation.  u = 2^-24 is the unit roundoff of fp32 round-to-nearest; t = 2^-23 bounds one fp32 truncation (round
toward zero), the worst a tensor core's internal alignment or normalisation can do.  h(x) is half an ulp of the output
type at |x|: 2^(floor(log2|x|) - 8) for bf16 (8 significant bits), 2^(floor(log2|x|) - 24) for fp32.  A stored value
is the fp32 result v rounded once, so |stored - ref| <= h(|ref| + e) + e whenever |v - ref| <= e (h is taken at the
largest |v| can be, so a rounding across a power of two is covered).

GEMM family (plain, conv, split-K, paired, B-resident, every epilogue)
-----------------------------------------------------------------------
Accumulation.  bf16 x bf16 products are exact in fp32.  wgmma adds them into the fp32 accumulator in blocks of at
most 16 products; whatever order and rounding it uses inside a block, each of the block's <= 17 inputs (16 products
and the accumulator) loses at most t times the block's largest magnitude when it is aligned and the result is
normalised.  Every partial accumulator is bounded by S = |A| |W|^T, so Ktot products (Ktot = K, or 9 K for the 3x3
convolution) cost at most   gamma_acc = (17 / 16) Ktot t   times S.  Split-K adds `splits` fp32 slabs in order
(splits u S).  The epilogue adds bias, row bias and the residual in fp32: one u per operation on the magnitudes
involved, 4 u S with S extended by |bias| + |rowbias| (+ |residual| after the activation).

LayerNorm fold (gemm_tc.cu:101-107, 137-141).  The output before bias is rstd (acc - mu colsum); with acc and
mu colsum both of size rstd |mu| |colsum|, the accumulation term uses S_ln = rstd (|A| |W'|^T + |mu| |colsum|).
mu and rstd come from the fp32 statistics the kernel sums over `slots` partials in a fixed order:
    |d s1| <= slots u sum|partials of s1|,  |d s2| <= slots u s2,  1 / K rounded (u),
    |d mu| <= (slots + 2) u sum|s1 partials| / K,
    |d var| <= (slots + 2) u E[x^2] + 2 |mu| |d mu| + u mu^2 + u (var + eps)   (E[x^2] - mu^2, + eps),
    |d rstd| / rstd <= |d var| / (2 (var + eps)) + 2 t                       (rsqrtf: 2 ulp).
The output carries these as  |d rstd| / rstd * |y_ln|  +  rstd |d mu| |colsum|.  This is the E[x^2] - E[x]^2 loss:
it grows like (mu / std)^2 u and is part of the bound, not hidden in a tolerance.

Activations (common.cuh).  An error e on the pre-activation becomes at most 1.13 e after SiLU / GELU / quick-GELU
(the largest slope of each is < 1.13).  The functions' own absolute errors:  GELU 2e-6 (erf_rational, 3.3e-7 on erf,
times |x| / 2, tests/test_erf_rational_cpu.py) plus 4 u |x| for its four fp32 operations;  GEGLU 4e-5 * |x-half| (erf_rational3: 1.5e-5 on
gelu(g), stated in common.cuh and checked by test_erf_rational_cpu.py, with a 2.5x margin for the fp32 products) ;
SiLU and quick-GELU use __expf (2 + 1.173 |arg| ulp, CUDA programming guide; arg = 1.702 x for quick-GELU) and
__fdividef (2 ulp), i.e. a relative error of (5 + 2.5 |x|) t.  The gate multiplies by |gate| and adds u.

Aggregate check (bf16 outputs).  A perfectly rounded result has rel-L2(round_bf16(ref64) - ref64) = r0.  A kernel
whose fp32 error is below 3/4 of the rounding error stays within sqrt(1 + 0.75^2) = 1.25 r0, so
rel-L2(got - ref64) <= 1.25 r0 is required.  The fp32 accumulation error of a correct kernel is ~ sqrt(Ktot / 16) u
relative (random) or Ktot / 16 u (all truncations one way), three orders below r0 ~ 1e-3 at every K used here.
An extra bf16 rounding (e.g. before the residual add), a dropped K step or a misplaced bias exceeds it.  The only
derived fp32 error that is not small is the LayerNorm statistics term above; the aggregate allows its rel-L2 on top.

Attention (attention.cu)
------------------------
The kernel computes o_i = sum_j P_j v_j / sum_j P_j with P_j = bf16(exp2(x_j)), x_j = s_j c - m c (c = scale log2 e
in fp32, m the running max of the key's 64-key tile), and l summed from the same rounded P (so the ratio is
consistent).  With P_j = p_j (1 + delta_j), p_j = exp2((s_j - m) c) exact,
    o_kernel - o = sum_j w_j delta_j (v_j - o) / (1 + sum_j w_j delta_j),    w_j = p_j / sum p,
so |o_kernel - o| <= sum_j w_j r_j |v_j - o| / (1 - max r) where |delta_j| <= r_j:
  * bf16 rounding of exp2 at the scale of the key's tile: h(y_j) / y_j with y_j = exp2((s_j - M_t) c), M_t the max up
    to and including that tile (the kernels visit key tiles in order) - between 2^-9 and 2^-8;
  * the exponential: 2^-22 on the MUFU (ex2.approx), eps_exp on the FMA pipe for the last `poly` of every 8 score pairs
    of a tile (ex2_poly3: 7.9e-4 max, tests/test_exp2_poly_cpu.py);
  * the score: the QK^T accumulation (gamma over d products of magnitude sum|q||k|, for key j and for the row max),
    the fmaf / m c roundings (u |x| and u |m c|) and c's own rounding (3 u), all times ln 2;
  * each later rescale by corr = exp2((m_old - m_new) c): 2^-22 plus 2 u |m_old - m_new| c ln 2.
ex2.approx flushes results below 2^-126 to zero: such keys get r_j = 1.  The P.V accumulation adds gamma over Lk
products of sum_j w_j |v_j|, the rescales of o_acc one u each, l's fp32 sum (each lane adds Lk / 4 values, two
butterfly steps, one rescale per tile) a relative (Lk / 4 + 2 ntiles + 4) u of |o|, and 1 / l and o * (1 / l) 3 t.
"""
from __future__ import annotations

import math
from dataclasses import dataclass, field

import torch

U = 2.0 ** -24
T = 2.0 ** -23
EPS_GELU = 2e-6
EPS_GEGLU = 4e-5
ACT_SLOPE = 1.13
EPS_EX2_MUFU = 2.0 ** -22
EPS_EX2_POLY = 7.9e-4
LN2 = math.log(2.0)


def half_ulp(x: torch.Tensor, dtype) -> torch.Tensor:
    """Half an ulp of `dtype` (bf16 or fp32) at |x| (fp64)."""
    bits = 8 if dtype == torch.bfloat16 else 24
    ax = x.abs().clamp_min(2.0 ** -126)
    return torch.exp2(torch.floor(torch.log2(ax)) - bits)


def round_to(x: torch.Tensor, dtype) -> torch.Tensor:
    return x.to(dtype).to(torch.float64)


def rel_l2(a, b):
    return ((a - b).norm() / b.norm().clamp_min(1e-300)).item()


@dataclass
class Report:
    """Worst ratio of |error| to the per-element bound, and of rel-L2 to its limit (<= 1 passes)."""
    what: str
    ratio: float
    agg_ratio: float = 0.0
    worst: str = ""
    extra: dict = field(default_factory=dict)

    @property
    def ok(self):
        return self.ratio <= 1.0 and self.agg_ratio <= 1.0

    def __str__(self):
        return f"{self.what}: elementwise {self.ratio:.3f} of bound, aggregate {self.agg_ratio:.3f} of limit {self.worst}"


def _elementwise(got64, ref64, err, dtype):
    bound = half_ulp(ref64.abs() + err, dtype) + err if dtype == torch.bfloat16 else err + U * (ref64.abs() + err)
    r = (got64 - ref64).abs() / bound
    i = int(torch.argmax(r))
    return r.reshape(-1)[i].item(), i, bound


def _matmul_abs(a, w, conv):
    """|A| |W|^T (fp64), as a GEMM or as the 3x3 convolution with zero padding."""
    K = a.shape[-1]
    A = a.reshape(-1, K).to(torch.float64).abs()
    W = w.to(torch.float64).abs()
    if conv is None:
        return A @ W.t()
    B, H, Wd = conv
    xp = torch.nn.functional.pad(A.reshape(B, H, Wd, K), (0, 0, 1, 1, 1, 1))
    wt = W.view(9, -1, K)
    return sum(xp[:, t // 3:t // 3 + H, t % 3:t % 3 + Wd].reshape(-1, K) @ wt[t].t() for t in range(9))


def gemm_check(got, a, w, bias=None, rowbias=None, rows_per_batch=1, act=0, gate=None, residual=None, geglu=False,
               conv=None, ln=None, splits=1, aggregate=True, what="gemm") -> Report:
    """Bound of the module docstring for one glg_gemm call (arguments as CudaOps.gemm; `got` the stored output)."""
    from ref_ops import RefOps
    f64 = torch.float64
    dev = got.device
    M = got.numel() // got.shape[-1]
    Nout = got.shape[-1]
    ref = torch.empty(got.shape, dtype=f64, device=dev)
    RefOps(dev, compute_dtype=f64).gemm(a, w, ref, bias=bias, rowbias=rowbias, rows_per_batch=rows_per_batch, act=act,
                                        gate=gate, residual=residual, geglu=geglu, conv=conv, ln=ln)
    ref = ref.reshape(M, Nout)
    got64 = got.reshape(M, Nout).to(f64)
    K = a.shape[-1]
    ktot = K * (9 if conv is not None else 1)
    gamma = 17.0 / 16.0 * ktot * T + (splits + 4) * U
    S = _matmul_abs(a, w, conv)                                   # [M, N]
    N = S.shape[1]
    extra = torch.zeros_like(S)                                   # LayerNorm-statistics error (not scaled by gamma)
    y_pre_abs = None
    if ln is not None:
        st, colsum, eps = ln
        st = st.to(f64)
        slots = st.shape[0]
        s1, s2 = st[:, :, 0].sum(0), st[:, :, 1].sum(0)
        s1abs = st[:, :, 0].abs().sum(0)
        mu = s1 / K
        ex2 = s2 / K
        var = (ex2 - mu * mu).clamp_min(0)
        rstd = torch.rsqrt(var + eps)
        dmu = (slots + 2) * U * s1abs / K
        dvar = (slots + 2) * U * ex2 + 2 * mu.abs() * dmu + U * mu * mu + U * (var + eps)
        drel = dvar / (2 * (var + eps)) + 2 * T
        cs = colsum.to(f64)
        A = a.reshape(-1, K).to(f64)
        y_ln = rstd[:, None] * (A @ w.to(f64).t() - mu[:, None] * cs[None])
        S = rstd[:, None] * (S + mu.abs()[:, None] * cs.abs()[None])
        extra = drel[:, None] * y_ln.abs() + (rstd * dmu)[:, None] * cs.abs()[None]
    if bias is not None:
        S = S + bias.to(f64).abs()[None]
    if rowbias is not None:
        idx = torch.arange(M, device=dev) // rows_per_batch
        S = S + rowbias.to(f64).abs()[idx]
    e = gamma * S + extra                                         # error of the pre-activation value
    if geglu:
        pre = torch.empty(M, N, dtype=f64, device=dev)
        RefOps(dev, compute_dtype=f64).gemm(a, w, pre, bias=bias, ln=ln)
        t4 = pre.view(M, N // 256, 2, 128)
        x, g = t4[:, :, 0], t4[:, :, 1]
        e4 = e.view(M, N // 256, 2, 128)
        ex, eg = e4[:, :, 0], e4[:, :, 1]
        gel = torch.nn.functional.gelu(g)
        err = (ex * (gel.abs() + ACT_SLOPE * eg) + x.abs() * (ACT_SLOPE * eg + EPS_GEGLU) + 2 * U * (x * gel).abs()).reshape(M, N // 2)
    else:
        err = e
        if act:
            pre = torch.empty(M, N, dtype=f64, device=dev)
            RefOps(dev, compute_dtype=f64).gemm(a, w, pre, bias=bias, rowbias=rowbias, rows_per_batch=rows_per_batch, ln=ln)
            post = ref if (gate is None and residual is None) else torch.empty_like(pre)
            if post is not ref:
                RefOps(dev, compute_dtype=f64).gemm(a, w, post, bias=bias, rowbias=rowbias, rows_per_batch=rows_per_batch, act=act, ln=ln)
            own = EPS_GELU + 4 * U * pre.abs() if act == 2 else (5 + 2.5 * pre.abs()) * T * post.abs()
            err = ACT_SLOPE * err + own
        if gate is not None:
            gv = float(gate.reshape(-1)[0])
            err = abs(gv) * err + U * (ref.abs() + err)
        if residual is not None:
            err = err + U * (ref.abs() + residual.reshape(M, -1).to(f64).abs() + err)
    dt = got.dtype
    ratio, i, _ = _elementwise(got64, ref, err, dt)
    agg = 0.0
    ex = {}
    if dt == torch.bfloat16 and aggregate:
        r0 = rel_l2(round_to(ref, torch.bfloat16), ref)
        allow = (extra.norm() / ref.norm().clamp_min(1e-300)).item() if ln is not None else 0.0
        r = rel_l2(got64, ref)
        agg = r / (1.25 * r0 + allow) if r0 > 0 else (0.0 if r == 0 else math.inf)
        ex = dict(rel_l2=r, r0=r0)
    row, col = divmod(i, Nout)
    worst = f"(worst at row {row} col {col}: got {got64.reshape(-1)[i].item():.6g} ref {ref.reshape(-1)[i].item():.6g})"
    return Report(what, ratio, agg, worst, ex)


def _heads(t, B, L, H, d):
    return t.reshape(B, L, H, d).permute(0, 2, 1, 3).to(torch.float64)


def attention_check_scores(got, s, v, c, d, poly=0, causal=False, qk_abs=None, what="attention") -> Report:
    """Bound for outputs `got` [n, Lq, dv] of rows with exact scores s [n, Lq, Lk] (fp64, before the scale), values
    v [n, Lk, dv] and exponent scale c (scale * log2 e).  qk_abs [n, Lq, Lk] = sum|q||k| (None: scores are exact inputs,
    d products per score otherwise)."""
    f64 = torch.float64
    n, Lq, Lk = s.shape
    s = s.to(f64)
    v = v.to(f64)
    if causal:
        s = s.masked_fill(torch.ones(Lq, Lk, dtype=torch.bool, device=s.device).triu(1), float("-inf"))
    ntiles = (Lk + 63) // 64
    pad = ntiles * 64 - Lk
    sp = torch.nn.functional.pad(s, (0, pad), value=float("-inf"))
    tile_max = sp.view(n, Lq, ntiles, 64).amax(-1)
    run = torch.cummax(tile_max, dim=-1).values                   # running max after each tile
    Mt = run.repeat_interleave(64, dim=-1)[..., :Lk]
    m = run[..., -1:]
    p = torch.exp2((s - m) * c)
    l = p.sum(-1, keepdim=True)
    w = p / l
    o = w @ v
    y = torch.exp2((s - Mt) * c)
    rho = torch.where(y > 0, half_ulp(y, torch.bfloat16) / y.clamp_min(1e-300), torch.zeros_like(y))
    lane = (torch.arange(Lk, device=s.device) % 64) // 8
    eps_exp = torch.where(lane >= 8 - poly, EPS_EX2_POLY, EPS_EX2_MUFU).to(f64)
    sfin = torch.where(torch.isfinite(s), s, m.expand_as(s))
    xabs = ((sfin - Mt) * c).abs()
    r = rho + eps_exp + LN2 * (U * xabs + U * (Mt * c).abs() + 3 * U * (sfin - m).abs() * c)
    if qk_abs is not None:
        ds = 17.0 / 16.0 * d * T * qk_abs
        ds_max = ds.amax(-1, keepdim=True)
        r = r + LN2 * c * (ds + ds_max)
    # later rescales: one per tile boundary where the running max moved
    step = torch.diff(run, dim=-1, prepend=run[..., :1])
    step = torch.where(torch.isfinite(step), step, torch.zeros_like(step))
    ecorr = EPS_EX2_MUFU + 2 * U * step.abs() * c * LN2
    later = torch.flip(torch.cumsum(torch.flip(ecorr, [-1]), -1), [-1]) - ecorr      # rescales after tile t
    r = r + later.repeat_interleave(64, dim=-1)[..., :Lk]
    r = torch.where(y < 2.0 ** -126, torch.ones_like(r), r)
    r = torch.where(torch.isfinite(s), r, torch.zeros_like(r))
    rmax = r.amax(-1, keepdim=True).clamp_max(0.5)
    e = _spread(w * r, v, o) / (1 - rmax)
    e = e + (17.0 / 16.0 * Lk * T + (ntiles + 3) * T) * (w @ v.abs()) + (Lk / 4 + 2 * ntiles + 4) * U * o.abs()
    got64 = got.to(f64)
    ratio, i, _ = _elementwise(got64, o, e, torch.bfloat16)
    dv = o.shape[-1]
    hq, col = divmod(i, dv)
    hh, row = divmod(hq, Lq)
    return Report(what, ratio, 0.0, f"(worst at row {row} col {col} of slice {hh}: got {got64.reshape(-1)[i].item():.6g} "
                                    f"ref {o.reshape(-1)[i].item():.6g})")


def _spread(wr, v, o):
    """sum_j wr_ij |v_j - o_i| (fp64), in row chunks so that the [rows, Lk, dv] intermediate stays near 1 GB."""
    out = torch.empty_like(o)
    step = max(1, 2 ** 27 // (wr.shape[0] * wr.shape[-1] * v.shape[-1]))
    for i in range(0, wr.shape[1], step):
        out[:, i:i + step] = torch.einsum("nij,nijc->nic", wr[:, i:i + step], (v[:, None, :, :] - o[:, i:i + step, None, :]).abs())
    return out


def attention_check(got, q, k, v, heads, d_head, poly=0, causal=False, what="attention", max_elems=2 ** 28) -> Report:
    """Bound for one glg_attention call (arguments as CudaOps.attention), in fp64 chunks of batch x heads."""
    B, Lq, _ = q.shape
    Lk = k.shape[1]
    scale = float(d_head) ** -0.5
    c = scale * 1.4426950408889634
    worst = Report(what, 0.0)
    G = B * heads
    per = max(1, max_elems // (Lq * Lk * 8))
    qh, kh, vh = _heads(q, B, Lq, heads, d_head), _heads(k, B, Lk, heads, d_head), _heads(v, B, Lk, heads, d_head)
    gh = _heads(got, B, Lq, heads, d_head)
    qh, kh, vh, gh = (t.reshape(G, t.shape[2], d_head) for t in (qh, kh, vh, gh))
    for g0 in range(0, G, per):
        sl = slice(g0, g0 + per)
        s = qh[sl] @ kh[sl].transpose(1, 2)
        qk = qh[sl].abs() @ kh[sl].abs().transpose(1, 2)
        rep = attention_check_scores(gh[sl], s, vh[sl], c, d_head, poly=poly, causal=causal, qk_abs=qk, what=what)
        if rep.ratio > worst.ratio:
            worst = rep
    return worst


def stats_restated(out):
    """gemm_tc.cu:130-169 on the stored bf16 output: per row and 32-column slot, lane q (columns 8 jj + 2 q + {0, 1})
    adds (x0 + x1) and fma(x0, x0, fma(x1, x1, sq)) over jj = 0..3, then the butterfly (q0 + q1) + (q2 + q3)."""
    M, N = out.shape
    f = out.float().view(M, N // 32, 4, 4, 2)            # row, slot, jj, q, pair
    s = torch.zeros(M, N // 32, 4, device=out.device)
    sq = torch.zeros_like(s)
    for jj in range(4):
        x0, x1 = f[:, :, jj, :, 0], f[:, :, jj, :, 1]
        s = s + (x0 + x1)
        sq = x0 * x0 + (x1 * x1 + sq)                     # bf16 squares are exact in fp32: fma == add of the product
    s = (s[..., 0] + s[..., 1]) + (s[..., 2] + s[..., 3])
    sq = (sq[..., 0] + sq[..., 1]) + (sq[..., 2] + sq[..., 3])
    return torch.stack([s, sq], -1).permute(1, 0, 2)     # slot-major [S, M, 2]
