"""Rounding-level checks of the kernels against a float64 statement of the same operation.

Each check bounds |got - ref64| per element by what the kernel's arithmetic can cost, derived below from the kernel
source (gligen_b200/csrc/gemm_tc.cu, attention.cu, norm.cu, elementwise.cu, frontend.cu, common.cuh).  Nothing here is fitted to measured errors.

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

Summation lemma (used below).  A floating-point sum, in any order and with any contraction into FMA, whose every term
passes through at most L roundings, errs by at most g(L) sum|terms| with g(L) = L u / (1 - L u): each rounding of a
partial costs u times that partial, and a partial is bounded by the sum of |terms| it contains.

GroupNorm (norm.cu: gn_reg_kernel, gn_small_kernel, gn_fused_kernel)
--------------------------------------------------------------------
Each (sample, group) of N = HW cpg elements is reduced as shifted moments S1 = sum d, S2 = sum d^2 with d = x - p
(one rounding: u |d|).  The pivot p differs per path:
  * reg: p = x[row 0, first channel of the group];
  * small: p = the fp32 mean of row 0 over the group's channels (any value near it serves: only |x - p| enters below);
  * fused: p_c = x[row 0, c] per channel, then S1' = S1 + n d_c, S2' = S2 + 2 d_c S1 + n d_c^2 with d_c = p_c - P,
    P = p of the group's first channel.  Every partial of S1' / S2' is then bounded by A1 = sum(|x - p_c| + |d_c|) /
    A2 = sum(|x - p_c| + |d_c|)^2 (for reg and small, A1 = sum|x - p|, A2 = sum (x - p)^2).
so |dS1| <= g(L1) A1 and |dS2| <= g(L2) A2 with the depths L of each path's summation order:
  * reg (n = ceil(N / 4 / 256) 4-element units per thread): L1 = 1 + 2 + n + 5 + 8 (d, the pair sums, the thread's
    running sum, warp_sum, the 8 warp partials); L2 = 2 + 4 n + 5 + 8 (d^2 carries d's rounding twice; four FMAs per unit);
  * small (n = ceil(N / 2 / 256) pairs per thread): L1 = 2 + n + 13, L2 = 2 + 2 n + 13;
  * fused (n_r rows per thread, rpi row lanes, cpg channels, the cross-CTA reduce of `chunks` partials by Q = threads /
    groups threads, then Q sums in order: depth D = ceil(chunks / Q) + Q): L1 = 1 + n_r + rpi + 2 + cpg + D;
    L2 = 2 + 2 (n_r + rpi + 1) + 5 + cpg + D (S1's own error enters S2' through 2 |d_c| |dS1|, bounded the same way).
    n_r and D depend on the grid: chunks = min(capacity / B, ceil(HW / (4 rpi))) with capacity between num_sms and
    8 num_sms CTAs; the bound takes the worst n_r and the worst D over that range.
Then m1 = S1 (1/N) and E2 = S2 (1/N) (1/N rounded, one product: g(2)), var = E2 - m1^2 (one rounding of m1^2 unless
contracted, one of the difference), + eps (u), the clamp at 0 (moves toward the truth), rsqrtf (2 ulp: 2 t):
    |d var| <= |dE2| + 2 |m1| |dm1| + dm1^2 + u (|m1| + dm1)^2 + u (var + eps + ...),
    rstd (1 + rho) with rho = (1 - |d var| / (var + eps))^(-1/2) (1 + 2 t) - 1,      mean = p + m1: |dmu| <= dm1 + u |mu|.
The variance term scales with A2 / N / var = E[(x - p)^2] / var: with a good pivot ~ 2, with the raw E[x^2] - E[x]^2
(p = 0) it is 1 + (mean / std)^2.  The affine step as each kernel writes it:
  * reg (and the LayerNorms below): t = fmaf((v - mu) rstd, gamma, beta): two roundings before the FMA (and one more if
    the product with gamma is not fused), so |dt| <= |gamma| (r |v - mu| ((1 + rho)(1 + u)^2 - 1) + r (1 + rho)(1 + u)^2 |dmu|)
    + u |gamma| |z| + u |t|;
  * fused / small: ga = gamma rstd, t = fmaf(v, ga, beta - mu ga): the same with (1 + u) in place of (1 + u)^2, plus
    u |mu ga| (the product mu ga) and u (|beta| + |mu ga|) (the difference) - the cancellation cost of folding mu into
    the bias.
SiLU (silu_fast: __expf, __fdividef) adds the activation terms above.  bf16 output: h(|y| + e) + e, and the aggregate
rel-L2 <= 1.25 r0 plus the rel-L2 of the statistics terms (as the LayerNorm fold of the GEMM).

Row LayerNorms (ln_kernel, layernorm_rows_kernel<bf16|f32>)
------------------------------------------------------------
One warp per row, two-pass in registers.  The mean: each lane adds its k = 8 ceil(C / 256) values in order, warp_sum,
/ C: |dmu| <= g(k + 5) sum|x| / C + u |mu|.  The variance sums d = v - mu_k (exact mean replaced by mu_k costs
C dmu^2: sum (v - mu_k)^2 = sum (v - mu)^2 + C (mu_k - mu)^2) with FMAs: g(2 + k + 5) sum d^2, then / C (u) and + eps
(u).  rho and the affine step as for gn_reg.  fp32 output (layernorm_rows_f32): e + u (|y| + e) per element.

softmax_rows (elementwise.cu)
-----------------------------
c = scale log2 e is formed on the host in fp32 (scale rounded to fp32, the constant rounded, the product: 3 u
relative).  x_j = fmaf(s_j, c, -(m c)) costs u |m c| + u |x_j|, and the 3 u of c times |s_j - m| c; exp2f (no fast
math) is within 2 ulp (2 t).  So each e_j = exp2(x_j) carries a relative error
    r_j = ln2 (u |m c| + u |x_j| + 3 u |s_j - m| c) + 2 t     (plus 2^-148 absolute below the normal range).
The fp32 sum: each thread adds 4 values per 1024-column stride (3 roundings inside the group, one into its running
sum), then warp_sum (5) and the 8 warp partials in order (8): L = 3 + ceil(cols / 1024) + 13, all terms positive, so
tot (1 + tau) with |tau| <= g(L) + max r_j.  1.0f / tot (correctly rounded) and e_j * inv: 2 u.  Relative error of
p_j: r_j + tau + 2 u (first order; the bound uses the exact quotient (1 + r_j)(1 + u)^2 / (1 - tau) - 1).

CUDA-core edge convolutions (conv_in_kernel, conv_in_px4_kernel, conv_out_kernel, conv_out_px8_kernel)
--------------------------------------------------------------------------------------------------------
conv_in: fp32 FMA chains from the bias over 9 Cin taps x channels: g(9 Cin) (|bias| + sum|x||w|), then bf16.
conv_out: per lane, 8 products summed (1 + 7 roundings) into the running sum, 9 ceil(Cin / 256) such steps, warp_sum
(5), + bias (1): g(8 + 9 ceil(Cin / 256) + 6) (|bias| + sum|x||w|), fp32 out.  For fp32 outputs this worst case is far
above the error of a correct kernel; the precision teeth are the exact tests on inputs whose every partial sum is
representable (tests/test_norm_edge_kernels_gpu.py).

LayerNorm of a computed input (clip_vision_embed, dwconv7_ln, clip_image_head)
-------------------------------------------------------------------------------
The kernel normalises x' = x + delta with |delta| <= eta (clip_vision_embed: the fp32 add, eta = u |cls or patch + pos|;
dwconv7_ln: an FMA chain from the bias over <= 49 taps, eta = g(49) (|bias| + sum |x||w|)).  Exactly,
(x'_i - mu') r' - (x_i - mu) r = (delta_i - mean delta) r' + (x_i - mu)(r' - r), and |var' - var| <= 2 mean(|x - mu|
(eta + mean eta)) + mean((eta + mean eta)^2) = dv, so r' = r (1 + rho_in) with rho_in = (1 - dv / (var + eps))^(-1/2) - 1.
The row LayerNorm bound above is then taken at the magnitudes of x' (|x| + eta, var + dv) and its rho composed with
rho_in.  dwconv7_ln's lanes add channel pairs (depth 2 ceil(C / 64) + 5); clip_image_head's block reduction adds
ceil(C / 256) values per thread, a warp butterfly and 8 warp partials (depth ceil(C / 256) + 13), fp32 out; its
projection is an FMA chain over C / 32 columns per lane and a butterfly: |W| |pooled_kernel - pooled| +
g(C / 32 + 5) |pooled| |W|^T.

Embeddings, token rows, the sampler update (elementwise.cu, frontend.cu)
------------------------------------------------------------------------
CUDA math API accuracy (no fast math): expf, sinf, cosf 2 ulp, powf 4 ulp; an ulp is at most 2^-23 of the result.
  * timestep_embedding: freq = expf(c k / half), c = -ln 1e4 in fp32: the exponent a carries 3 roundings (3 u |a|),
    expf 2 t, arg = t freq one more u; sinf / cosf (slope <= 1) add 2 t |result|; bf16.
  * position_features: f = powf(100, k / freqs): the rounded exponent costs ln(100) (k / freqs) u relative, powf 4 t,
    a = f coord u; sin / cos as above; v = e m + (1 - m) null: g(3) over |e m| + |(1 - m) null|; zero padding exact.
  * embed_tokens: one fp32 add (u |t + p|); spatial_tokens: x m + null (1 - m) + pos, g(4) over the three terms.
  * cast: exact (one round-to-nearest-even to bf16).
  * sampler_update, against float64 with the fp32 scalars the kernel receives: e = u + g (e_c - u): g(3) (|u| +
    |g| |e_c - u|); ep = sum c_i o_i: |c0| de + g(5) sum |c_i o_i|; pred = (x - s1 ep) / s0 (the division correctly
    rounded): (g(2) (|x| + |s1 ep|) + s1 dep) / s0 + u |pred|; x_prev = s2 pred + s3 ep: s2 dpred + s3 dep +
    g(3) (|s2 pred| + |s3 ep|); fp32 outputs.
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


class _Worst:
    """The elementwise worst over row chunks, and per-row sums of squares for the aggregate rel-L2.  The sums over all
    rows are taken once at the end, so a report does not depend on how its rows were chunked."""

    def __init__(self, rows, cols, dev):
        self.cols = cols
        self.ratio, self.i, self.vals = -math.inf, 0, (0.0, 0.0)
        self.sq = torch.zeros(4, rows, dtype=torch.float64, device=dev)  # |got - ref|^2, |ref|^2, |bf16(ref) - ref|^2, stats^2

    def add(self, r0, got64, ref, err, dtype, stats=None, sums=True):
        """Rows [r0, r0 + len(ref)) of the output ([rows, cols] float64 views; dtype the stored output's)."""
        ratio, i, _ = _elementwise(got64, ref, err, dtype)
        if not math.isnan(self.ratio) and not ratio <= self.ratio:         # a NaN ratio is kept
            self.ratio, self.i = ratio, r0 * self.cols + i
            self.vals = (got64.reshape(-1)[i].item(), ref.reshape(-1)[i].item())
        if sums and dtype == torch.bfloat16:
            rows = slice(r0, r0 + ref.shape[0])
            self.sq[0, rows] = ((got64 - ref) ** 2).sum(1)
            self.sq[1, rows] = (ref ** 2).sum(1)
            self.sq[2, rows] = ((round_to(ref, torch.bfloat16) - ref) ** 2).sum(1)
            if stats is not None:
                st = torch.where(torch.isfinite(stats), stats, torch.zeros_like(stats))
                self.sq[3, rows] = (st ** 2).sum(1)

    def aggregate(self):
        """(rel-L2 over the limit 1.25 r0 + the rel-L2 of the statistics term, details) for bf16 outputs."""
        d, nref, d0, st = self.sq.sum(1).sqrt().tolist()
        nref = max(nref, 1e-300)
        r, r0, allow = d / nref, d0 / nref, st / nref
        agg = r / (1.25 * r0 + allow) if r0 > 0 else (0.0 if r == 0 else math.inf)
        return agg, dict(rel_l2=r, r0=r0)


def _row_chunks(rows, cols, max_elems, conv=None):
    """Row ranges (compute c0, c1, keep k0, k1, conv of the compute rows) such that one float64 [rows, cols] intermediate
    of a chunk stays within `max_elems` bytes (None: one chunk of every row).  A 3x3 convolution is chunked by whole
    image rows and computes one halo row above and below each chunk (kept rows only are checked), so every kept output
    sees the same taps and zero padding as in the whole image."""
    if max_elems is None:
        yield 0, rows, 0, rows, conv
        return
    if conv is None:
        step = max(1, max_elems // (8 * cols))
        for r in range(0, rows, step):
            yield r, min(rows, r + step), r, min(rows, r + step), None
        return
    B, H, Wd = conv
    step = max(1, max_elems // (8 * cols * Wd))
    for b in range(B):
        for y0 in range(0, H, step):
            y1 = min(H, y0 + step)
            ys, ye = max(0, y0 - 1), min(H, y1 + 1)
            base = b * H * Wd
            yield base + ys * Wd, base + ye * Wd, base + y0 * Wd, base + y1 * Wd, (1, ye - ys, Wd)


def _gemm_rows(a, w, bias, rowbias, act, gate, residual, geglu, conv, ln, gamma):
    """(ref, error bound, LayerNorm-statistics part) of the GEMM rows a [M, K] (rowbias already one row per output row)."""
    from ref_ops import RefOps
    f64 = torch.float64
    dev = a.device
    M, K = a.shape
    ref64 = RefOps(dev, compute_dtype=f64)
    N = w.shape[0] // (9 if conv is not None else 1)
    Nout = N // 2 if geglu else N
    ref = torch.empty(M, Nout, dtype=f64, device=dev)
    ref64.gemm(a, w, ref, bias=bias, rowbias=rowbias, act=act, gate=gate, residual=residual, geglu=geglu, conv=conv, ln=ln)
    S = _matmul_abs(a, w, conv)                                   # [M, N]
    extra = torch.zeros_like(S)                                   # LayerNorm-statistics error (not scaled by gamma)
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
        A = a.to(f64)
        y_ln = rstd[:, None] * (A @ w.to(f64).t() - mu[:, None] * cs[None])
        S = rstd[:, None] * (S + mu.abs()[:, None] * cs.abs()[None])
        extra = drel[:, None] * y_ln.abs() + (rstd * dmu)[:, None] * cs.abs()[None]
    if bias is not None:
        S = S + bias.to(f64).abs()[None]
    if rowbias is not None:
        S = S + rowbias.to(f64).abs()
    e = gamma * S + extra                                         # error of the pre-activation value
    if geglu:
        pre = torch.empty(M, N, dtype=f64, device=dev)
        ref64.gemm(a, w, pre, bias=bias, ln=ln)
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
            ref64.gemm(a, w, pre, bias=bias, rowbias=rowbias, ln=ln)
            post = ref if (gate is None and residual is None) else torch.empty_like(pre)
            if post is not ref:
                ref64.gemm(a, w, post, bias=bias, rowbias=rowbias, act=act, ln=ln)
            own = EPS_GELU + 4 * U * pre.abs() if act == 2 else (5 + 2.5 * pre.abs()) * T * post.abs()
            err = ACT_SLOPE * err + own
        if gate is not None:
            gv = float(gate.reshape(-1)[0])
            err = abs(gv) * err + U * (ref.abs() + err)
        if residual is not None:
            err = err + U * (ref.abs() + residual.to(f64).abs() + err)
    return ref, err, extra


def gemm_check(got, a, w, bias=None, rowbias=None, rows_per_batch=1, act=0, gate=None, residual=None, geglu=False,
               conv=None, ln=None, splits=1, aggregate=True, what="gemm", max_elems=None) -> Report:
    """Bound of the module docstring for one glg_gemm call (arguments as CudaOps.gemm; `got` the stored output).
    max_elems: evaluate in row chunks whose float64 [rows, max(N, K)] intermediates stay within that many bytes (None:
    all rows at once).  The report is the same either way."""
    f64 = torch.float64
    dev = got.device
    M = got.numel() // got.shape[-1]
    Nout = got.shape[-1]
    K = a.shape[-1]
    ktot = K * (9 if conv is not None else 1)
    gamma = 17.0 / 16.0 * ktot * T + (splits + 4) * U
    A, G = a.reshape(-1, K), got.reshape(M, Nout)
    R = None if residual is None else residual.reshape(M, -1)
    dt = got.dtype
    acc = _Worst(M, Nout, dev)
    for c0, c1, k0, k1, cv in _row_chunks(M, max(w.shape[0] // (9 if conv is not None else 1), K), max_elems, conv):
        rb = None if rowbias is None else rowbias[torch.arange(c0, c1, device=rowbias.device) // rows_per_batch]
        lnc = None if ln is None else (ln[0][:, c0:c1], ln[1], ln[2])
        ref, err, extra = _gemm_rows(A[c0:c1], w, bias, rb, act, gate, None if R is None else R[c0:c1], geglu, cv, lnc, gamma)
        keep = slice(k0 - c0, k1 - c0)
        acc.add(k0, G[k0:k1].to(f64), ref[keep], err[keep], dt, extra[keep] if ln is not None else None, sums=aggregate)
    agg, ex = acc.aggregate() if dt == torch.bfloat16 and aggregate else (0.0, {})
    row, col = divmod(acc.i, Nout)
    worst = f"(worst at row {row} col {col}: got {acc.vals[0]:.6g} ref {acc.vals[1]:.6g})"
    return Report(what, acc.ratio, agg, worst, ex)


def _heads(t, B, L, H, d):
    return t.reshape(B, L, H, d).permute(0, 2, 1, 3).to(torch.float64)


def attention_check_scores(got, s, v, c, d, poly=0, causal=False, qk_abs=None, what="attention", row0=0) -> Report:
    """Bound for outputs `got` [n, Lq, dv] of rows with exact scores s [n, Lq, Lk] (fp64, before the scale), values
    v [n, Lk, dv] and exponent scale c (scale * log2 e).  qk_abs [n, Lq, Lk] = sum|q||k| (None: scores are exact inputs,
    d products per score otherwise).  row0: query index of the first row (the causal mask and the report)."""
    f64 = torch.float64
    n, Lq, Lk = s.shape
    s = s.to(f64)
    v = v.to(f64)
    if causal:
        s = s.masked_fill(torch.ones(Lq, Lk, dtype=torch.bool, device=s.device).triu(1 + row0), float("-inf"))
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
    return Report(what, ratio, 0.0, f"(worst at row {row0 + row} col {col} of slice {hh}: got {got64.reshape(-1)[i].item():.6g} "
                                    f"ref {o.reshape(-1)[i].item():.6g})")


def _spread(wr, v, o):
    """sum_j wr_ij |v_j - o_i| (fp64), in row chunks so that the [rows, Lk, dv] intermediate stays near 1 GB."""
    out = torch.empty_like(o)
    step = max(1, 2 ** 27 // (wr.shape[0] * wr.shape[-1] * v.shape[-1]))
    for i in range(0, wr.shape[1], step):
        out[:, i:i + step] = torch.einsum("nij,nijc->nic", wr[:, i:i + step], (v[:, None, :, :] - o[:, i:i + step, None, :]).abs())
    return out


def attention_check(got, q, k, v, heads, d_head, poly=0, causal=False, what="attention", max_elems=2 ** 28) -> Report:
    """Bound for one glg_attention call (arguments as CudaOps.attention), in fp64 chunks of batch x heads, and of query
    rows when one head's [Lq, Lk] scores exceed max_elems bytes."""
    B, Lq, _ = q.shape
    Lk = k.shape[1]
    scale = float(d_head) ** -0.5
    c = scale * 1.4426950408889634
    worst = Report(what, 0.0)
    G = B * heads
    per = max(1, max_elems // (Lq * Lk * 8))
    rows = max(1, min(Lq, max_elems // (Lk * 8)))
    qh, kh, vh = _heads(q, B, Lq, heads, d_head), _heads(k, B, Lk, heads, d_head), _heads(v, B, Lk, heads, d_head)
    gh = _heads(got, B, Lq, heads, d_head)
    qh, kh, vh, gh = (t.reshape(G, t.shape[2], d_head) for t in (qh, kh, vh, gh))
    for g0 in range(0, G, per):
        sl = slice(g0, g0 + per)
        for r0 in range(0, Lq, rows):
            rs = slice(r0, r0 + rows)
            s = qh[sl, rs] @ kh[sl].transpose(1, 2)
            qk = qh[sl, rs].abs() @ kh[sl].abs().transpose(1, 2)
            rep = attention_check_scores(gh[sl, rs], s, vh[sl], c, d_head, poly=poly, causal=causal, qk_abs=qk, what=what, row0=r0)
            if not math.isnan(worst.ratio) and not rep.ratio <= worst.ratio:     # a NaN ratio is kept
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


# ---------------------------------------------------------------------------------------------------------------------
def g_n(L):
    """g(L) = L u / (1 - L u): the summation lemma of the module docstring."""
    return L * U / (1 - L * U)


def _stats_error(N, A1, A2, L1, L2, m1, E2, var, eps):
    """(|d mean - p| bound dm1, |d var| bound) of the kernel's fp32 statistics (module docstring, GroupNorm)."""
    dS1, dS2 = g_n(L1) * A1, g_n(L2) * A2
    dm1 = dS1 / N + g_n(2) * (m1.abs() + dS1 / N)
    dE2 = dS2 / N + g_n(2) * (E2 + dS2 / N)
    dv0 = dE2 + 2 * m1.abs() * dm1 + dm1 * dm1
    dvar = dv0 + U * (m1.abs() + dm1) ** 2 * (1 + U)
    dvar = dvar + U * (var + dvar) * (1 + U)
    dvar = dvar + U * (var + eps + dvar) * (1 + U)
    return dm1, dvar


def _rstd_rho(dvar, var, eps):
    """Relative error bound of rsqrtf(var_kernel + eps) against rsqrt(var + eps) (inf when the bound is vacuous)."""
    delta = dvar / (var + eps)
    rho = (1 - delta).clamp_min(0).rsqrt() * (1 + 2 * T) - 1
    return torch.where(delta < 1, rho, torch.full_like(rho, math.inf))


def _affine_error(v, mu, dmu, r, rho, gamma, beta, fold):
    """(error bound of the fp32 affine output t, its statistics part) for z = (v - mu) r, t = z gamma + beta
    (module docstring: `fold` = fused / small form fmaf(v, gamma r, beta - mu gamma r), else (v - mu) r then fmaf)."""
    k = 1 if fold else 2
    dz = v - mu
    z = dz * r
    ga = gamma.abs()
    stats = ga * r * (dz.abs() * ((1 + rho) - 1) + (1 + rho) * dmu)
    e = ga * r * (dz.abs() * ((1 + rho) * (1 + U) ** k - 1) + (1 + rho) * (1 + U) ** k * dmu)
    if fold:
        mga = (mu.abs() + dmu) * ga * r * (1 + rho) * (1 + U)
        e = e + U * mga + U * (beta.abs() + mga * (1 + U))
    else:
        e = e + U * ga * (z.abs() + e)
    t = z * gamma + beta
    e = e + U * (t.abs() + e) * (1 + U)
    vacuous = ~torch.isfinite(rho).expand_as(e)
    return e.masked_fill(vacuous, math.inf), stats.masked_fill(vacuous, math.inf)


def _silu_error(t, e):
    post = torch.nn.functional.silu(t)
    return ACT_SLOPE * e + (5 + 2.5 * t.abs()) * T * post.abs(), post


def _finish(got, ref, err, stats, what, idx_desc):
    """Elementwise bound, and for bf16 outputs the aggregate (1.25 r0 plus the rel-L2 of the statistics term)."""
    f64 = torch.float64
    got64 = got.to(f64).reshape(ref.shape)
    ratio, i, _ = _elementwise(got64, ref, err, got.dtype)
    agg, ex = 0.0, {}
    if got.dtype == torch.bfloat16:
        r0 = rel_l2(round_to(ref, torch.bfloat16), ref)
        stats = torch.where(torch.isfinite(stats), stats, torch.zeros_like(stats))
        allow = (stats.norm() / ref.norm().clamp_min(1e-300)).item()
        r = rel_l2(got64, ref)
        agg = r / (1.25 * r0 + allow) if r0 > 0 else (0.0 if r == 0 else math.inf)
        ex = dict(rel_l2=r, r0=r0)
    worst = f"(worst at {idx_desc(i)}: got {got64.reshape(-1)[i].item():.6g} ref {ref.reshape(-1)[i].item():.6g})"
    return Report(what, ratio, agg, worst, ex)


def gn_dispatch(B, HW, C, groups, aligned8=True, small_mode=True):
    """glg_groupnorm's kernel choice (norm.cu), restated: "reg5" | "reg10" | "reg20" | "small" | "fused"."""
    cpg = C // groups
    units = HW * (cpg // 4)
    if small_mode and cpg % 4 == 0 and units <= 256 * 20 and aligned8 and C % 4 == 0:
        return "reg5" if units <= 256 * 5 else "reg10" if units <= 256 * 10 else "reg20"
    if small_mode and HW <= 256 and cpg % 2 == 0:
        return "small"
    return "fused"


def gn_fused_geometry(B, HW, C, groups, num_sms=132, chunks=None):
    """(rpi, Q, worst rows per thread, worst cross-CTA reduce depth) of gn_fused_kernel's launch (norm.cu glg_groupnorm).
    `chunks` pins the grid (a restatement); otherwise every capacity from num_sms to 8 num_sms CTAs is allowed."""
    vec = C // 8
    rpi = max(1, 256 // vec)
    threads = vec * rpi
    Q = threads // groups
    max_chunks = (HW + rpi * 4 - 1) // (rpi * 4)

    def grid(cap):
        ch = max(1, min(cap // B, max_chunks))
        rpc = (HW + ch - 1) // ch
        return (HW + rpc - 1) // rpc, rpc

    options = [grid(num_sms), grid(8 * num_sms)] if chunks is None else [grid(chunks * B)]
    n_r = max((rpc + rpi - 1) // rpi for _, rpc in options)
    depth = max((ch + Q - 1) // Q + Q for ch, _ in options)
    return rpi, Q, n_r, depth


def groupnorm_check(y, x, gamma, beta, groups, eps, silu, path, num_sms=132, chunks=None, what="groupnorm") -> Report:
    """Bound of the module docstring for one glg_groupnorm call (x, y [B, HW, C]; path as gn_dispatch returns)."""
    f64 = torch.float64
    B, HW, C = x.shape
    G, cpg = groups, C // groups
    N = HW * cpg
    xv = x.to(f64).reshape(B, HW, G, cpg)
    var, mu = torch.var_mean(xv, dim=(1, 3), correction=0, keepdim=True)          # [B, 1, G, 1]
    if path.startswith("reg"):
        p = xv[:, :1, :, :1]
        dev = (xv - p).abs()
        A1, A2 = dev.sum((1, 3), keepdim=True), (dev * dev).sum((1, 3), keepdim=True)
        n = -(-N // 4 // 256)
        L1, L2 = 3 + n + 13, 2 + 4 * n + 13
    elif path == "small":
        p = x.reshape(B, HW, G, cpg)[:, :1].float().sum(3, keepdim=True).to(f64) / cpg
        dev = (xv - p).abs()
        A1, A2 = dev.sum((1, 3), keepdim=True), (dev * dev).sum((1, 3), keepdim=True)
        n = -(-N // 2 // 256)
        L1, L2 = 2 + n + 13, 2 + 2 * n + 13
    elif path == "fused":
        pc = xv[:, :1]                                                             # per-channel pivots [B, 1, G, cpg]
        p = pc[..., :1]
        dev = (xv - pc).abs() + (pc - p).abs()
        A1, A2 = dev.sum((1, 3), keepdim=True), (dev * dev).sum((1, 3), keepdim=True)
        rpi, Q, n_r, depth = gn_fused_geometry(B, HW, C, G, num_sms, chunks)
        L1 = 1 + n_r + rpi + 2 + cpg + depth
        L2 = 2 + 2 * (n_r + rpi + 1) + 5 + cpg + depth
    else:
        raise ValueError(path)
    m1 = mu - p
    E2 = var + m1 * m1
    dm1, dvar = _stats_error(N, A1, A2, L1, L2, m1, E2, var, eps)
    dmu = dm1 + U * (mu.abs() + dm1)
    r = torch.rsqrt(var + eps)
    rho = _rstd_rho(dvar, var, eps)
    ga = gamma.to(f64).view(1, 1, G, cpg)
    be = beta.to(f64).view(1, 1, G, cpg)
    err, stats = _affine_error(xv, mu, dmu, r, rho, ga, be, fold=not path.startswith("reg"))
    ref = (xv - mu) * r * ga + be
    if silu:
        stats = ACT_SLOPE * stats
        err, ref = _silu_error(ref, err)
    ref, err, stats = (t.reshape(B, HW, C) for t in (ref, err, stats))

    def where(i):
        b, rem = divmod(i, HW * C)
        row, c = divmod(rem, C)
        return f"sample {b} row {row} channel {c} (group {c // cpg})"
    return _finish(y, ref, err, stats, f"{what} [{path}]", where)


def layernorm_check(y, x, gamma, beta, eps, what="layernorm", x_err=None, depth=None) -> Report:
    """Bound for the row LayerNorms: x [..., C] the exact input rows (float64 statement), y the output likewise.
    x_err: bound on |kernel's fp32 input - x| per element (clip_vision_embed's add, dwconv7_ln's taps), None = exact.
    depth: roundings of a term of the mean's sum (default: the warp-per-row kernels' 8 ceil(C / 256) + 5)."""
    f64 = torch.float64
    C = x.shape[-1]
    xv = x.to(f64).reshape(-1, C)
    var, mu = torch.var_mean(xv, dim=1, correction=0, keepdim=True)
    k = depth if depth is not None else 8 * (-(-C // 256)) + 5
    eta = torch.zeros_like(xv) if x_err is None else x_err.to(f64).reshape(-1, C)
    eta_m = eta.mean(1, keepdim=True)
    # the kernel normalises x' = x + delta (|delta| <= eta): its statistics are bounded at the magnitudes of x'
    dv_in = 2 * ((xv - mu).abs() * (eta + eta_m)).mean(1, keepdim=True) + ((eta + eta_m) ** 2).mean(1, keepdim=True)
    var_k = var + dv_in
    dmu = g_n(k) * (xv.abs() + eta).sum(1, keepdim=True) / C + U * (mu.abs() + eta_m)
    dmu = dmu * (1 + U)
    dQ = g_n(2 + k) * C * (var_k + dmu * dmu)
    dvar = dQ / C + dmu * dmu
    dvar = dvar + U * (var_k + dvar) * (1 + U)
    dvar = dvar + U * (var_k + eps + dvar) * (1 + U)
    r = torch.rsqrt(var + eps)
    # input perturbation: (x'_i - mu') r' - (x_i - mu) r = (delta_i - mean delta) r' + (x_i - mu)(r' - r)
    rho_in = _rstd_rho(dv_in, var, eps)
    rho = (1 + rho_in) * (1 + _rstd_rho(dvar, var_k, eps)) - 1
    g64, b64 = gamma.to(f64)[None], beta.to(f64)[None]
    err, stats = _affine_error(xv, mu, dmu + eta + eta_m, r, rho, g64, b64, fold=False)
    err = err + g64.abs() * r * (1 + rho) * U * 2 * (eta + eta_m)          # the roundings of x' - mu at |x' - mu|
    ref = (xv - mu) * r * g64 + b64
    return _finish(y, ref, err, stats, what, lambda i: f"row {i // C} col {i % C}")


def softmax_check(p, s, scale, what="softmax_rows", max_elems=None) -> Report:
    """Bound for one glg_softmax_rows call: s fp32 [rows, cols], p bf16 [rows, cols].  max_elems: as gemm_check's, row
    chunks whose float64 [rows, cols] intermediates stay within that many bytes (None: all rows at once)."""
    f64 = torch.float64
    rows, cols = s.shape
    c = scale * 1.4426950408889634
    L = 3 + -(-cols // 1024) + 13
    acc = _Worst(rows, cols, s.device)
    for r0, r1, _, _, _ in _row_chunks(rows, cols, max_elems):
        s64 = s[r0:r1].to(f64)
        m = s64.amax(1, keepdim=True)
        x = (s64 - m) * c
        e = torch.exp2(x)
        ref = e / e.sum(1, keepdim=True)
        r = LN2 * (U * (m * c).abs() + U * x.abs() + 3 * U * x.abs()) + 2 * T
        tiny = 2.0 ** -148 / e.clamp_min(2.0 ** -1074)
        r = r + torch.where(e < 2.0 ** -126, tiny, torch.zeros_like(tiny))
        tau = g_n(L) * (1 + r.amax(1, keepdim=True)) + (r * e).sum(1, keepdim=True) / e.sum(1, keepdim=True)
        rel = (1 + r) * (1 + U) ** 2 / (1 - tau) - 1
        err = (ref * rel).clamp_max(1.0)
        err = err + 2.0 ** -149 * 2                                               # the subnormal range of the fp32 product
        acc.add(r0, p[r0:r1].to(f64), ref, err, p.dtype)
    agg, ex = acc.aggregate() if p.dtype == torch.bfloat16 else (0.0, {})
    worst = f"(worst at row {acc.i // cols} col {acc.i % cols}: got {acc.vals[0]:.6g} ref {acc.vals[1]:.6g})"
    return Report(what, acc.ratio, agg, worst, ex)


def conv_check(got, x, w, bias, kind, H=None, W=None, extra=None, what=None) -> Report:
    """Bound for glg_conv_in (kind "in": x [B, C0, H, W] fp32 (+ extra), w [9, Cin, Cout], out bf16 [B, HW, Cout]) and
    glg_conv_out (kind "out": x [B, HW, Cin] bf16, w [9, Cout, Cin], out fp32 [B, Cout, H, W])."""
    f64 = torch.float64
    F = torch.nn.functional
    if kind == "in":
        xin = x if extra is None else torch.cat([x, extra], 1)
        B, Cin, H, W = xin.shape
        Cout = w.shape[2]
        wk = w.to(f64).view(3, 3, Cin, Cout).permute(3, 2, 0, 1)
        xi = xin.to(f64)
        L = 9 * Cin
    else:
        B, _, Cin = x.shape
        Cout = w.shape[1]
        wk = w.to(f64).view(3, 3, Cout, Cin).permute(2, 3, 0, 1)
        xi = x.to(f64).reshape(B, H, W, Cin).permute(0, 3, 1, 2)
        L = 8 + 9 * (-(-Cin // 256)) + 6
    ref = F.conv2d(xi, wk, bias.to(f64), padding=1)
    S = F.conv2d(xi.abs(), wk.abs(), bias.to(f64).abs(), padding=1)
    err = g_n(L) * S
    if kind == "in":
        ref, err = (t.permute(0, 2, 3, 1).reshape(B, H * W, Cout) for t in (ref, err))
    dims = tuple(ref.shape)

    def where(i):
        return "index " + str(list(torch.unravel_index(torch.tensor(i), dims)))
    return _finish(got, ref, err, torch.zeros_like(ref), what or f"conv_{kind}", where)


def _plain_check(got, ref, err, what):
    dims = tuple(ref.shape)
    return _finish(got, ref, err, torch.zeros_like(ref), what,
                   lambda i: "index " + str([int(v) for v in torch.unravel_index(torch.tensor(i), dims)]))


def embed_tokens_check(out, ids, table, pos, what="embed_tokens") -> Report:
    """out = bf16(table[ids] + pos[:L]): one fp32 add, then bf16."""
    f64 = torch.float64
    t, p = table.to(f64)[ids], pos.to(f64)[: ids.shape[1]][None]
    return _plain_check(out.reshape(t.shape), t + p, U * (t.abs() + p.abs()), what)


def spatial_tokens_check(y, x, mask, null_feat, pos, n, what="spatial_tokens") -> Report:
    """y = bf16(x m + null (1 - m) + pos): at most 3 roundings per term (g(4) with the 1 - m)."""
    f64 = torch.float64
    C = x.shape[-1]
    xv = x.to(f64).reshape(-1, n, C)
    m = mask.to(f64).view(-1, 1, 1)
    nf, ps = null_feat.to(f64).view(1, 1, C), pos.to(f64).view(1, n, C)
    ref = xv * m + nf * (1 - m) + ps
    err = g_n(4) * ((xv * m).abs() + (nf * (1 - m)).abs() + ps.abs())
    return _plain_check(y.reshape(ref.shape), ref, err, what)


def _sincos_error(arg_abs, rel, val_abs):
    """sinf / cosf (2 ulp, CUDA math API) of an fp32 argument within rel |arg| of the exact one (slope <= 1)."""
    da = arg_abs * rel
    return da + 2 * T * (val_abs + da) + 2.0 ** -148


def timestep_embedding_check(out, t, what="timestep_embedding") -> Report:
    """freq = expf(c k / half) with c = -ln 1e4 rounded (3 roundings of the exponent a, expf 2 ulp), arg = t freq (u),
    cosf / sinf 2 ulp, bf16."""
    f64 = torch.float64
    dim = out.shape[1]
    half = dim // 2
    k = torch.arange(half, dtype=f64, device=out.device)
    a = -math.log(10000.0) * k / half
    arg = t.to(f64)[:, None] * torch.exp(a)[None]
    rel = torch.exp(3 * U * a.abs() * (1 + U)) * (1 + 2 * T) * (1 + U) - 1
    ref = torch.cat([torch.cos(arg), torch.sin(arg)], 1)
    err = _sincos_error(arg.abs().repeat(1, 2), rel.repeat(2)[None], ref.abs())
    return _plain_check(out, ref, err, what)


def position_features_check(out, feat, feat_mask, null_feat, coords, pos_mask, null_pos, freqs, what="position_features") -> Report:
    """[feat m + (1 - m) null | sin / cos(f_k coords) pm + (1 - pm) null_pos | 0]: f_k = powf(100, k / freqs) (exponent
    rounded: relative ln(100) (k / freqs) u; powf 4 ulp), a = f_k coord (u), sinf / cosf 2 ulp, the masked mix g(3)."""
    f64 = torch.float64
    B, N, nc = coords.shape
    if feat.dim() == 2:
        feat = feat.unsqueeze(0).expand(B, -1, -1)
    F_ = feat.shape[-1]
    fm, pm = feat_mask.to(f64).unsqueeze(-1), pos_mask.to(f64).unsqueeze(-1)
    fe, nfe, npe = feat.to(f64), null_feat.to(f64).view(1, 1, -1), null_pos.to(f64).view(1, 1, -1)
    cs = coords.to(f64)
    args, rels = [], []
    for k in range(freqs):
        y = k / freqs
        f = 100.0 ** y
        rel = math.exp(math.log(100.0) * y * U * (1 + U)) * (1 + 4 * T) * (1 + U) - 1
        args += [f * cs, f * cs]
        rels += [rel, rel]
    arg = torch.cat(args, -1)
    rel = torch.tensor([r for r in rels for _ in range(nc)], dtype=f64, device=cs.device)
    kinds = torch.tensor(([0] * nc + [1] * nc) * freqs, device=cs.device).bool()
    e = torch.where(kinds, torch.cos(arg), torch.sin(arg))
    de = _sincos_error(arg.abs(), rel, e.abs())
    pe = e * pm + (1 - pm) * npe
    epe = pm.abs() * de + g_n(3) * ((e * pm).abs() + ((1 - pm) * npe).abs())
    fv = fe * fm + (1 - fm) * nfe
    efv = g_n(3) * ((fe * fm).abs() + ((1 - fm) * nfe).abs())
    ldo = out.shape[-1]
    ref = torch.zeros(B * N, ldo, dtype=f64, device=cs.device)
    err = torch.zeros_like(ref)
    ref[:, :F_], ref[:, F_:F_ + pe.shape[-1]] = fv.reshape(B * N, -1), pe.reshape(B * N, -1)
    err[:, :F_], err[:, F_:F_ + pe.shape[-1]] = efv.reshape(B * N, -1), epe.reshape(B * N, -1)
    return _plain_check(out, ref, err, what)


def sampler_update_check(e_out, x_prev, x, e_cond, e_uncond, guidance, olds, coefs, a_t, a_prev, what="sampler_update") -> Report:
    """glg_sampler_update against float64 with the fp32 scalars the kernel receives (guidance, coefficients, and
    sqrtf(a_t), sqrtf(1 - a_t), ... formed in fp32 on the host): e = u + g (e_c - u): g(3) (|u| + |g| |e_c - u|);
    ep = sum c_i o_i: |c0| de + g(5) sum |c_i o_i|; pred = (x - s1 ep) / s0: (g(2) (|x| + |s1 ep|) + s1 dep) / s0 + u |pred|;
    x_prev = s2 pred + s3 ep: s2 dpred + s3 dep + g(3) (|s2 pred| + |s3 ep|)."""
    import numpy as np
    f64 = torch.float64
    f32 = np.float32
    g = float(f32(guidance))
    c = [float(f32(v)) for v in coefs]
    at, ap = f32(a_t), f32(a_prev)
    s0, s1 = float(np.sqrt(at)), float(np.sqrt(f32(1) - at))
    s2, s3 = float(np.sqrt(ap)), float(np.sqrt(f32(1) - ap))
    ec = e_cond.to(f64)
    if e_uncond is not None:
        eu = e_uncond.to(f64)
        e = eu + g * (ec - eu)
        de = g_n(3) * (eu.abs() + abs(g) * (ec - eu).abs())
    else:
        e, de = ec, torch.zeros_like(ec)
    ep = c[0] * e
    mag = (c[0] * e).abs()
    for ci, o in zip(c[1:], olds):
        ep = ep + ci * o.to(f64)
        mag = mag + (ci * o.to(f64)).abs()
    dep = abs(c[0]) * de + g_n(5) * mag
    xv = x.to(f64)
    pred = (xv - s1 * ep) / s0
    dnum = g_n(2) * (xv.abs() + (s1 * ep).abs()) + s1 * dep
    dpred = dnum / s0 + U * (pred.abs() + dnum / s0)
    xp = s2 * pred + s3 * ep
    dxp = s2 * dpred + s3 * dep + g_n(3) * ((s2 * pred).abs() + (s3 * ep).abs())
    rep = _plain_check(x_prev.reshape(xp.shape), xp, dxp, what + " x_prev")
    if e_out is not None:
        r2 = _plain_check(e_out.reshape(e.shape), e, de, what + " e")
        if r2.ratio > rep.ratio:
            rep = r2
    return rep


def clip_image_head_check(pooled, embeds, x, gamma, beta, w_proj, eps, what="clip_image_head") -> Report:
    """pooled = LayerNorm of each image's row 0 (one CTA: each thread adds ceil(C / 256) values, warp butterfly, 8 warp
    partials in order); embeds = pooled w_proj^T (per lane an FMA chain over C / 32 columns, butterfly 5):
    |W| e_pooled + g(C / 32 + 5) |pooled| |W|^T."""
    f64 = torch.float64
    C = x.shape[-1]
    x0 = x[:, 0]
    rep = layernorm_check(pooled, x0, gamma, beta, eps, what=what + " pooled", depth=-(-C // 256) + 13)
    xv = x0.to(f64)
    var, mu = torch.var_mean(xv, dim=1, correction=0, keepdim=True)
    y = (xv - mu) * torch.rsqrt(var + eps) * gamma.to(f64)[None] + beta.to(f64)[None]
    dy = (pooled.to(f64) - y).abs()                                   # within the pooled bound just checked
    W = w_proj.to(f64)
    ref = y @ W.t()
    err = dy @ W.abs().t() + g_n(-(-C // 32) + 5) * ((y.abs() + dy) @ W.abs().t())
    r2 = _plain_check(embeds, ref, err, what + " embeds")
    return max(rep, r2, key=lambda r: (not r.ok, r.ratio))


def dwconv7_ln_check(y, x, w, bias, gamma, beta, B, H, W, C, eps, what="dwconv7_ln") -> Report:
    """Depthwise 7x7 (pad 3) + bias as an fp32 FMA chain from the bias over <= 49 taps (g(49) (|bias| + sum |x||w|)), then
    the row LayerNorm bound with that as its input error (lanes add channel pairs: 2 ceil(C / 64) + 5 roundings)."""
    f64 = torch.float64
    F = torch.nn.functional
    xv = x.reshape(B, H, W, -1)[..., :C].permute(0, 3, 1, 2).to(f64)
    wk = w.to(f64).t().reshape(C, 1, 7, 7)
    h = F.conv2d(xv, wk, bias.to(f64), padding=3, groups=C).permute(0, 2, 3, 1).reshape(-1, C)
    S = F.conv2d(xv.abs(), wk.abs(), bias.to(f64).abs(), padding=3, groups=C).permute(0, 2, 3, 1).reshape(-1, C)
    yv = y.reshape(B * H * W, -1)[:, :C]
    return layernorm_check(yv, h, gamma, beta, eps, what=what, x_err=g_n(49) * S, depth=2 * (-(-C // 64)) + 5)


def clip_vision_embed_check(x, patch, cls, pos, gamma, beta, P, eps, what="clip_vision_embed") -> Report:
    """Rows LN(cls + pos[0]) and LN(patch + pos[1 + p]): the add is one fp32 rounding (u |a + p|), then the row LayerNorm."""
    f64 = torch.float64
    C = pos.shape[1]
    p = patch.reshape(-1, P, C).to(f64)
    t = torch.cat([cls.to(f64).view(1, 1, C).expand(p.shape[0], 1, C), p], 1) + pos.to(f64)[None]
    t = t.reshape(-1, C)
    return layernorm_check(x.reshape(-1, C), t, gamma, beta, eps, what=what, x_err=U * t.abs())
