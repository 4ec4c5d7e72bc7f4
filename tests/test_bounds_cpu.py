"""The rounding-level bounds of tests/bounds.py have teeth: on the CPU, a torch restatement of each kernel's documented
arithmetic passes its bound, and each realistic mutant of that arithmetic fails it.

GEMM restatement (gemm_tc.cu): fp32 accumulation over 64-wide K steps, fp32 epilogue (bias, row bias, residual), one
bf16 rounding.  Attention restatement (attention.cu): 64-key tiles in order, 16-row fragments whose rows r and r + 8
share a warp, online softmax with corr = exp2((m_old - m_new) c), P rounded to bf16 and l summed from the rounded P,
the last `poly` of every 8 score pairs exponentiated by ex2_poly3 restated in fp32."""
import math

import pytest
import torch

import bounds
from ref_ops import RefOps

F32, F64, BF = torch.float32, torch.float64, torch.bfloat16


def _fma32(a, b, c):
    """fp32 fma: one rounding of the exact a * b + c."""
    return (a.to(F64) * b.to(F64) + c.to(F64)).to(F32)


def ex2_poly3(x):
    """common.cuh ex2_poly3, op for op in fp32."""
    x = x.clamp_min(-125.0)
    t = x + 12582912.0
    f = x - (t - 12582912.0)
    p = _fma32(torch.full_like(f, 0.05550411), f, torch.full_like(f, 0.24022651))
    p = _fma32(p, f, torch.full_like(f, 0.69314718))
    p = _fma32(p, f, torch.ones_like(f))
    return p * torch.exp2(t - 12582912.0)


def ex2_poly3_doubled(x):
    """A cruder FMA-pipe exp2: twice ex2_poly3's relative error."""
    e = torch.exp2(x.to(F64))
    return (e * (1 + 2 * (ex2_poly3(x).to(F64) / e - 1))).to(F32)


# ---------------------------------------------------------------------------------------------------------------------
def gemm_restated(a, w, bias=None, rowbias=None, rpb=1, residual=None, mutant=None):
    K = a.shape[1]
    acc = torch.zeros(a.shape[0], w.shape[0], dtype=F32)
    for k in range(0, K, 64):
        if mutant == "drop_k" and k == 64:
            continue
        acc = acc + a[:, k:k + 64].float() @ w[:, k:k + 64].float().t()
    v = acc
    if bias is not None:
        v = v + (bias.roll(8) if mutant == "bias_shift" else bias)[None]
    if rowbias is not None:
        rows = torch.arange(a.shape[0])
        idx = (rows + 1) // rpb if mutant == "rowbias_off" else rows // rpb
        v = v + rowbias[idx.clamp_max(rowbias.shape[0] - 1)]
    if residual is not None:
        if mutant == "double_round":
            v = v.to(BF).float()
        v = v + residual.float()
    return v.to(BF)


@pytest.mark.parametrize("mutant", [None, "drop_k", "bias_shift", "rowbias_off", "double_round"])
def test_gemm_bound(mutant):
    g = torch.Generator().manual_seed(3)
    M, N, K, rpb = 256, 192, 320, 64
    a = torch.randn(M, K, generator=g).to(BF)
    w = (torch.randn(N, K, generator=g) * K ** -0.5).to(BF)
    bias = torch.randn(N, generator=g)
    rowbias = torch.randn(M // rpb, N, generator=g)
    res = (0.25 * torch.randn(M, N, generator=g)).to(BF)
    out = gemm_restated(a, w, bias, rowbias, rpb, res, mutant)
    rep = bounds.gemm_check(out, a, w, bias=bias, rowbias=rowbias, rows_per_batch=rpb, residual=res)
    print(rep)
    assert rep.ok == (mutant is None), str(rep)


def test_ref_ops_fp64_conv_matches_fp32():
    """RefOps(float64) states the 3x3 convolution as nine shifted GEMMs; it must be the same operation as F.conv2d."""
    g = torch.Generator().manual_seed(1)
    a = torch.randn(2, 6 * 5, 64, generator=g).to(BF)
    w = (torch.randn(9 * 16, 64, generator=g) * 0.05).to(BF)
    o32, o64 = torch.empty(60, 16), torch.empty(60, 16, dtype=F64)
    RefOps().gemm(a, w, o32, conv=(2, 6, 5))
    RefOps(compute_dtype=F64).gemm(a, w, o64, conv=(2, 6, 5))
    assert (o32.double() - o64).abs().max() < 1e-5


# ---------------------------------------------------------------------------------------------------------------------
def attn_restated(s, v, c, Lk, poly=0, mutant=None, exp_poly=ex2_poly3):
    """s [rows, Lk] fp32 scores (before the scale), v [Lk, dv] bf16 -> o [rows, dv] bf16.  Rows are taken 16 at a time
    (one warp's fragment: r and r + 8 share lanes)."""
    rows = s.shape[0]
    nkt = (Lk + 63) // 64
    sp = torch.zeros(rows, nkt * 64, dtype=F32)
    sp[:, :Lk] = s                                         # keys past Lk: zero-filled K rows -> score 0, V rows 0
    vp = torch.zeros(nkt * 64, v.shape[1], dtype=F32)
    vp[:Lk] = v.float()
    c32 = torch.tensor(c, dtype=F32)
    m = torch.full((rows,), -math.inf, dtype=F32)
    l = torch.zeros(rows, dtype=F32)
    o = torch.zeros(rows, v.shape[1], dtype=F32)
    keys = torch.arange(64)
    lane = keys // 8
    cut = Lk + 1 if mutant == "mask_under" else Lk - 1 if mutant == "mask_over" else Lk
    for kt in range(nkt - 1 if mutant == "drop_last_tile" else nkt):
        sc = sp[:, kt * 64:(kt + 1) * 64].clone()
        sc[:, kt * 64 + keys >= cut] = -math.inf
        mn = torch.maximum(m, sc.max(1).values)
        corr = torch.exp2((m - mn) * c32)
        if mutant == "corr_row8":
            corr = corr.view(-1, 2, 8)[:, [0, 0]].reshape(-1)   # row r's factor also on row r + 8
        m = mn
        ms = mn * c32
        x = _fma32(sc, c32.expand_as(sc), -ms[:, None].expand_as(sc))
        e = torch.where(lane[None] >= 8 - poly, exp_poly(x), torch.exp2(x))
        p = e.to(BF).float()
        l = (l if mutant == "l_not_rescaled" else l * corr) + p.sum(1)
        o = o * corr[:, None] + p @ vp[kt * 64:(kt + 1) * 64]
    return (o * (1.0 / l)[:, None]).to(BF)


def _check_attn(out, s, v, c, poly):
    return bounds.attention_check_scores(out[None], s.double()[None], v.double()[None], c, 0, poly=poly)


def _scores_row_tiles(rows, Lk, std, seed):
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(rows, Lk, generator=g) * std).float()


@pytest.mark.parametrize("std", [1.0, 4.0, 10.0, 30.0])
@pytest.mark.parametrize("poly", [0, 2])
def test_attention_faithful_passes(std, poly):
    rows, Lk, c = 32, 333, 0.7
    s = _scores_row_tiles(rows, Lk, std, 5)
    v = torch.randn(Lk, 24, generator=torch.Generator().manual_seed(6)).to(BF)
    rep = _check_attn(attn_restated(s, v, c, Lk, poly), s, v, c, poly)
    print(rep)
    assert rep.ok, str(rep)


def test_attention_mask_under_rejected():
    """All real logits strongly negative: a zero-filled key let through by the ragged mask takes the softmax."""
    rows, Lk, c = 16, 100, 0.5
    s = _scores_row_tiles(rows, Lk, 1.0, 7) - 40.0
    v = (torch.randn(Lk, 16, generator=torch.Generator().manual_seed(8)) + 1.0).to(BF)
    assert _check_attn(attn_restated(s, v, c, Lk), s, v, c, 0).ok
    rep = _check_attn(attn_restated(s, v, c, Lk, mutant="mask_under"), s, v, c, 0)
    assert not rep.ok, str(rep)


def test_attention_mask_over_rejected():
    """The argmax key is the last real key (in the ragged last tile): masking it moves the output by O(1)."""
    rows, Lk, c = 16, 100, 0.5
    s = _scores_row_tiles(rows, Lk, 1.0, 9)
    s[:, Lk - 1] = 20.0
    v = torch.randn(Lk, 16, generator=torch.Generator().manual_seed(10)).to(BF)
    assert _check_attn(attn_restated(s, v, c, Lk), s, v, c, 0).ok
    rep = _check_attn(attn_restated(s, v, c, Lk, mutant="mask_over"), s, v, c, 0)
    assert not rep.ok, str(rep)


@pytest.mark.parametrize("std,lift", [(1.0, 8.0), (10.0, 0.0)])
def test_attention_fuser_length_drop_last_tile_rejected(std, lift):
    """The fuser's key length at a 768^2 image: T = 9216 visual tokens + 30 grounding tokens, so the last 64-key tile
    holds only the 30 grounding keys.  The faithful restatement passes; one that stops before that ragged tile fails.
    With logits of std 1 the grounding keys score `lift` above the visual ones (5 % of the softmax mass): 30 keys of
    equal weight among 9246 move the output less than the P.V accumulation term of the bound."""
    rows, Lk, c = 16, 9216 + 30, 0.5
    s = _scores_row_tiles(rows, Lk, std, 13)
    s[:, 9216:] += lift
    v = torch.randn(Lk, 16, generator=torch.Generator().manual_seed(14)).to(BF)
    good = _check_attn(attn_restated(s, v, c, Lk), s, v, c, 0)
    assert good.ok, str(good)
    bad = _check_attn(attn_restated(s, v, c, Lk, mutant="drop_last_tile"), s, v, c, 0)
    print(good, bad)
    assert not bad.ok, str(bad)


@pytest.mark.parametrize("mutant", ["l_not_rescaled", "corr_row8"])
def test_attention_rescale_mutants_rejected(mutant):
    """Logits of std 10 whose level rises from tile to tile: corr is far from 1 and differs between rows."""
    rows, Lk, c = 32, 300, 0.7
    s = _scores_row_tiles(rows, Lk, 10.0, 11) + torch.arange(Lk).float()[None] * 0.05 * torch.arange(1, rows + 1).float()[:, None]
    v = torch.randn(Lk, 16, generator=torch.Generator().manual_seed(12)).to(BF)
    assert _check_attn(attn_restated(s, v, c, Lk), s, v, c, 0).ok
    rep = _check_attn(attn_restated(s, v, c, Lk, mutant=mutant), s, v, c, 0)
    assert not rep.ok, str(rep)


def test_attention_exp2_twice_the_error_rejected():
    """An FMA-pipe exp2 with twice ex2_poly3's error.  The rounding of P to bf16 absorbs small exp errors, so the rows are
    built where it cannot: key 0 is the max (v = 0); keys 1..31 (MUFU lanes) sit just above a bf16 rounding midpoint and
    round up by their full half ulp (v = -1); keys 32..63 (FMA-pipe lanes with poly = 4) sit a relative eta above a
    midpoint, eta between ex2_poly3's error there and twice it (v = +1).  The faithful kernel rounds them up, the mutant
    down: their error exceeds half an ulp plus the documented 7.9e-4 and the two groups' errors add."""
    c, poly, Lk = 1.0, 4, 64                              # scores in log2 units
    mid_a = 0.5 + 107 / 512                               # bf16 rounding midpoints of [0.5, 1)
    mid_b = 0.5 + 109 / 512
    xa = math.log2(mid_a * (1 + 1e-6))
    x0 = math.log2(mid_b * 1.0012)
    xt = torch.tensor([x0], dtype=F32)
    err_doubled = 1 - ex2_poly3_doubled(xt).double().item() / 2 ** xt.double().item()
    eta = 0.92 * err_doubled                              # faithful error ~ err_doubled / 2 < eta < err_doubled
    xb = math.log2(mid_b * (1 + eta))
    s = torch.zeros(1, Lk, dtype=F32)
    s[0, 1:32], s[0, 32:] = xa, xb
    v = torch.zeros(Lk, 8)
    v[1:32], v[32:] = -1.0, 1.0
    v = v.to(BF)
    assert err_doubled / 2 < eta < err_doubled and err_doubled / 2 <= bounds.EPS_EX2_POLY < eta
    good = _check_attn(attn_restated(s, v, c, Lk, poly), s, v, c, poly)
    assert good.ok, str(good)
    bad = _check_attn(attn_restated(s, v, c, Lk, poly, exp_poly=ex2_poly3_doubled), s, v, c, poly)
    print(good, bad)
    assert not bad.ok, str(bad)


# ---------------------------------------------------------------------------------------------------------------------
def _gemm_case(case):
    """(stored output, gemm_check kwargs, [rows, max(N, K)] columns) of one small GEMM of each epilogue family."""
    g = torch.Generator().manual_seed(len(case))
    B, H, Wd, K, N = 2, 5, 7, 64, 32
    M = B * H * Wd
    a = torch.randn(M, K, generator=g).to(BF)
    kw = dict(bias=torch.randn(N, generator=g))
    if case == "conv":
        w = (torch.randn(9 * N, K, generator=g) * (9 * K) ** -0.5).to(BF)
        kw.update(rowbias=torch.randn(B, N, generator=g), rows_per_batch=H * Wd, residual=torch.randn(M, N, generator=g).to(BF),
                  conv=(B, H, Wd))
    elif case == "geglu":
        w = (torch.randn(512, K, generator=g) * K ** -0.5).to(BF)
        kw.update(bias=torch.randn(512, generator=g), geglu=True)
    else:
        w = (torch.randn(N, K, generator=g) * K ** -0.5).to(BF)
        if case == "ln":
            kw.update(ln=(bounds.stats_restated(a), w.float().sum(1), 1e-5))
        elif case == "act":
            kw.update(act=1, gate=torch.tensor([0.7]), residual=torch.randn(M, N, generator=g).to(BF),
                      rowbias=torch.randn(7, N, generator=g), rows_per_batch=10)
    out = torch.empty(M, w.shape[0] // (9 if case == "conv" else 2 if case == "geglu" else 1), dtype=F32 if case == "fp32" else BF)
    o32 = torch.empty(out.shape)
    RefOps().gemm(a, w, o32, **kw)
    out.copy_(o32 + 0.01 * torch.randn(o32.shape, generator=g) * (o32.abs() > 1).float())   # a few elements off their bound
    return out, a, w, kw


def _same_report(a, b):
    """The same worst element and ratio, bit for bit; the aggregates are float64 sums over per-row partials and may
    differ in their last bits when a chunk is a single row (torch reduces one row in another order)."""
    assert (a.ratio, a.worst) == (b.ratio, b.worst)
    assert math.isclose(a.agg_ratio, b.agg_ratio, rel_tol=1e-13)
    assert a.extra.keys() == b.extra.keys() and all(math.isclose(a.extra[k], b.extra[k], rel_tol=1e-13) for k in a.extra)


@pytest.mark.parametrize("case", ["plain", "fp32", "conv", "ln", "geglu", "act"])
@pytest.mark.parametrize("max_elems", [1, 8 * 64 * 7 * 2, 8 * 64 * 13])
def test_gemm_check_chunked_equals_unchunked(case, max_elems):
    """Row chunks (one row, two image rows of a 3x3 convolution with their halo, 13 rows) report exactly what the
    whole-matrix evaluation reports: the worst element, its ratio and the aggregate."""
    out, a, w, kw = _gemm_case(case)
    whole = bounds.gemm_check(out, a, w, splits=8, **kw)
    chunked = bounds.gemm_check(out, a, w, splits=8, max_elems=max_elems, **kw)
    print(whole)
    _same_report(chunked, whole)
    assert not whole.ok                                                   # the perturbed elements are found either way


@pytest.mark.parametrize("max_elems", [1, 8 * 100 * 3])
def test_softmax_check_chunked_equals_unchunked(max_elems):
    import test_bounds_norm_cpu as N
    g = torch.Generator().manual_seed(4)
    s = torch.randn(21, 100, generator=g) * 8
    p = N.softmax_restated(s, 0.25)
    p[7, 3] = p[7, 3] * 1.1
    whole, chunked = bounds.softmax_check(p, s, 0.25), bounds.softmax_check(p, s, 0.25, max_elems=max_elems)
    print(whole)
    _same_report(chunked, whole)
    assert not whole.ok


@pytest.mark.parametrize("causal", [False, True])
def test_attention_check_row_chunks_equal_whole(causal):
    """Query-row chunks of one head (and the causal mask offset by the chunk's first row) report what one chunk does."""
    g = torch.Generator().manual_seed(5)
    B, heads, d, L = 1, 2, 16, 90
    q, k, v = (torch.randn(B, L, heads * d, generator=g).to(BF) for _ in range(3))
    out = torch.empty(B, L, heads * d, dtype=BF)
    RefOps().attention(q, k, v, out, heads, d, causal=causal)
    out[0, 50, 3] = out[0, 50, 3] + 0.05
    whole = bounds.attention_check(out, q, k, v, heads, d, causal=causal)
    chunked = bounds.attention_check(out, q, k, v, heads, d, causal=causal, max_elems=8 * L * 7)
    print(whole)
    assert (chunked.ratio, chunked.worst) == (whole.ratio, whole.worst)
    assert not whole.ok and "row 50 col 3 of slice 0" in whole.worst
