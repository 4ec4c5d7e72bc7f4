"""GEMM and attention kernels on inputs built so that bugs show.

Exact constructions (torch.equal): attention rows with one key ahead by a logit margin >= 30 must return that key's V
row bit for bit; GEMMs with one-hot A rows and 3x3 convolutions with isolated one-hot pixels must return the selected
weights; stats_out must equal a torch-fp32 restatement of its documented summation order on the kernel's own output.
Bounded constructions use the float64 bounds of tests/bounds.py: attention logits of std 1..30, strongly negative
logits, the argmax key in the ragged last tile, V with a common offset; LayerNorm fold at row mean / std up to 100."""
import math

import pytest
import torch

import bounds

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
BF = torch.bfloat16


@pytest.fixture(scope="module")
def ops():
    from gligen_b200.ops import CudaOps
    return CudaOps(DEV)


def gen(seed):
    return torch.Generator(device="cpu").manual_seed(seed)


class debug_modes:
    """Set the library's test hooks for one call and always restore the defaults."""

    def __init__(self, ops, attn=0, poly=0, bn=0, cta2=0, bres=0, splitk=0):
        self.ops, self.v = ops, (attn, poly, bn, cta2, bres, splitk)

    def __enter__(self):
        L = self.ops.lib
        attn, poly, bn, cta2, bres, splitk = self.v
        L.glg_debug_attn_mode(attn); L.glg_debug_attn_poly_share(poly); L.glg_debug_force_bn(bn)
        L.glg_debug_gemm_cta2(cta2); L.glg_debug_gemm_bres(bres); L.glg_debug_splitk(splitk)

    def __exit__(self, *a):
        L = self.ops.lib
        L.glg_debug_attn_mode(0); L.glg_debug_attn_poly_share(0); L.glg_debug_force_bn(0)
        L.glg_debug_gemm_cta2(0); L.glg_debug_gemm_bres(0); L.glg_debug_splitk(0)


# attention kernels: (glg_debug_attn_mode, FMA-pipe share): auto, streamed mma.sync, wgmma / TMA, short-key mma.sync
ATTN_KERNELS = {"auto": (0, 0), "mma_sync": (1, 0), "wgmma": (2, 0), "short_key": (3, 0),
                "wgmma_fma1": (2, 1), "wgmma_fma2": (2, 2), "mma_sync_fma1": (1, 1), "mma_sync_fma2": (1, 2)}


def kernels_for(Lk):
    return [k for k in ATTN_KERNELS if k != "short_key" or Lk <= 128]


def run_attention(ops, q, k, v, heads, d, kernel, causal=False):
    out = torch.zeros(q.shape[0], q.shape[1], heads * d, device=DEV, dtype=BF)
    with debug_modes(ops, *ATTN_KERNELS[kernel]):
        ops.attention(q, k, v, out, heads, d, causal=causal)
        torch.cuda.synchronize()
    return out


# ---- exact: one dominant key per query row --------------------------------------------------------------------------
def onehot_attention(B, heads, d, Lq, Lk, causal, seed):
    """Keys are distinct +-1 vectors; q_i = beta k_pi(i) with beta = ceil(15 sqrt(d)), so key pi(i) leads every other key
    by >= 2 beta / sqrt(d) >= 30 in scaled logits.  pi(i) runs through the first tile, keys 63 / 64 / 127 / 128, a middle
    tile and the ragged last tile."""
    g = gen(seed)
    nbits = min(d, 20)
    assert Lk <= 2 ** nbits
    beta = float(math.ceil(15 * math.sqrt(d)))
    K = torch.empty(B, Lk, heads, d)
    for b in range(B):
        for h in range(heads):
            codes = torch.randperm(2 ** nbits, generator=g)[:Lk]
            bits = (codes[:, None] >> torch.arange(nbits)[None]) & 1
            rest = torch.randint(0, 2, (Lk, d - nbits), generator=g)
            K[b, :, h] = torch.cat([bits, rest], 1).float() * 2 - 1
    special = [0, 63, 64, 127, 128, Lk // 2, ((Lk - 1) // 64) * 64, Lk - 1]
    special = [s for s in special if s < Lk]
    pi = torch.tensor([special[i % len(special)] if i % 3 else int(torch.randint(0, Lk, (1,), generator=g)) for i in range(Lq)])
    if causal:
        pi = torch.minimum(pi, torch.arange(Lq))
    Q = beta * K[:, pi]
    V = torch.randn(B, Lk, heads, d, generator=g)
    f = lambda t: t.reshape(t.shape[0], t.shape[1], heads * d).to(DEV, BF)
    Vb = f(V)
    return f(Q), f(K), Vb, Vb[:, pi]


EXACT_ATTN = [  # B, heads, d, Lq, Lk
    (1, 2, 8, 130, 250), (2, 2, 16, 200, 333), (1, 2, 32, 70, 77), (2, 3, 40, 200, 333), (1, 2, 40, 256, 4126),
    (1, 2, 64, 129, 128), (1, 2, 80, 100, 200), (1, 2, 96, 64, 65), (2, 2, 104, 150, 333), (1, 2, 128, 80, 129),
    (2, 2, 136, 150, 333), (1, 2, 136, 64, 100), (1, 2, 160, 100, 300), (1, 2, 104, 77, 77),
]


@pytest.mark.parametrize("B,heads,d,Lq,Lk", EXACT_ATTN)
def test_attention_dominant_key_exact(ops, B, heads, d, Lq, Lk):
    q, k, v, want = onehot_attention(B, heads, d, Lq, Lk, False, seed=d + Lk)
    for kernel in kernels_for(Lk):
        out = run_attention(ops, q, k, v, heads, d, kernel)
        bad = (out != want).any(-1)
        assert not bad.any(), f"{kernel} d={d} {Lq}x{Lk}: rows {bad.nonzero()[:8].tolist()} differ from V[pi(i)]"


@pytest.mark.parametrize("d", [40, 64, 104, 136])
def test_attention_dominant_key_exact_causal(ops, d):
    """The CLIP text encoder's causal 77-token attention (short-key kernel): pi(i) <= i."""
    q, k, v, want = onehot_attention(2, 2, d, 77, 77, True, seed=d)
    out = run_attention(ops, q, k, v, 2, d, "auto", causal=True)
    assert torch.equal(out, want)


# ---- bounded attention ----------------------------------------------------------------------------------------------
def attention_inputs(kind, B, heads, d, Lq, Lk, seed):
    g = gen(seed)
    if kind.startswith("std"):
        sd = math.sqrt(float(kind[3:]))                   # scaled logits q.k / sqrt(d) of std sd^2
        q = torch.randn(B, Lq, heads * d, generator=g) * sd
        k = torch.randn(B, Lk, heads * d, generator=g) * sd
        v = torch.randn(B, Lk, heads * d, generator=g)
    elif kind == "negative":                              # every real logit about -40: a leaked zero key would dominate
        u = torch.ones(heads * d) / math.sqrt(d)
        q = (torch.randn(B, Lq, heads * d, generator=g) * 0.2 + 6.0 * u)
        k = (torch.randn(B, Lk, heads * d, generator=g) * 0.2 - 6.6 * math.sqrt(d) * u / 1.0)
        v = torch.randn(B, Lk, heads * d, generator=g) + 0.5
    elif kind == "argmax_last":                           # the largest logit on the last key (ragged last tile)
        q = torch.randn(B, Lq, heads * d, generator=g) * 0.5 + 1.0
        k = torch.randn(B, Lk, heads * d, generator=g) * 0.5
        k[:, Lk - 1] = 2.0                                # its scaled logit ~ 2 sqrt(d), the others ~ N(0, 1.25)
        v = torch.randn(B, Lk, heads * d, generator=g)
    else:                                                 # "v_offset": V with a common offset
        q = torch.randn(B, Lq, heads * d, generator=g) * 2
        k = torch.randn(B, Lk, heads * d, generator=g)
        v = torch.randn(B, Lk, heads * d, generator=g) + 8.0
    return q.to(DEV, BF), k.to(DEV, BF), v.to(DEV, BF)


BOUNDED_ATTN = [(2, 4, 40, 300, 333), (1, 2, 104, 130, 200), (1, 2, 136, 96, 77), (1, 2, 64, 256, 1000), (1, 3, 160, 70, 128)]


@pytest.mark.parametrize("kind", ["std1", "std4", "std10", "std30", "negative", "argmax_last", "v_offset"])
@pytest.mark.parametrize("B,heads,d,Lq,Lk", BOUNDED_ATTN)
def test_attention_bounded(ops, kind, B, heads, d, Lq, Lk):
    q, k, v = attention_inputs(kind, B, heads, d, Lq, Lk, seed=Lk + d)
    for kernel in kernels_for(Lk):
        out = run_attention(ops, q, k, v, heads, d, kernel)
        poly = ATTN_KERNELS[kernel][1]
        rep = bounds.attention_check(out, q, k, v, heads, d, poly=poly, what=f"attention {kind} d={d} {Lq}x{Lk} {kernel}")
        assert rep.ok, str(rep)


def test_attention_bounded_causal(ops):
    q, k, v = attention_inputs("std10", 2, 2, 64, 77, 77, seed=3)
    out = run_attention(ops, q, k, v, 2, 64, "auto", causal=True)
    rep = bounds.attention_check(out, q, k, v, 2, 64, causal=True, what="causal attention")
    assert rep.ok, str(rep)


# ---- exact: one-hot GEMM and convolution ----------------------------------------------------------------------------
GEMM_MODES = {  # name -> debug_modes kwargs
    "bn64": dict(bn=64, cta2=1), "bn128": dict(bn=128, cta2=1), "bn160": dict(bn=160, cta2=1), "bn256": dict(bn=256, cta2=1),
    "pair128": dict(bn=128, cta2=2), "pair256": dict(bn=256, cta2=2), "resident": dict(cta2=1, bres=2),
    "splitk": dict(cta2=1, splitk=2),
}


@pytest.mark.parametrize("mode", list(GEMM_MODES))
def test_gemm_onehot_exact(ops, mode):
    """A row m is 2^(m % 3) e_sigma(m) with sigma spread over every K step: out[m] = 2^(m % 3) W[:, sigma(m)] exactly.
    Checks A / B addressing, the rotated K order, the slab reduction and the ragged last row block."""
    M, N, K = 300, 1280, 640
    sigma = (torch.arange(M) * 37 + 5) % K
    a = torch.zeros(M, K)
    a[torch.arange(M), sigma] = 2.0 ** (torch.arange(M) % 3).float()
    a = a.to(DEV, BF)
    w = torch.randn(N, K, generator=gen(1)).to(DEV, BF)
    out = torch.zeros(M, N, device=DEV, dtype=BF)
    with debug_modes(ops, **GEMM_MODES[mode]):
        ops.gemm(a, w, out)
        torch.cuda.synchronize()
    want = (w.t()[sigma.to(DEV)].float() * (2.0 ** (torch.arange(M, device=DEV) % 3).float())[:, None]).to(BF)
    assert torch.equal(out, want)


CONV_EXACT = [(2, 4, 128, 64, 128), (2, 2, 256, 64, 128), (1, 2, 512, 128, 64), (2, 8, 8, 128, 256), (3, 4, 4, 64, 128),
              (2, 16, 16, 64, 320)]


@pytest.mark.parametrize("B,H,W,Cin,Cout", CONV_EXACT)
@pytest.mark.parametrize("mode", ["single", "pair", "splitk"])
def test_conv_onehot_exact(ops, B, H, W, Cin, Cout, mode):
    """Isolated one-hot pixels on a 3-pixel grid (origin per image, so borders and the 128-pixel segment edges of wide
    rows are hit): every output pixel sees at most one non-zero input, so out = the selected tap weight exactly."""
    x = torch.zeros(B, H, W, Cin)
    for b in range(B):
        for y in range(b % 3, H, 3):
            for xx in range((b + 1) % 3, W, 3):
                x[b, y, xx, (y * 7 + xx * 13) % Cin] = 1.0
    a = x.reshape(B, H * W, Cin).to(DEV, BF)
    w = (torch.randn(9 * Cout, Cin, generator=gen(2))).to(DEV, BF)
    out = torch.zeros(B, H * W, Cout, device=DEV, dtype=BF)
    kw = {"single": dict(cta2=1), "pair": dict(cta2=2), "splitk": dict(cta2=1, splitk=2)}[mode]
    with debug_modes(ops, **kw):
        ops.gemm(a, w, out, conv=(B, H, W))
        torch.cuda.synchronize()
    from ref_ops import RefOps
    ref = torch.empty(B, H * W, Cout, device=DEV, dtype=torch.float64)
    RefOps(DEV, compute_dtype=torch.float64).gemm(a, w, ref, conv=(B, H, W))
    assert torch.equal(out, ref.to(BF)), f"{(out.float() != ref.to(BF).float()).sum().item()} outputs differ"


# ---- exact: stats_out summation order -------------------------------------------------------------------------------
STATS_CASES = [  # M, N, K, flags
    (300, 1280, 320, dict()), (77, 640, 768, dict(gate=True)), (512, 960, 320, dict(gate=True, residual=True)),
    (1000, 640, 640, dict(residual=True, slot_view=True)), (64, 320, 640, dict(residual=True, gate=True, slot_view=True)),
]


@pytest.mark.parametrize("M,N,K,fl", STATS_CASES)
@pytest.mark.parametrize("mode", ["bn64", "bn128", "bn160", "bn256", "pair128", "pair256", "resident", "auto"])
def test_stats_out_order_exact(ops, M, N, K, fl, mode):
    kw = GEMM_MODES.get(mode, {})
    if kw.get("bn") and N % kw["bn"]:
        pytest.skip("tile width does not divide N")
    g = gen(M + N)
    a = torch.randn(M, K, generator=g).to(DEV, BF)
    w = (torch.randn(N, K, generator=g) * K ** -0.5).to(DEV, BF)
    gate = torch.tensor([0.61], device=DEV) if fl.get("gate") else None
    res = (torch.randn(M, N, generator=g) * 2 + 0.7).to(DEV, BF) if fl.get("residual") else None
    out = torch.zeros(M, N, device=DEV, dtype=BF)
    if fl.get("slot_view"):
        big = torch.full((N // 32, M + 40, 2), 7.0, device=DEV)
        st = big[:, 10:10 + M]
    else:
        st = torch.full((N // 32, M, 2), 7.0, device=DEV)
    with debug_modes(ops, **kw):
        ops.gemm(a, w, out, gate=gate, residual=res, stats_out=st)
        torch.cuda.synchronize()
    assert torch.equal(st, bounds.stats_restated(out)), f"max diff {(st - bounds.stats_restated(out)).abs().max().item()}"
    if fl.get("slot_view"):
        assert (big[:, :10] == 7.0).all() and (big[:, 10 + M:] == 7.0).all(), "wrote outside the slot-strided view"
    rep = bounds.gemm_check(out, a, w, gate=gate, residual=res, what=f"stats producer {M}x{N}x{K} {mode}")
    assert rep.ok, str(rep)


# ---- LayerNorm fold at large row means -------------------------------------------------------------------------------
def ln_fold_inputs(M, K, N, ratio, seed):
    g = gen(seed)
    mean = ratio * (1 + 0.3 * torch.rand(M, 1, generator=g)) * torch.where(torch.rand(M, 1, generator=g) < 0.5, -1.0, 1.0)
    x = (torch.randn(M, K, generator=g) + mean).to(BF)
    xd = x.double()
    parts = xd.view(M, K // 32, 32)
    st = torch.stack([parts.sum(-1), (parts * parts).sum(-1)], -1).permute(1, 0, 2).float().contiguous()
    gamma = 1 + 0.2 * torch.randn(K, generator=g)
    wf = (torch.randn(N, K, generator=g) * K ** -0.5 * gamma[None]).to(BF)
    colsum = wf.double().sum(1).float()
    bias = torch.randn(N, generator=g)
    return x.to(DEV), st.to(DEV), wf.to(DEV), colsum.to(DEV), bias.to(DEV)


@pytest.mark.parametrize("ratio", [0.0, 10.0, 30.0, 100.0])
@pytest.mark.parametrize("mode", ["bn128", "pair256", "resident"])
def test_ln_fold_large_mean(ops, ratio, mode):
    """Rows of mean / std up to 100 (post-residual streams): the fold's fp32 E[x^2] - E[x]^2 against the float64
    LayerNorm of the same bf16 rows (statistics: exact per-slot sums, rounded once to fp32), within the statistics
    error derived in tests/bounds.py."""
    M, K, N = 512, 640, 1280
    x, st, wf, colsum, bias = ln_fold_inputs(M, K, N, ratio, seed=int(ratio) + 1)
    out = torch.zeros(M, N, device=DEV, dtype=BF)
    with debug_modes(ops, **GEMM_MODES[mode]):
        ops.gemm(x, wf, out, bias=bias, ln=(st, colsum, 1e-5))
        torch.cuda.synchronize()
    rep = bounds.gemm_check(out, x, wf, bias=bias, ln=(st, colsum, 1e-5), what=f"ln fold mean/std={ratio} {mode}")
    print(rep)
    assert rep.ok, str(rep)


def test_ln_fold_slot_strided_into_batch_strided_output(ops):
    """The fuser's grounding rows: statistics are a row range ostat[:, lo:hi] of a larger tensor (slot stride != M) and
    the output is a batch-strided [B, T, :] view of a [B, T + G, 3C] buffer."""
    B, T, G, K, N = 2, 128, 30, 320, 960
    x, st, wf, colsum, bias = ln_fold_inputs(B * T, K, N, 10.0, seed=5)
    big_st = torch.full((K // 32, B * T + 70, 2), 7.0, device=DEV)
    big_st[:, 40:40 + B * T] = st
    view = big_st[:, 40:40 + B * T]
    big = torch.zeros(B, T + G, N, device=DEV, dtype=BF)
    ops.gemm(x, wf, big[:, :T], bias=bias, ln=(view, colsum, 1e-5))
    torch.cuda.synchronize()
    assert big[:, T:].abs().max().item() == 0, "wrote outside the batch-strided view"
    rep = bounds.gemm_check(big[:, :T].reshape(B * T, N), x, wf, bias=bias, ln=(st, colsum, 1e-5), what="slot-strided ln fold")
    assert rep.ok, str(rep)


# ---- real call shapes the kernel suite did not reach ----------------------------------------------------------------
def test_vae_attention_gemms(ops):
    """The VAE mid-block attention at 64 x 64 latents (vae.py:110-120): W_v as the A operand (V^T = W_v hn^T), the fp32
    T x T score matrix, and P.V with K = T = 4096."""
    T, C = 4096, 512
    g = gen(7)
    hn = torch.randn(T, C, generator=g).to(DEV, BF)
    wv = (torch.randn(C, C, generator=g) * C ** -0.5).to(DEV, BF)
    q = torch.randn(T, C, generator=g).to(DEV, BF)
    k = torch.randn(T, C, generator=g).to(DEV, BF)
    vt = torch.zeros(C, T, device=DEV, dtype=BF)
    s = torch.zeros(T, T, device=DEV)
    ops.gemm(wv, hn, vt)
    ops.gemm(q, k, s)
    torch.cuda.synchronize()
    for rep in (bounds.gemm_check(vt, wv, hn, what="V^T = W_v hn^T"), bounds.gemm_check(s, q, k, what="S = Q K^T fp32")):
        assert rep.ok, str(rep)
    p = torch.softmax(torch.randn(T, T, generator=g) * 3, -1).to(DEV, BF)
    bv = torch.randn(C, generator=g).to(DEV)
    o = torch.zeros(T, C, device=DEV, dtype=BF)
    ops.gemm(p, vt, o, bias=bv)
    torch.cuda.synchronize()
    rep = bounds.gemm_check(o, p, vt, bias=bv, what="O = P V + b (K = 4096)")
    assert rep.ok, str(rep)


@pytest.mark.parametrize("B,H,W,Cin,Cout", [(2, 8, 8, 1280, 1280), (4, 16, 16, 1280, 1280), (2, 8, 8, 2560, 1280)])
def test_split_k_conv_with_time_rowbias(ops, B, H, W, Cin, Cout):
    """The UNet's small-image 3x3 convolutions carry the time-embedding row bias (one row per image) and take split-K
    when the tile grid leaves SMs idle."""
    g = gen(B * H + Cin)
    a = torch.randn(B, H * W, Cin, generator=g).to(DEV, BF)
    w = (torch.randn(9 * Cout, Cin, generator=g) * (9 * Cin) ** -0.5).to(DEV, BF)
    bias = torch.randn(Cout, generator=g).to(DEV)
    rowbias = torch.randn(B, Cout, generator=g).to(DEV)
    res = torch.randn(B, H * W, Cout, generator=g).to(DEV, BF)
    for splitk in (0, 2):
        out = torch.zeros(B, H * W, Cout, device=DEV, dtype=BF)
        with debug_modes(ops, splitk=splitk):
            ops.gemm(a, w, out, bias=bias, rowbias=rowbias, rows_per_batch=H * W, residual=res, conv=(B, H, W))
            torch.cuda.synchronize()
        rep = bounds.gemm_check(out, a, w, bias=bias, rowbias=rowbias, rows_per_batch=H * W, residual=res, conv=(B, H, W),
                                splits=8, what=f"conv {B}x{H}x{W} {Cin}->{Cout} splitk={splitk}")
        assert rep.ok, str(rep)


@pytest.mark.parametrize("B,H,W,C", [(1, 4, 256, 128), (1, 2, 512, 128), (1, 8, 128, 256)])
def test_wide_conv_bounded(ops, B, H, W, C):
    """VAE decoder widths: a 128-row block is a segment of one image row (x0 != 0 for W > 128)."""
    g = gen(W + C)
    a = torch.randn(B, H * W, C, generator=g).to(DEV, BF)
    w = (torch.randn(9 * C, C, generator=g) * (9 * C) ** -0.5).to(DEV, BF)
    bias = torch.randn(C, generator=g).to(DEV)
    res = torch.randn(B, H * W, C, generator=g).to(DEV, BF)
    out = torch.zeros(B, H * W, C, device=DEV, dtype=BF)
    ops.gemm(a, w, out, bias=bias, residual=res, conv=(B, H, W))
    torch.cuda.synchronize()
    rep = bounds.gemm_check(out, a, w, bias=bias, residual=res, conv=(B, H, W), what=f"wide conv W={W}")
    assert rep.ok, str(rep)


@pytest.mark.parametrize("act,geglu", [(1, False), (2, False), (3, False), (0, True)])
def test_gemm_epilogues_bounded(ops, act, geglu):
    M, N, K = 700, 1280 if not geglu else 2560, 640
    g = gen(act + 10 * geglu)
    a = torch.randn(M, K, generator=g).to(DEV, BF)
    w = (torch.randn(N, K, generator=g) * K ** -0.5).to(DEV, BF)
    bias = torch.randn(N, generator=g).to(DEV)
    out = torch.zeros(M, N // 2 if geglu else N, device=DEV, dtype=BF)
    ops.gemm(a, w, out, bias=bias, act=act, geglu=geglu)
    torch.cuda.synchronize()
    rep = bounds.gemm_check(out, a, w, bias=bias, act=act, geglu=geglu, what=f"epilogue act={act} geglu={geglu}")
    assert rep.ok, str(rep)
