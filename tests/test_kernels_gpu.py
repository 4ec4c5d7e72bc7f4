"""Per-kernel parity on the GPU: every CudaOps method (C-ABI call into libgligen_b200.so) against the
same-named torch-fp32 statement in tests/ref_ops.py, on identical bf16-rounded inputs.

Tolerances (floating point): outputs are bf16, accumulation fp32 -> rel-L2 <= 6e-3, max-abs <= 3% of max|ref|
(attention: P is rounded to bf16 before PV, rel-L2 <= 1e-2)."""
import pytest
import torch

from conftest import assert_close
from ref_ops import RefOps
from gligen_b200.ops import gn_scratch_floats

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ops():
    from gligen_b200.ops import CudaOps
    return CudaOps("cuda:0")


@pytest.fixture(scope="module")
def ref():
    return RefOps("cuda:0", torch.float32)


def rnd(*shape, scale=1.0, seed=0, dtype=torch.bfloat16):
    g = torch.Generator(device="cpu").manual_seed(seed + sum(shape))
    return (torch.randn(*shape, generator=g) * scale).to("cuda:0").to(dtype)


GEMM_CASES = [
    # M, N, K, flags
    (256, 320, 320, dict()),
    (1000, 640, 768, dict(bias=True)),
    (300, 1280, 1280, dict(bias=True, residual=True, gate=True)),
    (4, 5120, 1280, dict(bias=True, fp32=True)),
    (2 * 77, 640, 768, dict()),
    (512, 1920, 640, dict(bias=True, act=True)),
    (16384, 960, 320, dict()),
    (4096, 320, 1280, dict(bias=True, residual=True, strided=True)),
    (4096, 2560, 320, dict(geglu=True)),
    (700, 1024, 256, dict(geglu=True)),
    (512, 640, 320, dict(bias=True, rowbias=128)),
]


@pytest.mark.parametrize("M,N,K,fl", GEMM_CASES)
@pytest.mark.parametrize("force_bn", [0, 64, 128, 160, 256])
@pytest.mark.parametrize("cta2", [0, 1, 2])
def test_gemm(ops, ref, M, N, K, fl, force_bn, cta2):
    """cta2: 0 = tile heuristic, 1 = single-CTA kernel, 2 = paired kernel (cluster of 2, B tile multicast to both CTAs)."""
    if force_bn and (N % force_bn or fl.get("geglu")):
        pytest.skip("BN does not divide N")
    if force_bn and M > 5000:
        pytest.skip("large case only with the heuristic tile")
    if cta2 == 2 and (force_bn == 64 or M <= 128):
        pytest.skip("pairs need BN >= 128 and M > 128")
    if cta2 == 0 and force_bn:
        pytest.skip("forced tiles are covered by the explicit modes")
    a = rnd(M, K)
    w = rnd(N, K, scale=K ** -0.5, seed=1)
    geglu = fl.get("geglu", False)
    No = N // 2 if geglu else N
    bias = rnd(N, seed=2, dtype=torch.float32) if (fl.get("bias") or geglu) else None
    gate = torch.tensor([0.37], device="cuda:0") if fl.get("gate") else None
    rows_per_batch = fl.get("rowbias", 0)
    rowbias = rnd(M // rows_per_batch, N, seed=3, dtype=torch.float32) if rows_per_batch else None
    odt = torch.float32 if fl.get("fp32") else torch.bfloat16
    if fl.get("strided"):
        big = torch.zeros(M, No + 64, device="cuda:0", dtype=odt)
        out, out_r = big[:, 64:], torch.zeros(M, No, device="cuda:0", dtype=odt)
        resb = rnd(M, No + 128, seed=4)
        residual = resb[:, 128:]
    else:
        out, out_r = torch.zeros(M, No, device="cuda:0", dtype=odt), torch.zeros(M, No, device="cuda:0", dtype=odt)
        residual = rnd(M, No, seed=4) if fl.get("residual") else None
    kw = dict(bias=bias, rowbias=rowbias, rows_per_batch=max(rows_per_batch, 1), act=1 if fl.get("act") else 0,
              gate=gate, residual=residual, geglu=geglu)
    ops.lib.glg_debug_force_bn(force_bn)
    ops.lib.glg_debug_gemm_cta2(cta2)
    try:
        ops.gemm(a, w, out, **kw)
        torch.cuda.synchronize()
    finally:
        ops.lib.glg_debug_force_bn(0)
        ops.lib.glg_debug_gemm_cta2(0)
    ref.gemm(a, w, out_r, **kw)
    assert_close(out, out_r, what=f"gemm {M}x{N}x{K} {fl} bn={force_bn} cta2={cta2}")
    if fl.get("strided"):
        assert big[:, :64].abs().max().item() == 0.0, "wrote outside the output slice"


@pytest.mark.parametrize("M,N,K,fl", GEMM_CASES + [(32768, 320, 320, dict(bias=True, residual=True)), (9000, 1920, 640, dict(bias=True)),
                                                   (20000, 2560, 320, dict(geglu=True)), (130, 320, 320, dict(bias=True))])
@pytest.mark.parametrize("force_bn", [0, 64, 128, 160, 256])
def test_gemm_weights_resident(ops, ref, M, N, K, fl, force_bn):
    """B-resident mode forced wherever the weight tile fits in shared memory (one n-tile per CTA for its lifetime, the
    weight tile loaded once, only A streams): same results as the torch statement, incl. CTAs that own no m-block."""
    if force_bn and (N % force_bn or fl.get("geglu")):
        pytest.skip("BN does not divide N")
    if fl.get("fp32") or fl.get("strided") or fl.get("rowbias"):
        pytest.skip("covered by the streaming-mode test (same epilogue code)")
    import ctypes as C
    pick = (C.c_int32 * 3)()
    ops.lib.glg_debug_force_bn(force_bn)
    ops.lib.glg_debug_gemm_cta2(1)
    ops.lib.glg_debug_gemm_bres(2)
    try:
        ops.lib.glg_debug_pick_tile(M, N, K, 1 if fl.get("geglu") else 0, 0, 0, 0, pick)
        if not (pick[1] >> 8):
            pytest.skip("weight tile does not fit beside three A stages")
        a = rnd(M, K)
        w = rnd(N, K, scale=K ** -0.5, seed=1)
        geglu = fl.get("geglu", False)
        No = N // 2 if geglu else N
        bias = rnd(N, seed=2, dtype=torch.float32) if (fl.get("bias") or geglu) else None
        gate = torch.tensor([0.37], device="cuda:0") if fl.get("gate") else None
        residual = rnd(M, No, seed=4) if fl.get("residual") else None
        out, out_r = torch.zeros(M, No, device="cuda:0", dtype=torch.bfloat16), torch.zeros(M, No, device="cuda:0", dtype=torch.bfloat16)
        kw = dict(bias=bias, act=1 if fl.get("act") else 0, gate=gate, residual=residual, geglu=geglu)
        ops.gemm(a, w, out, **kw)
        torch.cuda.synchronize()
        out2 = torch.zeros_like(out)
        ops.gemm(a, w, out2, **kw)
        torch.cuda.synchronize()
    finally:
        ops.lib.glg_debug_force_bn(0)
        ops.lib.glg_debug_gemm_cta2(0)
        ops.lib.glg_debug_gemm_bres(0)
    ref.gemm(a, w, out_r, **kw)
    assert_close(out, out_r, what=f"B-resident gemm {M}x{N}x{K} {fl} bn={force_bn}")
    assert torch.equal(out, out2)


@pytest.mark.parametrize("M,N,K,geglu", [(4096, 960, 320, False), (1000, 1920, 640, False), (300, 1280, 1280, False),
                                         (4096, 2560, 320, True), (520, 1024, 128, True)])
@pytest.mark.parametrize("cta2,bres", [(1, 1), (2, 1), (1, 2)])
def test_gemm_layernorm_fold(ops, ref, M, N, K, geglu, cta2, bres):
    """bres: 1 = streaming tiles only, 2 = weights-resident tiles wherever they fit."""
    ops.lib.glg_debug_gemm_cta2(cta2)
    ops.lib.glg_debug_gemm_bres(bres)
    try:
        _ln_fold_case(ops, ref, M, N, K, geglu)
    finally:
        ops.lib.glg_debug_gemm_cta2(0)
        ops.lib.glg_debug_gemm_bres(0)


def _ln_fold_case(ops, ref, M, N, K, geglu):
    """producer GEMM (stats_out) -> consumer GEMM (ln fold) == explicit LayerNorm followed by the GEMM."""
    import torch.nn.functional as F
    a0 = rnd(M, 64)
    w0 = rnd(K, 64, scale=0.3, seed=1)
    res = rnd(M, K, seed=2) * 2 + 0.7                      # non-zero row means: exercises the mu * colsum cancellation
    x = torch.zeros(M, K, device="cuda:0", dtype=torch.bfloat16)
    slots = K // 32
    st = torch.full((slots, M, 2), 7.0, device="cuda:0")   # slot-major; poisoned: every slot must be written by the kernel
    ops.gemm(a0, w0, x, residual=res, stats_out=st)
    torch.cuda.synchronize()
    xf = x.float()
    assert_close(st[:, :, 0].sum(0), xf.sum(1), rel=1e-5, max_rel=1e-4, what="row sums")
    assert_close(st[:, :, 1].sum(0), (xf * xf).sum(1), rel=1e-5, max_rel=1e-4, what="row sums of squares")
    gamma = 1 + 0.2 * rnd(K, seed=3, dtype=torch.float32)
    beta = 0.2 * rnd(K, seed=4, dtype=torch.float32)
    w = rnd(N, K, scale=K ** -0.5, seed=5, dtype=torch.float32)
    bias = rnd(N, seed=6, dtype=torch.float32)
    wf = (w * gamma[None]).to(torch.bfloat16)
    colsum = wf.float().sum(1)
    bfold = bias + w @ beta
    No = N // 2 if geglu else N
    out = torch.zeros(M, No, device="cuda:0", dtype=torch.bfloat16)
    ops.gemm(x, wf, out, bias=bfold, geglu=geglu, ln=(st, colsum, 1e-5))
    torch.cuda.synchronize()
    y = F.linear(F.layer_norm(xf, (K,), gamma, beta, 1e-5), w, bias)
    if geglu:
        t = y.view(M, N // 256, 2, 128)
        y = (t[:, :, 0] * F.gelu(t[:, :, 1])).reshape(M, No)
    assert_close(out, y, what=f"ln-fold gemm {M}x{N}x{K} geglu={geglu}")


@pytest.mark.parametrize("M,N,K,conv", [(512, 1280, 1280, None), (512, 1280, 5120, None), (200, 640, 2560, None),
                                         (512, 1280, 1280, (8, 8, 8)), (128, 1280, 2560, (2, 8, 8)), (512, 256, 256, (8, 8, 8))])
def test_gemm_split_k(ops, ref, M, N, K, conv):
    """forced split-K (fp32 slabs + fixed-order reduce) against the unsplit statement; twice -> bit-reproducible."""
    a = rnd(conv[0], conv[1] * conv[2], K) if conv else rnd(M, K)
    w = rnd((9 if conv else 1) * N, K, scale=((9 if conv else 1) * K) ** -0.5, seed=1)
    bias = rnd(N, seed=2, dtype=torch.float32)
    res = rnd(M, N, seed=3)
    rowbias = rnd(M // 64, N, seed=4, dtype=torch.float32) if M % 64 == 0 else None
    outs = []
    ops.lib.glg_debug_splitk(2)
    try:
        for _ in range(2):
            out = torch.zeros(M, N, device="cuda:0", dtype=torch.bfloat16)
            ops.gemm(a, w, out, bias=bias, rowbias=rowbias, rows_per_batch=64, residual=res, conv=conv)
            torch.cuda.synchronize()
            outs.append(out)
    finally:
        ops.lib.glg_debug_splitk(0)
    out_r = torch.zeros(M, N, device="cuda:0", dtype=torch.bfloat16)
    ref.gemm(a, w, out_r, bias=bias, rowbias=rowbias, rows_per_batch=64, residual=res, conv=conv)
    assert_close(outs[0], out_r, what=f"split-K gemm {M}x{N}x{K} conv={conv}")
    assert torch.equal(outs[0], outs[1])


def test_gemm_batch_strided_output(ops, ref):
    B, T, G, C = 3, 200, 30, 320
    a = rnd(B * T, C)
    w = rnd(3 * C, C, scale=C ** -0.5, seed=1)
    big = torch.zeros(B, T + G, 3 * C, device="cuda:0", dtype=torch.bfloat16)
    big_r = torch.zeros_like(big)
    ops.gemm(a, w, big[:, :T])
    torch.cuda.synchronize()
    ref.gemm(a, w, big_r[:, :T])
    assert_close(big, big_r, what="batch-strided gemm")
    assert big[:, T:].abs().max().item() == 0


CONV_CASES = [
    # B, H, W, Cin, Cout, flags
    (2, 64, 64, 320, 320, dict(rowbias=True)),
    (2, 32, 32, 640, 1280, dict(residual=True)),
    (1, 16, 16, 2560, 1280, dict()),
    (3, 8, 8, 1280, 1280, dict(rowbias=True, residual=True)),
    (1, 8, 8, 1280, 1280, dict()),
    (2, 16, 16, 64, 64, dict()),
    (2, 2, 2, 256, 256, dict(residual=True)),
    (2, 4, 4, 128, 256, dict()),
    (2, 64, 64, 320, 320, dict(strided=True)),
]


@pytest.mark.parametrize("B,H,W,Cin,Cout,fl", CONV_CASES)
@pytest.mark.parametrize("cta2", [1, 2])
def test_conv3x3(ops, ref, B, H, W, Cin, Cout, fl, cta2):
    if cta2 == 2 and (B * H * W <= 128 or Cout % 128):
        pytest.skip("pairs need M > 128 and Cout % 128 == 0")
    ops.lib.glg_debug_gemm_cta2(cta2)
    try:
        _conv_case(ops, ref, B, H, W, Cin, Cout, fl)
    finally:
        ops.lib.glg_debug_gemm_cta2(0)


def _conv_case(ops, ref, B, H, W, Cin, Cout, fl):
    if fl.get("strided"):
        big = rnd(B, H * W, Cin + 192)
        a = big[:, :, 64:64 + Cin]
    else:
        a = rnd(B, H * W, Cin)
    w = rnd(9 * Cout, Cin, scale=(9 * Cin) ** -0.5, seed=1)
    bias = rnd(Cout, seed=2, dtype=torch.float32)
    rowbias = rnd(B, Cout, seed=3, dtype=torch.float32) if fl.get("rowbias") else None
    residual = rnd(B, H * W, Cout, seed=4) if fl.get("residual") else None
    out = torch.zeros(B, H * W, Cout, device="cuda:0", dtype=torch.bfloat16)
    out_r = torch.zeros_like(out)
    kw = dict(bias=bias, rowbias=rowbias, rows_per_batch=H * W, residual=residual, conv=(B, H, W))
    ops.gemm(a, w, out, **kw)
    torch.cuda.synchronize()
    ref.gemm(a, w, out_r, **kw)
    assert_close(out, out_r, what=f"conv {B}x{H}x{W} {Cin}->{Cout} {fl}")


ATTN_CASES = [
    # B, heads, d, Lq, Lk, packed
    (1, 8, 40, 4096, 4096, "qkv"),
    (2, 8, 40, 1024, 1054, "fuser"),
    (2, 8, 80, 1024, 1084, "fuser"),
    (2, 8, 160, 256, 286, "fuser"),
    (3, 8, 160, 64, 94, "fuser"),
    (2, 8, 40, 4096, 77, "kv"),
    (2, 8, 80, 1024, 77, "kv"),
    (2, 8, 160, 64, 77, "kv"),
    (2, 8, 8, 256, 262, "fuser"),
    (2, 8, 16, 64, 70, "fuser"),
    (2, 8, 32, 16, 22, "fuser"),
    (2, 4, 64, 200, 333, "plain"),
    (1, 2, 40, 128, 64, "plain"),
    (1, 2, 40, 128, 8192, "plain"),
    (8, 8, 40, 4096, 4126, "fuser"),
    (2, 8, 80, 1024, 1024, "qkv"),
    (1, 4, 96, 300, 555, "plain"),
    (1, 4, 128, 256, 200, "plain"),
    (1, 4, 72, 128, 130, "plain"),
    (2, 8, 40, 1000, 128, "kv"),          # short-key kernel: ragged last query tile of a 4-tile CTA, two full K tiles
    (2, 8, 80, 257, 1, "kv"),
    (1, 8, 160, 320, 65, "kv"),
    (2, 8, 40, 300, 257, "plain"),         # ragged query tile, 5 key tiles (last: 1 key)
    (1, 8, 24, 512, 1000, "plain"),
    (1, 4, 64, 257, 384, "plain"),
    (2, 8, 40, 200, 64, "plain"),          # one key tile: the second softmax warpgroup of the two-warpgroup kernel sees none
    (1, 8, 40, 384, 129, "plain"),         # three key tiles (2 + 1), last one a single key
    (1, 4, 56, 130, 640, "plain"),
]


# path -> (glg_debug_attn_mode, FMA-pipe exp2 share of 8).  The path names are those of the kernels of the
# project's Blackwell build; each selects one H100 configuration: 0 = auto dispatch, 1 = streamed mma.sync kernel,
# 2 = wgmma / TMA kernel, 3 = short-key mma.sync kernel.
ATTN_PATHS = {"auto": (0, 0), "mma_sync": (1, 0), "tcgen05": (2, 0), "tcgen05_sum": (2, 1), "short_tc": (3, 0), "tc2": (2, 2), "tc3": (1, 2)}


@pytest.mark.parametrize("B,heads,d,Lq,Lk,mode", ATTN_CASES)
@pytest.mark.parametrize("path", ["auto", "mma_sync", "tcgen05", "tcgen05_sum", "short_tc", "tc2", "tc3"])
def test_attention(ops, ref, B, heads, d, Lq, Lk, mode, path):
    """auto: the short-key mma.sync kernel (K/V resident, <= 128 keys: the text context) or the wgmma / TMA flash kernel
    (longer key sets).  The other paths force one kernel for every case it accepts (ATTN_PATHS): the streamed mma.sync
    kernel, the wgmma kernel (also for short key sets), the short-key kernel (Lk <= 128 only); tcgen05_sum / tc2 / tc3 run
    the wgmma or streamed kernel with 1 or 2 of every 8 score pairs exponentiated on the FMA pipe."""
    if path == "short_tc" and Lk > 128:
        pytest.skip("short-key kernel: all keys in at most two resident tiles")
    C = heads * d
    if mode == "qkv":
        qkv = rnd(B, Lk, 3 * C)
        q, k, v = qkv[:, :, :C], qkv[:, :, C:2 * C], qkv[:, :, 2 * C:]
    elif mode == "fuser":
        qkv = rnd(B, Lk, 3 * C)
        q, k, v = qkv[:, :Lq, :C], qkv[:, :, C:2 * C], qkv[:, :, 2 * C:]
    elif mode == "kv":
        q = rnd(B, Lq, C)
        kv = rnd(B, Lk, 2 * C, seed=1)
        k, v = kv[:, :, :C], kv[:, :, C:]
    else:
        q, k, v = rnd(B, Lq, C), rnd(B, Lk, C, seed=1), rnd(B, Lk, C, seed=2)
    out = torch.zeros(B, Lq, C, device="cuda:0", dtype=torch.bfloat16)
    out_r = torch.zeros_like(out)
    kernel, poly = ATTN_PATHS[path]
    ops.lib.glg_debug_attn_mode(kernel)
    ops.lib.glg_debug_attn_poly_share(poly)
    try:
        ops.attention(q, k, v, out, heads, d)
        torch.cuda.synchronize()
    finally:
        ops.lib.glg_debug_attn_mode(0)
        ops.lib.glg_debug_attn_poly_share(0)
    ref.attention(q, k, v, out_r, heads, d)
    assert_close(out, out_r, rel=1e-2, max_rel=5e-2, what=f"attention d={d} {Lq}x{Lk} {mode} {path}")


@pytest.mark.parametrize("mode", [4, 5])
@pytest.mark.parametrize("poly", [1, 2, 3])
def test_attention_fma_pipe_exp2(ops, ref, poly, mode):
    """long-key kernels with `poly` of every 8 score pairs exponentiated on the FMA pipe (Cody-Waite + Taylor cubic, rel error
    1.2e-4 mean / 7.9e-4 max), on a wider score range than the default cases.  mode 4: the wgmma kernel, 5: the streamed
    mma.sync kernel."""
    B, heads, d, Lq, Lk = 2, 8, 40, 1024, 1054
    C = heads * d
    qkv = rnd(B, Lk, 3 * C) * 2.0
    q, k, v = qkv[:, :Lq, :C], qkv[:, :, C:2 * C], qkv[:, :, 2 * C:]
    out = torch.zeros(B, Lq, C, device="cuda:0", dtype=torch.bfloat16)
    out_r = torch.zeros_like(out)
    ops.lib.glg_debug_attn_mode({4: 2, 5: 1}[mode])
    ops.lib.glg_debug_attn_poly_share(poly)
    try:
        ops.attention(q, k, v, out, heads, d)
        torch.cuda.synchronize()
    finally:
        ops.lib.glg_debug_attn_mode(0)
        ops.lib.glg_debug_attn_poly_share(0)
    ref.attention(q, k, v, out_r, heads, d)
    assert_close(out, out_r, rel=1e-2, max_rel=5e-2, what=f"attention poly={poly} mode={mode}")


@pytest.mark.parametrize("B,HW,C,ld,eps,silu", [(2, 4096, 320, 320, 1e-5, True), (2, 1024, 960, 960, 1e-5, True),
                                                (1, 256, 2560, 2560, 1e-5, True), (3, 64, 1280, 1280, 1e-6, False),
                                                (2, 1024, 640, 1280, 1e-5, True), (2, 4, 256, 256, 1e-5, True),
                                                (2, 256, 64, 128, 1e-6, False)])
def test_groupnorm(ops, ref, B, HW, C, ld, eps, silu):
    big = rnd(B, HW, ld) * 1.7 + 0.3
    x = big[:, :, ld - C:]
    gamma = 1 + 0.1 * rnd(C, seed=1, dtype=torch.float32)
    beta = 0.1 * rnd(C, seed=2, dtype=torch.float32)
    stats = torch.zeros(gn_scratch_floats(B), device="cuda:0")
    y, y_r = torch.zeros(B, HW, C, device="cuda:0", dtype=torch.bfloat16), torch.zeros(B, HW, C, device="cuda:0", dtype=torch.bfloat16)
    ops.groupnorm(x, y, gamma, beta, stats, 32, eps, silu)
    torch.cuda.synchronize()
    ref.groupnorm(x, y_r, gamma, beta, stats, 32, eps, silu)
    assert_close(y, y_r, what="groupnorm")
    y2 = torch.zeros_like(y)
    ops.groupnorm(x, y2, gamma, beta, stats, 32, eps, silu)
    assert torch.equal(y, y2), "groupnorm must be bit-reproducible"


@pytest.mark.parametrize("B,HW,C,mean", [(2, 4096, 320, 40.0), (8, 4096, 320, -25.0), (2, 1024, 1920, 60.0), (16, 1024, 640, 10.0),
                                         (3, 256, 1280, 50.0), (2, 64, 2560, -80.0), (64, 256, 64, 30.0)])
def test_groupnorm_large_mean(ops, B, HW, C, mean):
    """Post-residual streams carry channel groups whose mean is far from 0: |mean| / std up to ~100 here.  The raw
    E[x^2] - E[x]^2 form loses the variance in fp32 there; the reference's GroupNorm32 (util.py:223-225, F.group_norm in
    fp32: two-pass) does not.  Checked against torch's fp32 group_norm on the same bf16 input; also covers up to 64
    samples per call (one barrier counter each) and bit-reproducibility of the in-kernel barrier path."""
    g = torch.Generator(device="cpu").manual_seed(11)
    base = torch.randn(B, HW, C, generator=g) * 0.8
    # per-group offsets around `mean` (groups of C/32 channels), a few channels with their own offset inside a group
    off = mean * (1.0 + 0.5 * torch.randn(B, 1, 32, generator=g)).repeat_interleave(C // 32, dim=2)
    off[:, :, ::7] += 3.0
    x = (base + off).to("cuda:0", torch.bfloat16)
    gamma = (1 + 0.1 * torch.randn(C, generator=g)).cuda()
    beta = (0.1 * torch.randn(C, generator=g)).cuda()
    stats = torch.zeros(gn_scratch_floats(B), device="cuda:0")
    y = torch.zeros(B, HW, C, device="cuda:0", dtype=torch.bfloat16)
    ops.groupnorm(x, y, gamma, beta, stats, 32, 1e-5, False)
    torch.cuda.synchronize()
    want = torch.nn.functional.group_norm(x.float().transpose(1, 2), 32, gamma, beta, 1e-5).transpose(1, 2)
    assert_close(y, want, rel=4e-3, max_rel=1e-2, what=f"groupnorm large mean {mean}")     # bf16 output rounding only
    y2 = torch.zeros_like(y)
    ops.groupnorm(x, y2, gamma, beta, stats, 32, 1e-5, False)
    assert torch.equal(y, y2), "groupnorm must be bit-reproducible"
    assert int(stats[:128].view(torch.int32).abs().sum()) == 0, "barrier counters must re-arm themselves"


@pytest.mark.parametrize("B,rows,C", [(2, 4096, 320), (2, 30, 640), (3, 64, 1280), (2, 16, 64), (2, 7, 2048)])
def test_layernorm(ops, ref, B, rows, C):
    x = rnd(B, rows, C) * 2 + 0.5
    gamma = 1 + 0.1 * rnd(C, seed=1, dtype=torch.float32)
    beta = 0.1 * rnd(C, seed=2, dtype=torch.float32)
    big = torch.zeros(B, rows + 5, C, device="cuda:0", dtype=torch.bfloat16)
    big_r = torch.zeros_like(big)
    ops.layernorm(x, big[:, 5:], gamma, beta)
    torch.cuda.synchronize()
    ref.layernorm(x, big_r[:, 5:], gamma, beta)
    assert_close(big, big_r, what="layernorm")


def test_small_ops(ops, ref):
    dev = "cuda:0"
    # conv_in (4 and 9 input channels)
    for C1 in (0, 5):
        x = rnd(2, 4, 64, 64, dtype=torch.float32)
        extra = rnd(2, C1, 64, 64, seed=1, dtype=torch.float32) if C1 else None
        w = rnd(9, 4 + C1, 320, scale=0.2, seed=2, dtype=torch.float32)
        b = rnd(320, seed=3, dtype=torch.float32)
        big = torch.zeros(2, 4096, 640, device=dev, dtype=torch.bfloat16)
        out_r = torch.zeros(2, 4096, 320, device=dev, dtype=torch.bfloat16)
        ops.conv_in(x, extra, w, b, big[:, :, 320:])
        ref.conv_in(x, extra, w, b, out_r)
        assert_close(big[:, :, 320:], out_r, what="conv_in")
        assert big[:, :, :320].abs().max().item() == 0
    # conv_out
    x = rnd(2, 4096, 320)
    w = rnd(9, 4, 320, scale=0.02, seed=1, dtype=torch.float32)
    b = rnd(4, seed=2, dtype=torch.float32)
    out, out_r = torch.zeros(2, 4, 64, 64, device=dev), torch.zeros(2, 4, 64, 64, device=dev)
    ops.conv_out(x, w, b, out, 64, 64)
    ref.conv_out(x, w, b, out_r, 64, 64)
    assert_close(out, out_r, rel=2e-3, max_rel=5e-3, what="conv_out")   # torch reference conv runs in TF32
    # odd widths take the per-pixel kernels (the wide-latent variants need W % 4 / W % 8 == 0)
    x = rnd(2, 4, 10, 10, dtype=torch.float32)
    w = rnd(9, 4, 64, scale=0.2, seed=2, dtype=torch.float32)
    b = rnd(64, seed=3, dtype=torch.float32)
    o, o_r = torch.zeros(2, 100, 64, device=dev, dtype=torch.bfloat16), torch.zeros(2, 100, 64, device=dev, dtype=torch.bfloat16)
    ops.conv_in(x, None, w, b, o)
    ref.conv_in(x, None, w, b, o_r)
    assert_close(o, o_r, what="conv_in 10x10")
    x = rnd(2, 100, 64)
    w = rnd(9, 4, 64, scale=0.05, seed=1, dtype=torch.float32)
    b = rnd(4, seed=2, dtype=torch.float32)
    out, out_r = torch.zeros(2, 4, 10, 10, device=dev), torch.zeros(2, 4, 10, 10, device=dev)
    ops.conv_out(x, w, b, out, 10, 10)
    ref.conv_out(x, w, b, out_r, 10, 10)
    assert_close(out, out_r, rel=2e-3, max_rel=5e-3, what="conv_out 10x10")
    # upsample / im2col
    x = rnd(2, 256, 640)
    y, y_r = torch.zeros(2, 1024, 640, device=dev, dtype=torch.bfloat16), torch.zeros(2, 1024, 640, device=dev, dtype=torch.bfloat16)
    ops.upsample2x(x, y, 16, 16); ref.upsample2x(x, y_r, 16, 16)
    assert torch.equal(y, y_r)
    col, col_r = torch.zeros(2 * 64, 9 * 640, device=dev, dtype=torch.bfloat16), torch.zeros(2 * 64, 9 * 640, device=dev, dtype=torch.bfloat16)
    ops.im2col_s2(x, col, 16, 16); ref.im2col_s2(x, col_r, 16, 16)
    assert torch.equal(col, col_r)
    # the VAE encoder's Downsample pads only right / bottom (model.py:73-77)
    ops.im2col_s2(x, col, 16, 16, pad_lo=0); ref.im2col_s2(x, col_r, 16, 16, pad_lo=0)
    assert torch.equal(col, col_r)
    xin = x.float().reshape(2, 16, 16, 640).permute(0, 3, 1, 2)
    wgt = torch.randn(64, 640, 3, 3, device=dev) * 0.01
    want = torch.nn.functional.conv2d(torch.nn.functional.pad(xin, (0, 1, 0, 1)), wgt, stride=2)            # the reference's statement
    got = (col.float() @ wgt.permute(0, 2, 3, 1).reshape(64, -1).t()).reshape(2, 8, 8, 64).permute(0, 3, 1, 2)
    assert_close(got, want, rel=1e-3, max_rel=5e-3, what="asymmetric-pad stride-2 conv through im2col")
    # timestep embedding
    t = torch.tensor([981, 1, 500, 21], device=dev)
    o, o_r = torch.zeros(4, 320, device=dev, dtype=torch.bfloat16), torch.zeros(4, 320, device=dev, dtype=torch.bfloat16)
    ops.timestep_embedding(t, o); ref.timestep_embedding(t, o_r)
    assert_close(o, o_r, rel=4e-3, max_rel=1e-2, what="timestep_embedding")
    # position features (text: F=768, 4 coords; keypoint: broadcast table, 2 coords, padded K)
    for F_, nc, ldo, bc in ((768, 4, 832, False), (768, 2, 832, True)):
        B, N = 3, 30
        feat = rnd(N, F_, dtype=torch.float32) if bc else rnd(B, N, F_, dtype=torch.float32)
        fm = (torch.rand(B, N, device=dev) > 0.4).float()
        pm = (torch.rand(B, N, device=dev) > 0.4).float()
        coords = torch.rand(B, N, nc, device=dev)
        nf, npos = rnd(F_, seed=5, dtype=torch.float32), rnd(16 * nc, seed=6, dtype=torch.float32)
        o, o_r = torch.ones(B * N, ldo, device=dev, dtype=torch.bfloat16), torch.ones(B * N, ldo, device=dev, dtype=torch.bfloat16)
        ops.position_features(feat, fm, nf, coords, pm, npos, o, 8); ref.position_features(feat, fm, nf, coords, pm, npos, o_r, 8)
        assert_close(o, o_r, rel=4e-3, max_rel=1e-2, what="position_features")
    # cast
    x = rnd(1000, 77, dtype=torch.float32)
    y = torch.zeros(1000, 77, device=dev, dtype=torch.bfloat16)
    ops.cast(x, y)
    assert torch.equal(y, x.to(torch.bfloat16))
    # sampler update
    n = (4, 4, 64, 64)
    xs, ec, eu, o1, o2, o3 = (rnd(*n, seed=s, dtype=torch.float32) for s in range(6))
    for olds, coefs in (([], (1.0, 0, 0, 0)), ([o1], (1.5, -0.5, 0, 0)), ([o1, o2, o3], (55 / 24, -59 / 24, 37 / 24, -9 / 24))):
        e, xp, e_r, xp_r = (torch.zeros(n, device=dev) for _ in range(4))
        ops.sampler_update(xs, ec, eu, 7.5, olds, coefs, 0.5, 0.6, e, xp)
        ref.sampler_update(xs, ec, eu, 7.5, olds, coefs, 0.5, 0.6, e_r, xp_r)
        assert_close(e, e_r, rel=1e-5, max_rel=1e-4, what="sampler e")
        assert_close(xp, xp_r, rel=1e-5, max_rel=1e-4, what="sampler x_prev")
    torch.cuda.synchronize()
