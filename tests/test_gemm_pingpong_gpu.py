"""The ping-pong GEMM schedule (each consumer warpgroup owns whole 128 x BN items, MMA token between them) forced wherever
legal, against the torch statement, in every mode the cooperative schedule has: streaming / B-resident / paired CTAs,
split-K, LayerNorm fold + statistics, GEGLU, 3x3 convolution.  The schedule must not change the arithmetic: at the same
tile width its output is bit-identical to the cooperative schedule's."""
import pytest
import torch

from conftest import assert_close
from ref_ops import RefOps
from test_kernels_gpu import CONV_CASES, GEMM_CASES, _conv_case, _ln_fold_case, rnd

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ops():
    from gligen_b200.ops import CudaOps
    return CudaOps("cuda:0")


@pytest.fixture(scope="module")
def ref():
    return RefOps("cuda:0", torch.float32)


class modes:
    """Set the picker's test hooks for the duration of a block; reset them after."""

    def __init__(self, ops, pp=2, cta2=1, bres=1, bn=0, splitk=0):
        self.lib, self.v = ops.lib, dict(pp=pp, cta2=cta2, bres=bres, bn=bn, splitk=splitk)

    def _set(self, pp, cta2, bres, bn, splitk):
        self.lib.glg_debug_gemm_pp(pp); self.lib.glg_debug_gemm_cta2(cta2); self.lib.glg_debug_gemm_bres(bres)
        self.lib.glg_debug_force_bn(bn); self.lib.glg_debug_splitk(splitk)

    def __enter__(self):
        self._set(**self.v)

    def __exit__(self, *exc):
        self._set(0, 0, 0, 0, 0)


def _gemm_inputs(M, N, K, fl):
    geglu = fl.get("geglu", False)
    No = N // 2 if geglu else N
    a = rnd(M, K)
    w = rnd(N, K, scale=K ** -0.5, seed=1)
    bias = rnd(N, seed=2, dtype=torch.float32) if (fl.get("bias") or geglu) else None
    gate = torch.tensor([0.37], device="cuda:0") if fl.get("gate") else None
    rows_per_batch = fl.get("rowbias", 0)
    rowbias = rnd(M // rows_per_batch, N, seed=3, dtype=torch.float32) if rows_per_batch else None
    residual = rnd(M, No, seed=4) if fl.get("residual") else None
    kw = dict(bias=bias, rowbias=rowbias, rows_per_batch=max(rows_per_batch, 1), act=1 if fl.get("act") else 0,
              gate=gate, residual=residual, geglu=geglu)
    odt = torch.float32 if fl.get("fp32") else torch.bfloat16
    return a, w, kw, (M, No), odt


@pytest.mark.parametrize("M,N,K,fl", GEMM_CASES)
@pytest.mark.parametrize("bn", [0, 64, 128])
@pytest.mark.parametrize("cta2,bres", [(1, 1), (2, 1), (1, 2)])
def test_gemm_pingpong(ops, ref, M, N, K, fl, bn, cta2, bres):
    """cta2 1 / 2: single CTAs / CTA pairs; bres 2: weights-resident tiles wherever they fit."""
    if bn and (N % bn or fl.get("geglu")):
        pytest.skip("BN does not divide N")
    if cta2 == 2 and (bn == 64 or M <= 128):
        pytest.skip("pairs need BN >= 128 and M > 128")
    a, w, kw, oshape, odt = _gemm_inputs(M, N, K, fl)
    out, out_co, out_r = (torch.zeros(*oshape, device="cuda:0", dtype=odt) for _ in range(3))
    with modes(ops, pp=2, cta2=cta2, bres=bres, bn=bn):
        pp = ops.lib.glg_debug_pick_pingpong(M, N, K, int(bool(fl.get("geglu"))), 0, 0, 0)
        tile_pp = _tile(ops, M, N, K, fl)
        ops.gemm(a, w, out, **kw)
        torch.cuda.synchronize()
    ref.gemm(a, w, out_r, **kw)
    assert_close(out, out_r, what=f"ping-pong gemm {M}x{N}x{K} {fl} bn={bn} cta2={cta2} bres={bres} pp={pp}")
    if pp and bn and not fl.get("geglu"):
        with modes(ops, pp=1, cta2=cta2, bres=bres, bn=bn):
            if _tile(ops, M, N, K, fl) != tile_pp:
                return                                   # the cooperative schedule picks another split / pairing
            ops.gemm(a, w, out_co, **kw)
            torch.cuda.synchronize()
        assert torch.equal(out, out_co), "ping-pong and cooperative schedules differ at the same tile"


def _tile(ops, M, N, K, fl):
    import ctypes as C
    pick = (C.c_int32 * 3)()
    can_split = not (fl.get("geglu") or fl.get("fp32"))
    ops.lib.glg_debug_pick_tile(M, N, K, int(bool(fl.get("geglu"))), 0, int(can_split), ops.splitk_ws.numel() * 4, pick)
    return tuple(pick)


def test_pingpong_is_legal_for_the_short_k_shapes(ops):
    """The forced hook reaches the ping-pong kernels for GEGLU and the BN <= 128 plain tiles."""
    with modes(ops, pp=2):
        assert ops.lib.glg_debug_pick_pingpong(32768, 2560, 320, 1, 0, 0, 0) == 1
        assert ops.lib.glg_debug_pick_pingpong(8192, 640, 640, 0, 0, 0, 0) == 1
    with modes(ops, pp=1):
        assert ops.lib.glg_debug_pick_pingpong(32768, 2560, 320, 1, 0, 0, 0) == 0


@pytest.mark.parametrize("M,N,K,geglu", [(4096, 960, 320, False), (1000, 1920, 640, False), (4096, 2560, 320, True),
                                         (520, 1024, 128, True)])
@pytest.mark.parametrize("cta2,bres", [(1, 1), (2, 1), (1, 2)])
def test_pingpong_layernorm_fold(ops, ref, M, N, K, geglu, cta2, bres):
    with modes(ops, pp=2, cta2=cta2, bres=bres):
        _ln_fold_case(ops, ref, M, N, K, geglu)


@pytest.mark.parametrize("M,N,K,conv", [(512, 1280, 1280, None), (200, 640, 2560, None), (512, 1280, 1280, (8, 8, 8)),
                                         (128, 1280, 2560, (2, 8, 8)), (512, 256, 256, (8, 8, 8))])
def test_pingpong_split_k(ops, ref, M, N, K, conv):
    a = rnd(conv[0], conv[1] * conv[2], K) if conv else rnd(M, K)
    w = rnd((9 if conv else 1) * N, K, scale=((9 if conv else 1) * K) ** -0.5, seed=1)
    bias = rnd(N, seed=2, dtype=torch.float32)
    res = rnd(M, N, seed=3)
    outs = []
    with modes(ops, pp=2, splitk=2):
        for _ in range(2):
            out = torch.zeros(M, N, device="cuda:0", dtype=torch.bfloat16)
            ops.gemm(a, w, out, bias=bias, residual=res, conv=conv)
            torch.cuda.synchronize()
            outs.append(out)
    out_r = torch.zeros(M, N, device="cuda:0", dtype=torch.bfloat16)
    ref.gemm(a, w, out_r, bias=bias, residual=res, conv=conv)
    assert_close(outs[0], out_r, what=f"ping-pong split-K gemm {M}x{N}x{K} conv={conv}")
    assert torch.equal(outs[0], outs[1])


@pytest.mark.parametrize("B,H,W,Cin,Cout,fl", CONV_CASES)
@pytest.mark.parametrize("cta2", [1, 2])
def test_pingpong_conv3x3(ops, ref, B, H, W, Cin, Cout, fl, cta2):
    if cta2 == 2 and (B * H * W <= 128 or Cout % 128):
        pytest.skip("pairs need M > 128 and Cout % 128 == 0")
    with modes(ops, pp=2, cta2=cta2):
        _conv_case(ops, ref, B, H, W, Cin, Cout, fl)


def test_pingpong_batch_strided_output(ops, ref):
    B, T, C = 3, 200, 320
    a = rnd(B * T, C)
    w = rnd(3 * C, C, scale=C ** -0.5, seed=1)
    big = torch.zeros(B, T + 30, 3 * C, device="cuda:0", dtype=torch.bfloat16)
    big_r = torch.zeros_like(big)
    with modes(ops, pp=2):
        ops.gemm(a, w, big[:, :T])
        torch.cuda.synchronize()
    ref.gemm(a, w, big_r[:, :T])
    assert_close(big, big_r, what="ping-pong batch-strided gemm")
    assert big[:, T:].abs().max().item() == 0
