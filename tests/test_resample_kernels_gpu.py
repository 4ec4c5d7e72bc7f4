"""GPU: the resampling kernels of the spatial modalities (csrc/frontend.cu resize_plane, conv2d_small, patchify_nchw) against
float64 at the bounds of tests/bounds_resample.py, on conditioning maps of any size and aspect ratio: non-square sources and
outputs, down- and upscaling (also one axis each way), ratios with many distinct bicubic fractions, 1- and 2-pixel sources,
1-pixel outputs, a phone-sized source, output sizes that are not powers of two (inexact coordinates), channel subsets of
wider maps, odd virtual grids whose last row and column get partial windows, and every Cout instantiation of conv2d_small."""
import pytest
import torch

import bounds_resample

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


@pytest.fixture(scope="module")
def ops():
    from gligen_b200.ops import CudaOps
    return CudaOps(DEV)


def rnd(*shape, scale=1.0, seed=0):
    g = torch.Generator(device="cpu").manual_seed(seed + sum(shape))
    return (torch.randn(*shape, generator=g) * scale).to(DEV)


RESIZE = [  # (B, Cx, C, Hs, Ws, Ho, Wo)
    (2, 3, 1, 480, 640, 256, 256), (1, 3, 3, 300, 224, 128, 128), (4, 3, 1, 640, 480, 256, 256),     # 4:3 photos: many fractions
    (2, 3, 3, 192, 320, 256, 256), (1, 3, 2, 320, 192, 64, 400), (1, 3, 3, 96, 120, 256, 200),        # one axis up, one down; both up
    (1, 1, 1, 1, 1, 64, 64), (2, 1, 1, 1, 37, 16, 16), (2, 3, 1, 2, 29, 8, 24), (1, 1, 1, 45, 2, 10, 3), (1, 3, 2, 33, 1, 5, 4),
    (2, 3, 3, 480, 640, 1, 1), (1, 3, 1, 300, 224, 1, 100), (1, 2, 2, 7, 5, 9, 1),                      # 1-pixel outputs
    (1, 3, 1, 4032, 3024, 256, 256),                                                                   # phone-sized source
    (2, 3, 3, 512, 512, 100, 100), (1, 3, 3, 480, 640, 224, 224), (3, 4, 2, 150, 200, 100, 224),       # inexact coordinates
    (4, 5, 3, 75, 61, 100, 224), (4, 3, 1, 300, 224, 128, 128),                                         # C < Cx, B = 4
]


@pytest.mark.parametrize("mode", ["nearest", "bicubic"])
@pytest.mark.parametrize("B,Cx,C,Hs,Ws,Ho,Wo", RESIZE)
def test_resize_plane(ops, mode, B, Cx, C, Hs, Ws, Ho, Wo):
    x = rnd(B, Cx, Hs, Ws)
    y = torch.full((B, C, Ho, Wo), float("nan"), device=DEV)
    ops.resize_plane(x, y, C, mode)
    torch.cuda.synchronize()
    rep = bounds_resample.resize_check(y, x, mode, what=f"resize_plane {mode} {Hs}x{Ws} -> {Ho}x{Wo}")
    print(rep)
    assert rep.ok, str(rep)


CONV = [  # (B, Cin, Cout, Hs, Ws, virtual, k, stride, pad, silu): the downsamplers' 4/2/1, the sem in_conv's 3/1/1
    (2, 1, 4, 192, 320, (129, 97), 4, 2, 1, True),       # canny / depth conv0 shape, virtual grid shrinking on one axis only
    (1, 3, 4, 300, 224, None, 4, 2, 1, True),            # normal conv0 on a non-square plane
    (2, 4, 8, 65, 47, None, 4, 2, 1, False),             # conv2: odd, partial last windows
    (1, 152, 16, 300, 224, (257, 255), 4, 2, 1, True),   # sem conv0: 152 one-hot classes, enlarging
    (1, 152, 16, 640, 480, (129, 131), 4, 2, 1, False),  # shrinking
    (1, 16, 8, 129, 63, None, 4, 2, 1, False),
    (1, 152, 3, 480, 640, (129, 127), 3, 1, 1, False),   # sem in_conv, shrinking
    (2, 24, 3, 100, 60, (131, 77), 3, 1, 1, False),      # sem in_conv, enlarging
    (1, 7, 3, 31, 45, (45, 31), 3, 1, 1, True),
    (3, 2, 16, 50, 70, (33, 95), 4, 2, 1, False),        # one axis up, one down
    (2, 1, 8, 33, 21, (17, 40), 3, 1, 1, True),
    (1, 5, 4, 1, 9, (5, 3), 3, 1, 1, False),             # 1-pixel source rows
]


@pytest.mark.parametrize("B,Cin,Cout,Hs,Ws,virtual,k,stride,pad,silu", CONV)
def test_conv2d_small(ops, B, Cin, Cout, Hs, Ws, virtual, k, stride, pad, silu):
    x = rnd(B, Cin, Hs, Ws)
    w, bias = rnd(Cin * k * k, Cout, scale=(Cin * k * k) ** -0.5, seed=1), 0.1 * rnd(Cout, seed=2)
    Hv, Wv = virtual or (Hs, Ws)
    Ho, Wo = (Hv + 2 * pad - k) // stride + 1, (Wv + 2 * pad - k) // stride + 1
    y = torch.full((B, Cout, Ho, Wo), float("nan"), device=DEV)
    ops.conv2d_small(x, w, bias, y, k, stride, pad, silu, virtual=virtual)
    torch.cuda.synchronize()
    rep = bounds_resample.conv2d_small_check(y, x, w, bias, k, stride, pad, silu, virtual, what=f"conv2d_small Cin={Cin} Cout={Cout} {Hs}x{Ws} -> {virtual}")
    print(rep)
    assert rep.ok, str(rep)


@pytest.mark.parametrize("Cout,k,stride,pad", [(3, 3, 1, 1), (4, 4, 2, 1), (8, 4, 2, 1), (16, 4, 2, 1)])
def test_conv2d_small_exact(ops, Cout, k, stride, pad):
    """Small integers: every partial sum is an integer below 2^24, exact in fp32 in any order, so the kernel must equal the
    float64 convolution bit for bit - a wrong tap, weight or padding cannot hide under a rounding bound."""
    g = torch.Generator(device="cpu").manual_seed(Cout)
    B, Cin, Hs, Ws, virtual = 2, 11, 37, 52, (41, 29)
    x = torch.randint(-3, 4, (B, Cin, Hs, Ws), generator=g).float().to(DEV)
    w = torch.randint(-2, 3, (Cin * k * k, Cout), generator=g).float().to(DEV)
    bias = torch.randint(-5, 6, (Cout,), generator=g).float().to(DEV)
    Ho, Wo = (virtual[0] + 2 * pad - k) // stride + 1, (virtual[1] + 2 * pad - k) // stride + 1
    y = torch.full((B, Cout, Ho, Wo), float("nan"), device=DEV)
    ops.conv2d_small(x, w, bias, y, k, stride, pad, False, virtual=virtual)
    torch.cuda.synchronize()
    F = torch.nn.functional
    xv = x.double()[:, :, bounds_resample.nearest_index(virtual[0], Hs, DEV)][:, :, :, bounds_resample.nearest_index(virtual[1], Ws, DEV)]
    ref = F.conv2d(xv, w.double().reshape(Cin, k, k, Cout).permute(3, 0, 1, 2), bias.double(), stride=stride, padding=pad)
    assert torch.equal(y.double(), ref), f"max diff {(y.double() - ref).abs().max().item()}"


@pytest.mark.parametrize("B,C,Hs,Ws,R,k,ldo", [(2, 3, 480, 640, 128, 4, 64), (1, 3, 300, 224, 256, 4, 64), (1, 3, 192, 320, 128, 4, 64),
                                             (2, 5, 97, 61, 64, 2, 24), (1, 3, 61, 97, 32, 2, 16)])
def test_patchify_nchw(ops, B, C, Hs, Ws, R, k, ldo):
    """A gather onto the virtual R x R grid and one round-to-nearest-even to bf16: bit-exact; columns [k^2 C, ldo) zero."""
    x = rnd(B, C, Hs, Ws)
    rows = B * (R // k) ** 2
    out = torch.full((rows, ldo), 7.0, device=DEV, dtype=torch.bfloat16)
    ops.patchify_nchw(x, out, R, R, k)
    torch.cuda.synchronize()
    xv = x[:, :, bounds_resample.nearest_index(R, Hs, DEV)][:, :, :, bounds_resample.nearest_index(R, Ws, DEV)]
    want = torch.zeros(rows, ldo, device=DEV, dtype=torch.bfloat16)
    want[:, : k * k * C] = xv.view(B, C, R // k, k, R // k, k).permute(0, 2, 4, 3, 5, 1).reshape(rows, k * k * C).to(torch.bfloat16)
    assert torch.equal(out[:, k * k * C:], torch.zeros_like(out[:, k * k * C:])), "padding columns not zero"
    assert torch.equal(out, want)
