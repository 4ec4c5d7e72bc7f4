"""CPU: the FMA-pipe exp2 of the long-key attention kernels (csrc/common.cuh ex2_poly3: Cody-Waite split by the 1.5 * 2^23 magic
constant + Taylor cubic on [-0.5, 0.5] + exponent insertion), restated in numpy fp32 exactly as the kernel computes it: relative error
against exp2 over the whole range the softmax feeds it - 1.2e-4 on average, 7.9e-4 at worst (|f| = 0.5) - below the bf16 rounding of P
(half an ulp = 2^-9 = 2e-3), and exact zero-ish results for masked / underflowing scores."""
import numpy as np


def ex2_poly3(x):
    x = np.maximum(x.astype(np.float32), np.float32(-125.0))
    magic = np.float32(12582912.0)
    t = (x + magic).astype(np.float32)
    f = (x - (t - magic)).astype(np.float32)
    p = np.float32(0.05550411) * f + np.float32(0.24022651)
    p = (p * f + np.float32(0.69314718)).astype(np.float32)
    p = (p * f + np.float32(1.0)).astype(np.float32)
    bits = p.view(np.int32) + (t.view(np.int32) << 23)
    return bits.view(np.float32)


def test_relative_error():
    x = np.concatenate([np.linspace(-124.9, 8.0, 400001), -np.random.default_rng(0).random(100000) * 20]).astype(np.float32)
    got, ref = ex2_poly3(x).astype(np.float64), np.exp2(x.astype(np.float64))
    rel = np.abs(got - ref) / ref
    assert rel.max() < 8.5e-4 and rel.mean() < 1.5e-4, (rel.max(), rel.mean())
    assert np.all(ex2_poly3(np.array([-200.0, -1e30, -np.inf], dtype=np.float32)) < 1e-37)      # masked keys / underflow: ~0, never garbage
    assert ex2_poly3(np.array([0.0], dtype=np.float32))[0] == 1.0
