"""Edges of the consumer loop of the long-key attention kernel (attn_wgmma_kernel), reached on purpose rather than by
chance: 1, 2, STAGES (3), STAGES + 1 and 2 STAGES + 1 key tiles, each with a full and with a ragged last tile (the K/V
ring wraps after 3 tiles); query counts whose second warpgroup has no valid row or only some (Lq % 128 in {1, 64, 65});
head dims 40 / 64 / 80 / 160 (DPAD 48 / 64 / 80 / 160); the branch-free MUFU exponentials (poly = 0) and the FMA-pipe
share (poly = 2), which are separate compile-time instantiations.  Every case is checked in the dominant-key exact form
(with poly = 2 up to the 2^-125 floor of ex2_poly3, see FMA_FLOOR) and against the float64 bound of tests/bounds.py.
Query rows whose dominant keys sit in different tiles move their running max on different tiles, so the warp-uniform
vote that skips the unity rescale sees both outcomes."""
import math

import pytest
import torch

import bounds
from test_kernel_stress_gpu import DEV, BF, debug_modes, gen, onehot_attention

pytestmark = pytest.mark.gpu

WGMMA = 2                                     # glg_debug_attn_mode: the wgmma kernel for every key length
KEY_LENGTHS = [64, 50, 128, 100, 192, 170, 256, 230, 448, 420]    # 1, 2, 3, 4, 7 tiles: full and ragged last tile
QUERY_LENGTHS = [129, 192, 193]              # Lq % 128 = 1, 64, 65
HEAD_DIMS = [40, 64, 80, 160]
POLYS = [0, 2]
# ex2_poly3 clamps its argument at -125 and never returns 0, so with poly > 0 every non-dominant key on an FMA-pipe lane
# adds about 2^-125 |V| to the output: an element where V[pi(i)] is exactly 0 comes back as a value of order 1e-37
# (d = 160, 193 x 448 has one).  Up to this floor the output is V[pi(i)] bit for bit.
FMA_FLOOR = 2.0 ** -100


@pytest.fixture(scope="module")
def ops():
    from gligen_b200.ops import CudaOps
    return CudaOps(DEV)


def run(ops, q, k, v, heads, d, poly):
    out = torch.zeros(q.shape[0], q.shape[1], heads * d, device=DEV, dtype=BF)
    with debug_modes(ops, attn=WGMMA, poly=poly):
        ops.attention(q, k, v, out, heads, d)
        torch.cuda.synchronize()
    return out


@pytest.mark.parametrize("Lk", KEY_LENGTHS)
@pytest.mark.parametrize("d", HEAD_DIMS)
def test_pipeline_dominant_key_exact(ops, d, Lk):
    for Lq in QUERY_LENGTHS:
        q, k, v, want = onehot_attention(1, 2, d, Lq, Lk, False, seed=7 * d + Lk + Lq)
        for poly in POLYS:
            out = run(ops, q, k, v, 2, d, poly)
            if poly:
                bad = (~((out.float() - want.float()).abs() <= FMA_FLOOR)).any(-1)     # NaN counts as bad
            else:
                bad = (out != want).any(-1)
            assert not bad.any(), f"d={d} {Lq}x{Lk} poly={poly}: rows {bad.nonzero()[:8].tolist()} differ from V[pi(i)]"


def staggered_max_inputs(B, heads, d, Lq, Lk, seed):
    """Scaled logits of std 1, plus a boost of 6 on one key per query row, in key tile (i // 3) % ntiles: the 16 rows of
    a warp reach their running max in different tiles, so on a given tile only some rows move it, and after the last
    boosted tile none do (the rescale is skipped there)."""
    g = gen(seed)
    q = torch.randn(B, Lq, heads * d, generator=g)
    k = torch.randn(B, Lk, heads * d, generator=g)
    v = torch.randn(B, Lk, heads * d, generator=g)
    ntiles = (Lk + 63) // 64
    alpha = 6.0 / math.sqrt(d)                   # q_i . k_j / sqrt(d) grows by ~ alpha |k_j|^2 / sqrt(d) = 6
    for i in range(Lq):
        t = (i // 3) % ntiles
        j = min(t * 64 + (i * 7) % 64, Lk - 1)
        q[:, i] += alpha * k[:, j]
    return q.to(DEV, BF), k.to(DEV, BF), v.to(DEV, BF)


@pytest.mark.parametrize("Lk", KEY_LENGTHS)
@pytest.mark.parametrize("d", HEAD_DIMS)
def test_pipeline_bounded(ops, d, Lk):
    for Lq in QUERY_LENGTHS:
        q, k, v = staggered_max_inputs(1, 2, d, Lq, Lk, seed=11 * d + Lk + Lq)
        for poly in POLYS:
            out = run(ops, q, k, v, 2, d, poly)
            rep = bounds.attention_check(out, q, k, v, 2, d, poly=poly, what=f"attention d={d} {Lq}x{Lk} poly={poly}")
            assert rep.ok, str(rep)


@pytest.mark.parametrize("d", [40, 80])
def test_pipeline_poly_shares_match_modes(ops, d):
    """Every FMA-pipe share 0..3 under every kernel mode 0..3 stays inside the bound (the POLY instantiation is chosen
    from the share at launch)."""
    Lq, Lk = 193, 420
    q, k, v = staggered_max_inputs(1, 2, d, Lq, Lk, seed=d)
    for mode in range(4):
        for poly in range(4):
            out = torch.zeros(1, Lq, 2 * d, device=DEV, dtype=BF)
            with debug_modes(ops, attn=mode, poly=poly):
                ops.attention(q, k, v, out, 2, d)
                torch.cuda.synchronize()
            # Lk > 128: every mode runs a long-key kernel, which applies the share
            rep = bounds.attention_check(out, q, k, v, 2, d, poly=poly, what=f"mode {mode} poly {poly} d={d}")
            assert rep.ok, str(rep)
