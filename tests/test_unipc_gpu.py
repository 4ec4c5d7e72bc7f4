"""GPU: the UniPC update kernel (glg_unipc_update) against float64 at its rounding limit (tests/bounds_unipc.py), and UniPCSampler
over the drop-in UNetModel against the oracle fixtures (tests/golden/unipc_*.pt, oracle/gen_golden_unipc.py) and on a non-square
latent.  Loop tolerance as tests/test_engine_gpu.py: rel-L2 <= 6e-2 and max-abs <= 10 % of max|latent| (bf16 UNet against the
fp32 oracle)."""
import os
from functools import partial

import numpy as np
import pytest
import torch

from bounds_unipc import unipc_update_check
from conftest import GOLD, assert_close
from gligen_b200 import synth
from ldm.models.diffusion import dpm_solver as DS
from ldm.models.diffusion import unipc as UP
from oracle import sampler_oracle as SO

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


@pytest.fixture(scope="module")
def ops():
    from gligen_b200.ops import CudaOps
    return CudaOps(DEV)


def _schedule(S, order):
    ac = SO.make_schedule()["alphas_cumprod"]
    alpha, sigma = DS.grid_alpha_sigma(ac, np.flip(SO.ddim_timesteps(S)))
    orders = DS.step_orders(len(alpha) - 1, order)
    return alpha, sigma, orders, UP.step_coefficients(alpha, sigma, orders)


def _inputs(shape, seed):
    g = torch.Generator(device=DEV).manual_seed(seed)
    return [torch.randn(shape, generator=g, device=DEV) for _ in range(7)]       # x, xc_prev, e_c, e_u, m1, m2, m3


def _run(ops, x, xcp, ec, eu, m1, m2, m3, a, s, coefs):
    """The kernel's three outputs, each in the middle of a guarded buffer: nothing outside them may be written."""
    n = x.numel()
    guard = 64
    buf = torch.full((3, n + 2 * guard), float("nan"), device=DEV)
    m0, xc, xn = (buf[j, guard:guard + n].view(x.shape) for j in range(3))
    ops.unipc_update(x, xcp, ec, eu, 7.5, m1, m2, m3, a, s, coefs, m0, xc, xn)
    torch.cuda.synchronize()
    assert torch.isnan(buf[:, :guard]).all() and torch.isnan(buf[:, guard + n:]).all(), "write outside the outputs"
    return m0, xc, xn


SHAPES = [(4, 4, 64, 64), (2, 4, 16, 24), (1001,), (3, 5, 7, 11)]


@pytest.mark.parametrize("shape", SHAPES)
@pytest.mark.parametrize("S", [10, 15, 20])
@pytest.mark.parametrize("order", [1, 2, 3])
def test_kernel_against_float64(ops, shape, S, order):
    """Every step of the schedule (the i = 0 form without xc_prev included), CFG on and off, history pointers null where the
    step does not read them; the inputs are left as they were."""
    alpha, sigma, orders, coefs = _schedule(S, order)
    x, xcp, ec, eu, m1, m2, m3 = _inputs(shape, seed=S * 10 + order)
    before = [t.clone() for t in (x, xcp, ec, eu, m1, m2, m3)]
    worst = None
    for i in range(len(orders)):
        a, s = float(alpha[i]), float(sigma[i])
        depth = UP.history_depth(orders, i)
        h1, h2, h3 = (m if j <= depth else None for j, m in ((1, m1), (2, m2), (3, m3)))
        prev = xcp if i > 0 else None
        for u in (eu, None):
            m0, xc, xn = _run(ops, x, prev, ec, u, h1, h2, h3, a, s, coefs[i])
            rep = unipc_update_check(m0, xc, xn, x, prev, ec, u, 7.5, h1, h2, h3, a, s, coefs[i],
                                     what=f"unipc_update {shape} S={S} step {i} order {orders[i]} cfg={u is not None}")
            assert rep.ok, rep
            if prev is None:
                assert torch.equal(xc, x)
            worst = rep if worst is None or rep.ratio > worst.ratio else worst
    assert all(torch.equal(t, b) for t, b in zip((x, xcp, ec, eu, m1, m2, m3), before))
    print(worst)


def test_kernel_scalar_path_and_repeat(ops):
    """Views 4 bytes off 16-byte alignment take the scalar path, with the same results; a repeat run is bit-identical."""
    alpha, sigma, orders, coefs = _schedule(20, 3)
    n = 4 * 64 * 64 + 3
    base = _inputs((n + 1,), seed=5)
    a, s, c = float(alpha[5]), float(sigma[5]), coefs[5]
    aligned = [t[:n] for t in base]
    buf = [torch.empty(n + 1, device=DEV) for _ in base]
    for b, t in zip(buf, aligned):
        b[1:].copy_(t)
    shifted = [b[1:] for b in buf]
    outs_a = _run(ops, *aligned, a, s, c)
    out = torch.empty(3, n + 1, device=DEV)
    ops.unipc_update(shifted[0], shifted[1], shifted[2], shifted[3], 7.5, shifted[4], shifted[5], shifted[6], a, s, c,
                     out[0, 1:], out[1, 1:], out[2, 1:])
    torch.cuda.synchronize()
    assert all(torch.equal(out[j, 1:], outs_a[j]) for j in range(3))
    rep = unipc_update_check(*outs_a, aligned[0], aligned[1], aligned[2], aligned[3], 7.5, *aligned[4:], a, s, c,
                             what="unipc_update n % 4 = 3")
    assert rep.ok, rep
    outs_b = _run(ops, *aligned, a, s, c)
    assert all(torch.equal(p, q) for p, q in zip(outs_a, outs_b))


# ---- the sampler over the drop-in UNetModel -------------------------------------------------------------------------------------
class cpu_rng_noise:
    """The fixtures' q_sample noise comes from the CPU generator: draw the same noise in the same order (test_engine_gpu.py)."""

    def __enter__(self):
        self.orig = torch.randn_like
        torch.randn_like = lambda x, **kw: torch.randn(x.shape, dtype=x.dtype).to(x.device)
        return self

    def __exit__(self, *a):
        torch.randn_like = self.orig


def _sample(cfg, B, max_objs, S, order, alpha_type, x=None):
    """(cfg, model, final latent) of one seeded run; x replaces make_inputs' x_T (the non-square case)."""
    from gligen_b200.pipeline import alpha_generator, build_model, sampler_inputs, set_alpha_scale, to_device
    from ldm.models.diffusion.ldm import LatentDiffusion
    cfg, model = build_model(cfg, DEV)
    inp = synth.make_inputs(cfg, B, max_objs, seed=2)
    if x is not None:
        inp["x"] = x
    dinp = to_device({k: v for k, v in inp.items() if k in ("x", "context", "uc", "z0")}, DEV)
    input, mask, x0 = sampler_inputs(cfg, model, dinp, to_device(inp["batch"], DEV))
    diffusion = LatentDiffusion(linear_start=0.00085, linear_end=0.012, timesteps=1000).to(DEV)
    sampler = UP.UniPCSampler(diffusion, model, alpha_generator_func=partial(alpha_generator, type=alpha_type),
                              set_alpha_scale=set_alpha_scale, order=order)
    cwd = os.getcwd()
    os.chdir(GOLD)                  # SD_input_conv_weight_bias.pth is read CWD-relative, like the reference
    try:
        torch.manual_seed(1234)
        with cpu_rng_noise():
            lat = sampler.sample(S=S, shape=tuple(dinp["x"].shape), input=input, uc=dinp["uc"], guidance_scale=7.5, mask=mask, x0=x0)
    finally:
        os.chdir(cwd)
    return cfg, model, lat


def _fixture_cfg(name):
    from gligen_b200.spec import NAMED_CONFIGS, SAMPLING_GATED_CA
    return SAMPLING_GATED_CA if name == "sampling_gated_ca" else NAMED_CONFIGS[name]


@pytest.mark.parametrize("gold_file", ["unipc_tiny_o2.pt", "unipc_tiny_o3.pt", "unipc_tiny_o2_s16.pt", "unipc_tiny_inpaint_o2.pt",
                                       "unipc_sampling_gated_ca_o2.pt", "unipc_sd14_box_text_o2.pt"])
def test_loop_matches_oracle(gold_file):
    gold = torch.load(os.path.join(GOLD, gold_file))
    cfg, model, lat = _sample(_fixture_cfg(gold["config"]), gold["B"], gold["max_objs"], gold["S"], gold["order"], gold["alpha_type"])
    if gold["alpha_type"][0] < 1 and not cfg.inpaint_mode:
        assert model.first_conv_type == "SD"
    r, m = assert_close(lat, gold["latent"], rel=6e-2, max_rel=0.1, what=f"{gold_file} latent")
    print(f"{gold_file}: S={gold['S']} order {gold['order']} alpha={gold['alpha_type']}: latent rel-L2 {r:.3e} max-rel {m:.3e}")


def test_non_square_latent_matches_oracle():
    """A 16 x 24 latent of the tiny model, order 2, S = 6, against the oracle loop run here on the CPU."""
    from gligen_b200.spec import NAMED_CONFIGS, synthetic_state_dict
    from oracle import gen_golden_dpm as GD
    from oracle import gen_golden_unipc as GU
    cfg = NAMED_CONFIGS["tiny"]
    x = torch.randn(2, 4, 16, 24, generator=torch.Generator().manual_seed(16024))
    _, _, lat = _sample(cfg, 2, 6, 6, 2, [1, 0, 0], x=x)
    inp, extra, mask, z0 = GD.case_inputs(cfg, 2, 6)
    ref = GU.oracle_latent(cfg, synthetic_state_dict(cfg, 0), inp, extra, mask, z0, 6, 2, [1, 0, 0], x=x)
    r, m = assert_close(lat, ref, rel=6e-2, max_rel=0.1, what="tiny 16x24 order 2 latent")
    print(f"tiny 16x24 order 2 S=6: latent rel-L2 {r:.3e} max-rel {m:.3e}")
