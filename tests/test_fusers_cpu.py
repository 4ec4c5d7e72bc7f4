"""CPU: UNets built with the gatedCA and gatedSA2 fusers (reference attention.py:190-297).

State-dict inventory and strict loads of the drop-in UNetModel, the oracle and the engine's plan (run with the fp32 checker ops)
against the reference fixtures of oracle/gen_golden_fusers.py, set_alpha_scale semantics per fuser type, the refusals, a checkpoint
round trip, and the arithmetic of glg_grid_resample_gate restated in torch against the float64 bound of tests/fuser_checks.py -
which accepts the faithful arithmetic and rejects realistic mistakes."""
import os
from dataclasses import replace

import pytest
import torch

from conftest import GOLD
from fuser_checks import FuserRefOps, resample_gate_check, stats_check
from gligen_b200 import synth
from gligen_b200.engine import Engine
from gligen_b200.spec import NAMED_CONFIGS, TINY, synthetic_state_dict, unet_param_shapes
from oracle import fuser_oracle as FO
from oracle import unet_oracle as UO

CASES = [("tiny_gated_ca", None), ("tiny_text_image_gated_ca", None), ("tiny_keypoint_gated_ca", None), ("tiny_hed_gated_sa2", None),
         ("tiny_gated_sa2_text", replace(TINY, fuser_type="gatedSA2"))]


def _case(name, cfg):
    gold = torch.load(os.path.join(GOLD, f"fuser_{name}.pt"))
    cfg = cfg or NAMED_CONFIGS[name]
    return cfg, gold, synth.make_inputs(cfg, gold["B"], gold["max_objs"], seed=gold["seed"])


def _model(cfg):
    from gligen_b200.pipeline import model_config
    from ldm.util import instantiate_from_config
    return instantiate_from_config(model_config(cfg))


@pytest.mark.parametrize("name", ["tiny_gated_ca", "tiny_hed_gated_sa2", "sd14_box_text_gated_ca", "sd14_hed_gated_sa2"])
def test_state_dict_inventory(name):
    """The drop-in UNetModel has exactly unet_param_shapes' keys; gatedCA drops fuser.linear and projects K / V from context_dim,
    gatedSA2 has gatedSA's key set; a synthetic state dict loads strictly."""
    cfg = NAMED_CONFIGS[name]
    shapes = unet_param_shapes(cfg)
    sa = unet_param_shapes(replace(cfg, fuser_type="gatedSA"))
    if cfg.fuser_type == "gatedSA2":
        assert shapes == sa
    else:
        fk = [k for k in shapes if ".fuser." in k]
        assert not any(".fuser.linear." in k for k in fk)
        assert all(shapes[k] == (int(shapes[k][0]), cfg.context_dim) for k in fk if k.endswith(("attn.to_k.weight", "attn.to_v.weight")))
        assert set(sa) - set(shapes) == {k for k in sa if ".fuser.linear." in k}
    if name.startswith("sd14"):
        return
    m = _model(cfg)
    body = {k: v for k, v in shapes.items() if not k.startswith(("position_net.", "downsample_net."))}
    sd = m.state_dict()
    assert all(tuple(sd[k].shape) == tuple(v) for k, v in body.items())
    m.load_state_dict(synthetic_state_dict(cfg, 0), strict=True)


@pytest.mark.parametrize("name,cfg", CASES)
def test_fixture_pins_reference_inventory(name, cfg):
    cfg, gold, _ = _case(name, cfg)
    assert gold["n_keys"] == len(unet_param_shapes(cfg)) and gold["fuser_type"] == cfg.fuser_type


@pytest.mark.parametrize("name,cfg", CASES)
def test_oracle_matches_reference(name, cfg):
    cfg, gold, inp = _case(name, cfg)
    sd = synthetic_state_dict(cfg, 0)
    ge = inp.get("grounding_extra_input")
    for scale, f in gold["forward"].items():
        e_c = FO.unet_forward(cfg, sd, inp["x"], gold["timesteps"], inp["context"], inp["grounding_input"], scale, grounding_extra_input=ge)
        e_u = FO.unet_forward(cfg, sd, inp["x"], gold["timesteps"], inp["uc"], UO.null_grounding(cfg, inp["grounding_input"]), scale,
                              grounding_extra_input=ge)
        assert (e_c - f["eps_cond"]).abs().max() <= 2e-5 and (e_u - f["eps_null"]).abs().max() <= 2e-5


@pytest.mark.parametrize("name,cfg", CASES)
def test_engine_plan_matches_reference(name, cfg):
    """The engine's gatedCA / gatedSA2 plans (weight packing, K/V-only GEMM, grounding-row attention, resample step, stats
    wiring) with the fp32 checker ops, single and CFG-batched, against the reference eps."""
    cfg, gold, inp = _case(name, cfg)
    eng = Engine(cfg, FuserRefOps())
    eng.load_state_dict(synthetic_state_dict(cfg, 0))
    ts, ge = gold["timesteps"], inp.get("grounding_extra_input")
    for scale, f in gold["forward"].items():
        eng.set_scale(scale)
        e_c = eng.forward(inp["x"], ts, inp["context"], inp["grounding_input"], None, ge)
        c2, u2 = eng.forward_cfg(inp["x"], ts, inp["context"], inp["uc"], inp["grounding_input"], None, ge)
        for got, ref in ((e_c, f["eps_cond"]), (c2, f["eps_cond"]), (u2, f["eps_null"])):
            assert (got - ref).abs().max() < 5e-5
    P = next(iter(eng.plans.values()))
    names = [n for n, fu, st, _ in P.steps if fu and not st]
    per_layer = 5 if cfg.fuser_type == "gatedCA" else 6          # (q | kv), core, out, [resample,] ff.1, ff.2
    assert len(names) == 16 * per_layer
    assert sum(n.endswith(".fuser.resample") for n in names) == (16 if cfg.fuser_type == "gatedSA2" else 0)


def test_set_alpha_scale_semantics():
    """The reference's set_alpha_scale matches GatedCrossAttentionDense (scheduled sampling drives gatedCA fusers) but not
    GatedSelfAttentionDense2 (those stay at 1); a scale set by hand on any fuser reaches the engine."""
    from gligen_b200.pipeline import set_alpha_scale
    from ldm.modules.attention import GatedCrossAttentionDense, GatedSelfAttentionDense, GatedSelfAttentionDense2
    for name, cls in (("tiny_gated_ca", GatedCrossAttentionDense), ("tiny_hed_gated_sa2", GatedSelfAttentionDense2), ("tiny", GatedSelfAttentionDense)):
        m = _model(NAMED_CONFIGS[name])
        fusers = [x for x in m.modules() if type(x) == cls]
        assert len(fusers) == 16 and fusers == m._fusers
        set_alpha_scale(m, 0.0)
        assert all(f.scale == (1 if cls is GatedSelfAttentionDense2 else 0.0) for f in fusers)
        fusers[3].scale = 0.25

        class Eng:
            scales = None

            def set_scale(self, s):
                self.scales = s
        e = Eng()
        m._sync_scales(e)
        assert e.scales[3] == 0.25 and len(e.scales) == 16


def test_refusals():
    """gatedSA2: a non-square grounding token count fails with the reference's message; a non-square latent is refused."""
    cfg = replace(TINY, fuser_type="gatedSA2")
    eng = Engine(cfg, FuserRefOps())
    eng.load_state_dict(synthetic_state_dict(cfg, 0))
    inp = synth.make_inputs(cfg, 1, 6, seed=2)
    with pytest.raises(AssertionError, match="Grounding tokens must be square rootable"):
        eng.forward(inp["x"], torch.tensor([981]), inp["context"], inp["grounding_input"])
    inp = synth.make_inputs(cfg, 1, 16, seed=2)
    x = torch.randn(1, 4, 16, 24)
    with pytest.raises(ValueError, match="square"):
        eng.forward(x, torch.tensor([981]), inp["context"], inp["grounding_input"])
    # gatedCA has neither restriction
    ca = NAMED_CONFIGS["tiny_gated_ca"]
    eng = Engine(ca, FuserRefOps())
    eng.load_state_dict(synthetic_state_dict(ca, 0))
    inp = synth.make_inputs(ca, 1, 6, seed=2)
    e = eng.forward(torch.randn(1, 4, 16, 24), torch.tensor([981]), inp["context"], inp["grounding_input"])
    assert e.shape == (1, 4, 16, 24) and torch.isfinite(e).all()


def test_constructor_accepts_every_reference_fuser_type():
    """UNetModel takes the three fuser types the reference asserts (openaimodel.py:276); what it still refuses is refused for its
    own reason (here an unknown tokenizer), never for the fuser type."""
    from ldm.modules.diffusionmodules.openaimodel import UNetModel
    for ft in ("gatedSA", "gatedCA", "gatedSA2"):
        m = _model(replace(TINY, fuser_type=ft))
        assert m.fuser_type == ft and len(m._fusers) == 16
        with pytest.raises(NotImplementedError) as e:
            UNetModel(16, 4, 64, 4, 2, [1], fuser_type=ft, context_dim=128, grounding_tokenizer=dict(target="x"))
        assert "fuser" not in str(e.value) and "grounding_tokenizer target" in str(e.value)
    with pytest.raises(AssertionError):
        UNetModel(16, 4, 64, 4, 2, [1], fuser_type="gatedXY", context_dim=128, grounding_tokenizer=dict(target="x"))


def test_checkpoint_round_trip_gated_ca(tmp_path):
    """save_ckpt -> load_ckpt keeps fuser_type in the model config: the model it builds has gatedCA fusers and every tensor."""
    from gligen_b200 import checkpoint as CK
    from gligen_b200.pipeline import GROUNDING_INPUT, model_config
    from ldm.modules.attention import GatedCrossAttentionDense
    cfg = NAMED_CONFIGS["tiny_gated_ca"]
    sd = synthetic_state_dict(cfg, 0)
    path = os.path.join(str(tmp_path), "gligen_gated_ca.pth")
    conf = {"model": model_config(cfg), "grounding_tokenizer_input": {"target": GROUNDING_INPUT[cfg.tokenizer]},
            "diffusion": {"target": "ldm.models.diffusion.ldm.LatentDiffusion", "params": dict(linear_start=0.00085, linear_end=0.012, timesteps=1000)}}
    CK.save_ckpt(path, conf, sd)
    model, _, _, _, config = CK.load_ckpt(path, device="cpu", with_text_encoder=False)
    assert config["model"]["params"]["fuser_type"] == "gatedCA" and model.fuser_type == "gatedCA"
    assert len(model._fusers) == 16 and all(type(f) == GatedCrossAttentionDense for f in model._fusers)
    got = model.state_dict()
    assert set(got) == set(sd) and all(torch.equal(got[k], sd[k]) for k in sd)


# ---- the kernel's arithmetic, restated --------------------------------------------------------------------------------------
def _fma(a, b, c):
    return (a.double() * b.double() + c.double()).float()


def _restate(grid, x, gate, g, n, A=-0.75, align_corners=False, clamp=True, gate_after_round=False, stats_unrounded=False):
    """glg_grid_resample_gate in fp32 torch (FMA chains as in csrc/fuser.cu), with optional mistakes."""
    B, _, C = grid.shape
    o = torch.arange(n, dtype=torch.float32)
    if align_corners:
        r = o * (float(g - 1) / float(n - 1) if n > 1 else 0.0)
    else:
        r = _fma(torch.tensor(float(g) / float(n), dtype=torch.float32).expand(n), o + 0.5, torch.full((n,), -0.5))
    fl = torch.floor(r)
    t = r - fl
    c1 = lambda a: ((A + 2.0) * a - (A + 3.0)) * a * a + 1.0
    c2 = lambda a: ((A * a - 5.0 * A) * a + 8.0 * A) * a - 4.0 * A
    w = torch.stack([c2(t + 1.0), c1(t), c1(1.0 - t), c2(2.0 - t)], 1).float()      # [n, 4]
    idx = fl.long()[:, None] - 1 + torch.arange(4)[None]
    valid = (idx >= 0) & (idx < g)
    if not clamp:
        w = torch.where(valid, w, torch.zeros_like(w))
    idx = idx.clamp(0, g - 1)
    src = grid.reshape(B, g, g, C)
    acc = torch.zeros(B, n, n, C)
    for j in range(4):
        rr = torch.zeros(B, n, n, C)
        for k in range(4):
            v = src[:, idx[:, j]][:, :, idx[:, k]]                              # [B, n, n, C]
            rr = _fma(w[None, None, :, k, None].expand_as(v), v, rr)
        acc = _fma(w[None, :, j, None, None].expand_as(rr), rr, acc)
    acc = acc.reshape(B, n * n, C)
    xf = x.float()
    if gate_after_round:
        v = _fma(torch.full_like(acc, gate), acc.to(torch.bfloat16).float(), xf)
    else:
        v = _fma(torch.full_like(acc, gate), acc, xf)
    out = v.to(torch.bfloat16)
    sv = (v if stats_unrounded else out.float()).reshape(B * n * n, C // 32, 32)
    stats = torch.stack([sv.sum(2).t(), (sv * sv).sum(2).t()], -1)
    return out, stats


def _suite():
    gen = torch.Generator().manual_seed(7)
    for g, n in ((1, 4), (2, 4), (2, 2), (4, 8), (4, 2), (8, 16), (8, 8), (4, 1), (8, 4)):
        for gate in (0.7, -1.3, 3.1):
            grid = torch.randn(2, g * g, 64, generator=gen)
            x = (0.1 * torch.randn(2, n * n, 64, generator=gen)).to(torch.bfloat16)
            yield g, n, gate, grid, x


def test_resample_bound_accepts_faithful_arithmetic():
    for g, n, gate, grid, x in _suite():
        out, stats = _restate(grid, x, gate, g, n)
        rep = resample_gate_check(out, x, grid, gate, g, n, what=f"g={g} n={n} gate={gate}")
        assert rep.ok, str(rep)
        assert stats_check(stats, out.reshape(-1, 64)).ok


@pytest.mark.parametrize("mutant", [dict(A=-0.5), dict(align_corners=True), dict(clamp=False), dict(gate_after_round=True),
                                    dict(stats_unrounded=True)])
def test_resample_bound_rejects_mutants(mutant):
    rejected = False
    for g, n, gate, grid, x in _suite():
        out, stats = _restate(grid, x, gate, g, n, **mutant)
        if mutant.get("stats_unrounded"):
            rejected |= not stats_check(stats, out.reshape(-1, 64)).ok
        else:
            rejected |= not resample_gate_check(out, x, grid, gate, g, n).ok
    assert rejected, mutant
