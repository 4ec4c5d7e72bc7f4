"""CPU: spatial grounding modalities (hed / depth / normal / sem; SURVEY 8f-4).
  * the oracle (oracle/spatial_oracle.py + the grounding_extra_input path of oracle/unet_oracle.py) against the fixtures written from
    the UNMODIFIED reference (oracle/gen_golden_spatial.py: strict state-dict load, outputs bit-identical at generation time);
  * the engine's plan for these models (gligen_b200/spatial.py: ConvNeXt packing with padded 96-channel rows, folded layer scale,
    patch-row convolutions, fused resize, downsampler planes into the first conv, SD first-conv swap by zero weights) executed with the
    torch-fp32 checker ops;
  * the drop-in module surface (UNetModel with grounding_downsampler, adapters at the reference's import paths)."""
import os

import pytest
import torch

from conftest import GOLD
from gligen_b200 import synth
from gligen_b200.engine import Engine
from gligen_b200.spec import NAMED_CONFIGS, SPATIAL_MAP_KEY, synthetic_state_dict
from oracle import unet_oracle as UO
from ref_ops import RefOps

TINY = ["tiny_hed", "tiny_canny", "tiny_depth", "tiny_normal", "tiny_sem"]
NON_SQUARE = ["tiny_hed_192x320", "tiny_normal_300x224", "tiny_sem_300x224"]       # fixtures of H x W maps


def _load(name):
    g = torch.load(os.path.join(GOLD, f"spatial_{name}.pt"))
    cfg = NAMED_CONFIGS[g["config"]]
    inp = synth.make_inputs(cfg, g["B"], seed=g["seed"], map_size=g.get("map_size"))
    return cfg, g, inp, torch.tensor(g["timesteps"])


@pytest.mark.parametrize("name", NON_SQUARE)
def test_non_square_fixture(name):
    """The fixture's map is the non-square one its name says, and the oracle matched the reference on it when it was written."""
    cfg, g, inp, _ = _load(name)
    H, W = (int(v) for v in name.rsplit("_", 1)[1].split("x"))
    assert tuple(g["map_size"]) == (H, W) and H != W
    assert tuple(inp["grounding_extra_input"].shape[2:]) == (H, W)
    assert max(g["oracle_vs_reference_max_abs"].values()) <= 2e-4


@pytest.mark.parametrize("name", TINY + NON_SQUARE)
def test_oracle_matches_reference_fixture(name):
    cfg, g, inp, ts = _load(name)
    sd = synthetic_state_dict(cfg, 0)
    taps = {}
    e_c = UO.unet_forward(cfg, sd, inp["x"], ts, inp["context"], inp["grounding_input"], 1.0, taps=taps, grounding_extra_input=inp["grounding_extra_input"])
    e_n = UO.unet_forward(cfg, sd, inp["x"], ts, inp["uc"], UO.null_grounding(cfg, inp["grounding_input"]), 1.0,
                          grounding_extra_input=inp["grounding_extra_input"])
    for got, key in ((taps["objs"], "objs"), (taps["downsample_net"], "ds"), (e_c, "eps_cond"), (e_n, "eps_null")):
        assert (got - g[key]).abs().max() <= 2e-5, key


@pytest.mark.parametrize("name", TINY + NON_SQUARE)
def test_engine_plan_matches_reference(name):
    cfg, g, inp, ts = _load(name)
    eng = Engine(cfg, RefOps())
    eng.load_state_dict(synthetic_state_dict(cfg, 0))
    gx = inp["grounding_extra_input"]
    e_c = eng.forward(inp["x"], ts, inp["context"], inp["grounding_input"], None, gx)
    e_n = eng.forward(inp["x"], ts, inp["uc"], None, None, gx)
    c2, n2 = eng.forward_cfg(inp["x"], ts, inp["context"], inp["uc"], inp["grounding_input"], None, gx)
    for got, key in ((e_c, "eps_cond"), (e_n, "eps_null"), (c2, "eps_cond"), (n2, "eps_null")):
        assert (got - g[key]).abs().max() < 1e-4, key
    # the tokenizer and the downsampler are static steps: a second timestep does not re-run them
    P = eng.plans[(g["B"], cfg.spatial_tokens, 77)]
    names = [n for n, _, st, _ in P.steps if st]
    assert any(n.startswith("cx.s2.8") for n in names) and "pn.l4" in names and any(n.startswith("ds.") for n in names)
    before = eng.ops.launches
    eng.forward(inp["x"], ts, inp["context"], inp["grounding_input"], None, gx)          # (re)computes the static part for these inputs
    with_static = eng.ops.launches - before
    before = eng.ops.launches
    eng.forward(inp["x"], ts - 1, inp["context"], inp["grounding_input"], None, gx)
    per_step = eng.ops.launches - before
    assert with_static - per_step == len(names)


def test_sd_first_conv_swap_on_a_spatial_model():
    """restore_first_conv_from_SD on a model with a grounding downsampler: the reference swaps in a 4-channel conv and stops
    concatenating the downsampler planes (openaimodel.py:407-411, 441); the engine keeps its plan and zeroes those weights."""
    cfg, g, inp, ts = _load("tiny_depth")
    sd = synthetic_state_dict(cfg, 0)
    eng = Engine(cfg, RefOps())
    eng.load_state_dict(sd)
    gx = inp["grounding_extra_input"]
    eng.forward(inp["x"], ts, inp["context"], inp["grounding_input"], None, gx)
    gen = torch.Generator().manual_seed(4)
    w4, b4 = torch.randn(cfg.model_channels, 4, 3, 3, generator=gen) * 0.2, torch.randn(cfg.model_channels, generator=gen) * 0.1
    nplans = len(eng.plans)
    eng.set_first_conv(w4, b4)
    assert len(eng.plans) == nplans
    got = eng.forward(inp["x"], ts, inp["context"], inp["grounding_input"], None, gx)
    sd2 = dict(sd); sd2["input_blocks.0.0.weight"], sd2["input_blocks.0.0.bias"] = w4, b4
    ref = UO.unet_forward(cfg, sd2, inp["x"], ts, inp["context"], inp["grounding_input"], 1.0, grounding_extra_input=None)   # "SD": no planes
    assert (got - ref).abs().max() < 1e-4


def test_drop_in_surface():
    from gligen_b200.pipeline import build_model, sampler_inputs
    for name in ("tiny_hed", "tiny_sem"):
        cfg, model = build_model(name, device="cpu")
        assert model.first_conv_type == "GLIGEN" and model.additional_channel_from_downsampler == cfg.ds_out_dim
        assert type(model.downsample_net).__module__ == f"ldm.modules.diffusionmodules.{cfg.tokenizer}_grounding_downsampler"
        assert type(model.position_net).__module__ == f"ldm.modules.diffusionmodules.{cfg.tokenizer}_grounding_net"
        assert set(model.state_dict()) == set(synthetic_state_dict(cfg, 0))
        inp = synth.make_inputs(cfg, 2, seed=3)
        input, mask, x0 = sampler_inputs(cfg, model, inp, inp["batch"])
        key = SPATIAL_MAP_KEY[cfg.tokenizer]
        assert input["grounding_extra_input"] is inp["batch"][key] and set(input["grounding_input"]) == {key, "mask"}
        null = model.grounding_tokenizer_input.get_null_input()
        assert null[key].shape == inp["batch"][key].shape and float(null[key].abs().sum()) == 0 and null["mask"].shape == (2,)
        with pytest.raises(RuntimeError):
            model(input)                 # CUDA only: no CPU fallback
        # the SD first-conv swap narrows the module's conv to 4 channels (like the reference); loading a checkpoint afterwards restores it
        import os
        from conftest import GOLD
        if cfg.model_channels == 320:
            continue                     # the bundled SD conv has 320 output channels: only full-size models can take it
        sdw = {"weight": torch.randn(cfg.model_channels, 4, 3, 3), "bias": torch.randn(cfg.model_channels)}
        cwd = os.getcwd()
        import tempfile
        with tempfile.TemporaryDirectory() as d:
            torch.save(sdw, os.path.join(d, "SD_input_conv_weight_bias.pth"))
            os.chdir(d)
            try:
                model.restore_first_conv_from_SD()
            finally:
                os.chdir(cwd)
        assert model.first_conv_type == "SD" and model.input_blocks[0][0].weight.shape[1] == 4
        model.load_state_dict(synthetic_state_dict(cfg, 0))
        assert model.first_conv_type == "GLIGEN" and model.input_blocks[0][0].weight.shape[1] == cfg.first_conv_in
