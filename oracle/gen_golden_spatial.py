"""Pin the spatial-modality oracle (oracle/spatial_oracle.py + the grounding_extra_input path of oracle/unet_oracle.py) against
the REAL reference and write tests/golden/spatial_*.pt.   (authoring container only: needs /root/reference)

    python oracle/gen_golden_spatial.py [--full]

For every configuration: the unmodified reference UNetModel (with its ConvNeXt PositionNet and GroundingDownsampler) is built
from /root/reference, the seeded synthetic weights are loaded STRICTLY (pins gligen_b200.spec's key / shape inventory), one
conditional and one null-grounding forward run on seeded maps; the oracle must agree to fp32 round-off; the reference outputs
(grounding tokens, downsampler planes, eps) become the fixtures.  `timm` / the ImageNet download are stood in for as documented
in oracle/ref_harness.shim_timm.
"""
from __future__ import annotations

import argparse
import os
import sys
import time

import torch

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)
from oracle import ref_harness as RH  # noqa: E402

ROOT = RH.mount("dir")

from gligen_b200 import synth  # noqa: E402
from gligen_b200.spec import NAMED_CONFIGS, SPATIAL_MAP_KEY, synthetic_state_dict  # noqa: E402
from oracle import unet_oracle as UO  # noqa: E402

GOLD = os.path.join(REPO, "tests", "golden")
TS = [981, 501]


def run(name: str, B: int, seed: int, plms: bool = False, map_size=None) -> None:
    """Writes spatial_{name}.pt, or spatial_{name}_{H}x{W}.pt for a map of `map_size` (H, W) instead of the default square one."""
    cfg = NAMED_CONFIGS[name]
    t0 = time.time()
    sd = synthetic_state_dict(cfg, 0)
    model = RH.ref_model(cfg)
    assert RH.is_reference_module(type(model)) and RH.is_reference_module(type(model.position_net)) and RH.is_reference_module(type(model.downsample_net))
    missing, unexpected = model.load_state_dict(sd, strict=True)
    assert not missing and not unexpected
    model.grounding_tokenizer_input = RH.ref_grounding_input(cfg)
    inp = synth.make_inputs(cfg, B, seed=seed, map_size=map_size)
    batch = inp["batch"]
    grounding = model.grounding_tokenizer_input.prepare(batch)
    ts = torch.tensor(TS[:B])
    out = {}
    with torch.no_grad():
        out["objs"] = model.position_net(**grounding)
        out["ds"] = model.downsample_net(inp["grounding_extra_input"])
        full = dict(x=inp["x"], timesteps=ts, context=inp["context"], grounding_input=grounding, inpainting_extra_input=None,
                    grounding_extra_input=inp["grounding_extra_input"])
        out["eps_cond"] = model(full)
        null = dict(full, context=inp["uc"])
        del null["grounding_input"]                    # -> get_null_input(): zero map, mask 0 (openaimodel.py:422-426)
        out["eps_null"] = model(null)
        assert model.first_conv_type == "GLIGEN"
    # the oracle on the same bits
    taps = {}
    o_c = UO.unet_forward(cfg, sd, inp["x"], ts, inp["context"], inp["grounding_input"], 1.0, taps=taps, grounding_extra_input=inp["grounding_extra_input"])
    o_n = UO.unet_forward(cfg, sd, inp["x"], ts, inp["uc"], UO.null_grounding(cfg, inp["grounding_input"]), 1.0, grounding_extra_input=inp["grounding_extra_input"])
    errs = {"objs": (taps["objs"] - out["objs"]).abs().max().item(), "ds": (taps["downsample_net"] - out["ds"]).abs().max().item(),
            "eps_cond": (o_c - out["eps_cond"]).abs().max().item(), "eps_null": (o_n - out["eps_null"]).abs().max().item()}
    print(f"{name}: B={B} oracle vs reference max-abs {errs}  ({time.time() - t0:.1f} s)", flush=True)
    for k, v in errs.items():
        assert v <= 2e-4, (name, k, v)
    extra = {}
    if plms:
        # a short reference PLMS loop with scheduled sampling: from step S/2 on the reference swaps in SD's 4-channel first conv
        # (restore_first_conv_from_SD) and stops concatenating the downsampler planes
        lat, secs = RH.run_reference_sampler(cfg, sd, inp, "plms", 4, [0.5, 0.0, 0.5], guidance=5.0, verbose=False)
        extra["plms"] = {"S": 4, "alpha_type": [0.5, 0.0, 0.5], "guidance": 5.0, "latent": lat.clone()}
        print(f"{name}: reference PLMS S=4 [0.5,0,0.5] latent std {lat.std():.3f} ({secs:.1f} s)", flush=True)
    shape = tuple(inp["grounding_extra_input"].shape[2:])
    print(f"{name}: map {shape[0]} x {shape[1]}", flush=True)
    tag = "" if map_size is None else f"_{map_size[0]}x{map_size[1]}"
    torch.save({"config": name, **extra, "B": B, "seed": seed, "timesteps": TS[:B], "map_key": SPATIAL_MAP_KEY[cfg.tokenizer],
                **({} if map_size is None else {"map_size": shape}),
                "oracle_vs_reference_max_abs": errs, **{k: v.clone() for k, v in out.items()}},
               os.path.join(GOLD, f"spatial_{name}{tag}.pt"))


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("--full", action="store_true", help="also the full-size SD-1.4 hed / sem models (1.07 B parameters each)")
    a = ap.parse_args()
    os.chdir(ROOT)
    only = os.environ.get("ONLY")
    for name in ("tiny_hed", "tiny_canny", "tiny_depth", "tiny_normal", "tiny_sem"):
        if only is None or name in only.split(","):
            run(name, 2, 11)
    # non-square maps (a 3:5 landscape and a 4:3 portrait): bicubic only (hed), bicubic + conv (normal), nearest fused into the
    # convolutions (sem); every resampling ratio there is not an integer and differs between the axes
    for name, size in (("tiny_hed", (192, 320)), ("tiny_normal", (300, 224)), ("tiny_sem", (300, 224))):
        if only is None or f"{name}_{size[0]}x{size[1]}" in only.split(","):
            run(name, 2, 11, map_size=size)
    if a.full:
        for name in ("sd14_hed", "sd14_sem"):
            run(name, 1, 12, plms=(name == "sd14_hed"))
