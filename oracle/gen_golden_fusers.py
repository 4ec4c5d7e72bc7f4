"""Pin the gatedCA / gatedSA2 oracle (oracle/fuser_oracle.py) against the REAL reference and write tests/golden/fuser_*.pt.
(authoring container only: needs /root/reference)

    python oracle/gen_golden_fusers.py [--full]

For every configuration the unmodified reference UNetModel is built with fuser_type="gatedCA" or "gatedSA2", the seeded synthetic
weights (gligen_b200.spec.synthetic_state_dict) are loaded STRICTLY - which pins the key / shape inventory of
gligen_b200.spec.unet_param_shapes for both fusers - and one grounded and one null-grounding forward run at fuser scale 1 and 0.5
on seeded inputs.  The oracle must agree to fp32 round-off; the reference eps become the fixtures (inputs are regenerated from the
seeds by gligen_b200.synth.make_inputs, weights by synthetic_state_dict).  Two reference PLMS loops with scheduled sampling on small
320-channel gatedCA / gatedSA2 models (fuser_plms_*.pt) pin the samplers' handling of each fuser type end to end.
"""
from __future__ import annotations

import argparse
import os
import sys
import time
from dataclasses import replace

import torch

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)
from oracle import ref_harness as RH  # noqa: E402

ROOT = RH.mount("dir")

from gligen_b200 import synth  # noqa: E402
from gligen_b200.spec import NAMED_CONFIGS, SAMPLING_GATED_CA, SAMPLING_HED_GATED_SA2, TINY, synthetic_state_dict  # noqa: E402
from oracle import fuser_oracle as FO  # noqa: E402
from oracle import unet_oracle as UO  # noqa: E402

GOLD = os.path.join(REPO, "tests", "golden")
SEED = 2
# (fixture name, config, batch, grounding objects passed to synth.make_inputs); a text-tokenizer gatedSA2 model is not a named
# config (make_inputs' default object count, 30, is not square): it runs at 16 boxes = a 4 x 4 grid, which the 2 x 2 middle block
# of the tiny UNet downsamples
TINY_CASES = [("tiny_gated_ca", NAMED_CONFIGS["tiny_gated_ca"], 2, 6), ("tiny_text_image_gated_ca", NAMED_CONFIGS["tiny_text_image_gated_ca"], 2, 5),
              ("tiny_keypoint_gated_ca", NAMED_CONFIGS["tiny_keypoint_gated_ca"], 2, 0), ("tiny_hed_gated_sa2", NAMED_CONFIGS["tiny_hed_gated_sa2"], 2, 0),
              ("tiny_gated_sa2_text", replace(TINY, fuser_type="gatedSA2"), 2, 16)]
FULL_CASES = [("sd14_box_text_gated_ca", NAMED_CONFIGS["sd14_box_text_gated_ca"], 1, 30), ("sd14_hed_gated_sa2", NAMED_CONFIGS["sd14_hed_gated_sa2"], 1, 0)]


def ref_model(cfg):
    """The reference UNetModel for `cfg`, with its fuser type (oracle/ref_harness.ref_model builds gatedSA only)."""
    from ldm.modules.diffusionmodules.openaimodel import UNetModel
    assert RH.is_reference_module(UNetModel)
    kw = {}
    if cfg.spatial:
        RH.shim_timm()
        kw["grounding_tokenizer"], kw["grounding_downsampler"] = RH.spatial_configs(cfg)
    else:
        tok = {
            "text": ("ldm.modules.diffusionmodules.text_grounding_net.PositionNet", dict(in_dim=cfg.tok_in_dim, out_dim=cfg.tok_out_dim)),
            "text_image": ("ldm.modules.diffusionmodules.text_image_grounding_net.PositionNet", dict(in_dim=cfg.tok_in_dim, out_dim=cfg.tok_out_dim)),
            "keypoint": ("ldm.modules.diffusionmodules.keypoint_grounding_net.PositionNet", dict(max_persons_per_image=cfg.max_persons, out_dim=cfg.tok_out_dim)),
        }[cfg.tokenizer]
        kw["grounding_tokenizer"] = dict(target=tok[0], params=tok[1])
    m = UNetModel(image_size=cfg.image_size, in_channels=cfg.in_channels, out_channels=cfg.out_channels, model_channels=cfg.model_channels,
                  attention_resolutions=list(cfg.attention_resolutions), num_res_blocks=cfg.num_res_blocks, channel_mult=list(cfg.channel_mult),
                  num_heads=cfg.num_heads, transformer_depth=1, context_dim=cfg.context_dim, fuser_type=cfg.fuser_type, use_checkpoint=True,
                  inpaint_mode=cfg.inpaint_mode, **kw)
    return m.eval()


def set_scale(model, scale):
    """Every fuser's .scale, whatever its type (set_alpha_scale of gligen_inference.py:24-28 does not match GatedSelfAttentionDense2)."""
    from ldm.modules.attention import GatedCrossAttentionDense, GatedSelfAttentionDense, GatedSelfAttentionDense2
    n = 0
    for m in model.modules():
        if type(m) in (GatedCrossAttentionDense, GatedSelfAttentionDense, GatedSelfAttentionDense2):
            m.scale = scale
            n += 1
    assert n > 0


@torch.no_grad()
def run(name, cfg, B, max_objs):
    t0 = time.time()
    sd = synthetic_state_dict(cfg, 0)
    model = ref_model(cfg)
    ref_keys = [(k, tuple(v.shape)) for k, v in model.state_dict().items()]
    missing, unexpected = model.load_state_dict(sd, strict=True)
    assert not missing and not unexpected
    mine = [(k, tuple(v.shape)) for k, v in sd.items()]
    assert sorted(ref_keys) == sorted(mine), f"{name}: state-dict keys / shapes differ from the reference"
    gin = RH.ref_grounding_input(cfg)
    model.grounding_tokenizer_input = gin
    inp = synth.make_inputs(cfg, B, max_objs, seed=SEED)
    grounding = gin.prepare(inp["batch"])
    ts = torch.tensor([981, 501][:B])
    gextra = inp.get("grounding_extra_input")
    out = {"config": name, "fuser_type": cfg.fuser_type, "tokenizer": cfg.tokenizer, "B": B, "max_objs": max_objs, "seed": SEED,
           "timesteps": ts, "n_keys": len(ref_keys), "forward": {}, "oracle_vs_reference_max_abs": {}}
    for scale in (1.0, 0.5):
        set_scale(model, scale)
        full = dict(x=inp["x"], timesteps=ts, context=inp["context"], grounding_input=grounding, inpainting_extra_input=None,
                    grounding_extra_input=gextra)
        e_c = model(full)
        null = dict(full, context=inp["uc"])
        del null["grounding_input"]                    # -> get_null_input() (openaimodel.py:422-426)
        e_u = model(null)
        o_c = FO.unet_forward(cfg, sd, inp["x"], ts, inp["context"], inp["grounding_input"], scale, grounding_extra_input=gextra)
        o_u = FO.unet_forward(cfg, sd, inp["x"], ts, inp["uc"], UO.null_grounding(cfg, inp["grounding_input"]), scale, grounding_extra_input=gextra)
        errs = ((o_c - e_c).abs().max().item(), (o_u - e_u).abs().max().item())
        print(f"{name}: scale {scale} oracle vs reference max-abs cond {errs[0]:.3e} null {errs[1]:.3e} (eps max {e_c.abs().max():.3f})", flush=True)
        assert max(errs) <= 2e-5 * max(1.0, e_c.abs().max().item()), (name, errs)
        out["forward"][scale] = {"eps_cond": e_c.clone(), "eps_null": e_u.clone()}
        out["oracle_vs_reference_max_abs"][scale] = errs
    torch.save(out, os.path.join(GOLD, f"fuser_{name}.pt"))
    print(f"{name}: {len(ref_keys)} keys, wrote fuser_{name}.pt ({time.time() - t0:.1f} s)", flush=True)


# reference PLMS loops with scheduled sampling (S = 4, alpha_type [0.3, 0, 0.7] -> alphas [1, 0, 0, 0]): from step 2 on the
# reference's set_alpha_scale sets gatedCA fusers to 0 but leaves gatedSA2 fusers at 1, and restore_first_conv_from_SD swaps in SD's
# first conv (for the hed model: the 4-channel conv, the downsampler planes dropped)
PLMS_CASES = [("sampling_gated_ca", SAMPLING_GATED_CA, 2, 6), ("sampling_hed_gated_sa2", SAMPLING_HED_GATED_SA2, 1, 0)]
PLMS_S, PLMS_ALPHA, PLMS_GUIDANCE = 4, [0.3, 0.0, 0.7], 7.5


@torch.no_grad()
def run_plms(name, cfg, B, max_objs):
    t0 = time.time()
    sd = synthetic_state_dict(cfg, 0)
    model = ref_model(cfg)
    missing, unexpected = model.load_state_dict(sd, strict=True)
    assert not missing and not unexpected
    inp = synth.make_inputs(cfg, B, max_objs, seed=SEED)
    lat, secs = RH.run_reference_sampler(cfg, sd, inp, "plms", PLMS_S, PLMS_ALPHA, guidance=PLMS_GUIDANCE, model=model, verbose=False)
    assert model.first_conv_type == "SD"
    scales = sorted({m.scale for m in model.modules() if type(m).__name__ in ("GatedCrossAttentionDense", "GatedSelfAttentionDense2")})
    assert scales == ([1] if cfg.fuser_type == "gatedSA2" else [0]), scales      # the fusers' scale at the last step
    torch.save({"config": name, "fuser_type": cfg.fuser_type, "B": B, "max_objs": max_objs, "seed": SEED, "S": PLMS_S, "alpha_type": PLMS_ALPHA,
                "guidance": PLMS_GUIDANCE, "noise_seed": 1234, "latent": lat.clone(), "final_fuser_scales": scales},
               os.path.join(GOLD, f"fuser_plms_{name}.pt"))
    print(f"{name}: reference PLMS S={PLMS_S} alpha={PLMS_ALPHA}: latent std {lat.std():.3f}, final fuser scales {scales} "
          f"({secs:.1f} s sampling, {time.time() - t0:.1f} s total); wrote fuser_plms_{name}.pt", flush=True)


def refusal_message():
    """The reference's own message for a gatedSA2 model fed a non-square token count (6 boxes)."""
    cfg = replace(TINY, fuser_type="gatedSA2")
    model = ref_model(cfg)
    model.load_state_dict(synthetic_state_dict(cfg, 0), strict=True)
    gin = RH.ref_grounding_input(cfg)
    model.grounding_tokenizer_input = gin
    inp = synth.make_inputs(cfg, 1, 6, seed=SEED)
    try:
        with torch.no_grad():
            model(dict(x=inp["x"], timesteps=torch.tensor([981]), context=inp["context"], grounding_input=gin.prepare(inp["batch"])))
    except AssertionError as e:
        print(f"gatedSA2 with 6 grounding tokens: AssertionError: {e}")
        return
    raise RuntimeError("the reference accepted a non-square grounding token count")


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("--full", action="store_true", help="also the SD-1.4-sized gatedCA / gatedSA2 models")
    a = ap.parse_args()
    torch.set_num_threads(os.cpu_count())
    os.chdir(ROOT)
    only = os.environ.get("ONLY")
    refusal_message()
    for name, cfg, B, n in TINY_CASES + (FULL_CASES if a.full else []):
        if only is None or name in only.split(","):
            run(name, cfg, B, n)
    for name, cfg, B, n in PLMS_CASES:
        if only is None or name in only.split(","):
            run_plms(name, cfg, B, n)
