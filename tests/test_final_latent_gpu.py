"""The tolerance the north star asks for, on the path the metric is quoted on: the FINAL LATENT of
`PLMSSampler.sample(S=50, guidance 7.5)` (102 UNet forwards) at full size, this repo's bf16 engine against the reference's
fp32 result on identical seeds, schedule and grounding inputs.

Golden: tests/golden/sd14_box_text_B1_G30_plms50.pt - the UNMODIFIED reference run on the CPU in fp32 (oracle/gen_golden.py
--plms50), alpha_type [1,0,0] and the script default [0.3,0,0.7] (scheduled sampling + first-conv swap).

Denominator (SURVEY 8d "Parity gate"): the reference's OWN reduced-precision gap, measured in the same run on the same GPU:
the reference under torch.autocast(bf16) (and fp16, fp32 eager for information) against the same fp32 golden, via
oracle/ref_run.py on the archived reference (oracle/_ref).  Stated tolerance: max-abs and rel-L2 of the engine's final
latent <= 2x the reference's bf16-autocast gap.  When the archive is absent the committed measurement
(tests/golden/final_latent_gaps.json, printed by this test where the archive was present) supplies the denominator."""
import json
import os
import subprocess
import sys
from functools import partial

import pytest
import torch

from conftest import GOLD, ROOT, rel_l2
from gligen_b200 import synth
from gligen_b200.pipeline import alpha_generator, build_model, sampler_inputs, set_alpha_scale, to_device

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
GAPS_FILE = os.path.join(GOLD, "final_latent_gaps.json")
FACTOR = 2.0


def engine_final_latent(name, B, max_objs, S, atype):
    from ldm.models.diffusion.ldm import LatentDiffusion
    from ldm.models.diffusion.plms import PLMSSampler
    cfg, model = build_model(name, DEV)
    inp = synth.make_inputs(cfg, B, max_objs, seed=2)
    diffusion = LatentDiffusion(linear_start=0.00085, linear_end=0.012, timesteps=1000).to(DEV)
    sampler = PLMSSampler(diffusion, model, alpha_generator_func=partial(alpha_generator, type=atype), set_alpha_scale=set_alpha_scale)
    t = {k: v.to(DEV) for k, v in inp.items() if isinstance(v, torch.Tensor)}
    input, mask, x0 = sampler_inputs(cfg, model, t, to_device(inp["batch"], DEV))
    cwd = os.getcwd()
    os.chdir(GOLD)                         # SD_input_conv_weight_bias.pth (restore_first_conv_from_SD reads it CWD-relative)
    try:
        torch.manual_seed(1234)
        lat = sampler.sample(S=S, shape=(B, cfg.in_channels, cfg.image_size, cfg.image_size), input=input, uc=t["uc"],
                             guidance_scale=7.5, mask=mask, x0=x0)
    finally:
        os.chdir(cwd)
    return lat.float().cpu()


def reference_on_gpu(name, B, max_objs, S, atype, tmp_path):
    """reference fp32 / bf16-autocast / fp16-autocast final latents on this GPU (None when oracle/_ref is absent)."""
    if not os.path.exists(os.path.join(ROOT, "oracle", "_ref", "gligen_reference.zip")):
        return None
    out = os.path.join(str(tmp_path), "ref.pt")
    cmd = [sys.executable, os.path.join(ROOT, "oracle", "ref_run.py"), "--config", name, "--B", str(B), "--max-objs", str(max_objs),
           "--S", str(S), "--alpha", ",".join(str(a) for a in atype), "--device", DEV, "--autocasts", "none,bf16,fp16", "--out", out]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=1500, cwd=ROOT)
    assert r.returncode == 0, r.stdout[-1500:] + r.stderr[-3000:]
    return torch.load(out)["latents"]


def gap(a, ref):
    d = (a.float() - ref.float())
    return {"max_abs": d.abs().max().item(), "rel_l2": (d.norm() / ref.float().norm()).item()}


@pytest.mark.parametrize("atype", [[1, 0, 0], [0.3, 0, 0.7]])
def test_final_latent_plms50(atype, tmp_path):
    gold = torch.load(os.path.join(GOLD, "sd14_box_text_B1_G30_plms50.pt"))
    run = gold["runs"][str(list(atype))]
    ref = run["latent"]
    S, B, max_objs = gold["S"], gold["B"], gold["max_objs"]
    mine = gap(engine_final_latent(gold["cfg"], B, max_objs, S, atype), ref)
    key = f"{gold['cfg']}_B{B}_G{max_objs}_plms{S}_{atype}"
    refs = reference_on_gpu(gold["cfg"], B, max_objs, S, atype, tmp_path)
    rec = {"latent_max": ref.abs().max().item(), "latent_std": ref.std().item(), "engine_bf16": mine}
    if refs is not None:
        rec.update({"reference_bf16_autocast": gap(refs["bf16"], ref), "reference_fp16_autocast": gap(refs["fp16"], ref),
                    "reference_fp32_gpu_eager": gap(refs["none"], ref), "denominator": "measured in this run (oracle/_ref on this GPU)"})
        print(f"\nGAPS {json.dumps({key: rec})}")      # the record tests/golden/final_latent_gaps.json keeps per key
        den = rec["reference_bf16_autocast"]
    else:
        assert os.path.exists(GAPS_FILE), "neither oracle/_ref nor the committed denominator (tests/golden/final_latent_gaps.json) is present"
        den = json.load(open(GAPS_FILE))[key]["reference_bf16_autocast"]
        rec["denominator"] = "committed measurement (tests/golden/final_latent_gaps.json)"
    print(f"\nFINAL LATENT {key}: max|latent| {rec['latent_max']:.2f} std {rec['latent_std']:.2f}")
    for k, v in rec.items():
        if isinstance(v, dict):
            print(f"   {k:28s} max-abs {v['max_abs']:.4f}  rel-L2 {v['rel_l2']:.4e}")
    print(f"   tolerance: {FACTOR} x reference bf16-autocast gap = max-abs {FACTOR * den['max_abs']:.4f}, rel-L2 {FACTOR * den['rel_l2']:.4e}  [{rec['denominator']}]")
    assert mine["max_abs"] <= FACTOR * den["max_abs"], (mine, den)
    assert mine["rel_l2"] <= FACTOR * den["rel_l2"], (mine, den)
