#!/usr/bin/env python
"""Pin tests/clip_vision_oracle.py against the installed `transformers` CLIPVisionModelWithProjection (the image tower of the
CLIPModel that gligen_inference.prepare_batch builds) and write tests/golden/clip_vision_{tiny,sd14}.pt.
    python scripts/gen_golden_clip_vision.py

Weights, pixel values and the projection matrix are seeded synthetic (gligen_b200.clip_vision); the weights are loaded strictly.
To keep the fixtures small they hold what the tests cannot regenerate: the library's pooler_output and image_embeds, the
float64 'after_reproject' features (gligen_inference.py:114-116) with synthetic_projection_matrix(768, PROJ_SEED), the rows
TOKENS of last_hidden_state (class token, first / middle / last patches), a corner of the pixel values (checks that the seeded
pixels are regenerated bit for bit), and the library model's own bf16-autocast gap over the FULL outputs (CPU
torch.autocast(bfloat16) against fp32: rel-L2 and max-abs / max|ref|), the tolerance denominator of the GPU tests."""
import os
import sys

import torch

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)
sys.path.insert(0, os.path.join(REPO, "tests"))
from gligen_b200.clip_vision import (NAMED_CLIP_VISION_CONFIGS, synthetic_clip_vision_state_dict, synthetic_pixel_values,  # noqa: E402
                                     synthetic_projection_matrix)
from clip_vision_oracle import clip_vision_forward, gligen_image_feature  # noqa: E402

GOLD = os.path.join(REPO, "tests", "golden")
TOKENS = [0, 1, 2, 127, 128, 255, 256]
PROJ_SEED = 7


def gap(a, b):
    a, b = a.float(), b.float()
    return ((a - b).norm() / b.norm()).item(), ((a - b).abs().max() / b.abs().max()).item()


def run_vision(name, N, seed):
    import transformers
    from transformers import CLIPVisionConfig, CLIPVisionModelWithProjection
    cfg = NAMED_CLIP_VISION_CONFIGS[f"{name}_clip_vision"]
    hf = CLIPVisionConfig(hidden_size=cfg.width, intermediate_size=cfg.ffn, num_hidden_layers=cfg.layers, num_attention_heads=cfg.heads,
                          image_size=cfg.image_size, patch_size=cfg.patch, projection_dim=cfg.projection, hidden_act="quick_gelu",
                          layer_norm_eps=cfg.eps, attn_implementation="eager")
    model = CLIPVisionModelWithProjection(hf).eval()
    sd = synthetic_clip_vision_state_dict(cfg, 0)
    missing, unexpected = model.load_state_dict(sd, strict=False)
    assert not unexpected and all(k.endswith("position_ids") for k in missing), (missing, unexpected)
    px = synthetic_pixel_values(N, seed)
    P = synthetic_projection_matrix(cfg.projection, PROJ_SEED)
    post = model.vision_model.post_layernorm
    with torch.no_grad():
        out = model(pixel_values=px)
        pooler = post(out.last_hidden_state[:, 0])
        z, pooled, emb = clip_vision_forward(cfg, sd, px)
        with torch.autocast("cpu", dtype=torch.bfloat16):
            lo = model(pixel_values=px)
            feat_lo = gligen_image_feature(lo.image_embeds, P)
        pooler_lo = post(lo.last_hidden_state[:, 0].float())
    errs = tuple((a - b).abs().max().item() for a, b in ((z, out.last_hidden_state), (pooled, pooler), (emb, out.image_embeds)))
    print(f"{name}: N={N} oracle vs transformers {transformers.__version__} max-abs last_hidden_state / pooler_output / image_embeds {errs}")
    assert max(errs) <= 2e-4
    feature64 = gligen_image_feature(out.image_embeds.double(), P.double())
    gaps = {"last_hidden_state": gap(lo.last_hidden_state, out.last_hidden_state), "pooler_output": gap(pooler_lo, pooler),
            "image_embeds": gap(lo.image_embeds, out.image_embeds), "feature": gap(feat_lo, feature64)}
    print(f"{name}: bf16-autocast gap (rel-L2, max-rel) {gaps}")
    torch.save({"config": f"{name}_clip_vision", "N": N, "seed": seed, "proj_seed": PROJ_SEED, "transformers": transformers.__version__,
                "pixel_corner": px[:, :, :4, :4].clone(), "tokens": TOKENS, "last_hidden_state_rows": out.last_hidden_state[:, TOKENS].clone(),
                "pooler_output": pooler.clone(), "image_embeds": out.image_embeds.clone(), "feature64": feature64,
                "autocast_bf16_gap": gaps, "oracle_vs_library_max_abs": errs}, os.path.join(GOLD, f"clip_vision_{name}.pt"))


if __name__ == "__main__":
    run_vision("tiny", 3, 5)
    run_vision("sd14", 2, 6)
