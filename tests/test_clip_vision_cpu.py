"""CPU: the CLIP image tower and prepare_batch's grounding features.  The oracle (tests/clip_vision_oracle.py) against the fixture
written from the installed transformers' CLIPVisionModelWithProjection (scripts/gen_golden_clip_vision.py); the engine's wiring
(conv-weight repack, patch padding columns, class and position rows, the head, the keys of a full CLIPModel dict, a second N
with its own workspace) executed with the torch-fp32 checker ops; ClipGroundingEncoder + pipeline.prepare_batch against the
one-item-at-a-time restatement of gligen_inference.py:146-187; the CUDA-only error."""
import os

import pytest
import torch

from clip_vision_oracle import clip_vision_forward, gligen_image_feature, prepare_batch as oracle_prepare_batch
from ref_ops import RefOps
from conftest import GOLD
from gligen_b200.clip_text import TINY_CLIP_TEXT, synthetic_clip_state_dict, synthetic_token_ids
from gligen_b200.clip_vision import (NAMED_CLIP_VISION_CONFIGS, TINY_CLIP_VISION, ClipVisionEngine, clip_vision_param_shapes,
                                     synthetic_clip_vision_state_dict, synthetic_pixel_values, synthetic_projection_matrix)
from oracle.clip_oracle import clip_text_forward

NAMES = ["tiny", "sd14"]


def fixture(name):
    """The stored library outputs plus the regenerated seeded pixel values (checked against the stored corner)."""
    g = torch.load(os.path.join(GOLD, f"clip_vision_{name}.pt"))
    g["pixel_values"] = synthetic_pixel_values(g["N"], g["seed"])
    assert torch.equal(g["pixel_values"][:, :, :4, :4], g["pixel_corner"])
    return g


def projection_matrix(D=768):
    return synthetic_projection_matrix(D, 7)


def clip_model_state_dict(text_cfg, vision_cfg, seed=0):
    """A full CLIPModel state dict: both towers, text_projection, logit_scale and the position_ids buffers older releases save."""
    sd = dict(synthetic_clip_state_dict(text_cfg, seed, prefix=""))
    sd.update(synthetic_clip_vision_state_dict(vision_cfg, seed))
    sd["text_projection.weight"] = torch.randn(vision_cfg.projection, text_cfg.width)
    sd["logit_scale"] = torch.tensor(2.6592)
    sd["text_model.embeddings.position_ids"] = torch.arange(text_cfg.max_length)[None]
    sd["vision_model.embeddings.position_ids"] = torch.arange(vision_cfg.tokens)[None]
    return sd


def test_param_shapes_are_transformers_keys():
    from transformers import CLIPVisionConfig, CLIPVisionModelWithProjection
    c = TINY_CLIP_VISION
    m = CLIPVisionModelWithProjection(CLIPVisionConfig(hidden_size=c.width, intermediate_size=c.ffn, num_hidden_layers=c.layers,
                                                       num_attention_heads=c.heads, projection_dim=c.projection, image_size=c.image_size,
                                                       patch_size=c.patch))
    ref = {k: tuple(v.shape) for k, v in m.state_dict().items() if not k.endswith("position_ids")}
    assert ref == dict(clip_vision_param_shapes(c))


@pytest.mark.parametrize("name", NAMES)
def test_oracle_matches_library_fixture(name):
    g = fixture(name)
    cfg = NAMED_CLIP_VISION_CONFIGS[f"{name}_clip_vision"]
    z, pooled, emb = clip_vision_forward(cfg, synthetic_clip_vision_state_dict(cfg, 0), g["pixel_values"])
    for got, key in ((z[:, g["tokens"]], "last_hidden_state_rows"), (pooled, "pooler_output"), (emb, "image_embeds")):
        assert (got - g[key]).abs().max() <= 2e-5, key
    assert g["proj_seed"] == 7
    f = gligen_image_feature(g["image_embeds"], projection_matrix())
    assert (f.double() - g["feature64"]).abs().max() <= 2e-5
    assert torch.allclose(g["feature64"].norm(dim=-1), torch.full((g["N"],), 28.7, dtype=torch.float64))


@pytest.mark.parametrize("name", NAMES)
def test_engine_wiring(name):
    g = fixture(name)
    cfg = NAMED_CLIP_VISION_CONFIGS[f"{name}_clip_vision"]
    eng = ClipVisionEngine(cfg, RefOps())
    eng.load_state_dict(clip_model_state_dict(TINY_CLIP_TEXT, cfg))           # the text tower's keys are ignored
    z, pooled, emb = eng.forward(g["pixel_values"])
    for got, key in ((z[:, g["tokens"]], "last_hidden_state_rows"), (pooled, "pooler_output"), (emb, "image_embeds")):
        err = (got - g[key]).abs().max().item()
        assert err <= 1e-4, (key, err)
    z_oracle = clip_vision_forward(cfg, synthetic_clip_vision_state_dict(cfg, 0), g["pixel_values"])[0]
    assert (z - z_oracle).abs().max() <= 1e-4                                  # every token row
    P = projection_matrix()
    f = eng.grounding_features(g["pixel_values"], P)
    assert (f.double() - g["feature64"]).abs().max() <= 1e-4
    z1, _, emb1 = eng.forward(g["pixel_values"][-1:])                          # another N gets its own workspace
    assert len(eng._ws) == 2
    assert (z1 - z_oracle[-1:]).abs().max() <= 1e-4 and (emb1 - g["image_embeds"][-1:]).abs().max() <= 1e-4


def test_engine_accepts_vision_model_and_bare_keys():
    g = fixture("tiny")
    cfg = TINY_CLIP_VISION
    sd = synthetic_clip_vision_state_dict(cfg, 0)
    bare = {k[len("vision_model."):] if k.startswith("vision_model.") else k: v for k, v in sd.items()}
    for d in (sd, bare):
        eng = ClipVisionEngine(cfg, RefOps())
        eng.load_state_dict(d)
        assert (eng.forward(g["pixel_values"])[2] - g["image_embeds"]).abs().max() <= 1e-4


# ---- ClipGroundingEncoder + prepare_batch ------------------------------------------------------------------------------------
def phrases(n, seed):
    """n CLIPTokenizer-style id rows of different lengths, as the processor returns one phrase: BOS, words, EOT, no padding."""
    ids = synthetic_token_ids(TINY_CLIP_TEXT, n, seed)
    eot = TINY_CLIP_TEXT.vocab_size - 1
    return [r[: int((r == eot).nonzero()[0]) + 1] for r in ids]


@pytest.fixture(scope="module")
def grounding():
    from gligen_b200.clip_grounding import ClipGroundingEncoder
    sd = clip_model_state_dict(TINY_CLIP_TEXT, TINY_CLIP_VISION)
    P = projection_matrix()
    enc = ClipGroundingEncoder(sd, P, text_config=TINY_CLIP_TEXT, vision_config=TINY_CLIP_VISION, ops=RefOps())

    def text_feature(ids):
        return clip_text_forward(TINY_CLIP_TEXT, sd, ids[None], prefix="text_model.")[1]

    def image_feature(px):
        return gligen_image_feature(clip_vision_forward(TINY_CLIP_VISION, sd, px.reshape(1, *px.shape[-3:]))[2], P)

    return enc, text_feature, image_feature


def metas():
    ph, px = phrases(4, 11), synthetic_pixel_values(4, 12)
    boxes = [[0.1, 0.1, 0.6, 0.5], [0.3, 0.2, 0.9, 0.9], [0.0, 0.5, 0.4, 1.0], [0.5, 0.0, 1.0, 0.4]]
    return {
        # generation_box_text_style: both objects carry a phrase and an image; the masks keep the text of one, the image of the other
        "style": dict(locations=boxes[:2], phrases=ph[:2], images=[px[0], px[1]], text_mask=[1, 0], image_mask=[0, 1]),
        "phrases_only": dict(locations=boxes[:3], phrases=ph[:3]),
        "images_only": dict(locations=boxes, images=[px[0], None, px[2][None], px[3]], image_mask=0.5),
        "mixed_none": dict(locations=boxes, phrases=[ph[0], None, ph[2], ph[3]], images=[None, px[1], px[2], None]),
    }


@pytest.mark.parametrize("scenario", ["style", "phrases_only", "images_only", "mixed_none"])
def test_prepare_batch_matches_reference_restatement(grounding, scenario):
    from gligen_b200.pipeline import prepare_batch
    enc, tf, imf = grounding
    meta = metas()[scenario]
    got = prepare_batch(meta, batch=2, max_objs=30, encoder=enc)
    want = oracle_prepare_batch(meta, tf, imf, batch=2, max_objs=30, text_dim=TINY_CLIP_TEXT.width, image_dim=768)
    assert set(got) == set(want) == {"boxes", "masks", "text_masks", "image_masks", "text_embeddings", "image_embeddings"}
    for k in want:
        assert got[k].shape == want[k].shape, k
        assert (got[k] - want[k]).abs().max() <= 1e-4, (scenario, k)
    n = len(meta["locations"])
    assert got["masks"][:, n:].abs().sum() == 0 and got["boxes"][:, n:].abs().sum() == 0           # padding to max_objs
    assert got["text_embeddings"][:, n:].abs().sum() == 0 and got["image_embeddings"][:, n:].abs().sum() == 0
    norms = got["image_embeddings"][0].norm(dim=-1)
    used = norms > 0
    assert torch.allclose(norms[used], torch.full_like(norms[used], 28.7), rtol=1e-5)
    assert int(used.sum()) == sum(im is not None for im in (meta.get("images") or []))


def test_phrase_batch_padding_is_invisible(grounding):
    """Phrases of different lengths in one padded forward give each phrase's own pooled EOT state."""
    enc, tf, _ = grounding
    ph = phrases(5, 21)
    batched = enc.text_features(enc.phrase_ids(ph))
    for i, p in enumerate(ph):
        assert (batched[i] - tf(p)[0]).abs().max() <= 1e-4


def test_grounding_encoder_is_cuda_only():
    from gligen_b200.clip_grounding import ClipGroundingEncoder
    from gligen_b200.pipeline import prepare_batch
    sd = clip_model_state_dict(TINY_CLIP_TEXT, TINY_CLIP_VISION)
    with pytest.raises(RuntimeError, match="CUDA"):
        ClipGroundingEncoder(sd, projection_matrix(), device="cpu", text_config=TINY_CLIP_TEXT, vision_config=TINY_CLIP_VISION)
    with pytest.raises(ValueError):
        prepare_batch(dict(locations=[[0, 0, 1, 1]], phrases=["a"]))


def test_projection_matrix_default_path_is_cwd_relative(monkeypatch, tmp_path):
    from gligen_b200.clip_grounding import ClipGroundingEncoder
    torch.save(projection_matrix(), tmp_path / "projection_matrix")
    monkeypatch.chdir(tmp_path)
    sd = clip_model_state_dict(TINY_CLIP_TEXT, TINY_CLIP_VISION)
    enc = ClipGroundingEncoder(sd, text_config=TINY_CLIP_TEXT, vision_config=TINY_CLIP_VISION, ops=RefOps())
    assert torch.equal(enc.P, projection_matrix())
