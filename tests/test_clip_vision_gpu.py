"""GPU: the CLIP image tower and prepare_batch's grounding features through the C ABI.

* glg_clip_vision_embed against its float64 statement rounded to bf16: every element within one bf16 ulp plus the fp32 error
  of rstd, 99.9 % within one ulp alone, on rows with |mean| / std up to 100, strided input and output rows.
* glg_clip_image_head against float64: rel-L2 <= 1e-5 per output row, feature norm 28.7 to 1e-5 relative.
* Attention at the tower's shape (N = 2, 16 heads of 64, 257 x 257: the wgmma kernel with a one-key last key tile and a one-row
  last query tile) within the float64 bounds of tests/bounds.py and in the exact dominant-key form.
* The whole tower, tiny and ViT-L/14: rel-L2 <= 2x the library model's own bf16-autocast gap (stored in the fixture) and
  max-rel <= 6 % on pooler_output, image_embeds and the after-reproject feature against the library fixture, and on
  last_hidden_state against the fixture's stored rows and, all 257 rows, against the CPU oracle (pinned to the library by
  tests/test_clip_vision_cpu.py).
* Rows of an N = 1 pass against the same rows of an N = 30 pass (not bitwise: M changes the GEMM tiles).
* The chain prepare_batch -> tiny_text_image UNet forward against the oracles, per-forward tolerance of DESIGN 2."""
import os
from dataclasses import replace

import pytest
import torch

import bounds
from conftest import GOLD, assert_close, rel_l2
from gligen_b200.clip_vision import synthetic_projection_matrix
from test_kernel_stress_gpu import attention_inputs, kernels_for, onehot_attention, run_attention

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
BF = torch.bfloat16


@pytest.fixture(scope="module")
def ops():
    from gligen_b200.ops import CudaOps
    return CudaOps(DEV)


def gen(seed):
    return torch.Generator(device="cpu").manual_seed(seed)


def bf16_ulp(v):
    """Spacing of bf16 numbers at |v| (8 significant bits); the smallest normal spacing at 0."""
    _, e = torch.frexp(v.abs().clamp_min(2.0 ** -126))
    return torch.ldexp(torch.ones_like(v), e - 8)


@pytest.mark.parametrize("N,C,ratio", [(3, 1024, 100.0), (2, 128, 30.0), (1, 1024, 0.0), (4, 512, 1.0)])
def test_clip_vision_embed_within_one_ulp(ops, N, C, ratio):
    """Inputs on a 2^-6 grid with |x| < 128 and C a power of two: the fp32 add, the row sum and the mean are exact in any order,
    so the only fp32 error left before the bf16 rounding is that of rstd (sum of C squares, rsqrtf), which scales with the
    normalised term |gamma (x - mean) rstd|.  Bound per element: one bf16 ulp of the rounded float64 result plus
    (C / 2 + 8) 2^-24 of that term (the term is beta-cancelled near zero, where one ulp alone would be below fp32 round-off)."""
    from ref_ops import RefOps
    P = 256
    g = gen(C + N)
    q = lambda t: torch.round(t * 64) / 64
    # rows whose sum with pos has |mean| / std = ratio: a per-row offset on top of unit-variance noise
    patch_full = torch.randn(N * P, C + 16, generator=g)
    patch_full[:, :C] += ratio * torch.randn(N * P, 1, generator=g).sign()
    patch_full, cls, pos = q(patch_full), q(torch.randn(C, generator=g) * 0.5 + ratio), q(torch.randn(P + 1, C, generator=g) * 0.1)
    gamma, beta = 1 + 0.1 * torch.randn(C, generator=g), 0.1 * torch.randn(C, generator=g)
    d = lambda t: t.to(DEV).contiguous()
    patch = d(patch_full)[:, :C]                                          # ldp = C + 16
    x_full = torch.zeros(N * (P + 1), C + 64, device=DEV, dtype=BF)
    x = x_full[:, :C]                                                     # ldx = C + 64
    ops.clip_vision_embed(patch, d(cls), d(pos), d(gamma), d(beta), x, P, 1e-5)
    want = torch.zeros(N * (P + 1), C, device=DEV, dtype=torch.float64)
    RefOps(DEV, torch.float64, torch.float64).clip_vision_embed(patch, d(cls), d(pos), d(gamma), d(beta), want, P, 1e-5)
    want_bf = want.to(BF).double()
    term = (want - d(beta).double()).abs()
    tol = bf16_ulp(want_bf) + (C / 2 + 8) * 2.0 ** -24 * term
    err = (x.double() - want_bf).abs()
    assert (err <= tol).all(), f"max err / tol {(err / tol).max().item():.2f}"
    assert (err <= bf16_ulp(want_bf)).float().mean() >= 0.999               # almost every element: one ulp alone
    assert x_full[:, C:].abs().sum() == 0                                 # nothing written past C


@pytest.mark.parametrize("proj", [True, False])
def test_clip_image_head_vs_float64(ops, proj):
    N, T, C, D = 5, 257, 1024, 768
    g = gen(7)
    buf = torch.zeros(N, T, C + 64, dtype=BF)
    buf[:, 0, :C] = (torch.randn(N, C, generator=g) * 3 + 0.5).to(BF)
    buf[:, 1:, :C] = 1e4                                                  # only the CLS rows may be read
    x = buf.to(DEV)[:, :, :C]                                             # batch stride T * (C + 64)
    gamma, beta = 1 + 0.1 * torch.randn(C, generator=g), 0.1 * torch.randn(C, generator=g)
    w = torch.randn(D, C, generator=g) * C ** -0.5
    P = synthetic_projection_matrix(D, 7)
    pooled, emb = torch.empty(N, C, device=DEV), torch.empty(N, D, device=DEV)
    feat = torch.empty(N, D, device=DEV) if proj else None
    ops.clip_image_head(x, gamma.to(DEV), beta.to(DEV), w.to(DEV), pooled, emb, P.to(DEV) if proj else None, feat, 28.7, 1e-5)
    torch.cuda.synchronize()
    xd = buf[:, 0, :C].double()
    y = torch.nn.functional.layer_norm(xd, (C,), gamma.double(), beta.double(), 1e-5)
    e = y @ w.double().t()
    f = e @ P.double()
    f = f / f.norm(dim=-1, keepdim=True) * 28.7
    for got, ref, what in ((pooled, y, "pooler_output"), (emb, e, "image_embeds")) + (((feat, f, "feature"),) if proj else ()):
        rel = ((got.cpu().double() - ref).norm(dim=-1) / ref.norm(dim=-1)).max().item()
        assert rel <= 1e-5, f"{what}: rel-L2 {rel:.2e}"
    if proj:
        n = feat.cpu().double().norm(dim=-1)
        assert ((n - 28.7).abs() / 28.7).max() <= 1e-5
    # deterministic: a second call gives the same bits
    pooled2, emb2 = torch.empty_like(pooled), torch.empty_like(emb)
    ops.clip_image_head(x, gamma.to(DEV), beta.to(DEV), w.to(DEV), pooled2, emb2)
    assert torch.equal(pooled, pooled2) and torch.equal(emb, emb2)


# ---- attention at the tower's shape -----------------------------------------------------------------------------------------
@pytest.mark.parametrize("kind", ["std1", "std4", "std10", "argmax_last", "v_offset"])
def test_attention_tower_shape_bounded(ops, kind):
    q, k, v = attention_inputs(kind, 2, 16, 64, 257, 257, seed=257)
    out = run_attention(ops, q, k, v, 16, 64, "auto")
    rep = bounds.attention_check(out, q, k, v, 16, 64, what=f"attention {kind} 16x64 257x257")
    assert rep.ok, str(rep)


def test_attention_tower_shape_dominant_key_exact(ops):
    q, k, v, want = onehot_attention(2, 16, 64, 257, 257, False, seed=257)
    for kernel in kernels_for(257):
        out = run_attention(ops, q, k, v, 16, 64, kernel)
        bad = (out != want).any(-1)
        assert not bad.any(), f"{kernel}: rows {bad.nonzero()[:8].tolist()} differ from V[pi(i)]"


# ---- the whole tower ------------------------------------------------------------------------------------------------------------
def engine(name):
    from gligen_b200.clip_vision import NAMED_CLIP_VISION_CONFIGS, ClipVisionEngine, synthetic_clip_vision_state_dict
    from gligen_b200.ops import CudaOps
    cfg = NAMED_CLIP_VISION_CONFIGS[f"{name}_clip_vision"]
    eng = ClipVisionEngine(cfg, CudaOps(DEV))
    eng.load_state_dict(synthetic_clip_vision_state_dict(cfg, 0))
    return eng


def fixture(name):
    """The stored library outputs plus the regenerated seeded pixel values (checked against the stored corner)."""
    from gligen_b200.clip_vision import synthetic_pixel_values
    g = torch.load(os.path.join(GOLD, f"clip_vision_{name}.pt"))
    g["pixel_values"] = synthetic_pixel_values(g["N"], g["seed"])
    assert torch.equal(g["pixel_values"][:, :, :4, :4], g["pixel_corner"])
    return g


def oracle_last_hidden_state(name, px):
    from clip_vision_oracle import clip_vision_forward
    from gligen_b200.clip_vision import NAMED_CLIP_VISION_CONFIGS, synthetic_clip_vision_state_dict
    cfg = NAMED_CLIP_VISION_CONFIGS[f"{name}_clip_vision"]
    with torch.no_grad():
        return clip_vision_forward(cfg, synthetic_clip_vision_state_dict(cfg, 0), px.cpu())[0]


def check_outputs(outs, g, z_ref, rows=slice(None), what=""):
    """outs: last_hidden_state [n, 257, C], pooler_output, image_embeds, feature of the fixture's images `rows`; z_ref: the full
    last_hidden_state of the oracle.  rel-L2 <= 2x the stored autocast gap, max-rel <= 6 %."""
    z, pooled, emb, feat = outs
    gap = g["autocast_bf16_gap"]
    pairs = (("last_hidden_state", z, z_ref), ("last_hidden_state rows", z[:, g["tokens"]], g["last_hidden_state_rows"][rows]),
             ("pooler_output", pooled, g["pooler_output"][rows]), ("image_embeds", emb, g["image_embeds"][rows]),
             ("feature", feat, g["feature64"][rows]))
    report = []
    for key, got, ref in pairs:
        den = gap[key.split()[0]][0]
        r = assert_close(got, ref, rel=2 * den, max_rel=6e-2, what=f"{what} {key}")
        report.append(f"{key} rel-L2 {r[0]:.3e} (gap {den:.3e}, x{r[0] / den:.2f}) max-rel {r[1]:.3e}")
    print(f"\n{what}: " + "; ".join(report))


@pytest.mark.parametrize("name", ["tiny", "sd14"])
def test_tower_vs_library_fixture(name):
    g = fixture(name)
    P = synthetic_projection_matrix(768, g["proj_seed"]).to(DEV)
    eng = engine(name)
    px = g["pixel_values"].to(DEV)
    z, pooled, emb = eng.forward(px)
    feat = eng.grounding_features(px, P)
    torch.cuda.synchronize()
    check_outputs((z, pooled, emb, feat), g, oracle_last_hidden_state(name, g["pixel_values"]), what=name)


def test_batch_rows_match_single_image_pass():
    from gligen_b200.clip_vision import synthetic_pixel_values
    g = fixture("sd14")
    P = synthetic_projection_matrix(768, g["proj_seed"]).to(DEV)
    eng = engine("sd14")
    px = synthetic_pixel_values(30, 9).to(DEV)
    px[0], px[29] = g["pixel_values"][0].to(DEV), g["pixel_values"][1].to(DEV)
    z30, p30, e30 = eng.forward(px)
    f30 = eng.grounding_features(px, P)
    gap = g["autocast_bf16_gap"]
    for i in (0, 29):
        one = px[i: i + 1]
        z1, p1, e1 = eng.forward(one)
        f1 = eng.grounding_features(one, P)
        for a, b, key in ((z30[i], z1[0], "last_hidden_state"), (p30[i], p1[0], "pooler_output"), (e30[i], e1[0], "image_embeds"), (f30[i], f1[0], "feature")):
            assert_close(a, b, rel=2 * gap[key][0], max_rel=6e-2, what=f"N=30 row {i} vs N=1 {key}")
    # and both against the fixture's images
    sel = [0, 29]
    check_outputs((z30[sel], p30[sel], e30[sel], f30[sel]), g, oracle_last_hidden_state("sd14", g["pixel_values"]),
                  what="sd14 rows of an N=30 pass")


# ---- the chain: prepare_batch -> UNet forward -----------------------------------------------------------------------------------
def test_prepare_batch_into_text_image_unet():
    from clip_vision_oracle import clip_vision_forward, gligen_image_feature, prepare_batch as oracle_prepare_batch
    from gligen_b200 import synth
    from gligen_b200.clip_grounding import ClipGroundingEncoder
    from gligen_b200.clip_text import TINY_CLIP_TEXT, synthetic_clip_state_dict, synthetic_token_ids
    from gligen_b200.clip_vision import TINY_CLIP_VISION, synthetic_clip_vision_state_dict, synthetic_pixel_values
    from gligen_b200.pipeline import build_model, prepare_batch
    from gligen_b200.spec import synthetic_state_dict
    from oracle import unet_oracle as UO
    from oracle.clip_oracle import clip_text_forward
    cfg, model = build_model("tiny_text_image", device=DEV)
    # the tiny UNet's PositionNet reads 128-d features: a 128-d projection and a seeded 128 x 128 reprojection matrix
    vcfg = replace(TINY_CLIP_VISION, projection=cfg.tok_in_dim)
    sd = dict(synthetic_clip_state_dict(TINY_CLIP_TEXT, 0, prefix=""))
    sd.update(synthetic_clip_vision_state_dict(vcfg, 0))
    P = torch.randn(vcfg.projection, vcfg.projection, generator=gen(3)) * vcfg.projection ** -0.5
    enc = ClipGroundingEncoder(sd, P, device=DEV, text_config=TINY_CLIP_TEXT, vision_config=vcfg)
    eot = TINY_CLIP_TEXT.vocab_size - 1
    ph = [r[: int((r == eot).nonzero()[0]) + 1] for r in synthetic_token_ids(TINY_CLIP_TEXT, 3, 4)]
    px = synthetic_pixel_values(3, 5)
    meta = dict(locations=[[0.1, 0.1, 0.6, 0.5], [0.3, 0.2, 0.9, 0.9], [0.0, 0.5, 0.4, 1.0]], phrases=[ph[0], ph[1], None],
                images=[None, px[1], px[2]], text_mask=[1, 1, 0], image_mask=[0, 1, 1])
    B, G = 2, 6
    batch = prepare_batch(meta, batch=B, max_objs=G, encoder=enc)
    want = oracle_prepare_batch(meta, lambda ids: clip_text_forward(TINY_CLIP_TEXT, sd, ids[None], prefix="text_model.")[1],
                                lambda im: gligen_image_feature(clip_vision_forward(vcfg, sd, im[None])[2], P),
                                batch=B, max_objs=G, text_dim=TINY_CLIP_TEXT.width, image_dim=vcfg.projection)
    for k in ("text_embeddings", "image_embeddings"):
        assert_close(batch[k], want[k], rel=2e-2, max_rel=6e-2, what=k)
    for k in ("boxes", "masks", "text_masks", "image_masks"):
        assert torch.equal(batch[k].cpu(), want[k]), k
    inp = synth.make_inputs(cfg, B, G, seed=8)
    ts = torch.tensor([981, 501])
    eps = model(dict(x=inp["x"].to(DEV), timesteps=ts.to(DEV), context=inp["context"].to(DEV),
                     grounding_input=model.grounding_tokenizer_input.prepare(batch), inpainting_extra_input=None, grounding_extra_input=None))
    ref = UO.unet_forward(cfg, synthetic_state_dict(cfg, 0), inp["x"], ts, inp["context"], synth.grounding_kwargs(cfg, want), 1.0)
    torch.cuda.synchronize()
    r = assert_close(eps, ref, rel=2.5e-2, max_rel=9e-2, what="tiny_text_image eps from prepare_batch features")
    print(f"\nchain prepare_batch -> tiny_text_image: eps rel-L2 {r[0]:.3e} max-rel {r[1]:.3e}; "
          f"features rel-L2 text {rel_l2(batch['text_embeddings'].cpu(), want['text_embeddings']):.3e} "
          f"image {rel_l2(batch['image_embeddings'].cpu(), want['image_embeddings']):.3e}")
