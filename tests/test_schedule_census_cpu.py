"""CPU: the enumeration of the kernel variants production plans select (tests/schedule_census.py) is complete and right.

Plain facts about the tile picker must show in its output, every key must map to a float64 check the GPU census runs,
every key keeps its representatives, an op the key map does not know fails the enumeration, and a wrong split-K
permission changes keys (the helper is not vacuous)."""
import importlib

import pytest
import torch

import schedule_census as S


@pytest.fixture(scope="module")
def census():
    c = S.enumerate_variants()
    print("\n" + S.summary(c))
    return c


def _gemms(census):
    for key, reps in census.keys.items():
        if key[0] == "gemm":
            for r in reps:
                yield dict(key[1:]), r


def test_enumeration_covers_every_engine(census):
    ops = {key[0] for key in census.keys}
    assert {"gemm", "attention", "groupnorm", "conv_in", "conv_out", "softmax_rows", "embed_tokens", "clip_vision_embed",
            "grid_resample_gate", "resize_plane", "conv2d_small", "layernorm_rows_f32"} <= ops, ops
    origins = {r.origin.split()[0] for reps in census.keys.values() for r in reps}
    assert {"sd14_vae", "sd14_clip_text", "sd14_clip_vision"} <= origins
    assert census.skipped and all("latent pixels" in s for s in census.skipped)
    assert sum(1 for k in census.keys if k[0] == "gemm") >= 75


def test_splits_only_where_allowed(census):
    """Split-K only with glg_gemm's permission, and each split keeps >= 16 K blocks (test_abi_cpu.py's rules)."""
    for f, r in _gemms(census):
        if f["splits"] > 1:
            assert S.can_split(r.args), (f, r.origin)
            M, N, K = S.gemm_dims(r.args)
            assert (K // 64) * (9 if f["conv"] else 1) // f["splits"] >= 16, (f, r.origin)


def test_pairs_only_where_allowed(census):
    """CTA pairs only for plain GEMMs with M >= 4096, N % 256 == 0 on 256-wide tiles without a split, and for 3x3
    convolutions with M >= 2048 on tiles >= 128 (test_abi_cpu.py::test_tile_picker_choices_are_valid)."""
    for f, r in _gemms(census):
        assert f["bres"] == 0, "weights-resident tiles are opt-in"
        if f["pair"]:
            M, N, K = S.gemm_dims(r.args)
            if f["conv"]:
                assert M >= 2048 and f["bn"] >= 128 and f["splits"] == 1, (f, r.origin)
            else:
                assert M >= 4096 and N % 256 == 0 and f["bn"] == 256 and f["splits"] == 1, (f, r.origin)


def test_uneven_splits_and_odd_levels():
    """576^2 images (72^2 latent) reach 7 K splits; 320 x 448 images (40 x 56) reach a 5 x 7 bottom level (M = 35) with a
    ping-pong GEGLU there."""
    c = S.enumerate_variants(configs=["sd14_box_text"], rows=(1,), latents=((72, 72),), vae_batches=(), clip_text=(), clip_vision=())
    assert any(k[0] == "gemm" and dict(k[1:])["splits"] == 7 for k in c.keys), [S.key_id(k) for k in c.keys]
    c = S.enumerate_variants(configs=["sd14_box_text"], rows=(1,), latents=((40, 56),), vae_batches=(), clip_text=(), clip_vision=())
    m35 = [(dict(k[1:]), r) for k, reps in c.keys.items() if k[0] == "gemm" for r in reps if S.gemm_dims(r.args)[0] == 35]
    assert m35 and any(f["pp"] and f["geglu"] for f, _ in m35), [S.key_id(k) for k in c.keys]


def test_every_key_has_a_float64_check(census):
    """Each op maps to an existing float64 check (or the exact statement for data movement), and CheckedOps of
    tests/test_op_census_gpu.py, which the GPU census runs every representative through, checks that op."""
    from test_op_census_gpu import SMALL_OPS, CheckedOps
    for key in census.keys:
        op = key[0]
        name = S.CHECKERS[op]
        if name == "exact":
            assert op in SMALL_OPS, op
        else:
            mod, fn = name.split(".")
            assert callable(getattr(importlib.import_module(mod), fn)), name
            assert op in vars(CheckedOps), f"CheckedOps passes {op} through unchecked"


def test_every_key_keeps_its_representatives(census):
    """One or two representatives per key (smallest work, largest M), each mapping back to its own key, each buildable:
    its outputs are among its tensor arguments."""
    for key, reps in census.keys.items():
        assert 1 <= len(reps) <= 2, S.key_id(key)
        for r in reps:
            assert S.variant_key(r.op, r.args) == key, (S.key_id(key), r.origin)
            assert any(r.args.get(o) is not None for o in S.OUTPUTS[r.op]), (r.op, r.origin)
        if len(reps) == 2:
            (w0, m0), (w1, m1) = (S.size_of(r.op, r.args) for r in reps)
            assert w0 <= w1 and m0 <= m1, S.key_id(key)
    ids = [S.key_id(k) for k in census.keys]
    assert len(set(ids)) == len(ids), "key ids must name one schedule each"


def test_unknown_op_fails_the_enumeration():
    rec = S.RecordingOps()
    rec.new_kernel(torch.zeros(4))
    col = S._Collector(S.Census())
    with pytest.raises(KeyError, match="new_kernel"):
        col.add(rec, "test")


def test_wrong_split_permission_changes_keys():
    """A can_split that also forbade split-K for residual epilogues (glg_gemm allows them: the reduce pass adds the
    residual) maps real representatives to unsplit keys.  (One that allowed split-K with stats_out changes no key: every
    stats_out call has K <= 1280, 20 K blocks, too few to split.)"""
    census = S.enumerate_variants(configs=["sd14_box_text"], rows=(1,), latents=((40, 56),), vae_batches=(), clip_text=(), clip_vision=())

    def wrong(args):
        return S.can_split(args) and args["residual"] is None
    changed = [(S.key_id(k), S.key_id(S.gemm_key(r.args, split_rule=wrong)), r.origin)
               for k, reps in census.keys.items() if k[0] == "gemm" for r in reps if S.gemm_key(r.args, split_rule=wrong) != k]
    print("\n".join(f"{a} -> {b} ({o})" for a, b, o in changed[:5]))
    assert changed and all("splits" in a and "residual" in a and "splits" not in b for a, b, _ in changed)
