"""CPU: which compiled epilogue kind each production GEMM call runs (csrc/gemm_tc.cuh, glg_debug_epilogue_kind).

The GEMM epilogue is compiled once per epilogue kind, a fixed set of flags, for the tiles the plans pick with it; any
other call runs the generic kernel, which reads its flags at run time.  Every GEMM call of the benchmark's plan
(SD-1.4 box+text, 8 UNet rows at 64 x 64, static and per-step parts) must get the kind equal to its own flags (0 for a
split-K call, whose tile kernel only stores partial sums), never the generic one; and no call anywhere in the schedule
census may get a kind whose flags differ from its own."""
import pytest

import schedule_census as S

EPI = dict(ln=1, bias=2, rowbias=4, gate=8, residual=16, stats_out=32, fp32=64, bstrided=128)
EPI_ACT, EPI_GENERIC = 256, 512


def flags(f):
    return sum(bit for name, bit in EPI.items() if f[name]) | (EPI_ACT if f["act"] else 0)


def kind_of(call):
    M, N, K = S.gemm_dims(call.args)
    f = dict(S.gemm_key(call.args)[1:])
    lib = S._lib()
    kind = lib.glg_debug_epilogue_kind(M, N, K, int(f["geglu"]), int(f["conv"]), int(S.can_split(call.args)),
                                       S.SPLITK_WS_BYTES, flags(f))
    return f, kind


def _gemm_calls(census):
    return [(key, r) for key, reps in census.keys.items() if key[0] == "gemm" for r in reps]


@pytest.fixture(scope="module")
def bench_census():
    return S.enumerate_variants(configs=["sd14_box_text"], rows=(8,), latents=((64, 64),), vae_batches=(), clip_text=(),
                                clip_vision=())


def test_benchmark_plan_runs_only_specialised_kinds(bench_census):
    calls = _gemm_calls(bench_census)
    assert len(calls) >= 30, len(calls)
    bad = []
    for key, r in calls:
        f, kind = kind_of(r)
        want = 0 if f["splits"] > 1 else flags(f)
        if kind != want:
            bad.append(f"{S.key_id(key)} from {r.origin}: kind {kind}, flags {want}")
    assert not bad, "\n".join(bad)


def test_every_call_runs_its_own_flags_or_the_generic_kernel():
    census = S.enumerate_variants(configs=["sd14_box_text", "sd14_keypoint"], rows=(1, 8, 64), latents=((64, 64), (40, 56)))
    generic = 0
    for key, r in _gemm_calls(census):
        f, kind = kind_of(r)
        want = 0 if f["splits"] > 1 else flags(f)
        assert kind in (want, EPI_GENERIC), (S.key_id(key), r.origin, kind, want)
        generic += kind == EPI_GENERIC
    # the VAE and the CLIP towers' GELU / quick-GELU and fp32-only calls stay generic
    assert generic > 0
