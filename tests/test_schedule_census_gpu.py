"""Every kernel variant production plans select, checked against float64 on this device, and the benchmark's workloads
censused at their batch sizes.

tests/schedule_census.py enumerates the production calls of every SD-1.4-sized engine at module import, on this
device's SM count (the tile picker reads it), and keys each call by the variant it runs.  Each key's representatives
(the smallest M*N*K and the largest M call) are rebuilt with their exact shapes, strides and aliasing on seeded data,
run once with the picker choosing on its own, and checked by CheckedOps of tests/test_op_census_gpu.py within the
float64 bounds of tests/bounds.py (row-chunked), stats_out bit for bit; every element of the call's storages outside
its outputs must be unchanged (guard bands and padding columns), so a split or pair writing out of range fails.  A
profiled child process confirms that each gemm key launches the gemm_tc_kernel template and split-K reduce its key
names."""
import json
import os
import pickle
import re
import subprocess
import sys

import pytest
import torch

import schedule_census as S
from test_large_resolution_gpu import CHUNK_BYTES, _census
from test_op_census_gpu import CheckedOps

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

CENSUS = S.enumerate_variants() if torch.cuda.is_available() else None
KEYS = list(CENSUS.keys) if CENSUS else []
if CENSUS:
    print("\n" + S.summary(CENSUS))


@pytest.fixture(scope="module")
def ops():
    from gligen_b200.ops import CudaOps
    return CudaOps(DEV)


def test_census_device(ops):
    sms = torch.cuda.get_device_properties(DEV).multi_processor_count
    print(f"\nschedule census on {torch.cuda.get_device_name(DEV)}: {sms} SMs, {len(KEYS)} keys, {CENSUS.calls} production calls")
    assert CENSUS.sms == sms and len(KEYS) > 0


@pytest.mark.parametrize("key", KEYS, ids=[S.key_id(k) for k in KEYS])
def test_representative(ops, key):
    bad = []
    torch.cuda.empty_cache()
    torch.cuda.reset_peak_memory_stats(DEV)
    for i, call in enumerate(CENSUS.keys[key]):
        args, store, mask = S.materialize(call, DEV, seed=i)
        before = {g: t.clone() for g, t in store.items()}
        checked = CheckedOps(ops, max_elems=CHUNK_BYTES)
        getattr(checked, call.op)(**args)
        torch.cuda.synchronize()
        what = f"{S.key_id(key)} from {call.origin}"
        rec = [r for rs in checked.records.values() for r in rs]
        print(f"{what}: worst {max((r[0] for r in rec), default=0.0):.3f}, peak memory "
              f"{torch.cuda.max_memory_allocated(DEV) / 2 ** 30:.1f} GiB")
        assert rec or call.op in ("cast", "upsample2x", "im2col_s2", "patchify_nchw", "patchify_nhwc"), f"{what}: no check ran"
        bad += [f"{what}: {f}" for f in checked.failures]
        for g, t in store.items():
            moved = (t != before[g]) & ~mask[g]
            if moved.any():
                bad.append(f"{what}: {int(moved.sum())} elements outside the outputs changed (storage {g}, first at "
                           f"{int(moved.nonzero()[0]) - S.GUARD} from the view base)")
        del args, store, mask, before
    assert not bad, "\n".join(bad)


# ---- the launched template of every gemm key --------------------------------------------------------------------------
_PROFILE = r"""
import json, pickle, sys
sys.path[:0] = [{root!r}, {tests!r}]
import torch
from torch.profiler import ProfilerActivity, profile
import schedule_census as S
from gligen_b200.ops import CudaOps
ops = CudaOps("cuda:0")
calls = pickle.load(open({calls!r}, "rb"))
with profile(activities=[ProfilerActivity.CUDA]) as prof:
    for call in calls:
        args, store, mask = S.materialize(call, "cuda:0")
        ops.gemm(**args)
        torch.cuda.synchronize()
        del args, store, mask
prof.export_chrome_trace({trace!r})
with open({trace!r}) as f:
    ev = [e for e in json.load(f)["traceEvents"] if str(e.get("cat", "")).lower() == "kernel"]
names = [e["name"] for e in sorted(ev, key=lambda e: e["ts"]) if "gemm_tc_kernel" in e["name"] or "splitk_reduce_kernel" in e["name"]]
print("GEMM_KERNELS " + json.dumps(names))
"""


def _expected_template(f):
    bn = 128 if f["pp"] and f["geglu"] else f["bn"]
    b = lambda v: "true" if v else "false"
    return f"{bn}, {b(f['geglu'])}, {b(f['pair'])}, {b(f['pp'])}"


def test_launched_templates(tmp_path):
    """One profiled region in a short child process (as test_large_resolution_gpu.py's GroupNorm trace): every gemm
    representative launches gemm_tc_kernel<BN, GEGLU, CTA2, PP> as its key says, followed by splitk_reduce_kernel exactly
    when the key splits K."""
    gemm = [(k, c) for k in KEYS if k[0] == "gemm" for c in CENSUS.keys[k]]
    path, trace = str(tmp_path / "calls.pkl"), str(tmp_path / "trace.json")
    with open(path, "wb") as f:
        pickle.dump([c for _, c in gemm], f)
    code = _PROFILE.format(root=ROOT, tests=os.path.join(ROOT, "tests"), calls=path, trace=trace)
    r = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, timeout=1200)
    line = next((ln for ln in r.stdout.splitlines() if ln.startswith("GEMM_KERNELS ")), None)
    assert r.returncode == 0 and line, r.stdout[-2000:] + r.stderr[-4000:]
    launches = []
    for name in json.loads(line[len("GEMM_KERNELS "):]):
        if "gemm_tc_kernel" in name:
            launches.append([re.search(r"gemm_tc_kernel<([^>]*)>", name).group(1), False])
        else:
            assert launches, name
            launches[-1][1] = True
    assert len(launches) == len(gemm), (len(launches), len(gemm))
    bad = []
    for (key, call), (tmpl, reduced) in zip(gemm, launches):
        f = dict(key[1:])
        want = _expected_template(f)
        if tmpl.replace(" ", "") != want.replace(" ", "") or reduced != (f["splits"] > 1):
            bad.append(f"{S.key_id(key)} from {call.origin}: launched <{tmpl}> reduce={reduced}, key says <{want}> reduce={f['splits'] > 1}")
    print(f"\n{len(gemm)} gemm representatives launched their keys' templates" if not bad else "")
    assert not bad, "\n".join(bad)


# ---- whole forwards at the benchmark's batch sizes ---------------------------------------------------------------------
def _unet_forward(name, B, cfg_batch, latent=None):
    """One forward of a seeded SD-1.4-sized model: CFG (2B rows) or a single pass (B rows), at its native latent or (H, W)."""
    from gligen_b200 import synth
    from gligen_b200.engine import Engine
    from gligen_b200.spec import NAMED_CONFIGS, SPATIAL_MAP_KEY, synthetic_state_dict
    from inpaint_mask_func import draw_masks_from_boxes
    cfg = NAMED_CONFIGS[name]

    def forward(checked):
        eng = Engine(cfg, checked, use_graphs=False)
        eng.load_state_dict(synthetic_state_dict(cfg, 0))
        inp = synth.make_inputs(cfg, B, seed=2)
        x = inp["x"] if latent is None else torch.randn(B, cfg.in_channels, *latent, generator=torch.Generator().manual_seed(sum(latent)))
        x, ctx, uc = x.to(DEV), inp["context"].to(DEV), inp["uc"].to(DEV)
        ts = torch.tensor([981, 501, 21, 700] * (B // 4 + 1), device=DEV)[:B]
        gr = {k: v.to(DEV) for k, v in inp["grounding_input"].items()}
        extra = gextra = None
        if cfg.inpaint_mode:
            mask = draw_masks_from_boxes(inp["batch"]["boxes"], cfg.image_size).to(DEV)
            extra = torch.cat([inp["z0"].to(DEV) * mask, mask], 1)
        if cfg.spatial:
            gextra = inp["batch"][SPATIAL_MAP_KEY[cfg.tokenizer]].to(DEV)
        outs = eng.forward_cfg(x, ts, ctx, uc, gr, extra, gextra) if cfg_batch else (eng.forward(x, ts, ctx, gr, extra, gextra),)
        torch.cuda.synchronize()
        assert all(torch.isfinite(o).all() for o in outs)
    return forward


BENCH_FORWARDS = [  # name, B, CFG, latent: bench.py's PRESETS at their UNet rows, and the odd-sided latents
    ("sd14_box_text_image", 8, True, None), ("sd14_inpaint_box_text", 8, True, None), ("sd14_keypoint", 4, True, None),
    ("sd14_keypoint", 64, False, None), ("sd14_box_text", 1, True, (72, 72)), ("sd14_box_text", 1, True, (40, 56)),
]


@pytest.mark.parametrize("name,B,cfg_batch,latent", BENCH_FORWARDS,
                         ids=[f"{n}-B{b}{'-cfg' if c else ''}{f'-{l[0]}x{l[1]}' if l else ''}" for n, b, c, l in BENCH_FORWARDS])
def test_census_benchmark_forwards(ops, name, B, cfg_batch, latent):
    title = f"{name} B={B}{' cfg' if cfg_batch else ''}{f' {latent[0]}x{latent[1]}' if latent else ''}"
    _census(ops, title, _unet_forward(name, B, cfg_batch, latent))
