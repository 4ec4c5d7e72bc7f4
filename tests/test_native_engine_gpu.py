"""Engine-level C ABI (include/gligen_b200.h: glg_engine_*): a plan exported by gligen_b200/export.py and replayed by the
library alone gives, bit for bit, the eps of the Python-driven engine (same kernels, same order, same buffers layout) -
for the tiny model in every tokenizer / inpaint variant and, once, for the full SD-1.4-sized model."""
import os

import pytest
import torch

from gligen_b200 import synth
from gligen_b200.export import export_plan
from gligen_b200.pipeline import build_model, to_device
from native_plan import _case

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


@pytest.mark.parametrize("name,max_objs", [("tiny", 6), ("tiny_text_image", 5), ("tiny_keypoint", 34), ("tiny_inpaint", 6), ("tiny_sem", 0), ("tiny_hed", 0)])
def test_exported_plan_matches_python_engine_tiny(name, max_objs, tmp_path):
    info = _case(name, 2, max_objs, tmp_path)
    assert info["ops"] > 300


def test_exported_plan_matches_python_engine_sd14(tmp_path):
    info = _case("sd14_box_text", 1, 30, tmp_path, scales=(1.0,))
    print(f"\nsd14 plan: {info}")


def _c_host(tmp_path):
    """examples/host_c/unet_host.c compiled against the library (skips without gcc)."""
    import shutil
    import subprocess
    if shutil.which("gcc") is None:
        pytest.skip("no gcc")
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    exe = os.path.join(str(tmp_path), "unet_host")
    r = subprocess.run(["gcc", "-O2", "-I", os.path.join(root, "include"), os.path.join(root, "examples", "host_c", "unet_host.c"),
                        "-L", os.path.join(root, "gligen_b200"), "-lgligen_b200", f"-Wl,-rpath,{os.path.join(root, 'gligen_b200')}", "-o", exe],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    return exe


def _c_host_run(exe, tmp_path, plan_path, files, shape):
    """Runs the C host on `plan_path` with the named inputs `files`; returns its "out" buffer as fp32 of `shape` (CPU)."""
    import subprocess
    import numpy as np
    args = []
    for name, t in files.items():
        fn = os.path.join(str(tmp_path), name.replace(":", "_") + ".bin")
        t.contiguous().cpu().numpy().tofile(fn)
        args.append(f"{name}={fn}")
    outp = os.path.join(str(tmp_path), "out.bin")
    r = subprocess.run([exe, plan_path, outp] + args, capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr
    print("\n" + r.stdout.strip())
    return torch.from_numpy(np.fromfile(outp, dtype=np.float32)).view(shape)


def test_c_host_replays_plan(tmp_path):
    """The plan of the tiny model replayed by examples/host_c/unet_host.c (plain C, no Python, no CUDA headers) gives the Python-driven
    engine's eps bit for bit."""
    exe = _c_host(tmp_path)
    B, G = 2, 6
    cfg, model = build_model("tiny", DEV)
    inp = synth.make_inputs(cfg, B, G, seed=4)
    ts = torch.tensor([981, 401], dtype=torch.long, device=DEV)
    x, ctx, uc = inp["x"].to(DEV), inp["context"].to(DEV), inp["uc"].to(DEV)
    batch = to_device(inp["batch"], DEV)
    grounding = model.grounding_tokenizer_input.prepare(batch)
    e_c, e_u = model.forward_cfg(dict(x=x, timesteps=ts, context=ctx, grounding_input=grounding, inpainting_extra_input=None), uc)
    want = torch.cat([e_c, e_u]).clone().cpu()
    eng = model.engine()
    path = os.path.join(str(tmp_path), "tiny.glgplan")
    export_plan(eng, 2 * B, G, ctx.shape[1], path)
    z = lambda t: torch.cat([t, torch.zeros_like(t)])
    files = {"in:x": torch.cat([x, x]), "in:t": torch.cat([ts, ts]), "in:context": torch.cat([ctx, uc]), "in:coords": z(batch["boxes"]),
             "in:masks": z(batch["masks"]), "in:feat0": z(batch["text_embeddings"]), "in:fmask0": z(batch["masks"]), "W:gates": eng.W["gates"]}
    got = _c_host_run(exe, tmp_path, path, files, want.shape)
    assert torch.equal(got, want), f"C host: max diff {(got - want).abs().max().item():.3e}"


@pytest.mark.parametrize("name,map_size", [("tiny_sem", (300, 224)), ("tiny_hed", (192, 320))])
def test_exported_plan_non_square_map(name, map_size, tmp_path):
    """A spatial model planned for a non-square conditioning map: the exported plan replays the Python-driven engine bit for bit."""
    _case(name, 2, 0, tmp_path, map_size=map_size)


def test_c_host_replays_non_square_map_plan(tmp_path):
    """The plan of the tiny sem model for a 300 x 224 map (nearest resampling fused into both convolutions, partial windows)
    replayed by the plain-C host gives the Python-driven engine's eps bit for bit."""
    from gligen_b200.spec import SPATIAL_MAP_KEY
    exe = _c_host(tmp_path)
    B = 2
    cfg, model = build_model("tiny_sem", DEV)
    inp = synth.make_inputs(cfg, B, seed=4, map_size=(300, 224))
    ts = torch.tensor([981, 401], dtype=torch.long, device=DEV)
    x, ctx, uc = inp["x"].to(DEV), inp["context"].to(DEV), inp["uc"].to(DEV)
    batch = to_device(inp["batch"], DEV)
    grounding = model.grounding_tokenizer_input.prepare(batch)
    gmap = batch[SPATIAL_MAP_KEY[cfg.tokenizer]]
    e_c, e_u = model.forward_cfg(dict(x=x, timesteps=ts, context=ctx, grounding_input=grounding, inpainting_extra_input=None,
                                      grounding_extra_input=gmap), uc)
    want = torch.cat([e_c, e_u]).clone().cpu()
    eng = model.engine()
    path = os.path.join(str(tmp_path), "tiny_sem.glgplan")
    export_plan(eng, 2 * B, cfg.spatial_tokens, ctx.shape[1], path)
    z = lambda t: torch.cat([t, torch.zeros_like(t)])
    files = {"in:x": torch.cat([x, x]), "in:t": torch.cat([ts, ts]), "in:context": torch.cat([ctx, uc]), "in:map": z(gmap),
             "in:gmask": z(batch["mask"]), "in:extra_map": torch.cat([gmap, gmap]), "W:gates": eng.W["gates"]}
    got = _c_host_run(exe, tmp_path, path, files, want.shape)
    assert torch.equal(got, want), f"C host: max diff {(got - want).abs().max().item():.3e}"
