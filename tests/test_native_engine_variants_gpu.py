"""Engine-level C ABI (include/gligen_b200.h: glg_engine_*) beyond one forward of the gatedSA models:

- every fuser variant (gatedCA on box+text, text+image and keypoint tokens; gatedSA2 with glg_grid_resample_gate) at fuser scales
  1, 0.5 and 0, and the 320-channel sampling models, replayed bit for bit against model.forward_cfg;
- non-square latents (the im2col-TMA convolutions at H != W), tiny and SD-1.4-sized;
- the per-step part captured in a CUDA graph and replayed with new inputs;
- a 4-step DDIM loop whose host writes in:x / in:t every step, against the same loop through model.forward_cfg (state that one
  forward does not show: GroupNorm barrier counters, static buffers the per-step part could overwrite);
- plan files that are truncated, stale or edited: glg_engine_load refuses each one, naming the op and the problem, before it
  allocates or launches anything, and a valid plan still loads and replays bit for bit afterwards.
"""
import copy
import ctypes as C
import os
import struct
import subprocess

import pytest
import torch

from gligen_b200 import lib as L
from gligen_b200.spec import SAMPLING_GATED_CA, SAMPLING_HED_GATED_SA2
from native_plan import DEV, PlanCase, _case

pytestmark = pytest.mark.gpu


# ---- variants, bit for bit against the Python-driven engine --------------------------------------------------------------
@pytest.mark.parametrize("name,max_objs", [("tiny_gated_ca", 6), ("tiny_text_image_gated_ca", 5), ("tiny_keypoint_gated_ca", 0),
                                           ("tiny_hed_gated_sa2", 0)])
def test_fuser_plan_matches_python_engine(name, max_objs, tmp_path):
    """Scale 0.5 halves every gate (W:gates); scale 0 skips the fuser ops of the per-step part."""
    info = _case(name, 2, max_objs, tmp_path, scales=(1.0, 0.5, 0.0))
    assert info["ops"] > 300


@pytest.mark.parametrize("cfg,B,max_objs", [(SAMPLING_GATED_CA, 2, 6), (SAMPLING_HED_GATED_SA2, 1, 0)], ids=["sampling_gated_ca", "sampling_hed_gated_sa2"])
def test_sampling_model_plan_matches_python_engine(cfg, B, max_objs, tmp_path):
    """The 320-channel models of the scheduled-sampling tests (SD-width GEMMs and convolutions), scale 1."""
    _case(cfg, B, max_objs, tmp_path, scales=(1.0,))


@pytest.mark.parametrize("name,B,max_objs,H,W,scales", [("tiny", 2, 6, 16, 24, (1.0, 0.0)), ("tiny", 2, 6, 24, 16, (1.0, 0.0)),
                                                        ("tiny_inpaint", 2, 6, 16, 24, (1.0, 0.0)), ("tiny_inpaint", 2, 6, 24, 16, (1.0, 0.0)),
                                                        ("sd14_box_text", 1, 30, 64, 96, (1.0,))])
def test_non_square_plan_matches_python_engine(name, B, max_objs, H, W, scales, tmp_path):
    _case(name, B, max_objs, tmp_path, scales=scales, H=H, W=W)


# ---- the per-step part in a CUDA graph ------------------------------------------------------------------------------------
def _new_step(c, seed):
    g = torch.Generator().manual_seed(seed)
    return torch.randn(tuple(c.x.shape), generator=g).to(DEV), torch.tensor([501, 61, 7, 3][:c.B], dtype=torch.long, device=DEV)


@pytest.mark.parametrize("name,max_objs", [("tiny", 6), ("tiny_hed_gated_sa2", 0)])
def test_per_step_part_replays_from_cuda_graph(name, max_objs, tmp_path):
    """glg_engine_run(static_part = 0) captured by torch.cuda.graph: a replay gives the eager native result, and after the host
    writes new in:x / in:t a replay gives the Python engine's eps for them."""
    c = PlanCase(name, 2, max_objs, tmp_path)
    c.set_scale(1.0)
    want = c.python(c.x, c.ts)
    c.run(static_part=True)
    c.run(static_part=False)
    eager = c.out()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        c.run(static_part=False)
    graph.replay()
    replay = c.out()
    x2, t2 = _new_step(c, seed=11)
    want2 = c.python(x2, t2)
    c.write_step(x2, t2)
    graph.replay()
    replay2 = c.out()
    c.run(static_part=False)
    eager2 = c.out()
    torch.cuda.synchronize()
    assert torch.equal(eager, want), f"eager: max diff {(eager - want).abs().max().item():.3e}"
    assert torch.equal(replay, eager), f"replay: max diff {(replay - eager).abs().max().item():.3e}"
    assert not torch.equal(want2, want)
    assert torch.equal(replay2, want2), f"replay with new inputs: max diff {(replay2 - want2).abs().max().item():.3e}"
    assert torch.equal(eager2, want2)
    del graph
    c.plan.close()


# ---- a sampler loop through the plan --------------------------------------------------------------------------------------
class _PlanUNet:
    """The samplers' model interface (forward_cfg) served by the exported plan, the way a host without Python drives it: the
    static part once, then per step write in:x / in:t and run the per-step part."""

    def __init__(self, case):
        self.c, self.static_done = case, False

    def forward_cfg(self, input, uc):
        c = self.c
        c.write_step(input["x"], input["timesteps"])
        if not self.static_done:
            c.run(static_part=True)
            self.static_done = True
        c.run(static_part=False)
        out = c.out()
        return out[:c.B], out[c.B:]


@pytest.mark.parametrize("name,max_objs", [("tiny", 6), ("tiny_hed_gated_sa2", 0)])
def test_ddim_loop_through_plan_matches_python_engine(name, max_objs, tmp_path):
    """DDIMSampler.sample(S=4), CFG 7.5, once over model.forward_cfg and once over the plan: the final latents are equal."""
    from ldm.models.diffusion.ddim import DDIMSampler
    from ldm.models.diffusion.ldm import LatentDiffusion
    c = PlanCase(name, 2, max_objs, tmp_path)
    c.set_scale(1.0)
    diffusion = LatentDiffusion(linear_start=0.00085, linear_end=0.012, timesteps=1000).to(DEV)

    def sample(model):
        return DDIMSampler(diffusion, model).sample(S=4, shape=tuple(c.x.shape), input=c.input(c.x.clone(), None), uc=c.uc,
                                                    guidance_scale=7.5).clone()

    want = sample(c.model)
    c.plan.write("W:gates", c.eng.W["gates"])          # the engine's gates at this scale, set by the Python loop
    got = sample(_PlanUNet(c))
    torch.cuda.synchronize()
    assert torch.isfinite(want).all() and not torch.equal(want, c.x)
    assert torch.equal(got, want), f"{name} DDIM S=4: max diff {(got - want).abs().max().item():.3e}"
    c.plan.close()


# ---- malformed plan files -------------------------------------------------------------------------------------------------
# The GLGPLAN1 layout gligen_b200/export.py writes: magic, ABI version, buffers (size, has-data flag, 48-byte name, contents),
# then ops (32-byte name, flags, argument count, tagged arguments).
MAGIC = b"GLGPLAN1"
NULLBUF = 0xFFFFFFFF


def _read_plan(path):
    data = open(path, "rb").read()
    pos = 0

    def take(n):
        nonlocal pos
        b = data[pos:pos + n]
        assert len(b) == n
        pos += n
        return b

    def u32():
        return struct.unpack("<I", take(4))[0]

    assert take(8) == MAGIC
    plan = {"magic": MAGIC, "abi": u32(), "bufs": [], "ops": []}
    for _ in range(u32()):
        nbytes, has_data = struct.unpack("<QI", take(12))
        name = take(48)
        plan["bufs"].append([nbytes, name, take(nbytes) if has_data else None])
    for _ in range(u32()):
        name = take(32).rstrip(b"\0").decode()
        flags, na = struct.unpack("<II", take(8))
        args = []
        for _ in range(na):
            tag = take(1).decode()
            if tag == "P":
                args.append(["P", *struct.unpack("<IQ", take(12))])
            elif tag in "IF":
                args.append([tag, take(8 if tag == "I" else 4)])
            elif tag == "T":
                args.append(["T"])
            else:
                assert tag == "S"
                raw = take(u32())
                args.append(["S", raw, [list(struct.unpack("<IIQ", take(16))) for _ in range(u32())]])
        plan["ops"].append([name, flags, args])
    assert pos == len(data)
    return plan


def _write_plan(path, plan):
    out = [plan["magic"], struct.pack("<II", plan["abi"], len(plan["bufs"]))]
    for nbytes, name, contents in plan["bufs"]:
        out += [struct.pack("<QI", nbytes, contents is not None), name] + ([contents] if contents is not None else [])
    out.append(struct.pack("<I", len(plan["ops"])))
    for name, flags, args in plan["ops"]:
        out += [name.encode().ljust(32, b"\0"), struct.pack("<II", flags, len(args))]
        for a in args:
            out.append(a[0].encode())
            if a[0] == "P":
                out.append(struct.pack("<IQ", a[1], a[2]))
            elif a[0] in "IF":
                out.append(a[1])
            elif a[0] == "S":
                out += [struct.pack("<I", len(a[1])), a[1], struct.pack("<I", len(a[2]))] + [struct.pack("<IIQ", *f) for f in a[2]]
    with open(path, "wb") as f:
        f.write(b"".join(out))


def _first(plan, pred):
    return next(k for k, op in enumerate(plan["ops"]) if pred(op))


def _corruptions(plan, raw):
    """name -> (file contents, fragment of the refusal message); each is `plan` with one thing wrong."""
    ops, bufs = plan["ops"], plan["bufs"]
    gn = _first(plan, lambda op: op[0] == "glg_groupnorm")
    gemm = _first(plan, lambda op: op[0] == "glg_gemm")
    # the first pointer argument into a buffer (not NULL), and the first such pointer field of a GlgGemmArgs
    pk = _first(plan, lambda op: op[0] != "glg_gemm" and any(a[0] == "P" and a[1] != NULLBUF for a in op[2]))
    pj = next(j for j, a in enumerate(ops[pk][2]) if a[0] == "P" and a[1] != NULLBUF)
    pname, pbuf = ops[pk][0], ops[pk][2][pj][1]
    fx = next(i for i, f in enumerate(ops[gemm][2][0][2]) if f[1] != NULLBUF)
    field, fbuf = ops[gemm][2][0][2][fx][:2]
    gemm_bytes = C.sizeof(L.GlgGemmArgs)
    assert len(ops[gemm][2][0][1]) == gemm_bytes

    def edit(fn):
        p = copy.deepcopy(plan)
        fn(p)
        return p

    def set_arg(k, j, a):
        return lambda p: p["ops"][k][2].__setitem__(j, a)

    def set_fix(k, x, f):
        return lambda p: p["ops"][k][2][0][2].__setitem__(x, f)

    ops_at = 16 + sum(60 + (0 if contents is None else len(contents)) for _, _, contents in bufs)     # where the op count is
    return {
        "truncated_in_weights": (raw[:ops_at // 2], "truncated or corrupt plan file"),
        "truncated_in_ops": (raw[:-5], "truncated or corrupt plan file"),
        "magic": (b"GLGPLAN2" + raw[8:], "not a GLGPLAN1 file"),
        "abi_version": (edit(lambda p: p.__setitem__("abi", p["abi"] + 1)), "plan was exported for another ABI version"),
        "unknown_op": (edit(lambda p: p["ops"].insert(10, ["glg_no_such_op", 0, [["T"]]])), "op 10: unknown op 'glg_no_such_op'"),
        "dropped_argument": (edit(lambda p: p["ops"][gn][2].pop(1)), f"op {gn}: glg_groupnorm has 13 arguments, expected 14"),
        "int_for_pointer": (edit(set_arg(pk, pj, ["I", struct.pack("<q", 0)])),
                            f"op {pk}: {pname} argument {pj} is tagged 'I', expected 'P'"),
        "short_gemm_args": (edit(lambda p: p["ops"][gemm][2][0].__setitem__(1, p["ops"][gemm][2][0][1][:-8])),
                            f"op {gemm}: glg_gemm argument 0 holds {gemm_bytes - 8} bytes, expected {gemm_bytes}"),
        "offset_at_buffer_end": (edit(set_arg(pk, pj, ["P", pbuf, bufs[pbuf][0]])),
                                 f"op {pk}: {pname} argument {pj} points at byte {bufs[pbuf][0]} of buffer"),
        "gemm_field_offset_at_buffer_end": (edit(set_fix(gemm, fx, [field, fbuf, bufs[fbuf][0]])),
                                            f"op {gemm}: glg_gemm argument 0 field at byte {field} points at byte {bufs[fbuf][0]} of buffer"),
        "buffer_index_out_of_range": (edit(set_arg(pk, pj, ["P", len(bufs), 0])),
                                      f"op {pk}: {pname} argument {pj} names buffer {len(bufs)}, but the plan has {len(bufs)}"),
    }


@pytest.fixture(scope="module")
def corrupt_plans(tmp_path_factory):
    """(valid tiny PlanCase with its plan closed, {name: (corrupted file path, expected message fragment)})."""
    d = tmp_path_factory.mktemp("plans")
    c = PlanCase("tiny", 2, 6, d)
    c.plan.close()
    raw = open(c.path, "rb").read()
    plan = _read_plan(c.path)
    _write_plan(str(d / "roundtrip.glgplan"), plan)
    assert open(d / "roundtrip.glgplan", "rb").read() == raw          # the writer reproduces an exported plan byte for byte
    files = {}
    for name, (contents, msg) in _corruptions(plan, raw).items():
        path = str(d / f"{name}.glgplan")
        if isinstance(contents, bytes):
            with open(path, "wb") as f:
                f.write(contents)
        else:
            _write_plan(path, contents)
        files[name] = (path, msg)
    return c, files


def _refused(path):
    """glg_engine_load on `path`: (return code, glg_last_error, kernels launched meanwhile).  A plan it accepts is destroyed at
    once: a corrupted plan is never run."""
    lib = L.load()
    n0 = lib.glg_launch_count()
    h = C.c_void_p()
    rc = lib.glg_engine_load(path.encode(), C.byref(h))
    msg = lib.glg_last_error().decode()
    if rc == 0:
        lib.glg_engine_destroy(h)
    torch.cuda.synchronize()
    return rc, msg, lib.glg_launch_count() - n0


CORRUPTIONS = ["truncated_in_weights", "truncated_in_ops", "magic", "abi_version", "unknown_op", "dropped_argument", "int_for_pointer",
               "short_gemm_args", "offset_at_buffer_end", "gemm_field_offset_at_buffer_end", "buffer_index_out_of_range"]


@pytest.mark.parametrize("corruption", CORRUPTIONS)
def test_load_refuses_malformed_plan(corrupt_plans, corruption):
    _, files = corrupt_plans
    assert sorted(files) == sorted(CORRUPTIONS)
    path, fragment = files[corruption]
    rc, msg, launched = _refused(path)
    assert rc < 0, f"{corruption}: glg_engine_load accepted the plan"
    assert msg.startswith("glg_engine_load: ") and fragment in msg, msg
    assert launched == 0


def test_valid_plan_replays_after_refusals(corrupt_plans):
    """Every refusal in a row, then the original plan loads and replays bit for bit (nothing stale is left behind)."""
    c, files = corrupt_plans
    for name, (path, _) in files.items():
        assert _refused(path)[0] < 0, name
    c.load()
    c.set_scale(1.0)
    want = c.python(c.x, c.ts)
    c.run(static_part=True)
    c.run(static_part=False)
    got = c.out()
    torch.cuda.synchronize()
    c.plan.close()
    assert torch.equal(got, want), f"max diff {(got - want).abs().max().item():.3e}"


def test_c_host_reports_load_refusal(corrupt_plans, tmp_path):
    """examples/host_c/unet_host.c exits with glg_last_error's message on a refused plan."""
    from test_native_engine_gpu import _c_host
    exe = _c_host(tmp_path)
    path, fragment = corrupt_plans[1]["unknown_op"]
    r = subprocess.run([exe, path, os.path.join(str(tmp_path), "out.bin")], capture_output=True, text=True)
    assert r.returncode == 1 and f"unet_host: {path}: glg_engine_load: {fragment}" in r.stderr, r.stderr
