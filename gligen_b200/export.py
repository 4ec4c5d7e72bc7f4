"""Export one plan of the UNet engine to a file that `glg_engine_load` (csrc/engine_capi.cu) can replay without Python:
packed weights + workspace sizes + the ordered op-level C-ABI calls with every pointer as (buffer, byte offset).

    eng = model.engine();  export_plan(eng, rows=2 * B, n_objs=30, n_ctx=77, path="unet_b8.glgplan")

`NativePlan` below is a minimal host of such a file through ctypes - the stand-in for a C / C++ / Go / Rust host, and what
tests/test_native_engine_gpu.py uses to check the exported plan bit for bit against the Python-driven engine.
"""
from __future__ import annotations

import ctypes as C
import struct
from typing import Dict, List, Optional, Tuple

import torch

from . import lib as L

MAGIC = b"GLGPLAN1"
NULLBUF = 0xFFFFFFFF


class _Recorder:
    """Stands in for the ctypes library object inside CudaOps: records (name, args) instead of launching."""

    def __init__(self):
        self.calls: List[Tuple[str, tuple]] = []

    def __getattr__(self, name):
        def rec(*args):
            out = []
            for a in args:
                if hasattr(a, "_obj"):                      # ctypes.byref(struct): keep a COPY of the struct
                    st = a._obj
                    out.append(type(st).from_buffer_copy(bytes(st)))
                else:
                    out.append(a)
            self.calls.append((name, tuple(out)))
            return 0
        return rec


def _registry(eng, P) -> List[Tuple[str, torch.Tensor, bool]]:
    """(name, tensor, has_data) of every device allocation an op may point into."""
    reg = [(f"W:{k}", v, True) for k, v in sorted(eng.W.items())]
    reg.append(("splitk_ws", eng.ops.splitk_ws, False))
    named = {id(t): f"in:{k}" for k, t in P.inp.items()}
    named[id(P.out)] = "out"
    for i, t in enumerate(P.buffers):
        reg.append((named.get(id(t), f"B:{i}"), t, False))
    return reg


def export_plan(eng, rows: int, n_objs: int, n_ctx: int, path: str, H: Optional[int] = None, W: Optional[int] = None,
                fractional_t: bool = False) -> Dict[str, int]:
    """Write the plan for (rows, n_objs, n_ctx) at an H x W latent (default: the config's square size) - rows = 2B when cond +
    uncond run as one batch.  The latent size is baked into the recorded calls and the sizes of "in:x" / "out".  Returns counts.
    "in:t" is int64 [rows], the integer DDPM steps; with fractional_t it is fp32 [rows], model time that may lie between them
    (the continuous-time grids of the Karras samplers), embedded by glg_timestep_embedding_f32.
    Spatial-map models: n_objs = cfg.spatial_tokens, and the engine must have seen one grounded call (or `eng._n_objs(grounding)`)
    so that it knows the (C, H, W) of the conditioning map its static buffers are sized for; the named inputs are then
    "in:map", "in:gmask" and "in:extra_map"."""
    P = eng._plan(rows, n_objs, n_ctx, H=H, W=W, fractional_t=fractional_t)
    reg = _registry(eng, P)
    spans = []
    for bi, (name, t, _) in enumerate(reg):
        base = t.untyped_storage().data_ptr()
        spans.append((base, base + t.untyped_storage().nbytes(), bi))

    def locate(ptr):
        if ptr is None or ptr == 0:
            return NULLBUF, 0
        for lo, hi, bi in spans:
            if lo <= ptr < hi:
                return bi, ptr - lo
        raise RuntimeError(f"export: pointer {ptr:#x} is not inside any registered engine buffer")

    rec = _Recorder()
    ops = eng.ops
    saved = ops._c
    ops._c = rec
    records = []
    try:
        for name, fuser, static, fn in P.steps:
            n0 = len(rec.calls)
            fn()
            for call in rec.calls[n0:]:
                records.append((call, (1 if fuser else 0) | (2 if static else 0)))
    finally:
        ops._c = saved
    with open(path, "wb") as f:
        f.write(MAGIC)
        f.write(struct.pack("<I", L.load().glg_abi_version()))
        f.write(struct.pack("<I", len(reg)))
        for name, t, has_data in reg:
            nbytes = t.untyped_storage().nbytes()
            f.write(struct.pack("<QI", nbytes, 1 if has_data else 0))
            f.write(name.encode()[:47].ljust(48, b"\0"))
            if has_data:
                assert t.is_contiguous() and t.numel() * t.element_size() == nbytes, f"{name}: packed weights own their storage"
                f.write(t.detach().reshape(-1).view(torch.uint8).cpu().numpy().tobytes())
        f.write(struct.pack("<I", len(records)))
        for (name, args), flags in records:
            sig = L.SIGNATURES[name][1]
            f.write(name.encode().ljust(32, b"\0"))
            f.write(struct.pack("<II", flags, len(args)))
            for ai, (a, ty) in enumerate(zip(args, sig)):
                last = ai == len(args) - 1
                if isinstance(a, C.Structure):
                    raw = bytearray(bytes(a))
                    fix = []
                    for fname, ftype in a._fields_:
                        if ftype is C.c_void_p:
                            off = getattr(type(a), fname).offset
                            bi, bo = locate(getattr(a, fname))
                            raw[off:off + 8] = b"\0" * 8
                            fix.append((off, bi, bo))
                    f.write(b"S" + struct.pack("<I", len(raw)) + bytes(raw) + struct.pack("<I", len(fix)))
                    for off, bi, bo in fix:
                        f.write(struct.pack("<IIQ", off, bi, bo))
                elif ty is C.c_void_p and last:
                    f.write(b"T")                                  # the stream argument
                elif ty is C.c_void_p:
                    bi, bo = locate(a)
                    f.write(b"P" + struct.pack("<IQ", bi, bo))
                elif ty is C.c_float:
                    f.write(b"F" + struct.pack("<f", float(a)))
                else:
                    f.write(b"I" + struct.pack("<q", int(a)))
    return {"buffers": len(reg), "ops": len(records)}


class NativePlan:
    """Host of an exported plan through the engine-level C ABI (no gligen_b200.engine at run time)."""

    def __init__(self, path: str):
        self.lib = L.load()
        h = C.c_void_p()
        L.check(self.lib.glg_engine_load(path.encode(), C.byref(h)), "glg_engine_load")
        self.h = h

    def buffer(self, name: str):
        p, n = C.c_void_p(), C.c_int64()
        L.check(self.lib.glg_engine_buffer(self.h, name.encode(), C.byref(p), C.byref(n)), "glg_engine_buffer")
        return p.value, n.value

    def write(self, name: str, t: torch.Tensor) -> None:
        """copy a (host or device) tensor into a named buffer on the current stream"""
        _, n = self.buffer(name)
        t = t.contiguous()
        assert t.numel() * t.element_size() == n, (name, tuple(t.shape), n)
        L.check(self.lib.glg_engine_write(self.h, name.encode(), t.data_ptr(), n, torch.cuda.current_stream().cuda_stream), "glg_engine_write")

    def read(self, name: str, shape, dtype=torch.float32) -> torch.Tensor:
        _, n = self.buffer(name)
        out = torch.empty(shape, dtype=dtype, device="cuda")
        assert out.numel() * out.element_size() == n
        L.check(self.lib.glg_engine_read(self.h, name.encode(), out.data_ptr(), n, torch.cuda.current_stream().cuda_stream), "glg_engine_read")
        return out

    def run(self, static_part: bool, fuser_on: bool = True) -> None:
        st = torch.cuda.current_stream().cuda_stream
        L.check(self.lib.glg_engine_run(self.h, 1 if static_part else 0, 1 if fuser_on else 0, st), "glg_engine_run")

    def close(self) -> None:
        if self.h:
            self.lib.glg_engine_destroy(self.h)
            self.h = None
