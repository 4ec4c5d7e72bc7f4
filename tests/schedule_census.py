"""The kernel variants production plans select, enumerated from the plans themselves (host only, no GPU work).

Every engine of the product is built on `RecordingOps`, an ops backend whose methods record their arguments and compute
nothing, and each plan is run once (static and per-step parts).  Each recorded call is mapped to a *variant key*: for
`gemm` the tile picker's choice (`glg_debug_pick_tile` / `glg_debug_pick_pingpong`, on the SM count of the device the
picker sees: the GPU's, or 132 without one) and the epilogue flags; for the other kernels with several code paths the
path their dispatcher takes (restated below); for the rest the op name.  Per key two production calls are kept as
representatives, the smallest M*N*K and the largest M, with every tensor argument described by shape, strides, dtype,
storage offset and which arguments share a storage, so that `materialize` rebuilds the call exactly on a device.

The plans only depend on the weights' shapes, so engines are loaded with zero weights of the checkpoint's shapes.
An op name that KEYS does not know fails the enumeration: a new kernel cannot enter production unchecked."""
from __future__ import annotations

import ctypes as C
import inspect
import math
from dataclasses import dataclass, field
from typing import Dict, List, Tuple

import torch

ROWS = (1, 2, 4, 8, 16, 64)
LATENTS = ((64, 64), (64, 96), (96, 64), (96, 96), (128, 128), (48, 128), (72, 72), (40, 56))
VAE_BATCHES = (1, 4, 8)
CLIP_TEXT_BATCHES = (1, 2, 8)      # one prompt with or without its uncond; prepare_batch's phrases of 1-8 boxes in one forward
CLIP_VISION_BATCHES = (1, 30)      # one image; max_objs grounding images in one forward
HOST_CAP_BYTES = 48 << 30          # estimated plan buffers above this are skipped (buffers are allocated, never written)
# Plans above these latent pixels per call are skipped: the float64 attention check of one call of 64 rows at 128^2
# takes minutes.  The caps keep the benchmark's largest call (a 64-row chunk at 64^2) and the 1024^2 decode.
UNET_PIXEL_CAP = 64 * 64 * 64      # rows * H * W
VAE_PIXEL_CAP = 128 * 128          # B * H * W of the latent
SPLITK_WS_BYTES = 8 * 1024 * 2560 * 4      # CudaOps.splitk_ws


@dataclass(frozen=True)
class TSpec:
    """One tensor argument: storage group (arguments with the same group share memory), element offset, shape, strides."""
    group: int
    offset: int
    shape: Tuple[int, ...]
    stride: Tuple[int, ...]
    dtype: str

    def dim(self):
        return len(self.shape)

    def numel(self):
        return math.prod(self.shape)

    def extent(self):
        """One past the last element the view addresses, from the storage start."""
        return self.offset + 1 + sum((s - 1) * st for s, st in zip(self.shape, self.stride)) if self.numel() else self.offset

    def esize(self):
        return torch.empty(0, dtype=getattr(torch, self.dtype)).element_size()


@dataclass
class Call:
    op: str
    args: Dict[str, object]            # bound arguments of the CudaOps method (tensors as TSpec)
    origin: str                        # the production call: engine, config, rows, latent


@dataclass
class Census:
    keys: Dict[tuple, List[Call]] = field(default_factory=dict)      # key -> [smallest M*N*K, largest M] (one if equal)
    skipped: List[str] = field(default_factory=list)
    refused: List[str] = field(default_factory=list)
    calls: int = 0
    sms: int = 132


# ---- the ops' signatures and the arguments each op writes ---------------------------------------------------------------
OUTPUTS = {
    "gemm": ("out", "stats_out"), "attention": ("out",), "groupnorm": ("y", "stats"), "layernorm": ("y",),
    "layernorm_rows": ("y",), "layernorm_rows_f32": ("y",), "conv_in": ("out",), "conv_out": ("out",),
    "upsample2x": ("y",), "im2col_s2": ("y",), "timestep_embedding": ("out",), "position_features": ("out",),
    "patchify_nchw": ("out",), "patchify_nhwc": ("out",), "embed_tokens": ("out",), "clip_vision_embed": ("x",),
    "clip_image_head": ("pooled", "embeds", "feature"), "dwconv7_ln": ("y",), "spatial_tokens": ("y",),
    "resize_plane": ("y",), "grid_resample_gate": ("x", "stats_out"), "conv2d_small": ("y",), "softmax_rows": ("p",),
    "cast": ("y",), "sampler_update": ("e_out", "x_prev"),
}


def _signature(op):
    from gligen_b200.ops import CudaOps
    return inspect.signature(getattr(CudaOps, op))


class RecordingOps:
    """The CudaOps interface on the CPU: every op records (op, args, kwargs) and returns without computing."""
    name = "record"
    act_dtype = torch.bfloat16

    def __init__(self):
        self.device = torch.device("cpu")
        self.calls: List[Tuple[str, tuple, dict]] = []

    def launch_count(self):
        return 0

    def reset_launch_count(self):
        pass

    def __getattr__(self, op):
        if op.startswith("_"):
            raise AttributeError(op)
        return lambda *a, **kw: self.calls.append((op, a, kw))


def describe(op, a, kw) -> Dict[str, object]:
    """Bound arguments of one recorded call with every tensor replaced by its TSpec (storage groups local to the call)."""
    if op not in OUTPUTS:
        raise KeyError(f"op {op!r} has no variant key (schedule_census.OUTPUTS / KEYS): add one before production calls it")
    bound = _signature(op).bind(None, *a, **kw)
    bound.apply_defaults()
    groups: Dict[Tuple[int, torch.dtype], int] = {}

    def spec(v):
        if isinstance(v, torch.Tensor):
            g = groups.setdefault((v.untyped_storage().data_ptr(), v.dtype), len(groups))
            return TSpec(g, v.storage_offset(), tuple(v.shape), tuple(v.stride()), str(v.dtype)[6:])
        if isinstance(v, (tuple, list)):
            return tuple(spec(t) for t in v)
        return v
    return {k: spec(v) for k, v in bound.arguments.items() if k != "self"}


# ---- variant keys ----------------------------------------------------------------------------------------------------
def _rows_view(t: TSpec):
    """(rows, cols, ld) as gligen_b200.ops._rows_view."""
    if t.dim() == 1:
        return 1, t.shape[0], t.shape[0]
    return math.prod(t.shape[:-1]), t.shape[-1], t.stride[-2]


def gemm_dims(args):
    """(M, N, K) of glg_gemm as CudaOps.gemm passes them (N: the packed GEGLU width)."""
    M, K, _ = _rows_view(args["a"])
    No = args["out"].shape[-1]
    return M, No * (2 if args["geglu"] else 1), K


def batch_strided(out: TSpec) -> bool:
    return out.dim() == 3 and out.shape[0] > 1 and out.stride[0] != out.stride[1] * out.shape[1]


def can_split(args) -> bool:
    """glg_gemm's split-K permission (gligen_b200/csrc/gemm_tc.cu:658), for CudaOps' always-present 16-byte aligned
    workspace: no GEGLU, no LayerNorm fold, no stats_out, bf16 output."""
    return not args["geglu"] and args["ln"] is None and args["stats_out"] is None and args["out"].dtype != "float32"


_LIB = None


def _lib():
    global _LIB
    if _LIB is None:
        from gligen_b200 import lib as L
        _LIB = L.load()
    return _LIB


def pick(M, N, K, geglu, conv, split_ok):
    """(BN, paired CTAs, B-resident, K splits, ping-pong) the tile picker chooses."""
    out = (C.c_int32 * 3)()
    lib = _lib()
    lib.glg_debug_pick_tile(M, N, K, int(geglu), int(conv), int(split_ok), SPLITK_WS_BYTES, out)
    pp = lib.glg_debug_pick_pingpong(M, N, K, int(geglu), int(conv), int(split_ok), SPLITK_WS_BYTES)
    return out[0], out[1] & 255, out[1] >> 8, out[2], int(pp)


def gemm_key(args, split_rule=can_split):
    M, N, K = gemm_dims(args)
    conv = args["conv"] is not None
    bn, pair, bres, sp, pp = pick(M, N, K, args["geglu"], conv, split_rule(args))
    return ("gemm", ("bn", bn), ("pair", pair), ("bres", bres), ("splits", sp), ("pp", pp), ("conv", conv),
            ("geglu", bool(args["geglu"])), ("ln", args["ln"] is not None), ("stats_out", args["stats_out"] is not None),
            ("fp32", args["out"].dtype == "float32"), ("bstrided", batch_strided(args["out"])),
            ("bias", args["bias"] is not None), ("rowbias", args["rowbias"] is not None), ("gate", args["gate"] is not None),
            ("residual", args["residual"] is not None), ("act", int(args["act"])))


def attention_variant(Lk, d_head, causal):
    """glg_attention's kernel (csrc/attention.cu): the short-key mma.sync kernel for Lk <= 128 (causal calls always),
    the wgmma kernel above; both instantiated at d_head padded to 16."""
    return "short" if Lk <= 128 or causal else "wgmma", (d_head + 15) // 16 * 16


def attention_key(args):
    Lq, Lk = args["q"].shape[1], args["k"].shape[1]
    kern, dpad = attention_variant(Lk, args["d_head"], args["causal"])
    return ("attention", ("kernel", kern), ("dpad", dpad), ("causal", bool(args["causal"])),
            ("lq_rag64", Lq % 64 != 0), ("lq_rag128", Lq % 128 != 0), ("lk_rag64", Lk % 64 != 0), ("lk_rag128", Lk % 128 != 0))


def groupnorm_key(args):
    import bounds
    x, y = args["x"], args["y"]
    B, HW, Cc = x.shape
    aligned8 = ((x.offset * x.esize()) | (y.offset * y.esize())) % 8 == 0
    return ("groupnorm", ("path", bounds.gn_dispatch(B, HW, Cc, args["groups"], aligned8=aligned8)))


def conv_out_kernel(W, Cout):
    """glg_conv_out's choice (csrc/elementwise.cu)."""
    return f"conv_out_px8_kernel<{Cout}>" if W % 8 == 0 and Cout in (3, 4) else f"conv_out_kernel<{Cout}>"


def conv_in_kernel(B, C0, C1, H, W, Cout):
    """glg_conv_in's choice (csrc/elementwise.cu): the 4-pixel kernel with weights in shared memory when W % 4 == 0, the
    weights fit in 110 KiB and the grid is large."""
    wbytes = 9 * (C0 + C1) * Cout * 4
    return "conv_in_px4_kernel" if W % 4 == 0 and wbytes <= 110 * 1024 and B * H * W * (Cout // 8) >= 4 * 256 * 64 else "conv_in_kernel"


def conv_in_key(args):
    B, C0, H, W = args["x"].shape
    C1 = 0 if args["extra"] is None else args["extra"].shape[1]
    return ("conv_in", ("kernel", conv_in_kernel(B, C0, C1, H, W, args["out"].shape[-1])))


def layernorm_maxv(C):
    """glg_layernorm's ln_kernel<MAXV> (csrc/norm.cu)."""
    vec = C // 8
    return 2 if vec <= 64 else 5 if vec <= 160 else 8


def resample_direction(g, n):
    return "up" if g < n else "identity" if g == n else "down"


KEYS = {
    "gemm": gemm_key,
    "attention": attention_key,
    "groupnorm": groupnorm_key,
    "conv_out": lambda a: ("conv_out", ("kernel", conv_out_kernel(a["W"], a["out"].shape[1]))),
    "conv_in": conv_in_key,
    "layernorm": lambda a: ("layernorm", ("maxv", layernorm_maxv(a["x"].shape[-1]))),
    "grid_resample_gate": lambda a: ("grid_resample_gate", ("resample", resample_direction(a["g"], a["n"]))),
}

# the float64 check each op's calls go through (CheckedOps of tests/test_op_census_gpu.py runs them)
CHECKERS = {
    "gemm": "bounds.gemm_check", "attention": "bounds.attention_check", "groupnorm": "bounds.groupnorm_check",
    "layernorm": "bounds.layernorm_check", "layernorm_rows": "bounds.layernorm_check", "layernorm_rows_f32": "bounds.layernorm_check",
    "softmax_rows": "bounds.softmax_check", "conv_in": "bounds.conv_check", "conv_out": "bounds.conv_check",
    "timestep_embedding": "bounds.timestep_embedding_check", "position_features": "bounds.position_features_check",
    "embed_tokens": "bounds.embed_tokens_check", "spatial_tokens": "bounds.spatial_tokens_check",
    "dwconv7_ln": "bounds.dwconv7_ln_check", "clip_vision_embed": "bounds.clip_vision_embed_check",
    "clip_image_head": "bounds.clip_image_head_check", "sampler_update": "bounds.sampler_update_check",
    "resize_plane": "bounds_resample.resize_check", "conv2d_small": "bounds_resample.conv2d_small_check",
    "grid_resample_gate": "fuser_checks.resample_gate_check",
    # pure data movement: the float64 statement (RefOps) bit for bit
    "cast": "exact", "upsample2x": "exact", "im2col_s2": "exact", "patchify_nchw": "exact", "patchify_nhwc": "exact",
}


def variant_key(op, args):
    if op not in OUTPUTS:
        raise KeyError(f"op {op!r} has no variant key")
    return KEYS[op](args) if op in KEYS else (op,)


def key_id(key) -> str:
    """A readable id: the op, then every field that is not false / zero / 1 split."""
    parts = [key[0]]
    for name, v in key[1:]:
        if v is True:
            parts.append(name)
        elif v in (False, None, 0) or (name in ("splits",) and v == 1):
            continue
        else:
            parts.append(f"{name}{v}")
    return "-".join(parts)


def size_of(op, args):
    """(work, M): M*N*K (taps included) and M for gemm; the first tensor's element count (twice) otherwise."""
    if op == "gemm":
        M, N, K = gemm_dims(args)
        return M * N * K * (9 if args["conv"] is not None else 1), M
    if op == "attention":
        q, k = args["q"], args["k"]
        return q.shape[0] * q.shape[1] * k.shape[1] * args["heads"] * args["d_head"], q.shape[0] * q.shape[1]
    first = next(v for v in args.values() if isinstance(v, TSpec))
    return first.numel(), first.numel()


# ---- enumeration -----------------------------------------------------------------------------------------------------
def _zeros_like_shapes(shapes):
    return {k: torch.zeros(v) for k, v in shapes.items()}


def unet_configs():
    from gligen_b200.spec import NAMED_CONFIGS
    return sorted(n for n in NAMED_CONFIGS if n.startswith("sd14_"))


def _unet_bytes(eng, rows, N, H, W):
    return 2 * sum(eng._sizes(rows, N, 77, H, W).values())


def _vae_bytes(B, H, W, decode):
    T = H * W
    px = 64 * T
    return B * px * 128 * 2 * (6 if decode else 3) + T * T * 6


class _Collector:
    def __init__(self, census: Census):
        self.c = census
        self.best: Dict[tuple, Dict[str, tuple]] = {}

    def add(self, rec: RecordingOps, origin: str):
        for op, a, kw in rec.calls:
            args = describe(op, a, kw)
            key = variant_key(op, args)
            work, m = size_of(op, args)
            b = self.best.setdefault(key, {})
            call = Call(op, args, origin)
            if "small" not in b or work < b["small"][0]:
                b["small"] = (work, m, call)
            if "large" not in b or m > b["large"][1]:
                b["large"] = (work, m, call)
            self.c.calls += 1
        rec.calls.clear()

    def finish(self):
        for key, b in sorted(self.best.items(), key=lambda kv: key_id(kv[0])):
            reps = [b["small"][2]]
            if b["large"][2] is not b["small"][2]:
                reps.append(b["large"][2])
            self.c.keys[key] = reps


def _enumerate_unet(col, name, rows_set, latents):
    from gligen_b200 import synth
    from gligen_b200.engine import Engine
    from gligen_b200.spec import NAMED_CONFIGS, unet_param_shapes
    cfg = NAMED_CONFIGS[name]
    rec = RecordingOps()
    eng = Engine(cfg, rec, use_graphs=False)
    eng.load_state_dict(_zeros_like_shapes(unet_param_shapes(cfg)))
    g = torch.Generator().manual_seed(0)
    N = eng._n_objs(synth.grounding_kwargs(cfg, synth.make_grounding_batch(cfg, 1, 30, g)))
    for H, W in latents:
        try:
            eng.check_latent_size(H, W)
        except ValueError as e:
            col.c.refused.append(f"{name} {H}x{W}: {str(e).split(':', 1)[1].strip()[:60]}")
            continue
        for rows in rows_set:
            where = f"{name} rows={rows} {H}x{W}"
            est = _unet_bytes(eng, rows, N, H, W)
            if rows * H * W > UNET_PIXEL_CAP:
                col.c.skipped.append(f"{where}: {rows * H * W} latent pixels per call > {UNET_PIXEL_CAP}")
                continue
            if est > HOST_CAP_BYTES:
                col.c.skipped.append(f"{where}: ~{est / 2 ** 30:.0f} GiB of plan buffers")
                continue
            P = eng._plan(rows, N, 77, H=H, W=W)
            P.run(True, True)
            P.run(True, False)
            col.add(rec, where)
            eng.plans.clear()
            eng._plan_allocs.clear()
    del eng
    _release()


def _release():
    """Hand freed engine memory back to the system: glibc keeps freed weight-sized blocks on its heap otherwise, and
    each config's engine would add its weights to the resident set."""
    import ctypes.util
    import gc
    gc.collect()
    name = ctypes.util.find_library("c")
    if name:
        try:
            C.CDLL(name).malloc_trim(0)
        except AttributeError:          # not glibc
            pass


def _enumerate_vae(col, batches, latents):
    from gligen_b200.spec import NAMED_VAE_CONFIGS, vae_decoder_param_shapes, vae_encoder_param_shapes
    from gligen_b200.vae import VAEDecoderEngine, VAEEncoderEngine
    cfg = NAMED_VAE_CONFIGS["sd14_vae"]
    rec = RecordingOps()
    dec, enc = VAEDecoderEngine(cfg, rec), VAEEncoderEngine(cfg, rec)
    dec.load_state_dict(_zeros_like_shapes(vae_decoder_param_shapes(cfg)))
    enc.load_state_dict(_zeros_like_shapes(vae_encoder_param_shapes(cfg)))
    for H, W in latents:
        for B in batches:
            for decode in (True, False):
                where = f"sd14_vae {'decode' if decode else 'encode'} B={B} {H}x{W}"
                est = _vae_bytes(B, H, W, decode)
                if B * H * W > VAE_PIXEL_CAP:
                    col.c.skipped.append(f"{where}: {B * H * W} latent pixels per call > {VAE_PIXEL_CAP}")
                    continue
                if est > HOST_CAP_BYTES:
                    col.c.skipped.append(f"{where}: ~{est / 2 ** 30:.0f} GiB of buffers")
                    continue
                if decode:
                    dec.decode(torch.empty(B, cfg.embed_dim, H, W))
                else:
                    enc.encode_moments(torch.empty(B, 3, 8 * H, 8 * W))
                col.add(rec, where)


def _enumerate_clip(col, text_batches, vision_batches):
    from gligen_b200.clip_text import NAMED_CLIP_CONFIGS, ClipTextEngine, clip_text_param_shapes, synthetic_token_ids
    from gligen_b200.clip_vision import NAMED_CLIP_VISION_CONFIGS, ClipVisionEngine, clip_vision_param_shapes
    rec = RecordingOps()
    cfg = NAMED_CLIP_CONFIGS["sd14_clip_text"]
    eng = ClipTextEngine(cfg, rec)
    eng.load_state_dict(_zeros_like_shapes(clip_text_param_shapes(cfg)))
    for B in text_batches:
        eng.forward(synthetic_token_ids(cfg, B, 0))
        col.add(rec, f"sd14_clip_text B={B}")
    vcfg = NAMED_CLIP_VISION_CONFIGS["sd14_clip_vision"]
    veng = ClipVisionEngine(vcfg, rec)
    veng.load_state_dict(_zeros_like_shapes(clip_vision_param_shapes(vcfg)))
    for N in vision_batches:
        veng.forward(torch.zeros(N, 3, 224, 224))
        col.add(rec, f"sd14_clip_vision N={N}")


def enumerate_variants(configs=None, rows=ROWS, latents=LATENTS, vae_batches=VAE_BATCHES, clip_text=CLIP_TEXT_BATCHES,
                       clip_vision=CLIP_VISION_BATCHES) -> Census:
    """Every production call of the given space, keyed; see the module docstring."""
    census = Census()
    census.sms = _device_sms()
    col = _Collector(census)
    with torch.no_grad():
        for name in (unet_configs() if configs is None else configs):
            _enumerate_unet(col, name, rows, latents)
        if vae_batches:
            _enumerate_vae(col, vae_batches, latents)
        _enumerate_clip(col, clip_text, clip_vision)
    col.finish()
    return census


def _device_sms():
    return torch.cuda.get_device_properties(0).multi_processor_count if torch.cuda.is_available() else 132


def summary(census: Census) -> str:
    per_op: Dict[str, int] = {}
    for key in census.keys:
        per_op[key[0]] = per_op.get(key[0], 0) + 1
    lines = [f"schedule census: {census.calls} production calls, {len(census.keys)} keys on {census.sms} SMs"]
    lines += [f"schedule census: {op:<22} {n:>4} keys" for op, n in sorted(per_op.items())]
    lines += [f"schedule census: skipped {s}" for s in census.skipped]
    lines += [f"schedule census: refused by the engine {s}" for s in census.refused]
    return "\n".join(lines)


# ---- rebuilding a representative on a device ---------------------------------------------------------------------------
GUARD = 64          # elements of each storage before and after every view


def _specs(v):
    if isinstance(v, TSpec):
        yield v
    elif isinstance(v, tuple):
        for t in v:
            yield from _specs(t)


def materialize(call: Call, device, seed=0):
    """(args, storages, output mask per storage) of one representative: every storage group one guarded buffer holding
    seeded values, every tensor argument a view with the recorded offset, shape and strides (so leading dimensions,
    batch strides and aliasing are the production call's).  Integer inputs are valid indices; the GroupNorm scratch is
    zero, as glg_groupnorm requires; a folded LayerNorm's statistics and column sums are those of the call's own A and W."""
    import bounds
    g = torch.Generator(device=device).manual_seed(seed)
    groups: Dict[int, Tuple[str, int]] = {}
    for v in call.args.values():
        for t in _specs(v):
            dt, ext = groups.get(t.group, (t.dtype, 0))
            groups[t.group] = (dt, max(ext, t.extent()))
    store = {}
    for gi, (dt, ext) in groups.items():
        n = ext + 2 * GUARD
        dtype = getattr(torch, dt)
        if dtype == torch.int64:
            store[gi] = torch.randint(0, 1000, (n,), generator=g, device=device)
        else:
            store[gi] = torch.randn(n, generator=g, device=device, dtype=torch.float32).to(dtype)

    def view(t):
        return store[t.group].as_strided(t.shape, t.stride, GUARD + t.offset)

    def build(v):
        if isinstance(v, TSpec):
            return view(v)
        if isinstance(v, tuple):
            return tuple(build(t) for t in v)
        return v
    args = {k: build(v) for k, v in call.args.items()}
    if call.op == "gemm":
        K = args["a"].shape[-1]
        args["w"].mul_(K ** -0.5)
        if args["ln"] is not None:
            st, colsum, eps = args["ln"]
            st.copy_(bounds.stats_restated(args["a"].reshape(-1, K)))
            colsum.copy_(args["w"].float().sum(1))
    elif call.op == "groupnorm":
        args["stats"].zero_()
    elif call.op == "embed_tokens":
        args["ids"].copy_(torch.randint(0, args["table"].shape[0], tuple(args["ids"].shape), generator=g, device=device))
    mask = {gi: torch.zeros(s.numel(), dtype=torch.bool, device=device) for gi, s in store.items()}
    for name in OUTPUTS[call.op]:
        for t in _specs(call.args.get(name)):
            mask[t.group].as_strided(t.shape, t.stride, GUARD + t.offset).fill_(True)
    return args, store, mask
