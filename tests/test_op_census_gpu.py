"""Every kernel call of real forwards, checked one call at a time.

CheckedOps wraps CudaOps: each call snapshots its inputs (the residual is often the output itself), runs the kernel,
synchronises and checks the output against RefOps(float64) on the snapshot - the GEMM family and attention with the
rounding-level bounds of tests/bounds.py, stats_out bit for bit against its documented summation order, the other ops
at the tolerances of tests/test_kernels_gpu.py.  The forwards run with seeded synthetic weights and no CUDA graphs, so
every call of the plan is seen.  A failure lists every violating call with its shapes, strides, flags and tile choice."""
import ctypes as C
import inspect
from collections import defaultdict

import pytest
import torch

import bounds
from conftest import assert_close
from ref_ops import RefOps

pytestmark = pytest.mark.gpu
DEV = "cuda:0"

# outputs of the ops checked at the kernel suite's tolerances: name -> (output arguments, rel-L2, max-rel)
SMALL_OPS = {
    "groupnorm": (("y",), 6e-3, 3e-2), "layernorm": (("y",), 6e-3, 3e-2), "layernorm_rows": (("y",), 6e-3, 3e-2),
    "layernorm_rows_f32": (("y",), 2e-3, 5e-3), "conv_in": (("out",), 6e-3, 3e-2), "conv_out": (("out",), 2e-3, 5e-3),
    "timestep_embedding": (("out",), 4e-3, 1e-2), "position_features": (("out",), 4e-3, 1e-2),
    "softmax_rows": (("p",), 6e-3, 3e-2), "sampler_update": (("e_out", "x_prev"), 1e-5, 1e-4), "cast": (("y",), 4e-3, 1e-2),
    "upsample2x": (("y",), 0.0, 0.0), "im2col_s2": (("y",), 0.0, 0.0), "embed_tokens": (("out",), 4e-3, 1e-2),
    "dwconv7_ln": (("y",), 6e-3, 3e-2), "spatial_tokens": (("y",), 4e-3, 1e-2), "resize_plane": (("y",), 2e-3, 5e-3),
    "conv2d_small": (("y",), 2e-3, 5e-3), "patchify_nchw": (("out",), 0.0, 0.0), "patchify_nhwc": (("out",), 0.0, 0.0),
}


def _snap(x):
    return x.clone() if isinstance(x, torch.Tensor) else (type(x)(_snap(t) for t in x) if isinstance(x, (list, tuple)) else x)


def _desc(t):
    return f"{tuple(t.shape)}/{tuple(t.stride())}/{str(t.dtype)[6:]}" if isinstance(t, torch.Tensor) else repr(t)


class CheckedOps:
    """CudaOps with a float64 check after every call (records, never raises)."""

    def __init__(self, inner):
        self.inner = inner
        self.ref = RefOps(DEV, compute_dtype=torch.float64)
        self.records = defaultdict(list)          # kind -> [(elementwise ratio, aggregate ratio)]
        self.failures = []

    def __getattr__(self, name):
        attr = getattr(self.inner, name)
        if name in SMALL_OPS:
            return lambda *a, **kw: self._small(name, attr, *a, **kw)
        return attr

    def _fail(self, msg):
        self.failures.append(msg)

    def gemm(self, a, w, out, **kw):
        snap = {k: _snap(v) for k, v in kw.items()}
        a0 = a.clone()
        self.inner.gemm(a, w, out, **kw)
        torch.cuda.synchronize()
        M, No = out.numel() // out.shape[-1], out.shape[-1]
        pick = (C.c_int32 * 3)()
        self.inner.lib.glg_debug_pick_tile(M, No * (2 if kw.get("geglu") else 1), a.shape[-1], int(bool(kw.get("geglu"))),
                                            int(kw.get("conv") is not None), 1, self.inner.splitk_ws.numel() * 4, pick)
        flags = {k: (_desc(v) if isinstance(v, torch.Tensor) else v) for k, v in kw.items() if v is not None and k != "ln"}
        what = (f"gemm a={_desc(a)} w={_desc(w)} out={_desc(out)} {flags} ln={kw.get('ln') is not None} "
                f"tile(BN={pick[0]}, pair={pick[1] & 255}, resident={pick[1] >> 8}, splits={pick[2]})")
        so = snap.pop("stats_out", None)
        if so is not None:
            st = kw["stats_out"]
            if not torch.equal(st, bounds.stats_restated(out.reshape(M, No))):
                self._fail(f"stats_out order: {what}")
        rep = bounds.gemm_check(out, a0, w, splits=8, what=what, **snap)
        kind = "conv3x3" if kw.get("conv") is not None else "gemm+ln" if kw.get("ln") is not None else "gemm"
        self.records[kind + (" fp32" if out.dtype == torch.float32 else "")].append((rep.ratio, rep.agg_ratio))
        if not rep.ok:
            self._fail(str(rep))

    def attention(self, q, k, v, out, heads, d_head, causal=False):
        q0, k0, v0 = q.clone(), k.clone(), v.clone()
        self.inner.attention(q, k, v, out, heads, d_head, causal=causal)
        torch.cuda.synchronize()
        rep = bounds.attention_check(out, q0, k0, v0, heads, d_head, causal=causal,
                                     what=f"attention q={_desc(q)} k={_desc(k)} out={_desc(out)} heads={heads} d={d_head} causal={causal}")
        self.records["attention"].append((rep.ratio, 0.0))
        if not rep.ok:
            self._fail(str(rep))

    def _small(self, name, fn, *a, **kw):
        outs, rel, max_rel = SMALL_OPS[name]
        bound = inspect.signature(getattr(RefOps, name)).bind(None, *a, **kw)
        args = {k: v for k, v in bound.arguments.items() if k != "self"}
        snap = {k: _snap(v) for k, v in args.items()}
        fn(*a, **kw)
        torch.cuda.synchronize()
        getattr(self.ref, name)(**snap)
        worst = 0.0
        for o in outs:
            got, want = args.get(o), snap.get(o)
            if got is None:
                continue
            what = f"{name} {o}={_desc(got)}"
            if rel == 0.0:
                ok = torch.equal(got.to(torch.float64), want.to(got.dtype).to(torch.float64))
                if not ok:
                    self._fail(f"{what}: not bit-identical")
                continue
            try:
                r, m = assert_close(got, want.to(got.dtype), rel=rel, max_rel=max_rel, what=what)
                worst = max(worst, r / rel, m / max_rel)
            except AssertionError as e:
                self._fail(str(e))
        self.records[name].append((worst, 0.0))


def _summary(title, ops):
    lines = [f"census {title}: {'op kind':<22} {'calls':>5} {'worst elem':>10} {'worst agg':>9}"]
    for kind, rs in sorted(ops.records.items()):
        lines.append(f"census {title}: {kind:<22} {len(rs):>5} {max(r[0] for r in rs):>10.3f} {max(r[1] for r in rs):>9.3f}")
    print("\n".join(lines))
    assert not ops.failures, f"{len(ops.failures)} calls out of bounds:\n" + "\n".join(ops.failures[:40])
    assert sum(len(r) for r in ops.records.values()) > 0


@pytest.fixture(scope="module")
def cuda_ops():
    from gligen_b200.ops import CudaOps
    return CudaOps(DEV)


def _unet_forward(cuda_ops, name, B, cfg_batch):
    from gligen_b200 import synth
    from gligen_b200.engine import Engine
    from gligen_b200.spec import NAMED_CONFIGS, SPATIAL_MAP_KEY, synthetic_state_dict
    from inpaint_mask_func import draw_masks_from_boxes
    cfg = NAMED_CONFIGS[name]
    ops = CheckedOps(cuda_ops)
    eng = Engine(cfg, ops, use_graphs=False)
    eng.load_state_dict(synthetic_state_dict(cfg, 0))
    inp = synth.make_inputs(cfg, B, seed=2)
    x, ctx, uc = (inp[k].to(DEV) for k in ("x", "context", "uc"))
    ts = torch.tensor([981, 501, 21, 700][:B] * (B // 4 + 1), device=DEV)[:B]
    gr = {k: v.to(DEV) for k, v in inp["grounding_input"].items()}
    extra = gextra = None
    if cfg.inpaint_mode:
        mask = draw_masks_from_boxes(inp["batch"]["boxes"], cfg.image_size).to(DEV)
        extra = torch.cat([inp["z0"].to(DEV) * mask, mask], 1)
    if cfg.spatial:
        gextra = inp["batch"][SPATIAL_MAP_KEY[cfg.tokenizer]].to(DEV)
    if cfg_batch:
        eng.forward_cfg(x, ts, ctx, uc, gr, extra, gextra)
    else:
        eng.forward(x, ts, ctx, gr, extra, gextra)
    torch.cuda.synchronize()
    _summary(f"{name} B={B}{' cfg' if cfg_batch else ''}", ops)


def test_census_sd14_box_text_cfg_b4(cuda_ops):
    """The benchmark's workload: one CFG forward of the SD-1.4-sized box+text model at a batch of 4 (8 UNet rows)."""
    _unet_forward(cuda_ops, "sd14_box_text", 4, True)


@pytest.mark.parametrize("name", ["sd14_keypoint", "sd14_inpaint_box_text"])
def test_census_sd14_variants(cuda_ops, name):
    _unet_forward(cuda_ops, name, 1, False)


def _tiny_names():
    from gligen_b200.spec import NAMED_CONFIGS
    return sorted(n for n in NAMED_CONFIGS if n.startswith("tiny"))


@pytest.mark.parametrize("name", _tiny_names())
def test_census_tiny(cuda_ops, name):
    _unet_forward(cuda_ops, name, 2, True)


def test_census_vae_sd14(cuda_ops):
    from gligen_b200.spec import NAMED_VAE_CONFIGS, synthetic_vae_encoder_state_dict, synthetic_vae_state_dict
    from gligen_b200.vae import VAEDecoderEngine, VAEEncoderEngine
    cfg = NAMED_VAE_CONFIGS["sd14_vae"]
    ops = CheckedOps(cuda_ops)
    dec = VAEDecoderEngine(cfg, ops)
    dec.load_state_dict(synthetic_vae_state_dict(cfg, 0))
    g = torch.Generator().manual_seed(4)
    dec.decode(torch.randn(1, 4, cfg.latent_size, cfg.latent_size, generator=g).to(DEV))
    enc = VAEEncoderEngine(cfg, ops)
    enc.load_state_dict(synthetic_vae_encoder_state_dict(cfg, 1))
    enc.encode_moments(torch.rand(1, 3, 8 * cfg.latent_size, 8 * cfg.latent_size, generator=g).to(DEV) * 2 - 1)
    torch.cuda.synchronize()
    _summary("sd14_vae decode + encode", ops)


def test_census_clip_text_sd14(cuda_ops):
    from gligen_b200.clip_text import NAMED_CLIP_CONFIGS, ClipTextEngine, synthetic_clip_state_dict, synthetic_token_ids
    cfg = NAMED_CLIP_CONFIGS["sd14_clip_text"]
    ops = CheckedOps(cuda_ops)
    eng = ClipTextEngine(cfg, ops)
    eng.load_state_dict(synthetic_clip_state_dict(cfg, 0))
    eng.forward(synthetic_token_ids(cfg, 2, 3).to(DEV))
    torch.cuda.synchronize()
    _summary("sd14_clip_text", ops)
