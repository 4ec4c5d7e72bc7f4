"""Every kernel call of real forwards, checked one call at a time.

CheckedOps wraps CudaOps: each call snapshots its inputs (the residual is often the output itself), runs the kernel,
synchronises and checks the output against RefOps(float64) on the snapshot - the GEMM family and attention with the
rounding-level bounds of tests/bounds.py, GroupNorm, the LayerNorms, softmax_rows and the edge convolutions with
the bounds derived for them there, as are the embeddings, token rows, dwconv7_ln, the CLIP vision embed / head, the
sampler update, and the resampling ops of the spatial modalities (resize_plane, conv2d_small) with the bounds of
tests/bounds_resample.py, the gatedSA2 grid_resample_gate with that of tests/fuser_checks.py; stats_out bit for bit
against its documented summation order; cast, the copies and the patch gathers exactly.  The forwards run with seeded synthetic weights and no CUDA graphs, so
every call of the plan is seen.  A failure lists every violating call with its shapes, strides, flags and tile choice."""
import ctypes as C
import inspect
from collections import defaultdict

import pytest
import torch

import bounds
import bounds_resample
from conftest import assert_close
from fuser_checks import resample_gate_check, stats_check
from ref_ops import RefOps

pytestmark = pytest.mark.gpu
DEV = "cuda:0"

# outputs of the ops that move values without arithmetic, checked bit for bit: name -> (output arguments, rel-L2, max-rel)
SMALL_OPS = {
    "cast": (("y",), 0.0, 0.0), "upsample2x": (("y",), 0.0, 0.0), "im2col_s2": (("y",), 0.0, 0.0),
    "patchify_nchw": (("out",), 0.0, 0.0), "patchify_nhwc": (("out",), 0.0, 0.0),
}


def _snap(x):
    return x.clone() if isinstance(x, torch.Tensor) else (type(x)(_snap(t) for t in x) if isinstance(x, (list, tuple)) else x)


def _desc(t):
    return f"{tuple(t.shape)}/{tuple(t.stride())}/{str(t.dtype)[6:]}" if isinstance(t, torch.Tensor) else repr(t)


class CheckedOps:
    """CudaOps with a float64 check after every call (records, never raises)."""

    def __init__(self, inner, max_elems=None):
        """max_elems: bytes of one float64 intermediate of the GEMM, softmax and attention checks, which then run in row
        chunks (bounds.gemm_check); None checks each GEMM and softmax call whole."""
        self.inner = inner
        self.max_elems = max_elems
        self.ref = RefOps(DEV, compute_dtype=torch.float64)
        self.records = defaultdict(list)          # kind -> [(elementwise ratio, aggregate ratio)]
        self.failures = []
        self.sms = torch.cuda.get_device_properties(DEV).multi_processor_count

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
        rep = bounds.gemm_check(out, a0, w, splits=8, what=what, max_elems=self.max_elems, **snap)
        kind = "conv3x3" if kw.get("conv") is not None else "gemm+ln" if kw.get("ln") is not None else "gemm"
        self.records[kind + (" fp32" if out.dtype == torch.float32 else "")].append((rep.ratio, rep.agg_ratio))
        if not rep.ok:
            self._fail(str(rep))

    def attention(self, q, k, v, out, heads, d_head, causal=False):
        q0, k0, v0 = q.clone(), k.clone(), v.clone()
        self.inner.attention(q, k, v, out, heads, d_head, causal=causal)
        torch.cuda.synchronize()
        chunk = {} if self.max_elems is None else dict(max_elems=self.max_elems)
        rep = bounds.attention_check(out, q0, k0, v0, heads, d_head, causal=causal, **chunk,
                                     what=f"attention q={_desc(q)} k={_desc(k)} out={_desc(out)} heads={heads} d={d_head} causal={causal}")
        self.records["attention"].append((rep.ratio, 0.0))
        if not rep.ok:
            self._fail(str(rep))

    def _record(self, kind, rep):
        self.records[kind].append((rep.ratio, rep.agg_ratio))
        if not rep.ok:
            self._fail(str(rep))

    def groupnorm(self, x, y, gamma, beta, stats, groups, eps, silu):
        x0 = x.clone()
        self.inner.groupnorm(x, y, gamma, beta, stats, groups, eps, silu)
        torch.cuda.synchronize()
        B, HW, Cc = x.shape
        path = bounds.gn_dispatch(B, HW, Cc, groups, aligned8=(x.data_ptr() | y.data_ptr()) % 8 == 0)
        self._record("groupnorm", bounds.groupnorm_check(y, x0, gamma, beta, groups, eps, silu, path, num_sms=self.sms,
                                                         what=f"groupnorm x={_desc(x)} y={_desc(y)} silu={silu} eps={eps}"))

    def layernorm(self, x, y, gamma, beta, eps=1e-5):
        x0 = x.clone()
        self.inner.layernorm(x, y, gamma, beta, eps)
        torch.cuda.synchronize()
        self._record("layernorm", bounds.layernorm_check(y, x0, gamma, beta, eps, what=f"layernorm x={_desc(x)} y={_desc(y)}"))

    def layernorm_rows(self, x, y, gamma, beta, C, eps):
        x0 = x.clone()
        self.inner.layernorm_rows(x, y, gamma, beta, C, eps)
        torch.cuda.synchronize()
        what = f"layernorm_rows x={_desc(x)} y={_desc(y)} C={C}"
        self._record("layernorm_rows", bounds.layernorm_check(y[..., :C], x0[..., :C], gamma, beta, eps, what=what))
        if not torch.equal(y[..., C:], torch.zeros_like(y[..., C:])):
            self._fail(f"{what}: padding columns not zero")

    def layernorm_rows_f32(self, x, y, gamma, beta, eps):
        x0 = x.clone()
        self.inner.layernorm_rows_f32(x, y, gamma, beta, eps)
        torch.cuda.synchronize()
        self._record("layernorm_rows_f32", bounds.layernorm_check(y, x0, gamma, beta, eps, what=f"layernorm_rows_f32 x={_desc(x)}"))

    def softmax_rows(self, s, p, scale):
        s0 = s.clone()
        self.inner.softmax_rows(s, p, scale)
        torch.cuda.synchronize()
        self._record("softmax_rows", bounds.softmax_check(p, s0, scale, what=f"softmax_rows s={_desc(s)}", max_elems=self.max_elems))

    def conv_in(self, x, extra, w, bias, out):
        self.inner.conv_in(x, extra, w, bias, out)
        torch.cuda.synchronize()
        self._record("conv_in", bounds.conv_check(out, x, w, bias, "in", extra=extra, what=f"conv_in x={_desc(x)} out={_desc(out)}"))

    def conv_out(self, x, w, bias, out, H, W):
        self.inner.conv_out(x, w, bias, out, H, W)
        torch.cuda.synchronize()
        self._record("conv_out", bounds.conv_check(out, x, w, bias, "out", H, W, what=f"conv_out x={_desc(x)} out={_desc(out)}"))

    def timestep_embedding(self, t, out):
        self.inner.timestep_embedding(t, out)
        torch.cuda.synchronize()
        self._record("timestep_embedding", bounds.timestep_embedding_check(out, t, what=f"timestep_embedding out={_desc(out)}"))

    def position_features(self, feat, feat_mask, null_feat, coords, pos_mask, null_pos, out, freqs):
        self.inner.position_features(feat, feat_mask, null_feat, coords, pos_mask, null_pos, out, freqs)
        torch.cuda.synchronize()
        self._record("position_features", bounds.position_features_check(out, feat, feat_mask, null_feat, coords, pos_mask, null_pos, freqs,
                                                                         what=f"position_features out={_desc(out)}"))

    def sampler_update(self, x, e_cond, e_uncond, guidance, olds, coefs, a_t, a_prev, e_out, x_prev):
        snap = [_snap(v) for v in (x, e_cond, e_uncond, olds)]
        self.inner.sampler_update(x, e_cond, e_uncond, guidance, olds, coefs, a_t, a_prev, e_out, x_prev)
        torch.cuda.synchronize()
        self._record("sampler_update", bounds.sampler_update_check(e_out, x_prev, snap[0], snap[1], snap[2], guidance, snap[3], coefs, a_t, a_prev))

    def embed_tokens(self, ids, table, pos, out):
        self.inner.embed_tokens(ids, table, pos, out)
        torch.cuda.synchronize()
        self._record("embed_tokens", bounds.embed_tokens_check(out, ids, table, pos, what=f"embed_tokens out={_desc(out)}"))

    def spatial_tokens(self, x, mask, null_feat, pos, y, n):
        x0 = x.clone()
        self.inner.spatial_tokens(x, mask, null_feat, pos, y, n)
        torch.cuda.synchronize()
        self._record("spatial_tokens", bounds.spatial_tokens_check(y, x0, mask, null_feat, pos, n, what=f"spatial_tokens y={_desc(y)}"))

    def dwconv7_ln(self, x, y, w, bias, gamma, beta, B, H, W, C, eps):
        x0 = x.clone()
        self.inner.dwconv7_ln(x, y, w, bias, gamma, beta, B, H, W, C, eps)
        torch.cuda.synchronize()
        what = f"dwconv7_ln x={_desc(x)} y={_desc(y)} C={C}"
        self._record("dwconv7_ln", bounds.dwconv7_ln_check(y, x0, w, bias, gamma, beta, B, H, W, C, eps, what=what))
        yv = y.reshape(B * H * W, -1)
        if not torch.equal(yv[:, C:], torch.zeros_like(yv[:, C:])):
            self._fail(f"{what}: padding columns not zero")

    def clip_vision_embed(self, patch, cls, pos, gamma, beta, x, P, eps):
        self.inner.clip_vision_embed(patch, cls, pos, gamma, beta, x, P, eps)
        torch.cuda.synchronize()
        self._record("clip_vision_embed", bounds.clip_vision_embed_check(x, patch, cls, pos, gamma, beta, P, eps, what=f"clip_vision_embed x={_desc(x)}"))

    def clip_image_head(self, x, gamma, beta, w_proj, pooled, embeds, proj=None, feature=None, target_norm=28.7, eps=1e-5):
        self.inner.clip_image_head(x, gamma, beta, w_proj, pooled, embeds, proj, feature, target_norm, eps)
        torch.cuda.synchronize()
        self._record("clip_image_head", bounds.clip_image_head_check(pooled, embeds, x, gamma, beta, w_proj, eps))

    def resize_plane(self, x, y, C, mode):
        x0 = x.clone()
        self.inner.resize_plane(x, y, C, mode)
        torch.cuda.synchronize()
        self._record("resize_plane", bounds_resample.resize_check(y, x0, mode, what=f"resize_plane x={_desc(x)} y={_desc(y)} {mode}"))

    def conv2d_small(self, x, w, bias, y, k, stride, pad, silu, virtual=None):
        x0 = x.clone()
        self.inner.conv2d_small(x, w, bias, y, k, stride, pad, silu, virtual=virtual)
        torch.cuda.synchronize()
        what = f"conv2d_small x={_desc(x)} y={_desc(y)} k={k} stride={stride} pad={pad} silu={silu} virtual={virtual}"
        # with max_elems, one image at a time (the float64 check holds every tap of the batch at once)
        step = x.shape[0] if self.max_elems is None else 1
        reps = [bounds_resample.conv2d_small_check(y[b:b + step], x0[b:b + step], w, bias, k, stride, pad, silu, virtual, what=f"{what} b={b}")
                for b in range(0, x.shape[0], step)]
        self._record("conv2d_small", max(reps, key=lambda r: (r.ratio, r.agg_ratio)))

    def grid_resample_gate(self, grid, x, gate, stats_out, g, n):
        x0, grid0 = x.clone(), grid.clone()
        self.inner.grid_resample_gate(grid, x, gate, stats_out, g, n)
        torch.cuda.synchronize()
        B, C = grid.shape[0], grid.shape[2]
        gv = float(gate.item())
        worst = 0.0
        for b in range(B):                              # one image at a time keeps the float64 gather small
            rep = resample_gate_check(x[b:b + 1], x0[b:b + 1], grid0[b:b + 1], gv, g, n, what=f"grid_resample_gate g={g} n={n} C={C} b={b}")
            worst = max(worst, rep.ratio)
            if not rep.ok:
                self._fail(str(rep))
        rep = stats_check(stats_out, x.reshape(-1, C))
        if not rep.ok:
            self._fail(str(rep))
        self.records["grid_resample_gate"].append((worst, 0.0))

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


def _unet_forward(cuda_ops, name, B, cfg_batch, map_size=None):
    from gligen_b200 import synth
    from gligen_b200.engine import Engine
    from gligen_b200.spec import NAMED_CONFIGS, SPATIAL_MAP_KEY, synthetic_state_dict
    from inpaint_mask_func import draw_masks_from_boxes
    cfg = NAMED_CONFIGS[name]
    ops = CheckedOps(cuda_ops)
    eng = Engine(cfg, ops, use_graphs=False)
    eng.load_state_dict(synthetic_state_dict(cfg, 0))
    inp = synth.make_inputs(cfg, B, seed=2, map_size=map_size)
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
    _summary(f"{name} B={B}{' cfg' if cfg_batch else ''}{f' map {map_size[0]}x{map_size[1]}' if map_size else ''}", ops)


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


@pytest.mark.parametrize("name,map_size", [("tiny_hed", (192, 320)), ("tiny_normal", (300, 224)), ("tiny_sem", (300, 224)),
                                           ("tiny_depth", (480, 640))])
def test_census_tiny_non_square_map(cuda_ops, name, map_size):
    """The spatial front end on non-square maps: resampling ratios that are not integers and differ between the axes."""
    _unet_forward(cuda_ops, name, 2, True, map_size)


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
