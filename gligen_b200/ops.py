"""Operator layer of the engine: every method enqueues exactly the CUDA kernels of libgligen_b200.so on
the current torch stream.  torch is used for memory and streams only.

`CudaOps` is the product backend.  The engine is written against this interface so that tests can
inject a torch-fp32 checker backend (tests/ref_ops.py) to validate the engine's wiring on a CPU-only box;
the product never does.
"""
from __future__ import annotations

import ctypes as C
from typing import Optional

import torch

from . import lib as L


def _rows_view(t: torch.Tensor):
    """(ptr, rows, cols, ld) of a tensor whose last dim is contiguous and whose leading dims collapse to
    uniformly strided rows (e.g. a channel slice of a [B, HW, Ctot] concat buffer)."""
    assert t.stride(-1) == 1, "last dim must be contiguous"
    cols = t.shape[-1]
    if t.dim() == 1:
        return t.data_ptr(), 1, cols, cols
    ld = t.stride(-2)
    rows = t.shape[-2]
    for i in range(t.dim() - 3, -1, -1):
        assert t.shape[i] == 1 or t.stride(i) == t.stride(i + 1) * t.shape[i + 1], f"non-uniform row stride {t.shape} {t.stride()}"
        rows *= t.shape[i]
    return t.data_ptr(), rows, cols, ld


def gn_scratch_floats(B: int, groups: int = 32) -> int:
    """GLG_GN_SCRATCH_FLOATS of include/gligen_b200.h (the first 128 words must be zero before the first call)."""
    return 128 + 2 * groups * (8 * 148 + B)


def _ptr(t: Optional[torch.Tensor]):
    return None if t is None else t.data_ptr()


def round_up(x: int, m: int) -> int:
    return (x + m - 1) // m * m


class EngineBase:
    """What every engine shares: its ops backend, and weights staged on the ops' device in the activation dtype (`_a`) or in
    fp32 (`_f`)."""

    def __init__(self, ops):
        self.ops, self.dev, self.adt = ops, ops.device, ops.act_dtype

    def _a(self, t: torch.Tensor) -> torch.Tensor:
        return t.detach().to(device=self.dev, dtype=self.adt).contiguous()

    def _f(self, t: torch.Tensor) -> torch.Tensor:
        return t.detach().to(device=self.dev, dtype=torch.float32).contiguous()

    @staticmethod
    def _pack_conv3(w: torch.Tensor) -> torch.Tensor:
        """[Cout, Cin, 3, 3] -> [9*Cout, Cin] (tap-major), the weight of gemm(conv=...)."""
        co, ci = w.shape[:2]
        return w.permute(2, 3, 0, 1).reshape(9 * co, ci)


# gemm(act=...): the epilogue activation, GLG_ACT_* of include/gligen_b200.h
ACT_NONE, ACT_SILU, ACT_GELU, ACT_QUICK_GELU = 0, 1, 2, 3


class CudaOps:
    """bf16 activations / fp32 statistics on one CUDA device."""

    name = "cuda"
    act_dtype = torch.bfloat16

    def __init__(self, device):
        self.device = torch.device(device)
        if self.device.type != "cuda":
            raise L.GligenLibraryError("CudaOps needs a CUDA device (there is no CPU fallback)")
        self.lib = L.load()
        self._c = self.lib           # where op calls go: the library, or a recorder standing in for it (gligen_b200/export.py)
        self.trace = None          # set to a list to record (kind, algorithmic flops, algorithmic bytes) per op call
        # fp32 scratch for split-K GEMMs (8 slabs of the largest small-M output: 8 x 1024 x 2560 floats = 80 MiB)
        self.splitk_ws = torch.empty(8 * 1024 * 2560, device=self.device, dtype=torch.float32)

    def _note(self, kind, flops=0.0, nbytes=0.0):
        if self.trace is not None:
            self.trace.append((kind, float(flops), float(nbytes)))

    # -- helpers --------------------------------------------------------------------------------
    def _stream(self):
        return torch.cuda.current_stream(self.device).cuda_stream

    def launch_count(self) -> int:
        return int(self.lib.glg_launch_count())

    def reset_launch_count(self) -> None:
        self.lib.glg_reset_launch_count()

    # -- tensor-core GEMM / conv --------------------------------------------------------------
    def gemm(self, a, w, out, bias=None, rowbias=None, rows_per_batch=1, act=0, gate=None, residual=None,
             geglu=False, conv=None, ln=None, stats_out=None):
        """out = epilogue(a @ w.T).  `conv=(B,H,W)` selects the implicit 3x3 convolution (w is [9*N, K]).
        ln=(stats [S,M,2] fp32 slot-major, colsum [N] fp32, eps): LayerNorm of the A rows folded into the epilogue.
        stats_out [S,M,2] fp32: per-row partial (sum, sumsq) of the stored output, one slot per 32 columns.
        Both may be row ranges of a larger [S, rows, 2] tensor (views `t[:, lo:hi]`): the slot stride is passed on.
        `out` may be a [B, rows, N] view whose batch stride is not rows*ld (batch-strided rows)."""
        ap, M, K, lda = _rows_view(a)
        g = L.GlgGemmArgs()
        if out.dim() == 3 and out.shape[0] > 1 and out.stride(0) != out.stride(1) * out.shape[1]:
            assert out.stride(2) == 1
            op, Mo, No, ldc = out.data_ptr(), out.shape[0] * out.shape[1], out.shape[2], out.stride(1)
            g.out_rows_per_batch, g.out_batch_stride = out.shape[1], out.stride(0)
        else:
            op, Mo, No, ldc = _rows_view(out)
            g.out_rows_per_batch, g.out_batch_stride = 0, 0
        N = No * 2 if geglu else No
        assert Mo == M, (Mo, M)
        assert w.is_contiguous() and w.shape[1] == K and w.shape[0] == (9 * N if conv else N), (w.shape, N, K)
        g.A, g.lda, g.W, g.out, g.ldc = ap, lda, w.data_ptr(), op, ldc
        g.M, g.N, g.K = M, N, K
        g.out_fp32 = 1 if out.dtype == torch.float32 else 0
        g.bias = _ptr(bias)
        if rowbias is not None:
            rp, _, rc, rld = _rows_view(rowbias)
            assert rc == N and rowbias.dtype == torch.float32
            g.rowbias, g.ld_rowbias, g.rows_per_batch = rp, rld, rows_per_batch
        else:
            g.rowbias, g.ld_rowbias, g.rows_per_batch = None, 0, 1
        g.act = act
        g.gate = _ptr(gate)
        if residual is not None:
            rp, Mr, Nr, ldr = _rows_view(residual)
            assert Mr == M and Nr == No
            g.residual, g.ldr = rp, ldr
        else:
            g.residual, g.ldr = None, 0
        g.geglu = 1 if geglu else 0
        if conv is not None:
            g.conv_mode, g.Bn, g.H, g.Wd = 1, conv[0], conv[1], conv[2]
        else:
            g.conv_mode, g.Bn, g.H, g.Wd = 0, 0, 0, 0
        if ln is not None:
            st, colsum, eps = ln
            assert st.dtype == torch.float32 and st.dim() == 3 and st.shape[1] == M and st.shape[2] == 2 and st.stride(2) == 1 and st.stride(1) == 2
            assert colsum.dtype == torch.float32 and colsum.numel() == N
            g.ln_stats, g.ln_colsum, g.ln_slots, g.ln_eps = st.data_ptr(), colsum.data_ptr(), st.shape[0], eps
            g.ln_slot_stride = st.stride(0) // 2
        else:
            g.ln_stats, g.ln_colsum, g.ln_slots, g.ln_eps, g.ln_slot_stride = None, None, 0, 0.0, 0
        if stats_out is not None:
            so = stats_out
            assert so.dtype == torch.float32 and so.dim() == 3 and so.shape[1] == M and so.shape[2] == 2 and so.stride(2) == 1 and so.stride(1) == 2
            g.stats_out, g.stats_slots, g.stats_slot_stride = so.data_ptr(), so.shape[0], so.stride(0) // 2
        else:
            g.stats_out, g.stats_slots, g.stats_slot_stride = None, 0, 0
        g.splitk_ws, g.splitk_ws_bytes = self.splitk_ws.data_ptr(), self.splitk_ws.numel() * 4
        L.check(self._c.glg_gemm(C.byref(g), self._stream()), "glg_gemm")
        taps = 9 if conv is not None else 1
        self._note("conv3x3" if conv is not None else "gemm", 2.0 * M * N * K * taps,
                   2.0 * (M * K + N * K * taps + M * No) + (2.0 * M * No if residual is not None else 0.0))

    # -- attention ---------------------------------------------------------------------------------
    def attention(self, q, k, v, out, heads: int, d_head: int, causal: bool = False):
        """q [B, Lq, heads*d] / k, v [B, Lk, heads*d] strided views; out [B, Lq, heads*d]."""
        a = L.GlgAttnArgs()
        B, Lq, _ = q.shape
        Lk = k.shape[1]
        for t in (q, k, v, out):
            assert t.stride(-1) == 1
        a.q, a.k, a.v, a.out = q.data_ptr(), k.data_ptr(), v.data_ptr(), out.data_ptr()
        a.q_row, a.k_row, a.v_row, a.o_row = q.stride(1), k.stride(1), v.stride(1), out.stride(1)
        a.q_batch, a.k_batch, a.v_batch, a.o_batch = q.stride(0), k.stride(0), v.stride(0), out.stride(0)
        a.B, a.heads, a.d_head, a.Lq, a.Lk = B, heads, d_head, Lq, Lk
        a.scale = float(d_head) ** -0.5
        a.causal = 1 if causal else 0
        L.check(self._c.glg_attention(C.byref(a), self._stream()), "glg_attention")
        self._note("attention", 4.0 * B * heads * Lq * Lk * d_head, 2.0 * B * heads * d_head * (2 * Lq + 2 * Lk))

    # -- norms ---------------------------------------------------------------------------------------
    def groupnorm(self, x, y, gamma, beta, stats, groups: int, eps: float, silu: bool):
        """x, y: [B, HW, C] (strided rows); stats: fp32 scratch [B*groups*2]."""
        B, HW, Cc = x.shape
        xp, _, _, ldx = _rows_view(x)
        yp, _, _, ldy = _rows_view(y)
        L.check(self._c.glg_groupnorm(xp, ldx, yp, ldy, gamma.data_ptr(), beta.data_ptr(), stats.data_ptr(),
                                       B, HW, Cc, groups, eps, 1 if silu else 0, self._stream()), "glg_groupnorm")
        self._note("groupnorm", 0.0, 2.0 * B * HW * Cc * 3)

    def layernorm(self, x, y, gamma, beta, eps: float = 1e-5):
        """x [B, rows, C] with contiguous rows inside a batch; y likewise (batch strides may differ)."""
        B, rows, Cc = x.shape
        assert x.stride(2) == 1 and x.stride(1) == Cc and y.stride(2) == 1 and y.stride(1) == Cc
        L.check(self._c.glg_layernorm(x.data_ptr(), x.stride(0), y.data_ptr(), y.stride(0), gamma.data_ptr(), beta.data_ptr(),
                                       B, rows, Cc, eps, self._stream()), "glg_layernorm")
        self._note("layernorm", 0.0, 2.0 * B * rows * Cc * 2)

    # -- small ops -----------------------------------------------------------------------------------
    def conv_in(self, x, extra, w, bias, out):
        B, C0, H, W = x.shape
        assert x.is_contiguous() and x.dtype == torch.float32
        C1 = 0 if extra is None else extra.shape[1]
        if extra is not None:
            assert extra.is_contiguous() and extra.dtype == torch.float32
        op, _, Cout, ldo = _rows_view(out)
        L.check(self._c.glg_conv_in(x.data_ptr(), C0, _ptr(extra), C1, w.data_ptr(), bias.data_ptr(), op, ldo,
                                     B, H, W, Cout, self._stream()), "glg_conv_in")
        self._note("conv_in")

    def conv_out(self, x, w, bias, out, H: int, W: int):
        """x [B, HW, Cin] bf16 -> out [B, Cout, H, W] fp32."""
        B, _, Cin = x.shape
        xp, _, _, ldx = _rows_view(x)
        assert out.is_contiguous() and out.dtype == torch.float32
        L.check(self._c.glg_conv_out(xp, ldx, w.data_ptr(), bias.data_ptr(), out.data_ptr(), B, H, W, Cin, out.shape[1],
                                      self._stream()), "glg_conv_out")
        self._note("conv_out")

    def upsample2x(self, x, y, H: int, W: int):
        B, _, Cc = x.shape
        xp, _, _, ldx = _rows_view(x)
        yp, _, _, ldy = _rows_view(y)
        L.check(self._c.glg_upsample2x(xp, ldx, yp, ldy, B, H, W, Cc, self._stream()), "glg_upsample2x")
        self._note("upsample2x")

    def im2col_s2(self, x, y, H: int, W: int, pad_lo: int = 1):
        B, _, Cc = x.shape
        xp, _, _, ldx = _rows_view(x)
        assert y.is_contiguous()
        if pad_lo == 1:
            L.check(self._c.glg_im2col_s2(xp, ldx, y.data_ptr(), B, H, W, Cc, self._stream()), "glg_im2col_s2")
        else:
            L.check(self._c.glg_im2col_s2_pad(xp, ldx, y.data_ptr(), B, H, W, Cc, pad_lo, self._stream()), "glg_im2col_s2_pad")
        self._note("im2col_s2")

    def timestep_embedding(self, t, out):
        assert t.dtype == torch.int64 and out.is_contiguous()
        L.check(self._c.glg_timestep_embedding(t.data_ptr(), out.data_ptr(), out.shape[0], out.shape[1], self._stream()),
                "glg_timestep_embedding")
        self._note("timestep_embedding")

    def position_features(self, feat, feat_mask, null_feat, coords, pos_mask, null_pos, out, freqs: int):
        """feat [B,N,F] or [N,F] (broadcast) fp32; coords [B,N,nc]; out [B*N, ldo] bf16."""
        B, N, nc = coords.shape
        F_ = feat.shape[-1]
        fbs = 0 if feat.dim() == 2 else feat.stride(0)
        for t in (feat, feat_mask, null_feat, coords, pos_mask, null_pos):
            assert t.is_contiguous() and t.dtype == torch.float32
        assert out.is_contiguous()
        L.check(self._c.glg_position_features(feat.data_ptr(), fbs, feat_mask.data_ptr(), null_feat.data_ptr(), coords.data_ptr(),
                                               pos_mask.data_ptr(), null_pos.data_ptr(), out.data_ptr(), out.shape[-1],
                                               B, N, F_, nc, freqs, self._stream()), "glg_position_features")
        self._note("position_features")

    # -- spatial grounding modalities (ConvNeXt tokenizer, grounding downsamplers): once per sample -------------
    def patchify_nchw(self, x, out, Hv: int, Wv: int, k: int):
        """x fp32 [B, C, Hs, Ws] resampled (nearest) onto Hv x Wv, k x k stride-k patches -> out bf16 [B*(Hv/k)*(Wv/k), ldo]."""
        B, Cc, Hs, Ws = x.shape
        assert x.is_contiguous() and x.dtype == torch.float32 and out.is_contiguous() and out.dim() == 2
        L.check(self._c.glg_patchify_nchw(x.data_ptr(), out.data_ptr(), out.shape[1], B, Cc, Hs, Ws, Hv, Wv, k, self._stream()), "glg_patchify_nchw")
        self._note("patchify")

    def patchify_nhwc(self, x, out, H: int, W: int, C: int, k: int):
        """x bf16 rows [B*H*W, ldx] (first C columns used) -> out bf16 [B*(H/k)*(W/k), k*k*C]."""
        xp, rows, _, ldx = _rows_view(x)
        assert out.is_contiguous() and out.dim() == 2
        L.check(self._c.glg_patchify_nhwc(xp, ldx, out.data_ptr(), out.shape[1], rows // (H * W), H, W, C, k, self._stream()), "glg_patchify_nhwc")
        self._note("patchify")

    def layernorm_rows(self, x, y, gamma, beta, C: int, eps: float):
        """LayerNorm over the first C columns of each row of x [rows, Cpad]; y columns [C, Cpad) are zeroed."""
        xp, rows, cp, ldx = _rows_view(x)
        yp, _, cpy, ldy = _rows_view(y)
        L.check(self._c.glg_layernorm_rows(xp, ldx, yp, ldy, gamma.data_ptr(), beta.data_ptr(), rows, C, cpy, eps, self._stream()), "glg_layernorm_rows")
        self._note("layernorm_rows", 0.0, 4.0 * rows * C)

    def layernorm_rows_f32(self, x, y, gamma, beta, eps: float):
        """LayerNorm of bf16 rows x [rows, C] -> fp32 y [rows, C]."""
        xp, rows, Cc, ldx = _rows_view(x)
        yp, _, _, ldy = _rows_view(y)
        assert y.dtype == torch.float32
        L.check(self._c.glg_layernorm_rows_f32(xp, ldx, yp, ldy, gamma.data_ptr(), beta.data_ptr(), rows, Cc, eps, self._stream()), "glg_layernorm_rows_f32")
        self._note("layernorm_rows", 0.0, 6.0 * rows * Cc)

    def embed_tokens(self, ids, table, pos, out):
        """out[b, l] = table[ids[b, l]] + pos[l]  (ids int64 [B, L]; table fp32 [V, C]; pos fp32 [L, C]; out bf16 [B*L, C])."""
        B, Lt = ids.shape
        assert ids.dtype == torch.int64 and ids.is_contiguous() and table.is_contiguous() and pos.is_contiguous() and pos.shape[0] >= Lt
        op, _, Cc, ldo = _rows_view(out)
        L.check(self._c.glg_embed_tokens(ids.data_ptr(), table.data_ptr(), table.shape[0], pos.data_ptr(), op, ldo, B, Lt, Cc, self._stream()), "glg_embed_tokens")
        self._note("embed_tokens")

    def clip_vision_embed(self, patch, cls, pos, gamma, beta, x, P: int, eps: float):
        """x bf16 rows [N*(P+1), C]: row n*(P+1) = LN(cls + pos[0]), row n*(P+1)+1+p = LN(patch[n*P+p] + pos[1+p]); patch fp32 [N*P, C]."""
        pp, rows, Cc, ldp = _rows_view(patch)
        xp, xrows, _, ldx = _rows_view(x)
        assert patch.dtype == torch.float32 and rows % P == 0 and xrows == rows // P * (P + 1)
        assert cls.is_contiguous() and pos.is_contiguous() and pos.shape == (P + 1, Cc)
        L.check(self._c.glg_clip_vision_embed(pp, ldp, cls.data_ptr(), pos.data_ptr(), gamma.data_ptr(), beta.data_ptr(), xp, ldx, rows // P, P, Cc,
                                               eps, self._stream()), "glg_clip_vision_embed")
        self._note("clip_vision_embed", 0.0, 2.0 * xrows * Cc * 5)

    def clip_image_head(self, x, gamma, beta, w_proj, pooled, embeds, proj=None, feature=None, target_norm: float = 28.7, eps: float = 1e-5):
        """x bf16 [N, T, C] (row 0 of each image is read): pooled fp32 [N, C] = LN(x[:, 0]), embeds fp32 [N, D] = pooled w_proj^T,
        feature fp32 [N, D] = target_norm * f / |f| with f = embeds proj (when proj is given)."""
        N, _, Cc = x.shape
        D = w_proj.shape[0]
        assert x.stride(-1) == 1 and w_proj.is_contiguous() and w_proj.shape == (D, Cc)
        assert pooled.is_contiguous() and pooled.shape == (N, Cc) and embeds.is_contiguous() and embeds.shape == (N, D)
        assert (proj is None) == (feature is None)
        if proj is not None:
            assert proj.is_contiguous() and proj.shape == (D, D) and feature.is_contiguous() and feature.shape == (N, D)
        L.check(self._c.glg_clip_image_head(x.data_ptr(), x.stride(0), gamma.data_ptr(), beta.data_ptr(), w_proj.data_ptr(), _ptr(proj),
                                             float(target_norm), pooled.data_ptr(), embeds.data_ptr(), _ptr(feature), N, Cc, D, eps, self._stream()),
                "glg_clip_image_head")
        self._note("clip_image_head", 2.0 * N * D * (Cc + (D if proj is not None else 0)), 4.0 * D * (Cc + D))

    def dwconv7_ln(self, x, y, w, bias, gamma, beta, B: int, H: int, W: int, C: int, eps: float):
        """depthwise 7x7 + bias + LayerNorm over the first C channels: x, y bf16 rows [B*H*W, Cpad]; w fp32 [49, C]."""
        xp, _, _, ldx = _rows_view(x)
        yp, _, cpy, ldy = _rows_view(y)
        L.check(self._c.glg_dwconv7_ln(xp, ldx, yp, ldy, w.data_ptr(), bias.data_ptr(), gamma.data_ptr(), beta.data_ptr(), B, H, W, C, cpy, eps,
                                        self._stream()), "glg_dwconv7_ln")
        self._note("dwconv7_ln", 98.0 * B * H * W * C, 4.0 * B * H * W * C)

    def spatial_tokens(self, x, mask, null_feat, pos, y, n: int):
        """y[b, t] = x[b, t] * mask[b] + null_feat * (1 - mask[b]) + pos[t]; x, y bf16 [B*n, C]."""
        xp, rows, Cc, ldx = _rows_view(x)
        yp, _, _, ldy = _rows_view(y)
        L.check(self._c.glg_spatial_tokens(xp, ldx, mask.data_ptr(), null_feat.data_ptr(), pos.data_ptr(), yp, ldy, rows // n, n, Cc, self._stream()),
                "glg_spatial_tokens")
        self._note("spatial_tokens")

    def resize_plane(self, x, y, C: int, mode: str):
        """F.interpolate of channels 0..C-1 of x fp32 [B, Cx, Hs, Ws] -> y fp32 [B, C, Ho, Wo]; mode "nearest" | "bicubic"."""
        assert x.is_contiguous() and y.is_contiguous() and x.dtype == torch.float32 and y.dtype == torch.float32 and y.shape[1] == C
        L.check(self._c.glg_resize_plane(x.data_ptr(), x.stride(0), y.data_ptr(), x.shape[0], C, x.shape[2], x.shape[3], y.shape[2], y.shape[3],
                                          {"nearest": 0, "bicubic": 1}[mode], self._stream()), "glg_resize_plane")
        self._note("resize_plane")

    def conv2d_small(self, x, w, bias, y, k: int, stride: int, pad: int, silu: bool, virtual=None):
        """Direct Conv2d on fp32 NCHW, Cout in {3, 4, 8, 16}; w fp32 packed [Cin*k*k, Cout]; `virtual=(Hv, Wv)`: the input is x
        resampled (nearest) onto that grid first."""
        B, Cin, Hs, Ws = x.shape
        Hv, Wv = virtual or (Hs, Ws)
        assert x.is_contiguous() and y.is_contiguous() and w.is_contiguous() and w.shape == (Cin * k * k, y.shape[1])
        assert y.shape[2] == (Hv + 2 * pad - k) // stride + 1 and y.shape[3] == (Wv + 2 * pad - k) // stride + 1
        L.check(self._c.glg_conv2d_small(x.data_ptr(), w.data_ptr(), bias.data_ptr(), y.data_ptr(), B, Cin, Hs, Ws, Hv, Wv, y.shape[1], k, stride, pad,
                                          1 if silu else 0, self._stream()), "glg_conv2d_small")
        self._note("conv2d_small")

    def softmax_rows(self, s, p, scale: float):
        """s fp32 [rows, cols] (row stride free) -> p bf16 [rows, cols] = softmax(scale * s) along the last dim."""
        assert s.dtype == torch.float32 and s.dim() == 2 and s.stride(1) == 1 and p.dim() == 2 and p.stride(1) == 1 and p.shape == s.shape
        L.check(self._c.glg_softmax_rows(s.data_ptr(), s.stride(0), p.data_ptr(), p.stride(0), s.shape[0], s.shape[1], float(scale), self._stream()),
                "glg_softmax_rows")
        self._note("softmax_rows", 0.0, 6.0 * s.numel())

    def cast(self, x, y):
        """fp32 -> activation dtype, contiguous."""
        assert x.is_contiguous() and y.is_contiguous() and x.dtype == torch.float32 and x.numel() == y.numel()
        L.check(self._c.glg_cast_f32_bf16(x.data_ptr(), y.data_ptr(), x.numel(), self._stream()), "glg_cast_f32_bf16")
        self._note("cast_f32_bf16")

    def sampler_update(self, x, e_cond, e_uncond, guidance, olds, coefs, a_t, a_prev, e_out, x_prev):
        o = list(olds) + [None] * (3 - len(olds))
        for t in (x, e_cond, x_prev):
            assert t.is_contiguous() and t.dtype == torch.float32
        L.check(self._c.glg_sampler_update(x.data_ptr(), e_cond.data_ptr(), _ptr(e_uncond), float(guidance),
                                            _ptr(o[0]), _ptr(o[1]), _ptr(o[2]),
                                            float(coefs[0]), float(coefs[1]), float(coefs[2]), float(coefs[3]),
                                            float(a_t), float(a_prev), _ptr(e_out), x_prev.data_ptr(), x.numel(), self._stream()),
                "glg_sampler_update")
        self._note("sampler_update")
