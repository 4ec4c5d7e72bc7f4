"""VAE decoder and encoder on the engine's kernels (SURVEY 8f rank 1: the step right after the sampling loop; rank 3: the
inpainting front end `autoencoder.encode(image)`, gligen_inference.py:403-404).

    AutoencoderKL.decode      ldm/models/autoencoder.py:40-44       z / scale_factor -> post_quant_conv -> Decoder
    Decoder.forward           ldm/modules/diffusionmodules/model.py:535-568
    ResnetBlock.forward       model.py:121-141   (temb is None in the VAE)
    AttnBlock.forward         model.py:178-202   (single head over H*W tokens, head dim = C = 512)
    Upsample.forward          model.py:53-57     (nearest x2, then 3x3 conv)

Same building blocks as the UNet engine: channels-last bf16 activations, GroupNorm(+SiLU) as the single-launch kernel,
every 3x3 / 1x1 convolution as the wgmma implicit GEMM with bias / residual in its epilogue (tiles that are segments
of one image row for the 256- and 512-wide levels), nearest upsample as one gather pass.  Restructurings, exact in real
arithmetic:
  * z / scale_factor -> post_quant_conv (1x1) -> conv_in (3x3) is ONE 3x3 convolution over [z, 1]: the 1x1 weights and
    1 / scale_factor are folded into the 3x3 weights; post_quant_conv's bias travels through a constant ones channel so
    that the zero padding of conv_in still sees zeros outside the image;
  * the mid attention has one head of dim 512 (O would not fit in registers next to S), so it runs as three GEMMs with an fp32
    score matrix and a row-softmax kernel between them:  S = Q K^T,  P = softmax(S * C^-1/2),  O = P V  with
    V^T = W_v hn^T produced directly in the [C, HW] layout the second GEMM wants; the bias of v is added after P.V
    (rows of P sum to 1).
Encoder (model.py:434-459, autoencoder.py:34-38): conv_in from the fp32 NCHW image, ResnetBlocks as above, Downsample
(model.py:73-77: zero pad on the right / bottom only, 3x3 stride 2) as a gather (`im2col_s2` with pad_lo = 0) + GEMM, the same
mid attention, and conv_out -> quant_conv (1x1) folded into ONE 3x3 convolution (W' = W_q W_out, b' = W_q b_out + b_q) that
writes the fp32 moments; the posterior sample (clamp, exp, CPU-generator noise) stays with the caller, which owns the RNG.
There is no CPU fallback; a tensor-core tile needs every channel count to be a multiple of 64 (true for ch >= 64).
"""
from __future__ import annotations

from typing import Dict

import torch

from .ops import EngineBase, gn_scratch_floats
from .spec import VAEDecoderConfig


class _VAEEngineBase(EngineBase):
    def __init__(self, cfg: VAEDecoderConfig, ops):
        super().__init__(ops)
        self.cfg = cfg
        self.W: Dict[str, torch.Tensor] = {}
        self.loaded = False
        chans = [cfg.ch * m for m in cfg.ch_mult]
        if any(c % 64 for c in chans):
            raise ValueError(f"VAE channels {chans} must be multiples of 64 for the tensor-core tiles")

    # ---- weights ---------------------------------------------------------------------------------------------
    def _load_res(self, sd, prefix):
        W = self.W
        for n in ("norm1", "norm2"):
            W[f"{prefix}.{n}.g"], W[f"{prefix}.{n}.b"] = self._f(sd[f"{prefix}.{n}.weight"]), self._f(sd[f"{prefix}.{n}.bias"])
        for n in ("conv1", "conv2"):
            W[f"{prefix}.{n}.w"] = self._a(self._pack_conv3(sd[f"{prefix}.{n}.weight"]))
            W[f"{prefix}.{n}.b"] = self._f(sd[f"{prefix}.{n}.bias"])
        if f"{prefix}.nin_shortcut.weight" in sd:
            w = sd[f"{prefix}.nin_shortcut.weight"]
            W[f"{prefix}.nin.w"] = self._a(w.reshape(w.shape[0], w.shape[1]))
            W[f"{prefix}.nin.b"] = self._f(sd[f"{prefix}.nin_shortcut.bias"])

    def _load_attn(self, sd, a):
        W = self.W
        W[f"{a}.norm.g"], W[f"{a}.norm.b"] = self._f(sd[f"{a}.norm.weight"]), self._f(sd[f"{a}.norm.bias"])
        for n in ("q", "k", "v", "proj_out"):
            w = sd[f"{a}.{n}.weight"]
            W[f"{a}.{n}.w"] = self._a(w.reshape(w.shape[0], w.shape[1]))
            W[f"{a}.{n}.b"] = self._f(sd[f"{a}.{n}.bias"])

    # ---- shared blocks ---------------------------------------------------------------------------------------------
    def _buf(self, *shape, dtype=None):
        return torch.empty(*shape, device=self.dev, dtype=dtype or self.adt)

    def _gn(self, x, g, b, silu, stats):
        y = torch.empty_like(x)
        self.ops.groupnorm(x, y, g, b, stats, 32, 1e-6, silu)
        return y

    def _resblock(self, x, prefix, B, H, Wd, stats):
        ops, W = self.ops, self.W
        cout = W[f"{prefix}.conv1.b"].numel()
        h = self._gn(x, W[f"{prefix}.norm1.g"], W[f"{prefix}.norm1.b"], True, stats)
        h1 = self._buf(B, H * Wd, cout)
        ops.gemm(h, W[f"{prefix}.conv1.w"], h1, bias=W[f"{prefix}.conv1.b"], conv=(B, H, Wd))
        h = self._gn(h1, W[f"{prefix}.norm2.g"], W[f"{prefix}.norm2.b"], True, stats)
        if f"{prefix}.nin.w" in W:
            sk = self._buf(B, H * Wd, cout)
            ops.gemm(x, W[f"{prefix}.nin.w"], sk, bias=W[f"{prefix}.nin.b"])
        else:
            sk = x
        out = self._buf(B, H * Wd, cout)
        ops.gemm(h, W[f"{prefix}.conv2.w"], out, bias=W[f"{prefix}.conv2.b"], residual=sk, conv=(B, H, Wd))
        return out

    def _attn(self, x, a, B, H, Wd, stats):
        """T = H * Wd tokens; the P.V GEMM has K = T, so T must be a multiple of 64.  The fp32 T x T score matrix is
        materialised (1 GiB at T = 16384, a 1024 x 1024 image)."""
        ops, W = self.ops, self.W
        T, C = H * Wd, x.shape[-1]
        hn = self._gn(x, W[f"{a}.norm.g"], W[f"{a}.norm.b"], False, stats)
        q, k = self._buf(B, T, C), self._buf(B, T, C)
        ops.gemm(hn, W[f"{a}.q.w"], q, bias=W[f"{a}.q.b"])
        ops.gemm(hn, W[f"{a}.k.w"], k, bias=W[f"{a}.k.b"])
        o = self._buf(B, T, C)
        vt = self._buf(C, T)
        s = self._buf(T, T, dtype=torch.float32)
        pr = self._buf(T, T)
        for b in range(B):                                  # one image at a time: the score matrix is T x T
            ops.gemm(W[f"{a}.v.w"], hn[b], vt)              # V^T [C, T] = W_v hn_b^T   (bias added after P.V)
            ops.gemm(q[b], k[b], s)                         # S = Q K^T, fp32
            ops.softmax_rows(s, pr, float(C) ** -0.5)
            ops.gemm(pr, vt, o[b], bias=W[f"{a}.v.b"])      # O = P V + b_v
        out = self._buf(B, T, C)
        ops.gemm(o, W[f"{a}.proj_out.w"], out, bias=W[f"{a}.proj_out.b"], residual=x)
        return out


class VAEDecoderEngine(_VAEEngineBase):
    def load_state_dict(self, sd: Dict[str, torch.Tensor]) -> None:
        cfg, W = self.cfg, self.W
        W.clear()
        # (z / sf) -> post_quant_conv -> conv_in  ==  conv3x3 over [z, 1]
        wpq = sd["post_quant_conv.weight"].float().reshape(cfg.z_channels, cfg.embed_dim)        # [m, i]
        bpq = sd["post_quant_conv.bias"].float()
        win = sd["decoder.conv_in.weight"].float()                                                # [o, m, 3, 3]
        wz = torch.einsum("omyx,mi->oiyx", win, wpq) / cfg.scale_factor                          # z channels
        w1 = torch.einsum("omyx,m->oyx", win, bpq).unsqueeze(1)                                  # ones channel
        wfull = torch.cat([wz, w1], dim=1)                                                        # [o, embed+1, 3, 3]
        W["conv_in.w"] = self._f(wfull.permute(2, 3, 1, 0).reshape(9, cfg.embed_dim + 1, -1))     # [9][Cin][Cout]
        W["conv_in.b"] = self._f(sd["decoder.conv_in.bias"])

        res = lambda prefix: self._load_res(sd, prefix)
        res("decoder.mid.block_1")
        res("decoder.mid.block_2")
        self._load_attn(sd, "decoder.mid.attn_1")
        for i_level in range(len(cfg.ch_mult)):
            for i_block in range(cfg.num_res_blocks + 1):
                res(f"decoder.up.{i_level}.block.{i_block}")
            if i_level != 0:
                p = f"decoder.up.{i_level}.upsample.conv"
                W[f"{p}.w"], W[f"{p}.b"] = self._a(self._pack_conv3(sd[f"{p}.weight"])), self._f(sd[f"{p}.bias"])
        W["norm_out.g"], W["norm_out.b"] = self._f(sd["decoder.norm_out.weight"]), self._f(sd["decoder.norm_out.bias"])
        wo = sd["decoder.conv_out.weight"].float()                                               # [3, C, 3, 3]
        W["conv_out.w"] = self._f(wo.permute(2, 3, 0, 1).reshape(9, wo.shape[0], wo.shape[1]))   # [9][Cout][Cin]
        W["conv_out.b"] = self._f(sd["decoder.conv_out.bias"])
        self.loaded = True

    @torch.no_grad()
    def decode(self, z: torch.Tensor) -> torch.Tensor:
        """z: fp32 [B, embed_dim, h, w] (the sampler's latent) -> image fp32 [B, out_ch, 8h, 8w] (for 4 levels)."""
        assert self.loaded, "load_state_dict first"
        cfg, ops, W = self.cfg, self.ops, self.W
        B, _, H, Wd = z.shape
        if H <= 0 or Wd <= 0 or H % 8 or Wd % 8:
            # the mid attention's P.V GEMM reduces over h*w tokens, which must be a multiple of 64
            raise ValueError(f"latent {H}x{Wd}: both sides must be positive multiples of 8")
        z = z.to(device=self.dev, dtype=torch.float32).contiguous()
        ones = torch.ones(B, 1, H, Wd, device=self.dev, dtype=torch.float32)
        stats = torch.zeros(gn_scratch_floats(B), device=self.dev, dtype=torch.float32)
        block_in = cfg.ch * cfg.ch_mult[-1]
        h = self._buf(B, H * Wd, block_in)
        ops.conv_in(z, ones, W["conv_in.w"], W["conv_in.b"], h)
        h = self._resblock(h, "decoder.mid.block_1", B, H, Wd, stats)
        h = self._attn(h, "decoder.mid.attn_1", B, H, Wd, stats)
        h = self._resblock(h, "decoder.mid.block_2", B, H, Wd, stats)
        for i_level in reversed(range(len(cfg.ch_mult))):
            for i_block in range(cfg.num_res_blocks + 1):
                h = self._resblock(h, f"decoder.up.{i_level}.block.{i_block}", B, H, Wd, stats)
            if i_level != 0:
                C = h.shape[-1]
                up = self._buf(B, 4 * H * Wd, C)
                ops.upsample2x(h, up, H, Wd)
                H, Wd = 2 * H, 2 * Wd
                h = self._buf(B, H * Wd, C)
                p = f"decoder.up.{i_level}.upsample.conv"
                ops.gemm(up, W[f"{p}.w"], h, bias=W[f"{p}.b"], conv=(B, H, Wd))
        h = self._gn(h, W["norm_out.g"], W["norm_out.b"], True, stats)
        img = torch.empty(B, cfg.out_ch, H, Wd, device=self.dev, dtype=torch.float32)
        ops.conv_out(h, W["conv_out.w"], W["conv_out.b"], img, H, Wd)
        return img


class VAEEncoderEngine(_VAEEngineBase):
    """`encoder.*` + `quant_conv.*` -> posterior moments (mean | logvar), fp32 [B, 2 * embed_dim, h, w]."""

    def load_state_dict(self, sd: Dict[str, torch.Tensor]) -> None:
        cfg, W = self.cfg, self.W
        W.clear()
        wi = sd["encoder.conv_in.weight"].float()                                                 # [o, c, 3, 3]
        W["conv_in.w"] = self._f(wi.permute(2, 3, 1, 0).reshape(9, wi.shape[1], wi.shape[0]))     # [9][Cin][Cout]
        W["conv_in.b"] = self._f(sd["encoder.conv_in.bias"])
        nlev = len(cfg.ch_mult)
        for i_level in range(nlev):
            for i_block in range(cfg.num_res_blocks):
                self._load_res(sd, f"encoder.down.{i_level}.block.{i_block}")
            if i_level != nlev - 1:
                p = f"encoder.down.{i_level}.downsample.conv"
                w = sd[p + ".weight"]                                                             # [o, c, 3, 3]
                W[p + ".w"] = self._a(w.permute(0, 2, 3, 1).reshape(w.shape[0], 9 * w.shape[1]))  # k = tap * C + c (im2col order)
                W[p + ".b"] = self._f(sd[p + ".bias"])
        self._load_res(sd, "encoder.mid.block_1")
        self._load_res(sd, "encoder.mid.block_2")
        self._load_attn(sd, "encoder.mid.attn_1")
        W["norm_out.g"], W["norm_out.b"] = self._f(sd["encoder.norm_out.weight"]), self._f(sd["encoder.norm_out.bias"])
        # conv_out (3x3, C -> 2z) then quant_conv (1x1, 2z -> 2e): one 3x3 convolution
        wo, bo = sd["encoder.conv_out.weight"].float(), sd["encoder.conv_out.bias"].float()      # [m, C, 3, 3]
        wq = sd["quant_conv.weight"].float().reshape(2 * cfg.embed_dim, 2 * cfg.z_channels)      # [o, m]
        wf = torch.einsum("om,mcyx->ocyx", wq, wo)
        W["conv_out.w"] = self._f(wf.permute(2, 3, 0, 1).reshape(9, wf.shape[0], wf.shape[1]))   # [9][Cout][Cin]
        W["conv_out.b"] = self._f(wq @ bo + sd["quant_conv.bias"].float())
        self.loaded = True

    @torch.no_grad()
    def encode_moments(self, x: torch.Tensor) -> torch.Tensor:
        """x: fp32 image [B, in_channels, H, W] -> moments fp32 [B, 2 * embed_dim, H / 2^(levels-1), W / 2^(levels-1)]."""
        assert self.loaded, "load_state_dict first"
        cfg, ops, W = self.cfg, self.ops, self.W
        B, Cin, H, Wd = x.shape
        nlev = len(cfg.ch_mult)
        assert Cin == cfg.in_channels, (Cin, cfg.in_channels)
        f = 1 << (nlev - 1)
        if H <= 0 or Wd <= 0 or H % f or Wd % f:
            # one factor 2 per stride-2 downsample.  On the GPU the mid attention's P.V GEMM also needs (H/f)*(W/f) to be a
            # multiple of 64, which glg_gemm reports itself.
            raise ValueError(f"image {H}x{Wd}: both sides must be positive multiples of {f}")
        x = x.to(device=self.dev, dtype=torch.float32).contiguous()
        stats = torch.zeros(gn_scratch_floats(B), device=self.dev, dtype=torch.float32)
        h = self._buf(B, H * Wd, cfg.ch)
        ops.conv_in(x, None, W["conv_in.w"], W["conv_in.b"], h)
        for i_level in range(nlev):
            for i_block in range(cfg.num_res_blocks):
                h = self._resblock(h, f"encoder.down.{i_level}.block.{i_block}", B, H, Wd, stats)
            if i_level != nlev - 1:
                p = f"encoder.down.{i_level}.downsample.conv"
                C = h.shape[-1]
                col = self._buf(B * (H // 2) * (Wd // 2), 9 * C)
                ops.im2col_s2(h, col, H, Wd, pad_lo=0)
                H, Wd = H // 2, Wd // 2
                h = self._buf(B, H * Wd, C)
                ops.gemm(col, W[p + ".w"], h, bias=W[p + ".b"])
                del col
        h = self._resblock(h, "encoder.mid.block_1", B, H, Wd, stats)
        h = self._attn(h, "encoder.mid.attn_1", B, H, Wd, stats)
        h = self._resblock(h, "encoder.mid.block_2", B, H, Wd, stats)
        h = self._gn(h, W["norm_out.g"], W["norm_out.b"], True, stats)
        mom = torch.empty(B, 2 * cfg.embed_dim, H, Wd, device=self.dev, dtype=torch.float32)
        ops.conv_out(h, W["conv_out.w"], W["conv_out.b"], mom, H, Wd)
        return mom
