"""torch-fp32 CHECKER backend with the same operator interface as gligen_b200.ops.CudaOps.

Test infrastructure only (lives under tests/).  Two uses:
  * on a CPU-only box: run the engine's plan with these ops to verify weight packing / buffer wiring of
    gligen_b200.engine against the oracle and the golden fixtures;
  * on the GPU: per-kernel parity - every CudaOps method is compared against the same-named method here.
Each method is the plain-PyTorch statement of the contract documented in include/gligen_b200.h.
"""
from __future__ import annotations

import math

import torch
import torch.nn.functional as F


class RefOps:
    name = "ref"

    def __init__(self, device="cpu", act_dtype=torch.float32, compute_dtype=torch.float32):
        """compute_dtype: precision of the statement (fp32 by default; fp64 for the rounding-level bounds of tests/bounds.py)."""
        self.device = torch.device(device)
        self.act_dtype = act_dtype
        self.cd = compute_dtype
        self.launches = 0

    def launch_count(self):
        return self.launches

    def reset_launch_count(self):
        self.launches = 0

    # ------------------------------------------------------------------------------------------
    def gemm(self, a, w, out, bias=None, rowbias=None, rows_per_batch=1, act=0, gate=None, residual=None,
             geglu=False, conv=None, ln=None, stats_out=None):
        self.launches += 1
        K = a.shape[-1]
        A = a.reshape(-1, K).to(self.cd)
        Wf = w.to(self.cd)
        if conv is not None:
            B, H, Wd = conv
            N = w.shape[0] // 9
            if self.cd == torch.float64:      # fp64 convolution is slow on CUDA: nine shifted GEMMs instead
                xp = F.pad(A.reshape(B, H, Wd, K), (0, 0, 1, 1, 1, 1))
                wt = Wf.view(9, N, K)
                y = sum(xp[:, t // 3:t // 3 + H, t % 3:t % 3 + Wd].reshape(-1, K) @ wt[t].t() for t in range(9))
            else:
                x = A.reshape(B, H, Wd, K).permute(0, 3, 1, 2)
                wk = Wf.view(3, 3, N, K).permute(2, 3, 0, 1)
                y = F.conv2d(x, wk, padding=1).permute(0, 2, 3, 1).reshape(B * H * Wd, N)
        else:
            y = A @ Wf.t()
        M = y.shape[0]
        if ln is not None:       # LayerNorm fold: rstd * (x W'^T - mu * colsum)   (gamma in W', beta in the bias)
            st, colsum, eps = ln
            s1, s2 = st[:, :, 0].sum(0), st[:, :, 1].sum(0)          # slot-major [S, M, 2]
            mu = s1 / K
            rstd = torch.rsqrt((s2 / K - mu * mu).clamp_min(0) + eps)
            y = rstd[:, None] * (y - mu[:, None] * colsum.to(self.cd)[None])
        if geglu:
            y = y + bias.to(self.cd)[None]
            n2 = y.shape[1] // 2
            t = y.view(M, n2 // 128, 2, 128)
            v = (t[:, :, 0] * F.gelu(t[:, :, 1])).reshape(M, n2)
        else:
            v = y
            if bias is not None:
                v = v + bias.to(self.cd)[None]
            if rowbias is not None:
                idx = torch.arange(M, device=v.device) // rows_per_batch
                v = v + rowbias.to(self.cd)[idx]
            if act == 1:
                v = F.silu(v)
            elif act == 2:
                v = F.gelu(v)
            elif act == 3:
                v = v * torch.sigmoid(1.702 * v)
            if gate is not None:
                v = v * gate.to(self.cd)
            if residual is not None:
                v = v + residual.reshape(M, -1).to(self.cd)
        stored = v.view(out.shape).to(out.dtype)
        out.copy_(stored)
        if stats_out is not None:
            sv = stored.to(self.cd).reshape(M, -1, 32)               # one partial per 32-column chunk
            stats_out[:, :, 0] = sv.sum(2).t()                       # slot-major [S, M, 2]
            stats_out[:, :, 1] = (sv * sv).sum(2).t()

    def attention(self, q, k, v, out, heads, d_head, causal=False):
        self.launches += 1
        B, Lq, _ = q.shape
        Lk = k.shape[1]
        qf = q.to(self.cd).reshape(B, Lq, heads, d_head).permute(0, 2, 1, 3)
        kf = k.to(self.cd).reshape(B, Lk, heads, d_head).permute(0, 2, 1, 3)
        vf = v.to(self.cd).reshape(B, Lk, heads, d_head).permute(0, 2, 1, 3)
        sim = torch.einsum("bhic,bhjc->bhij", qf, kf) * (d_head ** -0.5)
        if causal:
            sim = sim.masked_fill(torch.ones(Lq, Lk, dtype=torch.bool, device=sim.device).triu(1), float("-inf"))
        o = torch.einsum("bhij,bhjc->bhic", sim.softmax(dim=-1), vf)
        out.copy_(o.permute(0, 2, 1, 3).reshape(B, Lq, heads * d_head).to(out.dtype))

    # -- spatial grounding modalities ----------------------------------------------------------------------------
    def patchify_nchw(self, x, out, Hv, Wv, k):
        self.launches += 1
        B, C = x.shape[:2]
        xv = F.interpolate(x.to(self.cd), (Hv, Wv))
        p = xv.view(B, C, Hv // k, k, Wv // k, k).permute(0, 2, 4, 3, 5, 1).reshape(-1, k * k * C)       # (b, oy, ox), (ky, kx, c)
        out.zero_()
        out[:, : k * k * C] = p.to(out.dtype)

    def patchify_nhwc(self, x, out, H, W, C, k):
        self.launches += 1
        xv = x.reshape(-1, H, W, x.shape[-1])[..., :C]
        B = xv.shape[0]
        out.copy_(xv.reshape(B, H // k, k, W // k, k, C).permute(0, 1, 3, 2, 4, 5).reshape(-1, k * k * C))

    def layernorm_rows(self, x, y, gamma, beta, C, eps):
        self.launches += 1
        v = F.layer_norm(x[..., :C].to(self.cd), (C,), gamma.to(self.cd), beta.to(self.cd), eps)
        y.zero_()
        y[..., :C] = v.to(y.dtype)

    def layernorm_rows_f32(self, x, y, gamma, beta, eps):
        self.launches += 1
        C = x.shape[-1]
        y.copy_(F.layer_norm(x.to(self.cd), (C,), gamma.to(self.cd), beta.to(self.cd), eps).reshape(y.shape))

    def embed_tokens(self, ids, table, pos, out):
        self.launches += 1
        Lt = ids.shape[1]
        out.copy_((table.to(self.cd)[ids] + pos.to(self.cd)[:Lt][None]).reshape(out.shape).to(out.dtype))

    def clip_vision_embed(self, patch, cls, pos, gamma, beta, x, P, eps):
        self.launches += 1
        C = pos.shape[1]
        p = patch.reshape(-1, P, C).to(self.cd)
        t = torch.cat([cls.to(self.cd).view(1, 1, C).expand(p.shape[0], 1, C), p], dim=1) + pos.to(self.cd)[None]
        x.copy_(F.layer_norm(t, (C,), gamma.to(self.cd), beta.to(self.cd), eps).reshape(x.shape).to(x.dtype))

    def clip_image_head(self, x, gamma, beta, w_proj, pooled, embeds, proj=None, feature=None, target_norm=28.7, eps=1e-5):
        self.launches += 1
        C = x.shape[-1]
        y = F.layer_norm(x[:, 0].to(self.cd), (C,), gamma.to(self.cd), beta.to(self.cd), eps)
        e = y @ w_proj.to(self.cd).t()
        pooled.copy_(y)
        embeds.copy_(e)
        if proj is not None:
            f = e @ proj.to(self.cd)
            feature.copy_(f * (target_norm / f.norm(dim=-1, keepdim=True)))

    def dwconv7_ln(self, x, y, w, bias, gamma, beta, B, H, W, C, eps):
        self.launches += 1
        xv = x.reshape(B, H, W, -1)[..., :C].permute(0, 3, 1, 2).to(self.cd)
        h = F.conv2d(xv, w.to(self.cd).t().reshape(C, 1, 7, 7), bias.to(self.cd), padding=3, groups=C).permute(0, 2, 3, 1)
        v = F.layer_norm(h, (C,), gamma.to(self.cd), beta.to(self.cd), eps).reshape(B * H * W, C)
        y.zero_()
        y.reshape(B * H * W, -1)[:, :C] = v.to(y.dtype)

    def spatial_tokens(self, x, mask, null_feat, pos, y, n):
        self.launches += 1
        C = x.shape[-1]
        xv = x.reshape(-1, n, C).to(self.cd)
        m = mask.to(self.cd).view(-1, 1, 1)
        y.copy_((xv * m + null_feat.to(self.cd).view(1, 1, -1) * (1 - m) + pos.to(self.cd).view(1, n, C)).reshape(y.shape).to(y.dtype))

    def resize_plane(self, x, y, C, mode):
        self.launches += 1
        y.copy_(F.interpolate(x[:, :C].to(self.cd), tuple(y.shape[2:]), mode=mode))

    def conv2d_small(self, x, w, bias, y, k, stride, pad, silu, virtual=None):
        self.launches += 1
        Cin, Cout = x.shape[1], y.shape[1]
        xv = x.to(self.cd) if virtual is None else F.interpolate(x.to(self.cd), tuple(virtual))
        v = F.conv2d(xv, w.to(self.cd).reshape(Cin, k, k, Cout).permute(3, 0, 1, 2), bias.to(self.cd), stride=stride, padding=pad)
        y.copy_(F.silu(v) if silu else v)

    def softmax_rows(self, s, p, scale):
        self.launches += 1
        p.copy_(torch.softmax(s.to(self.cd) * scale, dim=-1).to(p.dtype))

    def groupnorm(self, x, y, gamma, beta, stats, groups, eps, silu):
        self.launches += 2
        h = F.group_norm(x.to(self.cd).permute(0, 2, 1), groups, gamma.to(self.cd), beta.to(self.cd), eps)
        if silu:
            h = F.silu(h)
        y.copy_(h.permute(0, 2, 1).to(y.dtype))

    def layernorm(self, x, y, gamma, beta, eps=1e-5):
        self.launches += 1
        y.copy_(F.layer_norm(x.to(self.cd), (x.shape[-1],), gamma.to(self.cd), beta.to(self.cd), eps).to(y.dtype))

    def conv_in(self, x, extra, w, bias, out):
        self.launches += 1
        xin = x if extra is None else torch.cat([x, extra], dim=1)
        cin, cout = w.shape[1], w.shape[2]
        wk = w.to(self.cd).view(3, 3, cin, cout).permute(3, 2, 0, 1)
        y = F.conv2d(xin.to(self.cd), wk, bias.to(self.cd), padding=1)
        B = x.shape[0]
        out.copy_(y.permute(0, 2, 3, 1).reshape(B, -1, cout).to(out.dtype))

    def conv_out(self, x, w, bias, out, H, W):
        self.launches += 1
        B, _, cin = x.shape
        cout = w.shape[1]
        wk = w.to(self.cd).view(3, 3, cout, cin).permute(2, 3, 0, 1)
        xin = x.to(self.cd).reshape(B, H, W, cin).permute(0, 3, 1, 2)
        out.copy_(F.conv2d(xin, wk, bias.to(self.cd), padding=1))

    def upsample2x(self, x, y, H, W):
        self.launches += 1
        B, _, C = x.shape
        t = x.reshape(B, H, W, C)
        t = t.repeat_interleave(2, dim=1).repeat_interleave(2, dim=2)
        y.copy_(t.reshape(B, 4 * H * W, C))

    def im2col_s2(self, x, y, H, W, pad_lo=1):
        self.launches += 1
        B, _, C = x.shape
        xin = x.to(self.cd).reshape(B, H, W, C).permute(0, 3, 1, 2)
        xin = F.pad(xin, (pad_lo, 1, pad_lo, 1))                         # even H, W: one zero row / column on the far side
        u = F.unfold(xin, kernel_size=3, padding=0, stride=2)            # [B, C*9, L], (c, tap) ordering
        L = u.shape[-1]
        u = u.view(B, C, 9, L).permute(0, 3, 2, 1).reshape(B * L, 9 * C)   # -> k = tap*C + c
        y.copy_(u.to(y.dtype))

    def timestep_embedding(self, t, out):
        self.launches += 1
        dim = out.shape[1]
        half = dim // 2
        freqs = torch.exp(-math.log(10000.0) * torch.arange(half, dtype=self.cd, device=t.device) / half)
        args = t[:, None].to(self.cd) * freqs[None]
        out.copy_(torch.cat([torch.cos(args), torch.sin(args)], dim=-1).to(out.dtype))

    def position_features(self, feat, feat_mask, null_feat, coords, pos_mask, null_pos, out, freqs):
        self.launches += 1
        B, N, nc = coords.shape
        if feat.dim() == 2:
            feat = feat.unsqueeze(0).expand(B, -1, -1)
        fm = feat_mask.unsqueeze(-1)
        pm = pos_mask.unsqueeze(-1)
        bands = 100.0 ** (torch.arange(freqs, device=coords.device) / freqs)
        emb = []
        for f in bands:
            emb.append(torch.sin(f * coords))
            emb.append(torch.cos(f * coords))
        pe = torch.cat(emb, dim=-1)
        row = torch.cat([feat * fm + (1 - fm) * null_feat.view(1, 1, -1), pe * pm + (1 - pm) * null_pos.view(1, 1, -1)], dim=-1)
        full = torch.zeros(B * N, out.shape[-1], device=coords.device, dtype=self.cd)
        full[:, : row.shape[-1]] = row.reshape(B * N, -1)
        out.copy_(full.to(out.dtype))

    def cast(self, x, y):
        self.launches += 1
        y.copy_(x.reshape(y.shape).to(y.dtype))

    def sampler_update(self, x, e_cond, e_uncond, guidance, olds, coefs, a_t, a_prev, e_out, x_prev):
        self.launches += 1
        e = e_cond
        if e_uncond is not None:
            e = e_uncond + guidance * (e_cond - e_uncond)
        if e_out is not None:
            e_out.copy_(e)
        ep = coefs[0] * e
        for c, o in zip(coefs[1:], olds):
            ep = ep + c * o
        a_t = torch.tensor(a_t, dtype=self.cd)
        a_prev = torch.tensor(a_prev, dtype=self.cd)
        pred_x0 = (x - (1 - a_t).sqrt() * ep) / a_t.sqrt()
        x_prev.copy_(a_prev.sqrt() * pred_x0 + (1 - a_prev).sqrt() * ep)
