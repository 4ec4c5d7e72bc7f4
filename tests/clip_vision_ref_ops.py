"""The torch checker ops (tests/ref_ops.py) extended by the CLIP image tower's two kernels.  Test infrastructure only.

Each method is the plain-PyTorch statement of the contract in include/gligen_b200.h (glg_clip_vision_embed, glg_clip_image_head),
with the same arguments as the same-named gligen_b200.ops.CudaOps method."""
from __future__ import annotations

import torch
import torch.nn.functional as F

from ref_ops import RefOps


class ClipVisionRefOps(RefOps):
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
