"""CPU ORACLE for image-to-image sampling: the samplers started part-way down their grid.  TEST INFRASTRUCTURE ONLY.

A run at strength s over the L-step grid time_range = np.flip(ddim_timesteps(S)) runs its last n = min(L, int(s L)) steps from
t0 = time_range[L - n], at x = sqrt(abar_t0) init + sqrt(1 - abar_t0) noise.

  * PLMS / DDIM (ref_sample): the REFERENCE's own per-step methods, PLMSSampler.p_sample_plms / DDIMSampler.p_sample_ddim, over
    the truncated range, started with the reference's LatentDiffusion.q_sample.  Needs the reference mounted in this process
    (oracle/ref_harness.mount) before the first import of `ldm`.
  * DPM-Solver++ / UniPC (fast_sample): the float64 loops of oracle/dpm_solver_oracle.py and oracle/unipc_oracle.py on the
    truncated grid (its time steps, then alphas_cumprod[0]).

eps_fn(x, t, cond) is the model, as in oracle/sampler_oracle.py; on_alpha(alpha) runs before each step's model pass with the
scheduled-sampling alphas alpha_generator(n, alpha_type), over the steps run.
"""
from __future__ import annotations

import math
from typing import List, Optional

import numpy as np
import torch

from oracle import dpm_solver_oracle as DO
from oracle import sampler_oracle as SO
from oracle import unipc_oracle as UPO


def truncated_range(S: int, strength: float):
    """(the time steps run, L)."""
    full = np.flip(SO.ddim_timesteps(S))
    L = len(full)
    n = min(L, int(strength * L))
    return full[L - n:].copy(), L


def init_and_noise(shape, seed: int):
    """A seeded stand-in for an encoded image (smooth, std ~ 1) and the start noise."""
    g = torch.Generator().manual_seed(seed)
    B, C, H, W = shape
    coarse = torch.randn(B, C, max(H // 4, 1), max(W // 4, 1), generator=g)
    init = torch.nn.functional.interpolate(coarse, size=(H, W), mode="bilinear", align_corners=False)
    init = init / init.std() * 0.9
    return init, torch.randn(shape, generator=g)


def _alphas(n, alpha_type):
    return None if alpha_type is None else SO.alpha_generator(n, alpha_type)


@torch.no_grad()
def fast_sample(kind: str, eps_fn: SO.EpsFn, S: int, strength: float, init, noise, sched=None, use_cfg=True,
                guidance_scale=7.5, order: int = 2, alpha_type: Optional[List[float]] = None, on_alpha=None, mask=None, x0=None):
    """kind "dpm" (DPM-Solver++) or "unipc".  Generator draws: one q_sample noise per step with a mask."""
    sched = sched or SO.make_schedule()
    time_range, _ = truncated_range(S, strength)
    n = len(time_range)
    if n == 0:
        return init.float()
    b = init.shape[0]
    t0 = torch.full((b,), int(time_range[0]), dtype=torch.long)
    x = SO.q_sample(sched, init.float(), t0, noise.float()).double()
    ac = sched["alphas_cumprod"].double()
    grid = [float(ac[int(t)]) for t in time_range] + [float(ac[0])]
    al = [math.sqrt(v) for v in grid]
    sg = [math.sqrt(1.0 - v) for v in grid]
    alphas = _alphas(n, alpha_type)
    use_cfg = use_cfg and guidance_scale != 1

    def data_pred(i, xx):
        if alphas is not None and on_alpha is not None:
            on_alpha(alphas[i])
        ts = torch.full((b,), int(time_range[i]), dtype=torch.long)
        if mask is not None:
            xx = SO.q_sample(sched, x0, ts).double() * mask + (1.0 - mask) * xx
        e = SO._cfg_eps(eps_fn, xx.float(), ts, use_cfg, guidance_scale).double()
        return xx, (xx - sg[i] * e) / al[i]

    solve = DO.solve if kind == "dpm" else UPO.solve
    return solve(x, al, sg, order, data_pred).float()


class _EpsModel:
    """What the reference's per-step methods call as self.model(input): the grounded pass when input carries grounding_input,
    the unconditional one otherwise (their unconditional input dict has none)."""

    def __init__(self, eps_fn):
        self.eps_fn = eps_fn

    def __call__(self, input):
        return self.eps_fn(input["x"], input["timesteps"], "grounding_input" in input)


@torch.no_grad()
def ref_sample(kind: str, eps_fn: SO.EpsFn, S: int, strength: float, init, noise, guidance_scale=7.5,
               alpha_type: Optional[List[float]] = None, on_alpha=None, mask=None, x0=None):
    """kind "plms" or "ddim": the reference sampler's loop body (plms.py:84-106, ddim.py:81-104) over the truncated range.
    Generator draws as the reference's: one sigma = 0 noise per x_prev, one q_sample noise per step with a mask."""
    from oracle import ref_harness as RH
    RH.mount()
    from ldm.models.diffusion.ddim import DDIMSampler
    from ldm.models.diffusion.plms import PLMSSampler
    cls = PLMSSampler if kind == "plms" else DDIMSampler
    assert RH.is_reference_module(cls)
    diffusion = RH.ref_diffusion("cpu")
    sampler = cls(diffusion, _EpsModel(eps_fn))
    sampler.make_schedule(ddim_num_steps=S)
    time_range, L = truncated_range(S, strength)
    n = len(time_range)
    if n == 0:
        return init.float()
    b = init.shape[0]
    t0 = torch.full((b,), int(time_range[0]), dtype=torch.long)
    img = diffusion.q_sample(init.float(), t0, noise=noise.float())
    # the keys the reference's unconditional input copies; "grounding_input" marks the grounded pass for _EpsModel
    input = dict(x=img, timesteps=None, context=None, grounding_input=True, inpainting_extra_input=None, grounding_extra_input=None)
    alphas = _alphas(n, alpha_type)
    old_eps = []
    for i, step in enumerate(time_range):
        if alphas is not None and on_alpha is not None:
            on_alpha(alphas[i])
        index = L - (L - n + i) - 1                            # the full grid's index of this step
        ts = torch.full((b,), int(step), dtype=torch.long)
        if mask is not None:
            img = diffusion.q_sample(x0, ts) * mask + (1.0 - mask) * img
            input["x"] = img
        if kind == "plms":
            ts_next = torch.full((b,), int(time_range[min(i + 1, n - 1)]), dtype=torch.long)
            img, _, e_t = sampler.p_sample_plms(input, ts, index=index, uc=True, guidance_scale=guidance_scale, old_eps=old_eps,
                                                t_next=ts_next)
            old_eps.append(e_t)
            if len(old_eps) >= 4:
                old_eps.pop(0)
        else:
            input["timesteps"] = ts
            img, _ = sampler.p_sample_ddim(input, index=index, uc=True, guidance_scale=guidance_scale)
        input["x"] = img
    return img
