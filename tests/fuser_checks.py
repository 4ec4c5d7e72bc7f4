"""Checks shared by the gatedCA / gatedSA2 fuser tests: the torch statement of glg_grid_resample_gate (a RefOps with that method,
so that CPU checker plans of gatedSA2 models run) and its rounding-level bound against float64.

glg_grid_resample_gate (csrc/fuser.cu) computes, per output pixel and channel,
    acc~ = the fp32 bicubic interpolant of the fp32 grid (the arithmetic of resize_plane, bounded by bounds_resample.bicubic_axis:
           |acc~ - acc| <= E),
    v    = fma(gate, acc~, x)                      one fp32 rounding: |v - (x + gate acc)| <= |gate| E + u (|ref| + |gate| E) = e1,
    out  = bf16(v)                                 half a bf16 ulp at |v| <= |ref| + e1,
with ref = x + gate * acc in float64, x the bf16 input.  The statistics are fp32 sums over one 32-column slot of the stored bf16
values (and of their squares, each square exact in fp32): |s~ - s| <= g(32) sum |out|, |sq~ - sq| <= g(33) sum out^2.
"""
from __future__ import annotations

import torch
import torch.nn.functional as F

from bounds import U, Report, g_n, half_ulp
from bounds_resample import KEYS_SLOPE, bicubic_axis
from ref_ops import RefOps


class FuserRefOps(RefOps):
    """RefOps plus the gatedSA2 residual kernel."""

    def grid_resample_gate(self, grid, x, gate, stats_out, g, n):
        self.launches += 1
        B, GG, C = grid.shape
        up = F.interpolate(grid.to(self.cd).permute(0, 2, 1).reshape(B, C, g, g), (n, n), mode="bicubic")
        v = x.reshape(B, n * n, C).to(self.cd) + gate.to(self.cd) * up.reshape(B, C, n * n).permute(0, 2, 1)
        stored = v.to(x.dtype)
        x.copy_(stored.view(x.shape))
        sv = stored.to(self.cd).reshape(B * n * n, C // 32, 32)
        stats_out[:, :, 0] = sv.sum(2).t()
        stats_out[:, :, 1] = (sv * sv).sum(2).t()


def bicubic_tokens(grid, g, n):
    """(float64 bicubic_{g->n} of grid [B, g*g, C] as [B, n*n, C], the bound E of the kernel's fp32 value of it)."""
    f64 = torch.float64
    B, _, C = grid.shape
    dev = grid.device
    iy, cy, dcy, dy = bicubic_axis(g, n, dev)
    ix, cx, dcx, dx = bicubic_axis(g, n, dev)
    g4 = g_n(4)
    x = grid.to(f64).reshape(B, g, g, C)
    a = x.abs()
    tap, atap = x[:, :, ix], a[:, :, ix]                                  # [B, g rows, n, 4, C]
    cxv, dcxv = cx[None, None, :, :, None], dcx[None, None, :, :, None]
    rows = (tap * cxv).sum(3)                                             # [B, g, n, C]
    er = (atap * dcxv).sum(3) + g4 * (atap * (cxv.abs() + dcxv)).sum(3)
    R = (1 + g4) * (atap * (cxv.abs() + dcxv)).sum(3)
    A = atap.sum(3)
    cyv, dcyv = cy[None, :, :, None, None], dcy[None, :, :, None, None]  # [1, n, 4, 1, 1]
    ref = (rows[:, iy] * cyv).sum(2)                                      # rows[:, iy]: [B, n, 4, n, C]
    err = (cyv.abs() * er[:, iy]).sum(2) + (dcyv * R[:, iy]).sum(2) + g4 * ((cyv.abs() + dcyv) * R[:, iy]).sum(2)
    d = dy[None, :, None, None] + dx[None, None, :, None]
    xmax = a.amax(dim=(1, 2))[:, None, None, :]
    err = err + KEYS_SLOPE * d * A[:, iy].sum(2) + 0.75 * d * d * xmax
    return ref.reshape(B, n * n, C), err.reshape(B, n * n, C)


def resample_gate_check(out, x, grid, gate, g, n, what="grid_resample_gate") -> Report:
    """out: the stored rows [B, n*n, C] (bf16); x: the rows before the call; grid fp32 [B, g*g, C]; gate a float.
    Elementwise ratio to the bound above, and rel-L2 against 1.25x that of perfectly rounded bf16 outputs."""
    f64 = torch.float64
    acc, E = bicubic_tokens(grid, g, n)
    gv = float(gate)
    ref = x.to(f64) + gv * acc
    e1 = abs(gv) * E + U * (ref.abs() + abs(gv) * E)
    bound = e1 + half_ulp(ref.abs() + e1, torch.bfloat16)
    got = out.to(f64).reshape(ref.shape)
    diff = (got - ref).abs()
    r = torch.where(diff == 0, torch.zeros_like(diff), diff / bound)
    i = int(torch.argmax(r))
    ideal = (ref.to(torch.bfloat16).to(f64) - ref).norm().item()
    rl2 = (got - ref).norm().item()
    agg = 0.0 if rl2 == 0 else rl2 / (1.25 * ideal) if ideal > 0 else float("inf")
    idx = [int(v) for v in torch.unravel_index(torch.tensor(i), tuple(ref.shape))]
    return Report(what, r.reshape(-1)[i].item(), agg, f"(worst at {idx}: got {got.reshape(-1)[i].item():.6g} ref {ref.reshape(-1)[i].item():.6g})")


def stats_check(stats, out, what="grid_resample_gate stats") -> Report:
    """stats [C/32, rows, 2] against float64 sums of the stored values out [rows, C]."""
    f64 = torch.float64
    v = out.to(f64).reshape(-1, out.shape[-1] // 32, 32)
    s, sq = v.sum(2).t(), (v * v).sum(2).t()
    bs, bq = g_n(32) * v.abs().sum(2).t(), g_n(33) * (v * v).sum(2).t()
    r = torch.maximum(torch.where(bs > 0, (stats[..., 0].to(f64) - s).abs() / bs, (stats[..., 0].to(f64) - s).abs() * float("inf")),
                      torch.where(bq > 0, (stats[..., 1].to(f64) - sq).abs() / bq, (stats[..., 1].to(f64) - sq).abs() * float("inf")))
    r = torch.nan_to_num(r, nan=0.0)
    return Report(what, r.max().item())
