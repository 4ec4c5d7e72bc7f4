"""The denoising engine: weight packing, static workspace, and the per-timestep UNet forward expressed as
a flat list of kernel launches (a "plan") that is replayed - directly or as a CUDA graph - every step.

Mirrors UNetModel.forward (reference ldm/modules/diffusionmodules/openaimodel.py:420-464) with these
restructurings, all exact in real arithmetic:
  * channels-last bf16 activations; [B,C,H,W] <-> [B,(HW),C] rearranges of SpatialTransformer
    (attention.py:371,374) disappear;
  * skip connections are written by their producer straight into the channel slice of the concat buffer
    of the output block that will consume them (no torch.cat, openaimodel.py:461);
  * Q/K/V projections fused into one GEMM, GEGLU fused into the FF1 epilogue, bias / time-embedding /
    residual / tanh-gate adds fused into GEMM epilogues, the 22 ResBlock emb projections in one GEMM;
  * cond and uncond passes of classifier-free guidance can run as one 2B batch;
  * the gated self-attention fuser is skipped when scale == 0 (x + 0*f(x), attention.py:241-242).
"""
from __future__ import annotations

from dataclasses import dataclass
from typing import Callable, Dict, List, Optional, Tuple

import torch

from .ops import ACT_SILU, EngineBase, gn_scratch_floats, round_up
from .spec import UNetConfig, block_schedule


class Plan:
    """Static buffers + ordered launch list for one (batch rows, grounding tokens) shape."""

    def __init__(self):
        self.steps: List[Tuple[str, bool, bool, Callable[[], None]]] = []   # (name, fuser_only, static, fn)
        self.static_sig = None      # identity of the inputs the static (timestep-invariant) steps were last run for
        self.inp: Dict[str, torch.Tensor] = {}
        self.out: Optional[torch.Tensor] = None
        self.buffers: List[torch.Tensor] = []     # every device allocation of this plan (inputs, output, workspace)
        self.graphs: Dict[bool, object] = {}
        self.warm: Dict[bool, int] = {}
        self.nlaunch: Dict[bool, int] = {}

    def add(self, name: str, fn: Callable[[], None], fuser: bool = False, static: bool = False) -> None:
        self.steps.append((name, fuser, static, fn))

    def run(self, fuser_on: bool, static: bool) -> None:
        """static=True: only the timestep-invariant steps (functions of context / grounding inputs and weights:
        PositionNet, context cast, attn2 K/V projections, fuser.linear - recomputed 102x per image by the
        reference); static=False: everything else."""
        for _, fuser, st, fn in self.steps:
            if st != static or (fuser and not fuser_on and not static):
                continue
            fn()


class Engine(EngineBase):
    def __init__(self, cfg: UNetConfig, ops, use_graphs: bool = True):
        super().__init__(ops)
        self.cfg = cfg
        self.blocks = block_schedule(cfg)
        self.W: Dict[str, torch.Tensor] = {}
        self.plans: Dict[Tuple[int, ...], Plan] = {}
        self.scale = 1.0
        self.use_graphs = use_graphs and self.dev.type == "cuda"
        self.loaded = False
        self.weights_version = 0
        self._plan_allocs: List[torch.Tensor] = []
        self.kernel_launches = 0       # kernels of libgligen_b200.so executed on behalf of this engine (graph replays included)
        # (prefix of every SpatialTransformer, in execution order) -> index into the gate table
        self.st_prefixes = [ly.prefix for blk in self.blocks for ly in blk.layers if ly.kind == "st"]
        self.res_layers = [ly for blk in self.blocks for ly in blk.layers if ly.kind == "res"]
        self.emb_off: Dict[str, int] = {}
        off = 0
        for ly in self.res_layers:
            self.emb_off[ly.prefix] = off
            off += ly.cout
        self.emb_total = off
        self._last_N: Optional[int] = None      # grounding slots of the last grounded call (shape of the null input)
        self._map_shape: Optional[Tuple[int, int, int]] = None    # spatial modalities: (C, H, W) of the conditioning map
        self.n_streams = 2 if cfg.tokenizer == "text_image" else 1
        self.pos_k = round_up(cfg.tok_feat_dim + cfg.position_dim, 64)

    # ------------------------------------------------------------------------------------------
    # weights
    # ------------------------------------------------------------------------------------------
    @staticmethod
    def _pack_geglu(w: torch.Tensor, *vecs: torch.Tensor):
        """[x rows | gate rows] -> per 256-row tile [128 x | 128 gate] (glg_gemm geglu layout); per-row vectors
        (bias, column sums) are permuted the same way."""
        n2 = w.shape[0] // 2
        assert n2 % 128 == 0, "GEGLU inner dim must be a multiple of 128"
        wx, wg = w[:n2].reshape(n2 // 128, 128, -1), w[n2:].reshape(n2 // 128, 128, -1)
        out = [torch.stack([wx, wg], dim=1).reshape(2 * n2, -1)]
        for b in vecs:
            bx, bg = b[:n2].reshape(n2 // 128, 128), b[n2:].reshape(n2 // 128, 128)
            out.append(torch.stack([bx, bg], dim=1).reshape(2 * n2))
        return out

    def _fold_ln(self, w: torch.Tensor, bias, gamma: torch.Tensor, beta: torch.Tensor):
        """LayerNorm(gamma, beta) followed by Linear(w, bias)  ->  (w * gamma in the activation dtype,
        column sums of THAT rounded matrix, bias + w @ beta), all still in the reference row order."""
        w32 = w.float()
        wf = (w32 * gamma.float()[None, :]).to(self.adt)
        colsum = wf.float().sum(dim=1)
        b = w32 @ beta.float()
        if bias is not None:
            b = b + bias.float()
        return wf, colsum, b

    def load_state_dict(self, sd: Dict[str, torch.Tensor]) -> None:
        cfg, W = self.cfg, self.W
        W.clear()
        W["time_embed.0.w"], W["time_embed.0.b"] = self._a(sd["time_embed.0.weight"]), self._f(sd["time_embed.0.bias"])
        W["time_embed.2.w"], W["time_embed.2.b"] = self._a(sd["time_embed.2.weight"]), self._f(sd["time_embed.2.bias"])
        W["emb_all.w"] = self._a(torch.cat([sd[f"{ly.prefix}.emb_layers.1.weight"] for ly in self.res_layers], dim=0))
        W["emb_all.b"] = self._f(torch.cat([sd[f"{ly.prefix}.emb_layers.1.bias"] for ly in self.res_layers], dim=0))
        self.set_first_conv(sd["input_blocks.0.0.weight"], sd["input_blocks.0.0.bias"])
        for blk in self.blocks:
            for ly in blk.layers:
                p = ly.prefix
                if ly.kind == "res":
                    W[f"{p}.gn1.g"], W[f"{p}.gn1.b"] = self._f(sd[f"{p}.in_layers.0.weight"]), self._f(sd[f"{p}.in_layers.0.bias"])
                    W[f"{p}.conv1.w"] = self._a(self._pack_conv3(sd[f"{p}.in_layers.2.weight"]))
                    W[f"{p}.conv1.b"] = self._f(sd[f"{p}.in_layers.2.bias"])
                    W[f"{p}.gn2.g"], W[f"{p}.gn2.b"] = self._f(sd[f"{p}.out_layers.0.weight"]), self._f(sd[f"{p}.out_layers.0.bias"])
                    W[f"{p}.conv2.w"] = self._a(self._pack_conv3(sd[f"{p}.out_layers.3.weight"]))
                    W[f"{p}.conv2.b"] = self._f(sd[f"{p}.out_layers.3.bias"])
                    if ly.cin != ly.cout:
                        W[f"{p}.skip.w"] = self._a(sd[f"{p}.skip_connection.weight"].reshape(ly.cout, ly.cin))
                        W[f"{p}.skip.b"] = self._f(sd[f"{p}.skip_connection.bias"])
                elif ly.kind == "down":
                    w = sd[f"{p}.op.weight"]
                    W[f"{p}.w"] = self._a(w.permute(0, 2, 3, 1).reshape(w.shape[0], -1))      # [Cout, 9*Cin], k = tap*Cin + c
                    W[f"{p}.b"] = self._f(sd[f"{p}.op.bias"])
                elif ly.kind == "up":
                    W[f"{p}.w"] = self._a(self._pack_conv3(sd[f"{p}.conv.weight"]))
                    W[f"{p}.b"] = self._f(sd[f"{p}.conv.bias"])
                elif ly.kind == "st":
                    C = ly.cin
                    W[f"{p}.gn.g"], W[f"{p}.gn.b"] = self._f(sd[f"{p}.norm.weight"]), self._f(sd[f"{p}.norm.bias"])
                    W[f"{p}.proj_in.w"], W[f"{p}.proj_in.b"] = self._a(sd[f"{p}.proj_in.weight"].reshape(C, C)), self._f(sd[f"{p}.proj_in.bias"])
                    W[f"{p}.proj_out.w"], W[f"{p}.proj_out.b"] = self._a(sd[f"{p}.proj_out.weight"].reshape(C, C)), self._f(sd[f"{p}.proj_out.bias"])
                    tb = f"{p}.transformer_blocks.0"
                    # every LayerNorm -> Linear pair is folded (see include/gligen_b200.h "LayerNorm fold")
                    for a, nrm in (("attn1", "norm1"), ("fuser.attn", "fuser.norm1")):
                        wq = torch.cat([sd[f"{tb}.{a}.to_q.weight"], sd[f"{tb}.{a}.to_k.weight"], sd[f"{tb}.{a}.to_v.weight"]], dim=0)
                        wf, cs, b = self._fold_ln(wq, None, sd[f"{tb}.{nrm}.weight"], sd[f"{tb}.{nrm}.bias"])
                        W[f"{tb}.{a}.qkv.w"], W[f"{tb}.{a}.qkv.s"], W[f"{tb}.{a}.qkv.b"] = wf.to(self.dev).contiguous(), self._f(cs), self._f(b)
                        W[f"{tb}.{a}.out.w"], W[f"{tb}.{a}.out.b"] = self._a(sd[f"{tb}.{a}.to_out.0.weight"]), self._f(sd[f"{tb}.{a}.to_out.0.bias"])
                    wf, cs, b = self._fold_ln(sd[f"{tb}.attn2.to_q.weight"], None, sd[f"{tb}.norm2.weight"], sd[f"{tb}.norm2.bias"])
                    W[f"{tb}.attn2.q.w"], W[f"{tb}.attn2.q.s"], W[f"{tb}.attn2.q.b"] = wf.to(self.dev).contiguous(), self._f(cs), self._f(b)
                    W[f"{tb}.attn2.kv.w"] = self._a(torch.cat([sd[f"{tb}.attn2.to_k.weight"], sd[f"{tb}.attn2.to_v.weight"]], dim=0))
                    W[f"{tb}.attn2.out.w"], W[f"{tb}.attn2.out.b"] = self._a(sd[f"{tb}.attn2.to_out.0.weight"]), self._f(sd[f"{tb}.attn2.to_out.0.bias"])
                    for f, nrm in (("ff", "norm3"), ("fuser.ff", "fuser.norm2")):
                        wf, cs, b = self._fold_ln(sd[f"{tb}.{f}.net.0.proj.weight"], sd[f"{tb}.{f}.net.0.proj.bias"],
                                                  sd[f"{tb}.{nrm}.weight"], sd[f"{tb}.{nrm}.bias"])
                        w1, s1, b1 = self._pack_geglu(wf, cs, b)
                        W[f"{tb}.{f}.w1"], W[f"{tb}.{f}.s1"], W[f"{tb}.{f}.b1"] = w1.to(self.dev).contiguous(), self._f(s1), self._f(b1)
                        W[f"{tb}.{f}.w2"], W[f"{tb}.{f}.b2"] = self._a(sd[f"{tb}.{f}.net.2.weight"]), self._f(sd[f"{tb}.{f}.net.2.bias"])
                    W[f"{tb}.fuser.linear.w"], W[f"{tb}.fuser.linear.b"] = self._a(sd[f"{tb}.fuser.linear.weight"]), self._f(sd[f"{tb}.fuser.linear.bias"])
        W["out.gn.g"], W["out.gn.b"] = self._f(sd["out.0.weight"]), self._f(sd["out.0.bias"])
        W["out.w"] = self._f(sd["out.2.weight"].permute(2, 3, 0, 1).reshape(9, cfg.out_channels, cfg.model_channels))
        W["out.b"] = self._f(sd["out.2.bias"])
        # fuser gates: alpha table [n_st, 2] (attn, dense); gates = scale * tanh(alpha)
        alphas = torch.stack([torch.stack([sd[f"{p}.transformer_blocks.0.fuser.alpha_attn"].reshape(()),
                                           sd[f"{p}.transformer_blocks.0.fuser.alpha_dense"].reshape(())]) for p in self.st_prefixes])
        W["alphas"] = self._f(alphas)
        W["gates"] = torch.zeros_like(W["alphas"])
        self._pack_position_net(sd)
        self.loaded = True
        self.weights_version += 1
        for P in self.plans.values():
            P.static_sig = None
        self.set_scale(self.scale)

    def broadcast_packed(self, src: int = 0) -> int:
        """Frozen weights, once, over NCCL / NVLink (north star; SURVEY 8e): send the PACKED arena of `src` - bf16 GEMM /
        conv operands in their fused layouts (2.14 GB for SD-1.4 + GLIGEN) plus the small fp32 vectors - instead of the
        fp32 masters (4.3 GB).  Every rank must have called load_state_dict (any values) so the slots exist.
        Returns the bytes sent."""
        from .dist import broadcast_tensors
        assert self.loaded, "load_state_dict first (allocates the packed slots)"
        names = sorted(k for k in self.W if k != "gates")
        sent = broadcast_tensors([self.W[k] for k in names], src=src)
        self.weights_version += 1
        self.invalidate_static()
        self.set_scale(self.scales)
        return sent

    def _pack_position_net(self, sd) -> None:
        cfg, W, pn = self.cfg, self.W, "position_net"
        if cfg.spatial:                      # ConvNeXt tokenizer + grounding downsampler (gligen_b200/spatial.py)
            from . import spatial
            spatial.pack(self, sd)
            return

        def mlp(src: str, dst: str):
            w0 = sd[f"{pn}.{src}.0.weight"].float()
            w0p = torch.zeros(w0.shape[0], self.pos_k)
            w0p[:, : w0.shape[1]] = w0
            W[f"{dst}.0.w"], W[f"{dst}.0.b"] = self._a(w0p), self._f(sd[f"{pn}.{src}.0.bias"])
            W[f"{dst}.2.w"], W[f"{dst}.2.b"] = self._a(sd[f"{pn}.{src}.2.weight"]), self._f(sd[f"{pn}.{src}.2.bias"])
            W[f"{dst}.4.w"], W[f"{dst}.4.b"] = self._a(sd[f"{pn}.{src}.4.weight"]), self._f(sd[f"{pn}.{src}.4.bias"])

        if cfg.tokenizer == "text":
            mlp("linears", "pn.s0")
            W["pn.s0.null_feat"] = self._f(sd[f"{pn}.null_positive_feature"])
            W["pn.null_pos"] = self._f(sd[f"{pn}.null_position_feature"])
        elif cfg.tokenizer == "text_image":
            mlp("linears_text", "pn.s0")
            mlp("linears_image", "pn.s1")
            W["pn.s0.null_feat"] = self._f(sd[f"{pn}.null_text_feature"])
            W["pn.s1.null_feat"] = self._f(sd[f"{pn}.null_image_feature"])
            W["pn.null_pos"] = self._f(sd[f"{pn}.null_position_feature"])
        else:  # keypoint: person x keypoint embedding table is input independent (keypoint_grounding_net.py:39-42)
            mlp("linears", "pn.s0")
            P = cfg.max_persons
            pe = sd[f"{pn}.person_embeddings"].float().unsqueeze(1).repeat(1, 17, 1).reshape(P * 17, -1)
            ke = torch.cat([sd[f"{pn}.keypoint_embeddings"].float()] * P, dim=0)
            W["pn.table"] = self._f(pe + ke)
            W["pn.s0.null_feat"] = self._f(sd[f"{pn}.null_person_feature"])
            W["pn.null_pos"] = self._f(sd[f"{pn}.null_xy_feature"])

    def set_first_conv(self, weight: torch.Tensor, bias: torch.Tensor) -> None:
        """openaimodel.py:400-413 swaps input_blocks[0][0]; here: repack into the static weight slot."""
        weight = weight.float()
        cin = self.cfg.first_conv_in
        if weight.shape[1] < cin:
            # the SD first conv (4 input channels) swapped into a model whose GLIGEN first conv also reads the grounding
            # downsampler's planes (openaimodel.py:400-413, 441-443: with first_conv_type == "SD" they are not concatenated):
            # zero weights on those channels state the same thing without changing the plan
            weight = torch.cat([weight, weight.new_zeros(weight.shape[0], cin - weight.shape[1], 3, 3)], dim=1)
        w = self._f(weight.permute(2, 3, 1, 0).reshape(9, weight.shape[1], weight.shape[0]))   # [9][Cin][Cout]
        b = self._f(bias)
        if "conv_in.w" in self.W and self.W["conv_in.w"].shape == w.shape:
            self.W["conv_in.w"].copy_(w)          # in place: captured graphs keep pointing at this storage
            self.W["conv_in.b"].copy_(b)
        else:
            self.W["conv_in.w"], self.W["conv_in.b"] = w, b
            self.plans.clear()

    def set_scale(self, scale) -> None:
        """GatedSelfAttentionDense.scale: one float for every fuser (set_alpha_scale, gligen_inference.py:24-28)
        or one value per SpatialTransformer in execution order."""
        if isinstance(scale, (int, float)):
            scale = [float(scale)] * len(self.st_prefixes)
        scale = [float(s) for s in scale]
        assert len(scale) == len(self.st_prefixes)
        self.scales = scale
        self.scale = max(abs(s) for s in scale) if scale else 0.0     # 0 <=> every fuser is off
        if self.loaded:
            sv = torch.tensor(scale, dtype=torch.float32).view(-1, 1).to(self.dev)
            self.W["gates"].copy_(torch.tanh(self.W["alphas"]) * sv)

    # ------------------------------------------------------------------------------------------
    # plan construction
    # ------------------------------------------------------------------------------------------
    def _buf(self, numel: int, dtype=None) -> torch.Tensor:
        t = torch.empty(max(int(numel), 8), device=self.dev, dtype=dtype or self.adt)
        self._plan_allocs.append(t)          # every buffer a plan touches is known by base address (gligen_b200/export.py)
        return t

    def _zeros(self, *shape, dtype=torch.float32) -> torch.Tensor:
        t = torch.zeros(*shape, device=self.dev, dtype=dtype)
        self._plan_allocs.append(t)
        return t

    def _sizes(self, Bt: int, N: int, nctx: int, Hl: int, Wl: int) -> Dict[str, int]:
        s = dict(t0=0, sb=0, sc=0, sd=0, up=0, col=0, xs=0, qkv=0, ao=0, ffh=0, xstat=0, blk=0)
        for blk in self.blocks:
            hw = (Hl // blk.ds) * (Wl // blk.ds)
            for ly in blk.layers:
                if ly.kind == "res":
                    s["t0"] = max(s["t0"], Bt * hw * ly.cin)
                    for k in ("sb", "sc", "sd", "blk"):
                        s[k] = max(s[k], Bt * hw * ly.cout)
                elif ly.kind == "st":
                    C, T = ly.cin, hw
                    s["t0"] = max(s["t0"], Bt * T * C)
                    s["xs"] = max(s["xs"], Bt * T * C)
                    s["ao"] = max(s["ao"], Bt * T * C)
                    s["qkv"] = max(s["qkv"], Bt * T * 3 * C)
                    s["ffh"] = max(s["ffh"], Bt * T * 4 * C)
                    s["xstat"] = max(s["xstat"], Bt * T * (C // 32) * 2)
                    s["blk"] = max(s["blk"], Bt * T * C)
                elif ly.kind == "down":
                    s["col"] = max(s["col"], Bt * (hw // 4) * 9 * ly.cin)
                elif ly.kind == "up":
                    s["up"] = max(s["up"], Bt * hw * 4 * ly.cin)
        return s

    def _build_plan(self, Bt: int, N: int, nctx: int, Hl: int, Wl: int) -> Plan:
        """Plan for a [Bt, in_channels, Hl, Wl] latent."""
        cfg, ops, W = self.cfg, self.ops, self.W
        S = self.n_streams
        G = N * S
        P = Plan()
        self._plan_allocs = P.buffers = []
        sz = self._sizes(Bt, N, nctx, Hl, Wl)
        B_ = {k: self._buf(v, torch.float32 if k == "xstat" else None) for k, v in sz.items()}
        B_["blk2"] = self._buf(sz["blk"])
        stats = self._zeros(gn_scratch_floats(Bt))   # GLG_GN_SCRATCH_FLOATS, barrier counters zeroed once
        f32 = torch.float32

        def view(name, *shape):
            n = 1
            for d in shape:
                n *= d
            return B_[name][:n].view(*shape)

        # ---- static inputs -------------------------------------------------------------------
        P.inp["x"] = self._zeros(Bt, cfg.in_channels, Hl, Wl)
        if cfg.inpaint_mode:
            P.inp["extra"] = self._zeros(Bt, cfg.in_channels + 1, Hl, Wl)
        P.inp["t"] = self._zeros(Bt, dtype=torch.int64)
        P.inp["context"] = self._zeros(Bt, nctx, cfg.context_dim)
        if cfg.spatial:
            P.inp["map"] = self._zeros(Bt, *self._map_shape)          # the conditioning map (null rows: zeros)
            P.inp["gmask"] = self._zeros(Bt)
            if cfg.ds_out_dim:
                P.inp["extra_map"] = self._zeros(Bt, *self._map_shape)   # grounding_extra_input (shared by cond and uncond rows)
        elif cfg.tokenizer == "keypoint":
            P.inp["coords"] = self._zeros(Bt, N, 2)
            P.inp["masks"] = self._zeros(Bt, N)
        else:
            P.inp["coords"] = self._zeros(Bt, N, 4)
            P.inp["masks"] = self._zeros(Bt, N)
            for si in range(S):
                P.inp[f"feat{si}"] = self._zeros(Bt, N, cfg.tok_in_dim)
                P.inp[f"fmask{si}"] = self._zeros(Bt, N)
        P.out = self._zeros(Bt, cfg.out_channels, Hl, Wl)

        # ---- grounding tokens (PositionNet) -> objs [S, Bt*N, D] -----------------------------
        D = cfg.tok_out_dim
        objs = self._buf(S * Bt * N * D).view(S, Bt * N, D)
        ds_planes = None
        if cfg.spatial:
            from . import spatial
            spatial.emit_tokenizer(self, P, Bt, objs[0])
            if cfg.ds_out_dim:
                ds_planes = spatial.emit_downsampler(self, P, Bt)
        else:
            pos_rows = self._buf(Bt * N * self.pos_k).view(Bt * N, self.pos_k)
            hid1 = self._buf(Bt * N * cfg.tok_hidden).view(Bt * N, cfg.tok_hidden)
            hid2 = self._buf(Bt * N * cfg.tok_hidden).view(Bt * N, cfg.tok_hidden)
        for si in range(0 if cfg.spatial else S):
            if cfg.tokenizer == "keypoint":
                feat, fmask = W["pn.table"], P.inp["masks"]
            else:
                feat, fmask = P.inp[f"feat{si}"], P.inp[f"fmask{si}"]
            nf = W[f"pn.s{si}.null_feat"]
            P.add(f"pn{si}.features", lambda feat=feat, fmask=fmask, nf=nf: ops.position_features(
                feat, fmask, nf, P.inp["coords"], P.inp["masks"], W["pn.null_pos"], pos_rows, cfg.fourier_freqs), static=True)
            k = f"pn.s{si}"
            P.add(f"pn{si}.l0", lambda k=k: ops.gemm(pos_rows, W[f"{k}.0.w"], hid1, bias=W[f"{k}.0.b"], act=ACT_SILU), static=True)
            P.add(f"pn{si}.l2", lambda k=k: ops.gemm(hid1, W[f"{k}.2.w"], hid2, bias=W[f"{k}.2.b"], act=ACT_SILU), static=True)
            P.add(f"pn{si}.l4", lambda k=k, si=si: ops.gemm(hid2, W[f"{k}.4.w"], objs[si], bias=W[f"{k}.4.b"]), static=True)

        # ---- time embedding -------------------------------------------------------------------
        ted = cfg.time_embed_dim
        temb = self._buf(Bt * cfg.model_channels).view(Bt, cfg.model_channels)
        e1 = self._buf(Bt * ted).view(Bt, ted)
        e2 = self._buf(Bt * ted).view(Bt, ted)
        emb_all = self._zeros(Bt, self.emb_total)
        P.add("temb", lambda: ops.timestep_embedding(P.inp["t"], temb))
        P.add("time_embed.0", lambda: ops.gemm(temb, W["time_embed.0.w"], e1, bias=W["time_embed.0.b"], act=ACT_SILU))
        # only SiLU(emb) is ever consumed (openaimodel.py:171-177): fold the SiLU into this epilogue
        P.add("time_embed.2", lambda: ops.gemm(e1, W["time_embed.2.w"], e2, bias=W["time_embed.2.b"], act=ACT_SILU))
        P.add("emb_layers", lambda: ops.gemm(e2, W["emb_all.w"], emb_all, bias=W["emb_all.b"]))

        # ---- context -> bf16 -------------------------------------------------------------------
        ctx_a = self._buf(Bt * nctx * cfg.context_dim).view(Bt * nctx, cfg.context_dim)
        P.add("context.cast", lambda: ops.cast(P.inp["context"], ctx_a), static=True)

        # ---- concat buffers: one per output block; producers write their channel slice --------
        out_blocks = [b for b in self.blocks if b.where == "out"]
        in_blocks = [b for b in self.blocks if b.where == "in"]
        mid = [b for b in self.blocks if b.where == "mid"][0]
        cats = []
        for ob in out_blocks:
            hw = (Hl // ob.ds) * (Wl // ob.ds)
            ctot = ob.layers[0].cin
            cats.append(self._buf(Bt * hw * ctot).view(Bt, hw, ctot))
        dest: Dict[Tuple[str, int], torch.Tensor] = {}
        for j, ib in enumerate(in_blocks):                # skip stack pops in reverse order
            ob_i = len(in_blocks) - 1 - j
            ch_h = out_blocks[ob_i].layers[0].cin - out_blocks[ob_i].skip_ch
            assert out_blocks[ob_i].skip_ch == ib.out_ch
            dest[("in", ib.index)] = cats[ob_i][:, :, ch_h:]
        dest[("mid", 0)] = cats[0][:, :, : mid.out_ch]
        for i, ob in enumerate(out_blocks):
            if i + 1 < len(out_blocks):
                dest[("out", ob.index)] = cats[i + 1][:, :, : ob.out_ch]
            else:
                dest[("out", ob.index)] = self._buf(Bt * Hl * Wl * ob.out_ch).view(Bt, Hl * Wl, ob.out_ch)

        st_index = {p: i for i, p in enumerate(self.st_prefixes)}

        # ---- layer emitters --------------------------------------------------------------------
        def emit_res(ly, x, out, H, Wd):
            p, hw = ly.prefix, H * Wd
            a = view("t0", Bt, hw, ly.cin)
            h1 = view("sb", Bt, hw, ly.cout)
            a2 = view("sc", Bt, hw, ly.cout)
            off = self.emb_off[p]
            rb = emb_all[:, off: off + ly.cout]
            P.add(f"{p}.gn1", lambda: ops.groupnorm(x, a, W[f"{p}.gn1.g"], W[f"{p}.gn1.b"], stats, 32, 1e-5, True))
            P.add(f"{p}.conv1", lambda: ops.gemm(a, W[f"{p}.conv1.w"], h1, bias=W[f"{p}.conv1.b"], rowbias=rb,
                                                 rows_per_batch=hw, conv=(Bt, H, Wd)))
            P.add(f"{p}.gn2", lambda: ops.groupnorm(h1, a2, W[f"{p}.gn2.g"], W[f"{p}.gn2.b"], stats, 32, 1e-5, True))
            if ly.cin != ly.cout:
                sk = view("sd", Bt, hw, ly.cout)
                P.add(f"{p}.skip", lambda: ops.gemm(x, W[f"{p}.skip.w"], sk, bias=W[f"{p}.skip.b"]))
                res = sk
            else:
                res = x
            P.add(f"{p}.conv2", lambda: ops.gemm(a2, W[f"{p}.conv2.w"], out, bias=W[f"{p}.conv2.b"], residual=res, conv=(Bt, H, Wd)))

        def emit_st(ly, x_in, out, H, Wd):
            p, T, C = ly.prefix, H * Wd, ly.cin
            tb = f"{p}.transformer_blocks.0"
            heads, d = ly.heads, ly.d_head
            gi = st_index[p]
            NS = C // 32                                   # capacity of the per-row LayerNorm partial-sum slots
            t0 = view("t0", Bt, T, C)
            xs = view("xs", Bt, T, C)                      # the residual stream of the block (raw, bf16)
            ao = view("ao", Bt, T, C)
            ffh = view("ffh", Bt, T, 4 * C)
            qkv = view("qkv", Bt, T, 3 * C)
            xst = view("xstat", NS, Bt * T, 2)             # slot-major (sum, sumsq) partials of the CURRENT xs rows
            EPS = 1e-5
            P.add(f"{p}.gn", lambda: ops.groupnorm(x_in, t0, W[f"{p}.gn.g"], W[f"{p}.gn.b"], stats, 32, 1e-6, False))
            P.add(f"{p}.proj_in", lambda: ops.gemm(t0, W[f"{p}.proj_in.w"], xs, bias=W[f"{p}.proj_in.b"], stats_out=xst))
            # -- attn1 (attention.py:334); norm1 folded into the QKV GEMM
            P.add(f"{tb}.attn1.qkv", lambda: ops.gemm(xs, W[f"{tb}.attn1.qkv.w"], qkv, bias=W[f"{tb}.attn1.qkv.b"],
                                                      ln=(xst, W[f"{tb}.attn1.qkv.s"], EPS)))
            P.add(f"{tb}.attn1.core", lambda: ops.attention(qkv[:, :, :C], qkv[:, :, C:2 * C], qkv[:, :, 2 * C:], ao, heads, d))
            P.add(f"{tb}.attn1.out", lambda: ops.gemm(ao, W[f"{tb}.attn1.out.w"], xs, bias=W[f"{tb}.attn1.out.b"], residual=xs, stats_out=xst))
            # -- fuser: GatedSelfAttentionDense (attention.py:236-244); skipped when scale == 0.
            #    LN(cat[x, objs']) @ Wqkv is computed as two GEMMs into one per-layer [Bt, T+G, 3C] buffer: the
            #    visual rows every step, the grounding rows (objs' = linear(objs) is timestep-invariant) once.
            fu = f"{tb}.fuser"
            objp = self._buf(S * Bt * N * C).view(S, Bt * N, C)
            ostat = self._buf(S * Bt * N * NS * 2, f32).view(NS, S * Bt * N, 2)     # slot-major over all streams' rows
            qkv2 = self._buf(Bt * (T + G) * 3 * C).view(Bt, T + G, 3 * C)
            P.add(f"{fu}.linear", lambda: ops.gemm(objs.view(S * Bt * N, D), W[f"{fu}.linear.w"], objp.view(S * Bt * N, C),
                                                  bias=W[f"{fu}.linear.b"], stats_out=ostat), fuser=True, static=True)
            for si in range(S):
                P.add(f"{fu}.attn.qkv.objs{si}", lambda si=si: ops.gemm(
                    objp[si], W[f"{fu}.attn.qkv.w"], qkv2[:, T + si * N: T + (si + 1) * N], bias=W[f"{fu}.attn.qkv.b"],
                    ln=(ostat[:, si * Bt * N: (si + 1) * Bt * N], W[f"{fu}.attn.qkv.s"], EPS)), fuser=True, static=True)
            P.add(f"{fu}.attn.qkv", lambda: ops.gemm(xs, W[f"{fu}.attn.qkv.w"], qkv2[:, :T], bias=W[f"{fu}.attn.qkv.b"],
                                                    ln=(xst, W[f"{fu}.attn.qkv.s"], EPS)), fuser=True)
            P.add(f"{fu}.attn.core", lambda: ops.attention(qkv2[:, :T, :C], qkv2[:, :, C:2 * C], qkv2[:, :, 2 * C:], ao, heads, d), fuser=True)
            P.add(f"{fu}.attn.out", lambda: ops.gemm(ao, W[f"{fu}.attn.out.w"], xs, bias=W[f"{fu}.attn.out.b"],
                                                    gate=W["gates"][gi, 0:1], residual=xs, stats_out=xst), fuser=True)
            P.add(f"{fu}.ff.1", lambda: ops.gemm(xs, W[f"{fu}.ff.w1"], ffh, bias=W[f"{fu}.ff.b1"], geglu=True,
                                                ln=(xst, W[f"{fu}.ff.s1"], EPS)), fuser=True)
            P.add(f"{fu}.ff.2", lambda: ops.gemm(ffh, W[f"{fu}.ff.w2"], xs, bias=W[f"{fu}.ff.b2"], gate=W["gates"][gi, 1:2],
                                                residual=xs, stats_out=xst), fuser=True)
            # -- attn2: cross attention to the text context (attention.py:336); K/V of the context are static
            q = view("ao", Bt, T, C)            # ao is free between attention calls: reuse as Q, write O to t0
            kv = self._buf(Bt * nctx * 2 * C).view(Bt, nctx, 2 * C)  # per layer: static across timesteps
            P.add(f"{tb}.attn2.q", lambda: ops.gemm(xs, W[f"{tb}.attn2.q.w"], q, bias=W[f"{tb}.attn2.q.b"], ln=(xst, W[f"{tb}.attn2.q.s"], EPS)))
            P.add(f"{tb}.attn2.kv", lambda: ops.gemm(ctx_a, W[f"{tb}.attn2.kv.w"], kv), static=True)
            P.add(f"{tb}.attn2.core", lambda: ops.attention(q, kv[:, :, :C], kv[:, :, C:], t0, heads, d))
            P.add(f"{tb}.attn2.out", lambda: ops.gemm(t0, W[f"{tb}.attn2.out.w"], xs, bias=W[f"{tb}.attn2.out.b"], residual=xs, stats_out=xst))
            # -- ff (attention.py:337)
            P.add(f"{tb}.ff.1", lambda: ops.gemm(xs, W[f"{tb}.ff.w1"], ffh, bias=W[f"{tb}.ff.b1"], geglu=True, ln=(xst, W[f"{tb}.ff.s1"], EPS)))
            P.add(f"{tb}.ff.2", lambda: ops.gemm(ffh, W[f"{tb}.ff.w2"], xs, bias=W[f"{tb}.ff.b2"], residual=xs))
            P.add(f"{p}.proj_out", lambda: ops.gemm(xs, W[f"{p}.proj_out.w"], out, bias=W[f"{p}.proj_out.b"], residual=x_in))

        def emit_down(ly, x, out, H, Wd):
            p = ly.prefix
            col = view("col", Bt * (H // 2) * (Wd // 2), 9 * ly.cin)
            P.add(f"{p}.im2col", lambda: ops.im2col_s2(x, col, H, Wd))
            P.add(f"{p}.conv", lambda: ops.gemm(col, W[f"{p}.w"], out, bias=W[f"{p}.b"]))

        def emit_up(ly, x, out, H, Wd):
            p = ly.prefix
            up = view("up", Bt, 4 * H * Wd, ly.cin)
            P.add(f"{p}.upsample", lambda: ops.upsample2x(x, up, H, Wd))
            P.add(f"{p}.conv", lambda: ops.gemm(up, W[f"{p}.w"], out, bias=W[f"{p}.b"], conv=(Bt, 2 * H, 2 * Wd)))

        # ---- walk the blocks ---------------------------------------------------------------------
        h = None
        oi = 0
        for blk in self.blocks:
            H, Wd = Hl // blk.ds, Wl // blk.ds
            if blk.where == "out":
                h = cats[oi]
                oi += 1
            final = dest[(blk.where, blk.index)]
            tmp_names = ["blk", "blk2"]
            for li, ly in enumerate(blk.layers):
                last = li == len(blk.layers) - 1
                o = final if last else view(tmp_names[li % 2], Bt, H * Wd, ly.cout)
                if ly.kind == "conv_in":
                    extra = P.inp.get("extra") if ds_planes is None else ds_planes
                    P.add("conv_in", lambda o=o, extra=extra: ops.conv_in(P.inp["x"], extra, W["conv_in.w"], W["conv_in.b"], o))
                elif ly.kind == "res":
                    emit_res(ly, h, o, H, Wd)
                elif ly.kind == "st":
                    emit_st(ly, h, o, H, Wd)
                elif ly.kind == "down":
                    emit_down(ly, h, o, H, Wd)
                elif ly.kind == "up":
                    emit_up(ly, h, o, H, Wd)
                h = o
        # ---- out: GN + SiLU + conv3x3 -> eps (NCHW fp32) ----------------------------------------
        mc = cfg.model_channels
        fin = view("t0", Bt, Hl * Wl, mc)
        hl = h
        P.add("out.gn", lambda: ops.groupnorm(hl, fin, W["out.gn.g"], W["out.gn.b"], stats, 32, 1e-5, True))
        P.add("out.conv", lambda: ops.conv_out(fin, W["out.w"], W["out.b"], P.out, Hl, Wl))
        return P

    # ------------------------------------------------------------------------------------------
    # execution
    # ------------------------------------------------------------------------------------------
    def _plan(self, Bt: int, N: int, nctx: int, slot: int = 0, H: Optional[int] = None, W: Optional[int] = None) -> Plan:
        """Plan for Bt rows of an H x W latent (default: cfg.image_size square)."""
        H = self.cfg.image_size if H is None else H
        W = self.cfg.image_size if W is None else W
        self.check_latent_size(H, W)
        # one plan (and static-part cache) per latent size and batch chunk; the square default size keeps the short key
        size = () if H == W == self.cfg.image_size else (H, W)
        key = (Bt, N, nctx) + size + ((slot,) if slot else ())
        if key not in self.plans:
            self.plans[key] = self._build_plan(Bt, N, nctx, H, W)
        return self.plans[key]

    def check_latent_size(self, H: int, W: int) -> None:
        """Latent sides must survive every stride-2 downsample exactly (the reference fails on other sides at the skip
        concatenation, openaimodel.py:461).  A grounding downsampler writes planes of one fixed size (hed_grounding_downsampler.py:
        interpolate to 64 x 64) that conv_in concatenates, so those models run at their native latent size only - also after
        restore_first_conv_from_SD, where the reference itself would run at other sizes (the plan keeps reading the planes
        through zero weights)."""
        f = max(blk.ds for blk in self.blocks)
        if H <= 0 or W <= 0 or H % f or W % f:
            raise ValueError(f"latent {H}x{W}: both sides must be positive multiples of {f} (one per stride-2 downsample)")
        n = self.cfg.image_size
        if self.cfg.ds_out_dim and (H, W) != (n, n):
            raise ValueError(f"latent {H}x{W}: the grounding downsampler of {self.cfg.tokenizer} models writes {n}x{n} planes that "
                             f"conv_in concatenates with the latent, so this model runs at {n}x{n} only (also with the SD first conv restored)")

    def _n_objs(self, grounding: Dict[str, torch.Tensor]) -> int:
        if self.cfg.spatial:
            from .spec import SPATIAL_MAP_KEY
            shape = tuple(grounding[SPATIAL_MAP_KEY[self.cfg.tokenizer]].shape[1:])
            if shape != self._map_shape:            # static buffers are sized for the map: a new size means new plans
                self._map_shape = shape
                self.plans.clear()
            return self.cfg.spatial_tokens
        return (grounding["points"] if self.cfg.tokenizer == "keypoint" else grounding["boxes"]).shape[1]

    def _stage_grounding(self, P: Plan, grounding: Optional[Dict[str, torch.Tensor]], lo: int, hi: int) -> None:
        """Copy grounding kwargs (GroundingNetInput.prepare output) into rows [lo, hi) of the static inputs;
        None -> the null input (all zeros, grounding_input/*:get_null_input)."""
        cfg = self.cfg
        names = [k for k in P.inp if k in ("coords", "masks", "map", "gmask") or k.startswith(("feat", "fmask"))]
        if grounding is None:
            for k in names:
                P.inp[k][lo:hi].zero_()
            return
        if cfg.spatial:
            from .spec import SPATIAL_MAP_KEY
            P.inp["map"][lo:hi].copy_(grounding[SPATIAL_MAP_KEY[cfg.tokenizer]])
            P.inp["gmask"][lo:hi].copy_(grounding["mask"])
        elif cfg.tokenizer == "keypoint":
            P.inp["coords"][lo:hi].copy_(grounding["points"])
            P.inp["masks"][lo:hi].copy_(grounding["masks"])
        elif cfg.tokenizer == "text":
            P.inp["coords"][lo:hi].copy_(grounding["boxes"])
            P.inp["masks"][lo:hi].copy_(grounding["masks"])
            P.inp["feat0"][lo:hi].copy_(grounding["positive_embeddings"])
            P.inp["fmask0"][lo:hi].copy_(grounding["masks"])
        else:
            P.inp["coords"][lo:hi].copy_(grounding["boxes"])
            P.inp["masks"][lo:hi].copy_(grounding["masks"])
            P.inp["feat0"][lo:hi].copy_(grounding["text_embeddings"])
            P.inp["fmask0"][lo:hi].copy_(grounding["text_masks"])
            P.inp["feat1"][lo:hi].copy_(grounding["image_embeddings"])
            P.inp["fmask1"][lo:hi].copy_(grounding["image_masks"])

    def _run_part(self, P: Plan, fuser_on: bool, static: bool) -> None:
        ops = self.ops
        key = (fuser_on and not static, static)
        if not self.use_graphs or (P.graphs.get(key) is None and P.warm.get(key, 0) < 1):
            # eager pass (also the first call of a shape: creates tensor maps, sets kernel attributes)
            c0 = ops.launch_count()
            P.run(fuser_on, static)
            P.nlaunch[key] = ops.launch_count() - c0
            self.kernel_launches += P.nlaunch[key]
            P.warm[key] = P.warm.get(key, 0) + 1
            return
        g = P.graphs.get(key)
        if g is None:
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g):
                P.run(fuser_on, static)
            P.graphs[key] = g
        g.replay()
        self.kernel_launches += P.nlaunch[key]

    def _execute(self, P: Plan, static_sig, refs=None) -> None:
        fuser_on = self.scale != 0.0
        if static_sig is None or P.static_sig != static_sig:
            self._run_part(P, fuser_on, True)
            P.static_sig = static_sig
            # keep the caller's tensors alive: while we hold them their (data_ptr, _version) cannot be recycled
            # by the allocator for different contents, so an equal signature really means equal contents
            P.static_refs = refs
        self._run_part(P, fuser_on, False)

    def invalidate_static(self) -> None:
        """Forget which inputs the timestep-invariant steps were last run for.  Tensor identity (below) cannot see
        writes that bypass the version counter (`t.data.copy_()`, numpy / DLPack aliases, custom kernels), so callers
        that reuse buffers call this between sampling runs; the samplers of this repo do it at the start of sample()."""
        for P in self.plans.values():
            P.static_sig = None
            P.static_refs = None

    _sig_serial = 0

    @classmethod
    def _sig(cls, *tensors):
        """Identity of caller tensors: same storage, same version counter, same shape -> same contents.  Tensors
        without a version counter (inference-mode tensors) get a fresh serial: never equal, always recomputed."""
        def one(v):
            try:
                ver = v._version
            except RuntimeError:
                cls._sig_serial += 1
                ver = ("unversioned", cls._sig_serial)
            return (v.data_ptr(), ver, tuple(v.shape))
        out = []
        for t in tensors:
            if t is None:
                out.append(None)
            elif isinstance(t, dict):
                out.append(tuple((k,) + one(v) for k, v in sorted(t.items())))
            else:
                out.append(one(t))
        return tuple(out)

    # glg_groupnorm handles at most 64 samples per call (one ticket word each); larger batches - BASELINE's keypoint
    # sweep goes to 64 images = 128 CFG rows - run as chunks, each with its own plan, buffers and static-part cache.
    MAX_ROWS = 64

    @staticmethod
    def _rows(t, lo, hi):
        if t is None:
            return None
        if isinstance(t, dict):
            return {k: v[lo:hi] for k, v in t.items()}
        return t[lo:hi]

    @torch.no_grad()
    def forward(self, x, timesteps, context, grounding, inpainting_extra_input=None, grounding_extra_input=None) -> torch.Tensor:
        """One UNet pass (UNetModel.forward semantics).  grounding=None -> null grounding tokens.
        grounding_extra_input: the map the grounding downsampler reads (spatial modalities; None -> zero planes).
        Returns a NEW fp32 tensor [B, out_channels, H, W]."""
        assert self.loaded, "load_state_dict first"
        B = x.shape[0]
        if B <= self.MAX_ROWS:
            return self._forward_rows(x, timesteps, context, grounding, inpainting_extra_input, 0, grounding_extra_input).clone()
        outs = []
        for slot, lo in enumerate(range(0, B, self.MAX_ROWS)):
            hi = min(B, lo + self.MAX_ROWS)
            outs.append(self._forward_rows(x[lo:hi], timesteps[lo:hi], context[lo:hi], self._rows(grounding, lo, hi),
                                           self._rows(inpainting_extra_input, lo, hi), slot, self._rows(grounding_extra_input, lo, hi)).clone())
        return torch.cat(outs, 0)

    def _stage_extra_map(self, P: Plan, gextra, lo: int, hi: int) -> None:
        if "extra_map" in P.inp:
            if gextra is None:
                P.inp["extra_map"][lo:hi].zero_()
            else:
                P.inp["extra_map"][lo:hi].copy_(gextra)

    def _forward_rows(self, x, timesteps, context, grounding, inpainting_extra_input, slot, grounding_extra_input=None):
        B = x.shape[0]
        if grounding is not None:
            N = self._last_N = self._n_objs(grounding)
        elif self._last_N is None:
            raise RuntimeError("forward(grounding=None) before any grounded call: the null grounding input has the shape "
                               "of the last prepared one (GroundingNetInput.get_null_input asserts the same)")
        else:
            N = self._last_N
        P = self._plan(B, N, context.shape[1], slot, *x.shape[2:])
        P.inp["x"].copy_(x)
        P.inp["t"].copy_(timesteps)
        if self.cfg.inpaint_mode:
            P.inp["extra"].copy_(inpainting_extra_input)
        sig = ("single", self._sig(context, grounding, grounding_extra_input), self.weights_version)
        if P.static_sig != sig:
            P.inp["context"].copy_(context)
            self._stage_grounding(P, grounding, 0, B)
            self._stage_extra_map(P, grounding_extra_input, 0, B)
        self._execute(P, sig, (context, grounding, grounding_extra_input))
        return P.out

    @torch.no_grad()
    def forward_cfg(self, x, timesteps, context, uc, grounding, inpainting_extra_input=None, grounding_extra_input=None):
        """cond + uncond (null grounding, context = uc) as ONE 2B-row pass.  Returns (eps_cond, eps_uncond)
        as views of the static output (valid until the next call); batches above MAX_ROWS / 2 images run in chunks
        and return new tensors."""
        assert self.loaded
        B = x.shape[0]
        per = self.MAX_ROWS // 2
        if B <= per:
            return self._forward_cfg_rows(x, timesteps, context, uc, grounding, inpainting_extra_input, 0, grounding_extra_input)
        conds, unconds = [], []
        for slot, lo in enumerate(range(0, B, per)):
            hi = min(B, lo + per)
            c, u = self._forward_cfg_rows(x[lo:hi], timesteps[lo:hi], context[lo:hi], uc[lo:hi], self._rows(grounding, lo, hi),
                                          self._rows(inpainting_extra_input, lo, hi), slot, self._rows(grounding_extra_input, lo, hi))
            conds.append(c.clone()); unconds.append(u.clone())
        return torch.cat(conds, 0), torch.cat(unconds, 0)

    def _forward_cfg_rows(self, x, timesteps, context, uc, grounding, inpainting_extra_input, slot, grounding_extra_input=None):
        B = x.shape[0]
        N = self._n_objs(grounding)
        self._last_N = N
        P = self._plan(2 * B, N, context.shape[1], slot, *x.shape[2:])
        P.inp["x"][:B].copy_(x); P.inp["x"][B:].copy_(x)
        P.inp["t"][:B].copy_(timesteps); P.inp["t"][B:].copy_(timesteps)
        if self.cfg.inpaint_mode:
            P.inp["extra"][:B].copy_(inpainting_extra_input); P.inp["extra"][B:].copy_(inpainting_extra_input)
        sig = ("cfg", self._sig(context, uc, grounding, grounding_extra_input), self.weights_version)
        if P.static_sig != sig:
            P.inp["context"][:B].copy_(context); P.inp["context"][B:].copy_(uc)
            self._stage_grounding(P, grounding, 0, B)
            self._stage_grounding(P, None, B, 2 * B)
            self._stage_extra_map(P, grounding_extra_input, 0, B)        # plms.py:118: the uncond pass keeps grounding_extra_input
            self._stage_extra_map(P, grounding_extra_input, B, 2 * B)
        self._execute(P, sig, (context, uc, grounding, grounding_extra_input))
        return P.out[:B], P.out[B:]
