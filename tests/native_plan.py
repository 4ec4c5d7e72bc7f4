"""A model, its seeded inputs and its exported plan loaded through the engine-level C ABI (include/gligen_b200.h: glg_engine_*),
with the inputs written the way Engine._forward_cfg_rows stages them, so that the replay and model.forward_cfg can be compared
bit for bit.  Used by the native-engine GPU tests."""
import os

import torch

from gligen_b200 import synth
from gligen_b200.export import NativePlan, export_plan
from gligen_b200.pipeline import build_model, to_device

DEV = "cuda:0"


class PlanCase:
    """`name`: a NAMED_CONFIGS key or a UNetConfig.  H, W: a latent size other than the config's square one.  map_size: the
    spatial models' conditioning map size."""

    def __init__(self, name, B, max_objs, tmp_path, map_size=None, H=None, W=None):
        cfg, model = build_model(name, DEV)
        self.cfg, self.model, self.B, self.scale = cfg, model, B, 1.0
        inp = synth.make_inputs(cfg, B, max_objs, seed=4, map_size=map_size)
        self.ts = torch.tensor([981, 401, 21, 1][:B], dtype=torch.long, device=DEV)
        x, z0 = inp["x"], inp.get("z0")
        if H is not None:
            g = torch.Generator().manual_seed(H * 1000 + W)
            x, z0 = torch.randn(B, cfg.in_channels, H, W, generator=g), torch.randn(B, cfg.in_channels, H, W, generator=g) * 0.9
        self.x, self.ctx, self.uc = x.to(DEV), inp["context"].to(DEV), inp["uc"].to(DEV)
        batch = to_device(inp["batch"], DEV)
        self.grounding = model.grounding_tokenizer_input.prepare(batch)
        self.extra = None
        if cfg.inpaint_mode:
            from inpaint_mask_func import draw_masks_from_boxes
            h, w = x.shape[2:]
            mask = draw_masks_from_boxes(batch["boxes"], max(h, w))[:, :, :h, :w].to(DEV)
            self.extra = torch.cat([z0.to(DEV) * mask, mask], dim=1)
        self.eng = model.engine()
        self.gextra = None
        if cfg.spatial:
            from gligen_b200.spec import SPATIAL_MAP_KEY
            self.gextra = batch[SPATIAL_MAP_KEY[cfg.tokenizer]]
            self.eng._n_objs(self.grounding)       # tells the engine the map size the static buffers are planned for
            N = cfg.spatial_tokens
        else:
            N = (batch["points"] if cfg.tokenizer == "keypoint" else batch["boxes"]).shape[1]
        tag = name if isinstance(name, str) else "cfg"
        self.path = os.path.join(str(tmp_path), f"{tag}.glgplan")
        self.info = export_plan(self.eng, 2 * B, N, self.ctx.shape[1], self.path, H=H, W=W)
        self.batch = batch
        self.load()

    def load(self):
        """Loads the exported plan (self.plan) and writes every input but the fuser gates."""
        cfg, batch, gmap = self.cfg, self.batch, self.gextra
        self.plan = plan = NativePlan(self.path)
        # rows [0, B) cond, rows [B, 2B) uncond / null grounding
        self.write_step(self.x, self.ts)
        plan.write("in:context", torch.cat([self.ctx, self.uc]))
        if cfg.inpaint_mode:
            plan.write("in:extra", torch.cat([self.extra, self.extra]))
        z = lambda t: torch.cat([t, torch.zeros_like(t)])
        if cfg.spatial:
            plan.write("in:map", z(gmap)); plan.write("in:gmask", z(batch["mask"]))
            plan.write("in:extra_map", torch.cat([gmap, gmap]))              # the uncond rows keep grounding_extra_input (plms.py:118)
        elif cfg.tokenizer == "keypoint":
            plan.write("in:coords", z(batch["points"])); plan.write("in:masks", z(batch["masks"]))
        else:
            plan.write("in:coords", z(batch["boxes"])); plan.write("in:masks", z(batch["masks"]))
            if cfg.tokenizer == "text":
                plan.write("in:feat0", z(batch["text_embeddings"])); plan.write("in:fmask0", z(batch["masks"]))
            else:
                plan.write("in:feat0", z(batch["text_embeddings"])); plan.write("in:fmask0", z(batch["text_masks"]))
                plan.write("in:feat1", z(batch["image_embeddings"])); plan.write("in:fmask1", z(batch["image_masks"]))

    def input(self, x, ts):
        """The UNet input dict of model.forward_cfg / the samplers."""
        return dict(x=x, timesteps=ts, context=self.ctx, grounding_input=self.grounding, inpainting_extra_input=self.extra,
                    grounding_extra_input=self.gextra)

    def set_scale(self, scale):
        """Every fuser's scale, gatedSA2 included (set_alpha_scale leaves those at 1, like the reference's)."""
        for fu in self.model._fusers:
            fu.scale = scale
        self.scale = scale

    def python(self, x, ts):
        """[eps_cond; eps_uncond] of the Python-driven engine, and the plan's "W:gates" set to the scale it ran at."""
        e_c, e_u = self.model.forward_cfg(self.input(x, ts), self.uc)
        self.plan.write("W:gates", self.eng.W["gates"])          # scale * tanh(alpha): the host owns the scheduled-sampling scale
        return torch.cat([e_c, e_u]).clone()

    def write_step(self, x, ts):
        self.plan.write("in:x", torch.cat([x, x]))
        self.plan.write("in:t", torch.cat([ts, ts]))

    def run(self, static_part):
        self.plan.run(static_part=static_part, fuser_on=self.scale != 0.0)

    def out(self):
        return self.plan.read("out", (2 * self.B,) + tuple(self.x.shape[1:]))


def _case(name, B, max_objs, tmp_path, scales=(1.0, 0.0), map_size=None, H=None, W=None):
    """At each fuser scale: the plan's static and per-step parts replayed natively give model.forward_cfg's eps bit for bit."""
    c = PlanCase(name, B, max_objs, tmp_path, map_size=map_size, H=H, W=W)
    for scale in scales:
        c.set_scale(scale)
        want = c.python(c.x, c.ts)
        c.run(static_part=True)
        c.run(static_part=False)
        got = c.out()
        torch.cuda.synchronize()
        assert torch.equal(got, want), f"{name} scale={scale}: max diff {(got - want).abs().max().item():.3e}"
    c.plan.close()
    return c.info
