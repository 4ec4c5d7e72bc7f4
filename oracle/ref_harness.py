"""Drive the UNMODIFIED reference (gligen/GLIGEN) on the hot path.  TEST / BASELINE INFRASTRUCTURE ONLY.

The reference modules come either from /root/reference (authoring container) or from the archive that
oracle/build_ref.py writes (oracle/_ref/gligen_reference.zip, copied with the working tree to a GPU machine).  Nothing here is imported by the
product package; users are oracle/gen_golden.py, oracle/ref_run.py (CLI used by the GPU parity tests through a
subprocess) and bench.py's `--impl reference` / `cpu_baseline` legs.

What is restated here from gligen_inference.py (it cannot be imported: needs `clip` / `omegaconf`, absent and no
network): `set_alpha_scale` (:24-28) and `alpha_generator` (:31-66, via oracle.sampler_oracle) and the construction of
`input` exactly as `run()` does (:411-430) with synthetic embeddings in place of CLIP / VAE outputs.
"""
from __future__ import annotations

import os
import sys
import time
from functools import partial
from typing import Dict, Optional

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
REPO = os.path.dirname(HERE)
REF_DIR = "/root/reference"

_mounted: Optional[str] = None


def _pin_namespace(name: str, path: str) -> None:
    import importlib.machinery
    import types
    spec = importlib.machinery.ModuleSpec(name, None, is_package=True)
    spec.submodule_search_locations = [path]
    mod = types.ModuleType(name)
    mod.__path__ = [path]
    mod.__spec__ = spec
    sys.modules[name] = mod
    if "." in name:
        setattr(sys.modules[name.rsplit(".", 1)[0]], name.rsplit(".", 1)[1], mod)


def mount(prefer: str = "auto") -> str:
    """Make `ldm.*`, `grounding_input.*`, `inpaint_mask_func` resolve to REFERENCE code in this process.
    prefer: "dir" (/root/reference), "zip" (oracle/_ref archive) or "auto" (the archive when present, else the dir).
    Returns the directory that holds SD_input_conv_weight_bias.pth (the reference reads it CWD-relative)."""
    global _mounted
    if _mounted:
        return _mounted
    if REPO not in sys.path:
        sys.path.insert(0, REPO)
    from oracle import build_ref
    use_dir = os.path.isdir(REF_DIR) and (prefer == "dir" or (prefer == "auto" and not build_ref.available()))
    if not use_dir and not build_ref.available():
        raise RuntimeError("reference unavailable: neither /root/reference nor oracle/_ref/gligen_reference.zip exists")
    for name in ("ldm", "grounding_input", "inpaint_mask_func"):
        if name in sys.modules:
            raise RuntimeError(f"`{name}` already imported in this process (the repo's drop-in?): mount the reference first / in a fresh process")
    if use_dir:
        sys.path.insert(0, REF_DIR)
        for sub in ("ldm", "ldm.models", "ldm.modules"):
            _pin_namespace(sub, os.path.join(REF_DIR, *sub.split(".")))
        _mounted = REF_DIR
    else:
        _mounted = build_ref.mount()
    return _mounted


def shim_timm() -> None:
    """The reference's convnext.py imports `timm` (absent here, no network) for three names that never run on this path:
    `trunc_normal_` (init only, commented out), `DropPath` (drop_path = 0 -> nn.Identity is used) and `register_model` (a
    registry decorator).  Stand-ins for exactly those names let the UNMODIFIED reference module import.  `convnext_tiny(
    pretrained=True)` (hed_grounding_net.py:20) downloads ImageNet weights: torch.hub.load_state_dict_from_url is pointed at
    an empty state dict (strict=False load); the parity runs then load the seeded synthetic weights over every tensor."""
    import types
    if "timm" not in sys.modules:
        timm = types.ModuleType("timm"); models = types.ModuleType("timm.models")
        layers = types.ModuleType("timm.models.layers"); registry = types.ModuleType("timm.models.registry")
        layers.trunc_normal_ = lambda t, std=0.02: torch.nn.init.trunc_normal_(t, std=std)
        layers.DropPath = torch.nn.Identity
        registry.register_model = lambda fn: fn
        timm.models, models.layers, models.registry = models, layers, registry
        sys.modules.update({"timm": timm, "timm.models": models, "timm.models.layers": layers, "timm.models.registry": registry})
    torch.hub.load_state_dict_from_url = lambda *a, **k: {"model": {}}


def spatial_configs(cfg):
    """(grounding_tokenizer, grounding_downsampler) config dicts of a spatial modality, as configs/cc3m_hed.yaml etc. give them."""
    t = cfg.tokenizer
    tok = dict(resize_input=cfg.tok_resize, out_dim=cfg.tok_out_dim)
    ds = dict(out_dim=cfg.ds_out_dim)
    if t != "hed":
        ds["resize_input"] = cfg.ds_resize
    if t == "sem":
        tok["in_dim"] = ds["in_dim"] = cfg.sem_in_dim
    return (dict(target=f"ldm.modules.diffusionmodules.{t}_grounding_net.PositionNet", params=tok),
            dict(target=f"ldm.modules.diffusionmodules.{t}_grounding_downsampler.GroundingDownsampler", params=ds))


def is_reference_module(mod) -> bool:
    f = getattr(sys.modules[mod.__module__], "__file__", "") or ""
    return f.startswith(REF_DIR) or "gligen_reference.zip" in f


# ---- model / adapters ---------------------------------------------------------------------------------------
def ref_model(cfg, device="cpu"):
    """The reference UNetModel for a gligen_b200.spec.UNetConfig (yaml params as a plain dict, configs/*.yaml)."""
    mount()
    from ldm.modules.diffusionmodules.openaimodel import UNetModel
    assert is_reference_module(UNetModel)
    if cfg.spatial:
        shim_timm()
        tokc, dsc = spatial_configs(cfg)
        m = UNetModel(image_size=cfg.image_size, in_channels=cfg.in_channels, out_channels=cfg.out_channels,
                      model_channels=cfg.model_channels, attention_resolutions=list(cfg.attention_resolutions),
                      num_res_blocks=cfg.num_res_blocks, channel_mult=list(cfg.channel_mult), num_heads=cfg.num_heads,
                      transformer_depth=1, context_dim=cfg.context_dim, fuser_type="gatedSA", use_checkpoint=True,
                      inpaint_mode=cfg.inpaint_mode, grounding_tokenizer=tokc, grounding_downsampler=dsc)
        return m.to(device).eval()
    tok = {
        "text": ("ldm.modules.diffusionmodules.text_grounding_net.PositionNet", dict(in_dim=cfg.tok_in_dim, out_dim=cfg.tok_out_dim)),
        "text_image": ("ldm.modules.diffusionmodules.text_image_grounding_net.PositionNet", dict(in_dim=cfg.tok_in_dim, out_dim=cfg.tok_out_dim)),
        "keypoint": ("ldm.modules.diffusionmodules.keypoint_grounding_net.PositionNet", dict(max_persons_per_image=cfg.max_persons, out_dim=cfg.tok_out_dim)),
    }[cfg.tokenizer]
    m = UNetModel(image_size=cfg.image_size, in_channels=cfg.in_channels, out_channels=cfg.out_channels,
                  model_channels=cfg.model_channels, attention_resolutions=list(cfg.attention_resolutions),
                  num_res_blocks=cfg.num_res_blocks, channel_mult=list(cfg.channel_mult), num_heads=cfg.num_heads,
                  transformer_depth=1, context_dim=cfg.context_dim, fuser_type="gatedSA", use_checkpoint=True,
                  inpaint_mode=cfg.inpaint_mode, grounding_tokenizer=dict(target=tok[0], params=tok[1]))
    return m.to(device).eval()


def ref_grounding_input(cfg):
    mount()
    import importlib
    if cfg.spatial:
        return importlib.import_module(f"grounding_input.{cfg.tokenizer}_grounding_tokinzer_input").GroundingNetInput()
    name = {"text": "text_grounding_tokinzer_input", "text_image": "text_image_grounding_tokinzer_input",
            "keypoint": "keypoint_grounding_tokinzer_input"}[cfg.tokenizer]
    return importlib.import_module(f"grounding_input.{name}").GroundingNetInput()


def set_alpha_scale(model, alpha_scale):
    """gligen_inference.py:24-28."""
    from ldm.modules.attention import GatedCrossAttentionDense, GatedSelfAttentionDense
    for module in model.modules():
        if type(module) == GatedCrossAttentionDense or type(module) == GatedSelfAttentionDense:
            module.scale = alpha_scale


def ref_diffusion(device="cpu"):
    mount()
    from ldm.models.diffusion.ldm import LatentDiffusion
    return LatentDiffusion(linear_start=0.00085, linear_end=0.012, timesteps=1000).to(device)


def _to(d, device):
    if d is None:
        return None
    if isinstance(d, dict):
        return {k: _to(v, device) for k, v in d.items()}
    return d.to(device)


class cpu_rng_noise:
    """Draw randn_like noise from the CPU generator whatever the device, so CPU and GPU runs of the reference consume
    identical noise (only the inpainting q_sample noise enters the result; sigma_t == 0 elsewhere)."""

    def __enter__(self):
        self.orig = torch.randn_like
        torch.randn_like = lambda x, **kw: torch.randn(x.shape, dtype=x.dtype).to(x.device)
        return self

    def __exit__(self, *a):
        torch.randn_like = self.orig


@torch.no_grad()
def run_reference_sampler(cfg, sd: Dict[str, torch.Tensor], inp: Dict[str, object], kind: str, S: int, alpha_type,
                          guidance: float = 7.5, device="cpu", autocast: Optional[torch.dtype] = None, model=None,
                          verbose: bool = True):
    """reference PLMSSampler / DDIMSampler (.sample) around the reference UNetModel, the way gligen_inference.run()
    drives them (:384-430).  `inp` = gligen_b200.synth.make_inputs(...).  Returns (latent on the CPU, seconds)."""
    mount()
    from oracle import sampler_oracle as SO
    from ldm.models.diffusion.ddim import DDIMSampler
    from ldm.models.diffusion.plms import PLMSSampler
    if str(device).startswith("cuda"):
        torch.backends.cuda.matmul.allow_tf32 = False         # the fp32 reference must be fp32
        torch.backends.cudnn.allow_tf32 = False
    gin = ref_grounding_input(cfg)
    if model is None:
        model = ref_model(cfg, device)                        # fresh: restore_first_conv_from_SD mutates the model
        model.load_state_dict(sd, strict=True)
    model.grounding_tokenizer_input = gin
    grounding = gin.prepare(_to(inp["batch"], device))
    mask = z0 = extra = None
    if cfg.inpaint_mode:
        from inpaint_mask_func import draw_masks_from_boxes
        mask = draw_masks_from_boxes(inp["batch"]["boxes"], cfg.image_size).to(device)
        z0 = inp["z0"].to(device)
        extra = torch.cat([z0 * mask, mask], dim=1)            # gligen_inference.py:400-407
    diffusion = ref_diffusion(device)
    cls = PLMSSampler if kind == "plms" else DDIMSampler
    sampler = cls(diffusion, model, alpha_generator_func=partial(SO.alpha_generator, type=alpha_type), set_alpha_scale=set_alpha_scale)
    B = inp["x"].shape[0]
    input = dict(x=inp["x"].clone().to(device), timesteps=None, context=inp["context"].to(device), grounding_input=grounding,
                 inpainting_extra_input=extra, grounding_extra_input=_to(inp.get("grounding_extra_input"), device))
    shape = (B, cfg.in_channels, cfg.image_size, cfg.image_size)
    cwd = os.getcwd()
    os.chdir(_mounted)                                         # SD_input_conv_weight_bias.pth is read CWD-relative
    try:
        torch.manual_seed(1234)
        t0 = time.time()
        ctx = torch.autocast(device_type=str(device).split(":")[0], dtype=autocast) if autocast is not None else _null()
        with cpu_rng_noise(), ctx:
            lat = sampler.sample(S=S, shape=shape, input=input, uc=inp["uc"].to(device), guidance_scale=guidance, mask=mask, x0=z0)
        if str(device).startswith("cuda"):
            torch.cuda.synchronize()
        dt = time.time() - t0
    finally:
        os.chdir(cwd)
    if verbose:
        print(f"   reference {kind} S={S} alpha={alpha_type} device={device} autocast={autocast}: {dt:.1f}s  latent std {lat.float().std():.3f}", flush=True)
    return lat.float().cpu(), dt


class _null:
    def __enter__(self):
        return self

    def __exit__(self, *a):
        return False


@torch.no_grad()
def run_reference_forward(cfg, model, inp, timesteps, scale: float, cond: bool, device="cpu", autocast: Optional[torch.dtype] = None):
    """One reference UNetModel.forward(input) (openaimodel.py:420-464): cond (grounded) or the null / uncond pass."""
    gin = ref_grounding_input(cfg)
    model.grounding_tokenizer_input = gin
    set_alpha_scale(model, scale)
    extra = None
    if cfg.inpaint_mode:
        from inpaint_mask_func import draw_masks_from_boxes
        mask = draw_masks_from_boxes(inp["batch"]["boxes"], cfg.image_size).to(device)
        extra = torch.cat([inp["z0"].to(device) * mask, mask], dim=1)
    d = dict(x=inp["x"].to(device), timesteps=timesteps.to(device), context=(inp["context"] if cond else inp["uc"]).to(device),
             inpainting_extra_input=extra, grounding_extra_input=None)
    if cond:
        d["grounding_input"] = gin.prepare(_to(inp["batch"], device))
    ctx = torch.autocast(device_type=str(device).split(":")[0], dtype=autocast) if autocast is not None else _null()
    with ctx:
        return model(d).float().cpu()
