"""CPU: the C-ABI library builds for sm_90a, loads, and exports every symbol include/gligen_b200.h declares
(no compute calls - there is no GPU here); the drop-in surface and host logic behave like the reference's."""
import ctypes
import os
import re

import pytest
import torch

from conftest import GOLD, ROOT
from gligen_b200.spec import NAMED_CONFIGS, unet_param_shapes


def test_library_exports_every_declared_symbol():
    from gligen_b200 import build, lib
    path = build.build()
    assert os.path.exists(path)
    header = open(os.path.join(ROOT, "include", "gligen_b200.h")).read()
    declared = set(re.findall(r"\b(glg_[a-z0-9_]+)\s*\(", header))
    assert declared == set(lib.SIGNATURES), declared ^ set(lib.SIGNATURES)
    so = ctypes.CDLL(path)
    for name in declared:
        assert getattr(so, name) is not None
    L = lib.load()
    assert L.glg_abi_version() == 4
    assert L.glg_launch_count() == 0


def test_kernels_are_hopper_native():
    """SASS evidence: wgmma -> HGMMA, TMA loads -> UTMALDG (incl. the multicast of the paired GEMM), mma.sync -> HMMA."""
    import shutil
    import subprocess
    from gligen_b200 import build
    if not shutil.which("cuobjdump"):
        pytest.skip("cuobjdump not available")
    sass = subprocess.run(["cuobjdump", "-sass", build.build()], capture_output=True, text=True).stdout
    for mnemonic in ("HGMMA", "UTMALDG", "UTMALDG.2D.MULTICAST", "HMMA"):
        assert mnemonic in sass, mnemonic


def _tiny_model():
    from ldm.util import instantiate_from_config
    return instantiate_from_config(dict(target="ldm.modules.diffusionmodules.openaimodel.UNetModel", params=dict(
        image_size=16, in_channels=4, out_channels=4, model_channels=64, attention_resolutions=[4, 2, 1], num_res_blocks=2,
        channel_mult=[1, 2, 4, 4], num_heads=8, transformer_depth=1, context_dim=128, fuser_type="gatedSA", use_checkpoint=True,
        grounding_tokenizer=dict(target="ldm.modules.diffusionmodules.text_grounding_net.PositionNet", params=dict(in_dim=128, out_dim=128)))))


def test_dropin_unet_surface():
    from ldm.modules.attention import GatedCrossAttentionDense, GatedSelfAttentionDense
    from gligen_b200.spec import synthetic_state_dict
    m = _tiny_model().eval()
    ref = unet_param_shapes(NAMED_CONFIGS["tiny"])
    sd = m.state_dict()
    assert set(sd) == set(ref) and all(tuple(sd[k].shape) == tuple(ref[k]) for k in ref)
    m.load_state_dict(synthetic_state_dict(NAMED_CONFIGS["tiny"], 0), strict=True)
    fusers = [x for x in m.modules() if type(x) == GatedSelfAttentionDense or type(x) == GatedCrossAttentionDense]
    assert len(fusers) == 16 and all(f.scale == 1 for f in fusers)
    assert m.input_blocks[0][0].weight.shape == (64, 4, 3, 3)
    assert (m.image_size, m.in_channels, m.inpaint_mode, m.first_conv_type, m.grounding_tokenizer_input) == (16, 4, False, "SD", None)
    # fails loudly without a CUDA device: no CPU fallback on the product path
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        m(dict(x=torch.zeros(1, 4, 16, 16), timesteps=torch.zeros(1, dtype=torch.long), context=torch.zeros(1, 77, 128),
               grounding_input=dict(boxes=torch.zeros(1, 2, 4), masks=torch.zeros(1, 2), positive_embeddings=torch.zeros(1, 2, 128))))
    with pytest.raises(NotImplementedError):
        from ldm.modules.diffusionmodules.openaimodel import UNetModel
        UNetModel(16, 4, 64, 4, 2, [1], fuser_type="gatedCA", context_dim=128, grounding_tokenizer=dict(target="x"))


def test_restore_first_conv_reads_cwd_relative_file(tmp_path, monkeypatch):
    from ldm.util import instantiate_from_config
    m = instantiate_from_config(dict(target="ldm.modules.diffusionmodules.openaimodel.UNetModel", params=dict(
        image_size=8, in_channels=4, out_channels=4, model_channels=320, attention_resolutions=[], num_res_blocks=1,
        channel_mult=[1], num_heads=8, context_dim=64, fuser_type="gatedSA",
        grounding_tokenizer=dict(target="ldm.modules.diffusionmodules.text_grounding_net.PositionNet", params=dict(in_dim=64, out_dim=64)))))
    monkeypatch.chdir(GOLD)
    m.restore_first_conv_from_SD()
    w = torch.load(os.path.join(GOLD, "SD_input_conv_weight_bias.pth"))
    assert torch.equal(m.input_blocks[0][0].weight, w["weight"]) and torch.equal(m.input_blocks[0][0].bias, w["bias"])
    assert abs(w["weight"].sum().item() - 1.770429) < 1e-4 and abs(w["bias"].sum().item() - 1.551949) < 1e-4   # SURVEY 8c
    assert "weight" in m.GLIGEN_first_conv_state_dict and m.first_conv_type == "SD"


def test_host_schedule_and_adapters():
    import importlib
    from inpaint_mask_func import draw_masks_from_boxes
    from ldm.models.diffusion.ldm import LatentDiffusion
    from ldm.models.diffusion.plms import PLMSSampler
    from oracle import sampler_oracle as SO
    a = torch.load(os.path.join(GOLD, "scalar_anchors.pt"))
    d = LatentDiffusion(linear_start=0.00085, linear_end=0.012, timesteps=1000)
    assert torch.equal(d.alphas_cumprod, a["alphas_cumprod"]) and d.num_timesteps == 1000
    s = PLMSSampler(d, None)
    s.make_schedule(50)
    assert list(s.ddim_timesteps[:3]) == [1, 21, 41] and s.ddim_timesteps[-1] == 981
    assert torch.allclose(torch.as_tensor(s.ddim_alphas), a["ddim50_alphas"]) and float(s.ddim_sigmas.max()) == 0.0
    torch.manual_seed(0)
    x0, t = torch.randn(2, 4, 8, 8), torch.tensor([981, 1])
    torch.manual_seed(1); q1 = d.q_sample(x0, t)
    torch.manual_seed(1); q2 = SO.q_sample(SO.make_schedule(), x0, t)
    assert torch.equal(q1, q2)
    boxes = torch.tensor([[[0.1, 0.2, 0.5, 0.9], [0.0, 0.0, 0.0, 0.0]], [[0.26, 0.51, 0.99, 1.0], [0.3, 0.3, 0.31, 0.31]]])
    assert torch.equal(draw_masks_from_boxes(boxes, 64), SO.draw_masks_from_boxes(boxes, 64))
    for mod, batch in (("text_grounding_tokinzer_input", dict(boxes=torch.rand(2, 5, 4), masks=torch.ones(2, 5), text_embeddings=torch.randn(2, 5, 8))),
                       ("keypoint_grounding_tokinzer_input", dict(points=torch.rand(2, 34, 2), masks=torch.ones(2, 34)))):
        g = importlib.import_module(f"grounding_input.{mod}").GroundingNetInput()
        with pytest.raises(AssertionError):
            g.get_null_input()
        out = g.prepare(batch)
        null = g.get_null_input()
        assert set(null) == set(out) and all(null[k].shape == out[k].shape and null[k].abs().sum() == 0 for k in out)
        assert g.get_null_input(batch=3)[next(iter(out))].shape[0] == 3


def test_tile_picker_choices_are_valid():
    """Host-side tile picker (csrc/gemm_tc.cu pick_tile) over every GEMM / conv shape of the SD-1.4 forward at 2B = 8
    and at B = 1: the tile width divides N, GEGLU keeps the 256-wide interleaved tile, K is only split when allowed and
    when each split keeps >= 16 K blocks, CTA pairs only for large plain GEMMs with N % 256 == 0 and for 3x3 convolutions
    with M >= 2048."""
    import ctypes as C
    from gligen_b200 import lib as L
    lib = L.load()
    out = (C.c_int32 * 3)()
    ws = 80 << 20

    def pick(M, N, K, geglu=0, conv=0, can_split=1):
        lib.glg_debug_pick_tile(M, N, K, geglu, conv, can_split, ws, out)
        return out[0], out[1], out[2]

    for rows in (8, 1):
        for (T, Cc) in ((4096, 320), (1024, 640), (256, 1280), (64, 1280)):
            M = rows * T
            for (N, K, geglu) in ((3 * Cc, Cc, 0), (Cc, Cc, 0), (Cc, 4 * Cc, 0), (8 * Cc, Cc, 1), (2 * Cc, 768, 0)):
                for can_split in (0, 1):
                    bn, pair, sp = pick(M, N, K, geglu, 0, can_split)
                    assert bn in (64, 128, 160, 256) and N % bn == 0, (M, N, K, bn)
                    assert not geglu or bn == 256
                    assert sp >= 1 and (can_split or sp == 1)
                    assert sp == 1 or (K // 64) // sp >= 16
                    assert not (pair & 1) or (M >= 4096 and N % 256 == 0 and bn == 256 and sp == 1)
                    assert not (pair >> 8), "weights-resident tiles are opt-in (GLG_GEMM_BRES)"
        for (H, Cin, Cout) in ((64, 320, 320), (64, 960, 320), (32, 640, 640), (32, 1920, 640), (16, 1280, 1280), (16, 2560, 1280), (8, 1280, 1280), (8, 2560, 1280)):
            bn, pair, sp = pick(rows * H * H, Cout, Cin, 0, 1, 1)
            assert Cout % bn == 0 and sp >= 1 and (not (pair & 1) or (rows * H * H >= 2048 and sp == 1 and bn >= 128))
            assert sp == 1 or (9 * Cin // 64) // sp >= 16
    # the 8x8 level at 2B = 8 (M = 512) leaves most SMs idle without a K split
    assert pick(512, 1280, 2560, 0, 1, 1)[2] > 1


def test_read_official_ckpt_splits_by_prefix(tmp_path):
    """trainer.read_official_ckpt (reference trainer.py:64-85): the key routing a real SD checkpoint goes through."""
    import trainer
    sd = {"model.diffusion_model.input_blocks.0.0.weight": torch.zeros(1), "cond_stage_model.transformer.x": torch.ones(1),
          "first_stage_model.decoder.conv_in.bias": torch.zeros(2), "model_ema.decay": torch.tensor(0.9999),
          "model_ema.num_updates": torch.tensor(3), "betas": torch.zeros(4), "alphas_cumprod": torch.ones(4)}
    path = tmp_path / "sd.ckpt"
    torch.save({"state_dict": sd}, path)
    out = trainer.read_official_ckpt(str(path))
    assert set(out) == {"model", "text_encoder", "autoencoder", "unexpected", "diffusion"}
    assert list(out["model"]) == ["input_blocks.0.0.weight"]
    assert list(out["text_encoder"]) == ["transformer.x"]
    assert list(out["autoencoder"]) == ["decoder.conv_in.bias"]
    assert sorted(out["unexpected"]) == ["model_ema.decay", "model_ema.num_updates"]
    assert sorted(out["diffusion"]) == ["alphas_cumprod", "betas"]


def test_c_host_example_builds(tmp_path):
    """examples/host_c/unet_host.c (a host without Python over the engine-level C ABI) compiles against include/gligen_b200.h and
    links against the library with plain gcc - no CUDA headers, no torch."""
    import shutil
    import subprocess
    if shutil.which("gcc") is None:
        pytest.skip("no gcc")
    from gligen_b200 import lib as L
    L.load()
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    exe = os.path.join(str(tmp_path), "unet_host")
    r = subprocess.run(["gcc", "-O2", "-Wall", "-Werror", "-I", os.path.join(root, "include"), os.path.join(root, "examples", "host_c", "unet_host.c"),
                        "-L", os.path.join(root, "gligen_b200"), "-lgligen_b200", f"-Wl,-rpath,{os.path.join(root, 'gligen_b200')}", "-o", exe],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    r = subprocess.run([exe], capture_output=True, text=True)
    assert r.returncode == 2 and "usage" in r.stderr
