"""CPU tests of the drop-in boundary: the C-ABI library exports every symbol its headers declare, the Python shells
expose the reference's state_dict keys / attributes, host-side glue (scheduler, windows) matches the oracle."""
import ctypes
import os
import re

import pytest
import torch

from oracle import hv_oracle as O

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def header_symbols():
    names = []
    for h in ("hv_b200.h", "hv_b200_ops.h"):
        src = open(os.path.join(ROOT, "include", h)).read()
        src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
        names += re.findall(r"\b(hv_[a-z0-9_]+)\s*\(", src)
    return sorted(set(names))


def test_library_exports_every_declared_symbol():
    from humanvid_b200 import _native

    lib = ctypes.CDLL(_native.LIB_PATH)
    syms = header_symbols()
    assert len(syms) >= 31 and "hv_unet2d_reference_forward" in syms
    missing = [s for s in syms if not hasattr(lib, s)]
    assert not missing, missing


def test_unet_shell_has_reference_state_dict_keys():
    from humanvid_b200 import UNet3DConditionModel

    kw = dict(block_out_channels=(32, 64, 128, 128), cross_attention_dim=64, use_motion_module=True, use_inflated_groupnorm=True,
              motion_module_resolutions=(1, 2, 4, 8), motion_module_mid_block=True, motion_module_type="Vanilla",
              motion_module_kwargs=dict(num_attention_heads=8, num_transformer_block=1, attention_block_types=["Temporal_Self", "Temporal_Self"],
                                        temporal_position_encoding=True, temporal_position_encoding_max_len=32, temporal_attention_dim_div=1),
              unet_use_cross_frame_attention=False, unet_use_temporal_attention=False)
    m = UNet3DConditionModel(**kw)
    o = O.UNet3DConditionModel(block_out_channels=(32, 64, 128, 128), cross_attention_dim=64)
    sm, so = m.state_dict(), o.state_dict()
    assert set(sm) == set(so)
    assert all(sm[k].shape == so[k].shape for k in so)
    assert m.in_channels == 4 and m.config.block_out_channels == (32, 64, 128, 128)
    # reader order == reference order (pin_report.json)
    names = {id(b): n for n, b in m.named_modules()}
    order = [names[id(b)] for b in m.reader_blocks()]
    import json

    rep = json.load(open(os.path.join(ROOT, "tests", "golden", "pin_report.json")))
    assert order == rep["bank_order"]
    # image variant (config 1): no motion modules
    m1 = UNet3DConditionModel(block_out_channels=(32, 64, 128, 128), cross_attention_dim=64, unet_use_cross_frame_attention=False, unet_use_temporal_attention=False)
    o1 = O.UNet3DConditionModel(block_out_channels=(32, 64, 128, 128), cross_attention_dim=64, use_motion_module=False, use_inflated_groupnorm=False)
    assert set(m1.state_dict()) == set(o1.state_dict())


def test_reference_unet2d_shell_keys_and_writer_order():
    from humanvid_b200 import ReferenceAttentionControl, UNet2DConditionModel, UNet3DConditionModel

    m = UNet2DConditionModel(block_out_channels=(32, 64, 128, 128), cross_attention_dim=64)
    o = O.UNet2DConditionModel(block_out_channels=(32, 64, 128, 128), cross_attention_dim=64)
    sm, so = m.state_dict(), o.state_dict()
    assert set(sm) == set(so) and all(sm[k].shape == so[k].shape for k in so)
    names = {id(b): n for n, b in m.named_modules()}
    import json

    rep = json.load(open(os.path.join(ROOT, "tests", "golden", "pin_report.json")))
    assert [names[id(b)] for b, _ in m.writer_blocks()] == rep["bank_order"]   # same sorted order on writer and reader side
    assert [lvl for _, lvl in m.writer_blocks()] == [2] * 5 + [3] + [1] * 5 + [0] * 5
    w = ReferenceAttentionControl(m, do_classifier_free_guidance=True, mode="write", fusion_blocks="full")
    assert m._ref_write and all(b.bank == [] for b, _ in m.writer_blocks())
    with pytest.raises(TypeError):
        ReferenceAttentionControl(m, mode="read", fusion_blocks="full")
    with pytest.raises(NotImplementedError):
        UNet2DConditionModel(use_linear_projection=True)
    # update(): writer banks land on the reader's blocks in the same order
    r3 = UNet3DConditionModel(block_out_channels=(32, 64, 128, 128), cross_attention_dim=64, unet_use_cross_frame_attention=False, unet_use_temporal_attention=False)
    rd = ReferenceAttentionControl(r3, do_classifier_free_guidance=True, mode="read", fusion_blocks="full")
    for i, (b, _) in enumerate(m.writer_blocks()):
        b.bank.append(torch.full((2, 4, b.norm1.normalized_shape[0]), float(i)))
    rd.update(w, dtype=torch.float32)
    assert [float(b.bank[0][0, 0, 0]) for b in r3.reader_blocks()] == [float(i) for i in range(16)]
    rd.clear(); w.clear()
    assert all(len(b.bank) == 0 for b in r3.reader_blocks()) and all(len(b.bank) == 0 for b, _ in m.writer_blocks())


def test_pose_guider_and_camera_shells():
    from humanvid_b200 import CameraPoseEncoder, PoseGuider

    pg = PoseGuider(320, block_out_channels=(16, 32, 96, 256))
    assert set(pg.state_dict()) == set(O.PoseGuider().state_dict())
    assert float(pg.conv_out.weight.abs().sum()) == 0.0  # zero_module like the reference
    cam = CameraPoseEncoder(downscale_factor=8, channels=[320], nums_rb=2, cin=384, ksize=1, sk=True, use_conv=False, compression_factor=1,
                            temporal_attention_nhead=8, attention_block_types=["Temporal_Self"], temporal_position_encoding=True,
                            temporal_position_encoding_max_len=24)
    so = O.CameraPoseEncoder().state_dict()
    assert set(cam.state_dict()) == set(so)
    assert all(cam.state_dict()[k].shape == so[k].shape for k in so)


def test_forward_fails_loudly_without_cuda():
    from humanvid_b200 import PoseGuider

    pg = PoseGuider(320, block_out_channels=(16, 32, 96, 256))
    with pytest.raises(RuntimeError, match="CUDA"):
        pg(torch.zeros(1, 3, 1, 16, 16))


def test_unsupported_configs_are_rejected():
    from humanvid_b200 import UNet3DConditionModel

    with pytest.raises(NotImplementedError):
        UNet3DConditionModel(use_linear_projection=True)
    with pytest.raises(NotImplementedError):
        UNet3DConditionModel(layers_per_block=3)


def test_scheduler_matches_oracle_ddim():
    from humanvid_b200.scheduler import DDIMScheduler

    s = DDIMScheduler(beta_start=0.00085, beta_end=0.012, beta_schedule="linear", clip_sample=False, steps_offset=1, prediction_type="v_prediction",
                      rescale_betas_zero_snr=True, timestep_spacing="trailing")
    s.set_timesteps(25)
    o = O.DDIM()
    ot = o.set_timesteps(25)
    assert s.timesteps.tolist() == ot.tolist()
    g = torch.Generator().manual_seed(0)
    x, v = torch.randn(1, 4, 2, 8, 8, generator=g), torch.randn(1, 4, 2, 8, 8, generator=g)
    for t in (999, 519, 39):
        assert torch.allclose(s.step(v, t, x).prev_sample, o.step(v, t, x), atol=1e-6)


def test_pipeline_windows_match_oracle():
    from humanvid_b200.pipeline import uniform

    for nf in (24, 48, 87):
        assert [list(w) for w in uniform(0, 25, nf, 24, 1, 4)] == O.uniform_windows(0, nf, 24, 1, 4)


def test_from_pretrained_2d_loading_flow(tmp_path):
    """unet_3d.py:579-670: config.json -> model, 2-D weights (.safetensors preferred, else .bin), motion-module file merged on top (every key,
    `proj_out` keys dropped under mm_zero_proj_out), strict=False; same exceptions for a missing config / weights file / unknown suffix."""
    import json

    from safetensors.torch import save_file

    from humanvid_b200 import UNet3DConditionModel

    mmk = dict(num_attention_heads=8, num_transformer_block=1, attention_block_types=["Temporal_Self", "Temporal_Self"],
               temporal_position_encoding=True, temporal_position_encoding_max_len=32, temporal_attention_dim_div=1)
    extra = dict(use_motion_module=True, use_inflated_groupnorm=True, motion_module_resolutions=(1, 2, 4, 8), motion_module_mid_block=True,
                 motion_module_type="Vanilla", motion_module_kwargs=mmk, unet_use_cross_frame_attention=False, unet_use_temporal_attention=False)
    src = O.synthetic_init(O.UNet3DConditionModel(block_out_channels=(32, 64, 128, 128), cross_attention_dim=64), seed=3)
    full = {k: v.clone() for k, v in src.state_dict().items()}
    sd2d = {k: v.contiguous() for k, v in full.items() if "motion_modules" not in k}
    mm = {k: v.contiguous() for k, v in full.items() if "motion_modules" in k}
    root = tmp_path / "sd15"
    (root / "unet").mkdir(parents=True)
    cfg = {"_class_name": "UNet2DConditionModel", "_diffusers_version": "0.6.0", "in_channels": 4, "out_channels": 4, "block_out_channels": [32, 64, 128, 128],
           "cross_attention_dim": 64, "attention_head_dim": 8, "layers_per_block": 2, "norm_num_groups": 32, "act_fn": "silu",
           "down_block_types": ["CrossAttnDownBlock2D"] * 3 + ["DownBlock2D"], "up_block_types": ["UpBlock2D"] + ["CrossAttnUpBlock2D"] * 3,
           "sample_size": 64, "some_future_key": 1}
    json.dump(cfg, open(root / "unet" / "config.json", "w"))
    mm_file = tmp_path / "mm.ckpt"
    torch.save(mm, mm_file)

    with pytest.raises(FileNotFoundError):
        UNet3DConditionModel.from_pretrained_2d(root, mm_file, subfolder="unet", unet_additional_kwargs=extra)
    torch.save(sd2d, root / "unet" / "diffusion_pytorch_model.bin")
    m = UNet3DConditionModel.from_pretrained_2d(root, mm_file, subfolder="unet", unet_additional_kwargs=extra)
    got = m.state_dict()
    assert set(got) == set(full) and all(torch.equal(got[k], full[k]) for k in full)
    assert m.config.sample_size == 64 and m.config.block_out_channels == [32, 64, 128, 128]

    # .safetensors wins over .bin when both exist
    marked = {k: (v + 1.0 if k == "conv_in.bias" else v) for k, v in sd2d.items()}
    save_file(marked, str(root / "unet" / "diffusion_pytorch_model.safetensors"))
    m2 = UNet3DConditionModel.from_pretrained_2d(root, mm_file, subfolder="unet", unet_additional_kwargs=extra)
    assert torch.equal(m2.state_dict()["conv_in.bias"], full["conv_in.bias"] + 1.0)

    # mm_zero_proj_out: the motion modules' proj_out stay at their zero init (identity modules), everything else is loaded
    m3 = UNet3DConditionModel.from_pretrained_2d(root, mm_file, subfolder="unet", unet_additional_kwargs=extra, mm_zero_proj_out=True)
    for k, v in m3.state_dict().items():
        if "motion_modules" in k and "proj_out" in k:
            assert float(v.abs().sum()) == 0.0, k
        elif "motion_modules" in k:
            assert torch.equal(v, full[k]), k

    # a missing motion-module file is not an error (the reference only checks exists() and is_file()): motion modules keep their init
    m4 = UNet3DConditionModel.from_pretrained_2d(root, tmp_path / "absent.ckpt", subfolder="unet", unet_additional_kwargs=extra)
    assert float(m4.state_dict()["mid_block.motion_modules.0.temporal_transformer.proj_out.weight"].abs().sum()) == 0.0

    # a key of the motion-module file that the 2-D file also has overrides it (state_dict.update of every key)
    torch.save({**mm, "conv_in.bias": full["conv_in.bias"] + 2.0}, tmp_path / "mm_plus.ckpt")
    m5 = UNet3DConditionModel.from_pretrained_2d(root, tmp_path / "mm_plus.ckpt", subfolder="unet", unet_additional_kwargs=extra)
    assert torch.equal(m5.state_dict()["conv_in.bias"], full["conv_in.bias"] + 2.0)

    bad = tmp_path / "mm.weights"
    bad.write_bytes(b"x")
    with pytest.raises(RuntimeError):
        UNet3DConditionModel.from_pretrained_2d(root, bad, subfolder="unet", unet_additional_kwargs=extra)
    with pytest.raises(RuntimeError):
        UNet3DConditionModel.from_pretrained_2d(tmp_path / "nowhere", mm_file, unet_additional_kwargs=extra)


def test_reference_unet2d_from_pretrained(tmp_path):
    """The writer UNet's diffusers-style loader: config.json keys its __init__ does not take are dropped, SD checkpoint keys it has no
    parameter for (conv_norm_out / conv_out) are ignored, and a directory without a weights file raises FileNotFoundError."""
    import json

    from safetensors.torch import save_file

    from humanvid_b200 import UNet2DConditionModel

    src = O.synthetic_init(O.UNet2DConditionModel(block_out_channels=(32, 64, 128, 128), cross_attention_dim=64), seed=5)
    sd = {k: v.clone().contiguous() for k, v in src.state_dict().items()}
    d = tmp_path / "unet"
    d.mkdir()
    cfg = {"_class_name": "UNet2DConditionModel", "block_out_channels": [32, 64, 128, 128], "cross_attention_dim": 64, "sample_size": 64,
           "some_future_key": 1}
    json.dump(cfg, open(d / "config.json", "w"))
    with pytest.raises(FileNotFoundError):
        UNet2DConditionModel.from_pretrained(tmp_path, subfolder="unet")
    save_file({**sd, "conv_out.weight": torch.zeros(4, 32, 3, 3), "conv_out.bias": torch.zeros(4)}, str(d / "diffusion_pytorch_model.safetensors"))
    m = UNet2DConditionModel.from_pretrained(tmp_path, subfolder="unet")
    got = m.state_dict()
    assert set(got) == set(sd) and all(torch.equal(got[k], sd[k]) for k in sd)
    assert m.config.sample_size == 64 and m.config.block_out_channels == [32, 64, 128, 128]


def test_native_fingerprint_tracks_parameter_edits():
    """_NativeNet._versions() decides on every forward whether the packed device weights are stale.  Its tensor list is cached per epoch
    (3 ms of module-tree walking per forward otherwise); the fingerprint must still move on an in-place edit of ANY parameter or buffer, on
    load_state_dict(), on .to() / .half(), on refresh_native() -- and must not move otherwise."""
    from humanvid_b200 import PoseGuider, UNet3DConditionModel

    mmk = dict(num_attention_heads=8, num_transformer_block=1, attention_block_types=["Temporal_Self", "Temporal_Self"],
               temporal_position_encoding=True, temporal_position_encoding_max_len=32, temporal_attention_dim_div=1)
    m = UNet3DConditionModel(block_out_channels=(32, 64, 64, 64), cross_attention_dim=32, use_motion_module=True, use_inflated_groupnorm=True,
                             motion_module_resolutions=(1, 2, 4, 8), motion_module_mid_block=True, motion_module_type="Vanilla", motion_module_kwargs=mmk)
    v0 = m._versions()
    assert m._versions() == v0 and m._versions() == v0                               # stable
    n_tensors = len(list(m.parameters())) + len(list(m.buffers()))
    assert len(m.__dict__["_ver_cache"][1]) == n_tensors
    with torch.no_grad():
        m.up_blocks[3].attentions[2].transformer_blocks[0].ff.net[2].bias.add_(1.0)   # a deep parameter, edited in place
    v1 = m._versions()
    assert v1 != v0
    with torch.no_grad():
        m.mid_block.motion_modules[0].temporal_transformer.transformer_blocks[0].attention_blocks[1].pos_encoder.pe.mul_(0.5)   # a buffer
    v2 = m._versions()
    assert v2 != v1
    sd = {k: v.clone() for k, v in m.state_dict().items()}
    m.load_state_dict(sd)
    v3 = m._versions()
    assert v3 != v2 and v3[3] == v2[3] + 1
    m.half()
    v4 = m._versions()
    assert v4 != v3 and v4[2] == torch.float16
    assert all(t.dtype == torch.float16 for t in m.__dict__["_ver_cache"][1] if t.is_floating_point())   # the cache was rebuilt on the new tensors
    m.refresh_native()
    assert m._versions() != v4
    # reader blocks: cached walk == the reference's order (DFS down, up, mid; stable sort by descending width), a fresh list every call
    a, b = m.reader_blocks(), m.reader_blocks()
    assert a == b and a is not b and len(a) == 16
    assert [x.norm1.normalized_shape[0] for x in a] == [64] * 11 + [32] * 5
    names = {id(mod): n for n, mod in m.named_modules()}
    assert [names[id(x)] for x in a][:3] == ["down_blocks.1.attentions.0.transformer_blocks.0", "down_blocks.1.attentions.1.transformer_blocks.0",
                                             "down_blocks.2.attentions.0.transformer_blocks.0"]
    pg = PoseGuider(320, block_out_channels=(16, 32, 96, 256))
    p0 = pg._versions()
    with torch.no_grad():
        pg.blocks[3].weight.zero_()
    assert pg._versions() != p0
