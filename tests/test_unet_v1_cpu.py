"""CPU tests of the inference_v1 UNet layout (AnimateDiff v1 motion modules): GroupNorm statistics pooled over frames and no mid-block
motion module.  The native shell must expose the reference's keys and shapes and load a from_pretrained_2d checkpoint; the oracle
(tests/unet_v1_oracle.py) must reproduce the golden written from the reference's own UNet3DConditionModel (scripts/pin_unet_v1.py)."""
import json
import os

import torch

from oracle import hv_oracle as O
from unet_v1_oracle import V1_MAX_LEN, V1_UNET_KWARGS, unet3d_v1

GOLD = os.path.join(os.path.dirname(__file__), "golden")
CHS, XDIM = (32, 64, 128, 128), 64


def v1_shell(**kw):
    from humanvid_b200 import UNet3DConditionModel

    return UNet3DConditionModel(block_out_channels=CHS, cross_attention_dim=XDIM, attention_head_dim=8, **{**V1_UNET_KWARGS, **kw})


def test_v1_shell_has_the_oracle_keys_and_shapes():
    m = v1_shell()
    sm, so = m.state_dict(), unet3d_v1(CHS, XDIM).state_dict()
    assert set(sm) == set(so)
    assert all(sm[k].shape == so[k].shape for k in so)
    assert not any(k.startswith("mid_block.motion_modules") for k in sm)
    assert any(k.startswith("down_blocks.0.motion_modules.0.") for k in sm) and any(k.startswith("up_blocks.3.motion_modules.2.") for k in sm)
    pes = {k: v for k, v in sm.items() if k.endswith("pos_encoder.pe")}
    assert len(pes) == 2 * (2 * 4 + 3 * 4)
    assert all(tuple(v.shape) == (1, V1_MAX_LEN, v.shape[-1]) for v in pes.values())
    assert m.config.use_inflated_groupnorm is False and m.config.motion_module_mid_block is False
    cfg = m._hv_config()
    assert (cfg.gn_pool_frames, cfg.no_mid_motion_module, cfg.motion_max_len, cfg.use_motion_module) == (1, 1, V1_MAX_LEN, 1)


def test_v2_and_image_shells_keep_the_zero_config():
    v2 = v1_shell(use_inflated_groupnorm=True, motion_module_mid_block=True)
    assert any(k.startswith("mid_block.motion_modules.0.") for k in v2.state_dict())
    c = v2._hv_config()
    assert (c.gn_pool_frames, c.no_mid_motion_module) == (0, 0)
    # stage 1 (Pose2ImagePipeline): no motion module, plain nn.GroupNorm; it only ever runs one frame, where pooling is the per-frame path
    img = v1_shell(use_motion_module=False)
    c = img._hv_config()
    assert (c.gn_pool_frames, c.no_mid_motion_module, c.use_motion_module) == (1, 0, 0)


def test_oracle_reproduces_the_v1_reference_golden():
    g = torch.load(os.path.join(GOLD, "unet_narrow_v1.pt"), weights_only=False)
    assert g["max_abs_diff"] == 0.0 and g["x"].shape[2] >= 3
    m = O.synthetic_init(unet3d_v1(tuple(g["chs"]), g["xdim"]).eval(), seed=g["seed"])
    with torch.no_grad():
        y = m(g["x"], torch.tensor(g["t"]), g["ehs"], pose_cond_fea=g["pose"])[0]
    assert torch.allclose(y, g["y"], atol=1e-5, rtol=1e-5)
    # the pooled statistics matter at this input (its frames drift apart): per-frame GroupNorm in the same network gives another answer
    per_frame = {}
    for name, mod in m.named_modules():
        if name.endswith(("norm1", "norm2")) and isinstance(mod, torch.nn.GroupNorm) or name == "conv_norm_out":
            per_frame[name] = mod
    assert len(per_frame) == 2 * (2 * 4 + 2 + 3 * 4) + 1
    for mod in per_frame.values():
        mod.__class__ = O.InflatedGroupNorm
    with torch.no_grad():
        y_pf = m(g["x"], torch.tensor(g["t"]), g["ehs"], pose_cond_fea=g["pose"])[0]
    assert float((y_pf - g["y"]).norm() / g["y"].norm()) > 1e-2


def test_from_pretrained_2d_loads_a_v1_checkpoint(tmp_path):
    from humanvid_b200 import UNet3DConditionModel

    src = O.synthetic_init(unet3d_v1(CHS, XDIM), seed=5)
    full = {k: v.clone() for k, v in src.state_dict().items()}
    sd2d = {k: v.contiguous() for k, v in full.items() if "motion_modules" not in k}
    mm = {k: v.contiguous() for k, v in full.items() if "motion_modules" in k}
    root = tmp_path / "sd15"
    (root / "unet").mkdir(parents=True)
    cfg = {"_class_name": "UNet2DConditionModel", "in_channels": 4, "out_channels": 4, "block_out_channels": list(CHS), "cross_attention_dim": XDIM,
           "attention_head_dim": 8, "layers_per_block": 2, "norm_num_groups": 32, "act_fn": "silu",
           "down_block_types": ["CrossAttnDownBlock2D"] * 3 + ["DownBlock2D"], "up_block_types": ["UpBlock2D"] + ["CrossAttnUpBlock2D"] * 3}
    json.dump(cfg, open(root / "unet" / "config.json", "w"))
    torch.save(sd2d, root / "unet" / "diffusion_pytorch_model.bin")
    torch.save(mm, tmp_path / "mm_sd_v15.ckpt")
    m = UNet3DConditionModel.from_pretrained_2d(root, tmp_path / "mm_sd_v15.ckpt", subfolder="unet", unet_additional_kwargs=V1_UNET_KWARGS)
    got = m.state_dict()
    assert set(got) == set(full) and all(torch.equal(got[k], full[k]) for k in full)
    assert m.config.use_inflated_groupnorm is False and m.config.motion_module_mid_block is False
    assert m._hv_config().gn_pool_frames == 1
