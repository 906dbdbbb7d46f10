"""fp32 oracle of UNet3DConditionModel in the configs/inference/inference_v1.yaml layout (AnimateDiff v1 motion modules).

It is oracle/hv_oracle.py's UNet3DConditionModel with the three things inference_v1.yaml changes against inference_v2.yaml:
- use_inflated_groupnorm=False: the resnets' norm1 / norm2 and conv_norm_out are nn.GroupNorm on the 5-D (b, c, f, h, w) tensor, so
  their statistics span every frame of a batch item (resnet.py:153-190, unet_3d.py:235-246);
- motion_module_mid_block=False: the mid block has no motion module (unet_3d.py:173), so no mid_block.motion_modules.* keys;
- temporal_position_encoding_max_len=24: every motion module's pos_encoder.pe is (1, 24, C).
scripts/pin_unet_v1.py pins it bit for bit against the reference's own UNet3DConditionModel and writes tests/golden/unet_narrow_v1.pt.
"""
import torch.nn as nn

from oracle import hv_oracle as O

V1_MAX_LEN = 24

# unet_additional_kwargs of inference_v1.yaml (use_inflated_groupnorm is absent there, so the class default False applies)
V1_MM_KWARGS = dict(num_attention_heads=8, num_transformer_block=1, attention_block_types=["Temporal_Self", "Temporal_Self"],
                    temporal_position_encoding=True, temporal_position_encoding_max_len=V1_MAX_LEN, temporal_attention_dim_div=1)
V1_UNET_KWARGS = dict(unet_use_cross_frame_attention=False, unet_use_temporal_attention=False, use_motion_module=True,
                      motion_module_resolutions=[1, 2, 4, 8], motion_module_mid_block=False, motion_module_decoder_only=False,
                      motion_module_type="Vanilla", motion_module_kwargs=V1_MM_KWARGS)


def unet3d_v1(block_out_channels=(320, 640, 1280, 1280), cross_attention_dim=768, in_channels=4, out_channels=4) -> O.UNet3DConditionModel:
    m = O.UNet3DConditionModel(in_channels, out_channels, block_out_channels, cross_attention_dim=cross_attention_dim, use_motion_module=True,
                               use_inflated_groupnorm=False)
    m.mid_block.motion_modules = nn.ModuleList([None])
    for mod in m.modules():
        if isinstance(mod, O.PositionalEncoding):
            mod.pe = O.sinusoid_table(V1_MAX_LEN, mod.pe.shape[-1])
    return m
