"""The model runtime calls the same checked operator functions as the operator C ABI, so an operator the forward cannot run is rejected on
the host with HV_ERR_INVALID and the operator's own message, before its kernel is launched.  Here: a motion module whose position-encoding
table allows 64 frames passes the forward's video-length test at F = 33, and temporal attention (at most 32 frames) refuses it."""
import pytest
import torch

pytestmark = pytest.mark.gpu

if torch.cuda.is_available():
    import humanvid_b200 as hv
    from oracle import hv_oracle as O

MM_KW = dict(num_attention_heads=8, num_transformer_block=1, attention_block_types=["Temporal_Self", "Temporal_Self"],
             temporal_position_encoding=True, temporal_position_encoding_max_len=64, temporal_attention_dim_div=1)


def test_forward_past_the_temporal_attention_frame_limit_is_invalid():
    chs, xdim = (64, 128, 256, 256), 64
    ora = O.UNet3DConditionModel(block_out_channels=chs, cross_attention_dim=xdim, use_motion_module=True, use_inflated_groupnorm=True).eval()
    O.synthetic_init(ora, seed=7)
    nat = hv.UNet3DConditionModel(block_out_channels=chs, cross_attention_dim=xdim, unet_use_cross_frame_attention=False, unet_use_temporal_attention=False,
                                  use_motion_module=True, use_inflated_groupnorm=True, motion_module_resolutions=(1, 2, 4, 8), motion_module_mid_block=True,
                                  motion_module_type="Vanilla", motion_module_kwargs=MM_KW)
    # the oracle's tables hold 32 positions; the native model keeps its own 64-position tables
    sd = {k: v for k, v in ora.half().state_dict().items() if not k.endswith("pos_encoder.pe")}
    missing, unexpected = nat.load_state_dict(sd, strict=False)
    assert not unexpected and missing and all(k.endswith("pos_encoder.pe") for k in missing)
    nat = nat.to("cuda", torch.float16)
    B, F, h, w = 2, 33, 16, 16
    g = torch.Generator(device="cuda").manual_seed(1)
    x = torch.randn(B, 4, F, h, w, generator=g, device="cuda").half()
    ehs = torch.randn(B, 1, xdim, generator=g, device="cuda").half()
    pose = (torch.randn(B, chs[0], F, h, w, generator=g, device="cuda") * 0.5).half()
    with pytest.raises(RuntimeError) as e, torch.no_grad():
        nat(x, 10, ehs, pose_cond_fea=pose)
    torch.cuda.synchronize()
    msg = str(e.value)
    assert "error -1:" in msg, msg
    assert "temporal attention" in msg and "F=33" in msg and "F <= 32" in msg, msg
