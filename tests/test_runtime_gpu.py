"""Bookkeeping of the native runtime on an H100: what a forward reports about itself stays readable after the planning
passes (workspace sizing, tap plan) that follow it."""
import pytest
import torch

pytestmark = pytest.mark.gpu

if torch.cuda.is_available():
    import humanvid_b200 as hv
    from oracle import hv_oracle as O

CHS, XDIM = (64, 128, 256, 256), 64


@pytest.fixture(scope="module")
def narrow_unet():
    ora = O.UNet3DConditionModel(block_out_channels=CHS, cross_attention_dim=XDIM, use_motion_module=False, use_inflated_groupnorm=False)
    ora = O.synthetic_init(ora.eval(), seed=7)
    nat = hv.UNet3DConditionModel(block_out_channels=CHS, cross_attention_dim=XDIM, unet_use_cross_frame_attention=False,
                                  unet_use_temporal_attention=False)
    nat.load_state_dict(ora.state_dict())
    return nat.to("cuda", torch.float16)


def test_launch_count_survives_planning(narrow_unet):
    B, F, h, w = 2, 1, 16, 16
    g = torch.Generator(device="cuda").manual_seed(0)
    x = torch.randn(B, 4, F, h, w, generator=g, device="cuda").half()
    ehs = torch.randn(B, 1, XDIM, generator=g, device="cuda").half()
    with torch.no_grad():
        narrow_unet(x, 500, ehs, return_dict=False)
    torch.cuda.synchronize()
    n = narrow_unet.last_launch_count
    assert n > 0
    assert narrow_unet.workspace_bytes(B, F, h, w) > 0
    assert len(narrow_unet.debug_tap_plan(B, F, h, w)) > 0
    assert narrow_unet.last_launch_count == n
