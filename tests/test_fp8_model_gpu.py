"""FP8 mode of the native UNet3DConditionModel (enable_fp8_linears) on an H100.

The network is narrow (channels 64, 128, 256, 1280, cross-attention dim 64) so that the feed-forwards FP8 mode runs on e4m3 (width
>= 1280: the level-3 motion modules, the mid block's transformer and motion module) sit beside fp16 ones.

Accuracy (DESIGN.md §9):  rel(native_fp8, oracle_fp32) <= (1 + 1/4) rel(emulated_fp8, oracle_fp32) + rel(native_fp16, oracle_fp32).
The emulation (tests/fp8_emulation.emulate_fp8_linears) is the fp32 oracle with the FP8 path's quantise-dequantise steps; the native
FP8 forward differs from it by the fp16 path's own error and by the values whose e4m3 rounding flips because their input carries that
fp16 error.  A flip moves a value by one e4m3 step (<= 2^-3 of it) and happens to a fraction of about (fp16 error / e4m3 step) ~ 2^-11 /
2^-4 of the values, an rms of 2^-3 sqrt(2^-7) ~ 1.1 % of the values against the quantisation's own rms of at least 2^-4 / sqrt(12)
~ 1.8 %: the flips add at most about 0.6 of the emulation's error in quadrature, under 1/4 of it in the sum.  That is the margin.

Composition, all bitwise in FP8 mode: two runs, a batch item alone against the same item inside a batch of two, the CFG unit flags against
the joint CFG forward, and disable after enable against a model that never enabled it."""
import pytest
import torch

pytestmark = pytest.mark.gpu

from conftest import report
from fp8_emulation import emulate_fp8_linears

if torch.cuda.is_available():
    import humanvid_b200 as hv
    from oracle import hv_oracle as O

CHS, XDIM = (64, 128, 256, 1280), 64
MM_KW = dict(num_attention_heads=8, num_transformer_block=1, attention_block_types=["Temporal_Self", "Temporal_Self"],
             temporal_position_encoding=True, temporal_position_encoding_max_len=32, temporal_attention_dim_div=1)


def rel(a, b):
    a, b = a.float(), b.float()
    return float((a - b).norm() / b.norm())


def make(seed=7):
    ora = O.synthetic_init(O.UNet3DConditionModel(block_out_channels=CHS, cross_attention_dim=XDIM).eval(), seed=seed).half().float().cuda()
    kw = dict(block_out_channels=CHS, cross_attention_dim=XDIM, use_motion_module=True, use_inflated_groupnorm=True,
              motion_module_resolutions=(1, 2, 4, 8), motion_module_mid_block=True, motion_module_type="Vanilla", motion_module_kwargs=MM_KW,
              unet_use_cross_frame_attention=False, unet_use_temporal_attention=False)
    nat = hv.UNet3DConditionModel(**kw)
    nat.load_state_dict(ora.state_dict())
    return ora, nat.to("cuda", torch.float16)


def inputs(B=2, F=4, h=16, w=16, seed=1):
    g = torch.Generator(device="cuda").manual_seed(seed)
    x = torch.randn(B, 4, F, h, w, generator=g, device="cuda").half()
    ehs = torch.randn(B, 1, XDIM, generator=g, device="cuda").half()
    ehs[: B // 2] = 0
    pose = (torch.randn(B, CHS[0], F, h, w, generator=g, device="cuda") * 0.5).half()
    return x, ehs, pose


@pytest.fixture(scope="module")
def nets():
    return make()


def run(nat, x, ehs, pose, t=500):
    with torch.no_grad():
        y = nat(x, t, ehs, pose_cond_fea=pose, return_dict=False)[0]
    torch.cuda.synchronize()
    return y


def test_toggle_state(nets):
    _, nat = nets
    assert nat.fp8_linears is False
    e0 = nat._epoch
    nat.enable_fp8_linears()
    assert nat.fp8_linears is True and nat._epoch == e0 + 1
    nat.enable_fp8_linears()            # no change, no rebuild
    assert nat._epoch == e0 + 1
    nat.disable_fp8_linears()
    assert nat.fp8_linears is False and nat._epoch == e0 + 2


def test_network_bound(nets):
    ora, nat = nets
    x, ehs, pose = inputs()
    with torch.no_grad():
        y32 = ora(x.float(), torch.tensor(500, device="cuda"), ehs.float(), pose_cond_fea=pose.float())[0]
        with emulate_fp8_linears(ora):
            yemu = ora(x.float(), torch.tensor(500, device="cuda"), ehs.float(), pose_cond_fea=pose.float())[0]
    nat.disable_fp8_linears()
    y16 = run(nat, x, ehs, pose)
    nat.enable_fp8_linears()
    y8 = run(nat, x, ehs, pose)
    nat.disable_fp8_linears()
    e8, eemu, e16 = rel(y8, y32), rel(yemu, y32), rel(y16, y32)
    report(f"fp8 narrow UNet (64,128,256,1280): native fp8 {e8:.3e}, emulated fp8 {eemu:.3e}, native fp16 {e16:.3e} vs fp32 oracle; "
           f"native fp8 vs emulation {rel(y8, yemu):.3e}")
    assert torch.isfinite(y8).all()
    assert not torch.equal(y8, y16), "FP8 mode changed nothing: no feed-forward ran on e4m3"
    assert eemu > e16, "the emulation carries no quantisation error: no feed-forward was emulated"
    assert e8 <= 1.25 * eemu + e16, f"native fp8 {e8:.3e} > 1.25 x emulated {eemu:.3e} + native fp16 {e16:.3e}"


def test_composition_bitwise(nets):
    _, nat = nets
    x, ehs, pose = inputs()
    nat.enable_fp8_linears()
    try:
        a = run(nat, x, ehs, pose)
        b = run(nat, x, ehs, pose)
        assert torch.equal(a, b), "two FP8 forwards differ"
        one = run(nat, x[1:], ehs[1:], pose[1:])
        assert torch.equal(one[0], a[1]), "a batch item alone differs from the same item in a batch of two"
        # CFG as separate units: the unconditional and the conditional half through HV_FLAG_UNCOND_ONLY / HV_FLAG_COND_ONLY flags
        nat._forward_flags = 2
        u = run(nat, x[:1], ehs[:1], pose[:1])
        nat._forward_flags = 4
        c = run(nat, x[1:], ehs[1:], pose[1:])
        nat._forward_flags = None
        assert torch.equal(u[0], a[0]) and torch.equal(c[0], a[1]), "CFG unit forwards differ from the joint forward"
    finally:
        nat._forward_flags = None
        nat.disable_fp8_linears()
    off = run(nat, x, ehs, pose)
    _, fresh = make()
    never = run(fresh, x, ehs, pose)
    assert torch.equal(off, never), "disable after enable differs from a model that never enabled FP8"
