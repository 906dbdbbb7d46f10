"""The inference_v1 UNet layout on an H100: GroupNorm statistics pooled over the frames of a window in the resnets and conv_norm_out,
no mid-block motion module, a 24-row positional encoding.  Native against the fp32 oracle (tests/unet_v1_oracle.py) on identical
weights, with the tolerances of tests/test_model_gpu.py and tests/test_fullsize_gpu.py; CFG-half units bitwise equal to the halves of
the CFG batch; determinism.  The latents drift from frame to frame, and the same network with per-frame GroupNorm is checked to be far
from the oracle on them."""
import pytest
import torch

pytestmark = pytest.mark.gpu

from conftest import report
from unet_v1_oracle import V1_UNET_KWARGS, unet3d_v1

if torch.cuda.is_available():
    import humanvid_b200 as hv
    from oracle import hv_oracle as O

NARROW, XDIM = (64, 128, 256, 256), 64
FLAG_CFG, FLAG_UNCOND_ONLY, FLAG_COND_ONLY = 1, 2, 4


def rel(a, b):
    a, b = a.float(), b.float()
    return float((a - b).norm() / (b.norm() + 1e-12))


def make_v1(chs, xdim, seed=7, dtype=torch.float32):
    ora = O.synthetic_init(unet3d_v1(chs, xdim).eval(), seed=seed).half().to("cuda", dtype)   # fp16-representable weights
    nat = hv.UNet3DConditionModel(block_out_channels=chs, cross_attention_dim=xdim, attention_head_dim=8, **V1_UNET_KWARGS)
    nat.load_state_dict(ora.state_dict())
    return ora, nat.to("cuda", torch.float16)


def inputs(B, F, h, w, c0, xdim, seed=1, drift=0.25):
    g = torch.Generator(device="cuda").manual_seed(seed)
    x = torch.randn(B, 4, F, h, w, generator=g, device="cuda")
    x = (x + drift * torch.arange(F, device="cuda").view(1, 1, F, 1, 1)).half()
    ehs = torch.randn(B, 1, xdim, generator=g, device="cuda").half()
    ehs[: B // 2] = 0  # uncond half, like the pipeline
    pose = (torch.randn(B, c0, F, h, w, generator=g, device="cuda") * 0.5).half()
    return x, ehs, pose


@pytest.fixture(scope="module")
def narrow():
    return make_v1(NARROW, XDIM)


def set_banks(ora, nat, banks, cfg):
    ctl = hv.ReferenceAttentionControl(nat, do_classifier_free_guidance=cfg, mode="read", fusion_blocks="full")
    for blk, bk in zip(nat.reader_blocks(), banks):
        blk.bank = [bk]
    O.set_reference_banks(ora, [b.float() for b in banks], cfg=cfg)
    return ctl


@pytest.mark.parametrize("banks", [False, True])
@pytest.mark.parametrize("F", [3, 24])
def test_v1_narrow_parity(narrow, F, banks):
    ora, nat = narrow
    B, t = 2, 721
    x, ehs, pose = inputs(B, F, 16, 16, NARROW[0], XDIM, seed=F)
    ctl, bk = None, None
    if banks:
        g = torch.Generator(device="cuda").manual_seed(5)
        bk = [torch.randn(B, l, c, generator=g, device="cuda").half() for (l, c) in O.bank_shapes(ora, 16, 16)]
        ctl = set_banks(ora, nat, bk, cfg=True)
    try:
        with torch.no_grad():
            y32 = ora(x.float(), torch.tensor(t, device="cuda"), ehs.float(), pose_cond_fea=pose.float())[0]
            ora.half()
            if bk is not None:
                O.set_reference_banks(ora, bk, cfg=True)
            y16 = ora(x, torch.tensor(t, device="cuda"), ehs, pose_cond_fea=pose)[0]
            ora.float()
            yn = nat(x, t, ehs, pose_cond_fea=pose, return_dict=False)[0]
        torch.cuda.synchronize()
    finally:
        if ctl is not None:
            ctl.clear()
        O.set_reference_banks(ora, None)
    e_ref, e_nat, e_pair = rel(y16, y32), rel(yn, y32), rel(yn, y16)
    report(f"v1 narrow F={F} banks={int(banks)}: fp16-eager vs fp32 {e_ref:.2e}; native vs fp32 {e_nat:.2e}; native vs fp16-eager {e_pair:.2e}")
    assert torch.isfinite(yn).all()
    assert e_nat <= e_ref + 1e-4 or e_nat <= 1e-3
    assert e_pair <= 2.5e-3


def test_v1_cfg_half_units_are_bitwise_halves_of_the_cfg_batch(narrow):
    ora, nat = narrow
    B, F, t = 2, 7, 400
    x, ehs, pose = inputs(B, F, 16, 16, NARROW[0], XDIM, seed=11)
    g = torch.Generator(device="cuda").manual_seed(6)
    ctl = set_banks(ora, nat, [torch.randn(B, l, c, generator=g, device="cuda").half() for (l, c) in O.bank_shapes(ora, 16, 16)], cfg=True)
    try:
        with torch.no_grad():
            y = nat(x, t, ehs, pose_cond_fea=pose, return_dict=False)[0].clone()
            y_again = nat(x, t, ehs, pose_cond_fea=pose, return_dict=False)[0].clone()
            nat._forward_flags = FLAG_UNCOND_ONLY
            yu = nat(x[:1].contiguous(), t, ehs[:1].contiguous(), pose_cond_fea=pose[:1].contiguous(), return_dict=False)[0].clone()
            nat._forward_flags = FLAG_COND_ONLY
            yc = nat(x[1:].contiguous(), t, ehs[1:].contiguous(), pose_cond_fea=pose[1:].contiguous(), return_dict=False)[0].clone()
    finally:
        nat._forward_flags = None
        ctl.clear()
        O.set_reference_banks(ora, None)
    assert torch.equal(y, y_again)
    assert torch.equal(yu, y[:1]), "the uncond-only unit differs from the uncond half of the CFG batch"
    assert torch.equal(yc, y[1:]), "the cond-only unit differs from the cond half of the CFG batch"


def test_v1_pools_groupnorm_statistics_over_the_window(narrow):
    """The same network with per-frame GroupNorm (use_inflated_groupnorm=True, everything else v1) is far from the v1 oracle on these
    drifting latents, and the v1 native network is not: the parity above comes from the pooled statistics, not from tolerance."""
    ora, nat = narrow
    pf = hv.UNet3DConditionModel(block_out_channels=NARROW, cross_attention_dim=XDIM, attention_head_dim=8,
                                 **{**V1_UNET_KWARGS, "use_inflated_groupnorm": True})
    pf.load_state_dict(ora.state_dict())
    pf = pf.to("cuda", torch.float16)
    assert pf._hv_config().gn_pool_frames == 0 and nat._hv_config().gn_pool_frames == 1
    x, ehs, pose = inputs(2, 7, 16, 16, NARROW[0], XDIM, seed=4, drift=0.5)
    with torch.no_grad():
        y32 = ora(x.float(), torch.tensor(300, device="cuda"), ehs.float(), pose_cond_fea=pose.float())[0]
        yn = nat(x, 300, ehs, pose_cond_fea=pose, return_dict=False)[0]
        ypf = pf(x, 300, ehs, pose_cond_fea=pose, return_dict=False)[0]
    torch.cuda.synchronize()
    e_n, e_pf = rel(yn, y32), rel(ypf, y32)
    report(f"v1 narrow F=7, drift 0.5/frame: pooled native vs fp32 oracle {e_n:.2e}; per-frame GroupNorm network vs the same oracle {e_pf:.2e}")
    assert e_n < 2.5e-3 and e_pf > 10 * e_n


@pytest.mark.parametrize("layout", ["v1", "v2"])
def test_banked_forward_after_a_bankless_one_at_the_same_shape(layout):
    """The workspace is planned with the reference banks' K/V scratch: a forward with banks that follows a bank-less forward at the same
    shape must run and give what a fresh model gives (it failed with HV_ERR_STATE where the banks raise the workspace peak, as in v1)."""
    kw = dict(V1_UNET_KWARGS)
    if layout == "v2":
        kw.update(use_inflated_groupnorm=True, motion_module_mid_block=True,
                  motion_module_kwargs=dict(kw["motion_module_kwargs"], temporal_position_encoding_max_len=32))
    ora = O.synthetic_init((unet3d_v1(NARROW, XDIM) if layout == "v1" else O.UNet3DConditionModel(block_out_channels=NARROW, cross_attention_dim=XDIM))
                           .eval(), seed=9)
    nets = []
    for _ in range(2):
        n = hv.UNet3DConditionModel(block_out_channels=NARROW, cross_attention_dim=XDIM, attention_head_dim=8, **kw)
        n.load_state_dict(ora.state_dict())
        nets.append(n.to("cuda", torch.float16))
    B, F = 2, 3
    x, ehs, pose = inputs(B, F, 16, 16, NARROW[0], XDIM, seed=8)
    g = torch.Generator(device="cuda").manual_seed(2)
    banks = [torch.randn(B, l, c, generator=g, device="cuda").half() for (l, c) in O.bank_shapes(ora, 16, 16)]
    with torch.no_grad():
        nets[0](x, 500, ehs, pose_cond_fea=pose, return_dict=False)
        ys = []
        for n in nets:
            ctl = hv.ReferenceAttentionControl(n, do_classifier_free_guidance=True, mode="read", fusion_blocks="full")
            for blk, bk in zip(n.reader_blocks(), banks):
                blk.bank = [bk]
            ys.append(n(x, 500, ehs, pose_cond_fea=pose, return_dict=False)[0].clone())
            ctl.clear()
    assert torch.equal(ys[0], ys[1])


def test_v1_config2_shape_full_size():
    """(2, 4, 24, 96, 72) at full width: native is no further from the fp32 oracle than the oracle's own fp16 run."""
    CH, XD, F, H, W = (320, 640, 1280, 1280), 768, 24, 96, 72
    ora, nat = make_v1(CH, XD, dtype=torch.float16)
    x, ehs, pose = inputs(2, F, H, W, CH[0], XD, seed=42, drift=0.1)
    t = 519
    with torch.no_grad():
        yn = nat(x, t, ehs, pose_cond_fea=pose, return_dict=False)[0]
        y16 = ora(x, torch.tensor(t, device="cuda"), ehs, pose_cond_fea=pose)[0]
        ora.float()
        y32 = ora(x.float(), torch.tensor(t, device="cuda"), ehs.float(), pose_cond_fea=pose.float())[0]
    torch.cuda.synchronize()
    e_ref, e_nat, e_pair = rel(y16, y32), rel(yn, y32), rel(yn, y16)
    report(f"v1 config2 full size (2,4,24,96,72): fp16-eager vs fp32 {e_ref:.2e}; native vs fp32 {e_nat:.2e}; native vs fp16-eager {e_pair:.2e}")
    assert torch.isfinite(yn).all()
    assert e_nat <= e_ref
    assert e_pair <= 2.5e-3
    del ora, nat
    torch.cuda.empty_cache()
