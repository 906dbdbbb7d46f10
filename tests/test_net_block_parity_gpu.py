"""Every block of the native AutoencoderKL, CLIP vision encoder, PoseGuider and camera encoder against fp64 on its own input, per frame,
per token row and per element (tests/block_parity.py).

One native forward per configuration copies every block's output out through the debug taps, each tap buffer pre-filled with NaN so a
block that writes nothing, or writes only part of its output, shows up.  oracle/block_replay.py then applies the oracle module of each
block to the native tap of its predecessor -- the input the native block consumed -- twice: in fp64 with the fp16 weights upcast (R) and
in fp16 eager (E, the reference's deployment).  The native tap N is held to the bounds of tests/block_parity.py against R, E to the row and
element bounds, and every padding channel of N must be exactly zero.  One oracle is on the device at a time; its dtype is switched in place.
In every configuration the network's output with taps set equals its output without taps bit for bit.

Configurations (weights from oracle.synthetic_init, rounded to fp16):
- VAE decode at SD widths (128, 256, 512, 512) on latents of the scale the pipeline decodes (1 / 0.18215 x unit variance, each frame with
  its own spread and offsets, so statistics leaking between frames show): N = 2 at 96x72 (config 2, mid-block attention over 6912
  tokens), N = 1 at 72x128 (config 5, 9216 tokens) and N = 3 at 13x9 (odd sides through the parity upconv, 117 tokens: a partial 64-row
  tile).
- VAE encode: N = 2 at 768x576, a flat grey image next to a random one (statistics leaking between frames would show as a large error on
  the flat frame), and N = 1 at 576x1024.  With the whole plan set, a decode leaves every encoder buffer NaN and an encode every decoder one.
- CLIP ViT-L/14 at 224, B = 2, with the default, qk_scaled and offsets weights of test_clip_vision_gpu.make_hf; the small p = 32 config at
  B = 3 (50 tokens).  image_embeds is checked per element against fp64 visual_projection of the native post_layernorm tap.
- PoseGuider at three width tuples; the plan's channel counts and the profile's kernel labels show which layers ran the small-channel
  kernel and which the 64-padded implicit GEMM.
- Camera encoder at full width (320 channels, cin 384, 8 heads, 2 resnet / attention pairs): B = 1, F = 24 at 768x576 through forward, and
  B = 2, F = 16 at 576x1024 through forward_cameras (the on-device plücker producer).

The VAE's upsamplers run the parity upconv on weights that hv_pack_upconv2x2 sums per 2x2 parity and rounds to fp16, a rounding fp16 eager
(the 3x3 conv of the upsampled grid) does not make.  They are held to the same slice bound as every other block: measured on an H100 80GB
HBM3 at a 700 W power limit, they use at most 0.82 of it at the three decode shapes (the UNet's upsamplers 0.83), so the packing needs no
bound of its own.
"""
import csv
import ctypes as C
import os
import tempfile
import time

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

from block_parity import BlockReport, block_kind, check_fp16_block, check_pad, elem_ratio
from conftest import report

if torch.cuda.is_available():
    import humanvid_b200 as hv
    from humanvid_b200 import _native as N
    from oracle import hv_oracle as O
    from oracle.block_replay import (camera_tap_names, clip_tap_names, pose_guider_tap_names, replay_camera, replay_clip, replay_pose_guider,
                                     replay_vae, vae_tap_names)
    import vae_oracle as V

NAN = float("nan")


@pytest.fixture(scope="module", autouse=True)
def wall_time():
    t0 = time.time()
    yield
    report(f"net block parity: file wall time {time.time() - t0:.0f} s on {torch.cuda.get_device_name()}")


# --------------------------------------------------------------------------------------------------------------- the parity run
def native_run(nat, plan_shape, forward, only=None):
    """(plan, {name: tap}, output with taps set, output without).  only: the plan's names to tap (the others get no buffer)."""
    plan = nat.debug_tap_plan(*plan_shape)
    want = [n for n, _ in plan if only is None or n in only]
    taps = {n: torch.full(d, NAN, device="cuda", dtype=torch.float16) for n, d in plan if n in want}
    with torch.no_grad():
        ref = forward()
        nat.debug_set_taps([taps.get(n) for n, _ in plan])
        try:
            out = forward()
            torch.cuda.synchronize()
        finally:
            nat.debug_set_taps([])
    return plan, taps, out, ref


def assert_same(out, ref, label):
    outs = out if isinstance(out, (list, tuple)) else [out]
    refs = ref if isinstance(ref, (list, tuple)) else [ref]
    assert all(torch.equal(a, b) for a, b in zip(outs, refs)), f"{label}: the output with taps set differs from the output without"


def parity(ora, names, native, replay):
    """{block kind: BlockReport} of every tap: N against R, E against the row and element bounds, N's padding channels exactly zero."""
    reports = {}
    try:
        ora.half()
        E = {n: o.contiguous() for n, o in replay()}
        ora.double()
        for n, r in replay():
            rep = reports.setdefault(block_kind(n), BlockReport())
            c = r.shape[-1]
            check_fp16_block(rep, n, native[n][..., :c], r, E.pop(n)[..., :c])
            check_pad(rep, n, native[n], c)
            del r
    finally:
        ora.half()
        torch.cuda.empty_cache()
    return reports


def assert_reports(label, reports):
    for k, r in reports.items():
        report(f"net block parity {label} {k}: worst err/bound native slice {r.slice.ratio:.3f} row {r.row.ratio:.3f} element {r.elem.ratio:.3f}; "
               f"fp16 eager row {r.e_row.ratio:.3f} element {r.e_elem.ratio:.3f}")
    fails = [f"{k}: {f}" for k, r in reports.items() for f in r.failures()]
    assert not fails, f"{label}:\n" + "\n".join(fails)


# --------------------------------------------------------------------------------------------------------------- AutoencoderKL
@pytest.fixture(scope="module")
def vaes():
    ora = O.synthetic_init(V.AutoencoderKL().eval(), seed=21).half().cuda()
    nat = hv.AutoencoderKL()
    nat.load_state_dict(ora.state_dict())
    nat = nat.to("cuda", torch.float16)
    yield ora, nat
    del ora, nat
    torch.cuda.empty_cache()


def latents(N, h, w, seed):
    """Latents of the scale the pipeline decodes, 1 / 0.18215 x unit variance, each frame with its own spread (0.6 .. 1.4) and per-channel
    offsets.  Frames of i.i.d. latents have nearly the same GroupNorm statistics: with them, every VAE resnet pooling its statistics over
    a call's two frames stayed within 1.06 of the slice bound; with these, it exceeds the slice bound 60-fold and the element bound 7-fold."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    spread = torch.linspace(0.6, 1.4, N, device="cuda") if N > 1 else torch.ones(1, device="cuda")
    z = torch.randn(N, 4, h, w, generator=g, device="cuda") * spread.view(N, 1, 1, 1) + 0.5 * torch.randn(N, 4, 1, 1, generator=g, device="cuda")
    return (z / 0.18215).half()


def test_vae_plan(vaes):
    ora, nat = vaes
    plan = dict(nat.debug_tap_plan(2, 1, 13, 9))
    assert list(plan) == vae_tap_names(ora, "decoder") + vae_tap_names(ora, "encoder")
    assert plan["post_quant_conv"] == (2, 13, 9, 64) and plan["decoder.conv_out"] == (2, 104, 72, 8)
    assert plan["decoder.up_blocks.0.upsamplers.0"] == (2, 26, 18, 512) and plan["encoder.conv_in"] == (2, 104, 72, 128)
    assert plan["quant_conv"] == (2, 13, 9, 8)


@pytest.mark.parametrize("N, h, w", [(2, 96, 72), (1, 72, 128), (3, 13, 9)], ids=["config2", "config5", "odd13x9"])
def test_vae_decode(vaes, N, h, w):
    ora, nat = vaes
    z = latents(N, h, w, seed=h * w + N)
    names = vae_tap_names(ora, "decoder")
    _, taps, out, ref = native_run(nat, (N, 1, h, w), lambda: nat.decode(z).sample, only=names)
    assert_same(out, ref, "decode")
    assert torch.equal(taps["decoder.conv_out"][..., :3], out.permute(0, 2, 3, 1))
    del out, ref
    assert_reports(f"vae decode N={N} {h}x{w}", parity(ora, names, taps, lambda: replay_vae(ora, names, taps, z)))


@pytest.mark.parametrize("N, H, W", [(2, 768, 576), (1, 576, 1024)], ids=["config2_flat_frame", "config5"])
def test_vae_encode(vaes, N, H, W):
    ora, nat = vaes
    g = torch.Generator(device="cuda").manual_seed(H + W)
    x = (torch.rand(N, 3, H, W, generator=g, device="cuda") * 2 - 1).half()
    if N == 2:
        x[0] = 0.25                      # a flat grey frame next to a random one
    names = vae_tap_names(ora, "encoder")
    _, taps, out, ref = native_run(nat, (N, 1, H // 8, W // 8), lambda: nat.encode(x).latent_dist.mean, only=names)
    assert_same(out, ref, "encode")
    assert torch.equal(taps["quant_conv"][..., :4], out.permute(0, 2, 3, 1))
    del out, ref
    assert_reports(f"vae encode N={N} {H}x{W}", parity(ora, names, taps, lambda: replay_vae(ora, names, taps, x)))


def test_vae_tap_routing(vaes):
    """With the whole plan set, a decode fills every decoder buffer and leaves every encoder buffer NaN; an encode the other way round."""
    ora, nat = vaes
    N, h, w = 1, 13, 9
    dec = set(vae_tap_names(ora, "decoder"))
    z = latents(N, h, w, seed=3)
    x = (torch.rand(N, 3, 8 * h, 8 * w, device="cuda") * 2 - 1).half()
    for forward, filled in ((lambda: nat.decode(z).sample, dec), (lambda: nat.encode(x).latent_dist.mean, None)):
        _, taps, _, _ = native_run(nat, (N, 1, h, w), forward)
        for n, t in taps.items():
            if (n in dec) == (filled is not None):
                assert torch.isfinite(t).all(), f"{n}: not written"
            else:
                assert torch.isnan(t).all(), f"{n}: written by the other half's forward"


# --------------------------------------------------------------------------------------------------------------- CLIP
def clip_arms(cfg_name, variant):
    from test_clip_vision_gpu import CONFIGS, make_hf

    m, sd = make_hf(cfg_name, variant)
    nat = hv.CLIPVisionModelWithProjection(**CONFIGS[cfg_name])
    nat.load_state_dict(sd)
    return m.half().cuda(), nat.to("cuda", torch.float16)


@pytest.mark.parametrize("cfg_name, variant, B", [("vit_l14", "default", 2), ("vit_l14", "qk_scaled", 2), ("vit_l14", "offsets", 2),
                                                   ("small", "default", 3)])
def test_clip(cfg_name, variant, B):
    ora, nat = clip_arms(cfg_name, variant)
    g = torch.Generator(device="cuda").manual_seed(11)
    pix = (torch.randn(B, 3, 224, 224, generator=g, device="cuda") * 1.2).half()
    plan, taps, out, ref = native_run(nat, (B, 1, 224, 224), lambda: nat(pix))
    names = [n for n, _ in plan]
    assert names == clip_tap_names(ora)
    assert_same([out.image_embeds, out.last_hidden_state], [ref.image_embeds, ref.last_hidden_state], "clip")
    assert torch.equal(taps[names[-2]][:, 0], out.last_hidden_state)
    reps = parity(ora, names, taps, lambda: replay_clip(ora, names, taps, pix))
    # image_embeds per element against fp64 visual_projection of the native post_layernorm tap
    ora.double()
    with torch.no_grad():
        r = ora.visual_projection(taps[names[-1]][:, 0, 0].double())
    ora.half()
    rep = reps.setdefault("image_embeds", BlockReport())
    rep.elem.take(elem_ratio(out.image_embeds[:, None, None], r[:, None, None]), "image_embeds")
    del ora, nat
    torch.cuda.empty_cache()
    assert_reports(f"clip {cfg_name} {variant} B={B}", reps)


# --------------------------------------------------------------------------------------------------------------- PoseGuider
def profile_labels(nat, forward):
    """The labels of the categorised launches of one forward, in order (hv_dump_profile)."""
    h = nat._sync_native()
    N.check(N.lib().hv_set_profiling(h, N.i32(1)), h)
    try:
        with torch.no_grad():
            forward()
        with tempfile.TemporaryDirectory() as d:
            path = os.path.join(d, "profile.csv")
            N.check(N.lib().hv_dump_profile(h, path.encode()), h)
            with open(path) as f:
                return [row["label"] for row in csv.DictReader(f)]
    finally:
        N.check(N.lib().hv_set_profiling(h, N.i32(0)), h)


# widths: (channels of conv_in, blocks.0 .. blocks.5, conv_out in the plan, the launch labels of the convs)
PG = {
    (16, 32, 96, 256): ([16, 16, 32, 32, 128, 128, 256, 320],
                        ["pg_conv_in", "smallconv", "smallconv_s2", "smallconv", "smallconv_s2", "conv3", "conv3_s2", "conv3"]),
    (16, 32, 64, 128): ([16, 16, 32, 64, 64, 64, 128, 320],
                        ["pg_conv_in", "smallconv", "smallconv_s2", "smallconv", "conv3_s2", "conv3", "conv3_s2", "conv3"]),
    (32, 64, 128, 256): ([64, 64, 64, 64, 128, 128, 256, 320],
                         ["conv3", "conv3_s2", "conv3", "conv3_s2", "conv3", "conv3_s2", "conv3"]),     # conv_in: the direct kernel
}


@pytest.mark.parametrize("widths, F_, H, W", [((16, 32, 96, 256), 2, 768, 576), ((16, 32, 96, 256), 2, 576, 1024), ((16, 32, 96, 256), 3, 24, 40),
                                              ((16, 32, 64, 128), 2, 256, 192), ((32, 64, 128, 256), 2, 256, 192)],
                         ids=["16-32-96-256_768x576", "16-32-96-256_576x1024", "16-32-96-256_24x40", "16-32-64-128", "32-64-128-256"])
def test_pose_guider(widths, F_, H, W):
    ora = O.synthetic_init(O.PoseGuider(320, 3, widths).eval(), seed=11).half().cuda()     # conv_out non-zero (the module zero-inits it)
    nat = hv.PoseGuider(320, block_out_channels=widths)
    nat.load_state_dict(ora.state_dict())
    nat = nat.to("cuda", torch.float16)
    g = torch.Generator(device="cuda").manual_seed(H + F_)
    cond = torch.rand(1, 3, F_, H, W, generator=g, device="cuda").half()
    plan, taps, out, ref = native_run(nat, (1, F_, H, W), lambda: nat(cond))
    names = [n for n, _ in plan]
    assert names == pose_guider_tap_names(ora)
    chans, labels = PG[widths]
    assert [d[-1] for _, d in plan] == chans
    assert profile_labels(nat, lambda: nat(cond)) == labels
    assert_same(out, ref, "pose guider")
    assert torch.equal(taps["conv_out"], out.permute(0, 2, 3, 4, 1).flatten(0, 1))
    reps = parity(ora, names, taps, lambda: replay_pose_guider(ora, names, taps, cond))
    del ora, nat
    assert_reports(f"pose guider {widths} F={F_} {H}x{W}", reps)


# --------------------------------------------------------------------------------------------------------------- camera encoder
def cameras(B, F_, H, W, seed):
    """Intrinsics (B, F, 4) in pixels and c2w (B, F, 4, 4): a random rotation and translation per frame."""
    g = torch.Generator().manual_seed(seed)
    K = torch.tensor([0.9 * W, 0.9 * H, 0.5 * W, 0.5 * H]) * (1 + 0.05 * torch.randn(B, F_, 4, generator=g))
    q, r = torch.linalg.qr(torch.randn(B, F_, 3, 3, generator=g, dtype=torch.float64))
    q = q * torch.sign(torch.diagonal(r, dim1=-2, dim2=-1)).unsqueeze(-2)
    q[torch.det(q) < 0] *= -1
    c2w = torch.eye(4, dtype=torch.float64).repeat(B, F_, 1, 1)
    c2w[..., :3, :3] = q
    c2w[..., :3, 3] = torch.randn(B, F_, 3, generator=g, dtype=torch.float64)
    return K.float(), c2w.float()


@pytest.mark.parametrize("B, F_, H, W, rays", [(1, 24, 768, 576, False), (2, 16, 576, 1024, True)], ids=["forward_F24", "forward_cameras"])
def test_camera_encoder(B, F_, H, W, rays):
    ora = O.synthetic_init(O.CameraPoseEncoder().eval(), seed=13).half().cuda()          # zero_conv_layers non-zero
    nat = hv.CameraPoseEncoder(downscale_factor=8, channels=[320], nums_rb=2, cin=384, ksize=1, sk=True, use_conv=False, compression_factor=1,
                               temporal_attention_nhead=8, attention_block_types=["Temporal_Self"], temporal_position_encoding=True,
                               temporal_position_encoding_max_len=24)
    nat.load_state_dict(ora.state_dict())
    nat = nat.to("cuda", torch.float16)
    if rays:
        K, c2w = cameras(B, F_, H, W, seed=F_)
        Kd, Md = K.cuda().contiguous(), c2w.cuda().contiguous()
        # the embedding the encoder's producer makes, as test_model_gpu.py derives it: hv_op_plucker_unshuffle, then PixelShuffle back
        un = torch.empty(B * F_, H // 8, W // 8, 384, device="cuda", dtype=torch.float16)
        N.check(N.lib().hv_op_plucker_unshuffle(N.ptr(Kd), N.ptr(Md), N.ptr(un), N.i64(B * F_), N.i64(H), N.i64(W), N.i32(8), N.stream()))
        plucker = F.pixel_shuffle(un.permute(0, 3, 1, 2), 8).reshape(B, F_, 6, H, W).transpose(1, 2)
        forward = lambda: nat.forward_cameras(K, c2w, H, W)[0]
    else:
        g = torch.Generator(device="cuda").manual_seed(F_)
        plucker = torch.randn(B, 6, F_, H, W, generator=g, device="cuda").half()
        forward = lambda: nat(plucker)[0]
    plan, taps, out, ref = native_run(nat, (B, F_, H, W), forward)
    names = [n for n, _ in plan]
    assert names == camera_tap_names(ora)
    assert_same(out, ref, "camera encoder")
    assert torch.equal(taps["zero_conv_layers.0"], out.permute(0, 2, 3, 1))
    reps = parity(ora, names, taps, lambda: replay_camera(ora, names, taps, plucker))
    del ora, nat
    assert_reports(f"camera encoder B={B} F={F_} {H}x{W}{' rays' if rays else ''}", reps)
