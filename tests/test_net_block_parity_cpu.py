"""The per-block replays of the VAE, CLIP, PoseGuider and camera encoder (oracle/block_replay.py), proven on the CPU.

Each oracle runs one whole forward in fp64 at a tiny size, with forward hooks capturing the output of every tapped module in tap layout:
the captures are what a perfect native forward would copy out.  Fed to the replay as the native taps, every replayed block must equal its
capture bit for bit and the last one the network's output, which proves the tap names, their order and each block's predecessor.  Then one
fault is put into one block of the forward (the hook returns the altered output, so the blocks after it consume it as they would a faulty
native block's), and the checks of tests/block_parity.py must flag that block and no other."""
import pytest
import torch
import torch.nn.functional as F

import vae_oracle as V
from block_parity import BlockReport, block_kind, check_fp16_block, check_pad
from oracle import hv_oracle as O
from oracle.block_replay import (camera_tap_names, clip_tap_names, pose_guider_tap_names, replay_camera, replay_clip, replay_pose_guider,
                                 replay_vae, vae_tap_names)

transformers = pytest.importorskip("transformers")

DT = torch.float64


def nhwc(t):
    """A module's output as a tap: (NF, C, H, W) -> (NF, H, W, C); (b, c, f, h, w) -> (b f, h, w, c); (B, L, C) -> (B, 1, L, C);
    (B, C) -> (B, 1, 1, C)."""
    if t.dim() == 5:
        return t.permute(0, 2, 3, 4, 1).flatten(0, 1)
    if t.dim() == 4:
        return t.permute(0, 2, 3, 1)
    return t.unsqueeze(1) if t.dim() == 3 else t[:, None, None]


def capture(model, names, run, post=None, fault=None, pad=None):
    """Run ``run()`` with forward hooks on every module of ``names``: {name: its output in tap layout}.  post: {name: f} applied to the
    module output to make the tap (the SiLU after a conv or GroupNorm).  fault: (module name, f): that module's output is replaced by
    f(output) in the forward itself.  pad: {name: C}: the tap is zero-padded to C channels, as the native layout holds it.

    Every tapped module gets its inputs contiguous, as the replay hands them over: some oracle blocks return a channels-last strided
    tensor (the VAE attention's transpose), and a conv of the same values in another memory layout rounds differently in the last bit."""
    mods = dict(model.named_modules())
    post, pad = post or {}, pad or {}
    taps, hooks = {}, []

    def hook(name):
        def fn(mod, inp, out):
            if fault is not None and fault[0] == name:
                out = fault[1](out)
            t = nhwc(post.get(name, lambda x: x)(out)).contiguous()
            if name in pad:
                t = F.pad(t, (0, pad[name] - t.shape[-1]))
            if name in names:
                taps[name] = t
            return out
        return fn

    def contiguous(mod, args):
        return tuple(a.contiguous() if torch.is_tensor(a) else a for a in args)

    for n in set(names) | ({fault[0]} if fault else set()):
        hooks.append(mods[n].register_forward_hook(hook(n)))
    hooks += [mods[n].register_forward_pre_hook(contiguous) for n in names]
    try:
        with torch.no_grad():
            result = run()
    finally:
        for h in hooks:
            h.remove()
    assert set(taps) == set(names), f"never ran: {set(names) - set(taps)}"
    return taps, result


def replayed(replay, names, taps):
    """{name: replayed output}, and the replay's names in order must be the plan's."""
    out = {n: o.contiguous() for n, o in replay(taps)}
    assert list(out) == list(names)
    return out


def flagged(names, taps, reps):
    """The blocks the checks flag: each replayed block against its tap as N, R (no fp16 eager leg), padding channels included."""
    bad = []
    for n in names:
        rep = BlockReport()
        r = reps[n]
        check_fp16_block(rep, n, taps[n][..., : r.shape[-1]], r)
        check_pad(rep, n, taps[n], r.shape[-1])
        if rep.failures(with_eager=False):
            bad.append(n)
    return bad


def assert_exact(names, taps, reps):
    for n in names:
        c = reps[n].shape[-1]
        assert torch.equal(reps[n], taps[n][..., :c]), f"{n}: replay differs from the forward's own output"
        assert not taps[n][..., c:].any()


# ------------------------------------------------------------------------------------------------ networks
def vae():
    return O.synthetic_init(V.AutoencoderKL(block_out_channels=(32, 32, 64, 64), norm_num_groups=8).eval(), seed=1).to(DT)


def clip():
    cfg = transformers.CLIPVisionConfig(hidden_size=64, intermediate_size=128, projection_dim=32, num_hidden_layers=2, num_attention_heads=2,
                                        image_size=32, patch_size=8, attn_implementation="eager")
    torch.manual_seed(3)
    return transformers.CLIPVisionModelWithProjection(cfg).eval().to(DT)


def pose_guider():
    return O.synthetic_init(O.PoseGuider(32, 3, (16, 32, 96, 256)).eval(), seed=4).to(DT)


def camera():
    return O.synthetic_init(O.CameraPoseEncoder(channels=(64,), heads=8).eval(), seed=5).to(DT)


def rnd(*shape, seed=0):
    return torch.randn(*shape, generator=torch.Generator().manual_seed(seed), dtype=DT)


VAE_POST = {"decoder.conv_norm_out": F.silu, "encoder.conv_norm_out": F.silu}
VAE_PAD = {"post_quant_conv": 64, "decoder.conv_out": 8}     # the native layouts: post_quant_conv's 64-channel conv_in input, 3 -> 8


def swap_groups(c_per_group):
    """GroupNorm output with the channels of groups 0 and 1 exchanged."""
    def f(out):
        out = out.clone()
        g = c_per_group
        out[:, :g], out[:, g : 2 * g] = out[:, g : 2 * g].clone(), out[:, :g].clone()
        return out
    return f


def frame_copied(dst, src):
    def f(out):
        out = out.clone()
        out[dst] = out[src]
        return out
    return f


# ------------------------------------------------------------------------------------------------ the replays are exact
def run_vae_decode(m, z, fault=None):
    names = vae_tap_names(m, "decoder")
    taps, y = capture(m, names, lambda: m.decode(z).sample, VAE_POST, fault, VAE_PAD)
    return names, taps, y, replayed(lambda t: replay_vae(m, names, t, z), names, taps)


def run_vae_encode(m, x, fault=None):
    names = vae_tap_names(m, "encoder")
    taps, y = capture(m, names, lambda: m.moments(x), VAE_POST, fault)
    return names, taps, y, replayed(lambda t: replay_vae(m, names, t, x), names, taps)


def run_clip(m, pix, fault=None):
    names = clip_tap_names(m)
    taps, y = capture(m, names, lambda: m(pix), fault=fault)
    return names, taps, y, replayed(lambda t: replay_clip(m, names, t, pix), names, taps)


def run_pose_guider(m, cond, fault=None):
    names = pose_guider_tap_names(m)
    post = {n: F.silu for n in names if n != "conv_out"}
    taps, y = capture(m, names, lambda: m(cond), post, fault, {"blocks.3": 128, "blocks.4": 128, "conv_out": 32})
    return names, taps, y, replayed(lambda t: replay_pose_guider(m, names, t, cond), names, taps)


def run_camera(m, x, fault=None):
    names = camera_tap_names(m)
    b, _, f, H, W = x.shape
    h, w = H // 8, W // 8
    # an attention block's output is (b h w, f, c): the tap is (b f, h, w, c)
    post = {n: lambda t: t.reshape(b, h, w, f, -1).permute(0, 3, 4, 1, 2).flatten(0, 1) for n in names if "attention" in n}
    taps, y = capture(m, names, lambda: m(x)[0], post, fault)
    return names, taps, y, replayed(lambda t: replay_camera(m, names, t, x), names, taps)


def test_vae_decode_replay_is_exact():
    m = vae()
    z = rnd(2, 4, 5, 3)                     # odd latent sides
    names, taps, y, reps = run_vae_decode(m, z)
    assert names[0] == "post_quant_conv" and names[-1] == "decoder.conv_out" and len(names) == 22
    assert_exact(names, taps, reps)
    assert torch.equal(reps[names[-1]], nhwc(y))


def test_vae_encode_replay_is_exact():
    m = vae()
    x = rnd(2, 3, 16, 24, seed=1)
    names, taps, y, reps = run_vae_encode(m, x)
    assert names[0] == "encoder.conv_in" and names[-1] == "quant_conv" and len(names) == 18
    assert_exact(names, taps, reps)
    assert torch.equal(reps[names[-1]], nhwc(y))


def test_clip_replay_is_exact():
    m = clip()
    pix = rnd(2, 3, 32, 32, seed=2)
    names, taps, y, reps = run_clip(m, pix)
    assert_exact(names, taps, reps)
    assert torch.equal(reps[names[-2]][:, 0], y.last_hidden_state)
    assert torch.equal(m.visual_projection(reps[names[-1]][:, 0, 0]), y.image_embeds)


def test_pose_guider_replay_is_exact():
    m = pose_guider()
    cond = rnd(1, 3, 2, 32, 24, seed=3)
    names, taps, y, reps = run_pose_guider(m, cond)
    assert_exact(names, taps, reps)
    assert torch.equal(reps["conv_out"], nhwc(y))


def test_camera_replay_is_exact():
    m = camera()
    x = rnd(1, 6, 4, 32, 24, seed=4)
    names, taps, y, reps = run_camera(m, x)
    assert names == ["encoder_conv_in", "encoder_down_conv_blocks.0.0", "encoder_down_attention_blocks.0.0", "encoder_down_conv_blocks.0.1",
                     "encoder_down_attention_blocks.0.1", "zero_conv_layers.0"]
    assert_exact(names, taps, reps)
    assert torch.equal(reps[names[-1]], nhwc(y))


# ------------------------------------------------------------------------------------------------ one fault, one flagged block
def test_vae_decode_swapped_groupnorm_group_is_flagged():
    m = vae()
    z = rnd(2, 4, 5, 3)
    blk = "decoder.up_blocks.1.resnets.2"
    names, taps, _, reps = run_vae_decode(m, z, fault=(blk + ".norm2", swap_groups(64 // 8)))
    assert flagged(names, taps, reps) == [blk]


def test_vae_encode_frame_replaced_is_flagged():
    m = vae()
    x = rnd(2, 3, 16, 24, seed=1)
    blk = "encoder.down_blocks.1.resnets.0"
    names, taps, _, reps = run_vae_encode(m, x, fault=(blk, frame_copied(1, 0)))
    assert flagged(names, taps, reps) == [blk]


def test_vae_nonzero_pad_channel_is_flagged():
    m = vae()
    z = rnd(2, 4, 5, 3)
    names, taps, _, reps = run_vae_decode(m, z)
    taps["post_quant_conv"][1, 4, 2, 63] = float("nan")
    assert flagged(names, taps, reps) == ["post_quant_conv"]
    taps["post_quant_conv"][1, 4, 2, 63] = -0.0          # -0 is zero
    assert flagged(names, taps, reps) == []


def test_pose_guider_nonzero_pad_channel_is_flagged():
    m = pose_guider()
    cond = rnd(1, 3, 2, 32, 24, seed=3)
    names, taps, _, reps = run_pose_guider(m, cond)
    taps["blocks.3"][0, 0, 0, 100] = 2.0 ** -14             # one padding channel of the small-channel layer's 128-wide output
    assert flagged(names, taps, reps) == ["blocks.3"]


def test_camera_frame_replaced_is_flagged():
    m = camera()
    x = rnd(1, 6, 4, 32, 24, seed=4)
    blk = "encoder_down_attention_blocks.0.0"
    # the attention block's output is (b h w, f, c): frame 3 of every pixel replaced by frame 2
    def f(out):
        out = out.clone()
        out[:, 3] = out[:, 2]
        return out
    names, taps, _, reps = run_camera(m, x, fault=(blk, f))
    assert flagged(names, taps, reps) == [blk]


def test_clip_scaled_token_row_is_flagged():
    m = clip()
    pix = rnd(2, 3, 32, 32, seed=2)
    blk = "vision_model.encoder.layers.0"

    def f(out):
        out = out.clone()
        out[1, 5] *= 1 + 2.0 ** -5
        return out
    names, taps, _, reps = run_clip(m, pix, fault=(blk, f))
    assert flagged(names, taps, reps) == [blk]
    rep = BlockReport()
    check_fp16_block(rep, blk, taps[blk], reps[blk])
    assert rep.row.ratio > 1.0 and rep.row.where[1:3] == (1, 5)


def test_block_kinds():
    kinds = {"post_quant_conv": "conv1x1", "decoder.conv_in": "conv_in", "decoder.mid_block.attentions.0": "attentions",
             "decoder.up_blocks.2.upsamplers.0": "upsamplers", "decoder.conv_norm_out": "norm_out", "decoder.conv_out": "conv_out",
             "encoder.down_blocks.0.downsamplers.0": "downsamplers", "quant_conv": "conv1x1", "vision_model.pre_layrnorm": "clip_embed",
             "vision_model.encoder.layers.11": "clip_layer", "vision_model.post_layernorm": "clip_pool", "conv_in": "conv_in", "blocks.5": "pg_conv",
             "conv_out": "conv_out", "encoder_conv_in": "conv_in", "encoder_down_conv_blocks.0.1": "cam_res",
             "encoder_down_attention_blocks.0.1": "cam_attn", "zero_conv_layers.0": "conv1x1", "up_blocks.1.motion_modules.2": "motion_modules"}
    assert {n: block_kind(n) for n in kinds} == kinds
