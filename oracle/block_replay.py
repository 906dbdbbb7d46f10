"""Isolated per-block replay of the oracle networks on the native forward's own activations.  TEST INFRASTRUCTURE ONLY.

Every native network copies the activation leaving each block out through its debug taps (``debug_tap_plan`` / ``debug_set_taps``): one
channels-last (B*F, H, W, C) fp16 tensor per block, in execution order, C including any zero padding channels.  ``replay_blocks`` (the
UNets), ``replay_vae``, ``replay_clip``, ``replay_pose_guider`` and ``replay_camera`` apply the oracle module of the same name to the native
taps of that block's predecessors -- the input the native block itself consumed -- so the difference between its result and the native tap
is the error that block adds by itself, free of what its input already carried.  The replays yield (name, out) with out in tap layout at
the block's true channel width; a predecessor's tap is read at the width of the predecessor's replayed output, so padding channels never
reach the oracle.

The oracle runs in its own dtype (fp16, fp32 or fp64: whatever ``unet`` holds), so the same replay gives an fp64 reference, the
reference's fp16 deployment and, under ``tests/fp8_emulation.emulate_fp8_linears``, the e4m3 emulation.  Reference banks set with
``set_reference_banks`` (or the write hook of ``set_reference_write``) are bound to their blocks and act during the replay as they do in a
whole forward; the caller sets them in the oracle's dtype.
"""
from __future__ import annotations

from typing import Dict, Iterator, List, Optional, Sequence, Tuple

import torch
import torch.nn.functional as F

from oracle import hv_oracle as O


def to_nhwc(t: torch.Tensor) -> torch.Tensor:
    """(B, C, F, H, W) -> (B*F, H, W, C), the layout of a native tap."""
    b, c, f, h, w = t.shape
    return t.permute(0, 2, 3, 4, 1).reshape(b * f, h, w, c)


def to_ncfhw(t: torch.Tensor, B: int, dtype: torch.dtype) -> torch.Tensor:
    """A native tap (B*F, H, W, C) -> (B, C, F, H, W) in dtype."""
    nf, h, w, c = t.shape
    return t.reshape(B, nf // B, h, w, c).permute(0, 4, 1, 2, 3).to(dtype).contiguous()


def skip_stack(names: Sequence[str]) -> List[str]:
    """The taps the up-path resnets concatenate, in push order (unet_3d.py:486-506): conv_in, then the last module of every down layer,
    then each down block's downsampler."""
    skips = ["conv_in"]
    for n in names:
        if n.startswith("down_blocks"):
            kind = n.rsplit(".", 2)[1]
            if kind in ("downsamplers", "resnets"):
                skips.append(n)      # a resnet entry is provisional: the layer's later modules replace it below
            else:
                skips[-1] = n        # attentions.j / motion_modules.j follow resnets.j of the same layer
    return skips


def replay_blocks(unet: O.UNet3DConditionModel, names: Sequence[str], native: Dict[str, torch.Tensor], sample: torch.Tensor, timestep: int,
                  ehs: torch.Tensor, pose: Optional[torch.Tensor] = None) -> Iterator[Tuple[str, torch.Tensor]]:
    """For every tap in ``names`` (execution order), yield (name, out): the oracle module ``name`` applied, in the oracle's dtype, to the
    native taps of its predecessors (for an up-path resnet, the previous tap concatenated with its skip tap), out as (B*F, H, W, C).
    ``conv_in`` takes ``sample`` (B, C, F, H, W) -- or (B, C, H, W) for the 2-D UNet -- plus ``pose``.

    ``unet`` is an oracle UNet3DConditionModel (any layout) or UNet2DConditionModel; ``native`` maps each name to its tap."""
    dt = unet.conv_in.weight.dtype
    x = sample if sample.dim() == 5 else sample.unsqueeze(2)
    B = x.shape[0]
    mods = dict(unet.named_modules())
    with torch.no_grad():
        tt = torch.tensor([timestep], device=x.device).expand(B)
        emb = unet.time_embedding(O.timestep_sincos(tt, unet.conv_in.out_channels).to(dt))
        e = ehs.to(dt)
        h0 = unet.conv_in(x.to(dt))
        if pose is not None:
            h0 = h0 + pose.to(dt)
        yield "conv_in", to_nhwc(h0)
        del h0
        skips = skip_stack(names)
        prev = "conv_in"
        for n in names[1:]:
            kind = n.split(".")[-2]
            ins = (to_ncfhw(native[prev], B, dt),)
            if n.startswith("up_blocks") and kind == "resnets":
                ins = ins + (to_ncfhw(native[skips.pop()], B, dt),)
            m = mods[n]
            if kind == "resnets":
                out = m(torch.cat(ins, dim=1), emb)
            elif kind == "attentions":
                out = m(ins[0], e)
            elif kind == "upsamplers":
                out = m(ins[0], None)
            else:   # motion_modules, downsamplers
                out = m(ins[0])
            yield n, to_nhwc(out)
            del out, ins
            prev = n
        assert not skips, f"skip tensors left unconsumed: {skips}"


# --------------------------------------------------------------------------------------------- the other networks
def _nchw(t: torch.Tensor, c: int, dtype: torch.dtype) -> torch.Tensor:
    """A native tap (NF, H, W, C >= c) -> its first c channels as (NF, c, H, W) in dtype."""
    return t[..., :c].permute(0, 3, 1, 2).to(dtype).contiguous()


def _chain(names: Sequence[str], native: Dict[str, torch.Tensor], dt: torch.dtype, first: torch.Tensor, step) -> Iterator[Tuple[str, torch.Tensor]]:
    """The replay of a network whose blocks run one after another: block 0 takes ``first``, block i the native tap of block i - 1 (at the
    width of block i - 1's replayed output); step(name, x) applies block ``name`` to x (NF, C, H, W) and returns its output the same way."""
    x = first.to(dt)
    for i, n in enumerate(names):
        out = step(n, x)
        yield n, out.permute(0, 2, 3, 1)
        if i + 1 < len(names):
            x = _nchw(native[n], out.shape[1], dt)
        del out


def replay_vae(vae, names: Sequence[str], native: Dict[str, torch.Tensor], inp: torch.Tensor) -> Iterator[Tuple[str, torch.Tensor]]:
    """An AutoencoderKL (tests/vae_oracle.py, or anything with diffusers' module tree) on the native taps of one decode or one encode:
    ``names`` are the decoder's taps (inp = the latents z, (N, 4, h, w), as post_quant_conv takes them) or the encoder's (inp = the images,
    (N, 3, H, W), as encoder.conv_in takes them).  conv_norm_out is GroupNorm then SiLU, as the native tap holds it."""
    mods = dict(vae.named_modules())

    def step(n, x):
        out = mods[n](x)
        return F.silu(out) if n.endswith("conv_norm_out") else out

    with torch.no_grad():
        yield from _chain(names, native, vae.post_quant_conv.weight.dtype, inp, step)


def replay_pose_guider(pg, names: Sequence[str], native: Dict[str, torch.Tensor], cond: torch.Tensor) -> Iterator[Tuple[str, torch.Tensor]]:
    """A PoseGuider (oracle/hv_oracle.py: InflatedConv3d layers over (b, c, f, h, w)) on the native taps: conv_in takes the conditioning
    image ``cond`` (B, 3, F, H, W); every conv but conv_out is followed by SiLU."""
    mods = dict(pg.named_modules())

    def step(n, x):   # the frames of x as the f axis of one batch item
        out = mods[n](x.transpose(0, 1).unsqueeze(0))[0].transpose(0, 1)
        return out if n == "conv_out" else F.silu(out)

    b, c, f, h, w = cond.shape
    with torch.no_grad():
        yield from _chain(names, native, pg.conv_in.weight.dtype, cond.transpose(1, 2).reshape(b * f, c, h, w), step)


def replay_camera(cam, names: Sequence[str], native: Dict[str, torch.Tensor], plucker: torch.Tensor) -> Iterator[Tuple[str, torch.Tensor]]:
    """A CameraPoseEncoder (oracle/hv_oracle.py) on the native taps: encoder_conv_in takes PixelUnshuffle of the plücker map ``plucker``
    (B, 6, F, H, W); an attention block runs over the frames of each pixel, on the (b h w, f, c) reshape of the oracle's forward."""
    mods = dict(cam.named_modules())
    b, c, f, h, w = plucker.shape

    def step(n, x):
        if n == "encoder_conv_in":
            return mods[n](cam.unshuffle(x))
        if n.startswith("encoder_down_attention_blocks"):
            nf, ch, hh, ww = x.shape
            t = mods[n](x.reshape(b, f, ch, hh, ww).permute(0, 3, 4, 1, 2).reshape(b * hh * ww, f, ch))
            return t.reshape(b, hh, ww, f, ch).permute(0, 3, 4, 1, 2).reshape(nf, ch, hh, ww)
        return mods[n](x)

    with torch.no_grad():
        yield from _chain(names, native, cam.encoder_conv_in.weight.dtype, plucker.transpose(1, 2).reshape(b * f, c, h, w), step)


def replay_clip(clip, names: Sequence[str], native: Dict[str, torch.Tensor], pixels: torch.Tensor) -> Iterator[Tuple[str, torch.Tensor]]:
    """A CLIPVisionModelWithProjection (transformers' module tree, eager attention) on the native taps, which hold the residual stream of
    image i as slice i, (B, 1, L, C): vision_model.pre_layrnorm is the embeddings + pre-LN of ``pixels`` (B, 3, S, S), a layer is called as
    ``layer(h, None)``, vision_model.post_layernorm takes the class token of the last layer's tap and holds (B, 1, 1, C)."""
    vm = clip.vision_model
    mods = dict(clip.named_modules())
    dt = vm.pre_layrnorm.weight.dtype
    with torch.no_grad():
        for i, n in enumerate(names):
            if i == 0:
                assert n == "vision_model.pre_layrnorm", n
                out = vm.pre_layrnorm(vm.embeddings(pixels.to(dt)))
            else:
                h = native[names[i - 1]][:, 0].to(dt)
                out = vm.post_layernorm(h[:, :1]) if n == "vision_model.post_layernorm" else mods[n](h, None)
            yield n, out.unsqueeze(1)
            del out


# --------------------------------------------------------------------------------------------- the tap plans, from the module trees
def vae_tap_names(vae, half: str) -> List[str]:
    """The taps of one decode (half = "decoder") or encode ("encoder"), in execution order, named from an AutoencoderKL's module tree."""
    d = getattr(vae, half)
    names = ["post_quant_conv"] if half == "decoder" else []
    names.append(f"{half}.conv_in")
    mid = [f"{half}.mid_block.resnets.0", f"{half}.mid_block.attentions.0", f"{half}.mid_block.resnets.1"]
    blocks = []
    kind = "up_blocks" if half == "decoder" else "down_blocks"
    for i, b in enumerate(getattr(d, kind)):
        blocks += [f"{half}.{kind}.{i}.resnets.{j}" for j in range(len(b.resnets))]
        sampler = "upsamplers" if half == "decoder" else "downsamplers"
        if getattr(b, sampler, None) is not None:
            blocks.append(f"{half}.{kind}.{i}.{sampler}.0")
    names += mid + blocks if half == "decoder" else blocks + mid
    names += [f"{half}.conv_norm_out", f"{half}.conv_out"]
    return names + (["quant_conv"] if half == "encoder" else [])


def clip_tap_names(clip) -> List[str]:
    n = len(clip.vision_model.encoder.layers)
    return ["vision_model.pre_layrnorm"] + [f"vision_model.encoder.layers.{i}" for i in range(n)] + ["vision_model.post_layernorm"]


def pose_guider_tap_names(pg) -> List[str]:
    return ["conv_in"] + [f"blocks.{k}" for k in range(len(pg.blocks))] + ["conv_out"]


def camera_tap_names(cam) -> List[str]:
    n = len(cam.encoder_down_conv_blocks[0])
    pairs = [f"{kind}.0.{j}" for j in range(n) for kind in ("encoder_down_conv_blocks", "encoder_down_attention_blocks")]
    return ["encoder_conv_in"] + pairs + ["zero_conv_layers.0"]
