"""Isolated per-block replay of the oracle UNets on the native forward's own activations.  TEST INFRASTRUCTURE ONLY.

The native UNet copies the activation leaving each block out through its debug taps (``debug_tap_plan`` / ``debug_set_taps``): one
channels-last (B*F, H, W, C) fp16 tensor per resnet, transformer, motion module and sampler, in execution order.  ``replay_blocks`` applies
the oracle module of the same name to the native taps of that block's predecessors -- the input the native block itself consumed -- so the
difference between its result and the native tap is the error that block adds by itself, free of what its input already carried.

The oracle runs in its own dtype (fp16, fp32 or fp64: whatever ``unet`` holds), so the same replay gives an fp64 reference, the
reference's fp16 deployment and, under ``tests/fp8_emulation.emulate_fp8_linears``, the e4m3 emulation.  Reference banks set with
``set_reference_banks`` (or the write hook of ``set_reference_write``) are bound to their blocks and act during the replay as they do in a
whole forward; the caller sets them in the oracle's dtype.
"""
from __future__ import annotations

from typing import Dict, Iterator, List, Optional, Sequence, Tuple

import torch

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
