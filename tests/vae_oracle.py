"""PyTorch restatement of diffusers 0.24 ``AutoencoderKL`` (KL VAE of Stable Diffusion).  TEST INFRASTRUCTURE ONLY.

The pipelines make the reference latents with ``vae.encode(x).latent_dist.mean`` and the frames with ``vae.decode(z).sample``; this module
restates both with plain torch ops, under diffusers' module tree and state_dict key names, for the layout configs/prompts/stage2.yaml
points at (sd-vae-ft-mse: block_out_channels (128, 256, 512, 512), layers_per_block 2, 32 groups, 4 latent channels).  Like the other
diffusers primitives of oracle/hv_oracle.py it is "unpinned" (diffusers is not installed); tests/test_thirdparty_vae_port_cpu.py checks it
against an independent port of the same LDM architecture.  ``humanvid_b200`` never imports it.

  ResnetBlock2D (temb_channels=None)  GroupNorm(eps 1e-6) -> SiLU -> conv3x3 -> GroupNorm -> SiLU -> conv3x3, + x (1x1 conv_shortcut when
                                      the channel count changes)
  Attention (mid block)               group_norm(eps 1e-6) -> to_q / to_k / to_v (bias) -> one head, softmax(q k^T / sqrt(C)) v ->
                                      to_out.0 (bias) -> + x
  Downsample2D                        F.pad(x, (0, 1, 0, 1)) -> conv3x3 stride 2, padding 0
  Upsample2D                          nearest 2x -> conv3x3
"""
from __future__ import annotations

from types import SimpleNamespace
from typing import Sequence

import torch
import torch.nn as nn
import torch.nn.functional as F


class ResnetBlock2D(nn.Module):
    def __init__(self, cin: int, cout: int, groups: int = 32, eps: float = 1e-6):
        super().__init__()
        self.norm1 = nn.GroupNorm(groups, cin, eps=eps)
        self.conv1 = nn.Conv2d(cin, cout, 3, padding=1)
        self.norm2 = nn.GroupNorm(groups, cout, eps=eps)
        self.conv2 = nn.Conv2d(cout, cout, 3, padding=1)
        self.conv_shortcut = nn.Conv2d(cin, cout, 1) if cin != cout else None

    def forward(self, x):
        h = self.conv1(F.silu(self.norm1(x)))
        h = self.conv2(F.silu(self.norm2(h)))
        if self.conv_shortcut is not None:
            x = self.conv_shortcut(x)
        return x + h


class Attention(nn.Module):
    """diffusers Attention(query_dim=C, heads=1, dim_head=C, norm_num_groups=32, residual_connection=True, bias=True, upcast_softmax=True)."""

    def __init__(self, ch: int, groups: int = 32):
        super().__init__()
        self.group_norm = nn.GroupNorm(groups, ch, eps=1e-6)
        self.to_q = nn.Linear(ch, ch)
        self.to_k = nn.Linear(ch, ch)
        self.to_v = nn.Linear(ch, ch)
        self.to_out = nn.ModuleList([nn.Linear(ch, ch), nn.Dropout(0.0)])

    def forward(self, x):
        b, c, h, w = x.shape
        t = self.group_norm(x).view(b, c, h * w).transpose(1, 2)
        q, k, v = self.to_q(t), self.to_k(t), self.to_v(t)
        o = F.scaled_dot_product_attention(q[:, None], k[:, None], v[:, None])[:, 0]   # AttnProcessor2_0, one head
        o = self.to_out[0](o)
        return o.transpose(1, 2).reshape(b, c, h, w) + x


class Downsample2D(nn.Module):
    def __init__(self, ch: int):
        super().__init__()
        self.conv = nn.Conv2d(ch, ch, 3, stride=2, padding=0)

    def forward(self, x):
        return self.conv(F.pad(x, (0, 1, 0, 1)))


class Upsample2D(nn.Module):
    def __init__(self, ch: int):
        super().__init__()
        self.conv = nn.Conv2d(ch, ch, 3, padding=1)

    def forward(self, x):
        return self.conv(F.interpolate(x, scale_factor=2.0, mode="nearest"))


class DownEncoderBlock2D(nn.Module):
    def __init__(self, cin, cout, layers, groups, add_downsample):
        super().__init__()
        self.resnets = nn.ModuleList([ResnetBlock2D(cin if j == 0 else cout, cout, groups) for j in range(layers)])
        self.downsamplers = nn.ModuleList([Downsample2D(cout)]) if add_downsample else None

    def forward(self, x):
        for r in self.resnets:
            x = r(x)
        if self.downsamplers is not None:
            x = self.downsamplers[0](x)
        return x


class UpDecoderBlock2D(nn.Module):
    def __init__(self, cin, cout, layers, groups, add_upsample):
        super().__init__()
        self.resnets = nn.ModuleList([ResnetBlock2D(cin if j == 0 else cout, cout, groups) for j in range(layers)])
        self.upsamplers = nn.ModuleList([Upsample2D(cout)]) if add_upsample else None

    def forward(self, x):
        for r in self.resnets:
            x = r(x)
        if self.upsamplers is not None:
            x = self.upsamplers[0](x)
        return x


class UNetMidBlock2D(nn.Module):
    def __init__(self, ch, groups):
        super().__init__()
        self.attentions = nn.ModuleList([Attention(ch, groups)])
        self.resnets = nn.ModuleList([ResnetBlock2D(ch, ch, groups), ResnetBlock2D(ch, ch, groups)])

    def forward(self, x):
        x = self.resnets[0](x)
        x = self.attentions[0](x)
        return self.resnets[1](x)


class Encoder(nn.Module):
    def __init__(self, cin, ch: Sequence[int], latent, layers, groups):
        super().__init__()
        self.conv_in = nn.Conv2d(cin, ch[0], 3, padding=1)
        self.down_blocks = nn.ModuleList([DownEncoderBlock2D(ch[max(i - 1, 0)], c, layers, groups, i < len(ch) - 1) for i, c in enumerate(ch)])
        self.mid_block = UNetMidBlock2D(ch[-1], groups)
        self.conv_norm_out = nn.GroupNorm(groups, ch[-1], eps=1e-6)
        self.conv_out = nn.Conv2d(ch[-1], 2 * latent, 3, padding=1)

    def forward(self, x):
        x = self.conv_in(x)
        for b in self.down_blocks:
            x = b(x)
        x = self.mid_block(x)
        return self.conv_out(F.silu(self.conv_norm_out(x)))


class Decoder(nn.Module):
    def __init__(self, cout, ch: Sequence[int], latent, layers, groups):
        super().__init__()
        rev = list(ch)[::-1]
        self.conv_in = nn.Conv2d(latent, rev[0], 3, padding=1)
        self.mid_block = UNetMidBlock2D(rev[0], groups)
        self.up_blocks = nn.ModuleList([UpDecoderBlock2D(rev[max(i - 1, 0)], c, layers + 1, groups, i < len(rev) - 1) for i, c in enumerate(rev)])
        self.conv_norm_out = nn.GroupNorm(groups, ch[0], eps=1e-6)
        self.conv_out = nn.Conv2d(ch[0], cout, 3, padding=1)

    def forward(self, z):
        x = self.mid_block(self.conv_in(z))
        for b in self.up_blocks:
            x = b(x)
        return self.conv_out(F.silu(self.conv_norm_out(x)))


class AutoencoderKL(nn.Module):
    def __init__(self, in_channels=3, out_channels=3, block_out_channels=(128, 256, 512, 512), layers_per_block=2, latent_channels=4,
                 norm_num_groups=32, scaling_factor=0.18215):
        super().__init__()
        self.config = SimpleNamespace(in_channels=in_channels, out_channels=out_channels, block_out_channels=tuple(block_out_channels),
                                      layers_per_block=layers_per_block, latent_channels=latent_channels, norm_num_groups=norm_num_groups,
                                      scaling_factor=scaling_factor)
        self.encoder = Encoder(in_channels, block_out_channels, latent_channels, layers_per_block, norm_num_groups)
        self.decoder = Decoder(out_channels, block_out_channels, latent_channels, layers_per_block, norm_num_groups)
        self.quant_conv = nn.Conv2d(2 * latent_channels, 2 * latent_channels, 1)
        self.post_quant_conv = nn.Conv2d(latent_channels, latent_channels, 1)

    def moments(self, x):
        return self.quant_conv(self.encoder(x))

    def encode(self, x):
        m = self.moments(x)
        mean, logvar = torch.chunk(m, 2, dim=1)
        return SimpleNamespace(latent_dist=SimpleNamespace(mean=mean, logvar=logvar))

    def decode(self, z):
        return SimpleNamespace(sample=self.decoder(self.post_quant_conv(z)))


def decode_flops(n: int, h: int, w: int, ch=(128, 256, 512, 512), latent=4, out_ch=3, layers=2) -> float:
    """Algorithmic FLOPs (2 x multiply-adds; convolutions, linears and attention) of decoding n latents of h x w."""
    rev = list(ch)[::-1]
    f = 2.0 * h * w * latent * latent                      # post_quant_conv
    f += 2.0 * h * w * 9 * latent * rev[0]                 # conv_in
    f += _mid_flops(h, w, rev[0])
    H, W, cin = h, w, rev[0]
    for i, c in enumerate(rev):
        for j in range(layers + 1):
            f += _resnet_flops(H, W, cin if j == 0 else c, c)
        cin = c
        if i < len(rev) - 1:
            H, W = 2 * H, 2 * W
            f += 2.0 * H * W * 9 * c * c                   # Upsample2D conv (on the upsampled grid, as the library computes it)
    f += 2.0 * H * W * 9 * ch[0] * out_ch                  # conv_out
    return n * f


def encode_flops(n: int, H: int, W: int, ch=(128, 256, 512, 512), latent=4, in_ch=3, layers=2) -> float:
    """Algorithmic FLOPs of encoding n images of H x W."""
    f = 2.0 * H * W * 9 * in_ch * ch[0]
    cin = ch[0]
    for i, c in enumerate(ch):
        for j in range(layers):
            f += _resnet_flops(H, W, cin if j == 0 else c, c)
        cin = c
        if i < len(ch) - 1:
            H, W = H // 2, W // 2
            f += 2.0 * H * W * 9 * c * c
    f += _mid_flops(H, W, ch[-1])
    f += 2.0 * H * W * 9 * ch[-1] * 2 * latent + 2.0 * H * W * (2 * latent) ** 2
    return n * f


def _resnet_flops(H, W, cin, cout):
    f = 2.0 * H * W * 9 * (cin * cout + cout * cout)
    if cin != cout:
        f += 2.0 * H * W * cin * cout
    return f


def _mid_flops(H, W, c):
    L = H * W
    return 2 * _resnet_flops(H, W, c, c) + 2.0 * L * 4 * c * c + 4.0 * L * L * c
