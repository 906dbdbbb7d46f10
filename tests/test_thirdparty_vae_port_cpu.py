"""Third-party cross-check of the AutoencoderKL restatement (tests/vae_oracle.py; diffusers is not installed, so it is "unpinned").

torchtitan's Flux autoencoder (``torchtitan.experiments.flux.model.autoencoder``) is a port of the same LDM KL-autoencoder by a different
hand.  ``Encoder`` / ``Decoder`` with ch = 32, ch_mult = (1, 2, 2, 2), 2 resnets per level and 4 latent channels is the SD layout at a
quarter of the width.  That port has no quant_conv / post_quant_conv; the oracle's are applied around it.  The weights are mapped with the
standard LDM <-> diffusers conversion and the encoder moments and the decoder output must agree in fp32.  Skipped when torchtitan is not
importable.
"""
import pytest
import torch

import vae_oracle as V
from oracle import hv_oracle as O


def _port():
    try:
        from torchtitan.experiments.flux.model import autoencoder as A
    except Exception as e:  # pragma: no cover
        pytest.skip(f"torchtitan's Flux autoencoder is not importable: {e}")
    return A


_ATTN = {"norm": "group_norm", "q": "to_q", "k": "to_k", "v": "to_v", "proj_out": "to_out.0"}


def ldm_to_diffusers(key: str) -> str:
    """One key of the LDM (torchtitan) encoder / decoder state_dict -> its diffusers name (both prefixed with encoder. / decoder.)."""
    p = key.split(".")
    half, rest = p[0], p[1:]
    if rest[0] == "down":          # down.i.block.j.* / down.i.downsample.conv.*
        i = rest[1]
        if rest[2] == "block":
            tail = ["down_blocks", i, "resnets", rest[3]] + rest[4:]
        else:
            tail = ["down_blocks", i, "downsamplers", "0"] + rest[3:]
    elif rest[0] == "up":          # up.i.block.j.* / up.i.upsample.conv.*  (up.i is the level i from the top: up_blocks.(3 - i))
        i = str(3 - int(rest[1]))
        if rest[2] == "block":
            tail = ["up_blocks", i, "resnets", rest[3]] + rest[4:]
        else:
            tail = ["up_blocks", i, "upsamplers", "0"] + rest[3:]
    elif rest[0] == "mid":
        if rest[1] in ("block_1", "block_2"):
            tail = ["mid_block", "resnets", "0" if rest[1] == "block_1" else "1"] + rest[2:]
        else:                      # attn_1.{norm,q,k,v,proj_out}.*
            tail = ["mid_block", "attentions", "0"] + _ATTN[rest[2]].split(".") + rest[3:]
    elif rest[0] == "norm_out":
        tail = ["conv_norm_out"] + rest[1:]
    else:                          # conv_in, conv_out
        tail = rest
    return ".".join([half] + tail).replace("nin_shortcut", "conv_shortcut")


def _ported_pair(seed=5):
    A = _port()
    ch, mult = 32, (1, 2, 2, 2)
    ora = O.synthetic_init(V.AutoencoderKL(block_out_channels=[ch * m for m in mult]).eval(), seed=seed)
    enc = A.Encoder(resolution=64, in_channels=3, ch=ch, ch_mult=mult, num_res_blocks=2, z_channels=4).eval()
    dec = A.Decoder(ch=ch, out_ch=3, ch_mult=mult, num_res_blocks=2, in_channels=3, resolution=64, z_channels=4).eval()
    sd = ora.state_dict()
    for half, mod in (("encoder", enc), ("decoder", dec)):
        own = mod.state_dict()
        mapped = {}
        for k, v in own.items():
            src = sd[ldm_to_diffusers(f"{half}.{k}")]
            mapped[k] = src.reshape(v.shape)    # the port's attention projections are 1x1 convs, diffusers' are linears
        mod.load_state_dict(mapped)
    n_ours = sum(1 for k in sd if not k.startswith(("quant_conv", "post_quant_conv")))
    assert n_ours == len(enc.state_dict()) + len(dec.state_dict())   # every parameter of the oracle is covered by exactly one of the port's
    return ora, enc, dec


def test_key_mapping_is_a_bijection():
    ora, enc, dec = _ported_pair()
    names = [ldm_to_diffusers(f"encoder.{k}") for k in enc.state_dict()] + [ldm_to_diffusers(f"decoder.{k}") for k in dec.state_dict()]
    assert len(set(names)) == len(names)
    sd = ora.state_dict()
    assert set(names) == {k for k in sd if not k.startswith(("quant_conv", "post_quant_conv"))}


@torch.no_grad()
def test_oracle_vae_matches_torchtitan_flux_autoencoder():
    ora, enc, dec = _ported_pair()
    g = torch.Generator().manual_seed(0)
    x = torch.rand(2, 3, 48, 40, generator=g) * 2 - 1
    m_ora = ora.moments(x)
    m_port = ora.quant_conv(enc(x))
    assert m_ora.shape == (2, 8, 6, 5)
    e_enc = float((m_ora - m_port).norm() / m_port.norm())
    z = torch.randn(2, 4, 6, 5, generator=g)
    y_ora = ora.decode(z).sample
    y_port = dec(ora.post_quant_conv(z))
    assert y_ora.shape == (2, 3, 48, 40)
    e_dec = float((y_ora - y_port).norm() / y_port.norm())
    assert e_enc < 1e-5 and e_dec < 1e-5, (e_enc, e_dec)
