"""humanvid_b200.AutoencoderKL on the CPU: parameter names and shapes, legacy attention names, unsupported layouts, from_pretrained.
Nothing here touches a GPU (the native forwards are covered by tests/test_vae_gpu.py)."""
import json

import pytest
import torch

import humanvid_b200 as hv
import vae_oracle as V
from oracle import hv_oracle as O

LEGACY = {"to_q": "query", "to_k": "key", "to_v": "value", "to_out.0": "proj_attn"}


def _legacy(state):
    out = {}
    for k, v in state.items():
        for new, old in LEGACY.items():
            tag = f"mid_block.attentions.0.{new}."
            if tag in k:
                k = k.replace(tag, f"mid_block.attentions.0.{old}.")
        out[k] = v
    return out


def test_state_dict_matches_oracle():
    nat = hv.AutoencoderKL().state_dict()
    ora = V.AutoencoderKL().state_dict()
    assert {k: tuple(v.shape) for k, v in nat.items()} == {k: tuple(v.shape) for k, v in ora.items()}
    assert len(nat) == 248


def test_legacy_attention_names_load_identically():
    ora = O.synthetic_init(V.AutoencoderKL().eval(), seed=3)
    sd = ora.state_dict()
    old = _legacy(sd)
    assert any(".query." in k for k in old) and not any(".to_q." in k for k in old)
    # the oldest checkpoints store the attention projections as 1x1 convs
    old = {k: (v[:, :, None, None] if ".attentions.0." in k and k.endswith("weight") and "group_norm" not in k else v) for k, v in old.items()}
    a, b = hv.AutoencoderKL(), hv.AutoencoderKL()
    a.load_state_dict(sd)
    b.load_state_dict(old)
    sa, sb = a.state_dict(), b.state_dict()
    assert set(sa) == set(sb)
    for k in sa:
        assert torch.equal(sa[k], sb[k]), k
        assert torch.equal(sa[k], sd[k]), k


@pytest.mark.parametrize("kw, what", [
    (dict(block_out_channels=(64, 128, 256, 256)), "block_out_channels"),
    (dict(layers_per_block=1), "layers_per_block"),
    (dict(latent_channels=16), "latent_channels"),
    (dict(down_block_types=("DownEncoderBlock2D",) * 3, up_block_types=("UpDecoderBlock2D",) * 3), "block types"),
    (dict(act_fn="gelu"), "act_fn"),
    (dict(norm_num_groups=16), "norm_num_groups"),
])
def test_unsupported_layouts_raise(kw, what):
    with pytest.raises(NotImplementedError, match=what):
        hv.AutoencoderKL(**kw)


def test_config_and_ignored_keywords():
    v = hv.AutoencoderKL(sample_size=768, scaling_factor=0.18215, force_upcast=False, latents_mean=None, shift_factor=None)
    assert v.config.block_out_channels == (128, 256, 512, 512)
    assert v.config.scaling_factor == 0.18215 and v.config.latent_channels == 4
    assert v.dtype == torch.float32 and v.device.type == "cpu"
    with pytest.raises(RuntimeError, match="CUDA"):
        v.decode(torch.zeros(1, 4, 8, 8))


def test_from_pretrained_reads_config_and_legacy_safetensors(tmp_path):
    from safetensors.torch import save_file

    ora = O.synthetic_init(V.AutoencoderKL().eval(), seed=9)
    sd = ora.state_dict()
    sub = tmp_path / "vae"
    sub.mkdir()
    cfg = {"_class_name": "AutoencoderKL", "_diffusers_version": "0.4.2", "act_fn": "silu", "block_out_channels": [128, 256, 512, 512],
           "down_block_types": ["DownEncoderBlock2D"] * 4, "in_channels": 3, "latent_channels": 4, "layers_per_block": 2, "norm_num_groups": 32,
           "out_channels": 3, "sample_size": 256, "up_block_types": ["UpDecoderBlock2D"] * 4}
    (sub / "config.json").write_text(json.dumps(cfg))
    save_file({k: v.contiguous() for k, v in _legacy(sd).items()}, str(sub / "diffusion_pytorch_model.safetensors"))
    v = hv.AutoencoderKL.from_pretrained(str(tmp_path), subfolder="vae")
    assert v.config.sample_size == 256 and v.config.scaling_factor == 0.18215 and v.config.block_out_channels == (128, 256, 512, 512)
    assert v.device.type == "cpu" and v._handle is None
    got = v.state_dict()
    assert set(got) == set(sd)
    assert all(torch.equal(got[k], sd[k]) for k in sd)


def test_from_pretrained_bin_fallback_and_missing_weights(tmp_path):
    ora = O.synthetic_init(V.AutoencoderKL().eval(), seed=1)
    sd = ora.state_dict()
    (tmp_path / "config.json").write_text(json.dumps({"block_out_channels": [128, 256, 512, 512], "latent_channels": 4}))
    torch.save(sd, str(tmp_path / "diffusion_pytorch_model.bin"))
    v = hv.AutoencoderKL.from_pretrained(str(tmp_path), torch_dtype=torch.float16)
    assert v.dtype == torch.float16
    assert torch.equal(v.state_dict()["decoder.conv_out.weight"], sd["decoder.conv_out.weight"].half())
    del sd["decoder.conv_out.weight"]
    torch.save(sd, str(tmp_path / "diffusion_pytorch_model.bin"))
    with pytest.raises(RuntimeError, match="decoder.conv_out.weight"):
        hv.AutoencoderKL.from_pretrained(str(tmp_path))
