"""humanvid_b200.CLIPVisionModelWithProjection without a GPU: the state_dict key set of transformers' class, from_pretrained of a directory
written by transformers' save_pretrained and of a pytorch_model.bin that carries position_ids, and the configs it refuses."""
import json

import pytest
import torch

transformers = pytest.importorskip("transformers")

import humanvid_b200 as hv

SMALL = dict(hidden_size=256, intermediate_size=1024, projection_dim=192, num_hidden_layers=2, num_attention_heads=4, image_size=224, patch_size=32)


def hf_model(**kw):
    torch.manual_seed(0)
    return transformers.CLIPVisionModelWithProjection(transformers.CLIPVisionConfig(**kw)).eval()


@pytest.mark.parametrize("kw", [SMALL, dict(hidden_size=1024, intermediate_size=4096, projection_dim=768, num_hidden_layers=24, num_attention_heads=16,
                                            image_size=224, patch_size=14)], ids=["small", "vit_l14"])
def test_state_dict_keys_match_transformers(kw):
    ref = hf_model(**kw).state_dict()
    nat = hv.CLIPVisionModelWithProjection(**kw).state_dict()
    assert set(nat) == set(ref)
    for k in ref:
        assert nat[k].shape == ref[k].shape, k


def test_defaults_match_clip_vision_config():
    c = transformers.CLIPVisionConfig()
    n = hv.CLIPVisionModelWithProjection().config
    for k in ("hidden_size", "intermediate_size", "projection_dim", "num_hidden_layers", "num_attention_heads", "num_channels", "image_size",
              "patch_size", "hidden_act", "layer_norm_eps"):
        assert getattr(n, k) == getattr(c, k), k


def test_from_pretrained_save_pretrained(tmp_path):
    ref = hf_model(**SMALL)
    ref.save_pretrained(tmp_path / "image_encoder")
    assert json.load(open(tmp_path / "image_encoder" / "config.json"))["model_type"] == "clip_vision_model"
    nat = hv.CLIPVisionModelWithProjection.from_pretrained(tmp_path, subfolder="image_encoder", torch_dtype=torch.float16)
    assert nat.dtype == torch.float16 and nat.device.type == "cpu"
    assert next(nat.parameters()).dtype == torch.float16
    for k, v in ref.state_dict().items():
        assert torch.equal(nat.state_dict()[k], v.half()), k
    assert nat.config.num_hidden_layers == 2 and nat.config.patch_size == 32


def test_from_pretrained_bin_with_position_ids(tmp_path):
    ref = hf_model(**SMALL)
    state = dict(ref.state_dict())
    state["vision_model.embeddings.position_ids"] = torch.arange(50).unsqueeze(0)
    cfg = ref.config.to_dict()
    with open(tmp_path / "config.json", "w") as f:
        json.dump(cfg, f)
    torch.save(state, tmp_path / "pytorch_model.bin")
    nat = hv.CLIPVisionModelWithProjection.from_pretrained(tmp_path)
    for k, v in ref.state_dict().items():
        assert torch.equal(nat.state_dict()[k], v), k
    # the same checkpoint through load_state_dict(strict=True)
    nat2 = hv.CLIPVisionModelWithProjection(**SMALL)
    nat2.load_state_dict(state)


def test_from_pretrained_without_weights(tmp_path):
    hf_model(**SMALL).config.to_json_file(tmp_path / "config.json")
    with pytest.raises(FileNotFoundError):
        hv.CLIPVisionModelWithProjection.from_pretrained(tmp_path)


@pytest.mark.parametrize("kw, what", [
    (dict(hidden_act="gelu"), "hidden_act"),
    (dict(hidden_size=768, num_attention_heads=8), "head dim"),
    (dict(hidden_size=320, num_attention_heads=4, intermediate_size=1280), "head dim"),
    (dict(num_channels=1), "num_channels"),
    (dict(image_size=224, patch_size=15), "patch_size"),
    (dict(hidden_size=1408, num_attention_heads=22, intermediate_size=6144), "hidden_size"),
])
def test_unsupported_configs(kw, what):
    with pytest.raises(NotImplementedError, match=what):
        hv.CLIPVisionModelWithProjection(**kw)


def test_cpu_forward_raises():
    m = hv.CLIPVisionModelWithProjection(**SMALL)
    with pytest.raises(RuntimeError, match="CUDA"):
        m(torch.zeros(1, 3, 224, 224))


@pytest.mark.parametrize("kw", [dict(output_attentions=True), dict(output_hidden_states=True), dict(interpolate_pos_encoding=True)])
def test_unsupported_outputs(kw):
    m = hv.CLIPVisionModelWithProjection(**SMALL)
    with pytest.raises(NotImplementedError):
        m(torch.zeros(1, 3, 224, 224), **kw)


def test_wrong_pixel_size():
    m = hv.CLIPVisionModelWithProjection(**SMALL)
    with pytest.raises(ValueError, match="doesn't match"):
        m(torch.zeros(1, 3, 256, 256))
    with pytest.raises(ValueError):
        m(torch.zeros(1, 1, 224, 224))
