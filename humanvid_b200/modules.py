"""Reference-facing modules of the H100-native denoising path.

``UNet3DConditionModel``, ``PoseGuider`` and ``CameraPoseEncoder`` keep the reference's constructor arguments,
``forward`` signatures, attribute names and ``state_dict`` keys (SURVEY.md section 8b), so
``scripts/pose2vid.py``-style drivers build, load and call them unchanged:

  * ``UNet3DConditionModel.forward``  <->  src/models/unet_3d.py:397-577
  * ``PoseGuider.forward``            <->  src/models/pose_guider.py:51-61
  * ``CameraPoseEncoder.forward``     <->  src/cameractrl/pose_adaptor.py:232-248
  * ``UNet2DConditionModel.forward``  <->  src/models/unet_2d_condition.py:872-1308 (the reference / "writer" UNet, whose
    LayerNorm-1 outputs become the denoising UNet's K/V banks)
  * ``AutoencoderKL.encode / decode``  <->  diffusers 0.24 ``AutoencoderKL`` in the SD layout (sd-vae-ft-mse), what the pipelines
    call for the reference latents and the output frames
  * ``CLIPVisionModelWithProjection``  <->  transformers' class of the same name (the image encoder of scripts/pose2vid.py:17,152),
    whose ``image_embeds`` condition both UNets

The ``nn.Module`` tree below only *holds parameters* under the reference's names (torch is plumbing: device memory,
``load_state_dict``, ``.to()``); none of its sub-modules' ``forward`` is ever executed.  All arithmetic happens in
``libhv_b200.so`` (hand-written sm_90a CUDA) through the C ABI in ``include/hv_b200.h``.  There is no PyTorch or
CPU fallback: without the library, or on a non-CUDA tensor, ``forward`` raises.
"""
from __future__ import annotations

import ctypes as C
import inspect
import json
import math
import os
import warnings
from dataclasses import dataclass
from types import SimpleNamespace
from typing import List, Optional, Sequence, Tuple, Union

import torch
import torch.nn as nn

from . import _native as N


# --------------------------------------------------------------------------------------------- parameter shells
class _Shell(nn.Module):
    """Parameter container; never called."""

    def forward(self, *a, **k):  # pragma: no cover
        raise RuntimeError("humanvid_b200 parameter shells are not executable; call the owning network's forward")


def _conv(cin, cout, k, **kw):
    return nn.Conv2d(cin, cout, k, **kw)


class _Attention(_Shell):
    """diffusers Attention parameter names: to_q/to_k/to_v (no bias), to_out.0 (bias)."""

    def __init__(self, dim, cross_dim=None):
        super().__init__()
        self.to_q = nn.Linear(dim, dim, bias=False)
        self.to_k = nn.Linear(cross_dim or dim, dim, bias=False)
        self.to_v = nn.Linear(cross_dim or dim, dim, bias=False)
        self.to_out = nn.ModuleList([nn.Linear(dim, dim), nn.Dropout(0.0)])


class _GEGLU(_Shell):
    def __init__(self, dim):
        super().__init__()
        self.proj = nn.Linear(dim, dim * 8)


class _FeedForward(_Shell):
    def __init__(self, dim):
        super().__init__()
        self.net = nn.ModuleList([_GEGLU(dim), nn.Dropout(0.0), nn.Linear(dim * 4, dim)])


class TemporalBasicTransformerBlock(_Shell):
    """Parameter shell of src/models/attention.py:298-379; ``bank`` is what ReferenceAttentionControl.update fills."""

    def __init__(self, dim, cross_attention_dim):
        nn.Module.__init__(self)   # not super(): an adopted reference class (see _adopt_reference_class) sits later in the MRO
        self.attn1 = _Attention(dim)
        self.norm1 = nn.LayerNorm(dim)
        self.attn2 = _Attention(dim, cross_attention_dim)
        self.norm2 = nn.LayerNorm(dim)
        self.ff = _FeedForward(dim)
        self.norm3 = nn.LayerNorm(dim)
        self.bank: List[torch.Tensor] = []


class BasicTransformerBlock(TemporalBasicTransformerBlock):
    """Writer-side block of the 2-D reference UNet (src/models/attention.py BasicTransformerBlock): same parameters."""


_ADOPTED = {}


def _adopt_reference_class(cls):
    """Inside the reference tree its own ``ReferenceAttentionControl`` finds the blocks to hook with
    ``isinstance(module, src.models.attention.TemporalBasicTransformerBlock / BasicTransformerBlock)``
    (mutual_self_attention.py:284-300, 321-330).  A native UNet built there must not silently present zero blocks (banks
    would never arrive): when ``src.models.attention`` is loaded, the shells are instantiated from a subclass that also derives
    from the reference's class of the same name, so the reference's control walks, sorts, hooks and fills ``.bank`` on them
    exactly as on its own modules.  (The hooked ``forward`` is never called; the native forward reads ``.bank``.)"""
    import sys

    ref_mod = sys.modules.get("src.models.attention")
    ref = getattr(ref_mod, cls.__name__, None) if ref_mod is not None else None
    if not (isinstance(ref, type) and issubclass(ref, nn.Module)) or issubclass(cls, ref):
        return cls
    key = (cls, ref)
    if key not in _ADOPTED:
        _ADOPTED[key] = type(cls.__name__, (cls, ref), {"__module__": cls.__module__, "__doc__": cls.__doc__})
    return _ADOPTED[key]


class _Transformer3D(_Shell):
    def __init__(self, ch, cross_attention_dim, groups, block_cls=None):
        super().__init__()
        self.norm = nn.GroupNorm(groups, ch, eps=1e-6)
        self.proj_in = _conv(ch, ch, 1)
        self.transformer_blocks = nn.ModuleList([_adopt_reference_class(block_cls or TemporalBasicTransformerBlock)(ch, cross_attention_dim)])
        self.proj_out = _conv(ch, ch, 1)


def _sinusoid(max_len, dim):
    pos = torch.arange(max_len).unsqueeze(1)
    div = torch.exp(torch.arange(0, dim, 2) * (-math.log(10000.0) / dim))
    pe = torch.zeros(1, max_len, dim)
    pe[0, :, 0::2] = torch.sin(pos * div)
    pe[0, :, 1::2] = torch.cos(pos * div)
    return pe


class _PosEnc(_Shell):
    def __init__(self, dim, max_len):
        super().__init__()
        self.register_buffer("pe", _sinusoid(max_len, dim))


class _TemporalAttention(_Attention):
    def __init__(self, dim, max_len):
        super().__init__(dim)
        self.pos_encoder = _PosEnc(dim, max_len)


class _TemporalBlock(_Shell):
    def __init__(self, dim, n_attn, max_len):
        super().__init__()
        self.attention_blocks = nn.ModuleList([_TemporalAttention(dim, max_len) for _ in range(n_attn)])
        self.norms = nn.ModuleList([nn.LayerNorm(dim) for _ in range(n_attn)])
        self.ff = _FeedForward(dim)
        self.ff_norm = nn.LayerNorm(dim)


class _TemporalTransformer3D(_Shell):
    def __init__(self, ch, max_len, groups):
        super().__init__()
        self.norm = nn.GroupNorm(groups, ch, eps=1e-6)
        self.proj_in = nn.Linear(ch, ch)
        self.transformer_blocks = nn.ModuleList([_TemporalBlock(ch, 2, max_len)])
        self.proj_out = nn.Linear(ch, ch)
        nn.init.zeros_(self.proj_out.weight)   # zero_module (motion_module.py:72-75): an unloaded motion module is the identity
        nn.init.zeros_(self.proj_out.bias)


class _MotionModule(_Shell):
    def __init__(self, ch, max_len, groups):
        super().__init__()
        self.temporal_transformer = _TemporalTransformer3D(ch, max_len, groups)


class _Resnet(_Shell):
    def __init__(self, cin, cout, temb, groups):
        super().__init__()
        self.norm1 = nn.GroupNorm(groups, cin, eps=1e-5)
        self.conv1 = _conv(cin, cout, 3, padding=1)
        self.time_emb_proj = nn.Linear(temb, cout)
        self.norm2 = nn.GroupNorm(groups, cout, eps=1e-5)
        self.conv2 = _conv(cout, cout, 3, padding=1)
        if cin != cout:
            self.conv_shortcut = _conv(cin, cout, 1)


class _Sampler(_Shell):
    def __init__(self, ch, stride):
        super().__init__()
        self.conv = _conv(ch, ch, 3, stride=stride, padding=1)


def _torch_dfs(m):
    """Every module under `m` in pre-order, like the reference's torch_dfs (mutual_self_attention.py): no deduplication."""
    out = [m]
    for c in m.children():
        out += _torch_dfs(c)
    return out


class _Block(_Shell):
    def __init__(self, res_io, ch, attn, motion, xdim, temb, groups, max_len, sampler=None, block_cls=None):
        super().__init__()
        if attn:
            self.attentions = nn.ModuleList([_Transformer3D(ch, xdim, groups, block_cls) for _ in range(attn)])
        self.resnets = nn.ModuleList([_Resnet(i, o, temb, groups) for i, o in res_io])
        if block_cls is None:   # the 2-D reference UNet's blocks (block_cls given) have no motion_modules attribute
            self.motion_modules = nn.ModuleList([_MotionModule(ch, max_len, groups) if motion else None for _ in range(max(attn, len(res_io)) if sampler != "mid" else 1)])
        if sampler == "down":
            self.downsamplers = nn.ModuleList([_Sampler(ch, 2)])
        elif sampler == "up":
            self.upsamplers = nn.ModuleList([_Sampler(ch, 1)])


class _TimestepEmbedding(_Shell):
    def __init__(self, cin, cout):
        super().__init__()
        self.linear_1 = nn.Linear(cin, cout)
        self.linear_2 = nn.Linear(cout, cout)


def _sd15_unsupported(c, dim):
    """The SD1.5 layout checks both UNets share, on config `c`; `dim` ("2D" / "3D") ends the block type names."""
    unsupported = []
    if tuple(c.down_block_types) != (f"CrossAttnDownBlock{dim}",) * 3 + (f"DownBlock{dim}",) \
            or tuple(c.up_block_types) != (f"UpBlock{dim}",) + (f"CrossAttnUpBlock{dim}",) * 3:
        unsupported.append("block types other than the SD1.5 layout")
    if c.layers_per_block != 2 or len(c.block_out_channels) != 4:
        unsupported.append("layers_per_block != 2 / depth != 4")
    if c.center_input_sample or not c.flip_sin_to_cos or c.freq_shift != 0 or c.use_linear_projection or c.dual_cross_attention:
        unsupported.append("center_input_sample / flip_sin_to_cos=False / freq_shift / use_linear_projection / dual_cross_attention")
    if c.class_embed_type is not None or c.num_class_embeds is not None:
        unsupported.append("class embeddings")
    if c.resnet_time_scale_shift != "default" or c.act_fn not in ("silu", "swish") or c.mid_block_scale_factor != 1 \
            or not isinstance(c.attention_head_dim, int):
        unsupported.append("non-default resnet/act options")
    return unsupported


def _build_sd15_unet(unet, in_channels, ch, xdim, groups, motion=False, mid_motion=False, max_len=0, block_cls=None):
    """conv_in, time_embedding and the down / mid / up ``_Block`` tree of the SD1.5 layout on `unet`.  ``block_cls=None`` builds the
    denoising UNet's blocks, each with ``motion_modules`` (motion modules where `motion` / `mid_motion`, else None entries); the writer UNet
    passes its ``BasicTransformerBlock``.  down_blocks and up_blocks are registered before mid_block: the module walk, and so the bank
    order, is down, up, mid as in the reference."""
    temb = ch[0] * 4
    unet.conv_in = _conv(in_channels, ch[0], 3, padding=1)
    unet.time_embedding = _TimestepEmbedding(ch[0], temb)
    unet.down_blocks = nn.ModuleList([])
    unet.up_blocks = nn.ModuleList([])
    prev = ch[0]
    for i, c in enumerate(ch):
        last = i == 3
        unet.down_blocks.append(_Block([(prev, c), (c, c)], c, 0 if last else 2, motion, xdim, temb, groups, max_len, None if last else "down", block_cls))
        prev = c
    unet.mid_block = _Block([(ch[3], ch[3]), (ch[3], ch[3])], ch[3], 1, mid_motion, xdim, temb, groups, max_len, "mid", block_cls)
    rev = ch[::-1]
    prev = rev[0]
    for i, c in enumerate(rev):
        cin = rev[min(i + 1, 3)]
        io = [((prev if j == 0 else c) + (cin if j == 2 else c), c) for j in range(3)]
        unet.up_blocks.append(_Block(io, c, 0 if i == 0 else 3, motion, xdim, temb, groups, max_len, "up" if i < 3 else None, block_cls))
        prev = c


def _sd15_hv_config(c, kind):
    """The HvConfig fields both UNets fill from their config."""
    cfg = HvConfig()
    cfg.kind = kind
    cfg.in_channels, cfg.out_channels = c.in_channels, c.out_channels
    cfg.block_out_channels = (C.c_int32 * 4)(*c.block_out_channels)
    cfg.heads, cfg.cross_attention_dim, cfg.norm_groups = c.attention_head_dim, c.cross_attention_dim, c.norm_num_groups
    return cfg


def _read_state(path):
    """A checkpoint file's state dict on the CPU: safetensors by suffix, else a torch pickle of tensors."""
    if os.path.splitext(path)[1].lower() == ".safetensors":
        from safetensors.torch import load_file

        return load_file(path, device="cpu")
    return torch.load(path, map_location="cpu", weights_only=True)


def _from_pretrained(cls, pretrained_model_path, subfolder=None, overrides=None, weights=("diffusion_pytorch_model.safetensors",
                     "diffusion_pytorch_model.bin"), require_all=False, torch_dtype=None):
    """``<path>[/<subfolder>]/config.json`` without its ``_`` keys -> ``cls`` from the keywords its ``__init__`` takes, then `overrides`;
    weights from ``weights[0]`` (safetensors) or else ``weights[1]``, loaded with strict=False.  With `require_all`, a parameter the
    checkpoint lacks raises.  Builds on the CPU."""
    path = os.path.join(str(pretrained_model_path), subfolder) if subfolder is not None else str(pretrained_model_path)
    with open(os.path.join(path, "config.json")) as f:
        cfg = {k: v for k, v in json.load(f).items() if not k.startswith("_")}
    allowed = set(inspect.signature(cls.__init__).parameters) - {"self", "unused"}
    model = cls(**{**{k: v for k, v in cfg.items() if k in allowed}, **(overrides or {})})
    st_path, bin_path = (os.path.join(path, w) for w in weights)
    if os.path.exists(st_path):
        state = _read_state(st_path)
    elif os.path.isfile(bin_path):
        state = _read_state(bin_path)
    else:
        raise FileNotFoundError(f"no weights file found in {path}")
    missing = model.load_state_dict(state, strict=False).missing_keys
    if require_all and missing:
        raise RuntimeError(f"{path}: weights missing from the checkpoint: {missing[:5]}{' ...' if len(missing) > 5 else ''}")
    return model.to(torch_dtype) if torch_dtype is not None else model


@dataclass
class UNet3DConditionOutput:
    sample: torch.Tensor


# --------------------------------------------------------------------------------------------- native base
class _NativeNet(nn.Module):
    """Owns one ``hv_handle``; pushes the module's state_dict into it whenever parameters changed."""

    def __init__(self):
        super().__init__()
        self._handle = None
        self._pushed_versions = None
        self._epoch = 0
        self._bank_fp = None
        self._bank_refs = None
        self._reserved = set()

    def _hv_config(self) -> "HvConfig":  # pragma: no cover - overridden
        raise NotImplementedError

    @property
    def dtype(self):
        return next(self.parameters()).dtype

    @property
    def device(self):
        return next(self.parameters()).device

    def _versions(self):
        # fingerprint checked on every forward: in-place edits of ANY parameter / buffer (sum of their version counters), a
        # re-allocation or dtype change of the first one, and load_state_dict()/.to()/.half() (the epoch) all force a re-push.
        # The flat tensor list is cached per epoch: walking the module tree (~600 modules, 1270 tensors) cost 3 ms of host time per
        # forward, which the end-to-end step (copy in -> forward -> copy out, nothing to hide behind) paid in full.  A Parameter OBJECT
        # replaced by attribute assignment is not seen by the cache: call refresh_native() after such surgery (in-place edits are seen).
        cache = self.__dict__.get("_ver_cache")
        if cache is None or cache[0] != self._epoch:
            cache = (self._epoch, list(self.parameters()) + list(self.buffers()))
            self.__dict__["_ver_cache"] = cache
        tensors = cache[1]
        p = tensors[0]
        ver = 0
        for t in tensors:
            ver += t._version
        return (p.data_ptr(), ver, p.dtype, self._epoch)

    def _apply(self, fn, *a, **k):
        self._epoch = getattr(self, "_epoch", 0) + 1
        return super()._apply(fn, *a, **k)

    def load_state_dict(self, *a, **k):
        self._epoch = getattr(self, "_epoch", 0) + 1
        return super().load_state_dict(*a, **k)

    def refresh_native(self):
        """Call after modifying parameters in place: the packed device copy is rebuilt on the next forward."""
        self._epoch = getattr(self, "_epoch", 0) + 1

    def _destroy(self):
        if self._handle is not None:
            N.lib().hv_destroy(self._handle)
            self._handle = None
        # a new handle may be created at the same address: nothing cached against the old one may survive it
        self._bank_fp = None
        self._bank_refs = None
        self._reserved = set()

    def _reserve(self, h, B, F, H, W, variant=()):
        """The C forwards never allocate: grow the handle's private workspace here, once per new shape (and `variant`: whatever
        else the plan depends on, such as the reference banks of the denoising UNet)."""
        key = (B, F, H, W, variant)
        if key not in self._reserved:
            N.check(N.lib().hv_reserve_workspace(h, N.i32(B), N.i32(F), N.i32(H), N.i32(W)), h)
            self._reserved.add(key)

    def _workspace_bytes(self, B, F, H, W) -> int:
        hd = self._sync_native()
        return int(N.lib().hv_workspace_bytes(hd, N.i32(B), N.i32(F), N.i32(H), N.i32(W)))

    def _run(self, entry, h, shape, *args):
        """Reserve the workspace for `shape` (``_reserve``'s B, F, H, W[, variant]), call the C forward `entry` as
        ``entry(h, *args, NULL workspace, 0, current stream)`` and raise with the handle's message on a non-zero status."""
        self._reserve(h, *shape)
        N.check(entry(h, *args, None, C.c_size_t(0), N.stream()), h)

    def __del__(self):
        try:
            self._destroy()
        except Exception:
            pass

    def _sync_native(self):
        if self.device.type != "cuda":
            raise RuntimeError("humanvid_b200 runs on CUDA (H100) only: move the module with .to('cuda', torch.float16); there is no CPU path")
        ver = self._versions()
        if self._handle is not None and ver == self._pushed_versions:
            return self._handle
        self._destroy()
        lib = N.lib()
        cfg = self._hv_config()
        h = C.c_void_p()
        N.check(lib.hv_create(C.byref(cfg), C.byref(h)))
        st = N.stream()
        for k, v in self.state_dict().items():
            if v.dtype == torch.float16:
                dt = 0
            elif v.dtype == torch.float32:
                dt = 1
            else:
                raise RuntimeError(f"parameter {k} has dtype {v.dtype}; humanvid_b200 ingests fp16 or fp32 weights")
            t = v.detach().contiguous()
            shape = (C.c_int64 * max(t.dim(), 1))(*(t.shape if t.dim() else (1,)))
            N.check(lib.hv_set_weight(h, k.encode(), N.ptr(t), shape, N.i32(max(t.dim(), 1)), N.i32(dt), st), h)
        N.check(lib.hv_finalize(h, st), h)
        torch.cuda.current_stream().synchronize()
        self._handle = h
        self._pushed_versions = ver
        return h

    @staticmethod
    def _as_half(x: torch.Tensor, what: str) -> torch.Tensor:
        if not x.is_cuda:
            raise RuntimeError(f"{what} must be a CUDA tensor (humanvid_b200 has no CPU path)")
        return x.to(torch.float16).contiguous()

    @staticmethod
    def _from_half(t: torch.Tensor, dtype: torch.dtype) -> torch.Tensor:
        """A forward's fp16 result in the caller's dtype."""
        return t if dtype == torch.float16 else t.to(dtype)

    @property
    def last_launch_count(self) -> int:
        if self._handle is None:
            return 0
        return int(N.lib().hv_last_launch_count(self._handle))

    # ---- debug taps (per-block parity tests, scripts/error_ladder.py) ------------------------------------------------------
    def debug_tap_plan(self, B, F, h, w):
        """[(reference module path, (NF, H, W, C))] of the activations the native forward can copy out, in execution order, at the shape
        ``hv_workspace_bytes`` takes: (B, F, h, w) latent for the UNets (F = 1 for the 2-D one), (n, 1, h, w) latent for the VAE (the
        decoder's taps at h x w, then the encoder's at 8h x 8w), (B, 1, S, S) for CLIP, (B, F, H, W) image for the PoseGuider and the
        camera encoder.  C includes the zero channels of a padded layout."""
        hd = self._sync_native()
        lib = N.lib()
        n = lib.hv_debug_tap_count(hd, N.i32(B), N.i32(F), N.i32(h), N.i32(w))
        if n < 0:
            N.check(n, hd)
        plan = []
        for i in range(n):
            name = C.create_string_buffer(128)
            dims = (C.c_int64 * 4)()
            N.check(lib.hv_debug_tap_info(hd, N.i32(i), name, N.i32(128), dims), hd)
            plan.append((name.value.decode(), tuple(int(d) for d in dims)))
        return plan

    def debug_set_taps(self, tensors):
        """tensors[i] (or None) receives tap i of ``debug_tap_plan`` as channels-last fp16 (NF, H, W, C) on the next forwards; [] disables."""
        hd = self._sync_native()
        self._tap_refs = list(tensors)
        arr = (C.c_void_p * max(len(tensors), 1))(*[None if t is None else t.data_ptr() for t in tensors])
        N.check(N.lib().hv_debug_set_taps(hd, arr if tensors else None, N.i32(len(tensors))), hd)


class HvConfig(C.Structure):
    _fields_ = [
        ("kind", C.c_int32),
        ("in_channels", C.c_int32),
        ("out_channels", C.c_int32),
        ("block_out_channels", C.c_int32 * 4),
        ("heads", C.c_int32),
        ("cross_attention_dim", C.c_int32),
        ("norm_groups", C.c_int32),
        ("use_motion_module", C.c_int32),
        ("motion_max_len", C.c_int32),
        ("pg_cond_channels", C.c_int32),
        ("pg_block_channels", C.c_int32 * 4),
        ("pg_out_channels", C.c_int32),
        ("cam_downscale", C.c_int32),
        ("cam_cin", C.c_int32),
        ("cam_channels", C.c_int32),
        ("cam_nums_rb", C.c_int32),
        ("cam_heads", C.c_int32),
        ("cam_max_len", C.c_int32),
        ("vae_latent_channels", C.c_int32),
        ("clip_hidden_size", C.c_int32),
        ("clip_layers", C.c_int32),
        ("clip_heads", C.c_int32),
        ("clip_intermediate_size", C.c_int32),
        ("clip_patch_size", C.c_int32),
        ("clip_image_size", C.c_int32),
        ("clip_projection_dim", C.c_int32),
        ("clip_layer_norm_eps", C.c_float),
        ("gn_pool_frames", C.c_int32),
        ("no_mid_motion_module", C.c_int32),
        ("fp8_linears", C.c_int32),
    ]


# --------------------------------------------------------------------------------------------- UNet3DConditionModel
class UNet3DConditionModel(_NativeNet):
    """Drop-in for src/models/unet_3d.py:30-577 (inference): same ctor keywords, forward signature, state_dict keys."""

    def __init__(
        self,
        sample_size: Optional[int] = None,
        in_channels: int = 4,
        out_channels: int = 4,
        center_input_sample: bool = False,
        flip_sin_to_cos: bool = True,
        freq_shift: int = 0,
        down_block_types: Tuple[str, ...] = ("CrossAttnDownBlock3D", "CrossAttnDownBlock3D", "CrossAttnDownBlock3D", "DownBlock3D"),
        mid_block_type: str = "UNetMidBlock3DCrossAttn",
        up_block_types: Tuple[str, ...] = ("UpBlock3D", "CrossAttnUpBlock3D", "CrossAttnUpBlock3D", "CrossAttnUpBlock3D"),
        only_cross_attention=False,
        block_out_channels: Tuple[int, ...] = (320, 640, 1280, 1280),
        layers_per_block: int = 2,
        downsample_padding: int = 1,
        mid_block_scale_factor: float = 1,
        act_fn: str = "silu",
        norm_num_groups: int = 32,
        norm_eps: float = 1e-5,
        cross_attention_dim: int = 1280,
        attention_head_dim=8,
        dual_cross_attention: bool = False,
        use_linear_projection: bool = False,
        class_embed_type=None,
        num_class_embeds=None,
        upcast_attention: bool = False,
        resnet_time_scale_shift: str = "default",
        use_inflated_groupnorm=False,
        use_motion_module=False,
        motion_module_resolutions=(1, 2, 4, 8),
        motion_module_mid_block=False,
        motion_module_decoder_only=False,
        motion_module_type=None,
        motion_module_kwargs=None,
        unet_use_cross_frame_attention=None,
        unet_use_temporal_attention=None,
    ):
        super().__init__()
        self.config = SimpleNamespace(**{k: v for k, v in locals().items() if k not in ("self", "__class__")})
        mmk = dict(motion_module_kwargs or {})
        unsupported = _sd15_unsupported(self.config, "3D")
        if unet_use_temporal_attention or unet_use_cross_frame_attention:
            unsupported.append("unet_use_temporal_attention / cross_frame_attention")
        if use_motion_module and (
            tuple(motion_module_resolutions) != (1, 2, 4, 8) or motion_module_decoder_only
            or motion_module_type != "Vanilla" or mmk.get("num_transformer_block", 1) != 1
            or tuple(mmk.get("attention_block_types", ("Temporal_Self", "Temporal_Self"))) != ("Temporal_Self", "Temporal_Self")
            or not mmk.get("temporal_position_encoding", False) or mmk.get("temporal_attention_dim_div", 1) != 1
        ):
            unsupported.append("motion-module layout other than configs/inference/inference_v1.yaml / inference_v2.yaml")
        if unsupported:
            raise NotImplementedError("humanvid_b200.UNet3DConditionModel implements the inference_v1 / inference_v2 hot path only; unsupported: "
                                      + "; ".join(unsupported))
        self.sample_size = sample_size
        self.in_channels = in_channels
        ch = list(block_out_channels)
        self._mm = mm = bool(use_motion_module)
        self._max_len = mmk.get("temporal_position_encoding_max_len", 24)
        # inference_v1.yaml: no motion module in the mid block
        _build_sd15_unet(self, in_channels, ch, cross_attention_dim, norm_num_groups, mm, mm and bool(motion_module_mid_block), self._max_len)
        self.conv_norm_out = nn.GroupNorm(norm_num_groups, ch[0], eps=norm_eps)
        self.conv_out = _conv(ch[0], out_channels, 3, padding=1)
        self._ref_cfg = True
        self._forward_flags = None   # humanvid_b200.distributed sets HV_FLAG_UNCOND_ONLY / HV_FLAG_COND_ONLY for one-half units

    # ---- reference banks (ReferenceAttentionControl, read side) -----------------------------------------------
    def reader_blocks(self) -> List[TemporalBasicTransformerBlock]:
        """fusion_blocks='full' order of mutual_self_attention.py:284-300."""
        cached = self.__dict__.get("_reader_blocks_cache")
        if cached is None:      # the module tree is fixed after __init__: walk it once (1 ms per forward otherwise)
            mods = [m for m in _torch_dfs(self) if isinstance(m, TemporalBasicTransformerBlock)]
            cached = sorted(mods, key=lambda m: -m.norm1.normalized_shape[0])
            self.__dict__["_reader_blocks_cache"] = cached
        return list(cached)

    def _push_banks(self, h):
        lib = N.lib()
        blocks = self.reader_blocks()
        any_bank = any(len(b.bank) > 0 for b in blocks)
        # the banks are step-invariant (written once per clip): skip the 16 device copies when nothing changed since the last push
        # (the pushed tensors are kept referenced so that their addresses cannot be recycled under the fingerprint)
        tensors = [t for b in blocks for t in b.bank]
        fp = (h.value if hasattr(h, "value") else h, self._epoch) + tuple((t.data_ptr(), t._version, tuple(t.shape), t.dtype) for t in tensors)
        if getattr(self, "_bank_fp", None) == fp:
            return
        self._bank_fp, self._bank_refs = fp, tensors
        N.check(lib.hv_clear_ref_banks(h), h)
        if not any_bank:
            # A reader control is registered (ours, or the reference's: its register_reference_hooks leaves an instance-level `forward` on every
            # block, mutual_self_attention.py:302-330) but no bank has been written: the reference would then attend over the clip's own tokens
            # only, and so does this forward -- legal, but almost always a missing `reader.update(writer)`.  Say so once.
            hooked = getattr(self, "_reader_registered", False) or any("forward" in b.__dict__ for b in blocks)
            if hooked and not getattr(self, "_warned_no_bank", False):
                self._warned_no_bank = True
                warnings.warn("humanvid_b200.UNet3DConditionModel: a ReferenceAttentionControl reader is registered but every reference bank is "
                              "empty; this forward runs without reference attention (call reader.update(writer) after the writer forward)",
                              RuntimeWarning, stacklevel=3)
            return
        st = N.stream()
        for i, b in enumerate(blocks):
            if len(b.bank) == 0:
                continue
            if len(b.bank) != 1:
                raise NotImplementedError("one reference bank per block is supported (the pipeline writes exactly one)")
            t = self._as_half(b.bank[0], "reference bank")
            N.check(lib.hv_set_ref_bank(h, N.i32(i), N.ptr(t), N.i64(t.shape[0]), N.i64(t.shape[1]), N.i64(t.shape[2]), st), h)

    def _hv_config(self):
        c = self.config
        cfg = _sd15_hv_config(c, N.HV_KIND_UNET3D)
        cfg.use_motion_module, cfg.motion_max_len = int(self._mm), self._max_len
        # use_inflated_groupnorm=False: the resnets and conv_norm_out apply nn.GroupNorm to (b, c, f, h, w), pooling over the frames
        cfg.gn_pool_frames = int(not c.use_inflated_groupnorm)
        cfg.no_mid_motion_module = int(self._mm and not c.motion_module_mid_block)
        cfg.fp8_linears = int(self.__dict__.get("_fp8", False))
        return cfg

    # ---- FP8 mode (DESIGN.md §9) -----------------------------------------------------------------------------------------
    @property
    def fp8_linears(self) -> bool:
        """True while the wide feed-forwards run on e4m3 (enable_fp8_linears)."""
        return bool(self.__dict__.get("_fp8", False))

    def enable_fp8_linears(self):
        """Run the LayerNorm -> FF1 -> FF2 chains of the transformers and motion modules of width >= 1280 on e4m3 (per-row weight scales,
        per-token and per-128 activation scales).  Faster at those widths on an H100, at the cost of the e4m3 quantisation error; the next
        forward rebuilds the native handle, as a weight change does."""
        self._set_fp8(True)
        return self

    def disable_fp8_linears(self):
        """Back to the fp16 path (the outputs of a model that never enabled FP8)."""
        self._set_fp8(False)
        return self

    def _set_fp8(self, on):
        if self.fp8_linears != bool(on):
            self.__dict__["_fp8"] = bool(on)
            self._epoch = getattr(self, "_epoch", 0) + 1

    def workspace_bytes(self, B, F, h, w) -> int:
        return self._workspace_bytes(B, F, h, w)

    @torch.no_grad()
    def forward(
        self,
        sample: torch.Tensor,
        timestep: Union[torch.Tensor, float, int],
        encoder_hidden_states: torch.Tensor,
        class_labels: Optional[torch.Tensor] = None,
        pose_cond_fea: Optional[torch.Tensor] = None,
        attention_mask: Optional[torch.Tensor] = None,
        down_block_additional_residuals: Optional[Tuple[torch.Tensor]] = None,
        mid_block_additional_residual: Optional[torch.Tensor] = None,
        return_dict: bool = True,
    ):
        if class_labels is not None or attention_mask is not None or down_block_additional_residuals is not None or mid_block_additional_residual is not None:
            raise NotImplementedError("class_labels / attention_mask / additional residuals are not part of the CamAnimate inference path")
        if sample.dim() != 5:
            raise ValueError(f"Expected sample to have ndim=5 (b c f h w), got {sample.dim()}")
        B, Cc, F, H, W = sample.shape
        if Cc != self.in_channels:
            raise ValueError(f"sample has {Cc} channels, model expects {self.in_channels}")
        h = self._sync_native()
        self._push_banks(h)
        x = self._as_half(sample, "sample")
        ehs = self._as_half(encoder_hidden_states, "encoder_hidden_states")
        if ehs.shape[0] != B or ehs.shape[1] != 1:
            raise ValueError(f"encoder_hidden_states must be (batch, 1, dim) with batch {B}; got {tuple(ehs.shape)}")
        pose = None if pose_cond_fea is None else self._as_half(pose_cond_fea, "pose_cond_fea")
        if pose is not None and tuple(pose.shape) != (B, self.config.block_out_channels[0], F, H, W):
            raise ValueError(f"pose_cond_fea must be {(B, self.config.block_out_channels[0], F, H, W)}, got {tuple(pose.shape)}")
        t = int(timestep.reshape(-1)[0].item()) if torch.is_tensor(timestep) else int(timestep)
        out = torch.empty((B, self.config.out_channels, F, H, W), device=x.device, dtype=torch.float16)
        flags = self._forward_flags if self._forward_flags is not None else (1 if self._ref_cfg else 0)
        banks = tuple(tuple(t.shape) for t in (self._bank_refs or ()))   # the banks' K/V scratch is planned too
        self._run(N.lib().hv_unet3d_forward, h, (B, F, H, W, banks), N.ptr(x), N.i64(t), N.ptr(ehs), N.ptr(pose), N.ptr(out), N.i32(B), N.i32(F),
                  N.i32(H), N.i32(W), C.c_uint32(flags))
        out = self._from_half(out, sample.dtype)
        if not return_dict:
            return (out,)
        return UNet3DConditionOutput(sample=out)

    # ---- loading (unet_3d.py:579-670) ---------------------------------------------------------------------------
    @classmethod
    def from_pretrained_2d(cls, pretrained_model_path, motion_module_path, subfolder=None, unet_additional_kwargs=None, mm_zero_proj_out=False):
        config_file = os.path.join(str(pretrained_model_path), subfolder or "", "config.json")
        if not os.path.isfile(config_file):
            raise RuntimeError(f"{config_file} does not exist or is not a file")
        blocks = dict(down_block_types=["CrossAttnDownBlock3D"] * 3 + ["DownBlock3D"], up_block_types=["UpBlock3D"] + ["CrossAttnUpBlock3D"] * 3,
                      mid_block_type="UNetMidBlock3DCrossAttn")
        model = _from_pretrained(cls, pretrained_model_path, subfolder, {**blocks, **(unet_additional_kwargs or {})})
        mp = str(motion_module_path)
        if os.path.isfile(mp):
            suffix = os.path.splitext(mp)[1].lower()
            if suffix not in (".pth", ".pt", ".ckpt", ".safetensors"):
                raise RuntimeError(f"unknown file format for motion module weights: {suffix}")
            mm_state = _read_state(mp)
            if mm_zero_proj_out:
                mm_state = {k: v for k, v in mm_state.items() if "proj_out" not in k}
            # every key, like the reference (unet_3d.py:657-658): one the 2-D file also has is overwritten, one the model lacks is dropped
            model.load_state_dict(mm_state, strict=False)
        return model

# --------------------------------------------------------------------------------------------- reference ("writer") UNet
@dataclass
class UNet2DConditionOutput:
    sample: torch.Tensor


class UNet2DConditionModel(_NativeNet):
    """Drop-in for the reference ("writer") UNet, src/models/unet_2d_condition.py (SD1.5 layout), inference only.

    ``forward(sample (b,4,h,w), timestep, encoder_hidden_states (b,1,dim))`` returns what the reference returns -- the last
    up block's output (b, 320, h, w); the post-process is removed there (unet_2d_condition.py:1295-1299).  Under
    ``ReferenceAttentionControl(self, mode="write", fusion_blocks="full")`` every transformer block's LayerNorm-1 output
    is left in ``block.bank`` (mutual_self_attention.py:137-146), ready for ``reader.update(writer)``.  The native forward
    (``hv_unet2d_reference_forward``) is the denoising UNet's own kernels at one frame without motion modules.
    """

    def __init__(
        self,
        sample_size: Optional[int] = None,
        in_channels: int = 4,
        out_channels: int = 4,
        center_input_sample: bool = False,
        flip_sin_to_cos: bool = True,
        freq_shift: int = 0,
        down_block_types: Tuple[str, ...] = ("CrossAttnDownBlock2D", "CrossAttnDownBlock2D", "CrossAttnDownBlock2D", "DownBlock2D"),
        mid_block_type: Optional[str] = "UNetMidBlock2DCrossAttn",
        up_block_types: Tuple[str, ...] = ("UpBlock2D", "CrossAttnUpBlock2D", "CrossAttnUpBlock2D", "CrossAttnUpBlock2D"),
        only_cross_attention=False,
        block_out_channels: Tuple[int, ...] = (320, 640, 1280, 1280),
        layers_per_block=2,
        downsample_padding: int = 1,
        mid_block_scale_factor: float = 1,
        act_fn: str = "silu",
        norm_num_groups: Optional[int] = 32,
        norm_eps: float = 1e-5,
        cross_attention_dim=1280,
        attention_head_dim=8,
        dual_cross_attention: bool = False,
        use_linear_projection: bool = False,
        class_embed_type: Optional[str] = None,
        num_class_embeds: Optional[int] = None,
        upcast_attention: bool = False,
        resnet_time_scale_shift: str = "default",
        **unused,
    ):
        super().__init__()
        self.config = SimpleNamespace(**{k: v for k, v in locals().items() if k not in ("self", "unused", "__class__")})
        unsupported = _sd15_unsupported(self.config, "2D")
        if mid_block_type != "UNetMidBlock2DCrossAttn" or only_cross_attention or norm_num_groups is None:
            unsupported.append("mid_block_type / only_cross_attention / norm_num_groups=None")
        if unsupported:
            raise NotImplementedError("humanvid_b200.UNet2DConditionModel implements the SD1.5 reference-UNet layout only; unsupported: " + "; ".join(unsupported))
        self.sample_size = sample_size
        self.in_channels = in_channels
        _build_sd15_unet(self, in_channels, list(block_out_channels), cross_attention_dim, norm_num_groups, block_cls=BasicTransformerBlock)
        self._ref_write = False

    # ---- banks (ReferenceAttentionControl, write side) ---------------------------------------------------------
    def writer_blocks(self) -> List[Tuple[BasicTransformerBlock, int]]:
        """(block, level) in ``update()`` order: DFS(down_blocks, up_blocks, mid_block), stable sort by descending width."""
        out = []
        for i, b in enumerate(self.down_blocks):
            for a in getattr(b, "attentions", []):
                out.append((a.transformer_blocks[0], i))
        for i, b in enumerate(self.up_blocks):
            for a in getattr(b, "attentions", []):
                out.append((a.transformer_blocks[0], 3 - i))
        out.append((self.mid_block.attentions[0].transformer_blocks[0], 3))
        return sorted(out, key=lambda t: -t[0].norm1.normalized_shape[0])

    def _hv_config(self):
        return _sd15_hv_config(self.config, N.HV_KIND_UNET2D_REF)

    @torch.no_grad()
    def forward(self, sample: torch.Tensor, timestep: Union[torch.Tensor, float, int], encoder_hidden_states: torch.Tensor,
                class_labels: Optional[torch.Tensor] = None, timestep_cond=None, attention_mask=None, cross_attention_kwargs=None,
                added_cond_kwargs=None, down_block_additional_residuals=None, mid_block_additional_residual=None,
                down_intrablock_additional_residuals=None, encoder_attention_mask=None, return_dict: bool = True):
        if any(v is not None for v in (class_labels, timestep_cond, attention_mask, cross_attention_kwargs, added_cond_kwargs, down_block_additional_residuals,
                                       mid_block_additional_residual, down_intrablock_additional_residuals, encoder_attention_mask)):
            raise NotImplementedError("only (sample, timestep, encoder_hidden_states) are part of the CamAnimate reference-UNet call")
        if sample.dim() != 4:
            raise ValueError(f"Expected sample to have ndim=4 (b c h w), got {sample.dim()}")
        B, Cc, H, W = sample.shape
        if Cc != self.in_channels:
            raise ValueError(f"sample has {Cc} channels, model expects {self.in_channels}")
        h = self._sync_native()
        x = self._as_half(sample, "sample")
        ehs = self._as_half(encoder_hidden_states, "encoder_hidden_states")
        if ehs.shape[0] != B or ehs.shape[1] != 1:
            raise ValueError(f"encoder_hidden_states must be (batch, 1, dim) with batch {B}; got {tuple(ehs.shape)}")
        t = int(timestep.reshape(-1)[0].item()) if torch.is_tensor(timestep) else int(timestep)
        blocks = self.writer_blocks()
        banks = [torch.empty((B, (H >> lvl) * (W >> lvl), blk.norm1.normalized_shape[0]), device=x.device, dtype=torch.float16) for blk, lvl in blocks]
        hidden = torch.empty((B, self.config.block_out_channels[0], H, W), device=x.device, dtype=torch.float16)
        ptrs = (C.c_void_p * len(banks))(*[b.data_ptr() for b in banks])
        self._run(N.lib().hv_unet2d_reference_forward, h, (B, 1, H, W), N.ptr(x), N.i64(t), N.ptr(ehs), N.ptr(hidden), ptrs, N.i32(len(banks)),
                  N.i32(B), N.i32(H), N.i32(W))
        if self._ref_write:
            for (blk, _), bank in zip(blocks, banks):
                blk.bank.append(bank)
        hidden = self._from_half(hidden, sample.dtype)
        if not return_dict:
            return (hidden,)
        return UNet2DConditionOutput(sample=hidden)

    @classmethod
    def from_pretrained(cls, pretrained_model_path, subfolder=None, **kwargs):
        """diffusers-style loader (scripts/pose2vid.py:72-75): ``<path>/<subfolder>/config.json`` + ``diffusion_pytorch_model.{safetensors,bin}``."""
        return _from_pretrained(cls, pretrained_model_path, subfolder)   # SD checkpoints also carry conv_norm_out / conv_out, unused by the reference UNet


# --------------------------------------------------------------------------------------------- PoseGuider
class PoseGuider(_NativeNet):
    """Drop-in for src/models/pose_guider.py:16-61."""

    def __init__(self, conditioning_embedding_channels: int, conditioning_channels: int = 3, block_out_channels: Tuple[int, ...] = (16, 32, 64, 128)):
        super().__init__()
        if len(block_out_channels) != 4:
            raise NotImplementedError("PoseGuider with 4 resolution levels only")
        ch = list(block_out_channels)
        self._cfg = (conditioning_embedding_channels, conditioning_channels, ch)
        self.conv_in = _conv(conditioning_channels, ch[0], 3, padding=1)
        self.blocks = nn.ModuleList([])
        for a, b in zip(ch[:-1], ch[1:]):
            self.blocks.append(_conv(a, a, 3, padding=1))
            self.blocks.append(_conv(a, b, 3, padding=1, stride=2))
        self.conv_out = _conv(ch[-1], conditioning_embedding_channels, 3, padding=1)
        nn.init.zeros_(self.conv_out.weight)  # zero_module (pose_guider.py:42)
        nn.init.zeros_(self.conv_out.bias)

    def _hv_config(self):
        out, cin, ch = self._cfg
        cfg = HvConfig()
        cfg.kind = N.HV_KIND_POSE_GUIDER
        cfg.pg_cond_channels, cfg.pg_out_channels = cin, out
        cfg.pg_block_channels = (C.c_int32 * 4)(*ch)
        cfg.norm_groups = 32
        return cfg

    @torch.no_grad()
    def forward(self, conditioning: torch.Tensor) -> torch.Tensor:
        if conditioning.dim() != 5:
            raise ValueError("conditioning must be (b, c, f, h, w)")
        B, Cc, F, H, W = conditioning.shape
        h = self._sync_native()
        x = self._as_half(conditioning, "conditioning")
        out = torch.empty((B, self._cfg[0], F, H // 8, W // 8), device=x.device, dtype=torch.float16)
        self._run(N.lib().hv_pose_guider_forward, h, (B, F, H, W), N.ptr(x), N.ptr(out), N.i32(B), N.i32(F), N.i32(H), N.i32(W))
        return self._from_half(out, conditioning.dtype)


# --------------------------------------------------------------------------------------------- CameraPoseEncoder
class _CamResnet(_Shell):
    def __init__(self, ch, ksize):
        super().__init__()
        self.block1 = _conv(ch, ch, 3, padding=1)
        self.block2 = _conv(ch, ch, ksize, padding=ksize // 2)


class CameraPoseEncoder(_NativeNet):
    """Drop-in for src/cameractrl/pose_adaptor.py:160-248 with configs/inference/inference_v2.yaml pose_encoder_kwargs."""

    def __init__(self, downscale_factor, channels=(320, 640, 1280, 1280), nums_rb=3, cin=64, ksize=3, sk=False, use_conv=True,
                 compression_factor=1, temporal_attention_nhead=8, attention_block_types=("Temporal_Self",), temporal_position_encoding=False,
                 temporal_position_encoding_max_len=16, rescale_output_factor=1.0):
        super().__init__()
        channels = list(channels)
        if len(channels) != 1 or ksize != 1 or not sk or compression_factor != 1 or tuple(attention_block_types) != ("Temporal_Self",) \
                or not temporal_position_encoding or rescale_output_factor != 1.0:
            raise NotImplementedError("CameraPoseEncoder: only the inference_v2.yaml layout (one level, ksize=1, sk=True, Temporal_Self + PE) is implemented")
        c = channels[0]
        self._cfg = dict(downscale=downscale_factor, cin=cin, c=c, nums_rb=nums_rb, heads=temporal_attention_nhead, max_len=temporal_position_encoding_max_len)
        self.channels = channels
        self.nums_rb = nums_rb
        self.encoder_down_conv_blocks = nn.ModuleList([nn.ModuleList([_CamResnet(c, ksize) for _ in range(nums_rb)])])
        att = []
        for _ in range(nums_rb):
            blk = _Shell()
            blk.attention_blocks = nn.ModuleList([_TemporalAttention(c, temporal_position_encoding_max_len)])
            blk.norms = nn.ModuleList([nn.LayerNorm(c)])
            blk.ff = _FeedForward(c)
            blk.ff_norm = nn.LayerNorm(c)
            att.append(blk)
        self.encoder_down_attention_blocks = nn.ModuleList([nn.ModuleList(att)])
        zc = _conv(c, c, 1, bias=False)
        nn.init.zeros_(zc.weight)
        self.zero_conv_layers = nn.ModuleList([zc])
        self.encoder_conv_in = _conv(cin, c, 3, padding=1)

    def _hv_config(self):
        d = self._cfg
        cfg = HvConfig()
        cfg.kind = N.HV_KIND_CAMERA_ENCODER
        cfg.cam_downscale, cfg.cam_cin, cfg.cam_channels = d["downscale"], d["cin"], d["c"]
        cfg.cam_nums_rb, cfg.cam_heads, cfg.cam_max_len = d["nums_rb"], d["heads"], d["max_len"]
        cfg.heads = d["heads"]
        cfg.norm_groups = 32
        return cfg

    @torch.no_grad()
    def forward(self, x: torch.Tensor) -> List[torch.Tensor]:
        if x.dim() != 5:
            raise ValueError("plucker embedding must be (b, c, f, h, w)")
        B, Cc, F, H, W = x.shape
        r = self._cfg["downscale"]
        if Cc * r * r != self._cfg["cin"]:
            raise ValueError(f"plucker embedding has {Cc} channels; encoder expects {self._cfg['cin'] // (r * r)}")
        h = self._sync_native()
        xin = self._as_half(x, "plucker embedding")
        out = torch.empty((B * F, self._cfg["c"], H // r, W // r), device=xin.device, dtype=torch.float16)
        self._run(N.lib().hv_camera_encoder_forward, h, (B, F, H, W), N.ptr(xin), N.ptr(out), N.i32(B), N.i32(F), N.i32(H), N.i32(W))
        return [self._from_half(out, x.dtype)]


    @torch.no_grad()
    def forward_cameras(self, intrinsics: torch.Tensor, c2w: torch.Tensor, height: int, width: int) -> List[torch.Tensor]:
        """``forward(ray_condition(intrinsics, c2w, height, width) as (b, 6, f, h, w))`` without building the embedding
        (SURVEY 8f-3): intrinsics (b, f, 4) in pixels, c2w (b, f, 4, 4), see humanvid_b200.camera.relative_cameras."""
        if intrinsics.dim() != 3 or intrinsics.shape[-1] != 4 or c2w.shape != (*intrinsics.shape[:2], 4, 4):
            raise ValueError("intrinsics must be (b, f, 4) and c2w (b, f, 4, 4)")
        B, F = intrinsics.shape[:2]
        r = self._cfg["downscale"]
        if self._cfg["cin"] != 6 * r * r:
            raise ValueError("the Plucker producer feeds a 6-channel encoder")
        h = self._sync_native()
        dev = self.device
        K = intrinsics.to(dev, torch.float32).contiguous()
        M = c2w.to(dev, torch.float32).contiguous()
        out = torch.empty((B * F, self._cfg["c"], height // r, width // r), device=dev, dtype=torch.float16)
        self._run(N.lib().hv_camera_encoder_forward_rays, h, (B, F, height, width), N.ptr(K), N.ptr(M), N.ptr(out), N.i32(B), N.i32(F),
                  N.i32(height), N.i32(width))
        return [self._from_half(out, self.dtype)]


# --------------------------------------------------------------------------------------------- ReferenceAttentionControl (reader)
class ReferenceAttentionControl:
    """src/models/mutual_self_attention.py for the native UNets: same constructor keywords / ``update(writer)`` / ``clear()``.

    ``mode="read"`` wraps a native ``UNet3DConditionModel`` (the denoising UNet): ``update`` hands the banks to the native
    attention kernel, which reads them as a second key/value segment (the reference monkey-patches every block's forward
    and concatenates).  ``mode="write"`` wraps a native ``UNet2DConditionModel`` (the reference UNet): its next forward
    leaves every block's LayerNorm-1 output in ``block.bank``.  ``update`` also accepts the reference's own PyTorch writer
    (anything exposing ``.unet`` whose transformer blocks carry ``norm1`` and a ``bank`` list); banks are matched in the
    same sorted order (mutual_self_attention.py:302-339).
    """

    def __init__(self, unet, mode="read", do_classifier_free_guidance=False, attention_auto_machine_weight=float("inf"),
                 gn_auto_machine_weight=1.0, style_fidelity=1.0, reference_attn=True, reference_adain=False, fusion_blocks="midup",
                 batch_size=1):
        if mode not in ("read", "write"):
            raise ValueError("mode must be 'read' or 'write'")
        if fusion_blocks != "full" or reference_adain or not reference_attn:
            raise NotImplementedError("only fusion_blocks='full', reference_attn=True (what pipeline_pose2vid_long.py uses)")
        self.unet = unet
        self.mode = mode
        if mode == "read":
            if not isinstance(unet, UNet3DConditionModel):
                raise TypeError("mode='read' needs a humanvid_b200.UNet3DConditionModel")
            unet._ref_cfg = bool(do_classifier_free_guidance)
            unet._reader_registered = True
            for m in unet.reader_blocks():
                m.bank = []
        else:
            if not isinstance(unet, UNet2DConditionModel):
                raise TypeError("mode='write' needs a humanvid_b200.UNet2DConditionModel (or use the reference's own writer around its PyTorch UNet)")
            unet._ref_write = True
            for m, _ in unet.writer_blocks():
                m.bank = []

    @staticmethod
    def _writer_blocks(writer):
        root = writer.unet if hasattr(writer, "unet") else writer
        if isinstance(root, UNet2DConditionModel):
            return [m for m, _ in root.writer_blocks()]
        mods = [m for m in _torch_dfs(root) if hasattr(m, "bank") and hasattr(m, "norm1") and hasattr(m, "attn1")]
        return sorted(mods, key=lambda m: -m.norm1.normalized_shape[0])

    def update(self, writer, dtype=torch.float16):
        if self.mode != "read":
            raise RuntimeError("update() is called on the reader")
        readers = self.unet.reader_blocks()
        writers = self._writer_blocks(writer)
        for r, w in zip(readers, writers):
            r.bank = [v.clone().to(dtype) for v in w.bank]

    def clear(self):
        if self.mode == "read":
            for r in self.unet.reader_blocks():
                r.bank.clear()
        else:
            for m, _ in self.unet.writer_blocks():
                m.bank.clear()


# --------------------------------------------------------------------------------------------- AutoencoderKL
class _VaeResnet(_Shell):
    """diffusers ResnetBlock2D with temb_channels=None (no time_emb_proj), GroupNorm eps 1e-6."""

    def __init__(self, cin, cout, groups):
        super().__init__()
        self.norm1 = nn.GroupNorm(groups, cin, eps=1e-6)
        self.conv1 = _conv(cin, cout, 3, padding=1)
        self.norm2 = nn.GroupNorm(groups, cout, eps=1e-6)
        self.conv2 = _conv(cout, cout, 3, padding=1)
        if cin != cout:
            self.conv_shortcut = _conv(cin, cout, 1)


class _VaeAttention(_Shell):
    """diffusers Attention of the VAE mid block: group_norm, to_q / to_k / to_v WITH bias, one head, to_out.0."""

    def __init__(self, ch, groups):
        super().__init__()
        self.group_norm = nn.GroupNorm(groups, ch, eps=1e-6)
        self.to_q = nn.Linear(ch, ch)
        self.to_k = nn.Linear(ch, ch)
        self.to_v = nn.Linear(ch, ch)
        self.to_out = nn.ModuleList([nn.Linear(ch, ch), nn.Dropout(0.0)])


class _VaeDownsample(_Shell):
    """Downsample2D(use_conv=True, padding=0): F.pad(x, (0, 1, 0, 1)) then a 3x3 stride-2 conv."""

    def __init__(self, ch):
        super().__init__()
        self.conv = _conv(ch, ch, 3, stride=2, padding=0)


class _VaeBlock(_Shell):
    def __init__(self, cin, cout, n, groups, sampler=None):
        super().__init__()
        self.resnets = nn.ModuleList([_VaeResnet(cin if j == 0 else cout, cout, groups) for j in range(n)])
        if sampler == "down":
            self.downsamplers = nn.ModuleList([_VaeDownsample(cout)])
        elif sampler == "up":
            self.upsamplers = nn.ModuleList([_Sampler(cout, 1)])


class _VaeMid(_Shell):
    def __init__(self, ch, groups):
        super().__init__()
        self.attentions = nn.ModuleList([_VaeAttention(ch, groups)])
        self.resnets = nn.ModuleList([_VaeResnet(ch, ch, groups), _VaeResnet(ch, ch, groups)])


class _VaeEncoder(_Shell):
    def __init__(self, cin, ch, latent, groups, layers):
        super().__init__()
        self.conv_in = _conv(cin, ch[0], 3, padding=1)
        self.down_blocks = nn.ModuleList([_VaeBlock(ch[max(i - 1, 0)], c, layers, groups, "down" if i < len(ch) - 1 else None) for i, c in enumerate(ch)])
        self.mid_block = _VaeMid(ch[-1], groups)
        self.conv_norm_out = nn.GroupNorm(groups, ch[-1], eps=1e-6)
        self.conv_out = _conv(ch[-1], 2 * latent, 3, padding=1)


class _VaeDecoder(_Shell):
    def __init__(self, cout, ch, latent, groups, layers):
        super().__init__()
        rev = list(ch)[::-1]
        self.conv_in = _conv(latent, rev[0], 3, padding=1)
        self.mid_block = _VaeMid(rev[0], groups)
        self.up_blocks = nn.ModuleList([_VaeBlock(rev[max(i - 1, 0)], c, layers + 1, groups, "up" if i < len(rev) - 1 else None) for i, c in enumerate(rev)])
        self.conv_norm_out = nn.GroupNorm(groups, ch[0], eps=1e-6)
        self.conv_out = _conv(ch[0], cout, 3, padding=1)


class DiagonalGaussianDistribution:
    """The posterior ``encode`` returns: ``moments`` = [mean | logvar] over the channel axis (diffusers' class of the same name; what the
    pipelines read is ``mean``)."""

    def __init__(self, parameters: torch.Tensor):
        self.parameters = parameters
        self.mean, logvar = torch.chunk(parameters, 2, dim=1)
        self.logvar = torch.clamp(logvar, -30.0, 20.0)

    @property
    def std(self):
        return torch.exp(0.5 * self.logvar)

    @property
    def var(self):
        return torch.exp(self.logvar)

    def mode(self):
        return self.mean


@dataclass
class AutoencoderKLOutput:
    latent_dist: DiagonalGaussianDistribution


@dataclass
class DecoderOutput:
    sample: torch.Tensor


# attention parameter names of diffusers < 0.14 checkpoints -> the current ones (diffusers converts them the same way on load)
_VAE_LEGACY_ATTN = {"query": "to_q", "key": "to_k", "value": "to_v", "proj_attn": "to_out.0"}


def _convert_legacy_vae_keys(state):
    out = {}
    for k, v in state.items():
        parts = k.split(".")
        if len(parts) == 6 and parts[0] in ("encoder", "decoder") and parts[1:4] == ["mid_block", "attentions", "0"] and parts[4] in _VAE_LEGACY_ATTN:
            k = ".".join(parts[:4] + [_VAE_LEGACY_ATTN[parts[4]], parts[5]])
            if parts[5] == "weight" and v.dim() == 4:   # stored as a 1x1 conv
                v = v[:, :, 0, 0]
        out[k] = v
    return out


class AutoencoderKL(_NativeNet):
    """Drop-in for diffusers' ``AutoencoderKL`` (0.24) in the SD layout that configs/prompts/stage2.yaml points at (sd-vae-ft-mse):
    same constructor keywords, ``config``, ``state_dict`` keys, ``from_pretrained``, ``encode(x).latent_dist.mean`` and
    ``decode(z).sample``.  Both run on libhv_b200 (``hv_vae_encode`` / ``hv_vae_decode``); every frame of a call is computed independently of
    the others.  Inference only: no tiling / slicing, no ``latent_dist.sample()``.
    """

    def __init__(
        self,
        in_channels: int = 3,
        out_channels: int = 3,
        down_block_types: Tuple[str, ...] = ("DownEncoderBlock2D",) * 4,
        up_block_types: Tuple[str, ...] = ("UpDecoderBlock2D",) * 4,
        block_out_channels: Tuple[int, ...] = (128, 256, 512, 512),
        layers_per_block: int = 2,
        act_fn: str = "silu",
        latent_channels: int = 4,
        norm_num_groups: int = 32,
        sample_size: int = 512,
        scaling_factor: float = 0.18215,
        force_upcast: bool = True,
        **unused,
    ):
        super().__init__()
        unsupported = []
        if tuple(down_block_types) != ("DownEncoderBlock2D",) * 4 or tuple(up_block_types) != ("UpDecoderBlock2D",) * 4:
            unsupported.append(f"block types {tuple(down_block_types)} / {tuple(up_block_types)} (4 x DownEncoderBlock2D / UpDecoderBlock2D)")
        if tuple(block_out_channels) != (128, 256, 512, 512):
            unsupported.append(f"block_out_channels {tuple(block_out_channels)} (128, 256, 512, 512)")
        if layers_per_block != 2:
            unsupported.append(f"layers_per_block {layers_per_block} (2)")
        if act_fn not in ("silu", "swish"):
            unsupported.append(f"act_fn {act_fn!r} (silu)")
        if norm_num_groups != 32:
            unsupported.append(f"norm_num_groups {norm_num_groups} (32)")
        if latent_channels != 4:
            unsupported.append(f"latent_channels {latent_channels} (4)")
        if not (1 <= in_channels <= 64 and 1 <= out_channels <= 64):
            unsupported.append(f"in_channels / out_channels {in_channels} / {out_channels} (1..64)")
        if unsupported:
            raise NotImplementedError("humanvid_b200.AutoencoderKL implements the SD VAE layout only; unsupported: " + "; ".join(unsupported))
        self.config = SimpleNamespace(in_channels=in_channels, out_channels=out_channels, down_block_types=tuple(down_block_types),
                                      up_block_types=tuple(up_block_types), block_out_channels=tuple(block_out_channels),
                                      layers_per_block=layers_per_block, act_fn=act_fn, latent_channels=latent_channels,
                                      norm_num_groups=norm_num_groups, sample_size=sample_size, scaling_factor=scaling_factor,
                                      force_upcast=force_upcast)
        ch = list(block_out_channels)
        self.encoder = _VaeEncoder(in_channels, ch, latent_channels, norm_num_groups, layers_per_block)
        self.decoder = _VaeDecoder(out_channels, ch, latent_channels, norm_num_groups, layers_per_block)
        self.quant_conv = _conv(2 * latent_channels, 2 * latent_channels, 1)
        self.post_quant_conv = _conv(latent_channels, latent_channels, 1)

    def _hv_config(self):
        c = self.config
        cfg = HvConfig()
        cfg.kind = N.HV_KIND_VAE
        cfg.in_channels, cfg.out_channels = c.in_channels, c.out_channels
        cfg.block_out_channels = (C.c_int32 * 4)(*c.block_out_channels)
        cfg.norm_groups = c.norm_num_groups
        cfg.vae_latent_channels = c.latent_channels
        return cfg

    def load_state_dict(self, state_dict, *a, **k):
        """Also accepts the mid-block attention names written before diffusers 0.14 (query / key / value / proj_attn)."""
        return super().load_state_dict(_convert_legacy_vae_keys(state_dict), *a, **k)

    def workspace_bytes(self, n, h, w) -> int:
        """Device workspace of decoding n latents of h x w and of encoding n images of 8h x 8w."""
        return self._workspace_bytes(n, 1, h, w)

    def reserve_workspace(self, n, h, w):
        """Grow the native workspace for n latents of h x w (and n images of 8h x 8w) now, e.g. before capturing a CUDA graph."""
        self._reserve(self._sync_native(), n, 1, h, w)

    @torch.no_grad()
    def encode(self, x: torch.Tensor, return_dict: bool = True):
        if x.dim() != 4:
            raise ValueError(f"Expected x to have ndim=4 (n c h w), got {x.dim()}")
        B, Cc, H, W = x.shape
        if Cc != self.config.in_channels:
            raise ValueError(f"image has {Cc} channels, model expects {self.config.in_channels}")
        if B == 0 or H % 8 or W % 8:
            raise ValueError(f"encode needs a non-empty batch of images whose sides are multiples of 8; got {tuple(x.shape)}")
        h = self._sync_native()
        xin = self._as_half(x, "image")
        moments = torch.empty((B, 2 * self.config.latent_channels, H // 8, W // 8), device=xin.device, dtype=torch.float16)
        self._run(N.lib().hv_vae_encode, h, (B, 1, H // 8, W // 8), N.ptr(xin), N.ptr(moments), N.i32(B), N.i32(H), N.i32(W))
        dist = DiagonalGaussianDistribution(self._from_half(moments, x.dtype))
        if not return_dict:
            return (dist,)
        return AutoencoderKLOutput(latent_dist=dist)

    @torch.no_grad()
    def decode(self, z: torch.Tensor, return_dict: bool = True, generator=None):
        if z.dim() != 4:
            raise ValueError(f"Expected z to have ndim=4 (n c h w), got {z.dim()}")
        B, Cc, H, W = z.shape
        if Cc != self.config.latent_channels:
            raise ValueError(f"latents have {Cc} channels, model expects {self.config.latent_channels}")
        if B == 0:
            raise ValueError("decode needs a non-empty batch")
        h = self._sync_native()
        zin = self._as_half(z, "latents")
        out = torch.empty((B, self.config.out_channels, 8 * H, 8 * W), device=zin.device, dtype=torch.float16)
        self._run(N.lib().hv_vae_decode, h, (B, 1, H, W), N.ptr(zin), N.ptr(out), N.i32(B), N.i32(H), N.i32(W))
        out = self._from_half(out, z.dtype)
        if not return_dict:
            return (out,)
        return DecoderOutput(sample=out)

    def forward(self, sample: torch.Tensor, sample_posterior: bool = False, return_dict: bool = True, generator=None):
        if sample_posterior:
            raise NotImplementedError("sampling the posterior is not implemented (inference uses its mean)")
        return self.decode(self.encode(sample).latent_dist.mode(), return_dict=return_dict)

    @classmethod
    def from_pretrained(cls, pretrained_model_path, subfolder=None, torch_dtype=None, **kwargs):
        """diffusers-style loader: ``<path>[/<subfolder>]/config.json`` + ``diffusion_pytorch_model.safetensors`` (or ``.bin``); old
        attention names are converted.  Builds on the CPU; move it with ``.to("cuda", torch.float16)``."""
        return _from_pretrained(cls, pretrained_model_path, subfolder, require_all=True, torch_dtype=torch_dtype)


# --------------------------------------------------------------------------------------------- CLIPVisionModelWithProjection
class _ClipEmbeddings(_Shell):
    def __init__(self, hidden, channels, image_size, patch_size):
        super().__init__()
        self.class_embedding = nn.Parameter(torch.zeros(hidden))
        self.patch_embedding = nn.Conv2d(channels, hidden, patch_size, stride=patch_size, bias=False)
        self.position_embedding = nn.Embedding((image_size // patch_size) ** 2 + 1, hidden)


class _ClipAttention(_Shell):
    def __init__(self, hidden):
        super().__init__()
        self.k_proj = nn.Linear(hidden, hidden)
        self.v_proj = nn.Linear(hidden, hidden)
        self.q_proj = nn.Linear(hidden, hidden)
        self.out_proj = nn.Linear(hidden, hidden)


class _ClipMLP(_Shell):
    def __init__(self, hidden, intermediate):
        super().__init__()
        self.fc1 = nn.Linear(hidden, intermediate)
        self.fc2 = nn.Linear(intermediate, hidden)


class _ClipEncoderLayer(_Shell):
    def __init__(self, hidden, intermediate, eps):
        super().__init__()
        self.self_attn = _ClipAttention(hidden)
        self.layer_norm1 = nn.LayerNorm(hidden, eps=eps)
        self.mlp = _ClipMLP(hidden, intermediate)
        self.layer_norm2 = nn.LayerNorm(hidden, eps=eps)


class _ClipEncoder(_Shell):
    def __init__(self, hidden, intermediate, layers, eps):
        super().__init__()
        self.layers = nn.ModuleList([_ClipEncoderLayer(hidden, intermediate, eps) for _ in range(layers)])


class _ClipVisionTransformer(_Shell):
    def __init__(self, c):
        super().__init__()
        self.embeddings = _ClipEmbeddings(c.hidden_size, c.num_channels, c.image_size, c.patch_size)
        self.pre_layrnorm = nn.LayerNorm(c.hidden_size, eps=c.layer_norm_eps)
        self.encoder = _ClipEncoder(c.hidden_size, c.intermediate_size, c.num_hidden_layers, c.layer_norm_eps)
        self.post_layernorm = nn.LayerNorm(c.hidden_size, eps=c.layer_norm_eps)


@dataclass
class CLIPVisionModelOutput:
    """transformers' output class of the same name: ``image_embeds`` (B, projection_dim), ``last_hidden_state`` (B, 1 + patches, hidden)."""

    image_embeds: torch.Tensor
    last_hidden_state: torch.Tensor
    hidden_states: Optional[tuple] = None
    attentions: Optional[tuple] = None

    def __getitem__(self, i):
        return self.to_tuple()[i]

    def to_tuple(self):
        return (self.image_embeds, self.last_hidden_state)


class CLIPVisionModelWithProjection(_NativeNet):
    """Drop-in for ``transformers.CLIPVisionModelWithProjection`` (the pipelines' image encoder): ``CLIPVisionConfig``'s keyword names and
    defaults, the same ``state_dict`` keys, ``from_pretrained``, and ``model(pixel_values).image_embeds`` / ``.last_hidden_state``.  The forward
    runs on libhv_b200 (``hv_clip_vision_forward``); every image of a batch is computed independently of the others.  OpenAI CLIP ViTs are
    supported: quick-GELU MLPs, heads of dimension 64, RGB input.  Inference only.
    """

    def __init__(
        self,
        hidden_size: int = 768,
        intermediate_size: int = 3072,
        projection_dim: int = 512,
        num_hidden_layers: int = 12,
        num_attention_heads: int = 12,
        num_channels: int = 3,
        image_size: int = 224,
        patch_size: int = 32,
        hidden_act: str = "quick_gelu",
        layer_norm_eps: float = 1e-5,
        attention_dropout: float = 0.0,
        initializer_range: float = 0.02,
        initializer_factor: float = 1.0,
        **unused,
    ):
        super().__init__()
        unsupported = []
        if hidden_act != "quick_gelu":
            unsupported.append(f"hidden_act {hidden_act!r} (quick_gelu)")
        if num_attention_heads <= 0 or hidden_size != 64 * num_attention_heads:
            unsupported.append(f"head dim hidden_size / num_attention_heads = {hidden_size} / {num_attention_heads} (64)")
        if hidden_size > 1280:
            unsupported.append(f"hidden_size {hidden_size} (<= 1280)")
        if intermediate_size <= 0 or intermediate_size % 8:
            unsupported.append(f"intermediate_size {intermediate_size} (a positive multiple of 8)")
        if num_channels != 3:
            unsupported.append(f"num_channels {num_channels} (3)")
        if patch_size <= 0 or image_size <= 0 or image_size % patch_size:
            unsupported.append(f"image_size {image_size} not a multiple of patch_size {patch_size}")
        if unsupported:
            raise NotImplementedError("humanvid_b200.CLIPVisionModelWithProjection implements OpenAI CLIP ViTs only; unsupported: " + "; ".join(unsupported))
        self.config = SimpleNamespace(hidden_size=hidden_size, intermediate_size=intermediate_size, projection_dim=projection_dim,
                                      num_hidden_layers=num_hidden_layers, num_attention_heads=num_attention_heads, num_channels=num_channels,
                                      image_size=image_size, patch_size=patch_size, hidden_act=hidden_act, layer_norm_eps=layer_norm_eps,
                                      attention_dropout=attention_dropout, initializer_range=initializer_range,
                                      initializer_factor=initializer_factor, model_type="clip_vision_model")
        self.vision_model = _ClipVisionTransformer(self.config)
        self.visual_projection = nn.Linear(hidden_size, projection_dim, bias=False)

    def _hv_config(self):
        c = self.config
        cfg = HvConfig()
        cfg.kind = N.HV_KIND_CLIP_VISION
        cfg.clip_hidden_size, cfg.clip_layers, cfg.clip_heads = c.hidden_size, c.num_hidden_layers, c.num_attention_heads
        cfg.clip_intermediate_size, cfg.clip_patch_size, cfg.clip_image_size = c.intermediate_size, c.patch_size, c.image_size
        cfg.clip_projection_dim, cfg.clip_layer_norm_eps = c.projection_dim, c.layer_norm_eps
        return cfg

    def load_state_dict(self, state_dict, *a, **k):
        """Also accepts checkpoints that carry the ``position_ids`` buffer older transformers versions saved."""
        return super().load_state_dict({n: v for n, v in state_dict.items() if not n.endswith("embeddings.position_ids")}, *a, **k)

    def workspace_bytes(self, batch) -> int:
        """Device workspace of one forward over `batch` images."""
        s = self.config.image_size
        return self._workspace_bytes(batch, 1, s, s)

    def reserve_workspace(self, batch):
        """Grow the native workspace for `batch` images now, e.g. before capturing a CUDA graph."""
        s = self.config.image_size
        self._reserve(self._sync_native(), batch, 1, s, s)

    @torch.no_grad()
    def forward(self, pixel_values: torch.Tensor, output_attentions: Optional[bool] = None, output_hidden_states: Optional[bool] = None,
                interpolate_pos_encoding: bool = False, return_dict: Optional[bool] = None):
        if output_attentions or output_hidden_states:
            raise NotImplementedError("humanvid_b200.CLIPVisionModelWithProjection returns image_embeds and last_hidden_state only "
                                      "(output_attentions / output_hidden_states are not implemented)")
        if interpolate_pos_encoding:
            raise NotImplementedError("interpolate_pos_encoding=True is not implemented (the model takes image_size x image_size pixels)")
        c = self.config
        if pixel_values.dim() != 4 or pixel_values.shape[1] != c.num_channels:
            raise ValueError(f"pixel_values must be (batch, {c.num_channels}, height, width), got {tuple(pixel_values.shape)}")
        B, _, H, W = pixel_values.shape
        if H != c.image_size or W != c.image_size:
            raise ValueError(f"Input image size ({H}*{W}) doesn't match model ({c.image_size}*{c.image_size}).")
        if B == 0:
            raise ValueError("pixel_values is an empty batch")
        h = self._sync_native()
        pix = self._as_half(pixel_values, "pixel_values")
        embeds = torch.empty((B, c.projection_dim), device=pix.device, dtype=torch.float16)
        hidden = torch.empty((B, (c.image_size // c.patch_size) ** 2 + 1, c.hidden_size), device=pix.device, dtype=torch.float16)
        self._run(N.lib().hv_clip_vision_forward, h, (B, 1, c.image_size, c.image_size), N.ptr(pix), N.ptr(embeds), N.ptr(hidden), N.i32(B))
        dtype = self.dtype
        embeds, hidden = self._from_half(embeds, dtype), self._from_half(hidden, dtype)
        if return_dict is False:
            return (embeds, hidden)
        return CLIPVisionModelOutput(image_embeds=embeds, last_hidden_state=hidden)

    @classmethod
    def from_pretrained(cls, pretrained_model_path, subfolder=None, torch_dtype=None, **kwargs):
        """transformers-style loader: ``<path>[/<subfolder>]/config.json`` (a ``clip_vision_model`` config) + ``model.safetensors`` (or
        ``pytorch_model.bin``).  Builds on the CPU; move it with ``.to("cuda", torch.float16)``."""
        return _from_pretrained(cls, pretrained_model_path, subfolder, weights=("model.safetensors", "pytorch_model.bin"), require_all=True,
                                torch_dtype=torch_dtype)
