"""Per-slice, per-row and per-element checks of one native block's output against a high-precision reference, shared by
tests/test_block_parity_gpu.py (native taps of the whole UNet), tests/test_net_block_parity_gpu.py (the VAE, CLIP, PoseGuider and camera
encoder) and the CPU self-tests tests/test_block_parity_cpu.py and tests/test_net_block_parity_cpu.py.

A tap is (NF, H, W, C): NF = batch items x frames.  A slice s is one (item, frame), all H W C elements; a row r one token of it.  For a
block whose output N and the fp16 eager result E are compared with the fp64 result R of the same block on the same input:

    slice    rel_s(N, R) <= 1e-3  and  rel_s(N, R) <= max(1.25 rel_s(E, R), 2^-12)
    row      ||N_r - R_r|| <= 2^-8 (||R_r|| + rms_r(R))          rms_r(R) = the rms over the slice's rows of ||R_r||
    element  |N - R| <= 2^-6 (|R| + rms_s(R))                    rms_s(R) = the rms of the slice's elements

The slice bound is the per-tensor target (one fp16 rounding of the output, about 2^-12, plus the block's fp32 arithmetic) asked of every
frame, and no worse than the reference's own fp16 path on the same input.  The row bound is four times the per-tensor target on one token:
it fails a wrong query row -- the last row of a partial key tile, the first row after a frame boundary -- that one slice's L2 dilutes.  The
element bound allows a few fp16 roundings of the element's magnitude or of the slice's scale; a wrong key, bank item, frame or GroupNorm
group moves elements by O(|R|) and fails it.

For a block whose feed-forward runs on e4m3 (FP8 mode) R is replaced by the e4m3 emulation Emu in fp64 and the slice bound is the flip
budget of tests/test_fp8_model_gpu.py, rel_s(N8, Emu) <= 0.6 rel_s(Emu, R) + 2^-10; the row and element bounds add ``extra`` (see
tests/fp8_emulation.ff_flip_bound).  That term is the worst case of every GEGLU value of a token flipping at once, far above what flips
do, so for these blocks the slice budget is the tight check and the row and element bounds catch only gross faults.

A tap whose layout carries padding channels (the 64-channel input of an implicit-GEMM conv, a conv output rounded up to 8 channels) is
compared on its true channels, and every padding channel must be exactly zero (check_pad).
"""
from dataclasses import dataclass, field

import torch

REL_MAX = 1e-3            # per-tensor target, asked per slice
REL_FLOOR = 2.0 ** -12    # below it, "no worse than fp16 eager" is rounding noise either way
ROW_K = 2.0 ** -8
ELEM_K = 2.0 ** -6
FP8_FLIP = 0.6            # share of the emulation's own error the native FP8 path may add by flipped e4m3 roundings
FP8_FLOOR = 2.0 ** -10


def _slices(t):
    return t.reshape(t.shape[0], -1, t.shape[-1]).double()      # (NF, L, C)


def slice_rel(a, r):
    """rel_s(a, r) per slice: (NF,) fp64."""
    a, r = _slices(a), _slices(r)
    return (a - r).flatten(1).norm(dim=1) / r.flatten(1).norm(dim=1).clamp_min(1e-300)


def row_ratio(a, r, extra=None):
    """||a_r - r_r|| / (2^-8 (||r_r|| + rms_r(r)) + ||extra_r||) per row: (NF, L)."""
    a, r = _slices(a), _slices(r)
    rn = r.norm(dim=2)
    bound = ROW_K * (rn + rn.pow(2).mean(1, keepdim=True).sqrt())
    if extra is not None:
        bound = bound + _slices(extra).norm(dim=2)
    return (a - r).norm(dim=2) / bound.clamp_min(1e-300)


def elem_ratio(a, r, extra=None):
    """|a - r| / (2^-6 (|r| + rms_s(r)) + extra) per element: (NF, L, C)."""
    a, r = _slices(a), _slices(r)
    bound = ELEM_K * (r.abs() + r.pow(2).mean((1, 2), keepdim=True).sqrt())
    if extra is not None:
        bound = bound + _slices(extra)
    return (a - r).abs() / bound.clamp_min(1e-300)


@dataclass
class Worst:
    """Worst err/bound ratio of one check and where it is: (tap, slice[, row[, channel]])."""
    ratio: float = 0.0
    where: tuple = ()

    def take(self, ratios, label):
        v, i = ratios.flatten().max(0)
        if float(v) > self.ratio or not self.where:
            idx = list(torch.unravel_index(i, ratios.shape))
            self.ratio, self.where = float(v), (label, *[int(j) for j in idx])


@dataclass
class BlockReport:
    """The worst ratio of each bound over the blocks fed to it."""
    slice: Worst = field(default_factory=Worst)
    row: Worst = field(default_factory=Worst)
    elem: Worst = field(default_factory=Worst)
    e_row: Worst = field(default_factory=Worst)     # the fp16 eager result against the row and element bounds
    e_elem: Worst = field(default_factory=Worst)
    nonfinite: list = field(default_factory=list)
    pad: list = field(default_factory=list)         # taps with a padding channel that is not exactly zero

    def worst(self):
        return max(self.slice.ratio, self.row.ratio, self.elem.ratio)

    def failures(self, with_eager=True):
        out = [f"non-finite output in {n}" for n in self.nonfinite] + [f"non-zero padding channel in {p}" for p in self.pad]
        checks = [("slice", self.slice), ("row", self.row), ("element", self.elem)]
        if with_eager:
            checks += [("fp16-eager row", self.e_row), ("fp16-eager element", self.e_elem)]
        for name, w in checks:
            if w.ratio > 1.0:
                out.append(f"{name} bound: err/bound {w.ratio:.3g} at {w.where[0]} (slice, row[, channel]) = {w.where[1:]}")
        return out


def check_fp16_block(rep: BlockReport, label: str, N, R, E=None):
    """Add one fp16 block's native output N to rep: the three bounds against the fp64 R; E (fp16 eager), when given, sets the slice
    bound's relative leg and is held to the row and element bounds too."""
    if not torch.isfinite(N).all():
        rep.nonfinite.append(label)
        return
    rn = slice_rel(N, R)
    cap = torch.full_like(rn, REL_MAX)
    if E is not None:
        cap = torch.minimum(cap, (1.25 * slice_rel(E, R)).clamp_min(REL_FLOOR))
        rep.e_row.take(row_ratio(E, R), label)
        rep.e_elem.take(elem_ratio(E, R), label)
    rep.slice.take(rn / cap, label)
    rep.row.take(row_ratio(N, R), label)
    rep.elem.take(elem_ratio(N, R), label)


def check_fp8_block(rep: BlockReport, label: str, N8, Emu, R, extra):
    """Add one e4m3 block's native output N8 to rep: the flip budget per slice against the fp64 emulation Emu, and the row and element
    bounds against Emu widened by ``extra`` (per element, the flip term of the block's e4m3 feed-forward)."""
    if not torch.isfinite(N8).all():
        rep.nonfinite.append(label)
        return
    rep.slice.take(slice_rel(N8, Emu) / (FP8_FLIP * slice_rel(Emu, R) + FP8_FLOOR), label)
    rep.row.take(row_ratio(N8, Emu, extra), label)
    rep.elem.take(elem_ratio(N8, Emu, extra), label)


def check_pad(rep: BlockReport, label: str, N, c: int):
    """Add the padding channels c.. of a native tap N (NF, H, W, C) to rep: each must be +0 or -0.  The next implicit-GEMM conv reads them
    through zero weight columns, and 0 * NaN or 0 * Inf would reach its real outputs."""
    bad = (N[..., c:] != 0).nonzero()                # NaN != 0 too
    if len(bad):
        n, h, w, ch = (int(i) for i in bad[0])
        rep.pad.append(f"{label} (slice, h, w, channel) = {(n, h, w, c + ch)}, {len(bad)} elements")


# tap names of the VAE, CLIP, PoseGuider and camera encoder that do not end in "<kind>.<index>": whole names, last components, prefixes
_NAMED = {"post_quant_conv": "conv1x1", "quant_conv": "conv1x1", "zero_conv_layers.0": "conv1x1", "vision_model.pre_layrnorm": "clip_embed",
          "vision_model.post_layernorm": "clip_pool"}
_LAST = {"conv_in": "conv_in", "encoder_conv_in": "conv_in", "conv_out": "conv_out", "conv_norm_out": "norm_out"}
_PREFIX = (("vision_model.encoder.layers.", "clip_layer"), ("blocks.", "pg_conv"), ("encoder_down_conv_blocks.", "cam_res"),
           ("encoder_down_attention_blocks.", "cam_attn"))


def block_kind(name: str) -> str:
    """The kind of a tap: conv_in, resnets, attentions, motion_modules, downsamplers, upsamplers (UNets, VAE), norm_out (GroupNorm + SiLU),
    conv_out, conv1x1, clip_embed, clip_layer, clip_pool, pg_conv (PoseGuider blocks), cam_res, cam_attn (camera encoder)."""
    if name in _NAMED:
        return _NAMED[name]
    last = name.rsplit(".", 1)[-1]
    if last in _LAST:
        return _LAST[last]
    for prefix, kind in _PREFIX:
        if name.startswith(prefix):
            return kind
    return name.split(".")[-2]
