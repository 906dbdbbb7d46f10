"""Every block of the native UNets against fp64 on its own input, per frame, per token row and per element (tests/block_parity.py).

One native forward per configuration copies every block's output out through the debug taps.  oracle/block_replay.py then applies the
oracle module of each block to the native taps of its predecessors -- the input the native block consumed -- three ways: in fp64 with the
fp16 weights upcast (R), in fp16 eager (E, the reference's deployment), and, in FP8 mode, in fp64 with the e4m3 quantise-dequantise steps
(Emu).  The native tap N of the block is held to the bounds of tests/block_parity.py against R (or Emu), and E to the row and element
bounds.  One oracle is held at a time and its dtype switched in place (the full-width fp64 copy is about 7 GB).

Configurations, at SD1.5 widths (320, 640, 1280, 1280), cross-attention dim 768 and 8 heads unless stated:
- v0 layout, CFG batch 2, no banks, latents 40x24 (5 frames) and 48x40 (3 frames): level-0 self-attention over 960 keys (a partial
  128-key tile) and 1920 (whole tiles), an odd 5x3 level-3 grid, the temporal attention's TMA kernel at d = 40 and at d = 80 (48x40) and
  its register kernel at d = 80 (40x24) and d = 160; the plans are read back from the library, not assumed.
- 16 reference banks, CFG on and off; with CFG on, every tap of the unconditional half equals the bank-free forward's bit for bit.
- a CFG batch of 4 with a 4-item bank (context_batch_size = 2): the frames of items 2 and 3 read bank items 2 and 3; at 16x8 the
  level-0 temporal attention runs the register kernel at d = 40.
- the inference_v1 layout (GroupNorm pooled over the window, no mid-block motion module, 24-row positional encoding), 24 frames, banks.
- FP8 mode, on the narrow (64, 128, 256, 1280) net and at full width: every tap before the first e4m3 feed-forward equals the fp16
  run's bit for bit, and the e4m3 blocks are checked against Emu.
- the reference ("writer") UNet2D at full width: its hidden taps, and every bank it writes per element against the oracle block's
  LayerNorm-1 output in fp64 on the native input.
- the narrow (64, 128, 256, 256) v0 net at the error ladder's 32x32, 6 frames.
"""
import ctypes as C
import time

import pytest
import torch

pytestmark = pytest.mark.gpu

from block_parity import BlockReport, block_kind, check_fp16_block, check_fp8_block
from conftest import report
from fp8_emulation import emulate_fp8_linears, ff_flip_bound
from unet_v1_oracle import V1_UNET_KWARGS, unet3d_v1

if torch.cuda.is_available():
    import humanvid_b200 as hv
    from humanvid_b200._native import check, i32, i64, lib
    from oracle import hv_oracle as O
    from oracle.block_replay import replay_blocks

SD, XDIM = (320, 640, 1280, 1280), 768
NARROW, NARROW_XDIM = (64, 128, 256, 256), 64
FP8_NARROW = (64, 128, 256, 1280)
T = 519
MM_KW = dict(num_attention_heads=8, num_transformer_block=1, attention_block_types=["Temporal_Self", "Temporal_Self"],
             temporal_position_encoding=True, temporal_position_encoding_max_len=32, temporal_attention_dim_div=1)
V0_KW = dict(use_motion_module=True, use_inflated_groupnorm=True, motion_module_resolutions=(1, 2, 4, 8), motion_module_mid_block=True,
             motion_module_type="Vanilla", motion_module_kwargs=MM_KW, unet_use_cross_frame_attention=False, unet_use_temporal_attention=False)


@pytest.fixture(scope="module", autouse=True)
def wall_time():
    t0 = time.time()
    yield
    report(f"block parity: file wall time {time.time() - t0:.0f} s on {torch.cuda.get_device_name()}")


# --------------------------------------------------------------------------------------------------------------- networks, inputs
def make_v0(chs, xdim, seed=7):
    """The oracle on the device in fp16 (so its fp64 copy holds the fp16-representable weights) and the native net with its weights."""
    ora = O.synthetic_init(O.UNet3DConditionModel(block_out_channels=chs, cross_attention_dim=xdim).eval(), seed=seed).half().cuda()
    nat = hv.UNet3DConditionModel(block_out_channels=chs, cross_attention_dim=xdim, **V0_KW)
    nat.load_state_dict(ora.state_dict())
    return ora, nat.to("cuda", torch.float16)


@pytest.fixture(scope="module")
def sd_v0():
    nets = make_v0(SD, XDIM)
    yield nets
    del nets
    torch.cuda.empty_cache()


def inputs(B, F, h, w, c0, xdim, seed=1, drift=0.0):
    g = torch.Generator(device="cuda").manual_seed(seed)
    x = torch.randn(B, 4, F, h, w, generator=g, device="cuda")
    x = (x + drift * torch.arange(F, device="cuda").view(1, 1, F, 1, 1)).half()
    ehs = torch.randn(B, 1, xdim, generator=g, device="cuda").half()
    ehs[: B // 2] = 0   # the uncond half, like the pipeline
    pose = (torch.randn(B, c0, F, h, w, generator=g, device="cuda") * 0.5).half()
    return x, ehs, pose


def make_banks(ora, B, h, w, seed=5):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return [torch.randn(B, l, c, generator=g, device="cuda").half() for (l, c) in O.bank_shapes(ora, h, w)]


class NativeBanks:
    """The reference banks on the native net (ReferenceAttentionControl read side) for the duration of a with block."""

    def __init__(self, nat, banks, cfg):
        self.nat, self.banks, self.cfg = nat, banks, cfg

    def __enter__(self):
        self.ctl = hv.ReferenceAttentionControl(self.nat, do_classifier_free_guidance=self.cfg, mode="read", fusion_blocks="full")
        for blk, bk in zip(self.nat.reader_blocks(), self.banks):
            blk.bank = [bk]

    def __exit__(self, *a):
        self.ctl.clear()


def native_taps(nat, x, ehs, pose, F):
    """(tap names in execution order, {name: (B*F, H, W, C) fp16}) of one native forward."""
    B, h, w = x.shape[0], x.shape[-2], x.shape[-1]
    plan = nat.debug_tap_plan(B, F, h, w)
    taps = [torch.empty(d, device="cuda", dtype=torch.float16) for _, d in plan]
    nat.debug_set_taps(taps)
    try:
        with torch.no_grad():
            if pose is None:
                nat(x, T, ehs, return_dict=False)
            else:
                nat(x, T, ehs, pose_cond_fea=pose, return_dict=False)
        torch.cuda.synchronize()
    finally:
        nat.debug_set_taps([])
    names = [n for n, _ in plan]
    return names, dict(zip(names, taps))


# --------------------------------------------------------------------------------------------------------------- the parity run
def e4m3_taps(ora, names):
    """{tap name: (feed-forward module, its block's proj_out weight as an (out, in) matrix)} for every block whose feed-forward FP8 mode
    runs on e4m3."""
    ffs = {id(m) for m in emulate_fp8_linears(ora).mods}
    out = {}
    for n, m in ora.named_modules():
        if id(m) in ffs:
            tap = max((t for t in names if n.startswith(t + ".")), key=len)
            blk = dict(ora.named_modules())[tap]
            po = blk.proj_out if hasattr(blk, "proj_out") else blk.temporal_transformer.proj_out
            out[tap] = (m, po.weight.reshape(po.weight.shape[0], -1))
    return out


def parity(label, ora, names, native, x, ehs, pose=None, banks=None, cfg=True, fp8=False, written=None):
    """Check every tap; returns {block kind: BlockReport}.  banks: fp16 reference banks read by the oracle's blocks.  written: the native
    writer's banks (reader order), checked against the oracle blocks' LayerNorm-1 output on the native input."""
    reports = {}

    def rep(kind):
        return reports.setdefault(kind, BlockReport())

    def set_banks(dt):
        if banks is not None:
            O.set_reference_banks(ora, [b.to(dt) for b in banks], cfg=cfg)
        if written is not None:
            O.set_reference_write(ora)

    try:
        # E: the reference's fp16 deployment on the native inputs
        ora.half()
        set_banks(torch.float16)
        E = {n: o.contiguous() for n, o in replay_blocks(ora, names, native, x, T, ehs, pose)}
        bank_e = [b.contiguous() for b in O.written_banks(ora)] if written is not None else None
        ora.double()
        # Emu: the e4m3 emulation in fp64, and the flip term of each e4m3 block's feed-forward carried through its proj_out
        emu, extra = {}, {}
        if fp8:
            blocks = e4m3_taps(ora, names)
            assert blocks, "no feed-forward of this net runs on e4m3"
            flips = {}
            hooks = [m.register_forward_hook(lambda mod, inp, o, t=t: flips.__setitem__(t, ff_flip_bound(mod, inp[0])))
                     for t, (m, _) in blocks.items()]
            set_banks(torch.float64)
            with emulate_fp8_linears(ora):
                for n, o in replay_blocks(ora, names, native, x, T, ehs, pose):
                    if n in blocks:
                        emu[n] = o.contiguous()
                        extra[n] = (flips.pop(n) @ blocks[n][1].abs().T).reshape(o.shape)
            for hk in hooks:
                hk.remove()
        # R: fp64
        set_banks(torch.float64)
        for n, r in replay_blocks(ora, names, native, x, T, ehs, pose):
            k = block_kind(n)
            if n in emu:
                check_fp8_block(rep(k + " (e4m3)"), n, native[n], emu.pop(n), r, extra.pop(n))
            else:
                check_fp16_block(rep(k), n, native[n], r, E.pop(n))
        if written is not None:
            R_b = O.written_banks(ora)
            assert len(R_b) == len(written) == len(bank_e)
            for i, (nb, rb, eb) in enumerate(zip(written, R_b, bank_e)):
                check_fp16_block(rep("written banks"), f"bank {i}", nb.unsqueeze(1), rb.unsqueeze(1), eb.unsqueeze(1))
    finally:
        O.set_reference_banks(ora, None)
        if written is not None:
            O.set_reference_write(ora, False)
        ora.half()
        torch.cuda.empty_cache()
    return reports


def assert_reports(label, reports):
    for k, r in reports.items():
        eager = "" if k.endswith("(e4m3)") else f"; fp16 eager row {r.e_row.ratio:.3f} element {r.e_elem.ratio:.3f}"
        report(f"block parity {label} {k}: worst err/bound native slice {r.slice.ratio:.3f} row {r.row.ratio:.3f} element {r.elem.ratio:.3f}{eager}")
    fails = [f"{k}: {f}" for k, r in reports.items() for f in r.failures(with_eager=not k.endswith("(e4m3)"))]
    assert not fails, f"{label}:\n" + "\n".join(fails)


# --------------------------------------------------------------------------------------------------------------- launch plans
def tplan(B, F, HW, heads, d):
    tma, hpb, grid = C.c_int32(), C.c_int32(), C.c_int32()
    check(lib().hv_dbg_temporal_attention_plan(i64(B), i64(F), i64(HW), i32(heads), i32(d), C.byref(tma), C.byref(hpb), C.byref(grid)))
    return "tma" if tma.value else "register"


def gplan(M, N, K, geglu=False):
    bn, st, grid = C.c_int32(), C.c_int32(), C.c_int32()
    check(lib().hv_dbg_gemm_plan(i64(M), i64(N), i64(K), i32(int(geglu)), C.byref(bn), C.byref(st), C.byref(grid)))
    return bn.value, "bstationary" if st.value > 0 else "ring"


def level_hw(h, w, chs):
    out = []
    for _ in chs:
        out.append((h, w))
        h, w = (h - 1) // 2 + 1, (w - 1) // 2 + 1
    return out


def temporal_plans(B, F, h, w, chs):
    """{d: plan} of the motion modules' temporal attention at each level (8 heads)."""
    return {c // 8: tplan(B, F, hh * ww, 8, c // 8) for c, (hh, ww) in zip(chs, level_hw(h, w, chs))}


# --------------------------------------------------------------------------------------------------------------- configurations
@pytest.mark.parametrize("h,w,F,tplans,full_tiles,l3", [
    (40, 24, 5, {40: "tma", 80: "register", 160: "register"}, False, (5, 3)),
    (48, 40, 3, {40: "tma", 80: "tma", 160: "register"}, True, (6, 5)),
], ids=["40x24xF5", "48x40xF3"])
def test_v0_sd15_cfg_no_banks(sd_v0, h, w, F, tplans, full_tiles, l3):
    ora, nat = sd_v0
    B = 2
    assert temporal_plans(B, F, h, w, SD) == tplans
    assert ((h * w) % 128 == 0) == full_tiles                      # level-0 self-attention keys: whole 128-key tiles or a partial one
    lv = level_hw(h, w, SD)
    assert lv[3] == l3
    # the GEMM launches of the transformers' linears (proj_in, GEGLU ff1, ff2) at every level of this shape
    gemms = sorted({gplan(B * F * hh * ww, n, k, g) for c, (hh, ww) in zip(SD, lv) for n, k, g in ((c, c, False), (8 * c, c, True), (c, 4 * c, False))})
    report(f"block parity v0 {h}x{w} F={F}: temporal plans {tplans}, GEMM (block_n, variant) {gemms}")
    assert {v for _, v in gemms} == {"ring", "bstationary"}
    x, ehs, pose = inputs(B, F, h, w, SD[0], XDIM, seed=h)
    names, taps = native_taps(nat, x, ehs, pose, F)
    assert_reports(f"v0 {h}x{w} F={F}", parity("v0", ora, names, taps, x, ehs, pose))


@pytest.mark.parametrize("cfg", [True, False], ids=["cfg", "no-cfg"])
def test_v0_sd15_16_banks(sd_v0, cfg):
    ora, nat = sd_v0
    B, F, h, w = 2, 5, 40, 24
    x, ehs, pose = inputs(B, F, h, w, SD[0], XDIM, seed=3)
    banks = make_banks(ora, B, h, w)
    assert len(banks) == 16
    with NativeBanks(nat, banks, cfg):
        names, taps = native_taps(nat, x, ehs, pose, F)
    if cfg:
        # the uncond half reads no bank: every one of its taps equals the bank-free forward's on the same input, bit for bit
        names0, taps0 = native_taps(nat, x, ehs, pose, F)
        assert names0 == names
        diff = [n for n in names if not torch.equal(taps[n][: (B // 2) * F], taps0[n][: (B // 2) * F])]
        assert not diff, f"uncond half differs from the bank-free forward first at {diff[0]}"
        assert not torch.equal(taps[names[-1]][(B // 2) * F:], taps0[names[-1]][(B // 2) * F:]), "the cond half read no bank"
        del taps0
    assert_reports(f"v0 16 banks cfg={int(cfg)}", parity("banks", ora, names, taps, x, ehs, pose, banks=banks, cfg=cfg))


def test_v0_sd15_batch4_bank4(sd_v0):
    """context_batch_size = 2: a CFG batch [u0, u1, c0, c1] with one bank item per batch item; frame n reads bank item n / F."""
    ora, nat = sd_v0
    B, F, h, w = 4, 3, 16, 8
    assert temporal_plans(B, F, h, w, SD)[40] == "register"
    x, ehs, pose = inputs(B, F, h, w, SD[0], XDIM, seed=4)
    banks = make_banks(ora, B, h, w, seed=6)
    with NativeBanks(nat, banks, True):
        names, taps = native_taps(nat, x, ehs, pose, F)
    assert_reports("v0 B=4 4-item bank", parity("b4", ora, names, taps, x, ehs, pose, banks=banks, cfg=True))


def test_v1_sd15_24_frames_banks():
    ora = O.synthetic_init(unet3d_v1(SD, XDIM).eval(), seed=7).half().cuda()
    nat = hv.UNet3DConditionModel(block_out_channels=SD, cross_attention_dim=XDIM, attention_head_dim=8, **V1_UNET_KWARGS)
    nat.load_state_dict(ora.state_dict())
    nat = nat.to("cuda", torch.float16)
    assert nat._hv_config().gn_pool_frames == 1
    B, F, h, w = 2, 24, 16, 16
    x, ehs, pose = inputs(B, F, h, w, SD[0], XDIM, seed=24, drift=0.1)
    banks = make_banks(ora, B, h, w, seed=7)
    with NativeBanks(nat, banks, True):
        names, taps = native_taps(nat, x, ehs, pose, F)
    assert not any(n.startswith("mid_block.motion_modules") for n in names)
    reps = parity("v1", ora, names, taps, x, ehs, pose, banks=banks, cfg=True)
    del ora, nat
    assert_reports("v1 F=24 banks", reps)


@pytest.mark.parametrize("width", ["narrow", "full"])
def test_fp8(width, request):
    if width == "narrow":
        ora, nat = make_v0(FP8_NARROW, 64)
        chs, xdim, (B, F, h, w) = FP8_NARROW, 64, (2, 4, 16, 16)
    else:
        ora, nat = request.getfixturevalue("sd_v0")
        chs, xdim, (B, F, h, w) = SD, XDIM, (2, 3, 24, 16)
    x, ehs, pose = inputs(B, F, h, w, chs[0], xdim, seed=8)
    nat.disable_fp8_linears()
    names, taps16 = native_taps(nat, x, ehs, pose, F)
    nat.enable_fp8_linears()
    try:
        names8, taps = native_taps(nat, x, ehs, pose, F)
    finally:
        nat.disable_fp8_linears()
    assert names8 == names
    blocks = e4m3_taps(ora, names)
    first = min(names.index(n) for n in blocks)
    diff = [n for n in names[:first] if not torch.equal(taps[n], taps16[n])]
    assert not diff, f"FP8 mode changed {diff[0]}, before the first e4m3 feed-forward ({names[first]})"
    assert not torch.equal(taps[names[first]], taps16[names[first]]), f"{names[first]} did not run on e4m3"
    del taps16
    assert_reports(f"fp8 {width}", parity("fp8", ora, names, taps, x, ehs, pose, fp8=True))


def test_unet2d_writer_sd15():
    ora = O.synthetic_init(O.UNet2DConditionModel(block_out_channels=SD, cross_attention_dim=XDIM).eval(), seed=11).half().cuda()
    nat = hv.UNet2DConditionModel(block_out_channels=SD, cross_attention_dim=XDIM)
    nat.load_state_dict(ora.state_dict())
    nat = nat.to("cuda", torch.float16)
    B, h, w = 2, 40, 24
    g = torch.Generator(device="cuda").manual_seed(12)
    x = torch.randn(B, 4, h, w, generator=g, device="cuda").half()
    ehs = torch.randn(B, 1, XDIM, generator=g, device="cuda").half()
    ehs[:1] = 0
    hv.ReferenceAttentionControl(nat, mode="write", fusion_blocks="full")
    names, taps = native_taps(nat, x, ehs, None, 1)
    written = [blk.bank[0] for blk, _ in nat.writer_blocks()]
    assert len(written) == 16
    reps = parity("writer", ora, names, taps, x, ehs, written=written)
    del ora, nat
    assert_reports("writer UNet2D", reps)


def test_v0_narrow_ladder_shape():
    """The error ladder's narrow net and shape (scripts/error_ladder.py --narrow --hw 32 32 --frames 6)."""
    ora, nat = make_v0(NARROW, NARROW_XDIM)
    B, F, h, w = 2, 6, 32, 32
    x, ehs, pose = inputs(B, F, h, w, NARROW[0], NARROW_XDIM, seed=42)
    names, taps = native_taps(nat, x, ehs, pose, F)
    assert len(names) >= 60
    assert_reports("v0 narrow 32x32 F=6", parity("narrow", ora, names, taps, x, ehs, pose))
