"""hv_op_groupnorm_pooled: GroupNorm whose statistics span the F frames of each batch item (nn.GroupNorm on (b, c, f, h, w)), the norm
of the inference_v1 UNet's resnets and conv_norm_out.

Every output element is compared with an fp64 reference computed from the same fp16 inputs, against a bound derived from the kernels'
arithmetic (u = 2^-24, fp32 throughout, one fp16 rounding at the store):
  * the sums S = sum(x - p), Q = sum((x - p)^2) are taken relative to the pivot p (the group's first channel in the first row of the
    item's first frame), in chains of at most D additions (per-thread row loop, the block's slot loop, the finalize's strided loop and
    its 7-level tree); with the roundings of x - p and of the squares, |dS| <= g(D + 1) A and |dQ| <= g(D + 3) Q, A = sum|x - p|,
    g(k) = k u / (1 - k u);
  * m' = S / N, mean = p + m', var = Q / N - m'^2: e(m') <= g(D + 1) A / N + 2u|m'|, e(mean) <= e(m') + u|mean|,
    e(var) <= g(D + 3) Q / N + 2|m'| e(m') + e(m')^2 + 4u (Q / N + m'^2);
  * rstd = rsqrtf(var + eps) (2 ulp): rel(rstd) <= e(var) / (2 (var + eps)) (1 + e(var) / (var + eps)) + 2^-22 + u;
  * sc = rstd gamma, sh = fma(-mean, sc, beta), y = fma(x, sc, sh):
    |dy| <= |x - mean| |gamma| rstd (rel(rstd) + u) + |sc| e(mean) + u (|sh| + |y|);
  * SiLU y / (1 + __expf(-y)) adds (5 + 1.2 |y|) 2^-23 |silu(y)| and scales dy by at most 1.1;
  * the fp16 store adds 2^-11 (|ref| + dy) + 2^-25.
The pivot is the item's frame-0 value, so frames that drift away from frame 0 make |m'| large; the bound carries that and the test
reports the worst err / bound.  Outputs sit in NaN-sentinel windows with guard rows; inputs are checked unchanged.
"""
import ctypes as C

import pytest
import torch

pytestmark = pytest.mark.gpu

from conftest import report
from guarded import Guarded, bits, check_inputs_unchanged
from norm_bounds import groupnorm_ref_and_bound

if torch.cuda.is_available():
    from humanvid_b200._native import check, i32, i64, lib, ptr, stream

G = 32
EPS = 1e-5
_worst = {}


def scratch_floats(C_, NF, HW, F):
    f = lib().hv_groupnorm_pooled_scratch_floats
    f.restype = C.c_size_t
    return int(f(i64(C_), i64(NF), i64(HW), i32(G), i64(F)))


def call(x1, x2, gamma, beta, out, NF, HW, F, silu, stats=None, groups=G):
    C1 = x1.shape[-1]
    C2 = x2.shape[-1] if x2 is not None else 0
    if stats is None:
        stats = torch.zeros(scratch_floats(C1 + C2, NF, HW, F), device="cuda", dtype=torch.float32)
    return lib().hv_op_groupnorm_pooled(ptr(x1), i64(C1), ptr(x2), i64(C2), ptr(gamma), ptr(beta), ptr(out), i64(NF), i64(HW), i32(groups),
                                        C.c_float(EPS), i32(silu), i64(F), ptr(stats), stream())


def pooled(x1, x2, gamma, beta, NF, HW, F, silu):
    Ct = x1.shape[-1] + (x2.shape[-1] if x2 is not None else 0)
    g = Guarded(NF * HW, Ct)
    before = [bits(t) for t in (x1, x2, gamma, beta) if t is not None]
    check(call(x1, x2, gamma, beta, g.out, NF, HW, F, silu))
    torch.cuda.synchronize()
    g.check_untouched(torch.ones(NF * HW, Ct, dtype=torch.bool, device="cuda"), "pooled groupnorm")
    check_inputs_unchanged(before, [t for t in (x1, x2, gamma, beta) if t is not None], "pooled groupnorm")
    return g.out.view(NF, HW, Ct)


def per_frame(x1, x2, gamma, beta, NF, HW, silu):
    C1 = x1.shape[-1]
    C2 = x2.shape[-1] if x2 is not None else 0
    f = lib().hv_groupnorm_scratch_floats
    f.restype = C.c_size_t
    stats = torch.zeros(int(f(i64(C1 + C2), i64(NF), i64(HW), i32(G))), device="cuda", dtype=torch.float32)
    out = torch.empty(NF, HW, C1 + C2, device="cuda", dtype=torch.half)
    check(lib().hv_op_groupnorm(ptr(x1), i64(C1), ptr(x2), i64(C2), ptr(gamma), ptr(beta), ptr(out), i64(NF), i64(HW), i32(G), C.c_float(EPS),
                                i32(silu), ptr(stats), stream()))
    return out


def check_against_fp64(y, x1, x2, gamma, beta, NF, HW, F, silu, label):
    x = torch.cat([x1, x2], -1) if x2 is not None else x1
    yr, bound = groupnorm_ref_and_bound(x.view(NF, HW, -1), gamma, beta, F, G, EPS, silu)
    err = (y.double().view_as(yr) - yr).abs()
    ratio = float((err / bound).max())
    relL2 = float((y.double().view_as(yr) - yr).norm() / yr.norm())
    _worst[label] = max(_worst.get(label, 0.0), ratio)
    assert torch.isfinite(y).all(), label
    assert ratio <= 1.0, f"{label}: worst err/bound {ratio:.3f}"
    assert relL2 < 1e-3, f"{label}: relative L2 {relL2:.2e}"
    return ratio


def inputs(NF, HW, C1, C2, F, seed, offset=0.0, drift=0.0):
    """Unit-variance noise, plus a common offset and a per-frame drift of `drift` standard deviations per frame from frame 0."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    Ct = C1 + C2
    x = torch.randn(NF, HW, Ct, generator=g, device="cuda") + offset
    if drift:
        f = (torch.arange(NF, device="cuda") % F).float()
        x = x + drift * f.view(NF, 1, 1)
    x = x.half()
    x1 = x[..., :C1].contiguous()
    x2 = x[..., C1:].contiguous() if C2 else None
    gamma = (1 + 0.1 * torch.randn(Ct, generator=g, device="cuda")).half()
    beta = (0.1 * torch.randn(Ct, generator=g, device="cuda")).half()
    return x1, x2, gamma, beta


# (C1, C2, level) of every resnet norm1 / norm2 (and conv_norm_out) of the SD1.5 UNet: down, mid and each up-block concat split
RESNET_SHAPES = {
    0: [(320, 0), (640, 320), (320, 320)],
    1: [(320, 0), (640, 0), (1280, 640), (640, 640), (640, 320)],
    2: [(640, 0), (1280, 0), (1280, 1280), (1280, 640)],
    3: [(1280, 0), (1280, 1280)],
}
# latent H*W per UNet level of bench config 2 (96 x 72: 6912, 1728, 432, 108) and config 5 (72 x 128: 9216, 2304, 576, 144)
LEVEL_HW = [(0, 6912), (1, 1728), (2, 432), (3, 108), (0, 9216), (1, 2304), (2, 576), (3, 144)]
SHAPE_CASES = [(C1, C2, HW) for lvl, HW in LEVEL_HW for (C1, C2) in RESNET_SHAPES[lvl]]


@pytest.mark.parametrize("silu", [1, 0])
@pytest.mark.parametrize("C1,C2,HW", SHAPE_CASES)
def test_pooled_resnet_shapes(C1, C2, HW, silu):
    F, B = 3, 2
    x1, x2, gamma, beta = inputs(B * F, HW, C1, C2, F, seed=C1 + C2 + HW)
    y = pooled(x1, x2, gamma, beta, B * F, HW, F, silu)
    check_against_fp64(y, x1, x2, gamma, beta, B * F, HW, F, silu, "resnet shapes")


@pytest.mark.parametrize("silu", [1, 0])
@pytest.mark.parametrize("B", [1, 2, 3])
@pytest.mark.parametrize("F", [1, 2, 7, 24])
@pytest.mark.parametrize("C1,C2,HW", [(1280, 640, 432), (320, 0, 1728), (1280, 1280, 108)])
def test_pooled_frames_and_batch(C1, C2, HW, F, B, silu):
    x1, x2, gamma, beta = inputs(B * F, HW, C1, C2, F, seed=F * 10 + B)
    y = pooled(x1, x2, gamma, beta, B * F, HW, F, silu)
    check_against_fp64(y, x1, x2, gamma, beta, B * F, HW, F, silu, "F x B")


@pytest.mark.parametrize("C1,C2,HW,F,B", [(640, 320, 9216, 24, 1), (320, 0, 6912, 24, 2), (1280, 640, 432, 7, 3), (1280, 1280, 108, 24, 2)])
@pytest.mark.parametrize("offset,drift", [(128.0, 0.0), (0.0, 4.0), (64.0, 2.0)])
def test_pooled_large_offset_and_drifting_frames(C1, C2, HW, F, B, offset, drift):
    """A 128-sigma common offset, and frames drifting 2-4 sigma per frame away from frame 0 (where the pivot sits): at F = 24 the last
    frame is ~92 sigma from the pivot and the pooled mean ~46 sigma."""
    x1, x2, gamma, beta = inputs(B * F, HW, C1, C2, F, seed=int(offset + 10 * drift), offset=offset, drift=drift)
    y = pooled(x1, x2, gamma, beta, B * F, HW, F, 1)
    check_against_fp64(y, x1, x2, gamma, beta, B * F, HW, F, 1, f"offset {offset:g}, drift {drift:g}")


@pytest.mark.parametrize("C1,C2,HW,NF", [(320, 0, 9216, 2), (640, 320, 6912, 3), (1280, 640, 432, 5), (1280, 1280, 108, 4)])
def test_f1_is_bitwise_per_frame_groupnorm(C1, C2, HW, NF):
    x1, x2, gamma, beta = inputs(NF, HW, C1, C2, 1, seed=HW, offset=16.0)
    for silu in (0, 1):
        assert torch.equal(bits(pooled(x1, x2, gamma, beta, NF, HW, 1, silu)), bits(per_frame(x1, x2, gamma, beta, NF, HW, silu)))


@pytest.mark.parametrize("C1,C2,HW,F", [(1280, 640, 432, 7), (320, 0, 6912, 24), (640, 640, 1728, 2)])
def test_items_are_independent_and_deterministic(C1, C2, HW, F):
    B = 3
    x1, x2, gamma, beta = inputs(B * F, HW, C1, C2, F, seed=5, drift=1.0)
    y = pooled(x1, x2, gamma, beta, B * F, HW, F, 1).clone()
    assert torch.equal(bits(y), bits(pooled(x1, x2, gamma, beta, B * F, HW, F, 1)))   # run to run
    # pooled over frames, not over items: three items differ from one item of the same frames
    for b in range(B):
        sl = slice(b * F, (b + 1) * F)
        yb = pooled(x1[sl].contiguous(), None if x2 is None else x2[sl].contiguous(), gamma, beta, F, HW, F, 1)
        assert torch.equal(bits(y[sl]), bits(yb)), f"item {b} of a B = {B} call differs from the item alone"
    # and it is not per-frame GroupNorm: the frames' statistics differ
    assert not torch.equal(bits(y), bits(per_frame(x1, x2, gamma, beta, B * F, HW, 1)))


def test_rejections_write_nothing():
    F, B, HW, C1, C2 = 3, 2, 108, 640, 640
    x1, x2, gamma, beta = inputs(B * F, HW, C1, C2, F, seed=9)
    raw = torch.empty(B * F * HW * (C1 + C2) + 64, device="cuda", dtype=torch.half)
    mis = raw[1: 1 + x1.numel()].view_as(x1)          # 2-byte aligned copy of x1
    mis.copy_(x1)
    g = Guarded(B * F * HW, C1 + C2)
    stats = torch.zeros(scratch_floats(C1 + C2, B * F, HW, F) + 2, device="cuda", dtype=torch.float32)
    cases = {
        "NF not a multiple of F": dict(NF=B * F, F=4),
        "F = 0": dict(F=0),
        "F < 0": dict(F=-3),
        "NF = 0": dict(NF=0),
        "misaligned X": dict(x1=mis),
        "misaligned out": dict(out=g.buf.view(torch.half).view(-1)[1 + 3 * (C1 + C2):]),
        "misaligned stats": dict(stats=stats[1:]),
        "C1 not a multiple of 8": dict(x1=x1[..., :636].contiguous(), x2=torch.cat([x1[..., 636:], x2], -1).contiguous()),
        "odd channels per group": dict(groups=128, x1=x1[..., :320].contiguous(), x2=x2[..., :320].contiguous()),
        "too many groups": dict(groups=320),
        "X2 NULL with C2 > 0": dict(x2_null=True),
        "C > 8192": dict(x1=torch.zeros(1, 1, 8192, device="cuda", dtype=torch.half), NF=1, F=1, HW=1),
    }
    for label, kw in cases.items():
        a1 = kw.get("x1", x1)
        a2 = kw.get("x2", x2)
        NF, FF, H = kw.get("NF", B * F), kw.get("F", F), kw.get("HW", HW)
        C1_, C2_ = a1.shape[-1], (a2.shape[-1] if a2 is not None else 0)
        p2 = None if kw.get("x2_null") else a2
        out = kw.get("out", g.out)
        st = kw.get("stats", stats)
        status = lib().hv_op_groupnorm_pooled(ptr(a1), i64(C1_), ptr(p2), i64(C2_), ptr(gamma), ptr(beta), ptr(out), i64(NF), i64(H),
                                              i32(kw.get("groups", G)), C.c_float(EPS), i32(1), i64(FF), ptr(st), stream())
        torch.cuda.synchronize()
        assert status == -1, f"{label}: status {status}, expected HV_ERR_INVALID"
        g.check_untouched(torch.zeros(g.rows, g.ld, dtype=torch.bool, device="cuda"), label)
        assert float(stats.abs().sum()) == 0.0, f"{label}: scratch written"
    # the same arguments with a valid F run
    check(call(x1, x2, gamma, beta, g.out, B * F, HW, F, 1, stats=stats[:-2]))


def test_report_worst_ratios():
    for k, v in sorted(_worst.items()):
        report(f"pooled groupnorm, {k}: worst err/bound {v:.3f}")
