"""The PoseGuider convolutions, the per-frame GroupNorm, the LayerNorm, the Plucker producer, the layout kernels, the small linear, the
timestep embedding and the weight packers, element by element against fp64 (or bit for bit), with guarded outputs.

Every output is a window into a NaN-sentinel buffer with guard rows (and a row stride wider than the written columns where the operator
takes one); every element outside the written set must still hold the sentinel.  Inputs with a row stride carry sentinel columns past
their width, and every input is checked unchanged bit for bit.  Each call goes through a wrapper that first checks, on the host, the
dtype and the byte extent of every tensor the operator reads or writes (guarded.need), from the extents its header states.

Pure data movement is compared bit for bit: the transposes (fp16 and fp32 sources), the pixel unshuffle, CLIP's patchify and the four
packers.
hv_pack_upconv2x2 sums up to four fp16 taps in fp32 (0 + w0 + w1 + ...); torch sums the same taps in the same order in fp32.

Everything that does arithmetic is held to a per-element bound, u = 2^-24, fp32 accumulation in any order, gamma_k = k u / (1 - k u):

  * Convolutions and the small linear (K = 9 Cin products, 27 for conv_in, K for the linear; the bias is the (K+1)-th term):
        v = sum_k x_k w_k + bias           |dv| <= gamma_{K+1} S,   S = sum |x_k| |w_k| + |bias|        (Higham, products rounded)
    The mma.sync kernels (hv_op_conv3x3_small, hv_op_pose_conv_in) accumulate on tensor cores, whose fp32 adds are not guaranteed to
    round to nearest; a truncating add errs by up to 2u, so their gamma uses 2u.  The activation then gives
        SiLU (silu_f = __fdividef(v, 1 + __expf(-v))):  dy <= 1.1 dv + (5 + 1.2 |v|) 2^-23 |silu(v)|   (slope of SiLU <= 1.1; the
                                                        second term is the pooled-GroupNorm docstring's bound of silu_f itself;
                                                        past |v| ~ 88 __expf overflows and the quotient is -0 or v, both within it)
        ReLU or none:                                   dy <= dv
    and hv_op_conv3x3_direct's `add`, applied after the activation, one more rounding: u (|act(v)| + |add|).
    For the small linear with act_in = SiLU the activation is on the inputs: S uses |silu(x_k)| and each input adds its silu_f error
    times |w_k|.
  * Per-frame GroupNorm: the bound of test_groupnorm_pooled_gpu.py at F = 1 (tests/norm_bounds.py).
  * LayerNorm (one row of C, LPR lanes per row, each lane summing its 8 ceil(C / 8 / LPR) values in order, then log2(LPR) shuffles:
    chains of D = 8 ceil(C / 8 / LPR) + log2(LPR) additions).  The statistics see v = x + pre_add as the kernel holds it, unrounded
    in fp32 (the reference uses the same fp32 sum; x_out holds it rounded to fp16 and is compared bit for bit):
        mean = sum / C                      e_m <= gamma_D sum |v| / C + u |m|
        var = sum (v - mean)^2 / C          sum (v_j - mean)^2 = C var + C (mean - m)^2, so with the roundings of the difference, the
                                            square, the D additions and the division:  e_var <= e_m^2 + (gamma_{D+3} + u)(var + e_m^2)
        rstd = rsqrtf(var + eps) (2 ulp)    rel(rstd) <= e_var / (2 (var + eps)) (1 + e_var / (var + eps)) + 2^-22 + u
        y = (v - mean) rstd g + b (+ pe)    |dy| <= |g| rstd (e_m (1 + u) + |v - m| (rel(rstd) + 3u)) + u |y| (+ u |y + pe|)
  * Plucker (fp32 per pixel: two divisions, three squares and two adds under sqrtf, three divisions by the norm, a 3x3 product with
    |R_ij| <= 1 and a cross product with t): dx, dy carry 2u relative, the squared norm 7u, the norm 4.5u, the unit direction 7.5u,
    so rays_d errs by at most 10.5u (1 + |x - cx| / fx + |y - cy| / fy) per component; the cross product adds 2 |t| times that and
    3u |t| |rays_d| twice.  With c = 32 >= 10.5 (2 + 1) + 6:
        |dv| <= 32 u (|t|_inf + 1)(1 + |x + 0.5 - cx| / fx + |y + 0.5 - cy| / fy)
    against an fp64 restatement of plucker_unshuffle_kernel on the same fp32 K and c2w.
  * Timestep embedding: freq = expf(-logf(10000) j / half): the argument a = -ln(10^4) j / half carries logf's 1 ulp, the product's and
    the division's u (4u relative), expf adds 2 ulp (4u), so rel(freq) <= 4u |a| + 4u; t freq adds u:  e_arg <= t freq (4u |a| + 5u).
    cosf / sinf add 2 ulp of the result: E = e_arg + 4u (|ref| + e_arg), against fp64 cos / sin of the fp64 argument.
Every arithmetic bound ends with the fp16 store:  |out - ref| <= 2^-11 (|ref| + E) + E + 2^-25, E the fp32 error above.  The store
term is tight (a value just above a power of two rounds by up to 2^-11 of itself), so over many elements the worst err / bound comes
close to 1 with a correct kernel; anything past 1 is an error beyond fp32 arithmetic and one rounding.  The worst err / bound per
operator family is reported.  A case over its bound is a finding, not a reason to widen it.

Not covered here: the strided (ldo > Cout, ldo > C) and device-timestep-table forms of hv_op_conv3x3_direct, hv_op_ncfhw_to_nhwc and
the timestep embedding.  Only the model runtime reaches them; the C ABI does not expose them.
"""
import math

import pytest
import torch
import torch.nn.functional as Fn

pytestmark = pytest.mark.gpu

from conftest import report
from guarded import Guarded, bits, check_inputs_unchanged, cols_mask, need, strided
from norm_bounds import U, gam, groupnorm_ref_and_bound, silu_error

if torch.cuda.is_available():
    import ctypes as C

    from humanvid_b200._native import check, i32, i64, lib, ptr, stream

HALF, F32 = torch.half, torch.float32
WORST = {}               # operator family -> worst err / bound seen
ALL = None               # "every element of the window is written"


@pytest.fixture(scope="module", autouse=True)
def _report_worst():
    yield
    for fam in sorted(WORST):
        report(f"small ops guarded: worst err/bound {fam} {WORST[fam]:.3f}")


def gen(seed):
    return torch.Generator(device="cuda").manual_seed(seed)


def randn(*shape, scale=1.0, seed=0, offset=0.0):
    return (torch.randn(*shape, generator=gen(seed), device="cuda") * scale + offset).half()


def judge(fam, label, y, ref, E):
    """y: the kernel's fp16 output; ref, E: fp64 reference and fp32 error bound of the same shape.  Bound: 2^-11 (|ref| + E) + E + 2^-25."""
    y = y.double().reshape(ref.shape)
    assert bool(torch.isfinite(y).all()), f"{label}: non-finite output"
    bound = 2.0 ** -11 * (ref.abs() + E) + E + 2.0 ** -25
    r = (y - ref).abs() / bound
    worst = float(r.max())
    WORST[fam] = max(WORST.get(fam, 0.0), worst)
    if worst > 1.0:
        i = int(r.flatten().argmax())
        pytest.fail(f"{label}: err/bound {worst:.3f} at flat index {i} (got {float(y.flatten()[i]):.6g}, ref {float(ref.flatten()[i]):.6g}, "
                    f"bound {float(bound.flatten()[i]):.3g})")


def finish(g, written, inputs, before, label):
    torch.cuda.synchronize()
    g.check_untouched(torch.ones(g.rows, g.ld, dtype=torch.bool, device="cuda") if written is ALL else written, label)
    check_inputs_unchanged(before, inputs, label)


# ------------------------------------------------------------------ wrappers: preflight, then the call
def op_conv3x3_small(x, wp, bias, out, ldo, NF, H, W, Cin, Cout, stride, act):
    Ho, Wo = (H, W) if stride == 1 else (H // 2, W // 2)
    need(x, HALF, NF * H * W * Cin * 2, "conv3x3_small X")
    need(wp, HALF, Cout * 9 * Cin * 2, "conv3x3_small Wp")
    if bias is not None:
        need(bias, HALF, Cout * 2, "conv3x3_small bias")
    need(out, HALF, ((NF * Ho * Wo - 1) * ldo + Cout) * 2, "conv3x3_small out")
    check(lib().hv_op_conv3x3_small(ptr(x), ptr(wp), ptr(bias), ptr(out), i64(ldo), i64(NF), i64(H), i64(W), i64(Cin), i64(Cout), i32(stride),
                                    i32(act), stream()))


def op_pose_conv_in(x, w, bias, out, B, F, H, W, act):
    need(x, HALF, B * 3 * F * H * W * 2, "pose_conv_in X")
    need(w, HALF, 16 * 27 * 2, "pose_conv_in W")
    if bias is not None:
        need(bias, HALF, 16 * 2, "pose_conv_in bias")
    need(out, HALF, B * F * H * W * 16 * 2, "pose_conv_in out")
    check(lib().hv_op_pose_conv_in(ptr(x), ptr(w), ptr(bias), ptr(out), i64(B), i64(F), i64(H), i64(W), i32(act), stream()))


def op_conv3x3_direct(x, w, bias, out, NF, H, W, Cin, Cout, stride, act, add):
    Ho, Wo = (H - 1) // stride + 1, (W - 1) // stride + 1
    need(x, HALF, NF * H * W * Cin * 2, "conv3x3_direct X")
    need(w, HALF, Cout * Cin * 9 * 2, "conv3x3_direct W")
    if bias is not None:
        need(bias, HALF, Cout * 2, "conv3x3_direct bias")
    need(out, HALF, NF * Ho * Wo * Cout * 2, "conv3x3_direct out")
    if add is not None:
        need(add, HALF, NF * Ho * Wo * Cout * 2, "conv3x3_direct add")
    check(lib().hv_op_conv3x3_direct(ptr(x), ptr(w), ptr(bias), ptr(out), i64(NF), i64(H), i64(W), i64(Cin), i64(Cout), i32(stride), i32(act),
                                     ptr(add), stream()))


def op_groupnorm(x1, x2, gamma, beta, out, NF, HW, groups, eps, silu, stats):
    C1, C2 = x1.shape[-1], (x2.shape[-1] if x2 is not None else 0)
    f = lib().hv_groupnorm_scratch_floats
    f.restype = C.c_size_t
    need(x1, HALF, NF * HW * C1 * 2, "groupnorm X")
    if C2:
        need(x2, HALF, NF * HW * C2 * 2, "groupnorm X2")
    need(gamma, HALF, (C1 + C2) * 2, "groupnorm gamma")
    need(beta, HALF, (C1 + C2) * 2, "groupnorm beta")
    need(out, HALF, NF * HW * (C1 + C2) * 2, "groupnorm out")
    need(stats, F32, int(f(i64(C1 + C2), i64(NF), i64(HW), i32(groups))) * 4, "groupnorm stats")
    check(lib().hv_op_groupnorm(ptr(x1), i64(C1), ptr(x2), i64(C2), ptr(gamma), ptr(beta), ptr(out), i64(NF), i64(HW), i32(groups), C.c_float(eps),
                                i32(silu), ptr(stats), stream()))


def op_layernorm(x, gamma, beta, out, rows, Cc, eps, pre_add, rpg, x_out, pe, hw, F):
    need(x, HALF, rows * Cc * 2, "layernorm X")
    need(gamma, HALF, Cc * 2, "layernorm gamma")
    need(beta, HALF, Cc * 2, "layernorm beta")
    need(out, HALF, rows * Cc * 2, "layernorm out")
    if pre_add is not None:
        need(pre_add, HALF, -(-rows // rpg) * Cc * 2, "layernorm pre_add")
    if x_out is not None:
        need(x_out, HALF, rows * Cc * 2, "layernorm x_out")
    if pe is not None:
        need(pe, HALF, F * Cc * 2, "layernorm pe")
    check(lib().hv_op_layernorm(ptr(x), ptr(gamma), ptr(beta), ptr(out), i64(rows), i64(Cc), C.c_float(eps), ptr(pre_add), i64(rpg), ptr(x_out),
                                ptr(pe), i64(hw), i64(F), stream()))


def op_plucker(K, c2w, out, NF, H, W, r):
    need(K, F32, NF * 4 * 4, "plucker K")
    need(c2w, F32, NF * 16 * 4, "plucker c2w")
    need(out, HALF, NF * H * W * 6 * 2, "plucker out")
    check(lib().hv_op_plucker_unshuffle(ptr(K), ptr(c2w), ptr(out), i64(NF), i64(H), i64(W), i32(r), stream()))


def op_ncfhw_to_nhwc(x, out, B, Cc, F, H, W, src_fp32):
    need(x, F32 if src_fp32 else HALF, B * Cc * F * H * W * (4 if src_fp32 else 2), "ncfhw_to_nhwc X")
    need(out, HALF, B * F * H * W * Cc * 2, "ncfhw_to_nhwc out")
    check(lib().hv_op_ncfhw_to_nhwc(ptr(x), ptr(out), i64(B), i64(Cc), i64(F), i64(H), i64(W), i32(src_fp32), stream()))


def op_nhwc_to_ncfhw(x, ldx, out, B, Cc, F, H, W):
    need(x, HALF, ((B * F * H * W - 1) * ldx + Cc) * 2, "nhwc_to_ncfhw X")
    need(out, HALF, B * Cc * F * H * W * 2, "nhwc_to_ncfhw out")
    check(lib().hv_op_nhwc_to_ncfhw(ptr(x), i64(ldx), ptr(out), i64(B), i64(Cc), i64(F), i64(H), i64(W), stream()))


def op_pixel_unshuffle(x, out, B, Cc, F, H, W, r):
    need(x, HALF, B * Cc * F * H * W * 2, "pixel_unshuffle X")
    need(out, HALF, B * Cc * F * H * W * 2, "pixel_unshuffle out")
    check(lib().hv_op_pixel_unshuffle(ptr(x), ptr(out), i64(B), i64(Cc), i64(F), i64(H), i64(W), i32(r), stream()))


def op_clip_patchify(x, out, B, Cc, S, p, Kpad):
    need(x, HALF, B * Cc * S * S * 2, "clip_patchify X")
    need(out, HALF, B * (S // p) ** 2 * Kpad * 2, "clip_patchify out")
    check(lib().hv_op_clip_patchify(ptr(x), ptr(out), i64(B), i64(Cc), i64(S), i64(p), i64(Kpad), stream()))


def op_small_linear(x, w, bias, out, M, N, K, act_in):
    need(x, HALF, M * K * 2, "small_linear X")
    need(w, HALF, N * K * 2, "small_linear W")
    if bias is not None:
        need(bias, HALF, N * 2, "small_linear bias")
    need(out, HALF, M * N * 2, "small_linear out")
    check(lib().hv_op_small_linear(ptr(x), ptr(w), ptr(bias), ptr(out), i64(M), i64(N), i64(K), i32(act_in), stream()))


def op_timestep_embedding(t, out, B, dim):
    need(out, HALF, B * dim * 2, "timestep_embedding out")
    check(lib().hv_op_timestep_embedding(i64(t), ptr(out), i64(B), i64(dim), stream()))


def op_pack_conv3x3(w, out, Cout, Cin, Cout_pad, Cin_pad):
    need(w, HALF, Cout * Cin * 9 * 2, "pack_conv3x3 W")
    need(out, HALF, Cout_pad * 9 * Cin_pad * 2, "pack_conv3x3 out")
    check(lib().hv_pack_conv3x3(ptr(w), ptr(out), i64(Cout), i64(Cin), i64(Cout_pad), i64(Cin_pad), stream()))


def op_pack_geglu(w, out, rows, K):
    need(w, HALF, rows * K * 2, "pack_geglu W")
    need(out, HALF, rows * K * 2, "pack_geglu out")
    check(lib().hv_pack_geglu(ptr(w), ptr(out), i64(rows), i64(K), stream()))


def op_pack_heads(w, out, heads, d, dpad, K):
    need(w, HALF, heads * d * K * 2, "pack_heads W")
    need(out, HALF, heads * dpad * K * 2, "pack_heads out")
    check(lib().hv_pack_heads(ptr(w), ptr(out), i32(heads), i32(d), i32(dpad), i64(K), stream()))


def op_pack_upconv2x2(w, out, Cout, Cin):
    need(w, HALF, Cout * Cin * 9 * 2, "pack_upconv2x2 W")
    need(out, HALF, 16 * Cout * Cin * 2, "pack_upconv2x2 out")
    check(lib().hv_pack_upconv2x2(ptr(w), ptr(out), i64(Cout), i64(Cin), stream()))


# ------------------------------------------------------------------ convolutions
ACT_NONE, ACT_RELU, ACT_SILU = 0, 1, 2


def conv_ref_bound(x, w, bias, stride, act, add=None, u=U):
    """fp64 conv (padding 1) + bias -> act (+ add) of one batch of frames x (n, H, W, Cin), w (Cout, Cin, 3, 3); returns (ref, E) channels-last."""
    K = w.shape[1] * 9
    xd, wd = x.permute(0, 3, 1, 2).double(), w.double()
    bd = bias.double() if bias is not None else None
    v = Fn.conv2d(xd, wd, bd, stride=stride, padding=1).permute(0, 2, 3, 1)
    S = Fn.conv2d(xd.abs(), wd.abs(), bd.abs() if bd is not None else None, stride=stride, padding=1).permute(0, 2, 3, 1)
    E = gam(K + 1, u) * S
    del S
    if act == ACT_SILU:
        E = 1.1 * E + silu_error(v)
        v = v * torch.sigmoid(v)
    elif act == ACT_RELU:
        v = v.clamp_min(0)
    if add is not None:
        a = add.double().view_as(v)
        E = E + U * (v.abs() + a.abs())
        v = v + a
    return v, E


# (NF, H, W, Cin, Cout, stride, act, bias, weight scale, label): the PoseGuider chain (pose_guider.py:25-49) at 768x576 and at config 5's
# 576x1024, then the edges; "hot" weights give pre-activations of +-100 and beyond (the __expf overflow branch of silu_f)
SMALL_CASES = [
    (1, 768, 576, 16, 16, 1, ACT_SILU, True, 1.0, "chain 768x576"),
    (1, 768, 576, 16, 32, 2, ACT_SILU, True, 1.0, "chain 768x576"),
    (1, 384, 288, 32, 32, 1, ACT_SILU, True, 1.0, "chain 768x576"),
    (1, 384, 288, 32, 96, 2, ACT_SILU, True, 1.0, "chain 768x576"),
    (1, 576, 1024, 16, 16, 1, ACT_SILU, True, 1.0, "chain 576x1024"),
    (1, 576, 1024, 16, 32, 2, ACT_SILU, True, 1.0, "chain 576x1024"),
    (1, 288, 512, 32, 32, 1, ACT_SILU, True, 1.0, "chain 576x1024"),
    (1, 288, 512, 32, 96, 2, ACT_SILU, True, 1.0, "chain 576x1024"),
    (3, 1, 1, 16, 16, 1, ACT_SILU, True, 1.0, "1x1"),
    (2, 1, 1, 32, 32, 1, ACT_NONE, False, 1.0, "1x1"),
    (3, 2, 2, 16, 32, 2, ACT_SILU, True, 1.0, "2x2 s2"),
    (2, 2, 2, 32, 96, 2, ACT_RELU, True, 1.0, "2x2 s2"),
    (2, 9, 1, 16, 16, 1, ACT_SILU, True, 1.0, "W = 1"),
    (3, 33, 31, 16, 16, 1, ACT_SILU, True, 30.0, "33x31 hot"),
    (2, 33, 31, 32, 32, 1, ACT_RELU, False, 1.0, "33x31"),
    (3, 9, 65, 32, 32, 1, ACT_NONE, True, 1.0, "9x65"),
    (2, 130, 19, 16, 16, 1, ACT_SILU, False, 30.0, "130x19 hot"),
    (3, 34, 66, 16, 32, 2, ACT_SILU, True, 30.0, "34x66 s2 hot"),
    (2, 130, 18, 32, 96, 2, ACT_SILU, True, 30.0, "130x18 s2 hot"),
    (4, 18, 130, 32, 96, 2, ACT_NONE, False, 1.0, "18x130 s2"),
]


@pytest.mark.parametrize("NF,H,W,Cin,Cout,stride,act,has_bias,scale,label", SMALL_CASES, ids=[f"{c[-1]}-{c[3]}-{c[4]}-s{c[5]}-act{c[6]}" for c in SMALL_CASES])
def test_conv3x3_small(NF, H, W, Cin, Cout, stride, act, has_bias, scale, label):
    x = randn(NF, H, W, Cin, seed=H * 7 + W + Cin)
    w = randn(Cout, Cin, 3, 3, scale=scale / math.sqrt(9 * Cin), seed=Cout + 1)
    bias = randn(Cout, scale=max(1.0, scale / 4), seed=Cout + 2) if has_bias else None
    wp = torch.empty(Cout, 9 * Cin, device="cuda", dtype=HALF)
    op_pack_conv3x3(w, wp, Cout, Cin, Cout, Cin)
    Ho, Wo = (H, W) if stride == 1 else (H // 2, W // 2)
    ldo = 128 if Cout == 96 else Cout + 8          # blocks.3 writes into the 128-channel k-block layout of the next implicit-GEMM conv
    g = Guarded(NF * Ho * Wo, ldo)
    ins = [t for t in (x, wp, bias) if t is not None]
    before = [bits(t) for t in ins]
    op_conv3x3_small(x, wp, bias, g.out, ldo, NF, H, W, Cin, Cout, stride, act)
    finish(g, cols_mask(g.rows, ldo, Cout), ins, before, f"conv3x3_small {label}")
    y = g.out[:, :Cout].reshape(NF, Ho, Wo, Cout)
    for n in range(NF):
        ref, E = conv_ref_bound(x[n : n + 1], w, bias, stride, act, u=2 * U)
        judge("conv3x3_small", f"conv3x3_small {label} frame {n}", y[n : n + 1], ref, E)
        del ref, E
    if scale > 1:
        pre = Fn.conv2d(x.permute(0, 3, 1, 2).double(), w.double(), bias.double() if bias is not None else None, stride=stride, padding=1)
        assert float(pre.abs().max()) > 90, "the hot case must reach the __expf overflow branch of silu_f"


# (B, F, H, W, act, bias, weight scale, label)
POSE_IN_CASES = [
    (1, 1, 768, 576, ACT_SILU, True, 1.0, "768x576"),
    (2, 2, 576, 1024, ACT_SILU, True, 1.0, "576x1024, B = 2, grid-stride wraps"),
    (2, 1, 768, 576, ACT_NONE, False, 1.0, "768x576, B = 2, no bias"),
    (1, 1, 1, 1, ACT_SILU, True, 1.0, "1x1"),
    (2, 2, 2, 2, ACT_RELU, True, 1.0, "2x2"),
    (2, 3, 33, 31, ACT_SILU, True, 60.0, "33x31 hot"),
    (1, 2, 9, 65, ACT_RELU, False, 1.0, "9x65"),
    (3, 1, 130, 19, ACT_SILU, True, 60.0, "130x19 hot"),
    (1, 1, 5, 7, ACT_NONE, True, 1.0, "5x7"),
]


@pytest.mark.parametrize("B,F,H,W,act,has_bias,scale,label", POSE_IN_CASES, ids=[c[-1] for c in POSE_IN_CASES])
def test_pose_conv_in(B, F, H, W, act, has_bias, scale, label):
    img = torch.rand(B, 3, F, H, W, generator=gen(H + W), device="cuda").half()
    w = randn(16, 3, 3, 3, scale=0.2 * scale, seed=36)
    bias = randn(16, seed=37) if has_bias else None
    g = Guarded(B * F * H * W, 16)
    ins = [t for t in (img, w, bias) if t is not None]
    before = [bits(t) for t in ins]
    op_pose_conv_in(img, w, bias, g.out, B, F, H, W, act)
    finish(g, ALL, ins, before, f"pose_conv_in {label}")
    y = g.out.view(B, F, H, W, 16)
    for b in range(B):
        for f in range(F):
            x = img[b, :, f].permute(1, 2, 0)[None]      # (1, H, W, 3)
            ref, E = conv_ref_bound(x, w, bias, 1, act, u=2 * U)
            judge("pose_conv_in", f"pose_conv_in {label} item {b} frame {f}", y[b, f][None], ref, E)
    if scale > 1:
        pre = Fn.conv2d(img[:, :, 0].double(), w.double(), bias.double() if bias is not None else None, padding=1)
        assert float(pre.abs().max()) > 90, "the hot case must reach the __expf overflow branch of silu_f"


# (NF, H, W, Cin, Cout, stride, act, bias, add, weight scale, label)
DIRECT_CASES = [
    (2, 768 // 8, 576 // 8, 3, 16, 1, ACT_SILU, True, False, 1.0, "conv_in 96x72"),
    (2, 32, 24, 3, 16, 2, ACT_SILU, True, False, 1.0, "Cin 3, s2"),
    (3, 17, 23, 4, 12, 1, ACT_SILU, True, True, 1.0, "Cout 12 (tail), add"),
    (2, 33, 31, 7, 5, 2, ACT_RELU, True, False, 1.0, "odd 33x31 s2, Cout 5"),
    (2, 9, 65, 16, 20, 2, ACT_NONE, False, True, 1.0, "odd 9x65 s2, no bias, add"),
    (3, 1, 40, 8, 16, 1, ACT_SILU, True, True, 1.0, "H = 1"),
    (2, 40, 1, 8, 9, 2, ACT_RELU, True, False, 1.0, "W = 1, s2"),
    (1, 1, 1, 3, 3, 1, ACT_SILU, True, False, 1.0, "1x1"),
    (2, 130, 19, 16, 16, 1, ACT_SILU, True, True, 25.0, "130x19 hot, add"),
    (4, 2, 2, 32, 96, 2, ACT_RELU, True, False, 1.0, "2x2 s2, Cout 96"),
]


@pytest.mark.parametrize("NF,H,W,Cin,Cout,stride,act,has_bias,has_add,scale,label", DIRECT_CASES, ids=[c[-1] for c in DIRECT_CASES])
def test_conv3x3_direct(NF, H, W, Cin, Cout, stride, act, has_bias, has_add, scale, label):
    Ho, Wo = (H - 1) // stride + 1, (W - 1) // stride + 1
    x = randn(NF, H, W, Cin, seed=H + W + Cin)
    w = randn(Cout, Cin, 3, 3, scale=scale / math.sqrt(9 * Cin), seed=Cout + 3)
    bias = randn(Cout, seed=Cout + 4) if has_bias else None
    add = randn(NF, Ho, Wo, Cout, scale=2.0, seed=5) if has_add else None
    g = Guarded(NF * Ho * Wo, Cout)
    ins = [t for t in (x, w, bias, add) if t is not None]
    before = [bits(t) for t in ins]
    op_conv3x3_direct(x, w, bias, g.out, NF, H, W, Cin, Cout, stride, act, add)
    finish(g, ALL, ins, before, f"conv3x3_direct {label}")
    ref, E = conv_ref_bound(x, w, bias, stride, act, add)
    judge("conv3x3_direct", f"conv3x3_direct {label}", g.out, ref, E)
    if scale > 1:
        pre = Fn.conv2d(x.permute(0, 3, 1, 2).double(), w.double(), bias.double() if bias is not None else None, stride=stride, padding=1)
        assert float(pre.abs().max()) > 90, "the hot case must reach the __expf overflow branch of silu_f"


# ------------------------------------------------------------------ norms
# (NF, HW, C1, C2, groups, silu, offset): resnet norms of the UNet at level-0 sizes of configs 2 and 5, then the block-shape edges:
# C = 960 (240 threads, not whole warps for the finalize fold), C = 1920, C = 8, groups other than 32
GN_CASES = [
    (2, 9216, 320, 0, 32, 1, 0.0),
    (2, 6912, 640, 320, 32, 1, 0.0),
    (3, 432, 1280, 640, 32, 0, 0.0),
    (3, 300, 960, 0, 32, 1, 0.0),
    (2, 77, 640, 320, 240, 1, 0.0),
    (2, 108, 1280, 640, 64, 1, 16.0),
    (3, 50, 8, 0, 4, 1, 0.0),
    (2, 33, 8, 0, 1, 0, 64.0),
    (2, 1728, 320, 0, 16, 1, 0.0),
    (4, 1, 64, 0, 32, 1, 0.0),
]


@pytest.mark.parametrize("NF,HW,C1,C2,groups,silu,offset", GN_CASES)
def test_groupnorm_per_frame(NF, HW, C1, C2, groups, silu, offset):
    Ct = C1 + C2
    # frames with different statistics, so that a per-frame offset error shows
    x = (torch.randn(NF, HW, Ct, generator=gen(Ct + HW), device="cuda") * (1 + torch.arange(NF, device="cuda").view(NF, 1, 1))
         + offset + 3 * torch.arange(NF, device="cuda").view(NF, 1, 1)).half()
    x1 = x[..., :C1].contiguous()
    x2 = x[..., C1:].contiguous() if C2 else None
    gamma = randn(Ct, scale=0.1, seed=1, offset=1.0)
    beta = randn(Ct, scale=0.1, seed=2)
    f = lib().hv_groupnorm_scratch_floats
    f.restype = C.c_size_t
    stats = torch.zeros(int(f(i64(Ct), i64(NF), i64(HW), i32(groups))), device="cuda", dtype=F32)
    g = Guarded(NF * HW, Ct)
    ins = [t for t in (x1, x2, gamma, beta) if t is not None]
    before = [bits(t) for t in ins]
    op_groupnorm(x1, x2, gamma, beta, g.out, NF, HW, groups, 1e-5, silu, stats)
    finish(g, ALL, ins, before, "groupnorm")
    ref, bound = groupnorm_ref_and_bound(x, gamma, beta, 1, groups, 1e-5, silu)
    y = g.out.double().view_as(ref)
    assert bool(torch.isfinite(y).all())
    ratio = float(((y - ref).abs() / bound).max())
    WORST["groupnorm"] = max(WORST.get("groupnorm", 0.0), ratio)
    assert ratio <= 1.0, f"groupnorm: worst err/bound {ratio:.3f}"


def layernorm_ref_and_E(v, gamma, beta, pe_rows, eps, LPR):
    """v: fp64 copy of the fp32 row values the kernel holds (x + pre_add); pe_rows: fp16 per-row pe or None.  Returns (ref, E)."""
    Cc = v.shape[-1]
    D = 8 * -(-(Cc // 8) // LPR) + int(math.log2(LPR))
    m = v.mean(-1, keepdim=True)
    var = ((v - m) ** 2).mean(-1, keepdim=True)
    e_m = gam(D) * v.abs().sum(-1, keepdim=True) / Cc + U * m.abs()
    e_var = e_m ** 2 + (gam(D + 3) + U) * (var + e_m ** 2)
    rstd = 1.0 / torch.sqrt(var + eps)
    rel = e_var / (2 * (var + eps)) * (1 + e_var / (var + eps)) + 2.0 ** -22 + U
    g, b = gamma.double(), beta.double()
    y = (v - m) * rstd * g + b
    E = g.abs() * rstd * (e_m * (1 + U) + (v - m).abs() * (rel + 3 * U)) + U * y.abs()
    if pe_rows is not None:
        y = y + pe_rows.double()
        E = E + U * y.abs()
    return y, E


# (rows, C, variant, hw, F, rows_per_group): rows that leave a tail warp (rows per warp 32 / LPR = 4, 2, 1), C at the lane-count switches
# (320 | 328: LPR 8 -> 16, 640 | 648: 16 -> 32) and the extremes 8 and 1280; the motion module's (b, f, p) rows with pe and the
# transformer's per-item pre_add
LN_CASES = [
    (2 * 24 * 108 + 1, 1280, "pe", 108, 24, 1),
    (2 * 3 * 432, 640, "pre_add+x_out+pe", 432, 3, 3 * 432),
    (4 * 433 + 3, 320, "plain", 1, 1, 1),
    (4 * 100 + 2, 328, "pre_add+x_out", 1, 1, 101),
    (2 * 200 + 1, 640, "pe", 7, 5, 1),
    (2 * 150 + 1, 648, "pre_add+x_out+pe", 10, 3, 37),
    (4 * 64 + 1, 8, "pre_add", 1, 1, 5),
    (4 * 30 + 3, 8, "pe", 3, 4, 1),
    (7, 1280, "pre_add+x_out+pe", 2, 3, 3),
    (1, 320, "plain", 1, 1, 1),
    (3 * 5 * 7 * 13 + 2, 1272, "pre_add+x_out+pe", 7, 5, 11),
]


@pytest.mark.parametrize("rows,Cc,variant,hw,F,rpg", LN_CASES)
def test_layernorm(rows, Cc, variant, hw, F, rpg):
    x = randn(rows, Cc, scale=2.0, seed=rows + Cc, offset=0.5)
    gamma = randn(Cc, scale=0.2, seed=3, offset=1.0)
    beta = randn(Cc, scale=0.2, seed=4)
    use_add, use_xo, use_pe = "pre_add" in variant, "x_out" in variant, "pe" in variant.split("+")
    add = randn(-(-rows // rpg), Cc, scale=3.0, seed=5) if use_add else None
    pe = randn(F, Cc, seed=6) if use_pe else None
    g = Guarded(rows, Cc)
    gx = Guarded(rows, Cc) if use_xo else None
    ins = [t for t in (x, gamma, beta, add, pe) if t is not None]
    before = [bits(t) for t in ins]
    op_layernorm(x, gamma, beta, g.out, rows, Cc, 1e-5, add, rpg if use_add else 1, gx.out if gx else None, pe, hw if use_pe else 1,
                 F if use_pe else 1)
    finish(g, ALL, ins, before, f"layernorm {variant}")
    r = torch.arange(rows, device="cuda")
    v32 = x.float() + add.float()[r // rpg] if use_add else x.float()   # the kernel's fp32 sum, unrounded
    if gx is not None:
        gx.check_untouched(torch.ones(rows, Cc, dtype=torch.bool, device="cuda"), "layernorm x_out")
        assert torch.equal(bits(gx.out), bits(v32.half())), "layernorm: x_out is not x + pre_add rounded once"
    vecs = Cc // 8
    LPR = 8 if vecs <= 40 else (16 if vecs <= 80 else 32)
    ref, E = layernorm_ref_and_E(v32.double(), gamma, beta, pe[(r // hw) % F] if use_pe else None, 1e-5, LPR)
    judge("layernorm", f"layernorm {variant} rows={rows} C={Cc}", g.out, ref, E)


# ------------------------------------------------------------------ Plucker producer
def cameras(NF, H, W, seed):
    """Per-frame intrinsics that differ (focal lengths, off-centre principal points) and rigid camera-to-world poses, fp32 on the host."""
    g = torch.Generator().manual_seed(seed)
    fx = W * (0.6 + torch.rand(NF, generator=g, dtype=torch.float64))
    fy = H * (0.6 + torch.rand(NF, generator=g, dtype=torch.float64))
    cx = W * (0.2 + 0.6 * torch.rand(NF, generator=g, dtype=torch.float64))
    cy = H * (0.2 + 0.6 * torch.rand(NF, generator=g, dtype=torch.float64))
    K = torch.stack([fx, fy, cx, cy], 1).float()
    Q, _ = torch.linalg.qr(torch.randn(NF, 3, 3, generator=g, dtype=torch.float64))
    M = torch.eye(4, dtype=torch.float64).repeat(NF, 1, 1)
    M[:, :3, :3] = Q
    M[:, :3, 3] = 3 * torch.randn(NF, 3, generator=g, dtype=torch.float64)
    M = M.float()
    assert float(M[:, :3, :3].abs().max()) <= 1.0
    return K, M.reshape(NF, 16)


def plucker_ref_and_E(K, c2w, H, W, r):
    """fp64 restatement of plucker_unshuffle_kernel on the same fp32 K and c2w: (NF, H/r, W/r, 6 r r) reference and E."""
    NF = K.shape[0]
    Kd, M = K.double().cuda(), c2w.double().cuda().view(NF, 4, 4)
    ys = torch.arange(H, device="cuda", dtype=torch.float64).view(1, H, 1) + 0.5
    xs = torch.arange(W, device="cuda", dtype=torch.float64).view(1, 1, W) + 0.5
    fx, fy, cx, cy = [Kd[:, i].view(NF, 1, 1) for i in range(4)]
    dx, dy = (xs - cx) / fx, (ys - cy) / fy
    dz = torch.ones_like(dx + dy)
    nrm = torch.sqrt(dx * dx + dy * dy + 1)
    d = torch.stack([dx / nrm, dy / nrm, dz / nrm], 1)                        # (NF, 3, H, W)
    R, t = M[:, :3, :3], M[:, :3, 3]
    rd = torch.einsum("nij,njhw->nihw", R, d)
    o = t.view(NF, 3, 1, 1).expand_as(rd)
    pl = torch.cat([torch.cross(o, rd, dim=1), rd], 1)                        # (NF, 6, H, W)
    tmax = t.abs().amax(1).view(NF, 1, 1, 1)
    E = (32 * U * (tmax + 1) * (1 + dx.abs() + dy.abs())[:, None]).expand_as(pl).contiguous()
    un = lambda a: Fn.pixel_unshuffle(a, r).permute(0, 2, 3, 1).contiguous()
    return un(pl), un(E)


PLUCKER_CASES = [(8, 64, 48, 8), (3, 33, 31, 1), (4, 18, 10, 2), (2, 768, 576, 8), (2, 576, 1024, 8), (5, 2, 2, 1), (3, 24, 40, 4)]


@pytest.mark.parametrize("NF,H,W,r", PLUCKER_CASES)
def test_plucker_unshuffle(NF, H, W, r):
    K, c2w = cameras(NF, H, W, seed=H + W + r)
    Kd, Md = K.cuda(), c2w.cuda()
    Ho, Wo = H // r, W // r
    g = Guarded(NF * Ho * Wo, 6 * r * r)
    before = [bits(Kd), bits(Md)]
    op_plucker(Kd, Md, g.out, NF, H, W, r)
    finish(g, ALL, [Kd, Md], before, "plucker")
    ref, E = plucker_ref_and_E(K, c2w, H, W, r)
    judge("plucker", f"plucker NF={NF} {H}x{W} r={r}", g.out, ref, E)


# ------------------------------------------------------------------ small linear, timestep embedding
# (M, N, K, act_in, bias, x scale): the time embedding (linear_1 320 -> 1280, linear_2 and the resnets' time_emb_proj on SiLU(emb)),
# CLIP's visual projection (1024 -> 768, no bias), the cross-attention collapse, and K off the 64-lane stride
LIN_CASES = [
    (2, 1280, 320, ACT_NONE, True, 1.0),
    (2, 1280, 1280, ACT_SILU, True, 1.0),
    (2, 320, 1280, ACT_SILU, True, 1.0),
    (1, 768, 1024, ACT_NONE, False, 1.0),
    (3, 17, 130, ACT_SILU, True, 40.0),
    (2, 33, 66, ACT_NONE, False, 1.0),
    (1, 5, 2, ACT_SILU, False, 50.0),
    (4, 64, 1282, ACT_SILU, True, 1.0),
]


@pytest.mark.parametrize("M,N,K,act_in,has_bias,xs", LIN_CASES)
def test_small_linear(M, N, K, act_in, has_bias, xs):
    x = randn(M, K, scale=xs, seed=M + K)
    if xs > 1:     # pre-activations at +-90 and beyond: the __expf overflow branch of silu_f
        x[0, :2] = torch.tensor([-90.0, 95.0], device="cuda").half()
    w = randn(N, K, scale=K ** -0.5, seed=N + 1)
    bias = randn(N, seed=N + 2) if has_bias else None
    g = Guarded(M, N)
    ins = [t for t in (x, w, bias) if t is not None]
    before = [bits(t) for t in ins]
    op_small_linear(x, w, bias, g.out, M, N, K, act_in)
    finish(g, ALL, ins, before, "small_linear")
    xd, wd = x.double(), w.double()
    ex = torch.zeros_like(xd)
    if act_in == ACT_SILU:
        ex = silu_error(xd)
        xd = xd * torch.sigmoid(xd)
    ref = xd @ wd.t()
    S = xd.abs() @ wd.abs().t()
    if bias is not None:
        ref, S = ref + bias.double(), S + bias.double().abs()
    E = gam(K + 1) * S + ex @ wd.abs().t()
    judge("small_linear", f"small_linear M={M} N={N} K={K} act_in={act_in}", g.out, ref, E)


@pytest.mark.parametrize("dim", [320, 2, 8, 1280, 322])
@pytest.mark.parametrize("t", [0, 1, 999, 959, 500])
def test_timestep_embedding(t, dim):
    B = 3
    g = Guarded(B, dim)
    op_timestep_embedding(t, g.out, B, dim)
    finish(g, ALL, [], [], "timestep_embedding")
    half = dim // 2
    j = torch.arange(half, device="cuda", dtype=torch.float64)
    a = -math.log(10000.0) * j / half
    freq = torch.exp(a)
    arg = t * freq
    ref = torch.cat([arg.cos(), arg.sin()])
    e_arg = t * freq * (4 * U * a.abs() + 5 * U) * 1.01
    e_arg = torch.cat([e_arg, e_arg])
    E = e_arg + 4 * U * (ref.abs() + e_arg)
    for b in range(B):
        judge("timestep_embedding", f"timestep_embedding t={t} dim={dim} row {b}", g.out[b], ref, E)


# ------------------------------------------------------------------ layout kernels (bitwise)
# (B, C, F, H, W): the latent (C = 4) and pose image (C = 3) at small sizes, C and H*W off the 32 x 32 tile, several tiles per grid dimension
LAYOUT_CASES = [(1, 4, 24, 12, 9), (2, 3, 3, 33, 31), (2, 70, 2, 9, 13), (1, 33, 1, 1, 1), (3, 65, 2, 7, 11), (1, 320, 2, 12, 9)]


@pytest.mark.parametrize("src_fp32", [0, 1])
@pytest.mark.parametrize("B,Cc,F,H,W", LAYOUT_CASES)
def test_ncfhw_to_nhwc(B, Cc, F, H, W, src_fp32):
    x32 = torch.randn(B, Cc, F, H, W, generator=gen(Cc * H), device="cuda") * 3
    x = x32 if src_fp32 else x32.half()
    g = Guarded(B * F * H * W, Cc)
    before = [bits(x)]
    op_ncfhw_to_nhwc(x, g.out, B, Cc, F, H, W, src_fp32)
    finish(g, ALL, [x], before, "ncfhw_to_nhwc")
    ref = x.half().permute(0, 2, 3, 4, 1).reshape(B * F * H * W, Cc)        # fp32 -> fp16 round to nearest even, like __float2half_rn
    assert torch.equal(bits(g.out), bits(ref)), "ncfhw_to_nhwc differs"


@pytest.mark.parametrize("B,Cc,F,H,W", LAYOUT_CASES)
def test_nhwc_to_ncfhw(B, Cc, F, H, W):
    ldx = (Cc + 7) // 8 * 8 + 8
    x = strided(B * F * H * W, Cc, ldx, seed=Cc + W)
    g = Guarded(B * Cc * F, H * W)
    before = [bits(x)]
    op_nhwc_to_ncfhw(x, ldx, g.out, B, Cc, F, H, W)
    finish(g, ALL, [x], before, "nhwc_to_ncfhw")
    ref = x.reshape(B, F, H, W, Cc).permute(0, 4, 1, 2, 3).reshape(B * Cc * F, H * W)
    assert torch.equal(bits(g.out), bits(ref)), "nhwc_to_ncfhw differs"


@pytest.mark.parametrize("B,Cc,F,H,W,r", [(1, 6, 2, 16, 24, 8), (2, 3, 3, 12, 18, 3), (1, 6, 1, 64, 48, 1), (2, 5, 2, 6, 4, 2), (1, 6, 2, 64, 48, 8)])
def test_pixel_unshuffle(B, Cc, F, H, W, r):
    x = randn(B, Cc, F, H, W, seed=H * W + r)
    g = Guarded(B * F * (H // r) * (W // r), Cc * r * r)
    before = [bits(x)]
    op_pixel_unshuffle(x, g.out, B, Cc, F, H, W, r)
    finish(g, ALL, [x], before, "pixel_unshuffle")
    ref = Fn.pixel_unshuffle(x.transpose(1, 2).reshape(B * F, Cc, H, W), r).permute(0, 2, 3, 1).reshape(g.rows, g.ld)
    assert torch.equal(bits(g.out), bits(ref)), "pixel_unshuffle differs"


# (B, C, S, p, Kpad): CLIP ViT-L/14 and ViT-B/32 at 224 (Kpad past C p^2: the zero-filled tail), a small image, p = 1
@pytest.mark.parametrize("B,Cc,S,p,Kpad", [(1, 3, 224, 14, 592), (3, 3, 224, 32, 3080), (2, 3, 56, 14, 640), (2, 5, 3, 1, 8)])
def test_clip_patchify(B, Cc, S, p, Kpad):
    x = randn(B, Cc, S, S, seed=S + p)
    g = Guarded(B * (S // p) ** 2, Kpad)
    before = [bits(x)]
    op_clip_patchify(x, g.out, B, Cc, S, p, Kpad)
    finish(g, ALL, [x], before, "clip_patchify")
    ref = torch.zeros(g.rows, Kpad, device="cuda", dtype=HALF)
    ref[:, : Cc * p * p] = Fn.unfold(x, kernel_size=p, stride=p).transpose(1, 2).reshape(g.rows, Cc * p * p)   # (c, ky, kx): the conv weight's order
    assert torch.equal(bits(g.out), bits(ref)), "clip_patchify differs (or the zero fill is not +0)"


# ------------------------------------------------------------------ weight packers (bitwise)
@pytest.mark.parametrize("Cout,Cin,Cout_pad,Cin_pad", [(16, 3, 16, 16), (96, 32, 128, 64), (320, 4, 320, 64), (13, 5, 24, 16), (32, 16, 32, 16)])
def test_pack_conv3x3(Cout, Cin, Cout_pad, Cin_pad):
    w = randn(Cout, Cin, 3, 3, seed=Cout + Cin)
    g = Guarded(Cout_pad, 9 * Cin_pad)
    before = [bits(w)]
    op_pack_conv3x3(w, g.out, Cout, Cin, Cout_pad, Cin_pad)
    finish(g, ALL, [w], before, "pack_conv3x3")
    ref = torch.zeros(Cout_pad, 9, Cin_pad, device="cuda", dtype=HALF)
    ref[:Cout, :, :Cin] = w.permute(0, 2, 3, 1).reshape(Cout, 9, Cin)
    assert torch.equal(bits(g.out), bits(ref.view(Cout_pad, 9 * Cin_pad))), "pack_conv3x3 differs (or the zero fill is not +0)"


@pytest.mark.parametrize("rows,K", [(2560, 320), (512, 24), (10240, 1280)])
def test_pack_geglu(rows, K):
    w = randn(rows, K, seed=rows)
    g = Guarded(rows, K)
    before = [bits(w)]
    op_pack_geglu(w, g.out, rows, K)
    finish(g, ALL, [w], before, "pack_geglu")
    hid, gate = w[: rows // 2].view(-1, 128, K), w[rows // 2 :].view(-1, 128, K)
    ref = torch.stack([hid, gate], 1).reshape(rows, K)
    assert torch.equal(bits(g.out), bits(ref)), "pack_geglu differs"


@pytest.mark.parametrize("heads,d,dpad,K", [(8, 40, 48, 320), (5, 8, 16, 64), (1, 160, 160, 1280), (8, 80, 80, 640), (3, 3, 16, 8)])
def test_pack_heads(heads, d, dpad, K):
    w = randn(heads * d, K, seed=heads * d)
    g = Guarded(heads * dpad, K)
    before = [bits(w)]
    op_pack_heads(w, g.out, heads, d, dpad, K)
    finish(g, ALL, [w], before, "pack_heads")
    ref = torch.zeros(heads, dpad, K, device="cuda", dtype=HALF)
    ref[:, :d] = w.view(heads, d, K)
    assert torch.equal(bits(g.out), bits(ref.view(heads * dpad, K))), "pack_heads differs (or the zero rows are not +0)"


@pytest.mark.parametrize("Cout,Cin", [(16, 8), (320, 64), (5, 3), (1280, 1280)])
def test_pack_upconv2x2(Cout, Cin):
    w = randn(Cout, Cin, 3, 3, seed=Cout * Cin)
    g = Guarded(4 * Cout, 4 * Cin)
    before = [bits(w)]
    op_pack_upconv2x2(w, g.out, Cout, Cin)
    finish(g, ALL, [w], before, "pack_upconv2x2")
    # output row 2y+py reads source rows {y-1, y, y} (py = 0) or {y, y, y+1} (py = 1): tap a collects the kernel rows below, b the columns
    rows_of = {(0, 0): [0], (0, 1): [1, 2], (1, 0): [0, 1], (1, 1): [2]}
    ref = torch.empty(4, Cout, 4, Cin, device="cuda", dtype=HALF)
    for py in (0, 1):
        for px in (0, 1):
            for a in (0, 1):
                for b in (0, 1):
                    s = torch.zeros(Cout, Cin, device="cuda", dtype=F32)
                    for dy in rows_of[(py, a)]:
                        for dx in rows_of[(px, b)]:
                            s = s + w[:, :, dy, dx].float()        # fp32, in the kernel's order
                    ref[py * 2 + px, :, a * 2 + b] = s.half()
    assert torch.equal(bits(g.out), bits(ref.view(4 * Cout, 4 * Cin))), "pack_upconv2x2 differs"
