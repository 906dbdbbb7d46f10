"""The e4m3 operators (include/hv_b200_fp8.h) on the device, per element against fp64, with guarded outputs: e4m3 outputs sit in
buffers filled with the e4m3 NaN byte 0x7F, scale arrays in NaN-filled ones, fp16 outputs in tests/guarded.py windows.

Bounds (DESIGN.md §9):
- quantisers: the scale is amax / 448 of the producer's fp32 value; every dequantised element is within half an e4m3 step of that value
  (tests/fp8_emulation.half_step, the subnormal step below 2^-6 s) plus the producer's own fp32 error against fp64.
- GEMM, against fp64 on the dequantised operands: the FP8 MMA adds each k32 product group into an accumulator that keeps at least 13
  fraction bits, so a chain of n adds is off by at most n 2^-13 of sum |a w| (n = K / 32 unpromoted, 4 per 128-k block when the k-blocks
  are promoted into fp32 with their A scale, plus 2^-24 per fp32 promotion add); then the fp32 epilogue (a few 2^-24) and the fp16
  rounding (2^-11 of the value)."""
import ctypes as C

import pytest
import torch

pytestmark = pytest.mark.gpu

from fp8_emulation import E4M3, dequantize, half_step, quantize
from guarded import GUARD_ROWS, Guarded, cols_mask, rand

if torch.cuda.is_available():
    from humanvid_b200._native import Epilogue, check, i64, lib, ptr, stream

NAN8 = 0x7F
U13 = 2.0 ** -13
CHUNK = 32768


class Guarded8:
    """rows x ld e4m3 output window with GUARD_ROWS rows of 0x7F on either side."""

    def __init__(self, rows, ld):
        self.rows, self.ld = rows, ld
        self.buf = torch.full((rows + 2 * GUARD_ROWS, ld), NAN8, dtype=torch.uint8, device="cuda")
        self.out = self.buf[GUARD_ROWS:GUARD_ROWS + rows]

    def check_untouched(self, cols, label):
        bad = self.buf != NAN8
        bad[GUARD_ROWS:GUARD_ROWS + self.rows, :cols] = False
        assert not bad.any(), f"{label}: {int(bad.sum())} e4m3 bytes written outside the output"

    def values(self, cols):
        return self.out[:, :cols].view(E4M3)


class GuardedF32:
    def __init__(self, rows, cols, pad=4):
        self.buf = torch.full((rows + 2 * pad, cols), float("nan"), device="cuda")
        self.pad, self.rows = pad, rows
        self.out = self.buf[pad:pad + rows]

    def check_untouched(self, label):
        assert torch.isnan(self.buf[:self.pad]).all() and torch.isnan(self.buf[self.pad + self.rows:]).all(), f"{label}: scale guard written"
        assert not torch.isnan(self.out).any(), f"{label}: scale not written"


def f32p(t):
    return C.cast(C.c_void_p(t.data_ptr()), C.POINTER(C.c_float))


def pack_rows(w):
    """hv_pack_fp8_rows of fp16 w [N][K] -> (e4m3 [N][K], fp32 [N])."""
    N, K = w.shape
    q = Guarded8(N, K)
    s = GuardedF32(N, 1)
    check(lib().hv_pack_fp8_rows(ptr(w), ptr(q.out), f32p(s.out), i64(N), i64(K), stream()))
    torch.cuda.synchronize()
    q.check_untouched(K, "hv_pack_fp8_rows")
    s.check_untouched("hv_pack_fp8_rows")
    return q.values(K), s.out[:, 0]


# ---------------------------------------------------------------- quantisers


@pytest.mark.parametrize("N,K", [(2560, 320), (960, 320), (1280, 5120), (10240, 1280), (37, 64)])
def test_pack_fp8_rows_matches_the_scheme(N, K):
    w = rand(N, K, scale=K ** -0.5, seed=N + K)
    w[3] = 0                     # an all-zero row: s = 0, zero bytes
    w[5, :16] = 60000            # a row whose fp32 products saturate at 448
    q, s = pack_rows(w)
    qe, se = quantize(w.float())
    # the same fp32 inputs through the same IEEE steps: the bytes and scales are the emulation's, exactly
    assert torch.equal(s, se)
    assert torch.equal(q.view(torch.uint8), qe.view(torch.uint8))
    assert s[3] == 0 and (q[3].view(torch.uint8) == 0).all()
    w64 = w.double()
    assert torch.equal(s.double(), (w64.abs().amax(1) / 448).float().double())
    assert ((dequantize(q, s).double() - w64).abs() <= half_step(w64, s.double().unsqueeze(1)) * (1 + 2 ** -18)).all()


@pytest.mark.parametrize("C_", [320, 640, 1280])
def test_layernorm_fp8(C_):
    rows, F, hw, rpg = 1003, 8, 17, 136
    x = rand(rows, C_, seed=1) * 3
    gamma, beta = rand(C_, seed=2) * 0.5 + 1, rand(C_, seed=3) * 0.1
    pre = rand((rows + rpg - 1) // rpg, C_, seed=4)
    pe = rand(F, C_, seed=5)
    q = Guarded8(rows, C_)
    s = GuardedF32(rows, 1)
    xo = Guarded(rows, C_)
    check(lib().hv_op_layernorm_fp8(ptr(x), ptr(gamma), ptr(beta), ptr(q.out), f32p(s.out), i64(rows), i64(C_), C.c_float(1e-5), ptr(pre),
                                    i64(rpg), ptr(xo.out), ptr(pe), i64(hw), i64(F), stream()))
    # the fp16 LayerNorm's x_out of the same call, for the bitwise check of the pre_add sum
    y16, xo16 = torch.empty(rows, C_, dtype=torch.half, device="cuda"), torch.empty(rows, C_, dtype=torch.half, device="cuda")
    check(lib().hv_op_layernorm(ptr(x), ptr(gamma), ptr(beta), ptr(y16), i64(rows), i64(C_), C.c_float(1e-5), ptr(pre), i64(rpg), ptr(xo16),
                                ptr(pe), i64(hw), i64(F), stream()))
    torch.cuda.synchronize()
    q.check_untouched(C_, "hv_op_layernorm_fp8")
    s.check_untouched("hv_op_layernorm_fp8")
    xo.check_untouched(cols_mask(rows, C_, C_), "hv_op_layernorm_fp8 x_out")
    assert torch.equal(xo.out.view(torch.int16), xo16.view(torch.int16))
    ridx = torch.arange(rows, device="cuda")
    xs = x.double() + pre.double()[ridx // rpg]   # the kernel normalises the fp32 sum; its fp16 copy x_out only feeds the residual
    ref = torch.nn.functional.layer_norm(xs, (C_,), eps=1e-5) * gamma.double() + beta.double() + pe.double()[(ridx // hw) % F]
    # fp32 LayerNorm against fp64: sums of C terms (C 2^-24 relative to the row's scale) and rsqrt (2 ulp); 1e-4 of the row's amax covers both
    amax = ref.abs().amax(1)
    sn = s.out[:, 0].double()
    assert ((sn - amax / 448).abs() <= 1e-4 * amax / 448).all()
    err = (dequantize(q.values(C_), s.out[:, 0]).double() - ref).abs()
    tol = half_step(ref.abs() * (1 + 1e-4), sn.unsqueeze(1)) * (1 + 2 ** -18) + 1e-4 * amax.unsqueeze(1)
    assert (err <= tol).all(), f"max excess {float((err - tol).max()):.3e}"


# ---------------------------------------------------------------- GEMM

def lvl(M, C_):
    return dict(M=M, C=C_)


# (config, level) -> tokens x frames and channels: config 2 (latent 96 x 72, 48 frames), config 5 level 0 (72 x 128, 48 frames)
LEVELS = {"c2l0": lvl(6912 * 48, 320), "c2l1": lvl(1728 * 48, 640), "c2l2": lvl(432 * 48, 1280), "c2l3": lvl(108 * 48, 1280),
          "c5l0": lvl(9216 * 48, 320)}
CASES = []
for name, L in LEVELS.items():
    CASES += [(f"{name}-qkv", L["M"], 3 * L["C"], L["C"], "rows", dict()),
              (f"{name}-ff1", L["M"], 8 * L["C"], L["C"], "geglu8", dict(bias=True)),
              (f"{name}-ff2", L["M"], L["C"], 4 * L["C"], "blocks", dict(bias=True, residual=True))]
CASES += [("edge-rowvec-res", 300, 320, 192, "rows", dict(bias=True, rowvec=True, residual=True)),   # M % 128, K = 1.5 k-blocks
          ("edge-geglu16", 1000, 2560, 320, "geglu16", dict(bias=True)),
          ("edge-geglu8-k64", 259, 512, 64, "geglu8", dict(bias=True)),                               # K = half a k-block
          ("edge-blocks-k320", 300, 640, 320, "blocks", dict(bias=True, residual=True)),                # per-128 scales, partial last block
          ("edge-blocks-1280", 517, 1280, 1280, "blocks", dict())]


def pack_geglu(w):
    out = torch.empty_like(w)
    check(lib().hv_pack_geglu(ptr(w), ptr(out), i64(w.shape[0]), i64(w.shape[1]), stream()))
    return out


@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_gemm_fp8(case):
    label, M, N, K, mode, opt = case
    geglu = mode.startswith("geglu")
    x = rand(M, K, seed=11)
    blk = 128 if mode == "blocks" else None
    if mode == "blocks":   # GEGLU-like activations: a few large values per row
        x = x * (1 + 8 * (rand(M, K, seed=12).float().abs() > 2.5))
    qa, sa = quantize(x.float(), blk)
    sa = sa.contiguous()
    w = rand(N, K, scale=K ** -0.5, seed=13)
    if geglu:
        w = pack_geglu(w)
    qw, sw = pack_rows(w)
    bias = rand(N, seed=14) * 0.1 if opt.get("bias") else None
    nout = N // 2 if geglu else N
    groups = 4
    rowvec = rand(groups, N, seed=15) * 0.1 if opt.get("rowvec") else None
    resid = rand(M, nout, seed=16) if opt.get("residual") else None
    ep = Epilogue()
    ep.bias = ptr(bias).value if bias is not None else None
    if rowvec is not None:
        ep.rowvec, ep.rowvec_ld, ep.rows_per_group = rowvec.data_ptr(), N, (M + groups - 1) // groups
    if resid is not None:
        ep.residual, ep.ldr = resid.data_ptr(), nout
    ep.geglu = 1 if geglu else 0
    if mode == "geglu8":
        out = Guarded8(M, nout + 16)
        osc = GuardedF32(M, N // 256 + 1)
        st = lib().hv_op_gemm_fp8(ptr(qa.view(torch.uint8)), i64(K), f32p(sa), i64(0), ptr(qw.view(torch.uint8)), f32p(sw), ptr(out.out),
                                  i64(nout + 16), f32p(osc.out), i64(N // 256 + 1), i64(M), i64(N), i64(K), C.byref(ep), stream())
    else:
        out = Guarded(M, nout + 8)
        st = lib().hv_op_gemm_fp8(ptr(qa.view(torch.uint8)), i64(K), f32p(sa), i64(sa.shape[1] if blk else 0), ptr(qw.view(torch.uint8)),
                                  f32p(sw), ptr(out.out), i64(nout + 8), None, i64(0), i64(M), i64(N), i64(K), C.byref(ep), stream())
    check(st)
    torch.cuda.synchronize()
    if mode == "geglu8":
        out.check_untouched(nout, label)
        sc = osc.out[:, : N // 256]
        assert torch.isnan(osc.out[:, N // 256:]).all() and torch.isnan(osc.buf[:osc.pad]).all() and torch.isnan(osc.buf[osc.pad + M:]).all(), label
        assert not torch.isnan(sc).any(), label
    else:
        out.check_untouched(cols_mask(M, nout + 8, nout), label)
    w64 = dequantize(qw, sw).double()
    b64 = bias.double() if bias is not None else None
    n_add = 4 if mode == "blocks" else (K + 31) // 32
    worst = 0.0
    for r0 in range(0, M, CHUNK):
        r1 = min(M, r0 + CHUNK)
        a64 = dequantize(qa[r0:r1], sa[r0:r1], blk).double()
        acc = a64 @ w64.T
        sabs = a64.abs() @ w64.abs().T
        e_acc = sabs * (n_add * U13 + 2 ** -22) + (sabs * ((K + 127) // 128) * 2 ** -24 if mode == "blocks" else 0)
        if b64 is not None:
            acc = acc + b64
        if rowvec is not None:
            acc = acc + rowvec.double()[torch.arange(r0, r1, device="cuda") // ((M + groups - 1) // groups)]
        if geglu:
            h, g = acc.view(r1 - r0, N // 256, 2, 128)[:, :, 0].reshape(r1 - r0, -1), acc.view(r1 - r0, N // 256, 2, 128)[:, :, 1].reshape(r1 - r0, -1)
            eh = e_acc.view(r1 - r0, N // 256, 2, 128)[:, :, 0].reshape(r1 - r0, -1)
            eg = e_acc.view(r1 - r0, N // 256, 2, 128)[:, :, 1].reshape(r1 - r0, -1)
            gel = torch.nn.functional.gelu(g)
            ref = h * gel
            # |d gelu / dg| <= 1.13; the erf polynomial and the approximate exp2 / rcp of geglu1: 1e-6 of |h| (|g| + 1)
            e_ref = gel.abs() * eh + (h.abs() + eh) * 1.13 * eg + 1e-6 * h.abs() * (g.abs() + 1)
        else:
            ref, e_ref = acc, e_acc
        if resid is not None:
            ref = ref + resid[r0:r1].double()
        if mode == "geglu8":
            s_n = sc[r0:r1].double()
            v = dequantize(out.values(nout)[r0:r1], sc[r0:r1], 128).double()
            # the block's scale: amax / 448 of the kernel's fp32 values, each within e_ref of fp64
            amax = ref.view(r1 - r0, -1, 128).abs().amax(-1)
            emax = e_ref.view(r1 - r0, -1, 128).amax(-1)
            assert ((s_n - amax / 448).abs() <= (emax + 2 ** -22 * amax) / 448).all(), f"{label}: block scales"
            sb = s_n.repeat_interleave(128, 1)
            tol = e_ref + half_step(ref.abs() + e_ref, sb) * (1 + 2 ** -18)
            err = (v - ref).abs()
            # aggregate: a rounding to nearest within half a step (<= 2^-4 of the value for normals) has an rms of at most 2^-4 / sqrt(3) of
            # the values; a scale a few percent off or a block's amax missing a lane would show as a larger error
            rel8 = float((v - ref).norm() / ref.norm())
            assert rel8 < 2 ** -4 / 3 ** 0.5, f"{label}: relative L2 of the e4m3 GEGLU output {rel8:.3e}"
        else:
            v = out.out[r0:r1, :nout].double()
            tol = e_ref + 2 ** -11 * ref.abs() * (1 + 2 ** -10) + 2 ** -22 * ref.abs() + 2 ** -25
            err = (v - ref).abs()
        bad = err > tol
        if bad.any():
            r, c = [int(t) for t in bad.nonzero()[0]]
            pytest.fail(f"{label}: {int(bad.sum())} elements out of bound, first row {r0 + r} col {c}: got {float(v[r, c])}, fp64 {float(ref[r, c])}, "
                        f"bound {float(tol[r, c]):.3e}")
        worst = max(worst, float((err / tol).max()))
        if mode != "geglu8":
            rel = float((v - ref).norm() / ref.norm())
            # expected error: the fp16 rounding (2^-11 / sqrt(3) rms) and the MMA's truncation well below it
            assert rel < 2e-3, f"{label}: relative L2 {rel:.2e}"
    print(f"{label}: worst error / bound {worst:.3f}")
