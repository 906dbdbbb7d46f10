"""Every launch path of the wgmma GEMM / implicit-GEMM conv kernel (csrc/gemm.cu) against an fp64 reference, with guarded outputs;
the edges of the d = 512 attention with the same harness.

The output of every call is a window into a larger buffer pre-filled with a NaN sentinel, with guard rows before and after it and a row
stride wider than the columns written.  After the call every element outside [0, M) x [0, n_valid) must still be the sentinel bit for
bit, and every input must be unchanged.  Each written element must be within one fp16 rounding plus fp32-accumulation noise of the fp64
result of the same fp16 inputs:

    |out - ref| <= 2^-10 |ref| + 1e-4 rms(ref)

so that one wrong column, row or tile fails the test even where it would barely move the relative L2 error of the whole output.

Linear shapes are derived from the device's SM count, and hv_dbg_gemm_plan (the host function hv_op_gemm launches with) confirms that
each case runs the tile width and variant (ring or B-stationary) it is named after.
"""
import ctypes as C

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

from conftest import report
from guarded import SENT, Guarded, bits, check_inputs_unchanged, cols_mask, rand, strided

if torch.cuda.is_available():
    from humanvid_b200._native import ACT_RELU, ACT_SILU, Epilogue, check, i32, i64, lib, ptr, stream


def check_close(out, ref, label, block_n=None, row_of=None):
    """Relative L2 < 1e-3 and the per-element bound; the first violation is reported with its row / column and CTA tile."""
    out64 = out.double()
    assert torch.isfinite(out64).all(), f"{label}: non-finite output at {(~torch.isfinite(out64)).nonzero()[0].tolist()}"
    err = (out64 - ref).abs()
    rms = float(ref.pow(2).mean().sqrt())
    bound = 2.0 ** -10 * ref.abs() + 1e-4 * rms
    rel = float((out64 - ref).norm() / (ref.norm() + 1e-30))
    viol = err > bound
    if viol.any():
        r, c = [int(v) for v in viol.nonzero()[0]]
        tile = f", tile (m {r // 128}, n {c // block_n})" if block_n else ""
        pytest.fail(f"{label}: {int(viol.sum())} elements over the bound, first at row {r}{'' if row_of is None else ' ' + row_of(r)}, column {c}"
                    f"{tile}: out {float(out64[r, c]):.6g} ref {float(ref[r, c]):.6g}; worst err/bound {float((err / bound).max()):.2f}; rel L2 {rel:.2e}")
    assert rel < 1e-3, f"{label}: rel L2 {rel:.2e}"
    return rel


def sms():
    return int(lib().hv_num_sms())


def gemm_plan(M, N, K, geglu=False):
    bn, st, grid = C.c_int32(), C.c_int32(), C.c_int32()
    check(lib().hv_dbg_gemm_plan(i64(M), i64(N), i64(K), i32(int(geglu)), C.byref(bn), C.byref(st), C.byref(grid)))
    return bn.value, st.value, grid.value


# ------------------------------------------------------------------------------------------------------------- linears
def m_for_bst(n_tiles, s, tail=37):
    """M whose m tiles are enough for the B-stationary variant (>= 2 per CTA sharing an n tile), with a partial last M tile and a
    tile count that is not a multiple of the grid (m_tiles % per_col != 0)."""
    per_col = s // n_tiles
    m_tiles = 2 * per_col + 3 if per_col > 3 else 2 * per_col + 1
    return m_tiles * 128 - tail


def m_for_ring(N, bn, s, tail=51):
    """M with enough tiles that pick_block_n keeps the widest tile (no SMs left idle), with a partial last M tile."""
    return (s // ((N + bn - 1) // bn) + 3) * 128 - tail


# name: (N, K, K1, bn, bst, epilogue, M rule).  K1 > 0: columns [K1, K) come from a second A source (split-K).
LINEAR = {
    "ring128": (384, 1280, 0, 128, False, "plain", "ring"),
    "ring160": (320, 1280, 0, 160, False, "plain", "ring"),
    "ring256": (1280, 1280, 0, 256, False, "plain", "ring"),
    "ring_idle_sms_128": (1280, 1280, 0, 128, False, "plain", 300),         # 256 wide would leave SMs idle -> 128
    "ring160_epilogue": (640, 1280, 0, 160, False, "full", "ring"),
    "bst128": (384, 320, 0, 128, True, "plain", "bst"),
    "bst160": (320, 320, 0, 160, True, "plain", "bst"),                     # level-0 linear
    "bst256": (1280, 320, 0, 256, True, "plain", "bst"),
    "bst128_epilogue": (384, 320, 0, 128, True, "full", "bst"),
    "bst160_epilogue": (320, 320, 0, 160, True, "full", "bst"),             # level-0 attention out-projection + residual
    "bst256_epilogue": (1280, 320, 0, 256, True, "full", "bst"),
    "bst256_geglu": (2560, 320, 0, 256, True, "geglu", "bst"),              # level-0 feed-forward
    "bst128_splitk": (384, 456, 256, 128, True, "plain", "bst"),
    "bst160_splitk": (320, 320, 192, 160, True, "plain", "bst"),
    "bst256_splitk": (1280, 320, 128, 256, True, "plain", "bst"),
    "bst128_partial_n": (328, 200, 0, 128, True, "bias", "bst"),            # last N tile: 72 of 128 columns
    "bst160_partial_n": (296, 200, 0, 160, True, "bias", "bst"),            # 136 of 160
    "bst256_partial_n": (488, 200, 0, 256, True, "bias", "bst"),            # 232 of 256
    "ring128_partial_n": (328, 1000, 0, 128, False, "bias", "ring"),
    "ring160_partial_n": (296, 1000, 0, 160, False, "bias", "ring"),
    "ring256_partial_n": (488, 1000, 0, 256, False, "bias", "ring"),
    "k40": (320, 40, 0, 160, None, "plain", "ring"),
    "k200": (320, 200, 0, 160, None, "plain", "ring"),
    "k328": (320, 328, 0, 160, None, "plain", "ring"),
    "k200_splitk64": (320, 200, 64, 160, None, "plain", "ring"),
    "k328_splitk256": (320, 328, 256, 160, None, "plain", "ring"),
    "k328_splitk256_bst": (384, 328, 256, 128, True, "bias", "bst"),
    "nvalid_relu": (320, 320, 0, 160, None, "nvalid_relu", "ring"),
}


@pytest.mark.parametrize("name", list(LINEAR))
def test_linear_path(name):
    N, K, K1, want_bn, want_bst, epi, mrule = LINEAR[name]
    s = sms()
    geglu = epi == "geglu"
    n_tiles_of = lambda bn: (N + bn - 1) // bn
    M = m_for_bst(n_tiles_of(want_bn), s) if mrule == "bst" else m_for_ring(N, want_bn, s) if mrule == "ring" else mrule
    bn, stages, grid = gemm_plan(M, N, K, geglu)
    m_tiles = (M + 127) // 128
    plan = f"{name}: M={M} N={N} K={K} K1={K1} -> BLOCK_N {bn}, {'BST ' + str(stages) + ' stages' if stages else 'ring'}, grid {grid}, {m_tiles * n_tiles_of(bn)} tiles on {s} SMs"
    report("gemm plan " + plan)
    assert bn == want_bn, plan
    if want_bst is not None:
        assert (stages > 0) == want_bst, plan
    if stages and mrule == "bst":
        assert (m_tiles * n_tiles_of(bn)) % grid != 0 and M % 128 != 0, plan

    # A (and A2) in wider allocations whose extra columns are NaN: a read past K (or K1) poisons the output
    if K1:
        A = strided(M, K1, K1 + 24, seed=1)
        A2 = strided(M, K - K1, K - K1 + 40, seed=2)
    else:
        A, A2 = strided(M, K, K + 16, seed=1), None
    W = rand(N, K, scale=K ** -0.5, seed=3)
    out_n = N // 2 if geglu else N
    n_valid = out_n - 40 if epi == "nvalid_relu" else out_n
    ldc = out_n + 24
    ep = Epilogue()
    inputs = [A, W] + ([A2] if K1 else [])
    a_full = torch.cat([A, A2], 1).double() if K1 else A.double()
    ref = a_full @ W.double().t()
    if epi in ("bias", "full", "geglu", "nvalid_relu"):
        bias = rand(N, seed=4)
        ep.bias = bias.data_ptr()
        inputs.append(bias)
        ref = ref + bias.double()
    if epi == "full":
        rpg = 1000                                                   # row groups end mid-tile (1000 % 128 != 0)
        groups = (M + rpg - 1) // rpg
        rv_ld = N + 8
        rowvec = strided(groups, N, rv_ld, seed=5)
        res_ld = N + 40
        res = strided(M, N, res_ld, seed=6)
        ep.rowvec, ep.rowvec_ld, ep.rows_per_group = rowvec.data_ptr(), rv_ld, rpg
        ep.residual, ep.ldr, ep.act = res.data_ptr(), res_ld, ACT_SILU
        inputs += [rowvec, res]
        ref = F.silu(ref + rowvec.double().repeat_interleave(rpg, 0)[:M]) + res.double()
    if epi == "nvalid_relu":
        ep.act, ep.n_valid = ACT_RELU, n_valid
        ref = F.relu(ref)
    if geglu:
        ep.geglu = 1
        # packed order: every 256-row block of W is [128 hidden | 128 gate]; output column j of block b is hidden row 128 b + j
        blk = ref.view(M, N // 256, 2, 128)
        ref = (blk[:, :, 0] * F.gelu(blk[:, :, 1])).reshape(M, N // 2)
    ref = ref[:, :n_valid]

    before = [bits(t) for t in inputs]
    g = Guarded(M, ldc)
    check(lib().hv_op_gemm(ptr(A), i64(A.stride(0)), ptr(A2), i64(A2.stride(0) if K1 else 0), i64(K1), ptr(W), ptr(g.out), i64(ldc), i64(M),
                           i64(N), i64(K), C.byref(ep), stream()))
    torch.cuda.synchronize()
    g.check_untouched(cols_mask(M, ldc, n_valid), name)
    check_inputs_unchanged(before, inputs, name)
    check_close(g.out[:, :n_valid], ref, name, block_n=bn // 2 if geglu else bn)


# ------------------------------------------------------------------------------------------------------------- convolutions
def conv_box(NF, H, W):
    """The (frames, rows, cols) box of 128 output pixels choose_conv_box picks (least padding, ties to the widest W)."""
    up = lambda a, b: -(-a // b) * b
    best, box = -1, None
    w = 128
    while w >= 1:
        h = 128 // w
        while h >= 1:
            n = 128 // (w * h)
            padded = up(NF, n) * up(H, h) * up(W, w)
            if best < 0 or padded < best:
                best, box = padded, (n, h, w)
            h >>= 1
        w >>= 1
    return box


def pack_conv(w):
    Cout, Cin = w.shape[:2]
    wp = torch.empty(Cout, 9 * Cin, device="cuda", dtype=torch.half)
    check(lib().hv_pack_conv3x3(ptr(w), ptr(wp), i64(Cout), i64(Cin), i64(Cout), i64(Cin), stream()))
    return wp


def conv_ref64(x, w, stride, pad_end):
    xc = x.permute(0, 3, 1, 2).double()
    if pad_end:
        y = F.conv2d(F.pad(xc, (0, 1, 0, 1)), w.double(), stride=2)
    else:
        y = F.conv2d(xc, w.double(), stride=stride, padding=1)
    return y.permute(0, 2, 3, 1).reshape(-1, w.shape[0])


# name: (NF, H, W, Cin, Cout, mode, epilogue, frames per rowvec group).  NF / H / W are not multiples of any power of two, so whatever
# box choose_conv_box picks, every box dimension has a tail; Cout = 200 is a partial last tile for every tile width.
CONV = {
    "s1_bias": (3, 13, 7, 128, 200, "s1", "bias", 0),
    "s2_bias": (5, 26, 14, 64, 200, "s2", "bias", 0),
    "s2_pad_end_bias": (5, 26, 14, 64, 200, "s2_end", "bias", 0),
    "s1_rowvec_silu": (6, 5, 7, 64, 200, "s1", "rowvec_silu", 3),            # the box spans frames of two batch items
    "s1_residual": (3, 13, 7, 128, 200, "s1", "residual", 0),
    "s2_rowvec_silu_residual": (6, 10, 14, 64, 136, "s2", "full", 3),
}


@pytest.mark.parametrize("name", list(CONV))
def test_conv_path(name):
    NF, H, W, Cin, Cout, mode, epi, fpg = CONV[name]
    x = rand(NF, H, W, Cin, seed=20)
    w = rand(Cout, Cin, 3, 3, scale=(9 * Cin) ** -0.5, seed=21)
    wp = pack_conv(w)
    Ho, Wo = (H, W) if mode == "s1" else (H // 2, W // 2)
    M = NF * Ho * Wo
    ldc = Cout + 24
    bias = rand(Cout, seed=22)
    ep = Epilogue(bias=bias.data_ptr())
    inputs = [x, wp, bias]
    ref = conv_ref64(x, w, 1 if mode == "s1" else 2, mode == "s2_end") + bias.double()
    if epi in ("rowvec_silu", "full"):
        box = conv_box(NF, Ho, Wo)
        assert box[0] > 1 and fpg % box[0] != 0, f"box {box} does not span two batch items"
        rpg = fpg * Ho * Wo
        rv_ld = Cout + 8
        rowvec = strided(NF // fpg, Cout, rv_ld, seed=23)
        ep.rowvec, ep.rowvec_ld, ep.rows_per_group, ep.act = rowvec.data_ptr(), rv_ld, rpg, ACT_SILU
        inputs.append(rowvec)
        ref = F.silu(ref + rowvec.double().repeat_interleave(rpg, 0))
    if epi in ("residual", "full"):
        res_ld = Cout + 40
        res = strided(M, Cout, res_ld, seed=24)
        ep.residual, ep.ldr = res.data_ptr(), res_ld
        inputs.append(res)
        ref = ref + res.double()
    before = [bits(t) for t in inputs]
    g = Guarded(M, ldc)
    if mode == "s2_end":
        st = lib().hv_op_conv3x3_s2_pad_end(ptr(x), ptr(wp), ptr(g.out), i64(ldc), i64(NF), i64(H), i64(W), i64(Cin), i64(Cout), C.byref(ep), stream())
    else:
        st = lib().hv_op_conv3x3(ptr(x), ptr(wp), ptr(g.out), i64(ldc), i64(NF), i64(H), i64(W), i64(Cin), i64(Cout), i32(1 if mode == "s1" else 2),
                                 C.byref(ep), stream())
    check(st)
    torch.cuda.synchronize()
    g.check_untouched(cols_mask(M, ldc, Cout), name)
    check_inputs_unchanged(before, inputs, name)
    row_of = lambda r: f"(frame {r // (Ho * Wo)}, y {r // Wo % Ho}, x {r % Wo})"
    check_close(g.out[:, :Cout], ref, f"{name} box {conv_box(NF, Ho, Wo)}", row_of=row_of)


@pytest.mark.parametrize("NF,H,W,Cin,Cout", [(3, 13, 7, 64, 256), (1, 5, 3, 128, 128)])
def test_upconv_path(NF, H, W, Cin, Cout):
    """Upsample + conv as four 2x2 convolutions: the fp64 reference is built from the packed weights read back (each parity's 2x2 taps),
    so the per-element bound applies; test_ops_gpu checks the packing itself against upsample + conv."""
    x = rand(NF, H, W, Cin, seed=25)
    w = rand(Cout, Cin, 3, 3, scale=(9 * Cin) ** -0.5, seed=26)
    bias = rand(Cout, seed=27)
    wp = torch.empty(4 * Cout, 4 * Cin, device="cuda", dtype=torch.half)
    check(lib().hv_pack_upconv2x2(ptr(w), ptr(wp), i64(Cout), i64(Cin), stream()))
    ldc = Cout + 24
    M = NF * 4 * H * W
    inputs = [x, wp, bias]
    before = [bits(t) for t in inputs]
    ep = Epilogue(bias=bias.data_ptr())
    g = Guarded(M, ldc)
    check(lib().hv_op_upconv2x2(ptr(x), ptr(wp), ptr(g.out), i64(ldc), i64(NF), i64(H), i64(W), i64(Cin), i64(Cout), C.byref(ep), stream()))
    # parity (py, px), tap 2a + b: output (2y + py, 2x + px) reads source (y + a + py - 1, x + b + px - 1), k = tap * Cin + c
    xp = F.pad(x.permute(0, 3, 1, 2).double(), (1, 1, 1, 1))
    ref = torch.empty(NF, 2 * H, 2 * W, Cout, dtype=torch.float64, device="cuda")
    for py in range(2):
        for px in range(2):
            k2 = wp[(2 * py + px) * Cout : (2 * py + px + 1) * Cout].double().view(Cout, 2, 2, Cin).permute(0, 3, 1, 2)
            y = F.conv2d(xp[:, :, py : py + H + 1, px : px + W + 1], k2) + bias.double()[None, :, None, None]
            ref[:, py::2, px::2] = y.permute(0, 2, 3, 1)
    torch.cuda.synchronize()
    g.check_untouched(cols_mask(M, ldc, Cout), "upconv")
    check_inputs_unchanged(before, inputs, "upconv")
    Ho, Wo = 2 * H, 2 * W
    check_close(g.out[:, :Cout], ref.reshape(M, Cout), f"upconv box {conv_box(NF, H, W)}",
                row_of=lambda r: f"(frame {r // (Ho * Wo)}, y {r // Wo % Ho}, x {r % Wo})")


# ------------------------------------------------------------------------------------------------------------- batched B (V^T)
@pytest.mark.parametrize("name,rows,K,rowbias,wide", [("t128_rows100", 100, 200, True, False), ("t128_rows300_small_grid", 300, 320, False, False),
                                                      ("t256_rows300", 300, 200, True, True), ("t256_rows129", 129, 512, False, True)])
def test_gemm_batched_b(name, rows, K, rowbias, wide):
    """out[m][n * out_stride + j] = A[m] . X[n][j] (+ rowbias[m]); the pad columns [rows, round8(rows)) are written as rowbias and the rest
    of each segment, and the columns past the last segment, keep the sentinel.  Tile width 256 is taken for rows > 128 once the grid is
    large enough (m_tiles * batch * ceil(rows / 256) >= SMs / 2), 128 otherwise."""
    s = sms()
    M = 200
    m_tiles = (M + 127) // 128
    per_256 = m_tiles * ((rows + 255) // 256)
    batch = (s // 2 + per_256 - 1) // per_256 + 1 if wide else 2
    assert (rows > 128 and m_tiles * batch * ((rows + 255) // 256) >= s // 2) == wide
    r8 = (rows + 7) // 8 * 8
    out_stride = r8 + 16
    ldc = batch * out_stride + 24
    A = strided(M, K, K + 8, scale=K ** -0.5, seed=30)
    X = rand(batch, rows, K, seed=31)
    rb = rand(M, seed=32) if rowbias else None
    inputs = [A, X] + ([rb] if rowbias else [])
    before = [bits(t) for t in inputs]
    g = Guarded(M, ldc)
    check(lib().hv_op_gemm_batched_b(ptr(A), i64(A.stride(0)), ptr(X), i64(K), ptr(g.out), i64(ldc), i64(M), i64(batch), i64(rows), i64(out_stride),
                                     i64(K), ptr(rb), stream()))
    torch.cuda.synchronize()
    written = torch.zeros(M, ldc, dtype=torch.bool, device="cuda")
    for n in range(batch):
        written[:, n * out_stride : n * out_stride + r8] = True
    g.check_untouched(written, name)
    check_inputs_unchanged(before, inputs, name)
    ref = torch.einsum("mk,njk->mnj", A.double(), X.double())
    rbd = rb.double()[:, None, None] if rowbias else torch.zeros(M, 1, 1, dtype=torch.float64, device="cuda")
    ref = ref + rbd
    out = g.out[:, : batch * out_stride].reshape(M, batch, out_stride)
    pad = out[:, :, rows:r8]
    assert torch.equal(pad.double(), rbd.expand_as(pad)), f"{name}: pad columns [rows, round8(rows)) are not 0 + rowbias"
    check_close(out[:, :, :rows].reshape(M, batch * rows), ref.reshape(M, batch * rows), name)


# ------------------------------------------------------------------------------------------------------------- d = 512 attention
@pytest.mark.parametrize("scale", [1.0, 8.0])
@pytest.mark.parametrize("L", [1, 7, 63, 64, 65, 127, 129])
def test_attention_d512_edges(L, scale):
    """hv_op_attention_d512 at a single partial query / key tile, exact multiples of the 64-row tiles and one past them, with Q and K
    optionally scaled x8 (scores of std 64: the lazy rescale fires and most exp2 arguments are far below zero), row strides wider than 512
    with NaN in the gaps, and a guarded output.  P is rounded to fp16, so the bound is relative L2 per query row (<= 3e-3), not per element."""
    NF, D = 3, 512
    ldq, ldk, ldo = D + 64, D + 128, D + 24
    q = strided(NF * L, D, ldq, scale=scale, seed=L)
    k = strided(NF * L, D, ldk, scale=scale, seed=L + 1)
    v = rand(NF, L, D, seed=L + 2)
    vt_stride = (L + 7) // 8 * 8 + 8
    vt = torch.full((D, NF * vt_stride + 8), SENT, dtype=torch.int16, device="cuda").view(torch.half)   # pad columns must never be read
    for n in range(NF):
        vt[:, n * vt_stride : n * vt_stride + L] = v[n].t()
    inputs = [q, k, vt]
    before = [bits(t) for t in inputs]
    g = Guarded(NF * L, ldo)
    check(lib().hv_op_attention_d512(ptr(q), i64(ldq), ptr(k), i64(ldk), ptr(vt), i64(vt.stride(0)), i64(vt_stride), ptr(g.out), i64(ldo), i64(NF),
                                     i64(L), stream()))
    torch.cuda.synchronize()
    label = f"attention d512 L={L} x{scale:g}"
    g.check_untouched(cols_mask(NF * L, ldo, D), label)
    check_inputs_unchanged(before, inputs, label)
    qd, kd = q.double().view(NF, L, D), k.double().view(NF, L, D)
    ref = (torch.softmax(qd @ kd.transpose(1, 2) / D ** 0.5, dim=-1) @ v.double()).reshape(NF * L, D)
    out = g.out[:, :D].double()
    assert torch.isfinite(out).all(), label
    e = (out - ref).norm(dim=1) / ref.norm(dim=1)
    worst = int(e.argmax())
    assert float(e.max()) <= 3e-3, f"{label}: query row {worst} (frame {worst // L}, token {worst % L}, query tile {worst % L // 64}) rel {float(e.max()):.3e}"
