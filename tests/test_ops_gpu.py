"""Operator-level parity tests on an H100: each C-ABI operator vs a plain torch fp32 reference of the same op."""
import ctypes as C

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

if torch.cuda.is_available():
    from humanvid_b200 import _native as N
    from humanvid_b200._native import Epilogue, check, i32, i64, lib, ptr, stream


def rel(a, b):
    a, b = a.float(), b.float()
    return float((a - b).norm() / (b.norm() + 1e-12))


def dev(*shape, scale=1.0, seed=0):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return (torch.randn(*shape, generator=g, device="cuda") * scale).half()


def gemm(A, W, M, N, K, ep=None, A2=None, K1=0, ldc=None):
    out_n = N // 2 if (ep is not None and ep.geglu) else N
    ldc = ldc or out_n
    out = torch.zeros(M, ldc, device="cuda", dtype=torch.half)
    check(lib().hv_op_gemm(ptr(A), i64(A.stride(0)), ptr(A2), i64(A2.stride(0) if A2 is not None else 0), i64(K1), ptr(W), ptr(out),
                           i64(ldc), i64(M), i64(N), i64(K), C.byref(ep) if ep is not None else None, stream()))
    return out


@pytest.mark.parametrize("M,N,K", [(128, 128, 64), (256, 256, 128), (1000, 320, 320), (6912, 640, 1280), (333, 2560, 320), (4096, 384, 320), (40000, 640, 1280), (38000, 320, 2560), (41000, 1280, 1024)])
def test_gemm_plain(M, N, K):
    A, W = dev(M, K, seed=1), dev(N, K, scale=K ** -0.5, seed=2)
    out = gemm(A, W, M, N, K)
    ref = A.float() @ W.float().t()
    # on-device cross-check with the slow CUDA-core kernel localises descriptor/layout faults
    dbg = torch.empty(M, N, device="cuda", dtype=torch.float32)
    check(lib().hv_dbg_gemm(ptr(A), i64(K), ptr(W), ptr(dbg), i64(M), i64(N), i64(K), stream()))
    torch.cuda.synchronize()
    assert rel(dbg, ref) < 1e-5
    assert rel(out, ref) < 1e-3, f"gemm mismatch rel={rel(out, ref)}"


def test_gemm_epilogue_bias_rowvec_residual_silu():
    M, N, K = 2 * 300, 320, 640
    A, W = dev(M, K, seed=3), dev(N, K, scale=K ** -0.5, seed=4)
    bias, rowvec, res = dev(N, seed=5), dev(2, N, seed=6), dev(M, N, seed=7)
    ep = Epilogue(bias=ptr(bias).value, rowvec=ptr(rowvec).value, rowvec_ld=N, rows_per_group=300, residual=ptr(res).value, ldr=N,
                  act=N_ACT_SILU, geglu=0, n_valid=0)
    out = gemm(A, W, M, N, K, ep)
    # fp32 through bias -> row vector -> SiLU -> residual, one rounding at the store (include/hv_b200_ops.h)
    v = A.float() @ W.float().t() + bias.float() + rowvec.float().repeat_interleave(300, 0)
    v = F.silu(v) + res.float()
    torch.cuda.synchronize()
    assert rel(out, v) < 1e-3


N_ACT_SILU = 2


def test_gemm_geglu():
    M, C_ = 700, 320
    A = dev(M, C_, seed=8)
    Wfull = dev(8 * C_, C_, scale=C_ ** -0.5, seed=9)
    bfull = dev(8 * C_, seed=10)
    Wp, bp = torch.empty_like(Wfull), torch.empty(8 * C_, 8, device="cuda", dtype=torch.half)
    check(lib().hv_pack_geglu(ptr(Wfull), ptr(Wp), i64(8 * C_), i64(C_), stream()))
    b8 = bfull[:, None].repeat(1, 8).contiguous()
    check(lib().hv_pack_geglu(ptr(b8), ptr(bp), i64(8 * C_), i64(8), stream()))
    bpk = bp[:, 0].contiguous()
    ep = Epilogue(bias=ptr(bpk).value, geglu=1)
    out = gemm(A, Wp, M, 8 * C_, C_, ep)
    proj = A.float() @ Wfull.float().t() + bfull.float()
    hid, gate = proj.chunk(2, dim=-1)
    ref = hid * F.gelu(gate)
    torch.cuda.synchronize()
    assert rel(out, ref) < 1e-3


def test_gemm_split_k_sources():
    M, K1, K2, N = 500, 640, 320, 320
    A1, A2, W = dev(M, K1, seed=11), dev(M, K2, seed=12), dev(N, K1 + K2, scale=(K1 + K2) ** -0.5, seed=13)
    out = gemm(A1, W, M, N, K1 + K2, A2=A2, K1=K1)
    ref = torch.cat([A1, A2], 1).float() @ W.float().t()
    torch.cuda.synchronize()
    assert rel(out, ref) < 1e-3


def conv_ref(x_nhwc, w, bias, stride):
    y = F.conv2d(x_nhwc.permute(0, 3, 1, 2).float(), w.float(), bias.float() if bias is not None else None, stride=stride, padding=1)
    return y.permute(0, 2, 3, 1).contiguous()


@pytest.mark.parametrize("NF,H,W,Cin,Cout,stride", [(2, 16, 16, 64, 128, 1), (3, 24, 18, 128, 320, 1), (4, 12, 9, 320, 64, 1),
                                                      (2, 96, 72, 64, 64, 1), (2, 16, 16, 64, 128, 2), (3, 24, 18, 128, 128, 2),
                                                      (2, 96, 72, 64, 64, 2), (5, 8, 8, 640, 8, 1), (8, 96, 72, 128, 320, 1), (24, 48, 36, 192, 640, 1), (48, 24, 18, 128, 1280, 1),
                                                      (16, 96, 72, 128, 320, 2)])
def test_conv3x3(NF, H, W, Cin, Cout, stride):
    x = dev(NF, H, W, Cin, seed=20)
    w = dev(Cout, Cin, 3, 3, scale=(9 * Cin) ** -0.5, seed=21)
    bias = dev(Cout, seed=22)
    wp = torch.empty(Cout, 9 * Cin, device="cuda", dtype=torch.half)
    check(lib().hv_pack_conv3x3(ptr(w), ptr(wp), i64(Cout), i64(Cin), i64(Cout), i64(Cin), stream()))
    Ho, Wo = (H, W) if stride == 1 else (H // 2, W // 2)
    out = torch.zeros(NF * Ho * Wo, Cout, device="cuda", dtype=torch.half)
    ep = Epilogue(bias=ptr(bias).value)
    check(lib().hv_op_conv3x3(ptr(x), ptr(wp), ptr(out), i64(Cout), i64(NF), i64(H), i64(W), i64(Cin), i64(Cout), i32(stride), C.byref(ep), stream()))
    ref = conv_ref(x, w, bias, stride).reshape(-1, Cout)
    torch.cuda.synchronize()
    assert rel(out, ref) < 1e-3, rel(out, ref)


@pytest.mark.parametrize("NF,H,W,Cin,Cout", [(2, 12, 9, 1280, 1280), (3, 24, 18, 640, 640), (2, 48, 36, 320, 320), (1, 5, 7, 64, 128), (48, 12, 9, 1280, 1280)])
def test_upconv2x2_is_upsample_then_conv(NF, H, W, Cin, Cout):
    """Upsample3D (resnet.py:68-71, :49): F.interpolate(nearest, 2x) + 3x3 conv, computed as four 2x2 convs of the source."""
    x = dev(NF, H, W, Cin, seed=25)
    w = dev(Cout, Cin, 3, 3, scale=(9 * Cin) ** -0.5, seed=26)
    bias = dev(Cout, seed=27)
    wp = torch.empty(4 * Cout, 4 * Cin, device="cuda", dtype=torch.half)
    check(lib().hv_pack_upconv2x2(ptr(w), ptr(wp), i64(Cout), i64(Cin), stream()))
    out = torch.zeros(NF * 4 * H * W, Cout, device="cuda", dtype=torch.half)
    ep = Epilogue(bias=ptr(bias).value)
    check(lib().hv_op_upconv2x2(ptr(x), ptr(wp), ptr(out), i64(Cout), i64(NF), i64(H), i64(W), i64(Cin), i64(Cout), C.byref(ep), stream()))
    up = F.interpolate(x.permute(0, 3, 1, 2).float(), scale_factor=2.0, mode="nearest")
    ref = F.conv2d(up, w.float(), bias.float(), padding=1).permute(0, 2, 3, 1).reshape(-1, Cout)
    torch.cuda.synchronize()
    assert rel(out, ref) < 1e-3, rel(out, ref)


@pytest.mark.parametrize("B,Fr,H,W", [(1, 3, 40, 56), (2, 2, 19, 130), (1, 1, 8, 64), (1, 4, 128, 1152), (1, 1, 5, 7)])
def test_pose_conv_in_from_planar_image(B, Fr, H, W):
    """pose_guider.py:25 conv_in (3 -> 16) + SiLU straight from the planar image: tiles of 8 x 64 outputs, ragged edges, several batch items,
    more tiles than resident blocks."""
    img = torch.rand(B, 3, Fr, H, W, device="cuda").half()
    w, b = dev(16, 3, 3, 3, scale=0.2, seed=36), dev(16, seed=37)
    out = torch.full((B * Fr, H, W, 16), 9.0, device="cuda", dtype=torch.half)
    check(lib().hv_op_pose_conv_in(ptr(img), ptr(w), ptr(b), ptr(out), i64(B), i64(Fr), i64(H), i64(W), i32(2), stream()))
    ref = torch.cat([F.silu(F.conv2d(img[i].permute(1, 0, 2, 3).float(), w.float(), b.float(), padding=1)).permute(0, 2, 3, 1) for i in range(B)])
    torch.cuda.synchronize()
    assert rel(out, ref) < 1e-3
    assert float((out.float() - ref).abs().max()) < 4e-3      # every pixel, edges included (fp16 half-ulp of |y| <= 4 is 1e-3)
    out2 = torch.empty_like(out)
    check(lib().hv_op_pose_conv_in(ptr(img), ptr(w), ptr(None), ptr(out2), i64(B), i64(Fr), i64(H), i64(W), i32(0), stream()))   # no bias, no activation
    ref2 = torch.cat([F.conv2d(img[i].permute(1, 0, 2, 3).float(), w.float(), None, padding=1).permute(0, 2, 3, 1) for i in range(B)])
    torch.cuda.synchronize()
    assert rel(out2, ref2) < 1e-3


@pytest.mark.parametrize("d,Fr", [(40, 24), (80, 24), (160, 24), (40, 8), (16, 5), (40, 32)])
def test_temporal_attention(d, Fr):
    B, HW, heads = 2, 37, 8
    Cc = heads * d
    qkv = dev(B * Fr * HW, 3 * Cc, seed=60)
    out = torch.zeros(B * Fr * HW, Cc, device="cuda", dtype=torch.half)
    check(lib().hv_op_temporal_attention(ptr(qkv), ptr(out), i64(B), i64(Fr), i64(HW), i32(heads), i32(d), stream()))
    q, k, v = qkv.float().reshape(B, Fr, HW, 3, heads, d).permute(3, 0, 2, 4, 1, 5)  # (b, hw, h, f, d)
    ref = F.scaled_dot_product_attention(q, k, v).permute(0, 3, 1, 2, 4).reshape(B * Fr * HW, Cc)
    torch.cuda.synchronize()
    assert rel(out, ref) < 1e-3


@pytest.mark.parametrize("d,Fr,HW", [(40, 24, 300), (80, 24, 300), (40, 8, 700), (40, 32, 300), (80, 5, 1100), (40, 17, 301)])
def test_temporal_attention_tma_staged(d, Fr, HW):
    """>= 4096 (pixel, head) problems at d = 40 / 80: the TMA-staged kernel (per-warp shared-memory slabs, ldmatrix fragments)."""
    B, heads = 2, 8
    Cc = heads * d
    qkv = dev(B * Fr * HW, 3 * Cc, seed=61)
    out = torch.zeros(B * Fr * HW, Cc, device="cuda", dtype=torch.half)
    check(lib().hv_op_temporal_attention(ptr(qkv), ptr(out), i64(B), i64(Fr), i64(HW), i32(heads), i32(d), stream()))
    q, k, v = qkv.float().reshape(B, Fr, HW, 3, heads, d).permute(3, 0, 2, 4, 1, 5)  # (b, hw, h, f, d)
    ref = F.scaled_dot_product_attention(q, k, v).permute(0, 3, 1, 2, 4).reshape(B * Fr * HW, Cc)
    torch.cuda.synchronize()
    assert torch.isfinite(out).all()
    assert rel(out, ref) < 1e-3


def attention_case(NF, L, heads, d, Lb=0, Fr=1, nf_nobank=0, seed=70):
    dpad = (d + 15) // 16 * 16
    q = dev(NF * L, heads, d, seed=seed)
    k = dev(NF * L, heads, d, seed=seed + 1)
    v = dev(NF * L, heads, d, seed=seed + 2)
    qk = torch.zeros(NF * L, 2, heads, dpad, device="cuda", dtype=torch.half)
    qk[:, 0, :, :d] = q
    qk[:, 1, :, :d] = k
    qk = qk.reshape(NF * L, 2 * heads * dpad)
    Lp = (L + 7) // 8 * 8
    ldvt = NF * Lp
    dv = (d + 1 + 15) // 16 * 16
    sel = torch.zeros(heads, dv, heads, d, device="cuda", dtype=torch.half)  # row h*dv+c picks channel h*d+c
    ones = torch.zeros(heads, dv, device="cuda", dtype=torch.half)
    for hh in range(heads):
        sel[hh, :d, hh, :] = torch.eye(d, device="cuda", dtype=torch.half)
        ones[hh, d] = 1
    sel = sel.reshape(heads * dv, heads * d).contiguous()
    vt = torch.zeros(heads * dv, NF, Lp, device="cuda", dtype=torch.half)
    check(lib().hv_op_gemm_batched_b(ptr(sel), i64(heads * d), ptr(v.reshape(NF * L, heads * d)), i64(heads * d), ptr(vt), i64(ldvt),
                                     i64(heads * dv), i64(NF), i64(L), i64(Lp), i64(heads * d), ptr(ones), stream()))
    torch.cuda.synchronize()
    vt4 = vt.reshape(heads, dv, NF, Lp)
    assert torch.equal(vt4[:, :d, :, :L], v.reshape(NF, L, heads, d).permute(2, 3, 0, 1)), "batched-B GEMM (V^T producer) mismatch"
    assert torch.equal(vt4[:, d, :, :L], torch.ones_like(vt4[:, d, :, :L]))
    out = torch.zeros(NF * L, heads * d, device="cuda", dtype=torch.half)
    kb = vbt = None
    B = NF // Fr
    if Lb:
        kbr = dev(B * Lb, heads, d, seed=seed + 3)
        vbr = dev(B * Lb, heads, d, seed=seed + 4)
        kb = torch.zeros(B * Lb, heads, dpad, device="cuda", dtype=torch.half)
        kb[:, :, :d] = kbr
        kb = kb.reshape(B * Lb, heads * dpad)
        Lbp = (Lb + 7) // 8 * 8
        vbt = torch.zeros(heads, dv, B, Lbp, device="cuda", dtype=torch.half)
        vbt[:, :d, :, :Lb] = vbr.reshape(B, Lb, heads, d).permute(2, 3, 0, 1)
        vbt[:, d, :, :Lb] = 1
        vbt = vbt.reshape(heads * dv, B * Lbp)
    k_view = qk[:, heads * dpad:]
    check(lib().hv_op_attention(ptr(qk), C.c_void_p(k_view.data_ptr()), ptr(vt), ptr(out), i64(NF), i64(L), i32(heads), i32(d),
                                i64(2 * heads * dpad), i64(2 * heads * dpad), i64(ldvt), i64(heads * d), ptr(kb), ptr(vbt), i64(Lb),
                                i64(heads * dpad), i64(vbt.stride(0) if vbt is not None else 0), i64(Fr), i64(nf_nobank), i64(Lp),
                                i64((Lb + 7) // 8 * 8), stream()))
    qf = q.float().reshape(NF, L, heads, d).transpose(1, 2)
    kf = k.float().reshape(NF, L, heads, d).transpose(1, 2)
    vf = v.float().reshape(NF, L, heads, d).transpose(1, 2)
    ref = torch.empty(NF, heads, L, d, device="cuda")
    for n in range(NF):
        kk, vv = kf[n], vf[n]
        if Lb and n >= nf_nobank:
            b = n // Fr
            kk = torch.cat([kk, kbr.float().reshape(B, Lb, heads, d)[b].transpose(0, 1)], 1)
            vv = torch.cat([vv, vbr.float().reshape(B, Lb, heads, d)[b].transpose(0, 1)], 1)
        ref[n] = F.scaled_dot_product_attention(qf[n], kk, vv)
    ref = ref.transpose(1, 2).reshape(NF * L, heads * d)
    torch.cuda.synchronize()
    return rel(out, ref)


@pytest.mark.parametrize("NF,L,heads,d", [(1, 128, 1, 40), (2, 256, 8, 40), (3, 432, 8, 160), (2, 300, 8, 80), (2, 1728, 8, 40), (2, 108, 8, 16), (3, 108, 8, 160), (2, 4, 8, 32),
                                          (1, 6912, 8, 40), (1, 9216, 8, 40), (1, 2304, 8, 80)])   # level-0 token counts of configs 2-4 (96x72) and 5 (72x128)
def test_attention_self(NF, L, heads, d):
    assert attention_case(NF, L, heads, d) < 1e-3


def test_attention_with_reference_bank():
    # 2 batch items x 3 frames; first batch item (uncond half) ignores the bank
    assert attention_case(6, 432, 8, 40, Lb=432, Fr=3, nf_nobank=3) < 1e-3
    assert attention_case(4, 200, 8, 80, Lb=200, Fr=2, nf_nobank=2, seed=90) < 1e-3
    # level-0 shape with banks (config 3: 6912 + 6912 keys; config 5: 9216 + 9216), one unconditional and one conditional frame
    assert attention_case(2, 6912, 8, 40, Lb=6912, Fr=1, nf_nobank=1, seed=91) < 1e-3
    assert attention_case(2, 9216, 8, 40, Lb=9216, Fr=1, nf_nobank=1, seed=92) < 1e-3
