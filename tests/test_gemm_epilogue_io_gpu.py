"""The GEMM / conv epilogue's output and residual tiles move by TMA, which needs 16-byte aligned rows: hv_op_gemm and hv_op_conv3x3
reject a residual stride that is not a positive multiple of 8 and a residual or output pointer off a 16-byte boundary with
HV_ERR_INVALID and write nothing.  An output that is also the residual (updated in place) gives the same bits as separate buffers."""
import ctypes as C

import pytest
import torch

pytestmark = pytest.mark.gpu

from guarded import SENT, Guarded, bits, rand

if torch.cuda.is_available():
    from humanvid_b200._native import Epilogue, check, i32, i64, lib, ptr, stream

HV_ERR_INVALID = -1
M, N, K = 300, 320, 320
NF, H, W, CIN = 2, 9, 13, 64


def gemm(A, Wt, out_ptr, ldc, ep):
    return lib().hv_op_gemm(ptr(A), i64(A.stride(0)), ptr(None), i64(0), i64(0), ptr(Wt), out_ptr, i64(ldc), i64(A.shape[0]), i64(Wt.shape[0]),
                            i64(A.shape[1]), C.byref(ep), stream())


def conv(x, wp, out_ptr, ldc, ep):
    return lib().hv_op_conv3x3(ptr(x), ptr(wp), out_ptr, i64(ldc), i64(NF), i64(H), i64(W), i64(CIN), i64(N), i32(1), C.byref(ep), stream())


def residual_cases(res_full):
    """(label, residual pointer, ldr) that must be rejected; res_full is a [rows][N + 8] buffer."""
    base = res_full.data_ptr()
    return [("ldr % 8", base, N + 4), ("ldr = 0", base, 0), ("ldr < 0", base, -8), ("residual off 16 B", base + 2, N + 8)]


@pytest.mark.parametrize("op", ["gemm", "conv3x3"])
def test_rejects_misaligned_epilogue_io(op):
    rows = M if op == "gemm" else NF * H * W
    if op == "gemm":
        a, wt = rand(M, K, seed=1), rand(N, K, scale=K ** -0.5, seed=2)
        run = lambda out_ptr, ldc, ep: gemm(a, wt, out_ptr, ldc, ep)
    else:
        a, wt = rand(NF, H, W, CIN, seed=1), rand(N, 9 * CIN, scale=(9 * CIN) ** -0.5, seed=2)
        run = lambda out_ptr, ldc, ep: conv(a, wt, out_ptr, ldc, ep)
    res_full = rand(rows + 1, N + 8, seed=3)
    ldc = N + 8
    g = Guarded(rows, ldc)
    for label, rp, ldr in residual_cases(res_full):
        ep = Epilogue()
        ep.residual, ep.ldr = rp, ldr
        assert run(C.c_void_p(g.out.data_ptr()), ldc, ep) == HV_ERR_INVALID, f"{op}: {label} accepted"
        assert "residual" in lib().hv_ops_last_error().decode(), label
    ep = Epilogue()
    # a window one element into the allocation: every row start is off the 16-byte grid
    assert run(C.c_void_p(g.out.data_ptr() + 2), ldc, ep) == HV_ERR_INVALID, f"{op}: misaligned out accepted"
    assert "aligned" in lib().hv_ops_last_error().decode()
    torch.cuda.synchronize()
    assert bool((g.buf == SENT).all()), f"{op}: a rejected call wrote to the output"


@pytest.mark.parametrize("op", ["gemm", "conv3x3"])
def test_residual_in_place(op):
    rows = M if op == "gemm" else NF * H * W
    ldc = N + 16
    if op == "gemm":
        a, wt = rand(M, K, seed=4), rand(N, K, scale=K ** -0.5, seed=5)
        run = lambda out, ep: check(gemm(a, wt, C.c_void_p(out.data_ptr()), ldc, ep))
    else:
        a, wt = rand(NF, H, W, CIN, seed=4), rand(N, 9 * CIN, scale=(9 * CIN) ** -0.5, seed=5)
        run = lambda out, ep: check(conv(a, wt, C.c_void_p(out.data_ptr()), ldc, ep))
    res = torch.zeros(rows, ldc, dtype=torch.half, device="cuda")
    res[:, :N] = rand(rows, N, seed=6)
    sep = torch.zeros_like(res)
    ep = Epilogue()
    ep.residual, ep.ldr = res.data_ptr(), ldc
    run(sep, ep)
    inplace = res.clone()
    ep.residual = inplace.data_ptr()
    run(inplace, ep)
    torch.cuda.synchronize()
    assert torch.equal(bits(inplace[:, :N]), bits(sep[:, :N])), f"{op}: in-place residual differs from separate buffers"
    assert torch.equal(bits(inplace[:, N:]), bits(res[:, N:])), f"{op}: columns past N were written"
