"""The FP8 quantisation scheme's emulation (tests/fp8_emulation.py) and the argument checks of the three e4m3 entry points
(include/hv_b200_fp8.h), without a GPU."""
import ctypes as C

import numpy as np
import pytest
import torch

from fp8_emulation import E4M3, dequantize, half_step, quantize

# ---------------------------------------------------------------- the scheme


def test_per_row_scale_and_step_order():
    g = torch.Generator().manual_seed(0)
    x = torch.randn(64, 320, generator=g) * torch.logspace(-3, 3, 64).unsqueeze(1)
    q, s = quantize(x)
    amax = x.abs().amax(1).numpy().astype(np.float32)
    np.testing.assert_array_equal(s.numpy(), amax / np.float32(448))              # s = amax / 448, one fp32 division
    inv = np.float32(448) / amax
    np.testing.assert_array_equal(q.float().numpy(), torch.from_numpy(x.numpy() * inv[:, None]).to(E4M3).float().numpy())
    assert (q.float().abs().amax(1) == 448).all()                                 # the row maximum lands on 448 exactly


def test_per_block_scales():
    g = torch.Generator().manual_seed(1)
    x = torch.randn(8, 320, generator=g)
    x[:, 128:256] *= 100
    q, s = quantize(x, 128)
    assert s.shape == (8, 3)
    for kb in range(3):
        blk = x[:, kb * 128:(kb + 1) * 128]
        assert torch.equal(s[:, kb], blk.abs().amax(1) / 448)
        assert torch.equal(q[:, kb * 128:(kb + 1) * 128].float(), quantize(blk)[0].float())
    assert torch.allclose(dequantize(q, s, 128), x, rtol=2 ** -4, atol=0)


def test_saturation_at_448():
    x = torch.tensor([[1.0, -1.0, 0.5]])
    inv = torch.tensor(448.0) / 1.0
    assert (x * inv).abs().max() == 448
    q, s = quantize(x)
    assert q.float().tolist() == [[448.0, -448.0, 224.0]]
    # a value whose fp32 product lands past 448 (rounding of x * inv) saturates instead of becoming NaN
    big = torch.tensor([[1.0, 1.0000001]])
    q, _ = quantize(big)
    assert q.float().abs().max() == 448 and not torch.isnan(q.float()).any()


def test_subnormals():
    # e4m3 subnormals are k * 2^-9, k = 1..7, below 2^-6
    x = torch.tensor([[448.0, 2.0 ** -9, 3 * 2.0 ** -9, 2.0 ** -10, 2.0 ** -11, 2.0 ** -7 + 2.0 ** -10]])
    q, s = quantize(x)
    assert s.item() == 1.0
    assert q.float().tolist() == [[448.0, 2.0 ** -9, 3 * 2.0 ** -9, 0.0, 0.0, 2.0 ** -7]]   # ties to even: 2^-10 -> 0, 2^-7 + 2^-10 -> 2^-7
    v = dequantize(q, s)
    assert ((v - x).abs() <= half_step(x, s.unsqueeze(1))).all()


def test_zero_rows_and_blocks():
    x = torch.zeros(3, 256)
    x[1, 5] = 3.0
    q, s = quantize(x)
    s3 = float(np.float32(3) / np.float32(448))
    assert s.tolist() == [0.0, s3, 0.0]
    assert (q[0].view(torch.uint8) == 0).all() and (q[2].view(torch.uint8) == 0).all()
    qb, sb = quantize(x, 128)
    assert sb[1].tolist() == [s3, 0.0] and (qb[1, 128:].view(torch.uint8) == 0).all()
    assert torch.equal(dequantize(q, s), x)


def test_half_step_bound_holds_for_random_rows():
    g = torch.Generator().manual_seed(2)
    x = torch.randn(256, 1280, generator=g) * torch.logspace(-4, 4, 256).unsqueeze(1)
    x[:, ::7] *= 1e-4   # spread values down into the subnormal range of each row
    q, s = quantize(x)
    v = dequantize(q, s)
    # + the fp32 roundings of x * inv and of q * s, each 2^-24 of a value at most 2^4 half steps large
    assert ((v - x).abs() <= half_step(x, s.unsqueeze(1)) * (1 + 2 ** -18)).all()


# ---------------------------------------------------------------- argument checks of the entry points

needs_no_gpu = pytest.mark.skipif(torch.cuda.is_available(), reason="hands fake device addresses to the library: only without a CUDA device")
HV_ERR_INVALID = -1
NULL = None


def P(i, off=0):
    return 0x7F0000000000 + (i << 20) + off


def _ptr(v):
    return C.c_void_p(v)


def _i64(v):
    return C.c_int64(v)


def _f32(v):
    return C.c_float(v)


def _ep(**kw):
    from humanvid_b200._native import Epilogue

    e = Epilogue()
    for k, v in kw.items():
        setattr(e, k, v)
    return C.byref(e)


GEMM = [("A", _ptr, P(1)), ("lda", _i64, 320), ("a_scale", _ptr, P(2)), ("a_scale_ld", _i64, 0), ("W", _ptr, P(3)), ("w_scale", _ptr, P(4)),
        ("out", _ptr, P(5)), ("ldc", _i64, 960), ("out_scale", _ptr, NULL), ("out_scale_ld", _i64, 0), ("M", _i64, 300), ("N", _i64, 960),
        ("K", _i64, 320), ("ep", None, lambda: _ep())]
GEGLU8 = dict(N=2560, ldc=1280, out_scale=P(6), out_scale_ld=10, ep=lambda: _ep(geglu=1))
OPS = {
    "hv_op_gemm_fp8": (GEMM, {
        "NULL A": dict(A=NULL), "NULL a_scale": dict(a_scale=NULL), "NULL W": dict(W=NULL), "NULL w_scale": dict(w_scale=NULL),
        "NULL out": dict(out=NULL), "M = 0": dict(M=0), "N = 0": dict(N=0), "K = 0": dict(K=0), "M past int32": dict(M=2 ** 31),
        "K % 16": dict(K=328, lda=336), "lda % 16": dict(lda=328), "lda < K": dict(lda=304), "N % 8": dict(N=964, ldc=968),
        "misaligned A": dict(A=P(1, 8)), "misaligned a_scale": dict(a_scale=P(2, 4)), "misaligned w_scale": dict(w_scale=P(4, 8)),
        "a_scale_ld < ceil(K/128)": dict(a_scale_ld=2), "a_scale_ld < 0": dict(a_scale_ld=-3), "geglu N % 256": dict(ep=lambda: _ep(geglu=1)),
        "geglu with per-block A scales": dict(N=2560, ldc=1280, a_scale_ld=3, ep=lambda: _ep(geglu=1)),
        "e4m3 out without geglu": dict(out_scale=P(6), out_scale_ld=10, ldc=960),
        "e4m3 out with residual": dict(GEGLU8, ep=lambda: _ep(geglu=1, residual=P(7), ldr=1280)),
        "e4m3 out with n_valid": dict(GEGLU8, ep=lambda: _ep(geglu=1, n_valid=640)),
        "e4m3 out ldc % 16": dict(GEGLU8, ldc=1288), "e4m3 out ldc < N/2": dict(GEGLU8, ldc=1264),
        "e4m3 out_scale_ld < N/256": dict(GEGLU8, out_scale_ld=9), "misaligned out_scale": dict(GEGLU8, out_scale=P(6, 4)),
        "e4m3 out misaligned": dict(GEGLU8, out=P(5, 8)),
        "fp16 out ldc % 8": dict(ldc=964), "fp16 out misaligned": dict(out=P(5, 2)),
        "residual ldr % 8": dict(ep=lambda: _ep(residual=P(7), ldr=964)), "residual misaligned": dict(ep=lambda: _ep(residual=P(7, 2), ldr=960)),
    }),
    "hv_op_layernorm_fp8": ([("X", _ptr, P(1)), ("gamma", _ptr, P(2)), ("beta", _ptr, P(3)), ("out", _ptr, P(4)), ("out_scale", _ptr, P(5)),
                             ("rows", _i64, 100), ("C", _i64, 320), ("eps", _f32, 1e-5), ("pre_add", _ptr, P(6)), ("rows_per_group", _i64, 50),
                             ("x_out", _ptr, P(7)), ("pe", _ptr, P(8)), ("hw", _i64, 10), ("F", _i64, 5)], {
        "NULL X": dict(X=NULL), "NULL gamma": dict(gamma=NULL), "NULL beta": dict(beta=NULL), "NULL out": dict(out=NULL),
        "NULL out_scale": dict(out_scale=NULL), "misaligned out": dict(out=P(4, 8)), "misaligned out_scale": dict(out_scale=P(5, 4)),
        "misaligned X": dict(X=P(1, 2)), "misaligned pre_add": dict(pre_add=P(6, 2)), "misaligned pe": dict(pe=P(8, 8)), "rows = 0": dict(rows=0),
        "C % 16": dict(C=328), "C = 1296": dict(C=1296), "F past int32": dict(F=2 ** 31)}),
    "hv_pack_fp8_rows": ([("W", _ptr, P(1)), ("out", _ptr, P(2)), ("scale", _ptr, P(3)), ("rows", _i64, 2560), ("K", _i64, 320)], {
        "NULL W": dict(W=NULL), "NULL out": dict(out=NULL), "NULL scale": dict(scale=NULL), "misaligned W": dict(W=P(1, 2)),
        "misaligned out": dict(out=P(2, 8)), "misaligned scale": dict(scale=P(3, 4)), "rows = 0": dict(rows=0), "K = 0": dict(K=0),
        "K % 16": dict(K=328), "rows past int32": dict(rows=2 ** 31)}),
}


def _call(fn, spec, over):
    from humanvid_b200._native import lib

    args = []
    for name, kind, value in spec:
        v = over.get(name, value)
        args.append(v() if kind is None else kind(v))
    return getattr(lib(), fn)(*args, C.c_void_p(0))


def test_every_fp8_entry_point_is_covered():
    import os
    import re

    src = open(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "include", "hv_b200_fp8.h")).read()
    assert set(re.findall(r"\b(hv_(?:op|pack)_[a-z0-9_]+)\s*\(", re.sub(r"/\*.*?\*/", "", src, flags=re.S))) == set(OPS)


@needs_no_gpu
@pytest.mark.parametrize("fn", sorted(OPS))
def test_rejected_before_any_cuda_call(fn):
    from humanvid_b200._native import lib

    spec, cases = OPS[fn]
    st = _call(fn, spec, {})
    assert st in (-2, -3), f"{fn}: the accepted argument set returned {st} ({lib().hv_ops_last_error().decode()})"
    if fn == "hv_op_gemm_fp8":   # the accepted e4m3-output and per-block-scale sets get past the checks too
        for over in (GEGLU8, dict(a_scale_ld=3), dict(GEGLU8, ep=lambda: _ep(geglu=1, bias=P(9)))):
            assert _call(fn, spec, over) in (-2, -3), lib().hv_ops_last_error().decode()
    for label, over in cases.items():
        st = _call(fn, spec, over)
        msg = lib().hv_ops_last_error().decode()
        assert st == HV_ERR_INVALID, f"{fn} {label}: status {st} ({msg}), expected HV_ERR_INVALID"
        assert msg.startswith(fn + ":") or msg.startswith(fn + " "), f"{fn} {label}: message {msg!r} does not name the operator"


def test_hv_config_fp8_field_is_mirrored():
    """hv_config.fp8_linears is the struct's last field, appended after the layout of earlier releases, and HvConfig mirrors it."""
    import os
    import re

    from humanvid_b200.modules import HvConfig

    src = open(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "include", "hv_b200.h")).read()
    body = re.sub(r"/\*.*?\*/", "", src[src.index("typedef struct hv_config"):src.index("} hv_config;")], flags=re.S)
    names = re.findall(r"\b(\w+)\s*(?:\[\d+\])?;", body)
    assert names[-2:] == ["no_mid_motion_module", "fp8_linears"]
    assert [f[0] for f in HvConfig._fields_] == names
    assert HvConfig.fp8_linears.offset == HvConfig.no_mid_motion_module.offset + 4
    assert HvConfig().fp8_linears == 0
