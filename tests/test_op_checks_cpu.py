"""Every operator entry point checks its arguments before it makes any CUDA call.  For each hv_op_* / hv_pack_* function this builds an
argument set the checks accept and, from it, sets that change one argument the operator cannot run; each of those must return
HV_ERR_INVALID (-1) with a message naming the operator.  On a machine without a GPU an accepted set gets as far as the device query or the
launch and fails there with HV_ERR_CUDA (or HV_ERR_TMA), so a check that is missing, or that runs after the device query, shows up as -2.

The addresses are fake (non-NULL, 256-byte aligned, never dereferenced on the host), so the module only runs where no CUDA device exists."""
import ctypes as C
import os
import re

import pytest
import torch

pytestmark = pytest.mark.skipif(torch.cuda.is_available(), reason="hands fake device addresses to the library: only without a CUDA device")

from humanvid_b200._native import Epilogue, lib  # noqa: E402

HV_ERR_INVALID = -1
NULL = None


def P(i, off=0):
    """Fake device address number i, `off` bytes past a 256-byte boundary."""
    return 0x7F0000000000 + (i << 20) + off


def ptr(v):
    return C.c_void_p(v)


def i64(v):
    return C.c_int64(v)


def i32(v):
    return C.c_int32(v)


def f32(v):
    return C.c_float(v)


def ep(**kw):
    e = Epilogue()
    for k, v in kw.items():
        setattr(e, k, v)
    return C.byref(e)


def ptrs(*vals):
    return (C.c_void_p * len(vals))(*vals)


# entry point -> (operator name in the message, [(argument, type, value the checks accept)], {case: {argument: value}})
EPI_IO = {"out off 16 B": dict(out=P(3, 2)), "ldr % 8": dict(ep=lambda: ep(residual=P(4), ldr=324)), "ldr = 0": dict(ep=lambda: ep(residual=P(4), ldr=0)),
          "ldr < 0": dict(ep=lambda: ep(residual=P(4), ldr=-8)), "residual off 16 B": dict(ep=lambda: ep(residual=P(4, 2), ldr=320))}
CONV = [("X", ptr, P(1)), ("Wp", ptr, P(2)), ("out", ptr, P(3)), ("ldc", i64, 320), ("NF", i64, 2), ("H", i64, 8), ("W", i64, 14), ("Cin", i64, 64),
        ("Cout", i64, 320)]
GN = [("X", ptr, P(1)), ("C1", i64, 640), ("X2", ptr, P(2)), ("C2", i64, 640), ("gamma", ptr, P(3)), ("beta", ptr, P(4)), ("out", ptr, P(5)),
      ("NF", i64, 6), ("HW", i64, 108), ("groups", i32, 32), ("eps", f32, 1e-5), ("silu", i32, 1)]
GN_CASES = {"NULL X": dict(X=NULL), "NULL gamma": dict(gamma=NULL), "NULL beta": dict(beta=NULL), "NULL out": dict(out=NULL),
            "NULL stats": dict(stats=NULL), "X2 NULL with C2 > 0": dict(X2=NULL), "NF = 0": dict(NF=0), "NF > 65535": dict(NF=65536),
            "HW = 0": dict(HW=0), "misaligned X": dict(X=P(1, 2)), "misaligned X2": dict(X2=P(2, 8)), "misaligned gamma": dict(gamma=P(3, 2)),
            "misaligned out": dict(out=P(5, 2)), "misaligned stats": dict(stats=P(6, 4)), "C1 not a multiple of 8": dict(C1=636, C2=644),
            "odd channels per group": dict(C1=320, C2=320, groups=128), "too many groups": dict(groups=320), "C > 8192": dict(C1=8192, C2=8),
            "C < 8": dict(C1=4, C2=0, X2=NULL, groups=2)}
ATTN = [("Q", ptr, P(1)), ("K", ptr, P(2)), ("Vt", ptr, P(3)), ("out", ptr, P(4)), ("NF", i64, 6), ("L", i64, 129), ("heads", i32, 3), ("d", i32, 40),
        ("ldq", i64, 144), ("ldk", i64, 144), ("ldvt", i64, 6 * 136), ("ldo", i64, 120), ("Kb", ptr, P(5)), ("Vbt", ptr, P(6)), ("Lb", i64, 200),
        ("ldkb", i64, 144), ("ldvbt", i64, 3 * 200), ("F", i64, 2), ("nf_nobank", i64, 2), ("vt_stride", i64, 136), ("vbt_stride", i64, 200)]

OPS = {
    "hv_op_gemm": ("hv_op_gemm",
                   [("A", ptr, P(1)), ("lda", i64, 320), ("A2", ptr, NULL), ("lda2", i64, 0), ("K1", i64, 0), ("W", ptr, P(2)), ("out", ptr, P(3)),
                    ("ldc", i64, 320), ("M", i64, 300), ("N", i64, 320), ("K", i64, 320), ("ep", None, lambda: ep())],
                   {"NULL A": dict(A=NULL), "NULL W": dict(W=NULL), "NULL out": dict(out=NULL), "M = 0": dict(M=0), "K % 8": dict(K=324),
                    "ldc % 8": dict(ldc=324), "split K1 % 64": dict(A2=P(5), lda2=320, K1=100), "geglu N % 256": dict(ep=lambda: ep(geglu=1)), **EPI_IO}),
    "hv_op_gemm_batched_b": ("hv_op_gemm_batched_b",
                             [("A", ptr, P(1)), ("lda", i64, 320), ("X", ptr, P(2)), ("ldx", i64, 320), ("out", ptr, P(3)), ("ldc", i64, 208),
                              ("M", i64, 200), ("batch", i64, 2), ("rows", i64, 100), ("out_stride", i64, 104), ("K", i64, 320), ("rowbias", ptr, NULL)],
                             {"NULL A": dict(A=NULL), "NULL X": dict(X=NULL), "NULL out": dict(out=NULL), "M = 0": dict(M=0), "batch = 0": dict(batch=0),
                              "out_stride < rows": dict(out_stride=96), "out_stride % 8": dict(out_stride=108)}),
    "hv_op_conv3x3": ("hv_op_conv3x3", CONV + [("stride", i32, 1), ("ep", None, lambda: ep())],
                      {"NULL X": dict(X=NULL), "NULL Wp": dict(Wp=NULL), "NULL out": dict(out=NULL), "Cin % 64": dict(Cin=32), "stride 3": dict(stride=3),
                       "NF = 0": dict(NF=0), **EPI_IO}),
    "hv_op_conv3x3_s2_pad_end": ("hv_op_conv3x3", CONV + [("ep", None, lambda: ep())],
                                 {"NULL X": dict(X=NULL), "Cout % 8": dict(Cout=324), "out off 16 B": dict(out=P(3, 2))}),
    "hv_op_upconv2x2": ("hv_op_upconv2x2", CONV + [("ep", None, lambda: ep())],
                        {"NULL X": dict(X=NULL), "NULL Wp": dict(Wp=NULL), "NULL out": dict(out=NULL), "Cin % 64": dict(Cin=96), "H = 0": dict(H=0),
                         "residual epilogue": dict(ep=lambda: ep(residual=P(4), ldr=320))}),
    "hv_pack_upconv2x2": ("hv_pack_upconv2x2", [("W", ptr, P(1)), ("out", ptr, P(2)), ("Cout", i64, 320), ("Cin", i64, 320)],
                          {"NULL W": dict(W=NULL), "NULL out": dict(out=NULL), "Cout = 0": dict(Cout=0), "Cin past int32": dict(Cin=2 ** 31)}),
    "hv_op_conv3x3_small": ("hv_op_conv3x3_small",
                            [("X", ptr, P(1)), ("Wp", ptr, P(2)), ("bias", ptr, P(3)), ("out", ptr, P(4)), ("ldo", i64, 16), ("NF", i64, 2),
                             ("H", i64, 16), ("W", i64, 32), ("Cin", i64, 16), ("Cout", i64, 16), ("stride", i32, 1), ("act", i32, 2)],
                            {"NULL X": dict(X=NULL), "NULL Wp": dict(Wp=NULL), "NULL out": dict(out=NULL), "(16, 16, 2)": dict(stride=2),
                             "misaligned X": dict(X=P(1, 2)), "misaligned Wp": dict(Wp=P(2, 8)), "misaligned out": dict(out=P(4, 2)),
                             "NF > 65535": dict(NF=65536), "odd H at stride 2": dict(Cout=32, stride=2, H=15), "ldo % 8": dict(ldo=20),
                             "ldo < Cout": dict(ldo=8)}),
    "hv_op_pose_conv_in": ("hv_op_pose_conv_in",
                           [("X", ptr, P(1)), ("W", ptr, P(2)), ("bias", ptr, P(3)), ("out", ptr, P(4)), ("B", i64, 1), ("F", i64, 2), ("H", i64, 16),
                            ("Wd", i64, 64), ("act", i32, 2)],
                           {"NULL X": dict(X=NULL), "NULL W": dict(W=NULL), "NULL out": dict(out=NULL), "misaligned out": dict(out=P(4, 2)),
                            "B = 0": dict(B=0), "H = 0": dict(H=0)}),
    "hv_op_clip_patchify": ("hv_op_clip_patchify",
                            [("X", ptr, P(1)), ("out", ptr, P(2)), ("B", i64, 1), ("C", i64, 3), ("S", i64, 224), ("p", i64, 14), ("Kpad", i64, 592)],
                            {"NULL X": dict(X=NULL), "NULL out": dict(out=NULL), "224 % 15": dict(p=15, Kpad=680), "Kpad < 588": dict(Kpad=584),
                             "Kpad % 8": dict(Kpad=596), "B = 0": dict(B=0)}),
    "hv_op_conv3x3_direct": ("hv_op_conv3x3_direct",
                             [("X", ptr, P(1)), ("W", ptr, P(2)), ("bias", ptr, P(3)), ("out", ptr, P(4)), ("NF", i64, 2), ("H", i64, 32), ("Wd", i64, 24),
                              ("Cin", i64, 3), ("Cout", i64, 16), ("stride", i32, 1), ("act", i32, 2), ("add", ptr, NULL)],
                             {"NULL X": dict(X=NULL), "NULL W": dict(W=NULL), "NULL out": dict(out=NULL), "stride 3": dict(stride=3), "Cin = 0": dict(Cin=0),
                              "NF = 0": dict(NF=0), "H past int32": dict(H=2 ** 31)}),
    "hv_op_groupnorm": ("hv_op_groupnorm", GN + [("stats", ptr, P(6))], GN_CASES),
    "hv_op_groupnorm_pooled": ("hv_op_groupnorm_pooled", GN + [("F", i64, 3), ("stats", ptr, P(6))],
                               {**GN_CASES, "NF not a multiple of F": dict(F=4), "F = 0": dict(F=0), "F < 0": dict(F=-3)}),
    "hv_op_layernorm": ("hv_op_layernorm",
                        [("X", ptr, P(1)), ("gamma", ptr, P(2)), ("beta", ptr, P(3)), ("out", ptr, P(4)), ("rows", i64, 100), ("C", i64, 320),
                         ("eps", f32, 1e-5), ("pre_add", ptr, P(5)), ("rows_per_group", i64, 50), ("x_out", ptr, P(6)), ("pe", ptr, P(7)), ("hw", i64, 10),
                         ("F", i64, 5)],
                        {"C = 1288": dict(C=1288), "misaligned X": dict(X=P(1, 2)), "NULL X": dict(X=NULL), "NULL gamma": dict(gamma=NULL),
                         "NULL beta": dict(beta=NULL), "NULL out": dict(out=NULL), "rows = 0": dict(rows=0), "C % 8": dict(C=324),
                         "misaligned pre_add": dict(pre_add=P(5, 2)), "misaligned x_out": dict(x_out=P(6, 2)), "misaligned pe": dict(pe=P(7, 8)),
                         "F past int32": dict(F=2 ** 31)}),
    "hv_op_attention": ("hv_op_attention", ATTN,
                        {"NF=0": dict(NF=0), "L=0": dict(L=0), "heads=0": dict(heads=0), "d=24": dict(d=24), "nf_nobank=-1": dict(nf_nobank=-1),
                         "nf_nobank>NF": dict(nf_nobank=7), "F does not divide NF": dict(F=4), "ldo<heads*d": dict(ldo=112),
                         "ldq<heads*dpad": dict(ldq=136), "ldk<heads*dpad": dict(ldk=136), "ldkb<heads*dpad": dict(ldkb=136),
                         "ldvt<NF*vt_stride": dict(ldvt=6 * 136 - 8), "ldvbt<B*vbt_stride": dict(ldvbt=3 * 200 - 8), "vbt_stride<Lb": dict(vbt_stride=192),
                         "Vbt NULL": dict(Vbt=NULL, nf_nobank=6), "F=0 with a bank": dict(F=0), "NULL Q": dict(Q=NULL), "NULL out": dict(out=NULL),
                         "NF>65535": dict(NF=65536, L=1, vt_stride=8, ldvt=65536 * 8, Kb=NULL),
                         "heads>65535": dict(heads=65536, d=8, ldq=65536 * 16, ldk=65536 * 16, ldo=65536 * 8, Kb=NULL)}),
    "hv_op_attention_d512": ("hv_op_attention_d512",
                             [("Q", ptr, P(1)), ("ldq", i64, 1024), ("K", ptr, P(2)), ("ldk", i64, 1024), ("Vt", ptr, P(3)), ("ldvt", i64, 2000),
                              ("vt_stride", i64, 1000), ("out", ptr, P(4)), ("ldo", i64, 512), ("NF", i64, 2), ("L", i64, 1000)],
                             {"NULL Q": dict(Q=NULL), "NULL out": dict(out=NULL), "NF = 0": dict(NF=0), "NF > 65535": dict(NF=65536), "L = 0": dict(L=0),
                              "ldq < 512": dict(ldq=504), "vt_stride < L": dict(vt_stride=992)}),
    "hv_op_temporal_attention": ("hv_op_temporal_attention",
                                 [("QKV", ptr, P(1)), ("out", ptr, P(2)), ("B", i64, 1), ("F", i64, 32), ("HW", i64, 37), ("heads", i32, 8), ("d", i32, 40)],
                                 {"B=0": dict(B=0), "F=0": dict(F=0), "F=33": dict(F=33), "HW=0": dict(HW=0), "heads=0": dict(heads=0), "d=24": dict(d=24),
                                  "d=64": dict(d=64, heads=5), "NULL QKV": dict(QKV=NULL), "NULL out": dict(out=NULL)}),
    "hv_op_ncfhw_to_nhwc": ("hv_op_ncfhw_to_nhwc",
                            [("X", ptr, P(1)), ("out", ptr, P(2)), ("B", i64, 2), ("C", i64, 4), ("F", i64, 3), ("H", i64, 16), ("W", i64, 12),
                             ("src_fp32", i32, 0)],
                            {"B*F = 65536": dict(F=32768), "NULL X": dict(X=NULL), "NULL out": dict(out=NULL), "C = 0": dict(C=0), "H = 0": dict(H=0),
                             "H*W past int32": dict(H=2 ** 20, W=2 ** 12)}),
    "hv_op_nhwc_to_ncfhw": ("hv_op_nhwc_to_ncfhw",
                            [("X", ptr, P(1)), ("ldx", i64, 8), ("out", ptr, P(2)), ("B", i64, 2), ("C", i64, 4), ("F", i64, 3), ("H", i64, 16),
                             ("W", i64, 12)],
                            {"ldx < C": dict(ldx=2), "NULL X": dict(X=NULL), "NULL out": dict(out=NULL), "B*F = 65536": dict(F=32768)}),
    "hv_op_pixel_unshuffle": ("hv_op_pixel_unshuffle",
                              [("X", ptr, P(1)), ("out", ptr, P(2)), ("B", i64, 1), ("C", i64, 6), ("F", i64, 2), ("H", i64, 16), ("W", i64, 24),
                               ("r", i32, 8)],
                              {"r = 0": dict(r=0), "H % r": dict(H=20), "W < r": dict(W=4), "NULL X": dict(X=NULL), "NULL out": dict(out=NULL), "B = 0": dict(B=0), "C r^2 past int32": dict(C=2 ** 26)}),
    "hv_op_plucker_unshuffle": ("hv_op_plucker_unshuffle",
                                [("K", ptr, P(1)), ("c2w", ptr, P(2)), ("out", ptr, P(3)), ("NF", i64, 2), ("H", i64, 64), ("W", i64, 64), ("r", i32, 8)],
                                {"NULL K": dict(K=NULL), "NULL c2w": dict(c2w=NULL), "NULL out": dict(out=NULL), "NF = 0": dict(NF=0), "r = 0": dict(r=0),
                                 "H % r": dict(H=60), "H past int32": dict(H=2 ** 33)}),
    "hv_op_small_linear": ("hv_op_small_linear",
                           [("X", ptr, P(1)), ("W", ptr, P(2)), ("bias", ptr, P(3)), ("out", ptr, P(4)), ("M", i64, 2), ("N", i64, 320), ("K", i64, 1280),
                            ("act_in", i32, 2)],
                           {"M = 0": dict(M=0), "NULL X": dict(X=NULL), "NULL W": dict(W=NULL), "NULL out": dict(out=NULL), "K odd": dict(K=1279),
                            "misaligned X": dict(X=P(1, 2))}),
    "hv_op_timestep_embedding": ("hv_op_timestep_embedding", [("t", i64, 959), ("out", ptr, P(1)), ("B", i64, 2), ("dim", i64, 320)],
                                 {"NULL out": dict(out=NULL), "B = 0": dict(B=0), "dim odd": dict(dim=321), "dim = 0": dict(dim=0)}),
    "hv_pack_conv3x3": ("hv_pack_conv3x3", [("W", ptr, P(1)), ("out", ptr, P(2)), ("Cout", i64, 16), ("Cin", i64, 3), ("Cout_pad", i64, 16), ("Cin_pad", i64, 64)],
                        {"NULL W": dict(W=NULL), "NULL out": dict(out=NULL), "Cout_pad < Cout": dict(Cout_pad=8), "Cin = 0": dict(Cin=0)}),
    "hv_pack_geglu": ("hv_pack_geglu", [("W", ptr, P(1)), ("out", ptr, P(2)), ("rows", i64, 2560), ("K", i64, 320)],
                      {"NULL W": dict(W=NULL), "NULL out": dict(out=NULL), "rows % 256": dict(rows=2568), "K = 0": dict(K=0)}),
    "hv_pack_heads": ("hv_pack_heads", [("W", ptr, P(1)), ("out", ptr, P(2)), ("heads", i32, 8), ("d", i32, 40), ("dpad", i32, 48), ("K", i64, 320)],
                      {"NULL W": dict(W=NULL), "NULL out": dict(out=NULL), "dpad < d": dict(dpad=32), "heads = 0": dict(heads=0)}),
    "hv_op_window_gather": ("hv_op_window_gather",
                            [("latents", ptr, P(1)), ("idx", ptr, P(2)), ("out", ptr, P(3)), ("Bl", i64, 1), ("C", i64, 4), ("Ftot", i64, 24),
                             ("Fw", i64, 16), ("HW", i64, 64), ("repeat", i32, 2)],
                            {"NULL latents": dict(latents=NULL), "NULL idx": dict(idx=NULL), "NULL out": dict(out=NULL), "repeat = 0": dict(repeat=0),
                             "Bl = 0": dict(Bl=0), "HW past int32": dict(HW=2 ** 31)}),
    "hv_op_cfg_ddim_step": ("hv_op_cfg_ddim_step",
                            [("uncond", None, lambda: ptrs(P(1), P(2))), ("cond", None, lambda: ptrs(P(3), P(4))), ("n", i32, 2), ("inv", ptr, P(5)),
                             ("K", i32, 2), ("coef", ptr, P(6)), ("step", ptr, P(7)), ("latents", ptr, P(8)), ("Bl", i64, 1), ("C", i64, 4),
                             ("Ftot", i64, 24), ("Fw", i64, 16), ("HW", i64, 64), ("guidance", f32, 3.5), ("ptype", i32, 0)],
                            {"NULL uncond": dict(uncond=lambda: None), "NULL window prediction": dict(cond=lambda: ptrs(P(3), None)),
                             "NULL inv": dict(inv=NULL), "NULL coef": dict(coef=NULL), "NULL latents": dict(latents=NULL), "0 windows": dict(n=0),
                             "33 windows": dict(n=33), "K = 0": dict(K=0), "prediction_type 2": dict(ptype=2), "misaligned coef": dict(coef=P(6, 4)),
                             "Bl = 0": dict(Bl=0)}),
    "hv_op_advance_index": ("hv_op_advance_index", [("index", ptr, P(1))], {"NULL index": dict(index=NULL)}),
}


def call(fn, spec, over):
    args = []
    for name, kind, value in spec:
        v = over.get(name, value)
        args.append(v() if kind is None else kind(v))
    return getattr(lib(), fn)(*args, C.c_void_p(0))


def test_every_entry_point_is_covered():
    src = open(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "include", "hv_b200_ops.h")).read()
    syms = set(re.findall(r"\b(hv_(?:op|pack)_[a-z0-9_]+)\s*\(", re.sub(r"/\*.*?\*/", "", src, flags=re.S)))
    assert syms == set(OPS), sorted(syms ^ set(OPS))


@pytest.mark.parametrize("fn", sorted(OPS))
def test_rejected_before_any_cuda_call(fn):
    name, spec, cases = OPS[fn]
    st = call(fn, spec, {})
    assert st in (-2, -3), f"{fn}: the accepted argument set returned {st} ({lib().hv_ops_last_error().decode()})"
    for label, over in cases.items():
        st = call(fn, spec, over)
        msg = lib().hv_ops_last_error().decode()
        assert st == HV_ERR_INVALID, f"{fn} {label}: status {st} ({msg}), expected HV_ERR_INVALID"
        assert msg.startswith(name + ":") or msg.startswith(name + " "), f"{fn} {label}: message {msg!r} does not name the operator"
