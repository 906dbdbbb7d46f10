"""fp16 against FP8 (e4m3) per covered linear of the denoising UNet, on one H100.

    python scripts/fp8_bench.py [--rounds R] [--out FILE]

For each layer shape the FP8 linears cover (spatial FF1 / FF2 and motion-module Q/K/V, FF1 / FF2; DESIGN.md §9) at config 2 levels
0-3 (latent 96 x 72, 48 frames = 2 CFG halves x 24) and config 5 level 0 (72 x 128, 48 frames), it times the fp16 GEMM (hv_op_gemm)
and the FP8 GEMM (hv_op_gemm_fp8) with their real epilogues (FF1: GEGLU, fp16 output against e4m3 output with per-128 scales; FF2:
bias + residual, per-128 A scales in FP8; Q/K/V: per-row A scales), and the fp16 LayerNorm against the e4m3 LayerNorm that feeds FF1
and Q/K/V.  The two arms alternate round by round; each round times `reps` launches between CUDA events; the medians and the spread
(min, max) over the rounds are reported with algorithmic TFLOP/s (2 M N K).  The relative L2 of each arm's output against fp32 (torch
matmul of the fp16 operands, first 8192 rows) is reported too.  Prints the card name, power limit and SM clock, then one JSON line.
Then the whole UNet3DConditionModel forward at config 2 (bench.py's model and seeded synthetic weights, CFG batch 2, 24 frames of latent
96 x 72): one model in fp16 and one with enable_fp8_linears(), alternating round by round, with the relative L2 of the FP8 output
against the fp16 one.
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

from fp8_emulation import quantize  # noqa: E402
from humanvid_b200._native import Epilogue, check, i64, lib, ptr, stream  # noqa: E402

LEVELS = [("config2-L0", 6912 * 48, 320), ("config2-L1", 1728 * 48, 640), ("config2-L2", 432 * 48, 1280), ("config2-L3", 108 * 48, 1280),
          ("config5-L0", 9216 * 48, 320)]


def f32p(t):
    return C.cast(C.c_void_p(t.data_ptr()), C.POINTER(C.c_float))


def gpu_info():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True, timeout=10).stdout
        name, plim, sm, smmax = [c.strip() for c in out.strip().split(",")]
        return dict(card=name, power_limit=plim, sm_clock=sm, sm_clock_max=smmax)
    except Exception as e:   # the card name from torch at least
        return dict(card=torch.cuda.get_device_name(0), power_limit=f"unavailable ({e})", sm_clock="unavailable", sm_clock_max="unavailable")


def time_arms(arms, rounds, target_ms=40.0):
    """arms: {name: fn}.  Alternating rounds; returns {name: (median_ms, min_ms, max_ms)} per launch."""
    for fn in arms.values():
        fn()
    torch.cuda.synchronize()
    reps = {}
    for k, fn in arms.items():   # launches per round so that a round lasts about target_ms
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        for _ in range(3):
            fn()
        b.record()
        torch.cuda.synchronize()
        reps[k] = max(3, int(target_ms / max(a.elapsed_time(b) / 3, 1e-3)))
    res = {k: [] for k in arms}
    for _ in range(rounds):
        for k, fn in arms.items():
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            for _ in range(reps[k]):
                fn()
            b.record()
            torch.cuda.synchronize()
            res[k].append(a.elapsed_time(b) / reps[k])
    return {k: (sorted(v)[len(v) // 2], min(v), max(v)) for k, v in res.items()}


def rel(a, b):
    return float((a.float() - b.float()).norm() / b.float().norm())


def layer(kind, M, Cc, rounds):
    g = torch.Generator(device="cuda").manual_seed(1)
    dev = "cuda"
    if kind == "qkv":
        N, K, geglu, blocks, res = 3 * Cc, Cc, False, False, False
    elif kind == "ff1":
        N, K, geglu, blocks, res = 8 * Cc, Cc, True, False, False
    else:
        N, K, geglu, blocks, res = Cc, 4 * Cc, False, True, True
    nout = N // 2 if geglu else N
    x = torch.randn(M, K, generator=g, device=dev).half()
    if blocks:
        x = (x.float() * (1 + 8 * (torch.randn(M, K, generator=g, device=dev).abs() > 2.5))).half()
    w = (torch.randn(N, K, generator=g, device=dev) * K ** -0.5).half()
    bias = (torch.randn(N, generator=g, device=dev) * 0.1).half()
    resid = torch.randn(M, nout, generator=g, device=dev).half() if res else None
    qa, sa = quantize(x.float(), 128 if blocks else None)
    qa, sa = qa.view(torch.uint8).contiguous(), sa.contiguous()
    qw = torch.empty(N, K, dtype=torch.uint8, device=dev)
    sw = torch.empty(N, dtype=torch.float32, device=dev)
    check(lib().hv_pack_fp8_rows(ptr(w), ptr(qw), f32p(sw), i64(N), i64(K), stream()))
    ep = Epilogue()
    ep.bias = bias.data_ptr()
    ep.geglu = int(geglu)
    if res:
        ep.residual, ep.ldr = resid.data_ptr(), nout
    out16 = torch.empty(M, nout, dtype=torch.half, device=dev)
    out8 = torch.empty(M, nout, dtype=torch.uint8, device=dev) if geglu else torch.empty(M, nout, dtype=torch.half, device=dev)
    osc = torch.empty(M, max(1, N // 256), dtype=torch.float32, device=dev)

    def f16():
        check(lib().hv_op_gemm(ptr(x), i64(K), None, i64(0), i64(0), ptr(w), ptr(out16), i64(nout), i64(M), i64(N), i64(K), C.byref(ep), stream()))

    def f8():
        check(lib().hv_op_gemm_fp8(ptr(qa), i64(K), f32p(sa), i64(sa.shape[1] if blocks else 0), ptr(qw), f32p(sw), ptr(out8), i64(nout),
                                   f32p(osc) if geglu else None, i64(osc.shape[1] if geglu else 0), i64(M), i64(N), i64(K), C.byref(ep), stream()))

    t = time_arms({"fp16": f16, "fp8": f8}, rounds)
    # fp32 reference on the first rows
    r = min(M, 8192)
    ref = x[:r].float() @ w.float().T + bias.float()
    if geglu:
        ref = ref.view(r, -1, 2, 128)
        ref = (ref[:, :, 0] * torch.nn.functional.gelu(ref[:, :, 1])).reshape(r, -1)
    if res:
        ref = ref + resid[:r].float()
    if geglu:
        v8 = (out8[:r].view(torch.float8_e4m3fn).float().view(r, -1, 128) * osc[:r].unsqueeze(-1)).reshape(r, -1)
    else:
        v8 = out8[:r].float()
    flop = 2.0 * M * N * K
    o16 = out16[:r].float()
    return dict(layer=kind, M=M, N=N, K=K, tflop=flop / 1e12,
                fp16_ms=t["fp16"][0], fp16_ms_spread=t["fp16"][1:], fp8_ms=t["fp8"][0], fp8_ms_spread=t["fp8"][1:],
                fp16_tflops=flop / t["fp16"][0] / 1e9, fp8_tflops=flop / t["fp8"][0] / 1e9, speedup=t["fp16"][0] / t["fp8"][0],
                rel_fp8_vs_fp16=rel(v8, o16), rel_fp8_vs_fp32=rel(v8, ref), rel_fp16_vs_fp32=rel(o16, ref))


def layernorm(name, M, Cc, rounds):
    g = torch.Generator(device="cuda").manual_seed(2)
    x = torch.randn(M, Cc, generator=g, device="cuda").half()
    gamma, beta = torch.ones(Cc, device="cuda").half(), torch.zeros(Cc, device="cuda").half()
    y16 = torch.empty_like(x)
    y8 = torch.empty(M, Cc, dtype=torch.uint8, device="cuda")
    s8 = torch.empty(M, dtype=torch.float32, device="cuda")

    def f16():
        check(lib().hv_op_layernorm(ptr(x), ptr(gamma), ptr(beta), ptr(y16), i64(M), i64(Cc), C.c_float(1e-5), None, i64(1), None, None, i64(0),
                                    i64(0), stream()))

    def f8():
        check(lib().hv_op_layernorm_fp8(ptr(x), ptr(gamma), ptr(beta), ptr(y8), f32p(s8), i64(M), i64(Cc), C.c_float(1e-5), None, i64(1), None,
                                        None, i64(0), i64(0), stream()))

    t = time_arms({"fp16": f16, "fp8": f8}, rounds)
    return dict(layer="layernorm", level=name, M=M, C=Cc, fp16_ms=t["fp16"][0], fp16_ms_spread=t["fp16"][1:], fp8_ms=t["fp8"][0],
                fp8_ms_spread=t["fp8"][1:], speedup=t["fp16"][0] / t["fp8"][0])


def whole_forward(rounds):
    import bench

    dev = "cuda"
    n16 = bench.build_native(dev)
    n8 = bench.build_native(dev)
    n8.enable_fp8_linears()
    g = torch.Generator(device=dev).manual_seed(3)
    B, F, h, w = 2, 24, 96, 72
    x = torch.randn(B, 4, F, h, w, generator=g, device=dev).half()
    ehs = torch.randn(B, 1, bench.XDIM, generator=g, device=dev).half()
    ehs[:1] = 0
    pose = (torch.randn(B, bench.CH[0], F, h, w, generator=g, device=dev) * 0.5).half()
    outs = {}

    def arm(net, key):
        def f():
            outs[key] = net(x, 500, ehs, pose_cond_fea=pose, return_dict=False)[0]
        return f

    t = time_arms({"fp16": arm(n16, "fp16"), "fp8": arm(n8, "fp8")}, rounds, target_ms=1000.0)
    r = dict(layer="unet3d_forward", config="config2", fp16_ms=t["fp16"][0], fp16_ms_spread=t["fp16"][1:], fp8_ms=t["fp8"][0],
             fp8_ms_spread=t["fp8"][1:], speedup=t["fp16"][0] / t["fp8"][0], rel_fp8_vs_fp16=rel(outs["fp8"], outs["fp16"]),
             fp8_finite=bool(torch.isfinite(outs["fp8"]).all()))
    del n16, n8
    torch.cuda.empty_cache()
    return r


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=7)
    ap.add_argument("--out", default=None, help="also write the JSON line to this file")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("fp8_bench.py needs a CUDA device")
    torch.cuda.set_device(0)
    info = gpu_info()
    print(f"card {info['card']}, power limit {info['power_limit']}, SM clock {info['sm_clock']} (max {info['sm_clock_max']})")
    rows = []
    with torch.no_grad():
        for name, M, Cc in LEVELS:
            for kind in ("qkv", "ff1", "ff2"):
                r = layer(kind, M, Cc, args.rounds)
                r["level"] = name
                rows.append(r)
                print(f"{name:11s} {kind:4s} M={M:6d} N={r['N']:5d} K={r['K']:5d}  fp16 {r['fp16_ms']:.3f} ms ({r['fp16_tflops']:.0f} TF/s)  "
                      f"fp8 {r['fp8_ms']:.3f} ms ({r['fp8_tflops']:.0f} TF/s)  x{r['speedup']:.2f}  rel L2 fp8/fp32 {r['rel_fp8_vs_fp32']:.2e} "
                      f"fp16/fp32 {r['rel_fp16_vs_fp32']:.2e}", flush=True)
                torch.cuda.empty_cache()
            r = layernorm(name, M, Cc, args.rounds)
            rows.append(r)
            print(f"{name:11s} LN   M={M:6d} C={Cc:5d}  fp16 {r['fp16_ms']:.3f} ms  fp8 {r['fp8_ms']:.3f} ms  x{r['speedup']:.2f}", flush=True)
        r = whole_forward(args.rounds)
        rows.append(r)
        print(f"config2 UNet forward  fp16 {r['fp16_ms']:.1f} ms  fp8 {r['fp8_ms']:.1f} ms  x{r['speedup']:.3f}  rel L2 fp8 vs fp16 "
              f"{r['rel_fp8_vs_fp16']:.2e}", flush=True)
    info2 = gpu_info()
    res = dict(metric="fp8_linears_per_layer", **info, sm_clock_after=info2["sm_clock"], rounds=args.rounds, layers=rows)
    line = json.dumps(res)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
