"""Times humanvid_b200.AutoencoderKL (the native VAE) against the PyTorch restatement run in fp16 eager on the same GPU, and prints one JSON line.

    python scripts/vae_bench.py [--iters N] [--warmup W] [--no-eager]

Workloads (random weights, seeded inputs; the SD VAE layout):
  decode  24 frames at 768x576 (latent 96x72) and 48 frames at 576x1024 (latent 72x128), each in calls of 8 frames (the pipeline's
          vae_decode_batch) and of 24 frames
  encode  one 768x576 reference image
Each workload is timed with CUDA events around the whole clip (all its calls), median of --iters after --warmup.  The fp16-eager bar runs
the same inputs through tests/vae_oracle.py in calls of 8 frames.  FLOPs are algorithmic (2 x multiply-adds of the convolutions, linears
and attention, computed from the shapes; vae_oracle.decode_flops / encode_flops), so TFLOP/s compares directly across the two arms.
The profile split is hv_get_profile's per-category device time of one 8-frame 768x576 decode.  The card's name, power limit and clocks
are read with nvidia-smi queries (bench.ClockSampler) during the timed runs.
"""
from __future__ import annotations

import argparse
import ctypes as C
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

CATEGORIES = ["gemm", "conv", "attention", "temporal_attention", "norm", "small_linear"]


def time_ms(fn, iters, warmup):
    import torch

    for _ in range(warmup):
        fn()
    times = []
    for _ in range(iters):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        times.append(a.elapsed_time(b))
    return statistics.median(times)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--no-eager", action="store_true", help="skip the fp16-eager oracle arm")
    args = ap.parse_args()

    import torch

    if not torch.cuda.is_available():
        raise SystemExit("vae_bench.py needs a CUDA device")
    import bench
    import humanvid_b200 as hv
    import vae_oracle as V
    from humanvid_b200 import _native as N
    from oracle import hv_oracle as O

    dev = "cuda"
    name = subprocess.run(["nvidia-smi", "--query-gpu=name", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True).stdout.strip()
    ora = O.synthetic_init(V.AutoencoderKL().eval(), seed=21).half()
    nat = hv.AutoencoderKL()
    nat.load_state_dict(ora.state_dict())
    nat = nat.to(dev, torch.float16)
    g = torch.Generator(device=dev).manual_seed(0)
    clips = {"768x576x24": (24, 96, 72), "576x1024x48": (48, 72, 128)}
    lat = {k: torch.randn(f, 4, h, w, generator=g, device=dev).half() for k, (f, h, w) in clips.items()}
    img = (torch.rand(1, 3, 768, 576, generator=g, device=dev) * 2 - 1).half()

    def decode_clip(model, z, n):
        with torch.no_grad():
            for i in range(0, z.shape[0], n):
                model.decode(z[i : i + n])

    res = {"gpu": name, "iters": args.iters, "warmup": args.warmup, "native": {}, "fp16_eager": {}}
    with bench.ClockSampler(0) as clk:
        for key, (f, h, w) in clips.items():
            flops = V.decode_flops(f, h, w)
            for n in (8, 24):
                ms = time_ms(lambda: decode_clip(nat, lat[key], n), args.iters, args.warmup)
                res["native"][f"decode_{key}_calls_of_{n}"] = {"ms": round(ms, 2), "tflops": round(flops / ms / 1e9, 1), "gflop": round(flops / 1e9, 1)}
        torch.cuda.empty_cache()
        eflops = V.encode_flops(1, 768, 576)
        ms = time_ms(lambda: nat.encode(img), args.iters, args.warmup)
        res["native"]["encode_768x576x1"] = {"ms": round(ms, 2), "tflops": round(eflops / ms / 1e9, 1), "gflop": round(eflops / 1e9, 1)}
        # per-category split of one 8-frame 768x576 decode
        h = nat._sync_native()
        N.check(N.lib().hv_set_profiling(h, N.i32(1)), h)
        with torch.no_grad():
            nat.decode(lat["768x576x24"][:8])
        ms6, fl6, cnt6 = (C.c_double * 6)(), (C.c_double * 6)(), (C.c_int64 * 6)()
        N.check(N.lib().hv_get_profile(h, ms6, fl6, cnt6, N.i32(6)), h)
        N.check(N.lib().hv_set_profiling(h, N.i32(0)), h)
        res["native"]["profile_decode_768x576x8"] = {
            c: {"ms": round(ms6[i], 2), "tflops": round(fl6[i] / ms6[i] / 1e9, 1) if ms6[i] > 0 else 0.0, "launches": cnt6[i]}
            for i, c in enumerate(CATEGORIES) if cnt6[i]}
        res["native"]["launches_decode_768x576x8"] = nat.last_launch_count
        # the native workspace is no longer needed: leave the memory to the eager arm
        nat._destroy()
        torch.cuda.empty_cache()
        if not args.no_eager:
            o16 = ora.to(dev)
            for key, (f, h, w) in clips.items():
                flops = V.decode_flops(f, h, w)
                ms = time_ms(lambda: decode_clip(o16, lat[key], 8), args.iters, args.warmup)
                res["fp16_eager"][f"decode_{key}_calls_of_8"] = {"ms": round(ms, 2), "tflops": round(flops / ms / 1e9, 1)}
            with torch.no_grad():
                ms = time_ms(lambda: o16.encode(img), args.iters, args.warmup)
            res["fp16_eager"]["encode_768x576x1"] = {"ms": round(ms, 2), "tflops": round(eflops / ms / 1e9, 1)}
            for key in clips:
                res[f"speedup_decode_{key}_calls_of_8"] = round(res["fp16_eager"][f"decode_{key}_calls_of_8"]["ms"] / res["native"][f"decode_{key}_calls_of_8"]["ms"], 2)
            res["speedup_encode_768x576x1"] = round(res["fp16_eager"]["encode_768x576x1"]["ms"] / res["native"]["encode_768x576x1"]["ms"], 2)
    res["clocks"] = clk.summary()
    peak_tflops, _, _, peak_src = bench.peaks()
    res["tensor_peak_tflops"], res["tensor_peak_source"] = peak_tflops, peak_src
    print(json.dumps(res))


if __name__ == "__main__":
    main()
