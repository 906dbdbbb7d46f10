"""Cost of the inference_v1 UNet layout on the GPU: frame-pooled against per-frame GroupNorm, and the v1 against the v2 UNet forward.

1. hv_op_groupnorm_pooled (statistics over the 24 frames of each batch item: statistics, finalize and apply launches) against
   hv_op_groupnorm (per frame: statistics and apply) at the resnet GroupNorm shapes of bench config 2, (2 x 24) frames of 96 x 72 at
   levels 0-3, SiLU on.  Both arms move the same HBM bytes (one read for the statistics, one read and one write for the apply).
2. The full-width UNet3DConditionModel forward at (2, 4, 24, 96, 72), inference_v1 layout (pooled GroupNorm, no mid-block motion module)
   against inference_v2, on the same random weights.
Both parts alternate the two arms round by round and take medians of CUDA-event times.  The card name, power limit and SM clock are
read in the same run.  Prints one JSON line.

    python scripts/gn_pooled_bench.py [--rounds 7] [--iters 50] [--no-unet]
"""
from __future__ import annotations

import argparse
import ctypes as C
import json
import os
import statistics
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

G, EPS = 32, 1e-5
B, F, H, W = 2, 24, 96, 72
# (level, C1, C2): down resnet norm1 / norm2 and the widest up-block concat of each level
SHAPES = [(0, 320, 0), (0, 640, 320), (1, 640, 0), (1, 1280, 640), (2, 1280, 0), (2, 1280, 1280), (3, 1280, 0), (3, 1280, 1280)]


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                       text=True).stdout.strip().splitlines()
    return q[torch.cuda.current_device()] if q else torch.cuda.get_device_name()


def time_ms(fn, iters):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b) / iters


def groupnorm_part(rounds, iters):
    from humanvid_b200._native import check, i32, i64, lib, ptr, stream

    L = lib()
    L.hv_groupnorm_scratch_floats.restype = C.c_size_t
    rows = []
    for lvl, C1, C2 in SHAPES:
        HW, NF, Ct = (H >> lvl) * (W >> lvl), B * F, C1 + C2
        g = torch.Generator(device="cuda").manual_seed(lvl)
        x1 = torch.randn(NF, HW, C1, generator=g, device="cuda").half()
        x2 = torch.randn(NF, HW, C2, generator=g, device="cuda").half() if C2 else None
        gamma, beta = torch.ones(Ct, device="cuda").half(), torch.zeros(Ct, device="cuda").half()
        out = torch.empty(NF, HW, Ct, device="cuda", dtype=torch.half)
        stats = torch.empty(int(L.hv_groupnorm_scratch_floats(i64(Ct), i64(NF), i64(HW), i32(G))), device="cuda", dtype=torch.float32)
        args = (ptr(x1), i64(C1), ptr(x2), i64(C2), ptr(gamma), ptr(beta), ptr(out), i64(NF), i64(HW), i32(G), C.c_float(EPS), i32(1))
        arms = {"per_frame": lambda: check(L.hv_op_groupnorm(*args, ptr(stats), stream())),
                "pooled": lambda: check(L.hv_op_groupnorm_pooled(*args, i64(F), ptr(stats), stream()))}
        for fn in arms.values():
            time_ms(fn, 5)
        t = {k: [] for k in arms}
        for _ in range(rounds):
            for k, fn in arms.items():
                t[k].append(time_ms(fn, iters))
        med = {k: statistics.median(v) for k, v in t.items()}
        gb = 3.0 * NF * HW * Ct * 2 / 1e9   # statistics read + apply read + apply write
        rows.append(dict(level=lvl, HW=HW, C1=C1, C2=C2, per_frame_us=round(1e3 * med["per_frame"], 2), pooled_us=round(1e3 * med["pooled"], 2),
                         ratio=round(med["pooled"] / med["per_frame"], 3), pooled_TBps=round(gb / med["pooled"], 2),
                         spread_per_frame=round((max(t["per_frame"]) - min(t["per_frame"])) / med["per_frame"], 3),
                         spread_pooled=round((max(t["pooled"]) - min(t["pooled"])) / med["pooled"], 3)))
        print(f"level {lvl} HW {HW:5d} C {C1}+{C2}: per-frame {rows[-1]['per_frame_us']:8.2f} us, pooled {rows[-1]['pooled_us']:8.2f} us, "
              f"ratio {rows[-1]['ratio']:.3f} ({rows[-1]['pooled_TBps']} TB/s)", file=sys.stderr)
    return rows


def unet_part(rounds):
    import humanvid_b200 as hv
    from oracle import hv_oracle as O
    from unet_v1_oracle import V1_MM_KWARGS, V1_UNET_KWARGS, unet3d_v1

    CH, XD = (320, 640, 1280, 1280), 768
    v2_mm = dict(V1_MM_KWARGS, temporal_position_encoding_max_len=32)
    v2_kw = dict(V1_UNET_KWARGS, use_inflated_groupnorm=True, motion_module_mid_block=True, motion_module_kwargs=v2_mm)
    nets = {}
    for name, ora, kw in (("v1", unet3d_v1(CH, XD), V1_UNET_KWARGS), ("v2", O.UNet3DConditionModel(block_out_channels=CH, cross_attention_dim=XD), v2_kw)):
        O.synthetic_init(ora, seed=7)
        nat = hv.UNet3DConditionModel(block_out_channels=CH, cross_attention_dim=XD, attention_head_dim=8, **kw)
        nat.load_state_dict(ora.state_dict())
        nets[name] = nat.to("cuda", torch.float16)
        del ora
    g = torch.Generator(device="cuda").manual_seed(0)
    x = torch.randn(B, 4, F, H, W, generator=g, device="cuda").half()
    ehs = torch.randn(B, 1, XD, generator=g, device="cuda").half()
    pose = (torch.randn(B, CH[0], F, H, W, generator=g, device="cuda") * 0.5).half()

    def fwd(n):
        with torch.no_grad():
            n(x, 500, ehs, pose_cond_fea=pose, return_dict=False)

    for n in nets.values():
        for _ in range(2):
            fwd(n)
    t = {k: [] for k in nets}
    for _ in range(rounds):
        for k, n in nets.items():
            t[k].append(time_ms(lambda: fwd(n), 3))
    med = {k: statistics.median(v) for k, v in t.items()}
    launches = {k: int(n.last_launch_count) for k, n in nets.items()}
    res = dict(v1_ms=round(med["v1"], 2), v2_ms=round(med["v2"], 2), ratio=round(med["v1"] / med["v2"], 4), launches=launches,
               spread_v1=round((max(t["v1"]) - min(t["v1"])) / med["v1"], 4), spread_v2=round((max(t["v2"]) - min(t["v2"])) / med["v2"], 4))
    print(f"UNet forward (2,4,24,96,72): v1 {res['v1_ms']} ms, v2 {res['v2_ms']} ms, ratio {res['ratio']}, launches {launches}", file=sys.stderr)
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=7)
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--no-unet", action="store_true")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("gn_pooled_bench.py needs a CUDA device")
    before = card()
    res = dict(card_before=before, groupnorm=groupnorm_part(args.rounds, args.iters))
    if not args.no_unet:
        res["unet"] = unet_part(args.rounds)
    res["card_after"] = card()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
