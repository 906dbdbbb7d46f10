"""Times the spatial attention operator (hv_op_attention) at the production shapes of bench configs 2, 3 and 5.

    python scripts/attn_bench.py [--lib PATH] [--iters N] [--warmup W] [--save DIR]
    python scripts/attn_bench.py --compare DIR_A DIR_B

Every shape runs on seeded inputs laid out as the model lays them out: Q and K interleaved per token with heads padded to
dpad, V^T[head * dv + channel][frame * Lp + token] with a row of ones at channel d (the softmax denominator).  `--lib` loads
any build of libhv_b200.so, so two builds can run the same script and `--save` / `--compare` checks that they compute the same.

Per shape it reports the median of `--iters` launches (CUDA events, after `--warmup`), algorithmic TFLOP/s (model.cu's
4 L C (NF L + (NF - nf_nobank) Lb)), exp2/s and the time over two floors computed from the tiles the kernel executes
(128 x 128 score tiles, padded key and query rows included) at the SM clock sampled during the run:
  MUFU floor    one ex2 per score at 16 per clock per SM
  tensor floor  S = QK^T (dpad) and O += PV (dv) at 4096 dense fp16 FLOP per clock per SM (989 TFLOP/s / 132 SMs / 1.83 GHz)
"""
from __future__ import annotations

import argparse
import ctypes as C
import json
import math
import os
import statistics
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

QT = KT = 128
MUFU_PER_CLK, TENSOR_FLOP_PER_CLK = 16, 4096

# name, NF, L, heads, d, Lb, F, nf_nobank (NF = 24 frames x CFG batch 2; the conditional half reads the bank)
SHAPES = [
    ("c2_l0", 48, 6912, 8, 40, 0, 24, 0),
    ("c2_l1", 48, 1728, 8, 80, 0, 24, 0),
    ("c2_l2", 48, 432, 8, 160, 0, 24, 0),
    ("c2_l3", 48, 108, 8, 160, 0, 24, 0),
    ("c3_l0", 48, 6912, 8, 40, 6912, 24, 24),
    ("c5_l0", 48, 9216, 8, 40, 9216, 24, 24),
    ("c5_l1", 48, 2304, 8, 80, 2304, 24, 24),
    ("c5_l2", 48, 576, 8, 160, 576, 24, 24),
    ("c5_l3", 48, 144, 8, 160, 144, 24, 24),
]


def load(path):
    lib = C.CDLL(path)
    lib.hv_ops_last_error.restype = C.c_char_p
    return lib


def make_inputs(NF, L, heads, d, Lb, F, seed):
    import torch

    g = torch.Generator(device="cuda").manual_seed(seed)
    dpad, dv = (d + 15) // 16 * 16, (d + 1 + 15) // 16 * 16
    qk = torch.zeros(NF * L, 2, heads, dpad, device="cuda", dtype=torch.half)
    qk[..., :d] = torch.randn(NF * L, 2, heads, d, generator=g, device="cuda").half()
    qk = qk.reshape(NF * L, 2 * heads * dpad)

    def vt_of(n, l):
        lp = (l + 7) // 8 * 8
        vt = torch.zeros(heads, dv, n, lp, device="cuda", dtype=torch.half)
        vt[:, :d, :, :l] = torch.randn(heads, d, n, l, generator=g, device="cuda").half()
        vt[:, d, :, :l] = 1
        return vt.reshape(heads * dv, n * lp), lp

    vt, Lp = vt_of(NF, L)
    kb = vbt = None
    Lbp = 0
    if Lb:
        B = NF // F
        kb = torch.zeros(B * Lb, heads, dpad, device="cuda", dtype=torch.half)
        kb[..., :d] = torch.randn(B * Lb, heads, d, generator=g, device="cuda").half()
        kb = kb.reshape(B * Lb, heads * dpad)
        vbt, Lbp = vt_of(B, Lb)
    out = torch.zeros(NF * L, heads * d, device="cuda", dtype=torch.half)
    return dict(qk=qk, vt=vt, Lp=Lp, kb=kb, vbt=vbt, Lbp=Lbp, out=out, dpad=dpad, dv=dv)


def launch(lib, x, NF, L, heads, d, Lb, F, nf_nobank, stream):
    i64, i32 = C.c_int64, C.c_int32
    p = lambda t: C.c_void_p(0 if t is None else t.data_ptr())  # noqa: E731
    ld = 2 * heads * x["dpad"]
    rc = lib.hv_op_attention(p(x["qk"]), C.c_void_p(x["qk"].data_ptr() + heads * x["dpad"] * 2), p(x["vt"]), p(x["out"]), i64(NF), i64(L),
                             i32(heads), i32(d), i64(ld), i64(ld), i64(x["vt"].stride(0)), i64(heads * d), p(x["kb"]), p(x["vbt"]), i64(Lb),
                             i64(heads * x["dpad"]), i64(x["vbt"].stride(0) if x["vbt"] is not None else 0), i64(F), i64(nf_nobank),
                             i64(x["Lp"]), i64(x["Lbp"]), C.c_void_p(stream))
    if rc != 0:
        raise RuntimeError(f"hv_op_attention failed ({rc}): {lib.hv_ops_last_error().decode()}")


def counts(NF, L, heads, d, Lb, nf_nobank):
    dpad, dv = (d + 15) // 16 * 16, (d + 1 + 15) // 16 * 16
    flops = 4.0 * L * heads * d * (NF * L + (NF - nf_nobank) * Lb)
    ex2 = float(heads) * L * (NF * L + (NF - nf_nobank) * Lb)
    qt, kt, kbt = math.ceil(L / QT), math.ceil(L / KT), math.ceil(Lb / KT) if Lb else 0
    tiles = heads * qt * (NF * kt + (NF - nf_nobank) * kbt)   # executed 128 x 128 score tiles
    mufu_cyc = tiles * QT * KT / MUFU_PER_CLK
    tensor_cyc = tiles * 2.0 * QT * KT * (dpad + dv) / TENSOR_FLOP_PER_CLK
    return flops, ex2, mufu_cyc, tensor_cyc


def run(args):
    import torch

    if not torch.cuda.is_available():
        raise SystemExit("attn_bench.py: no CUDA device (this script only measures on the GPU)")
    from bench import ClockSampler

    lib = load(args.lib)
    props = torch.cuda.get_device_properties(0)
    sms = props.multi_processor_count
    stream = torch.cuda.current_stream().cuda_stream
    if args.save:
        os.makedirs(args.save, exist_ok=True)
    rows = []
    for si, (name, NF, L, heads, d, Lb, F, nf_nobank) in enumerate(SHAPES):
        if args.only and name not in args.only.split(","):
            continue
        x = make_inputs(NF, L, heads, d, Lb, F, seed=1000 + si)
        for _ in range(args.warmup):
            launch(lib, x, NF, L, heads, d, Lb, F, nf_nobank, stream)
        ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(args.iters)]
        with ClockSampler(0) as cs:
            for a, b in ev:
                a.record()
                launch(lib, x, NF, L, heads, d, Lb, F, nf_nobank, stream)
                b.record()
            torch.cuda.synchronize()
        clk = cs.summary()
        ms = statistics.median(a.elapsed_time(b) for a, b in ev)
        flops, ex2, mufu_cyc, tensor_cyc = counts(NF, L, heads, d, Lb, nf_nobank)
        mhz = clk.get("sm_mhz")
        row = {"shape": name, "NF": NF, "L": L, "heads": heads, "d": d, "Lb": Lb, "nf_nobank": nf_nobank, "ms": round(ms, 4),
               "tflops": round(flops / ms / 1e9, 1), "ex2_per_s": f"{ex2 / ms * 1e3:.3e}", "sm_mhz": mhz}
        if mhz:
            row["x_mufu_floor"] = round(ms / (mufu_cyc / sms / (mhz * 1e3)), 3)
            row["x_tensor_floor"] = round(ms / (tensor_cyc / sms / (mhz * 1e3)), 3)
            row["cycles_per_sm"] = round(ms * mhz * 1e3)
        rows.append(row)
        print(json.dumps(row), flush=True)
        if args.save:
            import numpy as np

            np.save(os.path.join(args.save, f"{name}.npy"), x["out"].cpu().numpy())
        del x
        torch.cuda.empty_cache()
    print(json.dumps({"gpu": props.name, "power_limit_w": clk.get("power_limit_w"), "sm_max_mhz": clk.get("sm_max_mhz"),
                      "lib": os.path.abspath(args.lib), "iters": args.iters, "warmup": args.warmup}), flush=True)
    return rows


def compare(a_dir, b_dir):
    import numpy as np

    names = sorted(f for f in os.listdir(a_dir) if f.endswith(".npy"))
    if not names:
        raise SystemExit(f"no .npy files in {a_dir}")
    for f in names:
        a = np.load(os.path.join(a_dir, f)).astype(np.float64)
        b = np.load(os.path.join(b_dir, f)).astype(np.float64)
        diff = a != b
        rel = float(np.linalg.norm(a - b) / (np.linalg.norm(a) + 1e-30))
        print(json.dumps({"shape": f[:-4], "bitwise_equal": not bool(diff.any()), "n_diff": int(diff.sum()), "n": int(a.size),
                          "max_abs": float(np.abs(a - b).max()), "rel_l2": rel}), flush=True)


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--lib", default=os.path.join(ROOT, "humanvid_b200", "lib", "libhv_b200.so"))
    ap.add_argument("--iters", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--only", default="", help="comma-separated shape names (default: all)")
    ap.add_argument("--save", default="", help="write each shape's output as DIR/<shape>.npy")
    ap.add_argument("--compare", nargs=2, metavar=("A", "B"), help="compare the outputs saved in two directories")
    args = ap.parse_args()
    if args.compare:
        compare(*args.compare)
    else:
        if args.iters < 20:
            ap.error("--iters must be at least 20")
        run(args)


if __name__ == "__main__":
    main()
