"""Per-shape A/B of the GEMM / conv kernel between two builds of the library.

Each build is a source tree whose humanvid_b200/lib holds a built libhv_b200.so (for example this repository and a checkout of
another commit).  For each round, and alternating A, B, A, B, ..., a separate process runs `bench.py --config 2` in that tree
with the per-launch profile written out (HV_TRACE: one profiled UNet forward, CUDA events around every launch).  The
gemm_kernel launches (categories gemm_linear and implicit_gemm_conv3x3) are grouped by label and shape (M, N, K); per group and
build the script prints the median over rounds of the per-forward ms, the TFLOP/s, the bound (tensor or HBM, scored by
bench.gemm_classes) and the B / A time ratio, with the spread of each arm.  The card name, power limit and median SM clock
of every run are recorded.

  python scripts/gemm_bench.py --a /path/to/tree_a --b /path/to/tree_b [--rounds 3] [--json OUT]
"""
from __future__ import annotations

import argparse
import csv
import json
import os
import statistics
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def run_tree(tree, tmp, tag):
    trace = os.path.join(tmp, f"trace_{tag}.csv")
    env = dict(os.environ, HV_TRACE=trace)
    cmd = [sys.executable, "bench.py", "--config", "2", "--steps", "3", "--warmup", "3", "--no-extras", "--no-cpu-baseline", "--no-eager"]
    out = subprocess.run(cmd, cwd=tree, env=env, capture_output=True, text=True, check=True).stdout
    line = json.loads(out.strip().splitlines()[-1])
    rows = [r for r in csv.DictReader(open(trace)) if int(r["cat"]) in (0, 1) and r["label"]]
    return line, rows


def groups(rows):
    g = {}
    for r in rows:
        key = (r["label"], int(r["M"]), int(r["N"]), int(r["K"]))
        e = g.setdefault(key, {"ms": 0.0, "n": 0, "rows": []})
        e["ms"] += float(r["ms"])
        e["n"] += 1
        e["rows"].append(r)
    return g


def bound_of(rows, tmp):
    """'tensor' or 'hbm', as bench.gemm_classes scores these launches."""
    import bench

    p = os.path.join(tmp, "group.csv")
    with open(p, "w", newline="") as f:
        w = csv.DictWriter(f, fieldnames=list(rows[0].keys()))
        w.writeheader()
        w.writerows(rows)
    pk = bench.peaks()
    c = bench.gemm_classes(p, pk[0], pk[2])
    return "tensor" if c["tensor_bound"]["launches"] else "hbm"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--a", required=True, help="tree of build A (the baseline)")
    ap.add_argument("--b", required=True, help="tree of build B")
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--json", default=None, help="also write the table as JSON here")
    args = ap.parse_args()
    with tempfile.TemporaryDirectory() as tmp:
        runs = {"a": [], "b": []}
        for i in range(args.rounds):
            for arm in ("a", "b"):
                line, rows = run_tree(getattr(args, arm), tmp, f"{arm}{i}")
                runs[arm].append({"fps": line["value"], "gpu": line["gpu"], "clocks": line["clocks"], "groups": groups(rows)})
        keys = list(runs["a"][0]["groups"])
        table = []
        for k in keys:
            lab, M, N, K = k
            ms = {arm: [r["groups"][k]["ms"] for r in runs[arm] if k in r["groups"]] for arm in ("a", "b")}
            if not ms["a"] or not ms["b"]:
                continue
            med = {arm: statistics.median(v) for arm, v in ms.items()}
            n = runs["a"][0]["groups"][k]["n"]
            fl = 2.0 * M * N * K * n
            table.append({"label": lab, "M": M, "N": N, "K": K, "launches": n, "bound": bound_of(runs["a"][0]["groups"][k]["rows"], tmp),
                          "ms_a": med["a"], "ms_b": med["b"], "spread_a": max(ms["a"]) - min(ms["a"]), "spread_b": max(ms["b"]) - min(ms["b"]),
                          "tflops_a": fl / 1e9 / med["a"], "tflops_b": fl / 1e9 / med["b"], "ratio_b_over_a": med["b"] / med["a"]})
    r0 = runs["a"][0]
    head = {"gpu": r0["gpu"], "power_limit_w": r0["clocks"].get("power_limit_w"),
            "sm_mhz": {arm: [r["clocks"].get("sm_mhz") for r in runs[arm]] for arm in ("a", "b")},
            "frames_per_s": {arm: [r["fps"] for r in runs[arm]] for arm in ("a", "b")}}
    print(json.dumps(head))
    print(f"{'label':<22}{'M':>9}{'N':>6}{'K':>7}{'n':>4} {'bound':<7}{'ms A':>9}{'ms B':>9}{'±A':>7}{'±B':>7}{'TF/s A':>8}{'TF/s B':>8}{'B/A':>7}")
    for t in sorted(table, key=lambda t: -t["ms_a"]):
        print(f"{t['label']:<22}{t['M']:>9}{t['N']:>6}{t['K']:>7}{t['launches']:>4} {t['bound']:<7}{t['ms_a']:>9.3f}{t['ms_b']:>9.3f}"
              f"{t['spread_a']:>7.3f}{t['spread_b']:>7.3f}{t['tflops_a']:>8.0f}{t['tflops_b']:>8.0f}{t['ratio_b_over_a']:>7.3f}")
    tot_a, tot_b = sum(t["ms_a"] for t in table), sum(t["ms_b"] for t in table)
    print(f"{'total':<22}{'':>26} {'':<7}{tot_a:>9.3f}{tot_b:>9.3f}{'':>30}{tot_b / tot_a:>7.3f}")
    if args.json:
        json.dump({"head": head, "table": table}, open(args.json, "w"), indent=1)


if __name__ == "__main__":
    main()
