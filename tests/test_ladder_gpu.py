"""Accumulated drift through the network (scripts/error_ladder.py on the narrow UNet): at every block, native stays no further from the fp32
oracle than the reference's own fp16 path.  The isolated per-block error -- every block on its own input -- is asserted per frame, row and
element against fp64 by tests/test_block_parity_gpu.py, at this shape among others; here it is only reported."""
import os
import re
import subprocess
import sys

import pytest

from conftest import report

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_native_drift_never_exceeds_fp16_eager(tmp_path):
    out = str(tmp_path / "ladder.txt")
    p = subprocess.run([sys.executable, os.path.join(ROOT, "scripts", "error_ladder.py"), "--narrow", "--hw", "32", "32", "--frames", "6", "--out", out],
                       capture_output=True, text=True, timeout=900, cwd=ROOT)
    assert p.returncode == 0, p.stdout[-2000:] + p.stderr[-2000:]
    txt = open(out).read()
    iso = float(re.search(r"max isolated per-block error: ([0-9.e+-]+)", txt).group(1))
    rows = [l.split() for l in txt.splitlines() if l and not l.startswith("#")]
    nat, eag = [float(r[-4]) for r in rows], [float(r[-3]) for r in rows]
    report(f"error ladder (narrow UNet, 66 taps): max isolated per-block error {iso:.2e}; accumulated native/fp32 max {max(nat):.2e} vs fp16-eager/fp32 max {max(eag):.2e}")
    assert len(rows) >= 60
    # accumulated through the network, native never drifts further from fp32 than the reference's own fp16 path does (5 % slack per tap)
    assert all(n <= 1.05 * e + 1e-5 for n, e in zip(nat, eag)), [(r[0], n, e) for r, n, e in zip(rows, nat, eag) if n > 1.05 * e + 1e-5][:5]
