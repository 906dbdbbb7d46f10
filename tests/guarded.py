"""Guarded buffers for operator tests on the device: outputs are windows into sentinel-filled allocations and inputs sit in wider
allocations whose unused columns hold the sentinel, so a write outside the output or a read past an input's columns shows up."""
import pytest
import torch

SENT = 0x7E01   # a quiet-NaN bit pattern no arithmetic produces (NaNs the kernel computed would be 0x7E00 / 0x7FFF)
GUARD_ROWS = 3


def rand(*shape, scale=1.0, seed=0):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return (torch.randn(*shape, generator=g, device="cuda") * scale).half()


def strided(rows, cols, ld, scale=1.0, seed=0):
    """rows x cols fp16 random values in a [rows][ld] allocation whose columns [cols, ld) hold the sentinel NaN (must never be read)."""
    full = torch.full((rows, ld), SENT, dtype=torch.int16, device="cuda").view(torch.half)
    full[:, :cols] = rand(rows, cols, scale=scale, seed=seed)
    return full[:, :cols]


def bits(t):
    return t.contiguous().view(torch.int16)


class Guarded:
    """A rows x ld fp16 output window with GUARD_ROWS sentinel rows on either side; `out` is the [rows][ld] view handed to the kernel."""

    def __init__(self, rows, ld):
        self.rows, self.ld = rows, ld
        self.buf = torch.full(((rows + 2 * GUARD_ROWS), ld), SENT, dtype=torch.int16, device="cuda")
        self.out = self.buf.view(torch.half)[GUARD_ROWS : GUARD_ROWS + rows]

    def check_untouched(self, written, label):
        """`written`: bool [rows][ld] of the elements the call may write; everything else must still be the sentinel."""
        mask = torch.zeros(self.buf.shape, dtype=torch.bool, device="cuda")
        mask[GUARD_ROWS : GUARD_ROWS + self.rows] = written
        bad = (self.buf != SENT) & ~mask
        if bad.any():
            r, c = [int(v) for v in bad.nonzero()[0]]
            where = f"guard row {r - GUARD_ROWS}" if not GUARD_ROWS <= r < GUARD_ROWS + self.rows else f"row {r - GUARD_ROWS}"
            pytest.fail(f"{label}: {int(bad.sum())} elements written outside the output, first at {where}, column {c}")


def cols_mask(rows, ld, n_valid):
    m = torch.zeros(rows, ld, dtype=torch.bool, device="cuda")
    m[:, :n_valid] = True
    return m


def check_inputs_unchanged(before, after, label):
    for i, (b, a) in enumerate(zip(before, after)):
        assert torch.equal(b, bits(a)), f"{label}: input {i} was modified"
