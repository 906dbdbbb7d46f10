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


def need(t, dtype, nbytes, label):
    """Preflight of one operand, on the host and before the launch: `t` is a CUDA tensor of `dtype` (what the operator reads it as)
    and its storage spans at least `nbytes` from the data pointer on, so the extent the operator's header states stays inside the
    allocation."""
    assert isinstance(t, torch.Tensor) and t.is_cuda, f"{label}: not a CUDA tensor"
    assert t.dtype == dtype, f"{label}: dtype {t.dtype}, the operator reads {dtype}"
    st = t.untyped_storage()
    span = st.data_ptr() + st.nbytes() - t.data_ptr()
    assert span >= nbytes, f"{label}: {span} bytes from the data pointer to the end of the allocation, the operator may touch {nbytes}"


def check_step_tables(inv, n_windows, Fw, frame_idx=None, Ftot=None, step_index=None, coef_rows=None):
    """Host-side check of the index tables the step glue reads on the device, before they are uploaded: every `inv` [Ftot][K] entry is -1
    or window * Fw + position with window < n_windows (any other entry reads through a NULL prediction slot), every row has at least one
    entry (a frame no window covers is outside the operator's contract), every `frame_idx` entry is a frame < Ftot, and `step_index`
    names a row of the coefficient table."""
    inv = torch.as_tensor(inv)
    assert not inv.is_cuda and inv.dtype == torch.int32 and inv.dim() == 2, "inv: host int32 [Ftot][K]"
    assert bool(((inv == -1) | ((inv >= 0) & (inv < n_windows * Fw))).all()), "inv: an entry is neither -1 nor a slot of a window"
    assert bool((inv >= 0).any(1).all()), "inv: a frame no window covers"
    if frame_idx is not None:
        fi = torch.as_tensor(frame_idx)
        assert not fi.is_cuda and fi.dtype == torch.int32 and fi.numel() == Fw, "frame_idx: host int32 [Fw]"
        assert bool(((fi >= 0) & (fi < Ftot)).all()), "frame_idx: a frame outside [0, Ftot)"
    if step_index is not None:
        assert 0 <= int(step_index) < coef_rows, f"step_index {int(step_index)} outside the {coef_rows} coefficient rows"
