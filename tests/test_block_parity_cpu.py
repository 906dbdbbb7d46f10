"""Self-test of the per-block checks (tests/block_parity.py) on synthetic taps: an fp16 rounding of the fp64 reference passes, and each
of the faults the bounds exist for -- one element, one token row, one frame, two frames swapped, one CFG half in place of the other -- is
flagged, by the bound meant to catch it."""
import pytest
import torch

from block_parity import BlockReport, check_fp16_block, check_fp8_block, elem_ratio, row_ratio, slice_rel

B, F, H, W, C = 2, 3, 6, 10, 64      # 60 tokens per frame: a partial 128-key tile


def reference(seed=0):
    """fp64 tap (B*F, H, W, C) with a different scale per slice and a per-channel offset, like a block's output."""
    g = torch.Generator().manual_seed(seed)
    r = torch.randn(B * F, H, W, C, generator=g, dtype=torch.float64)
    r = r * torch.linspace(0.5, 2.0, B * F, dtype=torch.float64).view(-1, 1, 1, 1) + 0.3 * torch.randn(C, generator=g, dtype=torch.float64)
    return r


def fp16(t):
    return t.half().double()


def run(N, R, E):
    rep = BlockReport()
    check_fp16_block(rep, "synthetic", N, R, E)
    return rep


def test_fp16_rounding_passes():
    R = reference()
    g = torch.Generator().manual_seed(1)
    E = fp16(R + 2.0 ** -13 * R.pow(2).mean().sqrt() * torch.randn(R.shape, generator=g, dtype=torch.float64))   # another fp16 path
    rep = run(fp16(R), R, E)
    assert rep.failures() == [], rep.failures()
    assert rep.row.ratio < 0.25 and rep.elem.ratio < 0.25, "fp16 rounding alone should use a small part of the row and element bounds"


def _element(N, R):
    s = 4
    i = int(R[s].abs().flatten().argmin())                 # |R| << rms_s: the bound is about 2^-6 rms_s there
    rms = float(R[s].pow(2).mean().sqrt())
    N[s].view(-1)[i] += 2.0 ** -5 * rms
    return "elem"


def _row(N, R):
    N[4, H - 1, W - 1] = fp16(R[4, H - 1, W - 1] * (1 + 2.0 ** -6))   # the last token of a frame
    return "row"


def _frame(N, R):
    N[F + 1] = fp16(R[F + 1] * (1 + 2.0 ** -9))
    return "slice"


def _swap(N, R):
    N[[1, 2]] = N[[2, 1]].clone()
    return "elem"


def _cfg_half(N, R):
    N[:F] = N[F:].clone()                                  # the uncond half computed as the cond half
    return "elem"


@pytest.mark.parametrize("fault", [_element, _row, _frame, _swap, _cfg_half], ids=["element", "row", "frame", "frame-swap", "cfg-half"])
def test_fault_is_flagged(fault):
    R = reference()
    N = fp16(R)
    bound = fault(N, R)
    rep = run(N, R, fp16(R))
    assert rep.failures(), f"{fault.__name__}: not flagged"
    assert getattr(rep, bound).ratio > 1.0, f"{fault.__name__}: not flagged by the {bound} bound (ratios {rep.slice.ratio:.2f} / {rep.row.ratio:.2f} / {rep.elem.ratio:.2f})"


def test_flagged_location():
    """The report names the slice and row of a fault."""
    R = reference()
    N = fp16(R)
    _row(N, R)
    rep = run(N, R, fp16(R))
    assert rep.row.where[:3] == ("synthetic", 4, H * W - 1)


def test_slice_bound_follows_the_eager_path():
    """A native slice within 1e-3 but over 1.25 x the fp16 eager path's error on the same input (and over 2^-12) fails."""
    R = reference()
    g = torch.Generator().manual_seed(2)
    N = fp16(R * (1 + 2.0 ** -10.5 * torch.randn(R.shape, generator=g, dtype=torch.float64)))
    assert float(slice_rel(N, R).max()) < 1e-3
    rep = run(N, R, fp16(R))
    assert rep.slice.ratio > 1.0 and rep.row.ratio <= 1.0 and rep.elem.ratio <= 1.0


def test_fp8_bounds():
    """The e4m3 check: within the flip budget of the emulation's own error it passes; the extra term widens the element and row bounds."""
    R = reference()
    g = torch.Generator().manual_seed(3)
    Emu = R * (1 + 2.0 ** -5 * torch.randn(R.shape, generator=g, dtype=torch.float64))   # ~3 % quantisation error
    N8 = fp16(Emu)
    rep = BlockReport()
    check_fp8_block(rep, "e4m3", N8, Emu, R, torch.zeros_like(R))
    assert rep.failures(with_eager=False) == []
    N8[2] = fp16(Emu[2] * 1.05)      # 5 % on one frame: more than flipped roundings can add to a 3 % quantisation error
    bad = BlockReport()
    check_fp8_block(bad, "e4m3", N8, Emu, R, torch.zeros_like(R))
    assert bad.slice.ratio > 1.0 and bad.slice.where[1] == 2
    wide = fp16(Emu + 2.0 ** -4 * Emu.abs())
    assert float(elem_ratio(wide, Emu).max()) > 1.0
    assert float(elem_ratio(wide, Emu, 2.0 ** -3 * Emu.abs()).max()) <= 1.0
    assert float(row_ratio(wide, Emu, 2.0 ** -3 * Emu.abs()).max()) <= 1.0
