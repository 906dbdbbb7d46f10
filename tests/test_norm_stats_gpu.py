"""GroupNorm and LayerNorm statistics at the sizes the UNet and the VAE run them, on inputs whose groups / rows carry large DC offsets.

A variance taken as E[x^2] - E[x]^2 from fp32 running sums loses its digits when a group's mean is large against its standard
deviation, and the VAE's full-resolution GroupNorm sums ~1700 rows per thread.  Each (frame, group) here gets its own offset of
0, 16, 64 or 128 standard deviations; the result must be within 1e-3 (relative L2) of F.group_norm in fp64 and no worse than 1.5x
PyTorch's own fp16 F.group_norm against the same reference, for every (frame, group).
"""
import ctypes as C

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

from conftest import report

if torch.cuda.is_available():
    from humanvid_b200._native import check, i32, i64, lib, ptr, stream

OFFSETS = (0.0, 16.0, 64.0, 128.0)
GROUPS = 32


def rand(*shape, seed=0):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return torch.randn(*shape, generator=g, device="cuda")


def groupnorm(x1, x2, gamma, beta, NF, HW, silu):
    C1 = x1.shape[-1]
    C2 = x2.shape[-1] if x2 is not None else 0
    f = lib().hv_groupnorm_scratch_floats
    f.restype = C.c_size_t
    stats = torch.zeros(int(f(i64(C1 + C2), i64(NF), i64(HW), i32(GROUPS))), device="cuda", dtype=torch.float32)
    out = torch.empty(NF, HW, C1 + C2, device="cuda", dtype=torch.half)
    check(lib().hv_op_groupnorm(ptr(x1), i64(C1), ptr(x2), i64(C2), ptr(gamma), ptr(beta), ptr(out), i64(NF), i64(HW), i32(GROUPS), C.c_float(1e-6),
                                i32(silu), ptr(stats), stream()))
    return out


def offset_input(NF, HW, Ct, seed):
    """(NF, HW, Ct) fp16: unit-variance noise plus, per (frame, group), a DC offset from OFFSETS (every offset in every frame)."""
    x = rand(NF, HW, Ct, seed=seed)
    cpg = Ct // GROUPS
    off = torch.tensor([OFFSETS[(g + n) % len(OFFSETS)] for n in range(NF) for g in range(GROUPS)], device="cuda").view(NF, 1, GROUPS, 1)
    return (x.view(NF, HW, GROUPS, cpg) + off).view(NF, HW, Ct).half(), off.view(NF, GROUPS)


def per_group_rel(y, ref, NF, HW, Ct):
    d = (y.double() - ref).view(NF, HW, GROUPS, Ct // GROUPS)
    r = ref.view(NF, HW, GROUPS, Ct // GROUPS)
    return d.pow(2).sum((1, 3)).sqrt() / r.pow(2).sum((1, 3)).sqrt()


# (C1, C2, HW, NF): the VAE's full-resolution (768 x 576 and 576 x 1024) and lower levels, the UNet's level 0 and a level-3 skip concat
SHAPES = [(128, 0, 768 * 576, 1), (128, 0, 576 * 1024, 1), (256, 0, 384 * 288, 1), (512, 0, 96 * 72, 2), (320, 0, 96 * 72, 2), (1280, 640, 24 * 18, 3)]


@pytest.mark.parametrize("silu", [0, 1])
@pytest.mark.parametrize("C1,C2,HW,NF", SHAPES)
def test_groupnorm_offsets(C1, C2, HW, NF, silu):
    Ct = C1 + C2
    x, off = offset_input(NF, HW, Ct, seed=HW + Ct)
    gamma = (rand(Ct, seed=1) * 0.1 + 1).half()
    beta = (rand(Ct, seed=2) * 0.1).half()
    x1 = x[..., :C1].contiguous()
    x2 = x[..., C1:].contiguous() if C2 else None
    y = groupnorm(x1, x2, gamma, beta, NF, HW, silu)
    xc = x.permute(0, 2, 1)
    ref = F.group_norm(xc.double(), GROUPS, gamma.double(), beta.double(), 1e-6).permute(0, 2, 1)
    y16 = F.group_norm(xc, GROUPS, gamma, beta, 1e-6).permute(0, 2, 1)
    if silu:
        ref, y16 = F.silu(ref), F.silu(y16)
    torch.cuda.synchronize()
    e_nat = per_group_rel(y, ref, NF, HW, Ct)
    e_t16 = per_group_rel(y16, ref, NF, HW, Ct)
    worst = []
    for k in OFFSETS:
        sel = off == k
        worst.append(f"{k:g}σ native {float(e_nat[sel].max()):.2e} torch-fp16 {float(e_t16[sel].max()):.2e}")
    report(f"groupnorm C={C1}+{C2} HW={HW} NF={NF} silu={silu}: " + "; ".join(worst))
    bad = (e_nat > 1e-3) | (e_nat > 1.5 * e_t16)
    if bad.any():
        n, g = [int(v) for v in bad.nonzero()[0]]
        pytest.fail(f"{int(bad.sum())} (frame, group) over the bound, first frame {n} group {g} (offset {float(off[n, g]):g}σ): native "
                    f"{float(e_nat[n, g]):.3e}, torch fp16 {float(e_t16[n, g]):.3e}")


def test_groupnorm_slab_tail():
    """HW = 1001 is not a multiple of the 63 rows each statistics block sums (nor of the 4-row unrolled step), with offsets."""
    NF, HW, Ct = 2, 1001, 320
    x, _ = offset_input(NF, HW, Ct, seed=5)
    gamma, beta = (rand(Ct, seed=6) * 0.1 + 1).half(), (rand(Ct, seed=7) * 0.1).half()
    y = groupnorm(x, None, gamma, beta, NF, HW, 1)
    ref = F.silu(F.group_norm(x.permute(0, 2, 1).double(), GROUPS, gamma.double(), beta.double(), 1e-6).permute(0, 2, 1))
    y16 = F.silu(F.group_norm(x.permute(0, 2, 1), GROUPS, gamma, beta, 1e-6).permute(0, 2, 1))
    e_nat, e_t16 = per_group_rel(y, ref, NF, HW, Ct), per_group_rel(y16, ref, NF, HW, Ct)
    assert bool((e_nat <= 1e-3).all()) and bool((e_nat <= 1.5 * e_t16).all()), (float(e_nat.max()), float(e_t16.max()))


@pytest.mark.parametrize("C1,C2,HW", [(320, 0, 96 * 72), (128, 0, 96 * 72 * 4), (640, 320, 48 * 36)])
def test_groupnorm_frame_independent(C1, C2, HW):
    """A frame normalised alone is bitwise equal to the same frame as frame 1 of NF = 3: the order the statistics are summed in depends on
    HW only, which the multi-GPU split of the CFG halves relies on."""
    Ct = C1 + C2
    x, _ = offset_input(3, HW, Ct, seed=9)
    gamma, beta = (rand(Ct, seed=10) * 0.1 + 1).half(), (rand(Ct, seed=11) * 0.1).half()
    split = lambda t: (t[..., :C1].contiguous(), t[..., C1:].contiguous() if C2 else None)
    y3 = groupnorm(*split(x), gamma, beta, 3, HW, 1)
    y1 = groupnorm(*split(x[1:2]), gamma, beta, 1, HW, 1)
    torch.cuda.synchronize()
    assert torch.equal(y3[1:2].view(torch.int16), y1.view(torch.int16))


@pytest.mark.parametrize("Cc", [320, 640, 1280])
def test_layernorm_offsets(Cc):
    """LayerNorm (two-pass) with per-row DC offsets, the per-batch-item pre-add and the per-frame positional encoding: every row within
    1e-3 (relative L2) of fp64."""
    B, Fr, hw = 2, 4, 300
    rows = B * Fr * hw
    off = torch.tensor(OFFSETS, device="cuda").repeat(rows // len(OFFSETS))[:, None]
    x = (rand(rows, Cc, seed=50) + off).half()
    g, b = (rand(Cc, seed=51) * 0.1 + 1).half(), (rand(Cc, seed=52) * 0.1).half()
    add, pe = rand(B, Cc, seed=53).half(), rand(Fr, Cc, seed=54).half()
    out, xo = torch.empty_like(x), torch.empty_like(x)
    check(lib().hv_op_layernorm(ptr(x), ptr(g), ptr(b), ptr(out), i64(rows), i64(Cc), C.c_float(1e-5), ptr(add), i64(Fr * hw), ptr(xo), ptr(pe),
                                i64(hw), i64(Fr), stream()))
    xn = x.double() + add.double().repeat_interleave(Fr * hw, 0)
    ref = F.layer_norm(xn, (Cc,), g.double(), b.double(), 1e-5) + pe.double().repeat_interleave(hw, 0).repeat(B, 1)
    torch.cuda.synchronize()
    assert torch.equal(xo, xn.half())
    e = (out.double() - ref).norm(dim=1) / ref.norm(dim=1)
    report(f"layernorm C={Cc} with offsets: worst row rel {float(e.max()):.2e}")
    assert bool((e <= 1e-3).all()), f"row {int(e.argmax())} (offset {float(off[int(e.argmax())]):g}σ): rel {float(e.max()):.3e}"
