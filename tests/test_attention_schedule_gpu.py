"""Spatial attention (hv_op_attention) against fp32 scaled_dot_product_attention over the cases its schedule distinguishes: every
head-dim instantiation, key segments (self and reference bank) that end on a full or a partial 128-key tile, odd and even
query-tile counts, frames that skip the bank, scores large enough to drive the lazy rescale and exp2 arguments below -126,
and run-to-run bitwise determinism."""
import ctypes as C

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

if torch.cuda.is_available():
    from humanvid_b200._native import check, i32, i64, lib, ptr, stream


def rel(a, b):
    a, b = a.float(), b.float()
    return float((a - b).norm() / (b.norm() + 1e-12))


def run_attention(NF, L, heads, d, Lb=0, Fr=1, nf_nobank=0, qk_scale=1.0, seed=0):
    """Inputs in the model's layout (Q and K interleaved per token, heads padded to dpad; V^T[head * dv + c][frame * Lp + t]
    with a row of ones at c = d), then the native output and the fp32 reference."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    rnd = lambda *s: torch.randn(*s, generator=g, device="cuda")  # noqa: E731
    dpad, dv = (d + 15) // 16 * 16, (d + 1 + 15) // 16 * 16
    q, k, v = (rnd(NF, L, heads, d) * qk_scale).half(), (rnd(NF, L, heads, d) * qk_scale).half(), rnd(NF, L, heads, d).half()
    qk = torch.zeros(NF * L, 2, heads, dpad, device="cuda", dtype=torch.half)
    qk[:, 0, :, :d] = q.reshape(NF * L, heads, d)
    qk[:, 1, :, :d] = k.reshape(NF * L, heads, d)
    qk = qk.reshape(NF * L, 2 * heads * dpad)

    def vt_of(x):   # x: (n, l, heads, d) -> V^T with the ones row
        n, l = x.shape[:2]
        lp = (l + 7) // 8 * 8
        vt = torch.zeros(heads, dv, n, lp, device="cuda", dtype=torch.half)
        vt[:, :d, :, :l] = x.permute(2, 3, 0, 1)
        vt[:, d, :, :l] = 1
        return vt.reshape(heads * dv, n * lp), lp

    vt, Lp = vt_of(v)
    B = NF // Fr
    kb = vbt = None
    Lbp = 0
    if Lb:
        kbr, vbr = (rnd(B, Lb, heads, d) * qk_scale).half(), rnd(B, Lb, heads, d).half()
        kb = torch.zeros(B * Lb, heads, dpad, device="cuda", dtype=torch.half)
        kb[:, :, :d] = kbr.reshape(B * Lb, heads, d)
        kb = kb.reshape(B * Lb, heads * dpad)
        vbt, Lbp = vt_of(vbr)
    out = torch.zeros(NF * L, heads * d, device="cuda", dtype=torch.half)

    def native():
        out.zero_()
        check(lib().hv_op_attention(ptr(qk), C.c_void_p(qk.data_ptr() + heads * dpad * 2), ptr(vt), ptr(out), i64(NF), i64(L), i32(heads),
                                    i32(d), i64(2 * heads * dpad), i64(2 * heads * dpad), i64(vt.stride(0)), i64(heads * d), ptr(kb), ptr(vbt),
                                    i64(Lb), i64(heads * dpad), i64(vbt.stride(0) if vbt is not None else 0), i64(Fr), i64(nf_nobank), i64(Lp),
                                    i64(Lbp), stream()))
        torch.cuda.synchronize()
        return out.clone()

    ref = torch.empty(NF, heads, L, d, device="cuda")
    for n in range(NF):
        kk, vv = k[n].float().transpose(0, 1), v[n].float().transpose(0, 1)
        if Lb and n >= nf_nobank:
            kk = torch.cat([kk, kbr[n // Fr].float().transpose(0, 1)], 1)
            vv = torch.cat([vv, vbr[n // Fr].float().transpose(0, 1)], 1)
        ref[n] = F.scaled_dot_product_attention(q[n].float().transpose(0, 1), kk, vv)
    return native, ref.transpose(1, 2).reshape(NF * L, heads * d)


@pytest.mark.parametrize("d", [8, 16, 32, 40, 80, 160])
def test_head_dims_full_tiles(d):
    # L = 256, Lb = 384: every key tile is full; two query tiles per (frame, head)
    native, ref = run_attention(4, 256, 2, d, Lb=384, Fr=2, nf_nobank=2, seed=d)
    out = native()
    assert torch.isfinite(out).all()
    assert rel(out, ref) < 1e-3


@pytest.mark.parametrize("NF,L,heads,d,Lb,Fr,nf_nobank", [
    (2, 384, 2, 40, 256, 1, 1),     # full tiles, three query tiles (odd)
    (2, 300, 2, 40, 256, 1, 1),     # partial last self tile, full bank tiles, three query tiles
    (2, 256, 2, 80, 200, 1, 1),     # full self tiles, partial last bank tile
    (4, 200, 2, 160, 136, 2, 2),    # both segments end on a partial tile, two query tiles
    (3, 108, 2, 160, 108, 3, 0),    # one partial tile per segment, one query tile, every frame reads the bank
    (2, 640, 2, 40, 0, 1, 0),       # self only, five query tiles
    (2, 1728, 2, 80, 1728, 1, 1),   # level-1 token count (config 2), odd query-tile count with partial tiles
])
def test_tile_and_segment_shapes(NF, L, heads, d, Lb, Fr, nf_nobank):
    native, ref = run_attention(NF, L, heads, d, Lb=Lb, Fr=Fr, nf_nobank=nf_nobank, seed=L + Lb)
    assert rel(native(), ref) < 1e-3


@pytest.mark.parametrize("L,d,Lb", [(512, 40, 384), (300, 40, 260), (300, 80, 130), (256, 160, 200)])
def test_large_scores(L, d, Lb):
    # q and k scaled by 8: row maxima grow by far more than the rescale threshold across tiles, and most exp2 arguments are < -126
    native, ref = run_attention(2, L, 2, d, Lb=Lb, Fr=1, nf_nobank=1, qk_scale=8.0, seed=7 * L + d)
    out = native()
    assert torch.isfinite(out).all()
    assert rel(out, ref) < 1e-3


def test_level0_with_bank_deterministic():
    # level-0 token count of configs 2-4 with a bank: one frame without the bank, one with it; two runs are bit for bit equal
    native, ref = run_attention(2, 6912, 8, 40, Lb=6912, Fr=1, nf_nobank=1, seed=5)
    a = native()
    b = native()
    assert torch.equal(a, b)
    assert rel(a, ref) < 1e-3
