"""The spatial (hv_op_attention) and temporal (hv_op_temporal_attention) attention kernels, element by element, against an fp64
reference of the same fp16 inputs, on every launch path, with guarded outputs.

Every output is a window into a buffer filled with a NaN sentinel, with guard rows around it (and, for the spatial op, a row stride wider
than the heads * d columns written); every input is checked unchanged bit for bit.  For query i, output column c, softmax weights p_ij
and keys j = 1..N_i, each element must satisfy

    |out_ic - ref_ic| <= (2^-10 + 2 delta_i) (|ref_ic| + sum_j p_ij |v_jc|) + N_i 2^-25 max_j |v_jc|
    delta_i = 2^-24 sqrt(d) max_j sum_k |q_ik| |k_jk|

2^-10 covers the fp16 rounding of the output and of P (the spatial kernel sums the same rounded P into its denominator through the
ones row of V^T; the temporal kernel divides by the fp32 sum of the unrounded exponentials), with headroom.  delta_i is the worst-case
fp32 error of a scaled score, as a relative error of p.  The last term covers P that falls below fp16's normal range.  Relative L2
< 1e-3 must hold as well.  The bound is derived, not fitted: a case over it is a finding, not a reason to widen it.

"Needle" keys score >= 30 nats above every other key of a chosen query, so that one key too many or too few under a mask (the last
valid key, the first key past a frame's or a bank item's end) moves that query's output by O(|v|), which a flat softmax over thousands
of keys would hide.
"""
import ctypes as C
import math

import pytest
import torch

pytestmark = pytest.mark.gpu

from conftest import report
from guarded import SENT, Guarded, bits, check_inputs_unchanged, cols_mask

if torch.cuda.is_available():
    from humanvid_b200._native import check, i32, i64, lib, ptr, stream

HV_ERR_INVALID = -1
BIG = 30000.0           # finite garbage in the V^T pad columns [L, vt_stride): read for a partial key tile, multiplied by P = 0
NEEDLE = 60.0           # score of a needle key against its query (nats); the other keys stay >= 30 below it (checked)
ELEMS = 1 << 24         # fp64 score elements per block of the reference
WORST = {}              # kernel family -> worst err / bound seen


@pytest.fixture(scope="module", autouse=True)
def _report_worst():
    yield
    for fam in sorted(WORST):
        report(f"attention guarded: worst err/bound {fam} {WORST[fam]:.3f}")


def round8(x):
    return (x + 7) // 8 * 8


def ref_and_bound(q, k, v):
    """fp64 softmax(q k^T / sqrt(d)) v of fp16 q [P][Nq][d], k and v [P][Nk][d], and the per-element bound of the module docstring;
    blocks of problems and query rows keep each score block <= ELEMS elements."""
    P, Nq, d = q.shape
    Nk = k.shape[1]
    ref = torch.empty(P, Nq, d, dtype=torch.float64, device=q.device)
    bound = torch.empty_like(ref)
    rows = max(1, ELEMS // Nk)
    pc, qc = (max(1, rows // Nq), Nq) if rows >= Nq else (1, rows)
    for p0 in range(0, P, pc):
        kd, vd = k[p0 : p0 + pc].double(), v[p0 : p0 + pc].double()
        vmax = vd.abs().amax(1, keepdim=True)
        for i0 in range(0, Nq, qc):
            qd = q[p0 : p0 + pc, i0 : i0 + qc].double()
            p = torch.softmax(qd @ kd.transpose(1, 2) / math.sqrt(d), -1)
            r = p @ vd
            delta = 2.0 ** -24 * math.sqrt(d) * (qd.abs() @ kd.abs().transpose(1, 2)).amax(-1, keepdim=True)
            ref[p0 : p0 + pc, i0 : i0 + qc] = r
            bound[p0 : p0 + pc, i0 : i0 + qc] = (2.0 ** -10 + 2 * delta) * (r.abs() + p @ vd.abs()) + Nk * 2.0 ** -25 * vmax
    return ref, bound


def check_close(out, ref, bound, family, label, where):
    """out (fp16), ref, bound: [P][Nq][d].  The first violation is reported as where(problem, query row) and column."""
    o = out.double()
    if not torch.isfinite(o).all():
        p, i, c = [int(x) for x in (~torch.isfinite(o)).nonzero()[0]]
        pytest.fail(f"{label}: non-finite output at {where(p, i)}, column {c}")
    err = (o - ref).abs()
    ratio = float((err / bound).max())
    WORST[family] = max(WORST.get(family, 0.0), ratio)
    rel = float((o - ref).norm() / (ref.norm() + 1e-30))
    viol = err > bound
    if viol.any():
        p, i, c = [int(x) for x in viol.nonzero()[0]]
        pytest.fail(f"{label}: {int(viol.sum())} elements over the bound, first at {where(p, i)}, column {c}: out {float(o[p, i, c]):.6g} "
                    f"ref {float(ref[p, i, c]):.6g} bound {float(bound[p, i, c]):.3g}; worst err/bound {ratio:.2f}; rel L2 {rel:.2e}")
    assert rel < 1e-3, f"{label}: rel L2 {rel:.2e}"


def directions(heads, d, n, seed):
    """n mutually orthogonal directions per head, each of squared norm d: [n][heads][d] (float32, on the device)."""
    g = torch.Generator().manual_seed(seed)
    qr = torch.linalg.qr(torch.randn(heads, d, d, generator=g, dtype=torch.float64)).Q
    return (qr[:, :, :n] * math.sqrt(d)).permute(2, 0, 1).float().cuda()


def needle_scale(d):
    """c with (c w) . (c w) / sqrt(d) = NEEDLE for |w|^2 = d."""
    return math.sqrt(NEEDLE / math.sqrt(d))


def assert_needle_gap(qv, target, others, label):
    """qv, target: [heads][d]; others: [heads][N][d] (the keys the needle must beat).  Checks the construction, not the kernel."""
    d = qv.shape[-1]
    if others.shape[1] == 0:
        return
    s_t = (qv.double() * target.double()).sum(-1) / math.sqrt(d)
    s_o = torch.einsum("hd,hnd->hn", qv.double(), others.double()).amax(-1) / math.sqrt(d)
    gap = float((s_t - s_o).min())
    assert gap >= 30, f"{label}: needle only {gap:.1f} nats above the other keys"


# ================================================================================================================= spatial
SPATIAL_ARGS = ("Q", "K", "Vt", "out", "NF", "L", "heads", "d", "ldq", "ldk", "ldvt", "ldo", "Kb", "Vbt", "Lb", "ldkb", "ldvbt", "F",
                "nf_nobank", "vt_stride", "vbt_stride")
PTR_ARGS = {"Q", "K", "Vt", "out", "Kb", "Vbt"}


def padded_heads(x, dpad, ld):
    """x [rows][heads][d] -> [rows][ld] with head h at columns [h dpad, h dpad + d), zeros up to (h + 1) dpad, the sentinel past heads dpad."""
    rows, heads, d = x.shape
    buf = torch.full((rows, ld), SENT, dtype=torch.int16, device="cuda").view(torch.half)
    body = buf[:, : heads * dpad]
    body.zero_()
    body.view(rows, heads, dpad)[:, :, :d] = x
    return buf


def vt_buffer(x, stride, extra):
    """x [n][l][heads][d] -> V^T [heads dv][n stride + extra]: rows h dv + c = channel c of head h, row h dv + d = ones, the rest zero, over
    columns [m stride, m stride + l) of item m; the pad columns [l, stride) of every item hold BIG; columns past n stride the sentinel."""
    n, l, heads, d = x.shape
    dv = (d + 1 + 15) // 16 * 16
    buf = torch.full((heads * dv, n * stride + extra), SENT, dtype=torch.int16, device="cuda").view(torch.half)
    body = buf[:, : n * stride]
    body.fill_(BIG)
    b4 = body.view(heads, dv, n, stride)
    b4[:, :, :, :l] = 0
    b4[:, :d, :, :l] = x.permute(2, 3, 0, 1)
    b4[:, d, :, :l] = 1
    return buf


class Spatial:
    """One hv_op_attention problem in separate, wider buffers (see the module docstring).  With needles (NF = 6 frames, F = 2 per batch
    item, B = 3 items), five queries get one key each:
      frame 4, row L-1   -> its own last key L-1                                   (read)
      frame 1, row L/2   -> the first key of frame 2, just past frame 1's segment  (masked)
      frame 3, row L-1   -> the last bank key Lb-1 of item 1                       (read)
      frame 2, row L/2   -> the first bank key of item 2, past item 1's segment    (masked)
      frame 0, row L-1   -> the last bank key of item 0                            (read only if nf_nobank = 0)"""

    def __init__(self, NF, L, heads, d, Lb=0, F=1, nf_nobank=0, scale=1.0, needles=False, seed=0):
        self.NF, self.L, self.heads, self.d, self.Lb, self.F, self.nf_nobank = NF, L, heads, d, Lb, F, nf_nobank
        self.dpad, self.dv = (d + 15) // 16 * 16, (d + 1 + 15) // 16 * 16
        self.B = B = NF // F
        g = torch.Generator(device="cuda").manual_seed(seed)
        rnd = lambda *s: torch.randn(*s, generator=g, device="cuda")  # noqa: E731
        q, k, v = rnd(NF, L, heads, d) * scale, rnd(NF, L, heads, d) * scale, rnd(NF, L, heads, d)
        kb, vb = rnd(B, Lb, heads, d) * scale, rnd(B, Lb, heads, d)
        self.needles = []
        if needles:
            assert (NF, F) == (6, 2)
            w = directions(heads, d, 5, seed) * needle_scale(d)
            plan = [(4, L - 1, "self", 4, L - 1), (1, L // 2, "self", 2, 0)]
            if Lb:
                plan += [(3, L - 1, "bank", 1, Lb - 1), (2, L // 2, "bank", 2, 0), (0, L - 1, "bank", 0, Lb - 1)]
            for m, (n, i, seg, item, t) in enumerate(plan):
                q[n, i] = w[m]
                (k if seg == "self" else kb)[item, t] = w[m]
                self.needles.append((n, i, seg, item, t))
        self.q, self.k, self.v, self.kb, self.vb = (x.half() for x in (q, k, v, kb, vb))
        hp = heads * self.dpad
        self.ldq, self.ldk, self.ldkb, self.ldo = hp + 24, hp + 40, hp + 56, heads * d + 24
        self.qbuf = padded_heads(self.q.reshape(NF * L, heads, d), self.dpad, self.ldq)
        self.kbuf = padded_heads(self.k.reshape(NF * L, heads, d), self.dpad, self.ldk)
        self.vt_stride = round8(L) + 16
        self.vt = vt_buffer(self.v, self.vt_stride, 24)
        self.inputs = [self.qbuf, self.kbuf, self.vt]
        self.kbbuf = self.vbt = None
        self.vbt_stride = 0
        if Lb:
            self.kbbuf = padded_heads(self.kb.reshape(B * Lb, heads, d), self.dpad, self.ldkb)
            self.vbt_stride = round8(Lb) + 16
            self.vbt = vt_buffer(self.vb, self.vbt_stride, 40)
            self.inputs += [self.kbbuf, self.vbt]
        for n, i, seg, item, t in self.needles:
            keys = self.keys(n)
            if seg == "self" and item == n:
                target, others = keys[:, t], torch.cat([keys[:, :t], keys[:, t + 1 :]], 1)
            elif seg == "bank" and self.uses_bank(n) and item == n // F:
                target, others = keys[:, L + t], torch.cat([keys[:, : L + t], keys[:, L + t + 1 :]], 1)
            else:
                target, others = (self.k if seg == "self" else self.kb)[item, t], keys
            assert_needle_gap(self.q[n, i], target, others, f"needle frame {n} row {i} -> {seg} {item} key {t}")

    def uses_bank(self, n):
        return self.Lb > 0 and n >= self.nf_nobank

    def keys(self, n):
        k = self.k[n].transpose(0, 1)
        return torch.cat([k, self.kb[n // self.F].transpose(0, 1)], 1) if self.uses_bank(n) else k

    def values(self, n):
        v = self.v[n].transpose(0, 1)
        return torch.cat([v, self.vb[n // self.F].transpose(0, 1)], 1) if self.uses_bank(n) else v

    def args(self, out, **override):
        a = dict(Q=self.qbuf, K=self.kbuf, Vt=self.vt, out=out, NF=self.NF, L=self.L, heads=self.heads, d=self.d, ldq=self.ldq, ldk=self.ldk,
                 ldvt=self.vt.stride(0), ldo=self.ldo, Kb=self.kbbuf, Vbt=self.vbt, Lb=self.Lb, ldkb=self.ldkb if self.Lb else 0,
                 ldvbt=self.vbt.stride(0) if self.Lb else 0, F=self.F, nf_nobank=self.nf_nobank, vt_stride=self.vt_stride,
                 vbt_stride=self.vbt_stride)
        a.update(override)
        return a

    def launch(self, out, **override):
        a = self.args(out, **override)
        conv = [ptr(a[n]) if n in PTR_ARGS else i32(a[n]) if n in ("heads", "d") else i64(a[n]) for n in SPATIAL_ARGS]
        return lib().hv_op_attention(*conv, stream())

    def run(self, label):
        g = Guarded(self.NF * self.L, self.ldo)
        before = [bits(t) for t in self.inputs]
        check(self.launch(g.out))
        torch.cuda.synchronize()
        g.check_untouched(cols_mask(self.NF * self.L, self.ldo, self.heads * self.d), label)
        check_inputs_unchanged(before, self.inputs, label)
        return g.out[:, : self.heads * self.d]

    def check(self, out, label):
        o = out.reshape(self.NF, self.L, self.heads, self.d)
        for n in range(self.NF):
            ref, bound = ref_and_bound(self.q[n].transpose(0, 1), self.keys(n), self.values(n))
            check_close(o[n].transpose(0, 1), ref, bound, "spatial", label, lambda h, i: f"frame {n}, head {h}, query row {i}")


SPATIAL_D = [8, 16, 32, 40, 64, 80, 160]
BANKS = [(0, 0), (1, 0), (1, 2), (128, 0), (128, 2), (200, 0), (200, 2)]   # (Lb, nf_nobank)


@pytest.mark.parametrize("Lb,nf_nobank", BANKS)
@pytest.mark.parametrize("L", [1, 127, 128, 129, 300])
@pytest.mark.parametrize("d", SPATIAL_D)
def test_spatial_attention(d, L, Lb, nf_nobank):
    """B = 3 bank items of F = 2 frames each (every item is read in one call), heads = 3, Q / K / Kb in separate buffers wider than
    heads * dpad, a guarded output with ldo > heads * d, vt_stride = round8(L) + 16 with finite garbage in the pad, and needle keys."""
    label = f"spatial d={d} L={L} Lb={Lb} nf_nobank={nf_nobank}"
    s = Spatial(6, L, 3, d, Lb=Lb, F=2, nf_nobank=nf_nobank, needles=True, seed=1000 * d + L + 7 * Lb + nf_nobank)
    out = s.run(label)
    if L == 1 and Lb == 0:
        assert torch.equal(bits(out), bits(s.v.reshape(6, 3 * d))), f"{label}: one key: the output is not V bit for bit"
    s.check(out, label)


@pytest.mark.parametrize("d", SPATIAL_D)
def test_spatial_attention_large_scores(d):
    """Q and K x8 (scores of std 8 sqrt(d)): row maxima grow past the lazy-rescale threshold across tiles and most exp2 arguments are
    below -126."""
    label = f"spatial x8 d={d}"
    s = Spatial(6, 300, 3, d, Lb=200, F=2, nf_nobank=2, scale=8.0, seed=d)
    s.check(s.run(label), label)


@pytest.mark.parametrize("L", [6912, 9216])
def test_spatial_attention_level0_bank(L):
    """The level-0 token counts with a bank of as many tokens: one frame without the bank, one with it."""
    label = f"spatial level-0 L={L}"
    s = Spatial(2, L, 8, 40, Lb=L, F=1, nf_nobank=1, seed=L)
    s.check(s.run(label), label)


def test_spatial_attention_rejects_bad_arguments():
    """Each rejected call returns HV_ERR_INVALID and writes nothing.  Every case would stay inside the buffers if its check were missing
    (the buffers are sized for it), so none can fault the device; NULL pointers the kernel would dereference are not passed."""
    NF, L, heads, d, Lb, F = 6, 129, 3, 40, 200, 2
    s = Spatial(NF, L, heads, d, Lb=Lb, F=F, nf_nobank=2, seed=3)
    hd, hp = heads * d, heads * s.dpad
    g = Guarded(NF * L, s.ldo)
    cases = {
        "NF=0": dict(NF=0), "L=0": dict(L=0), "heads=0": dict(heads=0), "d=24": dict(d=24),
        "nf_nobank=-1": dict(nf_nobank=-1), "nf_nobank>NF": dict(nf_nobank=NF + 1),
        "F does not divide NF": dict(F=4), "ldo<heads*d": dict(ldo=hd - 8), "ldq<heads*dpad": dict(ldq=hp - 8),
        "ldk<heads*dpad": dict(ldk=hp - 8), "ldkb<heads*dpad": dict(ldkb=hp - 8), "ldvt<NF*vt_stride": dict(ldvt=NF * s.vt_stride - 8),
        "ldvbt<B*vbt_stride": dict(ldvbt=s.B * s.vbt_stride - 8), "vbt_stride<Lb": dict(vbt_stride=round8(Lb) - 8),
        "Vbt NULL": dict(Vbt=None, nf_nobank=NF),
    }
    for name, over in cases.items():
        st = s.launch(g.out, **over)
        torch.cuda.synchronize()
        assert st == HV_ERR_INVALID, f"{name}: status {st}, expected HV_ERR_INVALID"
        g.check_untouched(torch.zeros(NF * L, s.ldo, dtype=torch.bool, device="cuda"), name)
    # F = 0 with a bank: without its check B would be NF, so the bank buffers hold NF items
    wide = Spatial(NF, L, heads, d, Lb=Lb, F=1, nf_nobank=0, seed=4)
    st = wide.launch(g.out, F=0)
    torch.cuda.synchronize()
    assert st == HV_ERR_INVALID, f"F=0 with a bank: status {st}"
    g.check_untouched(torch.zeros(NF * L, s.ldo, dtype=torch.bool, device="cuda"), "F=0")
    # grid limits: NF or heads above 65535, with buffers sized for the call
    for name, NFx, hx in (("NF>65535", 65536, 1), ("heads>65535", 1, 65536)):
        big = Spatial(NFx, 1, hx, 8, seed=5)
        gb = Guarded(NFx, big.ldo)
        st = big.launch(gb.out)
        torch.cuda.synchronize()
        assert st == HV_ERR_INVALID, f"{name}: status {st}"
        gb.check_untouched(torch.zeros(NFx, big.ldo, dtype=torch.bool, device="cuda"), name)


# ================================================================================================================= temporal
TT_WARPS = 12           # warps per CTA of the TMA-staged kernel (attn_temporal.cu)
GUARD = 2               # NaN rows before and after the qkv window


def tplan(B, F, HW, heads, d):
    tma, hpb, grid = C.c_int32(), C.c_int32(), C.c_int32()
    check(lib().hv_dbg_temporal_attention_plan(i64(B), i64(F), i64(HW), i32(heads), i32(d), C.byref(tma), C.byref(hpb), C.byref(grid)))
    return bool(tma.value), hpb.value, grid.value


class Temporal:
    """QKV rows (b, f, p) of [q | k | v] in a window with NaN guard rows; needles on key F-1 for three pixels of every batch item (all
    heads), each for one query frame."""

    def __init__(self, B, F, HW, heads, d, seed=0, needles=True, x=None):
        self.B, self.F, self.HW, self.heads, self.d = B, F, HW, heads, d
        self.C = heads * d
        if x is None:
            g = torch.Generator(device="cuda").manual_seed(seed)
            x = torch.randn(B, F, HW, 3, heads, d, generator=g, device="cuda")
            if needles and F > 1:
                c = needle_scale(d)
                for b in range(B):
                    for p in sorted({0, HW // 2, HW - 1}):
                        w = torch.randn(heads, d, generator=g, device="cuda")
                        w = w * (math.sqrt(d) / w.norm(dim=-1, keepdim=True)) * c
                        f = (b + p) % F
                        x[b, f, p, 0] = w
                        x[b, F - 1, p, 1] = w
                        assert_needle_gap(x[b, f, p, 0].half(), x[b, F - 1, p, 1].half(), x[b, : F - 1, p, 1].half().transpose(0, 1),
                                          f"needle b={b} p={p}")
            x = x.half()
        self.x = x
        rows = B * F * HW
        self.buf = torch.full((rows + 2 * GUARD, 3 * self.C), SENT, dtype=torch.int16, device="cuda").view(torch.half)
        self.qkv = self.buf[GUARD : GUARD + rows]
        self.qkv.copy_(x.reshape(rows, 3 * self.C))

    def launch(self, out, **override):
        a = dict(B=self.B, F=self.F, HW=self.HW, heads=self.heads, d=self.d, qkv=self.qkv, out=out)
        a.update(override)
        return lib().hv_op_temporal_attention(ptr(a["qkv"]), ptr(a["out"]), i64(a["B"]), i64(a["F"]), i64(a["HW"]), i32(a["heads"]), i32(a["d"]),
                                              stream())

    def run(self, label):
        rows = self.B * self.F * self.HW
        g = Guarded(rows, self.C)
        before = [bits(self.buf)]
        check(self.launch(g.out))
        torch.cuda.synchronize()
        g.check_untouched(cols_mask(rows, self.C, self.C), label)
        check_inputs_unchanged(before, [self.buf], label)
        return g.out

    def problems(self, t):
        """[B][F][HW][heads][d] -> [(b, p, h)][F][d]"""
        return t.reshape(self.B, self.F, self.HW, self.heads, self.d).permute(0, 2, 3, 1, 4).reshape(-1, self.F, self.d)

    def check(self, out, family, label):
        x = self.x
        if self.F == 1:
            assert torch.equal(bits(out), bits(x[:, :, :, 2].reshape(-1, self.C))), f"{label}: one frame: the output is not V bit for bit"
        q, k, v = (self.problems(x[:, :, :, j]) for j in range(3))
        ref, bound = ref_and_bound(q, k, v)
        HW, heads = self.HW, self.heads
        check_close(self.problems(out), ref, bound, family, label,
                    lambda P, i: f"batch item {P // (HW * heads)}, pixel {P // heads % HW}, head {P % heads}, query frame {i}")


TEMPORAL_REG_D = [8, 16, 32, 40, 80, 160]


@pytest.mark.parametrize("B", [1, 3])
@pytest.mark.parametrize("heads", [1, 3, 8])
@pytest.mark.parametrize("d", TEMPORAL_REG_D)
def test_temporal_register_kernel(d, heads, B):
    """The register kernel (HW * heads < 2048) at every F from 1 to 32."""
    HW = 37
    for F in range(1, 33):
        label = f"temporal register d={d} heads={heads} B={B} F={F}"
        assert not tplan(B, F, HW, heads, d)[0], label
        t = Temporal(B, F, HW, heads, d, seed=F + 100 * d + 10 * heads + B)
        t.check(t.run(label), "temporal register", label)


def tma_case(regime, d, heads=8):
    """(B, HW) on this device: 'few' has fewer (pixel, box) problems than the 12 * SMs resident warps; 'many' gives every warp of the
    persistent grid three or four problems (a remainder)."""
    sms = int(lib().hv_num_sms())
    hpb = 2 if d == 40 else 1
    if regime == "few":
        B, HW = 1, -(-2048 // heads) + 3
    else:
        B = 2
        target = 3 * TT_WARPS * sms + TT_WARPS * sms // 2 + 5
        HW = -(-target * hpb // (B * heads))
    tma, got_hpb, grid = tplan(B, 1, HW, heads, d)
    groups = B * HW * heads // hpb
    desc = f"B={B} HW={HW} heads={heads}: {groups} problems, grid {grid} x {TT_WARPS} warps on {sms} SMs"
    assert tma and got_hpb == hpb, desc
    if regime == "few":
        assert groups < TT_WARPS * sms and grid == -(-groups // TT_WARPS) and groups % TT_WARPS, desc
    else:
        assert grid == sms and groups > 3 * TT_WARPS * grid and groups % (TT_WARPS * grid), desc
    return B, HW, desc


TMA_CASES = [("few", 40), ("many", 40), ("many", 80)]


@pytest.mark.parametrize("regime,d", TMA_CASES)
def test_temporal_tma_kernel(regime, d):
    """The TMA-staged kernel (d = 40 two heads per box, d = 80 one) at every F from 1 to 32."""
    heads = 8
    B, HW, desc = tma_case(regime, d, heads)
    report(f"temporal TMA {regime} d={d}: {desc}")
    for F in range(1, 33):
        label = f"temporal TMA {regime} d={d} F={F} ({desc})"
        t = Temporal(B, F, HW, heads, d, seed=F + 100 * d)
        t.check(t.run(label), "temporal TMA", label)


@pytest.mark.parametrize("heads", [3, 5])
def test_temporal_odd_heads_keep_register_kernel(heads):
    """d = 40 with odd heads above the HW * heads >= 2048 threshold: two heads per box do not divide the heads, so the register kernel runs."""
    d, B = 40, 1
    HW = -(-2048 // heads) + 1
    for F in (1, 2, 7, 16, 31, 32):
        label = f"temporal d=40 odd heads={heads} HW={HW} F={F}"
        assert tplan(B, F, HW, heads, d) == (False, 1, -(-B * HW * heads // 8)), label
        t = Temporal(B, F, HW, heads, d, seed=F + heads)
        t.check(t.run(label), "temporal register", label)


def test_temporal_tma_stale_slab_rows_are_masked():
    """Rows >= F of the TMA kernel's q / k slabs are shared memory this launch never wrote; only the key mask keeps them out, and the v
    rows >= F are zeroed at the start of each launch.  A first launch with F = 32 fills the slabs: its keys all point along one direction
    per head and its values past frame 7 are NaN.  The next launch (F = 7, same shape otherwise, so the same warps and slabs) has every
    query along that direction: a stale key left unmasked would dominate its softmax, a stale value left unzeroed would make it NaN.
    That the second launch lands on the slabs the first wrote is likely (same grid, one CTA per SM), not guaranteed."""
    d, heads = 40, 8
    B, HW, desc = tma_case("many", d, heads)
    c = needle_scale(d)
    u = directions(heads, d, 1, 11)[0] * c                      # [heads][d]
    g = torch.Generator(device="cuda").manual_seed(12)
    x = torch.randn(B, 32, HW, 3, heads, d, generator=g, device="cuda")
    x[:, :, :, 1] = u
    x = x.half()
    x[:, 7:, :, 2] = torch.tensor(SENT, dtype=torch.int16).view(torch.half).item()
    stain = Temporal(B, 32, HW, heads, d, x=x)
    out = torch.empty(B * 32 * HW, heads * d, device="cuda", dtype=torch.half)
    check(stain.launch(out))
    y = torch.randn(B, 7, HW, 3, heads, d, generator=g, device="cuda")
    y[:, :, :, 0] = u
    t = Temporal(B, 7, HW, heads, d, x=y.half())
    label = f"temporal TMA F=7 after F=32 ({desc})"
    t.check(t.run(label), "temporal TMA", label)


@pytest.mark.parametrize("d", [40, 80])
def test_temporal_tma_equals_register_kernel(d):
    """The TMA kernel loads the same fragments, issues the same MMAs in the same order and runs the same softmax as the register kernel,
    so their outputs are equal bit for bit.  The register kernel's output comes from pixel chunks small enough (HW * heads < 2048) for it."""
    heads = 8
    B, HW, desc = tma_case("many", d, heads)
    chunk = 2047 // heads
    for F in range(1, 33):
        t = Temporal(B, F, HW, heads, d, seed=500 + F)
        tma_out = t.run(f"tma d={d} F={F}").clone()
        x = t.x.reshape(B, F, HW, 3 * heads * d)
        reg = torch.empty(B, F, HW, heads * d, device="cuda", dtype=torch.half)
        for p0 in range(0, HW, chunk):
            n = min(chunk, HW - p0)
            assert not tplan(B, F, n, heads, d)[0]
            part = Temporal(B, F, n, heads, d, x=x[:, :, p0 : p0 + n].reshape(B, F, n, 3, heads, d).contiguous())
            reg[:, :, p0 : p0 + n] = part.run(f"register chunk d={d} F={F} p0={p0}").reshape(B, F, n, heads * d)
        same = bits(tma_out) == bits(reg.reshape(-1, heads * d))
        if not same.all():
            r, col = [int(v) for v in (~same).nonzero()[0]]
            pytest.fail(f"d={d} F={F} ({desc}): TMA and register kernels differ in {int((~same).sum())} elements, first at batch item "
                        f"{r // (F * HW)}, frame {r // HW % F}, pixel {r % HW}, head {col // d}, column {col % d}")


@pytest.mark.parametrize("d", [40, 80])
@pytest.mark.parametrize("side", ["below", "above"])
def test_temporal_batch_independence_and_determinism(d, side):
    """The kernel choice depends on HW only: the B = 2 output equals two B = 1 outputs bit for bit, just below and just above the
    HW * heads >= 2048 threshold; two runs are bit for bit equal."""
    heads, F = 8, 13
    HW = 2048 // heads - (1 if side == "below" else 0)
    assert tplan(2, F, HW, heads, d)[0] == (side == "above") == tplan(1, F, HW, heads, d)[0]
    t = Temporal(2, F, HW, heads, d, seed=d + HW)
    both = t.run(f"B=2 d={d} HW={HW}").clone()
    assert torch.equal(bits(both), bits(t.run(f"B=2 again d={d} HW={HW}"))), f"d={d} HW={HW}: two runs differ"
    rows = F * HW
    for b in range(2):
        one = Temporal(1, F, HW, heads, d, x=t.x[b : b + 1].contiguous())
        assert torch.equal(bits(one.run(f"B=1 item {b}")), bits(both[b * rows : (b + 1) * rows])), f"d={d} HW={HW}: batch item {b} depends on B"


def test_temporal_attention_rejects_bad_arguments():
    """Each rejected call returns HV_ERR_INVALID and writes nothing.  The shapes stay on the register kernel and the qkv buffer holds
    33 frames, so none of the calls could leave the buffers without its check; NULL pointers are not passed."""
    B, HW, heads, d = 1, 37, 8, 40
    t = Temporal(B, 33, HW, heads, d, seed=9, needles=False)
    g = Guarded(B * 33 * HW, heads * d)
    cases = {"B=0": dict(B=0), "F=0": dict(F=0), "F=33": dict(F=33), "HW=0": dict(HW=0), "heads=0": dict(heads=0), "d=24": dict(d=24),
             "d=64": dict(d=64, heads=5)}
    for name, over in cases.items():
        st = t.launch(g.out, **{"F": 32, **over})
        torch.cuda.synchronize()
        assert st == HV_ERR_INVALID, f"{name}: status {st}, expected HV_ERR_INVALID"
        g.check_untouched(torch.zeros(B * 33 * HW, heads * d, dtype=torch.bool, device="cuda"), name)
