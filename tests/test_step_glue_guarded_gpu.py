"""The per-timestep glue of the device denoising loop -- hv_op_window_gather, hv_op_cfg_ddim_step and hv_op_advance_index -- against an
fp64 restatement of pipeline_pose2vid_long.py:516-563: gather each window's frames (repeated for the CFG batch), accumulate every
window's prediction onto its frames, divide by the count, apply classifier-free guidance, then take the DDIM step with eta = 0.

The gather is pure data movement and is compared bit for bit.  For the step, every latent element is held to a bound derived from the
kernel's fp32 arithmetic (u = 2^-24, gamma_k = k u / (1 - k u)), for a frame in n windows and guidance s:
    un = (sum of n fp16 predictions) * (1 / n)          e_un <= gamma_{n+1} A_un,  A_un = sum |p| / n     (n - 1 adds, the reciprocal,
                                                                                                          the product); tx likewise
    m = un + s (tx - un)                                e_m <= (1 + |s|) e_un + |s| e_tx + 2u |s| |tx - un| + u |m|      (m = un without CFG)
    v-prediction:  x0 = a x - b m,  eps = a m + b x     e_x0 <= b e_m + 2u (|a x| + |b m|),  e_eps <= a e_m + 2u (|a m| + |b x|)
    epsilon:       eps = m,  x0 = (x - b eps) / a       e_x0 <= (b e_m + 2u (|x| + |b m|)) / a + u |x0|
    x_prev = c x0 + d eps                               E <= c e_x0 + d e_eps + 2u (|c x0| + |d eps|)
and the fp16 store:  |out - ref| <= 2^-11 (|ref| + E) + E + 2^-25 (tight: worst ratios near 1 are expected).  (a, b, c, d) = (sqrt(a_t), sqrt(1 - a_t), sqrt(a_prev),
sqrt(1 - a_prev)) are the fp32 values of the coefficient table, used in fp64 by the reference.  Epsilon runs on a table without the
zero-terminal-SNR rescale: at a_t = 0 its x0 divides by zero, in the kernel and in diffusers alike.

Every table the kernels read on the device is checked on the host before upload (guarded.check_step_tables): `inv` entries are -1 or a
slot of one of the n_windows windows, `frame_idx` entries are frames of the clip, `step_index` names a coefficient row; every tensor
is checked for its dtype and byte extent (guarded.need).  Latents are updated in place: the latent buffer sits in a guarded window and
everything else is checked unchanged bit for bit.

A frame that no window covers is outside the operator's contract: the kernel leaves its mean prediction at 0 where the pipeline
computes 0 / 0.  No test pins that behaviour, and the table check rejects such tables.
"""
import ctypes as C

import pytest
import torch

pytestmark = pytest.mark.gpu

from conftest import report
from guarded import Guarded, bits, check_inputs_unchanged, check_step_tables, need
from norm_bounds import U, gam

if torch.cuda.is_available():
    from humanvid_b200._native import check, i32, i64, lib, ptr, stream

HALF, I32, F32 = torch.half, torch.int32, torch.float32
WORST = {}


@pytest.fixture(scope="module", autouse=True)
def _report_worst():
    yield
    for fam in sorted(WORST):
        report(f"step glue guarded: worst err/bound {fam} {WORST[fam]:.3f}")


def op_window_gather(lat, idx_dev, out, Bl, Cc, Ftot, Fw, HW, repeat):
    need(lat, HALF, Bl * Cc * Ftot * HW * 2, "window_gather latents")
    need(idx_dev, I32, Fw * 4, "window_gather frame_idx")
    need(out, HALF, repeat * Bl * Cc * Fw * HW * 2, "window_gather out")
    check(lib().hv_op_window_gather(ptr(lat), ptr(idx_dev), ptr(out), i64(Bl), i64(Cc), i64(Ftot), i64(Fw), i64(HW), i32(repeat), stream()))


def op_cfg_ddim_step(preds_u, preds_c, inv_dev, coef_dev, step_dev, lat, Bl, Cc, Ftot, Fw, HW, s, prediction_type):
    n = Bl * Cc * Fw * HW * 2
    for w, p in enumerate(preds_u):
        need(p, HALF, n, f"cfg_ddim_step pred_uncond[{w}]")
    for w, p in enumerate(preds_c or []):
        need(p, HALF, n, f"cfg_ddim_step pred_cond[{w}]")
    K = inv_dev.shape[1]
    need(inv_dev, I32, Ftot * K * 4, "cfg_ddim_step inv")
    need(coef_dev, F32, coef_dev.shape[0] * 16, "cfg_ddim_step coef")   # check_step_tables keeps step_index below the row count
    assert coef_dev.data_ptr() % 16 == 0, "cfg_ddim_step coef: read as float4"
    if step_dev is not None:
        need(step_dev, I32, 4, "cfg_ddim_step step_index")
    need(lat, HALF, Bl * Cc * Ftot * HW * 2, "cfg_ddim_step latents")
    nw = len(preds_u)
    pu = (C.c_void_p * nw)(*[p.data_ptr() for p in preds_u])
    pc = (C.c_void_p * nw)(*[p.data_ptr() for p in preds_c]) if preds_c is not None else None
    check(lib().hv_op_cfg_ddim_step(pu, pc, i32(nw), ptr(inv_dev), i32(K), ptr(coef_dev), ptr(step_dev), ptr(lat), i64(Bl), i64(Cc), i64(Ftot),
                                    i64(Fw), i64(HW), C.c_float(s), i32(prediction_type), stream()))


def op_advance_index(step_dev):
    need(step_dev, I32, 4, "advance_index index")
    check(lib().hv_op_advance_index(ptr(step_dev), stream()))


def coef_table(steps, prediction):
    from humanvid_b200.scheduler import DDIMScheduler

    sched = DDIMScheduler(prediction_type="v_prediction" if prediction == 0 else "epsilon", rescale_betas_zero_snr=prediction == 0)
    sched.set_timesteps(steps)
    return sched.coef_table()


def inverse_map(windows, Ftot, K=None):
    """[Ftot][K] int32 on the host: the (window * Fw + position) slots of each frame, -1 padded to K columns (K >= the widest coverage)."""
    Fw = len(windows[0])
    slots = [[] for _ in range(Ftot)]
    for w, win in enumerate(windows):
        for i, f in enumerate(win):
            slots[f].append(w * Fw + i)
    K = K or max(len(s) for s in slots)
    return torch.tensor([s + [-1] * (K - len(s)) for s in slots], dtype=I32)


def step_ref_and_E(lat, preds, windows, Bl, s, cfg, coef_row, prediction):
    """fp64 restatement of pipeline_pose2vid_long.py:550-563 and the bound E of the module docstring; lat (Bl, C, Ftot, HW) fp16,
    preds[w] (R * Bl, C, Fw, HW) fp16 (R = 2 with CFG: uncond half first)."""
    Ftot = lat.shape[2]
    shape = (Bl,) + tuple(lat.shape[1:])
    acc_u, abs_u = torch.zeros(shape, dtype=torch.float64, device="cuda"), torch.zeros(shape, dtype=torch.float64, device="cuda")
    acc_t, abs_t = torch.zeros_like(acc_u), torch.zeros_like(acc_u)
    cnt = torch.zeros(1, 1, Ftot, 1, dtype=torch.float64, device="cuda")
    for win, p in zip(windows, preds):
        pd = p.double()
        acc_u[:, :, win] += pd[:Bl]
        abs_u[:, :, win] += pd[:Bl].abs()
        if cfg:
            acc_t[:, :, win] += pd[Bl:]
            abs_t[:, :, win] += pd[Bl:].abs()
        cnt[:, :, win] += 1
    assert bool((cnt > 0).all())
    un, tx = acc_u / cnt, acc_t / cnt
    g = gam(cnt + 1)
    e_un, e_tx = g * abs_u / cnt, g * abs_t / cnt
    if cfg:
        m = un + s * (tx - un)
        e_m = (1 + abs(s)) * e_un + abs(s) * e_tx + 2 * U * abs(s) * (tx - un).abs() + U * m.abs()
    else:
        m, e_m = un, e_un
    a, b, c, d = [float(v) for v in coef_row]
    x = lat.double()
    if prediction == 0:
        x0, eps = a * x - b * m, a * m + b * x
        e_x0 = b * e_m + 2 * U * ((a * x).abs() + (b * m).abs())
        e_eps = a * e_m + 2 * U * ((a * m).abs() + (b * x).abs())
    else:
        eps = m
        x0 = (x - b * eps) / a
        e_x0 = (b * e_m + 2 * U * (x.abs() + (b * m).abs())) / a + U * x0.abs()
        e_eps = e_m
    ref = c * x0 + d * eps
    E = c * e_x0 + d * e_eps + 2 * U * ((c * x0).abs() + (d * eps).abs())
    return ref, E


def judge(fam, label, y, ref, E):
    y = y.double().reshape(ref.shape)
    assert bool(torch.isfinite(y).all()), f"{label}: non-finite latents"
    bound = 2.0 ** -11 * (ref.abs() + E) + E + 2.0 ** -25
    r = (y - ref).abs() / bound
    worst = float(r.max())
    WORST[fam] = max(WORST.get(fam, 0.0), worst)
    assert worst <= 1.0, f"{label}: worst err/bound {worst:.3f}"


def uniform_windows(Ftot, Fw):
    from humanvid_b200.pipeline import uniform

    return [list(w) for w in uniform(0, 20, Ftot, Fw, 1, 4)]


# (label, Ftot, Fw, windows): the shipped context of 24 frames with overlap 4 over 24 frames (configs 2-4) and 48 frames (config 5: three
# windows), a short clip, and a hand-built table in which frame 5 lies in three windows and the inverse map is wider than any frame's
# coverage (K = 5, the rest -1)
HAND = [[0, 1, 2, 3, 4, 5], [3, 4, 5, 6, 7, 8], [5, 9, 10, 11, 12, 13], [14, 15, 16, 17, 0, 1]]
TABLES = [
    ("24 frames, one window", 24, 24, lambda: uniform_windows(24, 24), None),
    ("48 frames, context 24", 48, 24, lambda: uniform_windows(48, 24), None),
    ("30 frames, context 8", 30, 8, lambda: uniform_windows(30, 8), None),
    ("hand-built, a frame in 3 windows, K = 5", 18, 6, lambda: HAND, 5),
]


@pytest.mark.parametrize("prediction", [0, 1], ids=["v_prediction", "epsilon"])
@pytest.mark.parametrize("cfg", [True, False], ids=["cfg", "no-cfg"])
@pytest.mark.parametrize("Bl", [1, 2])
@pytest.mark.parametrize("device_index", [True, False], ids=["step_index", "step_index NULL"])
@pytest.mark.parametrize("label,Ftot,Fw,make_windows,K", TABLES, ids=[t[0] for t in TABLES])
def test_window_gather_and_cfg_ddim_step(label, Ftot, Fw, make_windows, K, device_index, Bl, cfg, prediction):
    windows = make_windows()
    Cc, H, W = 4, 9, 7
    HW = H * W
    steps = 3
    s = 3.5
    R = 2 if cfg else 1
    coef = coef_table(steps, prediction)
    inv = inverse_map(windows, Ftot, K)
    assert K is None or int((inv >= 0).sum(1).max()) < inv.shape[1]
    check_step_tables(inv, len(windows), Fw)
    inv_dev, coef_dev = inv.cuda(), coef.cuda()
    step_dev = torch.zeros(1, dtype=I32, device="cuda") if device_index else None
    g = torch.Generator(device="cuda").manual_seed(Ftot * 10 + Bl)
    lat_g = Guarded(Bl * Cc * Ftot, HW)
    lat_g.out.copy_((torch.randn(Bl * Cc * Ftot, HW, generator=g, device="cuda")).half())
    lat = lat_g.out.view(Bl, Cc, Ftot, HW)
    for step in range(steps):
        row = step if device_index else 0
        check_step_tables(inv, len(windows), Fw, step_index=row, coef_rows=coef.shape[0])
        if device_index:
            assert int(step_dev.item()) == step
        preds = []
        lat_before = bits(lat).clone()
        for w, win in enumerate(windows):
            idx = torch.tensor(win, dtype=I32)
            check_step_tables(inv, len(windows), Fw, frame_idx=idx, Ftot=Ftot)
            idx_dev = idx.cuda()
            out = Guarded(R * Bl * Cc * Fw, HW)
            op_window_gather(lat, idx_dev, out.out, Bl, Cc, Ftot, Fw, HW, R)
            torch.cuda.synchronize()
            out.check_untouched(torch.ones(out.rows, HW, dtype=torch.bool, device="cuda"), f"window_gather {label} window {w}")
            ref = lat[:, :, win].repeat(R, 1, 1, 1).reshape(out.rows, HW)
            assert torch.equal(bits(out.out), bits(ref)), f"window_gather {label} window {w}: differs"
            assert torch.equal(bits(lat), lat_before) and torch.equal(bits(idx_dev), bits(idx.cuda())), "window_gather modified an input"
            # stand-in for the UNet's output on this window: (R * Bl, C, Fw, HW), the CFG halves in one allocation
            preds.append(torch.randn(R * Bl, Cc, Fw, HW, generator=g, device="cuda").half() * (1 + w))
        ins = preds + [inv_dev, coef_dev]
        before = [bits(t) for t in ins]
        ref, E = step_ref_and_E(lat, preds, windows, Bl, s, cfg, coef[row], prediction)
        op_cfg_ddim_step([p for p in preds], [p[Bl:] for p in preds] if cfg else None, inv_dev, coef_dev, step_dev, lat, Bl, Cc, Ftot, Fw, HW, s,
                         prediction)
        if device_index:
            op_advance_index(step_dev)
        torch.cuda.synchronize()
        lat_g.check_untouched(torch.ones(lat_g.rows, HW, dtype=torch.bool, device="cuda"), f"cfg_ddim_step {label}")
        check_inputs_unchanged(before, ins, f"cfg_ddim_step {label}")
        fam = ("v_prediction" if prediction == 0 else "epsilon") + (", cfg" if cfg else ", no cfg")
        judge(fam, f"cfg_ddim_step {label} step {step}", lat, ref, E)
    if device_index:
        assert int(step_dev.item()) == steps


def test_advance_index_counts():
    idx = torch.tensor([7, -1], dtype=I32, device="cuda")
    for _ in range(5):
        op_advance_index(idx)
    torch.cuda.synchronize()
    assert idx.tolist() == [12, -1], "advance_index must add 1 to the first int32 only"
