"""fp64 references and per-element error bounds of the GroupNorm kernels (hv_op_groupnorm, hv_op_groupnorm_pooled), shared by the tests
of both operators.  The derivation is in the docstring of test_groupnorm_pooled_gpu.py; hv_op_groupnorm is the pooled operator at F = 1."""
import torch

U = 2.0 ** -24


def gam(k, u=U):
    return k * u / (1 - k * u)


def chain_depth(Ct, HW, F, groups):
    """Longest chain of fp32 additions behind one (item, group) sum, from the launch plan of norm.cu (gn_plan)."""
    vecs = Ct // 8
    t = vecs * (1 if vecs >= 256 else 256 // vecs)
    if t > 1024:
        t = vecs
    rpi = t // vecs
    rpb = max(32, -(-HW // 16))
    slabs = -(-HW // rpb)
    cpg = Ct // groups
    rows = -(-rpb // rpi) + 1                      # per-thread row loop, each row adding a (d0 + d1) pair
    block = rpi * cpg // 2                         # the block's slot loop for one group
    combine = max(-(-F * slabs // 128) + 7, -(-slabs // 4) + 2)   # finalize (strided loop + tree) or the per-frame 4-lane fold
    return rows + block + combine


def groupnorm_ref_and_bound(x, gamma, beta, F, groups, eps, silu):
    """x: fp16 (NF, HW, C), frames [b*F, (b+1)*F) pooled.  Returns the fp64 reference and the per-element bound, both (NF, HW, C)."""
    NF, HW, Ct = x.shape
    cpg, B, N = Ct // groups, NF // F, F * HW * (Ct // groups)
    xd = x.double().view(B, F, HW, groups, cpg)
    p = xd[:, 0, 0, :, 0]                                              # (B, G) the kernel's pivot
    d = xd - p[:, None, None, :, None]
    A, Q = d.abs().sum((1, 2, 4)) / N, (d * d).sum((1, 2, 4)) / N      # per (item, group), divided by N
    mp = d.sum((1, 2, 4)) / N
    del d
    mean = p + mp
    var = (Q - mp * mp).clamp_min(0)
    rstd = 1.0 / torch.sqrt(var + eps)
    D = chain_depth(Ct, HW, F, groups)
    e_mp = gam(D + 1) * A + 2 * U * mp.abs()
    e_mean = e_mp + U * mean.abs()
    e_var = gam(D + 3) * Q + 2 * mp.abs() * e_mp + e_mp ** 2 + 4 * U * (Q + mp * mp)
    rel_rstd = e_var / (2 * (var + eps)) * (1 + e_var / (var + eps)) + 2.0 ** -22 + U
    gm, bt = gamma.double().view(groups, cpg), beta.double().view(groups, cpg)
    bc = lambda t: t[:, None, None, :, None]
    sc = bc(rstd) * gm
    sh = bt - bc(mean) * sc
    yr = (xd - bc(mean)) * sc + bt
    dy = (xd - bc(mean)).abs() * gm.abs() * bc(rstd) * (bc(rel_rstd) + U) + sc.abs() * bc(e_mean) + U * (sh.abs() + yr.abs())
    if silu:
        s = yr * torch.sigmoid(yr)
        dy = 1.1 * dy + silu_error(yr)
        yr = s
    bound = 2.0 ** -11 * (yr.abs() + dy) + dy + 2.0 ** -25
    return yr.view(NF, HW, Ct), bound.view(NF, HW, Ct)


def silu_error(y):
    """fp32 error of silu_f(y) = __fdividef(y, 1 + __expf(-y)) (ptx.cuh) beyond the error already in y: (5 + 1.2 |y|) 2^-23 |silu(y)|."""
    return (5 + 1.2 * y.abs()) * 2.0 ** -23 * (y * torch.sigmoid(y)).abs()
