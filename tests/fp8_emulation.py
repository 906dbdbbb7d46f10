"""The FP8 (e4m3) quantisation scheme of the FP8 linears (DESIGN.md §9) in PyTorch, on CPU or GPU: the reference the kernels' bytes and
scales are checked against.

For a row, or a block of `block` columns of a row, with absolute maximum amax (all fp32, each step one IEEE operation):
    inv = 448 / amax,  q = e4m3(x * inv) (round to nearest even, saturating),  s = amax / 448
and amax == 0 gives inv = 0, s = 0 and zero bytes.  The value a byte stands for is q * s."""
import torch

E4M3_MAX = 448.0
E4M3 = torch.float8_e4m3fn


def _blocks(x, block):
    """[..., K] -> [..., nb, block] (the last block zero-padded when block does not divide K)."""
    K = x.shape[-1]
    nb = (K + block - 1) // block
    if nb * block != K:
        x = torch.nn.functional.pad(x, (0, nb * block - K))
    return x.reshape(*x.shape[:-1], nb, block), K


def quantize(x, block=None):
    """fp32 x [..., K] -> (q float8_e4m3fn [..., K], s fp32 [...] per row, or [..., ceil(K / block)] per block of `block` columns)."""
    x = x.float()
    xb, K = _blocks(x, block) if block else (x.unsqueeze(-2), x.shape[-1])
    amax = xb.abs().amax(-1, keepdim=True)
    # tensor / tensor: PyTorch turns a division by a Python scalar into a multiplication by its reciprocal on CUDA, which is not the
    # IEEE division the kernels do
    c448 = torch.full_like(amax, E4M3_MAX)
    inv = torch.where(amax > 0, c448 / amax, torch.zeros_like(amax))
    # clamp-then-round equals the kernels' saturating round: every fp32 value above 448 lies above the e4m3 midpoint 464 or rounds to 448
    q = (xb * inv).clamp(-E4M3_MAX, E4M3_MAX).to(E4M3)
    s = (amax / c448).squeeze(-1)
    q = q.reshape(*x.shape[:-1], -1)[..., :K].contiguous()
    return q, (s if block else s.squeeze(-1))


def dequantize(q, s, block=None):
    """q [..., K] e4m3 with per-row s [...] or per-block s [..., nb] -> fp32."""
    v = q.float()
    if not block:
        return v * s.unsqueeze(-1)
    vb, K = _blocks(v, block)
    return (vb * s.unsqueeze(-1)).reshape(*v.shape[:-1], -1)[..., :K]


def qdq(x, block=None):
    """Quantise then dequantise: the value the FP8 path computes with in place of x."""
    q, s = quantize(x, block)
    return dequantize(q, s, block)


def half_step(v, s):
    """Half the e4m3 spacing at the magnitude of the dequantised value v with scale s: 2^(e - 4) for a normal value in [2^e, 2^(e+1))
    (3 mantissa bits), and 2^-10 below 2^-6 (the subnormal spacing 2^-9), both times s."""
    a = (v / torch.where(s > 0, s, torch.ones_like(s))).abs()
    e = torch.floor(torch.log2(torch.clamp(a, min=2.0 ** -6)))
    return torch.exp2(e - 4) * s


def _ff_emulated(ff, x):
    """oracle FeedForward (GEGLU proj -> Linear) with e4m3 quantise-dequantise at the FP8 path's points: the LayerNorm output per token,
    the weights per row, the GEGLU output per (token, 128 columns).  The scales and e4m3 values are formed in fp32 as the kernels form them;
    the arithmetic between the quantisation points runs in x's dtype (fp32, or fp64 for a reference of the emulation)."""
    proj, lin2 = ff.net[0].proj, ff.net[2]
    h = torch.nn.functional.linear(qdq(x).to(x.dtype), qdq(proj.weight).to(x.dtype), proj.bias)
    hidden, gate = h.chunk(2, dim=-1)
    y = qdq(hidden * torch.nn.functional.gelu(gate), 128).to(x.dtype)
    return torch.nn.functional.linear(y, qdq(lin2.weight).to(x.dtype), lin2.bias)


def ff_flip_bound(ff, x):
    """Per output element of the emulated FeedForward on x, the most that flipped e4m3 roundings of its GEGLU output can move it.

    The native FP8 path quantises a GEGLU output that carries the fp16 path's error; where that error carries a value across an e4m3
    rounding midpoint, the value lands one e4m3 spacing (two half_steps) from the emulation's.  Through ff2 this moves output i by at most
    sum_j |W2[i, j]| 2 half_step(y_j): the bound for every value of the row flipping at once."""
    proj, lin2 = ff.net[0].proj, ff.net[2]
    h = torch.nn.functional.linear(qdq(x).to(x.dtype), qdq(proj.weight).to(x.dtype), proj.bias)
    hidden, gate = h.chunk(2, dim=-1)
    v = hidden * torch.nn.functional.gelu(gate)
    q, s = quantize(v, 128)
    y = dequantize(q, s, 128)
    step = 2 * half_step(y, s.repeat_interleave(128, dim=-1)[..., : v.shape[-1]])
    return torch.nn.functional.linear(step.to(x.dtype), qdq(lin2.weight).to(x.dtype).abs())


class emulate_fp8_linears:
    """Context manager: the oracle UNet (fp32, or fp64) with the FP8 mode's quantisation inserted in the feed-forwards FP8 mode runs on e4m3 (those
    of width >= min_dim; the LayerNorm in front of each is the caller of FeedForward, so quantising its input is quantising the LayerNorm's
    output)."""

    def __init__(self, unet, min_dim=1280):
        self.mods = [m for m in unet.modules() if type(m).__name__ == "FeedForward" and m.net[0].proj.in_features >= min_dim]

    def __enter__(self):
        for m in self.mods:
            m.forward = (lambda mod: (lambda x: _ff_emulated(mod, x)))(m)
        return self

    def __exit__(self, *a):
        for m in self.mods:
            del m.forward
