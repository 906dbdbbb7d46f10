"""Per-layer error ladder at BASELINE config 2 (or any shape): after every resnet / transformer / motion module / sampler of the
denoising UNet, the relative L2 error of

    native (libhv_b200, fp16 storage, fp32 epilogues)   vs  the oracle in fp32
    the oracle in fp16 eager (the reference's deployment) vs  the oracle in fp32
    native                                               vs  the oracle in fp16 eager

on identical latents / timestep / conditioning.  Native activations come from the debug taps of the C ABI
(hv_debug_set_taps); oracle activations from forward hooks on the modules of the same name.

    python scripts/error_ladder.py [--out gpurun_out/error_ladder.txt] [--hw 96 72] [--frames 24] [--banks 0|1] [--narrow]
"""
import argparse
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import humanvid_b200 as hv  # noqa: E402
from oracle import hv_oracle as O  # noqa: E402
from oracle.block_replay import replay_blocks, to_nhwc  # noqa: E402

MM_KW = dict(num_attention_heads=8, num_transformer_block=1, attention_block_types=["Temporal_Self", "Temporal_Self"],
             temporal_position_encoding=True, temporal_position_encoding_max_len=32, temporal_attention_dim_div=1)


def rel(a, b):
    a, b = a.float(), b.float()
    return float((a - b).norm() / (b.norm() + 1e-20))


def run_oracle(ora, names, x, t, ehs, pose, visit):
    """Forward with hooks; visit(name, activation as (NF,H,W,C)) in execution order."""
    mods = dict(ora.named_modules())
    handles = []
    for n in names:
        if n == "conv_in":
            handles.append(mods[n].register_forward_hook(lambda m, i, o, n=n: visit(n, to_nhwc(o + pose.to(o.dtype)))))
        else:
            handles.append(mods[n].register_forward_hook(lambda m, i, o, n=n: visit(n, to_nhwc(o[0] if isinstance(o, tuple) else o))))
    with torch.no_grad():
        y = ora(x, torch.tensor(t, device=x.device), ehs, pose_cond_fea=pose)[0]
    for h in handles:
        h.remove()
    return y


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default="gpurun_out/error_ladder.txt")
    ap.add_argument("--hw", type=int, nargs=2, default=[96, 72])
    ap.add_argument("--frames", type=int, default=24)
    ap.add_argument("--banks", type=int, default=0)
    ap.add_argument("--narrow", action="store_true")
    ap.add_argument("--timestep", type=int, default=519)
    a = ap.parse_args()
    H, W = a.hw
    F = a.frames
    chs, xdim = ((64, 128, 256, 256), 64) if a.narrow else ((320, 640, 1280, 1280), 768)
    dev = "cuda"
    ora = O.UNet3DConditionModel(block_out_channels=chs, cross_attention_dim=xdim).eval()
    O.synthetic_init(ora, seed=7)
    ora = ora.half().to(dev)
    nat = hv.UNet3DConditionModel(block_out_channels=chs, cross_attention_dim=xdim, use_motion_module=True, use_inflated_groupnorm=True,
                                  motion_module_resolutions=(1, 2, 4, 8), motion_module_mid_block=True, motion_module_type="Vanilla",
                                  motion_module_kwargs=MM_KW, unet_use_cross_frame_attention=False, unet_use_temporal_attention=False)
    nat.load_state_dict(ora.state_dict())
    nat = nat.to(dev, torch.float16)
    g = torch.Generator(device=dev).manual_seed(42)
    x = torch.randn(2, 4, F, H, W, generator=g, device=dev).half()
    ehs = torch.randn(2, 1, xdim, generator=g, device=dev).half()
    ehs[:1] = 0
    pose = (torch.randn(2, chs[0], F, H, W, generator=g, device=dev) * 0.5).half()
    if a.banks:
        banks = [torch.randn(2, l, c, generator=g, device=dev).half() for (l, c) in O.bank_shapes(ora, H, W)]
        hv.ReferenceAttentionControl(nat, do_classifier_free_guidance=True, mode="read", fusion_blocks="full")
        for blk, bk in zip(nat.reader_blocks(), banks):
            blk.bank = [bk]
        O.set_reference_banks(ora, banks, cfg=True)

    plan = nat.debug_tap_plan(2, F, H, W)
    taps = [torch.empty(d, device=dev, dtype=torch.float16) for _, d in plan]
    nat.debug_set_taps(taps)
    with torch.no_grad():
        yn = nat(x, a.timestep, ehs, pose_cond_fea=pose, return_dict=False)[0]
    torch.cuda.synchronize()
    nat.debug_set_taps([])
    names = [n for n, _ in plan]
    native = dict(zip(names, taps))

    # fp16 eager first (keeps fp16 copies), then fp32: errors of both against fp32 are formed inside the fp32 pass
    eager = {}
    y16 = run_oracle(ora, names, x, a.timestep, ehs, pose, lambda n, t: eager.__setitem__(n, t.contiguous()))
    ora.float()
    if a.banks:
        O.set_reference_banks(ora, [b.float() for b in banks], cfg=True)
    rows = []

    def visit32(n, t32):
        rows.append((n, tuple(t32.shape), rel(native[n], t32), rel(eager[n], t32), rel(native[n], eager[n])))

    y32 = run_oracle(ora, names, x.float(), a.timestep, ehs.float(), pose.float(), visit32)
    rows.append(("conv_out (network output)", tuple(y32.shape), rel(yn, y32), rel(y16, y32), rel(yn, y16)))

    # ---- isolated per-block error: the oracle's block in fp32 applied to the NATIVE block's own input (the native taps of its
    # predecessors), against the native block's output -- "identical inputs, per tensor" (north_star), free of the error the input
    # already carried.  The banks set above are the oracle's fp32 banks, so the replay reads them as the whole forward did.
    iso = {}
    for n, out in replay_blocks(ora, names, native, x, a.timestep, ehs, pose):
        iso[n] = rel(native[n], out)
        del out

    os.makedirs(os.path.dirname(a.out) or ".", exist_ok=True)
    with open(a.out, "w") as f:
        f.write(f"# error ladder: latent {H}x{W}, {F} frames, CFG batch 2, widths {chs}, banks={a.banks}, timestep {a.timestep}, seed-7 synthetic init\n")
        f.write("# relative L2 error of the activation leaving each block (channels-last (NF,H,W,C))\n")
        f.write("# isolated = the oracle's block in fp32 applied to the native block's OWN input (native taps) vs the native block's output\n")
        f.write(f"# {'block':38s} {'shape':>22s} {'native/fp32':>12s} {'eager16/fp32':>13s} {'native/eager16':>15s} {'isolated':>10s}\n")
        for n, s, e1, e2, e3 in rows:
            f.write(f"{n:40s} {str(s):>22s} {e1:12.3e} {e2:13.3e} {e3:15.3e} " + (f"{iso[n]:10.3e}" if n in iso else f"{'-':>10s}") + "\n")
        if iso:
            wi = max(iso.items(), key=lambda kv: kv[1])
            f.write(f"# max isolated per-block error: {wi[1]:.3e} at {wi[0]}\n")
        worst = max(rows, key=lambda r: r[2])
        f.write(f"# max native/fp32 over the ladder: {worst[2]:.3e} at {worst[0]}; network output: native/fp32 {rows[-1][2]:.3e}, "
                f"eager16/fp32 {rows[-1][3]:.3e}, native/eager16 {rows[-1][4]:.3e}\n")
    print(open(a.out).read()[-1200:])


if __name__ == "__main__":
    main()
