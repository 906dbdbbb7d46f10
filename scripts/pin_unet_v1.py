"""Pin the inference_v1 oracle (tests/unet_v1_oracle.py) against the reference's OWN UNet3DConditionModel and write
tests/golden/unet_narrow_v1.pt.

    python scripts/pin_unet_v1.py [--reference /path/to/HumanVid]

The reference model is built with inference_v1.yaml's unet_additional_kwargs at narrow channels, takes the oracle's synthetic weights
(every key must match both ways) and runs on the CPU in fp32 at F = 4 with frames whose values drift away from frame 0.  The oracle
must reproduce it bit for bit; the script fails otherwise.  The other goldens (oracle/pin_against_reference.py) are not touched.
"""
import argparse
import contextlib
import io
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

from oracle import hv_oracle as O  # noqa: E402
from oracle import pin_against_reference as P  # noqa: E402
from unet_v1_oracle import V1_UNET_KWARGS, unet3d_v1  # noqa: E402

CHS, XDIM, SEED, B, F, HW, T = (32, 64, 128, 128), 64, 7, 2, 4, 16, 721


def inputs():
    g = torch.Generator().manual_seed(3)
    x = torch.randn(B, 4, F, HW, HW, generator=g)
    x = x + 0.75 * torch.arange(F).view(1, 1, F, 1, 1)   # frames drift away from frame 0: pooled statistics differ from per-frame ones
    ehs = torch.randn(B, 1, XDIM, generator=g)
    pose = torch.randn(B, CHS[0], F, HW, HW, generator=g) * 0.5
    return x, ehs, pose


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reference", default=P.REF)
    args = ap.parse_args()
    P.REF = args.reference
    P.install_stubs()
    from src.models.unet_3d import UNet3DConditionModel as RefUNet

    ref = RefUNet(in_channels=4, out_channels=4, block_out_channels=CHS, cross_attention_dim=XDIM, attention_head_dim=8, **V1_UNET_KWARGS).eval()
    ora = O.synthetic_init(unet3d_v1(CHS, XDIM).eval(), seed=SEED)
    sd = ora.state_dict()
    missing, unexpected = ref.load_state_dict(sd, strict=False)
    assert not missing and not unexpected, (missing[:5], unexpected[:5])
    assert set(ref.state_dict()) == set(sd)
    assert not any(k.startswith("mid_block.motion_modules") for k in sd)
    x, ehs, pose = inputs()
    t = torch.tensor(T)
    with contextlib.redirect_stdout(io.StringIO()), torch.no_grad():   # the reference print()s in forward
        y_ref = ref(x, t, ehs, pose_cond_fea=pose, return_dict=False)[0]
    with torch.no_grad():
        y_ora = ora(x, t, ehs, pose_cond_fea=pose)[0]
    d = float((y_ref.double() - y_ora.double()).abs().max())
    print(f"unet_narrow_v1: max |reference - oracle| = {d}")
    if d != 0.0:
        raise SystemExit("the inference_v1 oracle does not reproduce the reference bit for bit")
    torch.save(dict(chs=CHS, xdim=XDIM, seed=SEED, x=x, ehs=ehs, pose=pose, t=T, y=y_ref, max_abs_diff=d),
               os.path.join(ROOT, "tests", "golden", "unet_narrow_v1.pt"))


if __name__ == "__main__":
    main()
