"""Times humanvid_b200.CLIPVisionModelWithProjection (the native image encoder) against transformers' CLIPVisionModelWithProjection in fp16
eager (SDPA) on the same GPU, and prints one JSON line.

    python scripts/clip_bench.py [--iters N] [--warmup W] [--rounds R]

Workload: ViT-L/14 at 224 x 224 (hidden 1024, 24 layers, 16 heads, MLP 4096, projection 768; random init rounded to fp16), batches of 1 and
2 images.  Three arms run in one process, alternating round by round: the native encoder called eagerly, the native encoder replayed from a
CUDA graph (static buffers, captured once per batch size), and transformers in fp16.  Each figure is the median over all rounds of CUDA-event
times of single calls.  Accuracy is the relative L2 error of image_embeds and last_hidden_state against transformers in fp32 (TF32 off).
The algorithmic work per image is computed from the shapes (clip_flops), not measured.  The card's name, power limit and clocks are read
with nvidia-smi during the timed rounds (bench.ClockSampler).
"""
from __future__ import annotations

import argparse
import ctypes as C
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

VIT_L14 = dict(hidden_size=1024, intermediate_size=4096, projection_dim=768, num_hidden_layers=24, num_attention_heads=16, image_size=224,
               patch_size=14)


def clip_flops(B, hidden_size, intermediate_size, projection_dim, num_hidden_layers, image_size, patch_size, num_channels=3, **_):
    """2 x multiply-adds of one forward over B images: the patch conv, per layer q / k / v / out (4 h^2 per token), the MLP (2 h I per
    token; 12 h^2 at I = 4h) and attention (QK^T and PV: 2 L^2 h), and the projection of the class token."""
    L = (image_size // patch_size) ** 2 + 1
    patch = (L - 1) * hidden_size * num_channels * patch_size ** 2
    per_layer = L * (4 * hidden_size ** 2 + 2 * hidden_size * intermediate_size) + 2 * L * L * hidden_size
    return 2.0 * B * (patch + num_hidden_layers * per_layer + hidden_size * projection_dim)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20, help="timed calls per arm and round")
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()

    import torch

    if not torch.cuda.is_available():
        raise SystemExit("clip_bench.py needs a CUDA device")
    import transformers

    import bench
    import humanvid_b200 as hv
    from humanvid_b200 import _native as N

    dev = "cuda"
    name = subprocess.run(["nvidia-smi", "--query-gpu=name", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True).stdout.strip()
    torch.manual_seed(0)
    m32 = transformers.CLIPVisionModelWithProjection(transformers.CLIPVisionConfig(**VIT_L14, attn_implementation="eager")).eval()
    sd = {k: v.half().float() for k, v in m32.state_dict().items()}
    m32.load_state_dict(sd)
    m32 = m32.to(dev)
    m16 = transformers.CLIPVisionModelWithProjection(transformers.CLIPVisionConfig(**VIT_L14, attn_implementation="sdpa")).eval()
    m16.load_state_dict(sd)
    m16 = m16.half().to(dev)
    nat = hv.CLIPVisionModelWithProjection(**VIT_L14)
    nat.load_state_dict(sd)
    nat = nat.to(dev, torch.float16)
    h = nat._sync_native()

    batches = (1, 2)
    g = torch.Generator(device=dev).manual_seed(1)
    pix = {B: torch.randn(B, 3, 224, 224, generator=g, device=dev).half() for B in batches}
    res = {"gpu": name, "model": "ViT-L/14 @ 224", "iters": args.iters, "warmup": args.warmup, "rounds": args.rounds}

    # accuracy against fp32
    saved = torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = torch.backends.cudnn.allow_tf32 = False
    rel = lambda a, b: float((a.float() - b.float()).norm() / b.float().norm())
    with torch.no_grad():
        for B in batches:
            o32, o16, on = m32(pix[B].float()), m16(pix[B]), nat(pix[B])
            res[f"rel_l2_b{B}"] = {
                "native": {"image_embeds": rel(on.image_embeds, o32.image_embeds), "last_hidden_state": rel(on.last_hidden_state, o32.last_hidden_state)},
                "fp16_eager": {"image_embeds": rel(o16.image_embeds, o32.image_embeds), "last_hidden_state": rel(o16.last_hidden_state, o32.last_hidden_state)},
            }
    torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = saved
    del m32
    torch.cuda.empty_cache()

    # one CUDA graph per batch size around the C forward, static input / output buffers
    graphs = {}
    for B in batches:
        nat.reserve_workspace(B)
        emb = torch.empty(B, VIT_L14["projection_dim"], device=dev, dtype=torch.float16)
        hid = torch.empty(B, 257, VIT_L14["hidden_size"], device=dev, dtype=torch.float16)
        fwd = lambda B=B, emb=emb, hid=hid: N.check(N.lib().hv_clip_vision_forward(h, N.ptr(pix[B]), N.ptr(emb), N.ptr(hid), N.i32(B), None,
                                                                                    C.c_size_t(0), N.stream()), h)
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):
            fwd()
        torch.cuda.current_stream().wait_stream(s)
        gr = torch.cuda.CUDAGraph()
        with torch.cuda.graph(gr):
            fwd()
        graphs[B] = gr

    def times(fn):
        for _ in range(args.warmup):
            fn()
        out = []
        for _ in range(args.iters):
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            fn()
            b.record()
            b.synchronize()
            out.append(a.elapsed_time(b))
        return out

    arms = {"native_eager": lambda B: (lambda: nat(pix[B])), "native_graph": lambda B: graphs[B].replay, "transformers_fp16_sdpa": lambda B: (lambda: m16(pix[B]))}
    samples = {(a, B): [] for a in arms for B in batches}
    with torch.no_grad(), bench.ClockSampler(0) as clk:
        for _ in range(args.rounds):
            for B in batches:
                for a, make in arms.items():
                    samples[(a, B)] += times(make(B))
    for B in batches:
        fl = clip_flops(B, **VIT_L14)
        res[f"b{B}"] = {"gflop": round(fl / 1e9, 1)}
        for a in arms:
            ms = statistics.median(samples[(a, B)])
            res[f"b{B}"][a] = {"ms": round(ms, 3), "tflops": round(fl / ms / 1e9, 1)}
    nat(pix[1])
    res["native_launches_b1"] = nat.last_launch_count
    res["clocks"] = clk.summary()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
