"""humanvid_b200.AutoencoderKL on an H100: the d = 512 single-head attention op, the end-padded stride-2 conv op, decode / encode parity
against the PyTorch restatement (tests/vae_oracle.py) in fp32 and in fp16 eager, determinism, frame independence, CUDA-graph capture and
the Pose2VideoPipeline decode path.  Weights are random (oracle.synthetic_init), rounded to fp16 so every arm sees the same values."""
import ctypes as C
from types import SimpleNamespace

import pytest
import torch
import torch.nn as nn
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

from conftest import report

if torch.cuda.is_available():
    import humanvid_b200 as hv
    from humanvid_b200._native import Epilogue, check, i32, i64, lib, ptr, stream
    from oracle import hv_oracle as O
    import vae_oracle as V


def rel(a, b):
    a, b = a.float(), b.float()
    return float((a - b).norm() / (b.norm() + 1e-12))


@pytest.fixture
def exact_fp32():
    """The fp32 oracle runs in true fp32 (no TF32 convolutions / matmuls)."""
    saved = torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32
    torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False
    yield
    torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = saved


@pytest.fixture(scope="module")
def vaes():
    ora = O.synthetic_init(V.AutoencoderKL().eval(), seed=21).half().float().cuda()
    o16 = V.AutoencoderKL().eval()
    o16.load_state_dict(ora.state_dict())
    o16 = o16.half().cuda()
    nat = hv.AutoencoderKL()
    nat.load_state_dict(ora.state_dict())
    nat = nat.to("cuda", torch.float16)
    return ora, o16, nat


# ------------------------------------------------------------------------------------------------ operators
@pytest.mark.parametrize("L", [81, 960, 6912, 9216])
def test_attention_d512_op(L):
    NF, D = 2, 512
    g = torch.Generator(device="cuda").manual_seed(L)
    qk = torch.randn(NF * L, 2 * D, generator=g, device="cuda").half()       # [Q | K] per token, as the bias GEMM writes them
    v = torch.randn(NF, L, D, generator=g, device="cuda").half()
    Lp = (L + 7) // 8 * 8
    vt = torch.full((D, NF * Lp), float("nan"), device="cuda", dtype=torch.float16)   # pad columns must never be read
    for n in range(NF):
        vt[:, n * Lp : n * Lp + L] = v[n].t()
    out = torch.empty(NF * L, D, device="cuda", dtype=torch.float16)
    check(lib().hv_op_attention_d512(ptr(qk), i64(2 * D), C.c_void_p(qk.data_ptr() + 2 * D), i64(2 * D), ptr(vt), i64(NF * Lp), i64(Lp),
                                     ptr(out), i64(D), i64(NF), i64(L), stream()))
    q, k = qk[:, :D].float().view(NF, L, D), qk[:, D:].float().view(NF, L, D)
    ref = torch.softmax(q @ k.transpose(1, 2) / D ** 0.5, dim=-1) @ v.float()
    e = rel(out.view(NF, L, D), ref)
    report(f"attention d512 op NF={NF} L={L}: rel vs fp32 {e:.2e}")
    assert torch.isfinite(out).all() and e <= 1e-3


def test_attention_d512_op_rejects_bad_shapes():
    x = torch.zeros(64, 1024, device="cuda", dtype=torch.float16)
    vt = torch.zeros(512, 64, device="cuda", dtype=torch.float16)
    assert lib().hv_op_attention_d512(ptr(x), i64(1024), ptr(x), i64(1024), ptr(vt), i64(64), i64(60), ptr(x), i64(512), i64(1), i64(60), stream()) != 0
    assert lib().hv_op_attention_d512(ptr(x), i64(1024), ptr(x), i64(1024), ptr(vt), i64(64), i64(64), ptr(x), i64(512), i64(0), i64(64), stream()) != 0


@pytest.mark.parametrize("NF, H, W, Cin, Cout", [(2, 48, 40, 128, 128), (1, 24, 16, 256, 256), (3, 12, 18, 512, 512)])
def test_conv3x3_s2_pad_end_op(exact_fp32, NF, H, W, Cin, Cout):
    g = torch.Generator(device="cuda").manual_seed(H * W + Cin)
    x = torch.randn(NF, Cin, H, W, generator=g, device="cuda").half()
    w = (torch.randn(Cout, Cin, 3, 3, generator=g, device="cuda") / (9 * Cin) ** 0.5).half()
    b = (torch.randn(Cout, generator=g, device="cuda") * 0.1).half()
    xc = x.permute(0, 2, 3, 1).contiguous()
    wp = torch.empty(Cout, 9 * Cin, device="cuda", dtype=torch.float16)
    check(lib().hv_pack_conv3x3(ptr(w), ptr(wp), i64(Cout), i64(Cin), i64(Cout), i64(Cin), stream()))
    out = torch.empty(NF, H // 2, W // 2, Cout, device="cuda", dtype=torch.float16)
    ep = Epilogue(bias=ptr(b).value)
    check(lib().hv_op_conv3x3_s2_pad_end(ptr(xc), ptr(wp), ptr(out), i64(Cout), i64(NF), i64(H), i64(W), i64(Cin), i64(Cout), C.byref(ep), stream()))
    ref = F.conv2d(F.pad(x.float(), (0, 1, 0, 1)), w.float(), b.float(), stride=2)
    e = rel(out.permute(0, 3, 1, 2), ref)
    report(f"conv3x3 s2 pad-end op {NF}x{Cin}x{H}x{W} -> {Cout}: rel vs fp32 {e:.2e}")
    assert e <= 1e-3


# ------------------------------------------------------------------------------------------------ network
@pytest.mark.parametrize("N, h, w", [(3, 32, 32), (8, 96, 72)])
def test_decode_parity(vaes, exact_fp32, N, h, w):
    ora, o16, nat = vaes
    g = torch.Generator(device="cuda").manual_seed(h * w + N)
    z = torch.randn(N, 4, h, w, generator=g, device="cuda").half()
    with torch.no_grad():
        yn = nat.decode(z).sample
        y16 = o16.decode(z).sample
        y32 = ora.decode(z.float()).sample
    torch.cuda.synchronize()
    assert yn.shape == (N, 3, 8 * h, 8 * w) and yn.dtype == torch.float16
    e_nat, e_ref = rel(yn, y32), rel(y16, y32)
    per_frame = [rel(yn[i], y32[i]) for i in range(N)]
    report(f"vae decode N={N} latent {h}x{w}: native vs fp32 {e_nat:.2e}; fp16-eager vs fp32 {e_ref:.2e}; per-frame max {max(per_frame):.2e}")
    assert torch.isfinite(yn).all()
    assert e_nat <= e_ref
    assert max(per_frame) <= 3 * (sum(per_frame) / N)


@pytest.mark.parametrize("H, W", [(768, 576), (576, 1024)])
def test_encode_parity(vaes, exact_fp32, H, W):
    ora, o16, nat = vaes
    g = torch.Generator(device="cuda").manual_seed(H + W)
    x = (torch.rand(1, 3, H, W, generator=g, device="cuda") * 2 - 1).half()
    with torch.no_grad():
        mn = nat.encode(x).latent_dist.mean
        m16 = o16.encode(x).latent_dist.mean
        m32 = ora.encode(x.float()).latent_dist.mean
        (dist,) = nat.encode(x, return_dict=False)
    torch.cuda.synchronize()
    assert mn.shape == (1, 4, H // 8, W // 8) and torch.equal(dist.mean, mn)
    e_nat, e_ref = rel(mn, m32), rel(m16, m32)
    report(f"vae encode 1x3x{H}x{W}: native vs fp32 {e_nat:.2e}; fp16-eager vs fp32 {e_ref:.2e}")
    assert torch.isfinite(mn).all() and e_nat <= e_ref


def test_determinism_frame_independence_graph_and_profile(vaes):
    _, _, nat = vaes
    g = torch.Generator(device="cuda").manual_seed(5)
    z = torch.randn(3, 4, 32, 32, generator=g, device="cuda").half()
    with torch.no_grad():
        a = nat.decode(z).sample
        b = nat.decode(z).sample
        assert torch.equal(a, b)
        for i in range(3):
            assert torch.equal(nat.decode(z[i : i + 1]).sample[0], a[i]), i
        # float32 in -> float32 out (the dtype follows the input), same values
        assert torch.equal(nat.decode(z.float()).sample, a.float())
        # CUDA graph: the forward never allocates or synchronises once the workspace is reserved
        nat.reserve_workspace(3, 32, 32)
        zs = z.clone()
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):
            nat.decode(zs)
        torch.cuda.current_stream().wait_stream(s)
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            yg = nat.decode(zs).sample
        zs.copy_(torch.randn(3, 4, 32, 32, generator=g, device="cuda").half())
        graph.replay()
        torch.cuda.synchronize()
        assert torch.equal(yg, nat.decode(zs).sample)
        zs.copy_(z)
        graph.replay()
        torch.cuda.synchronize()
        assert torch.equal(yg, a)
        # launch count and profile categories: GEMMs 0, convs 1, attention 2 (one per decode), norms 4
        h = nat._sync_native()
        assert nat.last_launch_count > 50
        check(lib().hv_set_profiling(h, i32(1)), h)
        nat.decode(z)
        ms, fl = (C.c_double * 6)(), (C.c_double * 6)()
        cnt = (C.c_int64 * 6)()
        check(lib().hv_get_profile(h, ms, fl, cnt, i32(6)), h)
        check(lib().hv_set_profiling(h, i32(0)), h)
    assert cnt[2] == 1 and cnt[0] > 0 and cnt[1] > 0 and cnt[4] > 0 and cnt[3] == 0
    assert fl[2] == 4.0 * 3 * (32 * 32) ** 2 * 512 and ms[2] > 0


def test_bad_shapes_raise(vaes):
    _, _, nat = vaes
    with pytest.raises(ValueError):
        nat.encode(torch.zeros(1, 3, 100, 64, device="cuda", dtype=torch.float16))
    with pytest.raises(ValueError):
        nat.decode(torch.zeros(1, 3, 8, 8, device="cuda", dtype=torch.float16))
    h = nat._sync_native()
    x = torch.zeros(1, 3, 64, 64, device="cuda", dtype=torch.float16)
    m = torch.zeros(1, 8, 8, 8, device="cuda", dtype=torch.float16)
    assert lib().hv_vae_encode(h, ptr(x), ptr(m), i32(1), i32(60), i32(64), None, C.c_size_t(0), stream()) == -1
    assert b"multiples of 8" in lib().hv_last_error(h)
    assert lib().hv_vae_decode(h, ptr(m), ptr(x), i32(0), i32(8), i32(8), None, C.c_size_t(0), stream()) == -1


# ------------------------------------------------------------------------------------------------ pipeline
class StubCLIP(nn.Module):
    def __init__(self, dim):
        super().__init__()
        self.lin = nn.Linear(3, dim)

    def forward(self, pix):
        return SimpleNamespace(image_embeds=self.lin(pix.float().mean((2, 3)).to(self.lin.weight.dtype)))


MM_KW = dict(num_attention_heads=8, num_transformer_block=1, attention_block_types=["Temporal_Self", "Temporal_Self"],
             temporal_position_encoding=True, temporal_position_encoding_max_len=32, temporal_attention_dim_div=1)


def test_pose2video_pipeline_with_native_vae(vaes, exact_fp32):
    from humanvid_b200.pipeline import Pose2VideoPipeline

    ora_vae, o16_vae, vae = vaes
    dev = "cuda"
    chs, xdim, Fv, H, W = (64, 128, 256, 256), 64, 24, 128, 128
    ora = O.synthetic_init(O.UNet3DConditionModel(block_out_channels=chs, cross_attention_dim=xdim).eval(), seed=7).half().float()
    unet = hv.UNet3DConditionModel(block_out_channels=chs, cross_attention_dim=xdim, use_motion_module=True, use_inflated_groupnorm=True,
                                   motion_module_resolutions=(1, 2, 4, 8), motion_module_mid_block=True, motion_module_type="Vanilla",
                                   motion_module_kwargs=MM_KW, unet_use_cross_frame_attention=False, unet_use_temporal_attention=False)
    unet.load_state_dict(ora.state_dict())
    pg = hv.PoseGuider(64, block_out_channels=(16, 32, 96, 256))
    pg.load_state_dict(O.synthetic_init(O.PoseGuider(64, 3, (16, 32, 96, 256)).eval(), seed=11).half().float().state_dict())
    cam = hv.CameraPoseEncoder(downscale_factor=8, channels=[64], nums_rb=2, cin=384, ksize=1, sk=True, use_conv=False, compression_factor=1,
                               temporal_attention_nhead=8, attention_block_types=["Temporal_Self"], temporal_position_encoding=True,
                               temporal_position_encoding_max_len=24)
    cam.load_state_dict(O.synthetic_init(O.CameraPoseEncoder(channels=(64,), heads=8).eval(), seed=13).half().float().state_dict())
    ref_unet = hv.UNet2DConditionModel(block_out_channels=chs, cross_attention_dim=xdim)
    ref_unet.load_state_dict(O.synthetic_init(O.UNet2DConditionModel(block_out_channels=chs, cross_attention_dim=xdim).eval(), seed=17).half().float().state_dict())
    sched = hv.DDIMScheduler(beta_start=0.00085, beta_end=0.012, beta_schedule="linear", clip_sample=False, steps_offset=1,
                             prediction_type="v_prediction", rescale_betas_zero_snr=True, timestep_spacing="trailing")
    pipe = Pose2VideoPipeline(vae=vae, image_encoder=StubCLIP(xdim), reference_unet=ref_unet, denoising_unet=unet, pose_guider=pg,
                              camera_pose_encoder=cam, scheduler=sched).to(dev, torch.float16)
    g = torch.Generator(device=dev).manual_seed(3)
    ref = torch.rand(3, H, W, generator=g, device=dev) * 2 - 1
    poses = [torch.rand(1, 3, H, W, generator=g, device=dev) for _ in range(Fv)]
    camera = torch.randn(1, 6, Fv, H, W, generator=g, device=dev).half()
    run = lambda out_type: pipe(ref, poses, camera, W, H, Fv, 1, 3.5, generator=torch.Generator(device=dev).manual_seed(7), output_type=out_type)
    lat = pipe(ref, poses, camera, W, H, Fv, 1, 3.5, generator=torch.Generator(device=dev).manual_seed(7), output_type="latent", return_dict=False)
    vid = run("tensor").videos
    assert vid.shape == (1, 3, Fv, H, W) and float(vid.min()) >= 0.0 and float(vid.max()) <= 1.0
    # the same latents through the oracle VAE (fp32 and fp16 eager), 8 frames per call like the pipeline
    z = (1 / 0.18215 * lat).permute(0, 2, 1, 3, 4).reshape(Fv, 4, H // 8, W // 8)
    with torch.no_grad():
        v32 = torch.cat([ora_vae.decode(z[i : i + 8].float()).sample for i in range(0, Fv, 8)])
        v16 = torch.cat([o16_vae.decode(z[i : i + 8].half()).sample for i in range(0, Fv, 8)])
    to_video = lambda y: (y.float().reshape(1, Fv, 3, H, W).permute(0, 2, 1, 3, 4) / 2 + 0.5).clamp(0, 1).cpu()
    vid_t = torch.as_tensor(vid).float().cpu()
    e_nat, e_ref = rel(vid_t, to_video(v32)), rel(to_video(v16), to_video(v32))
    report(f"pipeline 24 frames 128x128 with native VAE: video vs oracle fp32 decode {e_nat:.2e}; fp16-eager decode vs fp32 {e_ref:.2e}")
    assert e_nat <= e_ref
    pipe.vae_decode_batch = 1
    vid1 = run("tensor").videos
    assert torch.equal(torch.as_tensor(vid1), torch.as_tensor(vid))
