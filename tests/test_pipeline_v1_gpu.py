"""Pose2VideoPipeline with the inference_v1 denoising UNet (GroupNorm statistics pooled over each 24-frame window, no mid-block motion
module) and DDIM as inference_v1.yaml's noise_scheduler_kwargs give it through diffusers' defaults: epsilon prediction, "leading"
timesteps, no zero-SNR rescale.  48 frames = three overlapping context windows, CFG, native writer UNet -> banks, on an H100 with the
stand-in VAE / CLIP of tests/test_pipeline_gpu.py.  The on-device loop (hv_op_cfg_ddim_step with pred_type = epsilon, one CUDA graph
per step) against the same call without the graph (bitwise), the host loop (humanvid_b200.DDIMScheduler.step), and the oracle's
restatement of the loop with the v1 oracle UNet and a closed-form epsilon DDIM step.  The camera encoder takes inference_v2.yaml's
pose_encoder_kwargs (inference_v1.yaml has none)."""
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

from conftest import report
from unet_v1_oracle import V1_UNET_KWARGS, unet3d_v1

if torch.cuda.is_available():
    import humanvid_b200 as hv
    from humanvid_b200.pipeline import Pose2VideoPipeline
    from oracle import hv_oracle as O
    from test_pipeline_gpu import StubCLIP, StubVAE, rel

V1_SCHED = dict(beta_start=0.00085, beta_end=0.012, beta_schedule="linear", steps_offset=1, clip_sample=False,
                prediction_type="epsilon", timestep_spacing="leading", rescale_betas_zero_snr=False)


def ddim_eps_step(sched, eps, t, x, steps):
    """diffusers DDIMScheduler.step, eta = 0, epsilon prediction, set_alpha_to_one: the closed form."""
    ac = sched.alphas_cumprod.double()
    prev = t - 1000 // steps
    a_t = ac[t]
    a_p = ac[prev] if prev >= 0 else torch.tensor(1.0, dtype=torch.float64)
    x0 = (x.double() - (1 - a_t).sqrt() * eps.double()) / a_t.sqrt()
    return (a_p.sqrt() * x0 + (1 - a_p).sqrt() * eps.double()).float()


def test_pose2video_v1_unet_epsilon_leading_three_windows():
    dev = "cuda"
    chs, xdim, Fv, H, W = (64, 128, 256, 256), 64, 48, 128, 128
    ora = O.synthetic_init(unet3d_v1(chs, xdim).eval(), seed=7).half().float().to(dev)
    opg = O.synthetic_init(O.PoseGuider(64, 3, (16, 32, 96, 256)).eval(), seed=11).half().float().to(dev)
    ocam = O.synthetic_init(O.CameraPoseEncoder(channels=(64,), heads=8).eval(), seed=13).half().float().to(dev)
    unet = hv.UNet3DConditionModel(block_out_channels=chs, cross_attention_dim=xdim, attention_head_dim=8, **V1_UNET_KWARGS)
    unet.load_state_dict(ora.state_dict())
    pg = hv.PoseGuider(64, block_out_channels=(16, 32, 96, 256))
    pg.load_state_dict(opg.state_dict())
    cam = hv.CameraPoseEncoder(downscale_factor=8, channels=[64], nums_rb=2, cin=384, ksize=1, sk=True, use_conv=False, compression_factor=1,
                               temporal_attention_nhead=8, attention_block_types=["Temporal_Self"], temporal_position_encoding=True,
                               temporal_position_encoding_max_len=24)
    cam.load_state_dict(ocam.state_dict())
    oref = O.synthetic_init(O.UNet2DConditionModel(block_out_channels=chs, cross_attention_dim=xdim).eval(), seed=17).half().float().to(dev)
    ref_unet = hv.UNet2DConditionModel(block_out_channels=chs, cross_attention_dim=xdim)
    ref_unet.load_state_dict(oref.state_dict())
    vae, clip = StubVAE().half().to(dev), StubCLIP(xdim).half().to(dev)
    sched = hv.DDIMScheduler(**V1_SCHED)
    steps, cfg = 2, 3.5
    sched.set_timesteps(steps)
    assert sched.timesteps.tolist() == [501, 1]   # leading spacing + steps_offset, as diffusers computes it
    pipe = Pose2VideoPipeline(vae=vae, image_encoder=clip, reference_unet=ref_unet, denoising_unet=unet, pose_guider=pg, camera_pose_encoder=cam,
                              scheduler=sched).to(dev, torch.float16)

    g = torch.Generator(device=dev).manual_seed(3)
    ref = torch.rand(3, H, W, generator=g, device=dev) * 2 - 1
    poses = [torch.rand(1, 3, H, W, generator=g, device=dev) for _ in range(Fv)]
    camera = torch.randn(1, 6, Fv, H, W, generator=g, device=dev).half()
    gen = torch.Generator(device=dev).manual_seed(42)
    out = pipe(ref, poses, camera, W, H, Fv, steps, cfg, generator=gen, output_type="latent", return_dict=False)
    assert out.shape == (1, 4, Fv, H // 8, W // 8) and torch.isfinite(out).all()
    assert pipe.device_step_loop and pipe.use_cuda_graph

    # the oracle's loop: v1 oracle UNet per window (oracle.denoise_step), closed-form epsilon DDIM
    gen = torch.Generator(device=dev).manual_seed(42)
    lat = torch.randn((1, 4, Fv, H // 8, W // 8), generator=gen, device=dev, dtype=torch.float16).float()
    with torch.no_grad():
        pix = F.interpolate(ref[None].float(), size=(224, 224), mode="bilinear", align_corners=False) * 0.5 + 0.5
        mean = torch.tensor(pipe.clip_image_processor.image_mean, device=dev).view(1, 3, 1, 1)
        std = torch.tensor(pipe.clip_image_processor.image_std, device=dev).view(1, 3, 1, 1)
        emb = clip(((pix - mean) / std).half()).image_embeds.float()
        ehs = torch.cat([torch.zeros_like(emb), emb]).unsqueeze(1)
        pose_cond = torch.cat([p.unsqueeze(2) for p in poses], dim=2).half().float()
        ref_lat = (vae.encode(ref[None].half()).latent_dist.mean * 0.18215).float()
        O.set_reference_write(oref)
        oref(ref_lat.repeat(2, 1, 1, 1), torch.tensor(0, device=dev), ehs)
        O.set_reference_banks(ora, O.written_banks(oref), cfg=True)
        for t in sched.timesteps.tolist():
            eps = O.denoise_step(ora, opg, ocam, lat, torch.tensor(t, device=dev), ehs, pose_cond, camera.float(), guidance_scale=cfg)
            lat = ddim_eps_step(sched, eps.cpu(), t, lat.cpu(), steps).to(dev)
    e = rel(out, lat)

    pipe.use_cuda_graph = False
    gen = torch.Generator(device=dev).manual_seed(42)
    out_nograph = pipe(ref, poses, camera, W, H, Fv, steps, cfg, generator=gen, output_type="latent", return_dict=False)
    pipe.device_step_loop = False
    gen = torch.Generator(device=dev).manual_seed(42)
    out_host = pipe(ref, poses, camera, W, H, Fv, steps, cfg, generator=gen, output_type="latent", return_dict=False)
    pipe.device_step_loop = pipe.use_cuda_graph = True
    e_host = rel(out_host, lat)
    report(f"pipeline v1 UNet, epsilon / leading DDIM, 48 frames / 3 windows / 2 steps: device-loop latents vs oracle loop {e:.2e}; "
           f"host-loop {e_host:.2e}; device vs host loop {rel(out, out_host):.2e}")
    assert torch.equal(out, out_nograph)
    # the tolerances of the inference_v2 pipeline test (tests/test_pipeline_gpu.py)
    assert e < 6e-3 and e_host < 6e-3 and rel(out, out_host) < 8e-3
    # and it is the epsilon branch that ran: the same call with v-prediction gives another clip
    sched_v = hv.DDIMScheduler(**{**V1_SCHED, "prediction_type": "v_prediction"})
    pipe_v = Pose2VideoPipeline(vae=vae, image_encoder=clip, reference_unet=ref_unet, denoising_unet=unet, pose_guider=pg, camera_pose_encoder=cam,
                                scheduler=sched_v).to(dev, torch.float16)
    gen = torch.Generator(device=dev).manual_seed(42)
    out_v = pipe_v(ref, poses, camera, W, H, Fv, steps, cfg, generator=gen, output_type="latent", return_dict=False)
    assert rel(out_v, out) > 1e-2
