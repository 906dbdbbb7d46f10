"""Pose2VideoPipeline / Pose2ImagePipeline around the native denoising path.

Keeps ``Pose2VideoPipeline.__call__``'s signature and control flow (src/pipelines/pipeline_pose2vid_long.py:340-588)
and ``Pose2ImagePipeline.__call__`` (src/pipelines/pipeline_pose2img.py:195-376): CLIP embed -> reference UNet once ->
DDIM loop over context windows with CFG -> VAE decode.  The VAE, the CLIP image encoder and the reference ("writer")
UNet stay whatever PyTorch modules the caller passes (the reference's own); the per-timestep hot path --
``pose_guider``, ``camera_pose_encoder``, ``denoising_unet`` -- are the humanvid_b200 modules.

Differences from the reference that do not change results: pose / camera features are computed once per context window
and reused across timesteps when ``cache_condition_features=True`` (the reference recomputes the step-invariant
features every step, :526-537); the reference's stray ``print`` calls are dropped.  One deliberate deviation: the reference's
window-batching loop reuses the name ``i`` (:511-517), so its ``callback`` receives ``num_context_batches - 1`` instead of the step index;
here ``callback(i, t, latents)`` gets the true step index.  A callback (or eta != 0, or unequal windows) selects the host loop below.
"""
from __future__ import annotations

import math
from dataclasses import dataclass
from typing import Callable, List, Optional, Union

import numpy as np
import torch


# ---- context windows (src/pipelines/context.py:7-42) -------------------------------------------------------------
def _ordered_halving(val: int) -> float:
    return int(f"{val:064b}"[::-1], 2) / (1 << 64)


def uniform(step: int = 0, num_steps: Optional[int] = None, num_frames: int = 0, context_size: Optional[int] = None,
            context_stride: int = 3, context_overlap: int = 4, closed_loop: bool = True):
    if num_frames <= context_size:
        yield list(range(num_frames))
        return
    context_stride = min(context_stride, int(np.ceil(np.log2(num_frames / context_size))) + 1)
    for context_step in 1 << np.arange(context_stride):
        pad = int(round(num_frames * _ordered_halving(step)))
        for j in range(int(_ordered_halving(step) * context_step) + pad, num_frames + pad + (0 if closed_loop else -context_overlap),
                       (context_size * context_step - context_overlap)):
            yield [e % num_frames for e in range(j, j + context_size * context_step, context_step)]


def get_total_steps(scheduler, timesteps, num_steps: Optional[int] = None, num_frames: int = 0, context_size: Optional[int] = None,
                    context_stride: int = 3, context_overlap: int = 4, closed_loop: bool = True) -> int:
    """context.py:50-76: number of UNet calls of a whole loop (note: like the reference, `closed_loop` is accepted and not forwarded)."""
    return sum(len(list(scheduler(i, num_steps, num_frames, context_size, context_stride, context_overlap))) for i in range(len(timesteps)))


# ---- latent interpolation (src/pipelines/utils.py) -----------------------------------------------------------------
tensor_interpolation = None


def get_tensor_interpolation_method():
    return tensor_interpolation


def set_tensor_interpolation_method(is_slerp):
    global tensor_interpolation
    tensor_interpolation = slerp if is_slerp else linear


def linear(v1, v2, t):
    return (1.0 - t) * v1 + t * v2


def slerp(v0: torch.Tensor, v1: torch.Tensor, t: float, DOT_THRESHOLD: float = 0.9995) -> torch.Tensor:
    u0, u1 = v0 / v0.norm(), v1 / v1.norm()
    dot = (u0 * u1).sum()
    if dot.abs() > DOT_THRESHOLD:
        return (1.0 - t) * v0 + t * v1
    omega = dot.acos()
    return (((1.0 - t) * omega).sin() * v0 + (t * omega).sin() * v1) / omega.sin()


def get_context_scheduler(name: str) -> Callable:
    if name == "uniform":
        return uniform
    raise ValueError(f"Unknown context_overlap policy {name}")


@dataclass
class Pose2VideoPipelineOutput:
    videos: Union[torch.Tensor, np.ndarray]


@dataclass
class Pose2ImagePipelineOutput:
    images: Union[torch.Tensor, np.ndarray]


def _to_tensor_image(img, height, width, lo_hi=(-1.0, 1.0)):
    """PIL image / ndarray / tensor -> (1, 3, H, W) float in [lo, hi] (VaeImageProcessor.preprocess equivalent)."""
    if torch.is_tensor(img):
        t = img.float()
        if t.dim() == 3:
            t = t.unsqueeze(0)
        if t.shape[-2:] != (height, width):
            t = torch.nn.functional.interpolate(t, size=(height, width), mode="bilinear", align_corners=False)
        return t
    if hasattr(img, "resize"):
        from PIL import Image

        img = img.convert("RGB").resize((width, height), resample=Image.LANCZOS)   # VaeImageProcessor's default resample
        arr = np.asarray(img).astype(np.float32) / 255.0
    else:
        arr = np.asarray(img).astype(np.float32)
        if arr.max() > 1.5:
            arr = arr / 255.0
    t = torch.from_numpy(arr).permute(2, 0, 1).unsqueeze(0)
    lo, hi = lo_hi
    return t * (hi - lo) + lo


class _PipelineBase:
    def __init__(self, vae, image_encoder, reference_unet, denoising_unet, pose_guider, camera_pose_encoder, scheduler,
                 image_proj_model=None, tokenizer=None, text_encoder=None, clip_image_processor=None):
        self.vae, self.image_encoder, self.reference_unet = vae, image_encoder, reference_unet
        self.denoising_unet, self.pose_guider, self.camera_pose_encoder = denoising_unet, pose_guider, camera_pose_encoder
        self.scheduler = scheduler
        if clip_image_processor is None:
            # the reference always builds one (pipeline_pose2vid_long.py:73): CLIP mean/std normalisation + bicubic resize
            from transformers import CLIPImageProcessor

            clip_image_processor = CLIPImageProcessor()
        self.clip_image_processor = clip_image_processor
        cfg = getattr(vae, "config", None)
        n = len(getattr(cfg, "block_out_channels", (1, 2, 3, 4))) if cfg is not None else 4
        self.vae_scale_factor = 2 ** (n - 1)
        self.cache_condition_features = True
        self.vae_decode_batch = 8
        self.device_step_loop = True     # window gather / accumulate / CFG / DDIM on the device, one CUDA graph per step (SURVEY 8f-2)
        self.use_cuda_graph = True
        self._cached_loop = None         # the last clip's loop (static buffers + captured graph), reused when the next clip has the same shapes
        self.reference_control_cls = None  # (writer_cls, reader_cls); set by the integrator, see INTEGRATION.md

    def to(self, device=None, dtype=None):
        for name in ("vae", "image_encoder", "reference_unet", "denoising_unet", "pose_guider", "camera_pose_encoder"):
            m = getattr(self, name)
            if m is not None and hasattr(m, "to"):
                if dtype is not None and device is not None:
                    m.to(device=device, dtype=dtype)
                elif device is not None:
                    m.to(device)
                elif dtype is not None:
                    m.to(dtype=dtype)
        return self

    def prepare_latents(self, batch_size, num_channels_latents, width, height, video_length, dtype, device, generator, latents=None):
        shape = (batch_size, num_channels_latents, video_length, height // self.vae_scale_factor, width // self.vae_scale_factor)
        if latents is None:
            gdev = generator.device if generator is not None else device
            latents = torch.randn(shape, generator=generator, device=gdev, dtype=dtype).to(device)
        else:
            latents = latents.to(device)
        return latents * self.scheduler.init_noise_sigma

    def _clip_embed(self, ref_image, device):
        if torch.is_tensor(ref_image):
            # tensor images (tests, already-decoded inputs) in [-1, 1]: resize, map to [0, 1], CLIP mean / std
            pix = _to_tensor_image(ref_image, 224, 224).to(device) * 0.5 + 0.5
            mean = torch.tensor(self.clip_image_processor.image_mean, device=pix.device).view(1, 3, 1, 1)
            std = torch.tensor(self.clip_image_processor.image_std, device=pix.device).view(1, 3, 1, 1)
            pix = (pix - mean) / std
        else:
            pix = self.clip_image_processor.preprocess(ref_image.resize((224, 224)), return_tensors="pt").pixel_values
        enc_dtype = next(self.image_encoder.parameters()).dtype if hasattr(self.image_encoder, "parameters") else torch.float16
        return self.image_encoder(pix.to(device, dtype=enc_dtype)).image_embeds

    def _begin(self, ref_image, num_inference_steps, guidance_scale):
        """(device, CFG on, host timesteps, encoder_hidden_states): the CLIP image embedding as (b, 1, dim), behind a zero unconditional
        half under CFG."""
        device = torch.device("cuda") if torch.cuda.is_available() else torch.device("cpu")
        cfg_on = guidance_scale > 1.0
        self.scheduler.set_timesteps(num_inference_steps, device=device)
        timesteps = getattr(self.scheduler, "_host_timesteps", None) or [int(t) for t in self.scheduler.timesteps]
        ehs = self._clip_embed(ref_image, device).unsqueeze(1)
        if cfg_on:
            ehs = torch.cat([torch.zeros_like(ehs), ehs], dim=0)
        return device, cfg_on, timesteps, ehs

    def _reference_controls(self, cfg_on):
        """(writer, reader) ReferenceAttentionControls: ``reference_control_cls`` if set, else this package's reader, and its writer around a
        native reference UNet (no writer otherwise)."""
        writer_cls, reader_cls = self.reference_control_cls or (None, None)
        if reader_cls is None:
            from .modules import ReferenceAttentionControl as reader_cls
        if writer_cls is None and self.reference_unet is not None:
            from .modules import ReferenceAttentionControl, UNet2DConditionModel
            if isinstance(self.reference_unet, UNet2DConditionModel):   # native reference UNet: the native control writes its banks
                writer_cls = ReferenceAttentionControl
        writer = writer_cls(self.reference_unet, do_classifier_free_guidance=cfg_on, mode="write", batch_size=1, fusion_blocks="full") \
            if writer_cls is not None else None
        reader = reader_cls(self.denoising_unet, do_classifier_free_guidance=cfg_on, mode="read", batch_size=1, fusion_blocks="full")
        return writer, reader

    def _reference_latents(self, ref_image, height, width, device):
        vae_dtype = next(self.vae.parameters()).dtype if hasattr(self.vae, "parameters") else torch.float16
        return self.vae.encode(_to_tensor_image(ref_image, height, width).to(dtype=vae_dtype, device=device)).latent_dist.mean * 0.18215

    def _write_banks(self, writer, reader, ref_latents, ehs, cfg_on, device):
        """One reference-UNet forward over the reference latents, then hand its banks to the denoising UNet."""
        if writer is not None:
            self.reference_unet(ref_latents.repeat((2 if cfg_on else 1), 1, 1, 1), torch.zeros((), dtype=torch.long, device=device),
                                encoder_hidden_states=ehs, return_dict=False)
            reader.update(writer)

    @staticmethod
    def _clear_controls(writer, reader):
        reader.clear()
        if writer is not None:
            writer.clear()

    def _output(self, latents, output_type, return_dict, output_cls):
        """The latents (output_type "latent") or the decoded frames (a tensor for "tensor", else an ndarray), in `output_cls` when
        return_dict."""
        out = latents
        if output_type != "latent":
            out = self.decode_latents(latents)
            if output_type == "tensor":
                out = torch.from_numpy(out)
        return output_cls(out) if return_dict else out

    def _device_loop_ok(self, eta, callback, context_batch_size, context_queue, latents, cfg_on=True) -> bool:
        """The on-device loop covers what scripts/pose2vid.py uses: native denoising UNet, this package's DDIM scheduler with
        eta = 0, no per-step host callback, one window per UNet call, equally long windows, and CFG on whenever windows overlap.
        (Without CFG the reference never divides the accumulated prediction by ``counter`` -- the division sits inside the CFG branch,
        pipeline_pose2vid_long.py:551-555 -- so overlapping windows are SUMMED; the glue kernel always averages, so that corner is
        left to the host loop below, which restates the reference line by line.)"""
        from .modules import UNet3DConditionModel
        from .scheduler import DDIMScheduler

        return (self.device_step_loop and isinstance(self.denoising_unet, UNet3DConditionModel) and isinstance(self.scheduler, DDIMScheduler)
                and eta == 0.0 and callback is None and context_batch_size == 1 and latents.is_cuda
                and len({len(c) for c in context_queue}) == 1 and len(context_queue) <= 32
                and (cfg_on or len(context_queue) == 1))

    def _loop_kwargs(self, context_queue, cfg_on):
        """Extra DeviceDenoiseLoop arguments; humanvid_b200.distributed overrides this to split (window x CFG-half) units over ranks."""
        return {}

    def interpolate_latents(self, latents: torch.Tensor, interpolation_factor: int, device):
        """pipeline_pose2vid_long.py:294-336: (factor - 1) interpolated latents between consecutive frames."""
        if interpolation_factor < 2:
            return latents
        if tensor_interpolation is None:
            raise RuntimeError("interpolation_factor >= 2 needs set_tensor_interpolation_method(is_slerp) first (src/pipelines/utils.py)")
        new_latents = torch.zeros((latents.shape[0], latents.shape[1], ((latents.shape[2] - 1) * interpolation_factor) + 1, latents.shape[3],
                                   latents.shape[4]), device=latents.device, dtype=latents.dtype)
        rate = [i / interpolation_factor for i in range(interpolation_factor)][1:]
        new_index = 0
        v1 = None
        for i0, i1 in zip(range(latents.shape[2]), range(latents.shape[2])[1:]):
            v0, v1 = latents[:, :, i0], latents[:, :, i1]
            new_latents[:, :, new_index] = v0
            new_index += 1
            for f in rate:
                new_latents[:, :, new_index] = tensor_interpolation(v0.to(device=device), v1.to(device=device), f).to(latents.device)
                new_index += 1
        new_latents[:, :, new_index] = v1
        return new_latents

    def decode_latents(self, latents):
        video_length = latents.shape[2]
        latents = 1 / 0.18215 * latents
        b = latents.shape[0]
        latents = latents.permute(0, 2, 1, 3, 4).reshape(b * video_length, *latents.shape[1:2], *latents.shape[3:])
        # the reference decodes one frame per call (:119-121); frames are independent in the VAE, so they go `vae_decode_batch` at a
        # time (SURVEY 8f-4).  vae_decode_batch = 1 reproduces the reference's call pattern exactly.
        n = max(1, int(self.vae_decode_batch))
        video = [self.vae.decode(latents[i : i + n]).sample for i in range(0, latents.shape[0], n)]
        video = torch.cat(video)
        video = video.reshape(b, video_length, *video.shape[1:]).permute(0, 2, 1, 3, 4)
        video = (video / 2 + 0.5).clamp(0, 1)
        return video.cpu().float().numpy()


class Pose2VideoPipeline(_PipelineBase):
    @torch.no_grad()
    def __call__(self, ref_image, pose_images, camera_embedding, width, height, video_length, num_inference_steps, guidance_scale,
                 num_images_per_prompt=1, eta: float = 0.0, generator=None, output_type: Optional[str] = "tensor", return_dict: bool = True,
                 callback: Optional[Callable] = None, callback_steps: Optional[int] = 1, context_schedule="uniform", context_frames=24,
                 context_stride=1, context_overlap=4, context_batch_size=1, interpolation_factor=1, **kwargs):
        device, cfg_on, timesteps, encoder_hidden_states = self._begin(ref_image, num_inference_steps, guidance_scale)
        writer, reader = self._reference_controls(cfg_on)
        latents = self.prepare_latents(num_images_per_prompt, self.denoising_unet.in_channels, width, height, video_length, encoder_hidden_states.dtype,
                                       device, generator)
        ref_image_latents = self._reference_latents(ref_image, height, width, device)

        pose_cond_tensor = torch.cat([_to_tensor_image(p, height, width, (0.0, 1.0)).unsqueeze(2) for p in pose_images], dim=2)
        pose_cond_tensor = pose_cond_tensor.to(device=device, dtype=self.pose_guider.dtype)
        camera_embedding = camera_embedding.to(device=device, dtype=self.camera_pose_encoder.dtype)
        assert camera_embedding.ndim == 5
        context_scheduler = get_context_scheduler(context_schedule)
        feature_cache = {}

        def window_features(context):
            key = tuple(tuple(c) for c in context)
            if self.cache_condition_features and key in feature_cache:
                return feature_cache[key]
            pose_fea = self.pose_guider(torch.cat([pose_cond_tensor[:, :, c] for c in context]))
            cur_cam = torch.cat([camera_embedding[:, :, c] for c in context])
            cam_b = cur_cam.shape[0]
            cam = self.camera_pose_encoder(cur_cam)[0]
            cam = cam.reshape(cam_b, -1, *cam.shape[1:]).permute(0, 2, 1, 3, 4)
            cond = (pose_fea + cam).repeat(2 if cfg_on else 1, 1, 1, 1, 1)
            if self.cache_condition_features:
                feature_cache[key] = cond
            return cond

        # the scheduler is always asked with step = 0 (:495-502): the windows are the same at every timestep
        context_queue = list(context_scheduler(0, num_inference_steps, latents.shape[2], context_frames, context_stride, context_overlap))
        if self._device_loop_ok(eta, callback, context_batch_size, context_queue, latents, cfg_on):
            # ---- SURVEY 8f-2: every per-timestep operation on the device, one CUDA graph per step -------------------------
            from .device_loop import DeviceDenoiseLoop

            self._write_banks(writer, reader, ref_image_latents, encoder_hidden_states, cfg_on, device)
            conds = [window_features([c]) for c in context_queue]
            extra = self._loop_kwargs(context_queue, cfg_on)
            loop = self._cached_loop
            if loop is not None and not extra and loop.matches(self.denoising_unet, self.scheduler, latents, context_queue, encoder_hidden_states, conds,
                                                               guidance_scale, cfg_on):
                # same shapes as the previous clip: the captured step is still valid -- refill its static buffers, no warm-up, no re-capture
                loop.reload(latents, encoder_hidden_states, conds)
            else:
                if loop is not None:
                    loop.close()
                loop = DeviceDenoiseLoop(self.denoising_unet, self.scheduler, latents, context_queue, encoder_hidden_states, conds, guidance_scale, cfg_on,
                                         **extra)
                self._cached_loop = loop if (self.use_cuda_graph and not extra) else None
            try:
                latents = loop.run(len(timesteps), use_graph=self.use_cuda_graph).to(latents.dtype).clone()
            finally:
                if self._cached_loop is loop:
                    loop.detach()
                else:
                    loop.close()
            timesteps = []

        for i, t in enumerate(timesteps):
            noise_pred = torch.zeros((latents.shape[0] * (2 if cfg_on else 1), *latents.shape[1:]), device=latents.device, dtype=latents.dtype)
            counter = torch.zeros((1, 1, latents.shape[2], 1, 1), device=latents.device, dtype=latents.dtype)
            if i == 0:
                self._write_banks(writer, reader, ref_image_latents, encoder_hidden_states, cfg_on, device)
            nb = math.ceil(len(context_queue) / context_batch_size)
            global_context = [context_queue[k * context_batch_size : (k + 1) * context_batch_size] for k in range(nb)]
            for context in global_context:
                latent_model_input = torch.cat([latents[:, :, c] for c in context]).to(device).repeat(2 if cfg_on else 1, 1, 1, 1, 1)
                latent_model_input = self.scheduler.scale_model_input(latent_model_input, t)
                b = latent_model_input.shape[0]
                cond = window_features(context)
                pred = self.denoising_unet(latent_model_input, t, encoder_hidden_states=encoder_hidden_states[:b], pose_cond_fea=cond,
                                           return_dict=False)[0]
                for c in context:
                    noise_pred[:, :, c] = noise_pred[:, :, c] + pred
                    counter[:, :, c] = counter[:, :, c] + 1
            if cfg_on:
                un, tx = (noise_pred / counter).chunk(2)
                noise_pred = un + guidance_scale * (tx - un)
            latents = self.scheduler.step(noise_pred, t, latents, eta=eta).prev_sample
            if callback is not None and i % callback_steps == 0:
                callback(i, t, latents)
        self._clear_controls(writer, reader)
        if interpolation_factor > 0:
            latents = self.interpolate_latents(latents, interpolation_factor, device)
        return self._output(latents, output_type, return_dict, Pose2VideoPipelineOutput)


class Pose2ImagePipeline(_PipelineBase):
    """Single-frame variant (config 1; src/pipelines/pipeline_pose2img.py:195-376): conditioning computed once outside the loop."""

    @torch.no_grad()
    def __call__(self, ref_image, pose_image, camera_embedding, width, height, num_inference_steps, guidance_scale, num_images_per_prompt=1,
                 eta: float = 0.0, generator=None, output_type: Optional[str] = "tensor", return_dict: bool = True, callback=None,
                 callback_steps: Optional[int] = 1, **kwargs):
        device, cfg_on, timesteps, ehs = self._begin(ref_image, num_inference_steps, guidance_scale)
        writer, reader = self._reference_controls(cfg_on)
        latents = self.prepare_latents(num_images_per_prompt, self.denoising_unet.in_channels, width, height, 1, ehs.dtype, device, generator)
        ref_latents = self._reference_latents(ref_image, height, width, device)
        pose = _to_tensor_image(pose_image, height, width, (0.0, 1.0)).unsqueeze(2).to(device=device, dtype=self.pose_guider.dtype)
        pose_fea = self.pose_guider(pose)
        camera_embedding = camera_embedding.to(device=device, dtype=self.camera_pose_encoder.dtype)
        if camera_embedding.ndim == 4:                    # (b, 6, h, w): the reference unsqueezes the frame axis itself (pipeline_pose2img.py:298)
            camera_embedding = camera_embedding.unsqueeze(2)
        assert camera_embedding.ndim == 5
        cb = camera_embedding.shape[0]
        cam = self.camera_pose_encoder(camera_embedding)[0]
        cam = cam.reshape(cb, -1, *cam.shape[1:]).permute(0, 2, 1, 3, 4)
        cond = pose_fea + cam
        if cond.shape[0] != latents.shape[0]:             # num_images_per_prompt > 1: one condition for every image of the prompt
            cond = cond.repeat(latents.shape[0] // cond.shape[0], 1, 1, 1, 1)
        cond = cond.repeat(2 if cfg_on else 1, 1, 1, 1, 1)
        for i, t in enumerate(timesteps):
            if i == 0:
                self._write_banks(writer, reader, ref_latents, ehs, cfg_on, device)
            x = self.scheduler.scale_model_input(latents.repeat(2 if cfg_on else 1, 1, 1, 1, 1), t)
            noise_pred = self.denoising_unet(x, t, encoder_hidden_states=ehs, pose_cond_fea=cond, return_dict=False)[0]
            if cfg_on:
                un, tx = noise_pred.chunk(2)
                noise_pred = un + guidance_scale * (tx - un)
            latents = self.scheduler.step(noise_pred, t, latents, eta=eta).prev_sample
            if callback is not None and i % callback_steps == 0:
                callback(i, t, latents)
        self._clear_controls(writer, reader)
        return self._output(latents, output_type, return_dict, Pose2ImagePipelineOutput)
