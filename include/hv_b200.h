/* hv_b200.h -- network-level C ABI of libhv_b200.so: the drop-in boundary for the CamAnimate denoising path.
 *
 * The reference (zhenzhiwang/HumanVid) is pure Python and has no FFI; these entry points are what a binding of its
 * three hot-path modules would call (see INTEGRATION.md for the ctypes stub):
 *
 *   HV_KIND_UNET3D        UNet3DConditionModel.forward   src/models/unet_3d.py:397-577
 *   HV_KIND_POSE_GUIDER   PoseGuider.forward             src/models/pose_guider.py:51-61
 *   HV_KIND_CAMERA_ENCODER CameraPoseEncoder.forward     src/cameractrl/pose_adaptor.py:232-248
 *   hv_set_ref_bank / hv_clear_ref_banks                 ReferenceAttentionControl.update / .clear
 *                                                        src/models/mutual_self_attention.py:302-363
 *   HV_KIND_VAE           AutoencoderKL.encode / .decode (diffusers 0.24, the SD layout configs/prompts/stage2.yaml points at):
 *                         what Pose2VideoPipeline / Pose2ImagePipeline call for the reference latents and the output frames
 *   HV_KIND_UNET2D_REF    UNet2DConditionModel.forward in "write" mode (the reference / "writer" UNet, once per clip)
 *                                                        src/models/unet_2d_condition.py:872-1308 (post-process removed
 *                                                        :1295-1299), write hook mutual_self_attention.py:137-146
 *   HV_KIND_CLIP_VISION   transformers' CLIPVisionModelWithProjection.forward (the image encoder whose image_embeds condition both UNets,
 *                         scripts/pose2vid.py:17,152)
 *
 * Contract: all tensor arguments are caller-owned CUDA device pointers (torch allocations), contiguous, fp16 unless
 * stated, in the reference's own layouts ((B,C,F,H,W) etc.).  The library owns only its packed weights, reference
 * banks and (unless the caller passes one) its workspace.  Every launch goes on the stream passed in and returns
 * without synchronising.  Functions return 0 or a negative hv_status and never throw; hv_last_error(handle) gives the
 * message.  A handle is bound to the device current at hv_create and is not thread-safe (the reference is
 * single-threaded Python under torch.no_grad).
 */
#ifndef HV_B200_H
#define HV_B200_H

#include "hv_b200_ops.h"

#ifdef __cplusplus
extern "C" {
#endif

typedef struct hv_model* hv_handle;

enum hv_kind { HV_KIND_UNET3D = 0, HV_KIND_POSE_GUIDER = 1, HV_KIND_CAMERA_ENCODER = 2, HV_KIND_UNET2D_REF = 3, HV_KIND_VAE = 4, HV_KIND_CLIP_VISION = 5 };
enum hv_dtype { HV_F16 = 0, HV_F32 = 1 };
enum hv_forward_flags {
  HV_FLAG_CFG = 1,         /* batch = [uncond half ; cond half]: the first half ignores the reference banks
                              (mutual_self_attention.py:166-186) */
  HV_FLAG_UNCOND_ONLY = 2, /* the batch is an unconditional CFG half only (one unit of a (window x CFG-half) split over
                              GPUs, SURVEY 8e): no item reads the banks */
  HV_FLAG_COND_ONLY = 4    /* the batch is a conditional CFG half only: its B items read the LAST B items of the banks
                              (banks are written for [uncond ; cond], pipeline_pose2vid_long.py:470-480) */
};

typedef struct hv_config {
  int32_t kind; /* hv_kind */
  /* UNet3DConditionModel (unet_3d.py:34-83 + configs/inference/inference_v2.yaml) */
  int32_t in_channels;           /* 4 */
  int32_t out_channels;          /* 4 */
  int32_t block_out_channels[4]; /* 320 640 1280 1280 */
  int32_t heads;                 /* attention_head_dim = 8 heads */
  int32_t cross_attention_dim;   /* 768 */
  int32_t norm_groups;           /* 32 */
  int32_t use_motion_module;     /* 1 (config 1 / pose2img: 0) */
  int32_t motion_max_len;        /* temporal_position_encoding_max_len = 32 */
  /* PoseGuider (pose_guider.py:17-49) */
  int32_t pg_cond_channels;      /* 3 */
  int32_t pg_block_channels[4];  /* 16 32 96 256 */
  int32_t pg_out_channels;       /* 320 */
  /* CameraPoseEncoder (pose_adaptor.py:162-230, pose_encoder_kwargs) */
  int32_t cam_downscale;         /* 8 */
  int32_t cam_cin;               /* 384 */
  int32_t cam_channels;          /* 320 */
  int32_t cam_nums_rb;           /* 2 */
  int32_t cam_heads;             /* 8 */
  int32_t cam_max_len;           /* 24 */
  /* AutoencoderKL (diffusers 0.24, SD layout): block_out_channels (128 256 512 512), norm_groups (32), in_channels /
   * out_channels (3 image channels) above, and: */
  int32_t vae_latent_channels;   /* 4 */
  /* CLIPVisionModelWithProjection (transformers CLIPVisionConfig; ViT-L/14 values shown).  Head dim hidden / heads must be 64, the MLP
   * activation is quick_gelu, 3 image channels. */
  int32_t clip_hidden_size;       /* 1024 */
  int32_t clip_layers;            /* num_hidden_layers = 24 */
  int32_t clip_heads;             /* num_attention_heads = 16 */
  int32_t clip_intermediate_size; /* 4096 */
  int32_t clip_patch_size;        /* 14 */
  int32_t clip_image_size;        /* 224 */
  int32_t clip_projection_dim;    /* 768 */
  float clip_layer_norm_eps;      /* 1e-5 */
  /* UNet3DConditionModel, configs/inference/inference_v1.yaml (AnimateDiff v1 motion-module layout).  0 keeps the inference_v2 behaviour. */
  int32_t gn_pool_frames;         /* 1: use_inflated_groupnorm = False -- the resnets' norm1 / norm2 and conv_norm_out take their statistics over
                                     all F frames of a batch item (nn.GroupNorm on (b, c, f, h, w)); the transformer and motion-module
                                     GroupNorms stay per frame.  A frame's output then depends on the other frames of its window. */
  int32_t no_mid_motion_module;   /* 1: motion_module_mid_block = False -- the mid block has no motion module */
  /* UNet3DConditionModel only.  0 keeps the fp16 path.  1: FP8 mode (DESIGN.md §9, include/hv_b200_fp8.h): hv_finalize keeps an e4m3 copy of
     the feed-forward weights of the spatial transformers and motion modules of width >= 1280, and those LayerNorm -> FF1 -> FF2 chains run on
     e4m3 with per-token / per-128 activation scales (the only covered shapes measured faster than fp16; every other linear stays fp16).
     Outputs then differ from the fp16 path by the e4m3 quantisation error. */
  int32_t fp8_linears;
} hv_config;

int hv_create(const hv_config* cfg, hv_handle* out);
void hv_destroy(hv_handle h);
const char* hv_last_error(hv_handle h);

/* Copies (and converts to fp16) one state_dict entry under the reference's key name, e.g.
 * "down_blocks.0.resnets.1.conv1.weight".  Unknown keys are accepted and ignored (returns 0). */
int hv_set_weight(hv_handle h, const char* key, const void* dev_ptr, const int64_t* shape, int32_t ndim, int32_t dtype,
                  hv_stream_t stream);
/* Packs all weights into their kernel layouts; fails with HV_ERR_MISSING naming the first absent key. */
int hv_finalize(hv_handle h, hv_stream_t stream);

/* Reference-attention K/V banks in reader order (all TemporalBasicTransformerBlocks of the UNet in DFS order
 * down_blocks, up_blocks, mid_block, stable-sorted by descending width).  bank: (B_ref, L, C) fp16. */
int hv_num_ref_blocks(hv_handle h);
int hv_ref_block_dim(hv_handle h, int32_t block_idx);
int hv_set_ref_bank(hv_handle h, int32_t block_idx, const void* dev_ptr, int64_t B_ref, int64_t L, int64_t C, hv_stream_t stream);
int hv_clear_ref_banks(hv_handle h);

/* Bytes of scratch one forward needs at this shape (h, w = spatial size of the tensor entering the network). */
size_t hv_workspace_bytes(hv_handle h, int32_t B, int32_t F, int32_t height, int32_t width);
/* Grows the handle's private workspace to what this shape needs (cudaMalloc here, never inside a forward).  A forward
 * called with workspace == NULL uses it and fails with HV_ERR_STATE if it is too small. */
int hv_reserve_workspace(hv_handle h, int32_t B, int32_t F, int32_t height, int32_t width);
/* Device-resident timestep for CUDA-graph replay of a denoising loop (pipeline_pose2vid_long.py:454-563): when set, every
 * UNet forward of this handle embeds dev_table[*dev_index] (read on the device when the kernel runs) and ignores its
 * `timestep` argument.  Both NULL restores the host argument. */
int hv_set_timestep_source(hv_handle h, const int64_t* dev_table, const int32_t* dev_index);

/* sample (B,4,F,h,w), encoder_hidden_states (B,1,cross_attention_dim), pose_cond_fea (B,320,F,h,w) or NULL,
 * out (B,4,F,h,w); all fp16.  workspace may be NULL: the handle's reserved workspace (hv_reserve_workspace) is used. */
int hv_unet3d_forward(hv_handle h, const void* sample, int64_t timestep, const void* encoder_hidden_states, const void* pose_cond_fea,
                      void* out, int32_t B, int32_t F, int32_t height, int32_t width, uint32_t flags, void* workspace,
                      size_t ws_bytes, hv_stream_t stream);
/* Reference ("writer") UNet, kind HV_KIND_UNET2D_REF (hv_config as for the UNet3D with use_motion_module = 0; no
 * conv_norm_out / conv_out weights).  sample (B,4,h,w), encoder_hidden_states (B,1,cross_attention_dim);
 * bank_out[i] (i in reader order, see hv_num_ref_blocks / hv_ref_block_dim) receives block i's LayerNorm-1 output
 * (B, h_i*w_i, C_i) fp16 -- exactly what hv_set_ref_bank of the denoising UNet takes; hidden_out (B,C0,h,w) or NULL is
 * the forward's return value (the last up block's output). */
int hv_unet2d_reference_forward(hv_handle h, const void* sample, int64_t timestep, const void* encoder_hidden_states, void* hidden_out,
                                void* const* bank_out, int32_t n_banks, int32_t B, int32_t height, int32_t width, void* workspace,
                                size_t ws_bytes, hv_stream_t stream);
/* conditioning (B,3,F,H,W) -> out (B,320,F,H/8,W/8) */
int hv_pose_guider_forward(hv_handle h, const void* conditioning, void* out, int32_t B, int32_t F, int32_t H, int32_t W,
                           void* workspace, size_t ws_bytes, hv_stream_t stream);
/* plucker (B,6,F,H,W) -> out (B*F,320,H/8,W/8) (the single feature map of the one-level encoder) */
int hv_camera_encoder_forward(hv_handle h, const void* plucker, void* out, int32_t B, int32_t F, int32_t H, int32_t W,
                              void* workspace, size_t ws_bytes, hv_stream_t stream);

/* The same encoder fed by the cameras themselves instead of the 6-channel Plucker image (SURVEY 8f-3): intrinsics DEVICE fp32
 * (B, F, 4) = (fx, fy, cx, cy) in pixels, c2w DEVICE fp32 (B, F, 4, 4) relative camera-to-world poses -- what
 * scripts/pose2vid.py:66-80 hands to ray_condition.  The embedding is generated inside the PixelUnshuffle producer. */
int hv_camera_encoder_forward_rays(hv_handle h, const float* intrinsics, const float* c2w, void* out, int32_t B, int32_t F, int32_t H,
                                   int32_t W, void* workspace, size_t ws_bytes, hv_stream_t stream);

/* AutoencoderKL (kind HV_KIND_VAE; weights under diffusers' key names: encoder.*, decoder.*, quant_conv, post_quant_conv, the mid-block
 * attention as mid_block.attentions.0.{group_norm,to_q,to_k,to_v,to_out.0}).
 * hv_vae_decode: z (N, latent, h, w) -> out (N, out_channels, 8h, 8w), post_quant_conv included; the 1/scaling_factor stays with the caller.
 * hv_vae_encode: x (N, in_channels, H, W), H and W multiples of 8 -> moments (N, 2*latent, H/8, W/8) = [mean | logvar], quant_conv included.
 * Every frame is computed independently of the others in the call.  For this kind hv_workspace_bytes(h, N, 1, h, w) and
 * hv_reserve_workspace(h, N, 1, h, w) take the LATENT size: the workspace covers both decoding N latents of h x w and encoding N images of
 * 8h x 8w.  Like the other forwards these never allocate or synchronise (CUDA-graph capturable after hv_reserve_workspace). */
int hv_vae_decode(hv_handle h, const void* z, void* out, int32_t N, int32_t height, int32_t width, void* workspace, size_t ws_bytes,
                  hv_stream_t stream);
int hv_vae_encode(hv_handle h, const void* x, void* moments, int32_t N, int32_t H, int32_t W, void* workspace, size_t ws_bytes,
                  hv_stream_t stream);

/* CLIPVisionModelWithProjection (kind HV_KIND_CLIP_VISION; weights under transformers' key names: vision_model.embeddings.*,
 * vision_model.pre_layrnorm.*, vision_model.encoder.layers.{i}.*, vision_model.post_layernorm.*, visual_projection.weight).
 * pixel_values (B, 3, S, S) with S = clip_image_size -> image_embeds (B, clip_projection_dim) = visual_projection(post_layernorm(class token
 * of the last layer)), and last_hidden_state (B, 1 + (S/p)^2, clip_hidden_size) (the last encoder layer's output, without post_layernorm) unless
 * it is NULL; all fp16.  Every image is computed independently of the others in the call.  For this kind hv_workspace_bytes(h, B, 1, S, S) and
 * hv_reserve_workspace(h, B, 1, S, S) take the pixel size.  Never allocates or synchronises (CUDA-graph capturable after hv_reserve_workspace). */
int hv_clip_vision_forward(hv_handle h, const void* pixel_values, void* image_embeds, void* last_hidden_state, int32_t B, void* workspace,
                           size_t ws_bytes, hv_stream_t stream);

/* Debug taps (per-block parity tests, scripts/error_ladder.py): the activation leaving each block of a forward is copied to dst[i] as
 * channels-last fp16 (NF, H, W, C), C including the zero channels a padded layout carries.  The blocks, in execution order:
 *   UNets          conv_in, every resnet / transformer / motion module / down- / up-sampler
 *   AutoencoderKL  the decoder's (post_quant_conv, decoder.conv_in, the mid block's resnets and attention, every up-block resnet and
 *                  upsampler, decoder.conv_norm_out (GroupNorm + SiLU), decoder.conv_out), then the encoder's (encoder.conv_in, ...,
 *                  encoder.conv_out, quant_conv); a decode fills only the decoder's entries and an encode only the encoder's
 *   CLIP vision    vision_model.pre_layrnorm (B, 1, L, C), every vision_model.encoder.layers.i, vision_model.post_layernorm (B, 1, 1, C)
 *   PoseGuider     conv_in, blocks.0 .. blocks.5, conv_out (before the output layout pass)
 *   camera encoder encoder_conv_in, then per resnet / attention pair encoder_down_conv_blocks.0.j, encoder_down_attention_blocks.0.j,
 *                  zero_conv_layers.0 (hv_camera_encoder_forward and _forward_rays alike)
 * hv_debug_tap_count plans the forward at the shape hv_workspace_bytes takes and returns the number of taps; hv_debug_tap_info names
 * tap i (the reference's module path) and gives dims4 = {NF, H, W, C}; hv_debug_set_taps(h, NULL, 0) disables.  With no taps set a
 * forward launches nothing more. */
int hv_debug_tap_count(hv_handle h, int32_t B, int32_t F, int32_t height, int32_t width);
int hv_debug_tap_info(hv_handle h, int32_t i, char* name, int32_t name_cap, int64_t* dims4);
int hv_debug_set_taps(hv_handle h, void* const* dst, int32_t n);

/* Kernel launches issued by the last forward on this handle (bench.py's gpu_launches).  hv_workspace_bytes,
 * hv_reserve_workspace and hv_debug_tap_count only plan a forward and leave it unchanged. */
int64_t hv_last_launch_count(hv_handle h);

/* Optional per-operator-category device timing of the next forwards (CUDA events around every launch on the caller's
 * stream).  Categories: 0 wgmma GEMM (linear / 1x1), 1 wgmma implicit-GEMM 3x3 conv, 2 spatial attention,
 * 3 temporal attention, 4 GroupNorm/LayerNorm, 5 small linears.  hv_get_profile synchronises on the last event and
 * returns summed milliseconds, algorithmic FLOPs (2*MAC, unpadded shapes) and launch counts of the LAST forward. */
int hv_set_profiling(hv_handle h, int32_t enable);
int hv_get_profile(hv_handle h, double* ms, double* flops, int64_t* count, int32_t ncat);
/* One CSV line per timed launch of the last profiled forward: idx,cat,label,M,N,K,ms,tflops. */
int hv_dump_profile(hv_handle h, const char* path);

#ifdef __cplusplus
}
#endif
#endif
