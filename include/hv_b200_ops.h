/* hv_b200_ops.h -- operator-level C ABI of libhv_b200.so (sm_90a only).
 *
 * Each entry point is one hot-path operator of the CamAnimate denoising forward, on channels-last fp16 device
 * tensors (activations are (N, H, W, C) with N = batch*frames; "tokens x C" matrices are the same memory).  They
 * replace, one to one, the library calls the reference reaches through torch/diffusers (SURVEY.md table 2c):
 *
 *   hv_op_gemm            nn.Linear / 1x1 InflatedConv3d           src/models/resnet.py:9-15,211, transformer_3d.py:64,93,
 *                                                                  diffusers Attention.to_q/k/v/out, FeedForward (GEGLU)
 *   hv_op_conv3x3         3x3 InflatedConv3d (stride 1 / 2)        src/models/resnet.py:163,192,104; pose_adaptor.py:123,223
 *   hv_op_groupnorm       InflatedGroupNorm / nn.GroupNorm (+SiLU) src/models/resnet.py:18-26,218-235; transformer_3d.py:58,124
 *   hv_op_layernorm       nn.LayerNorm (+ temporal PE add)         src/models/attention.py:389-427; motion_module.py:244,256,273-277
 *   hv_op_attention       F.scaled_dot_product_attention over the spatial tokens of a frame, optional reference-bank
 *                         keys (ReferenceAttentionControl read hook)  src/models/attention.py:405; mutual_self_attention.py:147-186
 *   hv_op_temporal_attention  SDPA over the frame axis per pixel   src/models/motion_module.py:351-388
 *   hv_op_attention_d512  the one-head d = 512 attention of AutoencoderKL's mid block (diffusers Attention, vae.encode / vae.decode)
 *   hv_op_conv3x3_s2_pad_end  AutoencoderKL's Downsample2D: F.pad(x, (0, 1, 0, 1)) + stride-2 conv
 *   hv_op_clip_patchify   the patch embedding of CLIPVisionModelWithProjection (Conv2d(3, hidden, p, stride=p)) as the A operand of hv_op_gemm
 *
 * All functions launch asynchronously on `stream`, never synchronise, return 0 on success or a negative hv_status,
 * and do not throw.  Pointers are caller-owned device memory, 16-byte aligned, row strides multiples of 8 elements.
 */
#ifndef HV_B200_OPS_H
#define HV_B200_OPS_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef void* hv_stream_t; /* cudaStream_t */

enum hv_status {
  HV_OK = 0,
  HV_ERR_INVALID = -1,   /* bad argument (shape / alignment / unsupported size) */
  HV_ERR_CUDA = -2,      /* a CUDA runtime / driver call failed */
  HV_ERR_TMA = -3,       /* tensor-map encoding failed */
  HV_ERR_MISSING = -4,   /* a required weight was never set */
  HV_ERR_STATE = -5      /* call order violation */
};

/* HV_ACT_QUICK_GELU: x * sigmoid(1.702 x), the MLP activation of OpenAI's CLIP ViTs (hv_op_gemm / hv_op_conv3x3 epilogues only). */
enum hv_act { HV_ACT_NONE = 0, HV_ACT_RELU = 1, HV_ACT_SILU = 2, HV_ACT_QUICK_GELU = 3 };

/* Fused epilogue of hv_op_gemm / hv_op_conv3x3, applied in this order in fp32 with ONE fp16 rounding at the store (the
 * reference's eager fp16 modules round after every step; the fp32 oracle is the parity anchor):  v = acc + bias;
 * v += rowvec[row / rows_per_group]; v = act(v); v += residual[row].  With geglu != 0 the packed weight holds [128 hidden | 128 gate] rows per 256-row block and the
 * output is hidden * gelu_erf(gate) with N/2 columns (hv_op_conv3x3 runs geglu only where it picks the 256-column tile). */
typedef struct hv_epilogue {
  const void* bias;      /* fp16 [N] or NULL */
  const void* rowvec;    /* fp16 [groups][rowvec_ld] or NULL (time-embedding projection per batch item) */
  int32_t rowvec_ld;
  int32_t rows_per_group;
  const void* residual;  /* fp16 [rows][ldr] or NULL; 16-byte aligned, ldr > 0 and a multiple of 8 (else HV_ERR_INVALID) */
  int32_t ldr;
  int32_t act;           /* hv_act */
  int32_t geglu;
  int32_t n_valid;       /* columns of the output actually written; 0 = all */
} hv_epilogue;

/* out[M, N] = A[M, K] * W[N, K]^T (+epilogue).  A may be split column-wise over two buffers (torch.cat of a skip
 * connection is never materialised): columns [0,K1) come from A (row stride lda), [K1,K) from A2 (row stride lda2);
 * K1 = 0 / A2 = NULL means a single source.  K1 must be a multiple of 64.  HV_ERR_INVALID for: A, W or out NULL, M, N or K <= 0, K, N, lda or ldc
 * not a multiple of 8, a split with K1 % 64, lda2 % 8 or K1 >= K, geglu with N % 256, and the epilogue I/O hv_epilogue rejects. */
int hv_op_gemm(const void* A, int64_t lda, const void* A2, int64_t lda2, int64_t K1, const void* W, void* out, int64_t ldc,
               int64_t M, int64_t N, int64_t K, const hv_epilogue* ep, hv_stream_t stream);

/* out[M][n*out_stride + j] = sum_k A[M][k] * X[n][j][k], n < batch, j < rows: the "swapped" GEMM that yields V^T with every
 * frame's token segment starting on a 16-byte boundary (out_stride % 8 == 0), as TMA readers of V^T require.  The pad columns
 * [rows, round8(rows)) of each segment are written too, as 0 + rowbias[m] (0 without rowbias); columns [round8(rows), out_stride)
 * and [batch*out_stride, ldc) are left untouched.  HV_ERR_INVALID for NULL A, X or out, M, batch or rows <= 0, K, lda, ldx, ldc or
 * out_stride not a multiple of 8, and out_stride < rows. */
int hv_op_gemm_batched_b(const void* A, int64_t lda, const void* X, int64_t ldx, void* out, int64_t ldc, int64_t M, int64_t batch,
                         int64_t rows, int64_t out_stride, int64_t K, const void* rowbias /* fp16 [M] added to row m, or NULL */,
                         hv_stream_t stream);

/* The small-channel 3x3 convolutions of the PoseGuider front (src/models/pose_guider.py:25-49) at their true channel counts (HBM-bound
 * layers at up to full image resolution; mma.sync implicit GEMM over a shared-memory halo tile): (Cin, Cout, stride) in
 * {(16,16,1), (16,32,2), (32,32,1), (32,96,2)}, padding 1, + bias, act.  X (NF, H, W, Cin) channels-last; Wp = hv_pack_conv3x3 with
 * Cin_pad = Cin, Cout_pad = Cout ([Cout][9 * Cin]); out (NF, Ho, Wo, ldo >= Cout), columns >= Cout are left untouched.
 * hv_op_pose_conv_in: the PoseGuider's conv_in (3 -> 16) read straight from the (B, 3, F, H, W) image, W in the reference layout (16,3,3,3),
 * out channels-last (B*F, H, W, 16).
 * HV_ERR_INVALID (hv_op_conv3x3_small) for: another (Cin, Cout, stride); X, Wp or out NULL or not 16-byte aligned; NF outside [1, 65535]; H or W
 * < 1 or odd at stride 2; more than 65535 rows of 8 output rows; ldo < Cout or not a multiple of 8.
 * HV_ERR_INVALID (hv_op_pose_conv_in) for: X, W or out NULL, out not 16-byte aligned, B, F, H or W < 1, B*F or H*W past int32. */
int hv_op_conv3x3_small(const void* X, const void* Wp, const void* bias, void* out, int64_t ldo, int64_t NF, int64_t H, int64_t W, int64_t Cin,
                        int64_t Cout, int32_t stride, int32_t act, hv_stream_t stream);
int hv_op_pose_conv_in(const void* X, const void* W, const void* bias, void* out, int64_t B, int64_t F, int64_t H, int64_t W_, int32_t act,
                       hv_stream_t stream);

/* Upsample3D (src/models/resnet.py:29-88): nearest 2x upsample followed by the 3x3 convolution, WITHOUT materialising the upsampled
 * tensor: every output parity (2y+py, 2x+px) is a 2x2 convolution of the source whose weights are sums of the 3x3 taps that land on
 * the same source pixel (4/9 of the multiply-adds; the summed weights are rounded to fp16 once, at packing).
 * X (NF, H, W, Cin) -> out (NF, 2H, 2W, Cout) given as [rows][ldc]; Wp = hv_pack_upconv2x2(W (Cout, Cin, 3, 3)) : [4][Cout][4 * Cin].
 * Epilogue: bias only.  Cin % 64 == 0; Cout a multiple of the 128/160/256-column tile the GEMM picks (320, 640, 1280 are).  HV_ERR_INVALID
 * for NULL pointers, the shapes above and NF, H or W <= 0; hv_pack_upconv2x2 for NULL pointers and Cout or Cin outside [1, INT32_MAX]. */
int hv_op_upconv2x2(const void* X, const void* Wp, void* out, int64_t ldc, int64_t NF, int64_t H, int64_t W, int64_t Cin, int64_t Cout,
                    const hv_epilogue* ep, hv_stream_t stream);
int hv_pack_upconv2x2(const void* W, void* out, int64_t Cout, int64_t Cin, hv_stream_t stream);

/* 3x3 convolution, padding 1, stride 1 or 2, over channels-last X (NF, H, W, Cin) -> out (NF, Ho, Wo, Cout) given as
 * a [rows][ldc] matrix.  Wp is the packed weight [Cout][9 * Cin] with k = (ky*3 + kx) * Cin + c (see hv_pack_conv3x3).
 * Cin must be a multiple of 64; stride 2 needs even H and W.  HV_ERR_INVALID for: X, Wp or out NULL, Cin % 64, Cout or ldc % 8, a stride
 * other than 1 or 2, NF, H or W <= 0, the epilogue I/O hv_epilogue rejects, and a geglu epilogue when the GEMM picks a tile narrower than
 * 256 columns for Cout. */
int hv_op_conv3x3(const void* X, const void* Wp, void* out, int64_t ldc, int64_t NF, int64_t H, int64_t W, int64_t Cin,
                  int64_t Cout, int32_t stride, const hv_epilogue* ep, hv_stream_t stream);

/* AutoencoderKL's Downsample2D: F.pad(x, (0, 1, 0, 1)) then a 3x3 convolution with stride 2 and padding 0, i.e. hv_op_conv3x3 at stride 2
 * with the padding at the bottom / right only (no padded copy is made; the rows / columns past the end read as zero).  Same X, Wp, out and
 * epilogue conventions as hv_op_conv3x3; H and W must be even, the output is (NF, H/2, W/2, Cout). */
int hv_op_conv3x3_s2_pad_end(const void* X, const void* Wp, void* out, int64_t ldc, int64_t NF, int64_t H, int64_t W, int64_t Cin, int64_t Cout,
                             const hv_epilogue* ep, hv_stream_t stream);

/* Patches of a stride-p, p x p convolution (CLIP's patch embedding) as the rows of a GEMM operand: X (B, C, S, S) fp16 NCHW, S % p == 0 ->
 * out [B * (S/p)^2][Kpad], row (b, gy, gx) in raster order, column k = c p^2 + ky p + kx holding X[b][c][gy p + ky][gx p + kx]; columns
 * [C p^2, Kpad) are written as zero.  Kpad >= C p^2 and a multiple of 8.  hv_op_gemm of this with the conv weight flattened to [hidden][C p^2]
 * and zero-padded to [hidden][Kpad] is the convolution, one output row per patch. */
int hv_op_clip_patchify(const void* X, void* out, int64_t B, int64_t C, int64_t S, int64_t p, int64_t Kpad, hv_stream_t stream);

/* Small-channel direct 3x3 convolution (any Cin/Cout, stride 1/2, padding 1) for conv_in and the PoseGuider stack.
 * W is the reference layout (Cout, Cin, 3, 3) fp16; act = hv_act.  HV_ERR_INVALID for: X, W or out NULL, a stride other than 1 or 2, NF < 1,
 * H, W, Cin or Cout outside [1, INT32_MAX]. */
int hv_op_conv3x3_direct(const void* X, const void* W, const void* bias, void* out, int64_t NF, int64_t H, int64_t Wd,
                         int64_t Cin, int64_t Cout, int32_t stride, int32_t act, const void* add, hv_stream_t stream);

/* GroupNorm over (H*W, C/groups) per frame, fp32 statistics (summed relative to one input value of the group, so a large mean does not
 * cancel the variance); optional SiLU; reads the channel concatenation of X
 * (C1 channels) and X2 (C2 channels, may be NULL/0) and writes one (NF, HW, C1+C2) tensor. stats: fp32 scratch
 * of hv_groupnorm_scratch_floats(...) floats (per-slab partial sums; the reduction is atomics-free and deterministic).
 * HV_ERR_INVALID, writing nothing, for what hv_op_groupnorm_pooled rejects at frames_per_item = 1. */
size_t hv_groupnorm_scratch_floats(int64_t C, int64_t NF, int64_t HW, int32_t groups);
int hv_op_groupnorm(const void* X, int64_t C1, const void* X2, int64_t C2, const void* gamma, const void* beta, void* out,
                    int64_t NF, int64_t HW, int32_t groups, float eps, int32_t silu, float* stats, hv_stream_t stream);
/* GroupNorm whose statistics span every frame of a batch item: nn.GroupNorm on a (b, c, f, h, w) tensor (unet_3d.py:235-246 and
 * resnet.py:153-190 with use_inflated_groupnorm=False).  Same layout and options as hv_op_groupnorm; frames [b*F, (b+1)*F) of the
 * (NF, HW, C1+C2) input are item b, F = frames_per_item.  One pivot per (item, group): the group's first channel in the first row of the
 * item's first frame.  The summation order depends on (F, HW, C) only, never on NF / F, so an item's output does not depend on the other
 * items in the call.  At F = 1 this is hv_op_groupnorm, bit for bit.  stats: hv_groupnorm_pooled_scratch_floats(...) fp32.
 * Returns HV_ERR_INVALID and writes nothing for: NULL pointers (X2 may be NULL only when C2 == 0), NF, HW or F <= 0, NF % F != 0,
 * NF > 65535, X / X2 / gamma / beta / out not 16-byte aligned or stats not 8-byte aligned, and the channel layouts hv_op_groupnorm cannot
 * run (C1 + C2 and C1 multiples of 8, C1 + C2 <= 8192, C / groups even, groups <= 256 and <= the block's thread count). */
size_t hv_groupnorm_pooled_scratch_floats(int64_t C, int64_t NF, int64_t HW, int32_t groups, int64_t frames_per_item);
int hv_op_groupnorm_pooled(const void* X, int64_t C1, const void* X2, int64_t C2, const void* gamma, const void* beta, void* out,
                           int64_t NF, int64_t HW, int32_t groups, float eps, int32_t silu, int64_t frames_per_item, float* stats,
                           hv_stream_t stream);

/* LayerNorm over C per row.  Optional: `pre_add` fp16 [ceil(rows / rows_per_group)][C] (row r adds row r / rows_per_group) is added to
 * x first and the sum is written to `x_out` (the cross-attention residual, see DESIGN.md; x_out is written only with pre_add; the
 * statistics use the unrounded fp32 sum); `pe` fp16 [F][C] is added to the normalised row
 * (row -> frame (row / hw) % F) as the motion module does before q/k/v.  HV_ERR_INVALID for: X, gamma, beta or out NULL, any tensor
 * (pre_add, x_out and pe included) not 16-byte aligned, rows < 1, C not a multiple of 8 in [8, 1280], hw or F past INT32_MAX. */
int hv_op_layernorm(const void* X, const void* gamma, const void* beta, void* out, int64_t rows, int64_t C, float eps,
                    const void* pre_add, int64_t rows_per_group, void* x_out, const void* pe, int64_t hw, int64_t F,
                    hv_stream_t stream);

/* Spatial multi-head attention.  Q: [NF*L][ldq] (head h at columns h*dpad, dpad = d rounded up to 16, pad columns zero), K
 * likewise.  Vt: [heads*dv][ldvt], dv = (d+1) rounded up to 16: rows h*dv..h*dv+d-1 = V of head h transposed, row h*dv+d = ONES (its
 * P*V column is the softmax denominator), remaining rows zero; holding
 * V transposed: frame n's tokens occupy columns [n*vt_stride, n*vt_stride + L), vt_stride % 8 == 0.  Optional bank keys/values per batch item (frame n uses bank n / F):
 * Kb [B][Lb][ldkb], Vbt [heads*dv][B*vbt_stride] (same row layout).  Frames with n < nf_nobank attend to their own L keys only (the
 * unconditional CFG half).  out: [NF*L][ldo], columns [0, heads*d) written.  d is one of 8, 16, 32, 40, 64, 80, 160; other head dims
 * return an error.  Kb = NULL or Lb = 0 means no bank (the other bank arguments are then ignored).
 * A frame's last key tile of 128 is read whole: when L % 128 != 0 the columns [L, vt_stride) of its V^T segment (and the first columns of
 * the next frame's segment) are loaded and multiplied by P = 0, and likewise [Lb, vbt_stride) of a bank item's segment.  Those columns
 * must hold finite values (NaN or Inf times 0 is NaN); hv_op_gemm_batched_b writes the pad [rows, round8(rows)) as 0 + rowbias, which
 * meets this with vt_stride = round8(L).  Columns at or past NF*vt_stride (B*vbt_stride) are never read.
 * HV_ERR_INVALID unless: the pointers are non-NULL; 1 <= NF <= 65535, 1 <= heads <= 65535, L >= 1, NF*L and NF*vt_stride fit an int32;
 * 0 <= nf_nobank <= NF; ldo >= heads*d; ldq, ldk >= heads*dpad; ldvt >= NF*vt_stride; vt_stride >= L.  With a bank also: Vbt non-NULL,
 * F >= 1 divides NF (B = NF/F), vbt_stride >= Lb, ldkb >= heads*dpad, ldvbt >= B*vbt_stride. */
int hv_op_attention(const void* Q, const void* K, const void* Vt, void* out, int64_t NF, int64_t L, int32_t heads,
                    int32_t d, int64_t ldq, int64_t ldk, int64_t ldvt, int64_t ldo, const void* Kb, const void* Vbt,
                    int64_t Lb, int64_t ldkb, int64_t ldvbt, int64_t F, int64_t nf_nobank, int64_t vt_stride, int64_t vbt_stride,
                    hv_stream_t stream);

/* Single-head attention with d = 512 (the mid-block attention of AutoencoderKL): out = softmax(Q K^T / sqrt(512)) V over the L tokens of
 * each of NF frames, softmax statistics in fp32, P rounded to fp16 for P*V.  Q: [NF*L][ldq] and K: [NF*L][ldk] (512 columns used);
 * Vt: [512][ldvt] = V transposed, frame n's tokens in columns [n*vt_stride, n*vt_stride + L) (vt_stride % 8 == 0, >= L; the
 * layout hv_op_gemm_batched_b writes); out: [NF*L][ldo].  Any L >= 1. */
int hv_op_attention_d512(const void* Q, int64_t ldq, const void* K, int64_t ldk, const void* Vt, int64_t ldvt, int64_t vt_stride, void* out,
                         int64_t ldo, int64_t NF, int64_t L, hv_stream_t stream);

/* Attention over the frame axis: tokens are rows (b, f, p) of QKV [B*F*HW][3*C] (q | k | v), one problem per
 * (b, p, head) with F <= 32 keys. out [B*F*HW][C].  HV_ERR_INVALID unless the pointers are non-NULL, B, HW, heads >= 1, 1 <= F <= 32,
 * d is one of 8, 16, 32, 40, 80, 160 and B*F*HW and B*HW*heads fit an int32. */
int hv_op_temporal_attention(const void* QKV, void* out, int64_t B, int64_t F, int64_t HW, int32_t heads, int32_t d,
                             hv_stream_t stream);

/* Layout / glue kernels.  HV_ERR_INVALID for: NULL pointers, B, C, F, H or W < 1, H*W past int32, B*F > 65535 (ncfhw_to_nhwc,
 * nhwc_to_ncfhw; also ldx < C), and for pixel_unshuffle r < 1 or not dividing H and W, or B*F, C*r*r past int32. */
int hv_op_ncfhw_to_nhwc(const void* X, void* out, int64_t B, int64_t C, int64_t F, int64_t H, int64_t W, int32_t src_fp32,
                        hv_stream_t stream);
int hv_op_nhwc_to_ncfhw(const void* X, int64_t ldx, void* out, int64_t B, int64_t C, int64_t F, int64_t H, int64_t W,
                        hv_stream_t stream);
int hv_op_pixel_unshuffle(const void* X, void* out, int64_t B, int64_t C, int64_t F, int64_t H, int64_t W, int32_t r,
                          hv_stream_t stream);
/* Plucker-embedding producer on the device (Camera + ray_condition, src/dataset/dance_image_h_v_camera.py:17-130; called from
 * scripts/pose2vid.py:52-84) fused with CameraPoseEncoder's PixelUnshuffle(r) (pose_adaptor.py:222,233-236):
 * K: DEVICE fp32 [NF][4] = (fx, fy, cx, cy) in pixels; c2w: DEVICE fp32 [NF][16] row-major camera-to-world (relative poses);
 * out: channels-last fp16 (NF, H/r, W/r, 6*r*r) with channel = c*r*r + dy*r + dx, i.e. pixel_unshuffle(plucker (NF, 6, H, W)).
 * HV_ERR_INVALID for NULL pointers, NF < 1, r < 1 or not dividing H and W, H or W past INT32_MAX. */
int hv_op_plucker_unshuffle(const float* K, const float* c2w, void* out, int64_t NF, int64_t H, int64_t W, int32_t r, hv_stream_t stream);
/* y[M][N] = act_in(x[M][K]) * W[N][K]^T + bias, tiny M (time embedding, cross-attention collapse); fp32 math,
 * fp16 rounding of the result. act_in: hv_act applied to x first.  HV_ERR_INVALID for: X, W or out NULL, X or W not 4-byte aligned, M, N,
 * K outside [1, INT32_MAX], K odd, more than INT32_MAX blocks of 8 outputs. */
int hv_op_small_linear(const void* X, const void* W, const void* bias, void* out, int64_t M, int64_t N, int64_t K,
                       int32_t act_in, hv_stream_t stream);
/* Timesteps(320, flip_sin_to_cos=True, shift=0): out[b] = [cos(t w_i) | sin(t w_i)] rounded to fp16.  HV_ERR_INVALID for NULL out, B < 1,
 * dim < 2 or odd, B*dim past INT32_MAX. */
int hv_op_timestep_embedding(int64_t timestep, void* out, int64_t B, int64_t dim, hv_stream_t stream);

/* ---- per-timestep glue of Pose2VideoPipeline.__call__ on the device (src/pipelines/pipeline_pose2vid_long.py:516-563) ----
 * hv_op_window_gather: out[(r*Bl + b), c, i] = latents[b, c, frame_idx[i]] for r < repeat -- `latents[:, :, c].repeat(2, ...)` (:516-523).
 *   latents (Bl, C, Ftot, HW) fp16; frame_idx: DEVICE int32[Fw]; out (repeat*Bl, C, Fw, HW) fp16.
 * hv_op_cfg_ddim_step: for every latent element, mean over the windows that contain its frame of the window predictions
 *   (`noise_pred[:, :, c] += pred; counter[:, :, c] += 1; noise_pred / counter`, :550-556), classifier-free guidance
 *   `uncond + s (text - uncond)` (:557-559; skipped when pred_cond == NULL) and the DDIM update with eta = 0 (:561-563;
 *   diffusers DDIMScheduler.step): x0, eps from the model output (prediction_type 0 = v_prediction, 1 = epsilon),
 *   x_prev = sqrt(a_prev) x0 + sqrt(1 - a_prev) eps, all in fp32, latents updated in place (one fp16 rounding).
 *   pred_uncond / pred_cond: HOST arrays of n_windows device pointers, each (Bl, C, Fw, HW) fp16 (the two halves of a
 *   CFG-doubled UNet output are pred and pred + Bl*C*Fw*HW); inv: DEVICE int32 [Ftot][K], entry = window*Fw + position of
 *   a window slot holding that frame, or -1; coef: DEVICE float [steps][4] = sqrt(a_t), sqrt(1-a_t), sqrt(a_prev),
 *   sqrt(1-a_prev); step_index: DEVICE int32 (row of coef used; NULL = row 0), read when the kernel runs so that a captured
 *   CUDA graph of one step replays for every timestep.
 * hv_op_advance_index: *index += 1 on the device (end of a graph-captured step).
 * HV_ERR_INVALID for NULL pointers (a NULL prediction of a window included), Bl, C, Ftot, Fw or HW outside [1, INT32_MAX], repeat < 1,
 * n_windows outside [1, 32], K < 1, another prediction_type and a coef table not 16-byte aligned. */
int hv_op_window_gather(const void* latents, const int32_t* frame_idx, void* out, int64_t Bl, int64_t C, int64_t Ftot, int64_t Fw, int64_t HW,
                        int32_t repeat, hv_stream_t stream);
int hv_op_cfg_ddim_step(const void* const* pred_uncond, const void* const* pred_cond, int32_t n_windows, const int32_t* inv, int32_t K,
                        const float* coef, const int32_t* step_index, void* latents, int64_t Bl, int64_t C, int64_t Ftot, int64_t Fw, int64_t HW,
                        float guidance_scale, int32_t prediction_type, hv_stream_t stream);
int hv_op_advance_index(int32_t* index, hv_stream_t stream);

/* Weight packing (device to device).  conv: fp16 (Cout, Cin, 3, 3) -> [Cout_pad][9*Cin_pad] (zero padded); geglu: rows of a [8C][K] matrix
 * (and its bias) interleaved in 128-row hidden/gate blocks; heads: [heads*d][K] -> [heads*dpad][K] with zero rows.  HV_ERR_INVALID for
 * NULL pointers, sizes < 1 or past INT32_MAX, a padded size below its true size, and geglu rows not a multiple of 256. */
int hv_pack_conv3x3(const void* W, void* out, int64_t Cout, int64_t Cin, int64_t Cout_pad, int64_t Cin_pad, hv_stream_t stream);
int hv_pack_geglu(const void* W, void* out, int64_t rows, int64_t K, hv_stream_t stream);
int hv_pack_heads(const void* W, void* out, int32_t heads, int32_t d, int32_t dpad, int64_t K, hv_stream_t stream);

/* Debug cross-checks (slow CUDA-core kernels, used by tests to localise a fault on the device). */
int hv_dbg_gemm(const void* A, int64_t lda, const void* W, float* out, int64_t M, int64_t N, int64_t K, hv_stream_t stream);
/* The launch hv_op_gemm makes for an M x N x K linear on this device (the same host function decides both): the CTA tile width
 * *block_n (128, 160 or 256), *bst_stages > 0 for the B-stationary variant (the CTA's N x K weight panel stays in shared memory and
 * A streams through that many stages) or 0 for the ring variant, and the persistent *grid.  Launches nothing. */
int hv_dbg_gemm_plan(int64_t M, int64_t N, int64_t K, int32_t geglu, int32_t* block_n, int32_t* bst_stages, int32_t* grid);
/* The launch hv_op_temporal_attention makes for these arguments on this device (the same host function decides both): *tma = 1 for the
 * TMA-staged kernel (HW*heads >= 2048 and d = 80, or d = 40 with even heads) with *heads_per_box heads fetched per box and a persistent
 * *grid of at most one CTA per SM, or *tma = 0 for the register kernel (one warp per problem, *grid blocks of 8).  Launches nothing. */
int hv_dbg_temporal_attention_plan(int64_t B, int64_t F, int64_t HW, int32_t heads, int32_t d, int32_t* tma, int32_t* heads_per_box, int32_t* grid);

const char* hv_ops_last_error(void);
int hv_num_sms(void);

#ifdef __cplusplus
}
#endif
#endif
