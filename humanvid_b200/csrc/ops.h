// The operator layer: one function per operator, defined next to its kernel, shared by the operator C ABI (capi_ops.cu) and the model
// runtime (model.cu).  Each checks its arguments before any CUDA call, then plans and launches; it returns an hv_status
// (include/hv_b200_ops.h) and records a message that names the operator.  Arguments mirror the hv_op_* / hv_pack_* entry points.
#pragma once
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/hv_b200_fp8.h"
#include "../../include/hv_b200_ops.h"

namespace hv {

int device_sms();
void set_error(const char* fmt, ...);
const char* last_error();
// HV_OK for cudaSuccess, else HV_ERR_CUDA with "what: <CUDA message>"
int cuda_status(cudaError_t e, const char* what);
inline bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; }
inline bool int32_ok(int64_t v) { return v >= 1 && v <= INT32_MAX; }   // a size >= 1 that an int holds

// ---- GEMM / implicit-GEMM convolution (ops.cu)
// The tile width and launch plan op_gemm would use for out[M, N] = A[M, K] W[N, K]^T (bst_stages 0: ring variant).
int plan_linear(int64_t M, int64_t N, int64_t K, bool geglu, int* block_n, int* bst_stages, int* grid);
int op_gemm(const __half* A, int64_t lda, const __half* A2, int64_t lda2, int64_t K1, const __half* W, __half* out, int64_t ldc,
            int64_t M, int64_t N, int64_t K, const hv_epilogue* ep, cudaStream_t stream);
// out[M][n*out_stride + j] = sum_k A[M][k] * X[n][j][k] for n < batch, j < rows (X: [batch][rows][ldx]); out_stride % 8 == 0.
// e4m3 operands with fp32 scales (hv_op_gemm_fp8): out is fp16 [M][ldc], or e4m3 [M][ldc] with out_scale for a GEGLU epilogue.
int op_gemm_fp8(const uint8_t* A, int64_t lda, const float* a_scale, int64_t a_scale_ld, const uint8_t* W, const float* w_scale, void* out,
                int64_t ldc, float* out_scale, int64_t out_scale_ld, int64_t M, int64_t N, int64_t K, const hv_epilogue* ep, cudaStream_t stream);
int op_gemm_batched_b(const __half* A, int64_t lda, const __half* X, int64_t ldx, __half* out, int64_t ldc, int64_t M, int64_t batch,
                      int64_t rows, int64_t out_stride, int64_t K, const __half* rowbias, cudaStream_t stream);
// pad_end (stride 2 only): padding (0, 1, 0, 1) instead of 1 on every side -- F.pad(x, (0, 1, 0, 1)) then a stride-2 conv with padding 0.
int op_conv3x3(const __half* X, const __half* Wp, __half* out, int64_t ldc, int64_t NF, int64_t H, int64_t W, int64_t Cin,
               int64_t Cout, int stride, const hv_epilogue* ep, cudaStream_t stream, bool pad_end = false);
// out (NF, 2H, 2W, Cout) = conv3x3(nearest_upsample_2x(X (NF, H, W, Cin))) + bias; Wp from op_pack_upconv2x2: [4][Cout][4 * Cin].
int op_upconv2x2(const __half* X, const __half* Wp, __half* out, int64_t ldc, int64_t NF, int64_t H, int64_t W, int64_t Cin, int64_t Cout,
                 const hv_epilogue* ep, cudaStream_t stream);

// ---- attention (attn_spatial.cu, attn_vae.cu, attn_temporal.cu)
int op_attention(const __half* Q, const __half* K, const __half* Vt, __half* out, int64_t NF, int64_t L, int heads, int d, int64_t ldq,
                 int64_t ldk, int64_t ldvt, int64_t ldo, const __half* Kb, const __half* Vbt, int64_t Lb, int64_t ldkb, int64_t ldvbt, int64_t F,
                 int64_t nf_nobank, int64_t vt_stride, int64_t vbt_stride, cudaStream_t stream);
int op_attention_d512(const __half* Q, int64_t ldq, const __half* K, int64_t ldk, const __half* Vt, int64_t ldvt, int64_t vt_stride, __half* out,
                      int64_t ldo, int64_t NF, int64_t L, cudaStream_t stream);
int op_temporal_attention(const __half* QKV, __half* out, int64_t B, int64_t F, int64_t HW, int heads, int d, cudaStream_t stream);
// The kernel op_temporal_attention runs (one host function decides both the launch and hv_dbg_temporal_attention_plan): the
// TMA-staged kernel with heads_per_box heads per (pixel, box) and a persistent grid of at most one CTA per SM, or the register kernel,
// one warp per (batch item, pixel, head).  `what` names the caller in the message of a rejected shape.
struct TemporalPlan {
  bool tma;
  int heads_per_box;
  unsigned grid;
};
int plan_temporal_attention(const char* what, int64_t B, int64_t F, int64_t HW, int heads, int d, TemporalPlan* plan);

// ---- normalisation (norm.cu)
size_t groupnorm_scratch_floats(int C, int NF, int HW, int groups);
int op_groupnorm(const __half* X, int64_t C1, const __half* X2, int64_t C2, const __half* gamma, const __half* beta, __half* out, int64_t NF,
                 int64_t HW, int groups, float eps, int silu, float* stats, cudaStream_t stream);
int op_groupnorm_pooled(const __half* X, int64_t C1, const __half* X2, int64_t C2, const __half* gamma, const __half* beta, __half* out,
                        int64_t NF, int64_t HW, int groups, float eps, int silu, int64_t F, float* stats, cudaStream_t stream);
int op_layernorm(const __half* X, const __half* gamma, const __half* beta, __half* out, int64_t rows, int64_t C, float eps, const __half* pre_add,
                 int64_t rows_per_group, __half* x_out, const __half* pe, int64_t hw, int64_t F, cudaStream_t stream);
int op_layernorm_fp8(const __half* X, const __half* gamma, const __half* beta, uint8_t* out, float* out_scale, int64_t rows, int64_t C, float eps,
                     const __half* pre_add, int64_t rows_per_group, __half* x_out, const __half* pe, int64_t hw, int64_t F, cudaStream_t stream);
// CLIP vision embeddings: row (b, t) of B x L tokens = LayerNorm((t == 0 ? cls : patch[b * (L - 1) + t - 1]) + pos[t]); rows = B * L.
int op_clip_embed_ln(const __half* patch, const __half* cls, const __half* pos, const __half* gamma, const __half* beta, __half* out, int64_t rows,
                     int64_t L, int64_t C, float eps, cudaStream_t stream);

// ---- layout, glue, direct convolutions and weight packing (misc.cu)
// ldo: row stride of out (0 = C); channels C .. ldo are left untouched.
int op_ncfhw_to_nhwc(const void* X, __half* out, int64_t B, int64_t C, int64_t F, int64_t H, int64_t W, int src_fp32, cudaStream_t stream,
                     int64_t ldo = 0);
int op_nhwc_to_ncfhw(const __half* X, int64_t ldx, __half* out, int64_t B, int64_t C, int64_t F, int64_t H, int64_t W, cudaStream_t stream);
int op_pixel_unshuffle(const __half* X, __half* out, int64_t B, int64_t C, int64_t F, int64_t H, int64_t W, int r, cudaStream_t stream);
int op_plucker_unshuffle(const float* K, const float* c2w, __half* out, int64_t NF, int64_t H, int64_t W, int r, cudaStream_t stream);
int op_small_linear(const __half* X, const __half* W, const __half* bias, __half* out, int64_t M, int64_t N, int64_t K, int act_in,
                    cudaStream_t stream);
// table != NULL: the timestep is table[*index], read on the device (graph replay of a denoising loop)
int op_timestep_embedding(int64_t timestep, const long long* table, const int* index, __half* out, int64_t B, int64_t dim, cudaStream_t stream);
// ldo: row stride of out (>= Cout; the channels past Cout are left untouched); add: NULL or a tensor of out's layout added last
int op_conv3x3_direct(const __half* X, const __half* W, const __half* bias, __half* out, int64_t NF, int64_t H, int64_t Wd, int64_t Cin,
                      int64_t Cout, int stride, int act, const __half* add, int64_t ldo, cudaStream_t stream);
int op_clip_patchify(const __half* X, __half* out, int64_t B, int64_t C, int64_t S, int64_t p, int64_t Kpad, cudaStream_t stream);
int op_pack_conv3x3(const __half* W, __half* out, int64_t Cout, int64_t Cin, int64_t Cout_pad, int64_t Cin_pad, cudaStream_t stream);
int op_pack_upconv2x2(const __half* W, __half* out, int64_t Cout, int64_t Cin, cudaStream_t stream);
int op_pack_geglu(const __half* W, __half* out, int64_t rows, int64_t K, cudaStream_t stream);
int op_pack_heads(const __half* W, __half* out, int heads, int d, int dpad, int64_t K, cudaStream_t stream);
int op_pack_fp8_rows(const __half* W, uint8_t* out, float* scale, int64_t rows, int64_t K, cudaStream_t stream);
int op_dbg_gemm(const __half* A, int64_t lda, const __half* W, float* out, int64_t M, int64_t N, int64_t K, cudaStream_t stream);

// ---- small-channel convolutions of the PoseGuider front (smallconv.cu)
bool smallconv_supported(int64_t cin, int64_t cout, int stride);
int op_conv3x3_small(const __half* X, const __half* Wp, const __half* bias, __half* out, int64_t ldo, int64_t NF, int64_t H, int64_t W, int64_t Cin,
                     int64_t Cout, int stride, int act, cudaStream_t stream);
int op_pose_conv_in(const __half* X, const __half* W, const __half* bias, __half* out, int64_t B, int64_t F, int64_t H, int64_t Wd, int act,
                    cudaStream_t stream);

// ---- per-timestep glue of the denoising loop (step.cu)
int op_window_gather(const __half* latents, const int32_t* frame_idx, __half* out, int64_t Bl, int64_t C, int64_t Ftot, int64_t Fw, int64_t HW,
                     int repeat, cudaStream_t stream);
int op_cfg_ddim_step(const void* const* pred_uncond, const void* const* pred_cond, int n_windows, const int32_t* inv, int K, const float* coef,
                     const int32_t* step_index, __half* latents, int64_t Bl, int64_t C, int64_t Ftot, int64_t Fw, int64_t HW, float guidance_scale,
                     int prediction_type, cudaStream_t stream);
int op_advance_index(int32_t* index, cudaStream_t stream);

}  // namespace hv
