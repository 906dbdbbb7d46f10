// Internal launcher declarations shared by the operator C ABI (capi_ops.cu) and the model runtime (model.cu).
#pragma once
#include <cuda_fp16.h>
#include <cuda_runtime.h>

namespace hv {

cudaError_t launch_groupnorm(const __half* x1, int C1, const __half* x2, int C2, const __half* gamma, const __half* beta,
                             __half* out, int NF, int HW, int groups, float eps, int silu, float* stats, cudaStream_t stream);
size_t groupnorm_scratch_floats(int C, int NF, int HW, int groups);
// GroupNorm whose statistics span the F frames of each batch item (frames [b*F, (b+1)*F) are item b); NF % F == 0.  Takes the scratch of
// groupnorm_scratch_floats(C, NF, HW, groups); at F = 1 it is launch_groupnorm.
cudaError_t launch_groupnorm_pooled(const __half* x1, int C1, const __half* x2, int C2, const __half* gamma, const __half* beta,
                                    __half* out, int NF, int HW, int groups, float eps, int silu, int F, float* stats, cudaStream_t stream);
// The channel / group layouts both GroupNorm launchers accept.
bool groupnorm_shape_ok(int C1, int C2, int HW, int groups);
cudaError_t launch_layernorm(const __half* x, const __half* gamma, const __half* beta, __half* out, long long rows, int C, float eps,
                             const __half* pre_add, long long rows_per_group, __half* x_out, const __half* pe, int hw, int F,
                             cudaStream_t stream);
// CLIP vision embeddings: row (b, t) of B x L tokens = LayerNorm((t == 0 ? cls : patch[b * (L - 1) + t - 1]) + pos[t]); rows = B * L.
cudaError_t launch_clip_embed_ln(const __half* patch, const __half* cls, const __half* pos, const __half* gamma, const __half* beta, __half* out,
                                 long long rows, int L, int C, float eps, cudaStream_t stream);
cudaError_t launch_temporal_attention(const __half* qkv, __half* out, int B, int F, int HW, int heads, int d, cudaStream_t stream);
// The kernel launch_temporal_attention runs (one host function decides both the launch and hv_dbg_temporal_attention_plan): the
// TMA-staged kernel with heads_per_box heads per (pixel, box) and a persistent grid of at most `sms` CTAs, or the register kernel,
// one warp per (batch item, pixel, head).
struct TemporalPlan {
  bool tma;
  int heads_per_box;
  unsigned grid;
};
TemporalPlan plan_temporal_attention(int B, int HW, int heads, int d, int sms);

struct AttnArgs {
  const __half* q; const __half* k; const __half* vt; __half* out;
  int NF, L, heads, d, dpad;
  long long ldq, ldk, ldvt, ldo;
  const __half* kb; const __half* vbt;   // bank keys [B][Lb][ldkb], bank values transposed [heads*d][ldvbt]
  int Lb; long long ldkb, ldvbt;
  int F, nf_nobank;
  long long vt_stride, vbt_stride;       // columns between consecutive frames / bank items in V^T (multiples of 8)
};
cudaError_t launch_attention(const AttnArgs& a, int num_sms, cudaStream_t stream);
// Single-head attention, d = 512 (AutoencoderKL mid block, attn_vae.cu): Q [NF*L][ldq], K [NF*L][ldk], V^T [512][ldvt] with frame n's
// tokens at columns [n*vt_stride, n*vt_stride + L), out [NF*L][ldo]; scale 512^-1/2.
cudaError_t launch_attention_d512(const __half* q, long long ldq, const __half* k, long long ldk, const __half* vt, long long ldvt, long long vt_stride,
                                  __half* out, long long ldo, int NF, int L, cudaStream_t stream);

cudaError_t launch_ncfhw_to_nhwc(const void* x, __half* out, int B, int C, int F, int H, int W, int src_fp32, cudaStream_t s, int ldo = 0);
cudaError_t launch_nhwc_to_ncfhw(const __half* x, int ldx, __half* out, int B, int C, int F, int H, int W, cudaStream_t s);
cudaError_t launch_pixel_unshuffle(const __half* x, __half* out, int B, int C, int F, int H, int W, int r, int num_sms, cudaStream_t s);
cudaError_t launch_plucker_unshuffle(const float* K, const float* c2w, __half* out, long long NF, int H, int W, int r, int num_sms, cudaStream_t s);
cudaError_t launch_small_linear(const __half* x, const __half* w, const __half* bias, __half* out, int M, int N, int K, int act_in,
                                cudaStream_t s);
cudaError_t launch_timestep_embedding(long long timestep, const long long* table, const int* index, __half* out, int B, int dim, cudaStream_t s);
cudaError_t launch_conv3x3_direct(const __half* x, const __half* w, const __half* bias, __half* out, long long NF, int H, int W, int Cin,
                                  int Cout, int stride, int act, const __half* add, int num_sms, cudaStream_t s);
cudaError_t launch_pack_conv3x3(const __half* w, __half* out, int Cout, int Cin, int Cout_pad, int Cin_pad, int num_sms, cudaStream_t s);
cudaError_t launch_conv3x3_direct_padded(const __half* x, const __half* w, const __half* bias, __half* out, long long NF, int H, int W,
                                         int Cin, int Cout, int ldo, int act, int num_sms, cudaStream_t s);
cudaError_t launch_pack_upconv2x2(const __half* w, __half* out, int Cout, int Cin, int num_sms, cudaStream_t s);
cudaError_t launch_pack_geglu(const __half* w, __half* out, int rows, int K, int num_sms, cudaStream_t s);
cudaError_t launch_pack_heads(const __half* w, __half* out, int heads, int d, int dpad, int K, int num_sms, cudaStream_t s);
// pixels (B, Cin, S, S) -> [B * (S/p)^2][Kpad] patch rows, k = c p^2 + ky p + kx, pad columns zero (see hv_op_clip_patchify)
cudaError_t launch_clip_patchify(const __half* x, __half* out, int B, int Cin, int S, int p, int Kpad, int num_sms, cudaStream_t s);
// ---- small-channel convolutions of the PoseGuider front (smallconv.cu)
bool smallconv_supported(int cin, int cout, int stride);
cudaError_t launch_smallconv(const __half* x, const __half* wp, const __half* bias, __half* out, int NF, int H, int W, int cin, int cout, int stride,
                             int ldo, int act, cudaStream_t s);
cudaError_t launch_pg_conv_in(const __half* x, const __half* w, const __half* bias, __half* out, int B, int F, int H, int W, int act, int num_sms,
                              cudaStream_t s);

// ---- per-timestep glue of the denoising loop (step.cu)
constexpr int kMaxWindows = 32;
struct StepPreds {                       // window w's UNet prediction, (Bl, C, Fw, HW) fp16 each; cond unused without CFG
  const __half* uncond[kMaxWindows];
  const __half* cond[kMaxWindows];
};
cudaError_t launch_window_gather(const __half* latents, const int* idx, __half* out, int Bl, int C, int Ftot, int Fw, int HW, int R, int num_sms,
                                 cudaStream_t s);
cudaError_t launch_cfg_ddim_step(const StepPreds& preds, const int* inv, int K, const float* coef, const int* step_idx, __half* latents, int Bl, int C,
                                 int Ftot, int Fw, int HW, float guidance, int cfg, int epsilon, int num_sms, cudaStream_t s);
cudaError_t launch_advance_index(int* idx, cudaStream_t s);

cudaError_t launch_dbg_gemm(const __half* a, long long lda, const __half* w, float* out, int M, int N, int K, cudaStream_t s);

}  // namespace hv
