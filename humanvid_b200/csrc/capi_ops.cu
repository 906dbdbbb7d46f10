// extern "C" operator entry points declared in include/hv_b200_ops.h: each is the checked operator function of ops.h.
#include "../../include/hv_b200_fp8.h"
#include "../../include/hv_b200_ops.h"
#include "ops.h"

using namespace hv;

#define H(p) static_cast<const __half*>(p)
#define HM(p) static_cast<__half*>(p)
#define ST(s) static_cast<cudaStream_t>(s)

extern "C" {

const char* hv_ops_last_error(void) { return last_error(); }
int hv_num_sms(void) { return device_sms(); }

int hv_op_gemm(const void* A, int64_t lda, const void* A2, int64_t lda2, int64_t K1, const void* W, void* out, int64_t ldc,
               int64_t M, int64_t N, int64_t K, const hv_epilogue* ep, hv_stream_t stream) {
  return op_gemm(H(A), lda, H(A2), lda2, K1, H(W), HM(out), ldc, M, N, K, ep, ST(stream));
}
int hv_op_gemm_batched_b(const void* A, int64_t lda, const void* X, int64_t ldx, void* out, int64_t ldc, int64_t M, int64_t batch,
                         int64_t rows, int64_t out_stride, int64_t K, const void* rowbias, hv_stream_t stream) {
  return op_gemm_batched_b(H(A), lda, H(X), ldx, HM(out), ldc, M, batch, rows, out_stride, K, H(rowbias), ST(stream));
}
int hv_op_conv3x3(const void* X, const void* Wp, void* out, int64_t ldc, int64_t NF, int64_t Hh, int64_t W, int64_t Cin,
                  int64_t Cout, int32_t stride, const hv_epilogue* ep, hv_stream_t stream) {
  return op_conv3x3(H(X), H(Wp), HM(out), ldc, NF, Hh, W, Cin, Cout, stride, ep, ST(stream));
}
int hv_op_conv3x3_s2_pad_end(const void* X, const void* Wp, void* out, int64_t ldc, int64_t NF, int64_t Hh, int64_t W, int64_t Cin, int64_t Cout,
                             const hv_epilogue* ep, hv_stream_t stream) {
  return op_conv3x3(H(X), H(Wp), HM(out), ldc, NF, Hh, W, Cin, Cout, 2, ep, ST(stream), true);
}
int hv_op_upconv2x2(const void* X, const void* Wp, void* out, int64_t ldc, int64_t NF, int64_t Hh, int64_t W, int64_t Cin, int64_t Cout,
                    const hv_epilogue* ep, hv_stream_t stream) {
  return op_upconv2x2(H(X), H(Wp), HM(out), ldc, NF, Hh, W, Cin, Cout, ep, ST(stream));
}
int hv_pack_upconv2x2(const void* W, void* out, int64_t Cout, int64_t Cin, hv_stream_t stream) {
  return op_pack_upconv2x2(H(W), HM(out), Cout, Cin, ST(stream));
}
int hv_op_conv3x3_small(const void* X, const void* Wp, const void* bias, void* out, int64_t ldo, int64_t NF, int64_t Hh, int64_t W, int64_t Cin,
                        int64_t Cout, int32_t stride, int32_t act, hv_stream_t stream) {
  return op_conv3x3_small(H(X), H(Wp), H(bias), HM(out), ldo, NF, Hh, W, Cin, Cout, stride, act, ST(stream));
}
int hv_op_pose_conv_in(const void* X, const void* W, const void* bias, void* out, int64_t B, int64_t F, int64_t Hh, int64_t Wd, int32_t act, hv_stream_t stream) {
  return op_pose_conv_in(H(X), H(W), H(bias), HM(out), B, F, Hh, Wd, act, ST(stream));
}
int hv_op_clip_patchify(const void* X, void* out, int64_t B, int64_t Cc, int64_t S, int64_t p, int64_t Kpad, hv_stream_t stream) {
  return op_clip_patchify(H(X), HM(out), B, Cc, S, p, Kpad, ST(stream));
}
int hv_op_conv3x3_direct(const void* X, const void* W, const void* bias, void* out, int64_t NF, int64_t Hh, int64_t Wd,
                         int64_t Cin, int64_t Cout, int32_t stride, int32_t act, const void* add, hv_stream_t stream) {
  return op_conv3x3_direct(H(X), H(W), H(bias), HM(out), NF, Hh, Wd, Cin, Cout, stride, act, H(add), Cout, ST(stream));
}

size_t hv_groupnorm_scratch_floats(int64_t C, int64_t NF, int64_t HW, int32_t groups) {
  return groupnorm_scratch_floats((int)C, (int)NF, (int)HW, groups);
}
int hv_op_groupnorm(const void* X, int64_t C1, const void* X2, int64_t C2, const void* gamma, const void* beta, void* out,
                    int64_t NF, int64_t HW, int32_t groups, float eps, int32_t silu, float* stats, hv_stream_t stream) {
  return op_groupnorm(H(X), C1, H(X2), C2, H(gamma), H(beta), HM(out), NF, HW, groups, eps, silu, stats, ST(stream));
}
size_t hv_groupnorm_pooled_scratch_floats(int64_t C, int64_t NF, int64_t HW, int32_t groups, int64_t frames_per_item) {
  (void)frames_per_item;   // the per-frame partials dominate; the items' {mean, rstd} fit where the per-frame ones would go
  return groupnorm_scratch_floats((int)C, (int)NF, (int)HW, groups);
}
int hv_op_groupnorm_pooled(const void* X, int64_t C1, const void* X2, int64_t C2, const void* gamma, const void* beta, void* out,
                           int64_t NF, int64_t HW, int32_t groups, float eps, int32_t silu, int64_t frames_per_item, float* stats,
                           hv_stream_t stream) {
  return op_groupnorm_pooled(H(X), C1, H(X2), C2, H(gamma), H(beta), HM(out), NF, HW, groups, eps, silu, frames_per_item, stats, ST(stream));
}
int hv_op_layernorm(const void* X, const void* gamma, const void* beta, void* out, int64_t rows, int64_t C, float eps,
                    const void* pre_add, int64_t rows_per_group, void* x_out, const void* pe, int64_t hw, int64_t F,
                    hv_stream_t stream) {
  return op_layernorm(H(X), H(gamma), H(beta), HM(out), rows, C, eps, H(pre_add), rows_per_group, HM(x_out), H(pe), hw, F, ST(stream));
}

int hv_op_attention(const void* Q, const void* K, const void* Vt, void* out, int64_t NF, int64_t L, int32_t heads, int32_t d,
                    int64_t ldq, int64_t ldk, int64_t ldvt, int64_t ldo, const void* Kb, const void* Vbt, int64_t Lb,
                    int64_t ldkb, int64_t ldvbt, int64_t F, int64_t nf_nobank, int64_t vt_stride, int64_t vbt_stride, hv_stream_t stream) {
  return op_attention(H(Q), H(K), H(Vt), HM(out), NF, L, heads, d, ldq, ldk, ldvt, ldo, H(Kb), H(Vbt), Lb, ldkb, ldvbt, F, nf_nobank, vt_stride,
                      vbt_stride, ST(stream));
}
int hv_op_attention_d512(const void* Q, int64_t ldq, const void* K, int64_t ldk, const void* Vt, int64_t ldvt, int64_t vt_stride, void* out,
                         int64_t ldo, int64_t NF, int64_t L, hv_stream_t stream) {
  return op_attention_d512(H(Q), ldq, H(K), ldk, H(Vt), ldvt, vt_stride, HM(out), ldo, NF, L, ST(stream));
}
int hv_op_temporal_attention(const void* QKV, void* out, int64_t B, int64_t F, int64_t HW, int32_t heads, int32_t d, hv_stream_t stream) {
  return op_temporal_attention(H(QKV), HM(out), B, F, HW, heads, d, ST(stream));
}

int hv_op_ncfhw_to_nhwc(const void* X, void* out, int64_t B, int64_t C, int64_t F, int64_t Hh, int64_t W, int32_t src_fp32, hv_stream_t stream) {
  return op_ncfhw_to_nhwc(X, HM(out), B, C, F, Hh, W, src_fp32, ST(stream));
}
int hv_op_nhwc_to_ncfhw(const void* X, int64_t ldx, void* out, int64_t B, int64_t C, int64_t F, int64_t Hh, int64_t W, hv_stream_t stream) {
  return op_nhwc_to_ncfhw(H(X), ldx, HM(out), B, C, F, Hh, W, ST(stream));
}
int hv_op_pixel_unshuffle(const void* X, void* out, int64_t B, int64_t C, int64_t F, int64_t Hh, int64_t W, int32_t r, hv_stream_t stream) {
  return op_pixel_unshuffle(H(X), HM(out), B, C, F, Hh, W, r, ST(stream));
}
int hv_op_plucker_unshuffle(const float* K, const float* c2w, void* out, int64_t NF, int64_t Hh, int64_t W, int32_t r, hv_stream_t stream) {
  return op_plucker_unshuffle(K, c2w, HM(out), NF, Hh, W, r, ST(stream));
}
int hv_op_small_linear(const void* X, const void* W, const void* bias, void* out, int64_t M, int64_t N, int64_t K, int32_t act_in, hv_stream_t stream) {
  return op_small_linear(H(X), H(W), H(bias), HM(out), M, N, K, act_in, ST(stream));
}
int hv_op_timestep_embedding(int64_t timestep, void* out, int64_t B, int64_t dim, hv_stream_t stream) {
  return op_timestep_embedding(timestep, nullptr, nullptr, HM(out), B, dim, ST(stream));
}
int hv_pack_conv3x3(const void* W, void* out, int64_t Cout, int64_t Cin, int64_t Cout_pad, int64_t Cin_pad, hv_stream_t stream) {
  return op_pack_conv3x3(H(W), HM(out), Cout, Cin, Cout_pad, Cin_pad, ST(stream));
}
int hv_pack_geglu(const void* W, void* out, int64_t rows, int64_t K, hv_stream_t stream) {
  return op_pack_geglu(H(W), HM(out), rows, K, ST(stream));
}
int hv_pack_heads(const void* W, void* out, int32_t heads, int32_t d, int32_t dpad, int64_t K, hv_stream_t stream) {
  return op_pack_heads(H(W), HM(out), heads, d, dpad, K, ST(stream));
}
int hv_op_window_gather(const void* latents, const int32_t* frame_idx, void* out, int64_t Bl, int64_t C, int64_t Ftot, int64_t Fw, int64_t HW,
                        int32_t repeat, hv_stream_t stream) {
  return op_window_gather(H(latents), frame_idx, HM(out), Bl, C, Ftot, Fw, HW, repeat, ST(stream));
}
int hv_op_cfg_ddim_step(const void* const* pred_uncond, const void* const* pred_cond, int32_t n_windows, const int32_t* inv, int32_t K,
                        const float* coef, const int32_t* step_index, void* latents, int64_t Bl, int64_t C, int64_t Ftot, int64_t Fw, int64_t HW,
                        float guidance_scale, int32_t prediction_type, hv_stream_t stream) {
  return op_cfg_ddim_step(pred_uncond, pred_cond, n_windows, inv, K, coef, step_index, HM(latents), Bl, C, Ftot, Fw, HW, guidance_scale,
                          prediction_type, ST(stream));
}
int hv_op_advance_index(int32_t* index, hv_stream_t stream) {
  return op_advance_index(index, ST(stream));
}

int hv_op_gemm_fp8(const void* A, int64_t lda, const float* a_scale, int64_t a_scale_ld, const void* W, const float* w_scale, void* out,
                   int64_t ldc, float* out_scale, int64_t out_scale_ld, int64_t M, int64_t N, int64_t K, const hv_epilogue* ep, hv_stream_t stream) {
  return op_gemm_fp8(static_cast<const uint8_t*>(A), lda, a_scale, a_scale_ld, static_cast<const uint8_t*>(W), w_scale, out, ldc, out_scale,
                     out_scale_ld, M, N, K, ep, ST(stream));
}
int hv_op_layernorm_fp8(const void* X, const void* gamma, const void* beta, void* out, float* out_scale, int64_t rows, int64_t C, float eps,
                        const void* pre_add, int64_t rows_per_group, void* x_out, const void* pe, int64_t hw, int64_t F, hv_stream_t stream) {
  return op_layernorm_fp8(H(X), H(gamma), H(beta), static_cast<uint8_t*>(out), out_scale, rows, C, eps, H(pre_add), rows_per_group, HM(x_out), H(pe),
                          hw, F, ST(stream));
}
int hv_pack_fp8_rows(const void* W, void* out, float* scale, int64_t rows, int64_t K, hv_stream_t stream) {
  return op_pack_fp8_rows(H(W), static_cast<uint8_t*>(out), scale, rows, K, ST(stream));
}

int hv_dbg_gemm(const void* A, int64_t lda, const void* W, float* out, int64_t M, int64_t N, int64_t K, hv_stream_t stream) {
  return op_dbg_gemm(H(A), lda, H(W), out, M, N, K, ST(stream));
}
int hv_dbg_gemm_plan(int64_t M, int64_t N, int64_t K, int32_t geglu, int32_t* block_n, int32_t* bst_stages, int32_t* grid) {
  return plan_linear(M, N, K, geglu != 0, block_n, bst_stages, grid);
}
int hv_dbg_temporal_attention_plan(int64_t B, int64_t F, int64_t HW, int32_t heads, int32_t d, int32_t* tma, int32_t* heads_per_box, int32_t* grid) {
  TemporalPlan p;
  if (int rc = plan_temporal_attention("hv_dbg_temporal_attention_plan", B, F, HW, heads, d, &p)) return rc;
  if (tma) *tma = p.tma ? 1 : 0;
  if (heads_per_box) *heads_per_box = p.heads_per_box;
  if (grid) *grid = (int32_t)p.grid;
  return HV_OK;
}

}  // extern "C"
