// extern "C" operator entry points declared in include/hv_b200_ops.h.
#include "../../include/hv_b200_ops.h"
#include "gemm.cuh"
#include "kernels.h"
#include "ops.h"
#include "tma.h"

using namespace hv;

#define H(p) static_cast<const __half*>(p)
#define HM(p) static_cast<__half*>(p)
#define ST(s) static_cast<cudaStream_t>(s)
#define CK(call, what)                          \
  do {                                          \
    cudaError_t _e = (call);                    \
    if (_e != cudaSuccess) return cuda_fail(_e, what); \
    return HV_OK;                               \
  } while (0)

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
  if (!device_sms()) return HV_ERR_CUDA;
  CK(launch_pack_upconv2x2(H(W), HM(out), (int)Cout, (int)Cin, device_sms(), ST(stream)), "hv_pack_upconv2x2");
}

int hv_op_conv3x3_small(const void* X, const void* Wp, const void* bias, void* out, int64_t ldo, int64_t NF, int64_t Hh, int64_t W, int64_t Cin,
                        int64_t Cout, int32_t stride, int32_t act, hv_stream_t stream) {
  if (!smallconv_supported((int)Cin, (int)Cout, stride)) { set_error("hv_op_conv3x3_small: (Cin, Cout, stride) = (%lld, %lld, %d) is not one of (16,16,1) (16,32,2) (32,32,1) (32,96,2)", (long long)Cin, (long long)Cout, stride); return HV_ERR_INVALID; }
  CK(launch_smallconv(H(X), H(Wp), H(bias), HM(out), (int)NF, (int)Hh, (int)W, (int)Cin, (int)Cout, stride, (int)ldo, act, ST(stream)), "hv_op_conv3x3_small");
}
int hv_op_pose_conv_in(const void* X, const void* W, const void* bias, void* out, int64_t B, int64_t F, int64_t Hh, int64_t Wd, int32_t act, hv_stream_t stream) {
  if (!device_sms()) return HV_ERR_CUDA;
  CK(launch_pg_conv_in(H(X), H(W), H(bias), HM(out), (int)B, (int)F, (int)Hh, (int)Wd, act, device_sms(), ST(stream)), "hv_op_pose_conv_in");
}

int hv_op_clip_patchify(const void* X, void* out, int64_t B, int64_t Cc, int64_t S, int64_t p, int64_t Kpad, hv_stream_t stream) {
  if (!device_sms()) return HV_ERR_CUDA;
  if (!X || !out || B <= 0 || Cc <= 0 || p <= 0 || S <= 0 || (S % p) || (Kpad % 8) || Kpad < Cc * p * p || B * S * S * Cc > INT32_MAX) {
    set_error("hv_op_clip_patchify: bad shape B=%lld C=%lld S=%lld p=%lld Kpad=%lld (S %% p == 0, Kpad >= C p^2 and a multiple of 8)", (long long)B,
              (long long)Cc, (long long)S, (long long)p, (long long)Kpad);
    return HV_ERR_INVALID;
  }
  CK(launch_clip_patchify(H(X), HM(out), (int)B, (int)Cc, (int)S, (int)p, (int)Kpad, device_sms(), ST(stream)), "hv_op_clip_patchify");
}

int hv_op_conv3x3_direct(const void* X, const void* W, const void* bias, void* out, int64_t NF, int64_t Hh, int64_t Wd,
                         int64_t Cin, int64_t Cout, int32_t stride, int32_t act, const void* add, hv_stream_t stream) {
  if (!device_sms()) return HV_ERR_CUDA;
  CK(launch_conv3x3_direct(H(X), H(W), H(bias), HM(out), NF, (int)Hh, (int)Wd, (int)Cin, (int)Cout, stride, act, H(add), device_sms(), ST(stream)),
     "hv_op_conv3x3_direct");
}

size_t hv_groupnorm_scratch_floats(int64_t C, int64_t NF, int64_t HW, int32_t groups) {
  return groupnorm_scratch_floats((int)C, (int)NF, (int)HW, groups);
}

int hv_op_groupnorm(const void* X, int64_t C1, const void* X2, int64_t C2, const void* gamma, const void* beta, void* out,
                    int64_t NF, int64_t HW, int32_t groups, float eps, int32_t silu, float* stats, hv_stream_t stream) {
  if (!device_sms()) return HV_ERR_CUDA;
  CK(launch_groupnorm(H(X), (int)C1, H(X2), (int)C2, H(gamma), H(beta), HM(out), (int)NF, (int)HW, groups, eps, silu, stats, ST(stream)),
     "hv_op_groupnorm");
}

size_t hv_groupnorm_pooled_scratch_floats(int64_t C, int64_t NF, int64_t HW, int32_t groups, int64_t frames_per_item) {
  (void)frames_per_item;   // the per-frame partials dominate; the items' {mean, rstd} fit where the per-frame ones would go
  return groupnorm_scratch_floats((int)C, (int)NF, (int)HW, groups);
}

int hv_op_groupnorm_pooled(const void* X, int64_t C1, const void* X2, int64_t C2, const void* gamma, const void* beta, void* out,
                           int64_t NF, int64_t HW, int32_t groups, float eps, int32_t silu, int64_t frames_per_item, float* stats,
                           hv_stream_t stream) {
  if (!device_sms()) return HV_ERR_CUDA;
  const int64_t F = frames_per_item;
  auto a16 = [](const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; };
  const bool ok = X && gamma && beta && out && stats && (C2 == 0 || X2) && C1 > 0 && C2 >= 0 && C1 + C2 <= 8192 && NF > 0 && HW > 0 &&
                  HW <= INT32_MAX && F > 0 && NF % F == 0 && NF <= 65535 && a16(X) && (C2 == 0 || a16(X2)) && a16(gamma) && a16(beta) &&
                  a16(out) && (reinterpret_cast<uintptr_t>(stats) & 7) == 0 && groupnorm_shape_ok((int)C1, (int)C2, (int)HW, groups);
  if (!ok) {
    set_error("hv_op_groupnorm_pooled: bad arguments C1=%lld C2=%lld NF=%lld HW=%lld groups=%d frames_per_item=%lld (NF %% F == 0, 16-byte aligned "
              "tensors, 8-byte aligned stats, a channel layout hv_op_groupnorm supports)", (long long)C1, (long long)C2, (long long)NF, (long long)HW,
              groups, (long long)F);
    return HV_ERR_INVALID;
  }
  CK(launch_groupnorm_pooled(H(X), (int)C1, C2 ? H(X2) : nullptr, (int)C2, H(gamma), H(beta), HM(out), (int)NF, (int)HW, groups, eps, silu, (int)F,
                             stats, ST(stream)),
     "hv_op_groupnorm_pooled");
}

int hv_op_layernorm(const void* X, const void* gamma, const void* beta, void* out, int64_t rows, int64_t C, float eps,
                    const void* pre_add, int64_t rows_per_group, void* x_out, const void* pe, int64_t hw, int64_t F,
                    hv_stream_t stream) {
  CK(launch_layernorm(H(X), H(gamma), H(beta), HM(out), rows, (int)C, eps, H(pre_add), rows_per_group, HM(x_out), H(pe), (int)hw, (int)F, ST(stream)),
     "hv_op_layernorm");
}

int hv_op_attention(const void* Q, const void* K, const void* Vt, void* out, int64_t NF, int64_t L, int32_t heads, int32_t d,
                    int64_t ldq, int64_t ldk, int64_t ldvt, int64_t ldo, const void* Kb, const void* Vbt, int64_t Lb,
                    int64_t ldkb, int64_t ldvbt, int64_t F, int64_t nf_nobank, int64_t vt_stride, int64_t vbt_stride, hv_stream_t stream) {
  if (!device_sms()) return HV_ERR_CUDA;
  if ((vt_stride % 8) || (vbt_stride % 8) || vt_stride < L) { set_error("hv_op_attention: V^T frame strides must be multiples of 8 and >= L"); return HV_ERR_INVALID; }
  if ((ldq % 8) || (ldk % 8) || (ldvt % 8) || (ldo % 8) || (d % 8)) { set_error("hv_op_attention: strides / head dim must be multiples of 8"); return HV_ERR_INVALID; }
  // every token, V^T column and TMA coordinate below is an int, and NF / heads are grid dimensions (<= 65535)
  const bool d_ok = d == 8 || d == 16 || d == 32 || d == 40 || d == 64 || d == 80 || d == 160;
  const int64_t dpad = (d + 15) / 16 * 16;
  if (!Q || !K || !Vt || !out || NF < 1 || NF > 65535 || L < 1 || L > INT32_MAX || vt_stride > INT32_MAX || heads < 1 || heads > 65535 || !d_ok ||
      NF * L > INT32_MAX || NF * vt_stride > INT32_MAX || nf_nobank < 0 || nf_nobank > NF || ldo < heads * d || ldq < heads * dpad || ldk < heads * dpad ||
      ldvt < NF * vt_stride) {
    set_error("hv_op_attention: bad arguments NF=%lld L=%lld heads=%d d=%d ldq=%lld ldk=%lld ldvt=%lld ldo=%lld vt_stride=%lld nf_nobank=%lld "
              "(pointers non-NULL, 1 <= NF, heads <= 65535, 0 <= nf_nobank <= NF, ldo >= heads*d, ldq and ldk >= heads*dpad, ldvt >= NF*vt_stride)",
              (long long)NF, (long long)L, heads, d, (long long)ldq, (long long)ldk, (long long)ldvt, (long long)ldo, (long long)vt_stride,
              (long long)nf_nobank);
    return HV_ERR_INVALID;
  }
  const bool bank = Kb != nullptr && Lb > 0;   // a NULL Kb (or Lb = 0) means no bank, whatever the other bank arguments hold
  if (bank && (!Vbt || F < 1 || NF % F || Lb > INT32_MAX || vbt_stride > INT32_MAX || vbt_stride < Lb || NF / F * Lb > INT32_MAX || NF / F * vbt_stride > INT32_MAX || ldkb < heads * dpad ||
               (ldkb % 8) || (ldvbt % 8) || ldvbt < NF / F * vbt_stride)) {
    set_error("hv_op_attention: bad bank arguments NF=%lld F=%lld Lb=%lld ldkb=%lld ldvbt=%lld vbt_stride=%lld (Vbt non-NULL, F divides NF, "
              "vbt_stride >= Lb, ldkb >= heads*dpad, ldvbt >= (NF/F)*vbt_stride)", (long long)NF, (long long)F, (long long)Lb, (long long)ldkb,
              (long long)ldvbt, (long long)vbt_stride);
    return HV_ERR_INVALID;
  }
  AttnArgs a;
  a.q = H(Q); a.k = H(K); a.vt = H(Vt); a.out = HM(out);
  a.NF = (int)NF; a.L = (int)L; a.heads = heads; a.d = d; a.dpad = (int)dpad;  // V^T rows per head: (d + 1 + 15) / 16 * 16, row d of every head = ones
  a.ldq = ldq; a.ldk = ldk; a.ldvt = ldvt; a.ldo = ldo;
  a.kb = H(Kb); a.vbt = H(Vbt); a.Lb = bank ? (int)Lb : 0; a.ldkb = ldkb; a.ldvbt = ldvbt;
  a.F = (int)F; a.nf_nobank = (int)nf_nobank; a.vt_stride = vt_stride; a.vbt_stride = vbt_stride;
  cudaError_t e = launch_attention(a, device_sms(), ST(stream));
  if (e != cudaSuccess) { set_error("hv_op_attention: %s (%s)", cudaGetErrorString(e), tma_last_error()); return HV_ERR_CUDA; }
  return HV_OK;
}

int hv_op_attention_d512(const void* Q, int64_t ldq, const void* K, int64_t ldk, const void* Vt, int64_t ldvt, int64_t vt_stride, void* out,
                         int64_t ldo, int64_t NF, int64_t L, hv_stream_t stream) {
  if (!device_sms()) return HV_ERR_CUDA;
  if (!Q || !K || !Vt || !out || NF <= 0 || NF > 65535 || L <= 0 || L > (1 << 24) || (ldq % 8) || (ldk % 8) || (ldvt % 8) || (ldo % 8) ||
      (vt_stride % 8) || vt_stride < L || ldq < 512 || ldk < 512 || ldo < 512) {
    set_error("hv_op_attention_d512: bad shape NF=%lld L=%lld ldq=%lld ldk=%lld ldvt=%lld vt_stride=%lld ldo=%lld (strides multiples of 8, rows >= 512 wide, "
              "vt_stride >= L)", (long long)NF, (long long)L, (long long)ldq, (long long)ldk, (long long)ldvt, (long long)vt_stride, (long long)ldo);
    return HV_ERR_INVALID;
  }
  cudaError_t e = launch_attention_d512(H(Q), ldq, H(K), ldk, H(Vt), ldvt, vt_stride, HM(out), ldo, (int)NF, (int)L, ST(stream));
  if (e != cudaSuccess) { set_error("hv_op_attention_d512: %s (%s)", cudaGetErrorString(e), tma_last_error()); return HV_ERR_CUDA; }
  return HV_OK;
}

// rows (b, f, p) and the one-warp-per-problem grid of the register kernel are indexed with ints
static bool temporal_args_ok(const char* what, int64_t B, int64_t F, int64_t HW, int32_t heads, int32_t d) {
  const bool d_ok = d == 8 || d == 16 || d == 32 || d == 40 || d == 80 || d == 160;
  if (B < 1 || B > INT32_MAX || F < 1 || F > 32 || HW < 1 || HW > INT32_MAX || heads < 1 || !d_ok || B * F > INT32_MAX || B * F * HW > INT32_MAX ||
      B * HW * heads > INT32_MAX || static_cast<int64_t>(heads) * d * 3 > INT32_MAX) {
    set_error("%s: bad shape B=%lld F=%lld HW=%lld heads=%d d=%d (B, HW, heads >= 1, 1 <= F <= 32, d one of 8, 16, 32, 40, 80, 160)", what,
              (long long)B, (long long)F, (long long)HW, heads, d);
    return false;
  }
  return true;
}

int hv_op_temporal_attention(const void* QKV, void* out, int64_t B, int64_t F, int64_t HW, int32_t heads, int32_t d, hv_stream_t stream) {
  if (!QKV || !out) { set_error("hv_op_temporal_attention: NULL pointer"); return HV_ERR_INVALID; }
  if (!temporal_args_ok("hv_op_temporal_attention", B, F, HW, heads, d)) return HV_ERR_INVALID;
  CK(launch_temporal_attention(H(QKV), HM(out), (int)B, (int)F, (int)HW, heads, d, ST(stream)), "hv_op_temporal_attention");
}

int hv_op_ncfhw_to_nhwc(const void* X, void* out, int64_t B, int64_t C, int64_t F, int64_t Hh, int64_t W, int32_t src_fp32, hv_stream_t stream) {
  CK(launch_ncfhw_to_nhwc(X, HM(out), (int)B, (int)C, (int)F, (int)Hh, (int)W, src_fp32, ST(stream)), "hv_op_ncfhw_to_nhwc");
}
int hv_op_nhwc_to_ncfhw(const void* X, int64_t ldx, void* out, int64_t B, int64_t C, int64_t F, int64_t Hh, int64_t W, hv_stream_t stream) {
  CK(launch_nhwc_to_ncfhw(H(X), (int)ldx, HM(out), (int)B, (int)C, (int)F, (int)Hh, (int)W, ST(stream)), "hv_op_nhwc_to_ncfhw");
}
int hv_op_pixel_unshuffle(const void* X, void* out, int64_t B, int64_t C, int64_t F, int64_t Hh, int64_t W, int32_t r, hv_stream_t stream) {
  if (!device_sms()) return HV_ERR_CUDA;
  CK(launch_pixel_unshuffle(H(X), HM(out), (int)B, (int)C, (int)F, (int)Hh, (int)W, r, device_sms(), ST(stream)), "hv_op_pixel_unshuffle");
}
int hv_op_plucker_unshuffle(const float* K, const float* c2w, void* out, int64_t NF, int64_t Hh, int64_t W, int32_t r, hv_stream_t stream) {
  if (!device_sms()) return HV_ERR_CUDA;
  if (!K || !c2w || !out || NF <= 0 || r < 1 || (Hh % r) || (W % r)) { set_error("hv_op_plucker_unshuffle: bad argument"); return HV_ERR_INVALID; }
  CK(launch_plucker_unshuffle(K, c2w, HM(out), NF, (int)Hh, (int)W, r, device_sms(), ST(stream)), "hv_op_plucker_unshuffle");
}
int hv_op_small_linear(const void* X, const void* W, const void* bias, void* out, int64_t M, int64_t N, int64_t K, int32_t act_in, hv_stream_t stream) {
  CK(launch_small_linear(H(X), H(W), H(bias), HM(out), (int)M, (int)N, (int)K, act_in, ST(stream)), "hv_op_small_linear");
}
int hv_op_timestep_embedding(int64_t timestep, void* out, int64_t B, int64_t dim, hv_stream_t stream) {
  CK(launch_timestep_embedding(timestep, nullptr, nullptr, HM(out), (int)B, (int)dim, ST(stream)), "hv_op_timestep_embedding");
}
int hv_pack_conv3x3(const void* W, void* out, int64_t Cout, int64_t Cin, int64_t Cout_pad, int64_t Cin_pad, hv_stream_t stream) {
  if (!device_sms()) return HV_ERR_CUDA;
  CK(launch_pack_conv3x3(H(W), HM(out), (int)Cout, (int)Cin, (int)Cout_pad, (int)Cin_pad, device_sms(), ST(stream)), "hv_pack_conv3x3");
}
int hv_pack_geglu(const void* W, void* out, int64_t rows, int64_t K, hv_stream_t stream) {
  if (!device_sms()) return HV_ERR_CUDA;
  CK(launch_pack_geglu(H(W), HM(out), (int)rows, (int)K, device_sms(), ST(stream)), "hv_pack_geglu");
}
int hv_pack_heads(const void* W, void* out, int32_t heads, int32_t d, int32_t dpad, int64_t K, hv_stream_t stream) {
  if (!device_sms()) return HV_ERR_CUDA;
  CK(launch_pack_heads(H(W), HM(out), heads, d, dpad, (int)K, device_sms(), ST(stream)), "hv_pack_heads");
}
int hv_op_window_gather(const void* latents, const int32_t* frame_idx, void* out, int64_t Bl, int64_t C, int64_t Ftot, int64_t Fw, int64_t HW,
                        int32_t repeat, hv_stream_t stream) {
  if (!device_sms()) return HV_ERR_CUDA;
  if (!latents || !frame_idx || !out || Bl <= 0 || C <= 0 || Ftot <= 0 || Fw <= 0 || HW <= 0 || repeat < 1) { set_error("hv_op_window_gather: bad argument"); return HV_ERR_INVALID; }
  CK(launch_window_gather(H(latents), frame_idx, HM(out), (int)Bl, (int)C, (int)Ftot, (int)Fw, (int)HW, repeat, device_sms(), ST(stream)), "hv_op_window_gather");
}
int hv_op_cfg_ddim_step(const void* const* pred_uncond, const void* const* pred_cond, int32_t n_windows, const int32_t* inv, int32_t K,
                        const float* coef, const int32_t* step_index, void* latents, int64_t Bl, int64_t C, int64_t Ftot, int64_t Fw, int64_t HW,
                        float guidance_scale, int32_t prediction_type, hv_stream_t stream) {
  if (!device_sms()) return HV_ERR_CUDA;
  if (!pred_uncond || !inv || !coef || !latents || n_windows < 1 || n_windows > kMaxWindows || K < 1 || (prediction_type != 0 && prediction_type != 1)) {
    set_error("hv_op_cfg_ddim_step: bad argument (1..%d windows, prediction_type 0 = v_prediction / 1 = epsilon)", kMaxWindows);
    return HV_ERR_INVALID;
  }
  StepPreds sp{};
  for (int w = 0; w < n_windows; ++w) {
    sp.uncond[w] = H(pred_uncond[w]);
    sp.cond[w] = pred_cond ? H(pred_cond[w]) : nullptr;
    if (!sp.uncond[w] || (pred_cond && !sp.cond[w])) { set_error("hv_op_cfg_ddim_step: window %d has a NULL prediction", w); return HV_ERR_INVALID; }
  }
  CK(launch_cfg_ddim_step(sp, inv, K, coef, step_index, HM(latents), (int)Bl, (int)C, (int)Ftot, (int)Fw, (int)HW, guidance_scale, pred_cond ? 1 : 0,
                          prediction_type, device_sms(), ST(stream)), "hv_op_cfg_ddim_step");
}
int hv_op_advance_index(int32_t* index, hv_stream_t stream) {
  if (!index) return HV_ERR_INVALID;
  CK(launch_advance_index(index, ST(stream)), "hv_op_advance_index");
}
int hv_dbg_gemm(const void* A, int64_t lda, const void* W, float* out, int64_t M, int64_t N, int64_t K, hv_stream_t stream) {
  CK(launch_dbg_gemm(H(A), lda, H(W), out, (int)M, (int)N, (int)K, ST(stream)), "hv_dbg_gemm");
}
int hv_dbg_gemm_plan(int64_t M, int64_t N, int64_t K, int32_t geglu, int32_t* block_n, int32_t* bst_stages, int32_t* grid) {
  return plan_linear(M, N, K, geglu != 0, block_n, bst_stages, grid);
}
int hv_dbg_temporal_attention_plan(int64_t B, int64_t F, int64_t HW, int32_t heads, int32_t d, int32_t* tma, int32_t* heads_per_box, int32_t* grid) {
  const int sms = device_sms();
  if (!sms) return HV_ERR_CUDA;
  if (!temporal_args_ok("hv_dbg_temporal_attention_plan", B, F, HW, heads, d)) return HV_ERR_INVALID;
  const TemporalPlan p = plan_temporal_attention((int)B, (int)HW, heads, d, sms);
  if (tma) *tma = p.tma ? 1 : 0;
  if (heads_per_box) *heads_per_box = p.heads_per_box;
  if (grid) *grid = (int32_t)p.grid;
  return HV_OK;
}

}  // extern "C"
