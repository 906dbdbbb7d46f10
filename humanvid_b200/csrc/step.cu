// Per-timestep glue of the denoising loop on the device (SURVEY 8f-2): what Pose2VideoPipeline.__call__ does around the
// UNet forward with a dozen small eager ops per step (src/pipelines/pipeline_pose2vid_long.py:516-563):
//
//   window gather   latent_model_input = latents[:, :, window].repeat(2 if CFG)                          (:516-523)
//   step            noise_pred[:, :, window] += pred ; counter[:, :, window] += 1   for every window    (:550-552)
//                   noise_pred / counter ; uncond + s * (text - uncond)                                  (:555-559)
//                   DDIM update (eta = 0, v-prediction or epsilon): x_prev = sqrt(a_prev) x0 + sqrt(1 - a_prev) eps  (:561-563)
//
// One elementwise kernel does accumulate -> /counter -> CFG -> DDIM in fp32 with a single fp16 rounding at the latent store,
// reading the DDIM coefficients of the CURRENT step from a device table indexed by a device-resident step counter, so a
// captured CUDA graph of one step replays for every timestep (hv_op_advance_index bumps the counter at the end of the step).
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include "ops.h"

namespace hv {

constexpr int kMaxWindows = 32;
struct StepPreds {                       // window w's UNet prediction, (Bl, C, Fw, HW) fp16 each; cond unused without CFG
  const __half* uncond[kMaxWindows];
  const __half* cond[kMaxWindows];
};

namespace {

constexpr int kThreads = 256;

// out[(r*Bl + b), c, i, p] = latents[b, c, idx[i], p]   for r < R  (R = 2: the CFG-doubled batch)
__global__ void window_gather_kernel(const __half* __restrict__ latents, const int* __restrict__ idx, __half* __restrict__ out, int Bl, int C,
                                     int Ftot, int Fw, int HW, int R) {
  const long long total = static_cast<long long>(Bl) * C * Fw * HW;
  for (long long e = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; e < total; e += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int p = static_cast<int>(e % HW);
    long long t = e / HW;
    const int i = static_cast<int>(t % Fw);
    t /= Fw;   // t = b*C + c
    const __half v = latents[(t * Ftot + idx[i]) * HW + p];
    for (int r = 0; r < R; ++r) out[e + r * total] = v;
  }
}

__global__ void cfg_ddim_step_kernel(StepPreds preds, const int* __restrict__ inv, int K, const float* __restrict__ coef,
                                     const int* __restrict__ step_idx, __half* __restrict__ latents, int Bl, int C, int Ftot, int Fw, int HW,
                                     float guidance, int cfg, int epsilon) {
  const float4 cf = *reinterpret_cast<const float4*>(coef + 4 * (step_idx ? *step_idx : 0));   // sqrt(a_t), sqrt(1-a_t), sqrt(a_prev), sqrt(1-a_prev)
  const long long total = static_cast<long long>(Bl) * C * Ftot * HW;
  for (long long e = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; e < total; e += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int p = static_cast<int>(e % HW);
    long long t = e / HW;
    const int f = static_cast<int>(t % Ftot);
    t /= Ftot;   // t = b*C + c
    float un = 0.f, tx = 0.f;
    int cnt = 0;
    for (int k = 0; k < K; ++k) {
      const int j = inv[f * K + k];
      if (j < 0) continue;
      const int w = j / Fw, i = j - w * Fw;
      const long long off = (t * Fw + i) * HW + p;
      un += __half2float(preds.uncond[w][off]);
      if (cfg) tx += __half2float(preds.cond[w][off]);
      ++cnt;
    }
    const float inv_cnt = cnt > 0 ? 1.f / static_cast<float>(cnt) : 0.f;
    un *= inv_cnt;
    tx *= inv_cnt;
    const float m = cfg ? un + guidance * (tx - un) : un;
    const float x = __half2float(latents[e]);
    float x0, eps;
    if (!epsilon) {   // v-prediction
      x0 = cf.x * x - cf.y * m;
      eps = cf.x * m + cf.y * x;
    } else {
      eps = m;
      x0 = (x - cf.y * eps) / cf.x;
    }
    latents[e] = __float2half_rn(cf.z * x0 + cf.w * eps);
  }
}

__global__ void advance_index_kernel(int* idx) { *idx += 1; }

inline unsigned blocks_for(long long n, int num_sms) {
  long long b = (n + kThreads - 1) / kThreads;
  const long long cap = static_cast<long long>(num_sms) * 16;
  return static_cast<unsigned>(b < 1 ? 1 : (b > cap ? cap : b));
}

}  // namespace

int op_window_gather(const __half* latents, const int32_t* idx, __half* out, int64_t Bl, int64_t C, int64_t Ftot, int64_t Fw, int64_t HW, int R,
                     cudaStream_t s) {
  if (!latents || !idx || !out || !int32_ok(Bl) || !int32_ok(C) || !int32_ok(Ftot) || !int32_ok(Fw) || !int32_ok(HW) || R < 1) {
    set_error("hv_op_window_gather: bad argument (non-NULL pointers, Bl, C, Ftot, Fw, HW >= 1 within int32, repeat >= 1)");
    return HV_ERR_INVALID;
  }
  const int sms = device_sms();
  if (!sms) return HV_ERR_CUDA;
  const long long total = Bl * C * Fw * HW;
  window_gather_kernel<<<blocks_for(total, sms), kThreads, 0, s>>>(latents, idx, out, static_cast<int>(Bl), static_cast<int>(C), static_cast<int>(Ftot),
                                                                    static_cast<int>(Fw), static_cast<int>(HW), R);
  return cuda_status(cudaGetLastError(), "hv_op_window_gather");
}

// coef is read as float4
int op_cfg_ddim_step(const void* const* pred_uncond, const void* const* pred_cond, int n_windows, const int32_t* inv, int K, const float* coef,
                     const int32_t* step_index, __half* latents, int64_t Bl, int64_t C, int64_t Ftot, int64_t Fw, int64_t HW, float guidance_scale,
                     int prediction_type, cudaStream_t s) {
  if (!pred_uncond || !inv || !coef || !latents || n_windows < 1 || n_windows > kMaxWindows || K < 1 || (prediction_type != 0 && prediction_type != 1) ||
      !aligned16(coef) || !int32_ok(Bl) || !int32_ok(C) || !int32_ok(Ftot) || !int32_ok(Fw) || !int32_ok(HW)) {
    set_error("hv_op_cfg_ddim_step: bad argument (1..%d windows, prediction_type 0 = v_prediction / 1 = epsilon, 16-byte aligned coef, Bl, C, Ftot, "
              "Fw, HW >= 1 within int32)", kMaxWindows);
    return HV_ERR_INVALID;
  }
  StepPreds sp{};
  for (int w = 0; w < n_windows; ++w) {
    sp.uncond[w] = static_cast<const __half*>(pred_uncond[w]);
    sp.cond[w] = pred_cond ? static_cast<const __half*>(pred_cond[w]) : nullptr;
    if (!sp.uncond[w] || (pred_cond && !sp.cond[w])) { set_error("hv_op_cfg_ddim_step: window %d has a NULL prediction", w); return HV_ERR_INVALID; }
  }
  const int sms = device_sms();
  if (!sms) return HV_ERR_CUDA;
  const long long total = Bl * C * Ftot * HW;
  cfg_ddim_step_kernel<<<blocks_for(total, sms), kThreads, 0, s>>>(sp, inv, K, coef, step_index, latents, static_cast<int>(Bl), static_cast<int>(C),
                                                                    static_cast<int>(Ftot), static_cast<int>(Fw), static_cast<int>(HW), guidance_scale,
                                                                    pred_cond ? 1 : 0, prediction_type);
  return cuda_status(cudaGetLastError(), "hv_op_cfg_ddim_step");
}

int op_advance_index(int32_t* idx, cudaStream_t s) {
  if (!idx) { set_error("hv_op_advance_index: NULL index"); return HV_ERR_INVALID; }
  advance_index_kernel<<<1, 1, 0, s>>>(idx);
  return cuda_status(cudaGetLastError(), "hv_op_advance_index");
}

}  // namespace hv
