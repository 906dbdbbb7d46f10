// Single-head attention of width d = 512: the mid-block attention of AutoencoderKL (diffusers Attention with one head of 512
// channels, biased to_q / to_k / to_v, reached from vae.encode and vae.decode).  out = softmax(Q K^T / sqrt(512)) V over the
// tokens of one frame, flash-style: no L x L score matrix is ever stored.
//
// One CTA per (64-query tile, frame), 384 threads:
//   warpgroup 0     TMA producer : the Q tile (64 x 512) once, then K tiles (64 keys x 512) and V^T tiles (512 x 64 keys)
//   warpgroups 1-2  math         : both compute the same S = Q K^T tile (wgmma m64 n64 k16, 32 steps over d, both operands from
//                                  shared memory) and the same softmax; warpgroup w then accumulates its half of the output,
//                                  O[:, 256 w, 256 w + 256) += P V (wgmma m64 n256 k16, P from registers).
// A 64 x 512 fp32 O tile is 256 registers per thread in one warpgroup; split over two it is 128.  Issuing Q K^T twice costs about
// 1 % of the decoder's FLOPs and no P has to be exchanged between the warpgroups.
// Shared memory holds Q (64 KB) and one K slot and one V^T slot (64 KB each).  The K slot is released as soon as S has been
// computed, so K_{j+1} loads during the softmax and P V of tile j; V^T_{j+1} loads during S_{j+1}.
// Softmax statistics are fp32 with the lazy rescale of attn_spatial.cu (O is rescaled only when a row max grows by more than 2^8);
// P is rounded to fp16 for P V and the denominator is summed, in fp32, from the same rounded values.
// Q, K and V^T are read through 3-D tensor maps bounded at the frame's L tokens: the last key tile may be partial (L = 960 at a
// 40 x 24 latent), its missing keys read as zero and are masked out of the softmax.
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <math.h>
#include <stdint.h>

#include "ops.h"
#include "ptx.cuh"
#include "tma.h"
#include "wgmma.cuh"

namespace hv {

namespace {

constexpr int D = 512;
constexpr int QT = 64;                          // queries per CTA
constexpr int KT = 64;                          // keys per tile
constexpr int kChunks = D / 64;                 // 64-channel (128-byte) chunks of a Q / K row
constexpr int kQBytes = kChunks * QT * 128;     // 64 KB
constexpr int kKBytes = kChunks * KT * 128;     // 64 KB
constexpr int kVHalfBytes = (D / 2) * KT * 2;   // one warpgroup's V^T rows: 256 x 64 keys = 32 KB
constexpr int kVBytes = 2 * kVHalfBytes;
constexpr int kSmemBytes = kQBytes + kKBytes + kVBytes + 1024 + 64;   // + alignment slack, barriers
constexpr int kThreads = 384;
constexpr int kMathWarps = 8;
constexpr float kRescaleThreshold = 8.0f;       // log2 units
constexpr uint32_t kProducerRegs = 40, kMathRegs = 232;

struct D512Args {
  __half* out;
  long long ldo;
  int L;
  float scale_log2;
};

__global__ void __launch_bounds__(kThreads, 1)
attn_d512_kernel(const __grid_constant__ CUtensorMap map_q, const __grid_constant__ CUtensorMap map_k, const __grid_constant__ CUtensorMap map_vt,
                 const D512Args a) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* sQ = smem;
  uint8_t* sK = sQ + kQBytes;
  uint8_t* sV = sK + kKBytes;
  uint64_t* bars = reinterpret_cast<uint64_t*>(sV + kVBytes);
  uint64_t* bar_q = bars;
  uint64_t* bar_k_full = bars + 1;
  uint64_t* bar_k_empty = bars + 2;
  uint64_t* bar_v_full = bars + 3;
  uint64_t* bar_v_empty = bars + 4;

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int q0 = blockIdx.x * QT;
  const int n = blockIdx.y;
  const int T = (a.L + KT - 1) / KT;

  if (threadIdx.x == 0) {
    mbar_init(bar_q, 1);
    mbar_init(bar_k_full, 1);
    mbar_init(bar_k_empty, kMathWarps);
    mbar_init(bar_v_full, 1);
    mbar_init(bar_v_empty, kMathWarps);
    fence_mbar_init();
    tma_prefetch_desc(&map_q);
    tma_prefetch_desc(&map_k);
    tma_prefetch_desc(&map_vt);
  }
  __syncthreads();

  if (warp < 4) {
    setmaxnreg_dec<kProducerRegs>();
    if (warp == 0 && lane == 0) {
      mbar_arrive_expect_tx(bar_q, kQBytes);
#pragma unroll
      for (int kc = 0; kc < kChunks; ++kc) tma_load_3d(sQ + kc * QT * 128, &map_q, bar_q, kc * 64, q0, n);
      for (int j = 0; j < T; ++j) {
        const uint32_t ph = j & 1;
        mbar_wait(bar_k_empty, ph ^ 1);
        mbar_arrive_expect_tx(bar_k_full, kKBytes);
#pragma unroll
        for (int kc = 0; kc < kChunks; ++kc) tma_load_3d(sK + kc * KT * 128, &map_k, bar_k_full, kc * 64, j * KT, n);
        mbar_wait(bar_v_empty, ph ^ 1);
        mbar_arrive_expect_tx(bar_v_full, kVBytes);
        tma_load_3d(sV, &map_vt, bar_v_full, j * KT, n, 0);
        tma_load_3d(sV + kVHalfBytes, &map_vt, bar_v_full, j * KT, n, D / 2);
      }
    }
    return;
  }

  // ---------------------------------------------------------------- math warpgroups: both own query rows 16 wq + lane/4 (+ 8)
  setmaxnreg_inc<kMathRegs>();
  const int wg = (warp >> 2) - 1, wq = warp & 3, quad = lane & 3;
  const float sc = a.scale_log2;
  const uint32_t aQ = smem_u32(sQ), aK = smem_u32(sK), aV = smem_u32(sV) + wg * kVHalfBytes;
  float o[D / 4];           // this warpgroup's 64 x 256 slice of O
#pragma unroll
  for (int i = 0; i < D / 4; ++i) o[i] = 0.f;
  float m_used[2] = {-INFINITY, -INFINITY};
  float lsum[2] = {0.f, 0.f};   // this thread's share of the row's denominator (its 16 columns of every tile)
  float s[KT / 2];
  uint32_t pa[KT / 16][4];

  mbar_wait(bar_q, 0);
  for (int j = 0; j < T; ++j) {
    const uint32_t ph = j & 1;
    mbar_wait(bar_k_full, ph);
    wgmma_fence();
#pragma unroll
    for (int ks = 0; ks < D / 16; ++ks)
      wgmma_ss<KT>(s, gmma_desc_k_sw128(aQ + (ks / 4) * QT * 128) + 2 * (ks % 4), gmma_desc_k_sw128(aK + (ks / 4) * KT * 128) + 2 * (ks % 4),
                   ks != 0 ? 1u : 0u);
    wgmma_commit();
    wgmma_wait<0>();
    wgmma_fence_regs(s);
    if (lane == 0) mbar_arrive(bar_k_empty);

    // row max over the valid keys (keys past L read as zero through the map and are masked to -inf here)
    const int kv_valid = a.L - j * KT;
    float mx[2] = {-INFINITY, -INFINITY};
#pragma unroll
    for (int jj = 0; jj < KT / 8; ++jj)
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        const bool ok = 8 * jj + 2 * quad + e < kv_valid;
#pragma unroll
        for (int hh = 0; hh < 2; ++hh) {
          float& v = s[4 * jj + 2 * hh + e];
          v = ok ? v : -INFINITY;
          mx[hh] = fmaxf(mx[hh], v);
        }
      }
    // lazy rescale, branch-free: a factor of exactly 1 leaves O and the denominator bit for bit as they were
#pragma unroll
    for (int hh = 0; hh < 2; ++hh) {
      mx[hh] = fmaxf(mx[hh], __shfl_xor_sync(0xffffffffu, mx[hh], 1));
      mx[hh] = fmaxf(mx[hh], __shfl_xor_sync(0xffffffffu, mx[hh], 2));
      const float rowmax = mx[hh] * sc;
      const bool grow = rowmax > m_used[hh] + kRescaleThreshold;
      const float f = grow ? fast_exp2(m_used[hh] - rowmax) : 1.f;
      m_used[hh] = grow ? rowmax : m_used[hh];
      lsum[hh] *= f;
#pragma unroll
      for (int jj = 0; jj < D / 16; ++jj) {
        o[4 * jj + 2 * hh] *= f;
        o[4 * jj + 2 * hh + 1] *= f;
      }
    }
    // p = 2^(s*scale - m), rounded to fp16 into the A fragments of P V; the denominator adds the rounded values
#pragma unroll
    for (int kk = 0; kk < KT / 16; ++kk)
#pragma unroll
      for (int half = 0; half < 2; ++half)
#pragma unroll
        for (int hh = 0; hh < 2; ++hh) {
          const int i = 4 * (2 * kk + half) + 2 * hh;
          const uint32_t p2 = pack_h2(fast_exp2(fmaf(s[i], sc, -m_used[hh])), fast_exp2(fmaf(s[i + 1], sc, -m_used[hh])));
          const float2 pf = __half22float2(*reinterpret_cast<const __half2*>(&p2));
          lsum[hh] += pf.x + pf.y;
          pa[kk][2 * half + hh] = p2;
        }

    mbar_wait(bar_v_full, ph);
    wgmma_fence_regs(o);
    wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < KT / 16; ++kk) wgmma_rs<D / 2>(o, pa[kk], gmma_desc_k_sw128(aV) + 2 * kk, 1u);
    wgmma_commit();
    wgmma_wait<0>();
    wgmma_fence_regs(o);
    wgmma_fence_regs(pa);
    if (lane == 0) mbar_arrive(bar_v_empty);
  }

  // ---- epilogue: O / denominator (the row's four lanes hold disjoint column shares of it)
#pragma unroll
  for (int hh = 0; hh < 2; ++hh) {
    float den = lsum[hh];
    den += __shfl_xor_sync(0xffffffffu, den, 1);
    den += __shfl_xor_sync(0xffffffffu, den, 2);
    const int qrow = q0 + wq * 16 + (lane >> 2) + 8 * hh;
    if (qrow < a.L) {
      const float inv = 1.f / den;
      __half* dst = a.out + (static_cast<long long>(n) * a.L + qrow) * a.ldo + wg * (D / 2);
#pragma unroll
      for (int jj = 0; jj < D / 16; ++jj)
        *reinterpret_cast<uint32_t*>(dst + 8 * jj + 2 * quad) = pack_h2(o[4 * jj + 2 * hh] * inv, o[4 * jj + 2 * hh + 1] * inv);
    }
  }
}

}  // namespace

int op_attention_d512(const __half* q, int64_t ldq, const __half* k, int64_t ldk, const __half* vt, int64_t ldvt, int64_t vt_stride, __half* out,
                      int64_t ldo, int64_t NF, int64_t L, cudaStream_t stream) {
  if (!q || !k || !vt || !out || NF <= 0 || NF > 65535 || L <= 0 || L > (1 << 24) || (ldq % 8) || (ldk % 8) || (ldvt % 8) || (ldo % 8) ||
      (vt_stride % 8) || vt_stride < L || ldq < 512 || ldk < 512 || ldo < 512) {
    set_error("hv_op_attention_d512: bad shape NF=%lld L=%lld ldq=%lld ldk=%lld ldvt=%lld vt_stride=%lld ldo=%lld (strides multiples of 8, rows >= 512 wide, "
              "vt_stride >= L)", (long long)NF, (long long)L, (long long)ldq, (long long)ldk, (long long)ldvt, (long long)vt_stride, (long long)ldo);
    return HV_ERR_INVALID;
  }
  CUtensorMap mq, mk, mvt;
  if (!make_map_3d(&mq, q, NF, L, D, ldq, QT) || !make_map_3d(&mk, k, NF, L, D, ldk, KT) ||
      !make_map_col_batches(&mvt, vt, NF, D, L, ldvt, vt_stride, D / 2)) {
    set_error("hv_op_attention_d512 map: %s", tma_last_error());
    return HV_ERR_TMA;
  }
  D512Args ka;
  ka.out = out;
  ka.ldo = ldo;
  ka.L = static_cast<int>(L);
  ka.scale_log2 = 1.4426950408889634f / sqrtf(static_cast<float>(D));
  static bool attr = false;
  if (!attr) {
    cudaError_t e = cudaFuncSetAttribute(attn_d512_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kSmemBytes);
    if (e != cudaSuccess) return cuda_status(e, "hv_op_attention_d512");
    attr = true;
  }
  attn_d512_kernel<<<dim3(static_cast<unsigned>((L + QT - 1) / QT), static_cast<unsigned>(NF)), kThreads, kSmemBytes, stream>>>(mq, mk, mvt, ka);
  return cuda_status(cudaGetLastError(), "hv_op_attention_d512");
}

}  // namespace hv
