// Spatial multi-head self-attention over the tokens of one frame (reference: diffusers Attention + AttnProcessor2_0
// reached from src/models/attention.py:405-408, and the ReferenceAttentionControl read hook
// src/models/mutual_self_attention.py:147-186 that appends the reference image's tokens as extra keys/values).
//
// Flash-style on wgmma: one CTA per (128-query tile, head, frame).
//   warpgroup 0     TMA producer : Q tile once, then K / V^T tiles of 128 keys through two shared-memory rings
//   warpgroups 1-2  math         : each owns 64 query rows: S = Q K^T (wgmma m64 x 128 x dpad, both operands from shared
//                                  memory, S in registers), row max across the four lanes of a row, p = 2^(s*scale - m)
//                                  converted in registers into the A fragments of O += P V (wgmma m64 x dv x 128, A from
//                                  registers).  O stays in registers across key tiles; V^T carries a row of ones per head so
//                                  O's extra column IS the softmax denominator (summed from the same fp16 P the MMA sees).
//                                  O is rescaled only when a row max grows by more than 2^8 (lazy rescale).
//                                  Pipelined by one key tile: S_{j+1} = Q K_{j+1} and O += P_j V_j are issued together and the
//                                  softmax of S_{j+1} runs while P_j V_j is on the tensor cores (DESIGN.md section 3).
// Keys come from two segments: the frame's own L tokens and, for frames of the conditional CFG half, the Lb tokens of
// the batch item's reference bank -- the reference instead materialises cat([x, bank.repeat(F)]) per frame and
// recomputes the unconditional half (mutual_self_attention.py:158-186).
// V is consumed transposed (V^T[channel][token], produced directly by a GEMM with swapped operands) so every shared-memory
// operand in this file is K-major and shares one descriptor format with gemm.cu.
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

constexpr int QT = 128;   // queries per CTA (two math warpgroups of 64)
constexpr int KT = 128;   // keys per tile
constexpr float kRescaleThreshold = 8.0f;  // log2 units: O is rescaled only when the row max grows by more than 2^8
constexpr int ATT_THREADS = 384;
constexpr int kMathWarps = 8;
constexpr uint32_t kProducerRegs = 40, kMathRegs = 232;

struct AttnArgs {
  const __half* q; const __half* k; const __half* vt; __half* out;
  int NF, L, heads, d, dpad;
  long long ldq, ldk, ldvt, ldo;
  const __half* kb; const __half* vbt;   // bank keys [B][Lb][ldkb], bank values transposed [heads*d][ldvbt]
  int Lb; long long ldkb, ldvbt;
  int F, nf_nobank;
  long long vt_stride, vbt_stride;       // columns between consecutive frames / bank items in V^T (multiples of 8)
};

template <int D>
struct ACfg {
  static constexpr int kDpad = (D + 15) / 16 * 16;             // Q/K head stride (zero padded)
  static constexpr int kDv = (D + 1 + 15) / 16 * 16;           // V^T rows per head: d values, one row of ones, zero pad
  static constexpr int kKC = (kDpad + 63) / 64;               // 64-column chunks of Q / K rows
  static constexpr int kQBytes = kKC * QT * 128;
  static constexpr int kKBytes = kKC * KT * 128;
  static constexpr int kVChunk = kDv * 128;                    // [dv rows][64 keys]
  static constexpr int kVBytes = 2 * kVChunk;
  static constexpr int kStageBytes = kKBytes + kVBytes;
  static constexpr int kMisc = 256 + 1024;                     // barriers, alignment
  static constexpr int kStagesFit = (227 * 1024 - kQBytes - kMisc) / kStageBytes;
  static constexpr int kStages = kStagesFit > 4 ? 4 : kStagesFit;
  static constexpr int kSmemBytes = kQBytes + kStages * kStageBytes + kMisc;
  // The one-tile software pipeline needs K_{j+1} resident while P_j V_j runs.  With a single stage (d = 160) K_{j+1} shares the
  // slot of K_j and arrives late, and the pipelined loop measured 12 % slower than the serial one (H100 SXM, 400 W), so that case
  // stays serial.
  static constexpr bool kPipelined = kStages >= 2;
};

// Online softmax of one 64 x 128 score tile held in wgmma accumulator layout (thread row r = lane/4 (+8 for hh = 1), columns
// 8 jj + 2 quad + e): row max across the four lanes of a row, the lazy-rescale decision (grow, alpha = 2^(m_old - m_new) for O),
// then s <- 2^(s*scale - m) in place.  MASK sets keys >= kv_valid to -inf first.
template <bool MASK>
__device__ __forceinline__ void tile_softmax(float (&s)[KT / 2], int kv_valid, int quad, float sc, float (&m_used)[2], bool (&grow)[2],
                                             float (&alpha)[2]) {
  float mx[2] = {-INFINITY, -INFINITY};
#pragma unroll
  for (int jj = 0; jj < KT / 8; ++jj)
#pragma unroll
    for (int e = 0; e < 2; ++e) {
      const bool ok = !MASK || 8 * jj + 2 * quad + e < kv_valid;
#pragma unroll
      for (int hh = 0; hh < 2; ++hh) {
        float& v = s[4 * jj + 2 * hh + e];
        if (MASK) v = ok ? v : -INFINITY;
        mx[hh] = fmaxf(mx[hh], v);
      }
    }
#pragma unroll
  for (int hh = 0; hh < 2; ++hh) {
    mx[hh] = fmaxf(mx[hh], __shfl_xor_sync(0xffffffffu, mx[hh], 1));
    mx[hh] = fmaxf(mx[hh], __shfl_xor_sync(0xffffffffu, mx[hh], 2));
    const float rowmax = mx[hh] * sc;
    grow[hh] = rowmax > m_used[hh] + kRescaleThreshold;
    if (grow[hh]) {
      alpha[hh] = fast_exp2(m_used[hh] - rowmax);
      m_used[hh] = rowmax;
    }
  }
#pragma unroll
  for (int jj = 0; jj < KT / 8; ++jj)
#pragma unroll
    for (int hh = 0; hh < 2; ++hh)
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        float& v = s[4 * jj + 2 * hh + e];
        v = fast_exp2(fmaf(v, sc, -m_used[hh]));
      }
}

struct AttnKernelArgs {
  __half* out;
  long long ldo;
  int L, Lb, F, nf_nobank, heads;
  int vt_stride, vbt_stride;
  float scale_log2;
};

template <int D>
__global__ void __launch_bounds__(ATT_THREADS, 1)
attn_kernel(const __grid_constant__ CUtensorMap map_q, const __grid_constant__ CUtensorMap map_k,
            const __grid_constant__ CUtensorMap map_vt, const __grid_constant__ CUtensorMap map_kb,
            const __grid_constant__ CUtensorMap map_vbt, const AttnKernelArgs a) {
  using C = ACfg<D>;
  constexpr int DP = C::kDpad, DV = C::kDv, NS = C::kStages;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* sQ = smem;
  uint8_t* sKV = sQ + C::kQBytes;
  uint64_t* bars = reinterpret_cast<uint64_t*>(sKV + NS * C::kStageBytes);
  uint64_t* bar_q = bars;
  // K and V tiles travel through separate rings: a K slot is free again as soon as its S = Q K^T has been computed (before
  // the softmax and the P V of the same tile), so the next K tile is in flight a whole phase earlier than a combined stage allows
  uint64_t* bar_k_full = bars + 1;
  uint64_t* bar_k_empty = bars + 1 + NS;
  uint64_t* bar_v_full = bars + 1 + 2 * NS;
  uint64_t* bar_v_empty = bars + 1 + 3 * NS;

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int q0 = blockIdx.x * QT;
  const int h = blockIdx.y;
  const int n = blockIdx.z;
  const bool use_bank = a.Lb > 0 && n >= a.nf_nobank;
  const int Ts = (a.L + KT - 1) / KT;
  const int T = Ts + (use_bank ? (a.Lb + KT - 1) / KT : 0);
  const int bidx = n / a.F;

  if (threadIdx.x == 0) {
    mbar_init(bar_q, 1);
    for (int s = 0; s < NS; ++s) {
      mbar_init(&bar_k_full[s], 1);
      mbar_init(&bar_k_empty[s], kMathWarps);
      mbar_init(&bar_v_full[s], 1);
      mbar_init(&bar_v_empty[s], kMathWarps);
    }
    fence_mbar_init();
    tma_prefetch_desc(&map_q);
    tma_prefetch_desc(&map_k);
    tma_prefetch_desc(&map_vt);
  }
  __syncthreads();

  if (warp < 4) {
    setmaxnreg_dec<kProducerRegs>();
    if (warp == 0 && lane == 0) {
      mbar_arrive_expect_tx(bar_q, C::kQBytes);
#pragma unroll
      for (int kc = 0; kc < C::kKC; ++kc) tma_load_2d(sQ + kc * QT * 128, &map_q, bar_q, h * DP + kc * 64, n * a.L + q0);
      int stage = 0;
      uint32_t phase = 0;
      for (int j = 0; j < T; ++j) {
        uint8_t* sK = sKV + stage * C::kStageBytes;
        uint8_t* sV = sK + C::kKBytes;
        const bool self = j < Ts;
        const CUtensorMap* mk = self ? &map_k : &map_kb;
        const CUtensorMap* mv = self ? &map_vt : &map_vbt;
        const int tok = self ? n * a.L + j * KT : bidx * a.Lb + (j - Ts) * KT;
        const int vcol = self ? n * a.vt_stride + j * KT : bidx * a.vbt_stride + (j - Ts) * KT;
        mbar_wait(&bar_k_empty[stage], phase ^ 1);
        mbar_arrive_expect_tx(&bar_k_full[stage], C::kKBytes);
#pragma unroll
        for (int kc = 0; kc < C::kKC; ++kc) tma_load_2d(sK + kc * KT * 128, mk, &bar_k_full[stage], h * DP + kc * 64, tok);
        mbar_wait(&bar_v_empty[stage], phase ^ 1);
        mbar_arrive_expect_tx(&bar_v_full[stage], C::kVBytes);
        tma_load_2d(sV, mv, &bar_v_full[stage], vcol, h * DV);
        tma_load_2d(sV + C::kVChunk, mv, &bar_v_full[stage], vcol + 64, h * DV);
        if (++stage == NS) { stage = 0; phase ^= 1; }
      }
    }
    return;
  }

  // ---------------------------------------------------------------- math warpgroups: rows 64 wg + 16 wq + lane/4 (+ 8)
  setmaxnreg_inc<kMathRegs>();
  const int wg = (warp >> 2) - 1, wq = warp & 3, quad = lane & 3;
  const float sc = a.scale_log2;
  const uint32_t aQ = smem_u32(sQ) + wg * 64 * 128;   // this warpgroup's 64 query rows (8 swizzle atoms)
  float o[DV / 2];
#pragma unroll
  for (int i = 0; i < DV / 2; ++i) o[i] = 0.f;
  float m_used[2] = {-INFINITY, -INFINITY};
  float s[KT / 2];          // scores of the next key tile, then its p = 2^(s*scale - m) in fp32
  uint32_t pa[KT / 16][4];  // p of the current tile as the packed fp16 A fragments of O += P V (16 keys per fragment)
  bool grow[2];
  float alpha[2];

  auto issue_qk = [&](int st) {
    const uint32_t aK = smem_u32(sKV + st * C::kStageBytes);
#pragma unroll
    for (int ks = 0; ks < DP / 16; ++ks)
      wgmma_ss<KT>(s, gmma_desc_k_sw128(aQ + (ks / 4) * QT * 128) + 2 * (ks % 4), gmma_desc_k_sw128(aK + (ks / 4) * KT * 128) + 2 * (ks % 4),
                   ks != 0 ? 1u : 0u);
    wgmma_commit();
  };
  // keys past the segment's end are masked; only a segment's last tile can be partial, every other tile skips the mask
  auto softmax = [&](int j) {
    const int kv_valid = j < Ts ? a.L - j * KT : a.Lb - (j - Ts) * KT;
    if (kv_valid < KT)
      tile_softmax<true>(s, kv_valid, quad, sc, m_used, grow, alpha);
    else
      tile_softmax<false>(s, KT, quad, sc, m_used, grow, alpha);
  };
  // Pipelined, O is rescaled branch-free (a factor of exactly 1 leaves O bit for bit as it was): ptxas serialises every wgmma of
  // the kernel when a data-dependent branch writes O between two MMAs that accumulate into it.
  auto rescale_o = [&] {
#pragma unroll
    for (int hh = 0; hh < 2; ++hh) {
      if (!C::kPipelined && !grow[hh]) continue;
      const float f = grow[hh] ? alpha[hh] : 1.f;
#pragma unroll
      for (int jj = 0; jj < DV / 8; ++jj) {
        o[4 * jj + 2 * hh] *= f;
        o[4 * jj + 2 * hh + 1] *= f;
      }
    }
  };
  auto pack_p = [&] {
#pragma unroll
    for (int kk = 0; kk < KT / 16; ++kk)
#pragma unroll
      for (int half = 0; half < 2; ++half)
#pragma unroll
        for (int hh = 0; hh < 2; ++hh) pa[kk][2 * half + hh] = pack_h2(s[4 * (2 * kk + half) + 2 * hh], s[4 * (2 * kk + half) + 2 * hh + 1]);
  };

  mbar_wait(bar_q, 0);
  int stage = 0;
  uint32_t phase = 0;
  if constexpr (!C::kPipelined) {
    // ---- one key tile at a time: S_j, softmax, O += P_j V_j
    for (int j = 0; j < T; ++j) {
      mbar_wait(&bar_k_full[stage], phase);
      wgmma_fence();
      issue_qk(stage);
      wgmma_wait<0>();
      wgmma_fence_regs(s);
      if (lane == 0) mbar_arrive(&bar_k_empty[stage]);
      softmax(j);
      rescale_o();
      pack_p();
      mbar_wait(&bar_v_full[stage], phase);
      const uint32_t aV = smem_u32(sKV + stage * C::kStageBytes + C::kKBytes);
      wgmma_fence_regs(o);
      wgmma_fence();
#pragma unroll
      for (int kk = 0; kk < KT / 16; ++kk) wgmma_rs<DV>(o, pa[kk], gmma_desc_k_sw128(aV + (kk / 4) * C::kVChunk) + 2 * (kk % 4), 1u);
      wgmma_commit();
      wgmma_wait<0>();
      wgmma_fence_regs(o);
      if (lane == 0) mbar_arrive(&bar_v_empty[stage]);
      if (++stage == NS) { stage = 0; phase ^= 1; }
    }
  } else {
    // ---- prologue: S_0, its softmax and P_0
    mbar_wait(&bar_k_full[0], 0);
    wgmma_fence();
    issue_qk(0);
    wgmma_wait<0>();
    wgmma_fence_regs(s);
    if (lane == 0) mbar_arrive(&bar_k_empty[0]);
    softmax(0);
    rescale_o();
    pack_p();

    // ---- steady state, one key tile per iteration: S_{j+1} = Q K_{j+1} and O += P_j V_j are issued back to back; the softmax of
    // S_{j+1} runs while P_j V_j is still on the tensor cores.  O is rescaled (and P_{j+1} written over P_j) once P_j V_j has completed,
    // so O accumulates in the same order, with the same rescale decisions, as a strictly serial loop.
    // `next`: tile j + 1 exists.  Called with a constant, so the last tile's copy has no conditional MMA issue (ptxas serialises
    // wgmma behind any divergent path around one).
    auto step = [&](int j, bool next) {
      const int nstage = stage + 1 == NS ? 0 : stage + 1;
      const uint32_t nphase = stage + 1 == NS ? phase ^ 1 : phase;
      if (next) mbar_wait(&bar_k_full[nstage], nphase);
      mbar_wait(&bar_v_full[stage], phase);
      wgmma_fence_regs(o);
      wgmma_fence();
      if (next) issue_qk(nstage);
      const uint32_t aV = smem_u32(sKV + stage * C::kStageBytes + C::kKBytes);
#pragma unroll
      for (int kk = 0; kk < KT / 16; ++kk) wgmma_rs<DV>(o, pa[kk], gmma_desc_k_sw128(aV + (kk / 4) * C::kVChunk) + 2 * (kk % 4), 1u);
      wgmma_commit();
      if (next) {
        wgmma_wait<1>();
        wgmma_fence_regs(s);
        if (lane == 0) mbar_arrive(&bar_k_empty[nstage]);
        softmax(j + 1);
      }
      wgmma_wait<0>();
      wgmma_fence_regs(o);
      wgmma_fence_regs(pa);
      if (lane == 0) mbar_arrive(&bar_v_empty[stage]);
      if (next) {
        rescale_o();
        pack_p();
      }
      stage = nstage;
      phase = nphase;
    };
    for (int j = 0; j + 1 < T; ++j) step(j, true);
    step(T - 1, false);
  }

  // ---- epilogue: O / denominator (column D of O, held by lane quad (D % 8) / 2 of the row)
#pragma unroll
  for (int hh = 0; hh < 2; ++hh) {
    const float den = __shfl_sync(0xffffffffu, o[4 * (D / 8) + 2 * hh + (D & 1)], (lane & ~3) | ((D % 8) / 2));
    const int qrow = q0 + wg * 64 + wq * 16 + (lane >> 2) + 8 * hh;
    if (qrow < a.L) {
      const float inv = 1.f / den;
      __half* dst = a.out + (static_cast<long long>(n) * a.L + qrow) * a.ldo + h * D;
#pragma unroll
      for (int jj = 0; jj < D / 8; ++jj)
        *reinterpret_cast<uint32_t*>(dst + 8 * jj + 2 * quad) = pack_h2(o[4 * jj + 2 * hh] * inv, o[4 * jj + 2 * hh + 1] * inv);
    }
  }
}

template <int D>
int launch_attn_t(const AttnArgs& a, cudaStream_t stream) {
  using C = ACfg<D>;
  static_assert(C::kStages >= 1, "one K/V stage must fit in shared memory");
  CUtensorMap mq, mk, mvt, mkb, mvbt;
  const long long tokens = static_cast<long long>(a.NF) * a.L;
  // the maps span the heads * dpad columns that exist: the last head's 64-column box then ends in TMA's zero fill instead of
  // reading past the row (past the buffer's end for K's last token, where K sits after Q in an interleaved row)
  const long long cols = static_cast<long long>(a.heads) * C::kDpad;
  bool maps = make_map_2d(&mq, a.q, tokens, cols, a.ldq, QT) && make_map_2d(&mk, a.k, tokens, cols, a.ldk, KT) &&
              make_map_2d(&mvt, a.vt, static_cast<long long>(a.heads) * C::kDv, static_cast<long long>(a.NF) * a.vt_stride, a.ldvt, C::kDv);
  mkb = mk;
  mvbt = mvt;
  const int B = a.NF / (a.F > 0 ? a.F : 1);
  if (maps && a.Lb > 0)
    maps = make_map_2d(&mkb, a.kb, static_cast<long long>(B) * a.Lb, a.ldkb, a.ldkb, KT) &&
           make_map_2d(&mvbt, a.vbt, static_cast<long long>(a.heads) * C::kDv, static_cast<long long>(B) * a.vbt_stride, a.ldvbt, C::kDv);
  if (!maps) {
    set_error("hv_op_attention (d = %d) map: %s", D, tma_last_error());
    return HV_ERR_TMA;
  }
  AttnKernelArgs ka;
  ka.out = a.out;
  ka.ldo = a.ldo;
  ka.L = a.L;
  ka.Lb = a.Lb;
  ka.F = a.F > 0 ? a.F : 1;
  ka.nf_nobank = a.nf_nobank;
  ka.heads = a.heads;
  ka.vt_stride = static_cast<int>(a.vt_stride);
  ka.vbt_stride = static_cast<int>(a.vbt_stride);
  ka.scale_log2 = 1.4426950408889634f / sqrtf(static_cast<float>(D));
  static bool attr = false;
  if (!attr) {
    cudaError_t e = cudaFuncSetAttribute(attn_kernel<D>, cudaFuncAttributeMaxDynamicSharedMemorySize, C::kSmemBytes);
    if (e != cudaSuccess) return cuda_status(e, "hv_op_attention");
    attr = true;
  }
  dim3 grid((a.L + QT - 1) / QT, a.heads, a.NF);
  attn_kernel<D><<<grid, ATT_THREADS, C::kSmemBytes, stream>>>(mq, mk, mvt, mkb, mvbt, ka);
  return cuda_status(cudaGetLastError(), "hv_op_attention");
}

}  // namespace

int op_attention(const __half* Q, const __half* K, const __half* Vt, __half* out, int64_t NF, int64_t L, int heads, int d, int64_t ldq,
                 int64_t ldk, int64_t ldvt, int64_t ldo, const __half* Kb, const __half* Vbt, int64_t Lb, int64_t ldkb, int64_t ldvbt, int64_t F,
                 int64_t nf_nobank, int64_t vt_stride, int64_t vbt_stride, cudaStream_t stream) {
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
  a.q = Q; a.k = K; a.vt = Vt; a.out = out;
  a.NF = (int)NF; a.L = (int)L; a.heads = heads; a.d = d; a.dpad = (int)dpad;  // V^T rows per head: (d + 1 + 15) / 16 * 16, row d of every head = ones
  a.ldq = ldq; a.ldk = ldk; a.ldvt = ldvt; a.ldo = ldo;
  a.kb = Kb; a.vbt = Vbt; a.Lb = bank ? (int)Lb : 0; a.ldkb = ldkb; a.ldvbt = ldvbt;
  a.F = (int)F; a.nf_nobank = (int)nf_nobank; a.vt_stride = vt_stride; a.vbt_stride = vbt_stride;
  switch (d) {
    case 8: return launch_attn_t<8>(a, stream);
    case 16: return launch_attn_t<16>(a, stream);
    case 32: return launch_attn_t<32>(a, stream);
    case 40: return launch_attn_t<40>(a, stream);
    case 64: return launch_attn_t<64>(a, stream);
    case 80: return launch_attn_t<80>(a, stream);
    default: return launch_attn_t<160>(a, stream);   // d_ok above
  }
}

}  // namespace hv
