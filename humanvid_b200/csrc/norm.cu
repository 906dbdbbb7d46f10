// GroupNorm (+SiLU) and LayerNorm (+cross-attention residual, +temporal positional encoding) on channels-last fp16.
// Both are HBM-bound passes: fp32 statistics and fp32 arithmetic through norm -> SiLU / PE add, one fp16 rounding at the store.
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdlib.h>

#include "ops.h"
#include "ptx.cuh"

namespace hv {

namespace {

__device__ __forceinline__ void unpack8(const uint4& u, float* v) {
  const __half2* h = reinterpret_cast<const __half2*>(&u);
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    float2 f = __half22float2(h[i]);
    v[2 * i] = f.x;
    v[2 * i + 1] = f.y;
  }
}
__device__ __forceinline__ uint4 pack8(const float* v) {
  uint4 u;
  u.x = pack_h2(v[0], v[1]);
  u.y = pack_h2(v[2], v[3]);
  u.z = pack_h2(v[4], v[5]);
  u.w = pack_h2(v[6], v[7]);
  return u;
}

// ---------------------------------------------------------------- GroupNorm statistics (deterministic: no atomics)
// The sums are taken of x - p, with one pivot p per (frame, group): the group's first channel in the frame's first row, read by every
// block that needs it.  var = E[(x-p)^2] - E[x-p]^2 then cancels only as much as p is away from the mean, about one standard deviation,
// where E[x^2] - E[x]^2 loses all its digits once a group's mean is ~100x its standard deviation (fp32 sums of ~1700 rows per thread
// at the VAE's full resolution).
__device__ __forceinline__ float gn_pivot(const __half* __restrict__ x1, int C1, const __half* __restrict__ x2, int C2, int HW, int n, int c) {
  return c < C1 ? __half2float(__ldg(x1 + static_cast<long long>(n) * HW * C1 + c)) : __half2float(__ldg(x2 + static_cast<long long>(n) * HW * C2 + (c - C1)));
}

// grid (slabs, NF); thread = (row lane, 8-channel vector).  Each block writes its per-group {sum, sumsq} of x - pivot to
// partial[n][slab][g]; gn_apply_kernel adds the slabs in a fixed order -> {mean, rstd}.  The pivots are read from frame pn.
__device__ __forceinline__ void gn_stats_body(const __half* __restrict__ x1, int C1, const __half* __restrict__ x2, int C2, int HW, int groups,
                                              int rows_per_block, float* __restrict__ partial, int pn) {
  extern __shared__ float sred[];  // [blockDim.x][4][2]
  const int C = C1 + C2, vecs = C / 8, cpg = C / groups;
  const int n = blockIdx.y;
  const int rl = threadIdx.x / vecs, v = threadIdx.x % vecs, rpi = blockDim.x / vecs;
  const int c0 = v * 8;
  float s[4] = {0, 0, 0, 0}, q[4] = {0, 0, 0, 0}, pv[4];
#pragma unroll
  for (int i = 0; i < 4; ++i) pv[i] = gn_pivot(x1, C1, x2, C2, HW, pn, (c0 + 2 * i) / cpg * cpg);   // a half2 never straddles two groups
  {
    const __half* src;
    int ldc, cc;
    if (c0 < C1) { src = x1; ldc = C1; cc = c0; } else { src = x2; ldc = C2; cc = c0 - C1; }
    const int row_end = min(HW, (blockIdx.x + 1) * rows_per_block);
    const __half* base = src + static_cast<long long>(n) * HW * ldc + cc;
    int r = blockIdx.x * rows_per_block + rl;
    for (; r + 3 * rpi < row_end; r += 4 * rpi) {  // four independent 16-byte loads in flight per thread
      uint4 u[4];
#pragma unroll
      for (int k = 0; k < 4; ++k) u[k] = __ldg(reinterpret_cast<const uint4*>(base + static_cast<long long>(r + k * rpi) * ldc));
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        float f[8];
        unpack8(u[k], f);
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          const float d0 = f[2 * i] - pv[i], d1 = f[2 * i + 1] - pv[i];
          s[i] += d0 + d1;
          q[i] += d0 * d0 + d1 * d1;
        }
      }
    }
    for (; r < row_end; r += rpi) {
      uint4 u = __ldg(reinterpret_cast<const uint4*>(base + static_cast<long long>(r) * ldc));
      float f[8];
      unpack8(u, f);
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const float d0 = f[2 * i] - pv[i], d1 = f[2 * i + 1] - pv[i];
        s[i] += d0 + d1;
        q[i] += d0 * d0 + d1 * d1;
      }
    }
  }
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    sred[(threadIdx.x * 4 + i) * 2] = s[i];
    sred[(threadIdx.x * 4 + i) * 2 + 1] = q[i];
  }
  __syncthreads();
  // thread g sums, in a fixed order, every (row lane, half2) slot that belongs to group g (channels-per-group is even,
  // so a half2 never straddles two groups; the slots of a group are the contiguous half2 range [g*cpg/2, (g+1)*cpg/2))
  if (threadIdx.x < groups) {
    const int g = threadIdx.x, h0 = g * (cpg / 2), h1 = h0 + cpg / 2;
    float ss = 0.f, qq = 0.f;
    for (int r = 0; r < rpi; ++r)
      for (int hh = h0; hh < h1; ++hh) {
        const int slot = (r * vecs + hh / 4) * 4 + (hh & 3);
        ss += sred[slot * 2];
        qq += sred[slot * 2 + 1];
      }
    float* dst = partial + ((static_cast<long long>(n) * gridDim.x + blockIdx.x) * groups + g) * 2;
    dst[0] = ss;
    dst[1] = qq;
  }
}

// The launch bounds let ptxas use 56 registers: without them it keeps the kernel at 40 and issues the row loop's four loads one at a
// time (one 16-byte load in flight per thread; GroupNorm took 27 % longer in a VAE decode).
__global__ void __launch_bounds__(1024, 1) gn_stats_kernel(const __half* __restrict__ x1, int C1, const __half* __restrict__ x2, int C2, int HW, int groups,
                                int rows_per_block, float* __restrict__ partial) {
  gn_stats_body(x1, C1, x2, C2, HW, groups, rows_per_block, partial, blockIdx.y);
}

// Frame-pooled statistics: the same per-frame partial sums, taken relative to the pivot of the batch item's first frame (frames
// [b*F, (b+1)*F) are item b), so that the F frames' partials of one (item, group) add up without a per-frame correction.
__global__ void __launch_bounds__(1024, 1) gn_stats_pooled_kernel(const __half* __restrict__ x1, int C1, const __half* __restrict__ x2, int C2, int HW,
                                                                  int groups, int rows_per_block, float* __restrict__ partial, int F) {
  gn_stats_body(x1, C1, x2, C2, HW, groups, rows_per_block, partial, blockIdx.y - blockIdx.y % F);
}

// grid (groups, items), 128 threads: {mean, rstd} of one (item, group) from the F * slabs partials of its frames.  Thread t adds partials
// t, t + 128, ... in order, then a fixed tree over the block: the order depends on F * slabs only, never on the number of items.
constexpr int kGnFinalizeThreads = 128;
__global__ void __launch_bounds__(kGnFinalizeThreads) gn_finalize_pooled_kernel(const __half* __restrict__ x1, int C1, const __half* __restrict__ x2,
                                                                                int C2, int HW, int groups, const float* __restrict__ partial,
                                                                                int slabs, int F, float inv_cnt, float eps, float2* __restrict__ stat) {
  __shared__ float2 sh[kGnFinalizeThreads / 32];
  const int g = blockIdx.x, b = blockIdx.y, P = F * slabs;
  const float* base = partial + (static_cast<long long>(b) * P * groups + g) * 2;   // partial[b*F + f][slab][g] = base[(f * slabs + slab) * groups * 2]
  float ss = 0.f, qq = 0.f;
  for (int p = threadIdx.x; p < P; p += kGnFinalizeThreads) {
    const float2 pp = __ldg(reinterpret_cast<const float2*>(base + static_cast<long long>(p) * groups * 2));
    ss += pp.x;
    qq += pp.y;
  }
#pragma unroll
  for (int o = 16; o; o >>= 1) {
    ss += __shfl_xor_sync(0xffffffffu, ss, o);
    qq += __shfl_xor_sync(0xffffffffu, qq, o);
  }
  if ((threadIdx.x & 31) == 0) sh[threadIdx.x >> 5] = make_float2(ss, qq);
  __syncthreads();
  if (threadIdx.x == 0) {
    ss = (sh[0].x + sh[1].x) + (sh[2].x + sh[3].x);
    qq = (sh[0].y + sh[1].y) + (sh[2].y + sh[3].y);
    const float m = ss * inv_cnt;   // mean - pivot
    const int cpg = (C1 + C2) / groups;
    stat[static_cast<long long>(b) * groups + g] =
        make_float2(gn_pivot(x1, C1, x2, C2, HW, b * F, g * cpg) + m, rsqrtf(fmaxf(qq * inv_cnt - m * m, 0.f) + eps));
  }
}

// Normalises rows [blockIdx.x * rows_per_block, ...) of frame blockIdx.y with the per-group {mean, rstd} in sstat.  (gn_apply_kernel keeps
// its own copy of this loop: calling this function from it reorders its SASS.)
__device__ __forceinline__ void gn_apply_rows(const __half* __restrict__ x1, int C1, const __half* __restrict__ x2, int C2,
                                              const __half* __restrict__ gamma, const __half* __restrict__ beta, __half* __restrict__ out,
                                              int HW, int groups, int rows_per_block, int silu, const float2* sstat) {
  const int C = C1 + C2, vecs = C / 8, cpg = C / groups;
  const int n = blockIdx.y;
  const int rl = threadIdx.x / vecs, v = threadIdx.x % vecs, rpi = blockDim.x / vecs;
  const int c0 = v * 8;
  float sc[8], sh[8];
  {
    float gm[8], bt[8];
    unpack8(__ldg(reinterpret_cast<const uint4*>(gamma + c0)), gm);
    unpack8(__ldg(reinterpret_cast<const uint4*>(beta + c0)), bt);
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const float2 st = sstat[(c0 + 2 * k) / cpg];
#pragma unroll
      for (int j = 0; j < 2; ++j) {
        sc[2 * k + j] = st.y * gm[2 * k + j];
        sh[2 * k + j] = fmaf(-st.x, sc[2 * k + j], bt[2 * k + j]);
      }
    }
  }
  const __half* src;
  int ldc;
  if (c0 < C1) { src = x1 + static_cast<long long>(n) * HW * C1 + c0; ldc = C1; } else { src = x2 + static_cast<long long>(n) * HW * C2 + (c0 - C1); ldc = C2; }
  __half* dst = out + static_cast<long long>(n) * HW * C + c0;
  const int row_end = min(HW, (blockIdx.x + 1) * rows_per_block);
  auto emit = [&](const uint4& u, int r) {
    float f[8];
    unpack8(u, f);
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      float y = fmaf(f[j], sc[j], sh[j]);
      if (silu) y = __fdividef(y, 1.0f + __expf(-y));
      f[j] = y;
    }
    *reinterpret_cast<uint4*>(dst + static_cast<long long>(r) * C) = pack8(f);
  };
  int r = blockIdx.x * rows_per_block + rl;
  for (; r + 3 * rpi < row_end; r += 4 * rpi) {
    uint4 u[4];
#pragma unroll
    for (int k = 0; k < 4; ++k) u[k] = __ldg(reinterpret_cast<const uint4*>(src + static_cast<long long>(r + k * rpi) * ldc));
#pragma unroll
    for (int k = 0; k < 4; ++k) emit(u[k], r + k * rpi);
  }
  for (; r < row_end; r += rpi) emit(__ldg(reinterpret_cast<const uint4*>(src + static_cast<long long>(r) * ldc)), r);
}

// grid (slabs, NF), thread = (row lane, 8-channel vector) like the statistics kernel: the thread's channels are fixed, so
// gamma/beta/mean/rstd fold into one per-channel scale and shift kept in registers, and the row loop has no integer
// division and one FFMA + SiLU per element.
__global__ void gn_apply_kernel(const __half* __restrict__ x1, int C1, const __half* __restrict__ x2, int C2,
                                const __half* __restrict__ gamma, const __half* __restrict__ beta, __half* __restrict__ out,
                                int HW, int groups, int rows_per_block, int silu, const float* __restrict__ partial, int slabs, float inv_cnt,
                                float eps) {
  const int C = C1 + C2, vecs = C / 8, cpg = C / groups;
  const int n = blockIdx.y;
  const int rl = threadIdx.x / vecs, v = threadIdx.x % vecs, rpi = blockDim.x / vecs;
  const int c0 = v * 8;
  // {mean, rstd} of this frame's groups: four lanes per group add the per-slab partial sums (each lane its slabs in order, then a fixed
  // two-step tree -> deterministic), full warps only so that the shuffles are well defined whatever the block size
  extern __shared__ float2 sstat[];   // [groups]
  {
    const int full = (blockDim.x >> 5) << 5;
    if (static_cast<int>(threadIdx.x) < full) {
      for (int g0 = 0; g0 < groups; g0 += full / 4) {
        const int g = g0 + static_cast<int>(threadIdx.x) / 4, l = threadIdx.x & 3;
        float ss = 0.f, qq = 0.f;
        if (g < groups)
          for (int sl = l; sl < slabs; sl += 4) {
            const float2 pp = __ldg(reinterpret_cast<const float2*>(partial + ((static_cast<long long>(n) * slabs + sl) * groups + g) * 2));
            ss += pp.x;
            qq += pp.y;
          }
        ss += __shfl_xor_sync(0xffffffffu, ss, 1);
        qq += __shfl_xor_sync(0xffffffffu, qq, 1);
        ss += __shfl_xor_sync(0xffffffffu, ss, 2);
        qq += __shfl_xor_sync(0xffffffffu, qq, 2);
        if (g < groups && l == 0) {
          const float m = ss * inv_cnt;   // mean - pivot
          sstat[g] = make_float2(gn_pivot(x1, C1, x2, C2, HW, n, g * cpg) + m, rsqrtf(fmaxf(qq * inv_cnt - m * m, 0.f) + eps));
        }
      }
    }
    __syncthreads();
  }
  float sc[8], sh[8];
  {
    float gm[8], bt[8];
    unpack8(__ldg(reinterpret_cast<const uint4*>(gamma + c0)), gm);
    unpack8(__ldg(reinterpret_cast<const uint4*>(beta + c0)), bt);
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const float2 st = sstat[(c0 + 2 * k) / cpg];
#pragma unroll
      for (int j = 0; j < 2; ++j) {
        sc[2 * k + j] = st.y * gm[2 * k + j];
        sh[2 * k + j] = fmaf(-st.x, sc[2 * k + j], bt[2 * k + j]);
      }
    }
  }
  const __half* src;
  int ldc;
  if (c0 < C1) { src = x1 + static_cast<long long>(n) * HW * C1 + c0; ldc = C1; } else { src = x2 + static_cast<long long>(n) * HW * C2 + (c0 - C1); ldc = C2; }
  __half* dst = out + static_cast<long long>(n) * HW * C + c0;
  const int row_end = min(HW, (blockIdx.x + 1) * rows_per_block);
  auto emit = [&](const uint4& u, int r) {
    float f[8];
    unpack8(u, f);
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      float y = fmaf(f[j], sc[j], sh[j]);
      if (silu) y = __fdividef(y, 1.0f + __expf(-y));
      f[j] = y;
    }
    *reinterpret_cast<uint4*>(dst + static_cast<long long>(r) * C) = pack8(f);
  };
  int r = blockIdx.x * rows_per_block + rl;
  for (; r + 3 * rpi < row_end; r += 4 * rpi) {
    uint4 u[4];
#pragma unroll
    for (int k = 0; k < 4; ++k) u[k] = __ldg(reinterpret_cast<const uint4*>(src + static_cast<long long>(r + k * rpi) * ldc));
#pragma unroll
    for (int k = 0; k < 4; ++k) emit(u[k], r + k * rpi);
  }
  for (; r < row_end; r += rpi) emit(__ldg(reinterpret_cast<const uint4*>(src + static_cast<long long>(r) * ldc)), r);
}

// Frame-pooled apply: frame n of item n / F reads the item's {mean, rstd} written by gn_finalize_pooled_kernel.
__global__ void gn_apply_pooled_kernel(const __half* __restrict__ x1, int C1, const __half* __restrict__ x2, int C2,
                                       const __half* __restrict__ gamma, const __half* __restrict__ beta, __half* __restrict__ out,
                                       int HW, int groups, int rows_per_block, int silu, const float2* __restrict__ stat, int F) {
  gn_apply_rows(x1, C1, x2, C2, gamma, beta, out, HW, groups, rows_per_block, silu, stat + static_cast<long long>(blockIdx.y / F) * groups);
}

// ---------------------------------------------------------------- LayerNorm: one warp per row
// LPR lanes cooperate on one row (32/LPR rows per warp), each lane owning up to 5 vectors of 8 halves: C = 320 -> 8 lanes
// x 5 vectors, 640 -> 16 x 5, 1280 -> 32 x 5, so every lane is busy and five 16-byte loads per lane are in flight.
// FP8: the normalised fp32 row (after affine and pe) is quantised to e4m3 into out8 [rows][C] with one scale per row, out_scale[row]
// (ptx.cuh e4m3_inv / e4m3_scale); out is not written.
template <int LPR, bool FP8>
__global__ void __launch_bounds__(256) layernorm_kernel(const __half* __restrict__ x, const __half* __restrict__ gamma, const __half* __restrict__ beta,
                                 __half* __restrict__ out, long long rows, int C, float eps, const __half* __restrict__ pre_add,
                                 long long rows_per_group, __half* __restrict__ x_out, const __half* __restrict__ pe, int hw, int F,
                                 uint8_t* __restrict__ out8, float* __restrict__ out_scale) {
  constexpr int MAXV = 5;
  constexpr int RPW = 32 / LPR;   // rows per warp
  const int lane = threadIdx.x & 31;
  const int sub = lane % LPR, rsel = lane / LPR;
  const int vecs = C / 8;
  const long long warps_total = static_cast<long long>(gridDim.x) * (blockDim.x >> 5);
  // grid-stride over row groups: a few resident blocks per SM stream the whole tensor (10 368 one-shot blocks at level 0 spent a third of
  // the kernel in block turnover: 4.1 TB/s against the 6.5 TB/s a copy reaches)
  for (long long warp_global = blockIdx.x * static_cast<long long>(blockDim.x >> 5) + (threadIdx.x >> 5); warp_global * RPW < rows; warp_global += warps_total) {
  const long long row = warp_global * RPW + rsel;
  const bool row_ok = row < rows;
  float v[MAXV][8];
  float sum = 0.f;
  const __half* add = (pre_add && row_ok) ? pre_add + (row / rows_per_group) * C : nullptr;
#pragma unroll
  for (int k = 0; k < MAXV; ++k) {
    const int vi = sub + LPR * k;
    if (row_ok && vi < vecs) unpack8(__ldg(reinterpret_cast<const uint4*>(x + row * C + vi * 8)), v[k]);
    else {
#pragma unroll
      for (int j = 0; j < 8; ++j) v[k][j] = 0.f;
    }
  }
#pragma unroll
  for (int k = 0; k < MAXV; ++k) {
    const int vi = sub + LPR * k;
    if (row_ok && vi < vecs) {
      if (add) {
        float a[8];
        unpack8(__ldg(reinterpret_cast<const uint4*>(add + vi * 8)), a);
#pragma unroll
        for (int j = 0; j < 8; ++j) v[k][j] += a[j];
        if (x_out) *reinterpret_cast<uint4*>(x_out + row * C + vi * 8) = pack8(v[k]);
      }
#pragma unroll
      for (int j = 0; j < 8; ++j) sum += v[k][j];
    }
  }
#pragma unroll
  for (int o = LPR / 2; o; o >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
  const float mean = sum / C;
  float sq = 0.f;
#pragma unroll
  for (int k = 0; k < MAXV; ++k) {
    const int vi = sub + LPR * k;
    if (vi < vecs) {
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const float d = v[k][j] - mean;
        sq += d * d;
      }
    }
  }
#pragma unroll
  for (int o = LPR / 2; o; o >>= 1) sq += __shfl_xor_sync(0xffffffffu, sq, o);
  const float rstd = rsqrtf(sq / C + eps);
  const __half* pe_row = (pe && row_ok) ? pe + static_cast<long long>((row / hw) % F) * C : nullptr;
#pragma unroll
  for (int k = 0; k < MAXV; ++k) {
    const int vi = sub + LPR * k;
    if (row_ok && vi < vecs) {
      float gm[8], bt[8];
      unpack8(__ldg(reinterpret_cast<const uint4*>(gamma + vi * 8)), gm);
      unpack8(__ldg(reinterpret_cast<const uint4*>(beta + vi * 8)), bt);
#pragma unroll
      for (int j = 0; j < 8; ++j) v[k][j] = (v[k][j] - mean) * rstd * gm[j] + bt[j];
      if (pe_row) {
        float pv[8];
        unpack8(__ldg(reinterpret_cast<const uint4*>(pe_row + vi * 8)), pv);
#pragma unroll
        for (int j = 0; j < 8; ++j) v[k][j] += pv[j];
      }
      if constexpr (!FP8) *reinterpret_cast<uint4*>(out + row * C + vi * 8) = pack8(v[k]);
    }
  }
  if constexpr (FP8) {
    float amax = 0.f;
#pragma unroll
    for (int k = 0; k < MAXV; ++k)
      if (row_ok && sub + LPR * k < vecs)
#pragma unroll
        for (int j = 0; j < 8; ++j) amax = fmaxf(amax, fabsf(v[k][j]));
#pragma unroll
    for (int o = LPR / 2; o; o >>= 1) amax = fmaxf(amax, __shfl_xor_sync(0xffffffffu, amax, o));
    const float inv = e4m3_inv(amax);
#pragma unroll
    for (int k = 0; k < MAXV; ++k) {
      const int vi = sub + LPR * k;
      if (row_ok && vi < vecs) {
        uint2 q;
        q.x = e4m3x2(v[k][0], v[k][1], inv) | (static_cast<uint32_t>(e4m3x2(v[k][2], v[k][3], inv)) << 16);
        q.y = e4m3x2(v[k][4], v[k][5], inv) | (static_cast<uint32_t>(e4m3x2(v[k][6], v[k][7], inv)) << 16);
        *reinterpret_cast<uint2*>(out8 + row * C + vi * 8) = q;
      }
    }
    if (row_ok && sub == 0) out_scale[row] = e4m3_scale(amax);
  }
  }
}

// ---------------------------------------------------------------- CLIP token assembly + pre_layrnorm: one 128-thread block per token row
// Row (b, t) of the B x L tokens is x = (t == 0 ? class_embedding : patch row b * (L - 1) + t - 1) + position_embedding[t], normalised over C
// in fp32 and written once in fp16 (the residual stream entering the first encoder layer).  Each thread holds up to 2 vectors of 8: C <= 2048.
__device__ __forceinline__ float block_sum128(float v, float* sh) {
#pragma unroll
  for (int o = 16; o; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  if ((threadIdx.x & 31) == 0) sh[threadIdx.x >> 5] = v;
  __syncthreads();
  const float s = (sh[0] + sh[1]) + (sh[2] + sh[3]);
  __syncthreads();
  return s;
}

__global__ void __launch_bounds__(128) clip_embed_ln_kernel(const __half* __restrict__ patch, const __half* __restrict__ cls,
                                                            const __half* __restrict__ pos, const __half* __restrict__ gamma,
                                                            const __half* __restrict__ beta, __half* __restrict__ out, int L, int C, float eps) {
  constexpr int MAXV = 2;
  __shared__ float sh[4];
  const long long row = blockIdx.x;
  const int t = static_cast<int>(row % L);
  const long long b = row / L;
  const __half* src = t == 0 ? cls : patch + (b * (L - 1) + t - 1) * C;
  const __half* pr = pos + static_cast<long long>(t) * C;
  const int vecs = C / 8;
  float v[MAXV][8];
  float sum = 0.f;
#pragma unroll
  for (int k = 0; k < MAXV; ++k) {
    const int vi = threadIdx.x + 128 * k;
    if (vi < vecs) {
      float p[8];
      unpack8(__ldg(reinterpret_cast<const uint4*>(src + vi * 8)), v[k]);
      unpack8(__ldg(reinterpret_cast<const uint4*>(pr + vi * 8)), p);
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        v[k][j] += p[j];
        sum += v[k][j];
      }
    }
  }
  const float mean = block_sum128(sum, sh) / C;
  float sq = 0.f;
#pragma unroll
  for (int k = 0; k < MAXV; ++k)
    if (threadIdx.x + 128 * k < vecs)
#pragma unroll
      for (int j = 0; j < 8; ++j) sq += (v[k][j] - mean) * (v[k][j] - mean);
  const float rstd = rsqrtf(block_sum128(sq, sh) / C + eps);
#pragma unroll
  for (int k = 0; k < MAXV; ++k) {
    const int vi = threadIdx.x + 128 * k;
    if (vi < vecs) {
      float gm[8], bt[8];
      unpack8(__ldg(reinterpret_cast<const uint4*>(gamma + vi * 8)), gm);
      unpack8(__ldg(reinterpret_cast<const uint4*>(beta + vi * 8)), bt);
#pragma unroll
      for (int j = 0; j < 8; ++j) v[k][j] = (v[k][j] - mean) * rstd * gm[j] + bt[j];
      *reinterpret_cast<uint4*>(out + row * C + vi * 8) = pack8(v[k]);
    }
  }
}

}  // namespace

int op_clip_embed_ln(const __half* patch, const __half* cls, const __half* pos, const __half* gamma, const __half* beta, __half* out, int64_t rows,
                     int64_t L, int64_t C, float eps, cudaStream_t stream) {
  if (!patch || !cls || !pos || !gamma || !beta || !out || !aligned16(patch) || !aligned16(cls) || !aligned16(pos) || !aligned16(gamma) ||
      !aligned16(beta) || !aligned16(out) || C % 8 || C / 8 > 256 || L < 1 || rows <= 0 || rows % L || rows > INT32_MAX) {
    set_error("clip_embed_ln: bad arguments rows=%lld L=%lld C=%lld (16-byte aligned tensors, C a multiple of 8 <= 2048, L divides rows)",
              (long long)rows, (long long)L, (long long)C);
    return HV_ERR_INVALID;
  }
  clip_embed_ln_kernel<<<static_cast<unsigned>(rows), 128, 0, stream>>>(patch, cls, pos, gamma, beta, out, static_cast<int>(L), static_cast<int>(C), eps);
  return cuda_status(cudaGetLastError(), "clip_embed_ln");
}

// scratch floats needed by op_groupnorm: final {mean, rstd} + per-slab partials
// The split of a frame's rows into slabs (= the order its statistics are summed in) depends on HW only, never on the number of frames in
// the batch: a forward of one CFG half (a unit of the multi-GPU split) is then bitwise equal to that half of a CFG batch.
// (Measured and rejected: normalising ~56 MB chunks of frames at a time so that the apply pass re-reads from L2 what the statistics pass
// just pulled in -- the smaller launches lose far more bandwidth than the L2 hits return: 135 us -> 250 us at level 0.)
static void gn_plan(int C, int HW, int* threads, int* slabs, int* rows_per_block) {
  const int vecs = C / 8;
  int t = vecs * (vecs >= 256 ? 1 : 256 / vecs);
  if (t > 1024) t = vecs;
  int sl = 16;
  int rpb = (HW + sl - 1) / sl;
  if (rpb < 32) rpb = 32;
  sl = (HW + rpb - 1) / rpb;
  *threads = t;
  *slabs = sl;
  *rows_per_block = rpb;
}
size_t groupnorm_scratch_floats(int C, int NF, int HW, int groups) {
  int t, sl, rpb;
  gn_plan(C, HW, &t, &sl, &rpb);
  return static_cast<size_t>(2) * NF * groups * (1 + sl);
}

// The arguments both GroupNorms can run: F = frames per item (1 for op_groupnorm).  The kernels load X, X2, gamma, beta and out 16 bytes
// at a time and stats as float2; NF is the grid's y dimension.
static int check_groupnorm(const char* op, const __half* X, int64_t C1, const __half* X2, int64_t C2, const __half* gamma, const __half* beta,
                           const __half* out, int64_t NF, int64_t HW, int groups, int64_t F, const float* stats) {
  bool ok = X && gamma && beta && out && stats && (C2 == 0 || X2) && C1 > 0 && C2 >= 0 && C1 + C2 <= 8192 && NF > 0 && HW > 0 && HW <= INT32_MAX &&
            F > 0 && NF % F == 0 && NF <= 65535 && aligned16(X) && (C2 == 0 || aligned16(X2)) && aligned16(gamma) && aligned16(beta) &&
            aligned16(out) && (reinterpret_cast<uintptr_t>(stats) & 7) == 0;
  const int C = static_cast<int>(C1 + C2);
  // the channel layouts the kernels run; gn_plan divides by C / 8, so it comes after C % 8 == 0 (and C1 > 0)
  ok = ok && groups > 0 && C % 8 == 0 && C1 % 8 == 0 && C % groups == 0 && ((C / groups) & 1) == 0 && groups <= 32 * 8;
  if (ok) {
    int threads, slabs, rows_per_block;
    gn_plan(C, static_cast<int>(HW), &threads, &slabs, &rows_per_block);
    ok = threads >= groups && threads >= 32;
  }
  if (!ok)
    set_error("%s: bad arguments C1=%lld C2=%lld NF=%lld HW=%lld groups=%d frames_per_item=%lld (NF %% F == 0, NF <= 65535, 16-byte aligned "
              "tensors, 8-byte aligned stats, C1 and C1 + C2 multiples of 8, C1 + C2 <= 8192, C / groups even, groups <= 256)", op, (long long)C1,
              (long long)C2, (long long)NF, (long long)HW, groups, (long long)F);
  return ok ? HV_OK : HV_ERR_INVALID;
}

int op_groupnorm(const __half* x1, int64_t C1, const __half* x2, int64_t C2, const __half* gamma, const __half* beta, __half* out, int64_t NF,
                 int64_t HW, int groups, float eps, int silu, float* stats, cudaStream_t stream) {
  if (int rc = check_groupnorm("hv_op_groupnorm", x1, C1, x2, C2, gamma, beta, out, NF, HW, groups, 1, stats)) return rc;
  const int C = static_cast<int>(C1 + C2);
  int threads, slabs, rows_per_block;
  gn_plan(C, static_cast<int>(HW), &threads, &slabs, &rows_per_block);
  float* partial = stats + static_cast<size_t>(2) * NF * groups;
  gn_stats_kernel<<<dim3(slabs, static_cast<unsigned>(NF)), threads, threads * 8 * sizeof(float), stream>>>(x1, static_cast<int>(C1), x2, static_cast<int>(C2),
                                                                                                          static_cast<int>(HW), groups, rows_per_block, partial);
  // (the {mean, rstd} finalize is folded into the apply kernel: one launch less per GroupNorm, 83 per forward)
  gn_apply_kernel<<<dim3(slabs, static_cast<unsigned>(NF)), threads, groups * sizeof(float2), stream>>>(
      x1, static_cast<int>(C1), x2, static_cast<int>(C2), gamma, beta, out, static_cast<int>(HW), groups, rows_per_block, silu, partial, slabs,
      1.f / (static_cast<float>(static_cast<int>(HW)) * (C / groups)), eps);
  return cuda_status(cudaGetLastError(), "hv_op_groupnorm");
}

// Statistics pooled over the F frames of each batch item (nn.GroupNorm on a (b, c, f, h, w) tensor).  Same scratch as op_groupnorm:
// the per-frame partials at the same offset, and the items' {mean, rstd} in the first 2 * (NF / F) * groups floats.  At F = 1 this is
// op_groupnorm itself.
int op_groupnorm_pooled(const __half* x1, int64_t C1, const __half* x2, int64_t C2, const __half* gamma, const __half* beta, __half* out,
                        int64_t NF, int64_t HW, int groups, float eps, int silu, int64_t F, float* stats, cudaStream_t stream) {
  if (int rc = check_groupnorm("hv_op_groupnorm_pooled", x1, C1, x2, C2, gamma, beta, out, NF, HW, groups, F, stats)) return rc;
  if (C2 == 0) x2 = nullptr;
  if (F == 1) return op_groupnorm(x1, C1, x2, C2, gamma, beta, out, NF, HW, groups, eps, silu, stats, stream);
  const int C = static_cast<int>(C1 + C2), Fi = static_cast<int>(F), HWi = static_cast<int>(HW);
  int threads, slabs, rows_per_block;
  gn_plan(C, HWi, &threads, &slabs, &rows_per_block);
  float2* stat = reinterpret_cast<float2*>(stats);
  float* partial = stats + static_cast<size_t>(2) * NF * groups;
  const dim3 grid(slabs, static_cast<unsigned>(NF));
  gn_stats_pooled_kernel<<<grid, threads, threads * 8 * sizeof(float), stream>>>(x1, static_cast<int>(C1), x2, static_cast<int>(C2), HWi, groups,
                                                                                 rows_per_block, partial, Fi);
  gn_finalize_pooled_kernel<<<dim3(groups, static_cast<unsigned>(NF / F)), kGnFinalizeThreads, 0, stream>>>(
      x1, static_cast<int>(C1), x2, static_cast<int>(C2), HWi, groups, partial, slabs, Fi, 1.f / (static_cast<float>(Fi) * HWi * (C / groups)), eps, stat);
  gn_apply_pooled_kernel<<<grid, threads, 0, stream>>>(x1, static_cast<int>(C1), x2, static_cast<int>(C2), gamma, beta, out, HWi, groups,
                                                       rows_per_block, silu, stat, Fi);
  return cuda_status(cudaGetLastError(), "hv_op_groupnorm_pooled");
}

// The kernel holds up to 160 vectors of 8 per row (C <= 1280) and loads x, pre_add, gamma, beta and pe and stores out and x_out 16 bytes at a time.
template <bool FP8>
static int run_layernorm(const char* op, const __half* x, const __half* gamma, const __half* beta, __half* out, int64_t rows, int64_t C, float eps,
                         const __half* pre_add, int64_t rows_per_group, __half* x_out, const __half* pe, int64_t hw, int64_t F, uint8_t* out8,
                         float* out_scale, cudaStream_t stream) {
  const int vecs = static_cast<int>(C / 8);
  if (rows_per_group <= 0) rows_per_group = 1;
  if (hw <= 0) hw = 1;
  if (F <= 0) F = 1;
  const int lpr = vecs <= 40 ? 8 : (vecs <= 80 ? 16 : 32);
  const int wpb = 8;
  const long long warps = (rows + (32 / lpr) - 1) / (32 / lpr);
  const int sms = device_sms();
  if (!sms) return HV_ERR_CUDA;
  long long blocks = (warps + wpb - 1) / wpb;
  if (blocks > 8LL * sms) blocks = 8LL * sms;   // persistent grid: 8 blocks per SM
  const unsigned grid = static_cast<unsigned>(blocks);
  const int Ci = static_cast<int>(C), hwi = static_cast<int>(hw), Fi = static_cast<int>(F);
  if (lpr == 8)
    layernorm_kernel<8, FP8><<<grid, wpb * 32, 0, stream>>>(x, gamma, beta, out, rows, Ci, eps, pre_add, rows_per_group, x_out, pe, hwi, Fi, out8, out_scale);
  else if (lpr == 16)
    layernorm_kernel<16, FP8><<<grid, wpb * 32, 0, stream>>>(x, gamma, beta, out, rows, Ci, eps, pre_add, rows_per_group, x_out, pe, hwi, Fi, out8, out_scale);
  else
    layernorm_kernel<32, FP8><<<grid, wpb * 32, 0, stream>>>(x, gamma, beta, out, rows, Ci, eps, pre_add, rows_per_group, x_out, pe, hwi, Fi, out8, out_scale);
  return cuda_status(cudaGetLastError(), op);
}

int op_layernorm(const __half* x, const __half* gamma, const __half* beta, __half* out, int64_t rows, int64_t C, float eps, const __half* pre_add,
                 int64_t rows_per_group, __half* x_out, const __half* pe, int64_t hw, int64_t F, cudaStream_t stream) {
  if (!x || !gamma || !beta || !out || !aligned16(x) || !aligned16(gamma) || !aligned16(beta) || !aligned16(out) || !aligned16(pre_add) ||
      !aligned16(x_out) || !aligned16(pe) || rows < 1 || C < 8 || C > 1280 || C % 8 || hw > INT32_MAX || F > INT32_MAX) {
    set_error("hv_op_layernorm: bad arguments rows=%lld C=%lld hw=%lld F=%lld (non-NULL, 16-byte aligned tensors, rows >= 1, C a multiple of 8 "
              "<= 1280, hw and F <= INT32_MAX)", (long long)rows, (long long)C, (long long)hw, (long long)F);
    return HV_ERR_INVALID;
  }
  return run_layernorm<false>("hv_op_layernorm", x, gamma, beta, out, rows, C, eps, pre_add, rows_per_group, x_out, pe, hw, F, nullptr, nullptr, stream);
}

int op_layernorm_fp8(const __half* x, const __half* gamma, const __half* beta, uint8_t* out, float* out_scale, int64_t rows, int64_t C, float eps,
                     const __half* pre_add, int64_t rows_per_group, __half* x_out, const __half* pe, int64_t hw, int64_t F, cudaStream_t stream) {
  if (!x || !gamma || !beta || !out || !out_scale || !aligned16(x) || !aligned16(gamma) || !aligned16(beta) || !aligned16(out) ||
      !aligned16(out_scale) || !aligned16(pre_add) || !aligned16(x_out) || !aligned16(pe) || rows < 1 || C < 16 || C > 1280 || C % 16 ||
      hw > INT32_MAX || F > INT32_MAX) {
    set_error("hv_op_layernorm_fp8: bad arguments rows=%lld C=%lld hw=%lld F=%lld (non-NULL out and out_scale, 16-byte aligned tensors, rows >= 1, "
              "C a multiple of 16 <= 1280, hw and F <= INT32_MAX)", (long long)rows, (long long)C, (long long)hw, (long long)F);
    return HV_ERR_INVALID;
  }
  return run_layernorm<true>("hv_op_layernorm_fp8", x, gamma, beta, nullptr, rows, C, eps, pre_add, rows_per_group, x_out, pe, hw, F, out, out_scale,
                             stream);
}

}  // namespace hv
