// Attention over the frame axis (AnimateDiff motion module, reference src/models/motion_module.py:351-388 and
// src/cameractrl/motion_module.py:323-388): for every (batch item, pixel, head) a softmax(q k^T / sqrt(d)) v with
// F <= 32 frames.  The reference materialises "(b f) d c -> (b d) f c" transposes around SDPA; here the frame axis is
// simply the strided axis of the channels-last token matrix, so nothing is transposed in memory.
//
// One warp per (b, pixel, head).  Q K^T and P V run on mma.sync.m16n8k16 register fragments (problems are 24x24xd:
// far too small for a wgmma tile; the op is bound by HBM traffic of q,k,v,o, ~0.2% of the step's FLOPs), the
// softmax row max / row sum are warp-shuffle reductions over the 4 lanes that share a row.
#include <cuda.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdlib.h>

#include "ops.h"
#include "ptx.cuh"
#include "tma.h"

namespace hv {

namespace {

__device__ __forceinline__ void mma16816(float (&c)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
  asm volatile(
      "mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
      : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}

__device__ __forceinline__ uint32_t ldg_h2(const __half* p) { return __ldg(reinterpret_cast<const unsigned int*>(p)); }
__device__ __forceinline__ uint32_t pack2(float a, float b) {
  __half2 h = __floats2half2_rn(a, b);
  return *reinterpret_cast<uint32_t*>(&h);
}
__device__ __forceinline__ uint32_t pack2h(__half a, __half b) {
  __half2 h = __halves2half2(a, b);
  return *reinterpret_cast<uint32_t*>(&h);
}

// QKV: [B*F*HW][3*C] rows (b, f, p); q at column h*D, k at C + h*D, v at 2C + h*D.
template <int D>
__global__ void __launch_bounds__(256, (D <= 40) ? 3 : 1) temporal_attn_kernel(const __half* __restrict__ qkv, __half* __restrict__ out, int B,
                                                           int F, int HW, int heads, float scale_log2) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int g = lane >> 2, t = lane & 3;
  const long long prob = static_cast<long long>(blockIdx.x) * (blockDim.x >> 5) + warp;
  const long long nprob = static_cast<long long>(B) * HW * heads;
  if (prob >= nprob) return;
  const int h = static_cast<int>(prob % heads);
  const long long bp = prob / heads;
  const int p = static_cast<int>(bp % HW);
  const int b = static_cast<int>(bp / HW);
  const int C = heads * D;
  const long long ld = 3LL * C;
  const long long fstride = static_cast<long long>(HW) * ld;  // elements between consecutive frames of one pixel
  const __half* qb = qkv + (static_cast<long long>(b) * F * HW + p) * ld + h * D;
  const __half* kb = qb + C;
  const __half* vb = qb + 2 * C;

  constexpr int KS = (D + 15) / 16;  // k16 steps of Q K^T
  // ---- S = Q K^T : 2 m-tiles (frames 0..31) x 4 n-tiles (keys 0..31)
  float s[2][4][4];
#pragma unroll
  for (int mt = 0; mt < 2; ++mt)
#pragma unroll
    for (int nt = 0; nt < 4; ++nt)
#pragma unroll
      for (int i = 0; i < 4; ++i) s[mt][nt][i] = 0.f;

#pragma unroll
  for (int ks = 0; ks < KS; ++ks) {
    const int c_lo = ks * 16 + 2 * t, c_hi = c_lo + 8;
    const bool lo_ok = ks * 16 < D, hi_ok = ks * 16 + 8 < D;
    uint32_t a[2][4];
#pragma unroll
    for (int mt = 0; mt < 2; ++mt) {
      const int r0 = mt * 16 + g, r1 = r0 + 8;
      a[mt][0] = (lo_ok && r0 < F) ? ldg_h2(qb + r0 * fstride + c_lo) : 0u;
      a[mt][1] = (lo_ok && r1 < F) ? ldg_h2(qb + r1 * fstride + c_lo) : 0u;
      a[mt][2] = (hi_ok && r0 < F) ? ldg_h2(qb + r0 * fstride + c_hi) : 0u;
      a[mt][3] = (hi_ok && r1 < F) ? ldg_h2(qb + r1 * fstride + c_hi) : 0u;
    }
#pragma unroll
    for (int nt = 0; nt < 4; ++nt) {
      const int j = nt * 8 + g;
      const uint32_t b0 = (lo_ok && j < F) ? ldg_h2(kb + j * fstride + c_lo) : 0u;
      const uint32_t b1 = (hi_ok && j < F) ? ldg_h2(kb + j * fstride + c_hi) : 0u;
      mma16816(s[0][nt], a[0], b0, b1);
      mma16816(s[1][nt], a[1], b0, b1);
    }
  }

  // ---- prefetch V (issued before the softmax so the loads overlap it): the B fragment of P V needs
  // (V[2t][c], V[2t+1][c]) with c = nt*8 + g, i.e. two rows of one column.  Each lane instead loads one half2
  // (row 2t + (g&1), columns c&~1, c|1) and swaps halves with its partner lane g^1 (lane ^ 4): 4-byte loads, half as many.
  constexpr int NTV = D / 8;
  constexpr bool kPrefetchV = D <= 40;
  uint32_t vfr[kPrefetchV ? NTV : 1][2][2];
  auto load_v = [&](int nt, int kk, int hi) -> uint32_t {
    const int j = kk * 16 + hi * 8 + 2 * t + (g & 1);
    const int c = nt * 8 + (g & ~1);
    return j < F ? ldg_h2(vb + j * fstride + c) : 0u;
  };
  auto fix_v = [&](uint32_t x) -> uint32_t {
    const uint32_t y = __shfl_xor_sync(0xffffffffu, x, 4);
    // even g: (x.lo, y.lo)   odd g: (y.hi, x.hi)
    return (g & 1) ? __byte_perm(y, x, 0x7632) : __byte_perm(x, y, 0x5410);
  };
  if constexpr (kPrefetchV) {
#pragma unroll
    for (int nt = 0; nt < NTV; ++nt)
#pragma unroll
      for (int kk = 0; kk < 2; ++kk) {
        vfr[nt][kk][0] = load_v(nt, kk, 0);
        vfr[nt][kk][1] = load_v(nt, kk, 1);
      }
  }

  // ---- softmax over keys (columns); rows g / g+8 of each m-tile; quad (t) shares a row
  uint32_t pa[2][2][4];  // P as A fragments: [m-tile][k16 step over keys][4]
  float inv_sum[2][2];
#pragma unroll
  for (int mt = 0; mt < 2; ++mt) {
#pragma unroll
    for (int half = 0; half < 2; ++half) {  // half 0: row g (regs 0,1), half 1: row g+8 (regs 2,3)
      float m = -INFINITY;
#pragma unroll
      for (int nt = 0; nt < 4; ++nt) {
        const int j0 = nt * 8 + 2 * t;
        if (j0 < F) m = fmaxf(m, s[mt][nt][half * 2]);
        if (j0 + 1 < F) m = fmaxf(m, s[mt][nt][half * 2 + 1]);
      }
      m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, 1));
      m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, 2));
      float sum = 0.f;
#pragma unroll
      for (int nt = 0; nt < 4; ++nt) {
        const int j0 = nt * 8 + 2 * t;
        float e0 = j0 < F ? exp2f((s[mt][nt][half * 2] - m) * scale_log2) : 0.f;
        float e1 = j0 + 1 < F ? exp2f((s[mt][nt][half * 2 + 1] - m) * scale_log2) : 0.f;
        sum += e0 + e1;
        s[mt][nt][half * 2] = e0;
        s[mt][nt][half * 2 + 1] = e1;
      }
      sum += __shfl_xor_sync(0xffffffffu, sum, 1);
      sum += __shfl_xor_sync(0xffffffffu, sum, 2);
      inv_sum[mt][half] = 1.f / sum;
    }
#pragma unroll
    for (int kk = 0; kk < 2; ++kk) {
      pa[mt][kk][0] = pack2(s[mt][2 * kk][0], s[mt][2 * kk][1]);
      pa[mt][kk][1] = pack2(s[mt][2 * kk][2], s[mt][2 * kk][3]);
      pa[mt][kk][2] = pack2(s[mt][2 * kk + 1][0], s[mt][2 * kk + 1][1]);
      pa[mt][kk][3] = pack2(s[mt][2 * kk + 1][2], s[mt][2 * kk + 1][3]);
    }
  }

  // ---- O = P V, one n8 tile of the head dim at a time
  __half* ob = out + (static_cast<long long>(b) * F * HW + p) * C + h * D;
  const long long ostride = static_cast<long long>(HW) * C;
#pragma unroll
  for (int nt = 0; nt < NTV; ++nt) {
    float o[2][4] = {{0.f, 0.f, 0.f, 0.f}, {0.f, 0.f, 0.f, 0.f}};
#pragma unroll
    for (int kk = 0; kk < 2; ++kk) {
      uint32_t x0, x1;
      if constexpr (kPrefetchV) {
        x0 = vfr[nt][kk][0];
        x1 = vfr[nt][kk][1];
      } else {
        x0 = load_v(nt, kk, 0);
        x1 = load_v(nt, kk, 1);
      }
      const uint32_t b0 = fix_v(x0), b1 = fix_v(x1);
      mma16816(o[0], pa[0][kk], b0, b1);
      mma16816(o[1], pa[1][kk], b0, b1);
    }
#pragma unroll
    for (int mt = 0; mt < 2; ++mt) {
      const int r0 = mt * 16 + g, r1 = r0 + 8;
      const int col = nt * 8 + 2 * t;
      if (r0 < F)
        *reinterpret_cast<__half2*>(ob + r0 * ostride + col) = __floats2half2_rn(o[mt][0] * inv_sum[mt][0], o[mt][1] * inv_sum[mt][0]);
      if (r1 < F)
        *reinterpret_cast<__half2*>(ob + r1 * ostride + col) = __floats2half2_rn(o[mt][2] * inv_sum[mt][1], o[mt][3] * inv_sum[mt][1]);
    }
  }
}

// ---------------------------------------------------------------------------------------------------------------------
// TMA-staged variant (d = 40 / 80, the two high-resolution levels = 80 % of the temporal-attention time).  The register
// kernel above gathers every operand with 4-byte loads at a (pixels x 3C x 2)-byte stride: 88 LDG/STG per lane and problem
// and half-used sectors held it at ~38 % of HBM speed.  Here every warp owns a private shared-memory slab; one elected
// lane fetches the F rows of q, k and v of its (pixel, head) with three 3-D TMA boxes (d x 1 x F: rows of 2d bytes, stride
// = one frame), the fragments come from ldmatrix (the row pitch of 2d bytes = 80 is bank-conflict free for 16-byte rows),
// and O goes back through the q slab with one TMA store.  d = 40: two slabs per warp, the next problem's boxes are in flight
// while this one is computed.
constexpr int TT_WARPS = 12;

// HPB = heads fetched per box: d = 40 takes two heads per slab row (160-byte rows -- 80-byte TMA rows ran at 2.6 TB/s, the
// request rate of the TMA unit being the limit), the warp then computes them one after the other.
template <int D, int HPB>
struct TTCfg {
  static constexpr int kPitch = D * HPB * 2;                 // bytes per slab row
  static constexpr int kSlab = 32 * kPitch;                  // 32 rows (F <= 32; rows >= F: garbage for q/k, zeros for v)
  static constexpr int kBuf = 3 * kSlab;                     // q | k | v
  static constexpr int kNBuf = (TT_WARPS * 2 * kBuf <= 200 * 1024) ? 2 : 1;
  static constexpr int kSmemBytes = TT_WARPS * kNBuf * kBuf + TT_WARPS * kNBuf * 8 + 1024;
};

__device__ __forceinline__ void ldsm_x4(uint32_t addr, uint32_t& r0, uint32_t& r1, uint32_t& r2, uint32_t& r3) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0,%1,%2,%3}, [%4];" : "=r"(r0), "=r"(r1), "=r"(r2), "=r"(r3) : "r"(addr));
}
__device__ __forceinline__ void ldsm_x2(uint32_t addr, uint32_t& r0, uint32_t& r1) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x2.shared.b16 {%0,%1}, [%2];" : "=r"(r0), "=r"(r1) : "r"(addr));
}
__device__ __forceinline__ void ldsm_x1(uint32_t addr, uint32_t& r0) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x1.shared.b16 {%0}, [%1];" : "=r"(r0) : "r"(addr));
}
__device__ __forceinline__ void ldsm_x2_t(uint32_t addr, uint32_t& r0, uint32_t& r1) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x2.trans.shared.b16 {%0,%1}, [%2];" : "=r"(r0), "=r"(r1) : "r"(addr));
}

template <int D, int HPB>
__global__ void __launch_bounds__(TT_WARPS * 32, 1)
temporal_attn_tma_kernel(const __grid_constant__ CUtensorMap map_qkv, const __grid_constant__ CUtensorMap map_out, int B, int F, int HW,
                         int heads, float scale_log2) {
  using C = TTCfg<D, HPB>;
  constexpr int PITCH = C::kPitch, NB = C::kNBuf;
  constexpr int KS = (D + 15) / 16;          // k16 steps of Q K^T (the last one is half wide when D % 16 == 8)
  constexpr bool kHalfLast = (D % 16) == 8;
  constexpr int NTV = D / 8;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 127) & ~uintptr_t(127));
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int g = lane >> 2, t = lane & 3;
  uint8_t* wbuf = smem + warp * (NB * C::kBuf);
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + TT_WARPS * NB * C::kBuf) + warp * NB;
  const int Cc = heads * D;

  // v rows F..31 take part in P V with p = 0: they must be finite, so zero them once (TMA only ever writes rows < F)
  for (int b = 0; b < NB; ++b) {
    uint8_t* v = wbuf + b * C::kBuf + 2 * C::kSlab;
    for (int i = F * PITCH + lane * 16; i < 32 * PITCH; i += 32 * 16) *reinterpret_cast<uint4*>(v + i) = make_uint4(0, 0, 0, 0);
  }
  if (lane == 0) {
    for (int b = 0; b < NB; ++b) mbar_init(&bars[b], 1);
    fence_mbar_init();
    fence_proxy_async();
  }
  __syncwarp();

  const int hgroups = heads / HPB;
  const long long nprob = static_cast<long long>(B) * HW * hgroups;      // one problem = HPB heads of one (batch item, pixel)
  const long long nwarps = static_cast<long long>(gridDim.x) * TT_WARPS;
  const long long first = static_cast<long long>(blockIdx.x) * TT_WARPS + warp;
  auto issue = [&](long long prob, int buf) {   // lane 0 only
    const int h = static_cast<int>(prob % hgroups) * HPB;
    const long long bp = prob / hgroups;
    const int p = static_cast<int>(bp % HW), b = static_cast<int>(bp / HW);
    uint8_t* dst = wbuf + buf * C::kBuf;
    mbar_arrive_expect_tx(&bars[buf], 3 * F * PITCH);
    tma_load_3d(dst, &map_qkv, &bars[buf], h * D, p, b * F);
    tma_load_3d(dst + C::kSlab, &map_qkv, &bars[buf], Cc + h * D, p, b * F);
    tma_load_3d(dst + 2 * C::kSlab, &map_qkv, &bars[buf], 2 * Cc + h * D, p, b * F);
  };
  if (lane == 0 && first < nprob) issue(first, 0);
  int buf = 0;
  uint32_t phase[2] = {0, 0};
  for (long long prob = first; prob < nprob; prob += nwarps) {
    if (NB == 2 && lane == 0) {
      tma_store_wait_read();                               // the store that read the other slab's q region has drained it
      if (prob + nwarps < nprob) issue(prob + nwarps, buf ^ 1);
    }
    mbar_wait(&bars[buf], phase[buf]);
    phase[buf] ^= 1;
#pragma unroll 1
    for (int hh = 0; hh < HPB; ++hh) {
    const uint32_t sq = smem_u32(wbuf + buf * C::kBuf) + hh * D * 2, sk = sq + C::kSlab, sv = sq + 2 * C::kSlab;

    // ---- S = Q K^T : 2 m-tiles (frames) x 4 n-tiles (keys)
    float s[2][4][4];
#pragma unroll
    for (int mt = 0; mt < 2; ++mt)
#pragma unroll
      for (int nt = 0; nt < 4; ++nt)
#pragma unroll
        for (int i = 0; i < 4; ++i) s[mt][nt][i] = 0.f;
#pragma unroll
    for (int ks = 0; ks < KS; ++ks) {
      const bool half = kHalfLast && ks == KS - 1;
      uint32_t a[2][4];
#pragma unroll
      for (int mt = 0; mt < 2; ++mt) {
        if (!half) {
          ldsm_x4(sq + (mt * 16 + (lane & 15)) * PITCH + (ks * 16 + (lane >> 4) * 8) * 2, a[mt][0], a[mt][1], a[mt][2], a[mt][3]);
        } else {
          ldsm_x2(sq + (mt * 16 + (lane & 15)) * PITCH + ks * 32, a[mt][0], a[mt][1]);
          a[mt][2] = a[mt][3] = 0u;
        }
      }
#pragma unroll
      for (int nt = 0; nt < 4; ++nt) {
        uint32_t b0, b1 = 0u;
        if (!half) ldsm_x2(sk + (nt * 8 + (lane & 7)) * PITCH + (ks * 16 + ((lane >> 3) & 1) * 8) * 2, b0, b1);
        else ldsm_x1(sk + (nt * 8 + (lane & 7)) * PITCH + ks * 32, b0);
        mma16816(s[0][nt], a[0], b0, b1);
        mma16816(s[1][nt], a[1], b0, b1);
      }
    }

    // ---- softmax over keys (columns); rows g / g+8 of each m-tile; quad (t) shares a row
    uint32_t pa[2][2][4];
    float inv_sum[2][2];
#pragma unroll
    for (int mt = 0; mt < 2; ++mt) {
#pragma unroll
      for (int hh = 0; hh < 2; ++hh) {
        float m = -INFINITY;
#pragma unroll
        for (int nt = 0; nt < 4; ++nt) {
          const int j0 = nt * 8 + 2 * t;
          if (j0 < F) m = fmaxf(m, s[mt][nt][hh * 2]);
          if (j0 + 1 < F) m = fmaxf(m, s[mt][nt][hh * 2 + 1]);
        }
        m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, 1));
        m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, 2));
        float sum = 0.f;
#pragma unroll
        for (int nt = 0; nt < 4; ++nt) {
          const int j0 = nt * 8 + 2 * t;
          const float e0 = j0 < F ? exp2f((s[mt][nt][hh * 2] - m) * scale_log2) : 0.f;
          const float e1 = j0 + 1 < F ? exp2f((s[mt][nt][hh * 2 + 1] - m) * scale_log2) : 0.f;
          sum += e0 + e1;
          s[mt][nt][hh * 2] = e0;
          s[mt][nt][hh * 2 + 1] = e1;
        }
        sum += __shfl_xor_sync(0xffffffffu, sum, 1);
        sum += __shfl_xor_sync(0xffffffffu, sum, 2);
        inv_sum[mt][hh] = 1.f / sum;
      }
#pragma unroll
      for (int kk = 0; kk < 2; ++kk) {
        pa[mt][kk][0] = pack2(s[mt][2 * kk][0], s[mt][2 * kk][1]);
        pa[mt][kk][1] = pack2(s[mt][2 * kk][2], s[mt][2 * kk][3]);
        pa[mt][kk][2] = pack2(s[mt][2 * kk + 1][0], s[mt][2 * kk + 1][1]);
        pa[mt][kk][3] = pack2(s[mt][2 * kk + 1][2], s[mt][2 * kk + 1][3]);
      }
    }

    // ---- O = P V, one n8 tile of the head dim at a time; rows of O overwrite the q slab (q is dead after S)
    __syncwarp();
#pragma unroll
    for (int nt = 0; nt < NTV; ++nt) {
      float o[2][4] = {{0.f, 0.f, 0.f, 0.f}, {0.f, 0.f, 0.f, 0.f}};
#pragma unroll
      for (int kk = 0; kk < 2; ++kk) {
        uint32_t b0, b1;
        ldsm_x2_t(sv + (kk * 16 + (lane & 15)) * PITCH + nt * 16, b0, b1);
        mma16816(o[0], pa[0][kk], b0, b1);
        mma16816(o[1], pa[1][kk], b0, b1);
      }
      uint8_t* qs = wbuf + buf * C::kBuf + hh * D * 2;
#pragma unroll
      for (int mt = 0; mt < 2; ++mt) {
        const int r0 = mt * 16 + g, r1 = r0 + 8;
        const int colb = (nt * 8 + 2 * t) * 2;
        if (r0 < F) *reinterpret_cast<__half2*>(qs + r0 * PITCH + colb) = __floats2half2_rn(o[mt][0] * inv_sum[mt][0], o[mt][1] * inv_sum[mt][0]);
        if (r1 < F) *reinterpret_cast<__half2*>(qs + r1 * PITCH + colb) = __floats2half2_rn(o[mt][2] * inv_sum[mt][1], o[mt][3] * inv_sum[mt][1]);
      }
    }
    }  // heads of this box
    fence_proxy_async();
    __syncwarp();
    if (lane == 0) {
      const int h = static_cast<int>(prob % hgroups) * HPB;
      const long long bp = prob / hgroups;
      const int p = static_cast<int>(bp % HW), b = static_cast<int>(bp / HW);
      tma_store_3d(&map_out, wbuf + buf * C::kBuf, h * D, p, b * F);
      tma_store_commit();
      if (NB == 1) {
        tma_store_wait_read();
        if (prob + nwarps < nprob) issue(prob + nwarps, 0);
      }
    }
    __syncwarp();
    if (NB == 2) buf ^= 1;
  }
  if (lane == 0) tma_store_wait_all();
}

template <int D, int HPB>
static int launch_tt(const __half* qkv, __half* out, int B, int F, int HW, int heads, float scale_log2, unsigned grid, cudaStream_t stream) {
  using C = TTCfg<D, HPB>;
  const int Cc = heads * D;
  CUtensorMap mq, mo;
  if (!make_map_frames(&mq, qkv, static_cast<int64_t>(B) * F, HW, 3LL * Cc, 3LL * Cc, D * HPB, F) ||
      !make_map_frames(&mo, out, static_cast<int64_t>(B) * F, HW, Cc, Cc, D * HPB, F)) {
    set_error("hv_op_temporal_attention map: %s", tma_last_error());
    return HV_ERR_TMA;
  }
  static bool attr = false;
  if (!attr) {
    cudaError_t e = cudaFuncSetAttribute(temporal_attn_tma_kernel<D, HPB>, cudaFuncAttributeMaxDynamicSharedMemorySize, C::kSmemBytes);
    if (e != cudaSuccess) return cuda_status(e, "hv_op_temporal_attention");
    attr = true;
  }
  temporal_attn_tma_kernel<D, HPB><<<grid, TT_WARPS * 32, C::kSmemBytes, stream>>>(mq, mo, B, F, HW, heads, scale_log2);
  return cuda_status(cudaGetLastError(), "hv_op_temporal_attention");
}

constexpr int kRegWarpsPerBlock = 8;

}  // namespace

// rows (b, f, p) and the one-warp-per-problem grid of the register kernel are indexed with ints
int plan_temporal_attention(const char* what, int64_t B, int64_t F, int64_t HW, int heads, int d, TemporalPlan* plan) {
  const bool d_ok = d == 8 || d == 16 || d == 32 || d == 40 || d == 80 || d == 160;
  if (B < 1 || B > INT32_MAX || F < 1 || F > 32 || HW < 1 || HW > INT32_MAX || heads < 1 || !d_ok || B * F > INT32_MAX || B * F * HW > INT32_MAX ||
      B * HW * heads > INT32_MAX || static_cast<int64_t>(heads) * d * 3 > INT32_MAX) {
    set_error("%s: bad shape B=%lld F=%lld HW=%lld heads=%d d=%d (B, HW, heads >= 1, 1 <= F <= 32, d one of 8, 16, 32, 40, 80, 160)", what,
              (long long)B, (long long)F, (long long)HW, heads, d);
    return HV_ERR_INVALID;
  }
  const int sms = device_sms();
  if (!sms) return HV_ERR_CUDA;
  TemporalPlan& p = *plan;
  const long long nprob = B * HW * heads;
  // the two high-resolution levels; small problems keep the register kernel.  The choice depends on HW only, not on the batch size
  // (a one-half unit of the multi-GPU split must run the same kernel as that half of a CFG batch).
  if (HW * heads >= 2048 && ((d == 40 && heads % 2 == 0) || d == 80)) {
    p.tma = true;
    p.heads_per_box = d == 40 ? 2 : 1;
    const long long ctas = (nprob / p.heads_per_box + TT_WARPS - 1) / TT_WARPS;   // persistent: at most one CTA per SM
    p.grid = static_cast<unsigned>(ctas < sms ? ctas : sms);
  } else {
    p.tma = false;
    p.heads_per_box = 1;
    p.grid = static_cast<unsigned>((nprob + kRegWarpsPerBlock - 1) / kRegWarpsPerBlock);
  }
  return HV_OK;
}

int op_temporal_attention(const __half* qkv, __half* out, int64_t B64, int64_t F64, int64_t HW64, int heads, int d, cudaStream_t stream) {
  if (!qkv || !out) { set_error("hv_op_temporal_attention: NULL pointer"); return HV_ERR_INVALID; }
  TemporalPlan plan;
  if (int rc = plan_temporal_attention("hv_op_temporal_attention", B64, F64, HW64, heads, d, &plan)) return rc;
  const int B = static_cast<int>(B64), F = static_cast<int>(F64), HW = static_cast<int>(HW64);
  const unsigned grid = plan.grid;
  const int wpb = kRegWarpsPerBlock;
  const float scale_log2 = 1.4426950408889634f / sqrtf(static_cast<float>(d));
  if (plan.tma) {
    if (d == 40) return launch_tt<40, 2>(qkv, out, B, F, HW, heads, scale_log2, grid, stream);
    return launch_tt<80, 1>(qkv, out, B, F, HW, heads, scale_log2, grid, stream);
  }
  switch (d) {
    case 40: temporal_attn_kernel<40><<<grid, wpb * 32, 0, stream>>>(qkv, out, B, F, HW, heads, scale_log2); break;
    case 80: temporal_attn_kernel<80><<<grid, wpb * 32, 0, stream>>>(qkv, out, B, F, HW, heads, scale_log2); break;
    case 160: temporal_attn_kernel<160><<<grid, wpb * 32, 0, stream>>>(qkv, out, B, F, HW, heads, scale_log2); break;
    case 32: temporal_attn_kernel<32><<<grid, wpb * 32, 0, stream>>>(qkv, out, B, F, HW, heads, scale_log2); break;
    case 16: temporal_attn_kernel<16><<<grid, wpb * 32, 0, stream>>>(qkv, out, B, F, HW, heads, scale_log2); break;
    default: temporal_attn_kernel<8><<<grid, wpb * 32, 0, stream>>>(qkv, out, B, F, HW, heads, scale_log2); break;   // d = 8 (checked above)
  }
  return cuda_status(cudaGetLastError(), "hv_op_temporal_attention");
}

}  // namespace hv
