// Small-channel 3x3 convolutions of the PoseGuider front (src/models/pose_guider.py:25-49: 3 -> 16 -> 16 -> 32 (s2) -> 32 -> 96 (s2) at up
// to 768x576 x 24 frames).  These layers are HBM-bound (a few hundred FLOP per byte of activation at most); padding their 16 / 32
// channels to the 64-channel k-block of the implicit-GEMM kernel would move 2-4x the necessary bytes.  Here they run at their true
// channel counts:
//
//   pg_conv_in_kernel            Cin = 3, read straight from the (B, 3, F, H, W) pose image (no layout pass), mma.sync with K = 27 -> 32
//   smallconv_mma_kernel<CIN, COUT, STRIDE>
//                                channels-last fp16, implicit GEMM on mma.sync.m16n8k16 (the problems are far below a wgmma tile):
//                                a CTA stages the (8 x 32 output) tile's input halo in shared memory with cp.async (zero fill = padding),
//                                each warp owns one output row of 32 pixels (two m16 tiles), A fragments come from ldmatrix at the
//                                tap-shifted halo pixels (no im2col), B fragments from the [Cout][9 * Cin] weight panel in shared
//                                memory, fp32 accumulators, bias + SiLU in fp32, one rounding, rows leave through shared memory as
//                                16-byte coalesced stores.
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include "ops.h"
#include "ptx.cuh"

namespace hv {

namespace {

__device__ __forceinline__ void cp_async16(void* smem, const void* gmem) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(smem_u32(smem)), "l"(gmem) : "memory");
}
__device__ __forceinline__ void cp_async_wait_all() { asm volatile("cp.async.wait_all;" ::: "memory"); }
__device__ __forceinline__ void ldsm_x4(const void* p, uint32_t& r0, uint32_t& r1, uint32_t& r2, uint32_t& r3) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0, %1, %2, %3}, [%4];" : "=r"(r0), "=r"(r1), "=r"(r2), "=r"(r3) : "r"(smem_u32(p)));
}
__device__ __forceinline__ void mma_16816(float (&c)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
  asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0, %1, %2, %3}, {%4, %5, %6, %7}, {%8, %9}, {%0, %1, %2, %3};"
               : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
               : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}

constexpr int SC_TH = 8, SC_TW = 32, SC_THREADS = 256;

template <int CIN, int COUT, int STRIDE>
struct SCfg {
  static constexpr int IH = (SC_TH - 1) * STRIDE + 3, IW = (SC_TW - 1) * STRIDE + 3;
  static constexpr int PIXP = CIN * 2 + 16;            // bytes per halo pixel (+16: ldmatrix rows of consecutive pixels hit distinct banks)
  static constexpr int WP = 9 * CIN * 2 + 16;          // bytes per weight row [cout][(ky*3+kx)*CIN + c]
  static constexpr int kHalo = IH * IW * PIXP;
  static constexpr int kW = COUT * WP;
  static constexpr int kOut = SC_TH * SC_TW * COUT * 2;  // output staging, aliases the halo
  static constexpr int kSmem = (kHalo > kOut ? kHalo : kOut) + kW + COUT * 4;
};

template <int CIN, int COUT, int STRIDE>
__global__ void __launch_bounds__(SC_THREADS)
smallconv_mma_kernel(const __half* __restrict__ x, const __half* __restrict__ wp, const __half* __restrict__ bias, __half* __restrict__ out, int H, int W,
                     int Ho, int Wo, int ldo, int act) {
  using C = SCfg<CIN, COUT, STRIDE>;
  extern __shared__ __align__(16) uint8_t smem[];
  uint8_t* halo = smem;
  uint8_t* wsm = smem + (C::kHalo > C::kOut ? C::kHalo : C::kOut);
  float* bsm = reinterpret_cast<float*>(wsm + C::kW);
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int n = blockIdx.z, y0 = blockIdx.y * SC_TH, x0 = blockIdx.x * SC_TW;

  // ---- stage the weight panel, the bias and the input halo (out-of-image pixels are the conv's zero padding)
  constexpr int WCH = 9 * CIN * 2 / 16;   // 16-byte chunks per weight row
  for (int i = tid; i < COUT * WCH; i += SC_THREADS) {
    const int r = i / WCH, c = i - r * WCH;
    cp_async16(wsm + r * C::WP + c * 16, wp + static_cast<size_t>(r) * 9 * CIN + c * 8);
  }
  for (int i = tid; i < COUT; i += SC_THREADS) bsm[i] = bias ? __half2float(bias[i]) : 0.f;
  constexpr int PCH = CIN * 2 / 16;       // 16-byte chunks per pixel
  const int iy0 = y0 * STRIDE - 1, ix0 = x0 * STRIDE - 1;
  for (int i = tid; i < C::IH * C::IW * PCH; i += SC_THREADS) {
    const int c = i % PCH, p = i / PCH;
    const int px = p % C::IW, py = p / C::IW;
    const int gy = iy0 + py, gx = ix0 + px;
    uint8_t* dst = halo + p * C::PIXP + c * 16;
    if (gy >= 0 && gy < H && gx >= 0 && gx < W) cp_async16(dst, x + ((static_cast<size_t>(n) * H + gy) * W + gx) * CIN + c * 8);
    else *reinterpret_cast<uint4*>(dst) = make_uint4(0, 0, 0, 0);
  }
  cp_async_wait_all();
  __syncthreads();

  // ---- implicit GEMM: this warp = output row (y0 + warp), 32 pixels = two m16 tiles; N = COUT; K = 9 taps x CIN
  float acc[2][COUT / 8][4];
#pragma unroll
  for (int mt = 0; mt < 2; ++mt)
#pragma unroll
    for (int nt = 0; nt < COUT / 8; ++nt)
#pragma unroll
      for (int i = 0; i < 4; ++i) acc[mt][nt][i] = 0.f;
  const int a_row = (lane & 7) + ((lane >> 3) & 1) * 8, a_kh = lane >> 4;          // ldmatrix.x4 lane -> (pixel of the m16 tile, k half)
  const int b_row = (lane & 7) + (lane >> 4) * 8, b_kh = (lane >> 3) & 1;          // ldmatrix.x4 lane -> (cout of the n16 pair, k half)
#pragma unroll 1
  for (int tap = 0; tap < 9; ++tap) {
    const int dy = tap / 3, dx = tap - dy * 3;
#pragma unroll
    for (int kb = 0; kb < CIN / 16; ++kb) {
      uint32_t a[2][4];
#pragma unroll
      for (int mt = 0; mt < 2; ++mt) {
        const int px = (mt * 16 + a_row) * STRIDE + dx, py = warp * STRIDE + dy;
        ldsm_x4(halo + (py * C::IW + px) * C::PIXP + kb * 32 + a_kh * 16, a[mt][0], a[mt][1], a[mt][2], a[mt][3]);
      }
#pragma unroll
      for (int np = 0; np < COUT / 16; ++np) {
        uint32_t b0, b1, b2, b3;
        ldsm_x4(wsm + (np * 16 + b_row) * C::WP + (tap * CIN + kb * 16 + b_kh * 8) * 2, b0, b1, b2, b3);
#pragma unroll
        for (int mt = 0; mt < 2; ++mt) {
          mma_16816(acc[mt][2 * np], a[mt], b0, b1);
          mma_16816(acc[mt][2 * np + 1], a[mt], b2, b3);
        }
      }
    }
  }
  __syncthreads();   // every warp is done reading the halo: its memory becomes the output staging buffer

  // ---- epilogue: bias + SiLU in fp32, one rounding; this warp's 32 x COUT row goes through shared memory and leaves in 16-byte pieces
  __half* orow = reinterpret_cast<__half*>(halo) + warp * SC_TW * COUT;
  const int r0 = lane >> 2, c0 = (lane & 3) * 2;
#pragma unroll
  for (int mt = 0; mt < 2; ++mt)
#pragma unroll
    for (int nt = 0; nt < COUT / 8; ++nt)
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int col = nt * 8 + c0;
        float v0 = acc[mt][nt][2 * h] + bsm[col], v1 = acc[mt][nt][2 * h + 1] + bsm[col + 1];
        if (act == 2) { v0 = silu_f(v0); v1 = silu_f(v1); } else if (act == 1) { v0 = fmaxf(v0, 0.f); v1 = fmaxf(v1, 0.f); }
        *reinterpret_cast<uint32_t*>(orow + (mt * 16 + r0 + 8 * h) * COUT + col) = pack_h2(v0, v1);
      }
  __syncwarp();
  const int y = y0 + warp;
  if (y < Ho) {
    constexpr int OCH = COUT * 2 / 16;    // 16-byte chunks per output pixel
    for (int i = lane; i < SC_TW * OCH; i += 32) {
      const int p = i / OCH, c = i - p * OCH;
      const int xo = x0 + p;
      if (xo < Wo)
        *reinterpret_cast<uint4*>(out + ((static_cast<size_t>(n) * Ho + y) * Wo + xo) * ldo + c * 8) = *reinterpret_cast<const uint4*>(orow + p * COUT + c * 8);
    }
  }
}

// conv_in of the PoseGuider: (B, 3, F, H, W) fp16 planes -> channels-last (B*F, H, W, 16), 3x3, padding 1, + bias, SiLU -- as an implicit
// GEMM on mma.sync.m16n8k16: M = pixels, N = 16, K = (ci, ky, kx) = 27 padded to 32 (the weight tensor (16, 3, 3, 3) IS the [n][k] operand).
// A block stages the 3 x (8 + 2) x (64 + 2) input halo of an 8 x 64 output tile in shared memory (zero fill = padding); a warp owns one
// output row = four m16 tiles; a lane builds its A fragment from 16 two-byte shared loads at compile-time-constant tap offsets (no im2col
// buffer), the 8 B-fragment registers are loaded once per thread.  Rows leave through shared memory as 16-byte coalesced stores.
constexpr int PG_TH = 8, PG_TW = 64, PG_ROWS = PG_TH + 2, PG_COLS = PG_TW + 2, PG_RS = PG_TW + 4, PG_OP = 24;   // PG_OP: halves per staged output pixel (16 + 8 pad: conflict-free)

__global__ void __launch_bounds__(256) pg_conv_in_kernel(const __half* __restrict__ x, const __half* __restrict__ w, const __half* __restrict__ bias,
                                                         __half* __restrict__ out, int B, int F, int H, int W, int act, int tiles_x, int tiles_y) {
  __shared__ __align__(16) __half tile[3 * PG_ROWS * PG_RS];
  __shared__ __align__(16) __half ostage[8][PG_TW * PG_OP];
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int g = lane >> 2, t = lane & 3;
  const long long HW = static_cast<long long>(H) * W;

  // ---- per-thread constants: B fragments (weights as [n][k], k >= 27 is zero) and the shared-memory offsets of this lane's 8 k indices
  uint32_t bf[2][2][2];   // [k16 step][n8 tile][k half]
  int koff[2][2][2];      // [k16 step][k half][element]
#pragma unroll
  for (int s = 0; s < 2; ++s)
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int k0 = s * 16 + h * 8 + 2 * t;
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        const int k = k0 + e;
        koff[s][h][e] = k < 27 ? ((k / 9) * PG_ROWS + (k % 9) / 3) * PG_RS + (k % 3) : 0;   // k >= 27: any finite value, its weight is zero
      }
#pragma unroll
      for (int j = 0; j < 2; ++j) {
        const __half lo = k0 < 27 ? w[(j * 8 + g) * 27 + k0] : __float2half(0.f);
        const __half hi = k0 + 1 < 27 ? w[(j * 8 + g) * 27 + k0 + 1] : __float2half(0.f);
        bf[s][j][h] = static_cast<uint32_t>(__half_as_ushort(lo)) | (static_cast<uint32_t>(__half_as_ushort(hi)) << 16);
      }
    }
  float bia[2][2];
#pragma unroll
  for (int j = 0; j < 2; ++j) {
    bia[j][0] = bias ? __half2float(bias[j * 8 + 2 * t]) : 0.f;
    bia[j][1] = bias ? __half2float(bias[j * 8 + 2 * t + 1]) : 0.f;
  }

  const long long ntiles = static_cast<long long>(B) * F * tiles_y * tiles_x;
  for (long long tl = blockIdx.x; tl < ntiles; tl += gridDim.x) {
    const int tx = static_cast<int>(tl % tiles_x);
    long long r = tl / tiles_x;
    const int ty = static_cast<int>(r % tiles_y);
    const long long nf = r / tiles_y;
    const int b = static_cast<int>(nf / F), f = static_cast<int>(nf % F);
    const int y0 = ty * PG_TH, x0 = tx * PG_TW;

    // ---- stage the halo of the three input planes; outside the image = the conv's zero padding
    for (int i = tid; i < 3 * PG_ROWS * PG_COLS; i += 256) {
      const int c = i % PG_COLS;
      const int rr = (i / PG_COLS) % PG_ROWS;
      const int ci = i / (PG_COLS * PG_ROWS);
      const int gy = y0 - 1 + rr, gx = x0 - 1 + c;
      __half v = __float2half(0.f);
      if (gy >= 0 && gy < H && gx >= 0 && gx < W) v = __ldg(x + ((static_cast<long long>(b) * 3 + ci) * F + f) * HW + static_cast<long long>(gy) * W + gx);
      tile[(ci * PG_ROWS + rr) * PG_RS + c] = v;
    }
    __syncthreads();

    // ---- this warp: output row y0 + warp, 64 pixels = four m16 tiles
    const unsigned short* tl16 = reinterpret_cast<const unsigned short*>(tile);
    __half* orow = ostage[warp];
#pragma unroll
    for (int mt = 0; mt < 4; ++mt) {
      const int pa = warp * PG_RS + mt * 16 + g, pb = pa + 8;
      float acc[2][4] = {{0.f, 0.f, 0.f, 0.f}, {0.f, 0.f, 0.f, 0.f}};
#pragma unroll
      for (int s = 0; s < 2; ++s) {
        uint32_t a[4];
        a[0] = static_cast<uint32_t>(tl16[koff[s][0][0] + pa]) | (static_cast<uint32_t>(tl16[koff[s][0][1] + pa]) << 16);   // row g,     k = 2t, 2t+1
        a[1] = static_cast<uint32_t>(tl16[koff[s][0][0] + pb]) | (static_cast<uint32_t>(tl16[koff[s][0][1] + pb]) << 16);   // row g + 8
        a[2] = static_cast<uint32_t>(tl16[koff[s][1][0] + pa]) | (static_cast<uint32_t>(tl16[koff[s][1][1] + pa]) << 16);   // row g,     k = 2t+8, 2t+9
        a[3] = static_cast<uint32_t>(tl16[koff[s][1][0] + pb]) | (static_cast<uint32_t>(tl16[koff[s][1][1] + pb]) << 16);   // row g + 8
        mma_16816(acc[0], a, bf[s][0][0], bf[s][0][1]);
        mma_16816(acc[1], a, bf[s][1][0], bf[s][1][1]);
      }
#pragma unroll
      for (int j = 0; j < 2; ++j)
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          float v0 = acc[j][2 * h] + bia[j][0], v1 = acc[j][2 * h + 1] + bia[j][1];
          if (act == 2) { v0 = silu_f(v0); v1 = silu_f(v1); } else if (act == 1) { v0 = fmaxf(v0, 0.f); v1 = fmaxf(v1, 0.f); }
          *reinterpret_cast<uint32_t*>(orow + (mt * 16 + g + 8 * h) * PG_OP + j * 8 + 2 * t) = pack_h2(v0, v1);
        }
    }
    __syncwarp();
    const int y = y0 + warp;
    if (y < H) {
      __half* dst = out + ((static_cast<size_t>(nf) * H + y) * W + x0) * 16;
      for (int i = lane; i < PG_TW * 2; i += 32) {
        const int p = i >> 1, c = i & 1;
        if (x0 + p < W) *reinterpret_cast<uint4*>(dst + p * 16 + c * 8) = *reinterpret_cast<const uint4*>(orow + p * PG_OP + c * 8);
      }
    }
    __syncthreads();   // every warp is done with the halo (and its staging row) before the next tile overwrites them
  }
}

template <int CIN, int COUT, int STRIDE>
int launch_sc(const __half* x, const __half* wp, const __half* bias, __half* out, int NF, int H, int W, int ldo, int act, cudaStream_t s) {
  using C = SCfg<CIN, COUT, STRIDE>;
  static bool attr = false;
  if (!attr) {
    cudaError_t e = cudaFuncSetAttribute(smallconv_mma_kernel<CIN, COUT, STRIDE>, cudaFuncAttributeMaxDynamicSharedMemorySize, C::kSmem);
    if (e != cudaSuccess) return cuda_status(e, "hv_op_conv3x3_small");
    attr = true;
  }
  const int Ho = STRIDE == 1 ? H : H / 2, Wo = STRIDE == 1 ? W : W / 2;
  dim3 grid((Wo + SC_TW - 1) / SC_TW, (Ho + SC_TH - 1) / SC_TH, NF);
  smallconv_mma_kernel<CIN, COUT, STRIDE><<<grid, SC_THREADS, C::kSmem, s>>>(x, wp, bias, out, H, W, Ho, Wo, ldo, act);
  return cuda_status(cudaGetLastError(), "hv_op_conv3x3_small");
}

}  // namespace

bool smallconv_supported(int64_t cin, int64_t cout, int stride) {
  return (cin == 16 && cout == 16 && stride == 1) || (cin == 16 && cout == 32 && stride == 2) || (cin == 32 && cout == 32 && stride == 1) ||
         (cin == 32 && cout == 96 && stride == 2);
}

// x (NF, H, W, cin) channels-last, wp [cout][9 * cin] (op_pack_conv3x3 with no padding), out (NF, Ho, Wo, ldo >= cout; pad columns untouched).
// x and wp are staged with 16-byte cp.async and out is written 16 bytes at a time; NF and the output's 8-row tiles are the grid's z and y.
int op_conv3x3_small(const __half* x, const __half* wp, const __half* bias, __half* out, int64_t ldo, int64_t NF, int64_t H, int64_t W, int64_t cin,
                     int64_t cout, int stride, int act, cudaStream_t s) {
  if (!smallconv_supported(cin, cout, stride)) {
    set_error("hv_op_conv3x3_small: (Cin, Cout, stride) = (%lld, %lld, %d) is not one of (16,16,1) (16,32,2) (32,32,1) (32,96,2)", (long long)cin,
              (long long)cout, stride);
    return HV_ERR_INVALID;
  }
  if (!x || !wp || !out || !aligned16(x) || !aligned16(wp) || !aligned16(out) || NF < 1 || NF > 65535 || H < 1 || W < 1 || H > INT32_MAX ||
      W > INT32_MAX || (H / stride + SC_TH - 1) / SC_TH > 65535 || (stride == 2 && ((H | W) & 1)) || (ldo % 8) || ldo < cout || ldo > INT32_MAX) {
    set_error("hv_op_conv3x3_small: bad arguments NF=%lld H=%lld W=%lld ldo=%lld (16-byte aligned X, Wp and out, 1 <= NF <= 65535, even H and W at "
              "stride 2, ldo >= Cout and a multiple of 8)", (long long)NF, (long long)H, (long long)W, (long long)ldo);
    return HV_ERR_INVALID;
  }
  const int n = static_cast<int>(NF), h = static_cast<int>(H), w = static_cast<int>(W), ld = static_cast<int>(ldo);
  if (cin == 16 && cout == 16) return launch_sc<16, 16, 1>(x, wp, bias, out, n, h, w, ld, act, s);
  if (cin == 16) return launch_sc<16, 32, 2>(x, wp, bias, out, n, h, w, ld, act, s);
  if (cout == 32) return launch_sc<32, 32, 1>(x, wp, bias, out, n, h, w, ld, act, s);
  return launch_sc<32, 96, 2>(x, wp, bias, out, n, h, w, ld, act, s);
}

// out (B*F, H, W, 16) is written 16 bytes at a time
int op_pose_conv_in(const __half* x, const __half* w, const __half* bias, __half* out, int64_t B, int64_t F, int64_t H, int64_t W, int act, cudaStream_t s) {
  if (!x || !w || !out || !aligned16(out) || B < 1 || F < 1 || H < 1 || W < 1 || B * F > INT32_MAX || H * W > INT32_MAX) {
    set_error("hv_op_pose_conv_in: bad arguments B=%lld F=%lld H=%lld W=%lld (non-NULL X, W and out, 16-byte aligned out, B, F, H, W >= 1, B*F and "
              "H*W within int32)", (long long)B, (long long)F, (long long)H, (long long)W);
    return HV_ERR_INVALID;
  }
  const int sms = device_sms();
  if (!sms) return HV_ERR_CUDA;
  const int Hi = static_cast<int>(H), Wi = static_cast<int>(W);
  const int tiles_x = (Wi + PG_TW - 1) / PG_TW, tiles_y = (Hi + PG_TH - 1) / PG_TH;
  long long blocks = B * F * tiles_y * tiles_x;
  if (blocks > static_cast<long long>(sms) * 7) blocks = static_cast<long long>(sms) * 7;   // 7 x 28.6 KB of static shared memory per SM
  pg_conv_in_kernel<<<static_cast<unsigned>(blocks), 256, 0, s>>>(x, w, bias, out, static_cast<int>(B), static_cast<int>(F), Hi, Wi, act, tiles_x, tiles_y);
  return cuda_status(cudaGetLastError(), "hv_op_pose_conv_in");
}

}  // namespace hv
