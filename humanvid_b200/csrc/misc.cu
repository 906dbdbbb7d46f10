// Glue kernels of the denoising path: layout changes at the (B,C,F,H,W) boundary, pixel unshuffle and the Plucker producer of
// the camera encoder, the tiny linears of the time embedding / cross-attention collapse, the timestep embedding, small-channel
// direct convolutions (PoseGuider conv_in), CLIP's patchify, weight packing, and a slow CUDA-core GEMM used only to localise faults in tests.
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include "ops.h"
#include "ptx.cuh"

namespace hv {

namespace {

constexpr int kThreads = 256;
inline unsigned blocks_for(long long n, int num_sms) {
  long long b = (n + kThreads - 1) / kThreads;
  long long cap = static_cast<long long>(num_sms) * 32;
  return static_cast<unsigned>(b < 1 ? 1 : (b > cap ? cap : b));
}

// (B, C, F, H, W) [fp16 or fp32] -> (B*F, H, W, C) fp16.  Tiled transpose of the (C, HW) plane of each (b, f).
template <typename T>
__global__ void ncfhw_to_nhwc_kernel(const T* __restrict__ x, __half* __restrict__ out, int B, int C, int F, int HW, int ldo) {
  __shared__ float tile[32][33];
  const int n = blockIdx.z;  // b*F + f
  const int b = n / F, f = n % F;
  const int p0 = blockIdx.x * 32, c0 = blockIdx.y * 32;
  for (int i = threadIdx.y; i < 32; i += blockDim.y) {
    const int c = c0 + i, p = p0 + threadIdx.x;
    if (c < C && p < HW) tile[i][threadIdx.x] = static_cast<float>(x[((static_cast<long long>(b) * C + c) * F + f) * HW + p]);
  }
  __syncthreads();
  for (int i = threadIdx.y; i < 32; i += blockDim.y) {
    const int p = p0 + i, c = c0 + threadIdx.x;
    if (c < C && p < HW) out[(static_cast<long long>(n) * HW + p) * ldo + c] = __float2half_rn(tile[threadIdx.x][i]);
  }
}

// (B*F, HW, ldx) fp16 (first C columns) -> (B, C, F, H, W) fp16
__global__ void nhwc_to_ncfhw_kernel(const __half* __restrict__ x, int ldx, __half* __restrict__ out, int B, int C, int F, int HW) {
  __shared__ __half tile[32][34];
  const int n = blockIdx.z;
  const int b = n / F, f = n % F;
  const int p0 = blockIdx.x * 32, c0 = blockIdx.y * 32;
  for (int i = threadIdx.y; i < 32; i += blockDim.y) {
    const int p = p0 + i, c = c0 + threadIdx.x;
    if (c < C && p < HW) tile[i][threadIdx.x] = x[(static_cast<long long>(n) * HW + p) * ldx + c];
  }
  __syncthreads();
  for (int i = threadIdx.y; i < 32; i += blockDim.y) {
    const int c = c0 + i, p = p0 + threadIdx.x;
    if (c < C && p < HW) out[((static_cast<long long>(b) * C + c) * F + f) * HW + p] = tile[threadIdx.x][i];
  }
}

// PixelUnshuffle(r) of (B, C, F, H, W) fp16 -> channels-last (B*F, H/r, W/r, C*r*r), channel = c*r*r + dy*r + dx
__global__ void pixel_unshuffle_kernel(const __half* __restrict__ x, __half* __restrict__ out, long long total, int B, int C, int F,
                                       int H, int W, int r) {
  const int Ho = H / r, Wo = W / r, Co = C * r * r;
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int co = static_cast<int>(i % Co);
    long long t = i / Co;
    const int xo = static_cast<int>(t % Wo);
    t /= Wo;
    const int yo = static_cast<int>(t % Ho);
    const long long n = t / Ho;
    const int b = static_cast<int>(n / F), f = static_cast<int>(n % F);
    const int c = co / (r * r), dy = (co / r) % r, dx = co % r;
    out[i] = x[(((static_cast<long long>(b) * C + c) * F + f) * H + (yo * r + dy)) * W + (xo * r + dx)];
  }
}

// Plucker-embedding producer (ray_condition, src/dataset/dance_image_h_v_camera.py:88-130) fused with PixelUnshuffle(r): writes the
// channels-last (B*F, H/r, W/r, 6*r*r) tensor encoder_conv_in reads, straight from the per-frame intrinsics K = (fx, fy, cx, cy) in
// pixels and camera-to-world matrices (row-major 4x4) -- the (B, 6, F, H, W) embedding (127 MB in fp16 at 24x768x576) is never built.
//   d = normalize((x + .5 - cx) / fx, (y + .5 - cy) / fy, 1);  rays_d = R d;  rays_o = t;  plucker = [rays_o x rays_d, rays_d]
// fp32 math like the reference (which runs it on the CPU), one rounding to fp16 (the pipeline's `.to(dtype=fp16)`).
__global__ void plucker_unshuffle_kernel(const float* __restrict__ K, const float* __restrict__ c2w, __half* __restrict__ out, long long total,
                                         int H, int W, int r) {
  const int Ho = H / r, Wo = W / r, rr = r * r;
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < total; i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int sub = static_cast<int>(i % rr);           // dy * r + dx: consecutive threads fill consecutive channels of one source plane
    long long t = i / rr;
    const int xo = static_cast<int>(t % Wo);
    t /= Wo;
    const int yo = static_cast<int>(t % Ho);
    const long long n = t / Ho;                          // b * F + f
    const int y = yo * r + sub / r, x = xo * r + sub % r;
    const float* k = K + n * 4;
    const float* m = c2w + n * 16;
    float dx = (static_cast<float>(x) + 0.5f - k[2]) / k[0];
    float dy = (static_cast<float>(y) + 0.5f - k[3]) / k[1];
    float dz = 1.0f;
    const float nrm = sqrtf(dx * dx + dy * dy + dz * dz);
    dx /= nrm; dy /= nrm; dz /= nrm;
    const float rx = dx * m[0] + dy * m[1] + dz * m[2];
    const float ry = dx * m[4] + dy * m[5] + dz * m[6];
    const float rz = dx * m[8] + dy * m[9] + dz * m[10];
    const float ox = m[3], oy = m[7], oz = m[11];
    const float v[6] = {oy * rz - oz * ry, oz * rx - ox * rz, ox * ry - oy * rx, rx, ry, rz};
    __half* dst = out + ((n * Ho + yo) * Wo + xo) * (6LL * rr) + sub;
#pragma unroll
    for (int c = 0; c < 6; ++c) dst[c * rr] = __float2half_rn(v[c]);
  }
}

// y[m][n] = fp16( sum_k act(x[m][k]) * w[n][k] + bias[n] ); one warp per output element (M is tiny).
__global__ void small_linear_kernel(const __half* __restrict__ x, const __half* __restrict__ w, const __half* __restrict__ bias,
                                    __half* __restrict__ out, int M, int N, int K, int act_in) {
  const long long wid = (blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (wid >= static_cast<long long>(M) * N) return;
  const int m = static_cast<int>(wid / N), n = static_cast<int>(wid % N);
  float acc = 0.f;
  for (int k = lane * 2; k < K; k += 64) {
    float2 xv = __half22float2(*reinterpret_cast<const __half2*>(x + static_cast<long long>(m) * K + k));
    float2 wv = __half22float2(*reinterpret_cast<const __half2*>(w + static_cast<long long>(n) * K + k));
    if (act_in == 2) {
      xv.x = silu_f(xv.x);
      xv.y = silu_f(xv.y);
    }
    acc += xv.x * wv.x + xv.y * wv.y;
  }
#pragma unroll
  for (int o = 16; o; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
  if (lane == 0) out[static_cast<long long>(m) * N + n] = __float2half_rn(acc + (bias ? __half2float(bias[n]) : 0.f));
}

__global__ void timestep_embedding_kernel(float t, const long long* __restrict__ table, const int* __restrict__ index,
                                          __half* __restrict__ out, int B, int dim) {
  if (table != nullptr) t = static_cast<float>(table[*index]);   // device-resident timestep (graph replay of a denoising loop)
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  const int half = dim / 2;
  if (i >= B * half) return;
  const int b = i / half, j = i % half;
  const float freq = expf(-logf(10000.0f) * static_cast<float>(j) / static_cast<float>(half));
  const float arg = t * freq;
  out[b * dim + j] = __float2half_rn(cosf(arg));
  out[b * dim + half + j] = __float2half_rn(sinf(arg));
}

// Direct 3x3 conv for small channel counts: one thread per (pixel, 8 output channels).  X (NF,H,W,Cin) channels-last,
// W (Cout, Cin, 3, 3).  fp32 accumulate; optional add (same shape as out) applied after bias (+act).
__global__ void conv3x3_direct_kernel(const __half* __restrict__ x, const __half* __restrict__ w, const __half* __restrict__ bias,
                                      __half* __restrict__ out, long long total, int H, int W, int Cin, int Cout, int stride,
                                      int act, const __half* __restrict__ add, int ldo) {
  const int Ho = (H - 1) / stride + 1, Wo = (W - 1) / stride + 1;
  const int cgroups = (Cout + 7) / 8;
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int cg = static_cast<int>(i % cgroups);
    long long t = i / cgroups;
    const int xo = static_cast<int>(t % Wo);
    t /= Wo;
    const int yo = static_cast<int>(t % Ho);
    const long long n = t / Ho;
    float acc[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) acc[j] = 0.f;
    for (int ky = 0; ky < 3; ++ky) {
      const int yi = yo * stride + ky - 1;
      if (yi < 0 || yi >= H) continue;
      for (int kx = 0; kx < 3; ++kx) {
        const int xi = xo * stride + kx - 1;
        if (xi < 0 || xi >= W) continue;
        const __half* xp = x + ((n * H + yi) * W + xi) * Cin;
        for (int c = 0; c < Cin; ++c) {
          const float xv = __half2float(__ldg(xp + c));
#pragma unroll
          for (int j = 0; j < 8; ++j) {
            const int co = cg * 8 + j;
            if (co < Cout) acc[j] += xv * __half2float(__ldg(w + ((static_cast<long long>(co) * Cin + c) * 3 + ky) * 3 + kx));
          }
        }
      }
    }
    const long long obase = ((n * Ho + yo) * Wo + xo) * ldo;
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const int co = cg * 8 + j;
      if (co < Cout) {
        float v = acc[j] + (bias ? __half2float(bias[co]) : 0.f);
        if (act == 2) v = silu_f(v);
        else if (act == 1) v = fmaxf(v, 0.f);
        if (add) v = v + __half2float(add[obase + co]);
        out[obase + co] = __float2half_rn(v);
      }
    }
  }
}

// ---------------------------------------------------------------- weight packing
template <typename T>
__global__ void pack_conv3x3_kernel(const T* __restrict__ w, __half* __restrict__ out, long long total, int Cout, int Cin, int CinPad) {
  // out[co][tap*CinPad + c] = w[co][c][tap]; zero for padded output rows / input channels
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int c = static_cast<int>(i % CinPad);
    long long t = i / CinPad;
    const int tap = static_cast<int>(t % 9);
    const long long co = t / 9;
    out[i] = (co < Cout && c < Cin) ? __float2half_rn(static_cast<float>(w[(co * Cin + c) * 9 + tap])) : __float2half_rn(0.f);
  }
}

// rows: [hidden 0..R/2) | gate R/2..R) -> blocks of 256: [128 hidden | 128 gate]
__global__ void pack_geglu_kernel(const __half* __restrict__ w, __half* __restrict__ out, long long total, int rows, int K) {
  const int half_rows = rows / 2;
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int k = static_cast<int>(i % K);
    const int prow = static_cast<int>(i / K);
    const int blk = prow / 256, within = prow % 256;
    const int src = within < 128 ? blk * 128 + within : half_rows + blk * 128 + (within - 128);
    out[i] = w[static_cast<long long>(src) * K + k];
  }
}

__global__ void pack_heads_kernel(const __half* __restrict__ w, __half* __restrict__ out, long long total, int d, int dpad, int K) {
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int k = static_cast<int>(i % K);
    const int prow = static_cast<int>(i / K);
    const int h = prow / dpad, j = prow % dpad;
    out[i] = j < d ? w[(static_cast<long long>(h) * d + j) * K + k] : __float2half_rn(0.f);
  }
}

__global__ void dbg_gemm_kernel(const __half* __restrict__ a, long long lda, const __half* __restrict__ w, float* __restrict__ out, int M,
                                int N, int K) {
  const long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x;
  if (i >= static_cast<long long>(M) * N) return;
  const int m = static_cast<int>(i / N), n = static_cast<int>(i % N);
  float acc = 0.f;
  for (int k = 0; k < K; ++k) acc += __half2float(a[m * lda + k]) * __half2float(w[static_cast<long long>(n) * K + k]);
  out[i] = acc;
}

// (Cout, Cin, 3, 3) -> [parity py*2+px][Cout][(2a+b)*Cin + c]: the 3x3 taps of a conv applied to a nearest-2x upsampled image, summed
// (fp32, one rounding) onto the 2x2 source pixels they read.  Output row 2y+py reads source rows {y-1, y, y} (py = 0) or {y, y, y+1}
// (py = 1) for dy = 0, 1, 2: a = 0 collects dy in {0} / {0, 1}, a = 1 collects {1, 2} / {2}; columns alike.
__global__ void pack_upconv2x2_kernel(const __half* __restrict__ w, __half* __restrict__ out, long long total, int Cout, int Cin) {
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < total; i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int c = static_cast<int>(i % Cin);
    long long t = i / Cin;
    const int tap = static_cast<int>(t % 4);
    t /= 4;
    const int co = static_cast<int>(t % Cout);
    const int par = static_cast<int>(t / Cout);
    const int py = par >> 1, px = par & 1, a = tap >> 1, b = tap & 1;
    const int dy0 = py == 0 ? (a == 0 ? 0 : 1) : (a == 0 ? 0 : 2), dy1 = py == 0 ? (a == 0 ? 0 : 2) : (a == 0 ? 1 : 2);
    const int dx0 = px == 0 ? (b == 0 ? 0 : 1) : (b == 0 ? 0 : 2), dx1 = px == 0 ? (b == 0 ? 0 : 2) : (b == 0 ? 1 : 2);
    float s = 0.f;
    for (int dy = dy0; dy <= dy1; ++dy)
      for (int dx = dx0; dx <= dx1; ++dx) s += __half2float(w[((static_cast<long long>(co) * Cin + c) * 3 + dy) * 3 + dx]);
    out[i] = __float2half_rn(s);
  }
}

// Conv2d(Cin, hidden, p, stride=p) as the A operand of a GEMM: pixels (B, Cin, S, S) -> rows (b, gy, gx) of [B * g * g][Kpad], g = S / p,
// column k = c p^2 + ky p + kx = pixels[b][c][gy p + ky][gx p + kx] (the flattening of the conv weight), columns [Cin p^2, Kpad) zero.
__global__ void clip_patchify_kernel(const __half* __restrict__ x, __half* __restrict__ out, long long total, int Cin, int S, int p, int Kpad) {
  const int g = S / p, K = Cin * p * p;
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < total; i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int k = static_cast<int>(i % Kpad);
    long long r = i / Kpad;
    const int gx = static_cast<int>(r % g);
    r /= g;
    const int gy = static_cast<int>(r % g);
    const long long b = r / g;
    __half v = __float2half_rn(0.f);
    if (k < K) {
      const int c = k / (p * p), rem = k - c * p * p, ky = rem / p, kx = rem - ky * p;
      v = x[((b * Cin + c) * S + gy * p + ky) * static_cast<long long>(S) + gx * p + kx];
    }
    out[i] = v;
  }
}

// e4m3 rows with one scale each (the FP8 weights: s_w[n] = amax(row n) / 448): one warp per row, 8 values per lane and step; the
// second pass re-reads the row from L2.
__global__ void pack_fp8_rows_kernel(const __half* __restrict__ w, uint8_t* __restrict__ out, float* __restrict__ scale, int rows, int K) {
  const int lane = threadIdx.x & 31;
  const long long row = static_cast<long long>(blockIdx.x) * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (row >= rows) return;
  const __half* src = w + row * K;
  float amax = 0.f;
  for (int c = lane * 8; c < K; c += 256) {
    const uint4 u = __ldg(reinterpret_cast<const uint4*>(src + c));
    const __half2* h = reinterpret_cast<const __half2*>(&u);
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const float2 f = __half22float2(h[j]);
      amax = fmaxf(amax, fmaxf(fabsf(f.x), fabsf(f.y)));
    }
  }
#pragma unroll
  for (int o = 16; o; o >>= 1) amax = fmaxf(amax, __shfl_xor_sync(0xffffffffu, amax, o));
  const float inv = e4m3_inv(amax);
  for (int c = lane * 8; c < K; c += 256) {
    const uint4 u = __ldg(reinterpret_cast<const uint4*>(src + c));
    const __half2* h = reinterpret_cast<const __half2*>(&u);
    uint32_t q[2];
#pragma unroll
    for (int j = 0; j < 2; ++j) {
      const float2 f0 = __half22float2(h[2 * j]), f1 = __half22float2(h[2 * j + 1]);
      q[j] = e4m3x2(f0.x, f0.y, inv) | (static_cast<uint32_t>(e4m3x2(f1.x, f1.y, inv)) << 16);
    }
    *reinterpret_cast<uint2*>(out + row * K + c) = make_uint2(q[0], q[1]);
  }
  if (lane == 0) scale[row] = e4m3_scale(amax);
}

}  // namespace

// Each operator below rejects NULL pointers and sizes its kernel would narrow out of int32 (or, where a size becomes gridDim.y / .z,
// past 65535) before it launches; the message lists what the operator needs.
static int invalid(const char* op, const char* needs) {
  set_error("%s: bad arguments (%s)", op, needs);
  return HV_ERR_INVALID;
}

int op_clip_patchify(const __half* x, __half* out, int64_t B, int64_t Cin, int64_t S, int64_t p, int64_t Kpad, cudaStream_t s) {
  if (!x || !out || B <= 0 || Cin <= 0 || p <= 0 || S <= 0 || (S % p) || (Kpad % 8) || Kpad < Cin * p * p || Kpad > INT32_MAX || B * S * S * Cin > INT32_MAX) {
    set_error("hv_op_clip_patchify: bad shape B=%lld C=%lld S=%lld p=%lld Kpad=%lld (S %% p == 0, Kpad >= C p^2 and a multiple of 8)", (long long)B,
              (long long)Cin, (long long)S, (long long)p, (long long)Kpad);
    return HV_ERR_INVALID;
  }
  const int sms = device_sms();
  if (!sms) return HV_ERR_CUDA;
  const long long total = B * (S / p) * (S / p) * Kpad;
  clip_patchify_kernel<<<blocks_for(total, sms), kThreads, 0, s>>>(x, out, total, static_cast<int>(Cin), static_cast<int>(S), static_cast<int>(p),
                                                                     static_cast<int>(Kpad));
  return cuda_status(cudaGetLastError(), "hv_op_clip_patchify");
}

// the tiled transposes: (C + 31) / 32 tiles and B * F frames are the grid's y and z dimensions
static bool transpose_ok(int64_t B, int64_t C, int64_t F, int64_t H, int64_t W) {
  return B >= 1 && F >= 1 && B * F <= 65535 && C >= 1 && (C + 31) / 32 <= 65535 && H >= 1 && W >= 1 && H * W <= INT32_MAX;
}

int op_ncfhw_to_nhwc(const void* x, __half* out, int64_t B, int64_t C, int64_t F, int64_t H, int64_t W, int src_fp32, cudaStream_t s, int64_t ldo) {
  if (ldo <= 0) ldo = C;
  if (!x || !out || !transpose_ok(B, C, F, H, W) || ldo < C || ldo > INT32_MAX)
    return invalid("hv_op_ncfhw_to_nhwc", "non-NULL pointers, B, C, F, H, W >= 1, B*F <= 65535, H*W and ldo >= C within int32");
  const int HW = static_cast<int>(H * W);
  dim3 grid((HW + 31) / 32, static_cast<unsigned>((C + 31) / 32), static_cast<unsigned>(B * F)), block(32, 8);
  if (src_fp32)
    ncfhw_to_nhwc_kernel<float><<<grid, block, 0, s>>>(static_cast<const float*>(x), out, static_cast<int>(B), static_cast<int>(C), static_cast<int>(F), HW,
                                                       static_cast<int>(ldo));
  else
    ncfhw_to_nhwc_kernel<__half><<<grid, block, 0, s>>>(static_cast<const __half*>(x), out, static_cast<int>(B), static_cast<int>(C), static_cast<int>(F), HW,
                                                        static_cast<int>(ldo));
  return cuda_status(cudaGetLastError(), "hv_op_ncfhw_to_nhwc");
}
int op_nhwc_to_ncfhw(const __half* x, int64_t ldx, __half* out, int64_t B, int64_t C, int64_t F, int64_t H, int64_t W, cudaStream_t s) {
  if (!x || !out || !transpose_ok(B, C, F, H, W) || ldx < C || ldx > INT32_MAX)
    return invalid("hv_op_nhwc_to_ncfhw", "non-NULL pointers, B, C, F, H, W >= 1, B*F <= 65535, H*W and ldx >= C within int32");
  const int HW = static_cast<int>(H * W);
  dim3 grid((HW + 31) / 32, static_cast<unsigned>((C + 31) / 32), static_cast<unsigned>(B * F)), block(32, 8);
  nhwc_to_ncfhw_kernel<<<grid, block, 0, s>>>(x, static_cast<int>(ldx), out, static_cast<int>(B), static_cast<int>(C), static_cast<int>(F), HW);
  return cuda_status(cudaGetLastError(), "hv_op_nhwc_to_ncfhw");
}
int op_pixel_unshuffle(const __half* x, __half* out, int64_t B, int64_t C, int64_t F, int64_t H, int64_t W, int r, cudaStream_t s) {
  if (!x || !out || !int32_ok(B) || !int32_ok(F) || !int32_ok(B * F) || !int32_ok(H) || !int32_ok(W) || r < 1 || (H % r) || (W % r) ||
      !int32_ok(C * r * r))
    return invalid("hv_op_pixel_unshuffle", "non-NULL pointers, r >= 1 dividing H and W, B, C, F, H, W >= 1, B*F and C*r*r within int32");
  const int sms = device_sms();
  if (!sms) return HV_ERR_CUDA;
  const long long total = B * F * C * H * W;
  pixel_unshuffle_kernel<<<blocks_for(total, sms), kThreads, 0, s>>>(x, out, total, static_cast<int>(B), static_cast<int>(C), static_cast<int>(F),
                                                                      static_cast<int>(H), static_cast<int>(W), r);
  return cuda_status(cudaGetLastError(), "hv_op_pixel_unshuffle");
}
int op_plucker_unshuffle(const float* K, const float* c2w, __half* out, int64_t NF, int64_t H, int64_t W, int r, cudaStream_t s) {
  if (!K || !c2w || !out || NF <= 0 || r < 1 || (H % r) || (W % r) || H > INT32_MAX || W > INT32_MAX)
    return invalid("hv_op_plucker_unshuffle", "non-NULL pointers, NF >= 1, r >= 1 dividing H and W, H and W within int32");
  const int sms = device_sms();
  if (!sms) return HV_ERR_CUDA;
  const long long total = NF * H * W;
  plucker_unshuffle_kernel<<<blocks_for(total, sms), kThreads, 0, s>>>(K, c2w, out, total, static_cast<int>(H), static_cast<int>(W), r);
  return cuda_status(cudaGetLastError(), "hv_op_plucker_unshuffle");
}
// one warp per output element, x and w read as half2
int op_small_linear(const __half* x, const __half* w, const __half* bias, __half* out, int64_t M, int64_t N, int64_t K, int act_in, cudaStream_t s) {
  if (!x || !w || !out || (reinterpret_cast<uintptr_t>(x) & 3) || (reinterpret_cast<uintptr_t>(w) & 3) || !int32_ok(M) || !int32_ok(N) || !int32_ok(K) ||
      (K % 2) || (M * N + 7) / 8 > INT32_MAX)
    return invalid("hv_op_small_linear", "non-NULL, 4-byte aligned X and W, M, N >= 1, K >= 2 and even, M*N/8 blocks within int32");
  const long long warps = M * N;
  small_linear_kernel<<<static_cast<unsigned>((warps * 32 + kThreads - 1) / kThreads), kThreads, 0, s>>>(x, w, bias, out, static_cast<int>(M),
                                                                                                         static_cast<int>(N), static_cast<int>(K), act_in);
  return cuda_status(cudaGetLastError(), "hv_op_small_linear");
}
int op_timestep_embedding(int64_t timestep, const long long* table, const int* index, __half* out, int64_t B, int64_t dim, cudaStream_t s) {
  if (!out || (table && !index) || B < 1 || dim < 2 || (dim % 2) || B * dim > INT32_MAX)
    return invalid("hv_op_timestep_embedding", "non-NULL out, B >= 1, dim >= 2 and even, B*dim within int32");
  const int n = static_cast<int>(B * dim / 2);
  timestep_embedding_kernel<<<(n + 127) / 128, 128, 0, s>>>(static_cast<float>(timestep), table, index, out, static_cast<int>(B), static_cast<int>(dim));
  return cuda_status(cudaGetLastError(), "hv_op_timestep_embedding");
}
int op_conv3x3_direct(const __half* x, const __half* w, const __half* bias, __half* out, int64_t NF, int64_t H, int64_t W, int64_t Cin, int64_t Cout,
                      int stride, int act, const __half* add, int64_t ldo, cudaStream_t s) {
  if (!x || !w || !out || NF < 1 || !int32_ok(H) || !int32_ok(W) || !int32_ok(Cin) || !int32_ok(Cout) || (stride != 1 && stride != 2) || ldo < Cout ||
      ldo > INT32_MAX)
    return invalid("hv_op_conv3x3_direct", "non-NULL X, W and out, stride 1 or 2, NF, H, W, Cin, Cout >= 1 within int32, Cout <= ldo within int32");
  const int sms = device_sms();
  if (!sms) return HV_ERR_CUDA;
  const int Hi = static_cast<int>(H), Wi = static_cast<int>(W), Ho = (Hi - 1) / stride + 1, Wo = (Wi - 1) / stride + 1;
  const long long total = NF * Ho * Wo * ((Cout + 7) / 8);
  conv3x3_direct_kernel<<<blocks_for(total, sms), kThreads, 0, s>>>(x, w, bias, out, total, Hi, Wi, static_cast<int>(Cin), static_cast<int>(Cout), stride,
                                                                     act, add, static_cast<int>(ldo));
  return cuda_status(cudaGetLastError(), "hv_op_conv3x3_direct");
}
int op_pack_conv3x3(const __half* w, __half* out, int64_t Cout, int64_t Cin, int64_t Cout_pad, int64_t Cin_pad, cudaStream_t s) {
  if (!w || !out || !int32_ok(Cout) || !int32_ok(Cin) || Cout_pad < Cout || Cin_pad < Cin || Cout_pad > INT32_MAX || Cin_pad > INT32_MAX)
    return invalid("hv_pack_conv3x3", "non-NULL pointers, 1 <= Cout <= Cout_pad and 1 <= Cin <= Cin_pad within int32");
  const int sms = device_sms();
  if (!sms) return HV_ERR_CUDA;
  const long long total = Cout_pad * 9 * Cin_pad;
  pack_conv3x3_kernel<__half><<<blocks_for(total, sms), kThreads, 0, s>>>(w, out, total, static_cast<int>(Cout), static_cast<int>(Cin),
                                                                           static_cast<int>(Cin_pad));
  return cuda_status(cudaGetLastError(), "hv_pack_conv3x3");
}
int op_pack_upconv2x2(const __half* w, __half* out, int64_t Cout, int64_t Cin, cudaStream_t s) {
  if (!w || !out || !int32_ok(Cout) || !int32_ok(Cin)) return invalid("hv_pack_upconv2x2", "non-NULL pointers, Cout and Cin >= 1 within int32");
  const int sms = device_sms();
  if (!sms) return HV_ERR_CUDA;
  const long long total = 16LL * Cout * Cin;
  pack_upconv2x2_kernel<<<blocks_for(total, sms), kThreads, 0, s>>>(w, out, total, static_cast<int>(Cout), static_cast<int>(Cin));
  return cuda_status(cudaGetLastError(), "hv_pack_upconv2x2");
}
// rows come in blocks of 256 = [128 hidden | 128 gate]
int op_pack_geglu(const __half* w, __half* out, int64_t rows, int64_t K, cudaStream_t s) {
  if (!w || !out || !int32_ok(rows) || (rows % 256) || !int32_ok(K))
    return invalid("hv_pack_geglu", "non-NULL pointers, rows a positive multiple of 256 and K >= 1 within int32");
  const int sms = device_sms();
  if (!sms) return HV_ERR_CUDA;
  const long long total = rows * K;
  pack_geglu_kernel<<<blocks_for(total, sms), kThreads, 0, s>>>(w, out, total, static_cast<int>(rows), static_cast<int>(K));
  return cuda_status(cudaGetLastError(), "hv_pack_geglu");
}
int op_pack_heads(const __half* w, __half* out, int heads, int d, int dpad, int64_t K, cudaStream_t s) {
  if (!w || !out || heads < 1 || d < 1 || dpad < d || !int32_ok(K) || static_cast<int64_t>(heads) * dpad > INT32_MAX)
    return invalid("hv_pack_heads", "non-NULL pointers, heads, d, K >= 1, dpad >= d, heads*dpad and K within int32");
  const int sms = device_sms();
  if (!sms) return HV_ERR_CUDA;
  const long long total = static_cast<long long>(heads) * dpad * K;
  pack_heads_kernel<<<blocks_for(total, sms), kThreads, 0, s>>>(w, out, total, d, dpad, static_cast<int>(K));
  return cuda_status(cudaGetLastError(), "hv_pack_heads");
}
int op_pack_fp8_rows(const __half* w, uint8_t* out, float* scale, int64_t rows, int64_t K, cudaStream_t s) {
  if (!w || !out || !scale || !aligned16(w) || !aligned16(out) || !aligned16(scale) || !int32_ok(rows) || !int32_ok(K) || (K % 16))
    return invalid("hv_pack_fp8_rows", "non-NULL, 16-byte aligned pointers, rows >= 1 and K a positive multiple of 16 within int32");
  constexpr int kWarps = 8;
  pack_fp8_rows_kernel<<<static_cast<unsigned>((rows + kWarps - 1) / kWarps), kWarps * 32, 0, s>>>(w, out, scale, static_cast<int>(rows), static_cast<int>(K));
  return cuda_status(cudaGetLastError(), "hv_pack_fp8_rows");
}
int op_dbg_gemm(const __half* a, int64_t lda, const __half* w, float* out, int64_t M, int64_t N, int64_t K, cudaStream_t s) {
  if (!a || !w || !out || !int32_ok(M) || !int32_ok(N) || !int32_ok(K) || M * N > INT32_MAX)
    return invalid("hv_dbg_gemm", "non-NULL pointers, M, N, K >= 1, M*N within int32");
  const long long total = M * N;
  dbg_gemm_kernel<<<static_cast<unsigned>((total + kThreads - 1) / kThreads), kThreads, 0, s>>>(a, lda, w, out, static_cast<int>(M), static_cast<int>(N),
                                                                                              static_cast<int>(K));
  return cuda_status(cudaGetLastError(), "hv_dbg_gemm");
}

}  // namespace hv
