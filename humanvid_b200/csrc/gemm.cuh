// Host-visible parameter block + launcher of the wgmma GEMM / implicit-GEMM convolution kernel.
#pragma once
#include <cuda.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>

namespace hv {

// A_CONV3X3_S2_END: stride 2 with the padding (0, 1, 0, 1) of F.pad + conv2d(stride=2, padding=0) (AutoencoderKL's Downsample2D):
// output (yo, xo) reads input rows 2 yo .. 2 yo + 2 and columns 2 xo .. 2 xo + 2, the ones past the end reading zero.
enum AMode : int { A_LINEAR = 0, A_CONV3X3 = 1, A_CONV3X3_S2 = 2, A_UPCONV2X2 = 3, A_CONV3X3_S2_END = 4 };
enum Act : int { ACT_NONE = 0, ACT_RELU = 1, ACT_SILU = 2, ACT_QUICK_GELU = 3 };

struct GemmEpilogue {
  __half* out = nullptr;           // [rows][ldc] fp16
  int ldc = 0;
  int n_valid = 0;                 // columns actually written (<= N)
  const __half* bias = nullptr;    // [N] (packed order)
  const __half* rowvec = nullptr;  // per-row-group vector added after bias: rowvec[(row / rows_per_group) * rowvec_ld + n]
  int rowvec_ld = 0;
  int rows_per_group = 1;
  const __half* residual = nullptr;  // [rows][ldr]
  int ldr = 0;
  int act = ACT_NONE;
  int geglu = 0;                   // BLOCK_N=256 tile = [128 hidden | 128 gate] -> 128 outputs
  const __half* rowbias = nullptr; // [M]: added to every column of output row m (the "ones" rows of V^T)
  // e4m3 GEMMs only (launch_gemm_fp8): acc is dequantised first, D = w_scale[n] * (a_scale * acc), then the steps above
  const float* a_scale = nullptr;  // a_scale_ld == 0: [M], one per row; else [M][a_scale_ld], one per (row, 128-k block)
  int a_scale_ld = 0;
  const float* w_scale = nullptr;  // [N] (packed order)
  uint8_t* out8 = nullptr;         // GEGLU only: e4m3 output [rows][ldc] instead of out, one scale per 128 output columns in
  float* out8_scale = nullptr;     //   out8_scale[row * out8_scale_ld + column / 128]
  int out8_scale_ld = 0;
};

struct GemmProblem {
  int M = 0, N = 0;                // logical rows / packed columns of D
  int num_k_blocks = 0;            // ceil(K / 64)
  int stages = 0;                  // set by launch_gemm: ring depth (A + B tiles, or A tiles only in the B-stationary variant)
  int epi_slabs = 0;               // set by launch_gemm: 128 x 32 staging slabs of the TMA-store epilogue (0: register stores)
  int a_mode = A_LINEAR;
  int k_split = 0;                 // A_LINEAR: k-blocks taken from tensor map a0 (rest from a1); 0 = all from a0
  int cin_blocks = 0;              // conv: 64-channel blocks per tap
  int cin = 0;                     // conv s2: channels of the source (parity offset in the folded 2C axis)
  int H = 0, W = 0, NF = 0;        // conv: OUTPUT height / width / frame count
  int bn = 1, bh = 1, bw = 128;    // conv: tile box (bn*bh*bw == 128 rows per CTA tile)
  int tiles_n = 0, tiles_y = 0, tiles_x = 0;
  int b_par_rows = 0;              // A_UPCONV2X2: rows of the packed weight per output parity (B is [4 parities][b_par_rows][4 * Cin])
  // batched B operand (V^T = Wv * X^T per frame): B is a 3-D map (K, b_rows, b_batch); output columns of batch n
  // start at n * b_out_stride (a multiple of 8) so every frame's token segment is 16-byte aligned for TMA readers.
  int b_batch = 0, b_rows = 0, b_out_stride = 0;
};

// How launch_gemm runs a problem.  bst_stages > 0: the B-stationary variant (each CTA keeps its BLOCK_N x K weight panel in shared
// memory and streams A through a ring of bst_stages tiles; grid is a multiple of the N tiles).  bst_stages == 0: the ring variant
// (A and B tiles stream together, `stages` deep), one persistent CTA per SM, grid = min(tiles, SMs).
// epi_slabs > 0: the tile leaves through that many 128-row x 32-column shared-memory slabs and TMA stores (the whole tile when
// they cover it, else in rounds); 0: register stores.
struct GemmPlan {
  int bst_stages = 0;
  int stages = 0;
  int epi_slabs = 0;
  int grid = 0;
};
// The plan launch_gemm follows for (p, block_n); false for a block_n or an empty problem it rejects.
bool plan_gemm(const GemmProblem& p, int block_n, int num_sms, GemmPlan* plan);

// C[M, N] = A[M, K] * B[N, K]^T  (fp16 in, fp32 accumulate in registers, fused epilogue, fp16 out), CTA tile 128 x block_n.
// a0/a1: TMA maps of the A operand with 128-row boxes (see make_* helpers in tma.h), b: TMA map of the packed weights [N][K].
// out / res: make_map_tile_* maps of e.out (ldc) and e.residual (ldr) over the written region [0, n_valid) x rows (linear: 2-D,
// 3x3 conv: 4-D over the output grid); unused by the up-convolution and batched-B paths, and res unused without a residual.
// block_n must be 128, 160 or 256 (256 required for geglu); 160 = two exact tiles for the 320-wide layers.  plan: plan_gemm(p, block_n).
cudaError_t launch_gemm(const CUtensorMap& a0, const CUtensorMap& a1, const CUtensorMap& b, const CUtensorMap& out, const CUtensorMap& res,
                        const GemmProblem& p, const GemmEpilogue& e, int block_n, const GemmPlan& plan, cudaStream_t stream);
// The same kernel on e4m3 operands (A_LINEAR only): a k-block is 128 e4m3 values (p.num_k_blocks = ceil(K / 128)), the maps are
// make_map_2d_e4m3 maps, and e.a_scale / e.w_scale dequantise the fp32 accumulators.  Per-(row, 128-k block) A scales
// (e.a_scale_ld > 0) need block_n 128 or 160: each k-block's products land in a second accumulator set and are added into the main
// one scaled by a_scale.
cudaError_t launch_gemm_fp8(const CUtensorMap& a, const CUtensorMap& b, const CUtensorMap& out, const CUtensorMap& res, const GemmProblem& p,
                            const GemmEpilogue& e, int block_n, const GemmPlan& plan, cudaStream_t stream);

// Picks the (bn, bh, bw) output-tile box of 128 output pixels with the least padding for an NF x H x W output
// (every box dimension is a power of two <= 128).
void choose_conv_box(int NF, int H, int W, int* bn, int* bh, int* bw);

}  // namespace hv
