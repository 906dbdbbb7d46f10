// Host-side construction of TMA tensor maps (cuTensorMapEncodeTiled resolved at run time through the CUDA
// runtime's driver-entry-point API, so the library has no link-time dependency on libcuda).
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <stdint.h>

namespace hv {

// fp16 row-major matrix [rows][ld] of which `cols` columns are valid; box = box_rows x 64 columns, 128B swizzle.
// Out-of-bounds box elements read as zero.
bool make_map_2d(CUtensorMap* m, const void* ptr, int64_t rows, int64_t cols, int64_t ld, int box_rows);

// Same with an explicit box width (<= 64 columns).
bool make_map_2d_box(CUtensorMap* m, const void* ptr, int64_t rows, int64_t cols, int64_t ld, int box_rows, int box_cols);

// e4m3 row-major matrix [rows][ld] (ld in bytes, a multiple of 16) of which `cols` columns are valid; box = box_rows x 128 columns
// (128-byte rows, the same 128B-swizzled tile as the fp16 box of 64 columns).  Out-of-bounds box elements read as zero.
bool make_map_2d_e4m3(CUtensorMap* m, const void* ptr, int64_t rows, int64_t cols, int64_t ld, int box_rows);

// channels-last activation (N, H, W, C) fp16 -> 4-D map (C, W, H, N), box (64, bw, bh, bn).
bool make_map_nhwc(CUtensorMap* m, const void* ptr, int64_t N, int64_t H, int64_t W, int64_t C, int bn, int bh, int bw);

// channels-last activation viewed as (N, H/2, 2, W/2, 2C) -> 5-D map, box (64, bw, 1, bh, bn): the operand view of a
// stride-2 3x3 convolution (H and W must be even).
bool make_map_nhwc_s2(CUtensorMap* m, const void* ptr, int64_t N, int64_t H, int64_t W, int64_t C, int bn, int bh, int bw);

// fp16 [batch][rows][ld] (cols valid) -> 3-D map (cols, rows, batch), box (64, box_rows, 1); rows beyond `rows` read as zero
// even when the next batch item follows in memory.
bool make_map_3d(CUtensorMap* m, const void* ptr, int64_t batch, int64_t rows, int64_t cols, int64_t ld, int box_rows);

// fp16 [rows][ld] matrix whose batch item n occupies columns [n * batch_stride, n * batch_stride + cols) (batch_stride % 8 == 0)
// -> 3-D map (cols, batch, rows), box (64, 1, box_rows), coordinates (col, item, row); columns beyond `cols` read as zero even
// when the next item follows (V^T with the frames side by side).
bool make_map_col_batches(CUtensorMap* m, const void* ptr, int64_t batch, int64_t rows, int64_t cols, int64_t ld, int64_t batch_stride,
                          int box_rows);

// Token matrix [frames][pixels][ld] (cols valid) viewed along the frame axis: 3-D map (cols, pixels, frames), unswizzled box
// (box_cols, 1, box_frames) = the box_frames rows of ONE pixel, box_cols channels wide (temporal attention operands).
bool make_map_frames(CUtensorMap* m, const void* ptr, int64_t frames, int64_t pixels, int64_t cols, int64_t ld, int box_cols, int box_frames);

// GEMM output / residual tiles, 32 columns per box with 64B swizzle (the staging slab of gemm_kernel's epilogue).  Only
// [0, cols) x rows is inside the map, so a store writes no element outside it and a load reads zero there.
//   2-D: [rows][ld] -> (cols, rows), box (32, 128)
//   4-D: channels-last (N, H, W, ld) -> (cols, W, H, N), box (32, bw, bh, bn)
bool make_map_tile_2d(CUtensorMap* m, const void* ptr, int64_t rows, int64_t cols, int64_t ld);
bool make_map_tile_nhwc(CUtensorMap* m, const void* ptr, int64_t N, int64_t H, int64_t W, int64_t cols, int64_t ld, int bn, int bh, int bw);

const char* tma_last_error();

}  // namespace hv
