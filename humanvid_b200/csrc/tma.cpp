#include "tma.h"

#include <cudaTypedefs.h>
#include <stdio.h>

#include <mutex>

namespace hv {

namespace {
thread_local char g_err[256] = "";
PFN_cuTensorMapEncodeTiled_v12000 g_encode = nullptr;
std::once_flag g_once;

void resolve() {
  void* fn = nullptr;
  cudaDriverEntryPointQueryResult q;
  cudaError_t e = cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &q);
  if (e == cudaSuccess && q == cudaDriverEntryPointSuccess) g_encode = reinterpret_cast<PFN_cuTensorMapEncodeTiled_v12000>(fn);
}

bool encode(CUtensorMap* m, const void* ptr, int rank, const cuuint64_t* dims, const cuuint64_t* strides_bytes,
            const cuuint32_t* box, CUtensorMapSwizzle swz = CU_TENSOR_MAP_SWIZZLE_128B,
            CUtensorMapDataType dtype = CU_TENSOR_MAP_DATA_TYPE_FLOAT16) {
  std::call_once(g_once, resolve);
  if (!g_encode) {
    snprintf(g_err, sizeof g_err, "cuTensorMapEncodeTiled entry point not available");
    return false;
  }
  cuuint32_t estr[5] = {1, 1, 1, 1, 1};
  CUresult r = g_encode(m, dtype, rank, const_cast<void*>(ptr), dims, strides_bytes, box, estr,
                        CU_TENSOR_MAP_INTERLEAVE_NONE, swz, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                        CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    snprintf(g_err, sizeof g_err, "cuTensorMapEncodeTiled failed (%d): rank %d dims %llu %llu %llu box %u %u %u ptr %p", (int)r,
             rank, (unsigned long long)dims[0], (unsigned long long)(rank > 1 ? dims[1] : 0),
             (unsigned long long)(rank > 2 ? dims[2] : 0), box[0], rank > 1 ? box[1] : 0, rank > 2 ? box[2] : 0, ptr);
    return false;
  }
  return true;
}
}  // namespace

const char* tma_last_error() { return g_err; }

bool make_map_2d_box(CUtensorMap* m, const void* ptr, int64_t rows, int64_t cols, int64_t ld, int box_rows, int box_cols) {
  cuuint64_t dims[2] = {(cuuint64_t)cols, (cuuint64_t)rows};
  cuuint64_t strides[1] = {(cuuint64_t)ld * 2};
  cuuint32_t box[2] = {(cuuint32_t)box_cols, (cuuint32_t)box_rows};
  return encode(m, ptr, 2, dims, strides, box);
}

bool make_map_2d(CUtensorMap* m, const void* ptr, int64_t rows, int64_t cols, int64_t ld, int box_rows) {
  return make_map_2d_box(m, ptr, rows, cols, ld, box_rows, 64);
}

bool make_map_2d_e4m3(CUtensorMap* m, const void* ptr, int64_t rows, int64_t cols, int64_t ld, int box_rows) {
  cuuint64_t dims[2] = {(cuuint64_t)cols, (cuuint64_t)rows};
  cuuint64_t strides[1] = {(cuuint64_t)ld};
  cuuint32_t box[2] = {128, (cuuint32_t)box_rows};
  return encode(m, ptr, 2, dims, strides, box, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_DATA_TYPE_UINT8);
}

bool make_map_3d(CUtensorMap* m, const void* ptr, int64_t batch, int64_t rows, int64_t cols, int64_t ld, int box_rows) {
  cuuint64_t dims[3] = {(cuuint64_t)cols, (cuuint64_t)rows, (cuuint64_t)batch};
  cuuint64_t strides[2] = {(cuuint64_t)ld * 2, (cuuint64_t)rows * ld * 2};
  cuuint32_t box[3] = {64, (cuuint32_t)box_rows, 1};
  return encode(m, ptr, 3, dims, strides, box);
}

bool make_map_col_batches(CUtensorMap* m, const void* ptr, int64_t batch, int64_t rows, int64_t cols, int64_t ld, int64_t batch_stride,
                          int box_rows) {
  // the batch axis is the middle one so that the strides grow outwards (batch_stride <= ld); a box of one item has the same
  // shared-memory layout as (64, box_rows)
  cuuint64_t dims[3] = {(cuuint64_t)cols, (cuuint64_t)batch, (cuuint64_t)rows};
  cuuint64_t strides[2] = {(cuuint64_t)batch_stride * 2, (cuuint64_t)ld * 2};
  cuuint32_t box[3] = {64, 1, (cuuint32_t)box_rows};
  return encode(m, ptr, 3, dims, strides, box);
}

bool make_map_frames(CUtensorMap* m, const void* ptr, int64_t frames, int64_t pixels, int64_t cols, int64_t ld, int box_cols, int box_frames) {
  cuuint64_t dims[3] = {(cuuint64_t)cols, (cuuint64_t)pixels, (cuuint64_t)frames};
  cuuint64_t strides[2] = {(cuuint64_t)ld * 2, (cuuint64_t)pixels * ld * 2};
  cuuint32_t box[3] = {(cuuint32_t)box_cols, 1, (cuuint32_t)box_frames};
  return encode(m, ptr, 3, dims, strides, box, CU_TENSOR_MAP_SWIZZLE_NONE);
}

bool make_map_nhwc(CUtensorMap* m, const void* ptr, int64_t N, int64_t H, int64_t W, int64_t C, int bn, int bh, int bw) {
  cuuint64_t dims[4] = {(cuuint64_t)C, (cuuint64_t)W, (cuuint64_t)H, (cuuint64_t)N};
  cuuint64_t strides[3] = {(cuuint64_t)C * 2, (cuuint64_t)W * C * 2, (cuuint64_t)H * W * C * 2};
  cuuint32_t box[4] = {64, (cuuint32_t)bw, (cuuint32_t)bh, (cuuint32_t)bn};
  return encode(m, ptr, 4, dims, strides, box);
}

bool make_map_nhwc_s2(CUtensorMap* m, const void* ptr, int64_t N, int64_t H, int64_t W, int64_t C, int bn, int bh, int bw) {
  if ((H & 1) || (W & 1)) {
    snprintf(g_err, sizeof g_err, "stride-2 view needs even H, W (got %lld x %lld)", (long long)H, (long long)W);
    return false;
  }
  cuuint64_t dims[5] = {(cuuint64_t)2 * C, (cuuint64_t)W / 2, 2, (cuuint64_t)H / 2, (cuuint64_t)N};
  cuuint64_t strides[4] = {(cuuint64_t)2 * C * 2, (cuuint64_t)W * C * 2, (cuuint64_t)2 * W * C * 2, (cuuint64_t)H * W * C * 2};
  cuuint32_t box[5] = {64, (cuuint32_t)bw, 1, (cuuint32_t)bh, (cuuint32_t)bn};
  return encode(m, ptr, 5, dims, strides, box);
}

bool make_map_tile_2d(CUtensorMap* m, const void* ptr, int64_t rows, int64_t cols, int64_t ld) {
  cuuint64_t dims[2] = {(cuuint64_t)cols, (cuuint64_t)rows};
  cuuint64_t strides[1] = {(cuuint64_t)ld * 2};
  cuuint32_t box[2] = {32, 128};
  return encode(m, ptr, 2, dims, strides, box, CU_TENSOR_MAP_SWIZZLE_64B);
}

bool make_map_tile_nhwc(CUtensorMap* m, const void* ptr, int64_t N, int64_t H, int64_t W, int64_t cols, int64_t ld, int bn, int bh, int bw) {
  cuuint64_t dims[4] = {(cuuint64_t)cols, (cuuint64_t)W, (cuuint64_t)H, (cuuint64_t)N};
  cuuint64_t strides[3] = {(cuuint64_t)ld * 2, (cuuint64_t)W * ld * 2, (cuuint64_t)H * W * ld * 2};
  cuuint32_t box[4] = {32, (cuuint32_t)bw, (cuuint32_t)bh, (cuuint32_t)bn};
  return encode(m, ptr, 4, dims, strides, box, CU_TENSOR_MAP_SWIZZLE_64B);
}

}  // namespace hv
