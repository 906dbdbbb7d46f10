// C++-level operator layer: argument checking + TMA map construction + kernel launch.  Used by both the operator
// C ABI and the model runtime.  Every function returns an hv_status (include/hv_b200_ops.h) and records a message.
#pragma once
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/hv_b200_ops.h"

namespace hv {

int device_sms();
void set_error(const char* fmt, ...);
const char* last_error();
int cuda_fail(cudaError_t e, const char* what);

// The tile width and launch plan op_gemm would use for out[M, N] = A[M, K] W[N, K]^T (bst_stages 0: ring variant).
int plan_linear(int64_t M, int64_t N, int64_t K, bool geglu, int* block_n, int* bst_stages, int* grid);
int op_gemm(const __half* A, int64_t lda, const __half* A2, int64_t lda2, int64_t K1, const __half* W, __half* out, int64_t ldc,
            int64_t M, int64_t N, int64_t K, const hv_epilogue* ep, cudaStream_t stream);
// out[M][n*out_stride + j] = sum_k A[M][k] * X[n][j][k] for n < batch, j < rows (X: [batch][rows][ldx]); out_stride % 8 == 0.
int op_gemm_batched_b(const __half* A, int64_t lda, const __half* X, int64_t ldx, __half* out, int64_t ldc, int64_t M, int64_t batch,
                      int64_t rows, int64_t out_stride, int64_t K, const __half* rowbias, cudaStream_t stream);
// pad_end (stride 2 only): padding (0, 1, 0, 1) instead of 1 on every side -- F.pad(x, (0, 1, 0, 1)) then a stride-2 conv with padding 0.
int op_conv3x3(const __half* X, const __half* Wp, __half* out, int64_t ldc, int64_t NF, int64_t H, int64_t W, int64_t Cin,
               int64_t Cout, int stride, const hv_epilogue* ep, cudaStream_t stream, bool pad_end = false);

// out (NF, 2H, 2W, Cout) = conv3x3(nearest_upsample_2x(X (NF, H, W, Cin))) + bias; Wp from launch_pack_upconv2x2: [4][Cout][4 * Cin].
int op_upconv2x2(const __half* X, const __half* Wp, __half* out, int64_t ldc, int64_t NF, int64_t H, int64_t W, int64_t Cin, int64_t Cout,
                 const hv_epilogue* ep, cudaStream_t stream);

}  // namespace hv
