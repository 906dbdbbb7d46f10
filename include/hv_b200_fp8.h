/* hv_b200_fp8.h -- the e4m3 (FP8) operators of libhv_b200.so (sm_90a only), for the feed-forward and motion-module Q/K/V linears
 * (DESIGN.md §9).  Same conventions as hv_b200_ops.h (include it first for hv_epilogue and hv_stream_t): asynchronous on `stream`,
 * 0 or a negative hv_status, every argument checked before any CUDA call.
 *
 * Quantisation (one definition for every producer): e4m3 "fn" (max 448, no infinities), round to nearest even, saturating.  For a row
 * (or block) with absolute maximum amax: inv = 448 / amax, q = e4m3(x * inv), s = amax / 448, each an IEEE fp32 operation; amax == 0
 * gives s = 0 and zero bytes.  The value a byte q stands for is q * s.
 *
 * Alignment: every e4m3 row stride (lda, ldc of an e4m3 output, K of a packed weight) is a multiple of 16 bytes, and every pointer,
 * scale arrays included, is 16-byte aligned.
 */
#ifndef HV_B200_FP8_H
#define HV_B200_FP8_H

#include <stddef.h>
#include <stdint.h>

#include "hv_b200_ops.h"

#ifdef __cplusplus
extern "C" {
#endif

/* out[M, N] = dequant(A)[M, K] * dequant(W)[N, K]^T (+epilogue):
 *   D[m, n] = w_scale[n] * sum_kb s_a(m, kb) * sum_{k in kb} A[m, k] W[n, k]   (kb: blocks of 128 k, the last one may be partial)
 * then hv_epilogue's steps in fp32.  A: e4m3 [M][lda]; W: e4m3 [N][K] with w_scale fp32 [N] (hv_pack_fp8_rows of the packed fp16 weight).
 * A scales: a_scale_ld == 0 -> one per row, s_a(m, kb) = a_scale[m]; a_scale_ld >= ceil(K / 128) -> one per (row, k-block),
 * s_a(m, kb) = a_scale[m * a_scale_ld + kb] (the e4m3 output of a GEGLU below).
 * Output: out_scale == NULL -> fp16 out [M][ldc] as hv_op_gemm.  out_scale != NULL -> GEGLU only: out is e4m3 [M][ldc] holding the N/2
 * outputs, quantised per row and 128-column block j with scale out_scale[m * out_scale_ld + j] from the fp32 GEGLU values.
 * HV_ERR_INVALID for: A, a_scale, W, w_scale or out NULL; M, N or K outside [1, INT32_MAX]; K or lda (< K) not a multiple of 16; N % 8; a
 * pointer off 16 bytes; a_scale_ld neither 0 nor >= ceil(K / 128); geglu with N % 256 or per-block A scales; an e4m3 output without geglu,
 * with residual, rowvec, act or n_valid, with ldc < N/2 or ldc % 16, or out_scale_ld < N/256; an fp16 output with ldc % 8 or the epilogue
 * I/O hv_op_gemm rejects. */
int hv_op_gemm_fp8(const void* A, int64_t lda, const float* a_scale, int64_t a_scale_ld, const void* W, const float* w_scale, void* out,
                   int64_t ldc, float* out_scale, int64_t out_scale_ld, int64_t M, int64_t N, int64_t K, const hv_epilogue* ep, hv_stream_t stream);

/* hv_op_layernorm (pre_add / x_out / pe included) whose normalised fp32 rows are quantised to e4m3 out [rows][C] with one scale per row,
 * out_scale fp32 [rows]; no fp16 copy of the row is written.  HV_ERR_INVALID for what hv_op_layernorm rejects, out_scale NULL or off 16
 * bytes, and C not a multiple of 16. */
int hv_op_layernorm_fp8(const void* X, const void* gamma, const void* beta, void* out, float* out_scale, int64_t rows, int64_t C, float eps,
                        const void* pre_add, int64_t rows_per_group, void* x_out, const void* pe, int64_t hw, int64_t F, hv_stream_t stream);

/* fp16 [rows][K] -> e4m3 [rows][K] with one scale per row, scale fp32 [rows] (weights: after hv_pack_geglu / hv_pack_heads, so row n of the
 * e4m3 weight is row n of the packed fp16 one).  HV_ERR_INVALID for NULL or misaligned pointers, rows < 1, K < 1 or not a multiple of 16,
 * rows or K past INT32_MAX. */
int hv_pack_fp8_rows(const void* W, void* out, float* scale, int64_t rows, int64_t K, hv_stream_t stream);

#ifdef __cplusplus
}
#endif
#endif
