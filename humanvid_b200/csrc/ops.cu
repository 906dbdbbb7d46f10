#include "ops.h"

#include <stdarg.h>

#include <stdio.h>
#include <stdlib.h>

#include "gemm.cuh"
#include "tma.h"

namespace hv {

namespace {
thread_local char g_msg[512] = "";
int g_sms = 0;
}  // namespace

void set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_msg, sizeof g_msg, fmt, ap);
  va_end(ap);
}
const char* last_error() { return g_msg; }
int cuda_status(cudaError_t e, const char* what) {
  if (e == cudaSuccess) return HV_OK;
  set_error("%s: %s", what, cudaGetErrorString(e));
  return HV_ERR_CUDA;
}

int device_sms() {
  if (g_sms == 0) {
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess) return 0;
    cudaDeviceProp prop;
    if (cudaGetDeviceProperties(&prop, dev) != cudaSuccess) return 0;
    if (prop.major != 9 || prop.minor != 0) {
      set_error("libhv_b200 needs an sm_90 device (found sm_%d%d)", prop.major, prop.minor);
      return 0;
    }
    g_sms = prop.multiProcessorCount;
  }
  return g_sms;
}

static void fill_epilogue(GemmEpilogue& e, const hv_epilogue* ep, __half* out, int64_t ldc, int64_t N) {
  e.out = out;
  e.ldc = static_cast<int>(ldc);
  e.n_valid = static_cast<int>(N);
  if (ep) {
    e.bias = static_cast<const __half*>(ep->bias);
    e.rowvec = static_cast<const __half*>(ep->rowvec);
    e.rowvec_ld = ep->rowvec_ld;
    e.rows_per_group = ep->rows_per_group > 0 ? ep->rows_per_group : 1;
    e.residual = static_cast<const __half*>(ep->residual);
    e.ldr = ep->ldr;
    e.act = ep->act;
    e.geglu = ep->geglu;
    if (ep->geglu) e.n_valid = static_cast<int>(N / 2);
    if (ep->n_valid > 0) e.n_valid = ep->n_valid;
  }
}

// The epilogue's TMA stores and residual loads need 16-byte aligned rows: out and residual on 16-byte boundaries, ldr % 8 == 0
// (ldc is checked with the shape).
static int check_epilogue_io(const char* op, const void* out, const hv_epilogue* ep) {
  if (reinterpret_cast<uintptr_t>(out) % 16) {
    set_error("%s: out %p is not 16-byte aligned", op, out);
    return HV_ERR_INVALID;
  }
  if (ep && ep->residual) {
    if (reinterpret_cast<uintptr_t>(ep->residual) % 16 || ep->ldr <= 0 || ep->ldr % 8) {
      set_error("%s: residual %p with ldr=%d: needs a 16-byte aligned pointer and ldr a positive multiple of 8", op, ep->residual,
                (int)ep->ldr);
      return HV_ERR_INVALID;
    }
  }
  return HV_OK;
}

// Output and residual maps of the staged epilogue: [M][n_valid] (linear) or the conv output grid (NF, H, W) x n_valid.
static int make_epilogue_maps(const char* op, const GemmProblem& p, const GemmEpilogue& e, CUtensorMap* mo, CUtensorMap* mr) {
  const bool lin = p.a_mode == A_LINEAR;
  bool ok = lin ? make_map_tile_2d(mo, e.out, p.M, e.n_valid, e.ldc) : make_map_tile_nhwc(mo, e.out, p.NF, p.H, p.W, e.n_valid, e.ldc, p.bn, p.bh, p.bw);
  if (ok && e.residual)
    ok = lin ? make_map_tile_2d(mr, e.residual, p.M, e.n_valid, e.ldr) : make_map_tile_nhwc(mr, e.residual, p.NF, p.H, p.W, e.n_valid, e.ldr, p.bn, p.bh, p.bw);
  else
    *mr = *mo;
  if (!ok) {
    set_error("%s epilogue map: %s", op, tma_last_error());
    return HV_ERR_TMA;
  }
  return HV_OK;
}

// Tile width: the candidate that pads N the least (N=320 -> 2 x 160, 640 -> 4 x 160, 384 -> 3 x 128, 1280 -> 5 x 256);
// ties go to the wider tile (fewer A re-reads per output) unless that leaves SMs idle.
static int pick_block_n(int64_t N, int64_t m_tiles, bool geglu, int sms) {
  if (geglu) return 256;
  const int cand[3] = {256, 160, 128};
  int best = 128;
  int64_t best_pad = -1;
  for (int bn : cand) {
    const int64_t padded = (N + bn - 1) / bn * bn;
    if (best_pad < 0 || padded < best_pad) { best_pad = padded; best = bn; }
  }
  if (best != 128 && m_tiles * ((N + best - 1) / best) < sms && m_tiles * ((N + 127) / 128) > m_tiles * ((N + best - 1) / best)) best = 128;
  return best;
}

// Problem block and tile width of the linear out[M, N] = A[M, K] W[N, K]^T over k-blocks of kb elements (64 fp16, 128 e4m3): what
// op_gemm and op_gemm_fp8 launch and plan_linear reports.
static GemmProblem linear_problem(int64_t M, int64_t N, int64_t K, int kb, bool geglu, int sms, int* block_n) {
  GemmProblem p;
  p.M = static_cast<int>(M);
  p.N = static_cast<int>(N);
  p.num_k_blocks = static_cast<int>((K + kb - 1) / kb);
  p.a_mode = A_LINEAR;
  *block_n = pick_block_n(N, (M + 127) / 128, geglu, sms);
  return p;
}

int plan_linear(int64_t M, int64_t N, int64_t K, bool geglu, int* block_n, int* bst_stages, int* grid) {
  if (M <= 0 || N <= 0 || K <= 0 || M > INT32_MAX || N > INT32_MAX || K > INT32_MAX) {
    set_error("hv_dbg_gemm_plan: bad shape M=%lld N=%lld K=%lld", (long long)M, (long long)N, (long long)K);
    return HV_ERR_INVALID;
  }
  const int sms = device_sms();
  if (!sms) return HV_ERR_CUDA;
  int bn;
  const GemmProblem p = linear_problem(M, N, K, 64, geglu, sms, &bn);
  GemmPlan plan;
  if (!plan_gemm(p, bn, sms, &plan)) {
    set_error("hv_dbg_gemm_plan: no plan for M=%lld N=%lld K=%lld", (long long)M, (long long)N, (long long)K);
    return HV_ERR_INVALID;
  }
  if (block_n) *block_n = bn;
  if (bst_stages) *bst_stages = plan.bst_stages;
  if (grid) *grid = plan.grid;
  return HV_OK;
}

// The launch of a problem the caller has checked and mapped (fp8: e4m3 operands, A in a0); HV_ERR_INVALID when no plan fits it.
// An e4m3 output (e.out8) leaves through register stores only.
static int run_gemm(const char* op, bool fp8, const CUtensorMap& a0, const CUtensorMap& a1, const CUtensorMap& b, const CUtensorMap& out,
                    const CUtensorMap& res, const GemmProblem& p, const GemmEpilogue& e, int bn, int sms, cudaStream_t stream) {
  GemmPlan plan;
  if (!plan_gemm(p, bn, sms, &plan) || (e.out8 && plan.epi_slabs)) {
    set_error("%s: no launch plan for M=%d N=%d with %d-column tiles", op, p.M, p.N, bn);
    return HV_ERR_INVALID;
  }
  return cuda_status(fp8 ? launch_gemm_fp8(a0, b, out, res, p, e, bn, plan, stream) : launch_gemm(a0, a1, b, out, res, p, e, bn, plan, stream), op);
}

int op_gemm(const __half* A, int64_t lda, const __half* A2, int64_t lda2, int64_t K1, const __half* W, __half* out, int64_t ldc,
            int64_t M, int64_t N, int64_t K, const hv_epilogue* ep, cudaStream_t stream) {
  if (!A || !W || !out || M <= 0 || N <= 0 || K <= 0 || (K % 8) || (lda % 8) || (ldc % 8) || (N % 8)) {
    set_error("hv_op_gemm: bad shape M=%lld N=%lld K=%lld lda=%lld ldc=%lld", (long long)M, (long long)N, (long long)K, (long long)lda,
              (long long)ldc);
    return HV_ERR_INVALID;
  }
  const bool split = A2 != nullptr && K1 > 0;
  if (split && ((K1 % 64) || (lda2 % 8) || K1 >= K)) {
    set_error("hv_op_gemm: split K1=%lld must be a multiple of 64 and < K", (long long)K1);
    return HV_ERR_INVALID;
  }
  const bool geglu = ep && ep->geglu;
  if (geglu && (N % 256)) {
    set_error("hv_op_gemm: geglu needs N %% 256 == 0 (N=%lld)", (long long)N);
    return HV_ERR_INVALID;
  }
  if (int rc = check_epilogue_io("hv_op_gemm", out, ep)) return rc;
  const int sms = device_sms();
  if (!sms) return HV_ERR_CUDA;
  CUtensorMap ma0, ma1, mb;
  const int64_t Ka = split ? K1 : K;
  int bn;
  GemmProblem p = linear_problem(M, N, K, 64, geglu, sms, &bn);
  p.k_split = split ? static_cast<int>(K1 / 64) : 0;
  if (!make_map_2d(&ma0, A, M, Ka, lda, 128)) { set_error("hv_op_gemm A map: %s", tma_last_error()); return HV_ERR_TMA; }
  ma1 = ma0;
  if (split && !make_map_2d(&ma1, A2, M, K - K1, lda2, 128)) { set_error("hv_op_gemm A2 map: %s", tma_last_error()); return HV_ERR_TMA; }
  if (!make_map_2d(&mb, W, N, K, K, bn)) { set_error("hv_op_gemm W map: %s", tma_last_error()); return HV_ERR_TMA; }
  GemmEpilogue e;
  fill_epilogue(e, ep, out, ldc, N);
  CUtensorMap mo, mr;
  if (int rc = make_epilogue_maps("hv_op_gemm", p, e, &mo, &mr)) return rc;
  return run_gemm("hv_op_gemm", false, ma0, ma1, mb, mo, mr, p, e, bn, sms, stream);
}

// e4m3 linear: the checks, then the kernel of op_gemm with KB = 128.  Tile width: GEGLU takes 256 (unpromoted, DESIGN §9); per-128 A
// scales need a second accumulator set, so 160 or 128, whichever pads N less (ties to 160: N = 320, 640 -> 160, 1280 -> 160); per-row
// scales follow pick_block_n as fp16 does.
int op_gemm_fp8(const uint8_t* A, int64_t lda, const float* a_scale, int64_t a_scale_ld, const uint8_t* W, const float* w_scale, void* out,
                int64_t ldc, float* out_scale, int64_t out_scale_ld, int64_t M, int64_t N, int64_t K, const hv_epilogue* ep, cudaStream_t stream) {
  const char* op = "hv_op_gemm_fp8";
  if (!A || !a_scale || !W || !w_scale || !out || !int32_ok(M) || !int32_ok(N) || !int32_ok(K) || (K % 16) || (N % 8) || lda < K || (lda % 16) ||
      !aligned16(A) || !aligned16(W) || !aligned16(a_scale) || !aligned16(w_scale) || !aligned16(out_scale)) {
    set_error("%s: bad arguments M=%lld N=%lld K=%lld lda=%lld (non-NULL A, a_scale, W, w_scale and out; 16-byte aligned pointers; K and lda >= K "
              "multiples of 16, N of 8)", op, (long long)M, (long long)N, (long long)K, (long long)lda);
    return HV_ERR_INVALID;
  }
  const int64_t kblocks = (K + 127) / 128;
  if (a_scale_ld != 0 && (a_scale_ld < kblocks || a_scale_ld > INT32_MAX)) {
    set_error("%s: a_scale_ld=%lld must be 0 (one scale per row) or >= ceil(K / 128) = %lld", op, (long long)a_scale_ld, (long long)kblocks);
    return HV_ERR_INVALID;
  }
  const bool geglu = ep && ep->geglu;
  if (geglu && ((N % 256) || a_scale_ld != 0)) {
    set_error("%s: geglu needs N %% 256 == 0 (N=%lld) and one A scale per row", op, (long long)N);
    return HV_ERR_INVALID;
  }
  if (out_scale) {
    if (!geglu || ep->residual || ep->rowvec || ep->act || ep->n_valid || (ldc % 16) || ldc < N / 2 || out_scale_ld < N / 256 ||
        out_scale_ld > INT32_MAX || !aligned16(out)) {
      set_error("%s: an e4m3 output (out_scale != NULL) needs a geglu epilogue without residual, rowvec, act or n_valid, a 16-byte aligned out, "
                "ldc >= N/2 a multiple of 16 and out_scale_ld >= N/256 (ldc=%lld out_scale_ld=%lld)", op, (long long)ldc, (long long)out_scale_ld);
      return HV_ERR_INVALID;
    }
  } else {
    if (ldc % 8) {
      set_error("%s: ldc=%lld must be a multiple of 8", op, (long long)ldc);
      return HV_ERR_INVALID;
    }
    if (int rc = check_epilogue_io(op, out, ep)) return rc;
  }
  const int sms = device_sms();
  if (!sms) return HV_ERR_CUDA;
  int bn;
  const GemmProblem p = linear_problem(M, N, K, 128, geglu, sms, &bn);
  if (a_scale_ld) bn = (N + 159) / 160 * 160 <= (N + 127) / 128 * 128 ? 160 : 128;   // replaces pick_block_n's width (see above)
  CUtensorMap ma, mb;
  if (!make_map_2d_e4m3(&ma, A, M, K, lda, 128)) { set_error("%s A map: %s", op, tma_last_error()); return HV_ERR_TMA; }
  if (!make_map_2d_e4m3(&mb, W, N, K, K, bn)) { set_error("%s W map: %s", op, tma_last_error()); return HV_ERR_TMA; }
  GemmEpilogue e;
  e.a_scale = a_scale;
  e.a_scale_ld = static_cast<int>(a_scale_ld);
  e.w_scale = w_scale;
  CUtensorMap mo = mb, mr = mb;
  if (out_scale) {
    e.ldc = static_cast<int>(ldc);
    e.n_valid = static_cast<int>(N / 2);
    e.bias = static_cast<const __half*>(ep->bias);
    e.geglu = 1;
    e.out8 = static_cast<uint8_t*>(out);
    e.out8_scale = out_scale;
    e.out8_scale_ld = static_cast<int>(out_scale_ld);
  } else {
    fill_epilogue(e, ep, static_cast<__half*>(out), ldc, N);
    if (int rc = make_epilogue_maps(op, p, e, &mo, &mr)) return rc;
  }
  return run_gemm(op, true, ma, ma, mb, mo, mr, p, e, bn, sms, stream);
}

int op_gemm_batched_b(const __half* A, int64_t lda, const __half* X, int64_t ldx, __half* out, int64_t ldc, int64_t M, int64_t batch,
                      int64_t rows, int64_t out_stride, int64_t K, const __half* rowbias, cudaStream_t stream) {
  if (!A || !X || !out || M <= 0 || batch <= 0 || rows <= 0 || (K % 8) || (lda % 8) || (ldx % 8) || (ldc % 8) || (out_stride % 8) || out_stride < rows) {
    set_error("hv_op_gemm_batched_b: bad shape M=%lld batch=%lld rows=%lld stride=%lld K=%lld", (long long)M, (long long)batch, (long long)rows,
              (long long)out_stride, (long long)K);
    return HV_ERR_INVALID;
  }
  const int sms = device_sms();
  if (!sms) return HV_ERR_CUDA;
  CUtensorMap ma, mb;
  if (!make_map_2d(&ma, A, M, K, lda, 128)) { set_error("gemm_batched_b A map: %s", tma_last_error()); return HV_ERR_TMA; }
  const int64_t m_tiles = (M + 127) / 128;
  const int bn = (rows > 128 && m_tiles * batch * ((rows + 255) / 256) >= sms / 2) ? 256 : 128;
  if (!make_map_3d(&mb, X, batch, rows, K, ldx, bn)) { set_error("gemm_batched_b X map: %s", tma_last_error()); return HV_ERR_TMA; }
  GemmProblem p;
  p.M = static_cast<int>(M);
  p.N = static_cast<int>(rows);
  p.num_k_blocks = static_cast<int>((K + 63) / 64);
  p.a_mode = A_LINEAR;
  p.b_batch = static_cast<int>(batch);
  p.b_rows = static_cast<int>(rows);
  p.b_out_stride = static_cast<int>(out_stride);
  GemmEpilogue e;
  e.out = out;
  e.ldc = static_cast<int>(ldc);
  e.n_valid = static_cast<int>(rows);
  e.rowbias = rowbias;
  return run_gemm("hv_op_gemm_batched_b", false, ma, ma, mb, mb, mb, p, e, bn, sms, stream);
}

// Tiling of an implicit-GEMM convolution over the NF x H x W grid of the pixels it computes: one M tile is a box of frames x rows x columns.
static void set_conv_tiles(GemmProblem& p, int64_t NF, int64_t H, int64_t W) {
  p.NF = static_cast<int>(NF);
  p.H = static_cast<int>(H);
  p.W = static_cast<int>(W);
  choose_conv_box(p.NF, p.H, p.W, &p.bn, &p.bh, &p.bw);
  p.tiles_n = (p.NF + p.bn - 1) / p.bn;
  p.tiles_y = (p.H + p.bh - 1) / p.bh;
  p.tiles_x = (p.W + p.bw - 1) / p.bw;
  p.M = p.NF * p.H * p.W;
}

int op_conv3x3(const __half* X, const __half* Wp, __half* out, int64_t ldc, int64_t NF, int64_t H, int64_t W, int64_t Cin,
               int64_t Cout, int stride, const hv_epilogue* ep, cudaStream_t stream, bool pad_end) {
  if (!X || !Wp || !out || (Cin % 64) || (Cout % 8) || (ldc % 8) || (stride != 1 && stride != 2) || (pad_end && stride != 2) || NF <= 0 || H <= 0 ||
      W <= 0) {
    set_error("hv_op_conv3x3: bad shape NF=%lld H=%lld W=%lld Cin=%lld Cout=%lld stride=%d (or NULL pointer)", (long long)NF, (long long)H,
              (long long)W, (long long)Cin, (long long)Cout, stride);
    return HV_ERR_INVALID;
  }
  if (int rc = check_epilogue_io("hv_op_conv3x3", out, ep)) return rc;
  const int sms = device_sms();
  if (!sms) return HV_ERR_CUDA;
  const int64_t Ho = stride == 1 ? H : H / 2, Wo = stride == 1 ? W : W / 2;
  GemmProblem p;
  p.a_mode = stride == 1 ? A_CONV3X3 : (pad_end ? A_CONV3X3_S2_END : A_CONV3X3_S2);
  p.N = static_cast<int>(Cout);
  p.cin_blocks = static_cast<int>(Cin / 64);
  p.cin = static_cast<int>(Cin);
  p.num_k_blocks = 9 * p.cin_blocks;
  set_conv_tiles(p, NF, Ho, Wo);
  const int bn = pick_block_n(Cout, (static_cast<int64_t>(NF) * Ho * Wo + 127) / 128, false, sms);
  if (ep && ep->geglu && bn != 256) {   // the GEGLU epilogue pairs the [128 hidden | 128 gate] halves of a 256-column tile
    set_error("hv_op_conv3x3: a geglu epilogue needs the 256-column tile, Cout=%lld gets %d columns", (long long)Cout, bn);
    return HV_ERR_INVALID;
  }
  CUtensorMap ma, mb;
  bool ok = stride == 1 ? make_map_nhwc(&ma, X, NF, H, W, Cin, p.bn, p.bh, p.bw) : make_map_nhwc_s2(&ma, X, NF, H, W, Cin, p.bn, p.bh, p.bw);
  if (!ok) { set_error("hv_op_conv3x3 X map: %s", tma_last_error()); return HV_ERR_TMA; }
  if (!make_map_2d(&mb, Wp, Cout, 9 * Cin, 9 * Cin, bn)) { set_error("hv_op_conv3x3 W map: %s", tma_last_error()); return HV_ERR_TMA; }
  GemmEpilogue e;
  fill_epilogue(e, ep, out, ldc, Cout);
  CUtensorMap mo, mr;
  if (int rc = make_epilogue_maps("hv_op_conv3x3", p, e, &mo, &mr)) return rc;
  return run_gemm("hv_op_conv3x3", false, ma, ma, mb, mo, mr, p, e, bn, sms, stream);
}

// Nearest-2x upsample + 3x3 conv (Upsample3D, resnet.py:68-71 + :49) as four 2x2 convolutions of the SOURCE tensor, one per output
// parity: the 4x larger upsampled tensor is never written or read and the conv does 4/9 of the multiply-adds.
int op_upconv2x2(const __half* X, const __half* Wp, __half* out, int64_t ldc, int64_t NF, int64_t H, int64_t W, int64_t Cin, int64_t Cout,
                 const hv_epilogue* ep, cudaStream_t stream) {
  if (!X || !Wp || !out || (Cin % 64) || (Cout % 8) || (ldc % 8) || NF <= 0 || H <= 0 || W <= 0 || (ep && (ep->residual || ep->rowvec || ep->geglu))) {
    set_error("hv_op_upconv2x2: bad shape NF=%lld H=%lld W=%lld Cin=%lld Cout=%lld (or NULL pointer, unsupported epilogue)", (long long)NF, (long long)H,
              (long long)W, (long long)Cin, (long long)Cout);
    return HV_ERR_INVALID;
  }
  const int sms = device_sms();
  if (!sms) return HV_ERR_CUDA;
  GemmProblem p;
  p.a_mode = A_UPCONV2X2;
  p.N = static_cast<int>(Cout);
  p.cin_blocks = static_cast<int>(Cin / 64);
  p.cin = static_cast<int>(Cin);
  p.num_k_blocks = 4 * p.cin_blocks;
  set_conv_tiles(p, NF, H, W);   // tile space = SOURCE pixels; the epilogue scatters to (2y + py, 2x + px)
  p.b_par_rows = static_cast<int>(Cout);
  const int64_t rows = NF * H * W;
  const int bn = pick_block_n(Cout, (4 * rows + 127) / 128, false, sms);
  if (Cout % bn) { set_error("hv_op_upconv2x2: Cout=%lld must be a multiple of the %d-column tile", (long long)Cout, bn); return HV_ERR_INVALID; }
  CUtensorMap ma, mb;
  if (!make_map_nhwc(&ma, X, NF, H, W, Cin, p.bn, p.bh, p.bw)) { set_error("hv_op_upconv2x2 X map: %s", tma_last_error()); return HV_ERR_TMA; }
  if (!make_map_2d(&mb, Wp, 4 * Cout, 4 * Cin, 4 * Cin, bn)) { set_error("hv_op_upconv2x2 W map: %s", tma_last_error()); return HV_ERR_TMA; }
  GemmEpilogue e;
  fill_epilogue(e, ep, out, ldc, Cout);
  return run_gemm("hv_op_upconv2x2", false, ma, ma, mb, mb, mb, p, e, bn, sms, stream);
}

}  // namespace hv
