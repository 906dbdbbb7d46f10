// wgmma GEMM / implicit-GEMM 3x3 convolution for sm_90a.
//
//   D[M, N] = A[M, K] * B[N, K]^T, fp16 operands, fp32 accumulation in registers, fused epilogue, fp16 output.
//
// One persistent CTA per SM, warp-specialised, CTA tile 128 x BLOCK_N:
//   warpgroup 0     TMA producer : one thread issues cp.async.bulk.tensor loads of the A tile (128 rows x 64 k) and the
//                                  B tile (BLOCK_N rows x 64 k) into a ring of 128B-swizzled shared-memory stages; the
//                                  warpgroup gives most of its registers to the math warpgroups (setmaxnreg)
//   warpgroups 1-2  math         : each owns 64 rows of the tile, issues wgmma m64 x BLOCK_N x 16 from the ring and keeps
//                                  its 64 x BLOCK_N accumulator in registers; then bias / time-embedding row vector /
//                                  activation / GEGLU / residual in fp32, one fp16 rounding at the store
// The producer runs ahead into the next tile's k-blocks while the math warpgroups run the epilogue.
// How a tile leaves the SM: the math warpgroups write the fp16 results into 128 x 32 staging slabs in shared memory (64B
// swizzle) and a second producer thread, the epilogue DMA, stores each slab with cp.async.bulk.tensor; the residual is
// TMA-loaded into the same slabs during the tile's MMAs and overwritten in place.  plan_gemm picks which launches do this;
// the others keep register stores straight from the accumulators.
// The A operand is addressed through TMA only, so a 3x3 convolution over a channels-last (N,H,W,C) tensor is the
// same kernel: k-block kb = (tap, 64-channel block) and the tile of 128 output pixels is a (bn x bh x bw) box whose
// input window is fetched with the box shifted by the tap offset; TMA's out-of-bounds zero fill is the padding.
// Stride-2 convolutions view the same memory as (N, H/2, 2, W/2, 2*C) so each tap is again a dense box; the end-padded
// variant (pad (0, 1, 0, 1), padding 0) is the same view with every tap shifted by one input pixel.
#include <cstdlib>

#include "gemm.cuh"
#include "ptx.cuh"
#include "wgmma.cuh"

namespace hv {

namespace {

constexpr int BLOCK_M = 128;
constexpr int BLOCK_K = 64;
constexpr int A_TILE_BYTES = BLOCK_M * BLOCK_K * 2;  // 16 KB
constexpr int kMaxStages = 8;
constexpr int kMaxRingStages = 6;
constexpr int kMaxSmem = 227 * 1024;
// Epilogue staging slab: 128 tile rows x 32 output columns, 64B-swizzled (16-byte chunk c of row r at chunk c ^ ((r >> 1) & 3)),
// the box of the output / residual tensor maps.  The accumulator fragment writes of one warp hit 32 distinct banks.
constexpr int SLAB_COLS = 32;
constexpr int SLAB_BYTES = BLOCK_M * SLAB_COLS * 2;  // 8 KB
constexpr int GEMM_THREADS = 384;   // warpgroup 0 TMA, warpgroups 1-2 wgmma + epilogue
constexpr int kMathWarps = 8;       // every math warp releases a ring slot once its warpgroup's MMAs on it are complete
// 65536 registers over 384 threads: the producer keeps 40, the two math warpgroups get 232 each (128 accumulators at N = 256)
constexpr uint32_t kProducerRegs = 40, kMathRegs = 232;

// Shared memory, from the 1024-byte aligned base: [B panel (BST): num_k_blocks B tiles] [ring: stages x (A tile [+ B tile])]
// [epilogue staging: slabs x SLAB_BYTES] [barriers: full[8] empty[8] bpanel epi_ready epi_staged].
struct SmemLayout {
  int b_tile, stage;  // bytes of one B tile and of one ring stage
  int bytes;          // the dynamic allocation, with the alignment slack
};
__host__ __device__ constexpr SmemLayout smem_layout(int block_n, bool bst, int num_k_blocks, int stages, int slabs) {
  SmemLayout l{};
  l.b_tile = block_n * BLOCK_K * 2;
  l.stage = A_TILE_BYTES + (bst ? 0 : l.b_tile);
  l.bytes = (bst ? num_k_blocks * l.b_tile : 0) + stages * l.stage + slabs * SLAB_BYTES + (2 * kMaxStages + 3) * 8 + 1024;
  return l;
}

// M tiles (conv: boxes, times the four output parities of the up-convolution) and N tiles (batched B: per item) of a problem.
struct TileCounts {
  int m, n, n_per_batch;
};
__host__ __device__ __forceinline__ TileCounts tile_counts(const GemmProblem& p, int block_n) {
  TileCounts t;
  t.m = p.a_mode == A_LINEAR ? (p.M + BLOCK_M - 1) / BLOCK_M : p.tiles_n * p.tiles_y * p.tiles_x * (p.a_mode == A_UPCONV2X2 ? 4 : 1);
  t.n_per_batch = p.b_batch ? (p.b_rows + block_n - 1) / block_n : 0;
  t.n = p.b_batch ? p.b_batch * t.n_per_batch : (p.N + block_n - 1) / block_n;
  return t;
}

// First output column of tile n_blk and the number of its 32-column slabs that hold written columns (< n_valid).
template <int BLOCK_N>
__device__ __forceinline__ int2 epi_tile_cols(const GemmEpilogue& e, int n_blk) {
  const int col0 = n_blk * BLOCK_N;
  const int v = (e.n_valid - col0 + SLAB_COLS - 1) / SLAB_COLS;
  return make_int2(col0, v < 0 ? 0 : (v > BLOCK_N / SLAB_COLS ? BLOCK_N / SLAB_COLS : v));
}

struct TileCoord {
  int m0;          // linear: first row.   conv: unused
  int n0, y0, x0;  // conv: first frame / output row / output col of the box
  int py, px;      // A_UPCONV2X2: output parity of this tile (output pixel (2y + py, 2x + px) for source pixel (y, x))
};

__device__ __forceinline__ TileCoord tile_coord(const GemmProblem& p, int m_blk) {
  TileCoord t;
  t.py = t.px = 0;
  if (p.a_mode == A_LINEAR) {
    t.m0 = m_blk * BLOCK_M;
    t.n0 = t.y0 = t.x0 = 0;
  } else {
    if (p.a_mode == A_UPCONV2X2) {   // the four parities of one source box are consecutive tiles (the box stays in L2 for all four)
      t.py = (m_blk >> 1) & 1;
      t.px = m_blk & 1;
      m_blk >>= 2;
    }
    int xb = m_blk % p.tiles_x;
    int r = m_blk / p.tiles_x;
    int yb = r % p.tiles_y;
    int nb = r / p.tiles_y;
    t.m0 = 0;
    t.n0 = nb * p.bn;
    t.y0 = yb * p.bh;
    t.x0 = xb * p.bw;
  }
  return t;
}

__device__ __forceinline__ float2 ldh2(const __half* p) { return __half22float2(__ldg(reinterpret_cast<const __half2*>(p))); }

// BST ("B-stationary"): every tile a CTA visits has the same n_blk (the host makes gridDim.x a multiple of n_tiles), so
// the CTA loads its BLOCK_N x K weight panel into shared memory once and streams only A afterwards.  For the K <= 640
// linears of the two high-resolution levels this removes the per-tile re-fetch of B from L2.
// FP8: e4m3 operands (A_LINEAR only).  A k-block is then 128 values: the same 128-byte swizzled rows, ring and descriptors.
template <int BLOCK_N, bool BST, bool FP8>
__global__ void __launch_bounds__(GEMM_THREADS, 1)
gemm_kernel(const __grid_constant__ CUtensorMap map_a0, const __grid_constant__ CUtensorMap map_a1,
            const __grid_constant__ CUtensorMap map_b, const __grid_constant__ CUtensorMap map_out,
            const __grid_constant__ CUtensorMap map_res, const GemmProblem p, const GemmEpilogue e) {
  constexpr int KB = FP8 ? 2 * BLOCK_K : BLOCK_K;   // elements per k-block
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  const int nstages = p.stages;
  const int nslab = p.epi_slabs;
  // smem_layout's regions, chained pointer by pointer: offsets from the base changed the SASS of every instantiation
  constexpr SmemLayout kL = smem_layout(BLOCK_N, BST, 0, 0, 0);
  uint8_t* ring = smem + (BST ? p.num_k_blocks * kL.b_tile : 0);
  uint8_t* stg = ring + nstages * kL.stage;
  uint64_t* bar_full = reinterpret_cast<uint64_t*>(stg + nslab * SLAB_BYTES);
  uint64_t* bar_empty = bar_full + kMaxStages;
  uint64_t* bar_bpanel = bar_empty + kMaxStages;
  uint64_t* bar_epi_ready = bar_bpanel + 1;    // staging slabs free (and the residual landed in them)
  uint64_t* bar_epi_staged = bar_bpanel + 2;   // the math warps wrote their part of the slabs

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;

  const TileCounts tiles = tile_counts(p, BLOCK_N);
  const int n_tiles = tiles.n, n_per_batch = tiles.n_per_batch, num_tiles = tiles.m * tiles.n;
  const int nkb = p.num_k_blocks;

  if (threadIdx.x == 0) {
    for (int s = 0; s < nstages; ++s) {
      mbar_init(&bar_full[s], 1);
      mbar_init(&bar_empty[s], kMathWarps);
    }
    mbar_init(bar_bpanel, 1);
    mbar_init(bar_epi_ready, 1);
    mbar_init(bar_epi_staged, kMathWarps);
    fence_mbar_init();
    tma_prefetch_desc(&map_a0);
    tma_prefetch_desc(&map_a1);
    tma_prefetch_desc(&map_b);
    if (nslab) {
      tma_prefetch_desc(&map_out);
      if (e.residual != nullptr) tma_prefetch_desc(&map_res);
    }
  }
  __syncthreads();

  if (warp < 4) {
    // ------------------------------------------------------------------ TMA producer
    setmaxnreg_dec<kProducerRegs>();
    if (warp == 0 && lane == 0) {
      int stage = 0;
      uint32_t phase = 0;
      if (BST && static_cast<int>(blockIdx.x) < num_tiles) {
        mbar_arrive_expect_tx(bar_bpanel, nkb * kL.b_tile);
        for (int kb = 0; kb < nkb; ++kb)
          tma_load_2d(smem + kb * kL.b_tile, &map_b, bar_bpanel, kb * KB, (blockIdx.x % n_tiles) * BLOCK_N);
      }
      for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
        const int m_blk = tile / n_tiles, n_blk = tile % n_tiles;
        const TileCoord tc = tile_coord(p, m_blk);
        for (int kb = 0; kb < nkb; ++kb) {
          mbar_wait(&bar_empty[stage], phase ^ 1);
          uint8_t* sa = ring + stage * kL.stage;
          uint8_t* sb = sa + A_TILE_BYTES;
          mbar_arrive_expect_tx(&bar_full[stage], kL.stage);
          if (p.a_mode == A_LINEAR) {
            if (p.k_split == 0 || kb < p.k_split)
              tma_load_2d(sa, &map_a0, &bar_full[stage], kb * KB, tc.m0);
            else
              tma_load_2d(sa, &map_a1, &bar_full[stage], (kb - p.k_split) * KB, tc.m0);
          } else {
            const int tap = kb / p.cin_blocks, cb = kb - tap * p.cin_blocks;
            const int dy = tap / 3, dx = tap - dy * 3;
            if (p.a_mode == A_CONV3X3) {
              tma_load_4d(sa, &map_a0, &bar_full[stage], cb * BLOCK_K, tc.x0 + dx - 1, tc.y0 + dy - 1, tc.n0);
            } else if (p.a_mode == A_UPCONV2X2) {
              // nearest-2x upsample folded into the conv: output (2y+py, 2x+px) reads the 2x2 source pixels (y + a + py - 1, x + b + px - 1)
              // with the 3x3 taps that land on each pre-summed in the packed weight (tap = 2a + b)
              const int a = tap >> 1, b = tap & 1;
              tma_load_4d(sa, &map_a0, &bar_full[stage], cb * BLOCK_K, tc.x0 + b + tc.px - 1, tc.y0 + a + tc.py - 1, tc.n0);
            } else if (p.a_mode == A_CONV3X3_S2) {  // stride 2: memory viewed as (N, H/2, 2, W/2, 2C); input row 2*yo+dy-1, col 2*xo+dx-1
              const int ph = dy == 1 ? 0 : 1, pw = dx == 1 ? 0 : 1;
              tma_load_5d(sa, &map_a0, &bar_full[stage], pw * p.cin + cb * BLOCK_K, tc.x0 - (dx == 0 ? 1 : 0), ph,
                          tc.y0 - (dy == 0 ? 1 : 0), tc.n0);
            } else {  // stride 2, padding at the end only: input row 2*yo+dy, col 2*xo+dx (the same view, the tap origin one pixel later)
              const int ph = dy & 1, pw = dx & 1;
              tma_load_5d(sa, &map_a0, &bar_full[stage], pw * p.cin + cb * BLOCK_K, tc.x0 + (dx >> 1), ph, tc.y0 + (dy >> 1), tc.n0);
            }
          }
          if (!BST) {
            if (p.b_batch)
              tma_load_3d(sb, &map_b, &bar_full[stage], kb * KB, (n_blk % n_per_batch) * BLOCK_N, n_blk / n_per_batch);
            else
              tma_load_2d(sb, &map_b, &bar_full[stage], kb * KB, n_blk * BLOCK_N + (tc.py * 2 + tc.px) * p.b_par_rows);
          }
          if (++stage == nstages) { stage = 0; phase ^= 1; }
        }
      }
    } else if (warp == 1 && lane == 0 && nslab) {
      // epilogue DMA: per round of up to nslab slabs, free the staging (loading the residual into it), wait for the math
      // warps to fill it, store it.  The first round's residual of a tile lands while that tile's MMAs run.
      const bool res = e.residual != nullptr;
      const bool lin = p.a_mode == A_LINEAR;
      uint32_t staged_phase = 0;
      for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
        const int m_blk = tile / n_tiles, n_blk = tile % n_tiles;
        const TileCoord tc = tile_coord(p, m_blk);
        const int2 cs = epi_tile_cols<BLOCK_N>(e, n_blk);
        for (int s0 = 0; s0 < cs.y; s0 += nslab) {
          const int ns = cs.y - s0 < nslab ? cs.y - s0 : nslab;
          if (res) {
            mbar_arrive_expect_tx(bar_epi_ready, ns * SLAB_BYTES);
            for (int i = 0; i < ns; ++i) {
              const int c = cs.x + (s0 + i) * SLAB_COLS;
              if (lin)
                tma_load_2d(stg + i * SLAB_BYTES, &map_res, bar_epi_ready, c, tc.m0);
              else
                tma_load_4d(stg + i * SLAB_BYTES, &map_res, bar_epi_ready, c, tc.x0, tc.y0, tc.n0);
            }
          } else {
            mbar_arrive(bar_epi_ready);
          }
          mbar_wait(bar_epi_staged, staged_phase);
          staged_phase ^= 1;
          for (int i = 0; i < ns; ++i) {
            const int c = cs.x + (s0 + i) * SLAB_COLS;
            if (lin)
              tma_store_2d(&map_out, stg + i * SLAB_BYTES, c, tc.m0);
            else
              tma_store_4d(&map_out, stg + i * SLAB_BYTES, c, tc.x0, tc.y0, tc.n0);
          }
          tma_store_commit();
          tma_store_wait_read();   // the slabs may be refilled
        }
      }
      tma_store_wait_all();
    }
    return;
  }

  // -------------------------------------------------------------------- math warpgroups
  setmaxnreg_inc<kMathRegs>();
  const int wg = (warp >> 2) - 1;          // 0 / 1: rows [64 wg, 64 wg + 64) of the tile
  const int wq = warp & 3;                 // warp inside the warpgroup: rows 16 wq .. 16 wq + 15 of the warpgroup's 64
  const int quad = lane & 3;
  int stage = 0;
  uint32_t phase = 0;
  uint32_t ready_phase = 0;
  if (BST && static_cast<int>(blockIdx.x) < num_tiles) mbar_wait(bar_bpanel, 0);
  for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
    const int m_blk = tile / n_tiles, n_blk = tile % n_tiles;
    float acc[BLOCK_N / 2];
#pragma unroll
    for (int i = 0; i < BLOCK_N / 2; ++i) acc[i] = 0.f;
    // FP8 with per-(row, k-block) A scales: the k-block's products go to `part` and are promoted into acc scaled by
    // s_a[row, kb] once its MMAs are complete (this also keeps the FP8 MMA's own limited-precision accumulation to one k-block).
    // Two accumulator sets fit beside the epilogue at BLOCK_N <= 160 only; the host never asks for it at 256.
    // launch_gemm_fp8 refuses per-block A scales at BLOCK_N = 256, where this kernel would compute without them.
    constexpr bool kPromote = FP8 && BLOCK_N <= 160;
    [[maybe_unused]] float part[kPromote ? BLOCK_N / 2 : 1];
    [[maybe_unused]] const float* sa_row[2] = {nullptr, nullptr};
    if constexpr (kPromote) {
      if (e.a_scale_ld) {
#pragma unroll
        for (int i = 0; i < BLOCK_N / 2; ++i) part[i] = 0.f;
#pragma unroll
        for (int hh = 0; hh < 2; ++hh) {
          const int row = m_blk * BLOCK_M + wg * 64 + wq * 16 + (lane >> 2) + 8 * hh;
          sa_row[hh] = row < p.M ? e.a_scale + static_cast<long long>(row) * e.a_scale_ld : nullptr;
        }
      }
    }
    int prev_stage = -1;
    for (int kb = 0; kb < nkb; ++kb) {
      mbar_wait(&bar_full[stage], phase);
      const uint32_t sa = smem_u32(ring + stage * kL.stage);
      const uint64_t adesc = gmma_desc_k_sw128(sa + wg * (A_TILE_BYTES / 2));
      const uint64_t bdesc = gmma_desc_k_sw128(BST ? smem_u32(smem + kb * kL.b_tile) : sa + A_TILE_BYTES);
      // the unpromoted FP8 k-block repeats the fp16 one: a shared helper changed the SASS of the 256-wide FP8 instantiations
      if constexpr (FP8) {
        bool promoted = false;
        if constexpr (kPromote) {
          if (e.a_scale_ld) {
            wgmma_fence_regs(part);
            wgmma_fence();
#pragma unroll
            for (int k = 0; k < KB / 32; ++k) wgmma_ss_e4m3<BLOCK_N>(part, adesc + 2 * k, bdesc + 2 * k, k ? 1u : 0u);
            wgmma_commit();
            wgmma_wait<0>();
            wgmma_fence_regs(part);
            const float s0 = sa_row[0] ? __ldg(sa_row[0] + kb) : 0.f, s1 = sa_row[1] ? __ldg(sa_row[1] + kb) : 0.f;
#pragma unroll
            for (int i = 0; i < BLOCK_N / 2; ++i) acc[i] = fmaf((i & 2) ? s1 : s0, part[i], acc[i]);
            promoted = true;
          }
        }
        if (!promoted) {
          wgmma_fence_regs(acc);
          wgmma_fence();
#pragma unroll
          for (int k = 0; k < KB / 32; ++k) wgmma_ss_e4m3<BLOCK_N>(acc, adesc + 2 * k, bdesc + 2 * k, 1u);
          wgmma_commit();
          wgmma_wait<1>();
          wgmma_fence_regs(acc);
        }
      } else {
      wgmma_fence_regs(acc);
      wgmma_fence();
#pragma unroll
      for (int k = 0; k < BLOCK_K / 16; ++k) wgmma_ss<BLOCK_N>(acc, adesc + 2 * k, bdesc + 2 * k, 1u);
      wgmma_commit();
      wgmma_wait<1>();                     // the previous k-block's MMAs are complete: its ring slot may be refilled
      wgmma_fence_regs(acc);
      }
      if (prev_stage >= 0 && lane == 0) mbar_arrive(&bar_empty[prev_stage]);
      prev_stage = stage;
      if (++stage == nstages) { stage = 0; phase ^= 1; }
    }
    wgmma_wait<0>();
    wgmma_fence_regs(acc);
    if (lane == 0) mbar_arrive(&bar_empty[prev_stage]);

    // ---------------------------------------------------------------- epilogue (fp32 all the way, ONE rounding at the store:
    // the fp32 oracle is the parity anchor; the reference's eager fp16 path rounds after every op)
    const TileCoord tc = tile_coord(p, m_blk);
    const bool has_bias = e.bias != nullptr && p.b_batch == 0;
    if (nslab) {
      // through the staging slabs: each thread writes its fp16 pairs at the swizzled position of (row, column); the residual,
      // when there is one, was loaded there by TMA and is read from the very word the result overwrites
      const int2 cs = epi_tile_cols<BLOCK_N>(e, n_blk);
      bool ok[2];
      const __half* rv[2];
      int rt[2];
      [[maybe_unused]] float rs[2];   // FP8: the per-row A scale (1 when the k-blocks were promoted with theirs)
#pragma unroll
      for (int hh = 0; hh < 2; ++hh) {
        rt[hh] = wg * 64 + wq * 16 + (lane >> 2) + 8 * hh;
        long long row;   // the register path's mapping without up-conv parities: one shared helper changed the fp16 SASS
        if (p.a_mode == A_LINEAR) {
          row = tc.m0 + rt[hh];
          ok[hh] = row < p.M;
        } else {
          const int ix = rt[hh] % p.bw, t2 = rt[hh] / p.bw;
          const int iy = t2 % p.bh, in = t2 / p.bh;
          const int n = tc.n0 + in, y = tc.y0 + iy, x = tc.x0 + ix;
          ok[hh] = n < p.NF && y < p.H && x < p.W;
          row = (static_cast<long long>(n) * p.H + y) * p.W + x;
        }
        rv[hh] = e.rowvec != nullptr && ok[hh] ? e.rowvec + (row / e.rows_per_group) * e.rowvec_ld : nullptr;
        if constexpr (FP8) rs[hh] = e.a_scale_ld == 0 && ok[hh] ? __ldg(e.a_scale + row) : 1.f;
      }
      const bool res = e.residual != nullptr;
      const float rowbias = 0.f;
      auto round_done = [&]() {
        fence_proxy_async();
        __syncwarp();
        if (lane == 0) mbar_arrive(bar_epi_staged);
      };
      auto slab_begin = [&](int s) -> uint8_t* {
        if (s % nslab == 0) {
          if (s) round_done();
          mbar_wait(bar_epi_ready, ready_phase);
          ready_phase ^= 1;
        }
        return stg + (s % nslab) * SLAB_BYTES;
      };
#pragma unroll
      for (int s = 0; s < BLOCK_N / SLAB_COLS; ++s) {
        if (s < cs.y) {
          uint8_t* slab = slab_begin(s);
#pragma unroll
          for (int hh = 0; hh < 2; ++hh) {
            if (!ok[hh]) continue;
#pragma unroll
            for (int jj = 0; jj < SLAB_COLS / 8; ++jj) {
              const int j = s * (SLAB_COLS / 8) + jj;
              const int col = cs.x + 8 * j + 2 * quad;
              if (col < e.n_valid) {
                uint32_t* w = reinterpret_cast<uint32_t*>(slab + rt[hh] * 64 + ((jj ^ ((rt[hh] >> 1) & 3)) << 4) + 4 * quad);
                float v0 = acc[4 * j + 2 * hh] + rowbias, v1 = acc[4 * j + 2 * hh + 1] + rowbias;
                if constexpr (FP8) {
                  const float2 sw = __ldg(reinterpret_cast<const float2*>(e.w_scale + col));
                  v0 = acc[4 * j + 2 * hh] * rs[hh] * sw.x;
                  v1 = acc[4 * j + 2 * hh + 1] * rs[hh] * sw.y;
                }
                if (has_bias) {
                  const float2 b = ldh2(e.bias + col);
                  v0 += b.x;
                  v1 += b.y;
                }
                if (rv[hh] != nullptr) {
                  const float2 t = ldh2(rv[hh] + col);
                  v0 += t.x;
                  v1 += t.y;
                }
                if (e.act == ACT_RELU) {
                  v0 = fmaxf(v0, 0.f);
                  v1 = fmaxf(v1, 0.f);
                } else if (e.act == ACT_SILU) {
                  v0 = silu_f(v0);
                  v1 = silu_f(v1);
                } else if (e.act == ACT_QUICK_GELU) {
                  v0 = quick_gelu_f(v0);
                  v1 = quick_gelu_f(v1);
                }
                if (res) add_h2(v0, v1, *w);
                *w = pack_h2(v0, v1);
              }
            }
          }
        }
      }
      if (cs.y > 0) round_done();
      continue;
    }
#pragma unroll
    for (int hh = 0; hh < 2; ++hh) {
      const int rt = wg * 64 + wq * 16 + (lane >> 2) + 8 * hh;   // row inside the CTA tile
      long long row;
      bool row_ok;
      if (p.a_mode == A_LINEAR) {
        row = tc.m0 + rt;
        row_ok = row < p.M;
      } else {
        const int ix = rt % p.bw, t2 = rt / p.bw;
        const int iy = t2 % p.bh, in = t2 / p.bh;
        const int n = tc.n0 + in, y = tc.y0 + iy, x = tc.x0 + ix;
        row_ok = n < p.NF && y < p.H && x < p.W;
        row = p.a_mode == A_UPCONV2X2 ? (static_cast<long long>(n) * 2 * p.H + 2 * y + tc.py) * (2 * p.W) + 2 * x + tc.px
                                      : (static_cast<long long>(n) * p.H + y) * p.W + x;
      }
      if (!row_ok) continue;
      const __half* __restrict__ rv = e.rowvec != nullptr ? e.rowvec + (row / e.rows_per_group) * e.rowvec_ld : nullptr;
      const __half* __restrict__ res = e.residual != nullptr ? e.residual + row * e.ldr : nullptr;
      const float rowbias = e.rowbias != nullptr ? __half2float(e.rowbias[row]) : 0.f;
      __half* __restrict__ out = e.out + row * e.ldc;
      [[maybe_unused]] float rs = 1.f;
      if constexpr (FP8) rs = e.a_scale_ld == 0 ? __ldg(e.a_scale + row) : 1.f;
      if (!e.geglu) {
        const int tile_col0 = p.b_batch ? (n_blk / n_per_batch) * p.b_out_stride + (n_blk % n_per_batch) * BLOCK_N : n_blk * BLOCK_N;
        const int col_lim = p.b_batch ? (n_blk / n_per_batch) * p.b_out_stride + ((p.b_rows + 7) & ~7) : e.n_valid;
#pragma unroll
        for (int j = 0; j < BLOCK_N / 8; ++j) {
          const int col = tile_col0 + 8 * j + 2 * quad;
          if (col < col_lim) {
            // the staged path's chain again: as one inlined helper it made every fp16 instantiation ~25 % longer
            float v0 = acc[4 * j + 2 * hh] + rowbias, v1 = acc[4 * j + 2 * hh + 1] + rowbias;
            if constexpr (FP8) {
              const float2 sw = __ldg(reinterpret_cast<const float2*>(e.w_scale + col));
              v0 = acc[4 * j + 2 * hh] * rs * sw.x;
              v1 = acc[4 * j + 2 * hh + 1] * rs * sw.y;
            }
            if (has_bias) {
              const float2 b = ldh2(e.bias + col);
              v0 += b.x;
              v1 += b.y;
            }
            if (rv != nullptr) {
              const float2 t = ldh2(rv + col);
              v0 += t.x;
              v1 += t.y;
            }
            if (e.act == ACT_RELU) {
              v0 = fmaxf(v0, 0.f);
              v1 = fmaxf(v1, 0.f);
            } else if (e.act == ACT_SILU) {
              v0 = silu_f(v0);
              v1 = silu_f(v1);
            } else if (e.act == ACT_QUICK_GELU) {
              v0 = quick_gelu_f(v0);
              v1 = quick_gelu_f(v1);
            }
            if (res != nullptr) {
              const float2 t = ldh2(res + col);
              v0 += t.x;
              v1 += t.y;
            }
            *reinterpret_cast<uint32_t*>(out + col) = pack_h2(v0, v1);
          }
        }
      } else {
        // GEGLU (BLOCK_N == 256): tile columns [0,128) are "hidden", [128,256) the matching "gate" rows of the packed weight.  FP8:
        // on dequantised accumulators; with out8 the 128 outputs of the row are quantised to e4m3 with one scale, their amax
        // reduced over the quad of lanes that hold the row (the geglu value replaces the hidden accumulator it came from)
        [[maybe_unused]] float amax = 0.f;
#pragma unroll
        for (int j = 0; j < BLOCK_N / 16; ++j) {
          const int hcol = n_blk * BLOCK_N + 8 * j + 2 * quad;
          const int ocol = n_blk * (BLOCK_N / 2) + 8 * j + 2 * quad;
          float h0 = acc[4 * j + 2 * hh], h1 = acc[4 * j + 2 * hh + 1];
          float g0 = acc[4 * (j + BLOCK_N / 16) + 2 * hh], g1 = acc[4 * (j + BLOCK_N / 16) + 2 * hh + 1];
          if constexpr (FP8) {
            const float2 swh = __ldg(reinterpret_cast<const float2*>(e.w_scale + hcol));
            const float2 swg = __ldg(reinterpret_cast<const float2*>(e.w_scale + hcol + BLOCK_N / 2));
            h0 = h0 * rs * swh.x;
            h1 = h1 * rs * swh.y;
            g0 = g0 * rs * swg.x;
            g1 = g1 * rs * swg.y;
          }
          if (has_bias) {
            const float2 bh = ldh2(e.bias + hcol), bg = ldh2(e.bias + hcol + BLOCK_N / 2);
            h0 += bh.x;
            h1 += bh.y;
            g0 += bg.x;
            g1 += bg.y;
          }
          if constexpr (FP8) {
            const float o0 = geglu1(h0, g0), o1 = geglu1(h1, g1);
            if (e.out8 != nullptr) {
              acc[4 * j + 2 * hh] = o0;
              acc[4 * j + 2 * hh + 1] = o1;
              amax = fmaxf(amax, fmaxf(fabsf(o0), fabsf(o1)));
            } else if (ocol < e.n_valid) {
              *reinterpret_cast<uint32_t*>(out + ocol) = pack_h2(o0, o1);
            }
          } else if (ocol < e.n_valid) {
            *reinterpret_cast<uint32_t*>(out + ocol) = pack_h2(geglu1(h0, g0), geglu1(h1, g1));
          }
        }
        if (FP8 && e.out8 != nullptr) {
          const unsigned qmask = 0xFu << (lane & 28);
          amax = fmaxf(amax, __shfl_xor_sync(qmask, amax, 1));
          amax = fmaxf(amax, __shfl_xor_sync(qmask, amax, 2));
          const float inv = e4m3_inv(amax);
          uint8_t* o8 = e.out8 + row * e.ldc + n_blk * (BLOCK_N / 2);
#pragma unroll
          for (int j = 0; j < BLOCK_N / 16; ++j)
            *reinterpret_cast<uint16_t*>(o8 + 8 * j + 2 * quad) = e4m3x2(acc[4 * j + 2 * hh], acc[4 * j + 2 * hh + 1], inv);
          if (quad == 0) e.out8_scale[row * e.out8_scale_ld + n_blk] = e4m3_scale(amax);
        }
      }
    }
  }
}

}  // namespace

void choose_conv_box(int NF, int H, int W, int* bn, int* bh, int* bw) {
  constexpr int rows = BLOCK_M;
  long long best = -1;
  int b_n = 1, b_h = 1, b_w = rows;
  for (int w = rows; w >= 1; w >>= 1) {
    for (int h = rows / w; h >= 1; h >>= 1) {
      int n = rows / (w * h);
      auto up = [](int a, int b) { return static_cast<long long>((a + b - 1) / b) * b; };
      long long padded = up(NF, n) * up(H, h) * up(W, w);
      if (best < 0 || padded < best) {  // ties keep the widest box along W (longest contiguous TMA rows)
        best = padded;
        b_n = n;
        b_h = h;
        b_w = w;
      }
    }
  }
  *bn = b_n;
  *bh = b_h;
  *bw = b_w;
}

// Shared-memory plan.  The staging covers the tile's output columns when it fits (then the residual is prefetched during the
// tile's MMAs), else it is used in rounds.  Ring variant: the whole tile is staged and the ring takes what is left, up to
// kMaxRingStages (6 stages at BLOCK_N 128, 5 at 160).  B-stationary: the BLOCK_N x K weight panel plus at least
// three A stages must fit beside at least one slab, and every CTA must get at least two tiles of its n_blk; slabs come before
// A stages beyond three.
static bool plan_smem(int block_n, bool bst, int slabs_wanted, int num_k_blocks, int* stages, int* slabs) {
  if (!bst) {
    const SmemLayout l = smem_layout(block_n, false, num_k_blocks, 0, slabs_wanted);
    *slabs = slabs_wanted;
    *stages = (kMaxSmem - l.bytes) / l.stage;
    if (*stages > kMaxRingStages) *stages = kMaxRingStages;
    return *stages >= 2;
  }
  const int stage = smem_layout(block_n, true, num_k_blocks, 0, 0).stage;
  int sl = (kMaxSmem - smem_layout(block_n, true, num_k_blocks, 3, 0).bytes) / SLAB_BYTES;
  if (sl > slabs_wanted) sl = slabs_wanted;
  if (sl < (slabs_wanted ? 1 : 0)) return false;
  int st = (kMaxSmem - smem_layout(block_n, true, num_k_blocks, 0, sl).bytes) / stage;
  if (st > kMaxStages) st = kMaxStages;
  if (st < 3) return false;
  *stages = st;
  *slabs = sl;
  return true;
}

template <int BN, bool BST, bool FP8>
static cudaError_t launch_t(const CUtensorMap& a0, const CUtensorMap& a1, const CUtensorMap& b, const CUtensorMap& out, const CUtensorMap& res,
                            GemmProblem p, const GemmEpilogue& e, const GemmPlan& plan, cudaStream_t stream) {
  static bool attr_set = false;
  if (!attr_set) {
    cudaError_t err = cudaFuncSetAttribute(gemm_kernel<BN, BST, FP8>, cudaFuncAttributeMaxDynamicSharedMemorySize, kMaxSmem);
    if (err != cudaSuccess) return err;
    attr_set = true;
  }
  p.stages = plan.stages;
  p.epi_slabs = plan.epi_slabs;
  const int smem = smem_layout(BN, BST, p.num_k_blocks, plan.stages, plan.epi_slabs).bytes;
  gemm_kernel<BN, BST, FP8><<<plan.grid, GEMM_THREADS, smem, stream>>>(a0, a1, b, out, res, p, e);
  return cudaGetLastError();
}

// The <BLOCK_N, BST> instantiation of the fp16 or the e4m3 kernel that runs (block_n, plan).
template <bool FP8>
static cudaError_t launch_any(const CUtensorMap& a0, const CUtensorMap& a1, const CUtensorMap& b, const CUtensorMap& out, const CUtensorMap& res,
                              const GemmProblem& p, const GemmEpilogue& e, int block_n, const GemmPlan& plan, cudaStream_t stream) {
  if (plan.bst_stages > 0) {
    if (block_n == 256) return launch_t<256, true, FP8>(a0, a1, b, out, res, p, e, plan, stream);
    if (block_n == 160) return launch_t<160, true, FP8>(a0, a1, b, out, res, p, e, plan, stream);
    return launch_t<128, true, FP8>(a0, a1, b, out, res, p, e, plan, stream);
  }
  if (block_n == 256) return launch_t<256, false, FP8>(a0, a1, b, out, res, p, e, plan, stream);
  if (block_n == 160) return launch_t<160, false, FP8>(a0, a1, b, out, res, p, e, plan, stream);
  return launch_t<128, false, FP8>(a0, a1, b, out, res, p, e, plan, stream);
}

bool plan_gemm(const GemmProblem& p, int block_n, int num_sms, GemmPlan* plan) {
  if (block_n != 128 && block_n != 160 && block_n != 256) return false;
  const TileCounts t = tile_counts(p, block_n);
  const int tiles = t.m * t.n;
  if (tiles <= 0 || p.num_k_blocks <= 0) return false;
  // Staged epilogue for tiles up to 160 wide on outputs up to 640 columns (the level-0/1 linears and the 3x3 convolutions up to 640
  // channels: up to 28 % faster per launch on an H100 SXM at 700 W, most of all with a residual).  Kept on register stores, where
  // staging measured slower: 256-wide tiles (the staging costs a ring stage, or rounds in the B-stationary variant) and wider
  // outputs (the N = 960 / 1920 projections, 1.9-2.2x); the up-convolution scatters its rows over two output parities and batched B
  // pads each item's columns.
  const bool staged = block_n <= 160 && p.N <= 640 && p.a_mode != A_UPCONV2X2 && !p.b_batch;
  const int slabs = staged ? block_n / SLAB_COLS : 0;
  plan->bst_stages = 0;
  plan->grid = tiles < num_sms ? tiles : num_sms;
  if (!plan_smem(block_n, false, slabs, p.num_k_blocks, &plan->stages, &plan->epi_slabs)) return false;
  if (p.a_mode == A_LINEAR && !p.b_batch && t.n <= num_sms) {
    const int per_col = num_sms / t.n;  // CTAs sharing one n_blk
    int st, sl;
    if (per_col >= 1 && t.m >= 2 * per_col && plan_smem(block_n, true, slabs, p.num_k_blocks, &st, &sl)) {
      plan->bst_stages = plan->stages = st;
      plan->epi_slabs = sl;
      plan->grid = per_col * t.n;   // gridDim.x a multiple of n_tiles: each CTA keeps one n_blk
    }
  }
  return true;
}

cudaError_t launch_gemm(const CUtensorMap& a0, const CUtensorMap& a1, const CUtensorMap& b, const CUtensorMap& out, const CUtensorMap& res,
                        const GemmProblem& p, const GemmEpilogue& e, int block_n, const GemmPlan& plan, cudaStream_t stream) {
  return launch_any<false>(a0, a1, b, out, res, p, e, block_n, plan, stream);
}

cudaError_t launch_gemm_fp8(const CUtensorMap& a, const CUtensorMap& b, const CUtensorMap& out, const CUtensorMap& res, const GemmProblem& p,
                            const GemmEpilogue& e, int block_n, const GemmPlan& plan, cudaStream_t stream) {
  // the 256-wide instantiations have no second accumulator set: they would ignore per-(row, k-block) A scales
  if (e.a_scale_ld != 0 && block_n == 256) return cudaErrorInvalidValue;
  return launch_any<true>(a, a, b, out, res, p, e, block_n, plan, stream);
}

}  // namespace hv
