// Persistent warp-specialised wgmma GEMM for sm_90a:   D[M,N] = A[M,K] * W[N,K]^T   (fp16 in, fp32 accumulate)
//
//   warpgroup 0      : TMA producer (one elected thread: cp.async.bulk.tensor 2-D, 128B-swizzled tiles, STAGES-deep
//                      mbarrier ring)
//   warpgroups 1, 2  : consumers.  Warpgroup g issues wgmma m64 x BLOCK_N x k16 for rows [64 (g-1), +64) of the 128-row
//                      tile, accumulators in registers, and then runs the fused epilogue of those rows itself.
//
// Epilogue: the accumulator fragment is staged through a warpgroup-private fp32 tile in shared memory so that the fused
// epilogue functors see it as "thread = row" -- warp w of the warpgroup owns rows [32 (w & 1), +32) and the
// 64-column block part = w >> 1 of the tile (BLOCK_N <= 128), lane = row; each 32-column chunk is handed to the functor, which stages its
// 128-byte-per-row output slab in warp-private shared memory (128B swizzle) and ships it with a TMA store.
//
// Tiles are statically strided over the persistent grid (tile = blockIdx.x + k * gridDim.x, N fastest so concurrently
// running CTAs share the same A rows in L2).  The step runs this kernel for the embedding (BLOCK_N = 128) and the output
// projection (96), once per step each; the per-layer projections run on gemm_f16_pingpong (gemm_pingpong.cuh), which
// takes its epilogue from the accumulator fragment.  A is [M,K] row-major (K contiguous), W is the torch nn.Linear
// layout [N,K] row-major -- both K-major wgmma operands, no transposes anywhere.  While the consumers run the epilogue
// of tile i the producer already streams the operands of tile i+1.  K tails / M tails / N tails rely on TMA
// out-of-bounds zero fill (loads) and clipping (stores).
#pragma once
#include "ptx.cuh"

namespace b200 {

constexpr int GEMM_BLOCK_M = 128;
constexpr int GEMM_BLOCK_K = 64;  // 64 fp16 = 128 B = one swizzle row
constexpr int GEMM_EPI_WARPS = 8;
constexpr int GEMM_THREADS = 384;
constexpr int GEMM_BAR_BYTES = 1024;
constexpr int GEMM_BIAS_BYTES = 8192;   // per-column epilogue vector (bias) of the whole GEMM, staged once per CTA: N <= 2048

// setmaxnreg: the producer warpgroup hands its registers to the consumers (40 + 2 x 232 <= 3 x 168, the pool of a
// 384-thread CTA).  The values are the ones the measured numbers in DESIGN.md section 5 were taken with.
constexpr int GEMM_REGS_PRODUCER = 40, GEMM_REGS_CONSUMER = 232;

template <int BLOCK_N>
constexpr int gemm_stage_ld() { return BLOCK_N + 4; }   // fp32 row pitch of the staging tile (bank spread)

template <int BLOCK_N, class Epi>
struct GemmSmem {
  static_assert(BLOCK_N <= 128, "the whole accumulator tile is staged for the epilogue at once");
  static constexpr int A_BYTES = GEMM_BLOCK_M * GEMM_BLOCK_K * 2;  // 16 KB
  static constexpr int B_BYTES = BLOCK_N * GEMM_BLOCK_K * 2;       // one k-block of the W tile
  static constexpr int STAGE_BYTES = A_BYTES + B_BYTES;
  static constexpr int ACC_BYTES = 2 * 64 * gemm_stage_ld<BLOCK_N>() * 4;   // one staging tile per consumer warpgroup
  static constexpr int EPI_BYTES = GEMM_EPI_WARPS * Epi::SMEM_PER_WARP;  // SMEM_PER_WARP is a multiple of 1024
  static constexpr int budget = 227 * 1024 - 1024 /*alignment slack*/ - ACC_BYTES - EPI_BYTES - GEMM_BIAS_BYTES - GEMM_BAR_BYTES;
  static constexpr int STAGES = (budget / STAGE_BYTES) > 6 ? 6 : (budget / STAGE_BYTES);
  static constexpr int TOTAL = 1024 + STAGES * STAGE_BYTES + EPI_BYTES + ACC_BYTES + GEMM_BIAS_BYTES + GEMM_BAR_BYTES;
  static_assert(STAGES >= 2, "not enough shared memory for a pipeline");
  static_assert(Epi::SMEM_PER_WARP % 1024 == 0, "epilogue slabs must keep 1024-byte alignment (128B swizzle)");
  static_assert(B_BYTES % 1024 == 0, "W tiles must keep 1024-byte alignment (128B swizzle)");
};

// Per-warp epilogue context handed to the functor (lives in registers for the whole persistent loop).
struct EpiCtx {
  uint8_t* smem;        // warp-private slab, Epi::SMEM_PER_WARP bytes, 1024-byte aligned
  const CUtensorMap* map_c;
  const float* bias_all; // CTA-shared copy of the functor's per-column vector for columns [0, N)
  int lane;
  int M, N;
  int col_base;         // first column of the tile in flight
  int col_end;          // first column after the tile in flight (col_base + BLOCK_N)
  uint32_t seq;         // running chunk / block counter (buffer rotation), functor-defined
};

// Write a warpgroup's accumulator fragment (rows [0, 64) of its half tile) into the fp32 staging tile.
template <int BLOCK_N>
__device__ __forceinline__ void stage_acc(float* st, const float (&acc)[BLOCK_N / 2], int wq, int lane) {
  constexpr int LD = gemm_stage_ld<BLOCK_N>();
  const int r = 16 * wq + (lane >> 2), c = 2 * (lane & 3);
#pragma unroll
  for (int j = 0; j < BLOCK_N / 8; ++j) {
    *reinterpret_cast<float2*>(st + r * LD + 8 * j + c) = make_float2(acc[4 * j], acc[4 * j + 1]);
    *reinterpret_cast<float2*>(st + (r + 8) * LD + 8 * j + c) = make_float2(acc[4 * j + 2], acc[4 * j + 3]);
  }
}
// thread = row: 32 consecutive fp32 accumulator columns of row `row` of the staging tile
template <int BLOCK_N>
__device__ __forceinline__ void load_row32(const float* st, int row, int col, uint32_t (&raw)[32]) {
  constexpr int LD = gemm_stage_ld<BLOCK_N>();
  const float4* p = reinterpret_cast<const float4*>(st + row * LD + col);
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const float4 v = p[i];
    raw[4 * i] = __float_as_uint(v.x); raw[4 * i + 1] = __float_as_uint(v.y);
    raw[4 * i + 2] = __float_as_uint(v.z); raw[4 * i + 3] = __float_as_uint(v.w);
  }
}

// Epi interface (all static, called by every lane of a consumer warp, warp-uniform arguments):
//   SMEM_PER_WARP                                   bytes of warp-private shared memory
//   preload(p, dst, N, tid, nthreads)               stage the per-column vector once per CTA (before the first tile)
//   tile_begin(ctx, p, row0, col_base)              before the tile's chunks
//   chunk(ctx, p, v, row0, col0, next_col0)         v[32] = accumulator row (row0+lane), columns [col0, col0+32);
//                                                   next_col0 = first column of this warp's next chunk in the tile, or -1
//   tile_end(ctx, p, row0, col_base)                after the last chunk
//   finish(ctx)                                     once, before the CTA exits (drain async stores)
template <int BLOCK_N, class Epi>
__global__ void __launch_bounds__(GEMM_THREADS, 1)
gemm_f16_wgmma(const __grid_constant__ CUtensorMap map_a, const __grid_constant__ CUtensorMap map_b,
               const __grid_constant__ CUtensorMap map_c, int M, int N, int K,
               const __grid_constant__ typename Epi::Params ep) {
  using SM = GemmSmem<BLOCK_N, Epi>;
  using MMA = Wgmma<BLOCK_N>;
  constexpr int STAGES = SM::STAGES;
  constexpr int NREG = BLOCK_N / 2;
  static_assert(BLOCK_N % 32 == 0, "epilogue works on 32-column chunks");

  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* tiles = smem;
  uint8_t* epi_smem = tiles + STAGES * SM::STAGE_BYTES;
  float* acc_stage = reinterpret_cast<float*>(epi_smem + SM::EPI_BYTES);
  float* bias_all = reinterpret_cast<float*>(epi_smem + SM::EPI_BYTES + SM::ACC_BYTES);
  uint64_t* bars = reinterpret_cast<uint64_t*>(epi_smem + SM::EPI_BYTES + SM::ACC_BYTES + GEMM_BIAS_BYTES);
  uint64_t* full_bar = bars;                    // [STAGES]
  uint64_t* empty_bar = bars + STAGES;          // [STAGES]  one arrival per consumer warp

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int tiles_m = (M + GEMM_BLOCK_M - 1) / GEMM_BLOCK_M;
  const int tiles_n = (N + BLOCK_N - 1) / BLOCK_N;
  const int num_tiles = tiles_m * tiles_n;
  const int num_kb = (K + GEMM_BLOCK_K - 1) / GEMM_BLOCK_K;

  pdl_launch_dependents();
  Epi::preload(ep, bias_all, N, threadIdx.x, blockDim.x);   // visible to the consumers after the barrier below
  if (threadIdx.x == 0) {
    tma_prefetch_desc(&map_a);
    tma_prefetch_desc(&map_b);
    tma_prefetch_desc(&map_c);
    for (int s = 0; s < STAGES; ++s) {
      mbar_init(&full_bar[s], 1);
      mbar_init(&empty_bar[s], GEMM_EPI_WARPS);
    }
    fence_barrier_init();
  }
  __syncthreads();
  pdl_wait();   // the prologue above overlapped the previous kernel's tail; its outputs are visible from here on

  if (warp < 4) {
    asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(GEMM_REGS_PRODUCER));
    // ------------------------------------------------------------ TMA producer
    if (warp == 0 && elect_one()) {
      int stage = 0;
      uint32_t phase = 0;
      for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
        const int m_blk = tile / tiles_n, n_blk = tile % tiles_n;
        for (int kb = 0; kb < num_kb; ++kb) {
          mbar_wait(&empty_bar[stage], phase ^ 1);
          uint8_t* sa = tiles + stage * SM::STAGE_BYTES;
          mbar_expect_tx(&full_bar[stage], SM::STAGE_BYTES);
          tma_load_2d(sa, &map_a, &full_bar[stage], kb * GEMM_BLOCK_K, m_blk * GEMM_BLOCK_M);
          tma_load_2d(sa + SM::A_BYTES, &map_b, &full_bar[stage], kb * GEMM_BLOCK_K, n_blk * BLOCK_N);
          if (++stage == STAGES) { stage = 0; phase ^= 1; }
        }
      }
    }
  } else {
    asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(GEMM_REGS_CONSUMER));
    // ------------------------------------------------------------ consumers: MMA + epilogue
    const int wg = (warp >> 2) - 1;    // 0 / 1: rows [64 wg, +64) of the tile
    const int wq = warp & 3;           // warp inside the warpgroup
    const int part = wq >> 1;          // which 64-column blocks of the tile this warp's epilogue owns
    const int rh = 32 * (wq & 1);      // first staging row of this warp's epilogue
    float* st = acc_stage + wg * 64 * gemm_stage_ld<BLOCK_N>();
    EpiCtx ctx;
    ctx.smem = epi_smem + (warp - 4) * Epi::SMEM_PER_WARP;
    ctx.map_c = &map_c;
    ctx.bias_all = bias_all;
    ctx.lane = lane;
    ctx.M = M;
    ctx.N = N;
    ctx.seq = 0;
    int stage = 0;
    uint32_t phase = 0;
    float acc[NREG];
    for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
      const int m_blk = tile / tiles_n, n_blk = tile % tiles_n;
      const int col_base = n_blk * BLOCK_N;
      // ---- main loop: one wgmma group in flight while the next stage is awaited
      int prev_stage = -1;
      for (int kb = 0; kb < num_kb; ++kb) {
        mbar_wait(&full_bar[stage], phase);
        const uint32_t sa = smem_u32(tiles + stage * SM::STAGE_BYTES) + wg * 64 * 128;
        const uint32_t sb = smem_u32(tiles + stage * SM::STAGE_BYTES) + SM::A_BYTES;
        const uint64_t da = wgmma_desc_k_sw128(sa);
        const uint64_t db = wgmma_desc_k_sw128(sb);
        wgmma_fence_acc(acc);
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < GEMM_BLOCK_K / 16; ++k) MMA::mma(acc, da + 2 * k, db + 2 * k, (kb | k) != 0);
        wgmma_commit();
        wgmma_fence_acc(acc);
        wgmma_wait<1>();
        if (prev_stage >= 0 && lane == 0) mbar_arrive(&empty_bar[prev_stage]);   // the group that read it is done
        prev_stage = stage;
        if (++stage == STAGES) { stage = 0; phase ^= 1; }
      }
      wgmma_wait<0>();
      wgmma_fence_acc(acc);
      if (lane == 0) mbar_arrive(&empty_bar[prev_stage]);
      // ---- epilogue
      const int row0 = m_blk * GEMM_BLOCK_M + 64 * wg + rh;
      const bool live = row0 < M;  // warp-uniform: this warp's 32 rows exist
      ctx.col_base = col_base;
      ctx.col_end = col_base + BLOCK_N;
      if (live) Epi::tile_begin(ctx, ep, row0, col_base);
      uint32_t raw[32];
      auto run = [&](int c, int cn) {
        if (live && col_base + c < N) {
          load_row32<BLOCK_N>(st, rh + lane, c, raw);
          Epi::chunk(ctx, ep, raw, row0, col_base + c, (cn < BLOCK_N && col_base + cn < N) ? col_base + cn : -1);
        }
      };
      named_bar_sync(1 + wg, 128);   // the previous tile's staging tile has been read by every warp of the warpgroup
      stage_acc<BLOCK_N>(st, acc, wq, lane);
      named_bar_sync(1 + wg, 128);
      const int c = part * 64;   // this warp owns one 64-column block of the tile
      if (c < BLOCK_N) {
        const bool two = c + 32 < BLOCK_N;                     // (BLOCK_N = 96: the last block is a single chunk)
        const int cnext = c + 128;
        run(c, two ? c + 32 : cnext);
        if (two) run(c + 32, cnext);
      }
      if (live) Epi::tile_end(ctx, ep, row0, col_base);
    }
    Epi::finish(ctx);
  }
}

}  // namespace b200
