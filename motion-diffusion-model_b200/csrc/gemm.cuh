// wgmma GEMMs for sm_90a:   D[M,N] = A[M,K] * W[N,K]^T   (fp16 in, fp32 accumulate)
//
// The operand pipeline shared by the three GEMM kernels (this file's gemm_f16_wgmma, gemm_f16_pingpong in
// gemm_pingpong.cuh, gemm_resid_ln_cluster in gemm_ln.cuh): a 384-thread CTA whose warpgroup 0 is the TMA producer
// (one elected thread, cp.async.bulk.tensor 2-D, 128B-swizzled A and W boxes) and warpgroups 1 and 2 the wgmma
// consumers.  The operands flow through a STAGES-deep ring of shared-memory stages, each with a `full` mbarrier (the
// producer's expect_tx + the TMA transactions) and an `empty` mbarrier (the consumer warps' arrivals once the MMAs that
// read the stage are done).  Ring tracks the stage and phase, produce_kblocks fills one tile's k-blocks and
// consume_kblocks issues their MMAs with one wgmma group in flight while the next stage is awaited.  A is [M,K]
// row-major (K contiguous), W is the torch nn.Linear layout [N,K] row-major -- both K-major wgmma operands, no
// transposes anywhere.  K tails / M tails / N tails rely on TMA out-of-bounds zero fill (loads) and clipping (stores).
//
// gemm_f16_wgmma, the staged kernel: persistent, tiles statically strided over the grid (tile = blockIdx.x + k *
// gridDim.x, N fastest so concurrently running CTAs share the same A rows in L2).  Consumer warpgroup g issues wgmma
// m64 x BLOCK_N x k16 for rows [64 (g-1), +64) of the 128-row tile and then runs the fused epilogue of those rows
// itself: the accumulator fragment is staged through a warpgroup-private fp32 tile in shared memory so that the
// epilogue functors see it as "thread = row" -- warp w of the warpgroup owns rows [32 (w & 1), +32) and the 64-column
// block part = w >> 1 of the tile (BLOCK_N <= 128), lane = row; each 32-column chunk is handed to the functor.  While
// the consumers run the epilogue of tile i the producer already streams the operands of tile i+1.  The step runs this
// kernel for the embedding (BLOCK_N = 128) and the output projection (96), once per step each; the per-layer
// projections run on gemm_f16_pingpong, which takes its epilogue from the accumulator fragment.
#pragma once
#include "ptx.cuh"

namespace b200 {

constexpr int GEMM_BLOCK_M = 128;
constexpr int GEMM_BLOCK_K = 64;  // 64 fp16 = 128 B = one swizzle row
constexpr int GEMM_EPI_WARPS = 8;
constexpr int GEMM_THREADS = 384;
constexpr int GEMM_BAR_BYTES = 1024;
constexpr int GEMM_BIAS_BYTES = 8192;   // gemm_f16_pingpong: per-column epilogue vector (bias), staged once per CTA: N <= 2048

// setmaxnreg: the producer warpgroup hands its registers to the consumers (40 + 2 x 232 <= 3 x 168, the pool of a
// 384-thread CTA).  The values are the ones the measured numbers in DESIGN.md section 5 were taken with.
constexpr int GEMM_REGS_PRODUCER = 40, GEMM_REGS_CONSUMER = 232;

// Bytes from smem_raw, the start of the dynamic shared memory, to its first 1024-byte boundary (128B-swizzled boxes).
// The kernels align by adding this offset to smem_raw itself, so that the compiler still sees shared-memory pointers
// (LDS / STS rather than generic LD / ST) and 32-bit address arithmetic.
__device__ __forceinline__ uint32_t smem_pad1024(const uint8_t* smem_raw) {
  return (1024u - (smem_u32(smem_raw) & 1023u)) & 1023u;
}

// Position in a STAGES-deep mbarrier ring: the stage and the parity of its current phase.  A consumer waits on the
// stage's full barrier at `phase`, the producer on its empty barrier at `phase ^ 1` (the first pass finds it free).
template <int STAGES>
struct Ring {
  int stage = 0;
  uint32_t phase = 0;
  Ring() = default;
  __device__ __forceinline__ explicit Ring(int pos) : stage(pos % STAGES), phase((pos / STAGES) & 1) {}
  __device__ __forceinline__ void advance() {
    if (++stage == STAGES) { stage = 0; phase ^= 1; }
  }
  // the position n stages further on
  __device__ __forceinline__ Ring ahead(int n) const {
    Ring r(stage + n);
    r.phase ^= phase;
    return r;
  }
};

// Producer: one tile's num_kb k-blocks into the ring, each once its stage is free -- the A box (rows from a_row) at the
// start of the stage, the W box (rows from w_row) w_off bytes into it, stage_bytes in all on the stage's full barrier.
// first() runs once the first k-block's stage is free.
template <int STAGES, class First>
__device__ __forceinline__ void produce_kblocks(Ring<STAGES>& ring, uint8_t* tiles, int stage_bytes, uint64_t* full_bar,
                                                uint64_t* empty_bar, const CUtensorMap* map_a, int a_row,
                                                const CUtensorMap* map_b, int w_off, int w_row, int num_kb, First&& first) {
  for (int kb = 0; kb < num_kb; ++kb) {
    mbar_wait(&empty_bar[ring.stage], ring.phase ^ 1);
    if (kb == 0) first();
    uint8_t* s = tiles + ring.stage * stage_bytes;
    mbar_expect_tx(&full_bar[ring.stage], stage_bytes);
    tma_load_2d(s, map_a, &full_bar[ring.stage], kb * GEMM_BLOCK_K, a_row);
    tma_load_2d(s + w_off, map_b, &full_bar[ring.stage], kb * GEMM_BLOCK_K, w_row);
    ring.advance();
  }
}

// Consumer: for each of num_kb k-blocks, wait until its stage has landed, run mma(shared address of the stage, kb) --
// one wgmma group with its accumulator fences: fence_acc, wgmma_fence, the MMAs (accumulating unless kb == 0 in the
// first k16 step), wgmma_commit, fence_acc -- and, once that group leaves one in flight, release the stage of the
// k-block before it (lane 0: one arrival per warp).  Returns the last k-block's stage, which the caller releases after
// wgmma_wait<0>.
template <int STAGES, class Mma>
__device__ __forceinline__ int consume_kblocks(Ring<STAGES>& ring, const uint8_t* tiles, int stage_bytes,
                                               uint64_t* full_bar, uint64_t* empty_bar, int num_kb, int lane, Mma&& mma) {
  int prev_stage = -1;
  for (int kb = 0; kb < num_kb; ++kb) {
    mbar_wait(&full_bar[ring.stage], ring.phase);
    mma(smem_u32(tiles + ring.stage * stage_bytes), kb);
    wgmma_wait<1>();
    if (prev_stage >= 0 && lane == 0) mbar_arrive(&empty_bar[prev_stage]);   // the group that read it is done
    prev_stage = ring.stage;
    ring.advance();
  }
  return prev_stage;
}

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
  static constexpr int budget = 227 * 1024 - 1024 /*alignment slack*/ - ACC_BYTES - EPI_BYTES - GEMM_BAR_BYTES;
  static constexpr int STAGES = (budget / STAGE_BYTES) > 6 ? 6 : (budget / STAGE_BYTES);
  static constexpr int TOTAL = 1024 + STAGES * STAGE_BYTES + EPI_BYTES + ACC_BYTES + GEMM_BAR_BYTES;
  static_assert(STAGES >= 2, "not enough shared memory for a pipeline");
  static_assert(Epi::SMEM_PER_WARP % 1024 == 0, "epilogue slabs must keep 1024-byte alignment (128B swizzle)");
  static_assert(B_BYTES % 1024 == 0, "W tiles must keep 1024-byte alignment (128B swizzle)");
};

// Per-warp epilogue context handed to the functor (lives in registers for the whole persistent loop).
struct EpiCtx {
  uint8_t* smem;        // warp-private slab, Epi::SMEM_PER_WARP bytes, 1024-byte aligned
  int lane;
  int M;
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
//   SMEM_PER_WARP                    bytes of warp-private shared memory
//   chunk(ctx, p, v, row0, col0)     v[32] = accumulator row (row0+lane), columns [col0, col0+32)
//   finish(ctx)                      once, before the CTA exits (drain async stores)
template <int BLOCK_N, class Epi>
__global__ void __launch_bounds__(GEMM_THREADS, 1)
gemm_f16_wgmma(const __grid_constant__ CUtensorMap map_a, const __grid_constant__ CUtensorMap map_b, int M, int N, int K,
               const __grid_constant__ typename Epi::Params ep) {
  using SM = GemmSmem<BLOCK_N, Epi>;
  using MMA = Wgmma<BLOCK_N>;
  constexpr int STAGES = SM::STAGES;
  constexpr int NREG = BLOCK_N / 2;
  static_assert(BLOCK_N % 32 == 0, "epilogue works on 32-column chunks");

  extern __shared__ uint8_t smem_raw[];
  uint8_t* tiles = smem_raw + smem_pad1024(smem_raw);
  uint8_t* epi_smem = tiles + STAGES * SM::STAGE_BYTES;
  float* acc_stage = reinterpret_cast<float*>(epi_smem + SM::EPI_BYTES);
  uint64_t* bars = reinterpret_cast<uint64_t*>(epi_smem + SM::EPI_BYTES + SM::ACC_BYTES);
  uint64_t* full_bar = bars;                    // [STAGES]
  uint64_t* empty_bar = bars + STAGES;          // [STAGES]  one arrival per consumer warp

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int tiles_m = (M + GEMM_BLOCK_M - 1) / GEMM_BLOCK_M;
  const int tiles_n = (N + BLOCK_N - 1) / BLOCK_N;
  const int num_tiles = tiles_m * tiles_n;
  const int num_kb = (K + GEMM_BLOCK_K - 1) / GEMM_BLOCK_K;

  pdl_launch_dependents();
  if (threadIdx.x == 0) {
    tma_prefetch_desc(&map_a);
    tma_prefetch_desc(&map_b);
    for (int s = 0; s < STAGES; ++s) {
      mbar_init(&full_bar[s], 1);
      mbar_init(&empty_bar[s], GEMM_EPI_WARPS);
    }
    fence_barrier_init();
  }
  __syncthreads();
  pdl_wait();   // the prologue above overlapped the previous kernel's tail; its outputs are visible from here on

  Ring<STAGES> ring;   // this thread's position in the operand ring
  if (warp < 4) {
    asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(GEMM_REGS_PRODUCER));
    // ------------------------------------------------------------ TMA producer
    if (warp == 0 && elect_one()) {
      for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
        const int m_blk = tile / tiles_n, n_blk = tile % tiles_n;
        produce_kblocks(ring, tiles, SM::STAGE_BYTES, full_bar, empty_bar, &map_a, m_blk * GEMM_BLOCK_M, &map_b,
                        SM::A_BYTES, n_blk * BLOCK_N, num_kb, [] {});
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
    ctx.lane = lane;
    ctx.M = M;
    ctx.seq = 0;
    float acc[NREG];
    auto mma = [&](uint32_t s, int kb) {
      const uint64_t da = wgmma_desc_k_sw128(s + wg * 64 * 128);
      const uint64_t db = wgmma_desc_k_sw128(s + SM::A_BYTES);
      wgmma_fence_acc(acc);
      wgmma_fence();
#pragma unroll
      for (int k = 0; k < GEMM_BLOCK_K / 16; ++k) MMA::mma(acc, da + 2 * k, db + 2 * k, (kb | k) != 0);
      wgmma_commit();
      wgmma_fence_acc(acc);
    };
    for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
      const int m_blk = tile / tiles_n, n_blk = tile % tiles_n;
      const int col_base = n_blk * BLOCK_N;
      const int last_stage = consume_kblocks(ring, tiles, SM::STAGE_BYTES, full_bar, empty_bar, num_kb, lane, mma);
      wgmma_wait<0>();
      wgmma_fence_acc(acc);
      if (lane == 0) mbar_arrive(&empty_bar[last_stage]);
      // ---- epilogue
      const int row0 = m_blk * GEMM_BLOCK_M + 64 * wg + rh;
      const bool live = row0 < M;  // warp-uniform: this warp's 32 rows exist
      uint32_t raw[32];
      auto run = [&](int c) {
        if (live && col_base + c < N) {
          load_row32<BLOCK_N>(st, rh + lane, c, raw);
          Epi::chunk(ctx, ep, raw, row0, col_base + c);
        }
      };
      named_bar_sync(1 + wg, 128);   // the previous tile's staging tile has been read by every warp of the warpgroup
      stage_acc<BLOCK_N>(st, acc, wq, lane);
      named_bar_sync(1 + wg, 128);
      const int c = part * 64;   // this warp owns one 64-column block of the tile (BLOCK_N = 96: the last is one chunk)
      if (c < BLOCK_N) run(c);
      if (c + 32 < BLOCK_N) run(c + 32);
    }
    Epi::finish(ctx);
  }
}

}  // namespace b200
