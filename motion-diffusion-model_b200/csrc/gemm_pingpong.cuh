// Projection GEMM with the epilogue under the MMAs, sm_90a:   out = epi(A[M,K] * W[N,K]^T)   (fp16 in, fp32 accumulate)
//
//   warpgroup 0      : the TMA producer of gemm.cuh, filling one PP_STAGES-deep ring in tile order
//   warpgroups 1, 2  : consumers.  Each owns a WHOLE 128 x 128 tile: two wgmma.m64n128k16 per k16 step (rows [0, 64) and
//                      [64, 128) of the tile against the same W tile), 128 fp32 accumulators per thread.
//
// Ping-pong: the CTA's tiles (tile = blockIdx.x + i * gridDim.x, N fastest so that concurrently running CTAs share A rows
// in L2) alternate between the consumer warpgroups, i even -> warpgroup 1, i odd -> warpgroup 2.  A pair of named
// barriers passes "the ring is yours" from one warpgroup to the other once it has waited for the last k-block of its tile
// and issued that k-block's MMAs, so the mainloops never interleave and the ring is consumed in tile order (ring position
// of tile i's first k-block = i * num_kb).  The epilogue of tile i then runs under the mainloop of tile i + 1.
//
// Epilogue straight from the accumulator fragment, no fp32 staging: thread (warp w, lane 4 g + t) holds rows
// 16 w + g (+8) of each 64-row half and columns 8 j + 2 t, +1 of every 8-column group j.  The functor (epilogues.cuh,
// "fragment interface") turns a column pair into fp16 and writes it into the warpgroup's 128-byte-swizzled output slabs
// ([128 rows x 128 B] per 64 columns: four TMA boxes of 32 rows).  Column pair 8 jj + 2 t of row r sits in 16-byte
// chunk jj ^ (r & 7) = jj ^ g, so the 32 lanes of a warp hit 32 distinct banks.  One thread per warpgroup ships the
// slabs with TMA stores and, before the next round overwrites them, waits until those stores have read them (they were
// issued a whole mainloop earlier).  Tails: loads zero-fill past M, N and K; stores clip at M and N, and boxes that lie
// wholly past M or N are not issued.
#pragma once
#include "epilogues.cuh"
#include "gemm.cuh"

namespace b200 {

constexpr int PP_BLOCK_N = 128;
constexpr int PP_A_BYTES = GEMM_BLOCK_M * GEMM_BLOCK_K * 2;                  // 16 KB
constexpr int PP_STAGE_BYTES = PP_A_BYTES + PP_BLOCK_N * GEMM_BLOCK_K * 2;    // 32 KB
constexpr int PP_SLAB_BYTES = 2 * GEMM_BLOCK_M * 128;                        // per consumer warpgroup: two 64-column slabs
constexpr int PP_STAGES = (227 * 1024 - 1024 /*alignment slack*/ - 2 * PP_SLAB_BYTES - GEMM_BIAS_BYTES - GEMM_BAR_BYTES) /
                          PP_STAGE_BYTES;
constexpr int PP_SMEM_BYTES = 1024 + PP_STAGES * PP_STAGE_BYTES + 2 * PP_SLAB_BYTES + GEMM_BIAS_BYTES + GEMM_BAR_BYTES;
static_assert(PP_STAGES == 4, "shared-memory budget: 4 operand stages of 32 KB");
// named barriers (0 is __syncthreads): 1 + g = "consumer warpgroup g may start its next mainloop", 3 + g = warpgroup g's
// epilogue
constexpr int PP_BAR_TURN = 1, PP_BAR_EPI = 3;

// Epi: EpiBiasF16<GELU>, EpiBiasF16Global or EpiBiasF16Wide<GELU> (PP_ROUND_COLS, pp_tile_bias, pp_pair, pp_store).
// map_a: A [M, K] fp16, box 128 rows x 64; map_b: W [N, K] fp16, box 128 rows x 64; map_c: output, box 32 rows x 64 cols.
template <class Epi>
__global__ void __launch_bounds__(GEMM_THREADS, 1)
gemm_f16_pingpong(const __grid_constant__ CUtensorMap map_a, const __grid_constant__ CUtensorMap map_b,
                  const __grid_constant__ CUtensorMap map_c, int M, int N, int K,
                  const __grid_constant__ typename Epi::Params ep) {
  constexpr int RC = Epi::PP_ROUND_COLS;
  static_assert(RC == 64 || RC == 128, "a round is one or two 64-column slabs");

  extern __shared__ uint8_t smem_raw[];
  uint8_t* tiles = smem_raw + smem_pad1024(smem_raw);
  uint8_t* slabs = tiles + PP_STAGES * PP_STAGE_BYTES;
  float* bias_all = reinterpret_cast<float*>(slabs + 2 * PP_SLAB_BYTES);
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(slabs + 2 * PP_SLAB_BYTES + GEMM_BIAS_BYTES);   // [STAGES]
  uint64_t* empty_bar = full_bar + PP_STAGES;   // [STAGES]  one arrival per warp of the consuming warpgroup

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int tiles_m = (M + GEMM_BLOCK_M - 1) / GEMM_BLOCK_M;
  const int tiles_n = (N + PP_BLOCK_N - 1) / PP_BLOCK_N;
  const int num_tiles = tiles_m * tiles_n;
  const int num_kb = (K + GEMM_BLOCK_K - 1) / GEMM_BLOCK_K;
  const int my_tiles = static_cast<int>(blockIdx.x) < num_tiles ? (num_tiles - 1 - blockIdx.x) / gridDim.x + 1 : 0;

  pdl_launch_dependents();
  Epi::preload(ep, bias_all, N, threadIdx.x, blockDim.x);   // visible to the consumers after the barrier below
  if (threadIdx.x == 0) {
    tma_prefetch_desc(&map_a);
    tma_prefetch_desc(&map_b);
    tma_prefetch_desc(&map_c);
    for (int s = 0; s < PP_STAGES; ++s) {
      mbar_init(&full_bar[s], 1);
      mbar_init(&empty_bar[s], 4);
    }
    fence_barrier_init();
  }
  __syncthreads();
  pdl_wait();   // the prologue above overlapped the previous kernel's tail; its outputs are visible from here on

  if (warp < 4) {
    asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(GEMM_REGS_PRODUCER));
    // ------------------------------------------------------------ TMA producer
    if (warp == 0 && elect_one()) {
      Ring<PP_STAGES> ring;
      for (int i = 0; i < my_tiles; ++i) {
        const int tile = blockIdx.x + i * gridDim.x;
        const int m_blk = tile / tiles_n, n_blk = tile % tiles_n;
        produce_kblocks(ring, tiles, PP_STAGE_BYTES, full_bar, empty_bar, &map_a, m_blk * GEMM_BLOCK_M, &map_b, PP_A_BYTES,
                        n_blk * PP_BLOCK_N, num_kb, [] {});
      }
    }
  } else {
    asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(GEMM_REGS_CONSUMER));
    // ------------------------------------------------------------ consumers: a whole tile's MMAs + its epilogue
    const int wg = (warp >> 2) - 1;          // 0 / 1: takes the CTA's tiles i = wg, wg + 2, ...
    const int wq = warp & 3;
    const int g = lane >> 2, t = lane & 3;
    const bool leader = wq == 0 && lane == 0;   // ships the warpgroup's slabs
    uint8_t* slab = slabs + wg * PP_SLAB_BYTES;
    // byte offset of this thread's column pair in row 16 wq + g of a slab, before the chunk index (row + 8: +1024,
    // the second 64-row half: +8192)
    const int toff = (16 * wq + g) * 128 + 4 * t;
    float acc0[64], acc1[64];   // rows [0, 64) and [64, 128) of the tile
    auto mma = [&](uint32_t s, int kb) {
      const uint64_t da0 = wgmma_desc_k_sw128(s);
      const uint64_t da1 = wgmma_desc_k_sw128(s + 64 * 128);
      const uint64_t db = wgmma_desc_k_sw128(s + PP_A_BYTES);
      wgmma_fence_acc(acc0);
      wgmma_fence_acc(acc1);
      wgmma_fence();
#pragma unroll
      for (int k = 0; k < GEMM_BLOCK_K / 16; ++k) {
        Wgmma<128>::mma(acc0, da0 + 2 * k, db + 2 * k, (kb | k) != 0);
        Wgmma<128>::mma(acc1, da1 + 2 * k, db + 2 * k, (kb | k) != 0);
      }
      wgmma_commit();
      wgmma_fence_acc(acc0);
      wgmma_fence_acc(acc1);
    };
    for (int i = wg; i < my_tiles; i += 2) {
      const int tile = blockIdx.x + i * gridDim.x;
      const int m_blk = tile / tiles_n, n_blk = tile % tiles_n;
      Ring<PP_STAGES> ring(i * num_kb);   // the tile's first k-block
      if (i > 0) named_bar_sync(PP_BAR_TURN + wg, 256);   // the other warpgroup has issued tile i - 1
      const int last_stage = consume_kblocks(ring, tiles, PP_STAGE_BYTES, full_bar, empty_bar, num_kb, lane, mma);
      if (i + 1 < my_tiles) named_bar_arrive(PP_BAR_TURN + (wg ^ 1), 256);   // hand the ring to the other warpgroup
      wgmma_wait<0>();
      wgmma_fence_acc(acc0);
      wgmma_fence_acc(acc1);
      if (lane == 0) mbar_arrive(&empty_bar[last_stage]);
      // ---- epilogue, in rounds of RC columns
      const int row_t = m_blk * GEMM_BLOCK_M, col_t = n_blk * PP_BLOCK_N;
      // (an epilogue that writes its scratch does so after this warpgroup's last read of the previous tile's bias: the
      // previous epilogue's final named barrier; the barrier of the first round below publishes it)
      const float* bs = Epi::pp_tile_bias(ep, bias_all, bias_all + wg * PP_BLOCK_N, col_t, N, threadIdx.x & 127);
#pragma unroll
      for (int c0 = 0; c0 < PP_BLOCK_N; c0 += RC) {
        if (col_t + c0 >= N) break;
        if (leader) bulk_wait_group_read<0>();   // the stores that last read the slabs are done
        named_bar_sync(PP_BAR_EPI + wg, 128);
#pragma unroll
        for (int jj = 0; jj < RC / 8; ++jj) {
          const int j = c0 / 8 + jj;
          const float2 b = *reinterpret_cast<const float2*>(bs + 8 * j + 2 * t);
          uint8_t* d = slab + (jj >> 3) * (GEMM_BLOCK_M * 128) + toff + (((jj & 7) ^ g) << 4);
          Epi::pp_pair(ep, b, acc0[4 * j], acc0[4 * j + 1], d);
          Epi::pp_pair(ep, b, acc0[4 * j + 2], acc0[4 * j + 3], d + 1024);
          Epi::pp_pair(ep, b, acc1[4 * j], acc1[4 * j + 1], d + 8192);
          Epi::pp_pair(ep, b, acc1[4 * j + 2], acc1[4 * j + 3], d + 8192 + 1024);
        }
        fence_proxy_async_smem();
        named_bar_sync(PP_BAR_EPI + wg, 128);
        if (leader) {
#pragma unroll
          for (int s = 0; s < RC / 64; ++s) {
            const int col = col_t + c0 + 64 * s;
            if (col < N)
              for (int r = 0; r < GEMM_BLOCK_M; r += 32)
                if (row_t + r < M) Epi::pp_store(&map_c, ep, slab + s * (GEMM_BLOCK_M * 128) + r * 128, col, row_t + r);
          }
          bulk_commit_group();
        }
      }
    }
    if (leader) bulk_wait_group<0>();   // the last stores have landed before the CTA exits
  }
}

}  // namespace b200
