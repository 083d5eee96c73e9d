// wgmma GEMM with residual add + LayerNorm fused into the epilogue, N = d_model = 512 split over a 2-CTA cluster:
//
//     h <- LayerNorm( h + A W^T + bias ; gamma, beta, eps )        in place on the residual stream (fp16 [hi | lo])
//     (post-norm nn.TransformerEncoderLayer of the reference, built at model/mdm.py:77-84)
//
// Both CTAs of a cluster work on the SAME 128 rows; CTA r owns columns [256 r, 256 r + 256) (its own 256 rows of W).
// The operand pipeline is gemm.cuh's: warpgroup 0 is the TMA producer; consumer warpgroup g (1, 2) issues wgmma
// m64n256k16 for rows [64 (g-1), +64) and keeps its 64 x 256 fp32 accumulator in registers (128 per thread) for the
// whole epilogue.
//
// The residual moves only as bulk TMA traffic.  After a tile's last k-block the producer loads the CTA's 256 residual
// columns as four 64-column groups, each a 128-row hi box + the matching lo box (2 x 16 KB, 128-byte swizzle), into the
// next four stages of the operand ring (the same Ring: group grp at ring.ahead(grp)), so the loads overlap the tail of
// the mainloop.  Epilogue:
//   pass 1    v = acc + bias + residual (read from the swizzled slab in the accumulator's fragment layout: the 8 rows of a
//             quad group land on distinct 16-byte chunks, no bank conflicts), kept in the accumulator registers;
//             per-row partial sum / sum of squares over the CTA's 256 columns (quad shuffles)
//   exchange  one lane per row pushes the CTA's partial into the PEER CTA's shared memory with st.async (data + mbarrier
//             complete_tx in one message, no release fence); both CTAs now own the statistics of the 512-wide rows
//   pass 2    y = (v - mean) rstd gamma + beta -> [hi | lo] fp16, written back over the slab element by element (only the
//             owning thread touches each one); group by group, each warpgroup ships its 64 rows with TMA stores and hands
//             the ring stage back once the store has read it, so the next tile's first k-blocks load under the epilogue.
// Tail rows: loads zero-fill past row M (a box that lies wholly past M is not loaded), stores clip at M.
#pragma once
#include "epilogues.cuh"
#include "gemm.cuh"

namespace b200 {

constexpr int GLN_THREADS = 384;
constexpr int GLN_D = 512;
constexpr int GLN_BN = 256;                       // columns per CTA
constexpr int GLN_STAGE_BYTES = (128 + GLN_BN) * GEMM_BLOCK_K * 2;   // 48 KB
constexpr int GLN_STAGES = 4;
// residual groups: 64 columns of the CTA's 256, hi slab [128 rows x 128 B] then lo slab, in one ring stage
constexpr int GLN_GROUPS = GLN_BN / 64;
constexpr int GLN_RES_BOX_ROWS = 64;                            // box of the residual map: one consumer warpgroup's rows
constexpr int GLN_RES_BOX_BYTES = GLN_RES_BOX_ROWS * 128;       // 8 KB
constexpr int GLN_RES_HALF = GEMM_BLOCK_M * 128;                // 16 KB: the hi (or lo) slab of a group
static_assert(2 * GLN_RES_HALF <= GLN_STAGE_BYTES, "a residual group fits in one ring stage");
static_assert(GLN_GROUPS <= GLN_STAGES, "a tile's residual groups occupy distinct ring stages");
// setmaxnreg: the producer warpgroup hands its registers to the consumers, whose 128 accumulators stay live through
// the epilogue (40 + 2 x 232 = 504 <= 3 x 168, the pool a 384-thread CTA gets at launch)
constexpr int GLN_REGS_PRODUCER = 40, GLN_REGS_CONSUMER = 232;
constexpr int GLN_AUX_BYTES = 3 * GLN_BN * 4 /*bias gamma beta*/ + 2 * 128 * 8 /*remote stats, 2 stages*/ + 1024 /*barriers*/;

struct GemmLnSmem {
  static constexpr int TOTAL = 1024 + GLN_STAGES * GLN_STAGE_BYTES + GLN_AUX_BYTES;
  static_assert(TOTAL <= 227 * 1024, "shared memory budget");
};

#ifdef B200_TRACE
// Instrumented build only: %globaltimer stamps per tile, [CTA][tile iteration][role][event], role 0 the producer thread,
// 1 + wg the store thread of consumer warpgroup wg; read (and cleared) by b200mdm_debug_ln_trace, see tools/ln_phases.py
// for the events.  Without B200_TRACE the stamps compile to nothing.
constexpr int GLN_TRACE_CTAS = 264, GLN_TRACE_ITERS = 16, GLN_TRACE_ROLES = 3, GLN_TRACE_EVENTS = 8;
__device__ uint64_t g_gln_trace[GLN_TRACE_CTAS * GLN_TRACE_ITERS * GLN_TRACE_ROLES * GLN_TRACE_EVENTS];
__device__ __forceinline__ void gln_stamp(int it, int role, int ev) {
  if (blockIdx.x < GLN_TRACE_CTAS && it < GLN_TRACE_ITERS)
    g_gln_trace[((blockIdx.x * GLN_TRACE_ITERS + it) * GLN_TRACE_ROLES + role) * GLN_TRACE_EVENTS + ev] = globaltimer_ns();
}
#define GLN_STAMP(cond, it, role, ev) if (cond) gln_stamp(it, role, ev)
#else
#define GLN_STAMP(cond, it, role, ev)
#endif

struct GemmLnParams {
  const float* bias;    // [512]
  const float* gamma;   // [512]
  const float* beta;    // [512]
  float eps;
};

// map_a: A [M, K] fp16, box 128 rows; map_b: W [512, K] fp16, box 256 rows;
// map_h: the residual stream h, fp16 [M, 1024] = [hi | lo] (hi + lo carries ~22 bits), box 64 rows x 64 columns,
// 128-byte swizzle; updated in place.
// The hi half doubles as the fp16 A operand of the next GEMM (the trans_dec engine feeds both halves, K = 1024).
__global__ void __cluster_dims__(2, 1, 1) __launch_bounds__(GLN_THREADS, 1)
gemm_resid_ln_cluster(const __grid_constant__ CUtensorMap map_a, const __grid_constant__ CUtensorMap map_b,
                      const __grid_constant__ CUtensorMap map_h, int M, int K, const GemmLnParams lp) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* tiles = smem_raw + smem_pad1024(smem_raw);
  float* prm = reinterpret_cast<float*>(tiles + GLN_STAGES * GLN_STAGE_BYTES);   // bias | gamma | beta  (this CTA's 256 cols)
  float2* st_remote = reinterpret_cast<float2*>(prm + 3 * GLN_BN);             // [2 stages][128 rows], written by the PEER
  uint64_t* bars = reinterpret_cast<uint64_t*>(st_remote + 256);
  uint64_t* full_bar = bars;                       // [STAGES]
  uint64_t* empty_bar = bars + GLN_STAGES;         // [STAGES]  8 arrivals: one per consumer warp (k-block), or 4 from
                                                   //           each warpgroup's store thread (residual group)
  uint64_t* xbar = bars + 2 * GLN_STAGES;          // [2 stages][8 consumer warps]  peer's statistics have landed

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const uint32_t rank = cluster_ctarank();
  const int cluster_id = blockIdx.x >> 1;
  const int num_clusters = gridDim.x >> 1;
  const int num_tiles = (M + GEMM_BLOCK_M - 1) / GEMM_BLOCK_M;   // one tile per cluster = 128 rows x 512 columns
  const int num_kb = (K + GEMM_BLOCK_K - 1) / GEMM_BLOCK_K;
  const int col_cta = static_cast<int>(rank) * GLN_BN;

  pdl_launch_dependents();
  for (int i = threadIdx.x; i < GLN_BN; i += blockDim.x) {
    prm[i] = lp.bias[col_cta + i];
    prm[GLN_BN + i] = lp.gamma[col_cta + i];
    prm[2 * GLN_BN + i] = lp.beta[col_cta + i];
  }
  if (threadIdx.x == 0) {
    tma_prefetch_desc(&map_a);
    tma_prefetch_desc(&map_b);
    tma_prefetch_desc(&map_h);
    for (int s = 0; s < GLN_STAGES; ++s) {
      mbar_init(&full_bar[s], 1);
      mbar_init(&empty_bar[s], 8);
    }
    for (int s = 0; s < 16; ++s) mbar_init(&xbar[s], 1);   // one expect_tx arrival; the peer's lanes deliver 128 bytes with st.async
    fence_barrier_init();
  }
  __syncthreads();
  cluster_sync_all();   // the peer's barriers exist before anybody signals them
  pdl_wait();           // everything above overlapped the previous kernel's tail

  if (warp < 4) {
    asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(GLN_REGS_PRODUCER));
    // ------------------------------------------------------------ TMA producer
    if (warp == 0 && elect_one()) {
      Ring<GLN_STAGES> ring;
      for (int tile = cluster_id; tile < num_tiles; tile += num_clusters) {
        GLN_STAMP(true, (tile - cluster_id) / num_clusters, 0, 0);
        produce_kblocks(ring, tiles, GLN_STAGE_BYTES, full_bar, empty_bar, &map_a, tile * GEMM_BLOCK_M, &map_b, 16384,
                        col_cta, num_kb, [&] { GLN_STAMP(true, (tile - cluster_id) / num_clusters, 0, 1); });
        // the tile's residual, group by group, into the next ring stages (hi slab | lo slab)
        const int r0 = tile * GEMM_BLOCK_M;
        const bool two = r0 + GLN_RES_BOX_ROWS < M;   // the second warpgroup's rows exist
        for (int grp = 0; grp < GLN_GROUPS; ++grp) {
          mbar_wait(&empty_bar[ring.stage], ring.phase ^ 1);
          uint64_t* fb = &full_bar[ring.stage];
          uint8_t* sr = tiles + ring.stage * GLN_STAGE_BYTES;
          const int c = col_cta + 64 * grp;
          mbar_expect_tx(fb, (two ? 4 : 2) * GLN_RES_BOX_BYTES);
          tma_load_2d(sr, &map_h, fb, c, r0);
          tma_load_2d(sr + GLN_RES_HALF, &map_h, fb, GLN_D + c, r0);
          if (two) {
            tma_load_2d(sr + GLN_RES_BOX_BYTES, &map_h, fb, c, r0 + GLN_RES_BOX_ROWS);
            tma_load_2d(sr + GLN_RES_HALF + GLN_RES_BOX_BYTES, &map_h, fb, GLN_D + c, r0 + GLN_RES_BOX_ROWS);
          }
          ring.advance();
        }
        GLN_STAMP(true, (tile - cluster_id) / num_clusters, 0, 2);
      }
    }
  } else {
    asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(GLN_REGS_CONSUMER));
    // ------------------------------------------------------------ consumers: MMA + LayerNorm epilogue
    const int wg = (warp >> 2) - 1;
    const int wq = warp & 3;
    const int cw = warp - 4;                          // consumer warp 0..7
    const int g = lane >> 2, t = lane & 3;
    const int lrow = 64 * wg + 16 * wq + g;           // first of this thread's two rows inside the tile (+8 for the second)
    const bool store_thread = wq == 0 && lane == 0;   // issues the warpgroup's residual stores
    // byte offset of this thread's column pair in row lrow of a 128-byte-swizzled slab, before the chunk index: column
    // 8 jj + 2 t of a group sits in 16-byte chunk jj ^ (row & 7) = jj ^ g (row lrow + 8 is 1024 bytes further, same chunk)
    const int toff = lrow * 128 + 4 * t;
    const float* bias_s = prm;
    const float* gamma_s = prm + GLN_BN;
    const float* beta_s = prm + 2 * GLN_BN;
    Ring<GLN_STAGES> ring;
    float acc[128];
    int it = 0;
    auto mma = [&](uint32_t s, int kb) {
      GLN_STAMP(kb == 0 && store_thread, it, 1 + wg, 1);
      const uint64_t da = wgmma_desc_k_sw128(s + wg * 64 * 128);
      const uint64_t db = wgmma_desc_k_sw128(s + 16384);
      wgmma_fence_acc(acc);
      wgmma_fence();
#pragma unroll
      for (int k = 0; k < GEMM_BLOCK_K / 16; ++k) Wgmma<256>::mma(acc, da + 2 * k, db + 2 * k, (kb | k) != 0);
      wgmma_commit();
      wgmma_fence_acc(acc);
    };
    for (int tile = cluster_id; tile < num_tiles; tile += num_clusters, ++it) {
      const int as = it & 1;
      const uint32_t aphase = (it >> 1) & 1;
      if (lane == 0) mbar_expect_tx(&xbar[as * 8 + cw], 16 * 8);   // the peer's partials of this warp's 16 rows
      GLN_STAMP(store_thread, it, 1 + wg, 0);
      const int last_stage = consume_kblocks(ring, tiles, GLN_STAGE_BYTES, full_bar, empty_bar, num_kb, lane, mma);
      wgmma_wait<0>();
      wgmma_fence_acc(acc);
      GLN_STAMP(store_thread, it, 1 + wg, 2);
      if (lane == 0) mbar_arrive(&empty_bar[last_stage]);
      // the residual groups sit in the next GLN_GROUPS ring stages: group grp at ring.ahead(grp)

      // ---- pass 1: v = residual + (acc + bias) in place, partial statistics of the two rows
      float sa = 0.f, qa = 0.f, sb = 0.f, qb = 0.f;
#pragma unroll
      for (int j = 0; j < GLN_BN / 8; ++j) {
        const int grp = j >> 3, jj = j & 7;
        const Ring<GLN_STAGES> rg = ring.ahead(grp);
        if (jj == 0) mbar_wait(&full_bar[rg.stage], rg.phase);
        GLN_STAMP(jj == 0 && (grp == 0 || grp == GLN_GROUPS - 1) && store_thread, it, 1 + wg, grp == 0 ? 3 : 4);
        const uint8_t* slab = tiles + rg.stage * GLN_STAGE_BYTES + toff + ((jj ^ g) << 4);
        const int c = 8 * j + 2 * t;                   // local column of acc[4j], acc[4j+1] (and of acc[4j+2..3], row b)
        const float2 bb = *reinterpret_cast<const float2*>(bias_s + c);
        float2 ra, rb;
        {
          const float2 h = __half22float2(*reinterpret_cast<const __half2*>(slab));
          const float2 l = __half22float2(*reinterpret_cast<const __half2*>(slab + GLN_RES_HALF));
          ra = make_float2(h.x + l.x, h.y + l.y);
        }
        {
          const float2 h = __half22float2(*reinterpret_cast<const __half2*>(slab + 1024));
          const float2 l = __half22float2(*reinterpret_cast<const __half2*>(slab + GLN_RES_HALF + 1024));
          rb = make_float2(h.x + l.x, h.y + l.y);
        }
        acc[4 * j] = ra.x + (acc[4 * j] + bb.x);
        acc[4 * j + 1] = ra.y + (acc[4 * j + 1] + bb.y);
        acc[4 * j + 2] = rb.x + (acc[4 * j + 2] + bb.x);
        acc[4 * j + 3] = rb.y + (acc[4 * j + 3] + bb.y);
        sa += acc[4 * j] + acc[4 * j + 1];
        qa = fmaf(acc[4 * j], acc[4 * j], fmaf(acc[4 * j + 1], acc[4 * j + 1], qa));
        sb += acc[4 * j + 2] + acc[4 * j + 3];
        qb = fmaf(acc[4 * j + 2], acc[4 * j + 2], fmaf(acc[4 * j + 3], acc[4 * j + 3], qb));
      }
#pragma unroll
      for (int o = 1; o < 4; o <<= 1) {
        sa += __shfl_xor_sync(0xffffffffu, sa, o);
        qa += __shfl_xor_sync(0xffffffffu, qa, o);
        sb += __shfl_xor_sync(0xffffffffu, sb, o);
        qb += __shfl_xor_sync(0xffffffffu, qb, o);
      }
      // ---- statistics of the full 512-wide rows: this CTA's 256 columns + the peer CTA's
      float2* rem = st_remote + as * 128;
      if (t == 0) {
        const uint32_t peer = rank ^ 1;
        const uint32_t pbar = mapa_shared(smem_u32(&xbar[as * 8 + cw]), peer);
        st_async_f32x2(mapa_shared(smem_u32(&rem[lrow]), peer), sa, qa, pbar);
        st_async_f32x2(mapa_shared(smem_u32(&rem[lrow + 8]), peer), sb, qb, pbar);
      }
      mbar_wait_cluster(&xbar[as * 8 + cw], aphase);   // the peer's lanes have delivered this warp's 16 partials
      GLN_STAMP(store_thread, it, 1 + wg, 5);
      const float2 pa = rem[lrow], pb = rem[lrow + 8];
      const float mean_a = (sa + pa.x) * (1.f / GLN_D), mean_b = (sb + pb.x) * (1.f / GLN_D);
      const float rstd_a = rsqrtf(fmaxf((qa + pa.y) * (1.f / GLN_D) - mean_a * mean_a, 0.f) + lp.eps);
      const float rstd_b = rsqrtf(fmaxf((qb + pb.y) * (1.f / GLN_D) - mean_b * mean_b, 0.f) + lp.eps);
      // ---- pass 2: y -> [hi | lo] over the slab, then out by TMA store, one group at a time
      const int row_wg = tile * GEMM_BLOCK_M + 64 * wg;   // first row of this warpgroup's half of the tile
#pragma unroll
      for (int j = 0; j < GLN_BN / 8; ++j) {
        const int grp = j >> 3, jj = j & 7;
        const int rs = ring.ahead(grp).stage;
        uint8_t* slab = tiles + rs * GLN_STAGE_BYTES + toff + ((jj ^ g) << 4);
        const int c = 8 * j + 2 * t;
        const float2 gg = *reinterpret_cast<const float2*>(gamma_s + c);
        const float2 ee = *reinterpret_cast<const float2*>(beta_s + c);
        {
          const float y0 = (acc[4 * j] - mean_a) * rstd_a * gg.x + ee.x, y1 = (acc[4 * j + 1] - mean_a) * rstd_a * gg.y + ee.y;
          const __half2 h = __floats2half2_rn(y0, y1);
          const float2 f = __half22float2(h);
          *reinterpret_cast<__half2*>(slab) = h;
          *reinterpret_cast<__half2*>(slab + GLN_RES_HALF) = __floats2half2_rn(y0 - f.x, y1 - f.y);
        }
        {
          const float y0 = (acc[4 * j + 2] - mean_b) * rstd_b * gg.x + ee.x, y1 = (acc[4 * j + 3] - mean_b) * rstd_b * gg.y + ee.y;
          const __half2 h = __floats2half2_rn(y0, y1);
          const float2 f = __half22float2(h);
          *reinterpret_cast<__half2*>(slab + 1024) = h;
          *reinterpret_cast<__half2*>(slab + GLN_RES_HALF + 1024) = __floats2half2_rn(y0 - f.x, y1 - f.y);
        }
        if (jj == 7) {   // the warpgroup's 64 rows of this group are complete
          GLN_STAMP(grp == GLN_GROUPS - 1 && store_thread, it, 1 + wg, 6);
          fence_proxy_async_smem();
          named_bar_sync(1 + wg, 128);
          if (store_thread) {
            uint8_t* sg = tiles + rs * GLN_STAGE_BYTES + wg * GLN_RES_BOX_BYTES;
            if (row_wg < M) {
              const int cg = col_cta + 64 * grp;
              tma_store_2d(&map_h, sg, cg, row_wg);
              tma_store_2d(&map_h, sg + GLN_RES_HALF, GLN_D + cg, row_wg);
              bulk_commit_group();
            }
            bulk_wait_group_read<0>();                   // the store has read the slab: the stage may be refilled
            GLN_STAMP(grp == GLN_GROUPS - 1, it, 1 + wg, 7);
            mbar_arrive_cnt(&empty_bar[rs], 4);
          }
        }
      }
      ring = ring.ahead(GLN_GROUPS);
    }
    if (store_thread) bulk_wait_group<0>();   // the last stores have landed before the CTA exits
  }

  // the peer may still be writing into this CTA's shared memory / signalling its barriers
  __syncwarp();
  cluster_sync_all();
}

}  // namespace b200
