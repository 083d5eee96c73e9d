// Self-attention core on warpgroup MMA (wgmma m64nNk16, fp16 operands, fp32 accumulation): one warpgroup per CTA, two
// CTAs per SM, each CTA walking query tiles of 64 rows of one (head, sample).  Every model has at most 256 keys, so a
// tile's whole score row (64 x KEYS fp32, KEYS / 2 registers per thread) stays in registers and the softmax takes one
// pass over the keys.
//   K, V of the (sample, head): all KEYS keys brought into shared memory by TMA (two 64-column atoms each, 128-byte
//                    swizzle, completion on one mbarrier for K and one for V); the per-sample 3-D tensor map has a box
//                    of exactly KEYS rows and zero-fills rows past the last token, so every row an MMA reads is either a
//                    token or zero (a masked P of 0 times stale NaN in V would be NaN)
//   Q                straight from global memory into registers, in the register-A fragment of wgmma (each element
//                    is used by exactly one thread)
//   S = Q K^T        wgmma.m64n{KEYS}k16, A = Q from registers, B = K from shared memory (K-major)
//   softmax          offset = exact row maximum over the valid keys (prefix key mask), p = exp2(s*scale - offset),
//                    row sum over the unrounded p in fp32, P rounded to fp16 in place: the accumulator fragment of
//                    16-bit values is the register-A fragment of the next wgmma
//   O += P V         wgmma.m64n128k16, A = P from registers, B = V from shared memory as stored ([key, dh], dh
//                    contiguous: an MN-major operand, read with the transpose bit -- no transpose pass), one k16 step per
//                    16-key block holding a valid key, in increasing key order
//   O / rowsum -> fp16 (WIDE: [hi | lo] pair with hi + lo = O to ~22 bits) -> global memory
// Every probability is computed once, against the row's true maximum (no online rescaling).
// (reference: nn.MultiheadAttention inside nn.TransformerEncoderLayer, built at model/mdm.py:77-84; the
//  key_padding_mask of model/mdm.py:241-247 is a prefix mask => per-sample valid-key count `kvlen`.)
#pragma once
#include <cuda_fp16.h>

#include "epilogues.cuh"
#include "ptx.cuh"

namespace b200 {

constexpr int ATC_THREADS = 128;         // one warpgroup
constexpr int ATC_QROWS = 64;            // query rows per tile (the M of one wgmma)
constexpr int ATC_TILES_PER_CTA = 4;     // query tiles each CTA walks (sharing one K / V load): all of them up to 256 tokens
constexpr int ATC_DH = 128;
constexpr int ATC_MAX_KEYS = 256;

// Key width the kernel is instantiated for: the smallest of 64 (DiP: 60 tokens, a2m: 61), 208 (HumanML3D: 197) and 256
// that holds round_up(S, 16).  The K / V tensor map's box height must be this width.
__host__ __device__ constexpr int atc_keys(int S) { return S <= 64 ? 64 : S <= 208 ? 208 : 256; }

struct AttnTcSmem {
  static __host__ __device__ int total(int keys) { return 1024 + 4 * keys * 128; }   // K and V: two [keys x 128 B] atoms each
};

// qkv : [n_samples * S, 3d] fp16 (q | k | v, head h at columns h * 128 of each)
// map_kv: the same tensor viewed [n_samples][S][3d], box {64, KEYS, 1}, SWIZZLE_128B
// out : [n_samples * S, kw * d] fp16; WIDE (kw = 2): [hi | lo]
// grid = (heads, n_samples, z): CTA z takes query tiles z, z + gridDim.z, ...; KEYS = atc_keys(S)
template <int KEYS, bool WIDE>
__global__ void __launch_bounds__(ATC_THREADS, 2)
attention_tc_kernel(const __grid_constant__ CUtensorMap map_kv, const __half* __restrict__ qkv, __half* __restrict__ out,
                    const int* __restrict__ kvlen, int S, int d, float scale_log2) {
  constexpr int ATOM = KEYS * 128;            // bytes of one 64-column atom (a multiple of 1024: KEYS % 8 == 0)
  constexpr int NS = KEYS / 2;                // score registers per thread
  constexpr int NB = KEYS / 16;               // 16-key blocks
  extern __shared__ uint8_t smem_raw[];
  __shared__ uint64_t bar_k, bar_v;
  uint8_t* sK = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* sV = sK + 2 * ATOM;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int h = blockIdx.x, smp = blockIdx.y;
  const int ld = 3 * d;
  const __half* base = qkv + static_cast<size_t>(smp) * S * ld;

  pdl_launch_dependents();
  if (threadIdx.x == 0) {
    tma_prefetch_desc(&map_kv);
    mbar_init(&bar_k, 1);
    mbar_init(&bar_v, 1);
    fence_barrier_init();
  }
  __syncthreads();
  pdl_wait();
  // ---- K and V by TMA (rows >= S are zero-filled, so masked probabilities never meet NaN garbage)
  if (threadIdx.x == 0) {
    mbar_expect_tx(&bar_k, 2 * ATOM);
    for (int a = 0; a < 2; ++a) tma_load_3d(sK + a * ATOM, &map_kv, &bar_k, d + h * ATC_DH + 64 * a, 0, smp);
    mbar_expect_tx(&bar_v, 2 * ATOM);
    for (int a = 0; a < 2; ++a) tma_load_3d(sV + a * ATOM, &map_kv, &bar_v, 2 * d + h * ATC_DH + 64 * a, 0, smp);
  }

  const int kvl = min(kvlen[smp], S);
  const int nblk = max(1, (kvl + 15) >> 4);          // 16-key blocks holding a valid key
  const int g = lane >> 2, t = lane & 3;
  // K: B of Q K^T, K-major; dh step ks (16 columns) lies in atom ks / 4 at byte 32 (ks % 4) of each swizzled row.
  // V: B of P V, MN-major; key block kk starts at row 16 kk (2048 B), the two dh atoms are ATOM bytes apart.
  const uint64_t desc_k = wgmma_desc_k_sw128(smem_u32(sK));
  const uint64_t desc_v = wgmma_desc_mn_sw128(smem_u32(sV), ATOM);
  const int ntiles = (S + ATC_QROWS - 1) / ATC_QROWS;
  const int ldo = (WIDE ? 2 : 1) * d;

  uint32_t qa[8][4];   // Q of this warp's 16 rows of a tile, register-A fragments of the 8 dh steps
  auto load_q = [&](int tile) {
    const int ra = tile * ATC_QROWS + warp * 16 + g, rb = ra + 8;
    const bool va = ra < S, vb = rb < S;
    const uint32_t* pa = reinterpret_cast<const uint32_t*>(base + static_cast<size_t>(va ? ra : 0) * ld + h * ATC_DH);
    const uint32_t* pb = reinterpret_cast<const uint32_t*>(base + static_cast<size_t>(vb ? rb : 0) * ld + h * ATC_DH);
#pragma unroll
    for (int ks = 0; ks < 8; ++ks) {
      qa[ks][0] = va ? pa[8 * ks + t] : 0u;
      qa[ks][1] = vb ? pb[8 * ks + t] : 0u;
      qa[ks][2] = va ? pa[8 * ks + 4 + t] : 0u;
      qa[ks][3] = vb ? pb[8 * ks + 4 + t] : 0u;
    }
  };
  if (static_cast<int>(blockIdx.z) < ntiles) load_q(blockIdx.z);
#pragma unroll 1
  for (int tile = blockIdx.z; tile < ntiles; tile += gridDim.z) {
    const int ra = tile * ATC_QROWS + warp * 16 + g, rb = ra + 8;   // this thread's two query rows
    const bool va = ra < S, vb = rb < S;
    // ---- S = Q K^T: s[4j + i] is row g + 8 (i / 2), key 8 j + 2 t + i % 2 of this warp's 16 rows
    float s[NS];
    mbar_wait(&bar_k, 0);
    wgmma_fence();
#pragma unroll
    for (int ks = 0; ks < 8; ++ks)
      WgmmaRA<KEYS, 0>::mma(s, qa[ks], desc_k + (((ks >> 2) * ATOM + (ks & 3) * 32) >> 4), ks != 0);
    wgmma_commit();
    wgmma_wait<0>();
    wgmma_fence_acc(s);
    // ---- row maxima over the valid keys
    float mxa = -INFINITY, mxb = -INFINITY;
#pragma unroll
    for (int j = 0; j < NS / 4; ++j)
#pragma unroll
      for (int i = 0; i < 2; ++i) {
        if (8 * j + 2 * t + i < kvl) {
          mxa = fmaxf(mxa, s[4 * j + i]);
          mxb = fmaxf(mxb, s[4 * j + 2 + i]);
        }
      }
#pragma unroll
    for (int o = 1; o < 4; o <<= 1) {
      mxa = fmaxf(mxa, __shfl_xor_sync(0xffffffffu, mxa, o));
      mxb = fmaxf(mxb, __shfl_xor_sync(0xffffffffu, mxb, o));
    }
    const float offa = (mxa == -INFINITY) ? 0.f : mxa * scale_log2;
    const float offb = (mxb == -INFINITY) ? 0.f : mxb * scale_log2;
    auto ex2 = [](float x) {
      float y;
      asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
      return y;
    };
    // ---- P (fp16, register-A fragment of key block kk: p[kk][0..3] = rows g, g+8 x keys 2t; rows g, g+8 x keys 8+2t)
    // and the row sums over the unrounded p, in key order, two keys at a time
    uint32_t p[NB][4];
    float suma = 0.f, sumb = 0.f;
#pragma unroll
    for (int j = 0; j < NS / 4; ++j) {
      const int key = 8 * j + 2 * t;
      const float p0 = key < kvl ? ex2(fmaf(s[4 * j], scale_log2, -offa)) : 0.f;
      const float p1 = key + 1 < kvl ? ex2(fmaf(s[4 * j + 1], scale_log2, -offa)) : 0.f;
      const float p2 = key < kvl ? ex2(fmaf(s[4 * j + 2], scale_log2, -offb)) : 0.f;
      const float p3 = key + 1 < kvl ? ex2(fmaf(s[4 * j + 3], scale_log2, -offb)) : 0.f;
      suma += p0 + p1;
      sumb += p2 + p3;
      p[j >> 1][2 * (j & 1)] = pack_half2(p0, p1);
      p[j >> 1][2 * (j & 1) + 1] = pack_half2(p2, p3);
    }
#pragma unroll
    for (int off = 1; off < 4; off <<= 1) {
      suma += __shfl_xor_sync(0xffffffffu, suma, off);
      sumb += __shfl_xor_sync(0xffffffffu, sumb, off);
    }
    const float inva = suma > 0.f ? 1.f / suma : 0.f;
    const float invb = sumb > 0.f ? 1.f / sumb : 0.f;
    // ---- O = P V over the blocks holding a valid key: o[4j + i] is row g + 8 (i / 2), dh column 8 j + 2 t + i % 2
    float o[64];
    mbar_wait(&bar_v, 0);
    wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < NB; ++kk)
      if (kk < nblk) WgmmaRA<128, 1>::mma(o, p[kk], desc_v + ((kk * 16 * 128) >> 4), kk != 0);
    wgmma_commit();
    // Q of the next tile loads while P V runs (qa is free once S is formed)
    if (tile + static_cast<int>(gridDim.z) < ntiles) load_q(tile + gridDim.z);
    wgmma_wait<0>();
    wgmma_fence_acc(o);
    // ---- O / rowsum -> fp16 (+ lo half)
    __half* oa = out + (static_cast<size_t>(smp) * S + (va ? ra : 0)) * ldo + h * ATC_DH + 2 * t;
    __half* ob = out + (static_cast<size_t>(smp) * S + (vb ? rb : 0)) * ldo + h * ATC_DH + 2 * t;
#pragma unroll
    for (int j = 0; j < 16; ++j) {
      const float x0 = o[4 * j] * inva, x1 = o[4 * j + 1] * inva, x2 = o[4 * j + 2] * invb, x3 = o[4 * j + 3] * invb;
      const __half2 ha = __floats2half2_rn(x0, x1), hb = __floats2half2_rn(x2, x3);
      if (va) *reinterpret_cast<__half2*>(oa + 8 * j) = ha;
      if (vb) *reinterpret_cast<__half2*>(ob + 8 * j) = hb;
      if (WIDE) {
        const float2 fa = __half22float2(ha), fb = __half22float2(hb);
        if (va) *reinterpret_cast<__half2*>(oa + d + 8 * j) = __floats2half2_rn(x0 - fa.x, x1 - fa.y);
        if (vb) *reinterpret_cast<__half2*>(ob + d + 8 * j) = __floats2half2_rn(x2 - fb.x, x3 - fb.y);
      }
    }
  }
}

}  // namespace b200
