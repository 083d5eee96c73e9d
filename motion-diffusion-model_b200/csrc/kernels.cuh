// Small HBM/L2-bound kernels around the GEMMs: input packing (transpose + fp16 hi/lo split), per-step
// conditioning token, LayerNorm rows, CFG blend of the hidden rows, weight repacking, table set-up.
#pragma once
#include <cuda_fp16.h>
#include <stdint.h>

#include "epilogues.cuh"

namespace b200 {

// ---------------------------------------------------------------------------------------------------------
// x [B, JF, T] fp32 (reference layout, T contiguous)  ->  xin16 [B*S, ld] fp16 rows (b, s = 1 + t_off + t):
//   columns [0,Kp) = hi, [Kp,2Kp) = lo, [2Kp,3Kp) = hi    (A' of the 3-pass split GEMM  A_hi*W_hi + A_lo*W_hi + A_hi*W_lo)
// Row s = 0 (conditioning token slot) and the pad columns stay zero from allocation time.
__global__ void pack_input_kernel(const float* __restrict__ x, __half* __restrict__ xin, int B, int JF, int T, int S,
                                  int Kp, int ld, int row_off) {
  pdl_launch_dependents();
  pdl_wait();
  __shared__ float tile[32][33];
  const int b = blockIdx.z;
  const int j0 = blockIdx.y * 32, t0 = blockIdx.x * 32;
  const int tx = threadIdx.x, ty = threadIdx.y;  // 32 x 8
  for (int i = ty; i < 32; i += 8) {
    const int j = j0 + i, t = t0 + tx;
    tile[i][tx] = (j < JF && t < T) ? x[(static_cast<size_t>(b) * JF + j) * T + t] : 0.f;
  }
  __syncthreads();
  for (int i = ty; i < 32; i += 8) {
    const int t = t0 + i, j = j0 + tx;
    if (t < T && j < JF) {
      const float v = tile[tx][i];
      const __half hi = __float2half_rn(v);
      const __half lo = __float2half_rn(v - __half2float(hi));
      __half* dst = xin + (static_cast<size_t>(b) * S + row_off + t) * ld + j;
      dst[0] = hi;
      dst[Kp] = lo;
      dst[2 * Kp] = hi;
    }
  }
}

// ---------------------------------------------------------------------------------------------------------
// Conditioning-token rows of the sequence (reference model/mdm.py:195,218-220,251-252):
//   h[b', s=0, :] = (condproj[b', :] + temb_table[t(b'), :]) + pe[0, :]
//   t(b') = tvec[b' % B] when tvec != nullptr (model called with explicit timesteps), else timestep_map[i] with
//   i = eval_index(state, back): the step in flight, or the one before it (PLMS improved Euler).  tvec is read through
//   L2: in slot mode slot_advance_kernel writes it inside the step graph (see load_step_state).
// With a target embedding g [B, d] (model/mdm.py:197-199, both CFG halves): (condproj + (temb + g[b' % B])) + pe[0].
// condproj == nullptr (the timestep token of trans_dec with emb_trans_dec, mdm.py:256): (temb + g) + pe[0], no text.
// Runs right after the embedding GEMM (which leaves placeholder values in these rows).
// The residual stream is an fp16 [hi | lo] pair per element (row = 2d halves, hi + lo carries ~22 bits).
__global__ void tok0_rows_kernel(__half* __restrict__ hres, const float* __restrict__ condproj,
                                 const float* __restrict__ temb_table, const float* __restrict__ pe,
                                 const int* __restrict__ tvec, const int* __restrict__ tmap,
                                 const StepState* __restrict__ state, const float* __restrict__ g, int B, int S, int d,
                                 int temb_rows, int back) {
  pdl_launch_dependents();
  pdl_wait();
  const int bp = blockIdx.x;
  int t = (tvec != nullptr) ? __ldcg(tvec + bp % B) : tmap[eval_index(load_step_state(state), back)];
  t = min(max(t, 0), temb_rows - 1);
  const size_t row = static_cast<size_t>(bp) * S;
  for (int c = threadIdx.x; c < d; c += blockDim.x) {
    float te = temb_table[static_cast<size_t>(t) * d + c];
    if (g != nullptr) te = te + g[static_cast<size_t>(bp % B) * d + c];
    const float v = (condproj != nullptr ? condproj[static_cast<size_t>(bp) * d + c] + te : te) + pe[c];
    const __half hi = __float2half_rn(v);
    hres[row * 2 * d + c] = hi;
    hres[row * 2 * d + d + c] = __float2half_rn(v - __half2float(hi));
  }
}

// pe_bias[s, c] = pe[s, c] + bias[c]  (per (B,T) workspace table for the embedding epilogue)
__global__ void pe_bias_kernel(float* __restrict__ out, const float* __restrict__ pe, const float* __restrict__ bias,
                               int S, int d) {
  const int s = blockIdx.x;
  for (int c = threadIdx.x; c < d; c += blockDim.x) out[static_cast<size_t>(s) * d + c] = bias[c] + pe[static_cast<size_t>(s) * d + c];
}

// dir = -1 walks the schedule down (sampling), +1 up (DDIM inversion: x at index i -> x at index i + 1).
__global__ void step_advance_kernel(StepState* state, int dir) {
  pdl_launch_dependents();
  pdl_wait();
  const StepState st = load_step_state(state);
  state->done = st.done + 1;
  state->cur = st.cur + dir;
}
__global__ void step_set_kernel(StepState* state, int done, int cur, const float* noise, long long noise_step_stride,
                                unsigned long long seed, long long sample_base, int n_steps) {
  state->done = done;
  state->cur = cur;
  state->n_steps = n_steps;
  state->noise = noise;
  state->noise_step_stride = noise_step_stride;
  state->seed = seed;
  state->sample_base = sample_base;
}

// Hand-off of an autoregressive chain (b200mdm_chain_loop_range) after the last step of a chunk: the final sample
// x [B, JF, T] goes to frames off .. off + T - 1 of the chain output out [B, JF, crop] (frames at or past crop are
// dropped) and, unless prefix is null (the last chunk), its last ctx frames to prefix [B, JF, ctx], which
// pack_input_kernel then packs into the embedding GEMM's A operand exactly as b200mdm_set_prefix packs y['prefix'].
// A copy: every value is moved, none is computed.
__global__ void chain_handoff_kernel(const float* __restrict__ x, float* __restrict__ out, float* __restrict__ prefix,
                                     long long rows, int T, int ctx, int off, int crop) {
  const long long n = rows * T;
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < n;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const long long row = i / T;
    const int t = static_cast<int>(i - row * T);
    const float v = x[i];
    if (off + t < crop) out[row * crop + off + t] = v;
    if (prefix != nullptr && t >= T - ctx) prefix[row * ctx + t - (T - ctx)] = v;
  }
}

// ---------------------------------------------------------------------------------------------------------
// The engine's own noise stream (B200MDM_FLAG_PHILOX_NOISE / b200mdm_philox_normal): replaces the reference's
// th.randn_like(x) per step (diffusion/gaussian_diffusion.py:525, :770) when the caller asks for a stream that does not
// depend on how the batch is split over GPUs or on how many steps are drawn at once.
//   Philox4x32-10 (Salmon et al., SC'11), key = (seed_lo, seed_hi),
//   counter = (q, step_id, g_lo, g_hi ^ 0x4d444d42)   q = element index / 4 inside the sample, g = global sample index
//   the 4 output words w0..w3 -> u_k = ((w_k >> 8) + 0.5) * 2^-24 in (0, 1);
//   elements 4q..4q+3 = r0 cos(2 pi u1), r0 sin(2 pi u1), r1 cos(2 pi u3), r1 sin(2 pi u3),  r0 = sqrt(-2 ln u0), r1 = sqrt(-2 ln u2)
// step_id = schedule index of the step that consumes the eps (state->cur when `state` != nullptr); x_T uses 0xffffffff.
__device__ __forceinline__ void philox4x32_10(uint32_t (&c)[4], uint32_t k0, uint32_t k1) {
#pragma unroll
  for (int r = 0; r < 10; ++r) {
    const uint32_t hi0 = __umulhi(0xD2511F53u, c[0]), lo0 = 0xD2511F53u * c[0];
    const uint32_t hi1 = __umulhi(0xCD9E8D57u, c[2]), lo1 = 0xCD9E8D57u * c[2];
    const uint32_t n0 = hi1 ^ c[1] ^ k0, n2 = hi0 ^ c[3] ^ k1;
    c[0] = n0; c[1] = lo1; c[2] = n2; c[3] = lo0;
    k0 += 0x9E3779B9u;
    k1 += 0xBB67AE85u;
  }
}
// Elements 4q .. 4q + 3 of one sample's eps (out: the sample's n elements), keyed by (seed, step_id, g).
__device__ __forceinline__ void philox_quad(float* out, long long n, long long q, unsigned long long seed,
                                            unsigned long long g, uint32_t step_id) {
  uint32_t c[4] = {static_cast<uint32_t>(q), step_id, static_cast<uint32_t>(g), static_cast<uint32_t>(g >> 32) ^ 0x4d444d42u};
  philox4x32_10(c, static_cast<uint32_t>(seed), static_cast<uint32_t>(seed >> 32));
  float z[4];
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const float u0 = (static_cast<float>(c[2 * h] >> 8) + 0.5f) * 5.9604644775390625e-08f;
    const float u1 = (static_cast<float>(c[2 * h + 1] >> 8) + 0.5f) * 5.9604644775390625e-08f;
    const float r = sqrtf(-2.0f * logf(u0));
    float sn, cs;
    sincospif(2.0f * u1, &sn, &cs);
    z[2 * h] = r * cs;
    z[2 * h + 1] = r * sn;
  }
  float* dst = out + 4 * q;
  if (4 * q + 3 < n && (reinterpret_cast<uintptr_t>(dst) & 15) == 0) {
    *reinterpret_cast<float4*>(dst) = make_float4(z[0], z[1], z[2], z[3]);
  } else {
#pragma unroll
    for (int j = 0; j < 4; ++j)
      if (4 * q + j < n) dst[j] = z[j];
  }
}
__global__ void philox_normal_kernel(float* __restrict__ out, int B, long long n, unsigned long long seed,
                                     long long sample_base, uint32_t step_id, const StepState* __restrict__ state) {
  pdl_launch_dependents();
  pdl_wait();
  if (state != nullptr) {
    const StepState st = load_step_state(state);
    seed = st.seed;
    sample_base = st.sample_base;
    step_id = static_cast<uint32_t>(st.cur);
  }
  const long long qn = (n + 3) / 4, total = qn * B;
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const long long b = i / qn, q = i - b * qn;
    philox_quad(out + b * n, n, q, seed, static_cast<unsigned long long>(sample_base + b), step_id);
  }
}

// philox_normal_kernel with every sample keyed by its own slot (seed, schedule index cur, global sample index g): the eps
// of each active slot's step, exactly as a uniform loop with noise_seed = seed draws it for sample g at index cur.
// Idle slots draw nothing.
__global__ void philox_slots_kernel(float* __restrict__ out, int B, long long n, const SlotState* slots) {
  pdl_launch_dependents();
  pdl_wait();
  const long long qn = (n + 3) / 4, total = qn * B;
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const long long b = i / qn, q = i - b * qn;
    const int cur = __ldcg(&slots[b].cur);
    if (cur < 0) continue;
    philox_quad(out + b * n, n, q, __ldcg(&slots[b].seed), static_cast<unsigned long long>(__ldcg(&slots[b].g)),
                static_cast<uint32_t>(cur));
  }
}

// ---------------------------------------------------------------------------------------------------------
// Continuous batching (b200mdm_slots_begin): every row of the workspace is a slot with its own schedule index.
// Every slot idle; tvec at a valid row for the idle forward, all keys valid, scale 0.
__global__ void slots_reset_kernel(SlotState* slots, int* tvec, int* kvlen, float* scale, int* action, const int* tmap, int B,
                                   int Bp, int S) {
  for (int b = blockIdx.x * blockDim.x + threadIdx.x; b < Bp; b += gridDim.x * blockDim.x) {
    kvlen[b] = S;
    if (b >= B) continue;
    slots[b].cur = -1;
    slots[b].seed = 0ull;
    slots[b].g = 0ll;
    tvec[b] = tmap[0];
    scale[b] = 0.f;
    if (action != nullptr) action[b] = 0;
  }
}
// Slot b's per-request scalars (b200mdm_slot_admit): its state at schedule index cur, the model timestep of its first
// step, its guidance scale and its valid-key count in each classifier-free half.  One thread.
__global__ void slot_admit_kernel(SlotState* slots, int* tvec, int* kvlen, float* scale, int* action, const int* tmap, int b,
                                  int B, int halves, int cur, unsigned long long seed, long long g, float sc, int kv,
                                  int act) {
  slots[b].cur = cur;
  slots[b].seed = seed;
  slots[b].g = g;
  tvec[b] = tmap[cur];
  scale[b] = sc;
  for (int h = 0; h < halves; ++h) kvlen[h * B + b] = kv;
  if (action != nullptr) action[b] = act;
}
// The last kernel of a slot step: every active slot moves one index down the schedule (after index 0 it is -1: done),
// and tvec takes the model timestep of its next step (idle slots: row 0, a valid row for the idle forward).
__global__ void slot_advance_kernel(SlotState* slots, int* tvec, const int* __restrict__ tmap, int B) {
  pdl_launch_dependents();
  pdl_wait();
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= B) return;
  int cur = __ldcg(&slots[b].cur);
  if (cur >= 0) slots[b].cur = --cur;
  tvec[b] = tmap[cur > 0 ? cur : 0];
}
// b200mdm_sample_step_at: slot b at schedule index tvec[b] (the caller's indices, uploaded there), tvec[b] <- its model
// timestep.  Noise comes from the caller, so no Philox key is set.
__global__ void slots_from_index_kernel(SlotState* slots, int* tvec, const int* __restrict__ tmap, int B) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= B) return;
  const int cur = tvec[b];
  slots[b].cur = cur;
  tvec[b] = tmap[cur];
}
// A token-memory slot session (b200mdm_chain_slot_admit / _handoff): slot b's padding mask [Mt] (1 = padding) into its
// row of every classifier-free half -- the rows pack_text_mask gives sample b with one prompt.  One block.
__global__ void slot_mask_kernel(unsigned char* __restrict__ memmask, const uint8_t* __restrict__ mask, int b, int B,
                                 int halves, int Mt) {
  for (int m = threadIdx.x; m < Mt; m += blockDim.x) {
    const unsigned char pad = mask[m] ? 1 : 0;
    for (int h = 0; h < halves; ++h) memmask[(static_cast<size_t>(h) * B + b) * Mt + m] = pad;
  }
}

// ---------------------------------------------------------------------------------------------------------
// CFG blend on the hidden rows + fp16 hi/lo split for the 3-pass output GEMM.
//   v = h_u + scale[b] * (h_c - h_u)   (same expression as utils/sampler_util.py:34, applied before the linear
//   OutputProcess: W(h_u + s(h_c-h_u)) + b == out_u + s(out_c - out_u) exactly in real arithmetic)
//   halves == 1: v = h.       g16 row layout: [hi | lo | hi], ld = 3*d.
// Handshakes between chained windows (hs != nullptr; layout HS_* below): window b continues window p = b - 1 when
// hs[HS_CHAIN(b)] != 0; handshake position j = 0 .. h-1 pairs frame n_p - h + j of p with frame j of b, and both rows
// receive H_j = (1 - a_j) v_p + a_j v_b with a_j = (j + 1) / (h + 1), each v the CFG blend of its own window (its own
// scale).  OutputProcess is linear per frame and the weights sum to 1, so this is the blend of the two x0 rows.  The two
// copies of a handshake frame evaluate the same expression on the same operands in the same order: identical g16 rows.
#define HS_H 0
#define HS_LEN(b) (1 + 2 * (b))
#define HS_CHAIN(b) (2 + 2 * (b))
__device__ __forceinline__ float2 cfg_blend_pair(const __half* hc, const __half* hu, float sc, int d, int c, bool guided) {
  const float2 ah = __half22float2(*reinterpret_cast<const __half2*>(hc + c));
  const float2 al = __half22float2(*reinterpret_cast<const __half2*>(hc + d + c));
  float2 a = make_float2(ah.x + al.x, ah.y + al.y);
  if (guided) {
    const float2 uh = __half22float2(*reinterpret_cast<const __half2*>(hu + c));
    const float2 ul = __half22float2(*reinterpret_cast<const __half2*>(hu + d + c));
    const float2 u = make_float2(uh.x + ul.x, uh.y + ul.y);
    a.x = __fadd_rn(u.x, __fmul_rn(sc, __fsub_rn(a.x, u.x)));
    a.y = __fadd_rn(u.y, __fmul_rn(sc, __fsub_rn(a.y, u.y)));
  }
  return a;
}
__global__ void blend_split_kernel(const __half* __restrict__ hres, __half* __restrict__ g16,
                                   const float* __restrict__ scale, int B, int S, int T, int s_off, int d, int halves,
                                   const int* __restrict__ hs) {
  pdl_launch_dependents();
  pdl_wait();
  // one warp per FRAME row: the rows s < s_off of a sequence (condition token / DiP prefix) never reach x, so g16
  // holds B*T rows only (12544 = 98 row tiles of 128 at B=64, T=196): the output GEMM computes no token-0 / prefix rows
  const int orow = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (orow >= B * T) return;
  const int b = orow / T;
  const int f = orow - b * T;
  // handshake: (earlier window wa, its frame fa) and (later window wb, its frame fb), weight a of the later one
  int wa = -1, fa = 0, wb = 0, fb = 0;
  float alpha = 0.f;
  if (hs != nullptr) {
    const int h = hs[HS_H];
    const int nb = hs[HS_LEN(b)];
    if (f < h && hs[HS_CHAIN(b)]) {                                      // prefix of b: partner is p's suffix
      wa = b - 1; fa = hs[HS_LEN(b - 1)] - h + f; wb = b; fb = f;
    } else if (b + 1 < B && hs[HS_CHAIN(b + 1)] && f >= nb - h && f < nb) {   // suffix of b: partner is b+1's prefix
      wa = b; fa = f; wb = b + 1; fb = f - (nb - h);
    }
    if (wa >= 0) alpha = __fdiv_rn(static_cast<float>(fb + 1), static_cast<float>(h + 1));
  }
  const bool guided = halves == 2;
  __half* dst = g16 + static_cast<size_t>(orow) * 3 * d;
  if (wa >= 0) {
    const int ra = wa * S + s_off + fa, rb = wb * S + s_off + fb;
    const __half *hca = hres + static_cast<size_t>(ra) * 2 * d, *hua = hres + (static_cast<size_t>(B) * S + ra) * 2 * d;
    const __half *hcb = hres + static_cast<size_t>(rb) * 2 * d, *hub = hres + (static_cast<size_t>(B) * S + rb) * 2 * d;
    const float sa = guided ? scale[wa] : 0.f, sb = guided ? scale[wb] : 0.f;
    const float beta = __fsub_rn(1.f, alpha);
    for (int c = lane * 2; c < d; c += 64) {
      const float2 va = cfg_blend_pair(hca, hua, sa, d, c, guided);
      const float2 vb = cfg_blend_pair(hcb, hub, sb, d, c, guided);
      const float2 a = make_float2(__fadd_rn(__fmul_rn(beta, va.x), __fmul_rn(alpha, vb.x)),
                                   __fadd_rn(__fmul_rn(beta, va.y), __fmul_rn(alpha, vb.y)));
      const __half2 hi = __floats2half2_rn(a.x, a.y);
      const float2 hif = __half22float2(hi);
      const __half2 lo = __floats2half2_rn(a.x - hif.x, a.y - hif.y);
      *reinterpret_cast<__half2*>(dst + c) = hi;
      *reinterpret_cast<__half2*>(dst + d + c) = lo;
      *reinterpret_cast<__half2*>(dst + 2 * d + c) = hi;
    }
    return;
  }
  const int row = b * S + s_off + f;
  const __half* hc = hres + static_cast<size_t>(row) * 2 * d;                         // [hi | lo] rows
  const __half* hu = hres + (static_cast<size_t>(B) * S + row) * 2 * d;
  const float sc = guided ? scale[b] : 0.f;
  for (int c = lane * 2; c < d; c += 64) {
    const float2 a = cfg_blend_pair(hc, hu, sc, d, c, guided);
    const __half2 hi = __floats2half2_rn(a.x, a.y);
    const float2 hif = __half22float2(hi);
    const __half2 lo = __floats2half2_rn(a.x - hif.x, a.y - hif.y);
    *reinterpret_cast<__half2*>(dst + c) = hi;
    *reinterpret_cast<__half2*>(dst + d + c) = lo;
    *reinterpret_cast<__half2*>(dst + 2 * d + c) = hi;
  }
}

// ---------------------------------------------------------------------------------------------------------
// Weight repacking (one-time, at load).
__global__ void f32_to_f16_kernel(const float* __restrict__ src, __half* __restrict__ dst, size_t n) {
  for (size_t i = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x; i < n;
       i += static_cast<size_t>(gridDim.x) * blockDim.x)
    dst[i] = __float2half_rn(src[i]);
}
// W [N, K] fp32 -> [W16 | W16] fp16 [N, 2K]: partner of activations stored as [hi | lo] along K (the trans_dec engine keeps
// its fp16 activations to ~22 mantissa bits this way; the product A_hi W + A_lo W accumulates in fp32 on the tensor core).
__global__ void f32_to_f16_dup_kernel(const float* __restrict__ src, __half* __restrict__ dst, int N, int K) {
  const size_t n = static_cast<size_t>(N) * K;
  for (size_t i = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x; i < n;
       i += static_cast<size_t>(gridDim.x) * blockDim.x) {
    const size_t r = i / K, k = i % K;
    const __half h = __float2half_rn(src[i]);
    dst[r * 2 * K + k] = h;
    dst[r * 2 * K + K + k] = h;
  }
}
// W [N, K] fp32 -> W' [Npad, 3*Kp] fp16 = [hi | hi | lo] (zero padding), partner of the [hi | lo | hi] activations.
__global__ void split_weight_kernel(const float* __restrict__ w, __half* __restrict__ out, int N, int K, int Kp) {
  const int n = blockIdx.x;
  for (int k = threadIdx.x; k < K; k += blockDim.x) {
    const float v = w[static_cast<size_t>(n) * K + k];
    const __half hi = __float2half_rn(v);
    const __half lo = __float2half_rn(v - __half2float(hi));
    __half* dst = out + static_cast<size_t>(n) * 3 * Kp + k;
    dst[0] = hi;
    dst[Kp] = hi;
    dst[2 * Kp] = lo;
  }
}

// y[r, c] = act( sum_k x[r, k] * w[c, k] + b[c] ), fp32, one warp per output element (tiny set-up GEMVs:
// timestep-embedding MLP for every model timestep, text projection once per loop)
template <int ACT>  // 0 none, 1 SiLU
__global__ void small_linear_kernel(const float* __restrict__ x, const float* __restrict__ w,
                                    const float* __restrict__ b, float* __restrict__ y, int R, int C, int K,
                                    int x_ld) {
  const size_t widx = (blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (widx >= static_cast<size_t>(R) * C) return;
  const int r = static_cast<int>(widx / C), c = static_cast<int>(widx % C);
  const float* xr = x + static_cast<size_t>(r) * x_ld;
  const float* wr = w + static_cast<size_t>(c) * K;
  float acc = 0.f;
  for (int k = lane; k < K; k += 32) acc = fmaf(xr[k], wr[k], acc);
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
  if (lane == 0) {
    acc += (b != nullptr) ? b[c] : 0.f;
    if (ACT == 1) acc = acc / (1.f + expf(-acc));
    y[static_cast<size_t>(r) * C + c] = acc;
  }
}

// Target-location encoder g[b, :] = embed_target_cond(target[b], valid[b]) (model/mdm.py:399-480), fp32, once per loop.
// The three encoders share one packed weight layout of G groups of width dj:
//   w0 [G][dj][in_dim], b0 [G][dj]: the first Linear; wk [layers][G][dj][dj], bk [layers][G][dj]: [SiLU, Linear] x layers
//   single (EmbedTargetLocSingle): G = 1, dj = d, in_dim = 4 n: one MLP on cat(target, valid) [4 n]
//   split  (EmbedTargetLocSplit) : G = n, dj = d / n, in_dim = 4: joint i's mini-MLP on (x, y, z, valid_i) writes
//                                  columns [i dj, (i+1) dj)
//   multi  (EmbedTargetLocMulti) : G = n, dj = d, in_dim = 3, layers = 1: joint i's MLP on (x, y, z), for valid joints
//                                  only (an invalid joint's row is zero), rows combined by WeightedSum:
//                                  g = sum_i (wsum[i] / sum(wsum)) row_i   (utils/misc.py:5-16)
// target [B, n, 3], valid [B, n] (1.0 / 0.0).  One CTA per sample, blockDim.x == d; dynamic shared memory (4 n + 2 d) floats.
__global__ void __launch_bounds__(512) target_embed_kernel(const float* __restrict__ target, const float* __restrict__ valid,
                                                           const float* __restrict__ w0, const float* __restrict__ b0,
                                                           const float* __restrict__ wk, const float* __restrict__ bk,
                                                           const float* __restrict__ wsum, float* __restrict__ g, int n,
                                                           int G, int dj, int in_dim, int layers, int multi) {
  extern __shared__ float tsm[];
  const int d = blockDim.x, b = blockIdx.x, c = threadIdx.x;
  float* x = tsm;          // [n][4] = (x, y, z, valid) of this sample
  float* s = x + 4 * n;    // SiLU of the hidden layer
  float* o = s + d;        // next hidden layer
  for (int k = c; k < 4 * n; k += d) {
    const int j = k >> 2, q = k & 3;
    x[k] = q < 3 ? target[(static_cast<size_t>(b) * n + j) * 3 + q] : valid[static_cast<size_t>(b) * n + j];
  }
  __syncthreads();
  float wtot = 0.f;
  if (multi)
    for (int i = 0; i < G; ++i) wtot += wsum[i];
  const int warp = c >> 5, lane = c & 31, nwarp = d >> 5;
  float acc = 0.f;
  for (int p = 0; p < (multi ? G : 1); ++p) {
    if (multi && x[4 * p + 3] == 0.f) continue;   // (uniform over the CTA)
    const int grp = multi ? p : c / dj, cl = multi ? c : c % dj;
    const float* xi = x + 4 * grp;
    const float* wr = w0 + (static_cast<size_t>(grp) * dj + cl) * in_dim;
    float h = 0.f;
    for (int k = 0; k < in_dim; ++k) h = fmaf(wr[k], xi[k], h);
    h += b0[grp * dj + cl];
    for (int l = 0; l < layers; ++l) {
      s[c] = h / (1.f + expf(-h));
      __syncthreads();
      // one warp per output q, reading its weight row contiguously
      for (int q = warp; q < d; q += nwarp) {
        const int gq = multi ? p : q / dj, ql = multi ? q : q % dj;
        const float* wq = wk + ((static_cast<size_t>(l) * G + gq) * dj + ql) * dj;
        const float* sq = s + (multi ? 0 : gq * dj);
        float a = 0.f;
        for (int k = lane; k < dj; k += 32) a = fmaf(wq[k], sq[k], a);
#pragma unroll
        for (int off = 16; off > 0; off >>= 1) a += __shfl_xor_sync(0xffffffffu, a, off);
        if (lane == 0) o[q] = a + bk[(static_cast<size_t>(l) * G + gq) * dj + ql];
      }
      __syncthreads();
      h = o[c];
    }
    acc = multi ? fmaf(wsum[p] / wtot, h, acc) : h;
  }
  g[static_cast<size_t>(b) * d + c] = acc;
}

// condproj rows for the packed batch: first B rows conditional, next B rows unconditional.
//   text  : cond = (W clip + b) already in proj[B, d];  uncond = bias          (mask_cond zeros => bias only)
//   action: cond = action_embedding[a[b]];              uncond = 0             (model/mdm.py:225-227)
//   none  : 0
__global__ void condproj_fill_kernel(float* __restrict__ condproj, const float* __restrict__ proj,
                                     const float* __restrict__ bias, const float* __restrict__ action_emb,
                                     const int* __restrict__ action, int B, int d, int rows, int first_uncond,
                                     int cond_mode) {
  const int bp = blockIdx.x;
  if (bp >= rows) return;
  const bool unc = first_uncond ? true : (bp >= B);
  const int b = bp % B;
  for (int c = threadIdx.x; c < d; c += blockDim.x) {
    float v = 0.f;
    if (cond_mode == 1) v = unc ? bias[c] : proj[static_cast<size_t>(b) * d + c];
    else if (cond_mode == 2) v = unc ? 0.f : action_emb[static_cast<size_t>(action[b]) * d + c];
    condproj[static_cast<size_t>(bp) * d + c] = v;
  }
}

// x_t = sqrt_ac * x0 + sqrt_1mac * noise   (q_sample, diffusion/gaussian_diffusion.py:226-244)
__global__ void q_sample_kernel(float* __restrict__ out, const float* __restrict__ x0, const float* __restrict__ noise,
                                float a, float b, size_t n) {
  for (size_t i = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x; i < n;
       i += static_cast<size_t>(gridDim.x) * blockDim.x) {
    const float s = (x0 != nullptr) ? x0[i] : 0.f;
    out[i] = __fadd_rn(__fmul_rn(a, s), __fmul_rn(b, noise[i]));
  }
}

// ---------------------------------------------------------------------------------------------------------
// The variational-bound loop (b200mdm_vb_loop_range).  Per step: vb_xt_kernel, the forward with the EpiOut<OutVb>
// epilogue, vb_reduce_kernel; after the last step, vb_final_kernel.
constexpr int VB_REDUCE_THREADS = 256;

// x_t = sqrt_ac[i] * x_start + sqrt_1mac[i] * eps at the step's schedule index (q_sample, gaussian_diffusion.py:226-244)
// eps: `noise` (one step, [B, n]) or the tape the step state describes
__global__ void vb_xt_kernel(float* __restrict__ x_t, const float* __restrict__ x_start, const float* noise,
                             const float* __restrict__ sched_vb, const StepState* __restrict__ state, size_t n) {
  pdl_launch_dependents();
  pdl_wait();
  const StepState st = load_step_state(state);
  const float* r = sched_vb + static_cast<size_t>(st.cur) * SCHED_VB_STRIDE;
  const float a = r[VB_SQ], b = r[VB_SQM1];
  const float* nz = noise != nullptr ? noise : st.noise + static_cast<long long>(st.done) * st.noise_step_stride;
  for (size_t i = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x; i < n; i += static_cast<size_t>(gridDim.x) * blockDim.x)
    x_t[i] = __fadd_rn(__fmul_rn(a, x_start[i]), __fmul_rn(b, nz[i]));
}

// Deterministic block sum of v[0 .. n): thread k adds v[k], v[k + 256], ... in that order, then a fixed shared-memory
// tree (stride 128, 64, ..., 1).  The result is in sh[0] after the call; every thread must call it.
__device__ __forceinline__ float vb_block_sum(float acc, float* sh) {
  sh[threadIdx.x] = acc;
  __syncthreads();
#pragma unroll
  for (int s = VB_REDUCE_THREADS / 2; s > 0; s >>= 1) {
    if (static_cast<int>(threadIdx.x) < s) sh[threadIdx.x] = __fadd_rn(sh[threadIdx.x], sh[threadIdx.x + s]);
    __syncthreads();
  }
  return sh[0];
}

// terms[k, b, n_steps - 1 - cur] = mean over the sample's J*T elements of term k (the sample's T*chunks partial sums, in
// the order of vb_block_sum), the vb term divided by log(2) (mean_flat(.) / np.log(2.0)).  grid (B, VB_TERMS).
__global__ void __launch_bounds__(VB_REDUCE_THREADS) vb_reduce_kernel(float* __restrict__ terms, int ld_terms,
                                                                     const float* __restrict__ part, int B, int per_sample,
                                                                     float count, const StepState* __restrict__ state) {
  __shared__ float sh[VB_REDUCE_THREADS];
  pdl_launch_dependents();
  pdl_wait();
  const int b = blockIdx.x, k = blockIdx.y;
  const float* v = part + (static_cast<size_t>(k) * B + b) * per_sample;
  float acc = 0.f;
  for (int i = threadIdx.x; i < per_sample; i += VB_REDUCE_THREADS) acc = __fadd_rn(acc, v[i]);
  const float sum = vb_block_sum(acc, sh);
  if (threadIdx.x == 0) {
    float m = __fdiv_rn(sum, count);
    if (k == 0) m = __fdiv_rn(m, 0.6931471805599453f);
    const StepState st = load_step_state(state);
    terms[(static_cast<size_t>(k) * B + b) * ld_terms + (st.n_steps - 1 - st.cur)] = m;
  }
}

// _prior_bpd and total_bpd (gaussian_diffusion.py:1527-1542, 1593): bpd[b] = sum_c vb[b, c] (c = 0 .. n - 1 in order) +
// prior[b], bpd[B + b] = prior[b] = mean(0.5 * (prior_c + (sqrt_ac * x_start)^2)) / log(2) with row n - 1 of the table.
// grid B.
__global__ void __launch_bounds__(VB_REDUCE_THREADS) vb_final_kernel(float* __restrict__ bpd, const float* __restrict__ terms,
                                                                    int ld_terms, const float* __restrict__ x_start,
                                                                    const float* __restrict__ sched_vb, int n_steps, int B,
                                                                    int per_sample) {
  __shared__ float sh[VB_REDUCE_THREADS];
  const int b = blockIdx.x;
  const float* r = sched_vb + static_cast<size_t>(n_steps - 1) * SCHED_VB_STRIDE;
  const float sq = r[VB_SQ], pc = r[VB_PRIOR_C];
  const float* xs = x_start + static_cast<size_t>(b) * per_sample;
  float acc = 0.f;
  for (int i = threadIdx.x; i < per_sample; i += VB_REDUCE_THREADS) {
    const float m = __fmul_rn(sq, xs[i]);
    acc = __fadd_rn(acc, __fmul_rn(0.5f, __fadd_rn(pc, __fmul_rn(m, m))));
  }
  const float sum = vb_block_sum(acc, sh);
  if (threadIdx.x == 0) {
    const float prior = __fdiv_rn(__fdiv_rn(sum, static_cast<float>(per_sample)), 0.6931471805599453f);
    const float* vb = terms + static_cast<size_t>(b) * ld_terms;
    float tot = 0.f;
    for (int c = 0; c < n_steps; ++c) tot = __fadd_rn(tot, vb[c]);
    bpd[b] = __fadd_rn(tot, prior);
    bpd[B + b] = prior;
  }
}

}  // namespace b200

// ===================================================================================================================
// trans_dec (DiP) helpers -- reference model/mdm.py:255-270 and torch nn.TransformerDecoderLayer cross-attention
namespace b200 {

// mem16[b', m, :] = [hi | lo] fp16 of ( memproj[b', m, :] + temb_table[t(b'), :] )   (emb = text_emb + time_emb,
// mdm.py:218-220; the time embedding is broadcast over the text tokens).  Rows are 2d wide.  grid = (Mt, Bp)
// With a target embedding g [B, d] (mdm.py:197-199, both CFG halves): memproj + (temb + g[b' % B]).
__global__ void mem_build_kernel(__half* __restrict__ mem16, const float* __restrict__ memproj,
                                 const float* __restrict__ temb_table, const int* __restrict__ tvec,
                                 const int* __restrict__ tmap, const StepState* __restrict__ state,
                                 const float* __restrict__ g, int B, int Mt, int d, int temb_rows, int back) {
  pdl_launch_dependents();
  pdl_wait();
  const int m = blockIdx.x, bp = blockIdx.y;
  int t = (tvec != nullptr) ? __ldcg(tvec + bp % B) : tmap[eval_index(load_step_state(state), back)];
  t = min(max(t, 0), temb_rows - 1);
  const size_t row = static_cast<size_t>(bp) * Mt + m;
  for (int c = threadIdx.x; c < d; c += blockDim.x) {
    float te = temb_table[static_cast<size_t>(t) * d + c];
    if (g != nullptr) te = te + g[static_cast<size_t>(bp % B) * d + c];
    const float v = memproj[row * d + c] + te;
    const __half hi = __float2half_rn(v);
    mem16[row * 2 * d + c] = hi;
    mem16[row * 2 * d + d + c] = __float2half_rn(v - __half2float(hi));
  }
}

// memproj rows of the packed batch (build_text_memory in engine.cu): the first cond_rows rows (K * B prompt rows, group-
// major as the packed batch; 0 when every row is unconditional) are W tokens + b (proj [cond_rows*Mt, d], rows
// (k*B + b, m)), the unconditional rows b.  grid = (Mt, Bp)
__global__ void memproj_group_fill_kernel(float* __restrict__ memproj, const float* __restrict__ proj,
                                          const float* __restrict__ bias, int cond_rows, int Mt, int d) {
  const int m = blockIdx.x, bp = blockIdx.y;
  const size_t row = static_cast<size_t>(bp) * Mt + m;
  for (int c = threadIdx.x; c < d; c += blockDim.x) memproj[row * d + c] = bp < cond_rows ? proj[row * d + c] : bias[c];
}

// enc_text [Mt, B, C] (reference layout, model/mdm.py:185) -> [B*Mt, C] rows (b, m) so that one small GEMM projects it
__global__ void permute_mbc_kernel(const float* __restrict__ src, float* __restrict__ dst, int Mt, int B, int C) {
  const int m = blockIdx.x, b = blockIdx.y;
  for (int c = threadIdx.x; c < C; c += blockDim.x)
    dst[(static_cast<size_t>(b) * Mt + m) * C + c] = src[(static_cast<size_t>(m) * B + b) * C + c];
}

// ---------------------------------------------------------------------------------------------------------
// trans_dec with a CLIP memory and the timestep token (emb_trans_dec, model/mdm.py:256-264).  The memory is ONE token
// per sample, m[b'] = textproj[b'] + (temb[t] + g[b]), without a mask: the softmax over a single key is exactly 1, so
// each layer's cross-attention block returns the same row for every query of the sample,
//   c_l[b'] = W_o,l (W_v,l m[b'] + b_v,l) + b_o,l .
// It is linear in m, so it splits into a per-sample part and a per-timestep part, both in fp32:
//   cb_l[b'] = W_o,l (W_v,l (textproj[b'] + g[b]) + b_v,l) + b_o,l   once per loop (set_cond_dec / set_target)
//   ct_l[t]  = W_o,l (W_v,l temb[t])                                  once per weight load, every model timestep
// and the step only adds them (cross_rows_kernel).  Against the reference's order this moves the fp32 rounding of the
// two GEMVs, a few ulp of each dot product (tests/test_dec_emb_gpu.py bounds it against fp64).

// mb[b', :] = textproj[b', :] + g[b' % B, :] (g == nullptr: textproj), the per-sample part of the memory row.
__global__ void cross_mem_kernel(float* __restrict__ mb, const float* __restrict__ textproj, const float* __restrict__ g,
                                 int B, int d) {
  const int bp = blockIdx.x;
  for (int c = threadIdx.x; c < d; c += blockDim.x) {
    const float p = textproj[static_cast<size_t>(bp) * d + c];
    mb[static_cast<size_t>(bp) * d + c] = g != nullptr ? p + g[static_cast<size_t>(bp % B) * d + c] : p;
  }
}

// c[l, b', :] = cb[l, b', :] + ct[l, t(b'), :]   (t as in tok0_rows_kernel).  grid = (Bp, L)
__global__ void cross_rows_kernel(float* __restrict__ c, const float* __restrict__ cb, const float* __restrict__ ct,
                                  const int* __restrict__ tvec, const int* __restrict__ tmap,
                                  const StepState* __restrict__ state, int B, int Bp, int d, int temb_rows, int back) {
  pdl_launch_dependents();
  pdl_wait();
  const int bp = blockIdx.x, l = blockIdx.y;
  int t = (tvec != nullptr) ? __ldcg(tvec + bp % B) : tmap[eval_index(load_step_state(state), back)];
  t = min(max(t, 0), temb_rows - 1);
  const size_t row = (static_cast<size_t>(l) * Bp + bp) * d, trow = (static_cast<size_t>(l) * temb_rows + t) * d;
  for (int i = threadIdx.x; i < d / 4; i += blockDim.x) {
    const float4 a = reinterpret_cast<const float4*>(cb + row)[i], b = reinterpret_cast<const float4*>(ct + trow)[i];
    reinterpret_cast<float4*>(c + row)[i] = make_float4(a.x + b.x, a.y + b.y, a.z + b.z, a.w + b.w);
  }
}

// h[r] <- LayerNorm(h[r] + c[r / S]; gamma, beta, eps) in place on the residual stream fp16 [M, 2 RBLN_D] = [hi | lo]
// (norm2 of the decoder layer with the cross-attention row c_l of the sample).  One warp per row; lane j holds columns
// [8j, 8j + 8) and [256 + 8j, 256 + 8j + 8) of both halves in 16-byte loads.  v = (hi + lo) + c in fp32; the mean and
// then the variance Σ(v - mean)² / d are two passes over the registers (no mean² cancellation);
// y = (v - mean) rstd gamma + beta, written back as hi = fp16(y), lo = fp16(y - hi).
constexpr int RBLN_D = 512;
constexpr int RBLN_ROWS_PER_CTA = 8;
__global__ void __launch_bounds__(32 * RBLN_ROWS_PER_CTA) row_bias_ln_kernel(__half* __restrict__ hres,
                                                                            const float* __restrict__ c,
                                                                            const float* __restrict__ gamma,
                                                                            const float* __restrict__ beta, int M, int S,
                                                                            float eps) {
  pdl_launch_dependents();
  pdl_wait();
  const int lane = threadIdx.x & 31;
  const int r = blockIdx.x * RBLN_ROWS_PER_CTA + (threadIdx.x >> 5);
  if (r >= M) return;
  __half* hrow = hres + static_cast<size_t>(r) * 2 * RBLN_D;
  const float* crow = c + static_cast<size_t>(r / S) * RBLN_D;
  float v[16];
#pragma unroll
  for (int k = 0; k < 2; ++k) {
    const int col = k * (RBLN_D / 2) + 8 * lane;
    const uint4 hv = *reinterpret_cast<const uint4*>(hrow + col);
    const uint4 lv = *reinterpret_cast<const uint4*>(hrow + RBLN_D + col);
    const float4 c0 = *reinterpret_cast<const float4*>(crow + col), c1 = *reinterpret_cast<const float4*>(crow + col + 4);
    const __half2* h2 = reinterpret_cast<const __half2*>(&hv);
    const __half2* l2 = reinterpret_cast<const __half2*>(&lv);
    const float cc[8] = {c0.x, c0.y, c0.z, c0.w, c1.x, c1.y, c1.z, c1.w};
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const float2 a = __half22float2(h2[j]), b = __half22float2(l2[j]);
      v[8 * k + 2 * j] = (a.x + b.x) + cc[2 * j];
      v[8 * k + 2 * j + 1] = (a.y + b.y) + cc[2 * j + 1];
    }
  }
  float s = 0.f;
#pragma unroll
  for (int i = 0; i < 16; ++i) s += v[i];
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  const float mean = s * (1.f / RBLN_D);
  float q = 0.f;
#pragma unroll
  for (int i = 0; i < 16; ++i) {
    const float dv = v[i] - mean;
    q = fmaf(dv, dv, q);
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) q += __shfl_xor_sync(0xffffffffu, q, o);
  const float rstd = rsqrtf(q * (1.f / RBLN_D) + eps);
#pragma unroll
  for (int k = 0; k < 2; ++k) {
    const int col = k * (RBLN_D / 2) + 8 * lane;
    const float4 g0 = *reinterpret_cast<const float4*>(gamma + col), g1 = *reinterpret_cast<const float4*>(gamma + col + 4);
    const float4 b0 = *reinterpret_cast<const float4*>(beta + col), b1 = *reinterpret_cast<const float4*>(beta + col + 4);
    const float gg[8] = {g0.x, g0.y, g0.z, g0.w, g1.x, g1.y, g1.z, g1.w};
    const float bb[8] = {b0.x, b0.y, b0.z, b0.w, b1.x, b1.y, b1.z, b1.w};
    uint4 ho, lo;
    __half2* h2 = reinterpret_cast<__half2*>(&ho);
    __half2* l2 = reinterpret_cast<__half2*>(&lo);
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const float y0 = (v[8 * k + 2 * j] - mean) * rstd * gg[2 * j] + bb[2 * j];
      const float y1 = (v[8 * k + 2 * j + 1] - mean) * rstd * gg[2 * j + 1] + bb[2 * j + 1];
      h2[j] = __floats2half2_rn(y0, y1);
      const float2 hf = __half22float2(h2[j]);
      l2[j] = __floats2half2_rn(y0 - hf.x, y1 - hf.y);
    }
    *reinterpret_cast<uint4*>(hrow + col) = ho;
    *reinterpret_cast<uint4*>(hrow + RBLN_D + col) = lo;
  }
}

// Cross-attention core: softmax(q k^T / sqrt(128) + mask) v with a handful of memory tokens (Mt <= 64).
//   q16 [n_samples*S, d] (head h at columns h*128), kv16 rows (sample, token) of pitch ld_kv holding k | v (v at +d), mask
//   [n_samples, Mt] (1 = ignore), out16 [n_samples*S, 2d]: the hi half only (the output projection reads K = d).
// 60 query rows x 16 tokens x 128 per (sample, head): far too small for a 128-row GEMM tile and bound by the ~40 MB
// of q / kv / out traffic, so each warp runs one 16-row m16n8k16 tile straight from registers:
//   * q and k fragments are read from global memory as 64 contiguous bytes per thread -- a dot product does not care
//     about the order of its terms, so thread t of a quad owns columns [32t, 32t+32) of the row for BOTH operands;
//   * softmax on the accumulator fragment (row statistics across the quad with two shuffles), exp2 with the scale
//     folded in; P is fed back as the A operand of the P.V product in two fp16 terms (hi + lo) so that the
//     probabilities carry fp32-like precision like the CUDA-core kernel this replaces;
//   * V is staged transposed in shared memory (pitch padded by 8 halves: conflict-free 32-bit fragment loads).
// A fully masked row yields 0 (the reference's softmax would give NaN there; it never occurs with a CLS token).
// grid = (heads, n_samples), block = 128 (4 warps x 16 rows per pass)
__device__ __forceinline__ void mma_m16n8k16(float (&c)[4], uint32_t a0, uint32_t a1, uint32_t a2, uint32_t a3, uint32_t b0,
                                             uint32_t b1) {
  asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};\n"
               : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
               : "r"(a0), "r"(a1), "r"(a2), "r"(a3), "r"(b0), "r"(b1));
}

__device__ __forceinline__ uint32_t pack_half2_u32(float x, float y) {
  const __half2 h = __floats2half2_rn(x, y);
  return *reinterpret_cast<const uint32_t*>(&h);
}

template <int MAX_NT>   // key tiles of 8 tokens: Mt <= 8 * MAX_NT, MAX_NT even
__global__ void __launch_bounds__(128) cross_attention_kernel(const __half* __restrict__ q16, const __half* __restrict__ kv16,
                                                              const unsigned char* __restrict__ mask,
                                                              __half* __restrict__ out16, int S, int Mt, int d, int ld_kv,
                                                              float scale_log2) {
  pdl_launch_dependents();
  pdl_wait();
  constexpr int KEYS = 8 * MAX_NT, VS = KEYS + 8;
  __shared__ __align__(16) __half sVt[128 * VS];
  __shared__ float sBias[KEYS];
  const int h = blockIdx.x, smp = blockIdx.y;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, g = lane >> 2, t = lane & 3;
  const __half* kv = kv16 + static_cast<size_t>(smp) * Mt * ld_kv + h * 128;
  for (int i = threadIdx.x; i < KEYS * 16; i += 128) {
    const int m = i >> 4, ch = i & 15;
    uint4 v = make_uint4(0u, 0u, 0u, 0u);
    if (m < Mt) v = *reinterpret_cast<const uint4*>(kv + static_cast<size_t>(m) * ld_kv + d + ch * 8);
    const __half* hv = reinterpret_cast<const __half*>(&v);
#pragma unroll
    for (int j = 0; j < 8; ++j) sVt[(ch * 8 + j) * VS + m] = hv[j];
  }
  if (threadIdx.x < KEYS)
    sBias[threadIdx.x] = (threadIdx.x < Mt && !mask[static_cast<size_t>(smp) * Mt + threadIdx.x]) ? 0.f : -INFINITY;
  __syncthreads();

  for (int m0 = warp * 16; m0 < S; m0 += 64) {
    const int r0 = m0 + g, r1 = r0 + 8;
    const size_t row0 = static_cast<size_t>(smp) * S + min(r0, S - 1), row1 = static_cast<size_t>(smp) * S + min(r1, S - 1);
    uint32_t qa[16], qb[16];
    {
      const uint4* p0 = reinterpret_cast<const uint4*>(q16 + row0 * d + h * 128 + t * 32);
      const uint4* p1 = reinterpret_cast<const uint4*>(q16 + row1 * d + h * 128 + t * 32);
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const uint4 a = p0[i], b = p1[i];
        qa[4 * i] = a.x; qa[4 * i + 1] = a.y; qa[4 * i + 2] = a.z; qa[4 * i + 3] = a.w;
        qb[4 * i] = b.x; qb[4 * i + 1] = b.y; qb[4 * i + 2] = b.z; qb[4 * i + 3] = b.w;
      }
    }
    float sc[MAX_NT][4];
#pragma unroll
    for (int nt = 0; nt < MAX_NT; ++nt) {
      sc[nt][0] = sc[nt][1] = sc[nt][2] = sc[nt][3] = 0.f;
      const int key = min(nt * 8 + g, Mt - 1);                        // padded tokens are masked through sBias
      const uint4* kp = reinterpret_cast<const uint4*>(kv + static_cast<size_t>(key) * ld_kv + t * 32);
      uint32_t kw[16];
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const uint4 a = kp[i];
        kw[4 * i] = a.x; kw[4 * i + 1] = a.y; kw[4 * i + 2] = a.z; kw[4 * i + 3] = a.w;
      }
#pragma unroll
      for (int j = 0; j < 8; ++j) mma_m16n8k16(sc[nt], qa[2 * j], qb[2 * j], qa[2 * j + 1], qb[2 * j + 1], kw[2 * j], kw[2 * j + 1]);
    }
    // softmax over the tokens: thread holds tokens nt*8 + 2t, +1 of rows g (c0, c1) and g+8 (c2, c3)
    float mx0 = -INFINITY, mx1 = -INFINITY;
#pragma unroll
    for (int nt = 0; nt < MAX_NT; ++nt) {
      const float b0 = sBias[nt * 8 + 2 * t], b1 = sBias[nt * 8 + 2 * t + 1];
      sc[nt][0] = fmaf(sc[nt][0], scale_log2, b0); sc[nt][1] = fmaf(sc[nt][1], scale_log2, b1);
      sc[nt][2] = fmaf(sc[nt][2], scale_log2, b0); sc[nt][3] = fmaf(sc[nt][3], scale_log2, b1);
      mx0 = fmaxf(mx0, fmaxf(sc[nt][0], sc[nt][1]));
      mx1 = fmaxf(mx1, fmaxf(sc[nt][2], sc[nt][3]));
    }
    mx0 = fmaxf(mx0, __shfl_xor_sync(0xffffffffu, mx0, 1)); mx0 = fmaxf(mx0, __shfl_xor_sync(0xffffffffu, mx0, 2));
    mx1 = fmaxf(mx1, __shfl_xor_sync(0xffffffffu, mx1, 1)); mx1 = fmaxf(mx1, __shfl_xor_sync(0xffffffffu, mx1, 2));
    const float off0 = (mx0 == -INFINITY) ? 0.f : mx0, off1 = (mx1 == -INFINITY) ? 0.f : mx1;
    float sum0 = 0.f, sum1 = 0.f;
    uint32_t phi[MAX_NT][2], plo[MAX_NT][2];
#pragma unroll
    for (int nt = 0; nt < MAX_NT; ++nt) {
      const float p0 = exp2f(sc[nt][0] - off0), p1 = exp2f(sc[nt][1] - off0);
      const float p2 = exp2f(sc[nt][2] - off1), p3 = exp2f(sc[nt][3] - off1);
      sum0 += p0 + p1; sum1 += p2 + p3;
      const __half2 h01 = __floats2half2_rn(p0, p1), h23 = __floats2half2_rn(p2, p3);
      const float2 f01 = __half22float2(h01), f23 = __half22float2(h23);
      phi[nt][0] = *reinterpret_cast<const uint32_t*>(&h01); phi[nt][1] = *reinterpret_cast<const uint32_t*>(&h23);
      plo[nt][0] = pack_half2_u32(p0 - f01.x, p1 - f01.y); plo[nt][1] = pack_half2_u32(p2 - f23.x, p3 - f23.y);
    }
    sum0 += __shfl_xor_sync(0xffffffffu, sum0, 1); sum0 += __shfl_xor_sync(0xffffffffu, sum0, 2);
    sum1 += __shfl_xor_sync(0xffffffffu, sum1, 1); sum1 += __shfl_xor_sync(0xffffffffu, sum1, 2);
    const float inv0 = (mx0 == -INFINITY || !(sum0 > 0.f)) ? 0.f : 1.f / sum0;
    const float inv1 = (mx1 == -INFINITY || !(sum1 > 0.f)) ? 0.f : 1.f / sum1;
    __half* o0 = out16 + (static_cast<size_t>(smp) * S + r0) * 2 * d + h * 128 + 2 * t;
    __half* o1 = out16 + (static_cast<size_t>(smp) * S + r1) * 2 * d + h * 128 + 2 * t;
#pragma unroll
    for (int nd = 0; nd < 16; ++nd) {
      float o[4] = {0.f, 0.f, 0.f, 0.f};
      const __half* vrow = sVt + (nd * 8 + g) * VS + 2 * t;
#pragma unroll
      for (int kk = 0; kk < MAX_NT / 2; ++kk) {
        const uint32_t b0 = *reinterpret_cast<const uint32_t*>(vrow + 16 * kk);
        const uint32_t b1 = *reinterpret_cast<const uint32_t*>(vrow + 16 * kk + 8);
        mma_m16n8k16(o, phi[2 * kk][0], phi[2 * kk][1], phi[2 * kk + 1][0], phi[2 * kk + 1][1], b0, b1);
        mma_m16n8k16(o, plo[2 * kk][0], plo[2 * kk][1], plo[2 * kk + 1][0], plo[2 * kk + 1][1], b0, b1);
      }
      if (r0 < S) *reinterpret_cast<__half2*>(o0 + nd * 8) = __floats2half2_rn(o[0] * inv0, o[1] * inv0);
      if (r1 < S) *reinterpret_cast<__half2*>(o1 + nd * 8) = __floats2half2_rn(o[2] * inv1, o[3] * inv1);
    }
  }
}

// Cross-attention core for long text memories (64 < Mt <= 512, DistilBERT's position limit): the interface of
// cross_attention_kernel, with the keys taken in blocks of 64 instead of all at once in registers.
//   * each block's K and V rows are staged in shared memory by cp.async, double-buffered: block kb + 1 is in flight
//     while block kb is used; keys past Mt are zero-filled (never read from global memory) and masked;
//   * scores: m16n8k16 with the q fragments held in registers for the whole launch.  Thread t of a quad owns the
//     16-byte chunks t, t + 4, t + 8, t + 12 of the 128 columns, for q and k alike (a dot product does not care about
//     the order of its terms), so a K row is read as four 16-byte shared-memory loads;
//   * online softmax in fp32 per query row: a running max m and sum l.  When a block raises m, O and l are scaled by
//     2^(m_old - m_new) (exactly 1 when m does not move, 0 when m_old = -inf).  While every key so far is masked m
//     stays -inf and the exponent offset is 0, so p = 0 and no -inf - -inf appears;
//   * P feeds P.V as hi + lo fp16 like the short core, V fragments come from row-major V by ldmatrix.trans, and O
//     [16 rows x 128] stays in registers across the blocks (16 n-tiles x 4 fp32 per thread).
// Shared-memory rows are unpadded: K chunk c of row r sits at c ^ 4 (r & 1), V chunk c at c ^ (r & 7), so a quad pair's
// 16-byte K loads and an ldmatrix's 8 row addresses each fall in distinct banks.
// A fully masked row yields 0.  grid = (heads, n_samples, ceil(S / 64)): one 64-row pass per CTA, so every CTA holds
// one warp tile of O and S = 196 runs as four CTAs per (sample, head), each streaming that head's K / V blocks from L2.
// block = 128 (4 warps x 16 rows), dynamic shared memory XAL_SMEM.
constexpr int XAL_KEYS = 64;                 // keys per block
constexpr int XAL_MAX_MT = 512;
constexpr int XAL_ROWS = 64;                 // query rows per CTA
constexpr int XAL_TILE = XAL_KEYS * 128;     // halves of one staged K or V block
constexpr size_t XAL_SMEM = 2 * 2 * XAL_TILE * sizeof(__half) + 2 * XAL_KEYS * sizeof(float);

__device__ __forceinline__ void cp_async16_zfill(uint32_t dst, const void* src, bool valid) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;\n" ::"r"(dst), "l"(src), "r"(valid ? 16 : 0) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;\n" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;\n" ::"n"(N) : "memory"); }

__global__ void __launch_bounds__(128) cross_attention_long_kernel(const __half* __restrict__ q16, const __half* __restrict__ kv16,
                                                                   const unsigned char* __restrict__ mask,
                                                                   __half* __restrict__ out16, int S, int Mt, int d, int ld_kv,
                                                                   float scale_log2) {
  pdl_launch_dependents();
  pdl_wait();
  extern __shared__ __align__(16) unsigned char xal_smem[];
  __half* sK = reinterpret_cast<__half*>(xal_smem);                    // [2][64 keys][128]
  __half* sV = sK + 2 * XAL_TILE;                                      // [2][64 keys][128]
  float* sBias = reinterpret_cast<float*>(sV + 2 * XAL_TILE);          // [2][64]
  const int h = blockIdx.x, smp = blockIdx.y;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, g = lane >> 2, t = lane & 3;
  const __half* kv = kv16 + static_cast<size_t>(smp) * Mt * ld_kv + h * 128;
  const unsigned char* mk = mask + static_cast<size_t>(smp) * Mt;
  const int nb = (Mt + XAL_KEYS - 1) / XAL_KEYS;

  auto stage = [&](int kb) {
    const int buf = kb & 1;
    const uint32_t ks = smem_u32(sK + buf * XAL_TILE), vs = smem_u32(sV + buf * XAL_TILE);
    for (int i = threadIdx.x; i < XAL_KEYS * 16; i += 128) {
      const int r = i >> 4, c = i & 15, key = kb * XAL_KEYS + r;
      const bool in = key < Mt;
      const __half* src = kv + static_cast<size_t>(in ? key : 0) * ld_kv + c * 8;
      cp_async16_zfill(ks + 2 * (r * 128 + 8 * (c ^ ((r & 1) << 2))), src, in);
      cp_async16_zfill(vs + 2 * (r * 128 + 8 * (c ^ (r & 7))), src + d, in);
    }
    if (threadIdx.x < XAL_KEYS) {
      const int key = kb * XAL_KEYS + threadIdx.x;
      sBias[buf * XAL_KEYS + threadIdx.x] = (key < Mt && !mk[key]) ? 0.f : -INFINITY;
    }
    cp_async_commit();
  };
  stage(0);

  const int m0 = blockIdx.z * XAL_ROWS + warp * 16, r0 = m0 + g, r1 = r0 + 8;
  const bool active = m0 < S;                  // idle warps still stage blocks and meet the barriers
  uint32_t qa[16], qb[16];
  {
    const size_t row0 = static_cast<size_t>(smp) * S + min(r0, S - 1), row1 = static_cast<size_t>(smp) * S + min(r1, S - 1);
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const uint4 a = *reinterpret_cast<const uint4*>(q16 + row0 * d + h * 128 + 8 * (4 * i + t));
      const uint4 b = *reinterpret_cast<const uint4*>(q16 + row1 * d + h * 128 + 8 * (4 * i + t));
      qa[4 * i] = a.x; qa[4 * i + 1] = a.y; qa[4 * i + 2] = a.z; qa[4 * i + 3] = a.w;
      qb[4 * i] = b.x; qb[4 * i + 1] = b.y; qb[4 * i + 2] = b.z; qb[4 * i + 3] = b.w;
    }
  }
  float o[16][4];
#pragma unroll
  for (int nd = 0; nd < 16; ++nd) o[nd][0] = o[nd][1] = o[nd][2] = o[nd][3] = 0.f;
  float mx0 = -INFINITY, mx1 = -INFINITY, l0 = 0.f, l1 = 0.f;   // l: this thread's share of the row sums

  for (int kb = 0; kb < nb; ++kb) {
    if (kb + 1 < nb) {
      stage(kb + 1);
      cp_async_wait<1>();
    } else {
      cp_async_wait<0>();
    }
    __syncthreads();
    if (active) {
      const int buf = kb & 1;
      const __half* kbuf = sK + buf * XAL_TILE;
      const float* bias = sBias + buf * XAL_KEYS;
      float sc[8][4];
#pragma unroll
      for (int nt = 0; nt < 8; ++nt) {
        sc[nt][0] = sc[nt][1] = sc[nt][2] = sc[nt][3] = 0.f;
        const __half* krow = kbuf + (nt * 8 + g) * 128;
        uint32_t kw[16];
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          const uint4 a = *reinterpret_cast<const uint4*>(krow + 8 * ((4 * i + t) ^ ((g & 1) << 2)));
          kw[4 * i] = a.x; kw[4 * i + 1] = a.y; kw[4 * i + 2] = a.z; kw[4 * i + 3] = a.w;
        }
#pragma unroll
        for (int j = 0; j < 8; ++j) mma_m16n8k16(sc[nt], qa[2 * j], qb[2 * j], qa[2 * j + 1], qb[2 * j + 1], kw[2 * j], kw[2 * j + 1]);
      }
      // thread holds keys nt*8 + 2t, +1 of rows g (c0, c1) and g+8 (c2, c3)
      float bm0 = -INFINITY, bm1 = -INFINITY;
#pragma unroll
      for (int nt = 0; nt < 8; ++nt) {
        const float b0 = bias[nt * 8 + 2 * t], b1 = bias[nt * 8 + 2 * t + 1];
        sc[nt][0] = fmaf(sc[nt][0], scale_log2, b0); sc[nt][1] = fmaf(sc[nt][1], scale_log2, b1);
        sc[nt][2] = fmaf(sc[nt][2], scale_log2, b0); sc[nt][3] = fmaf(sc[nt][3], scale_log2, b1);
        bm0 = fmaxf(bm0, fmaxf(sc[nt][0], sc[nt][1]));
        bm1 = fmaxf(bm1, fmaxf(sc[nt][2], sc[nt][3]));
      }
      bm0 = fmaxf(bm0, __shfl_xor_sync(0xffffffffu, bm0, 1)); bm0 = fmaxf(bm0, __shfl_xor_sync(0xffffffffu, bm0, 2));
      bm1 = fmaxf(bm1, __shfl_xor_sync(0xffffffffu, bm1, 1)); bm1 = fmaxf(bm1, __shfl_xor_sync(0xffffffffu, bm1, 2));
      const float mn0 = fmaxf(mx0, bm0), mn1 = fmaxf(mx1, bm1);
      const float al0 = (mn0 == mx0) ? 1.f : exp2f(mx0 - mn0), al1 = (mn1 == mx1) ? 1.f : exp2f(mx1 - mn1);
      mx0 = mn0; mx1 = mn1;
      const float off0 = (mn0 == -INFINITY) ? 0.f : mn0, off1 = (mn1 == -INFINITY) ? 0.f : mn1;
      float s0 = 0.f, s1 = 0.f;
#pragma unroll
      for (int nt = 0; nt < 8; ++nt) {
        sc[nt][0] = exp2f(sc[nt][0] - off0); sc[nt][1] = exp2f(sc[nt][1] - off0);
        sc[nt][2] = exp2f(sc[nt][2] - off1); sc[nt][3] = exp2f(sc[nt][3] - off1);
        s0 += sc[nt][0] + sc[nt][1]; s1 += sc[nt][2] + sc[nt][3];
      }
      l0 = l0 * al0 + s0; l1 = l1 * al1 + s1;
#pragma unroll
      for (int nd = 0; nd < 16; ++nd) {
        o[nd][0] *= al0; o[nd][1] *= al0; o[nd][2] *= al1; o[nd][3] *= al1;
      }
      // P.V: lane addresses row (lane & 7) of ldmatrix matrix lane >> 3 = (keys +8 if odd, columns +8 if >= 2)
      const uint32_t vbuf = smem_u32(sV + buf * XAL_TILE);
      const int mi = lane >> 3, lr = lane & 7;
#pragma unroll
      for (int kk = 0; kk < 4; ++kk) {
        uint32_t ph[4], pl[4];
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const float x = sc[2 * kk + (j >> 1)][2 * (j & 1)], y = sc[2 * kk + (j >> 1)][2 * (j & 1) + 1];
          const __half2 hv = __floats2half2_rn(x, y);
          const float2 hf = __half22float2(hv);
          ph[j] = *reinterpret_cast<const uint32_t*>(&hv);
          pl[j] = pack_half2_u32(x - hf.x, y - hf.y);
        }
        const int vr = 16 * kk + 8 * (mi & 1) + lr;
#pragma unroll
        for (int nd = 0; nd < 16; nd += 2) {
          uint32_t b[4];
          ldmatrix_x4_trans(b, vbuf + 2 * (vr * 128 + 8 * ((nd + (mi >> 1)) ^ lr)));
          mma_16816(o[nd], ph, b[0], b[1]);
          mma_16816(o[nd], pl, b[0], b[1]);
          mma_16816(o[nd + 1], ph, b[2], b[3]);
          mma_16816(o[nd + 1], pl, b[2], b[3]);
        }
      }
    }
    __syncthreads();   // the next iteration stages block kb + 2 into this buffer
  }
  if (!active) return;
  l0 += __shfl_xor_sync(0xffffffffu, l0, 1); l0 += __shfl_xor_sync(0xffffffffu, l0, 2);
  l1 += __shfl_xor_sync(0xffffffffu, l1, 1); l1 += __shfl_xor_sync(0xffffffffu, l1, 2);
  const float inv0 = (mx0 == -INFINITY || !(l0 > 0.f)) ? 0.f : 1.f / l0;
  const float inv1 = (mx1 == -INFINITY || !(l1 > 0.f)) ? 0.f : 1.f / l1;
  __half* o0 = out16 + (static_cast<size_t>(smp) * S + r0) * 2 * d + h * 128 + 2 * t;
  __half* o1 = out16 + (static_cast<size_t>(smp) * S + r1) * 2 * d + h * 128 + 2 * t;
#pragma unroll
  for (int nd = 0; nd < 16; ++nd) {
    if (r0 < S) *reinterpret_cast<__half2*>(o0 + nd * 8) = __floats2half2_rn(o[nd][0] * inv0, o[nd][1] * inv0);
    if (r1 < S) *reinterpret_cast<__half2*>(o1 + nd * 8) = __floats2half2_rn(o[nd][2] * inv1, o[nd][3] * inv1);
  }
}

}  // namespace b200
