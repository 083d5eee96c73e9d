// Fused GEMM epilogues.  EpiEmbed and EpiOut serve the staged kernel gemm_f16_wgmma (gemm.cuh: chunk / finish, thread
// = accumulator row, 32 columns at a time).  The projection epilogues (EpiBiasF16, EpiBiasF16Global, EpiBiasF16Wide)
// provide the fragment interface of gemm_pingpong.cuh instead (preload, then pp_*: one column pair of the wgmma
// accumulator fragment at a time).
//
// Row-major outputs are written as 128-byte-per-row slabs (32 rows of the warp x 64 fp16 or 32 fp32 columns = 4 KB)
// staged in warp-private shared memory in the TMA 128-byte swizzle and shipped with cp.async.bulk.tensor stores;
// residual inputs arrive the same way with TMA loads.  No global load/store instruction is issued by these
// epilogues except broadcast bias reads, and out-of-range rows / columns are clipped by the TMA unit.
// Feature-major outputs ([B, J, T], T contiguous) are written straight from registers because consecutive
// accumulator rows are consecutive frames (coalesced along T).
#pragma once
#include <cuda_fp16.h>

#include "gemm.cuh"
#include "ptx.cuh"

namespace b200 {

// byte offset of 16-byte chunk j (0..7) of row r inside a [32 x 128 B] slab with the TMA SWIZZLE_128B pattern
__device__ __forceinline__ uint32_t slab_off(int r, int j) { return r * 128 + ((j ^ (r & 7)) << 4); }
// byte offset of 16-byte chunk j (0..3) of row r inside a [32 x 64 B] half-slab with the TMA SWIZZLE_64B pattern
// (address bits 4-5 xor bits 7-8).  A residual-stream slab is two of these: hi halves at +0, lo halves at +2048.
__device__ __forceinline__ uint32_t slab64_off(int r, int j) { return r * 64 + ((j ^ ((r >> 1) & 3)) << 4); }

// 8 fp32 values -> 4 packed half2 "hi" words + 4 packed half2 "lo" words with hi + lo = v to ~22 bits
__device__ __forceinline__ void split_hi_lo8(const float (&v)[8], uint32_t (&hi)[4], uint32_t (&lo)[4]) {
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const __half2 h = __floats2half2_rn(v[2 * i], v[2 * i + 1]);
    const float2 f = __half22float2(h);
    const __half2 l = __floats2half2_rn(v[2 * i] - f.x, v[2 * i + 1] - f.y);
    hi[i] = *reinterpret_cast<const uint32_t*>(&h);
    lo[i] = *reinterpret_cast<const uint32_t*>(&l);
  }
}
// the inverse for one 16-byte group of hi and one of lo: 8 fp32 values
__device__ __forceinline__ void join_hi_lo8(const uint4& h, const uint4& l, float (&v)[8]) {
  const uint32_t hw[4] = {h.x, h.y, h.z, h.w}, lw[4] = {l.x, l.y, l.z, l.w};
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const float2 a = __half22float2(*reinterpret_cast<const __half2*>(&hw[i]));
    const float2 b = __half22float2(*reinterpret_cast<const __half2*>(&lw[i]));
    v[2 * i] = a.x + b.x;
    v[2 * i + 1] = a.y + b.y;
  }
}

// exact (erf) GELU, torch F.gelu default (reference model/mdm.py:80 activation="gelu"):  gelu(x) = x * Phi(x).
// Phi(-t) = 2^q(t) with q a degree-6 minimax fit of log2(0.5*erfc(t/sqrt 2)) on [0, 5.5] (|Phi error| < 1.5e-7);
// Phi(t) = 1 - Phi(-t).  Below x = -5.5 the result is 0: |gelu(x)| < |gelu(-5.5)| = 1.1e-7 there, while the clamped
// polynomial would return x * Phi(-5.5), an error that grows with |x| (1.8e-5 at x = -1000).  |gelu error| < 8e-7 +
// 2^-22 |gelu(x)| over all x: tests/test_epilogues_gpu.py::test_gelu_sweep checks it against fp64 erfc from -1008 to 6.
// 11 FP32 ops + one MUFU.EX2 instead of the ~25 of erff() -- the epilogue of the FFN up-projection runs 26 M of these
// per layer.
__device__ __forceinline__ float gelu_erf(float x) {
  const float t = fminf(fabsf(x), 5.5f);
  float q = 1.9175331544829533e-05f;
  q = fmaf(q, t, -0.0006586098461411893f);
  q = fmaf(q, t, 0.007754423655569553f);
  q = fmaf(q, t, -0.05296541005373001f);
  q = fmaf(q, t, -0.4590602517127991f);
  q = fmaf(q, t, -1.1511220932006836f);
  q = fmaf(q, t, -0.9999997019767761f);
  float a;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(a) : "f"(q));
  const float phi = (x >= 0.f) ? (1.0f - a) : (x < -5.5f ? 0.f : a);
  return x * phi;
}

__device__ __forceinline__ uint32_t pack_half2(float a, float b) {
  __half2 h = __floats2half2_rn(a, b);
  return *reinterpret_cast<uint32_t*>(&h);
}

// ---------------------------------------------------------------------------------------------------------
// out16[row, col] = fp16( act(acc + bias[col]) )          (QKV projection, FFN up-projection)
// map_c: fp16 [M, N], box {64 cols, 32 rows}, SWIZZLE_128B.  Fragment interface only (gemm_f16_pingpong), like
// EpiBiasF16Wide / EpiBiasF16Global.
template <bool GELU>
struct EpiBiasF16 {
  struct Params {
    const float* bias;
  };
  // the bias of ALL N columns is staged once per CTA (a per-tile global load sat on the epilogue's critical path:
  // 1-2.7 k cycles between "accumulator ready" and the first chunk, measured with clock64 stamps)
  static __device__ __forceinline__ void preload(const Params& p, float* dst, int N, int tid, int nthreads) {
    for (int i = tid; i < N; i += nthreads) dst[i] = p.bias[i];
  }
  // one column pair of one accumulator row at a time
  static constexpr int PP_ROUND_COLS = 128;   // a round fills two 64-column slabs (16 KB each) of the warpgroup's 128 rows
  // the bias of the tile's 128 columns (col_t = first column): here a view of the CTA's staged vector
  static __device__ __forceinline__ const float* pp_tile_bias(const Params&, const float* bias_all, float*, int col_t, int, int) {
    return bias_all + col_t;
  }
  static __device__ __forceinline__ void pp_pair(const Params&, float2 b, float a0, float a1, uint8_t* dst) {
    float x0 = a0 + b.x, x1 = a1 + b.y;
    if (GELU) {
      x0 = gelu_erf(x0); x1 = gelu_erf(x1);
    }
    *reinterpret_cast<uint32_t*>(dst) = pack_half2(x0, x1);
  }
  static __device__ __forceinline__ void pp_store(const CUtensorMap* map_c, const Params&, const uint8_t* box, int col, int row) {
    tma_store_2d(map_c, box, col, row);
  }
};

// EpiBiasF16 for a GEMM wider than the staged-vector limit (the cross-attention K/V projection of all decoder layers
// at once, N = L * 2d = 8192): the bias is read from global memory, one float2 per column pair.  Fragment interface
// only (gemm_f16_pingpong).
struct EpiBiasF16Global : EpiBiasF16<false> {
  static constexpr bool UNSTAGED = true;
  static __device__ __forceinline__ void preload(const Params&, float*, int, int, int) {}
  // thread `tid` (0..127) of the warpgroup copies one column of the tile's bias into the warpgroup's 128-float scratch
  // (visible to the warpgroup after its next named barrier)
  static __device__ __forceinline__ const float* pp_tile_bias(const Params& p, const float*, float* scratch, int col_t, int N,
                                                              int tid) {
    scratch[tid] = col_t + tid < N ? __ldg(p.bias + col_t + tid) : 0.f;
    return scratch;
  }
};

// ---------------------------------------------------------------------------------------------------------
// EpiBiasF16 with the result kept as a [hi | lo] fp16 pair: out16[row, col] = hi, out16[row, lo_col + col] = lo with
// hi + lo = act(acc + bias) to ~22 bits (trans_dec engine, where guidance 7.5 amplifies activation rounding; the
// consumer GEMM runs over K = 2N against [W | W]).  map_c: fp16 [M, 2N], box {64 cols, 32 rows}, SWIZZLE_128B.
// Fragment interface only (gemm_f16_pingpong).
template <bool GELU>
struct EpiBiasF16Wide {
  struct Params {
    const float* bias;
    int lo_col;
  };
  static __device__ __forceinline__ void preload(const Params& p, float* dst, int N, int tid, int nthreads) {
    for (int i = tid; i < N; i += nthreads) dst[i] = p.bias[i];
  }
  static constexpr int PP_ROUND_COLS = 64;    // a round fills one 64-column hi slab (16 KB) and its lo slab, 16 KB further
  static __device__ __forceinline__ const float* pp_tile_bias(const Params&, const float* bias_all, float*, int col_t, int, int) {
    return bias_all + col_t;
  }
  static __device__ __forceinline__ void pp_pair(const Params&, float2 b, float a0, float a1, uint8_t* dst) {
    float x0 = a0 + b.x, x1 = a1 + b.y;
    if (GELU) {
      x0 = gelu_erf(x0); x1 = gelu_erf(x1);
    }
    const __half2 h = __floats2half2_rn(x0, x1);
    const float2 f = __half22float2(h);
    const __half2 l = __floats2half2_rn(x0 - f.x, x1 - f.y);
    *reinterpret_cast<__half2*>(dst) = h;
    *reinterpret_cast<__half2*>(dst + 16384) = l;
  }
  static __device__ __forceinline__ void pp_store(const CUtensorMap* map_c, const Params& p, const uint8_t* box, int col, int row) {
    tma_store_2d(map_c, box, col, row);
    tma_store_2d(map_c, box + 16384, p.lo_col + col, row);
  }
};

// ---------------------------------------------------------------------------------------------------------
// InputProcess + positional encoding (reference model/mdm.py:238,252,343-349):
//   GEMM rows are (b, s) over B*S, s >= 1 is frame s-1:  h = acc + (bias + pe[s]).  The frame rows are identical for
//   the cond / uncond halves of the packed CFG batch, so every slab is TMA-stored twice (one tensor map per half --
//   the per-half maps also clip the rows of the last M tile that belong to the other half).  Row s == 0 (the
//   conditioning token, mdm.py:251) is produced by tok0_rows_kernel right after this GEMM.
//   Output: the residual stream as fp16 [hi | lo] (hi half = the next GEMM's A operand).
struct EpiEmbed {
  static constexpr int SMEM_PER_WARP = 2 * 4096;  // two [hi | lo] slabs
  struct Params {
    CUtensorMap res_c, res_u;                 // residual stream [rows, 2d] = [hi | lo] of the two CFG halves,
                                              // box {32 cols, 32 rows} (64-byte rows, SWIZZLE_64B)
    const float* pe_bias;                     // [S, d] = pe[s] + bias
    int S, d, halves;
  };
  static __device__ __forceinline__ void chunk(EpiCtx& ctx, const Params& p, uint32_t (&raw)[32], int row0, int col0) {
    uint8_t* slab = ctx.smem + (ctx.seq & 1) * 4096;
    if (ctx.lane == 0) bulk_wait_group_read<1>();  // the group that last read this slab (two chunks ago) is done
    __syncwarp();
    const int row = row0 + ctx.lane;
    const int s = (row < ctx.M) ? row % p.S : 0;
    const float* pb = p.pe_bias + static_cast<size_t>(s) * p.d + col0;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const float4 a0 = __ldg(reinterpret_cast<const float4*>(pb + 8 * j));
      const float4 a1 = __ldg(reinterpret_cast<const float4*>(pb + 8 * j + 4));
      const float o[8] = {__uint_as_float(raw[8 * j + 0]) + a0.x, __uint_as_float(raw[8 * j + 1]) + a0.y,
                          __uint_as_float(raw[8 * j + 2]) + a0.z, __uint_as_float(raw[8 * j + 3]) + a0.w,
                          __uint_as_float(raw[8 * j + 4]) + a1.x, __uint_as_float(raw[8 * j + 5]) + a1.y,
                          __uint_as_float(raw[8 * j + 6]) + a1.z, __uint_as_float(raw[8 * j + 7]) + a1.w};
      uint32_t hi[4], lo[4];
      split_hi_lo8(o, hi, lo);
      *reinterpret_cast<uint4*>(slab + slab64_off(ctx.lane, j)) = make_uint4(hi[0], hi[1], hi[2], hi[3]);
      *reinterpret_cast<uint4*>(slab + 2048 + slab64_off(ctx.lane, j)) = make_uint4(lo[0], lo[1], lo[2], lo[3]);
    }
    fence_proxy_async_smem();
    __syncwarp();
    if (ctx.lane == 0) {
      tma_store_2d(&p.res_c, slab, col0, row0);
      tma_store_2d(&p.res_c, slab + 2048, p.d + col0, row0);
      if (p.halves == 2) {
        tma_store_2d(&p.res_u, slab, col0, row0);
        tma_store_2d(&p.res_u, slab + 2048, p.d + col0, row0);
      }
      bulk_commit_group();
    }
    ctx.seq++;
  }
  static __device__ __forceinline__ void finish(EpiCtx& ctx) {
    if (ctx.lane == 0) bulk_wait_group<0>();
    __syncwarp();
  }
};

// ---------------------------------------------------------------------------------------------------------
// OutputProcess + (inpainting) + sampler update fused (reference model/mdm.py:372-386,
// diffusion/gaussian_diffusion.py:300-304, 254-257, 525-540, 757-778, 838-874, 992-1074).  GEMM rows are frames:
// row = b*T + t; column j < J is a feature.  All tensors are the reference layout [B, J*F, T].
// x0 = acc + bias, then the inpainting blend, then the clamp; then the update of `mode`, in fp32 in the reference's
// operation order with no contraction (bit-exact):
//   mode 0: out = x0                       (model forward only)
//   mode 1: DDPM   x_{t-1} = c1*x0 + c2*x_t + (nz*sigma)*eps
//   mode 2: DDIM   eps_hat = (sr*x_t - x0)/srm1 ; x_{t-1} = x0*sqrt_abp + coef*eps_hat + (nz*sigma)*eps
// PLMS (gaussian_diffusion.py:992-1074), eps = (sr*x - x0)/srm1 as in DDIM; sqrt_abp / sqrt(1 - abp) are columns 5 / 6
// of an eta = 0 table (sigma = 0 exactly, so 1 - abp - sigma^2 == 1 - abp).  eps of the k-th evaluation of the loop
// (k = StepState::done) lives in slot k % 3 of an eps history ring:
//   mode 3: Adams-Bashforth  eps' = combine(eps, ring[k-1], ring[k-2], ring[k-3]) at cur_order = min(order, k + 1);
//           ring[k] = eps; pred' = sr*x_t - srm1*eps'; x_{t-1} = (pred'*sqrt_abp + s1*eps')*nz + x0*(1 - nz)
//   mode 4: improved Euler, first evaluation: ring[k] = eps0; pred_xstart = x0; x_out = x0*sqrt_abp + s1*eps0 (mean1)
//   mode 5: improved Euler, second evaluation, of x_t = mean1 at schedule index i - 1 (`back` = 1): eps2 from the row
//           of i - 1; eps' = (ring[k] + eps2)/2; pred' from x_step (the step's x_t) and the row of i; the sample as
//           in mode 3 with x0 = pred_xstart (the first evaluation's)
// DDIM inversion (ddim_reverse_sample, gaussian_diffusion.py:838-874): x at schedule index i -> x at index i + 1
//   mode 6: eps = (sr*x - x0)/srm1 (row i of sched); x_next = x0*sqrt(abn) + sqrt(1 - abn)*eps (row i of sched_next)
// DPM-Solver++ multistep, data prediction (Lu et al. 2022, Algorithm 2; DESIGN.md section 1): x0 of evaluation k lives in
// slot k % 2 of an x0 history, row i of the DPM table holds (c_x, c0, c_cur, c_prev)
//   mode 7: cur_order = (k == 0 || i == 0) ? 1 : order;  history[k % 2] = x0;
//           order 1: x_out = fmaf(c0, x0, c_x*x);  order 2: x_out = fmaf(c_prev, history[(k-1) % 2], fmaf(c_cur, x0, c_x*x))
// Variational bound (calc_bpd_loop / _vb_terms_bpd, gaussian_diffusion.py:1189-1222, 1544-1599; diffusion/losses.py):
// x_t = q_sample(x_start, i, eps) was formed by vb_xt_kernel at the head of the step; row i of the bound table (VB_*)
//   mode 8: mean = c1*x0 + c2*x_t;  i > 0: true_mean = c1*x_start + c2*x_t, term = normal_kl(true_mean, lv_true, mean,
//           lv_model);  i == 0: term = -discretized_gaussian_log_likelihood(x_start, mean, 0.5*lv_model);
//           xm = (x0 - x_start)^2;  em = ((sr*x_t - x0)/srm1 - eps)^2.  The three are summed per (row, 32-column chunk)
//           in column order into fixed slots of a partial-sum buffer (vb_reduce_kernel finishes the per-sample means)
// Per-step scalars come from a device table indexed by the device-side step state, so the very same launch
// (and CUDA graph) serves every step of the loop.
constexpr int SCHED_STRIDE = 8;       // floats per schedule row: c1 c2 sig_ddpm sr srm1 sqrt_abp coef_eps sig_ddim
constexpr int SCHED_NEXT_STRIDE = 2;  // floats per row of the reverse table: sqrt(abn) sqrt(1 - abn)
constexpr int SCHED_DPM_STRIDE = 4;   // floats per row of the DPM-Solver++ table: c_x c0 c_cur c_prev
// floats per row of the bound table (b200mdm_set_schedule_vb), every entry fp32 as the reference's tensors hold it:
constexpr int SCHED_VB_STRIDE = 12;
enum VbCol : int {
  VB_C1 = 0, VB_C2 = 1,          // posterior_mean_coef1 / 2
  VB_LV_TRUE = 2, VB_LV_MODEL = 3,   // posterior_log_variance_clipped; the model's fixed log-variance
  VB_SR = 4, VB_SRM1 = 5,        // sqrt_recip_alphas_cumprod, sqrt_recipm1_alphas_cumprod
  VB_SQ = 6, VB_SQM1 = 7,        // sqrt_alphas_cumprod, sqrt_one_minus_alphas_cumprod (q_sample)
  VB_KL_C = 8,                   // ((-1 + lv_model) - lv_true) + exp(lv_true - lv_model)   (normal_kl's per-row part)
  VB_EXP_NEG_LV = 9,             // exp(-lv_model)
  VB_INV_STD = 10,               // exp(-(0.5 * lv_model))   (discretized_gaussian_log_likelihood's inv_stdv)
  VB_PRIOR_C = 11,               // (-1 - log(1 - ac)) + exp(log(1 - ac))   (the prior term's normal_kl part, _prior_bpd)
};
constexpr int VB_TERMS = 3;           // vb, xstart_mse, mse
constexpr int PLMS_RING = 3;          // eps history slots: AB4 combines this step's eps with the three before it
constexpr int DPM_SLOTS = 2;          // x0 history slots: 2M combines this step's x0 with the one before it
enum OutMode : int {
  MODE_X0 = 0, MODE_DDPM = 1, MODE_DDIM = 2,                      // B200MDM_MODE_*
  MODE_PLMS_AB = 3, MODE_PLMS_EULER1 = 4, MODE_PLMS_EULER2 = 5,   // internal: the steps of the PLMS loop
  MODE_DDIM_REVERSE = 6,                                          // B200MDM_MODE_DDIM_REVERSE
  MODE_DPM = 7,                                                   // internal: the step of the DPM-Solver++ loop
  MODE_VB = 8,                                                    // internal: the step of the bound loop
};
struct StepState {
  int done;      // steps completed so far (indexes the noise tape; PLMS: the evaluation count k)
  int cur;       // schedule index i of the step in flight
  int n_steps;   // schedule length (index i - 1 of the PLMS improved-Euler step wraps to n_steps - 1 at i = 0)
  const float* noise;            // loop mode: base of the noise tape (set per loop, so the step graph is reusable)
  long long noise_step_stride;   // loop mode: elements between consecutive steps of the tape
  unsigned long long seed;       // in-engine Philox noise (philox_normal_kernel): stream seed ...
  long long sample_base;         // ... and the global index of this workspace's sample 0
};

// One slot of a continuously batched workspace (b200mdm_slots_begin): the schedule index of the step its row takes next
// (-1: idle, or finished and waiting to be read), and the Philox key of its request -- the stream seed and the request's
// global sample index.  Written by the slot kernels inside the step graph, so every reader loads it through L2, as
// load_step_state below.
struct SlotState {
  int cur;
  int pad;
  unsigned long long seed;
  long long g;
};

// The step state as of the last step_set / step_advance.  Every reader goes through L2 (ld.global.cg), never through
// the SM's L1 / read-only cache: under programmatic dependent launch a kernel is resident on an SM before the
// step_advance it depends on has written the state, and an L1 line of the previous step's state -- brought in by another
// kernel still running on that SM, e.g. a reader through a const __restrict__ pointer (LDG.CONSTANT) -- is not
// invalidated by griddepcontrol.wait.  Such a line once served the previous schedule index to the first kernel of the
// next step (DESIGN.md section 1, "Step state").
__device__ __forceinline__ StepState load_step_state(const StepState* s) {
  StepState st;
  st.done = __ldcg(&s->done);
  st.cur = __ldcg(&s->cur);
  st.n_steps = __ldcg(&s->n_steps);
  st.noise = reinterpret_cast<const float*>(__ldcg(reinterpret_cast<const unsigned long long*>(&s->noise)));
  st.noise_step_stride = __ldcg(&s->noise_step_stride);
  st.seed = __ldcg(&s->seed);
  st.sample_base = __ldcg(&s->sample_base);
  return st;
}

// Schedule index a forward evaluates: the step's own (back = 0) or the one before it (back = 1, PLMS improved Euler).
// At i = 0, i - 1 = -1 indexes the reference's timestep map and tables from the end (gaussian_diffusion.py:1046).
__device__ __forceinline__ int eval_index(const StepState& st, int back) {
  const int i = st.cur - back;
  return i < 0 ? i + st.n_steps : i;
}

struct EpiOutParams {
  const float* bias;        // [J]
  const float* x_t;         // [B, J, T]
  const float* noise;       // modes 1-2: explicit eps for one step; nullptr => tape described by *state (loop mode)
  float* x_out;             // [B, J, T]
  float* pred_xstart;       // nullable, except in modes 4 and 5
  const unsigned char* inpaint_mask;  // nullable, bool [B, J, T]
  const float* inpaint_weight;        // nullable, soft inpainting weight [B, J, T] in [0, 1]; at most one of it and the mask
  const float* inpaint_motion;        // [B, J, T]
  const float* sched;       // [n_steps, SCHED_STRIDE]
  const float* sched_next;  // mode 6: [n_steps, SCHED_NEXT_STRIDE]
  const float* sched_dpm;   // mode 7: [n_steps, SCHED_DPM_STRIDE]
  float* eps_ring;          // modes 3-5: [PLMS_RING, B, J, T]
  float* x0_hist;           // mode 7: [DPM_SLOTS, B, J, T]
  const float* x_step;      // mode 5: x_t of the step (x_t above is mean1 there)
  const float* sched_vb;    // mode 8: [n_steps, SCHED_VB_STRIDE]
  const float* x_start;     // mode 8: [B, J, T]
  float* vb_part;           // mode 8: [VB_TERMS, B*T, vb_chunks] per-(row, 32-column chunk) sums
  float* vb_elem;           // mode 8, nullable: [VB_TERMS, B, J, T] the per-element terms (kernel tests)
  int vb_chunks;            // mode 8: ceil(J / 32)
  const StepState* state;
  long long noise_batch_stride;  // J*T normally, 0 for const_noise
  int B, T, J, mode;
  int clip_denoised;        // clamp x0 to [-1, 1] after the inpainting blend (gaussian_diffusion.py:348-352)
  int order;                // mode 3: 1..4; mode 7: 1..2
  int back;                 // modes 3-5: this forward evaluates schedule index eval_index(state, back)
  const SlotState* slots;   // OutStepSlots: [B] per-row schedule index (last, so the other fields keep their offsets)
};

// The update policies of EpiOut: the constructor reads the chunk's scalars, load() the extra inputs of one element
// (In), store() writes its outputs from x0.
struct OutStep {   // modes 0-2
  float c1 = 0.f, c2 = 0.f, sg = 0.f, sr = 0.f, srm1 = 1.f, sq = 0.f, ce = 0.f;
  const float* nz = nullptr;
  struct In { float x, n; };
  __device__ __forceinline__ OutStep(const EpiOutParams& p, int b) {
    if (p.mode == MODE_X0) return;
    const StepState st = load_step_state(p.state);
    set_row(p, st.cur);
    nz = (p.noise != nullptr ? p.noise : st.noise + static_cast<long long>(st.done) * st.noise_step_stride) +
         static_cast<long long>(b) * p.noise_batch_stride;
  }
  __device__ __forceinline__ OutStep() {}
  // the scalars of schedule row i
  __device__ __forceinline__ void set_row(const EpiOutParams& p, int i) {
    const float* row_s = p.sched + static_cast<size_t>(i) * SCHED_STRIDE;
    c1 = row_s[0]; c2 = row_s[1]; sr = row_s[3]; srm1 = row_s[4]; sq = row_s[5]; ce = row_s[6];
    sg = (p.mode == MODE_DDPM) ? row_s[2] : row_s[7];
  }
  __device__ __forceinline__ In load(const EpiOutParams& p, bool in, size_t idx, int col, int t) const {
    in = in && p.mode != MODE_X0;
    return {in ? p.x_t[idx] : 0.f, in ? nz[static_cast<size_t>(col) * p.T + t] : 0.f};
  }
  __device__ __forceinline__ void store(const EpiOutParams& p, size_t idx, float x0, const In& v) const {
    if (p.pred_xstart != nullptr) p.pred_xstart[idx] = x0;
    float o = x0;
    if (p.mode == MODE_DDPM) {
      const float mean = __fadd_rn(__fmul_rn(c1, x0), __fmul_rn(c2, v.x));
      o = __fadd_rn(mean, __fmul_rn(sg, v.n));
    } else if (p.mode == MODE_DDIM) {
      const float eh = __fdiv_rn(__fsub_rn(__fmul_rn(sr, v.x), x0), srm1);
      const float mean = __fadd_rn(__fmul_rn(x0, sq), __fmul_rn(ce, eh));
      o = __fadd_rn(mean, __fmul_rn(sg, v.n));
    }
    p.x_out[idx] = o;
  }
  __device__ __forceinline__ void end(const EpiOutParams&, int, int) const {}
};

// DDPM / DDIM with a schedule index per row (continuous batching, b200mdm_sample_step_at): row b takes the step of its
// slot's index, with OutStep's arithmetic, and an idle slot (index -1) writes nothing -- a finished sample stays in
// place until it is read.  The eps is always explicit (the caller's, or the slot Philox kernel's eps_buf).
struct OutStepSlots : OutStep {   // modes 1-2
  bool idle;
  __device__ __forceinline__ OutStepSlots(const EpiOutParams& p, int b) {
    const int i = __ldcg(&p.slots[b].cur);
    idle = i < 0;
    if (idle) return;
    set_row(p, i);
    nz = p.noise + static_cast<long long>(b) * p.noise_batch_stride;
  }
  __device__ __forceinline__ In load(const EpiOutParams& p, bool in, size_t idx, int col, int t) const {
    return OutStep::load(p, in && !idle, idx, col, t);
  }
  __device__ __forceinline__ void store(const EpiOutParams& p, size_t idx, float x0, const In& v) const {
    if (!idle) OutStep::store(p, idx, x0, v);
  }
};

struct OutPlms {   // modes 3-5
  float sr, srm1, sq, s1, sr_e, srm1_e, nzf;
  int cur_order;
  const float *h1, *h2, *h3;
  float* own;
  // mode 3: e1..e3 = eps of evaluations k-1..k-3;  mode 5: e1 = eps0, e2 = x_step, e3 = x0 of the first evaluation
  struct In { float x, e1, e2, e3; };
  __device__ __forceinline__ OutPlms(const EpiOutParams& p, int) {
    const StepState st = load_step_state(p.state);
    const int k = st.done;
    const float* row_s = p.sched + static_cast<size_t>(st.cur) * SCHED_STRIDE;
    const float* row_e = p.sched + static_cast<size_t>(eval_index(st, p.back)) * SCHED_STRIDE;
    sr = row_s[3]; srm1 = row_s[4]; sq = row_s[5]; s1 = row_s[6];
    sr_e = row_e[3]; srm1_e = row_e[4];
    nzf = st.cur != 0 ? 1.f : 0.f;                  // (t != 0), gaussian_diffusion.py:1071
    cur_order = min(p.order, k + 1);
    const size_t slot = static_cast<size_t>(p.B) * p.J * p.T;
    h1 = p.eps_ring + static_cast<size_t>((k + PLMS_RING - 1) % PLMS_RING) * slot;
    h2 = p.eps_ring + static_cast<size_t>((k + PLMS_RING - 2) % PLMS_RING) * slot;
    h3 = p.eps_ring + static_cast<size_t>(k % PLMS_RING) * slot;   // k - 3
    own = p.eps_ring + static_cast<size_t>(k % PLMS_RING) * slot;
  }
  __device__ __forceinline__ In load(const EpiOutParams& p, bool in, size_t idx, int, int) const {
    In v{in ? p.x_t[idx] : 0.f, 0.f, 0.f, 0.f};
    if (in && p.mode == MODE_PLMS_AB) {
      if (cur_order >= 2) v.e1 = h1[idx];
      if (cur_order >= 3) v.e2 = h2[idx];
      if (cur_order >= 4) v.e3 = h3[idx];
    } else if (in && p.mode == MODE_PLMS_EULER2) {
      v.e1 = own[idx];
      v.e2 = p.x_step[idx];
      v.e3 = p.pred_xstart[idx];
    }
    return v;
  }
  __device__ __forceinline__ void store(const EpiOutParams& p, size_t idx, float x0, const In& v) const {
    // _predict_eps_from_xstart (gaussian_diffusion.py:400-404) at the index this forward evaluates
    const float eps = __fdiv_rn(__fsub_rn(__fmul_rn(sr_e, v.x), x0), srm1_e);
    if (p.mode == MODE_PLMS_EULER1) {
      own[idx] = eps;
      p.pred_xstart[idx] = x0;
      p.x_out[idx] = __fadd_rn(__fmul_rn(x0, sq), __fmul_rn(s1, eps));   // :1045
      return;
    }
    float ep, x_t = v.x, x0s = x0;
    if (p.mode == MODE_PLMS_EULER2) {
      ep = __fdiv_rn(__fadd_rn(v.e1, eps), 2.f);                          // :1047
      x_t = v.e2;
      x0s = v.e3;
    } else {
      if (p.pred_xstart != nullptr) p.pred_xstart[idx] = x0;
      if (cur_order == 1) {                                               // :1055-1062
        ep = eps;
      } else if (cur_order == 2) {
        ep = __fdiv_rn(__fsub_rn(__fmul_rn(3.f, eps), v.e1), 2.f);
      } else if (cur_order == 3) {
        ep = __fdiv_rn(__fadd_rn(__fsub_rn(__fmul_rn(23.f, eps), __fmul_rn(16.f, v.e1)), __fmul_rn(5.f, v.e2)), 12.f);
      } else {
        ep = __fdiv_rn(__fsub_rn(__fadd_rn(__fsub_rn(__fmul_rn(55.f, eps), __fmul_rn(59.f, v.e1)), __fmul_rn(37.f, v.e2)),
                                 __fmul_rn(9.f, v.e3)),
                       24.f);
      }
      own[idx] = eps;                                                     // replaces evaluation k - 3
    }
    // _predict_xstart_from_eps (:381-388), then the mean and the (t != 0) blend (:1065-1072)
    const float pp = __fsub_rn(__fmul_rn(sr, x_t), __fmul_rn(srm1, ep));
    const float mean = __fadd_rn(__fmul_rn(pp, sq), __fmul_rn(s1, ep));
    p.x_out[idx] = __fadd_rn(__fmul_rn(mean, nzf), __fmul_rn(x0s, __fsub_rn(1.f, nzf)));
  }
  __device__ __forceinline__ void end(const EpiOutParams&, int, int) const {}
};

struct OutReverse {   // mode 6: no noise and no history
  float sr, srm1, sa, sb;
  struct In { float x; };
  __device__ __forceinline__ OutReverse(const EpiOutParams& p, int) {
    const int i = load_step_state(p.state).cur;
    const float* row_s = p.sched + static_cast<size_t>(i) * SCHED_STRIDE;
    const float* row_n = p.sched_next + static_cast<size_t>(i) * SCHED_NEXT_STRIDE;
    sr = row_s[3]; srm1 = row_s[4]; sa = row_n[0]; sb = row_n[1];
  }
  __device__ __forceinline__ In load(const EpiOutParams& p, bool in, size_t idx, int, int) const {
    return {in ? p.x_t[idx] : 0.f};
  }
  __device__ __forceinline__ void store(const EpiOutParams& p, size_t idx, float x0, const In& v) const {
    if (p.pred_xstart != nullptr) p.pred_xstart[idx] = x0;
    const float eps = __fdiv_rn(__fsub_rn(__fmul_rn(sr, v.x), x0), srm1);    // :862-865
    p.x_out[idx] = __fadd_rn(__fmul_rn(x0, sa), __fmul_rn(sb, eps));          // :869-872
  }
  __device__ __forceinline__ void end(const EpiOutParams&, int, int) const {}
};

struct OutDpm {   // mode 7: no noise; the x0 history replaces PLMS's eps ring
  float cx, c0, cc, cp;
  bool second;            // this step is second order
  const float* prev;      // x0 of evaluation k - 1
  float* own;             // slot of evaluation k
  struct In { float x, h; };
  __device__ __forceinline__ OutDpm(const EpiOutParams& p, int) {
    const StepState st = load_step_state(p.state);
    const int k = st.done, i = st.cur;
    const float* row = p.sched_dpm + static_cast<size_t>(i) * SCHED_DPM_STRIDE;
    cx = row[0]; c0 = row[1]; cc = row[2]; cp = row[3];
    second = p.order == 2 && k != 0 && i != 0;
    const size_t slot = static_cast<size_t>(p.B) * p.J * p.T;
    own = p.x0_hist + static_cast<size_t>(k & 1) * slot;
    prev = p.x0_hist + static_cast<size_t>((k + 1) & 1) * slot;
  }
  __device__ __forceinline__ In load(const EpiOutParams& p, bool in, size_t idx, int, int) const {
    return {in ? p.x_t[idx] : 0.f, in && second ? prev[idx] : 0.f};
  }
  __device__ __forceinline__ void store(const EpiOutParams& p, size_t idx, float x0, const In& v) const {
    own[idx] = x0;
    if (p.pred_xstart != nullptr) p.pred_xstart[idx] = x0;
    const float base = __fmul_rn(cx, v.x);
    p.x_out[idx] = second ? __fmaf_rn(cp, v.h, __fmaf_rn(cc, x0, base)) : __fmaf_rn(c0, x0, base);
  }
  __device__ __forceinline__ void end(const EpiOutParams&, int, int) const {}
};

// approx_standard_normal_cdf (diffusion/losses.py:42-47) in fp32 in torch's operation order: pow(x, 3) = (x*x)*x
__device__ __forceinline__ float vb_approx_cdf(float x) {
  const float x3 = __fmul_rn(__fmul_rn(x, x), x);
  const float in = __fmul_rn(0.7978845608028654f, __fadd_rn(x, __fmul_rn(0.044715f, x3)));
  return __fmul_rn(0.5f, __fadd_rn(1.f, tanhf(in)));
}
// -discretized_gaussian_log_likelihood(x, mean, log_scales) for one element (losses.py:50-77); inv_std = exp(-log_scales)
__device__ __forceinline__ float vb_decoder_nll(float x, float mean, float inv_std) {
  const float c = __fsub_rn(x, mean);
  const float cdf_plus = vb_approx_cdf(__fmul_rn(inv_std, __fadd_rn(c, 1.0f / 255.0f)));
  const float cdf_min = vb_approx_cdf(__fmul_rn(inv_std, __fsub_rn(c, 1.0f / 255.0f)));
  float lp;
  if (x < -0.999f) lp = logf(fmaxf(cdf_plus, 1e-12f));
  else if (x > 0.999f) lp = logf(fmaxf(__fsub_rn(1.f, cdf_min), 1e-12f));
  else lp = logf(fmaxf(__fsub_rn(cdf_plus, cdf_min), 1e-12f));
  return -lp;
}

struct OutVb {   // mode 8: writes no sample; the three terms of each element go into the chunk's sums
  float c1, c2, sr, srm1, klc, elv, isd;
  bool t0;
  const float* nz;
  mutable float s_vb = 0.f, s_x = 0.f, s_e = 0.f;
  struct In { float x, xs, n; };
  __device__ __forceinline__ OutVb(const EpiOutParams& p, int b) {
    const StepState st = load_step_state(p.state);
    const float* r = p.sched_vb + static_cast<size_t>(st.cur) * SCHED_VB_STRIDE;
    c1 = r[VB_C1]; c2 = r[VB_C2]; sr = r[VB_SR]; srm1 = r[VB_SRM1];
    klc = r[VB_KL_C]; elv = r[VB_EXP_NEG_LV]; isd = r[VB_INV_STD];
    t0 = st.cur == 0;
    nz = (p.noise != nullptr ? p.noise : st.noise + static_cast<long long>(st.done) * st.noise_step_stride) +
         static_cast<long long>(b) * p.noise_batch_stride;
  }
  __device__ __forceinline__ In load(const EpiOutParams& p, bool in, size_t idx, int col, int t) const {
    return {in ? p.x_t[idx] : 0.f, in ? p.x_start[idx] : 0.f, in ? nz[static_cast<size_t>(col) * p.T + t] : 0.f};
  }
  __device__ __forceinline__ void store(const EpiOutParams& p, size_t idx, float x0, const In& v) const {
    if (p.pred_xstart != nullptr) p.pred_xstart[idx] = x0;
    const float mean = __fadd_rn(__fmul_rn(c1, x0), __fmul_rn(c2, v.x));           // q_posterior of x0 (:254-257)
    float term;
    if (t0) {
      term = vb_decoder_nll(v.xs, mean, isd);
    } else {   // normal_kl (losses.py:12-39): 0.5 * (((-1 + lv2) - lv1) + exp(lv1 - lv2) + (m1 - m2)^2 * exp(-lv2))
      const float tm = __fadd_rn(__fmul_rn(c1, v.xs), __fmul_rn(c2, v.x));
      const float d = __fsub_rn(tm, mean);
      term = __fmul_rn(0.5f, __fadd_rn(klc, __fmul_rn(__fmul_rn(d, d), elv)));
    }
    const float dx = __fsub_rn(x0, v.xs);
    const float xm = __fmul_rn(dx, dx);
    const float eps = __fdiv_rn(__fsub_rn(__fmul_rn(sr, v.x), x0), srm1);           // _predict_eps_from_xstart
    const float de = __fsub_rn(eps, v.n);
    const float em = __fmul_rn(de, de);
    s_vb = __fadd_rn(s_vb, term);
    s_x = __fadd_rn(s_x, xm);
    s_e = __fadd_rn(s_e, em);
    if (p.vb_elem != nullptr) {
      const size_t slot = static_cast<size_t>(p.B) * p.J * p.T;
      p.vb_elem[idx] = term;
      p.vb_elem[slot + idx] = xm;
      p.vb_elem[2 * slot + idx] = em;
    }
  }
  // the chunk's sums into slot (row, col0 / 32) of each term: every slot has exactly one writer
  __device__ __forceinline__ void end(const EpiOutParams& p, int row, int col0) const {
    if (col0 >= p.J) return;
    const size_t rows = static_cast<size_t>(p.B) * p.T * p.vb_chunks;
    const size_t i = static_cast<size_t>(row) * p.vb_chunks + col0 / 32;
    p.vb_part[i] = s_vb;
    p.vb_part[rows + i] = s_x;
    p.vb_part[2 * rows + i] = s_e;
  }
};

// Soft inpainting of one x0 element (DESIGN.md, "Refined transitions"): w >= 1 takes the motion, w <= 0 keeps x0, so a
// 0 / 1 weight gives the bool mask's bits; in between (1 - w) x0 + w m in fp32 with no contraction.  The motion is read
// only where it is used.
__device__ __forceinline__ float soft_inpaint(float x0, float w, const float* motion) {
  if (w >= 1.f) return *motion;
  if (w <= 0.f) return x0;
  return __fadd_rn(__fmul_rn(__fsub_rn(1.f, w), x0), __fmul_rn(w, *motion));
}

// The per-element tail of the output step, after x0 is formed: inpainting (bool mask or soft weight), the clamp of
// clip_denoised, then the update's store.  The output epilogue and the joint-guidance step kernel (joint_guidance.cuh)
// share it.
template <class Update>
__device__ __forceinline__ void out_tail(const EpiOutParams& p, const Update& u, size_t idx, float x0,
                                         const typename Update::In& v) {
  if (p.inpaint_mask != nullptr && p.inpaint_mask[idx]) x0 = p.inpaint_motion[idx];
  if (p.inpaint_weight != nullptr) x0 = soft_inpaint(x0, p.inpaint_weight[idx], p.inpaint_motion + idx);
  if (p.clip_denoised) x0 = fminf(fmaxf(x0, -1.f), 1.f);
  u.store(p, idx, x0, v);
}

// One GEMM instantiation per update family, so that the PLMS, inversion, DPM-Solver++ and bound epilogues leave the
// DDPM / DDIM kernel as it is.
template <class Update>
struct EpiOut {
  static constexpr int SMEM_PER_WARP = 1024;  // unused
  using Params = EpiOutParams;
  static __device__ __forceinline__ void chunk(EpiCtx& ctx, const Params& p, uint32_t (&raw)[32], int row0, int col0) {
    const int row = row0 + ctx.lane;
    if (row >= ctx.M) return;
    const int b = row / p.T, t = row - b * p.T;
    const Update u(p, b);
    // x_out may alias x_t, x_step and the ring slots (in-place loop): every load of a 16-column group is issued before
    // its first store, so that they are all in flight together (consecutive lanes = consecutive frames => each load /
    // store is one coalesced line), and an element is only ever read and written by the thread that owns it.
    const size_t base = static_cast<size_t>(b) * p.J * p.T + t;
#pragma unroll
    for (int h = 0; h < 32; h += 16) {
      typename Update::In v[16];
#pragma unroll
      for (int j = 0; j < 16; ++j) {
        const int col = col0 + h + j;
        v[j] = u.load(p, col < p.J, base + static_cast<size_t>(col) * p.T, col, t);
      }
#pragma unroll
      for (int j = 0; j < 16; ++j) {
        const int col = col0 + h + j;
        if (col >= p.J) continue;
        const size_t idx = base + static_cast<size_t>(col) * p.T;
        out_tail(p, u, idx, __uint_as_float(raw[h + j]) + __ldg(p.bias + col), v[j]);
      }
    }
    u.end(p, row, col0);
  }
  static __device__ __forceinline__ void finish(EpiCtx&) {}
};

}  // namespace b200
