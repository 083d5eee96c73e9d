// Multi-prompt guidance (DESIGN.md, "Multi-prompt guidance"): the packed batch holds G = K + 1 groups of B motions, the
// K prompts' groups first and the unconditional group last.  The output GEMM writes every group's raw x0 into
// x0g [G, B, D, T]; compose_step_kernel forms
//   x0[b, f, t] = x0_u + sum_{k=0..K-1} w[b, k, f, t] (x0_k - x0_u)
// in fp32, k ascending, with no contraction, then runs the output step's per-element tail (out_tail: inpainting, the
// clamp of clip_denoised, the update of the sampler) exactly as the output epilogue does.
#pragma once
#include <cuda_runtime.h>

#include "epilogues.cuh"
#include "ptx.cuh"

namespace b200 {

constexpr int MP_MAX_PROMPTS = 8;      // B200MDM_MAX_PROMPTS
constexpr int MP_THREADS = 256;

// The prompt weights: a caller-owned fp32 tensor read as w[b * sb + k * sk + f * sf + t * st] (a stride of 0 broadcasts
// that dimension) and the prompt count K.
struct PromptWeight {
  const float* w;
  long long sb, sk, sf, st;
  int K;
};

// Every reader goes through L2 (as load_step_state): the step graph reads the descriptor the last
// b200mdm_set_prompt_weight uploaded.
__device__ __forceinline__ PromptWeight load_prompt_weight(const PromptWeight* d) {
  PromptWeight g;
  g.w = reinterpret_cast<const float*>(__ldcg(reinterpret_cast<const unsigned long long*>(&d->w)));
  g.sb = __ldcg(&d->sb);
  g.sk = __ldcg(&d->sk);
  g.sf = __ldcg(&d->sf);
  g.st = __ldcg(&d->st);
  g.K = __ldcg(&d->K);
  return g;
}

// The composed x0 of element (b, f, t) of x0g [K + 1, B, D, T]; n = D * T, i = f * T + t.
__device__ __forceinline__ float compose_x0(const PromptWeight& g, const float* x0g, int B, size_t n, int b, size_t i,
                                            int f, int t) {
  const size_t off = static_cast<size_t>(b) * n + i, group = static_cast<size_t>(B) * n;
  const float xu = __ldcg(x0g + static_cast<size_t>(g.K) * group + off);
  const float* wb = g.w + b * g.sb + f * g.sf + t * g.st;
  float x0 = xu;
  for (int k = 0; k < g.K; ++k) {
    const float xk = __ldcg(x0g + static_cast<size_t>(k) * group + off);
    x0 = __fadd_rn(x0, __fmul_rn(__ldg(wb + k * g.sk), __fsub_rn(xk, xu)));
  }
  return x0;
}

// One thread per element of motion blockIdx.y: the composed x0, then the step's tail of the Update family (OutStep for
// modes 0-2, OutPlms, OutDpm, OutReverse), reading x_t, noise and history as EpiOut does.  x_out may alias x_t: every
// element is read and written by the thread that owns it.
template <class Update>
__global__ void __launch_bounds__(MP_THREADS) compose_step_kernel(const PromptWeight* desc, const float* x0g,
                                                                  const EpiOutParams p) {
  pdl_launch_dependents();
  pdl_wait();
  const int b = blockIdx.y;
  const size_t n = static_cast<size_t>(p.J) * p.T;
  const size_t i = static_cast<size_t>(blockIdx.x) * MP_THREADS + threadIdx.x;
  if (i >= n) return;
  const PromptWeight g = load_prompt_weight(desc);
  const int f = static_cast<int>(i / p.T), t = static_cast<int>(i - static_cast<size_t>(f) * p.T);
  const Update u(p, b);
  const size_t idx = static_cast<size_t>(b) * n + i;
  const typename Update::In v = u.load(p, true, idx, f, t);
  out_tail(p, u, idx, compose_x0(g, x0g, p.B, n, b, i, f, t), v);
}

}  // namespace b200
