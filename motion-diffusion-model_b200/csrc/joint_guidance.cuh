// Joint-position control (DESIGN.md, "Joint-position control"): K gradient steps x0 <- x0 - step * grad G(x0) on
//   G(x0) = 1/2 sum_{t,j} w[j,t] |p(x0 * std + mean)[t,j] - c[j,:,t]|^2,   p = recover_from_ric (postprocess.cuh),
// then the output step's per-element tail.  One CTA per motion, one thread per frame (T <= 256); the features p depends
// on (the R = 4 + 3(J-1) "ric features": root yaw velocity, root XZ velocity, root height, root-relative joints) stay in
// shared memory, normalised, for all K iterations.  Per iteration:
//   forward   yaw[t] = sum_{u<t} r[u];  w[t] = rot(yaw[t]) v[t-1] (w[0] = 0);  P[t] = sum_{u<=t} w[u];
//             joint j > 0: rot(yaw[t]) q_j[t] + P[t] in x / z, q_j[t].y in y;  the root: (P.x, height, P.z)
//   adjoint   e = w (p - c);  dG/dq_j = rot(yaw)^T e;  gP[t] = sum_j e_xz;  gW[u] = sum_{t>=u} gP[t];
//             dG/dv[t-1] = rot(yaw[t])^T gW[t];  gyaw[t] = sum_j 2 (e_z r_x - e_x r_z) + 2 (gW_z w_x - gW_x w_z)
//             (d rot(yaw) a / d yaw = 2 (-(rot a)_z, (rot a)_x): the quaternion (cos yaw, 0, sin yaw, 0) turns by 2 yaw);
//             dG/dr[u] = sum_{t>u} gyaw[t];  dG/dx0 = dG/dx * std
// Per-frame arithmetic is fp32; the four scans and the loss accumulate in fp64 across the block (warp shuffles, then the
// warp totals), so their error does not grow with T.  Features a thread's frame alone reads (height, joints) are updated
// as soon as their gradient is known; the yaw and root velocities, which other frames read, after the last scan.
#pragma once
#include <cuda_runtime.h>

#include "epilogues.cuh"
#include "postprocess.cuh"
#include "ptx.cuh"

namespace b200 {

constexpr int JG_THREADS = 256;                 // one thread per frame
constexpr int JG_WARPS = JG_THREADS / 32;
constexpr int JG_MAX_FRAMES = JG_THREADS;
constexpr int JG_MAX_FEATS = 4 + 3 * 21;        // HumanML3D: 22 joints

// The guidance inputs: caller-owned device tensors (mean, std [D]; target [B, J, 3, T]; weight [B, J, T]) and the user's
// step size and iteration count.
struct JointGuide {
  const float* mean;
  const float* std;
  const float* target;
  const float* weight;
  float step;
  int iters;
};

// Shared memory of the guidance: xs [R, T] floats, mean / std of the R features, the velocity adjoints handed one frame
// back [2, T], and the scans' warp totals.
__host__ __device__ constexpr size_t jg_smem_bytes(int T, int R) {
  return static_cast<size_t>(JG_WARPS) * 3 * sizeof(double) + (static_cast<size_t>(R) * T + 2 * R + 2 * T) * sizeof(float);
}

// Inclusive scan over the block's threads (REV: from the last thread down) of N fp64 values per thread.  Every thread of
// the block calls it; it leaves `sh` free for the next call.
template <int N, bool REV>
__device__ __forceinline__ void jg_scan(double (&v)[N], double* sh) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
#pragma unroll
    for (int c = 0; c < N; ++c) {
      const double n = REV ? __shfl_down_sync(0xffffffffu, v[c], o) : __shfl_up_sync(0xffffffffu, v[c], o);
      if (REV ? lane + o < 32 : lane >= o) v[c] += n;
    }
  }
  if (lane == (REV ? 0 : 31)) {
#pragma unroll
    for (int c = 0; c < N; ++c) sh[warp * N + c] = v[c];
  }
  __syncthreads();
  double off[N];
#pragma unroll
  for (int c = 0; c < N; ++c) off[c] = 0.0;
  for (int w = 0; w < JG_WARPS; ++w) {
    if (REV ? w > warp : w < warp) {
#pragma unroll
      for (int c = 0; c < N; ++c) off[c] += sh[w * N + c];
    }
  }
#pragma unroll
  for (int c = 0; c < N; ++c) v[c] += off[c];
  __syncthreads();
}

// x0[f] <- x0[f] - (step * std[f]) * g; a zero gradient leaves x0 bit for bit (a -0 gradient would turn -0 into +0)
__device__ __forceinline__ void jg_descend(float* x0, float step_sd, float g) {
  if (g != 0.f) *x0 = __fsub_rn(*x0, __fmul_rn(step_sd, g));
}

// The K guidance iterations of motion b on xs (its R ric features, normalised, [R, T] in shared memory; mu / sd the
// features' mean and std).  loss (nullable) [K + 1, B] receives G before each iteration and after the last one.
// Every thread of the block calls it.
__device__ void joint_guidance_iterate(float* xs, const float* mu, const float* sd, float* gv, double* sh, const JointGuide& g,
                                       int b, int B, int T, int J, float* loss) {
  const int t = threadIdx.x;
  const bool act = t < T;
  const float* tg = g.target + static_cast<size_t>(b) * J * 3 * T + t;
  const float* wt = g.weight + static_cast<size_t>(b) * J * T + t;
  auto X = [&](int f, int u) { return __fadd_rn(__fmul_rn(xs[f * T + u], sd[f]), mu[f]); };
  for (int k = 0; k <= g.iters; ++k) {
    const bool upd = k < g.iters;
    if (!upd && loss == nullptr) break;
    // forward: yaw = exclusive prefix sum of the yaw velocity
    double a1[1] = {act && t > 0 ? static_cast<double>(X(0, t - 1)) : 0.0};
    jg_scan<1, false>(a1, sh);
    const float yaw = static_cast<float>(a1[0]);
    const float c = cosf(yaw), s = sinf(yaw);
    // world-frame root velocity, root XZ = its inclusive prefix sum
    float wx = 0.f, wz = 0.f;
    if (act && t > 0) ric_rot(c, s, X(1, t - 1), X(2, t - 1), &wx, &wz);
    double a2[2] = {wx, wz};
    jg_scan<2, false>(a2, sh);
    const float px = static_cast<float>(a2[0]), pz = static_cast<float>(a2[1]);
    // joints: residuals, loss, the position / yaw adjoints of this frame, and the descent on height and joints
    float gpx = 0.f, gpz = 0.f, gyaw = 0.f;
    double lsum = 0.0;
    if (act) {
      for (int j = 0; j < J; ++j) {
        const float w = __ldcg(wt + static_cast<size_t>(j) * T);
        if (w == 0.f) continue;   // a free joint: its target is never read
        const float* cj = tg + static_cast<size_t>(j) * 3 * T;
        const int f = j == 0 ? 3 : 4 + 3 * (j - 1);   // the feature of the y coordinate's first input
        float rx = 0.f, rz = 0.f, qx = 0.f, qy, qz = 0.f;
        if (j == 0) {
          qy = X(3, t);
        } else {
          qx = X(f, t); qy = X(f + 1, t); qz = X(f + 2, t);
          ric_rot(c, s, qx, qz, &rx, &rz);
        }
        const float dx = __fsub_rn(__fadd_rn(rx, px), __ldcg(cj));
        const float dy = __fsub_rn(qy, __ldcg(cj + T));
        const float dz = __fsub_rn(__fadd_rn(rz, pz), __ldcg(cj + 2 * T));
        lsum += 0.5 * static_cast<double>(w) * (static_cast<double>(dx) * dx + static_cast<double>(dy) * dy +
                                                static_cast<double>(dz) * dz);
        const float ex = __fmul_rn(w, dx), ey = __fmul_rn(w, dy), ez = __fmul_rn(w, dz);
        gpx = __fadd_rn(gpx, ex);
        gpz = __fadd_rn(gpz, ez);
        if (j == 0) {
          if (upd) jg_descend(&xs[3 * T + t], __fmul_rn(g.step, sd[3]), ey);
          continue;
        }
        gyaw = __fadd_rn(gyaw, __fmul_rn(2.f, __fsub_rn(__fmul_rn(ez, rx), __fmul_rn(ex, rz))));
        if (upd) {
          float gx, gz;
          ric_rot(c, -s, ex, ez, &gx, &gz);   // rot(yaw)^T = rot(-yaw)
          jg_descend(&xs[f * T + t], __fmul_rn(g.step, sd[f]), gx);
          jg_descend(&xs[(f + 1) * T + t], __fmul_rn(g.step, sd[f + 1]), ey);
          jg_descend(&xs[(f + 2) * T + t], __fmul_rn(g.step, sd[f + 2]), gz);
        }
      }
    }
    // gW = suffix sum of the position adjoint; the loss rides along as a third component (total at thread 0)
    double a3[3] = {gpx, gpz, lsum};
    jg_scan<3, true>(a3, sh);
    if (t == 0 && loss != nullptr) loss[static_cast<size_t>(k) * B + b] = static_cast<float>(a3[2]);
    if (!upd) break;
    const float gwx = static_cast<float>(a3[0]), gwz = static_cast<float>(a3[1]);
    if (act && t > 0) {
      gyaw = __fadd_rn(gyaw, __fmul_rn(2.f, __fsub_rn(__fmul_rn(gwz, wx), __fmul_rn(gwx, wz))));
      float gx, gz;
      ric_rot(c, -s, gwx, gwz, &gx, &gz);   // the adjoint of v[t - 1]
      gv[t - 1] = gx;
      gv[T + t - 1] = gz;
    }
    // the yaw-velocity adjoint: exclusive suffix sum of the yaw adjoint
    double a4[1] = {gyaw};
    jg_scan<1, true>(a4, sh);
    if (act) {
      const float gr = static_cast<float>(a4[0] - static_cast<double>(gyaw));
      jg_descend(&xs[t], __fmul_rn(g.step, sd[0]), gr);
      if (t < T - 1) {
        jg_descend(&xs[T + t], __fmul_rn(g.step, sd[1]), gv[t]);
        jg_descend(&xs[2 * T + t], __fmul_rn(g.step, sd[2]), gv[T + t]);
      }
    }
    __syncthreads();   // the next iteration reads the neighbours' velocities
  }
}

// The guidance of one motion around joint_guidance_iterate: shared memory carved, ric features of x0 [B, D, T] loaded
// (through L2: x0 was written by the kernel before).  Returns the shared-memory view of the guided features.
__device__ __forceinline__ float* joint_guidance_run(const JointGuide& g, const float* x0, int B, int T, int D, float* loss) {
  extern __shared__ double jg_smem[];
  const int J = D == 263 ? 22 : 21, R = 4 + 3 * (J - 1), b = blockIdx.x;
  double* sh = jg_smem;
  float* xs = reinterpret_cast<float*>(jg_smem + JG_WARPS * 3);
  float* mu = xs + R * T;
  float* sd = mu + R;
  float* gv = sd + R;
  const float* xb = x0 + static_cast<size_t>(b) * D * T;
  for (int i = threadIdx.x; i < R * T; i += blockDim.x) xs[i] = __ldcg(xb + i);
  for (int i = threadIdx.x; i < R; i += blockDim.x) {
    mu[i] = __ldcg(g.mean + i);
    sd[i] = __ldcg(g.std + i);
  }
  __syncthreads();
  joint_guidance_iterate(xs, mu, sd, gv, sh, g, b, B, T, J, loss);
  return xs;
}

// The guidance as read from its device descriptor (b200mdm_set_joint_guidance uploads it, so a captured step graph
// follows a new step size or new targets)
__device__ __forceinline__ JointGuide load_joint_guide(const JointGuide* d) {
  JointGuide g;
  g.mean = reinterpret_cast<const float*>(__ldcg(reinterpret_cast<const unsigned long long*>(&d->mean)));
  g.std = reinterpret_cast<const float*>(__ldcg(reinterpret_cast<const unsigned long long*>(&d->std)));
  g.target = reinterpret_cast<const float*>(__ldcg(reinterpret_cast<const unsigned long long*>(&d->target)));
  g.weight = reinterpret_cast<const float*>(__ldcg(reinterpret_cast<const unsigned long long*>(&d->weight)));
  g.step = __ldcg(&d->step);
  g.iters = __ldcg(&d->iters);
  return g;
}

// The guided step of motion blockIdx.x: x0 (the output projection + bias after the CFG blend, [B, D, T], written by the
// MODE_X0 output GEMM) -> guidance -> the output step's tail (inpainting, clamp, the DDPM / DDIM update of p.mode) for
// every element of the motion, reading the step's noise as OutStep does.  grid = B, block = JG_THREADS,
// dynamic shared memory jg_smem_bytes(T, R).
__global__ void __launch_bounds__(JG_THREADS) joint_guidance_step_kernel(const JointGuide* guide, const float* x0,
                                                                         const EpiOutParams p) {
  pdl_launch_dependents();
  pdl_wait();
  const int T = p.T, D = p.J, b = blockIdx.x, t = threadIdx.x;
  const JointGuide g = load_joint_guide(guide);
  const int R = D == 263 ? 67 : 64;
  const float* xs = joint_guidance_run(g, x0, p.B, T, D, nullptr);
  if (t >= T) return;
  const OutStep u(p, b);
  const size_t base = static_cast<size_t>(b) * D * T + t;
  for (int f = 0; f < D; ++f) {
    const size_t idx = base + static_cast<size_t>(f) * T;
    const OutStep::In v = u.load(p, true, idx, f, t);
    out_tail(p, u, idx, f < R ? xs[f * T + t] : __ldcg(x0 + idx), v);
  }
}

// b200mdm_test_joint_guidance: the guidance alone, x0_out [B, D, T] = guided x0 (features past the ric features copied).
__global__ void __launch_bounds__(JG_THREADS) joint_guidance_test_kernel(const JointGuide g, const float* x0, float* x0_out,
                                                                         float* loss, int B, int T, int D) {
  const int R = D == 263 ? 67 : 64, b = blockIdx.x;
  const float* xs = joint_guidance_run(g, x0, B, T, D, loss);
  const size_t base = static_cast<size_t>(b) * D * T;
  for (int i = threadIdx.x; i < D * T; i += blockDim.x) x0_out[base + i] = i < R * T ? xs[i] : x0[base + i];
}

}  // namespace b200
