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
// FOOT (DESIGN.md, "Foot contact and floor"): G gains 1/2 lc sum_{k,t} kappa_k[t] |Delta_k[t]|^2 over the four foot joints,
// Delta_k[t] = p[t+1, f_k] - p[t, f_k] formed from the root velocity w[t+1] and the rotated root-relative feet (never from
// world positions), and 1/2 lf sum_{t<L, j} min(p[t,j].y - h, 0)^2; both only add to e, the existing chain is unchanged.
// The neighbour frame's w and feet, and kappa * Delta of the previous pair, go through shared memory.
// SCENE (DESIGN.md, "Scene: obstacles and uneven ground"), on top of FOOT: two 2D grids over the XZ plane, sampled
// bilinearly at every joint's world XZ (scene_sample; read through L2).  G gains 1/2 lo sum_{t<L, j} max(r - S, 0)^2 with
// S the obstacles' signed distance, and the floor term's height becomes h + H(x, z) with H the terrain; both only add to e
// (in x / z through the grids' gradients), the existing chain is unchanged.
// INTER (DESIGN.md, "Several characters in one scene"), on top of SCENE: the B motions are B / C scenes of C characters,
// one thread-block cluster of C CTAs per scene.  Each CTA places its frame's joints in the scene frame, Q = rot(phi) p +
// (X, 0, Z), and writes them to its shared memory; after a cluster barrier every thread reads its partners' frame-t rows
// (mapa + ld.shared::cluster) and adds the avoidance adjoint la max(r - d, 0) and the reach rows' w max(d - delta, 0),
// along the unit vector between the joints and rotated back by rot(phi)^T, to e.  Every character reads the positions
// of the same iteration (Jacobi descent on the scene's energy): the next iteration's writes wait on a second cluster
// barrier that follows the reads.
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

// The foot-contact and floor terms (b200mdm_set_foot_guidance): contact [B, 4, T] fp32 (nullptr: kappa derived from x0's
// contact features), lengths [B] (nullptr: every frame), the weights lc / lf and the floor height.
struct FootGuide {
  const float* contact;
  const int* lengths;
  float contact_w, floor_w, floor_h;
};

// A 2D grid over the XZ plane (b200mdm_grid): values [gz, gx] fp32, sample b's at v + b * stride (stride 0: shared);
// row i at z = z0 + i * cell, column k at x = x0 + k * cell.  v == nullptr: no grid.
struct SceneGrid {
  const float* v;
  long long stride;
  int gz, gx;
  float x0, z0, cell;
};

// The scene terms (b200mdm_set_scene_guidance): the obstacles' signed distance (nullptr values: none) with weight lo and
// margin r, and the terrain heights H added to the floor height (nullptr values: a flat floor).
struct SceneGuide {
  SceneGrid sdf, terrain;
  float obstacle_w, margin;
};

// One reach row (b200mdm_set_interaction_guidance): joint j of scene-local character a toward joint k of character b,
// within `reach` metres
struct InterPair {
  int a, j, b, k;
  float reach;
};

// The interaction terms (b200mdm_set_interaction_guidance): C characters per scene, placement [B, 3] (x, z, phi) fp32,
// n_pairs reach rows and their per-frame weights [N, T] at pair_w + s * pw_stride for scene s (pw_stride 0: shared),
// the avoidance weight la and margin r.
struct InterGuide {
  const float* placement;
  const InterPair* pairs;
  const float* pair_w;
  long long pw_stride;
  int chars, n_pairs;
  float weight, margin;
};

// The guidance descriptor, which the step kernels read from the engine's device copy and the test kernels take by value:
// the foot terms follow the joint terms, the scene terms the foot terms and the interaction terms the scene terms, so a
// kernel without them reads what it always read
struct GuideDesc {
  JointGuide j;
  FootGuide f;
  SceneGuide s;
  InterGuide i;
};

// Shared memory of the guidance: xs [R, T] floats, mean / std of the R features, the velocity adjoints handed one frame
// back [2, T], and the scans' warp totals.
__host__ __device__ constexpr size_t jg_smem_bytes(int T, int R) {
  return static_cast<size_t>(JG_WARPS) * 3 * sizeof(double) + (static_cast<size_t>(R) * T + 2 * R + 2 * T) * sizeof(float);
}
// ... and with the foot terms: each frame's w and four rotated feet [14, FG_LD] and kappa * Delta of its pair [12, FG_LD]
// (a fixed row pitch, so every access is the thread's base address plus an immediate)
constexpr int FG_NB = 14, FG_CD = 12, FG_LD = JG_MAX_FRAMES;
__host__ __device__ constexpr size_t fg_smem_bytes(int T, int R) {
  return jg_smem_bytes(T, R) + static_cast<size_t>(FG_NB + FG_CD) * FG_LD * sizeof(float);
}
// ... and with the interaction terms: each frame's scene-frame joints [3 J, FG_LD] (J <= 22), which the cluster reads
constexpr int IG_ROWS = 3 * 22;
__host__ __device__ constexpr size_t ig_smem_bytes(int T, int R) {
  return fg_smem_bytes(T, R) + static_cast<size_t>(IG_ROWS) * FG_LD * sizeof(float);
}
constexpr int IG_MAX_CHARS = 8;   // the portable cluster size

// The foot joints of contact channels D - 4 .. D - 1 (the reference's cat([..., feet_l, feet_r]) with fid_l, fid_r)
__host__ __device__ constexpr int foot_joint(int J, int k) {
  return J == 22 ? (k == 0 ? 7 : k == 1 ? 10 : k == 2 ? 8 : 11) : (k == 0 ? 19 : k == 1 ? 20 : k == 2 ? 14 : 15);
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

// The bilinear interpolant of grid G (sample b) at (x, z) and its gradient (*dx, *dz), fp32: u = clamp((x - x0) / cell,
// 0, gx - 1), cell column k = min(floor(u), gx - 2), alpha = u - k (and v, i, beta in z); the gradient is the cell's,
// 0 along a clamped axis.
__device__ __forceinline__ float scene_sample(const SceneGrid& G, int b, float x, float z, float* dx, float* dz) {
  const float* V = G.v + static_cast<size_t>(b) * static_cast<size_t>(G.stride);
  const float ur = __fdiv_rn(__fsub_rn(x, G.x0), G.cell), vr = __fdiv_rn(__fsub_rn(z, G.z0), G.cell);
  const float u = fminf(fmaxf(ur, 0.f), static_cast<float>(G.gx - 1));
  const float v = fminf(fmaxf(vr, 0.f), static_cast<float>(G.gz - 1));
  const int k = min(static_cast<int>(u), G.gx - 2), i = min(static_cast<int>(v), G.gz - 2);
  const float a = __fsub_rn(u, static_cast<float>(k)), c = __fsub_rn(v, static_cast<float>(i));
  const float* r0 = V + static_cast<size_t>(i) * G.gx + k;
  const float v00 = __ldcg(r0), v01 = __ldcg(r0 + 1), v10 = __ldcg(r0 + G.gx), v11 = __ldcg(r0 + G.gx + 1);
  const float e0 = __fsub_rn(v01, v00), e1 = __fsub_rn(v11, v10);   // x differences of rows i, i + 1
  const float f0 = __fsub_rn(v10, v00), f1 = __fsub_rn(v11, v01);   // z differences of columns k, k + 1
  const bool cx = ur == u, cz = vr == v;                            // false on a clamped axis (or a NaN coordinate)
  *dx = cx ? __fdiv_rn(__fadd_rn(__fmul_rn(__fsub_rn(1.f, c), e0), __fmul_rn(c, e1)), G.cell) : 0.f;
  *dz = cz ? __fdiv_rn(__fadd_rn(__fmul_rn(__fsub_rn(1.f, a), f0), __fmul_rn(a, f1)), G.cell) : 0.f;
  const float w0 = __fadd_rn(v00, __fmul_rn(a, e0)), w1 = __fadd_rn(v10, __fmul_rn(a, e1));
  return __fadd_rn(w0, __fmul_rn(c, __fsub_rn(w1, w0)));
}

// x0[f] <- x0[f] - (step * std[f]) * g; a zero gradient leaves x0 bit for bit (a -0 gradient would turn -0 into +0)
__device__ __forceinline__ void jg_descend(float* x0, float step_sd, float g) {
  if (g != 0.f) *x0 = __fsub_rn(*x0, __fmul_rn(step_sd, g));
}

// The foot terms' per-frame constants: kappa_k[t] of this thread's pair (t, t + 1), whether the floor acts on its frame,
// and the shared-memory exchange buffers nb [FG_NB, T] and cd [FG_CD, T] (unused when !FOOT)
struct FootFrame {
  float kap[4];
  bool floor;
  float* nb;
  float* cd;
};

// The interaction terms' per-thread constants: this CTA's scene-frame joints q [IG_ROWS, FG_LD] (row 3 j + c), its rank
// in the scene and the scene's first motion, its placement (cos phi, sin phi, X, Z), and bit b of `live` set when
// frame t < L_ab for partner b (unused when !INTER)
struct InterFrame {
  float* q;
  int rank, first;
  float c, s, X, Z;
  unsigned live;
};

// The interaction adjoint of joint j at thread t's frame (own-frame e += rot(phi)^T dG/dQ) and the pairs' loss counted
// at the lower rank, reading the partners' rows of this iteration
__device__ __forceinline__ void inter_joint(const InterGuide& ig, const InterFrame& xf, int j, int J, int T, float* ex,
                                            float* ey, float* ez, double* lsum) {
  const int t = threadIdx.x;
  const float* qo = xf.q + t;
  const float ax = qo[3 * j * FG_LD], ay = qo[(3 * j + 1) * FG_LD], az = qo[(3 * j + 2) * FG_LD];
  const uint32_t q0 = smem_u32(qo);
  float gx = 0.f, gy = 0.f, gz = 0.f;
  // one pair term along Qa - Qb (partner p's joint k): coefficient cf of the unit vector, added to g
  auto pair = [&](int p, int k, float* dx, float* dy, float* dz) {
    const uint32_t r = mapa_shared(q0 + static_cast<uint32_t>(3 * k * FG_LD * sizeof(float)), static_cast<uint32_t>(p));
    *dx = __fsub_rn(ax, ld_shared_cluster_f32(r));
    *dy = __fsub_rn(ay, ld_shared_cluster_f32(r + FG_LD * sizeof(float)));
    *dz = __fsub_rn(az, ld_shared_cluster_f32(r + 2 * FG_LD * sizeof(float)));
    return __fsqrt_rn(__fadd_rn(__fadd_rn(__fmul_rn(*dx, *dx), __fmul_rn(*dy, *dy)), __fmul_rn(*dz, *dz)));
  };
  auto add = [&](float cf, float dx, float dy, float dz) {
    gx = __fadd_rn(gx, __fmul_rn(cf, dx));
    gy = __fadd_rn(gy, __fmul_rn(cf, dy));
    gz = __fadd_rn(gz, __fmul_rn(cf, dz));
  };
  if (ig.weight > 0.f) {   // avoidance against every joint of every partner: -la max(r - d, 0) (Qa - Qb) / d
#pragma unroll 1
    for (int p = 0; p < ig.chars; ++p) {
      if (p == xf.rank || !((xf.live >> p) & 1u)) continue;
#pragma unroll 1
      for (int k = 0; k < J; ++k) {
        float dx, dy, dz;
        const float d = pair(p, k, &dx, &dy, &dz);
        const float m = __fsub_rn(ig.margin, d);
        if (!(m > 0.f)) continue;
        if (xf.rank < p) *lsum += 0.5 * static_cast<double>(ig.weight) * (static_cast<double>(m) * m);
        if (d > 0.f) add(-__fdiv_rn(__fmul_rn(ig.weight, m), d), dx, dy, dz);   // 0 at d = 0
      }
    }
  }
  // the reach rows this joint belongs to, on either side: w max(d - delta, 0) (Qa - Qb) / d
  const float* pw = ig.pair_w + static_cast<size_t>(xf.first / ig.chars) * static_cast<size_t>(ig.pw_stride) + t;
#pragma unroll 1
  for (int n = 0; n < ig.n_pairs; ++n) {
    const InterPair* row = ig.pairs + n;
    const int a = __ldcg(&row->a), b = __ldcg(&row->b);
    int p, k;
    if (a == xf.rank && __ldcg(&row->j) == j) {
      p = b;
      k = __ldcg(&row->k);
    } else if (b == xf.rank && __ldcg(&row->k) == j) {
      p = a;
      k = __ldcg(&row->j);
    } else {
      continue;
    }
    if (!((xf.live >> p) & 1u)) continue;
    const float w = __ldcg(pw + static_cast<size_t>(n) * T);
    if (w == 0.f) continue;
    float dx, dy, dz;
    const float d = pair(p, k, &dx, &dy, &dz);
    const float m = __fsub_rn(d, __ldcg(&row->reach));
    if (!(m > 0.f)) continue;
    if (xf.rank < p) *lsum += 0.5 * static_cast<double>(w) * (static_cast<double>(m) * m);
    add(__fdiv_rn(__fmul_rn(w, m), d), dx, dy, dz);
  }
  if (gx == 0.f && gy == 0.f && gz == 0.f) return;
  // rot(phi)^T back to the character's own frame
  *ex = __fadd_rn(*ex, __fadd_rn(__fmul_rn(xf.c, gx), __fmul_rn(xf.s, gz)));
  *ey = __fadd_rn(*ey, gy);
  *ez = __fadd_rn(*ez, __fsub_rn(__fmul_rn(xf.c, gz), __fmul_rn(xf.s, gx)));
}

// Thread t's frame of this CTA in the scene frame: Q = rot(phi) p + (X, 0, Z) of every joint into xf.q, from the
// forward pass's yaw (c, s) and root position (px, pz)
__device__ __forceinline__ void inter_place(const InterFrame& xf, const float* xs, const float* mu, const float* sd, int T,
                                            int J, float c, float s, float px, float pz) {
  const int t = threadIdx.x;
  auto X = [&](int f) { return __fadd_rn(__fmul_rn(xs[f * T + t], sd[f]), mu[f]); };
  float* q = xf.q + t;
#pragma unroll 1
  for (int j = 0; j < J; ++j) {
    float x = px, y, z = pz;
    if (j == 0) {
      y = X(3);
    } else {
      const int f = 4 + 3 * (j - 1);
      float rx, rz;
      ric_rot(c, s, X(f), X(f + 2), &rx, &rz);
      x = __fadd_rn(rx, px);
      y = X(f + 1);
      z = __fadd_rn(rz, pz);
    }
    q[3 * j * FG_LD] = __fadd_rn(__fsub_rn(__fmul_rn(xf.c, x), __fmul_rn(xf.s, z)), xf.X);
    q[(3 * j + 1) * FG_LD] = y;
    q[(3 * j + 2) * FG_LD] = __fadd_rn(__fadd_rn(__fmul_rn(xf.s, x), __fmul_rn(xf.c, z)), xf.Z);
  }
}

// One iteration's joint pass with the foot terms, for thread t's frame (every thread of the block calls it): the
// neighbour exchange, kappa * Delta of pair (t, t + 1) and its loss, then per joint e = w (p - c) + the floor's and the
// contact pairs' adjoints, into the position / yaw adjoints and the descent on height and joints, as joint_guidance_iterate.
// SCENE: the floor's height gains the terrain, and the obstacles' adjoint joins (sg.obstacle_w is 0 on frames >= L).
// INTER: the frame's scene-frame joints are published to the cluster (after the partners' reads of the previous
// iteration, `wait`), and the interaction adjoint joins.
template <bool SCENE, bool INTER>
__device__ __forceinline__ void foot_iterate(float* xs, const float* mu, const float* sd, const JointGuide& g, const FootGuide& fg,
                                             const FootFrame& ff, const float* tg, const float* wt, int T, int J, bool upd,
                                             float c, float s, float wx, float wz, float px, float pz, float* gpx, float* gpz,
                                             float* gyaw, double* lsum, const SceneGuide& sg, int b, const InterGuide& ig,
                                             const InterFrame& xf, bool wait) {
  const int t = threadIdx.x;
  const bool act = t < T;
  if constexpr (INTER) {
    if (wait) cluster_wait_acquire();
    if (act) inter_place(xf, xs, mu, sd, T, J, c, s, px, pz);
    cluster_arrive_release();
    cluster_wait_acquire();
  }
  auto X = [&](int f) { return __fadd_rn(__fmul_rn(xs[f * T + t], sd[f]), mu[f]); };
  float* nb = ff.nb + t;   // row r of frame t + o: nb[r * FG_LD + o]
  float* cd = ff.cd + t;
  // this frame's root velocity and rotated feet, for frame t - 1
  float rfx[4], qfy[4], rfz[4];
  if (act) {
    nb[0] = wx;
    nb[FG_LD] = wz;
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const int f = 4 + 3 * (foot_joint(J, k) - 1);
      ric_rot(c, s, X(f), X(f + 2), &rfx[k], &rfz[k]);
      qfy[k] = X(f + 1);
      nb[(2 + 3 * k) * FG_LD] = rfx[k];
      nb[(3 + 3 * k) * FG_LD] = qfy[k];
      nb[(4 + 3 * k) * FG_LD] = rfz[k];
    }
  }
  __syncthreads();
  // Delta_k[t] = w[t+1] + rot(yaw[t+1]) q_f[t+1] - rot(yaw[t]) q_f[t] in x / z, q_f[t+1].y - q_f[t].y in y
  if (act) {
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      float dx = 0.f, dy = 0.f, dz = 0.f;
      if (ff.kap[k] != 0.f) {   // kappa is 0 on the last frame
        dx = __fsub_rn(__fadd_rn(nb[1], nb[(2 + 3 * k) * FG_LD + 1]), rfx[k]);
        dy = __fsub_rn(nb[(3 + 3 * k) * FG_LD + 1], qfy[k]);
        dz = __fsub_rn(__fadd_rn(nb[FG_LD + 1], nb[(4 + 3 * k) * FG_LD + 1]), rfz[k]);
        *lsum += 0.5 * static_cast<double>(fg.contact_w) * ff.kap[k] *
                 (static_cast<double>(dx) * dx + static_cast<double>(dy) * dy + static_cast<double>(dz) * dz);
        dx = __fmul_rn(ff.kap[k], dx);
        dy = __fmul_rn(ff.kap[k], dy);
        dz = __fmul_rn(ff.kap[k], dz);
      }
      cd[3 * k * FG_LD] = dx;
      cd[(3 * k + 1) * FG_LD] = dy;
      cd[(3 * k + 2) * FG_LD] = dz;
    }
  }
  __syncthreads();
  if (!act) return;
  // the contact adjoint at (t, f_k): lc (kappa[t-1] Delta[t-1] - kappa[t] Delta[t])
  auto ce = [&](int k, int a) {
    const float prev = t > 0 ? cd[(3 * k + a) * FG_LD - 1] : 0.f;
    return __fmul_rn(fg.contact_w, __fsub_rn(prev, cd[(3 * k + a) * FG_LD]));
  };
#pragma unroll 1
  for (int j = 0; j < J; ++j) {
    const float w = __ldcg(wt + static_cast<size_t>(j) * T);
    const int f = j == 0 ? 3 : 4 + 3 * (j - 1);
    float rx = 0.f, rz = 0.f, qx = 0.f, qy, qz = 0.f;
    if (j == 0) {
      qy = X(3);
    } else {
      qx = X(f); qy = X(f + 1); qz = X(f + 2);
      ric_rot(c, s, qx, qz, &rx, &rz);
    }
    float ex = 0.f, ey = 0.f, ez = 0.f;
    if (w != 0.f) {   // a free joint: its target is never read
      const float* cj = tg + static_cast<size_t>(j) * 3 * T;
      const float dx = __fsub_rn(__fadd_rn(rx, px), __ldcg(cj));
      const float dy = __fsub_rn(qy, __ldcg(cj + T));
      const float dz = __fsub_rn(__fadd_rn(rz, pz), __ldcg(cj + 2 * T));
      *lsum += 0.5 * static_cast<double>(w) * (static_cast<double>(dx) * dx + static_cast<double>(dy) * dy +
                                               static_cast<double>(dz) * dz);
      ex = __fmul_rn(w, dx); ey = __fmul_rn(w, dy); ez = __fmul_rn(w, dz);
    }
    if constexpr (SCENE) {
      const float x = __fadd_rn(rx, px), z = __fadd_rn(rz, pz);   // the joint's world XZ (rx = rz = 0 at the root)
      if (ff.floor) {   // the floor over the terrain: lf min(p.y - h - H, 0), and -lf m dH in x / z
        float hx = 0.f, hz = 0.f;
        const float H = sg.terrain.v != nullptr ? scene_sample(sg.terrain, b, x, z, &hx, &hz) : 0.f;
        const float m = fminf(__fsub_rn(__fsub_rn(qy, fg.floor_h), H), 0.f);
        if (m < 0.f) {
          *lsum += 0.5 * static_cast<double>(fg.floor_w) * (static_cast<double>(m) * m);
          const float lm = __fmul_rn(fg.floor_w, m);
          ey = __fadd_rn(ey, lm);
          ex = __fsub_rn(ex, __fmul_rn(lm, hx));
          ez = __fsub_rn(ez, __fmul_rn(lm, hz));
        }
      }
      if (sg.obstacle_w > 0.f) {   // the obstacles: lo max(r - S, 0), and -lo m dS in x / z
        float sx, sz;
        const float m = fmaxf(__fsub_rn(sg.margin, scene_sample(sg.sdf, b, x, z, &sx, &sz)), 0.f);
        if (m > 0.f) {
          *lsum += 0.5 * static_cast<double>(sg.obstacle_w) * (static_cast<double>(m) * m);
          const float lm = __fmul_rn(sg.obstacle_w, m);
          ex = __fsub_rn(ex, __fmul_rn(lm, sx));
          ez = __fsub_rn(ez, __fmul_rn(lm, sz));
        }
      }
      if constexpr (INTER) inter_joint(ig, xf, j, J, T, &ex, &ey, &ez, lsum);
    } else if (ff.floor) {   // the floor: lf min(p.y - h, 0)
      const float m = fminf(__fsub_rn(qy, fg.floor_h), 0.f);
      if (m < 0.f) {
        *lsum += 0.5 * static_cast<double>(fg.floor_w) * (static_cast<double>(m) * m);
        ey = __fadd_rn(ey, __fmul_rn(fg.floor_w, m));
      }
    }
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      if (j == foot_joint(J, k)) {
        ex = __fadd_rn(ex, ce(k, 0));
        ey = __fadd_rn(ey, ce(k, 1));
        ez = __fadd_rn(ez, ce(k, 2));
      }
    }
    if (ex == 0.f && ey == 0.f && ez == 0.f) continue;
    *gpx = __fadd_rn(*gpx, ex);
    *gpz = __fadd_rn(*gpz, ez);
    if (j == 0) {
      if (upd) jg_descend(&xs[3 * T + t], __fmul_rn(g.step, sd[3]), ey);
      continue;
    }
    *gyaw = __fadd_rn(*gyaw, __fmul_rn(2.f, __fsub_rn(__fmul_rn(ez, rx), __fmul_rn(ex, rz))));
    if (upd) {
      float gx, gz;
      ric_rot(c, -s, ex, ez, &gx, &gz);   // rot(yaw)^T = rot(-yaw)
      jg_descend(&xs[f * T + t], __fmul_rn(g.step, sd[f]), gx);
      jg_descend(&xs[(f + 1) * T + t], __fmul_rn(g.step, sd[f + 1]), ey);
      jg_descend(&xs[(f + 2) * T + t], __fmul_rn(g.step, sd[f + 2]), gz);
    }
  }
}

// The K guidance iterations of motion b on xs (its R ric features, normalised, [R, T] in shared memory; mu / sd the
// features' mean and std).  loss (nullable) [K + 1, B] receives G before each iteration and after the last one.
// Every thread of the block calls it.
template <bool FOOT, bool SCENE, bool INTER>
__device__ void joint_guidance_iterate(float* xs, const float* mu, const float* sd, float* gv, double* sh, const JointGuide& g,
                                       int b, int B, int T, int J, float* loss, const FootGuide& fg, const FootFrame& ff,
                                       const SceneGuide& sg, const InterGuide& ig, const InterFrame& xf) {
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
    if constexpr (FOOT) {
      foot_iterate<SCENE, INTER>(xs, mu, sd, g, fg, ff, tg, wt, T, J, upd, c, s, wx, wz, px, pz, &gpx, &gpz, &gyaw, &lsum, sg, b,
                                 ig, xf, k > 0);
      if constexpr (INTER) cluster_arrive_release();   // this iteration's reads of the partners' rows are done
    } else if (act) {
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
  if constexpr (INTER) cluster_wait_acquire();   // no CTA leaves while a partner may still read its rows
}

// The guidance of one motion around joint_guidance_iterate: shared memory carved, ric features of x0 [B, D, T] loaded
// (through L2: x0 was written by the kernel before).  Returns the shared-memory view of the guided features.
template <bool FOOT, bool SCENE, bool INTER>
__device__ __forceinline__ float* joint_guidance_run(const JointGuide& g, const FootGuide& fg, SceneGuide sg, const float* x0,
                                                     int B, int T, int D, float* loss, const InterGuide& ig) {
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
  FootFrame ff{};
  if constexpr (FOOT) {
    // kappa of pair (t, t + 1), read once: the guidance never changes the contact features
    const int t = threadIdx.x;
    const int L = fg.lengths != nullptr ? min(max(__ldcg(fg.lengths + b), 0), T) : T;
    for (int k = 0; k < 4; ++k) {
      float kap = 0.f;
      if (t + 1 < T) {
        if (fg.contact != nullptr) {
          kap = __ldcg(fg.contact + (static_cast<size_t>(b) * 4 + k) * T + t);
        } else if (t + 1 < L) {
          const int f = D - 4 + k;
          kap = __fadd_rn(__fmul_rn(__ldcg(xb + static_cast<size_t>(f) * T + t), __ldcg(g.std + f)), __ldcg(g.mean + f)) > 0.5f
                    ? 1.f : 0.f;
        }
      }
      ff.kap[k] = kap;
    }
    ff.floor = fg.floor_w > 0.f && t < L;
    if constexpr (SCENE) {
      if (t >= L) sg.obstacle_w = 0.f;   // the obstacles act on frames t < L
    }
    ff.nb = gv + 2 * T;
    ff.cd = ff.nb + FG_NB * FG_LD;
  }
  InterFrame xf{};
  if constexpr (INTER) {
    const int t = threadIdx.x;
    xf.q = ff.cd + FG_CD * FG_LD;
    xf.rank = b % ig.chars;
    xf.first = b - xf.rank;
    const float phi = __ldcg(ig.placement + 3 * b + 2);
    xf.c = cosf(phi);
    xf.s = sinf(phi);
    xf.X = __ldcg(ig.placement + 3 * b);
    xf.Z = __ldcg(ig.placement + 3 * b + 1);
    // partner p acts on frame t < min(L_self, L_p)
    auto len = [&](int m) { return fg.lengths != nullptr ? min(max(__ldcg(fg.lengths + m), 0), T) : T; };
    const int L = len(b);
    for (int p = 0; p < ig.chars; ++p)
      if (t < L && t < len(xf.first + p)) xf.live |= 1u << p;
  }
  __syncthreads();
  joint_guidance_iterate<FOOT, SCENE, INTER>(xs, mu, sd, gv, sh, g, b, B, T, J, loss, fg, ff, sg, ig, xf);
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
__device__ __forceinline__ FootGuide load_foot_guide(const FootGuide* d) {
  FootGuide f;
  f.contact = reinterpret_cast<const float*>(__ldcg(reinterpret_cast<const unsigned long long*>(&d->contact)));
  f.lengths = reinterpret_cast<const int*>(__ldcg(reinterpret_cast<const unsigned long long*>(&d->lengths)));
  f.contact_w = __ldcg(&d->contact_w);
  f.floor_w = __ldcg(&d->floor_w);
  f.floor_h = __ldcg(&d->floor_h);
  return f;
}
__device__ __forceinline__ SceneGrid load_scene_grid(const SceneGrid* d) {
  SceneGrid G;
  G.v = reinterpret_cast<const float*>(__ldcg(reinterpret_cast<const unsigned long long*>(&d->v)));
  G.stride = __ldcg(&d->stride);
  G.gz = __ldcg(&d->gz);
  G.gx = __ldcg(&d->gx);
  G.x0 = __ldcg(&d->x0);
  G.z0 = __ldcg(&d->z0);
  G.cell = __ldcg(&d->cell);
  return G;
}
__device__ __forceinline__ SceneGuide load_scene_guide(const SceneGuide* d) {
  SceneGuide s;
  s.sdf = load_scene_grid(&d->sdf);
  s.terrain = load_scene_grid(&d->terrain);
  s.obstacle_w = __ldcg(&d->obstacle_w);
  s.margin = __ldcg(&d->margin);
  return s;
}
__device__ __forceinline__ InterGuide load_inter_guide(const InterGuide* d) {
  InterGuide i;
  i.placement = reinterpret_cast<const float*>(__ldcg(reinterpret_cast<const unsigned long long*>(&d->placement)));
  i.pairs = reinterpret_cast<const InterPair*>(__ldcg(reinterpret_cast<const unsigned long long*>(&d->pairs)));
  i.pair_w = reinterpret_cast<const float*>(__ldcg(reinterpret_cast<const unsigned long long*>(&d->pair_w)));
  i.pw_stride = __ldcg(&d->pw_stride);
  i.chars = __ldcg(&d->chars);
  i.n_pairs = __ldcg(&d->n_pairs);
  i.weight = __ldcg(&d->weight);
  i.margin = __ldcg(&d->margin);
  return i;
}

// The guided step of motion blockIdx.x: x0 (the output projection + bias after the CFG blend, [B, D, T], written by the
// MODE_X0 output GEMM) -> guidance -> the output step's tail (inpainting, clamp, the DDPM / DDIM update of p.mode) for
// every element of the motion, reading the step's noise as OutStep does.  grid = B, block = JG_THREADS,
// dynamic shared memory jg_smem_bytes(T, R) (FOOT: fg_smem_bytes(T, R)).  FOOT asks for one CTA per SM (the B CTAs
// never share one at B <= 132), which lifts the register cap ptxas otherwise picks and keeps the step free of spills.
// SCENE (only with FOOT) adds the scene terms, INTER (only with SCENE) the interaction terms: the grid is then B / C
// clusters of C CTAs (C = the descriptor's chars) and the dynamic shared memory ig_smem_bytes(T, R).
template <bool FOOT, bool SCENE, bool INTER = false>
__global__ void __launch_bounds__(JG_THREADS, FOOT ? 1 : 0) joint_guidance_step_kernel(const GuideDesc* guide, const float* x0,
                                                                         const EpiOutParams p) {
  static_assert(FOOT || !SCENE, "the scene terms extend the foot family");
  static_assert(SCENE || !INTER, "the interaction terms extend the scene family");
  pdl_launch_dependents();
  pdl_wait();
  const int T = p.T, D = p.J, b = blockIdx.x, t = threadIdx.x;
  const JointGuide g = load_joint_guide(&guide->j);
  FootGuide fg{};
  if constexpr (FOOT) fg = load_foot_guide(&guide->f);
  SceneGuide sg{};
  if constexpr (SCENE) sg = load_scene_guide(&guide->s);
  InterGuide ig{};
  if constexpr (INTER) ig = load_inter_guide(&guide->i);
  const int R = D == 263 ? 67 : 64;
  const float* xs = joint_guidance_run<FOOT, SCENE, INTER>(g, fg, sg, x0, p.B, T, D, nullptr, ig);
  if (t >= T) return;
  const OutStep u(p, b);
  const size_t base = static_cast<size_t>(b) * D * T + t;
  for (int f = 0; f < D; ++f) {
    const size_t idx = base + static_cast<size_t>(f) * T;
    const OutStep::In v = u.load(p, true, idx, f, t);
    out_tail(p, u, idx, f < R ? xs[f * T + t] : __ldcg(x0 + idx), v);
  }
}

// b200mdm_test_joint_guidance / b200mdm_test_foot_guidance (FOOT) / b200mdm_test_scene_guidance (SCENE) /
// b200mdm_test_interaction_guidance (INTER, clusters as the step kernel's): the guidance of descriptor d alone,
// x0_out [B, D, T] = guided x0 (features past the ric features copied).
template <bool FOOT, bool SCENE, bool INTER = false>
__global__ void __launch_bounds__(JG_THREADS) joint_guidance_test_kernel(const GuideDesc d, const float* x0, float* x0_out,
                                                                         float* loss, int B, int T, int D) {
  static_assert(FOOT || !SCENE, "the scene terms extend the foot family");
  static_assert(SCENE || !INTER, "the interaction terms extend the scene family");
  const int R = D == 263 ? 67 : 64, b = blockIdx.x;
  const float* xs = joint_guidance_run<FOOT, SCENE, INTER>(d.j, d.f, d.s, x0, B, T, D, loss, d.i);
  const size_t base = static_cast<size_t>(b) * D * T;
  for (int i = threadIdx.x; i < D * T; i += blockDim.x) x0_out[base + i] = i < R * T ? xs[i] : x0[base + i];
}

}  // namespace b200
