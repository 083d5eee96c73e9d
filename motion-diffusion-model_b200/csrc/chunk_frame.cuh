// Goal-directed autoregressive chains (DESIGN.md, "Goals in the world frame"): a world-space goal re-expressed in the
// frame of the chunk about to be generated.  The chunk frame of returned frame g is recover_root_rot_pos's yaw and root
// position at g,
//   yaw_g = sum_{u<g} r[u];   P_g = sum_{u<=g} w[u],  w[u] = rot(yaw[u]) v[u-1],  w[0] = 0
// (r the root yaw velocity, v the root XZ velocity, rot the quaternion (cos yaw, 0, sin yaw, 0) of recover_from_ric,
// which turns by 2 yaw), and recover_from_ric(returned)[g + t] = M(recover_from_ric(chunk alone)[t]) with M = rot(yaw_g)
// then + P_g in XZ.  A per-sample fp64 carry (yaw, P.x, P.z, v.x, v.z of the last frame, has-a-frame) holds the sums over
// every frame seen so far, so a chunk boundary costs one pass over that chunk's frames whatever the chain's length.
#pragma once
#include <cuda_runtime.h>

#include "joint_guidance.cuh"

namespace b200 {

constexpr int CF_CARRY = 6;   // yaw, P.x, P.z, last v.x, last v.z, has-previous-frame

// (x, z) <- qrot(q, (x, 0, z)) for q = (c, 0, qy, 0), in the operation order of the reference's qrot (quaternion.py):
// qy = -sin yaw is recover_from_ric's qinv (the chunk-to-world rotation), qy = +sin yaw its inverse.
__device__ __forceinline__ void cf_rot(double c, double qy, double& x, double& z) {
  const double uvx = qy * z, uvz = -(qy * x);
  const double uuvx = qy * uvz, uuvz = -(qy * uvx);
  x = x + 2.0 * (c * uvx + uuvx);
  z = z + 2.0 * (c * uvz + uuvz);
}

// One CTA per sample, JG_THREADS threads, thread t <- frame t of frames [B, D, n] (normalised features, n <= JG_THREADS,
// n == 0 leaves the carry as it is).  Advances carry [B, CF_CARRY] over the n frames, then writes target [B, n_ext, 3]:
// every position entry of goal [B, n_ext, 3] mapped by M^-1 of the frame after the last one seen (XZ translated and
// rotated back, y unchanged), and the heading entry n_ext - 1 as wrap(heading + 2 yaw) in (-pi, pi] (M turns an
// atan2(x, z) heading by -2 yaw), its components 1 and 2 unchanged.  Features are de-normalised in fp32 as the
// reference's motion * std + mean; the scans, the carry and the transform are fp64.
__global__ void __launch_bounds__(JG_THREADS) chunk_frame_kernel(const float* __restrict__ frames, int D, int n,
                                                                  const float* __restrict__ mean,
                                                                  const float* __restrict__ std, double* __restrict__ carry,
                                                                  const float* __restrict__ goal, int n_ext,
                                                                  float* __restrict__ target) {
  __shared__ double sh[JG_WARPS * 2];
  __shared__ double vprev[2 * JG_THREADS];
  __shared__ double frame[5];   // the next chunk's frame: yaw, cos yaw, sin yaw, P.x, P.z
  const int b = blockIdx.x, t = threadIdx.x;
  double* cy = carry + static_cast<size_t>(b) * CF_CARRY;
  const double yaw0 = cy[0], has0 = cy[5];
  const bool live = t < n;
  double r = 0.0, vx = 0.0, vz = 0.0;
  if (live) {
    const float* x = frames + static_cast<size_t>(b) * D * n + t;
    r = __fadd_rn(__fmul_rn(x[0], std[0]), mean[0]);
    vx = __fadd_rn(__fmul_rn(x[n], std[1]), mean[1]);
    vz = __fadd_rn(__fmul_rn(x[2 * n], std[2]), mean[2]);
    vprev[2 * t] = vx;
    vprev[2 * t + 1] = vz;
  }
  double s1[1] = {r};
  jg_scan<1, false>(s1, sh);                   // also orders the vprev writes before the reads below
  double w[2] = {0.0, 0.0};
  if (live) {
    const double yaw = yaw0 + (s1[0] - r);     // yaw[t] = sum of the velocities before t
    double px, pz;
    bool prev = true;
    if (t > 0) {
      px = vprev[2 * (t - 1)];
      pz = vprev[2 * (t - 1) + 1];
    } else {
      px = cy[3];
      pz = cy[4];
      prev = has0 != 0.0;
    }
    if (prev) {
      cf_rot(cos(yaw), -sin(yaw), px, pz);
      w[0] = px;
      w[1] = pz;
    }
  }
  jg_scan<2, false>(w, sh);
  if (t == JG_THREADS - 1) {                   // the inclusive totals over the block (frames >= n add 0)
    const double yaw = yaw0 + s1[0];
    double Px = cy[1] + w[0], Pz = cy[2] + w[1], lx = cy[3], lz = cy[4], has = has0;
    if (n > 0) {
      lx = vprev[2 * (n - 1)];
      lz = vprev[2 * (n - 1) + 1];
      has = 1.0;
    }
    cy[0] = yaw; cy[1] = Px; cy[2] = Pz; cy[3] = lx; cy[4] = lz; cy[5] = has;
    const double c = cos(yaw), s = sin(yaw);
    if (has != 0.0) {                          // P_g = P_{g-1} + w[g]
      double ax = lx, az = lz;
      cf_rot(c, -s, ax, az);
      Px += ax;
      Pz += az;
    }
    frame[0] = yaw; frame[1] = c; frame[2] = s; frame[3] = Px; frame[4] = Pz;
  }
  __syncthreads();
  if (t < n_ext) {
    const float* g = goal + (static_cast<size_t>(b) * n_ext + t) * 3;
    float* o = target + (static_cast<size_t>(b) * n_ext + t) * 3;
    if (t == n_ext - 1) {
      const double pi = 3.141592653589793;
      double h = static_cast<double>(g[0]) + 2.0 * frame[0];
      if (h > pi || h <= -pi) h -= 2.0 * pi * ceil((h - pi) / (2.0 * pi));
      o[0] = static_cast<float>(h);
      o[2] = g[2];
    } else {
      double x = static_cast<double>(g[0]) - frame[3], z = static_cast<double>(g[2]) - frame[4];
      cf_rot(frame[1], frame[2], x, z);
      o[0] = static_cast<float>(x);
      o[2] = static_cast<float>(z);
    }
    o[1] = g[1];
  }
}

}  // namespace b200
