// nope_b200 -- symmetry-aware MSSD / MSPD of the BOP 2019 protocol (DESIGN.md section 15).
//
// For F rows (one object) x P estimates x S symmetry transforms over V model points:
//   MSSD = min_s max_x || (R_e x + t_e) - (R_g (R_s x + t_s) + t_g) ||_2                                    (mm)
//   MSPD = min_s max_x || proj(R_e x + t_e) - proj(R_g (R_s x + t_s) + t_g) ||_2,  u = fx X / Z + cx      (px)
// in float64, every product and sum rounded on its own (no FMA contraction):
//   composed pose   G = R_g R_s:  G_ij = ((g_i0 s_0j + g_i1 s_1j) + g_i2 s_2j),  t_i = ((g_i0 ts_0 + g_i1 ts_1) + g_i2 ts_2) + tg_i
//   transform       ((r_0 x + r_1 y) + r_2 z) + t, per row, the float32 point widened
//   squared norm    ((dx dx + dy dy) + dz dz), resp. (du du + dv dv)
//   projection      (fx X) / Z + cx, (fy Y) / Z + cy
// The max is taken over squared distances and sqrt.rn applied once: a correctly rounded sqrt is monotone, so this is
// the max of the norms as computed.  A symmetry under which any point has Z <= 0 (or NaN) for either pose gives MSPD
// +inf.  Max and min are exact, so the work splits freely: each CTA takes kPoseErrSyms symmetries of one (row,
// estimate), reduces the max over V per symmetry and the min over its symmetries, and atomicMin's the uint64 bits of
// the non-negative result into outputs filled with +inf.  The output does not depend on the launch shape.
// oracle/bop_oracle.py restates every step in numpy.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace nope {

constexpr int kPoseErrThreads = 256;
constexpr int kPoseErrSyms = 4;                          // symmetries per CTA: each estimated point serves 4 (8 spill)
constexpr unsigned long long kDoubleInfBits = 0x7ff0000000000000ull;

__global__ void pose_error_fill_kernel(unsigned long long* __restrict__ a, unsigned long long* __restrict__ b, int n) {
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    a[i] = kDoubleInfBits;
    b[i] = kDoubleInfBits;
  }
}

// row i of a 3x4 (R | t) pose applied to a point: ((r0 x + r1 y) + r2 z) + t
__device__ __forceinline__ double pose_row(const double* m, int i, double x, double y, double z) {
  return __dadd_rn(__dadd_rn(__dadd_rn(__dmul_rn(m[4 * i], x), __dmul_rn(m[4 * i + 1], y)), __dmul_rn(m[4 * i + 2], z)),
                   m[4 * i + 3]);
}

// grid (ceil(S / kPoseErrSyms), P, F), kPoseErrThreads threads.  points [V, 3] fp32; sym [S, 12], gt [F, 12],
// est [F, P, 12] row-major 3x4 (R | t) fp64; K [F, 4] (fx, fy, cx, cy) fp64; out_* [F, P] fp64 bits, +inf-filled.
__global__ void __launch_bounds__(kPoseErrThreads)
pose_error_kernel(const float* __restrict__ points, int V, const double* __restrict__ sym, int S,
                  const double* __restrict__ gt, const double* __restrict__ est, const double* __restrict__ K, int P,
                  unsigned long long* __restrict__ out_mssd, unsigned long long* __restrict__ out_mspd) {
  __shared__ double comp[kPoseErrSyms][12];              // R_g R_s | R_g t_s + t_g of this CTA's symmetries
  __shared__ double emat[12];
  __shared__ double red_e[kPoseErrThreads / 32][kPoseErrSyms], red_p[kPoseErrThreads / 32][kPoseErrSyms];
  const int s0 = blockIdx.x * kPoseErrSyms, p = blockIdx.y, f = blockIdx.z;
  const int ns = min(kPoseErrSyms, S - s0);
  const int t = threadIdx.x;
  if (t < kPoseErrSyms * 12) {
    const int j = t / 12, e = t % 12, r = e / 4, c = e % 4;
    if (j < ns) {
      const double* g = gt + 12 * f;
      const double* s = sym + 12 * (s0 + j);
      double v = __dadd_rn(__dadd_rn(__dmul_rn(g[4 * r], s[c]), __dmul_rn(g[4 * r + 1], s[4 + c])),
                           __dmul_rn(g[4 * r + 2], s[8 + c]));
      if (c == 3) v = __dadd_rn(v, g[4 * r + 3]);
      comp[j][e] = v;
    }
  } else if (t < kPoseErrSyms * 12 + 12) {
    emat[t - kPoseErrSyms * 12] = est[((size_t)f * P + p) * 12 + (t - kPoseErrSyms * 12)];
  }
  __syncthreads();
  const double fx = K[4 * f], fy = K[4 * f + 1], cx = K[4 * f + 2], cy = K[4 * f + 3];
  double me[kPoseErrSyms], mp[kPoseErrSyms];             // max squared distance, 3-D and projected
  bool bad[kPoseErrSyms];                                // some point at Z <= 0 under the symmetric ground truth
#pragma unroll
  for (int j = 0; j < kPoseErrSyms; ++j) { me[j] = 0.0; mp[j] = 0.0; bad[j] = false; }
  bool bad_e = false;                                    // some point at Z <= 0 under the estimate
  for (int i = t; i < V; i += kPoseErrThreads) {
    const double x = (double)points[3 * i], y = (double)points[3 * i + 1], z = (double)points[3 * i + 2];
    const double ex = pose_row(emat, 0, x, y, z), ey = pose_row(emat, 1, x, y, z), ez = pose_row(emat, 2, x, y, z);
    bad_e |= !(ez > 0.0);
    const double eu = __dadd_rn(__ddiv_rn(__dmul_rn(fx, ex), ez), cx);
    const double ev = __dadd_rn(__ddiv_rn(__dmul_rn(fy, ey), ez), cy);
#pragma unroll
    for (int j = 0; j < kPoseErrSyms; ++j) {
      if (j < ns) {
        const double gx = pose_row(comp[j], 0, x, y, z), gy = pose_row(comp[j], 1, x, y, z);
        const double gz = pose_row(comp[j], 2, x, y, z);
        const double dx = __dsub_rn(ex, gx), dy = __dsub_rn(ey, gy), dz = __dsub_rn(ez, gz);
        me[j] = fmax(me[j], __dadd_rn(__dadd_rn(__dmul_rn(dx, dx), __dmul_rn(dy, dy)), __dmul_rn(dz, dz)));
        bad[j] |= !(gz > 0.0);
        const double du = __dsub_rn(eu, __dadd_rn(__ddiv_rn(__dmul_rn(fx, gx), gz), cx));
        const double dv = __dsub_rn(ev, __dadd_rn(__ddiv_rn(__dmul_rn(fy, gy), gz), cy));
        mp[j] = fmax(mp[j], __dadd_rn(__dmul_rn(du, du), __dmul_rn(dv, dv)));
      }
    }
  }
  const int lane = t & 31, warp = t >> 5;
#pragma unroll
  for (int j = 0; j < kPoseErrSyms; ++j) {
    double pj = (bad[j] || bad_e) ? __longlong_as_double((long long)kDoubleInfBits) : mp[j];
    double ej = me[j];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      ej = fmax(ej, __shfl_xor_sync(0xffffffffu, ej, o));
      pj = fmax(pj, __shfl_xor_sync(0xffffffffu, pj, o));
    }
    if (lane == 0) { red_e[warp][j] = ej; red_p[warp][j] = pj; }
  }
  __syncthreads();
  if (t == 0) {
    double be = __longlong_as_double((long long)kDoubleInfBits), bp = be;
    for (int j = 0; j < ns; ++j) {
      double ej = red_e[0][j], pj = red_p[0][j];
      for (int w = 1; w < kPoseErrThreads / 32; ++w) { ej = fmax(ej, red_e[w][j]); pj = fmax(pj, red_p[w][j]); }
      be = fmin(be, ej);
      bp = fmin(bp, pj);
    }
    // non-negative doubles order as their bit patterns: sqrt.rn once, then the min over CTAs through the bits
    atomicMin(out_mssd + (size_t)f * P + p, (unsigned long long)__double_as_longlong(__dsqrt_rn(be)));
    atomicMin(out_mspd + (size_t)f * P + p, (unsigned long long)__double_as_longlong(__dsqrt_rn(bp)));
  }
}

}  // namespace nope
