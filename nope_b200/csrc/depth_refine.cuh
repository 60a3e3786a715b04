// nope_b200 -- pose refinement from the sensor depth (DESIGN.md section 19).
//
// Projective point-to-plane ICP of every rotation hypothesis against its frame's depth: the mesh is rendered at the
// current [R | t] with depth_raster_kernel (render.cuh, unchanged), each rendered pixel is paired with the sensor
// reading at the same pixel, and one damped Gauss-Newton step of the six pose parameters minimises the point-to-plane
// distances of the pairs.  Every float64 operation is rounded on its own (no contraction) and every per-pixel product
// is rounded to 64-bit fixed point before it is summed as an integer, so the sums -- and everything after them -- do
// not depend on the order of the pixels, the launch shape or the batch: tests/depth_refine_oracle.py restates it in
// numpy bit for bit.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "render.cuh"

namespace nope {

constexpr int kIcpThreads = 256;
constexpr int kIcpPixelsPerCta = kIcpThreads * 16;
constexpr int kIcpJJ = 21;                      // upper triangle of J J^T, row by row
constexpr int kIcpSums = 29;                    // 21 J J^T, 6 J e, e^2, n_in
constexpr double kIcpFixedScale = 4294967296.0;  // 2^32: one unit is 2^-32
constexpr double kIcpFixedClamp = 16.0;          // |product| <= 2^4, so |fixed| <= 2^36 and 2^26 pixels sum < 2^62
constexpr double kIcpDamping = 1e-2;             // mu = kIcpDamping max diag(A)

// a per-pixel product in fixed point: clamped to [-16, 16], times 2^32 (exact), rounded half to even
__device__ __forceinline__ long long icp_fixed(double x) {
  return __double2ll_rn(__dmul_rn(fmin(fmax(x, -kIcpFixedClamp), kIcpFixedClamp), kIcpFixedScale));
}

// back-projection X(r, c, z) = ((c + 1/2 - cx) z / fx, (r + 1/2 - cy) z / fy, z), in this order
__device__ __forceinline__ void icp_point(int r, int c, double z, double fx, double fy, double cx, double cy,
                                          double* X) {
  X[0] = __ddiv_rn(__dmul_rn(__dsub_rn(__dadd_rn((double)c, 0.5), cx), z), fx);
  X[1] = __ddiv_rn(__dmul_rn(__dsub_rn(__dadd_rn((double)r, 0.5), cy), z), fy);
  X[2] = z;
}

// a x b, each component (a1 b2 - a2 b1) etc.
__device__ __forceinline__ void icp_cross(const double* a, const double* b, double* o) {
  o[0] = __dsub_rn(__dmul_rn(a[1], b[2]), __dmul_rn(a[2], b[1]));
  o[1] = __dsub_rn(__dmul_rn(a[2], b[0]), __dmul_rn(a[0], b[2]));
  o[2] = __dsub_rn(__dmul_rn(a[0], b[1]), __dmul_rn(a[1], b[0]));
}

// (a0 b0 + a1 b1) + a2 b2
__device__ __forceinline__ double icp_dot(const double* a, const double* b) {
  return __dadd_rn(__dadd_rn(__dmul_rn(a[0], b[0]), __dmul_rn(a[1], b[1])), __dmul_rn(a[2], b[2]));
}

__device__ __forceinline__ bool icp_hit(unsigned bits) { return bits != kDepthInfBits; }

// One pair's fixed-point products added to a thread's 28 int64 registers: acc[0, 21) the upper triangle of J J^T row
// by row, acc[21, 27) J e, acc[27] e^2.
__device__ __forceinline__ void icp_add_pair(long long* acc, const double* J, double e) {
  int q = 0;
#pragma unroll
  for (int a = 0; a < 6; ++a) {
#pragma unroll
    for (int b = a; b < 6; ++b) acc[q++] += icp_fixed(__dmul_rn(J[a], J[b]));
  }
#pragma unroll
  for (int a = 0; a < 6; ++a) acc[kIcpJJ + a] += icp_fixed(__dmul_rn(J[a], e));
  acc[kIcpJJ + 6] += icp_fixed(__dmul_rn(e, e));
}

// The CTA's flush of an accumulate kernel: every thread's 28 registers acc and pair count n are reduced through warp
// shuffles and shared memory, and the CTA adds its partials to the hypothesis's sums [29] with one integer atomic per
// field.  kContour also reduces the contour pixel counts nc into *n_contour.  Called by every thread of the CTA.
template <bool kContour>
__device__ __forceinline__ void icp_flush_sums(const long long* acc, int n, int nc, unsigned long long* __restrict__ sums,
                                               int* __restrict__ n_contour) {
  constexpr int kFields = kIcpSums + (kContour ? 1 : 0);
  __shared__ long long part[kIcpThreads / 32][kFields];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
#pragma unroll
  for (int k = 0; k < kIcpSums - 1; ++k) {
    long long v = acc[k];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    if (lane == 0) part[warp][k] = v;
  }
  n = __reduce_add_sync(0xffffffffu, n);
  if (kContour) nc = __reduce_add_sync(0xffffffffu, nc);
  if (lane == 0) {
    part[warp][kIcpSums - 1] = n;
    if (kContour) part[warp][kIcpSums] = nc;
  }
  __syncthreads();
  if (threadIdx.x >= kFields) return;
  long long v = 0;
  for (int w = 0; w < kIcpThreads / 32; ++w) v += part[w][threadIdx.x];
  if (v == 0) return;
  if (!kContour || threadIdx.x < kIcpSums) atomicAdd(sums + threadIdx.x, (unsigned long long)v);   // wraps
  else atomicAdd(n_contour, (int)v);
}

// The pairs of one iteration: grid (ceil(H W / kIcpPixelsPerCta), P, F).  z [F, P, H, W] the render of hypothesis
// (f, p) (float bits, +inf where nothing is hit), S [F, H, W] the sensor depth (mm, 0 = no reading), masks [F, H, W]
// or null, K [F, 4], t [F, P, 3] the hypotheses' current origins.  Each pixel that takes part adds its fixed-point
// products to 28 int64 registers; the CTA reduces them through warp shuffles and shared memory and adds its partials
// to sums [F, P, 29] with one integer atomic per field.
__global__ void __launch_bounds__(kIcpThreads)
icp_accumulate_kernel(const unsigned* __restrict__ z, const double* __restrict__ S, const uint8_t* __restrict__ masks,
                      const double* __restrict__ K, const double* __restrict__ t, int P, int H, int W, double tau,
                      double rho, unsigned long long* __restrict__ sums) {
  const int p = blockIdx.y, f = blockIdx.z;
  const int hw = H * W;
  const size_t h = (size_t)f * P + p;
  const unsigned* zi = z + h * hw;
  const double* sf = S + (size_t)f * hw;
  const uint8_t* m = masks ? masks + (size_t)f * hw : nullptr;
  const double fx = K[4 * f], fy = K[4 * f + 1], cx = K[4 * f + 2], cy = K[4 * f + 3];
  const double to[3] = {t[3 * h], t[3 * h + 1], t[3 * h + 2]};
  const int lo = blockIdx.x * kIcpPixelsPerCta, hi = min(lo + kIcpPixelsPerCta, hw);
  long long acc[kIcpSums - 1];
#pragma unroll
  for (int k = 0; k < kIcpSums - 1; ++k) acc[k] = 0;
  int n = 0;
  for (int i = lo + (int)threadIdx.x; i < hi; i += kIcpThreads) {
    const int r = i / W, c = i - r * W;
    if (r == 0 || c == 0 || r == H - 1 || c == W - 1) continue;
    const unsigned d0 = zi[i];
    if (!icp_hit(d0) || (m && m[i] == 0)) continue;
    const double s = sf[i];
    const double d = (double)__uint_as_float(d0);
    if (!(s > 0.0) || !(fabs(__dsub_rn(s, d)) <= tau)) continue;
    const unsigned dl = zi[i - 1], dr = zi[i + 1], du = zi[i - W], dd = zi[i + W];
    if (!(icp_hit(dl) && icp_hit(dr) && icp_hit(du) && icp_hit(dd))) continue;
    double P0[3], Q[3], A[3], B[3], eu[3], ev[3], nr[3];
    icp_point(r, c, d, fx, fy, cx, cy, P0);
    icp_point(r, c, s, fx, fy, cx, cy, Q);
    icp_point(r, c + 1, (double)__uint_as_float(dr), fx, fy, cx, cy, A);
    icp_point(r, c - 1, (double)__uint_as_float(dl), fx, fy, cx, cy, B);
#pragma unroll
    for (int k = 0; k < 3; ++k) eu[k] = __dsub_rn(A[k], B[k]);
    icp_point(r + 1, c, (double)__uint_as_float(dd), fx, fy, cx, cy, A);
    icp_point(r - 1, c, (double)__uint_as_float(du), fx, fy, cx, cy, B);
#pragma unroll
    for (int k = 0; k < 3; ++k) ev[k] = __dsub_rn(A[k], B[k]);
    icp_cross(eu, ev, nr);
    const double len2 = icp_dot(nr, nr);
    if (len2 == 0.0) continue;
    const double len = __dsqrt_rn(len2);
    double J[6];
#pragma unroll
    for (int k = 0; k < 3; ++k) J[3 + k] = __ddiv_rn(nr[k], len);
    if (icp_dot(J + 3, P0) > 0.0) {
#pragma unroll
      for (int k = 0; k < 3; ++k) J[3 + k] = -J[3 + k];
    }
#pragma unroll
    for (int k = 0; k < 3; ++k) { A[k] = __dsub_rn(P0[k], to[k]); B[k] = __dsub_rn(P0[k], Q[k]); }
    icp_cross(A, J + 3, J);
#pragma unroll
    for (int k = 0; k < 3; ++k) J[k] = __ddiv_rn(J[k], rho);
    icp_add_pair(acc, J, __ddiv_rn(icp_dot(J + 3, B), tau));
    ++n;
  }
  icp_flush_sums<false>(acc, n, 0, sums + h * kIcpSums, nullptr);
}

// n_valid [F] += the pixels of each frame with a sensor reading inside its mask: grid (ceil(H W / kIcpPixelsPerCta),
// 1, F)
__global__ void __launch_bounds__(kIcpThreads)
icp_valid_kernel(const double* __restrict__ S, const uint8_t* __restrict__ masks, int H, int W,
                 int* __restrict__ n_valid) {
  const int f = blockIdx.z;
  const int hw = H * W;
  const double* sf = S + (size_t)f * hw;
  const uint8_t* m = masks ? masks + (size_t)f * hw : nullptr;
  const int lo = blockIdx.x * kIcpPixelsPerCta, hi = min(lo + kIcpPixelsPerCta, hw);
  int n = 0;
  for (int i = lo + (int)threadIdx.x; i < hi; i += kIcpThreads) n += (sf[i] > 0.0 && (!m || m[i] != 0)) ? 1 : 0;
  n = __reduce_add_sync(0xffffffffu, n);
  __shared__ int part[kIcpThreads / 32];
  if ((threadIdx.x & 31) == 0) part[threadIdx.x >> 5] = n;
  __syncthreads();
  if (threadIdx.x != 0) return;
  for (int w = 1; w < kIcpThreads / 32; ++w) n += part[w];
  if (n) atomicAdd(n_valid + f, n);
}

// a fixed-point sum as float64: rounded to nearest, times 2^-32 (exact)
__device__ __forceinline__ double icp_unfix(unsigned long long s) {
  return __dmul_rn(__ll2double_rn((long long)s), 1.0 / kIcpFixedScale);
}

// hypothesis i: R, t = the inputs, the first pose, its sums reset
__device__ __forceinline__ void icp_init_one(long long i, const double* __restrict__ R_in,
                                             const double* __restrict__ t_in, double* __restrict__ R,
                                             double* __restrict__ t, float* __restrict__ poses,
                                             unsigned long long* __restrict__ sums) {
#pragma unroll
  for (int k = 0; k < 9; ++k) R[9 * i + k] = R_in[9 * i + k];
#pragma unroll
  for (int k = 0; k < 3; ++k) t[3 * i + k] = t_in[3 * i + k];
  render_write_pose(R_in + 9 * i, t_in + 3 * i, poses + 16 * i);
  for (int k = 0; k < kIcpSums; ++k) sums[kIcpSums * i + k] = 0ull;
}

// One thread per (f, p), n = F P: R, t = the inputs, the first pose, every sum and n_valid reset.
__global__ void icp_init_kernel(const double* __restrict__ R_in, const double* __restrict__ t_in, int F, int P,
                                double* __restrict__ R, double* __restrict__ t, float* __restrict__ poses,
                                unsigned long long* __restrict__ sums, int* __restrict__ n_valid) {
  const long long n = (long long)F * P;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    icp_init_one(i, R_in, t_in, R, t, poses, sums);
    if (i < F) n_valid[i] = 0;
  }
}

// One update of one hypothesis from its sums s [29], DESIGN.md section 19, every float64 operation rounded on its own.
// With n_in >= 6: A = the 21 J J^T sums, g = the 6 J e sums, M = A + mu I with mu = kIcpDamping max diag(A), M = L L^T
// by Cholesky (column by column, every inner sum in ascending k), L y = -g forward and L^T delta = y backward (inner
// sums in ascending k); omega = (delta_w tau) / rho, v = delta_v tau; R <- R_delta R with R_delta the rotation of the
// unit quaternion (1, omega / 2) / sqrt(1 + |omega|^2 / 4), t <- t + v.  Fewer pairs or a non-positive pivot leave the
// pose unchanged.  tau is the hypothesis's metric tolerance (mm): the pairing tolerance of the depth fit, or the
// contour fit's pixel tolerance scaled to the object's distance (contour_refine.cuh).
__device__ __forceinline__ void icp_step(const unsigned long long* s, double tau, double rho, double* Ri, double* ti) {
  if ((long long)s[kIcpSums - 1] >= 6) {
    double M[6][6], g[6];
    int q = 0;
    for (int a = 0; a < 6; ++a)
      for (int b = a; b < 6; ++b) { M[a][b] = icp_unfix(s[q++]); M[b][a] = M[a][b]; }
    for (int a = 0; a < 6; ++a) g[a] = icp_unfix(s[kIcpJJ + a]);
    double dmax = M[0][0];
    for (int a = 1; a < 6; ++a) dmax = fmax(dmax, M[a][a]);
    const double mu = __dmul_rn(kIcpDamping, dmax);
    for (int a = 0; a < 6; ++a) M[a][a] = __dadd_rn(M[a][a], mu);
    double L[6][6];
    bool ok = true;
    for (int j = 0; j < 6 && ok; ++j) {
      double d = M[j][j];
      for (int k = 0; k < j; ++k) d = __dsub_rn(d, __dmul_rn(L[j][k], L[j][k]));
      if (!(d > 0.0)) { ok = false; break; }
      L[j][j] = __dsqrt_rn(d);
      for (int r = j + 1; r < 6; ++r) {
        double x = M[r][j];
        for (int k = 0; k < j; ++k) x = __dsub_rn(x, __dmul_rn(L[r][k], L[j][k]));
        L[r][j] = __ddiv_rn(x, L[j][j]);
      }
    }
    if (ok) {
      double y[6], dl[6];
      for (int r = 0; r < 6; ++r) {
        double x = -g[r];
        for (int k = 0; k < r; ++k) x = __dsub_rn(x, __dmul_rn(L[r][k], y[k]));
        y[r] = __ddiv_rn(x, L[r][r]);
      }
      for (int r = 5; r >= 0; --r) {
        double x = y[r];
        for (int k = r + 1; k < 6; ++k) x = __dsub_rn(x, __dmul_rn(L[k][r], dl[k]));
        dl[r] = __ddiv_rn(x, L[r][r]);
      }
      double h[3];
#pragma unroll
      for (int k = 0; k < 3; ++k) h[k] = __dmul_rn(__ddiv_rn(__dmul_rn(dl[k], tau), rho), 0.5);   // omega / 2
      const double sn = __dsqrt_rn(__dadd_rn(1.0, icp_dot(h, h)));
      const double qw = __ddiv_rn(1.0, sn), qx = __ddiv_rn(h[0], sn), qy = __ddiv_rn(h[1], sn),
                   qz = __ddiv_rn(h[2], sn);
      const double xx = __dmul_rn(qx, qx), yy = __dmul_rn(qy, qy), zz = __dmul_rn(qz, qz);
      const double xy = __dmul_rn(qx, qy), xz = __dmul_rn(qx, qz), yz = __dmul_rn(qy, qz);
      const double wx = __dmul_rn(qw, qx), wy = __dmul_rn(qw, qy), wz = __dmul_rn(qw, qz);
      const double Rd[9] = {
          __dsub_rn(1.0, __dmul_rn(2.0, __dadd_rn(yy, zz))), __dmul_rn(2.0, __dsub_rn(xy, wz)),
          __dmul_rn(2.0, __dadd_rn(xz, wy)),
          __dmul_rn(2.0, __dadd_rn(xy, wz)), __dsub_rn(1.0, __dmul_rn(2.0, __dadd_rn(xx, zz))),
          __dmul_rn(2.0, __dsub_rn(yz, wx)),
          __dmul_rn(2.0, __dsub_rn(xz, wy)), __dmul_rn(2.0, __dadd_rn(yz, wx)),
          __dsub_rn(1.0, __dmul_rn(2.0, __dadd_rn(xx, yy)))};
      double Rn[9];
#pragma unroll
      for (int r = 0; r < 3; ++r) {
#pragma unroll
        for (int c = 0; c < 3; ++c)
          Rn[3 * r + c] = __dadd_rn(__dadd_rn(__dmul_rn(Rd[3 * r], Ri[c]), __dmul_rn(Rd[3 * r + 1], Ri[3 + c])),
                                    __dmul_rn(Rd[3 * r + 2], Ri[6 + c]));
      }
#pragma unroll
      for (int k = 0; k < 9; ++k) Ri[k] = Rn[k];
#pragma unroll
      for (int k = 0; k < 3; ++k) ti[k] = __dadd_rn(ti[k], __dmul_rn(dl[3 + k], tau));
    }
  }
}

// One update per (f, p) at the pairing tolerance tau (icp_step); writes the next float32 pose and resets the sums for
// the next render.
__global__ void icp_solve_kernel(int F, int P, double tau, double rho, double* __restrict__ R, double* __restrict__ t,
                                 float* __restrict__ poses, unsigned long long* __restrict__ sums) {
  const long long n = (long long)F * P;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    unsigned long long* s = sums + kIcpSums * i;
    icp_step(s, tau, rho, R + 9 * i, t + 3 * i);
    render_write_pose(R + 9 * i, t + 3 * i, poses + 16 * i);
    for (int k = 0; k < kIcpSums; ++k) s[k] = 0ull;
  }
}

// hypothesis i's pose into R_out [F, P, 9], t_out [F, P, 3] and its sums into sums_out [F, P, 29] (when not null)
__device__ __forceinline__ void icp_out_one(long long i, const double* __restrict__ R, const double* __restrict__ t,
                                            const unsigned long long* __restrict__ sums, double* __restrict__ R_out,
                                            double* __restrict__ t_out, long long* __restrict__ sums_out) {
#pragma unroll
  for (int k = 0; k < 9; ++k) R_out[9 * i + k] = R[9 * i + k];
#pragma unroll
  for (int k = 0; k < 3; ++k) t_out[3 * i + k] = t[3 * i + k];
  if (sums_out) {
    for (int k = 0; k < kIcpSums; ++k) sums_out[kIcpSums * i + k] = (long long)sums[kIcpSums * i + k];
  }
}

// The outputs after the last render at tau: R_out [F, P, 9], t_out [F, P, 3], fit [F, P, 4] = (n_in, n_valid,
// rms = tau sqrt(sum e^2 / n_in), score = n_in / n_valid) -- rms is NaN when n_in = 0, score when n_valid = 0 --
// and sums_out [F, P, 29] (optional) the integer sums of the last render.
__global__ void icp_final_kernel(const double* __restrict__ R, const double* __restrict__ t,
                                 const unsigned long long* __restrict__ sums, const int* __restrict__ n_valid, int F,
                                 int P, double tau, double* __restrict__ R_out, double* __restrict__ t_out,
                                 double* __restrict__ fit, long long* __restrict__ sums_out) {
  const long long n = (long long)F * P;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const unsigned long long* s = sums + kIcpSums * i;
    icp_out_one(i, R, t, sums, R_out, t_out, sums_out);
    const double nin = (double)(long long)s[kIcpSums - 1], nv = (double)n_valid[i / P];
    fit[4 * i] = nin;
    fit[4 * i + 1] = nv;
    fit[4 * i + 2] = __dmul_rn(tau, __dsqrt_rn(__ddiv_rn(icp_unfix(s[kIcpSums - 2]), nin)));
    fit[4 * i + 3] = __ddiv_rn(nin, nv);
  }
}

}  // namespace nope
