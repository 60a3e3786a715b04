// nope_b200 -- pose tracking (DESIGN.md section 26): prior rotations to the centres of the joint roll and viewpoint
// refinement (section 14).
//
// For a prior rotation Rc in the crop camera and a grid T [N], the centre (D, seed, rho) with Rz(rho) D T[seed] = Rc
// whose residual D turns only about an axis in the camera's xy plane: for every grid pose n
//   M = Rc T[n]^T,      M_ij = ((Rc_i0 T_j0 + Rc_i1 T_j1) + Rc_i2 T_j2)
//   a = M00 + M11,  b = M10 - M01,  r = sqrt(a a + b b),  score_n = r + M22
// score_n is the trace of Rz(-rho_n) M at its best roll, so the largest score is the (roll, template) pair nearest
// to the prior.  seed = argmax_n score_n (ties -> the lowest n, a NaN never chosen), (c, s) = (a / r, b / r) or (1, 0)
// at r = 0, and D = [[c, s, 0], [-s, c, 0], [0, 0, 1]] M as
//   D_0j = c M0j + s M1j,  D_1j = c M1j - s M0j,  D_2j = M2j,
// each rounded to fp32 once, like (c, s).  float64, every product and sum rounded on its own (no FMA contraction),
// division and sqrt correctly rounded; tests/track_oracle.py restates it op by op.  A prior with a non-finite entry,
// or a grid without one score that is a number, gives seed 0, D = I and (1, 0): no index leaves the grid.
// One CTA per prior; the threads stride over N and the argmax is reduced across the CTA.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <climits>

namespace nope {

constexpr int kTrackThreads = 256;

// (v, i) ranks before (w, j): the larger score, ties -> the lower index; a NaN v never ranks first
__device__ __forceinline__ bool track_better(double v, int i, double w, int j) {
  return v > w || (v == w && i < j);
}

// M = Rc T^T, row-major, each entry ((x0 y0 + x1 y1) + x2 y2)
__device__ __forceinline__ void track_residual(const double* rc, const double* __restrict__ t, double* m) {
#pragma unroll
  for (int i = 0; i < 3; ++i)
#pragma unroll
    for (int j = 0; j < 3; ++j)
      m[3 * i + j] = __dadd_rn(__dadd_rn(__dmul_rn(rc[3 * i], __ldg(t + 3 * j)),
                                         __dmul_rn(rc[3 * i + 1], __ldg(t + 3 * j + 1))),
                               __dmul_rn(rc[3 * i + 2], __ldg(t + 3 * j + 2)));
}

// grid H, kTrackThreads threads.  Rc [H, 9], T [N, 9] fp64 row-major -> out_D [H, 9] fp32, out_seed [H] int32,
// out_cossin [H, 2] fp32
__global__ void __launch_bounds__(kTrackThreads)
track_seed_kernel(const double* __restrict__ Rc, const double* __restrict__ T, int N, float* __restrict__ out_D,
                  int32_t* __restrict__ out_seed, float* __restrict__ out_cossin) {
  __shared__ double red_v[kTrackThreads / 32];
  __shared__ int red_i[kTrackThreads / 32];
  const int h = blockIdx.x, t = threadIdx.x;
  double rc[9];
  bool finite = true;
#pragma unroll
  for (int e = 0; e < 9; ++e) {
    rc[e] = __ldg(Rc + 9 * (size_t)h + e);
    finite &= isfinite(rc[e]);
  }
  double best = -__longlong_as_double(0x7ff0000000000000ll);
  int bi = INT_MAX;
  if (finite) {
    for (int n = t; n < N; n += kTrackThreads) {
      double m[9];
      track_residual(rc, T + 9 * (size_t)n, m);
      const double a = __dadd_rn(m[0], m[4]), b = __dsub_rn(m[3], m[1]);
      const double r = __dsqrt_rn(__dadd_rn(__dmul_rn(a, a), __dmul_rn(b, b)));
      const double v = __dadd_rn(r, m[8]);
      if (track_better(v, n, best, bi)) best = v, bi = n;
    }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const double w = __shfl_xor_sync(0xffffffffu, best, o);
    const int j = __shfl_xor_sync(0xffffffffu, bi, o);
    if (track_better(w, j, best, bi)) best = w, bi = j;
  }
  if ((t & 31) == 0) red_v[t >> 5] = best, red_i[t >> 5] = bi;
  __syncthreads();
  if (t != 0) return;
  for (int w = 1; w < kTrackThreads / 32; ++w)
    if (track_better(red_v[w], red_i[w], best, bi)) best = red_v[w], bi = red_i[w];
  float* d = out_D + 9 * (size_t)h;
  if (bi == INT_MAX) {                                   // a non-finite prior, or no score that is a number
#pragma unroll
    for (int e = 0; e < 9; ++e) d[e] = e % 4 == 0 ? 1.f : 0.f;
    out_seed[h] = 0;
    out_cossin[2 * (size_t)h] = 1.f;
    out_cossin[2 * (size_t)h + 1] = 0.f;
    return;
  }
  double m[9];
  track_residual(rc, T + 9 * (size_t)bi, m);
  const double a = __dadd_rn(m[0], m[4]), b = __dsub_rn(m[3], m[1]);
  const double r = __dsqrt_rn(__dadd_rn(__dmul_rn(a, a), __dmul_rn(b, b)));
  const double c = r == 0.0 ? 1.0 : __ddiv_rn(a, r), s = r == 0.0 ? 0.0 : __ddiv_rn(b, r);
#pragma unroll
  for (int j = 0; j < 3; ++j) {
    d[j] = __double2float_rn(__dadd_rn(__dmul_rn(c, m[j]), __dmul_rn(s, m[3 + j])));
    d[3 + j] = __double2float_rn(__dsub_rn(__dmul_rn(c, m[3 + j]), __dmul_rn(s, m[j])));
    d[6 + j] = __double2float_rn(m[6 + j]);
  }
  out_seed[h] = bi;
  out_cossin[2 * (size_t)h] = __double2float_rn(c);
  out_cossin[2 * (size_t)h + 1] = __double2float_rn(s);
}

}  // namespace nope
