// Distinct pose hypotheses (DESIGN.md section 21): greedy non-maximum suppression of a similarity row in the
// project's ranking order, where two entries are "within theta" when their rotations are, modulo the object's
// symmetry group.  One CTA per row; tests/distinct_oracle.py restates every float64 step in the same order.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "rank.cuh"

namespace nope {

constexpr int kDistinctMaxSym = 32;                       // discrete rotations per group, the identity first
constexpr int kDistinctThreads = 512;
constexpr int kDistinctSmemWords = 4096;                  // 131 072 entries: 36 x 2562 in-plane rows fit

// One symmetry group: the discrete rotations d[0 .. n) (row-major 3x3, d[0] the identity) and the continuous axis
// (a unit vector, has_axis = 0 when there is none).
struct DistinctGroup {
  double d[kDistinctMaxSym * 9];
  double axis[3];
  int n;
  int has_axis;
};

// Correctly rounded sqrt of x (the value of __dsqrt_rn) without the call to the IEEE slow path that __dsqrt_rn
// compiles to.  x = F 2^(e - 52) with F the 53-bit integer significand; for M = F 2^(52 + (e & 1)) < 2^106,
// sqrt(x) = sqrt(M) 2^(floor(e / 2) - 52) with sqrt(M) in [2^52, 2^53).  S = floor(sqrt(M)) is found from a float64
// estimate and corrected by exact 128-bit integer compares; the result rounds up when M - S^2 > S, i.e. when
// sqrt(M) > S + 1/2 (M is an integer, so it never equals (S + 1/2)^2: sqrt has no ties).  S + 1 <= 2^53 and the
// power-of-two scale are exact.
__device__ __forceinline__ double distinct_sqrt_rn(double x) {
  if (!(x > 0.0) || isinf(x)) return x == 0.0 || isinf(x) ? x : __longlong_as_double(0x7ff8000000000000LL);
  int shift = 0;
  if (x < 0x1p-1000) { x = __dmul_rn(x, 0x1p108); shift = -54; }            // subnormal range: exact scaling
  const unsigned long long bits = (unsigned long long)__double_as_longlong(x);
  const int e = (int)((bits >> 52) & 0x7ff) - 1023;
  const unsigned long long F = (bits & 0xfffffffffffffULL) | (1ULL << 52);
  const int odd = e & 1;
  const unsigned __int128 M = (unsigned __int128)F << (52 + odd);
  // the estimate from the significand alone: m = F 2^(odd - 52) in [1, 4), y ~ 1 / sqrt(m) refined twice
  const double m = __dmul_rn((double)F, odd ? 0x1p-51 : 0x1p-52);
  double y = (double)rsqrtf((float)m);
  y = __dmul_rn(y, __dsub_rn(1.5, __dmul_rn(__dmul_rn(0.5, m), __dmul_rn(y, y))));
  y = __dmul_rn(y, __dsub_rn(1.5, __dmul_rn(__dmul_rn(0.5, m), __dmul_rn(y, y))));
  unsigned long long S = (unsigned long long)__dmul_rn(__dmul_rn(m, y), 0x1p52);
  while ((unsigned __int128)S * S > M) --S;
  while ((unsigned __int128)(S + 1) * (S + 1) <= M) ++S;
  if (M - (unsigned __int128)S * S > S) ++S;
  const int k = (e - odd) / 2 - 52 + shift;                                   // e - odd is even: exact halving
  return __dmul_rn((double)S, __longlong_as_double((long long)(k + 1023) << 52));
}

// Is entry j within theta of the selected entry i?  P = Rj^T Ri, M_d = D_d P; c_d = tr M_d without an axis, else
// a^T M_d a + sqrt((tr M_d - a^T M_d a)^2 + s^2) with s = a . (M21 - M12, M02 - M20, M10 - M01), the maximum of
// tr(M_d Rot(a, phi)) over phi.  Within when some c_d >= c_thr.  Each product, sum and root rounded on its own.
__device__ __forceinline__ bool distinct_within(const double* ri, const double* rj, const DistinctGroup& g,
                                                double c_thr) {
  double P[9];
#pragma unroll
  for (int a = 0; a < 3; ++a)
#pragma unroll
    for (int b = 0; b < 3; ++b)
      P[a * 3 + b] = __dadd_rn(__dadd_rn(__dmul_rn(rj[a], ri[b]), __dmul_rn(rj[3 + a], ri[3 + b])),
                               __dmul_rn(rj[6 + a], ri[6 + b]));
  for (int d = 0; d < g.n; ++d) {
    const double* D = g.d + d * 9;
    double c;
    if (!g.has_axis) {
      double M[3];
#pragma unroll
      for (int a = 0; a < 3; ++a)
        M[a] = __dadd_rn(__dadd_rn(__dmul_rn(D[a * 3], P[a]), __dmul_rn(D[a * 3 + 1], P[3 + a])),
                         __dmul_rn(D[a * 3 + 2], P[6 + a]));
      c = __dadd_rn(__dadd_rn(M[0], M[1]), M[2]);
    } else {
      double M[9], v[3];
#pragma unroll
      for (int a = 0; a < 3; ++a)
#pragma unroll
        for (int b = 0; b < 3; ++b)
          M[a * 3 + b] = __dadd_rn(__dadd_rn(__dmul_rn(D[a * 3], P[b]), __dmul_rn(D[a * 3 + 1], P[3 + b])),
                                   __dmul_rn(D[a * 3 + 2], P[6 + b]));
      const double* ax = g.axis;
#pragma unroll
      for (int a = 0; a < 3; ++a)
        v[a] = __dadd_rn(__dadd_rn(__dmul_rn(M[a * 3], ax[0]), __dmul_rn(M[a * 3 + 1], ax[1])),
                         __dmul_rn(M[a * 3 + 2], ax[2]));
      const double t = __dadd_rn(__dadd_rn(M[0], M[4]), M[8]);
      const double u = __dadd_rn(__dadd_rn(__dmul_rn(ax[0], v[0]), __dmul_rn(ax[1], v[1])), __dmul_rn(ax[2], v[2]));
      const double s = __dadd_rn(__dadd_rn(__dmul_rn(ax[0], __dsub_rn(M[7], M[5])),
                                           __dmul_rn(ax[1], __dsub_rn(M[2], M[6]))),
                                 __dmul_rn(ax[2], __dsub_rn(M[3], M[1])));
      const double w = __dsub_rn(t, u);
      c = __dadd_rn(u, distinct_sqrt_rn(__dadd_rn(__dmul_rn(w, w), __dmul_rn(s, s))));
    }
    if (c >= c_thr) return true;
  }
  return false;
}

// The scan of distinct_topk_kernel: a warp per 32-entry word of the mask, which marks the removed entries (taken,
// suppressed, or scored -inf / NaN).  Each round removes what lies within theta of the last pick.
struct DistinctSel : TopkOut {
  const float* row;                    // sim [N]
  int N, nwords;
  const double* rot;                   // [N, 9]
  const DistinctGroup* g;              // in shared memory
  double c_thr;
  unsigned* mask;                      // [nwords]

  __device__ __forceinline__ void scan(int t, const int* picks, float& bv, int& bi) const {
    const int lane = threadIdx.x & 31;
    const int pick = t > 0 ? picks[t - 1] : -1;
    double ri[9];
    if (t > 0)
#pragma unroll
      for (int e = 0; e < 9; ++e) ri[e] = rot[(long long)pick * 9 + e];
    for (int w = threadIdx.x >> 5; w < nwords; w += kDistinctThreads / 32) {
      const unsigned word = mask[w];
      if (word == 0xffffffffu) continue;
      const int j = (w << 5) + lane;
      bool dead = ((word >> lane) & 1u) || j >= N;
      if (!dead) {
        const float v = row[j];
        if (!(v > -INFINITY) || j == pick) {
          dead = true;
        } else if (t > 0 && distinct_within(ri, rot + (long long)j * 9, *g, c_thr)) {
          dead = true;
        } else {
          offer(v, j, bv, bi);
        }
      }
      const unsigned now = __ballot_sync(0xffffffffu, dead);
      if (lane == 0 && now != word) mask[w] = now;
    }
  }
};

// One CTA per row r of sim [R, N].  The row's rotations are rot [G_r, N, 9] at r / Q (0 when G_r = 1), its group
// groups[group[r]].  The removal mask lives in shared memory up to kDistinctSmemWords words, else at
// gmask + r * ceil(N / 32).  k picks cost k passes over the row (select_rounds); ranks with nothing left get -inf / -1.
__global__ void __launch_bounds__(kDistinctThreads)
distinct_topk_kernel(const float* __restrict__ sim, int N, const double* __restrict__ rot, int G_r, int Q,
                     const DistinctGroup* __restrict__ groups, const int* __restrict__ group, int k, double c_thr,
                     unsigned* __restrict__ gmask, long long* __restrict__ idx_out, float* __restrict__ score_out) {
  __shared__ DistinctGroup s_g;
  __shared__ unsigned s_mask[kDistinctSmemWords];
  __shared__ SelectSmem<kDistinctThreads> sm;
  const int r = blockIdx.x;
  const int nwords = (N + 31) >> 5;
  unsigned* mask = gmask ? gmask + (long long)r * nwords : s_mask;
  {
    const long long* src = reinterpret_cast<const long long*>(groups + group[r]);
    long long* dst = reinterpret_cast<long long*>(&s_g);
    for (int i = threadIdx.x; i < (int)(sizeof(DistinctGroup) / 8); i += blockDim.x) dst[i] = src[i];
  }
  for (int w = threadIdx.x; w < nwords; w += blockDim.x) mask[w] = 0u;
  __syncthreads();
  const long long o = (long long)r * k;
  select_rounds(DistinctSel{{score_out + o, idx_out + o, 0}, sim + (long long)r * N, N, nwords,
                            rot + (long long)(G_r == 1 ? 0 : r / Q) * N * 9, &s_g, c_thr, mask},
                k, sm);
}

}  // namespace nope
