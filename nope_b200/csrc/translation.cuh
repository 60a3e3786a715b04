// nope_b200 -- translation from the object mask (DESIGN.md section 18).
//
// For every frame f and rotation hypothesis p the translation t is moved so that the silhouette of the mesh rendered
// at [R | t] lines up with the frame's object mask: the distance is scaled by the ratio of the two bounding-box sizes,
// then the origin is moved so that the silhouette's box centre lands on the mask's.  The silhouette is the coverage of
// depth_raster_kernel (render.cuh), unchanged.  Everything that decides a result is an integer reduction (counts,
// bounding boxes) or one float64 operation rounded on its own, so the output is deterministic and does not depend on
// the batch: tests/translation_oracle.py restates it in numpy.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "render.cuh"

namespace nope {

constexpr int kFitThreads = 256;
constexpr int kFitPixelsPerCta = kFitThreads * 16;
constexpr int kFitStats = 6;                     // n, n_inter, r0, r1, c0, c1 (int32)

// the empty statistics: nothing counted, an empty box
__device__ __forceinline__ void fit_stats_reset(int* s) {
  s[0] = 0; s[1] = 0; s[2] = 0x7fffffff; s[3] = -1; s[4] = 0x7fffffff; s[5] = -1;
}

// Integer statistics of one image: grid (ceil(H W / kFitPixelsPerCta), P, F).  kSil: the silhouette of hypothesis
// (f, p), z [F, P, H, W] depth bits (+inf where nothing is hit), with its intersection with the mask of frame f, into
// stats [F, P, 6]; otherwise the mask of frame f (nonzero = object) into stats [F, 6] (n_inter unused).  occ
// [F, H, W] (nonzero = something may hide the object; DESIGN.md section 24) may be null: its pixels count for neither
// the silhouette nor the mask, so the statistics are those of S n U and M n U with U the pixels outside occ.  Each CTA
// reduces its pixels through warp reductions and shared memory and adds its partials with one integer atomic per
// field: integer sums, minima and maxima do not depend on the order, so neither does the result.
template <bool kSil>
__global__ void __launch_bounds__(kFitThreads)
fit_stats_kernel(const unsigned* __restrict__ z, const uint8_t* __restrict__ masks, const uint8_t* __restrict__ occ,
                 int P, int H, int W, int* __restrict__ stats) {
  const int p = blockIdx.y, f = blockIdx.z;
  const int hw = H * W;
  const uint8_t* m = masks + (size_t)f * hw;
  const uint8_t* o = occ ? occ + (size_t)f * hw : nullptr;
  const unsigned* zi = kSil ? z + ((size_t)f * P + p) * hw : nullptr;
  const int lo = blockIdx.x * kFitPixelsPerCta, hi = min(lo + kFitPixelsPerCta, hw);
  int n = 0, ni = 0, r0 = 0x7fffffff, r1 = -1, c0 = 0x7fffffff, c1 = -1;
  for (int i = lo + (int)threadIdx.x; i < hi; i += kFitThreads) {
    if (o && o[i] != 0) continue;                // unknown: neither silhouette nor mask
    const bool in_m = m[i] != 0;
    const bool in = kSil ? zi[i] != kDepthInfBits : in_m;
    if (!in) continue;
    const int row = i / W, col = i - row * W;
    ++n;
    ni += (kSil && in_m) ? 1 : 0;
    r0 = min(r0, row); r1 = max(r1, row); c0 = min(c0, col); c1 = max(c1, col);
  }
  n = __reduce_add_sync(0xffffffffu, n);
  ni = __reduce_add_sync(0xffffffffu, ni);
  r0 = __reduce_min_sync(0xffffffffu, r0);
  r1 = __reduce_max_sync(0xffffffffu, r1);
  c0 = __reduce_min_sync(0xffffffffu, c0);
  c1 = __reduce_max_sync(0xffffffffu, c1);
  __shared__ int part[kFitThreads / 32][kFitStats];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (lane == 0) {
    part[warp][0] = n; part[warp][1] = ni; part[warp][2] = r0; part[warp][3] = r1; part[warp][4] = c0;
    part[warp][5] = c1;
  }
  __syncthreads();
  if (threadIdx.x != 0) return;
  for (int w = 1; w < kFitThreads / 32; ++w) {
    n += part[w][0]; ni += part[w][1];
    r0 = min(r0, part[w][2]); r1 = max(r1, part[w][3]); c0 = min(c0, part[w][4]); c1 = max(c1, part[w][5]);
  }
  if (n == 0) return;                            // nothing to add
  int* s = stats + ((size_t)f * (kSil ? P : 1) + (kSil ? p : 0)) * kFitStats;
  atomicAdd(s, n);
  if (kSil) atomicAdd(s + 1, ni);
  atomicMin(s + 2, r0); atomicMax(s + 3, r1); atomicMin(s + 4, c0); atomicMax(s + 5, c1);
}

// box centre (lo + hi + 1) / 2 and size hi - lo + 1 of an integer pixel range, exact in float64
__device__ __forceinline__ double fit_centre(int lo, int hi) { return __dmul_rn((double)(lo + hi + 1), 0.5); }
__device__ __forceinline__ double fit_size(int lo, int hi) { return (double)(hi - lo + 1); }

// One thread per (f, p), n = F P: t = t_init, the first pose, every statistic reset.
__global__ void fit_init_kernel(const double* __restrict__ R, const double* __restrict__ t_init, int F, int P,
                                double* __restrict__ t, float* __restrict__ poses, int* __restrict__ sil_stats,
                                int* __restrict__ mask_stats) {
  const long long n = (long long)F * P;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    double ti[3];
#pragma unroll
    for (int k = 0; k < 3; ++k) { ti[k] = t_init[3 * i + k]; t[3 * i + k] = ti[k]; }
    render_write_pose(R + 9 * i, ti, poses + 16 * i);
    fit_stats_reset(sil_stats + kFitStats * i);
    if (i < F) fit_stats_reset(mask_stats + kFitStats * i);
  }
}

// One update per (f, p), DESIGN.md section 18, every float64 operation rounded on its own:
//   s = sqrt((w_S h_S) / (w_M h_M)), z' = z s, pu = (fx x) / z + cx, pv = (fy y) / z + cy, k = z / z',
//   u' = u_M - (u_S - pu) k, v' = v_M - (v_S - pv) k, x' = ((u' - cx) z') / fx, y' = ((v' - cy) z') / fy.
// An empty silhouette or an empty mask leaves t as it is.  Writes the next float32 pose and resets the silhouette's
// statistics for the next render.  K [F, 4] = (fx, fy, cx, cy).
__global__ void fit_update_kernel(const double* __restrict__ R, const double* __restrict__ K,
                                  const int* __restrict__ mask_stats, int F, int P, double* __restrict__ t,
                                  float* __restrict__ poses, int* __restrict__ sil_stats) {
  const long long n = (long long)F * P;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const int f = (int)(i / P);
    const int* ms = mask_stats + kFitStats * (size_t)f;
    int* ss = sil_stats + kFitStats * i;
    double ti[3] = {t[3 * i], t[3 * i + 1], t[3 * i + 2]};
    if (ss[0] > 0 && ms[0] > 0) {
      const double fx = K[4 * f], fy = K[4 * f + 1], cx = K[4 * f + 2], cy = K[4 * f + 3];
      const double x = ti[0], y = ti[1], z = ti[2];
      const double s = __dsqrt_rn(__ddiv_rn(__dmul_rn(fit_size(ss[4], ss[5]), fit_size(ss[2], ss[3])),
                                            __dmul_rn(fit_size(ms[4], ms[5]), fit_size(ms[2], ms[3]))));
      const double z1 = __dmul_rn(z, s);
      const double pu = __dadd_rn(__ddiv_rn(__dmul_rn(fx, x), z), cx);
      const double pv = __dadd_rn(__ddiv_rn(__dmul_rn(fy, y), z), cy);
      const double k = __ddiv_rn(z, z1);
      const double u1 = __dsub_rn(fit_centre(ms[4], ms[5]), __dmul_rn(__dsub_rn(fit_centre(ss[4], ss[5]), pu), k));
      const double v1 = __dsub_rn(fit_centre(ms[2], ms[3]), __dmul_rn(__dsub_rn(fit_centre(ss[2], ss[3]), pv), k));
      ti[0] = __ddiv_rn(__dmul_rn(__dsub_rn(u1, cx), z1), fx);
      ti[1] = __ddiv_rn(__dmul_rn(__dsub_rn(v1, cy), z1), fy);
      ti[2] = z1;
#pragma unroll
      for (int c = 0; c < 3; ++c) t[3 * i + c] = ti[c];
    }
    render_write_pose(R + 9 * i, ti, poses + 16 * i);
    fit_stats_reset(ss);
  }
}

// The outputs after the last render: t_out [F, P, 3], iou [F, P] = |S n M| / |S u M| (0 for an empty silhouette; S
// and M are restricted to the known pixels when there are occluders), both NaN for a frame whose mask is empty; stats_out [F, P, 6] (optional) the silhouette's statistics.
__global__ void fit_final_kernel(const double* __restrict__ t, const int* __restrict__ mask_stats,
                                 const int* __restrict__ sil_stats, int F, int P, double* __restrict__ t_out,
                                 double* __restrict__ iou, int* __restrict__ stats_out) {
  const long long n = (long long)F * P;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const int f = (int)(i / P);
    const int nm = mask_stats[kFitStats * (size_t)f];
    const int* ss = sil_stats + kFitStats * i;
    const double nan = __longlong_as_double(0x7ff8000000000000LL);
#pragma unroll
    for (int c = 0; c < 3; ++c) t_out[3 * i + c] = nm > 0 ? t[3 * i + c] : nan;
    iou[i] = nm > 0 ? __ddiv_rn((double)ss[1], (double)(ss[0] + nm - ss[1])) : nan;
    if (stats_out) {
#pragma unroll
      for (int c = 0; c < kFitStats; ++c) stats_out[kFitStats * i + c] = ss[c];
    }
  }
}

}  // namespace nope
