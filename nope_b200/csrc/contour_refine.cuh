// nope_b200 -- pose refinement from the object mask's contour (DESIGN.md section 20).
//
// The RGB counterpart of depth_refine.cuh: every pose hypothesis is rendered at its current [R | t] with
// depth_raster_kernel (render.cuh, unchanged), each contour pixel of the rendered silhouette is paired with the
// frame's mask through the mask's signed distance field phi, and one damped Gauss-Newton step of the six pose
// parameters (icp_step, shared with the depth fit) minimises phi along the contour.  phi comes from an exact
// separable Euclidean distance transform in integers; every float64 operation is rounded on its own and every
// per-pixel product is rounded to 64-bit fixed point before it is summed as an integer, so the result does not depend
// on the order of the pixels, the launch shape or the batch: tests/contour_refine_oracle.py restates it in numpy bit
// for bit.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "depth_refine.cuh"
#include "render.cuh"
#include "translation.cuh"

namespace nope {

constexpr int kSdfColThreads = 128;
constexpr int kSdfMaxRowsPerCta = 32;
constexpr int kSdfSmemBytes = 48 * 1024;         // the row pass's envelopes: 4 W bytes per row, W <= 8192

// ---------------------------------------------------------------------------------------------------------------
// The mask's signed distance field.  Pixels outside the frame are neither object nor background.
//   d2_out(r, c) = min over object pixels (r', c') of (r - r')^2 + (c - c')^2   (0 on the object),
//   d2_in(r, c)  = the same over background pixels                               (0 off the object),
//   phi = sqrt(d2_out) - 1/2 off the object, 1/2 - sqrt(d2_in) on it; NaN for a mask that is empty or covers the
// whole frame (it has no contour).  Both minima are exact integers, computed in two separable passes.
// ---------------------------------------------------------------------------------------------------------------

// Column pass: grid (ceil(W / kSdfColThreads), F), one thread per column.  g [F, H, W] packs, for each pixel, the row
// distance to the nearest object pixel of its column (low 16 bits) and to the nearest background pixel (high 16
// bits); "none in the column" is INF = H + W, which is larger than any distance in the frame.  occ [F, H, W] may be
// null; where it is nonzero the pixel is background, so the field is that of M n U (DESIGN.md section 24).  Adjacent
// threads read and write adjacent columns, so every row access is coalesced.
__global__ void __launch_bounds__(kSdfColThreads)
mask_sdf_cols_kernel(const uint8_t* __restrict__ masks, const uint8_t* __restrict__ occ, int H, int W,
                     unsigned* __restrict__ g) {
  const int f = blockIdx.y, c = blockIdx.x * kSdfColThreads + threadIdx.x;
  if (c >= W) return;
  const size_t base = (size_t)f * H * W + c;
  const uint8_t* m = masks + base;
  const uint8_t* o = occ ? occ + base : nullptr;
  unsigned* gc = g + base;
  const int inf = H + W;
  int lo = -inf, lb = -inf;                      // the last object / background row above
  for (int r = 0; r < H; ++r) {
    if (m[(size_t)r * W] && !(o && o[(size_t)r * W])) lo = r; else lb = r;
    gc[(size_t)r * W] = (unsigned)min(r - lo, inf) | ((unsigned)min(r - lb, inf) << 16);
  }
  lo = H - 1 + inf; lb = H - 1 + inf;            // the next object / background row below
  for (int r = H - 1; r >= 0; --r) {
    if (m[(size_t)r * W] && !(o && o[(size_t)r * W])) lo = r; else lb = r;
    const unsigned v = gc[(size_t)r * W];
    gc[(size_t)r * W] = (unsigned)min((int)(v & 0xffffu), lo - r) | ((unsigned)min((int)(v >> 16), lb - r) << 16);
  }
}

// rows of the row pass per CTA: each row's lower envelope takes 4 W bytes of shared memory
__host__ __device__ __forceinline__ int mask_sdf_rows_per_cta(int W) {
  return min(kSdfMaxRowsPerCta, kSdfSmemBytes / (4 * W));
}

// (x - i)^2 + g_i^2: the squared distance from column x to the nearest feature of column i, exact in int32 (< 2^29)
__device__ __forceinline__ int sdf_f(int x, int i, int gi) { return (x - i) * (x - i) + gi * gi; }

// Row pass: grid (ceil(H / rows), F) with rows = mask_sdf_rows_per_cta(W) threads, one per row, and 4 W bytes of
// dynamic shared memory each.  For each of the two features (object, background) the row's lower envelope of the
// parabolas (x - i)^2 + g(i)^2 is built left to right and read right to left (Meijster, Roerdink and Hesselink 2000),
// all in integers, so d2 is exact; phi [F, H, W] is written at the pixels whose own minimum it is: d2_out off the
// object, d2_in on it.  d2 >= INF^2 means the frame has no feature of that kind: phi is NaN.
__global__ void mask_sdf_rows_kernel(const unsigned* __restrict__ g, int H, int W, double* __restrict__ phi) {
  extern __shared__ unsigned sdf_envelope[];
  const int f = blockIdx.y, r = blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= H) return;
  const unsigned* gr = g + ((size_t)f * H + r) * W;
  double* pr = phi + ((size_t)f * H + r) * W;
  unsigned* env = sdf_envelope + (size_t)threadIdx.x * W;     // entry q: s_q | t_q << 16 (both < W <= 8192)
  const int inf2 = (H + W) * (H + W);
  const double nan = __longlong_as_double(0x7ff8000000000000LL);
  for (int ch = 0; ch < 2; ++ch) {
    const int sh = 16 * ch;
    int q = 0, sq = 0, tq = 0, gq = (int)((gr[0] >> sh) & 0xffffu);
    env[0] = 0u;
    for (int u = 1; u < W; ++u) {
      const int gu = (int)((gr[u] >> sh) & 0xffffu);
      while (q >= 0 && sdf_f(tq, sq, gq) > sdf_f(tq, u, gu)) {
        if (--q >= 0) {
          sq = (int)(env[q] & 0xffffu); tq = (int)(env[q] >> 16); gq = (int)((gr[sq] >> sh) & 0xffffu);
        }
      }
      if (q < 0) {
        q = 0; sq = u; tq = 0; gq = gu;
        env[0] = (unsigned)u;
      } else {
        // the first column where u is nearer than s_q: 1 + floor(N / D), N >= 0 because s_q wins at t_q >= 0
        const int w = 1 + (u * u - sq * sq + gu * gu - gq * gq) / (2 * (u - sq));
        if (w < W) {
          ++q; sq = u; tq = w; gq = gu;
          env[q] = (unsigned)u | ((unsigned)w << 16);
        }
      }
    }
    for (int u = W - 1; u >= 0; --u) {
      const int d2 = sdf_f(u, sq, gq);
      const bool on = (gr[u] & 0xffffu) == 0u;   // an object pixel: its d2_out is 0
      if (on == (ch == 1)) {
        const double d = __dsqrt_rn((double)d2);
        pr[u] = d2 >= inf2 ? nan : (ch == 0 ? __dsub_rn(d, 0.5) : __dsub_rn(0.5, d));
      }
      if (u == tq && --q >= 0) {
        sq = (int)(env[q] & 0xffffu); tq = (int)(env[q] >> 16); gq = (int)((gr[sq] >> sh) & 0xffffu);
      }
    }
  }
}

// ---------------------------------------------------------------------------------------------------------------
// The contour fit.  mask_stats [F, 6] are fit_stats_kernel<false>'s statistics of the masks (translation.cuh).
// ---------------------------------------------------------------------------------------------------------------

// Iteration i's pairing tolerance in px: tau_frac s_f with s_f = sqrt(w_M h_M) the mask's box size; NaN for a frame
// without a contour (an empty or a full mask)
__device__ __forceinline__ double contour_tau(double tau_frac, const int* ms, long long hw) {
  if (ms[0] == 0 || ms[0] == hw) return __longlong_as_double(0x7ff8000000000000LL);
  return __dmul_rn(tau_frac, __dsqrt_rn(__dmul_rn(fit_size(ms[4], ms[5]), fit_size(ms[2], ms[3]))));
}

// kappa = t_2 / sqrt(fx fy): one pixel in mm at the hypothesis's distance
__device__ __forceinline__ double contour_kappa(double t2, double fx, double fy) {
  return __ddiv_rn(t2, __dsqrt_rn(__dmul_rn(fx, fy)));
}

// The pairs of one iteration: grid (ceil(H W / kIcpPixelsPerCta), P, F).  z [F, P, H, W] the render of hypothesis
// (f, p) (float bits, +inf where nothing is hit), phi [F, H, W], K [F, 4], t [F, P, 3] the hypotheses' current
// origins.  A contour pixel (interior, hit, a neighbour not hit) is counted into n_contour [F, P]; with e = phi + 1/2
// in [-tau, tau] and a non-zero gradient of phi it adds its fixed-point products to 28 int64 registers.  occ [F, H, W]
// may be null; otherwise a contour pixel counts only when neither it nor a 4-neighbour is in occ (DESIGN.md section
// 24): next to an occluder the object's outline is unknown.  The CTA reduces the registers through warp shuffles and
// shared memory and adds its partials to sums [F, P, 29] with one integer atomic per field.
__global__ void __launch_bounds__(kIcpThreads)
contour_accumulate_kernel(const unsigned* __restrict__ z, const double* __restrict__ phi,
                          const uint8_t* __restrict__ occ, const double* __restrict__ K, const double* __restrict__ t,
                          const int* __restrict__ mask_stats, int P, int H, int W, double tau_frac, double rho,
                          unsigned long long* __restrict__ sums, int* __restrict__ n_contour) {
  const int p = blockIdx.y, f = blockIdx.z;
  const int hw = H * W;
  const size_t h = (size_t)f * P + p;
  const unsigned* zi = z + h * hw;
  const double* ph = phi + (size_t)f * hw;
  const uint8_t* o = occ ? occ + (size_t)f * hw : nullptr;
  const double fx = K[4 * f], fy = K[4 * f + 1], cx = K[4 * f + 2], cy = K[4 * f + 3];
  const double to[3] = {t[3 * h], t[3 * h + 1], t[3 * h + 2]};
  const double tau = contour_tau(tau_frac, mask_stats + kFitStats * f, hw);
  const double kappa = contour_kappa(to[2], fx, fy);
  const int lo = blockIdx.x * kIcpPixelsPerCta, hi = min(lo + kIcpPixelsPerCta, hw);
  long long acc[kIcpSums - 1];
#pragma unroll
  for (int k = 0; k < kIcpSums - 1; ++k) acc[k] = 0;
  int n = 0, nc = 0;
  for (int i = lo + (int)threadIdx.x; i < hi; i += kIcpThreads) {
    const int r = i / W, c = i - r * W;
    if (r == 0 || c == 0 || r == H - 1 || c == W - 1) continue;
    const unsigned d0 = zi[i];
    if (!icp_hit(d0)) continue;
    if (icp_hit(zi[i - 1]) && icp_hit(zi[i + 1]) && icp_hit(zi[i - W]) && icp_hit(zi[i + W])) continue;
    if (o && (o[i] | o[i - 1] | o[i + 1] | o[i - W] | o[i + W])) continue;
    ++nc;
    const double e = __dadd_rn(ph[i], 0.5);
    if (!(fabs(e) <= tau)) continue;
    const double gu = __dmul_rn(__dsub_rn(ph[i + 1], ph[i - 1]), 0.5);
    const double gv = __dmul_rn(__dsub_rn(ph[i + W], ph[i - W]), 0.5);
    if (gu == 0.0 && gv == 0.0) continue;
    double P0[3], A[3], J[6];
    icp_point(r, c, (double)__uint_as_float(d0), fx, fy, cx, cy, P0);
    const double zz = P0[2];
    const double au = __dmul_rn(gu, fx), av = __dmul_rn(gv, fy);
    // n = w kappa, w = the gradient of phi pulled back through the projection at P0
    J[3] = __dmul_rn(__ddiv_rn(au, zz), kappa);
    J[4] = __dmul_rn(__ddiv_rn(av, zz), kappa);
    J[5] = __dmul_rn(-__ddiv_rn(__ddiv_rn(__dadd_rn(__dmul_rn(au, P0[0]), __dmul_rn(av, P0[1])), zz), zz), kappa);
#pragma unroll
    for (int k = 0; k < 3; ++k) A[k] = __dsub_rn(P0[k], to[k]);
    icp_cross(A, J + 3, J);
#pragma unroll
    for (int k = 0; k < 3; ++k) J[k] = __ddiv_rn(J[k], rho);
    icp_add_pair(acc, J, __ddiv_rn(e, tau));
    ++n;
  }
  icp_flush_sums<true>(acc, n, nc, sums + h * kIcpSums, n_contour + h);
}

// One thread per (f, p), n = F P: R, t = the inputs, the first pose, the sums, n_contour and the silhouette and mask
// statistics reset.
__global__ void contour_init_kernel(const double* __restrict__ R_in, const double* __restrict__ t_in, int F, int P,
                                    double* __restrict__ R, double* __restrict__ t, float* __restrict__ poses,
                                    unsigned long long* __restrict__ sums, int* __restrict__ n_contour,
                                    int* __restrict__ sil_stats, int* __restrict__ mask_stats) {
  const long long n = (long long)F * P;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    icp_init_one(i, R_in, t_in, R, t, poses, sums);
    n_contour[i] = 0;
    fit_stats_reset(sil_stats + kFitStats * i);
    if (i < F) fit_stats_reset(mask_stats + kFitStats * i);
  }
}

// One update per (f, p): icp_step at the metric tolerance tau_m = tau kappa (mm), with kappa from the current t; a
// hypothesis at t_2 <= 0 keeps its pose.  Writes the next float32 pose and resets the sums and n_contour for the next
// render.
__global__ void contour_solve_kernel(int F, int P, long long hw, double tau_frac, double rho,
                                     const int* __restrict__ mask_stats, const double* __restrict__ K,
                                     double* __restrict__ R, double* __restrict__ t, float* __restrict__ poses,
                                     unsigned long long* __restrict__ sums, int* __restrict__ n_contour) {
  const long long n = (long long)F * P;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const int f = (int)(i / P);
    unsigned long long* s = sums + kIcpSums * i;
    double* ti = t + 3 * i;
    if (ti[2] > 0.0) {
      const double tau = contour_tau(tau_frac, mask_stats + kFitStats * f, hw);
      icp_step(s, __dmul_rn(tau, contour_kappa(ti[2], K[4 * f], K[4 * f + 1])), rho, R + 9 * i, ti);
    }
    render_write_pose(R + 9 * i, ti, poses + 16 * i);
    for (int k = 0; k < kIcpSums; ++k) s[k] = 0ull;
    n_contour[i] = 0;
  }
}

// The outputs after the last render: R_out [F, P, 9], t_out [F, P, 3], fit [F, P, 4] = (n_in, n_contour,
// rms = tau sqrt(sum e^2 / n_in) px, iou = |S n M| / |S u M| over the known pixels) -- rms is NaN when n_in = 0,
// rms and iou are NaN for a frame without a contour -- and sums_out [F, P, 29] (optional) the integer sums of the last
// render.
__global__ void contour_final_kernel(const double* __restrict__ R, const double* __restrict__ t,
                                     const unsigned long long* __restrict__ sums, const int* __restrict__ n_contour,
                                     const int* __restrict__ mask_stats, const int* __restrict__ sil_stats, int F,
                                     int P, long long hw, double tau_frac, double* __restrict__ R_out,
                                     double* __restrict__ t_out, double* __restrict__ fit,
                                     long long* __restrict__ sums_out) {
  const long long n = (long long)F * P;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const int* ms = mask_stats + kFitStats * (i / P);
    const int* ss = sil_stats + kFitStats * i;
    const unsigned long long* s = sums + kIcpSums * i;
    icp_out_one(i, R, t, sums, R_out, t_out, sums_out);
    const double nin = (double)(long long)s[kIcpSums - 1];
    const double tau = contour_tau(tau_frac, ms, hw);
    fit[4 * i] = nin;
    fit[4 * i + 1] = (double)n_contour[i];
    fit[4 * i + 2] = __dmul_rn(tau, __dsqrt_rn(__ddiv_rn(icp_unfix(s[kIcpSums - 2]), nin)));
    fit[4 * i + 3] = isnan(tau) ? tau : __ddiv_rn((double)ss[1], (double)(ss[0] + ms[0] - ss[1]));
  }
}

}  // namespace nope
