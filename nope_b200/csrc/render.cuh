// nope_b200 -- depth rasterizer and VSD kernels for the T-LESS evaluation (DESIGN.md section 12).
//
// Rasterizer: camera-Z depth of a triangle mesh under P poses (model -> OpenCV camera, row-major 4x4, mm), 0 where
// nothing is hit.  Pixel (r, c) samples the image point (c + 1/2, r + 1/2).  Vertices are transformed and projected in
// float32 with every product, quotient and sum rounded on its own; projected coordinates are snapped to fixed point
// with 8 sub-pixel bits and coverage is decided by exact int64 edge functions with a top-left fill rule, so shared
// edges are watertight and the result depends neither on face order nor on winding.  Depth interpolates 1/Z with
// barycentrics from the exact edge values in float64, rounded once to float32, and the z-buffer keeps the minimum
// through atomicMin on the bits of the positive depth: the output is deterministic.  oracle/render_oracle.py
// restates every step in torch.
//
// VSD: vsd_obj's per-pose body (reference src/poses/vsd.py:92-135 with src/poses/vsd_utils.py, visibility "bop19"),
// one 8-CTA cluster per (frame, pose), reduced over the image in a fixed order; one pass serves up to 16 tolerances tau
// (DESIGN.md section 15).
#pragma once
#include <cooperative_groups.h>
#include <cuda_runtime.h>
#include <stdint.h>

namespace nope {

constexpr int kRenderSubBits = 8;              // sub-pixel bits of the fixed-point vertex positions
constexpr float kRenderMaxCoord = 1048576.f;   // |u|, |v| <= 2^20 px, else the triangle is dropped (see DESIGN.md)
constexpr int kRenderMaxSide = 8192;           // H, W <= 8192 = 2^13: sample positions < 2^21 in fixed point
constexpr unsigned kDepthInfBits = 0x7f800000u;
constexpr int kVsdThreads = 512;
constexpr int kVsdCluster = 8;               // CTAs per (frame, pose): one image split 8 ways

__global__ void depth_fill_kernel(unsigned* __restrict__ z, long long n) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x)
    z[i] = kDepthInfBits;
}

// +inf (no surface) -> 0, in place
__global__ void depth_finish_kernel(unsigned* __restrict__ z, long long n) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x)
    if (z[i] == kDepthInfBits) z[i] = 0u;
}

// the rasterizer's pose: [R | t] (float64, R row-major 3x3) rounded to float32, row-major 4x4
__device__ __forceinline__ void render_write_pose(const double* R, const double* t, float* __restrict__ pose) {
#pragma unroll
  for (int r = 0; r < 3; ++r) {
#pragma unroll
    for (int c = 0; c < 3; ++c) pose[4 * r + c] = __double2float_rn(R[3 * r + c]);
    pose[4 * r + 3] = __double2float_rn(t[r]);
  }
  pose[12] = 0.f; pose[13] = 0.f; pose[14] = 0.f; pose[15] = 1.f;
}

struct RVert {
  float z;      // camera Z
  int x, y;     // fixed-point image position, 8 sub-pixel bits
  bool ok;      // Z >= znear and |u|, |v| <= 2^20
};

__device__ __forceinline__ RVert render_project(const float* __restrict__ vtx, int i, const float* m, float fx, float fy,
                                                float cx, float cy, float znear) {
  const float X = vtx[3 * i], Y = vtx[3 * i + 1], Z = vtx[3 * i + 2];
  // camera coordinates: ((m0 X + m1 Y) + m2 Z) + m3, per row
  const float xc = __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(m[0], X), __fmul_rn(m[1], Y)), __fmul_rn(m[2], Z)), m[3]);
  const float yc = __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(m[4], X), __fmul_rn(m[5], Y)), __fmul_rn(m[6], Z)), m[7]);
  const float zc = __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(m[8], X), __fmul_rn(m[9], Y)), __fmul_rn(m[10], Z)), m[11]);
  RVert r;
  r.z = zc;
  r.x = r.y = 0;
  r.ok = zc >= znear;                              // false for NaN too
  if (!r.ok) return r;
  const float u = __fadd_rn(__fdiv_rn(__fmul_rn(fx, xc), zc), cx);
  const float v = __fadd_rn(__fdiv_rn(__fmul_rn(fy, yc), zc), cy);
  r.ok = fabsf(u) <= kRenderMaxCoord && fabsf(v) <= kRenderMaxCoord;
  if (!r.ok) return r;
  r.x = __float2int_rn(__fmul_rn(u, 256.f));       // exact scaling, round half to even
  r.y = __float2int_rn(__fmul_rn(v, 256.f));
  return r;
}

// edge (a -> b) owns its zero-valued samples when it is a top edge (horizontal, pointing +x) or a left edge
// (pointing -y); in image coordinates (y down) with positive area this is the top-left rule
__device__ __forceinline__ bool render_top_left(int dx, int dy) { return dy < 0 || (dy == 0 && dx > 0); }

// One warp per (triangle, pose): grid (ceil(F / 8), P), 256 threads.  The warp's lanes walk the triangle's bounding box
// clipped to the image, 32 samples at a time.  z holds float bits, initialised to +inf.
__global__ void __launch_bounds__(256)
depth_raster_kernel(const float* __restrict__ vtx, int V, const int* __restrict__ faces, int F,
                    const float* __restrict__ poses, float fx, float fy, float cx, float cy, float znear, int H, int W,
                    unsigned* __restrict__ z) {
  const int f = blockIdx.x * 8 + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (f >= F) return;
  const int p = blockIdx.y;
  int i0 = faces[3 * f], i1 = faces[3 * f + 1], i2 = faces[3 * f + 2];
  if (i0 < 0 || i0 >= V || i1 < 0 || i1 >= V || i2 < 0 || i2 >= V) return;
  // canonical vertex order: the lowest index first (a rotation keeps the winding)
  if (i1 < i0 && i1 <= i2) { const int t = i0; i0 = i1; i1 = i2; i2 = t; }
  else if (i2 < i0 && i2 < i1) { const int t = i2; i2 = i1; i1 = i0; i0 = t; }
  float m[12];
#pragma unroll
  for (int k = 0; k < 12; ++k) m[k] = poses[16 * p + k];
  RVert a = render_project(vtx, i0, m, fx, fy, cx, cy, znear);
  RVert b = render_project(vtx, i1, m, fx, fy, cx, cy, znear);
  RVert c = render_project(vtx, i2, m, fx, fy, cx, cy, znear);
  if (!(a.ok && b.ok && c.ok)) return;
  long long area = (long long)(b.x - a.x) * (c.y - a.y) - (long long)(b.y - a.y) * (c.x - a.x);
  if (area == 0) return;
  if (area < 0) {                                  // orient to positive area: no culling
    const RVert t = b; b = c; c = t;
    area = -area;
  }
  const int xmin = min(a.x, min(b.x, c.x)), xmax = max(a.x, max(b.x, c.x));
  const int ymin = min(a.y, min(b.y, c.y)), ymax = max(a.y, max(b.y, c.y));
  // samples at 256 c + 128: c in [ceil((xmin - 128) / 256), floor((xmax - 128) / 256)]
  const int c0 = max(0, -((128 - xmin) >> kRenderSubBits)), c1 = min(W - 1, (xmax - 128) >> kRenderSubBits);
  const int r0 = max(0, -((128 - ymin) >> kRenderSubBits)), r1 = min(H - 1, (ymax - 128) >> kRenderSubBits);
  if (c0 > c1 || r0 > r1) return;
  const int bw = c1 - c0 + 1, n = bw * (r1 - r0 + 1);
  const bool tl0 = render_top_left(c.x - b.x, c.y - b.y);
  const bool tl1 = render_top_left(a.x - c.x, a.y - c.y);
  const bool tl2 = render_top_left(b.x - a.x, b.y - a.y);
  const double iza = __ddiv_rn(1.0, (double)a.z), izb = __ddiv_rn(1.0, (double)b.z), izc = __ddiv_rn(1.0, (double)c.z);
  const double darea = (double)area;
  unsigned* zp = z + (size_t)p * H * W;
  for (int i = lane; i < n; i += 32) {
    const int row = r0 + i / bw, col = c0 + i % bw;
    const int px = (col << kRenderSubBits) + 128, py = (row << kRenderSubBits) + 128;
    const long long w0 = (long long)(c.x - b.x) * (py - b.y) - (long long)(c.y - b.y) * (px - b.x);
    const long long w1 = (long long)(a.x - c.x) * (py - c.y) - (long long)(a.y - c.y) * (px - c.x);
    const long long w2 = (long long)(b.x - a.x) * (py - a.y) - (long long)(b.y - a.y) * (px - a.x);
    const bool in = (w0 > 0 || (w0 == 0 && tl0)) && (w1 > 0 || (w1 == 0 && tl1)) && (w2 > 0 || (w2 == 0 && tl2));
    if (!in) continue;
    const double s = __dadd_rn(__dadd_rn(__dmul_rn((double)w0, iza), __dmul_rn((double)w1, izb)),
                               __dmul_rn((double)w2, izc));
    const float d = __double2float_rn(__ddiv_rn(darea, s));
    atomicMin(zp + (size_t)row * W + col, __float_as_uint(d));
  }
}

// distance of the point that projects to integer pixel (x, y) at depth d: depth_im_to_dist_im_fast
// (vsd_utils.py:40-62), in numpy's order
__device__ __forceinline__ double vsd_dist(double prex, double prey, double d) {
  const double a = __dmul_rn(prex, d), b = __dmul_rn(prey, d);
  return __dsqrt_rn(__dadd_rn(__dadd_rn(__dmul_rn(a, a), __dmul_rn(b, b)), __dmul_rn(d, d)));
}

constexpr int kVsdMaxTaus = 16;              // misalignment tolerances served by one pass

struct VsdTaus {
  double v[kVsdMaxTaus];                       // v[0 .. T) are used
};

// One cluster of kVsdCluster CTAs per (pose p, frame f): grid (kVsdCluster * P, F).  CTA rank r of the cluster
// takes pixels r * kVsdThreads + t, r * kVsdThreads + t + kVsdCluster * kVsdThreads, ...; each CTA reduces its
// partial counts in a fixed tree order and rank 0 adds the kVsdCluster partials in rank order through distributed
// shared memory: no workspace, no atomics, and a result that does not depend on scheduling.  K [F, 4] =
// (fx, fy, cx, cy) float64.  cost_type 0 = "step", 1 = "tlinear".  One pass scores T <= kMaxT tolerances taus.v[j]:
// the distance images, the visibility masks and the intersection / union counts are shared, each tolerance keeps
// its own cost and is reduced through the same tree, one after the other.  out [F, P, T] float64.
template <int kMaxT>
__global__ void __cluster_dims__(kVsdCluster, 1, 1) __launch_bounds__(kVsdThreads)
vsd_kernel(const double* __restrict__ depth_test, const float* __restrict__ depth_gt, const float* __restrict__ depth_est,
           int P, int H, int W, const double* __restrict__ K, float delta, const VsdTaus taus, int T, int cost_type,
           double* __restrict__ out) {
  static_assert(kMaxT >= 1 && kMaxT <= kVsdMaxTaus, "1 <= kMaxT <= kVsdMaxTaus");
  namespace cg = cooperative_groups;
  cg::cluster_group cluster = cg::this_cluster();
  const int rank = (int)cluster.block_rank();
  const int p = blockIdx.x / kVsdCluster, f = blockIdx.y;
  const int hw = H * W;
  const double fx = K[4 * f], fy = K[4 * f + 1], cx = K[4 * f + 2], cy = K[4 * f + 3];
  const double* dt_f = depth_test + (size_t)f * hw;
  const float* dg_f = depth_gt + (size_t)f * hw;
  const float* de_f = depth_est + ((size_t)f * P + p) * hw;
  int n_inter = 0, n_union = 0, n_cost[kMaxT];
  double s_cost[kMaxT];
#pragma unroll
  for (int j = 0; j < kMaxT; ++j) { n_cost[j] = 0; s_cost[j] = 0.0; }
  for (int i = rank * kVsdThreads + threadIdx.x; i < hw; i += kVsdCluster * kVsdThreads) {
    const int y = i / W, x = i % W;
    const double prex = __ddiv_rn(__dsub_rn((double)x, cx), fx), prey = __ddiv_rn(__dsub_rn((double)y, cy), fy);
    const double d_test = vsd_dist(prex, prey, dt_f[i]);
    const double d_gt = vsd_dist(prex, prey, (double)dg_f[i]);
    const double d_est = vsd_dist(prex, prey, (double)de_f[i]);
    // _estimate_visib_mask (vsd_utils.py:91-95): d_diff in float32
    const float t32 = __double2float_rn(d_test);
    const bool test0 = d_test == 0.0;
    const bool vis_gt = (__fsub_rn(__double2float_rn(d_gt), t32) <= delta || test0) && d_gt > 0.0;
    const bool vis_est = ((__fsub_rn(__double2float_rn(d_est), t32) <= delta || test0) && d_est > 0.0) ||
                         (vis_gt && d_est > 0.0);
    n_union += (vis_gt || vis_est) ? 1 : 0;
    if (vis_gt && vis_est) {
      ++n_inter;
      const double dd = fabs(__dsub_rn(d_gt, d_est));
#pragma unroll
      for (int j = 0; j < kMaxT; ++j) {
        if (kMaxT == 1 || j < T) {                 // the T = 1 instantiation needs no test
          if (cost_type == 0) n_cost[j] += dd >= taus.v[j] ? 1 : 0;
          else s_cost[j] = __dadd_rn(s_cost[j], fmin(__ddiv_rn(dd, taus.v[j]), 1.0));
        }
      }
    }
  }
  __shared__ int si[3][kVsdThreads];
  __shared__ double sd[kVsdThreads];
  __shared__ int part_i[2 + kMaxT];                // this CTA's inter, union and per-tolerance costs
  __shared__ double part_d[kMaxT];
  const int t = threadIdx.x;
  si[0][t] = n_inter; si[1][t] = n_union;
#pragma unroll
  for (int j = 0; j < kMaxT; ++j) {
    if (kMaxT == 1 || j < T) {
      si[2][t] = n_cost[j]; sd[t] = s_cost[j];
      __syncthreads();
      for (int s = kVsdThreads / 2; s > 0; s >>= 1) {  // fixed tree order, the same for every tolerance
        if (t < s) {
          if (j == 0) { si[0][t] += si[0][t + s]; si[1][t] += si[1][t + s]; }
          si[2][t] += si[2][t + s];
          sd[t] = __dadd_rn(sd[t], sd[t + s]);
        }
        __syncthreads();
      }
      if (t == 0) {
        if (j == 0) { part_i[0] = si[0][0]; part_i[1] = si[1][0]; }
        part_i[2 + j] = si[2][0]; part_d[j] = sd[0];
      }
      __syncthreads();                             // si[2] / sd are rewritten for the next tolerance
    }
  }
  cluster.sync();                                  // every CTA's partials are in its shared memory
  if (rank == 0 && t < T) {                        // one thread per tolerance
    int inter = 0, uni = 0, cost = 0;
    double sum = 0.0;
    for (int r = 0; r < kVsdCluster; ++r) {        // rank order
      const int* ri = cluster.map_shared_rank(&part_i[0], r);
      const double* rd = cluster.map_shared_rank(&part_d[0], r);
      inter += ri[0]; uni += ri[1]; cost += ri[2 + t];
      sum = __dadd_rn(sum, rd[t]);
    }
    double e = 1.0;
    // (sum(costs) + (union - inter)) / union: an integer sum for "step", a float64 sum for "tlinear"
    if (uni > 0)
      e = cost_type == 0 ? __ddiv_rn((double)(cost + uni - inter), (double)uni)
                         : __ddiv_rn(__dadd_rn(sum, (double)(uni - inter)), (double)uni);
    out[((size_t)f * P + p) * T + t] = e;
  }
  cluster.sync();                                  // no CTA leaves while rank 0 reads its shared memory
}

}  // namespace nope
