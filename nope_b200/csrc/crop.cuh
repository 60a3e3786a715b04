// nope_b200 -- full-frame crops (DESIGN.md section 13): the reference's virtual-bounding-box crop with its
// dataloaders' input pipeline around it, bit for bit.  Crop b of side S is frame frame_idx[b] pasted onto black
// through its mask (PIL: DIV255(v m)), warped by cv2.warpPerspective (bilinear, constant border 0) through the
// destination -> source map inv_maps[b] (the inverse cv2 computes of crop_frame's M), then ToTensor and x*2-1.
// One thread per output pixel, all three channels; grid (ceil(S*S / 256), B).
//
// Every step follows OpenCV's fixed-point warp: float64 coordinates per 64-column block, each product and sum rounded
// on its own; 32 / W; clamp to the int32 range; round half to even; taps at X >> 5, fractions X & 31; the 32 x 32
// bilinear weight table from float32 products times 32768; (sum v_k w_k + 16384) >> 15.  oracle/crop_oracle.py
// restates it in numpy, and the CPU tests hold that to the live cv2 / PIL / torchvision pipeline.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace nope {

constexpr int kCropThreads = 256;
constexpr int kCropBlockW = 64;        // OpenCV builds coordinates per block of 64 output columns (16 rows x 64)
constexpr int kCropMaxSide = 16384;    // frame H, W: a tap X >> 5 saturated to int16 by OpenCV stays outside
constexpr int kCropMaxS = 4096;

__device__ __forceinline__ int crop_div255(int a) {
  a += 128;
  return ((a >> 8) + a) >> 8;
}

// x * W' clamped as std::max(INT_MIN, std::min(INT_MAX, x)) (NaN -> INT_MAX), rounded half to even
__device__ __forceinline__ int crop_fixed(double v) {
  v = v < 2147483647.0 ? v : 2147483647.0;
  v = -2147483648.0 < v ? v : -2147483648.0;
  return __double2int_rn(v);
}

// The sample of crop pixel (x, y) through the destination -> source map M [9]: the tap origin (sx, sy) and the
// fixed-point bilinear weights wt of taps (sx, sy), (sx+1, sy), (sx, sy+1), (sx+1, sy+1).  crop_warp_kernel and
// crop_hidden_kernel both sample through it.
__device__ __forceinline__ void crop_sample(const double* __restrict__ M, int x, int y, int& sx, int& sy, int wt[4]) {
  const int xb = x & ~(kCropBlockW - 1), x1 = x - xb;
  const double m0 = __ldg(M), m1 = __ldg(M + 1), m2 = __ldg(M + 2), m3 = __ldg(M + 3), m4 = __ldg(M + 4),
               m5 = __ldg(M + 5), m6 = __ldg(M + 6), m7 = __ldg(M + 7), m8 = __ldg(M + 8);
  const double dxb = (double)xb, dy = (double)y, dx1 = (double)x1;
  // block origin (M0 xb + M1 y) + M2, then + M0 x1: OpenCV's association
  const double X0 = __dadd_rn(__dadd_rn(__dmul_rn(m0, dxb), __dmul_rn(m1, dy)), m2);
  const double Y0 = __dadd_rn(__dadd_rn(__dmul_rn(m3, dxb), __dmul_rn(m4, dy)), m5);
  const double W0 = __dadd_rn(__dadd_rn(__dmul_rn(m6, dxb), __dmul_rn(m7, dy)), m8);
  double w = __dadd_rn(W0, __dmul_rn(m6, dx1));
  w = w != 0.0 ? __ddiv_rn(32.0, w) : 0.0;
  const int X = crop_fixed(__dmul_rn(__dadd_rn(X0, __dmul_rn(m0, dx1)), w));
  const int Y = crop_fixed(__dmul_rn(__dadd_rn(Y0, __dmul_rn(m3, dx1)), w));
  const int fx = X & 31, fy = Y & 31;
  sx = X >> 5;
  sy = Y >> 5;

  // float32 1-D weights (1 - i/32, i/32), their product times 32768 rounded, the sum brought to 32768 through the
  // largest (short) or smallest (over) one
  const float ax = __fmul_rn((float)fx, 0.03125f), ay = __fmul_rn((float)fy, 0.03125f);
  const float bx = __fsub_rn(1.f, ax), by = __fsub_rn(1.f, ay);
  wt[0] = __float2int_rn(__fmul_rn(__fmul_rn(by, bx), 32768.f));
  wt[1] = __float2int_rn(__fmul_rn(__fmul_rn(by, ax), 32768.f));
  wt[2] = __float2int_rn(__fmul_rn(__fmul_rn(ay, bx), 32768.f));
  wt[3] = __float2int_rn(__fmul_rn(__fmul_rn(ay, ax), 32768.f));
  const int diff = wt[0] + wt[1] + wt[2] + wt[3] - 32768;
  if (diff != 0) {
    int hi = 0, lo = 0, whi = wt[0], wlo = wt[0];      // first largest / smallest, no indexed register array
#pragma unroll
    for (int k = 1; k < 4; ++k) {
      if (wt[k] > whi) hi = k, whi = wt[k];
      if (wt[k] < wlo) lo = k, wlo = wt[k];
    }
    const int at = diff < 0 ? hi : lo;
#pragma unroll
    for (int k = 0; k < 4; ++k)
      if (k == at) wt[k] -= diff;
  }
}

template <int C>
__global__ void __launch_bounds__(kCropThreads) crop_warp_kernel(
    const uint8_t* __restrict__ frames, int F, int H, int W, const uint8_t* __restrict__ masks,
    const int32_t* __restrict__ frame_idx, const double* __restrict__ inv_maps, int S, float* __restrict__ out) {
  const int b = blockIdx.y;
  const int p = blockIdx.x * kCropThreads + threadIdx.x;
  const int SS = S * S;
  if (p >= SS) return;
  float* o = out + (size_t)b * 3 * SS + p;
  const int f = frame_idx ? __ldg(frame_idx + b) : b;
  if (f < 0 || f >= F) {
    o[0] = -1.f;
    o[SS] = -1.f;
    o[2 * SS] = -1.f;
    return;
  }
  const int y = p / S, x = p - y * S;
  int sx, sy, wt[4];
  crop_sample(inv_maps + 9 * (size_t)b, x, y, sx, sy, wt);

  int acc0 = 0, acc1 = 0, acc2 = 0;
  const uint8_t* fr = frames + (size_t)f * H * W * C;
  const uint8_t* mk = masks ? masks + (size_t)b * H * W : nullptr;
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    const int tx = sx + (k & 1), ty = sy + (k >> 1);
    if (tx < 0 || tx >= W || ty < 0 || ty >= H) continue;     // constant border: the tap reads 0
    const size_t at = (size_t)ty * W + tx;
    const uint8_t* px = fr + at * C;
    const int m = C == 4 ? (int)__ldg(px + 3) : (mk ? (int)__ldg(mk + at) : 255);
    acc0 += crop_div255((int)__ldg(px) * m) * wt[k];
    acc1 += crop_div255((int)__ldg(px + 1) * m) * wt[k];
    acc2 += crop_div255((int)__ldg(px + 2) * m) * wt[k];
  }
  const int acc[3] = {acc0, acc1, acc2};
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    const int u = min(max((acc[c] + 16384) >> 15, 0), 255);
    // ToTensor (u / 255) then x * 2 - 1, each operation rounded on its own
    o[(size_t)c * SS] = __fsub_rn(__fmul_rn(__fdiv_rn((float)u, 255.f), 2.f), 1.f);
  }
}

// The crop-space hidden mask (DESIGN.md section 27): crop pixel (x, y) of detection b is 1 when a tap of its
// crop_warp_kernel sample has a non-zero weight, lies inside the frame and is non-zero in occluders [B, H, W];
// otherwise 0.  out [B, S, S]; one thread per crop pixel, grid (ceil(S * S / 256), B).
__global__ void __launch_bounds__(kCropThreads) crop_hidden_kernel(
    const uint8_t* __restrict__ occluders, int H, int W, const double* __restrict__ inv_maps, int S,
    uint8_t* __restrict__ out) {
  const int b = blockIdx.y;
  const int p = blockIdx.x * kCropThreads + threadIdx.x;
  const int SS = S * S;
  if (p >= SS) return;
  const int y = p / S, x = p - y * S;
  int sx, sy, wt[4];
  crop_sample(inv_maps + 9 * (size_t)b, x, y, sx, sy, wt);
  const uint8_t* ob = occluders + (size_t)b * H * W;
  bool hidden = false;
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    const int tx = sx + (k & 1), ty = sy + (k >> 1);
    if (wt[k] != 0 && tx >= 0 && tx < W && ty >= 0 && ty < H) hidden |= __ldg(ob + (size_t)ty * W + tx) != 0;
  }
  out[(size_t)b * SS + p] = hidden ? 1 : 0;
}

// ---------------------------------------------------------------------------------
// The crop camera (DESIGN.md section 23).  crop_frame maps the square of side s around the object centre o, spanned
// by `upper` and `right`, onto the crop: the warp is the view of a pinhole camera at the real camera's centre with
// rotation R_v (rows right / |right|, -upper / |upper|, o / |o|) and K_v = [[S |o| / s, 0, S/2], [0, S |o| / s, S/2],
// [0, 0, 1]].  float64, every operation rounded on its own; norms sqrt((a a + b b) + c c), divisions per component,
// products (p0 + p1) + p2.  tests/crop_camera_oracle.py restates it op by op.
constexpr int kCropCamMax = 65535;     // F, P

__device__ __forceinline__ double crop_cam_norm(double a, double b, double c) {
  return __dsqrt_rn(__dadd_rn(__dadd_rn(__dmul_rn(a, a), __dmul_rn(b, b)), __dmul_rn(c, c)));
}

// a b - c d, each product rounded
__device__ __forceinline__ double crop_cam_cross(double a, double b, double c, double d) {
  return __dsub_rn(__dmul_rn(a, b), __dmul_rn(c, d));
}

// pose [F, 16] row-major (object -> camera) -> Rv [F, 9] row-major; one thread per pose
__global__ void __launch_bounds__(256) crop_camera_kernel(const double* __restrict__ pose, int F, int keep_inplane,
                                                          double* __restrict__ Rv) {
  for (int f = blockIdx.x * blockDim.x + threadIdx.x; f < F; f += gridDim.x * blockDim.x) {
    const double* p = pose + 16 * (size_t)f;
    const double ox = p[3], oy = p[7], oz = p[11];
    double ux, uy, uz, rx, ry, rz;                                  // upper, right
    if (keep_inplane) {
      ux = 0.0, uy = -oz, uz = oy;
      rx = __dadd_rn(__dmul_rn(oy, oy), __dmul_rn(oz, oz));
      ry = -__dmul_rn(ox, oy);
      rz = -__dmul_rn(ox, oz);
    } else {
      // up = pose . ([0, 0, 6] - o, 1); right = o x up; upper = right x o
      const double ax = __dsub_rn(0.0, ox), ay = __dsub_rn(0.0, oy), az = __dsub_rn(6.0, oz);
      double up[3];
#pragma unroll
      for (int i = 0; i < 3; ++i) {
        const double* r = p + 4 * i;
        up[i] = __dadd_rn(__dadd_rn(__dadd_rn(__dmul_rn(r[0], ax), __dmul_rn(r[1], ay)), __dmul_rn(r[2], az)), r[3]);
      }
      rx = crop_cam_cross(oy, up[2], oz, up[1]);
      ry = crop_cam_cross(oz, up[0], ox, up[2]);
      rz = crop_cam_cross(ox, up[1], oy, up[0]);
      ux = crop_cam_cross(ry, oz, rz, oy);
      uy = crop_cam_cross(rz, ox, rx, oz);
      uz = crop_cam_cross(rx, oy, ry, ox);
    }
    const double nu = crop_cam_norm(ux, uy, uz), nr = crop_cam_norm(rx, ry, rz), no = crop_cam_norm(ox, oy, oz);
    double* o = Rv + 9 * (size_t)f;
    if (nu == 0.0 && nr == 0.0) {
      // crop_frame's image-axes fallback: the square lies parallel to the image plane, R_v = I
#pragma unroll
      for (int i = 0; i < 9; ++i) o[i] = i % 4 == 0 ? 1.0 : 0.0;
      continue;
    }
    o[0] = __ddiv_rn(rx, nr), o[1] = __ddiv_rn(ry, nr), o[2] = __ddiv_rn(rz, nr);
    o[3] = -__ddiv_rn(ux, nu), o[4] = -__ddiv_rn(uy, nu), o[5] = -__ddiv_rn(uz, nu);
    o[6] = __ddiv_rn(ox, no), o[7] = __ddiv_rn(oy, no), o[8] = __ddiv_rn(oz, no);
  }
}

// out[f, p] = A R[f, p] with A = Rv[f]^T (to_camera) or Rv[f]; one thread per 3 x 3, which is read whole before it
// is written, so out may alias R
__global__ void __launch_bounds__(256) crop_rotate_kernel(const double* __restrict__ Rv, const double* R, int P,
                                                          long long n, int to_camera, double* out) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const double* v = Rv + 9 * (size_t)((unsigned)i / (unsigned)P);     // i < F P < 2^32: a 32-bit division
    double a[9], r[9];
#pragma unroll
    for (int k = 0; k < 9; ++k) a[k] = __ldg(v + (to_camera ? (k % 3) * 3 + k / 3 : k)), r[k] = R[9 * i + k];
#pragma unroll
    for (int row = 0; row < 3; ++row)
#pragma unroll
      for (int col = 0; col < 3; ++col)
        out[9 * i + 3 * row + col] = __dadd_rn(__dadd_rn(__dmul_rn(a[3 * row], r[col]),
                                                         __dmul_rn(a[3 * row + 1], r[3 + col])),
                                               __dmul_rn(a[3 * row + 2], r[6 + col]));
  }
}

}  // namespace nope
