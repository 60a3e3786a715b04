// nope_b200 -- Stable Diffusion VAE encoder and decoder (diffusers AutoencoderKL, SD v1 configuration), fp32-accurate.
// The decoder (nope_vae_decoder at the end of this file, DESIGN.md section 17) shares the host side below
// (nope::VaeEngine) and every kernel but its conv_in, its upsample repack and its output extraction.
//
// latent = AutoencoderKL.encode(x).latent_dist.mode() * 0.18215 for x [B, 3, 256, 256] in [-1, 1]
// (DESIGN.md section 16): conv_in 3x3 (3 -> 128); four down blocks of two ResnetBlock2D each
// (128, 256, 512, 512 channels; blocks 0-2 end in pad (0, 1, 0, 1) + 3x3 stride-2 conv); the mid block
// (ResnetBlock2D, one-head self-attention over 32x32 tokens, ResnetBlock2D); GroupNorm(32) + SiLU, conv_out
// 3x3 (512 -> 8) and quant_conv 1x1, of which the four mean channels are kept.
//
// Precision follows encoder.cuh: every convolution runs on the wgmma kernel (conv_tc2.cuh, the EXTRAS epilogue
// the template encoder already instantiates) with split-precision fp16 (hi, lo) operands -- three K-segments per
// filter tap.  GroupNorm statistics come from the fp32 outputs in a separate pass that sums in float64, per image
// in a fixed order, so they do not depend on the batch or the chunk.  The residual stream is kept as fp32 (for
// the statistics) and as (hi, lo) (for the identity shortcut, added in the conv2 epilogue, and for the 1x1
// shortcut, extra K-segments of conv2).  The attention core (q k^T, softmax, p v) runs on CUDA cores in fp32.
// The encoder's opt-in single-fp16 mode (precision 1, DESIGN.md section 22) packs one fp16 weight per tap, keeps one
// fp16 copy of every stored activation (the lo halves are not allocated; the kernels below skip a null lo) and runs
// one K-segment per tap and source; the fp32 stream, the float64 statistics and the attention core are unchanged.
//
// The 256 x 256 level is wider than one 128-pixel tile row, which the convolution's tile geometry requires.
// Its activations are therefore stored parity-planar: plane (py, px) = 2 py + px holds the pixels (2 Y + py,
// 2 X + px) of every image of the chunk as a [cap, 128, 128, C] NHWC tensor.  A 3x3 convolution at that level is
// four launches, one per output plane, each reading the four input planes with the tap offsets of its parity;
// the stride-2 downsample reads the planes as the four sub-lattices of its input.
#pragma once
#include "conv_tc2.cuh"
#include "encoder.cuh"

#include <cmath>
#include <map>
#include <string>
#include <tuple>
#include <vector>

namespace nope {

constexpr int kVaeSlab = 1024;   // pixels per GroupNorm partial sum (divides every level's H*W per plane)

// conv_in: 3x3 pad 1 (3 -> 128), fp32 direct, -> parity-planar fp32 + (hi, lo) (out_lo nullptr: hi only).
// w: [128][3][3][3] fp32.
// Block = 128 output channels x 2 pixels.
__global__ void __launch_bounds__(256)
vae_conv_in_kernel(const float* __restrict__ x, const float* __restrict__ w, const float* __restrict__ bias,
                   float* __restrict__ out32, __half* __restrict__ out_hi, __half* __restrict__ out_lo, int n,
                   int cap) {
  __shared__ float s_w[128 * 27];
  for (int i = threadIdx.x; i < 128 * 27; i += 256) s_w[i] = w[i];
  __syncthreads();
  const int o = threadIdx.x & 127;
  const int pix = blockIdx.x * 2 + (threadIdx.x >> 7);
  if (pix >= n * 65536) return;
  const int b = pix >> 16, y = (pix >> 8) & 255, xx = pix & 255;
  float acc = bias[o];
  for (int c = 0; c < 3; ++c)
    for (int ky = 0; ky < 3; ++ky) {
      const int yy = y + ky - 1;
      if (yy < 0 || yy > 255) continue;
      const float* xr = x + (((size_t)b * 3 + c) * 256 + yy) * 256;
      const float* wr = s_w + o * 27 + (c * 3 + ky) * 3;
#pragma unroll
      for (int kx = 0; kx < 3; ++kx) {
        const int xc = xx + kx - 1;
        if (xc >= 0 && xc < 256) acc = fmaf(xr[xc], wr[kx], acc);
      }
    }
  const size_t plane = (size_t)((y & 1) * 2 + (xx & 1));
  const size_t dst = (((plane * cap + b) * 128 + (y >> 1)) * 128 + (xx >> 1)) * 128 + o;
  out32[dst] = acc;
  const __half hi = __float2half_rn(acc);
  out_hi[dst] = hi;
  if (out_lo) out_lo[dst] = __float2half_rn(acc - __half2float(hi));
}

// GroupNorm(32) partial sums of fp32 NHWC activations: image b's pixels lie in `planes` planes of [cap, hw, C]
// (plane q of image b at x + (q * cap + b) * hw * C).  grid (planes * hw / kVaeSlab, n): block s sums slab s of
// image b in float64 in a fixed order -> part[(b * gridDim.x + s) * 32 + g] = (sum, sum of squares) of group g.
// C in {128, 256, 512}: a thread owns one 4-channel quad (groups have 4, 8 or 16 channels).
__global__ void __launch_bounds__(256)
vae_gn_partial_kernel(const float* __restrict__ x, int C, int hw, int cap, double2* __restrict__ part) {
  __shared__ double s1[256], s2[256];
  const int b = blockIdx.y, spp = hw / kVaeSlab;
  const int q = blockIdx.x / spp, s0 = (blockIdx.x - q * spp) * kVaeSlab;
  const float* base = x + (((size_t)q * cap + b) * hw + s0) * C;
  const int quads = C >> 2, rows = 256 / quads;
  const int qd = threadIdx.x % quads, r = threadIdx.x / quads;
  double a = 0.0, a2 = 0.0;
  for (int p = r; p < kVaeSlab; p += rows) {
    const float4 v = *reinterpret_cast<const float4*>(base + (size_t)p * C + qd * 4);
    const double v0 = v.x, v1 = v.y, v2 = v.z, v3 = v.w;
    a += (v0 + v1) + (v2 + v3);
    a2 += (v0 * v0 + v1 * v1) + (v2 * v2 + v3 * v3);
  }
  s1[threadIdx.x] = a;
  s2[threadIdx.x] = a2;
  __syncthreads();
  if (threadIdx.x < 32) {
    const int g = threadIdx.x, qpg = quads / 32;
    double t = 0.0, t2 = 0.0;
    for (int rr = 0; rr < rows; ++rr)
      for (int k = 0; k < qpg; ++k) {
        const int i = rr * quads + g * qpg + k;
        t += s1[i];
        t2 += s2[i];
      }
    part[((size_t)b * gridDim.x + blockIdx.x) * 32 + g] = make_double2(t, t2);
  }
}

// (mean, rstd) of every (image, group) from the partial sums, in slab order.  grid n, 32 threads.
__global__ void __launch_bounds__(32)
vae_gn_finalize_kernel(const double2* __restrict__ part, int nparts, double inv_cnt, double eps,
                       float2* __restrict__ stats) {
  const int b = blockIdx.x, g = threadIdx.x;
  double t = 0.0, t2 = 0.0;
  for (int k = 0; k < nparts; ++k) {
    const double2 v = part[((size_t)b * nparts + k) * 32 + g];
    t += v.x;
    t2 += v.y;
  }
  const double mean = t * inv_cnt;
  double var = t2 * inv_cnt - mean * mean;
  if (var < 0.0) var = 0.0;
  // 1 / sqrt(var + eps): rsqrtf refined by one Newton step in float64 (no call to the IEEE slow paths)
  const double v = var + eps, r0 = (double)rsqrtf((float)v);
  stats[b * 32 + g] = make_float2((float)mean, (float)(r0 * (1.5 - 0.5 * v * r0 * r0)));
}

// y = [SiLU]((x - mean) * rstd * gamma + beta) -> (hi, lo) (out_lo nullptr: hi only), same layout as x; 4 channels
// per thread.
// grid (ceil(hw * C / 1024), planes * n): blockIdx.y = q * n + b is image b of plane q (its cap slots hold the n
// images of the chunk first).
__global__ void __launch_bounds__(256)
vae_gn_apply_kernel(const float* __restrict__ x, const float2* __restrict__ stats, const float* __restrict__ gamma,
                    const float* __restrict__ beta, int C, int hw, int n, int cap, int silu,
                    __half* __restrict__ out_hi, __half* __restrict__ out_lo) {
  const int quads = C >> 2;
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= hw * quads) return;
  const int q = (int)blockIdx.y / n, b = (int)blockIdx.y - q * n;
  const int c4 = i % quads;
  const size_t off = ((size_t)q * cap + b) * hw * quads + i;
  const float4 v = reinterpret_cast<const float4*>(x)[off];
  const float2 ms = stats[b * 32 + c4 * 4 / (C >> 5)];
  const float4 ga = reinterpret_cast<const float4*>(gamma)[c4];
  const float4 be = reinterpret_cast<const float4*>(beta)[c4];
  float y[4] = {(v.x - ms.x) * ms.y * ga.x + be.x, (v.y - ms.x) * ms.y * ga.y + be.y,
                (v.z - ms.x) * ms.y * ga.z + be.z, (v.w - ms.x) * ms.y * ga.w + be.w};
  if (silu) {
#pragma unroll
    for (int k = 0; k < 4; ++k) y[k] = __fdividef(y[k], 1.f + expf(-y[k]));
  }
  reinterpret_cast<uint2*>(out_hi)[off] = make_uint2(pack_half2(y[0], y[1]), pack_half2(y[2], y[3]));
  if (!out_lo) return;
  float l[4];
#pragma unroll
  for (int k = 0; k < 4; ++k) l[k] = y[k] - __half2float(__float2half_rn(y[k]));
  reinterpret_cast<uint2*>(out_lo)[off] = make_uint2(pack_half2(l[0], l[1]), pack_half2(l[2], l[3]));
}

// Batched fp32 GEMM of the attention core, one image per blockIdx.z, 64 x 64 tile per block, 4 x 4 per thread,
// every output summed over k in ascending order:
//   C[m, j] = alpha * sum_k A[m, k] B(k, j),  B(k, j) = Bm[j * ldb + k] (KT) or Bm[k * ldb + j].
// SPLIT stores (hi, lo) halves (Clo nullptr: hi only), else fp32.  M, N multiples of 64, K a multiple of 16.
template <bool KT, bool SPLIT>
__global__ void __launch_bounds__(256)
vae_attn_gemm_kernel(const float* __restrict__ A, int lda, long long sa, const float* __restrict__ Bm, int ldb,
                     long long sb, int K, float alpha, float* __restrict__ C32, __half* __restrict__ Chi,
                     __half* __restrict__ Clo, int ldc, long long sc) {
  __shared__ float As[16][64 + 4], Bs[16][64 + 4];
  const int t = threadIdx.x, tx = t & 15, ty = t >> 4;
  const int m0 = blockIdx.y * 64, n0 = blockIdx.x * 64;
  A += blockIdx.z * sa;
  Bm += blockIdx.z * sb;
  float acc[4][4];
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;
  for (int k0 = 0; k0 < K; k0 += 16) {
#pragma unroll
    for (int l = t; l < 1024; l += 256) {
      const int m = l >> 4, k = l & 15;
      As[k][m] = A[(size_t)(m0 + m) * lda + k0 + k];
      if (KT) {
        Bs[k][m] = Bm[(size_t)(n0 + m) * ldb + k0 + k];
      } else {
        const int kk = l >> 6, j = l & 63;
        Bs[kk][j] = Bm[(size_t)(k0 + kk) * ldb + n0 + j];
      }
    }
    __syncthreads();
#pragma unroll
    for (int k = 0; k < 16; ++k) {
      float a[4], bv[4];
#pragma unroll
      for (int i = 0; i < 4; ++i) a[i] = As[k][ty + 16 * i];
#pragma unroll
      for (int j = 0; j < 4; ++j) bv[j] = Bs[k][tx + 16 * j];
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(a[i], bv[j], acc[i][j]);
    }
    __syncthreads();
  }
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const size_t o = blockIdx.z * sc + (size_t)(m0 + ty + 16 * i) * ldc + n0 + tx + 16 * j;
      const float v = acc[i][j] * alpha;
      if (SPLIT) {
        const __half hi = __float2half_rn(v);
        Chi[o] = hi;
        if (Clo) Clo[o] = __float2half_rn(v - __half2float(hi));
      } else {
        C32[o] = v;
      }
    }
}

// Row softmax in place over rows of 1024 fp32 scores: exp(s - max) / sum, both reductions in a fixed tree order.
__global__ void __launch_bounds__(256) vae_softmax_kernel(float* __restrict__ s) {
  __shared__ float red[8];
  float* row = s + (size_t)blockIdx.x * 1024;
  const int t = threadIdx.x, lane = t & 31, w = t >> 5;
  float v[4];
#pragma unroll
  for (int k = 0; k < 4; ++k) v[k] = row[t + 256 * k];
  float m = fmaxf(fmaxf(v[0], v[1]), fmaxf(v[2], v[3]));
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
  if (lane == 0) red[w] = m;
  __syncthreads();
  m = red[0];
#pragma unroll
  for (int k = 1; k < 8; ++k) m = fmaxf(m, red[k]);
  __syncthreads();
#pragma unroll
  for (int k = 0; k < 4; ++k) v[k] = expf(v[k] - m);
  float sum = (v[0] + v[1]) + (v[2] + v[3]);
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
  if (lane == 0) red[w] = sum;
  __syncthreads();
  sum = ((red[0] + red[1]) + (red[2] + red[3])) + ((red[4] + red[5]) + (red[6] + red[7]));
#pragma unroll
  for (int k = 0; k < 4; ++k) row[t + 256 * k] = __fdividef(v[k], sum);
}

// A convolution of the VAE: packed split-precision weights [cout][K] fp16, K = taps x (W_hi | W_lo | W_hi) x cin,
// then, for a ResnetBlock2D conv2 with a 1x1 shortcut, (S_hi | S_lo | S_hi) x cin_sc; bias = b2 (+ b_shortcut).
// In the single-fp16 mode each tap holds W_hi alone: K = taps x cin (+ cin_sc).
struct VaeConv {
  int cin = 0, cin_sc = 0, cout = 0, k = 1, K = 0, bn = 0;
  __half* w = nullptr;
  float* bias = nullptr;
  CUtensorMap wmap;
};

struct VaeNorm {
  float* gamma = nullptr;
  float* beta = nullptr;
};

// One tap of a convolution: input pair (hi map 2 * pair, lo map 2 * pair + 1; fp16 mode: map pair) at (dy, dx).
struct VaeTap {
  int pair, dy, dx;
};

// ---------------------------------------------------------------- decoder kernels (DESIGN.md section 17)

// post_quant_conv (1x1, 4 -> 4, the 1 / 0.18215 scale folded into pq_w) then decoder.conv_in (3x3 pad 1, 4 -> 512),
// fp32 direct, -> NHWC [n, 32, 32, 512] fp32 + (hi, lo).  z: [n, 4, 32, 32] NCHW; w: [512][4][3][3].  conv_in's zero
// padding applies to post_quant_conv's output, so a border pixel sees fewer of post_quant_conv's bias taps.
// grid (32 rows, n, 2 channel halves); one output channel per thread, the 32 pixels of the row in turn.
__global__ void __launch_bounds__(256)
vae_dec_conv_in_kernel(const float* __restrict__ z, const float* __restrict__ pq_w, const float* __restrict__ pq_b,
                       const float* __restrict__ w, const float* __restrict__ bias, float* __restrict__ out32,
                       __half* __restrict__ out_hi, __half* __restrict__ out_lo) {
  __shared__ float s_w[36 * 256];   // [tap][channel]
  __shared__ float s_p[3][34][4];   // post_quant_conv output of rows y - 1 .. y + 1, zero outside the image
  const int y = blockIdx.x, b = blockIdx.y, o0 = blockIdx.z * 256, t = threadIdx.x;
  for (int i = t; i < 36 * 256; i += 256) {
    const int o = i / 36, j = i - o * 36;
    s_w[j * 256 + o] = w[(size_t)o0 * 36 + i];
  }
  if (t < 3 * 34) {
    const int r = t / 34, xx = t - r * 34 - 1, yy = y + r - 1;
    float p[4] = {0.f, 0.f, 0.f, 0.f};
    if (yy >= 0 && yy < 32 && xx >= 0 && xx < 32) {
      float zc[4];
#pragma unroll
      for (int c = 0; c < 4; ++c) zc[c] = z[(((size_t)b * 4 + c) * 32 + yy) * 32 + xx];
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        float a = pq_b[k];
#pragma unroll
        for (int c = 0; c < 4; ++c) a = fmaf(pq_w[k * 4 + c], zc[c], a);
        p[k] = a;
      }
    }
#pragma unroll
    for (int k = 0; k < 4; ++k) s_p[r][xx + 1][k] = p[k];
  }
  __syncthreads();
  float wr[36];
#pragma unroll
  for (int j = 0; j < 36; ++j) wr[j] = s_w[j * 256 + t];
  const int o = o0 + t;
  const float bo = bias[o];
  for (int x = 0; x < 32; ++x) {
    float acc = bo;
#pragma unroll
    for (int c = 0; c < 4; ++c)
#pragma unroll
      for (int ky = 0; ky < 3; ++ky)
#pragma unroll
        for (int kx = 0; kx < 3; ++kx) acc = fmaf(s_p[ky][x + kx][c], wr[(c * 3 + ky) * 3 + kx], acc);
    const size_t dst = (((size_t)b * 32 + y) * 32 + x) * 512 + o;
    out32[dst] = acc;
    const __half hi = __float2half_rn(acc);
    out_hi[dst] = hi;
    out_lo[dst] = __float2half_rn(acc - __half2float(hi));
  }
}

// The four parity planes of an upsample's output ([4][cap][H][H][C]; plane (py, px) = 2 py + px holds the pixels
// (2 Y + py, 2 X + px)) -> plain NHWC [n, 2H, 2H, C], fp32 and (hi, lo); 4 channels per thread.
__global__ void __launch_bounds__(256)
vae_dec_repack_kernel(const float* __restrict__ p32, const __half* __restrict__ phi, const __half* __restrict__ plo,
                      int C, int H, int n, int cap, float* __restrict__ o32, __half* __restrict__ ohi,
                      __half* __restrict__ olo) {
  const int quads = C >> 2, W2 = 2 * H;
  const int total = n * W2 * W2 * quads;
  for (int i = blockIdx.x * 256 + threadIdx.x; i < total; i += gridDim.x * 256) {
    const int c4 = i % quads, pix = i / quads;
    const int xx = pix % W2, yy = (pix / W2) % W2, b = pix / (W2 * W2);
    const int q = (yy & 1) * 2 + (xx & 1);
    const size_t src = ((((size_t)q * cap + b) * H + (yy >> 1)) * H + (xx >> 1)) * quads + c4;
    reinterpret_cast<float4*>(o32)[i] = reinterpret_cast<const float4*>(p32)[src];
    reinterpret_cast<uint2*>(ohi)[i] = reinterpret_cast<const uint2*>(phi)[src];
    reinterpret_cast<uint2*>(olo)[i] = reinterpret_cast<const uint2*>(plo)[src];
  }
}

// conv_out's parity-planar fp32 output ([4][cap][128][128][ld], channels 0-2 real) -> NCHW [n, 3, 256, 256]
__global__ void __launch_bounds__(256)
vae_dec_extract_kernel(const float* __restrict__ t, int ld, int cap, int n, float* __restrict__ out) {
  const int total = n * 3 * 65536;
  for (int i = blockIdx.x * 256 + threadIdx.x; i < total; i += gridDim.x * 256) {
    const int xx = i & 255, yy = (i >> 8) & 255, bc = i >> 16, c = bc % 3, b = bc / 3;
    const int q = (yy & 1) * 2 + (xx & 1);
    out[i] = t[((((size_t)q * cap + b) * 128 + (yy >> 1)) * 128 + (xx >> 1)) * ld + c];
  }
}

// ---------------------------------------------------------------- host side shared by the encoder and the decoder
// The state_dict schema helpers, the split-precision weight packing, the workspace, and the launches of a
// convolution, GroupNorm, ResnetBlock2D and the mid-block attention.  Every buffer holds `cap` images.
struct VaeEngine {
  const int cap;                              // images per pass
  int device = 0, num_sms = 132;
  int precision = 0;                          // 0: split (hi, lo) operands; 1: single fp16 (encoder, before finalize)
  bool finalized = false;
  StagedWeights staged;
  std::map<std::string, VaeConv> convs;
  std::map<std::string, VaeNorm> norms;
  DeviceAllocs mem;                           // weights and workspace
  // workspace (alloc_workspace), each activation buffer sized for cap images of the widest level
  float* x32[2] = {nullptr, nullptr};         // residual stream, fp32
  ActPair xs[2];                              // residual stream, (hi, lo)
  ActPair nrm;                                // normalised activations / attention output, (hi, lo)
  float* t32 = nullptr;                       // conv1 / qkv / conv_out output, fp32
  double2* gn_part = nullptr;                 // GroupNorm partial sums
  float2* gn_stats = nullptr;                 // GroupNorm (mean, rstd)
  std::map<std::tuple<const void*, int, int, int>, CUtensorMap> tmaps;
  int64_t launches = 0;

  explicit VaeEngine(int cap_) : cap(cap_) {}

  // ---------------------------------------------------------------- schema (diffusers AutoencoderKL, SD v1)
  void expect_norm(const std::string& p, int c) {
    staged.expect(p + ".weight", {c});
    staged.expect(p + ".bias", {c});
  }
  void expect_conv(const std::string& p, int cout, int cin, int k) {
    staged.expect(p + ".weight", {cout, cin, k, k});
    staged.expect(p + ".bias", {cout});
  }
  void expect_resnet(const std::string& p, int cin, int cout) {
    expect_norm(p + ".norm1", cin);
    expect_conv(p + ".conv1", cout, cin, 3);
    expect_norm(p + ".norm2", cout);
    expect_conv(p + ".conv2", cout, cout, 3);
    if (cin != cout) expect_conv(p + ".conv_shortcut", cout, cin, 1);
  }
  void expect_attention(const std::string& a) {
    expect_norm(a + "group_norm", 512);
    for (const char* s : {"query", "key", "value", "proj_attn"}) {
      staged.expect(a + s + ".weight", {512, 512});
      staged.expect(a + s + ".bias", {512});
    }
  }

  // ---------------------------------------------------------------- weights
  const std::vector<float>& h(const std::string& k) const { return staged.at(k).data; }

  // W [cout_real][cin][k*k], bias [cout_real] (float64), optional 1x1 shortcut Ws [cout_real][cin_sc] + its bias
  int pack_conv(const std::string& name, int cout_real, int cin, int k, const std::vector<double>& W,
                const std::vector<double>& bias, int cin_sc = 0, const std::vector<double>* Ws = nullptr) {
    VaeConv L;
    L.cin = cin;
    L.cin_sc = cin_sc;
    L.k = k;
    L.cout = (cout_real + 63) / 64 * 64;
    const int taps = k * k, prods = tap_products(precision);
    L.K = (taps * cin + cin_sc) * prods;
    NOPE_CHECK(cin % 64 == 0 && cin_sc % 64 == 0, name + ": input channels must be a multiple of 64");
    L.bn = pick_bn(L.cout);
    std::vector<__half> packed((size_t)L.cout * L.K, __float2half_rn(0.f));
    auto put = [&](__half* dst, int c, int stride, double v) {
      const float wf = (float)v;
      const __half hi = __float2half_rn(wf);
      dst[c] = hi;
      if (prods == 1) return;
      dst[stride + c] = __float2half_rn(wf - __half2float(hi));
      dst[2 * stride + c] = hi;
    };
    for (int o = 0; o < cout_real; ++o) {
      for (int c = 0; c < cin; ++c)
        for (int t = 0; t < taps; ++t)
          put(&packed[(size_t)o * L.K + (size_t)t * prods * cin], c, cin, W[((size_t)o * cin + c) * taps + t]);
      for (int c = 0; c < cin_sc; ++c)
        put(&packed[(size_t)o * L.K + (size_t)taps * prods * cin], c, cin_sc, (*Ws)[(size_t)o * cin_sc + c]);
    }
    std::vector<float> b(L.cout, 0.f);
    for (int o = 0; o < cout_real; ++o) b[o] = (float)bias[o];
    if (mem.upload(&L.w, packed) || mem.upload(&L.bias, b)) return -1;
    if (make_weight_map(&L.wmap, L.w, L.cout, L.K, L.bn)) return -1;
    convs[name] = L;
    return 0;
  }
  std::vector<double> dvec(const std::string& k) {
    const auto& v = h(k);
    return std::vector<double>(v.begin(), v.end());
  }
  int make_plain(const std::string& name, int k) {
    const auto& s = staged.at(name + ".weight").shape;
    return pack_conv(name, (int)s[0], (int)s[1], k, dvec(name + ".weight"), dvec(name + ".bias"));
  }
  int make_norm(const std::string& name) {
    VaeNorm N;
    if (mem.upload(&N.gamma, h(name + ".weight")) || mem.upload(&N.beta, h(name + ".bias"))) return -1;
    norms[name] = N;
    return 0;
  }
  // planar: the block runs at the parity-planar 256 x 256 level, where a 1x1 shortcut is its own convolution (no
  // bias) whose (hi, lo) output is conv2's residual; elsewhere it rides in conv2 as extra K-segments.  Either way
  // the shortcut's bias is added to conv2's in float64.
  int make_resnet(const std::string& p, int cin, int cout, bool planar = false) {
    if (make_norm(p + ".norm1") || make_norm(p + ".norm2") || make_plain(p + ".conv1", 3)) return -1;
    std::vector<double> b = dvec(p + ".conv2.bias");
    if (cin == cout) return pack_conv(p + ".conv2", cout, cout, 3, dvec(p + ".conv2.weight"), b);
    const std::vector<double> ws = dvec(p + ".conv_shortcut.weight"), bs = dvec(p + ".conv_shortcut.bias");
    for (int o = 0; o < cout; ++o) b[o] += bs[o];
    if (!planar) return pack_conv(p + ".conv2", cout, cout, 3, dvec(p + ".conv2.weight"), b, cin, &ws);
    if (pack_conv(p + ".conv_shortcut", cout, cin, 1, ws, std::vector<double>(cout, 0.0))) return -1;
    return pack_conv(p + ".conv2", cout, cout, 3, dvec(p + ".conv2.weight"), b);
  }
  int make_attention(const std::string& a) {
    if (make_norm(a + "group_norm")) return -1;
    {  // q, k, v as one 1x1 convolution 512 -> 1536
      std::vector<double> W, b;
      for (const char* s : {"query", "key", "value"}) {
        const auto w = dvec(a + s + ".weight"), bb = dvec(a + s + ".bias");
        W.insert(W.end(), w.begin(), w.end());
        b.insert(b.end(), bb.begin(), bb.end());
      }
      if (pack_conv(a + "qkv", 1536, 512, 1, W, b)) return -1;
    }
    return pack_conv(a + "proj_attn", 512, 512, 1, dvec(a + "proj_attn.weight"), dvec(a + "proj_attn.bias"));
  }

  // workspace of E elements per activation buffer, allocated once so that no call allocates (or synchronises); the
  // lo halves only in split precision
  int alloc_workspace(size_t E) {
    const bool split = precision == 0;
    for (int s = 0; s < 2; ++s)
      if (mem.alloc(&x32[s], E) || mem.alloc(&xs[s].hi, E) || (split && mem.alloc(&xs[s].lo, E))) return -1;
    if (mem.alloc(&nrm.hi, E) || (split && mem.alloc(&nrm.lo, E)) || mem.alloc(&t32, E)) return -1;
    return mem.alloc(&gn_part, (size_t)cap * 64 * 32) || mem.alloc(&gn_stats, (size_t)cap * 32) ? -1 : 0;
  }

  // ---------------------------------------------------------------- launches
  // NHWC map of `cap` images of side H x H and C channels at base; lattice >= 0: the stride-2 sub-lattice
  // (lattice >> 1, lattice & 1) of a 2H x 2H tensor
  int get_map(const CUtensorMap** out, const void* base, int C, int H, int lattice) {
    const auto key = std::make_tuple(base, lattice, C, H);
    auto it = tmaps.find(key);
    if (it == tmaps.end()) {
      TileGeom g;
      if (make_geom(H, H, &g)) return -1;
      CUtensorMap m;
      const int rc = lattice < 0 ? make_act_map(&m, base, cap, C, g)
                                 : make_unshuffle_map(&m, base, cap, C, g, lattice >> 1, lattice & 1);
      if (rc) return -1;
      it = tmaps.emplace(key, m).first;
    }
    *out = &it->second;
    return 0;
  }
  // offset of plane q of a parity-planar level-0 tensor with C channels
  size_t plane_off(int q, int C) const { return (size_t)q * cap * 128 * 128 * C; }

  // out = conv(taps over the input pairs `in`) [+ shortcut taps over pair sc] + bias [+ res]; output H x H.
  // in: (hi, lo) base pointers of each input pair with their lattice (-1: plain NHWC of side H); fp16 mode: hi only.
  int conv(const VaeConv& L, const std::vector<std::pair<ActPair, int>>& in, int Hin_map,
           const std::vector<VaeTap>& taps, int sc_pair, int H, int n, __half* out_hi, __half* out_lo,
           float* out_f32, const ActPair* res, cudaStream_t st) {
    TileGeom g;
    if (make_geom(H, H, &g)) return -1;
    ConvParams p;
    memset(&p, 0, sizeof p);
    const CUtensorMap* m = nullptr;
    NOPE_CHECK(in.size() <= (size_t)kMaxAMaps / 2, "vae conv: too many input maps");
    const bool split = precision == 0;   // fp16 mode: one map per input (its hi), one segment per tap
    const int mps = split ? 2 : 1;       // maps per input
    for (size_t i = 0; i < in.size(); ++i) {
      const int C = (int)i == sc_pair ? L.cin_sc : L.cin;
      if (get_map(&m, in[i].first.hi, C, Hin_map, in[i].second)) return -1;
      p.amap[mps * i] = *m;
      if (!split) continue;
      if (get_map(&m, in[i].first.lo, C, Hin_map, in[i].second)) return -1;
      p.amap[2 * i + 1] = *m;
    }
    p.n_amaps = mps * (int)in.size();
    int nseg = 0, ksteps = 0;
    auto add = [&](const VaeTap& t, int nch) {
      p.seg[nseg++] = ConvSeg{(int16_t)(mps * t.pair), (int16_t)t.dy, (int16_t)t.dx, (int16_t)nch};     // A_hi W_hi
      ksteps += nch;
      if (!split) return;
      p.seg[nseg++] = ConvSeg{(int16_t)(2 * t.pair), (int16_t)t.dy, (int16_t)t.dx, (int16_t)nch};       // A_hi W_lo
      p.seg[nseg++] = ConvSeg{(int16_t)(2 * t.pair + 1), (int16_t)t.dy, (int16_t)t.dx, (int16_t)nch};   // A_lo W_hi
      ksteps += 2 * nch;
    };
    for (const VaeTap& t : taps) add(t, L.cin / 64);
    if (sc_pair >= 0) add(VaeTap{sc_pair, 0, 0}, L.cin_sc / 64);
    NOPE_CHECK(nseg <= kMaxSeg && ksteps * 64 == L.K, "vae conv: segment table");
    p.bmap = L.wmap;
    if (get_map(&m, out_hi, L.cout, H, -1)) return -1;
    p.omap[0] = *m;
    p.bias = L.bias;
    p.stats_hw = H * H;
    p.stats_noct = L.cout / 8;
    p.n_total = L.cout;
    p.m_valid = n * H * H;
    p.nseg = nseg;
    p.ksteps = ksteps;
    p.m_tiles = geom_m_tiles(g, n);
    p.n_par = 1;
    p.n_tiles_par = L.cout / L.bn;
    p.n_tiles = p.n_tiles_par;
    p.tiles_per_img = g.tiles_per_img;
    p.h_cnt = g.h_cnt;
    p.b_cnt = g.b_cnt;
    p.res_hi = res ? res->hi : nullptr;
    p.res_lo = res ? res->lo : nullptr;
    p.out_lo = out_lo;
    p.out_f32 = out_f32;
    ++launches;
    return launch_conv_tc2(p, L.bn, num_sms, st);
  }

  // 3x3 pad-1 convolution at the current level.  Level 0 (parity-planar): one launch per output plane (py, px);
  // tap (oy, ox) of that plane reads input plane ((py + oy) & 1, (px + ox) & 1) at offset ((py + oy) >> 1, ...).
  // Output: out_f32 (+ (hi, lo) when out_lo), residual res (same layout) or the conv's 1x1 shortcut over sc.
  int conv3(const VaeConv& L, const ActPair& in, int H, int n, const ActPair& out, bool want_lo, float* out_f32,
            const ActPair* res, const ActPair* sc, cudaStream_t st) {
    std::vector<VaeTap> taps;
    if (H < 256) {
      for (int oy = -1; oy <= 1; ++oy)
        for (int ox = -1; ox <= 1; ++ox) taps.push_back(VaeTap{0, oy, ox});
      std::vector<std::pair<ActPair, int>> src{{in, -1}};
      if (sc) src.push_back({*sc, -1});
      return conv(L, src, H, taps, sc ? 1 : -1, H, n, out.hi, want_lo ? out.lo : nullptr, out_f32, res, st);
    }
    NOPE_CHECK(!sc, "vae conv: no shortcut segments at the 256 x 256 level");
    std::vector<std::pair<ActPair, int>> src;
    for (int q = 0; q < 4; ++q) src.push_back({act_at(in, plane_off(q, L.cin)), -1});
    for (int q = 0; q < 4; ++q) {
      const int py = q >> 1, px = q & 1;
      taps.clear();
      for (int oy = -1; oy <= 1; ++oy)
        for (int ox = -1; ox <= 1; ++ox) {
          const int sy = py + oy, sx = px + ox;
          taps.push_back(VaeTap{(sy & 1) * 2 + (sx & 1), sy >> 1, sx >> 1});
        }
      const size_t o = plane_off(q, L.cout);
      ActPair r;
      if (res) r = act_at(*res, o);
      if (conv(L, src, 128, taps, -1, 128, n, out.hi + o, want_lo ? act_at(out, o).lo : nullptr, out_f32 + o,
               res ? &r : nullptr, st))
        return -1;
    }
    return 0;
  }

  // GroupNorm(32, eps 1e-6) [+ SiLU] of the fp32 tensor x (C channels, side H; parity-planar at 256) -> nrm
  int group_norm(const std::string& name, const float* x, int C, int H, int n, bool silu, cudaStream_t st) {
    const VaeNorm& N = norms.at(name);
    const int planes = H == 256 ? 4 : 1, hw = H == 256 ? 128 * 128 : H * H;
    const int nparts = planes * hw / kVaeSlab;
    vae_gn_partial_kernel<<<dim3(nparts, n), 256, 0, st>>>(x, C, hw, cap, gn_part);
    NOPE_CUDA(cudaGetLastError());
    vae_gn_finalize_kernel<<<n, 32, 0, st>>>(gn_part, nparts, 1.0 / ((double)planes * hw * (C / 32)), 1e-6,
                                             gn_stats);
    NOPE_CUDA(cudaGetLastError());
    vae_gn_apply_kernel<<<dim3((hw * C / 4 + 255) / 256, planes * n), 256, 0, st>>>(
        x, gn_stats, N.gamma, N.beta, C, hw, n, cap, silu ? 1 : 0, nrm.hi, nrm.lo);
    NOPE_CUDA(cudaGetLastError());
    launches += 3;
    return 0;
  }

  // ResnetBlock2D on the residual stream `cur` -> 1 - cur
  int resnet(const std::string& p, int cin, int cout, int H, int n, int& cur, cudaStream_t st) {
    const int nxt = 1 - cur;
    if (group_norm(p + ".norm1", x32[cur], cin, H, n, true, st)) return -1;
    const bool sc = cin != cout, planar_sc = sc && H == 256;
    ActPair sres;
    if (planar_sc) {
      // the 1x1 shortcut, one launch per plane, into x32[cur]'s memory (norm1 was its last reader)
      __half* s = reinterpret_cast<__half*>(x32[cur]);
      sres = ActPair{s, precision == 0 ? s + 4 * plane_off(1, cout) : nullptr};
      const VaeConv& S = convs.at(p + ".conv_shortcut");
      for (int q = 0; q < 4; ++q) {
        const size_t i = plane_off(q, cin), o = plane_off(q, cout);
        if (conv(S, {{act_at(xs[cur], i), -1}}, 128, {VaeTap{0, 0, 0}}, -1, 128, n, sres.hi + o, act_at(sres, o).lo,
                 nullptr, nullptr, st))
          return -1;
      }
    }
    // conv1 -> t32; its fp16 high halves land in xs[nxt].hi, which conv2 overwrites
    if (conv3(convs.at(p + ".conv1"), nrm, H, n, xs[nxt], false, t32, nullptr, nullptr, st)) return -1;
    if (group_norm(p + ".norm2", t32, cout, H, n, true, st)) return -1;
    const ActPair* res = !sc ? &xs[cur] : planar_sc ? &sres : nullptr;
    if (conv3(convs.at(p + ".conv2"), nrm, H, n, xs[nxt], true, x32[nxt], res, sc && !planar_sc ? &xs[cur] : nullptr,
              st))
      return -1;
    cur = nxt;
    return 0;
  }

  // mid-block attention (parameters under prefix a) on the 32 x 32 residual stream `cur` -> 1 - cur
  int attention(const std::string& a, int n, int& cur, cudaStream_t st) {
    const int nxt = 1 - cur;
    if (group_norm(a + "group_norm", x32[cur], 512, 32, n, false, st)) return -1;
    // qkv [n * 1024, 1536] fp32 -> t32 (high halves into xs[nxt].hi, overwritten by proj_attn)
    const VaeConv& qkv = convs.at(a + "qkv");
    if (conv(qkv, {{nrm, -1}}, 32, {VaeTap{0, 0, 0}}, -1, 32, n, xs[nxt].hi, nullptr, t32, nullptr, st)) return -1;
    // S = q k^T / sqrt(512) -> x32[nxt] (overwritten by proj_attn), softmax over keys in place
    float* S = x32[nxt];
    vae_attn_gemm_kernel<true, false><<<dim3(16, 16, n), 256, 0, st>>>(
        t32, 1536, 1024LL * 1536, t32 + 512, 1536, 1024LL * 1536, 512, (float)(1.0 / std::sqrt(512.0)), S, nullptr,
        nullptr, 1024, 1024LL * 1024);
    NOPE_CUDA(cudaGetLastError());
    vae_softmax_kernel<<<n * 1024, 256, 0, st>>>(S);
    NOPE_CUDA(cudaGetLastError());
    // O = P v -> nrm (hi, lo) [n * 1024, 512]
    vae_attn_gemm_kernel<false, true><<<dim3(8, 16, n), 256, 0, st>>>(
        S, 1024, 1024LL * 1024, t32 + 1024, 1536, 1024LL * 1536, 1024, 1.f, nullptr, nrm.hi, nrm.lo, 512,
        1024LL * 512);
    NOPE_CUDA(cudaGetLastError());
    launches += 3;
    // x + proj_attn(O)
    if (conv(convs.at(a + "proj_attn"), {{nrm, -1}}, 32, {VaeTap{0, 0, 0}}, -1, 32, n, xs[nxt].hi, xs[nxt].lo,
             x32[nxt], &xs[cur], st))
      return -1;
    cur = nxt;
    return 0;
  }

  // ---------------------------------------------------------------- one module on its own (run_block)
  // x [n, C, H, H] fp32 NCHW -> residual stream 0: x32[0] and xs[0] (parity-planar at 256)
  int stage_stream(const float* x, int C, int H, int n, cudaStream_t st) {
    nchw_f32_to_nhwc_f16_kernel<<<ew_grid((long long)n * C * H * H), 256, 0, st>>>(
        x, xs[0].hi, n, C, H * H, xs[0].lo, false, x32[0], H == 256 ? cap : 0);
    NOPE_CUDA(cudaGetLastError());
    return 0;
  }
  // residual stream `cur` -> out (fp32 stream) and out_pair (hi + lo, if given), [n, C, H, H] fp32 NCHW
  int extract_stream(int cur, int C, int H, int n, float* out, float* out_pair, cudaStream_t st) {
    const int pc = H == 256 ? cap : 0;
    const int g = ew_grid((long long)n * C * H * H);
    nhwc_f16_to_nchw_f32_kernel<<<g, 256, 0, st>>>(nullptr, out, n, C, H * H, nullptr, false, x32[cur], pc);
    if (out_pair)
      nhwc_f16_to_nchw_f32_kernel<<<g, 256, 0, st>>>(xs[cur].hi, out_pair, n, C, H * H, xs[cur].lo, false, nullptr,
                                                     pc);
    NOPE_CUDA(cudaGetLastError());
    return 0;
  }
  // the checks every run_block makes once the module's input shape (Ci, Hi) and output shape (Co, Ho) are known
  int check_block(const std::string& name, int chunk, int C, int H, int n, int Ci, int Hi, int Co, int Ho,
                  int64_t cap_floats) {
    NOPE_CHECK(Ci, "run_block: unknown module " + name);
    NOPE_CHECK(n >= 1 && n <= chunk, "run_block: n must be in [1, " + std::to_string(chunk) + "]");
    NOPE_CHECK(C == Ci && H == Hi, "run_block: " + name + " takes [n, " + std::to_string(Ci) + ", " +
                                       std::to_string(Hi) + ", " + std::to_string(Hi) + "] inputs, got C = " +
                                       std::to_string(C) + ", H = " + std::to_string(H));
    NOPE_CHECK(cap_floats >= (int64_t)n * Co * Ho * Ho, "run_block: output buffer too small");
    return 0;
  }
};

}  // namespace nope

// ---------------------------------------------------------------- encoder (DESIGN.md section 16)
struct nope_vae : nope::VaeEngine {
  static constexpr const char* kName = "VAE";
  static constexpr int kChunk = 16;           // images per pass: the workspace holds this many (~200 MB each)
  static constexpr int kCh[4] = {128, 256, 512, 512};
  float *in_w = nullptr, *in_b = nullptr;
  float* rot_stage = nullptr;                 // kChunk rotated crops

  nope_vae() : VaeEngine(kChunk) {}

  void build_schema() {
    expect_conv("encoder.conv_in", 128, 3, 3);
    int cin = 128;
    for (int i = 0; i < 4; ++i) {
      for (int j = 0; j < 2; ++j) {
        expect_resnet("encoder.down_blocks." + std::to_string(i) + ".resnets." + std::to_string(j), cin, kCh[i]);
        cin = kCh[i];
      }
      if (i < 3) expect_conv("encoder.down_blocks." + std::to_string(i) + ".downsamplers.0.conv", kCh[i], kCh[i], 3);
    }
    for (int j = 0; j < 2; ++j) expect_resnet("encoder.mid_block.resnets." + std::to_string(j), 512, 512);
    expect_attention("encoder.mid_block.attentions.0.");
    expect_norm("encoder.conv_norm_out", 512);
    expect_conv("encoder.conv_out", 8, 512, 3);
    expect_conv("quant_conv", 8, 8, 1);
  }

  // packs the staged weights (nope::engine_finalize: every schema key is present, device selected)
  int finalize() {
    using namespace nope;
    if (mem.upload(&in_w, h("encoder.conv_in.weight")) || mem.upload(&in_b, h("encoder.conv_in.bias"))) return -1;
    int cin = 128;
    for (int i = 0; i < 4; ++i) {
      const std::string blk = "encoder.down_blocks." + std::to_string(i);
      for (int j = 0; j < 2; ++j) {
        if (make_resnet(blk + ".resnets." + std::to_string(j), cin, kCh[i])) return -1;
        cin = kCh[i];
      }
      if (i < 3 && make_plain(blk + ".downsamplers.0.conv", 3)) return -1;
    }
    for (int j = 0; j < 2; ++j)
      if (make_resnet("encoder.mid_block.resnets." + std::to_string(j), 512, 512)) return -1;
    if (make_attention("encoder.mid_block.attentions.0.")) return -1;
    if (make_norm("encoder.conv_norm_out")) return -1;
    {  // conv_out followed by quant_conv rows 0-3 (the mean) and the 0.18215 scale, folded in float64
      const auto W = dvec("encoder.conv_out.weight"), b = dvec("encoder.conv_out.bias");
      const auto Q = dvec("quant_conv.weight"), qb = dvec("quant_conv.bias");
      constexpr double kScale = 0.18215;
      std::vector<double> Wf((size_t)4 * 512 * 9, 0.0), bf(4, 0.0);
      for (int o = 0; o < 4; ++o) {
        double bo = qb[o];
        for (int j = 0; j < 8; ++j) {
          bo += Q[o * 8 + j] * b[j];
          for (size_t i = 0; i < (size_t)512 * 9; ++i) Wf[(size_t)o * 512 * 9 + i] += Q[o * 8 + j] * W[(size_t)j * 512 * 9 + i];
        }
        bf[o] = kScale * bo;
        for (size_t i = 0; i < (size_t)512 * 9; ++i) Wf[(size_t)o * 512 * 9 + i] *= kScale;
      }
      if (pack_conv("conv_out", 4, 512, 3, Wf, bf)) return -1;
    }
    // workspace for kChunk images of the 256 x 256 x 128 level
    if (alloc_workspace((size_t)kChunk * 256 * 256 * 128)) return -1;
    return mem.alloc(&rot_stage, (size_t)kChunk * 3 * 256 * 256);
  }

  // Downsample2D: pad (0, 1, 0, 1) + 3x3 stride 2 from side 2H to H.  Tap (ky, kx) reads input (2y + ky, 2x + kx):
  // sub-lattice (ky & 1, kx & 1) at offset (ky >> 1, kx >> 1); the bottom / right zero padding is the TMA's
  // out-of-bounds fill of offset 1.  The 256 x 256 input's sub-lattices are its planes.
  int downsample(const nope::VaeConv& L, const nope::ActPair& in, int Hin, int n, const nope::ActPair& out,
                 float* out_f32, cudaStream_t st) {
    using namespace nope;
    const int H = Hin / 2;
    std::vector<std::pair<ActPair, int>> src;
    for (int q = 0; q < 4; ++q) {
      if (Hin == 256) {
        src.push_back({act_at(in, plane_off(q, L.cin)), -1});
      } else {
        src.push_back({in, q});
      }
    }
    std::vector<VaeTap> taps;
    for (int ky = 0; ky < 3; ++ky)
      for (int kx = 0; kx < 3; ++kx) taps.push_back(VaeTap{(ky & 1) * 2 + (kx & 1), ky >> 1, kx >> 1});
    return conv(L, src, H, taps, -1, H, n, out.hi, out.lo, out_f32, nullptr, st);
  }

  // n <= kChunk images [n, 3, 256, 256] -> out [n, 4, 32, 32]
  int encode(const float* images, int n, float* out, cudaStream_t st) {
    using namespace nope;
    launches = 0;
    vae_conv_in_kernel<<<n * 65536 / 2, 256, 0, st>>>(images, in_w, in_b, x32[0], xs[0].hi, xs[0].lo, n, kChunk);
    NOPE_CUDA(cudaGetLastError());
    ++launches;
    int cur = 0, H = 256, cin = 128;
    for (int i = 0; i < 4; ++i) {
      const std::string blk = "encoder.down_blocks." + std::to_string(i);
      for (int j = 0; j < 2; ++j) {
        if (resnet(blk + ".resnets." + std::to_string(j), cin, kCh[i], H, n, cur, st)) return -1;
        cin = kCh[i];
      }
      if (i < 3) {
        if (downsample(convs.at(blk + ".downsamplers.0.conv"), xs[cur], H, n, xs[1 - cur], x32[1 - cur], st))
          return -1;
        cur = 1 - cur;
        H /= 2;
      }
    }
    if (resnet("encoder.mid_block.resnets.0", 512, 512, 32, n, cur, st)) return -1;
    if (attention("encoder.mid_block.attentions.0.", n, cur, st)) return -1;
    if (resnet("encoder.mid_block.resnets.1", 512, 512, 32, n, cur, st)) return -1;
    if (group_norm("encoder.conv_norm_out", x32[cur], 512, 32, n, true, st)) return -1;
    const VaeConv& co = convs.at("conv_out");
    if (conv3(co, nrm, 32, n, xs[1 - cur], false, t32, nullptr, nullptr, st)) return -1;
    enc_extract_kernel<<<ew_grid((long long)n * 4 * 1024), 256, 0, st>>>(t32, out, n, 4, 1024, co.cout);
    NOPE_CUDA(cudaGetLastError());
    ++launches;
    return 0;
  }

  // Runs one module of encode() on its own (nope_vae_run_block): x [n, C, H, H] fp32 NCHW (images for conv_in)
  // staged as the residual stream -> out: the fp32 stream after the module, out_pair (nullable): its (hi, lo) pair
  // as hi + lo.  "encoder.conv_out" is conv_norm_out + SiLU + conv_out + quant_conv's mean x 0.18215 and has no pair.
  int run_block(const std::string& name, const float* x, int C, int H, int n, float* out, float* out_pair,
                int64_t cap_floats, cudaStream_t st) {
    using namespace nope;
    enum { kResnet, kDown, kAttention, kIn, kOut } kind = kResnet;
    int Ci = 0, Hi = 0, Co = 0, Ho = 0;
    if (name == "encoder.conv_in") {
      kind = kIn, Ci = 3, Hi = 256, Co = 128, Ho = 256;
    } else if (name == "encoder.conv_out") {
      kind = kOut, Ci = 512, Hi = 32, Co = 4, Ho = 32;
    } else if (name == "encoder.mid_block.attentions.0") {
      kind = kAttention, Ci = Co = 512, Hi = Ho = 32;
    } else if (name == "encoder.mid_block.resnets.0" || name == "encoder.mid_block.resnets.1") {
      Ci = Co = 512, Hi = Ho = 32;
    } else {
      int cin = 128;
      for (int i = 0; i < 4; ++i) {
        const std::string blk = "encoder.down_blocks." + std::to_string(i);
        for (int j = 0; j < 2; ++j) {
          if (name == blk + ".resnets." + std::to_string(j)) Ci = cin, Co = kCh[i], Hi = Ho = 256 >> i;
          cin = kCh[i];
        }
        if (i < 3 && name == blk + ".downsamplers.0") kind = kDown, Ci = Co = kCh[i], Hi = 256 >> i, Ho = Hi / 2;
      }
    }
    if (check_block(name, kChunk, C, H, n, Ci, Hi, Co, Ho, cap_floats)) return -1;
    NOPE_CHECK(!out_pair || kind != kOut, "run_block: encoder.conv_out has no (hi, lo) output");
    launches = 0;
    int cur = 0;
    if (kind == kIn) {
      vae_conv_in_kernel<<<n * 65536 / 2, 256, 0, st>>>(x, in_w, in_b, x32[0], xs[0].hi, xs[0].lo, n, kChunk);
      NOPE_CUDA(cudaGetLastError());
    } else if (stage_stream(x, C, H, n, st)) {
      return -1;
    }
    if (kind == kResnet) {
      if (resnet(name, Ci, Co, H, n, cur, st)) return -1;
    } else if (kind == kAttention) {
      if (attention(name + ".", n, cur, st)) return -1;
    } else if (kind == kDown) {
      if (downsample(convs.at(name + ".conv"), xs[cur], H, n, xs[1 - cur], x32[1 - cur], st)) return -1;
      cur = 1 - cur;
    } else if (kind == kOut) {
      if (group_norm("encoder.conv_norm_out", x32[cur], 512, 32, n, true, st)) return -1;
      const VaeConv& co = convs.at("conv_out");
      if (conv3(co, nrm, 32, n, xs[1 - cur], false, t32, nullptr, nullptr, st)) return -1;
      enc_extract_kernel<<<ew_grid((long long)n * 4 * 1024), 256, 0, st>>>(t32, out, n, 4, 1024, co.cout);
      NOPE_CUDA(cudaGetLastError());
    }
    if (kind != kOut && extract_stream(cur, Co, Ho, n, out, out_pair, st)) return -1;
    NOPE_CUDA(cudaStreamSynchronize(st));
    return 0;
  }

  // images [B, 3, 256, 256] x angles cossin [A, 2] -> out [B, A, 4, 32, 32]: the (image, angle) pairs in b-major
  // order, kChunk at a time rotated into rot_stage and encoded from there (the chunks encode() makes of that batch)
  int encode_inplane(const float* images, int B, const float* cossin, int A, float* out, cudaStream_t st) {
    using namespace nope;
    NOPE_CHECK((int64_t)B * A <= INT32_MAX, "too many (image, angle) pairs");
    const int pairs = B * A;
    int64_t total = 0;
    for (int lo = 0; lo < pairs; lo += kChunk) {
      const int n = pairs - lo < kChunk ? pairs - lo : kChunk;
      inplane_rotate_kernel<<<dim3(256 * 256 / 256, n), 256, 0, st>>>(images, cossin, A, 256, 256, lo, rot_stage);
      NOPE_CUDA(cudaGetLastError());
      if (encode(rot_stage, n, out + (size_t)lo * 4 * 32 * 32, st)) return -1;
      total += launches + 1;
    }
    launches = total;
    return 0;
  }

  // images [B, 3, 256, 256] x pairs (image_idx [P], cossin [P, 2]) -> out [P, 4, 32, 32], kChunk pairs at a time
  int encode_rotated(const float* images, int B, const int* image_idx, const float* cossin, int P, float* out,
                     cudaStream_t st) {
    using namespace nope;
    int64_t total = 0;
    for (int lo = 0; lo < P; lo += kChunk) {
      const int n = P - lo < kChunk ? P - lo : kChunk;
      inplane_rotate_pairs_kernel<<<dim3(256 * 256 / 256, n), 256, 0, st>>>(images, B, image_idx, cossin, 256, 256,
                                                                             lo, rot_stage);
      NOPE_CUDA(cudaGetLastError());
      if (encode(rot_stage, n, out + (size_t)lo * 4 * 32 * 32, st)) return -1;
      total += launches + 1;
    }
    launches = total;
    return 0;
  }
};

// ---------------------------------------------------------------- decoder (DESIGN.md section 17)
// image = AutoencoderKL.decode(z / 0.18215).sample for z [B, 4, 32, 32]: post_quant_conv 1x1 (4 -> 4); conv_in 3x3
// (4 -> 512); the mid block at 32 x 32; four up blocks of three ResnetBlock2D (512, 512, 256, 128 channels; blocks 0-2
// end in Upsample2D, nearest x2 + 3x3 conv); GroupNorm(32) + SiLU and conv_out 3x3 (128 -> 3).  Up block 3 runs at
// the parity-planar 256 x 256 level; the 64 x 64 and 128 x 128 levels are plain NHWC, as in the encoder.
struct nope_vae_decoder : nope::VaeEngine {
  static constexpr const char* kName = "VAE decoder";
  static constexpr int kChunk = 8;            // images per pass: 256 x 256 x 256 is 67 MB of fp32 per image
  static constexpr int kCh[4] = {512, 512, 256, 128};
  static constexpr const char* kAttn = "decoder.mid_block.attentions.0.";
  float *in_w = nullptr, *in_b = nullptr, *pq_w = nullptr, *pq_b = nullptr;

  nope_vae_decoder() : VaeEngine(kChunk) {}

  static std::string up(int i) { return "decoder.up_blocks." + std::to_string(i); }

  void build_schema() {
    expect_conv("post_quant_conv", 4, 4, 1);
    expect_conv("decoder.conv_in", 512, 4, 3);
    expect_resnet("decoder.mid_block.resnets.0", 512, 512);
    expect_attention(kAttn);
    expect_resnet("decoder.mid_block.resnets.1", 512, 512);
    int cin = 512;
    for (int i = 0; i < 4; ++i) {
      for (int j = 0; j < 3; ++j) {
        expect_resnet(up(i) + ".resnets." + std::to_string(j), cin, kCh[i]);
        cin = kCh[i];
      }
      if (i < 3) expect_conv(up(i) + ".upsamplers.0.conv", kCh[i], kCh[i], 3);
    }
    expect_norm("decoder.conv_norm_out", 128);
    expect_conv("decoder.conv_out", 3, 128, 3);
  }

  // Upsample2D's 3x3 kernel folded into one 2x2 kernel per output parity (py, px), in float64.  Output row 2 Y + py
  // with tap ky reads upsampled row 2 Y + py + ky - 1, i.e. source row Y + floor((py + ky - 1) / 2): offsets
  // py - 1 + a, a = 0, 1, and the fold adds the taps that land on the same source row (the same for columns).
  static int fold_dy(int p, int k) { return (p + k + 1) / 2 - 1; }
  int make_upsample(const std::string& name, int C) {
    const std::vector<double> W = dvec(name + ".weight"), b = dvec(name + ".bias");
    for (int q = 0; q < 4; ++q) {
      const int py = q >> 1, px = q & 1;
      std::vector<double> Wf((size_t)C * C * 4, 0.0);
      for (size_t oc = 0; oc < (size_t)C * C; ++oc)
        for (int ky = 0; ky < 3; ++ky)
          for (int kx = 0; kx < 3; ++kx) {
            const int a = fold_dy(py, ky) - py + 1, bb = fold_dy(px, kx) - px + 1;
            Wf[oc * 4 + a * 2 + bb] += W[oc * 9 + ky * 3 + kx];
          }
      if (pack_conv(name + ".p" + std::to_string(q), C, C, 2, Wf, b)) return -1;
    }
    return 0;
  }

  // packs the staged weights (nope::engine_finalize: every schema key is present, device selected)
  int finalize() {
    using namespace nope;
    {  // post_quant_conv with the 1 / 0.18215 scale folded into its weight in float64; its bias stays separate
      const auto W = dvec("post_quant_conv.weight");
      std::vector<float> w(16);
      for (int i = 0; i < 16; ++i) w[i] = (float)(W[i] / 0.18215);
      if (mem.upload(&pq_w, w) || mem.upload(&pq_b, h("post_quant_conv.bias"))) return -1;
    }
    if (mem.upload(&in_w, h("decoder.conv_in.weight")) || mem.upload(&in_b, h("decoder.conv_in.bias"))) return -1;
    if (make_resnet("decoder.mid_block.resnets.0", 512, 512) || make_attention(kAttn) ||
        make_resnet("decoder.mid_block.resnets.1", 512, 512))
      return -1;
    int cin = 512;
    for (int i = 0; i < 4; ++i) {
      for (int j = 0; j < 3; ++j) {
        if (make_resnet(up(i) + ".resnets." + std::to_string(j), cin, kCh[i], i == 3)) return -1;
        cin = kCh[i];
      }
      if (i < 3 && make_upsample(up(i) + ".upsamplers.0.conv", kCh[i])) return -1;
    }
    if (make_norm("decoder.conv_norm_out") || make_plain("decoder.conv_out", 3)) return -1;
    // workspace for kChunk images of the 256 x 256 x 256 level (the same 3.2 GB as the encoder's)
    return alloc_workspace((size_t)kChunk * 256 * 256 * 256);
  }

  // Upsample2D from side H (residual stream `cur`, plain NHWC) to 2H -> 1 - cur.  One launch per output parity
  // (py, px), four taps over the source; the zero padding one row / column past the source's edge is the TMA's
  // out-of-bounds fill.  Into the 256 x 256 level the parity planes are that level's layout; below it they go to
  // (t32, nrm) and are interleaved into plain NHWC.
  int upsample(const std::string& name, int C, int H, int n, int& cur, cudaStream_t st) {
    using namespace nope;
    const int nxt = 1 - cur;
    const bool planar = 2 * H == 256;
    for (int q = 0; q < 4; ++q) {
      const int py = q >> 1, px = q & 1;
      std::vector<VaeTap> taps;
      for (int a = 0; a < 2; ++a)
        for (int b = 0; b < 2; ++b) taps.push_back(VaeTap{0, py - 1 + a, px - 1 + b});
      const size_t o = (size_t)q * cap * H * H * C;
      float* f = (planar ? x32[nxt] : t32) + o;
      const ActPair d = planar ? ActPair{xs[nxt].hi + o, xs[nxt].lo + o} : ActPair{nrm.hi + o, nrm.lo + o};
      if (conv(convs.at(name + ".p" + std::to_string(q)), {{xs[cur], -1}}, H, taps, -1, H, n, d.hi, d.lo, f, nullptr,
               st))
        return -1;
    }
    if (!planar) {
      vae_dec_repack_kernel<<<ew_grid((long long)n * 4 * H * H * (C / 4)), 256, 0, st>>>(
          t32, nrm.hi, nrm.lo, C, H, n, cap, x32[nxt], xs[nxt].hi, xs[nxt].lo);
      NOPE_CUDA(cudaGetLastError());
      ++launches;
    }
    cur = nxt;
    return 0;
  }

  // n <= kChunk latents [n, 4, 32, 32] -> images out [n, 3, 256, 256] (unclamped)
  int decode(const float* z, int n, float* out, cudaStream_t st) {
    using namespace nope;
    launches = 0;
    vae_dec_conv_in_kernel<<<dim3(32, n, 2), 256, 0, st>>>(z, pq_w, pq_b, in_w, in_b, x32[0], xs[0].hi, xs[0].lo);
    NOPE_CUDA(cudaGetLastError());
    ++launches;
    int cur = 0, H = 32, cin = 512;
    if (resnet("decoder.mid_block.resnets.0", 512, 512, 32, n, cur, st) || attention(kAttn, n, cur, st) ||
        resnet("decoder.mid_block.resnets.1", 512, 512, 32, n, cur, st))
      return -1;
    for (int i = 0; i < 4; ++i) {
      for (int j = 0; j < 3; ++j) {
        if (resnet(up(i) + ".resnets." + std::to_string(j), cin, kCh[i], H, n, cur, st)) return -1;
        cin = kCh[i];
      }
      if (i < 3) {
        if (upsample(up(i) + ".upsamplers.0.conv", kCh[i], H, n, cur, st)) return -1;
        H *= 2;
      }
    }
    if (group_norm("decoder.conv_norm_out", x32[cur], 128, 256, n, true, st)) return -1;
    const VaeConv& co = convs.at("decoder.conv_out");
    if (conv3(co, nrm, 256, n, xs[1 - cur], false, t32, nullptr, nullptr, st)) return -1;
    vae_dec_extract_kernel<<<ew_grid((long long)n * 3 * 65536), 256, 0, st>>>(t32, co.cout, cap, n, out);
    NOPE_CUDA(cudaGetLastError());
    ++launches;
    return 0;
  }

  // Runs one module of decode() on its own (nope_vae_decoder_run_block), as nope_vae::run_block: "decoder.conv_in"
  // (post_quant_conv with 1 / 0.18215, then conv_in) takes latents [n, 4, 32, 32]; "decoder.conv_out"
  // (conv_norm_out + SiLU + conv_out) gives images [n, 3, 256, 256] and has no pair.
  int run_block(const std::string& name, const float* x, int C, int H, int n, float* out, float* out_pair,
                int64_t cap_floats, cudaStream_t st) {
    using namespace nope;
    enum { kResnet, kUp, kAttention, kIn, kOut } kind = kResnet;
    int Ci = 0, Hi = 0, Co = 0, Ho = 0;
    if (name == "decoder.conv_in") {
      kind = kIn, Ci = 4, Hi = 32, Co = 512, Ho = 32;
    } else if (name == "decoder.conv_out") {
      kind = kOut, Ci = 128, Hi = 256, Co = 3, Ho = 256;
    } else if (name + "." == kAttn) {
      kind = kAttention, Ci = Co = 512, Hi = Ho = 32;
    } else if (name == "decoder.mid_block.resnets.0" || name == "decoder.mid_block.resnets.1") {
      Ci = Co = 512, Hi = Ho = 32;
    } else {
      int cin = 512;
      for (int i = 0; i < 4; ++i) {
        for (int j = 0; j < 3; ++j) {
          if (name == up(i) + ".resnets." + std::to_string(j)) Ci = cin, Co = kCh[i], Hi = Ho = 32 << i;
          cin = kCh[i];
        }
        if (i < 3 && name == up(i) + ".upsamplers.0") kind = kUp, Ci = Co = kCh[i], Hi = 32 << i, Ho = 2 * Hi;
      }
    }
    if (check_block(name, kChunk, C, H, n, Ci, Hi, Co, Ho, cap_floats)) return -1;
    NOPE_CHECK(!out_pair || kind != kOut, "run_block: decoder.conv_out has no (hi, lo) output");
    launches = 0;
    int cur = 0;
    if (kind == kIn) {
      vae_dec_conv_in_kernel<<<dim3(32, n, 2), 256, 0, st>>>(x, pq_w, pq_b, in_w, in_b, x32[0], xs[0].hi, xs[0].lo);
      NOPE_CUDA(cudaGetLastError());
    } else if (stage_stream(x, C, H, n, st)) {
      return -1;
    }
    if (kind == kResnet) {
      if (resnet(name, Ci, Co, H, n, cur, st)) return -1;
    } else if (kind == kAttention) {
      if (attention(kAttn, n, cur, st)) return -1;
    } else if (kind == kUp) {
      if (upsample(name + ".conv", Co, H, n, cur, st)) return -1;
    } else if (kind == kOut) {
      if (group_norm("decoder.conv_norm_out", x32[cur], 128, 256, n, true, st)) return -1;
      const VaeConv& co = convs.at("decoder.conv_out");
      if (conv3(co, nrm, 256, n, xs[1 - cur], false, t32, nullptr, nullptr, st)) return -1;
      vae_dec_extract_kernel<<<ew_grid((long long)n * 3 * 65536), 256, 0, st>>>(t32, co.cout, cap, n, out);
      NOPE_CUDA(cudaGetLastError());
    }
    if (kind != kOut && extract_stream(cur, Co, Ho, n, out, out_pair, st)) return -1;
    NOPE_CUDA(cudaStreamSynchronize(st));
    return 0;
  }
};
