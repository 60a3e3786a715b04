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

struct VaeNorm {
  float* gamma = nullptr;
  float* beta = nullptr;
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
// The module kinds, the state_dict schema helpers, the workspace, the launches of a 3x3 convolution, GroupNorm,
// ResnetBlock2D and the mid-block attention, the forward pass over the plan and run_block.  Every buffer holds `cap`
// images (the engine's kChunk); mem also holds the workspace and rot_stage.
struct VaeEngine : ImageEngine {
  enum { kConvIn, kResnet, kDown, kUp, kAttention, kConvOut };
  std::vector<ImageModule> plan;              // conv_in first, conv_out last
  std::map<std::string, VaeNorm> norms;
  // workspace (alloc_workspace), each activation buffer sized for cap images of the widest level
  float* x32[2] = {nullptr, nullptr};         // residual stream, fp32
  ActPair xs[2];                              // residual stream, (hi, lo)
  ActPair nrm;                                // normalised activations / attention output, (hi, lo)
  float* t32 = nullptr;                       // conv1 / qkv / conv_out output, fp32
  double2* gn_part = nullptr;                 // GroupNorm partial sums
  float2* gn_stats = nullptr;                 // GroupNorm (mean, rstd)

  explicit VaeEngine(int cap_) { cap = cap_; }

  // module m of n inputs on the residual stream `cur` -> the new cur.  conv_in reads the raw inputs `in` (images or
  // latents) and starts stream 0; conv_out leaves its fp32 output in t32 for extract_output.  The launches of
  // conv_in and of extract_output are not counted (run_block reports neither; forward adds them).
  virtual int run(const ImageModule& m, int n, int& cur, const float* in, cudaStream_t st) = 0;
  // conv_out's output in t32 -> out, the engine's output layout
  virtual int extract_output(int n, float* out, cudaStream_t st) = 0;

  // n <= cap inputs through the plan -> out
  int forward(const float* in, int n, float* out, cudaStream_t st) {
    launches = 2;   // conv_in and extract_output
    int cur = 0;
    for (const ImageModule& m : plan)
      if (run(m, n, cur, in, st)) return -1;
    return extract_output(n, out, st);
  }

  // Runs one module of the forward pass on its own (nope_vae_run_block, nope_vae_decoder_run_block): x [n, C, H, H]
  // fp32 NCHW (the raw inputs for conv_in) staged as the residual stream -> out: the fp32 stream after the module,
  // out_pair (nullable): its (hi, lo) pair as hi + lo.  conv_out gives the engine's output and has no pair.
  int run_block(const std::string& name, const float* x, int C, int H, int n, float* out, float* out_pair,
                int64_t cap_floats, cudaStream_t st) {
    const ImageModule* m = find_module(plan, name);
    NOPE_CHECK(m, "run_block: unknown module " + name);
    if (check_block(*m, cap, C, H, n, cap_floats)) return -1;
    NOPE_CHECK(!out_pair || m->kind != kConvOut, "run_block: " + name + " has no (hi, lo) output");
    launches = 0;
    int cur = 0;
    if (m->kind != kConvIn && stage_stream(x, C, H, n, st)) return -1;
    if (run(*m, n, cur, x, st)) return -1;
    if (m->kind == kConvOut ? extract_output(n, out, st) : extract_stream(cur, m->Co, m->Ho, n, out, out_pair, st))
      return -1;
    NOPE_CUDA(cudaStreamSynchronize(st));
    return 0;
  }

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

  std::vector<double> dvec(const std::string& k) {
    const auto& v = h(k);
    return std::vector<double>(v.begin(), v.end());
  }
  // a convolution with the taps of `shape` from its staged weight and bias
  int make_plain(const std::string& name, const ConvLayer& shape) {
    const auto& s = staged.at(name + ".weight").shape;
    return pack_conv(name, shape, (int)s[0], (int)s[1], dvec(name + ".weight"), dvec(name + ".bias"));
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
    if (make_norm(p + ".norm1") || make_norm(p + ".norm2") || make_plain(p + ".conv1", conv3x3())) return -1;
    std::vector<double> b = dvec(p + ".conv2.bias");
    if (cin == cout) return pack_conv(p + ".conv2", conv3x3(), cout, cout, dvec(p + ".conv2.weight"), b);
    const std::vector<double> ws = dvec(p + ".conv_shortcut.weight"), bs = dvec(p + ".conv_shortcut.bias");
    for (int o = 0; o < cout; ++o) b[o] += bs[o];
    if (!planar) return pack_conv(p + ".conv2", conv3x3(), cout, cout, dvec(p + ".conv2.weight"), b, cin, &ws);
    if (pack_conv(p + ".conv_shortcut", conv1x1(), cout, cin, ws, std::vector<double>(cout, 0.0))) return -1;
    return pack_conv(p + ".conv2", conv3x3(), cout, cout, dvec(p + ".conv2.weight"), b);
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
      if (pack_conv(a + "qkv", conv1x1(), 1536, 512, W, b)) return -1;
    }
    return pack_conv(a + "proj_attn", conv1x1(), 512, 512, dvec(a + "proj_attn.weight"), dvec(a + "proj_attn.bias"));
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
  // offset of plane q of a parity-planar level-0 tensor with C channels
  size_t plane_off(int q, int C) const { return (size_t)q * cap * 128 * 128 * C; }

  // 3x3 pad-1 convolution at the current level.  Level 0 (parity-planar): one launch per output plane (py, px);
  // tap (oy, ox) of that plane reads input plane ((py + oy) & 1, (px + ox) & 1) at offset ((py + oy) >> 1, ...).
  // Output: out_f32 (+ (hi, lo) when out_lo), residual res (same layout) or the conv's 1x1 shortcut over sc.
  int conv3(const ConvLayer& L, const ActPair& in, int H, int n, const ActPair& out, bool want_lo, float* out_f32,
            const ActPair* res, const ActPair* sc, cudaStream_t st) {
    if (H < 256)
      return conv(L, {{in, -1}}, L.taps(), sc, H, n, false, res, out.hi, want_lo ? out.lo : nullptr, out_f32, st);
    NOPE_CHECK(!sc, "vae conv: no shortcut segments at the 256 x 256 level");
    std::vector<std::pair<ActPair, int>> src;
    for (int q = 0; q < 4; ++q) src.push_back({act_at(in, plane_off(q, L.cin)), -1});
    for (int q = 0; q < 4; ++q) {
      const int py = q >> 1, px = q & 1;
      const size_t o = plane_off(q, L.cout);
      ActPair r;
      if (res) r = act_at(*res, o);
      if (conv(L, src, conv_taps(3, 2, py - 1, px - 1), nullptr, 128, n, false, res ? &r : nullptr, out.hi + o,
               want_lo ? act_at(out, o).lo : nullptr, out_f32 + o, st))
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
      const ConvLayer& S = convs.at(p + ".conv_shortcut");
      for (int q = 0; q < 4; ++q) {
        const size_t i = plane_off(q, cin), o = plane_off(q, cout);
        if (conv(S, {{act_at(xs[cur], i), -1}}, S.taps(), nullptr, 128, n, false, nullptr, sres.hi + o,
                 act_at(sres, o).lo, nullptr, st))
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
    const ConvLayer& qkv = convs.at(a + "qkv");
    if (conv(qkv, {{nrm, -1}}, qkv.taps(), nullptr, 32, n, false, nullptr, xs[nxt].hi, nullptr, t32, st))
      return -1;
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
    const ConvLayer& proj = convs.at(a + "proj_attn");
    if (conv(proj, {{nrm, -1}}, proj.taps(), nullptr, 32, n, false, &xs[cur], xs[nxt].hi,
             xs[nxt].lo, x32[nxt], st))
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
};

}  // namespace nope


// ---------------------------------------------------------------- encoder (DESIGN.md section 16)
struct nope_vae final : nope::VaeEngine {
  static constexpr const char* kName = "VAE";
  static constexpr int kChunk = 16;           // images per pass: the workspace holds this many (~200 MB each)
  float *in_w = nullptr, *in_b = nullptr;
  float* rot_stage = nullptr;                 // kChunk rotated crops, allocated by the first rotated encode
  size_t out_floats() const { return 4 * 32 * 32; }   // per encoded image

  nope_vae() : VaeEngine(kChunk) {}

  void build_plan() {
    const int ch[4] = {128, 256, 512, 512};
    plan = {{"encoder.conv_in", kConvIn, 3, 256, 128, 256}};
    int cin = 128, H = 256;
    for (int i = 0; i < 4; ++i) {
      const std::string blk = "encoder.down_blocks." + std::to_string(i);
      for (int j = 0; j < 2; ++j) {
        plan.push_back({blk + ".resnets." + std::to_string(j), kResnet, cin, H, ch[i], H});
        cin = ch[i];
      }
      if (i < 3) {
        plan.push_back({blk + ".downsamplers.0", kDown, cin, H, cin, H / 2});
        H /= 2;
      }
    }
    plan.push_back({"encoder.mid_block.resnets.0", kResnet, 512, 32, 512, 32});
    plan.push_back({"encoder.mid_block.attentions.0", kAttention, 512, 32, 512, 32});
    plan.push_back({"encoder.mid_block.resnets.1", kResnet, 512, 32, 512, 32});
    // conv_norm_out + SiLU + conv_out + quant_conv's mean x 0.18215
    plan.push_back({"encoder.conv_out", kConvOut, 512, 32, 4, 32});
  }

  void build_schema() {
    for (const nope::ImageModule& m : plan) {
      if (m.kind == kConvIn) {
        expect_conv(m.name, m.Co, m.Ci, 3);
      } else if (m.kind == kResnet) {
        expect_resnet(m.name, m.Ci, m.Co);
      } else if (m.kind == kDown) {
        expect_conv(m.name + ".conv", m.Co, m.Ci, 3);
      } else if (m.kind == kAttention) {
        expect_attention(m.name + ".");
      } else {
        expect_norm("encoder.conv_norm_out", 512);
        expect_conv("encoder.conv_out", 8, 512, 3);
        expect_conv("quant_conv", 8, 8, 1);
      }
    }
  }

  // conv_out followed by quant_conv rows 0-3 (the mean) and the 0.18215 scale, folded in float64
  int make_conv_out() {
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
    return pack_conv("conv_out", nope::conv3x3(), 4, 512, Wf, bf);
  }

  // packs the staged weights (nope::engine_finalize: every schema key is present, device selected)
  int finalize() {
    for (const nope::ImageModule& m : plan) {
      int rc = 0;
      if (m.kind == kConvIn) {
        rc = mem.upload(&in_w, h(m.name + ".weight")) || mem.upload(&in_b, h(m.name + ".bias"));
      } else if (m.kind == kResnet) {
        rc = make_resnet(m.name, m.Ci, m.Co);
      } else if (m.kind == kDown) {
        rc = make_plain(m.name + ".conv", nope::conv_shape(3, 2, 0, 0));   // pad (0, 1): see downsample
      } else if (m.kind == kAttention) {
        rc = make_attention(m.name + ".");
      } else {
        rc = make_norm("encoder.conv_norm_out") || make_conv_out();
      }
      if (rc) return -1;
    }
    // workspace for kChunk images of the 256 x 256 x 128 level
    return alloc_workspace((size_t)kChunk * 256 * 256 * 128);
  }

  // Downsample2D: pad (0, 1, 0, 1) + 3x3 stride 2 from side 2H to H.  Tap (ky, kx) reads input (2y + ky, 2x + kx):
  // sub-lattice (ky & 1, kx & 1) at offset (ky >> 1, kx >> 1); the bottom / right zero padding is the TMA's
  // out-of-bounds fill of offset 1.  The 256 x 256 input's sub-lattices are its planes.
  int downsample(const nope::ConvLayer& L, const nope::ActPair& in, int Hin, int n, const nope::ActPair& out,
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
    return conv(L, src, L.taps(), nullptr, H, n, false, nullptr, out.hi, out.lo, out_f32, st);
  }

  int run(const nope::ImageModule& m, int n, int& cur, const float* images, cudaStream_t st) override {
    using namespace nope;
    switch (m.kind) {
      case kConvIn:
        vae_conv_in_kernel<<<n * 65536 / 2, 256, 0, st>>>(images, in_w, in_b, x32[0], xs[0].hi, xs[0].lo, n, cap);
        NOPE_CUDA(cudaGetLastError());
        cur = 0;
        return 0;
      case kResnet:
        return resnet(m.name, m.Ci, m.Co, m.Hi, n, cur, st);
      case kDown:
        if (downsample(convs.at(m.name + ".conv"), xs[cur], m.Hi, n, xs[1 - cur], x32[1 - cur], st)) return -1;
        cur = 1 - cur;
        return 0;
      case kAttention:
        return attention(m.name + ".", n, cur, st);
      default:
        if (group_norm("encoder.conv_norm_out", x32[cur], 512, 32, n, true, st)) return -1;
        return conv3(convs.at("conv_out"), nrm, 32, n, xs[1 - cur], false, t32, nullptr, nullptr, st);
    }
  }
  int extract_output(int n, float* out, cudaStream_t st) override {
    nope::enc_extract_kernel<<<nope::ew_grid((long long)n * 4 * 1024), 256, 0, st>>>(t32, out, n, 4, 1024,
                                                                                     convs.at("conv_out").cout);
    NOPE_CUDA(cudaGetLastError());
    return 0;
  }

  // n <= kChunk images [n, 3, 256, 256] -> out [n, 4, 32, 32]
  int encode(const float* images, int n, float* out, cudaStream_t st) { return forward(images, n, out, st); }
};

// ---------------------------------------------------------------- decoder (DESIGN.md section 17)
// image = AutoencoderKL.decode(z / 0.18215).sample for z [B, 4, 32, 32]: post_quant_conv 1x1 (4 -> 4); conv_in 3x3
// (4 -> 512); the mid block at 32 x 32; four up blocks of three ResnetBlock2D (512, 512, 256, 128 channels; blocks 0-2
// end in Upsample2D, nearest x2 + 3x3 conv); GroupNorm(32) + SiLU and conv_out 3x3 (128 -> 3).  Up block 3 runs at
// the parity-planar 256 x 256 level; the 64 x 64 and 128 x 128 levels are plain NHWC, as in the encoder.
struct nope_vae_decoder final : nope::VaeEngine {
  static constexpr const char* kName = "VAE decoder";
  static constexpr int kChunk = 8;            // images per pass: 256 x 256 x 256 is 67 MB of fp32 per image
  float *in_w = nullptr, *in_b = nullptr, *pq_w = nullptr, *pq_b = nullptr;
  size_t out_floats() const { return 3 * 256 * 256; }   // per decoded image

  nope_vae_decoder() : VaeEngine(kChunk) {}

  // "decoder.conv_in" is post_quant_conv with 1 / 0.18215, then conv_in, on latents [n, 4, 32, 32];
  // "decoder.conv_out" is conv_norm_out + SiLU + conv_out, giving images [n, 3, 256, 256]
  void build_plan() {
    const int ch[4] = {512, 512, 256, 128};
    plan = {{"decoder.conv_in", kConvIn, 4, 32, 512, 32}};
    plan.push_back({"decoder.mid_block.resnets.0", kResnet, 512, 32, 512, 32});
    plan.push_back({"decoder.mid_block.attentions.0", kAttention, 512, 32, 512, 32});
    plan.push_back({"decoder.mid_block.resnets.1", kResnet, 512, 32, 512, 32});
    int cin = 512, H = 32;
    for (int i = 0; i < 4; ++i) {
      const std::string blk = "decoder.up_blocks." + std::to_string(i);
      for (int j = 0; j < 3; ++j) {
        plan.push_back({blk + ".resnets." + std::to_string(j), kResnet, cin, H, ch[i], H});
        cin = ch[i];
      }
      if (i < 3) {
        plan.push_back({blk + ".upsamplers.0", kUp, cin, H, cin, 2 * H});
        H *= 2;
      }
    }
    plan.push_back({"decoder.conv_out", kConvOut, 128, 256, 3, 256});
  }

  void build_schema() {
    for (const nope::ImageModule& m : plan) {
      if (m.kind == kConvIn) {
        expect_conv("post_quant_conv", 4, 4, 1);
        expect_conv(m.name, m.Co, m.Ci, 3);
      } else if (m.kind == kResnet) {
        expect_resnet(m.name, m.Ci, m.Co);
      } else if (m.kind == kAttention) {
        expect_attention(m.name + ".");
      } else if (m.kind == kUp) {
        expect_conv(m.name + ".conv", m.Co, m.Ci, 3);
      } else {
        expect_norm("decoder.conv_norm_out", m.Ci);
        expect_conv(m.name, m.Co, m.Ci, 3);
      }
    }
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
      if (pack_conv(name + ".p" + std::to_string(q), nope::conv_shape(2, 1, py - 1, px - 1), C, C, Wf, b)) return -1;
    }
    return 0;
  }

  // packs the staged weights (nope::engine_finalize: every schema key is present, device selected)
  int finalize() {
    for (const nope::ImageModule& m : plan) {
      int rc = 0;
      if (m.kind == kConvIn) {
        // post_quant_conv with the 1 / 0.18215 scale folded into its weight in float64; its bias stays separate
        const auto W = dvec("post_quant_conv.weight");
        std::vector<float> w(16);
        for (int i = 0; i < 16; ++i) w[i] = (float)(W[i] / 0.18215);
        rc = mem.upload(&pq_w, w) || mem.upload(&pq_b, h("post_quant_conv.bias")) ||
             mem.upload(&in_w, h(m.name + ".weight")) || mem.upload(&in_b, h(m.name + ".bias"));
      } else if (m.kind == kResnet) {
        rc = make_resnet(m.name, m.Ci, m.Co, m.Hi == 256);
      } else if (m.kind == kAttention) {
        rc = make_attention(m.name + ".");
      } else if (m.kind == kUp) {
        rc = make_upsample(m.name + ".conv", m.Co);
      } else {
        rc = make_norm("decoder.conv_norm_out") || make_plain(m.name, nope::conv3x3());
      }
      if (rc) return -1;
    }
    // workspace for kChunk images of the 256 x 256 x 256 level (the same 3.2 GB as the encoder's)
    return alloc_workspace((size_t)kChunk * 256 * 256 * 256);
  }

  // Upsample2D from side H (residual stream `cur`, plain NHWC) to 2H -> 1 - cur.  One launch per output parity
  // (py, px), the four taps of its layer over the source; the zero padding one row / column past the source's edge is
  // the TMA's out-of-bounds fill.  Into the 256 x 256 level the parity planes are that level's layout; below it they go
  // to (t32, nrm) and are interleaved into plain NHWC.
  int upsample(const std::string& name, int C, int H, int n, int& cur, cudaStream_t st) {
    using namespace nope;
    const int nxt = 1 - cur;
    const bool planar = 2 * H == 256;
    for (int q = 0; q < 4; ++q) {
      const size_t o = (size_t)q * cap * H * H * C;
      float* f = (planar ? x32[nxt] : t32) + o;
      const ActPair d = planar ? ActPair{xs[nxt].hi + o, xs[nxt].lo + o} : ActPair{nrm.hi + o, nrm.lo + o};
      const ConvLayer& L = convs.at(name + ".p" + std::to_string(q));
      if (conv(L, {{xs[cur], -1}}, L.taps(), nullptr, H, n, false, nullptr, d.hi,
               d.lo, f, st))
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

  int run(const nope::ImageModule& m, int n, int& cur, const float* latents, cudaStream_t st) override {
    using namespace nope;
    switch (m.kind) {
      case kConvIn:
        vae_dec_conv_in_kernel<<<dim3(32, n, 2), 256, 0, st>>>(latents, pq_w, pq_b, in_w, in_b, x32[0], xs[0].hi,
                                                               xs[0].lo);
        NOPE_CUDA(cudaGetLastError());
        cur = 0;
        return 0;
      case kResnet:
        return resnet(m.name, m.Ci, m.Co, m.Hi, n, cur, st);
      case kAttention:
        return attention(m.name + ".", n, cur, st);
      case kUp:
        return upsample(m.name + ".conv", m.Co, m.Hi, n, cur, st);
      default:
        if (group_norm("decoder.conv_norm_out", x32[cur], 128, 256, n, true, st)) return -1;
        return conv3(convs.at(m.name), nrm, 256, n, xs[1 - cur], false, t32, nullptr, nullptr, st);
    }
  }
  int extract_output(int n, float* out, cudaStream_t st) override {
    nope::vae_dec_extract_kernel<<<nope::ew_grid((long long)n * 3 * 65536), 256, 0, st>>>(
        t32, convs.at("decoder.conv_out").cout, cap, n, out);
    NOPE_CUDA(cudaGetLastError());
    return 0;
  }

  // n <= kChunk latents [n, 4, 32, 32] -> images out [n, 3, 256, 256] (unclamped)
  int decode(const float* z, int n, float* out, cudaStream_t st) { return forward(z, n, out, st); }
};
