// nope_b200 -- the HBM-bound kernels around the tensor-core convolutions:
// weight packing, pose embedding, GroupNorm(+SiLU,+pose bias,+residual), linear
// attention, bottleneck attention, nearest upsample, the fused final 1x1 conv +
// l2 score, top-k.  All activations are NHWC fp16; statistics, softmax and
// scores are fp32.  Each kernel cites the reference code it reproduces (paths
// relative to the reference root).
#pragma once
#include "common.cuh"

namespace nope {

// ----------------------------------------------------------------------------
// weight packing (once, at load time)
// ----------------------------------------------------------------------------
// src fp32 [Cout][Cin][T] (OIHW with T = KH*KW, or the [Cout][Cin*4] weight of the
// 1x1 after pixel-unshuffle, whose input channel index is c*4 + p1*2 + p2,
// model_utils.py:168-172) -> dst fp16 [Cout][T][Cin]  (K-major for the GEMM).
// lo_off > 0 additionally writes the fp16 remainder W - fp16(W) at column lo_off + (t*cin + c):
// the "exact weights" K-segments of the split-precision modes (22 significant bits per weight).
__global__ void pack_weight_kernel(const float* __restrict__ src, __half* __restrict__ dst,
                                   int cout, int cin, int taps, int dst_row_stride,
                                   int dst_col_off, int lo_off = 0, int bf16 = 0) {
  const long long total = (long long)cout * cin * taps;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const int c = (int)(i % cin);
    const int t = (int)((i / cin) % taps);
    const int o = (int)(i / ((long long)cin * taps));
    const float w = src[((long long)o * cin + c) * taps + t];
    __half* d = dst + (long long)o * dst_row_stride + dst_col_off + t * cin + c;
    if (bf16) { st16(d, w, true); continue; }
    const __half hi = __float2half_rn(w);
    d[0] = hi;
    if (lo_off > 0) d[lo_off] = __float2half_rn(w - __half2float(hi));
  }
}

// HardUpsample = nearest x2 then conv3x3 (model_utils.py:161-165).  Output pixel
// (2y+py, 2x+px) only ever sees the 2x2 source neighbourhood {y+py-1, y+py} x {x+px-1, x+px},
// so the 3x3 kernel folds, per output parity, into a 2x2 kernel on the SOURCE resolution:
//   rows:  py=0: dy=-1 <- ky0,        dy=0 <- ky1+ky2;   py=1: dy=0 <- ky0+ky1, dy=+1 <- ky2
// (same for columns): 2.25x fewer MACs and no upsampled tensor.  Sums are taken in fp32.
// src fp32 [Cout][Cin][3][3] -> dst fp32 [4*Cout][Cin][2][2] (row = parity * Cout + o).
__global__ void fold_upconv_kernel(const float* __restrict__ src, float* __restrict__ dst, int cout,
                                   int cin) {
  const long long total = (long long)4 * cout * cin;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const int c = (int)(i % cin);
    const int o = (int)((i / cin) % cout);
    const int par = (int)(i / ((long long)cin * cout));
    const int py = par >> 1, px = par & 1;
    const float* w = src + ((long long)o * cin + c) * 9;
    float f[4] = {0.f, 0.f, 0.f, 0.f};
    for (int ky = 0; ky < 3; ++ky) {
      const int a = py == 0 ? (ky == 0 ? 0 : 1) : (ky == 2 ? 1 : 0);
      for (int kx = 0; kx < 3; ++kx) {
        const int b = px == 0 ? (kx == 0 ? 0 : 1) : (kx == 2 ? 1 : 0);
        f[a * 2 + b] += w[ky * 3 + kx];
      }
    }
    float* d = dst + i * 4;
    d[0] = f[0]; d[1] = f[1]; d[2] = f[2]; d[3] = f[3];
  }
}

// ----------------------------------------------------------------------------
// pose embedding: cs[h, :] = SiLU(W6 pose[h] + b)   (u_net.py:63-66 pose_mlp, then the
// SiLU that opens every ResnetBlock.mlp, model_utils.py:261-263)
// ----------------------------------------------------------------------------
__global__ void pose_embed_kernel(const float* __restrict__ poses, const float* __restrict__ w,
                                  const float* __restrict__ b, __half* __restrict__ cs, int n_hyp,
                                  int rot_dim, int cemb, bool bf = false) {
  pdl_sync();
  const int h = blockIdx.x;
  if (h >= n_hyp) return;
  __shared__ float sp[8];      // rot_dim <= 8 (6-D rotations); padded so vectorised reads stay inside
  if (threadIdx.x < 8) sp[threadIdx.x] = threadIdx.x < rot_dim ? poses[(long long)h * rot_dim + threadIdx.x] : 0.f;
  __syncthreads();
  for (int j = threadIdx.x; j < cemb; j += blockDim.x) {
    float a = b[j];
    for (int i = 0; i < rot_dim; ++i) a = fmaf(w[j * rot_dim + i], sp[i], a);
    st16(cs + (long long)h * cemb + j, silu_f(a), bf);
  }
}

// ----------------------------------------------------------------------------
// init_conv (u_net.py:77,161): fp32 NCHW latent [B,Cl,H,W] -> fp16 NHWC [B,H,W,Cout],
// direct 3x3, pad 1.  Runs once per reference image (pose independent).
// ----------------------------------------------------------------------------
__global__ void init_conv_kernel(const float* __restrict__ x, const float* __restrict__ w,
                                 const float* __restrict__ bias, __half* __restrict__ out, int B,
                                 int Cl, int H, int W, int Cout, __half* __restrict__ out_lo = nullptr,
                                 bool bf = false) {
  const long long total = (long long)B * H * W * Cout;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const int o = (int)(i % Cout);
    const int px = (int)((i / Cout) % W);
    const int py = (int)((i / ((long long)Cout * W)) % H);
    const int b = (int)(i / ((long long)Cout * W * H));
    float acc = bias[o];
    for (int c = 0; c < Cl; ++c)
      for (int ky = 0; ky < 3; ++ky) {
        const int yy = py + ky - 1;
        if (yy < 0 || yy >= H) continue;
        for (int kx = 0; kx < 3; ++kx) {
          const int xx = px + kx - 1;
          if (xx < 0 || xx >= W) continue;
          acc = fmaf(x[(((long long)b * Cl + c) * H + yy) * W + xx],
                     w[((o * Cl + c) * 3 + ky) * 3 + kx], acc);
        }
      }
    if (bf) { st16(out + i, acc, true); continue; }
    const __half hi = __float2half_rn(acc);
    out[i] = hi;
    if (out_lo) out_lo[i] = __float2half_rn(acc - __half2float(hi));
  }
}

// ----------------------------------------------------------------------------
// broadcast a per-reference tensor to every hypothesis of that reference, optionally
// adding the per-hypothesis pose projection (ResnetBlock.forward, model_utils.py:274-276,
// applied to the hoisted pose-independent block1 output).
// out[h, p, c] = src[ref_of[h], p, c] + pb[h, pb_off + c]
// ----------------------------------------------------------------------------
// With src_lo / out_lo (split precision) the sum src_hi + src_lo + pb is re-split into (hi, lo).
__global__ void bcast_add_kernel(const __half* __restrict__ src, const int* __restrict__ ref_of,
                                 const __half* __restrict__ pb, int pb_stride, int pb_off,
                                 __half* __restrict__ out, int n_hyp, int hw, int C,
                                 const __half* __restrict__ src_lo = nullptr,
                                 __half* __restrict__ out_lo = nullptr, bool bf = false) {
  pdl_sync();
  // grid (x: 16-byte pieces of one image, y: hypotheses): 32-bit index arithmetic only (the flat 64-bit index with
  // three divisions per 16 bytes held this pure copy at 2.6 TB/s)
  const int octs = C / 8;
  const int per_img = hw * octs;
  for (int h = blockIdx.y; h < n_hyp; h += gridDim.y) {
  const int r = ref_of[h];
  for (int j = blockIdx.x * blockDim.x + threadIdx.x; j < per_img; j += gridDim.x * blockDim.x) {
    const int p = j / octs;
    const int o = j - p * octs;
    uint4 v = *reinterpret_cast<const uint4*>(src + ((long long)r * hw + p) * C + o * 8);
    if (out_lo) {
      float f[8];
      const __half2* vv = reinterpret_cast<const __half2*>(&v);
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        const float2 x = __half22float2(vv[q]);
        f[2 * q] = x.x;
        f[2 * q + 1] = x.y;
      }
      if (src_lo) {
        const uint4 l = *reinterpret_cast<const uint4*>(src_lo + ((long long)r * hw + p) * C + o * 8);
        const __half2* ll = reinterpret_cast<const __half2*>(&l);
#pragma unroll
        for (int q = 0; q < 4; ++q) {
          const float2 x = __half22float2(ll[q]);
          f[2 * q] += x.x;
          f[2 * q + 1] += x.y;
        }
      }
      if (pb) {
        const uint4 a = *reinterpret_cast<const uint4*>(pb + (long long)h * pb_stride + pb_off + o * 8);
        const __half2* aa = reinterpret_cast<const __half2*>(&a);
#pragma unroll
        for (int q = 0; q < 4; ++q) {
          const float2 x = __half22float2(aa[q]);
          f[2 * q] += x.x;
          f[2 * q + 1] += x.y;
        }
      }
      uint4 wh, wl;
      uint32_t* ph = reinterpret_cast<uint32_t*>(&wh);
      uint32_t* pl = reinterpret_cast<uint32_t*>(&wl);
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        const __half2 hh2 = __floats2half2_rn(f[2 * q], f[2 * q + 1]);
        const float2 back = __half22float2(hh2);
        ph[q] = *reinterpret_cast<const uint32_t*>(&hh2);
        pl[q] = pack_half2(f[2 * q] - back.x, f[2 * q + 1] - back.y);
      }
      *reinterpret_cast<uint4*>(out + ((long long)h * hw + p) * C + o * 8) = wh;
      *reinterpret_cast<uint4*>(out_lo + ((long long)h * hw + p) * C + o * 8) = wl;
      continue;
    }
    if (pb) {
      const uint4 a = *reinterpret_cast<const uint4*>(pb + (long long)h * pb_stride + pb_off + o * 8);
      uint32_t* vv = reinterpret_cast<uint32_t*>(&v);
      const uint32_t* aa = reinterpret_cast<const uint32_t*>(&a);
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        const float2 x = unpack2(vv[q], bf), y = unpack2(aa[q], bf);
        vv[q] = pack2(x.x + y.x, x.y + y.y, bf);
      }
    }
    *reinterpret_cast<uint4*>(out + ((long long)h * hw + p) * C + o * 8) = v;
  }
  }
}

// ----------------------------------------------------------------------------
// GroupNorm (model_utils.py:241-252 Block.norm, :230 PreNorm, :401 to_out[1]), eps 1e-5,
// biased variance, fp32 statistics.  Two kernels: deterministic partial sums per
// (hypothesis, pixel slab, group), then a fused apply:
//   y = [SiLU](x * scale + shift) + pose_bias[h, c] + residual[res_of[h], p, c]
// Thread mapping: blockDim = octets * rows, thread -> (8-channel octet, pixel row);
// consecutive threads read consecutive 16-byte vectors of one pixel (coalesced).
// ----------------------------------------------------------------------------
__host__ __device__ inline int gn_rows(int C) {
  const int octs = C / 8;
  const int r = 384 / octs;
  return r < 1 ? 1 : r;
}

__global__ void gn_stats_kernel(const __half* __restrict__ x, float2* __restrict__ partial,
                                int hw, int C, int G, int nslab) {
  extern __shared__ float2 s_red[];
  const int octs = C / 8;
  const int rows = blockDim.x / octs;
  const int o = threadIdx.x % octs;
  const int r = threadIdx.x / octs;
  const int slab = blockIdx.x, h = blockIdx.y;
  const int pps = hw / nslab;
  const __half* base = x + ((long long)h * hw + (long long)slab * pps) * C + o * 8;
  float s = 0.f, ss = 0.f;
  for (int p = r; p < pps; p += rows) {
    const uint4 v = *reinterpret_cast<const uint4*>(base + (long long)p * C);
    const __half2* hv = reinterpret_cast<const __half2*>(&v);
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      const float2 f = __half22float2(hv[q]);
      s += f.x + f.y;
      ss = fmaf(f.x, f.x, ss);
      ss = fmaf(f.y, f.y, ss);
    }
  }
  s_red[threadIdx.x] = make_float2(s, ss);
  __syncthreads();
  if (threadIdx.x < G) {
    const int opg = octs / G;
    float a = 0.f, b = 0.f;
    for (int rr = 0; rr < rows; ++rr)
      for (int oo = 0; oo < opg; ++oo) {
        const float2 t = s_red[rr * octs + threadIdx.x * opg + oo];
        a += t.x;
        b += t.y;
      }
    partial[((long long)h * nslab + slab) * G + threadIdx.x] = make_float2(a, b);
  }
}

// Statistics of an NHWC fp16 tensor in the conv-epilogue format (parts of 32 pixels x
// 8-channel octets); used only behind the SIMT debug convolution.  grid (parts, img).
__global__ void stats_ref_kernel(const __half* __restrict__ x, float2* __restrict__ stats, int hw,
                                 int C) {
  const int part = blockIdx.x, img = blockIdx.y, parts = gridDim.x;
  const int noct = C / 8;
  const int npx = hw < 32 ? hw : 32;
  for (int o = threadIdx.x; o < noct; o += blockDim.x) {
    float s = 0.f, ss = 0.f;
    for (int p = 0; p < npx; ++p) {
      const __half* px = x + ((size_t)img * hw + part * 32 + p) * C + o * 8;
      for (int i = 0; i < 8; ++i) {
        const float f = __half2float(px[i]);
        s += f;
        ss = fmaf(f, f, ss);
      }
    }
    stats[((size_t)img * parts + part) * noct + o] = make_float2(s, ss);
  }
}

struct GnApplyArgs {
  const __half* x;
  __half* y;
  // Partial statistics [img][parts][noct] of (sum, sum of squares); the channels of group g
  // are covered by entries g*opg .. g*opg+opg-1 of each part (opg = noct / G).  Producers:
  // the conv epilogue (parts = max(1, hw/32), noct = C/8), gn_stats_kernel (parts = nslab,
  // noct = G) or a previous gn_apply with `emit` (parts = nslab, noct = 1, G = 1).
  // nullptr => no normalisation (y = x + ...).
  const float2* stats;
  int st_parts, st_noct;
  const float* gamma;
  const float* beta;
  const __half* pb;       // per-hypothesis channel bias (added after the activation) or nullptr
  const __half* res;      // residual or nullptr
  const int* res_of;      // hypothesis -> residual image index, nullptr => identity
  float2* emit;           // optional: per (img, fixed sub-slab) sum / sum of squares of y
  int emit_parts;         // fixed sub-slabs per image (independent of nslab)
  int pb_stride, pb_off;
  int hw, C, G, nslab;
  int silu;
  float eps;
  int bf16;               // 16-bit storage format of x / y / pb / res
};

__device__ __forceinline__ uint4 ld_stream16(const __half* p) {
  uint4 r;
  asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0, %1, %2, %3}, [%4];"
               : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w)
               : "l"(p));
  return r;
}

constexpr int kGnUnroll = 4;   // independent 16-byte loads in flight per thread

template <bool SILU, bool PB, bool RES>
__global__ void __launch_bounds__(384, 2) gn_apply_kernel(const GnApplyArgs a) {
  pdl_sync();
  __shared__ float2 s_red[256];
  __shared__ float2 s_grp[8];
  const int octs = a.C / 8;
  const int rows = blockDim.x / octs;
  const int o = threadIdx.x % octs;
  const int r = threadIdx.x / octs;
  const int slab = blockIdx.x, h = blockIdx.y;
  float scale[8], shift[8], pbv[8];
  const bool bf = a.bf16 != 0;
  if (a.stats) {
    // independent loads first (affine parameters), then the partial statistics
    float4 g0 = *reinterpret_cast<const float4*>(a.gamma + o * 8);
    float4 g1 = *reinterpret_cast<const float4*>(a.gamma + o * 8 + 4);
    float4 be0 = *reinterpret_cast<const float4*>(a.beta + o * 8);
    float4 be1 = *reinterpret_cast<const float4*>(a.beta + o * 8 + 4);
    // cooperative, fixed-order reduction of this image's partials: tpg threads per group
    const int opg = a.st_noct / a.G;
    const int E = a.st_parts * opg;
    int tpg = 256 / a.G;
    if (tpg > E) tpg = E;
    if ((int)threadIdx.x < a.G * tpg) {
      const int g = threadIdx.x / tpg, li = threadIdx.x - g * tpg;
      float s = 0.f, ss = 0.f;
      for (int e = li; e < E; e += tpg) {
        const int part = e / opg, oo = e - part * opg;
        const float2 t = a.stats[((size_t)h * a.st_parts + part) * a.st_noct + g * opg + oo];
        s += t.x;
        ss += t.y;
      }
      s_red[threadIdx.x] = make_float2(s, ss);
    }
    __syncthreads();
    if ((int)threadIdx.x < a.G) {
      float s = 0.f, ss = 0.f;
      for (int i = 0; i < tpg; ++i) {
        const float2 t = s_red[threadIdx.x * tpg + i];
        s += t.x;
        ss += t.y;
      }
      s_grp[threadIdx.x] = make_float2(s, ss);
    }
    __syncthreads();
    const float2 tot = s_grp[o / (octs / a.G)];
    const float cnt = (float)a.hw * (float)(a.C / a.G);
    const float mean = tot.x / cnt;
    const float var = fmaxf(tot.y / cnt - mean * mean, 0.f);
    const float rstd = rsqrtf(var + a.eps);
    const float gm[8] = {g0.x, g0.y, g0.z, g0.w, g1.x, g1.y, g1.z, g1.w};
    const float bt[8] = {be0.x, be0.y, be0.z, be0.w, be1.x, be1.y, be1.z, be1.w};
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      scale[i] = rstd * gm[i];
      shift[i] = bt[i] - mean * scale[i];
    }
  } else {
#pragma unroll
    for (int i = 0; i < 8; ++i) { scale[i] = 1.f; shift[i] = 0.f; }
  }
  if (PB) {
    const uint4 pv = *reinterpret_cast<const uint4*>(a.pb + (long long)h * a.pb_stride + a.pb_off + o * 8);
    const uint32_t* hp = reinterpret_cast<const uint32_t*>(&pv);
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      const float2 t = unpack2(hp[q], bf);
      pbv[2 * q] = t.x;
      pbv[2 * q + 1] = t.y;
    }
  }
  // The CTA covers pixel slab `slab` of nslab; statistics are emitted per FIXED sub-slab
  // (a.emit_parts per image, independent of nslab) and every sub-slab is reduced with the same
  // thread->pixel assignment and the same tree, so the emitted sums -- and everything
  // downstream -- do not depend on how many images share the launch.
  const int pps = a.hw / a.nslab;
  const int nsub = a.emit ? a.emit_parts / a.nslab : 1;   // fixed sub-slabs handled by this CTA
  const int spp = pps / nsub;                             // pixels per sub-slab
  const __half* xp = a.x + ((long long)h * a.hw + (long long)slab * pps) * a.C + o * 8;
  __half* yp = a.y + ((long long)h * a.hw + (long long)slab * pps) * a.C + o * 8;
  const __half* rp = nullptr;
  if (RES)
    rp = a.res + ((long long)(a.res_of ? a.res_of[h] : h) * a.hw + (long long)slab * pps) * a.C + o * 8;
  for (int sub = 0; sub < nsub; ++sub) {
    float es = 0.f, ess = 0.f;
    const int pbeg = sub * spp, pend = pbeg + spp;
    for (int p0 = pbeg + r; p0 < pend; p0 += rows * kGnUnroll) {
      uint4 xv[kGnUnroll], rv[kGnUnroll];
#pragma unroll
      for (int u = 0; u < kGnUnroll; ++u) {
        const int p = p0 + u * rows;
        if (p < pend) {
          xv[u] = ld_stream16(xp + (long long)p * a.C);
          if (RES) rv[u] = ld_stream16(rp + (long long)p * a.C);
        }
      }
#pragma unroll
      for (int u = 0; u < kGnUnroll; ++u) {
        const int p = p0 + u * rows;
        if (p >= pend) break;
        const uint32_t* hv = reinterpret_cast<const uint32_t*>(&xv[u]);
        float f[8];
#pragma unroll
        for (int q = 0; q < 4; ++q) {
          const float2 t = unpack2(hv[q], bf);
          f[2 * q] = t.x;
          f[2 * q + 1] = t.y;
        }
#pragma unroll
        for (int i = 0; i < 8; ++i) {
          float t = fmaf(f[i], scale[i], shift[i]);
          if (SILU) t = silu_f(t);
          if (PB) t += pbv[i];
          f[i] = t;
        }
        if (RES) {
          const uint32_t* hr = reinterpret_cast<const uint32_t*>(&rv[u]);
#pragma unroll
          for (int q = 0; q < 4; ++q) {
            const float2 t = unpack2(hr[q], bf);
            f[2 * q] += t.x;
            f[2 * q + 1] += t.y;
          }
        }
        uint4 w;
        w.x = pack2(f[0], f[1], bf);
        w.y = pack2(f[2], f[3], bf);
        w.z = pack2(f[4], f[5], bf);
        w.w = pack2(f[6], f[7], bf);
        *reinterpret_cast<uint4*>(yp + (long long)p * a.C) = w;
        if (a.emit) {
          // statistics of the values as stored (fp16-rounded), what the consumer will read
          const uint32_t* hw2 = reinterpret_cast<const uint32_t*>(&w);
#pragma unroll
          for (int q = 0; q < 4; ++q) {
            const float2 t = unpack2(hw2[q], bf);
            es += t.x + t.y;
            ess = fmaf(t.x, t.x, ess);
            ess = fmaf(t.y, t.y, ess);
          }
        }
      }
    }
    if (a.emit) {
      __syncthreads();   // s_red reuse
#pragma unroll
      for (int off2 = 16; off2 > 0; off2 >>= 1) {
        es += __shfl_xor_sync(0xffffffffu, es, off2);
        ess += __shfl_xor_sync(0xffffffffu, ess, off2);
      }
      if ((threadIdx.x & 31) == 0) s_red[threadIdx.x >> 5] = make_float2(es, ess);
      __syncthreads();
      if (threadIdx.x == 0) {
        float s = 0.f, ss = 0.f;
        for (int i = 0; i < (int)((blockDim.x + 31) >> 5); ++i) {
          s += s_red[i].x;
          ss += s_red[i].y;
        }
        a.emit[(size_t)h * a.emit_parts + slab * nsub + sub] = make_float2(s, ss);
      }
    }
  }
}

inline cudaError_t launch_gn_apply(const GnApplyArgs& a, dim3 grid, int threads, cudaStream_t st) {
  const int key = (a.silu ? 4 : 0) | (a.pb ? 2 : 0) | (a.res ? 1 : 0);
  switch (key) {
    case 0: return launch_pdl(gn_apply_kernel<false, false, false>, grid, dim3(threads), 0, st, a);
    case 1: return launch_pdl(gn_apply_kernel<false, false, true>, grid, dim3(threads), 0, st, a);
    case 2: return launch_pdl(gn_apply_kernel<false, true, false>, grid, dim3(threads), 0, st, a);
    case 3: return launch_pdl(gn_apply_kernel<false, true, true>, grid, dim3(threads), 0, st, a);
    case 4: return launch_pdl(gn_apply_kernel<true, false, false>, grid, dim3(threads), 0, st, a);
    case 5: return launch_pdl(gn_apply_kernel<true, false, true>, grid, dim3(threads), 0, st, a);
    case 6: return launch_pdl(gn_apply_kernel<true, true, false>, grid, dim3(threads), 0, st, a);
    default: return launch_pdl(gn_apply_kernel<true, true, true>, grid, dim3(threads), 0, st, a);
  }
}

// ----------------------------------------------------------------------------
// LinearAttention core (model_utils.py:403-417), heads = 4, dim_head = 32:
//   q = softmax_d(q) * scale ; k = softmax_n(k) ; ctx[d,e] = sum_n k[d,n] v[e,n]
//   out[e,n] = sum_d ctx[d,e] q[d,n]
// qkv: [n_hyp, n, 384] fp16 (q | k | v, each (head, 32)); out: [n_hyp, n, 128] fp16.
// One CTA per (head, hypothesis).
// ----------------------------------------------------------------------------
constexpr int kLinAttnThreads = 256;
constexpr int kLinAttnTile = 128;

__device__ __forceinline__ void load32h(const __half* p, float (&f)[32], bool bf = false) {
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    const uint4 v = *reinterpret_cast<const uint4*>(p + j * 8);
    const uint32_t* hv = reinterpret_cast<const uint32_t*>(&v);
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      const float2 t = unpack2(hv[q], bf);
      f[j * 8 + 2 * q] = t.x;
      f[j * 8 + 2 * q + 1] = t.y;
    }
  }
}

__global__ void __launch_bounds__(kLinAttnThreads)
linattn_kernel(const __half* __restrict__ qkv, __half* __restrict__ out, int n, bool bf = false) {
  pdl_sync();
  __shared__ float s_red[kLinAttnThreads / 32][32];
  __shared__ float s_kmax[32];
  __shared__ float s_ksum[32];
  __shared__ __align__(16) float s_ctx[32][32];
  __shared__ __align__(16) float s_ek[kLinAttnTile][32];
  __shared__ __align__(16) float s_v[kLinAttnTile][32];
  const int head = blockIdx.x, h = blockIdx.y;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const __half* base = qkv + (long long)h * n * 384;
  const __half* qb = base + head * 32;
  const __half* kb = base + 128 + head * 32;
  const __half* vb = base + 256 + head * 32;

  // ---- pass A: per-channel max of k over tokens
  float mx[32];
#pragma unroll
  for (int d = 0; d < 32; ++d) mx[d] = -INFINITY;
  for (int i = tid; i < n; i += kLinAttnThreads) {
    float f[32];
    load32h(kb + (long long)i * 384, f, bf);
#pragma unroll
    for (int d = 0; d < 32; ++d) mx[d] = fmaxf(mx[d], f[d]);
  }
#pragma unroll
  for (int d = 0; d < 32; ++d) {
    float m = mx[d];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
    if (lane == 0) s_red[warp][d] = m;
  }
  __syncthreads();
  if (tid < 32) {
    float m = s_red[0][tid];
    for (int w = 1; w < kLinAttnThreads / 32; ++w) m = fmaxf(m, s_red[w][tid]);
    s_kmax[tid] = m;
  }
  __syncthreads();

  // ---- pass B: ctx = exp(k - max)^T v, ksum.  Each thread owns a 4x4 block of ctx for one
  // quarter of the tokens (2 x LDS.128 per 16 FMA); the four token quarters are combined in a
  // fixed order afterwards.
  const int tq = tid & 63, tp = tid >> 6;
  const int cd = (tq >> 3) * 4;    // ctx rows d .. d+3
  const int ce = (tq & 7) * 4;     // ctx cols e .. e+3
  float c[4][4];
  float ks[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) c[i][j] = 0.f;
  for (int t0 = 0; t0 < n; t0 += kLinAttnTile) {
    const int tn = min(kLinAttnTile, n - t0);
    // stage: thread -> (token, 8-channel octet) for k and v
    for (int idx = tid; idx < tn * 4; idx += kLinAttnThreads) {
      const int t = idx >> 2, oc = (idx & 3) * 8;
      const uint4 kv = *reinterpret_cast<const uint4*>(kb + (long long)(t0 + t) * 384 + oc);
      const uint4 vv = *reinterpret_cast<const uint4*>(vb + (long long)(t0 + t) * 384 + oc);
      const uint32_t* hk = reinterpret_cast<const uint32_t*>(&kv);
      const uint32_t* hv = reinterpret_cast<const uint32_t*>(&vv);
      float ek[8], vf[8];
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        const float2 a = unpack2(hk[q], bf), b = unpack2(hv[q], bf);
        ek[2 * q] = __expf(a.x - s_kmax[oc + 2 * q]);
        ek[2 * q + 1] = __expf(a.y - s_kmax[oc + 2 * q + 1]);
        vf[2 * q] = b.x;
        vf[2 * q + 1] = b.y;
      }
      *reinterpret_cast<float4*>(&s_ek[t][oc]) = make_float4(ek[0], ek[1], ek[2], ek[3]);
      *reinterpret_cast<float4*>(&s_ek[t][oc + 4]) = make_float4(ek[4], ek[5], ek[6], ek[7]);
      *reinterpret_cast<float4*>(&s_v[t][oc]) = make_float4(vf[0], vf[1], vf[2], vf[3]);
      *reinterpret_cast<float4*>(&s_v[t][oc + 4]) = make_float4(vf[4], vf[5], vf[6], vf[7]);
    }
    __syncthreads();
    for (int t = tp; t < tn; t += 4) {
      const float4 e4 = *reinterpret_cast<const float4*>(&s_ek[t][cd]);
      const float4 v4 = *reinterpret_cast<const float4*>(&s_v[t][ce]);
      const float ee[4] = {e4.x, e4.y, e4.z, e4.w};
      const float vv4[4] = {v4.x, v4.y, v4.z, v4.w};
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        ks[i] += ee[i];
#pragma unroll
        for (int j = 0; j < 4; ++j) c[i][j] = fmaf(ee[i], vv4[j], c[i][j]);
      }
    }
    __syncthreads();
  }
  // combine the four token quarters (s_ek is free now: reuse it as [4][32][32] scratch)
  {
    float* part = &s_ek[0][0];
#pragma unroll
    for (int i = 0; i < 4; ++i)
      *reinterpret_cast<float4*>(part + (tp * 32 + cd + i) * 32 + ce) =
          make_float4(c[i][0], c[i][1], c[i][2], c[i][3]);
    float* pks = &s_v[0][0];                      // [4][32] partial column sums of exp(k)
    if ((tq & 7) == 0) {
#pragma unroll
      for (int i = 0; i < 4; ++i) pks[tp * 32 + cd + i] = ks[i];
    }
    __syncthreads();
    if (tid < 32) s_ksum[tid] = (pks[tid] + pks[32 + tid]) + (pks[64 + tid] + pks[96 + tid]);
    __syncthreads();
    for (int i = tid; i < 1024; i += kLinAttnThreads) {
      const int d = i >> 5;
      const float v = (part[i] + part[1024 + i]) + (part[2048 + i] + part[3072 + i]);
      s_ctx[d][i & 31] = v / s_ksum[d];
    }
  }
  __syncthreads();

  // ---- pass C: out[n, e] = sum_d softmax_d(q[n,:])[d] * scale * ctx[d][e]
  const float scale = 0.17677669529663687f;  // 32^-0.5
  for (int i = tid; i < n; i += kLinAttnThreads) {
    float q[32];
    load32h(qb + (long long)i * 384, q, bf);
    float m = q[0];
#pragma unroll
    for (int d = 1; d < 32; ++d) m = fmaxf(m, q[d]);
    float sum = 0.f;
#pragma unroll
    for (int d = 0; d < 32; ++d) { q[d] = __expf(q[d] - m); sum += q[d]; }
    const float qs = scale / sum;
    float o[32];
#pragma unroll
    for (int e = 0; e < 32; ++e) o[e] = 0.f;
#pragma unroll 4
    for (int d = 0; d < 32; ++d) {
      const float qd = q[d] * qs;
#pragma unroll
      for (int e4 = 0; e4 < 8; ++e4) {
        const float4 c = *reinterpret_cast<const float4*>(&s_ctx[d][e4 * 4]);
        o[e4 * 4 + 0] = fmaf(qd, c.x, o[e4 * 4 + 0]);
        o[e4 * 4 + 1] = fmaf(qd, c.y, o[e4 * 4 + 1]);
        o[e4 * 4 + 2] = fmaf(qd, c.z, o[e4 * 4 + 2]);
        o[e4 * 4 + 3] = fmaf(qd, c.w, o[e4 * 4 + 3]);
      }
    }
    __half* op = out + ((long long)h * n + i) * 128 + head * 32;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      uint4 w;
      w.x = pack2(o[j * 8 + 0], o[j * 8 + 1], bf);
      w.y = pack2(o[j * 8 + 2], o[j * 8 + 3], bf);
      w.z = pack2(o[j * 8 + 4], o[j * 8 + 5], bf);
      w.w = pack2(o[j * 8 + 6], o[j * 8 + 7], bf);
      *reinterpret_cast<uint4*>(op + j * 8) = w;
    }
  }
}

// ----------------------------------------------------------------------------
// Attention core at the bottleneck (model_utils.py:376-388), n <= 32 tokens:
//   sim = (q*scale)^T k ; softmax_j ; out[i,d] = sum_j attn[i,j] v[d,j]
// One CTA per hypothesis, one warp per head.
// ----------------------------------------------------------------------------
__global__ void __launch_bounds__(128)
midattn_kernel(const __half* __restrict__ qkv, __half* __restrict__ out, int n, bool bf = false) {
  pdl_sync();
  __shared__ float s_k[4][32][32];
  __shared__ float s_v[4][32][32];
  const int h = blockIdx.x, head = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const __half* base = qkv + (long long)h * n * 384;
  for (int t = lane; t < n; t += 32) {
    float f[32];
    load32h(base + (long long)t * 384 + 128 + head * 32, f, bf);
#pragma unroll
    for (int d = 0; d < 32; ++d) s_k[head][t][d] = f[d];
    load32h(base + (long long)t * 384 + 256 + head * 32, f, bf);
#pragma unroll
    for (int d = 0; d < 32; ++d) s_v[head][t][d] = f[d];
  }
  __syncwarp();
  const float scale = 0.17677669529663687f;
  for (int i = lane; i < n; i += 32) {
    float q[32];
    load32h(base + (long long)i * 384 + head * 32, q, bf);
#pragma unroll
    for (int d = 0; d < 32; ++d) q[d] *= scale;
    float sim[32];
    float m = -INFINITY;
    for (int j = 0; j < n; ++j) {
      float a = 0.f;
#pragma unroll
      for (int d = 0; d < 32; ++d) a = fmaf(q[d], s_k[head][j][d], a);
      sim[j] = a;
      m = fmaxf(m, a);
    }
    float sum = 0.f;
    for (int j = 0; j < n; ++j) { sim[j] = __expf(sim[j] - m); sum += sim[j]; }
    const float inv = 1.0f / sum;
    float o[32];
#pragma unroll
    for (int d = 0; d < 32; ++d) o[d] = 0.f;
    for (int j = 0; j < n; ++j) {
      const float p = sim[j] * inv;
#pragma unroll
      for (int d = 0; d < 32; ++d) o[d] = fmaf(p, s_v[head][j][d], o[d]);
    }
    __half* op = out + ((long long)h * n + i) * 128 + head * 32;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      uint4 w;
      w.x = pack2(o[j * 8 + 0], o[j * 8 + 1], bf);
      w.y = pack2(o[j * 8 + 2], o[j * 8 + 3], bf);
      w.z = pack2(o[j * 8 + 4], o[j * 8 + 5], bf);
      w.w = pack2(o[j * 8 + 6], o[j * 8 + 7], bf);
      *reinterpret_cast<uint4*>(op + j * 8) = w;
    }
  }
}

// ----------------------------------------------------------------------------
// nearest x2 upsample (HardUpsample[0], model_utils.py:161-163), NHWC fp16
// ----------------------------------------------------------------------------
__global__ void upsample2x_kernel(const __half* __restrict__ x, __half* __restrict__ y, int n_img,
                                  int H, int W, int C) {
  const int octs = C / 8;
  const int H2 = 2 * H, W2 = 2 * W;
  const long long total = (long long)n_img * H2 * W2 * octs;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const int o = (int)(i % octs);
    const int xx = (int)((i / octs) % W2);
    const int yy = (int)((i / ((long long)octs * W2)) % H2);
    const int b = (int)(i / ((long long)octs * W2 * H2));
    const uint4 v = *reinterpret_cast<const uint4*>(
        x + (((long long)b * H + (yy >> 1)) * W + (xx >> 1)) * C + o * 8);
    *reinterpret_cast<uint4*>(y + (((long long)b * H2 + yy) * W2 + xx) * C + o * 8) = v;
  }
}

// ----------------------------------------------------------------------------
// final_conv[1] (1x1, C -> Cl <= 8, u_net.py:156) fused with the reference's "l2" score
// (model.py:260-262):  score[h] = -sum_p sqrt( sum_c (q[c,p] - e[c,p])^4 ).
// x: [n_hyp, hw, C] fp16; w fp32 [Cl, C]; emb (optional) fp32 [n_hyp, Cl, hw] (NCHW);
// query (optional) fp32 [B, Cl, hw]; partial (optional) [n_hyp, nslab] positive sums.
// One thread per pixel, 128 pixels per CTA.
// ----------------------------------------------------------------------------
constexpr int kFinalThreads = 128;
constexpr int kFinalPPT = 4;                               // pixels per thread of final_conv_score_kernel
constexpr int kFinalPix = kFinalThreads * kFinalPPT;       // pixels per CTA (slab)
constexpr int kMaxLatent = 8;
constexpr int kScoreParts = 3;     // partial sums per (hypothesis, pixel slab): metric-dependent
// Similarity metrics (include/nope_b200.h): 0 the reference's "l2" (model.py:260-262); 1 cosine of the
// flattened C*H*W descriptors (extension, F.cosine_similarity semantics, eps 1e-8); 2 occlusion-aware
// cosine: the per-pixel cosine over channels (the encoder's `sim_distance = nn.CosineSimilarity(dim=1)`,
// template.py:45) with similarities <= threshold zeroed (`OcclusionAwareSimilarity`,
// base_template.py:67-75), averaged over the pixels.
__device__ __forceinline__ float finish_score(int metric, float a, float b, float c, int hw) {
  if (metric == 0) return -a;
  if (metric == 1) return a / (fmaxf(sqrtf(b), 1e-8f) * fmaxf(sqrtf(c), 1e-8f));
  return a / (float)hw;
}

__global__ void __launch_bounds__(kFinalThreads)
final_conv_score_kernel(const __half* __restrict__ x, const float* __restrict__ w,
                        const float* __restrict__ bias, float* __restrict__ emb,
                        const float* __restrict__ query, const int* __restrict__ ref_of,
                        float* __restrict__ partial, int hw, int C, int Cl,
                        const __half* __restrict__ x_lo = nullptr, int metric = 0, float occ_thr = 0.f,
                        bool bf = false) {
  pdl_sync();
  // weights transposed to [C][kMaxLatent] (zero beyond Cl): the 8 outputs of one input channel are two aligned 16-byte
  // broadcast loads, and every loaded weight serves the kFinalPPT pixels of the thread.  (With a [Cl][C] table and one
  // pixel per thread every FMA had its own 4-byte shared-memory load: 1.5 TB/s, bound by the load-store unit.)
  extern __shared__ __align__(16) float s_w[];
  __shared__ float s_part[kScoreParts][kFinalThreads / 32];
  const int slab = blockIdx.x, h = blockIdx.y, nslab = gridDim.x;
  for (int i = threadIdx.x; i < kMaxLatent * C; i += kFinalThreads) {
    const int k = i / kMaxLatent, c = i - k * kMaxLatent;
    s_w[i] = c < Cl ? w[c * C + k] : 0.f;
  }
  __syncthreads();
  static_assert(kMaxLatent == 8, "two float4 per input channel");
  float acc[kFinalPPT][kMaxLatent];
  int pix[kFinalPPT];
#pragma unroll
  for (int u = 0; u < kFinalPPT; ++u) {
    pix[u] = slab * kFinalPix + u * kFinalThreads + threadIdx.x;      // consecutive threads: consecutive pixels
#pragma unroll
    for (int c = 0; c < kMaxLatent; ++c) acc[u][c] = (c < Cl) ? bias[c] : 0.f;
  }
  for (int k0 = 0; k0 < C; k0 += 8) {
    float f[kFinalPPT][8];
#pragma unroll
    for (int u = 0; u < kFinalPPT; ++u) {
      uint4 v = make_uint4(0u, 0u, 0u, 0u);
      if (pix[u] < hw) v = *reinterpret_cast<const uint4*>(x + ((long long)h * hw + pix[u]) * C + k0);
      const uint32_t* hv = reinterpret_cast<const uint32_t*>(&v);
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        const float2 t = unpack2(hv[q], bf);
        f[u][2 * q] = t.x;
        f[u][2 * q + 1] = t.y;
      }
      if (x_lo && pix[u] < hw) {
        const uint4 l = *reinterpret_cast<const uint4*>(x_lo + ((long long)h * hw + pix[u]) * C + k0);
        const __half2* hl = reinterpret_cast<const __half2*>(&l);
#pragma unroll
        for (int q = 0; q < 4; ++q) {
          const float2 t = __half22float2(hl[q]);
          f[u][2 * q] += t.x;
          f[u][2 * q + 1] += t.y;
        }
      }
    }
#pragma unroll
    for (int i = 0; i < 8; ++i) {       // per output the channels are accumulated in ascending order
      const float4 w0 = *reinterpret_cast<const float4*>(s_w + (k0 + i) * kMaxLatent);
      const float4 w1 = *reinterpret_cast<const float4*>(s_w + (k0 + i) * kMaxLatent + 4);
#pragma unroll
      for (int u = 0; u < kFinalPPT; ++u) {
        acc[u][0] = fmaf(f[u][i], w0.x, acc[u][0]); acc[u][1] = fmaf(f[u][i], w0.y, acc[u][1]);
        acc[u][2] = fmaf(f[u][i], w0.z, acc[u][2]); acc[u][3] = fmaf(f[u][i], w0.w, acc[u][3]);
        acc[u][4] = fmaf(f[u][i], w1.x, acc[u][4]); acc[u][5] = fmaf(f[u][i], w1.y, acc[u][5]);
        acc[u][6] = fmaf(f[u][i], w1.z, acc[u][6]); acc[u][7] = fmaf(f[u][i], w1.w, acc[u][7]);
      }
    }
  }
  float dist = 0.f, d1 = 0.f, d2 = 0.f;      // metric-dependent partial sums over this thread's pixels
#pragma unroll
  for (int u = 0; u < kFinalPPT; ++u) {
    const int p = pix[u];
    if (p >= hw) continue;
    if (emb) {
#pragma unroll
      for (int c = 0; c < kMaxLatent; ++c)
        if (c < Cl) emb[((long long)h * Cl + c) * hw + p] = acc[u][c];
    }
    if (query) {
      const float* qp = query + (long long)ref_of[h] * Cl * hw + p;
      float s4 = 0.f, qe = 0.f, qq = 0.f, ee = 0.f;
#pragma unroll
      for (int c = 0; c < kMaxLatent; ++c)
        if (c < Cl) {
          const float qv = qp[(long long)c * hw];
          const float d = qv - acc[u][c];
          const float dd = d * d;
          s4 = fmaf(dd, dd, s4);
          qe = fmaf(qv, acc[u][c], qe);
          qq = fmaf(qv, qv, qq);
          ee = fmaf(acc[u][c], acc[u][c], ee);
        }
      if (metric == 0) {                 // reference "l2" (model.py:260-262)
        dist += sqrtf(s4);
      } else if (metric == 1) {          // cosine of the flattened descriptors: three global sums
        dist += qe; d1 += qq; d2 += ee;
      } else {                           // per-pixel cosine over channels, occlusion threshold
        const float sc = qe / (fmaxf(sqrtf(qq), 1e-8f) * fmaxf(sqrtf(ee), 1e-8f));
        dist += sc > occ_thr ? sc : 0.f;
      }
    }
  }
  if (partial) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      dist += __shfl_xor_sync(0xffffffffu, dist, o);
      d1 += __shfl_xor_sync(0xffffffffu, d1, o);
      d2 += __shfl_xor_sync(0xffffffffu, d2, o);
    }
    if ((threadIdx.x & 31) == 0) {
      s_part[0][threadIdx.x >> 5] = dist;
      s_part[1][threadIdx.x >> 5] = d1;
      s_part[2][threadIdx.x >> 5] = d2;
    }
    __syncthreads();
    if (threadIdx.x < kScoreParts) {
      float t = 0.f;
      for (int i = 0; i < kFinalThreads / 32; ++i) t += s_part[threadIdx.x][i];
      partial[((long long)h * nslab + slab) * kScoreParts + threadIdx.x] = t;
    }
  }
}

// Standalone score of materialised embeddings (PoseConditional.retrieval, model.py:254-266):
// emb fp32 [B, N, Cl, hw], query fp32 [B, Cl, hw].  metric 0: reference "l2";
// metric 1: cosine over the flattened descriptor (extension, eps 1e-8).
// One CTA per (b, n).
__global__ void __launch_bounds__(256)
score_kernel(const float* __restrict__ query, const float* __restrict__ emb,
             float* __restrict__ sim, int N, int Cl, int hw, int metric, float occ_thr) {
  __shared__ float s_a[8], s_b[8], s_c[8];
  const int n = blockIdx.x, b = blockIdx.y;
  const float* e = emb + ((long long)b * N + n) * Cl * hw;
  const float* q = query + (long long)b * Cl * hw;
  float a0 = 0.f, a1 = 0.f, a2 = 0.f;
  for (int p = threadIdx.x; p < hw; p += blockDim.x) {
    if (metric == 0) {
      float s4 = 0.f;
      for (int c = 0; c < Cl; ++c) {
        const float d = q[c * hw + p] - e[c * hw + p];
        const float d2 = d * d;
        s4 = fmaf(d2, d2, s4);
      }
      a0 += sqrtf(s4);
    } else if (metric == 1) {
      for (int c = 0; c < Cl; ++c) {
        const float x = q[c * hw + p], y = e[c * hw + p];
        a0 = fmaf(x, y, a0);
        a1 = fmaf(x, x, a1);
        a2 = fmaf(y, y, a2);
      }
    } else {
      float qe = 0.f, qq = 0.f, ee = 0.f;
      for (int c = 0; c < Cl; ++c) {
        const float x = q[c * hw + p], y = e[c * hw + p];
        qe = fmaf(x, y, qe);
        qq = fmaf(x, x, qq);
        ee = fmaf(y, y, ee);
      }
      const float sc = qe / (fmaxf(sqrtf(qq), 1e-8f) * fmaxf(sqrtf(ee), 1e-8f));
      a0 += sc > occ_thr ? sc : 0.f;
    }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    a0 += __shfl_xor_sync(0xffffffffu, a0, o);
    a1 += __shfl_xor_sync(0xffffffffu, a1, o);
    a2 += __shfl_xor_sync(0xffffffffu, a2, o);
  }
  if ((threadIdx.x & 31) == 0) {
    s_a[threadIdx.x >> 5] = a0;
    s_b[threadIdx.x >> 5] = a1;
    s_c[threadIdx.x >> 5] = a2;
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    float t0 = 0.f, t1 = 0.f, t2 = 0.f;
    for (int i = 0; i < (int)(blockDim.x >> 5); ++i) { t0 += s_a[i]; t1 += s_b[i]; t2 += s_c[i]; }
    sim[(long long)b * N + n] = finish_score(metric, t0, t1, t2, hw);
  }
}

// ----------------------------------------------------------------------------
// sim = -(sum of slab partials) and top-k (model.py:265 topk(k=5)); descending score,
// ties -> lowest index.  One CTA per batch row.  idx_base is added to the indices so a
// shard reports global pose indices.
// ----------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
sim_topk_kernel(const float* __restrict__ partial, int nslab, float* __restrict__ sim, int N,
                int k, float* __restrict__ top_val, long long* __restrict__ top_idx,
                long long idx_base, int nparts = 1, int metric = 0, int hw = 1) {
  pdl_sync();
  __shared__ float s_v[8];
  __shared__ int s_i[8];
  __shared__ int s_chosen[64];
  const int b = blockIdx.x;
  float* srow = sim + (long long)b * N;
  if (partial) {
    for (int n = threadIdx.x; n < N; n += blockDim.x) {
      float t[3] = {0.f, 0.f, 0.f};
      for (int s = 0; s < nslab; ++s)
        for (int q = 0; q < nparts; ++q) t[q] += partial[(((long long)b * N + n) * nslab + s) * nparts + q];
      srow[n] = finish_score(metric, t[0], t[1], t[2], hw);
    }
    __syncthreads();
  }
  if (k <= 0) return;
  for (int r = 0; r < k; ++r) {
    float bv = -INFINITY;
    int bi = 0x7fffffff;
    for (int n = threadIdx.x; n < N; n += blockDim.x) {
      bool used = false;
      for (int c = 0; c < r; ++c) used |= (s_chosen[c] == n);
      if (used) continue;
      const float v = srow[n];
      if (v > bv || (v == bv && n < bi) || bi == 0x7fffffff) { bv = v; bi = n; }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      const float ov = __shfl_xor_sync(0xffffffffu, bv, o);
      const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
      if (oi != 0x7fffffff && (bi == 0x7fffffff || ov > bv || (ov == bv && oi < bi))) {
        bv = ov;
        bi = oi;
      }
    }
    if ((threadIdx.x & 31) == 0) { s_v[threadIdx.x >> 5] = bv; s_i[threadIdx.x >> 5] = bi; }
    __syncthreads();
    if (threadIdx.x == 0) {
      for (int w = 1; w < (int)(blockDim.x >> 5); ++w) {
        const float ov = s_v[w];
        const int oi = s_i[w];
        if (oi != 0x7fffffff && (bi == 0x7fffffff || ov > bv || (ov == bv && oi < bi))) {
          bv = ov;
          bi = oi;
        }
      }
      s_chosen[r] = bi;
      top_val[(long long)b * k + r] = bv;
      top_idx[(long long)b * k + r] = (bi == 0x7fffffff) ? -1 : (long long)bi + idx_base;
    }
    __syncthreads();
  }
}

// ----------------------------------------------------------------------------
// Multi-GPU merge (SURVEY.md 8e): every rank contributes ONE packed record to a single all-gather,
//   [ topv: B*k f32 | pad to even | topi: B*k i64 | sim slice: B*n_local f32 (optional) ]      (`pack` floats)
// with GLOBAL pose indices (idx -1 = padding).  This kernel turns the W gathered records into the
// global top-k per batch row (descending score, ties -> lowest index: deterministic, identical on
// every rank) and the full similarity rows.  One CTA per batch row; candidates W*k <= 1024.
// rank r owns poses [r*per, min(N, (r+1)*per)).
// ----------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
topk_merge_kernel(const float* __restrict__ gathered, int world, long long pack, int B, int k, int N, int per,
                  int has_sim, float* __restrict__ out_sim, float* __restrict__ top_val,
                  long long* __restrict__ top_idx) {
  __shared__ float s_v[1024];
  __shared__ long long s_i[1024];
  const int b = blockIdx.x;
  const int kk = (B * k + 1) & ~1;                    // floats before the index block (8-byte aligned)
  const int ncand = world * k;
  for (int c = threadIdx.x; c < ncand; c += blockDim.x) {
    const int r = c / k, j = c - r * k;
    const float* rec = gathered + (long long)r * pack;
    const long long idx = reinterpret_cast<const long long*>(rec + kk)[b * k + j];
    s_i[c] = idx;
    s_v[c] = idx < 0 ? -INFINITY : rec[b * k + j];
  }
  __syncthreads();
  for (int c = threadIdx.x; c < ncand; c += blockDim.x) {
    const float v = s_v[c];
    const long long i = s_i[c];
    if (i < 0) continue;
    int rank = 0;                                     // candidates that beat this one
    for (int o = 0; o < ncand; ++o) {
      const long long io = s_i[o];
      if (io < 0 || o == c) continue;
      const float vo = s_v[o];
      rank += (vo > v || (vo == v && io < i)) ? 1 : 0;
    }
    if (rank < k) {
      top_val[(long long)b * k + rank] = v;
      top_idx[(long long)b * k + rank] = i;
    }
  }
  // fewer than k valid candidates (N < k cannot happen: the callers clamp k): nothing to pad
  if (has_sim && out_sim) {
    for (int n = threadIdx.x; n < N; n += blockDim.x) {
      const int r = n / per, j = n - r * per;
      const int lo = r * per, hi = min(N, lo + per);
      const float* rec = gathered + (long long)r * pack + kk + 2 * B * k;
      out_sim[(long long)b * N + n] = rec[(long long)b * (hi - lo) + j];
    }
  }
}

// ----------------------------------------------------------------------------
// SIMT implicit-GEMM convolution: a slow, obviously-correct CUDA-core twin of the
// wgmma kernel (same packed weights, same segment semantics).  Debug / bring-up
// only (NOPE_CONV_IMPL=simt); never the default path.
// mode 0: 3x3 pad 1; mode 1: 1x1; mode 2: pixel-unshuffle(2) + 1x1 (input is 2H x 2W);
// mode 3: parity-folded nearest-x2 upsample + 3x3 (input is H/2 x W/2, weights [4*Cout][4*Cin]).
// ----------------------------------------------------------------------------
struct SimtConvArgs {
  const __half* src0;
  const __half* src1;
  int C0, C1;
  const __half* w;   // [Cout][K]
  const float* bias;
  __half* out;
  int n_img, H, W, Cout, K, mode;
};

__global__ void conv_simt_kernel(const SimtConvArgs a) {
  const long long total = (long long)a.n_img * a.H * a.W * a.Cout;
  const int Ccat = a.C0 + a.C1;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const int o = (int)(i % a.Cout);
    const int px = (int)((i / a.Cout) % a.W);
    const int py = (int)((i / ((long long)a.Cout * a.W)) % a.H);
    const int b = (int)(i / ((long long)a.Cout * a.W * a.H));
    const int par = a.mode == 3 ? ((py & 1) * 2 + (px & 1)) : 0;
    const __half* wr = a.w + ((long long)par * a.Cout + o) * a.K;
    float acc = a.bias ? a.bias[o] : 0.f;
    const int taps = a.mode == 0 ? 9 : (a.mode == 1 ? 1 : 4);
    for (int t = 0; t < taps; ++t) {
      int yy, xx, Hs = a.H, Ws = a.W;
      if (a.mode == 0) { yy = py + t / 3 - 1; xx = px + t % 3 - 1; }
      else if (a.mode == 1) { yy = py; xx = px; }
      else if (a.mode == 2) { Hs = 2 * a.H; Ws = 2 * a.W; yy = 2 * py + t / 2; xx = 2 * px + t % 2; }
      else { Hs = a.H / 2; Ws = a.W / 2; yy = (py >> 1) + t / 2 - 1 + (py & 1); xx = (px >> 1) + t % 2 - 1 + (px & 1); }
      if (yy < 0 || yy >= Hs || xx < 0 || xx >= Ws) continue;
      const long long pix = ((long long)b * Hs + yy) * Ws + xx;
      const __half* s0 = a.src0 + pix * a.C0;
      const __half* wk = wr + t * Ccat;
      for (int c = 0; c < a.C0; c += 2) {
        const float2 x = __half22float2(*reinterpret_cast<const __half2*>(s0 + c));
        const float2 y = __half22float2(*reinterpret_cast<const __half2*>(wk + c));
        acc = fmaf(x.x, y.x, acc);
        acc = fmaf(x.y, y.y, acc);
      }
      if (a.src1) {
        const __half* s1 = a.src1 + pix * a.C1;
        for (int c = 0; c < a.C1; c += 2) {
          const float2 x = __half22float2(*reinterpret_cast<const __half2*>(s1 + c));
          const float2 y = __half22float2(*reinterpret_cast<const __half2*>(wk + a.C0 + c));
          acc = fmaf(x.x, y.x, acc);
          acc = fmaf(x.y, y.y, acc);
        }
      }
    }
    a.out[i] = __float2half_rn(acc);
  }
}

// fp32 NCHW <-> fp16 NHWC helpers for the per-op test entry points
__global__ void nchw_f32_to_nhwc_f16_kernel(const float* __restrict__ x, __half* __restrict__ y,
                                            int n_img, int C, int hw, __half* __restrict__ y_lo = nullptr,
                                            bool bf = false) {
  const long long total = (long long)n_img * C * hw;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const int c = (int)(i % C);
    const int p = (int)((i / C) % hw);
    const int b = (int)(i / ((long long)C * hw));
    const float v = x[((long long)b * C + c) * hw + p];
    if (bf) { st16(y + i, v, true); continue; }
    const __half hi = __float2half_rn(v);
    y[i] = hi;
    if (y_lo) y_lo[i] = __float2half_rn(v - __half2float(hi));
  }
}
__global__ void nhwc_f16_to_nchw_f32_kernel(const __half* __restrict__ x, float* __restrict__ y,
                                            int n_img, int C, int hw,
                                            const __half* __restrict__ x_lo = nullptr, bool bf = false) {
  const long long total = (long long)n_img * C * hw;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const int p = (int)(i % hw);
    const int c = (int)((i / hw) % C);
    const int b = (int)(i / ((long long)C * hw));
    const long long j = ((long long)b * hw + p) * C + c;
    y[i] = ld16(x + j, bf) + (x_lo ? __half2float(x_lo[j]) : 0.f);
  }
}

inline int ew_grid(long long total, int threads = 256, int cap = 132 * 16) {
  long long g = (total + threads - 1) / threads;
  if (g < 1) g = 1;
  if (g > cap) g = cap;
  return (int)g;
}

}  // namespace nope
