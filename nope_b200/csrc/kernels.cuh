// nope_b200 -- the HBM-bound kernels around the tensor-core convolutions:
// weight packing, pose embedding, linear attention, bottleneck attention, nearest
// upsample, the fused final 1x1 conv + score partials (scoring of materialised templates and every ranking kernel
// are in rank.cuh).  All activations are NHWC fp16; statistics, softmax and scores are fp32.  Each kernel cites the
// reference code it reproduces (paths relative to the reference root).
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

// hypotheses [h0, h0 + n) of the flattened (reference, pose) list -> their reference image: r[i] = (h0 + i) / N
__global__ void ref_of_kernel(int* r, int h0, int N, int n) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) r[i] = (h0 + i) / N;
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

// 16-byte load that does not allocate in L1: for tensors each thread reads exactly once
__device__ __forceinline__ uint4 ld_stream16(const __half* p) {
  uint4 r;
  asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0, %1, %2, %3}, [%4];"
               : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w)
               : "l"(p));
  return r;
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
// query fp32 [B, Q, Cl, hw] (Q queries per reference; needed when partial is set);
// partial (optional) [n_hyp, Q, nslab, kScoreParts] sums.  With kVis the sums skip the pixels that the visible map
// vis [B, Q, hw] of the (reference, query) row marks 0 (DESIGN.md section 27).
// kFinalPPT pixels per thread, kFinalPix pixels per CTA.
// ----------------------------------------------------------------------------
constexpr int kFinalThreads = 128;
constexpr int kFinalPPT = 4;                               // pixels per thread of final_conv_score_kernel
constexpr int kFinalPix = kFinalThreads * kFinalPPT;       // pixels per CTA (slab)
constexpr int kMaxLatent = 8;
constexpr int kScoreParts = 3;     // partial sums per (hypothesis, pixel slab): metric-dependent

template <bool kVis>
__global__ void __launch_bounds__(kFinalThreads)
final_conv_score_kernel(const __half* __restrict__ x, const float* __restrict__ w,
                        const float* __restrict__ bias, float* __restrict__ emb,
                        const float* __restrict__ query, const int* __restrict__ ref_of,
                        float* __restrict__ partial, int hw, int C, int Cl,
                        const __half* __restrict__ x_lo, int metric, float occ_thr,
                        bool bf, int Q, const uint8_t* __restrict__ vis) {
  pdl_sync();
  // weights transposed to [C][kMaxLatent] (zero beyond Cl): the 8 outputs of one input channel are two aligned 16-byte
  // broadcast loads, and every loaded weight serves the kFinalPPT pixels of the thread.  (With a [Cl][C] table and one
  // pixel per thread every FMA had its own 4-byte shared-memory load: 1.5 TB/s, bound by the load-store unit.)
  extern __shared__ __align__(16) float s_w[];
  __shared__ float s_part[2][kScoreParts][kFinalThreads / 32];
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
  if (emb) {                                 // the template is stored once, whatever the number of queries
#pragma unroll
    for (int u = 0; u < kFinalPPT; ++u) {
      if (pix[u] >= hw) continue;
#pragma unroll
      for (int c = 0; c < kMaxLatent; ++c)
        if (c < Cl) emb[((long long)h * Cl + c) * hw + pix[u]] = acc[u][c];
    }
  }
  if (!partial) return;
  // Every query of this hypothesis's reference is scored against the accumulators in registers.  The sums of
  // one (hypothesis, query) pair run in the same order for any Q, so a Q-query sweep reproduces Q one-query
  // sweeps bit for bit.  s_part is double-buffered: the writes of query q + 2 follow the barrier of q + 1,
  // which the readers of query q have passed.
  const long long qrow0 = (long long)ref_of[h] * Q;
#pragma unroll 1
  for (int qi = 0; qi < Q; ++qi) {
    float dist = 0.f, d1 = 0.f, d2 = 0.f;      // metric-dependent partial sums over this thread's pixels
#pragma unroll
    for (int u = 0; u < kFinalPPT; ++u) {
      const int p = pix[u];
      if (p >= hw) continue;
      if (kVis && !vis[(qrow0 + qi) * hw + p]) continue;
      const float* qp = query + (qrow0 + qi) * Cl * hw + p;     // coalesced: consecutive threads, consecutive pixels
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
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      dist += __shfl_xor_sync(0xffffffffu, dist, o);
      d1 += __shfl_xor_sync(0xffffffffu, d1, o);
      d2 += __shfl_xor_sync(0xffffffffu, d2, o);
    }
    float (*sp)[kFinalThreads / 32] = s_part[qi & 1];
    if ((threadIdx.x & 31) == 0) {
      sp[0][threadIdx.x >> 5] = dist;
      sp[1][threadIdx.x >> 5] = d1;
      sp[2][threadIdx.x >> 5] = d2;
    }
    __syncthreads();
    if (threadIdx.x < kScoreParts) {
      float t = 0.f;
      for (int i = 0; i < kFinalThreads / 32; ++i) t += sp[threadIdx.x][i];
      partial[(((long long)h * Q + qi) * nslab + slab) * kScoreParts + threadIdx.x] = t;
    }
  }
}

// fp32 NCHW <-> fp16 NHWC helpers for the per-op test entry points.  NHWC element (b, p, c) of image b's pixel p:
// plain [n_img, hw, C], or, with plane_cap > 0, the parity-planar layout of a 256 x 256 level (vae.cuh): plane
// (py, px) of a [4][plane_cap][128][128][C] tensor holds the pixels (2 Y + py, 2 X + px).
__device__ __forceinline__ long long nhwc_index(int b, int p, int c, int C, int hw, int plane_cap) {
  if (!plane_cap) return ((long long)b * hw + p) * C + c;
  const int y = p >> 8, x = p & 255, q = (y & 1) * 2 + (x & 1);
  return ((((long long)q * plane_cap + b) * 128 + (y >> 1)) * 128 + (x >> 1)) * C + c;
}
// y32 (optional) receives the fp32 values in the same NHWC layout
__global__ void nchw_f32_to_nhwc_f16_kernel(const float* __restrict__ x, __half* __restrict__ y,
                                            int n_img, int C, int hw, __half* __restrict__ y_lo = nullptr,
                                            bool bf = false, float* __restrict__ y32 = nullptr, int plane_cap = 0) {
  const long long total = (long long)n_img * C * hw;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const int c = (int)(i % C);
    const int p = (int)((i / C) % hw);
    const int b = (int)(i / ((long long)C * hw));
    const float v = x[((long long)b * C + c) * hw + p];
    const long long j = plane_cap ? nhwc_index(b, p, c, C, hw, plane_cap) : i;
    if (bf) { st16(y + j, v, true); continue; }
    const __half hi = __float2half_rn(v);
    y[j] = hi;
    if (y_lo) y_lo[j] = __float2half_rn(v - __half2float(hi));
    if (y32) y32[j] = v;
  }
}
// x32 (optional) is read instead of the fp16 pair
__global__ void nhwc_f16_to_nchw_f32_kernel(const __half* __restrict__ x, float* __restrict__ y,
                                            int n_img, int C, int hw,
                                            const __half* __restrict__ x_lo = nullptr, bool bf = false,
                                            const float* __restrict__ x32 = nullptr, int plane_cap = 0) {
  const long long total = (long long)n_img * C * hw;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const int p = (int)(i % hw);
    const int c = (int)((i / hw) % C);
    const int b = (int)(i / ((long long)C * hw));
    const long long j = nhwc_index(b, p, c, C, hw, plane_cap);
    y[i] = x32 ? x32[j] : ld16(x + j, bf) + (x_lo ? __half2float(x_lo[j]) : 0.f);
  }
}

inline int ew_grid(long long total, int threads = 256, int cap = 132 * 16) {
  long long g = (total + threads - 1) / threads;
  if (g < 1) g = 1;
  if (g > cap) g = cap;
  return (int)g;
}

// Packs one convolution weight with pack_weight_kernel (row_stride, col_off, lo_off and bf16 as there).  src is fp32
// [cout][cin][taps] in host or device memory; with fold_up it is a [cout][cin][3][3] kernel that fold_upconv_kernel
// first folds into 4 cout rows of four taps.  src is staged in temporary device memory, freed once `st` has run the
// packing.
inline int pack_conv_weight(const float* src, __half* dst, int cout, int cin, int taps, bool fold_up, int row_stride,
                            int col_off, int lo_off, int bf16, cudaStream_t st) {
  const size_t n = (size_t)cout * cin * (fold_up ? 9 : taps);
  const int rows = fold_up ? 4 * cout : cout;
  float *tmp = nullptr, *folded = nullptr;
  NOPE_CUDA(cudaMalloc(reinterpret_cast<void**>(&tmp), n * sizeof(float)));
  NOPE_CUDA(cudaMemcpyAsync(tmp, src, n * sizeof(float), cudaMemcpyDefault, st));
  const float* w = tmp;
  if (fold_up) {
    NOPE_CUDA(cudaMalloc(reinterpret_cast<void**>(&folded), (size_t)rows * cin * taps * sizeof(float)));
    fold_upconv_kernel<<<ew_grid((long long)4 * cout * cin), 256, 0, st>>>(tmp, folded, cout, cin);
    NOPE_CUDA(cudaGetLastError());
    w = folded;
  }
  pack_weight_kernel<<<ew_grid((long long)rows * cin * taps), 256, 0, st>>>(w, dst, rows, cin, taps, row_stride,
                                                                            col_off, lo_off, bf16);
  NOPE_CUDA(cudaGetLastError());
  NOPE_CUDA(cudaStreamSynchronize(st));
  NOPE_CUDA(cudaFree(tmp));
  if (folded) NOPE_CUDA(cudaFree(folded));
  return 0;
}

}  // namespace nope
