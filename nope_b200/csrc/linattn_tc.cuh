// nope_b200 -- LinearAttention core on wgmma tensor cores (model_utils.py:403-417), heads = 4, dim_head = 32:
//   q = softmax_d(q) * scale ; k = softmax_n(k) ; ctx[d,e] = sum_n k[d,n] v[e,n] ; out[e,n] = sum_d ctx[d,e] q[d,n]
// qkv: [n_img, n_tok, 384] fp16 (q | k | v, each (head, 32)); out: [n_img, n_tok, 128] fp16; n_tok % 128 == 0.
//
// The SIMT kernel (kernels.cuh) runs both contractions on CUDA cores: 16.8 MFLOP per image is ~0.2 ms of
// fp32 FMA per 642-image launch before any memory time.  Here they are two tensor-core GEMMs per image with
// all four heads stacked (the off-diagonal head blocks are wasted work, 4x of a negligible amount):
//   ctx [128 d x 128 e] += ek^T [128 d x 128 tok] * v [128 tok x 128 e]          per 128-token tile
//   out [128 tok x 128 e] = qs [128 tok x 128 d] * ctxm [128 d x 128 e]          ctxm = block-diagonal ctx / ksum
// ek = exp(k - max_n k) and qs = softmax_d(q) * scale are written back IN PLACE over the TMA-loaded tiles
// (fp16), so the token-major tiles serve directly as operands: token-major [tok][channel] is the canonical
// MN-major SWIZZLE_128B layout for ek^T / v (M resp. N = channel is contiguous, K = token runs over rows) and
// the canonical K-major layout for qs (K = channel).
//
// One persistent CTA per SM; per image: pass 1 streams k (column max), pass 2 streams (k, v) (second read of
// k comes from L2), pass 3 builds ctxm, pass 4 streams q and stores out.  Warp roles: 0 TMA producer,
// 4..11 (two warpgroups) SIMT transforms, wgmma and epilogues.  Warpgroup w owns rows [64 w, 64 w + 64) of
// each GEMM: ctx stays in its registers across pass 2, the out tile is written from registers to staging.
#pragma once
#include "conv_tc.cuh"

namespace nope {

constexpr int kLaSlots = 4;                       // ring of 32 KB slots: one [128 tok][128 ch] fp16 tile each
constexpr int kLaSlotBytes = 2 * kBM * 128;       // two 64-channel boxes
constexpr int kLaThreads = 384;
constexpr int kLaSimt = 256;

struct LinAttnParams {
  CUtensorMap qkv;        // [n_img][n_tok][384], box {64, 128, 1}
  CUtensorMap out;        // [n_img][n_tok][128], box {64, 128, 1}
  int n_img, n_tok;
  int bf16;               // qkv / out (and the ek / qs / ctxm operands written here) are bf16
};

struct LinAttnSmem {
  static constexpr int kRing = kLaSlots * kLaSlotBytes;          // 128 KB
  static constexpr int kCtxOff = kRing;                          // ctxm operand [128 e][128 d] fp16, 2 boxes
  static constexpr int kOutOff = kCtxOff + kLaSlotBytes;         // output staging, 2 boxes
  static constexpr int kBarOff = kOutOff + kLaSlotBytes;
  static constexpr int kVecOff = kBarOff + 256;                  // kmax[128], ksum[128] fp32, scratch [8][128]
  static constexpr int kTotal = kVecOff + (2 * 128 + 8 * 128) * 4 + 1024;
};

// MN-major SWIZZLE_128B wgmma descriptor: 64 MN-elements (128 B) contiguous, 8 K-rows per 1024-byte atom
// (SBO), the next 64 MN-elements 16 KB further (LBO = the second 64-channel box).
constexpr uint64_t kWgDescMN = (static_cast<uint64_t>(16384 >> 4) << 16) | (static_cast<uint64_t>(1024 >> 4) << 32) |
                               (static_cast<uint64_t>(1) << 62);

template <bool BF>
__device__ __forceinline__ void linattn_ctx_mma(float (&c)[64], uint32_t a_lo, uint32_t b_lo, int t) {
#pragma unroll
  for (int k = 0; k < kBM / 16; ++k)        // 16 tokens = two 8-row atoms = 2048 B
    Wgmma<128, BF, 1>::mma(c, kWgDescMN | (a_lo + k * 128), kWgDescMN | (b_lo + k * 128), (t | k) != 0 ? 1u : 0u);
}
template <bool BF>
__device__ __forceinline__ void linattn_out_mma(float (&o)[64], uint32_t a_lo, uint32_t b_lo) {
#pragma unroll
  for (int k = 0; k < 8; ++k) {             // K = 128 channels d: 4 steps of 16 per 64-channel box
    const uint32_t off = (k >> 2) * ((kBM * 128) >> 4) + (k & 3) * 2;
    Wgmma<128, BF>::mma(o, kWgDescK | (a_lo + off), kWgDescK | (b_lo + off), k != 0 ? 1u : 0u);
  }
}

__global__ void __launch_bounds__(kLaThreads, 1) linattn_tc_kernel(const __grid_constant__ LinAttnParams p) {
  using S = LinAttnSmem;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~static_cast<uintptr_t>(1023));
  uint8_t* s_ctx = smem + S::kCtxOff;
  uint8_t* s_out = smem + S::kOutOff;
  uint64_t* full = reinterpret_cast<uint64_t*>(smem + S::kBarOff);   // [slots] TMA landed
  uint64_t* empty = full + kLaSlots;                                 // [slots] slot may be refilled
  float* s_kmax = reinterpret_cast<float*>(smem + S::kVecOff);
  float* s_ksum = s_kmax + 128;
  float* s_scr = s_ksum + 128;                                       // [8 warps][128]

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int T = p.n_tok / kBM;                                       // 128-token tiles per image

  if (warp == 0 && lane == 0) {
    prefetch_tmap(&p.qkv);
    prefetch_tmap(&p.out);
  }
  if (warp == 1 && lane == 0) {
    for (int s = 0; s < kLaSlots; ++s) {
      mbar_init(&full[s], 1);
      mbar_init(&empty[s], 1);
    }
    fence_mbar_init();
  }
  __syncthreads();
  pdl_sync();       // the prologue above overlapped the previous kernel's tail; its output is read from here on

  // Ring protocol: items are consumed in production order; item i lives in slot i % kLaSlots and completes
  // exactly one phase of full[s] (TMA) and of empty[s] (the compute warps, once done with the tile), so both
  // flip with parity (i / kLaSlots) & 1.  Per image the item sequence is
  //   T x k (pass 1) | T x (k, v) (pass 2) | T x q (pass 4)
  if (warp == 0) {
    // ===================== TMA producer =====================
    uint32_t item = 0;
    auto load = [&](int ch0, int tok0, int img) {
      const int s = item % kLaSlots;
      mbar_wait(&empty[s], ((item / kLaSlots) & 1) ^ 1);
      if (elect_one()) {
        uint8_t* dst = smem + s * kLaSlotBytes;
        mbar_expect_tx(&full[s], kLaSlotBytes);
        tma_load_3d(dst, &p.qkv, &full[s], ch0, tok0, img);
        tma_load_3d(dst + kBM * 128, &p.qkv, &full[s], ch0 + 64, tok0, img);
      }
      __syncwarp();
      ++item;
    };
    for (int img = blockIdx.x; img < p.n_img; img += gridDim.x) {
      for (int t = 0; t < T; ++t) load(128, t * kBM, img);                 // k
      for (int t = 0; t < T; ++t) {
        load(128, t * kBM, img);                                           // k again (L2)
        load(256, t * kBM, img);                                           // v
      }
      for (int t = 0; t < T; ++t) load(0, t * kBM, img);                   // q
    }
  } else if (warp >= 4) {
    // ===================== SIMT transforms, wgmma, epilogues (8 warps) =====================
    const int tid = threadIdx.x - 128, w8 = warp - 4;
    const int cx = tid & 15;                       // 16-byte chunk column: channels [8 cx, 8 cx + 8)
    const int r0 = tid >> 4;                       // token rows r0 + 16 i
    const int box = cx >> 3, cin = cx & 7;
    const int wg = tid >> 7;                       // warpgroup: rows [64 wg, 64 wg + 64) of both GEMMs
    const int fr = 64 * wg + 16 * (w8 & 3) + (lane >> 2);    // accumulator fragment rows fr, fr + 8
    const int fc = 2 * (lane & 3);                           // fragment columns 8 i + fc, + 1
    const float scale = 0.17677669529663687f;      // 32^-0.5
    const bool bf = p.bf16 != 0;
    const uint32_t smem_base = smem_u32(smem);
    uint32_t item = 0;
    for (int img = blockIdx.x; img < p.n_img; img += gridDim.x) {
      // ---- pass 1: per-channel max of k over the image's tokens
      float mx[8];
#pragma unroll
      for (int i = 0; i < 8; ++i) mx[i] = -INFINITY;
      for (int t = 0; t < T; ++t, ++item) {
        const int s = item % kLaSlots;
        mbar_wait(&full[s], (item / kLaSlots) & 1);
        const uint8_t* tile = smem + s * kLaSlotBytes + box * (kBM * 128);
#pragma unroll
        for (int i = 0; i < 8; ++i) {
          const int r = r0 + 16 * i;
          const uint4 v = *reinterpret_cast<const uint4*>(tile + r * 128 + ((cin ^ (r & 7)) << 4));
          const uint32_t* h2 = reinterpret_cast<const uint32_t*>(&v);
#pragma unroll
          for (int k2 = 0; k2 < 4; ++k2) {
            const float2 f = unpack2(h2[k2], bf);
            mx[2 * k2] = fmaxf(mx[2 * k2], f.x);
            mx[2 * k2 + 1] = fmaxf(mx[2 * k2 + 1], f.y);
          }
        }
        asm volatile("bar.sync 1, 256;" ::: "memory");
        if (tid == 0) mbar_arrive(&empty[s]);
      }
#pragma unroll
      for (int i = 0; i < 8; ++i) mx[i] = fmaxf(mx[i], __shfl_xor_sync(0xffffffffu, mx[i], 16));
      if (lane < 16) {
#pragma unroll
        for (int i = 0; i < 8; ++i) s_scr[w8 * 128 + cx * 8 + i] = mx[i];
      }
      asm volatile("bar.sync 1, 256;" ::: "memory");
      if (tid < 128) {
        float m = s_scr[tid];
        for (int w = 1; w < 8; ++w) m = fmaxf(m, s_scr[w * 128 + tid]);
        s_kmax[tid] = m;
      }
      asm volatile("bar.sync 1, 256;" ::: "memory");
      float km[8], ks[8];
#pragma unroll
      for (int i = 0; i < 8; ++i) { km[i] = s_kmax[cx * 8 + i]; ks[i] = 0.f; }
      // ---- pass 2: ek = exp(k - max) in place; column sums of the stored values; ctx += ek^T v
      float c[64];
#pragma unroll
      for (int i = 0; i < 64; ++i) c[i] = 0.f;
      for (int t = 0; t < T; ++t, item += 2) {
        const int s = item % kLaSlots, sv = (item + 1) % kLaSlots;
        mbar_wait(&full[s], (item / kLaSlots) & 1);
        uint8_t* tile = smem + s * kLaSlotBytes + box * (kBM * 128);
#pragma unroll
        for (int i = 0; i < 8; ++i) {
          const int r = r0 + 16 * i;
          uint4* pv = reinterpret_cast<uint4*>(tile + r * 128 + ((cin ^ (r & 7)) << 4));
          uint4 v = *pv;
          uint32_t* h2 = reinterpret_cast<uint32_t*>(&v);
#pragma unroll
          for (int k2 = 0; k2 < 4; ++k2) {
            const float2 f = unpack2(h2[k2], bf);
            const uint32_t e2 = pack2(__expf(f.x - km[2 * k2]), __expf(f.y - km[2 * k2 + 1]), bf);
            const float2 b = unpack2(e2, bf);
            ks[2 * k2] += b.x;
            ks[2 * k2 + 1] += b.y;
            h2[k2] = e2;
          }
          *pv = v;
        }
        fence_proxy_async_smem();
        asm volatile("bar.sync 1, 256;" ::: "memory");
        mbar_wait(&full[sv], ((item + 1) / kLaSlots) & 1);              // v landed
        const uint32_t a_lo = (smem_base + s * kLaSlotBytes + wg * (kBM * 128)) >> 4;
        const uint32_t b_lo = (smem_base + sv * kLaSlotBytes) >> 4;
        wgmma_fence();
        if (bf) linattn_ctx_mma<true>(c, a_lo, b_lo, t);
        else linattn_ctx_mma<false>(c, a_lo, b_lo, t);
        wgmma_commit();
        wgmma_wait<0>();
        asm volatile("bar.sync 1, 256;" ::: "memory");
        if (tid == 0) {
          mbar_arrive(&empty[s]);
          mbar_arrive(&empty[sv]);
        }
      }
#pragma unroll
      for (int i = 0; i < 8; ++i) ks[i] += __shfl_xor_sync(0xffffffffu, ks[i], 16);
      if (lane < 16) {
#pragma unroll
        for (int i = 0; i < 8; ++i) s_scr[w8 * 128 + cx * 8 + i] = ks[i];
      }
      asm volatile("bar.sync 1, 256;" ::: "memory");
      if (tid < 128) {
        float a = 0.f;
        for (int w = 0; w < 8; ++w) a += s_scr[w * 128 + tid];
        s_ksum[tid] = a;
      }
      asm volatile("bar.sync 1, 256;" ::: "memory");
      // ---- pass 3: ctxm[e][d] = ctx[d][e] / ksum[d] inside a head, 0 across heads; fp16, K-major (K = d).
      // The previous image's out-tile MMAs have all retired, so the ctxm operand buffer is free to overwrite.
#pragma unroll
      for (int h8 = 0; h8 < 2; ++h8) {
        const int d = fr + 8 * h8;
        const float inv = 1.0f / s_ksum[d];
        uint8_t* cbox = s_ctx + (d >> 6) * (kBM * 128);
#pragma unroll
        for (int i = 0; i < 16; ++i) {
#pragma unroll
          for (int j = 0; j < 2; ++j) {
            const int e = 8 * i + fc + j;                       // row of the operand
            const float val = (e >> 5) == (d >> 5) ? c[4 * i + 2 * h8 + j] * inv : 0.f;
            st16(reinterpret_cast<__half*>(cbox + e * 128 + ((((d & 63) >> 3) ^ (e & 7)) << 4) + (d & 7) * 2), val, bf);
          }
        }
      }
      fence_proxy_async_smem();
      asm volatile("bar.sync 1, 256;" ::: "memory");
      // ---- pass 4: qs = softmax_d(q) * scale in place; out tile = qs ctxm -> staging -> TMA store
      for (int t = 0; t < T; ++t, ++item) {
        const int s = item % kLaSlots;
        mbar_wait(&full[s], (item / kLaSlots) & 1);
        {
          // thread -> (token row, 64-channel box = head pair): two softmaxes over 32 channels each
          const int r = tid & 127, bx = tid >> 7;
          uint8_t* rowp = smem + s * kLaSlotBytes + bx * (kBM * 128) + r * 128;
#pragma unroll
          for (int hd = 0; hd < 2; ++hd) {
            uint4 v[4];
            float f[32];
#pragma unroll
            for (int c4 = 0; c4 < 4; ++c4) {
              v[c4] = *reinterpret_cast<const uint4*>(rowp + (((hd * 4 + c4) ^ (r & 7)) << 4));
              const uint32_t* h2 = reinterpret_cast<const uint32_t*>(&v[c4]);
#pragma unroll
              for (int k2 = 0; k2 < 4; ++k2) {
                const float2 t2 = unpack2(h2[k2], bf);
                f[c4 * 8 + 2 * k2] = t2.x;
                f[c4 * 8 + 2 * k2 + 1] = t2.y;
              }
            }
            float m = f[0];
#pragma unroll
            for (int i = 1; i < 32; ++i) m = fmaxf(m, f[i]);
            float sum = 0.f;
#pragma unroll
            for (int i = 0; i < 32; ++i) { f[i] = __expf(f[i] - m); sum += f[i]; }
            const float qs = scale / sum;
#pragma unroll
            for (int c4 = 0; c4 < 4; ++c4) {
              uint4 w;
              w.x = pack2(f[c4 * 8 + 0] * qs, f[c4 * 8 + 1] * qs, bf);
              w.y = pack2(f[c4 * 8 + 2] * qs, f[c4 * 8 + 3] * qs, bf);
              w.z = pack2(f[c4 * 8 + 4] * qs, f[c4 * 8 + 5] * qs, bf);
              w.w = pack2(f[c4 * 8 + 6] * qs, f[c4 * 8 + 7] * qs, bf);
              *reinterpret_cast<uint4*>(rowp + (((hd * 4 + c4) ^ (r & 7)) << 4)) = w;
            }
          }
        }
        fence_proxy_async_smem();
        if (tid == 0) tma_store_wait_read0();      // the previous tile's store has read the staging buffer
        asm volatile("bar.sync 1, 256;" ::: "memory");
        float o[64];
        const uint32_t a_lo = (smem_base + s * kLaSlotBytes + wg * 64 * 128) >> 4;
        const uint32_t b_lo = (smem_base + S::kCtxOff) >> 4;
        wgmma_fence();
        if (bf) linattn_out_mma<true>(o, a_lo, b_lo);
        else linattn_out_mma<false>(o, a_lo, b_lo);
        wgmma_commit();
        wgmma_wait<0>();
#pragma unroll
        for (int h8 = 0; h8 < 2; ++h8) {
          const int row = fr + 8 * h8;
#pragma unroll
          for (int i = 0; i < 16; ++i) {
            const int e = 8 * i + fc;
            *reinterpret_cast<uint32_t*>(s_out + (e >> 6) * (kBM * 128) + row * 128 +
                                         ((((e & 63) >> 3) ^ (row & 7)) << 4) + (e & 7) * 2) =
                pack2(o[4 * i + 2 * h8], o[4 * i + 2 * h8 + 1], bf);
          }
        }
        fence_proxy_async_smem();
        asm volatile("bar.sync 1, 256;" ::: "memory");
        if (tid == 0) {
          mbar_arrive(&empty[s]);
          tma_store_3d(&p.out, s_out, 0, t * kBM, img);
          tma_store_3d(&p.out, s_out + kBM * 128, 64, t * kBM, img);
          tma_store_commit();
        }
      }
    }
    if (tid == 0) tma_store_wait_all();
  }
}

// fp16 3-D tensor map [n_img][n_tok][C], box {64, 128, 1}, 128-byte swizzle
inline int make_token_map(CUtensorMap* out, const void* base, int n_img, int n_tok, int C) {
  uint64_t dims[3] = {(uint64_t)C, (uint64_t)n_tok, (uint64_t)n_img};
  uint64_t str[2] = {(uint64_t)C * 2, (uint64_t)n_tok * C * 2};
  uint32_t box[3] = {64, (uint32_t)kBM, 1};
  return make_tmap_f16(out, base, 3, dims, str, box);
}

inline int launch_linattn_tc(const __half* qkv, __half* out, int n_img, int n_tok, int num_sms, cudaStream_t st,
                             bool bf16 = false) {
  if (n_tok % kBM != 0) return fail("linattn_tc: n_tok must be a multiple of 128");
  static bool attr_set[kMaxDevices];
  int dev = 0;
  NOPE_CUDA(cudaGetDevice(&dev));
  NOPE_CHECK(dev >= 0 && dev < kMaxDevices, "device index out of range");
  if (!attr_set[dev]) {
    NOPE_CUDA(cudaFuncSetAttribute(linattn_tc_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, LinAttnSmem::kTotal));
    attr_set[dev] = true;
  }
  LinAttnParams p;
  if (make_token_map(&p.qkv, qkv, n_img, n_tok, 384) || make_token_map(&p.out, out, n_img, n_tok, 128)) return -1;
  p.n_img = n_img;
  p.n_tok = n_tok;
  p.bf16 = bf16 ? 1 : 0;
  const int grid = n_img < num_sms ? n_img : num_sms;
  NOPE_CUDA(launch_pdl(linattn_tc_kernel, dim3(grid), dim3(kLaThreads), LinAttnSmem::kTotal, st, p));
  return 0;
}

}  // namespace nope
