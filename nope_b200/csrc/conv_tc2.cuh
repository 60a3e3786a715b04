// nope_b200 -- the implicit-GEMM convolution kernel, with the fused epilogues.
//
// Math, parameters, mainloop and plain epilogue come from conv_tc.cuh; CTAs are launched in
// thread-block clusters of 2 that walk the tile list in PAIRS of 128-pixel M-tiles (tile
// (m_pair, n_tile) -> M-tiles 2 m_pair and 2 m_pair + 1, one per CTA), so the two CTAs of a pair
// read the same weight tile at the same time and the second read is served by L2.  Each CTA
// TMA-loads its own 128 pixel rows of A and the whole BN-row weight tile, and its epilogue
// warpgroups run the wgmma mainloop (conv_mma_tile): warpgroups 0 and 1 accumulate 64 rows x all
// BN columns each in registers (a single warpgroup takes both row halves; a third one only joins the
// epilogue), the fp32 tile then passes through shared memory to the epilogue.  setmaxnreg moves
// registers from the control warpgroup (warps 0-3) to the math warpgroups (conv2_math_regs).
//
// Tile widths: 192 (the default UNet: every width is a multiple of 192), 256 (the LDM variant:
// multiples of 256), 128 / 64 (template encoder, GEGLU).  Tiles of <= 128 columns double-buffer
// the output staging.  EPI selects the epilogue at compile time: 0 plain (+ GroupNorm partial
// sums), 1 extras (ReLU, residual add, (hi, lo) split, fp32 store: template encoder, LDM out conv),
// 2 GEGLU (conv_tc.cuh), 4 GroupNorm fused (GnFuse, conv_tc.cuh) with the CTA split into math /
// statistics / store roles (conv_gn_* below): the default UNet's Block / ResnetBlock / to_qkv /
// to_out epilogues -- the normalised, activated tensor is the only thing that reaches HBM.
//
// Protocol (per CTA):
//   full[s]   count 1: the producer's arrive.expect_tx; the stage's TMA loads complete_tx on it
//   empty[s]  one arrive per mainloop warp (conv_mma_warps) once its wgmma reads of the stage retired
//   tempty    one arrive per epilogue warp once the accumulator tile has been read out of the ring;
//             the producer waits for it before it loads the next tile
#pragma once
#include "conv_tc.cuh"

namespace nope {

__device__ __forceinline__ uint32_t cluster_ctarank() {
  uint32_t r;
  asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r));
  return r;
}
__device__ __forceinline__ uint32_t cluster_id_x() {
  uint32_t r;
  asm volatile("mov.u32 %0, %%clusterid.x;" : "=r"(r));
  return r;
}
__device__ __forceinline__ uint32_t num_clusters_x() {
  uint32_t r;
  asm volatile("mov.u32 %0, %%nclusterid.x;" : "=r"(r));
  return r;
}
__device__ __forceinline__ void cluster_sync_all() {
  asm volatile("barrier.cluster.arrive.release.aligned;" ::: "memory");
  asm volatile("barrier.cluster.wait.acquire.aligned;" ::: "memory");
}
// shared-memory map of the EPI == 4 epilogue (conv_gn_* below), relative to Conv2Smem::kGnOffset
template <int BN>
struct GnSmem {
  static constexpr int kOct = BN / 8;
  static constexpr int kPart = 0;                          // fp32 [8 row segments][kOct][2]
  static constexpr int kMr = kPart + 8 * kOct * 8;         // float2 [2][64]: (mean, rstd) per (image, group) / image
  static constexpr int kTab = kMr + 2 * 64 * 8;            // fp32 [2][scale | shift][BN]
  static constexpr int kOg = kTab + 2 * 2 * BN * 4;        // int [kOct]: octet -> group of the tile
  static constexpr int kEm = kOg + kOct * 4;               // float2 [2 staging buffers][BN / 64][8]: emit partials per 16-row segment
  static constexpr int kX = kEm + 2 * 32 * 8;                  // fp32 [256]: gathered cross-CTA partials
  static constexpr int kBytes = kX + 256 * 4;
};

template <int BN, int STAGES, int EPI = 0>
struct Conv2Smem {
  static constexpr int kABytes = kBM * kBK * 2;
  static constexpr int kBBytes = BN * kBK * 2;
  static constexpr int kStageBytes = kABytes + kBBytes;
  static constexpr int kOutBytes = (BN / 64) * kBM * 128;
  // narrow tiles double-buffer the output staging: the TMA store of tile i drains while the
  // epilogue of tile i+1 fills the other buffer (the short-K 1x1 layers are epilogue bound).  At BN = 192 the
  // second buffer would cost a ring stage, and the fourth stage is worth more: with one wgmma group in flight
  // the mainloop holds two stages, so three stages leave the producer one stage of lead (fused GroupNorm at
  // BN = 192 on an H100 at 700 W: 3 stages + 2 buffers 45.0 ms per 642-pose step, 4 stages + 1 buffer 41.0-41.4,
  // every layer class faster, the short-K to_qkv / to_out launches included; DESIGN.md section 6)
  static constexpr int kOutBufs = BN <= 128 ? 2 : 1;
  static constexpr int kBarOffset = STAGES * kStageBytes + kOutBufs * kOutBytes;
  static constexpr int kBiasOffset = kBarOffset + 256;
  static constexpr int kGnOffset = kBiasOffset + BN * 4;
  static constexpr int kGnBytes = EPI == 4 ? GnSmem<BN>::kBytes : 0;
  static constexpr int kTotal = kGnOffset + kGnBytes + 1024;
  static_assert(STAGES * kStageBytes >= kBM * (BN + 4) * 4, "the fp32 accumulator tile must fit in the operand ring");
  static_assert(kTotal <= 227 * 1024, "shared memory per block");
};

// 8-byte {value, tag} words of the cross-CTA partial-sum exchange: single-copy atomic, L2-coherent
__device__ __forceinline__ uint2 ld_volatile_u2(const uint2* p) {
  uint2 r;
  asm volatile("ld.volatile.global.v2.u32 {%0, %1}, [%2];" : "=r"(r.x), "=r"(r.y) : "l"(p) : "memory");
  return r;
}
__device__ __forceinline__ void st_volatile_u2(uint2* p, uint2 v) {
  asm volatile("st.volatile.global.v2.u32 [%0], {%1, %2};" ::"l"(p), "r"(v.x), "r"(v.y) : "memory");
}

// ---------------------------------------------------------------------------------------------
// EPI == 4: the GroupNorm-fused epilogue (GnFuse, conv_tc.cuh), with the CTA split into roles.  Warps 2 and 3 take
// the bookkeeping -- the statistics exchange, the table build and the drain of the TMA store -- and talk to the math
// warps through mbarriers only, so none of it sits on the critical path of the warps that do the arithmetic:
//
//   warps 4..   math: wgmma mainloop, accumulator -> registers (+bias), release the ring, per-octet partial sums -> s_part,
//               arrive part_bar | wait stats_bar[b], res_bar | normalise / SiLU / pose bias / residual in place
//               in the staging tile | arrive out_bar, tabfree_bar[b].   No block-wide barrier anywhere.
//   warp 3      statistics: wait part_bar | per-(image, group) sums, publish {value, epoch} words, poll the peer
//               tiles, fixed-order totals | per-channel scale / shift table (or (mean, rstd) pairs) into buffer
//               b = tile parity | arrive stats_bar[b].  The pre-norm fold's per-image scalars are independent of
//               the accumulator, so for those launches this warp runs a tile ahead of the math warps.
//   warp 2      store: wait out_bar | GroupNorm(1) sums of the stored tile (emit) | TMA store | once the store has
//               read the staging buffer: TMA load of the NEXT tile's residual into it (or a plain arrive), res_bar.
//
// Per-channel parameters (bias, gamma, beta, pose-bias rows) are read through the read-only L1 path rather than
// staged in shared memory per tile, so no barrier has to publish them.
// ---------------------------------------------------------------------------------------------
// read-only shared-memory tables of pass 2: plain (non-volatile, no memory clobber) asm loads, so the
// compiler may hoist them above the in-place stores to the staging tile (same shared array: it must
// otherwise assume they alias and serialises every 8-channel octet).  `tok` is produced by a volatile asm
// after the mbarrier waits that publish the tables, which keeps the loads below those waits.
__device__ __forceinline__ float4 lds_f4(uint32_t addr) {
  float4 r;
  asm("ld.shared.v4.f32 {%0, %1, %2, %3}, [%4];" : "=f"(r.x), "=f"(r.y), "=f"(r.z), "=f"(r.w) : "r"(addr));
  return r;
}
__device__ __forceinline__ uint4 lds_u4(uint32_t addr) {
  uint4 r;
  asm("ld.shared.v4.u32 {%0, %1, %2, %3}, [%4];" : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w) : "r"(addr));
  return r;
}
__device__ __forceinline__ float2 lds_f2(uint32_t addr) {
  float2 r;
  asm("ld.shared.v2.f32 {%0, %1}, [%2];" : "=f"(r.x), "=f"(r.y) : "r"(addr));
  return r;
}
__device__ __forceinline__ uint32_t order_token(uint32_t v) {
  uint32_t r;
  asm volatile("mov.u32 %0, %1;" : "=r"(r) : "r"(v) : "memory");
  return r;
}

// x * sigmoid(x) on two MUFU ops and three FMA-pipe ops (flush-to-zero variants: the IEEE-denormal
// handling of __expf / __fdividef costs four more instructions per element in this issue-bound pass)
__device__ __forceinline__ float silu_ftz(float x) {
  float e, r;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(e) : "f"(x * -1.4426950408889634f));
  asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(1.0f + e));
  return x * r;
}

__host__ __device__ constexpr int gn_epi_warps(int BN) { return 4 * (BN / 64); }           // one (lane quarter, 64-column sub-tile) each
__host__ __device__ constexpr int gn_threads(int BN) { return 128 + 32 * gn_epi_warps(BN); }

struct GnBars {
  uint64_t* full;       // [STAGES] operand stage landed (producer -> math warps)
  uint64_t* empty;      // [STAGES] operand stage consumed (math warps -> producer)
  uint64_t* tempty;     // accumulator tile read out of the ring (math warps -> producer)
  uint64_t* res[2];     // per staging buffer: residual landed / buffer free (store warp -> math warps)
  uint64_t* part;       // s_part written (math warps -> statistics warp)
  uint64_t* stats;      // [2] tables of tile parity b ready (statistics warp -> math warps)
  uint64_t* tabfree;    // [2] last read of table buffer b done (math warps -> statistics warp)
  uint64_t* out;        // [staging buffers] staging tile written (math warps -> store warp)
};

// Pass 2 of the EPI == 4 epilogue for the hot epilogue shapes, one 8-channel octet at a time with every
// launch-uniform choice a template parameter: normalise, SiLU, pose bias / residual, pack and store of an octet form
// one straight-line block, so the MUFU chains of one octet overlap the FMA / shared-memory work of its neighbours
// (the phase-per-step form below runs all 128 MUFU operations of a thread back to back with the FMA pipe idle).
//   NORM 1: y = x * sc[c] + sh[c] (tables: one image per tile, or the folded pre-norm)
//        2: y = (x - mean) * rstd * gamma[c] + beta[c] ((mean, rstd) per (image, group): several images per tile)
//        3: folded pre-norm with several images per tile: y = x * rstd - rstd * mean * w1[c] + wb[c]
// Shared-memory operands are read with non-volatile asm loads whose address derives from the order token taken after
// the barrier waits: the compiler may hoist them above the in-place stores (other octets, other addresses).
template <int NORM, bool SILU, bool PB, bool RES, bool EMIT>
__device__ __forceinline__ void gn_pass2_octets(float* f, uint32_t a_sc, uint32_t a_sh, uint32_t a_mr, const int* og,
                                                int it_gpt, const float4* gm4, const float4* bt4, const uint4* pb4,
                                                bool img_ok, uint8_t* srow, uint32_t a_srow, int row, bool bf,
                                                float& e1, float& e2) {
  float2 mr3 = make_float2(0.f, 0.f);
  if (NORM == 3) mr3 = lds_f2(a_mr);
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    float* ff = f + j * 8;
    const int sw = (j ^ (row & 7)) << 4;
    uint4 rv = make_uint4(0u, 0u, 0u, 0u), pv = make_uint4(0u, 0u, 0u, 0u);
    if (RES) rv = lds_u4(a_srow + sw);
    if (PB && img_ok) pv = __ldg(pb4 + j);
    if (NORM == 1) {
      const float4 s0 = lds_f4(a_sc + j * 32), s1 = lds_f4(a_sc + j * 32 + 16);
      const float4 h0 = lds_f4(a_sh + j * 32), h1 = lds_f4(a_sh + j * 32 + 16);
      ff[0] = fmaf(ff[0], s0.x, h0.x); ff[1] = fmaf(ff[1], s0.y, h0.y);
      ff[2] = fmaf(ff[2], s0.z, h0.z); ff[3] = fmaf(ff[3], s0.w, h0.w);
      ff[4] = fmaf(ff[4], s1.x, h1.x); ff[5] = fmaf(ff[5], s1.y, h1.y);
      ff[6] = fmaf(ff[6], s1.z, h1.z); ff[7] = fmaf(ff[7], s1.w, h1.w);
    } else if (NORM == 2) {
      const float2 mr = lds_f2(a_mr + (it_gpt + og[j]) * 8);
      const float4 g0 = __ldg(gm4 + 2 * j), g1 = __ldg(gm4 + 2 * j + 1);
      const float4 t0 = __ldg(bt4 + 2 * j), t1 = __ldg(bt4 + 2 * j + 1);
      ff[0] = fmaf(ff[0] - mr.x, mr.y * g0.x, t0.x); ff[1] = fmaf(ff[1] - mr.x, mr.y * g0.y, t0.y);
      ff[2] = fmaf(ff[2] - mr.x, mr.y * g0.z, t0.z); ff[3] = fmaf(ff[3] - mr.x, mr.y * g0.w, t0.w);
      ff[4] = fmaf(ff[4] - mr.x, mr.y * g1.x, t1.x); ff[5] = fmaf(ff[5] - mr.x, mr.y * g1.y, t1.y);
      ff[6] = fmaf(ff[6] - mr.x, mr.y * g1.z, t1.z); ff[7] = fmaf(ff[7] - mr.x, mr.y * g1.w, t1.w);
    } else if (NORM == 3) {
      const float nm = -mr3.x * mr3.y;
      const float4 g0 = __ldg(gm4 + 2 * j), g1 = __ldg(gm4 + 2 * j + 1);
      const float4 t0 = __ldg(bt4 + 2 * j), t1 = __ldg(bt4 + 2 * j + 1);
      ff[0] = fmaf(ff[0], mr3.y, fmaf(nm, g0.x, t0.x)); ff[1] = fmaf(ff[1], mr3.y, fmaf(nm, g0.y, t0.y));
      ff[2] = fmaf(ff[2], mr3.y, fmaf(nm, g0.z, t0.z)); ff[3] = fmaf(ff[3], mr3.y, fmaf(nm, g0.w, t0.w));
      ff[4] = fmaf(ff[4], mr3.y, fmaf(nm, g1.x, t1.x)); ff[5] = fmaf(ff[5], mr3.y, fmaf(nm, g1.y, t1.y));
      ff[6] = fmaf(ff[6], mr3.y, fmaf(nm, g1.z, t1.z)); ff[7] = fmaf(ff[7], mr3.y, fmaf(nm, g1.w, t1.w));
    }
    if (SILU) {
#pragma unroll
      for (int i = 0; i < 8; ++i) ff[i] = silu_ftz(ff[i]);
    }
    if (PB) {
      const uint32_t* hp = reinterpret_cast<const uint32_t*>(&pv);
#pragma unroll
      for (int k2 = 0; k2 < 4; ++k2) {
        const float2 t = unpack2(hp[k2], bf);
        ff[2 * k2] += t.x;
        ff[2 * k2 + 1] += t.y;
      }
    }
    if (RES) {
      const uint32_t* hr = reinterpret_cast<const uint32_t*>(&rv);
#pragma unroll
      for (int k2 = 0; k2 < 4; ++k2) {
        const float2 t = unpack2(hr[k2], bf);
        ff[2 * k2] += t.x;
        ff[2 * k2 + 1] += t.y;
      }
    }
    uint4 w;
    w.x = pack2(ff[0], ff[1], bf);
    w.y = pack2(ff[2], ff[3], bf);
    w.z = pack2(ff[4], ff[5], bf);
    w.w = pack2(ff[6], ff[7], bf);
    *reinterpret_cast<uint4*>(srow + sw) = w;
    if (EMIT) {
      const uint32_t* hw2 = reinterpret_cast<const uint32_t*>(&w);
#pragma unroll
      for (int k2 = 0; k2 < 4; ++k2) {
        const float2 t = unpack2(hw2[k2], bf);     // statistics of the values as stored (what the consumer reads)
        e1 += t.x + t.y;
        e2 = fmaf(t.x, t.x, e2);
        e2 = fmaf(t.y, t.y, e2);
      }
    }
  }
}


template <int BN, int STAGES, bool MMA>
__device__ __forceinline__ void conv_gn_math_warps(const ConvParams& p, uint8_t* smem, uint8_t* gsm,
                                                   const GnBars& B, int tile0, int tile_step, int num_tiles,
                                                   uint32_t rank) {
  using S = Conv2Smem<BN, STAGES, 4>;
  using GS = GnSmem<BN>;
  constexpr int kOct = BN / 8;
  constexpr int kNB = S::kOutBufs;                   // staging buffers: tile i uses buffer i % kNB
  uint8_t* ost0 = smem + STAGES * S::kStageBytes;
  float* s_part = reinterpret_cast<float*>(gsm + GS::kPart);
  const int* s_og = reinterpret_cast<const int*>(gsm + GS::kOg);
  float2* s_em0 = reinterpret_cast<float2*>(gsm + GS::kEm);

  const GnFuse& g = p.gn;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int e = warp - 4;
  const int q = e & 3, cc = e >> 2;                  // row quarter, 64-column sub-tile of this warp
  const int row = q * 32 + lane;
  const int hw = p.stats_hw;
  const bool small = hw < 32;                        // 4x4 images: 16-row segments, two per warp
  const int it = hw < kBM ? (row >> g.hw_shift) : 0; // image of this thread's row inside the tile
  const bool use_tab = g.G > 0 && g.ipt == 1 && g.expected > 1;
  const bool pre = g.pre_stats != nullptr;
  const bool wait_stats = g.G > 0 || pre;
  const bool bf = p.bf16 != 0;
  const uint32_t gsm_off = (uint32_t)(gsm - smem);
  // pass-2 variant: the hot epilogue shapes run gn_pass2_octets, everything else the phase-per-step code
  int variant = -1;
  if (!(g.out_lo || g.res_lo)) {
    if (g.G > 0 && g.silu) {
      const int nm2 = use_tab ? 0 : 1;
      if (g.pb && !g.has_res && !g.emit) variant = nm2;                                   // Block 1: + pose bias
      else if (!g.pb && g.has_res) variant = 2 + 2 * nm2 + (g.emit ? 1 : 0);              // Block 2: + residual
    } else if (pre && g.G == 0 && !g.silu && !g.pb && !g.has_res && !g.emit) {
      variant = g.ipt > 1 ? 7 : 6;                                                        // folded pre-norm (to_qkv)
    }
  }

  int kstage = 0;
  uint32_t kphase = 0;
  float* s_acc = reinterpret_cast<float*>(smem);
  int iter = 0;
  for (int tile = tile0; tile < num_tiles; tile += tile_step, ++iter) {
    const int b = iter & 1;
    const int ob = kNB == 2 ? (iter & 1) : 0;
    uint8_t* ost = ost0 + ob * S::kOutBytes;
    float2* s_em = s_em0 + ob * 32;
    const int m_pair = tile / p.n_tiles;
    const int n_tile = tile - m_pair * p.n_tiles;
    const int m_tile = 2 * m_pair + (int)rank;
    const int n_chan0 = n_tile * BN;
    const bool live = m_tile < p.m_tiles;          // the peer of an odd last pair owns phantom tiles (its last ones)
    int b0, y0;
    conv_tile_coords(p, m_tile, b0, y0);
    const int img0 = p.tiles_per_img > 0 ? m_tile / g.mt : m_tile * g.ipt;   // first image of the tile
    const bool img_ok = img0 + it < g.n_img;
    const __half* pb_row = g.pb + (size_t)(img_ok ? img0 + it : 0) * g.pb_stride + g.pb_off + n_chan0 + cc * 64;
    if (g.pb && live) asm volatile("prefetch.global.L1 [%0];" ::"l"(pb_row));

    conv_mma_tile<BN, BN / 64, STAGES, S::kStageBytes, S::kABytes, MMA>(p, smem, B.full, B.empty, kstage, kphase, s_acc);
    // ---- pass 1: accumulator -> registers, free the ring, per-octet partial sums
    uint32_t a[64];
    {
      const float* a_row = s_acc + row * acc_ld(BN) + cc * 64;
      acc_ld_32(a_row, *reinterpret_cast<uint32_t(*)[32]>(&a[0]));
      acc_ld_32(a_row + 32, *reinterpret_cast<uint32_t(*)[32]>(&a[32]));
      acc_release(B.tempty, lane);
    }
    if (!live) continue;

    float* f = reinterpret_cast<float*>(a);
    if (p.bias) {
      const float4* b4 = reinterpret_cast<const float4*>(p.bias + n_chan0 + cc * 64);
#pragma unroll
      for (int j = 0; j < 16; ++j) {
        const float4 c = __ldg(b4 + j);
        f[4 * j + 0] += c.x;
        f[4 * j + 1] += c.y;
        f[4 * j + 2] += c.z;
        f[4 * j + 3] += c.w;
      }
    }
    if (g.G > 0) {
#pragma unroll
      for (int hh = 0; hh < 2; ++hh) {
        float st[8];
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const float* ff = f + hh * 32 + j * 8;
          const float sm = (ff[0] + ff[1]) + (ff[2] + ff[3]) + ((ff[4] + ff[5]) + (ff[6] + ff[7]));
          float q2 = ff[0] * ff[0];
#pragma unroll
          for (int i = 1; i < 8; ++i) q2 = fmaf(ff[i], ff[i], q2);
          st[2 * j] = sm;
          st[2 * j + 1] = q2;
        }
        const int idx = small ? butterfly8<16>(st, lane) : butterfly8<32>(st, lane);
        const bool writer = small ? ((lane & 1) == 0) : ((lane & 3) == 0);
        const int segi = small ? (q * 2 + (lane >> 4)) : q;
        if (writer) s_part[(segi * kOct + cc * 8 + hh * 4) * 2 + idx] = st[0];   // idx = octet * 2 + {sum, sumsq}
      }
      __syncwarp();
      if (lane == 0) mbar_arrive(B.part);
    }
    if (wait_stats) mbar_wait(&B.stats[b], (iter >> 1) & 1);
    mbar_wait(B.res[ob], (iter / kNB) & 1);      // residual tile landed in the staging buffer / the buffer is free

    // ---- pass 2: normalise / activate / add, in place in the swizzled staging tile
    float e1 = 0.f, e2 = 0.f;
    const uint32_t tok = order_token(smem_u32(smem));          // tables below are read after the waits above
    const uint32_t a_mr = tok + gsm_off + GS::kMr + b * 64 * 8;
    const uint32_t a_sc = tok + gsm_off + GS::kTab + b * 2 * BN * 4 + cc * 256;
    const uint32_t a_sh = a_sc + BN * 4;
    const int grow = m_tile * kBM + row;            // linear output pixel
    const bool row_ok = grow < p.m_valid;
    const long long rpix = g.res_div > 0
        ? (long long)((g.res_base + b0) / g.res_div) * hw + (m_tile % g.mt) * kBM + row
        : (long long)grow;
    uint8_t* srow = ost + cc * (kBM * 128) + row * 128;
    const bool do_norm = g.G > 0;
    const bool do_silu = g.silu;
    const bool want_emit = g.emit != nullptr;
    if (variant >= 0) {
      const uint32_t a_srow = tok + (uint32_t)(srow - smem);
      const float4* gm4 = reinterpret_cast<const float4*>((pre ? g.pre_w1 : g.gamma) + n_chan0 + cc * 64);
      const float4* bt4 = reinterpret_cast<const float4*>((pre ? g.pre_wb : g.beta) + n_chan0 + cc * 64);
      const uint4* pb4 = reinterpret_cast<const uint4*>(pb_row);
      const int* og = s_og + cc * 8;
      const int it_gpt = it * g.gpt;
      switch (variant) {
        case 0: gn_pass2_octets<1, true, true, false, false>(f, a_sc, a_sh, a_mr, og, it_gpt, gm4, bt4, pb4, img_ok, srow, a_srow, row, bf, e1, e2); break;
        case 1: gn_pass2_octets<2, true, true, false, false>(f, a_sc, a_sh, a_mr, og, it_gpt, gm4, bt4, pb4, img_ok, srow, a_srow, row, bf, e1, e2); break;
        case 2: gn_pass2_octets<1, true, false, true, false>(f, a_sc, a_sh, a_mr, og, it_gpt, gm4, bt4, pb4, img_ok, srow, a_srow, row, bf, e1, e2); break;
        case 3: gn_pass2_octets<1, true, false, true, true>(f, a_sc, a_sh, a_mr, og, it_gpt, gm4, bt4, pb4, img_ok, srow, a_srow, row, bf, e1, e2); break;
        case 4: gn_pass2_octets<2, true, false, true, false>(f, a_sc, a_sh, a_mr, og, it_gpt, gm4, bt4, pb4, img_ok, srow, a_srow, row, bf, e1, e2); break;
        case 5: gn_pass2_octets<2, true, false, true, true>(f, a_sc, a_sh, a_mr, og, it_gpt, gm4, bt4, pb4, img_ok, srow, a_srow, row, bf, e1, e2); break;
        case 6: gn_pass2_octets<1, false, false, false, false>(f, a_sc, a_sh, a_mr, og, it_gpt, gm4, bt4, pb4, img_ok, srow, a_srow, row, bf, e1, e2); break;
        default: gn_pass2_octets<3, false, false, false, false>(f, a_sc, a_sh, a_mr + it * 8, og, it_gpt, gm4, bt4, pb4, img_ok, srow, a_srow, row, bf, e1, e2); break;
      }
    } else {
    // every step runs over all 64 values of the thread with its (launch-uniform) condition tested outside the
    // unrolled loop: one long basic block per step
    if (pre && g.ipt > 1) {
      const float2 mr = lds_f2(a_mr + it * 8);
      const float nm = -mr.x * mr.y;
      const float4* w14 = reinterpret_cast<const float4*>(g.pre_w1 + n_chan0 + cc * 64);
      const float4* wb4 = reinterpret_cast<const float4*>(g.pre_wb + n_chan0 + cc * 64);
#pragma unroll
      for (int j = 0; j < 16; ++j) {
        const float4 w1 = __ldg(w14 + j), wb = __ldg(wb4 + j);
        f[4 * j + 0] = fmaf(f[4 * j + 0], mr.y, fmaf(nm, w1.x, wb.x));
        f[4 * j + 1] = fmaf(f[4 * j + 1], mr.y, fmaf(nm, w1.y, wb.y));
        f[4 * j + 2] = fmaf(f[4 * j + 2], mr.y, fmaf(nm, w1.z, wb.z));
        f[4 * j + 3] = fmaf(f[4 * j + 3], mr.y, fmaf(nm, w1.w, wb.w));
      }
    } else if ((do_norm && use_tab) || pre) {
#pragma unroll
      for (int j = 0; j < 16; ++j) {
        const float4 sc = lds_f4(a_sc + j * 16), sh = lds_f4(a_sh + j * 16);
        f[4 * j + 0] = fmaf(f[4 * j + 0], sc.x, sh.x);
        f[4 * j + 1] = fmaf(f[4 * j + 1], sc.y, sh.y);
        f[4 * j + 2] = fmaf(f[4 * j + 2], sc.z, sh.z);
        f[4 * j + 3] = fmaf(f[4 * j + 3], sc.w, sh.w);
      }
    } else if (do_norm) {
      const float4* gm4 = reinterpret_cast<const float4*>(g.gamma + n_chan0 + cc * 64);
      const float4* bt4 = reinterpret_cast<const float4*>(g.beta + n_chan0 + cc * 64);
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const float2 mr = lds_f2(a_mr + (it * g.gpt + s_og[cc * 8 + j]) * 8);
#pragma unroll
        for (int h2 = 0; h2 < 2; ++h2) {
          const float4 gm = __ldg(gm4 + j * 2 + h2), bt = __ldg(bt4 + j * 2 + h2);
          float* ff = f + j * 8 + h2 * 4;
          ff[0] = fmaf(ff[0] - mr.x, mr.y * gm.x, bt.x);
          ff[1] = fmaf(ff[1] - mr.x, mr.y * gm.y, bt.y);
          ff[2] = fmaf(ff[2] - mr.x, mr.y * gm.z, bt.z);
          ff[3] = fmaf(ff[3] - mr.x, mr.y * gm.w, bt.w);
        }
      }
    }
    if (do_silu) {
#pragma unroll
      for (int i = 0; i < 64; ++i) f[i] = silu_ftz(f[i]);
    }
    if (g.pb && img_ok) {
      const uint4* pb4 = reinterpret_cast<const uint4*>(pb_row);
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const uint4 pv = __ldg(pb4 + j);
        const uint32_t* hp = reinterpret_cast<const uint32_t*>(&pv);
#pragma unroll
        for (int k2 = 0; k2 < 4; ++k2) {
          const float2 t = unpack2(hp[k2], bf);
          f[j * 8 + 2 * k2] += t.x;
          f[j * 8 + 2 * k2 + 1] += t.y;
        }
      }
    }
    if (g.has_res) {
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const uint4 rv = *reinterpret_cast<const uint4*>(srow + ((j ^ (row & 7)) << 4));
        const uint32_t* hr = reinterpret_cast<const uint32_t*>(&rv);
#pragma unroll
        for (int k2 = 0; k2 < 4; ++k2) {
          const float2 t = unpack2(hr[k2], bf);
          f[j * 8 + 2 * k2] += t.x;
          f[j * 8 + 2 * k2 + 1] += t.y;
        }
      }
      if (g.res_lo && row_ok) {
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          const uint4 rl = *reinterpret_cast<const uint4*>(g.res_lo + rpix * p.n_total + n_chan0 + cc * 64 + j * 8);
          const __half2* hl = reinterpret_cast<const __half2*>(&rl);
#pragma unroll
          for (int k2 = 0; k2 < 4; ++k2) {
            const float2 t = __half22float2(hl[k2]);
            f[j * 8 + 2 * k2] += t.x;
            f[j * 8 + 2 * k2 + 1] += t.y;
          }
        }
      }
    }
    const bool want_lo = g.out_lo && row_ok;
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      uint4 w;
      w.x = pack2(f[j * 8 + 0], f[j * 8 + 1], bf);
      w.y = pack2(f[j * 8 + 2], f[j * 8 + 3], bf);
      w.z = pack2(f[j * 8 + 4], f[j * 8 + 5], bf);
      w.w = pack2(f[j * 8 + 6], f[j * 8 + 7], bf);
      *reinterpret_cast<uint4*>(srow + ((j ^ (row & 7)) << 4)) = w;
      if (want_lo || want_emit) {
        const uint32_t* hw2 = reinterpret_cast<const uint32_t*>(&w);
        uint4 wl;
        uint32_t* pl = reinterpret_cast<uint32_t*>(&wl);
#pragma unroll
        for (int k2 = 0; k2 < 4; ++k2) {
          const float2 t = unpack2(hw2[k2], bf);
          pl[k2] = pack_half2(f[j * 8 + 2 * k2] - t.x, f[j * 8 + 2 * k2 + 1] - t.y);
          e1 += t.x + t.y;                 // statistics of the values as stored (what the consumer reads)
          e2 = fmaf(t.x, t.x, e2);
          e2 = fmaf(t.y, t.y, e2);
        }
        if (want_lo)
          *reinterpret_cast<uint4*>(g.out_lo + (size_t)grow * p.n_total + n_chan0 + cc * 64 + j * 8) = wl;
      }
    }
    }   // phase-per-step pass 2
    if (want_emit) {
      // 16-row segments: every image is a whole number of them at every resolution
#pragma unroll
      for (int off = 8; off > 0; off >>= 1) {
        e1 += __shfl_xor_sync(0xffffffffu, e1, off);
        e2 += __shfl_xor_sync(0xffffffffu, e2, off);
      }
      if ((lane & 15) == 0) s_em[cc * 8 + (row >> 4)] = make_float2(e1, e2);
    }
    fence_proxy_async_smem();
    __syncwarp();
    if (lane == 0) {
      mbar_arrive(&B.out[ob]);
      if (wait_stats) mbar_arrive(&B.tabfree[b]);
    }
  }
}

// statistics warp (warp 3) of the EPI == 4 epilogue
template <int BN, int STAGES>
__device__ __forceinline__ void conv_gn_stats_warp(const ConvParams& p, uint8_t* gsm, const GnBars& B, int tile0,
                                                   int tile_step, int num_tiles, uint32_t rank) {
  using GS = GnSmem<BN>;
  constexpr int kOct = BN / 8;
  const float* s_part = reinterpret_cast<const float*>(gsm + GS::kPart);
  float2* s_mr = reinterpret_cast<float2*>(gsm + GS::kMr);
  float* s_tab = reinterpret_cast<float*>(gsm + GS::kTab);
  int* s_og = reinterpret_cast<int*>(gsm + GS::kOg);
  float* s_x = reinterpret_cast<float*>(gsm + GS::kX);
  const GnFuse& g = p.gn;
  const int lane = threadIdx.x & 31;
  const int hw = p.stats_hw;
  const bool small = hw < 32;
  const int npairs = g.ipt * g.gpt;
  const bool use_tab = g.G > 0 && g.ipt == 1 && g.expected > 1;
  const bool pre = g.pre_stats != nullptr;
  if (!(g.G > 0 || pre)) return;          // residual / pose-bias-only epilogues: nothing to hand over
  for (int o = lane; o < kOct; o += 32) s_og[o] = (g.G > 0 && g.cpg < BN) ? (o * 8) / g.cpg : 0;
  __syncwarp();
  // register-only exchange (see `fast` below): one image per tile, 128-row tiles, groups = whole octet blocks of the lanes
  constexpr int kOpl = kOct / 8;                       // octets per lane: 32 lanes = 4 row segments x 8 octet blocks
  const int cpt = g.cpg < BN ? g.cpg : BN;             // channels of a group inside the tile
  const bool fast = use_tab && hw >= kBM && cpt % (kOpl * 8) == 0 && (g.gpt & (g.gpt - 1)) == 0 && g.gpt <= 8 &&
                    g.gpt * cpt == BN;
  const int lpp = 32 / g.gpt;                          // lanes per (image, group) pair
  float gam[BN / 32], bet[BN / 32];
  int tab_n_tile = -1;
  int iter = 0;
  for (int tile = tile0; tile < num_tiles; tile += tile_step, ++iter) {
    const int b = iter & 1;
    const int m_pair = tile / p.n_tiles;
    const int n_tile = tile - m_pair * p.n_tiles;
    const int m_tile = 2 * m_pair + (int)rank;
    if (m_tile >= p.m_tiles) break;                      // phantom tiles are this CTA's last ones
    const int n_chan0 = n_tile * BN;
    const int img0 = p.tiles_per_img > 0 ? m_tile / g.mt : m_tile * g.ipt;
    float* t_sc = s_tab + b * 2 * BN;
    float* t_sh = t_sc + BN;
    float2* mr = s_mr + b * 64;
    if (iter >= 2) mbar_wait(&B.tabfree[b], ((iter >> 1) - 1) & 1);   // tile iter-2 has read buffer b
    if (fast) {
      // ---- one image per tile, groups aligned to the lanes' octet blocks: the whole exchange in registers.
      // lane -> (octet block lane >> 2 of kOct / 8 octets, row segment lane & 3); xor tree over the lanes of a group
      if (n_tile != tab_n_tile) {
        tab_n_tile = n_tile;
#pragma unroll
        for (int j = 0; j < BN / 32; ++j) {
          gam[j] = __ldg(g.gamma + n_chan0 + lane + 32 * j);
          bet[j] = __ldg(g.beta + n_chan0 + lane + 32 * j);
        }
      }
      mbar_wait(B.part, iter & 1);
      float ax = 0.f, aq = 0.f;
#pragma unroll
      for (int k = 0; k < kOpl; ++k) {
        const float2 t = *reinterpret_cast<const float2*>(s_part + ((lane & 3) * kOct + (lane >> 2) * kOpl + k) * 2);
        ax += t.x;
        aq += t.y;
      }
      for (int off = 1; off < lpp; off <<= 1) {
        ax += __shfl_xor_sync(0xffffffffu, ax, off);
        aq += __shfl_xor_sync(0xffffffffu, aq, off);
      }
      const int sg = (m_tile / g.mt) * (p.n_tiles / g.tpg) + n_tile / g.tpg;
      const int slot = (m_tile % g.mt) * g.tpg + (n_tile % g.tpg);
      uint2* xp = g.xpart + (size_t)sg * g.expected * npairs * 2;
      if ((lane & (lpp - 1)) == 0) {
        const int pr = lane / lpp;
        st_volatile_u2(xp + ((size_t)slot * npairs + pr) * 2, make_uint2(__float_as_uint(ax), g.epoch));
        st_volatile_u2(xp + ((size_t)slot * npairs + pr) * 2 + 1, make_uint2(__float_as_uint(aq), g.epoch));
      }
      // word w = (slot * npairs + pair) * 2 + stat; 2 * npairs divides 32, so every word of lane l (w = l + 32 k)
      // belongs to (pair, stat) = l mod (2 npairs): sum over k in registers, then over the lanes of that class
      const int nw = g.expected * npairs * 2;        // <= 256 (host check)
      uint2 u[8];
#pragma unroll
      for (int k = 0; k < 8; ++k) {
        const int w = lane + 32 * k;
        u[k] = make_uint2(0u, g.epoch);
        if (w < nw) u[k] = ld_volatile_u2(xp + w);
      }
      float tot = 0.f;
#pragma unroll
      for (int k = 0; k < 8; ++k) {
        const int w = lane + 32 * k;
        if (w < nw && u[k].y != g.epoch) {
          const long long t0 = clock64();
          do {
            u[k] = ld_volatile_u2(xp + w);
            if (clock64() - t0 > 4000000000LL) __trap();   // no printf: see mbar_wait
          } while (u[k].y != g.epoch);
        }
        tot += __uint_as_float(u[k].x);
      }
      for (int off = 2 * npairs; off < 32; off <<= 1) tot += __shfl_xor_sync(0xffffffffu, tot, off);
      const float o1 = __shfl_sync(0xffffffffu, tot, lane & ~1), o2 = __shfl_sync(0xffffffffu, tot, lane | 1);
      const float mean_l = o1 * g.inv_cnt;                                  // lane l: group (l mod 2 npairs) >> 1
      const float rstd_l = rsqrtf(fmaxf(o2 * g.inv_cnt - mean_l * mean_l, 0.f) + g.eps);
#pragma unroll
      for (int j = 0; j < BN / 32; ++j) {
        const int c = lane + 32 * j;
        const int gl = g.cpg < BN ? c / g.cpg : 0;
        const float mean = __shfl_sync(0xffffffffu, mean_l, 2 * gl);
        const float rstd = __shfl_sync(0xffffffffu, rstd_l, 2 * gl);
        const float sc = rstd * gam[j];
        t_sc[c] = sc;
        t_sh[c] = bet[j] - mean * sc;
      }
    } else
    if (g.G > 0) {
      mbar_wait(B.part, iter & 1);
      // sums of this tile per (image, group) pair: fixed order over row segments and channel octets
      float Sx[2], Qx[2];
#pragma unroll
      for (int k = 0; k < 2; ++k) {
        const int pr = lane + 32 * k;
        Sx[k] = 0.f;
        Qx[k] = 0.f;
        if (pr < npairs) {
          const int ii = pr / g.gpt, gl = pr - ii * g.gpt;
          const int spi = hw >= kBM ? 4 : (small ? 1 : (hw >> 5));   // row segments of this image in the tile
          const int s0 = hw >= kBM ? 0 : ii * spi;
          const int opg = (g.cpg < BN ? g.cpg : BN) >> 3;
          const int o0 = gl * opg;
          for (int sgm = s0; sgm < s0 + spi; ++sgm) {
#pragma unroll 4
            for (int o = o0; o < o0 + opg; ++o) {
              const float2 t = *reinterpret_cast<const float2*>(s_part + (sgm * kOct + o) * 2);
              Sx[k] += t.x;
              Qx[k] += t.y;
            }
          }
        }
      }
      if (g.expected > 1) {
        // publish {value, epoch}; poll the [slot][pair][2] block of the sync group until every word carries this
        // launch's epoch (all loads of the warp in flight at once)
        const int sg = (m_tile / g.mt) * (p.n_tiles / g.tpg) + n_tile / g.tpg;
        const int slot = (m_tile % g.mt) * g.tpg + (n_tile % g.tpg);
        uint2* xp = g.xpart + (size_t)sg * g.expected * npairs * 2;
#pragma unroll
        for (int k = 0; k < 2; ++k) {
          const int pr = lane + 32 * k;
          if (pr < npairs) {
            st_volatile_u2(xp + ((size_t)slot * npairs + pr) * 2, make_uint2(__float_as_uint(Sx[k]), g.epoch));
            st_volatile_u2(xp + ((size_t)slot * npairs + pr) * 2 + 1, make_uint2(__float_as_uint(Qx[k]), g.epoch));
          }
        }
        const int nw = g.expected * npairs * 2;        // <= 256 (host check)
        uint2 u[8];
#pragma unroll
        for (int k = 0; k < 8; ++k) {
          const int w = lane + 32 * k;
          u[k] = make_uint2(0u, g.epoch);
          if (w < nw) u[k] = ld_volatile_u2(xp + w);
        }
#pragma unroll
        for (int k = 0; k < 8; ++k) {
          const int w = lane + 32 * k;
          if (w < nw) {
            if (u[k].y != g.epoch) {
              const long long t0 = clock64();
              do {
                u[k] = ld_volatile_u2(xp + w);
                if (clock64() - t0 > 4000000000LL) __trap();   // no printf: see mbar_wait
              } while (u[k].y != g.epoch);
            }
            s_x[w] = __uint_as_float(u[k].x);
          }
        }
        __syncwarp();
        if (use_tab) {
          // one image per tile: totals per (group, statistic) in slot order, then per-channel scale / shift
          float tot = 0.f;
          if (lane < 2 * g.gpt)
            for (int sl = 0; sl < g.expected; ++sl) tot += s_x[(sl * npairs + (lane >> 1)) * 2 + (lane & 1)];
#pragma unroll
          for (int c = lane; c < BN; c += 32) {
            const int gl = s_og[c >> 3];
            const float s1 = __shfl_sync(0xffffffffu, tot, 2 * gl);
            const float s2 = __shfl_sync(0xffffffffu, tot, 2 * gl + 1);
            const float mean = s1 * g.inv_cnt;
            const float var = fmaxf(s2 * g.inv_cnt - mean * mean, 0.f);
            const float sc = rsqrtf(var + g.eps) * __ldg(g.gamma + n_chan0 + c);
            t_sc[c] = sc;
            t_sh[c] = __ldg(g.beta + n_chan0 + c) - mean * sc;
          }
        } else {
#pragma unroll
          for (int k = 0; k < 2; ++k) {
            const int pr = lane + 32 * k;
            if (pr < npairs) {
              float S1 = 0.f, S2 = 0.f;
              for (int sl = 0; sl < g.expected; ++sl) {
                S1 += s_x[(sl * npairs + pr) * 2];
                S2 += s_x[(sl * npairs + pr) * 2 + 1];
              }
              const float mean = S1 * g.inv_cnt;
              const float var = fmaxf(S2 * g.inv_cnt - mean * mean, 0.f);
              mr[pr] = make_float2(mean, rsqrtf(var + g.eps));
            }
          }
        }
      } else {
#pragma unroll
        for (int k = 0; k < 2; ++k) {
          const int pr = lane + 32 * k;
          if (pr < npairs) {
            const float mean = Sx[k] * g.inv_cnt;
            const float var = fmaxf(Qx[k] * g.inv_cnt - mean * mean, 0.f);
            mr[pr] = make_float2(mean, rsqrtf(var + g.eps));
          }
        }
      }
    }
    if (pre) {
      // folded pre-norm: (mean, rstd) of each input image of the tile from its producer's partial sums
      // (all loads issued together, summed in part order)
      if (g.ipt == 1) {
        float s1 = 0.f, s2 = 0.f;
        for (int k0 = 0; k0 < g.pre_parts; k0 += 32) {
          float2 t = make_float2(0.f, 0.f);
          if (k0 + lane < g.pre_parts) t = g.pre_stats[(size_t)img0 * g.pre_parts + k0 + lane];
          const int n = g.pre_parts - k0 < 32 ? g.pre_parts - k0 : 32;
          for (int k = 0; k < n; ++k) {
            s1 += __shfl_sync(0xffffffffu, t.x, k);
            s2 += __shfl_sync(0xffffffffu, t.y, k);
          }
        }
        const float mean = s1 * g.pre_inv_cnt;
        const float rstd = rsqrtf(fmaxf(s2 * g.pre_inv_cnt - mean * mean, 0.f) + g.eps);
#pragma unroll
        for (int c = lane; c < BN; c += 32) {
          t_sc[c] = rstd;
          t_sh[c] = __ldg(g.pre_wb + n_chan0 + c) - rstd * mean * __ldg(g.pre_w1 + n_chan0 + c);
        }
      } else if (lane < g.ipt) {
        float2 t[8];
#pragma unroll
        for (int k = 0; k < 8; ++k) {
          t[k] = make_float2(0.f, 0.f);
          if (k < g.pre_parts && img0 + lane < g.n_img) t[k] = g.pre_stats[(size_t)(img0 + lane) * g.pre_parts + k];
        }
        float s1 = 0.f, s2 = 0.f;
#pragma unroll
        for (int k = 0; k < 8; ++k)
          if (k < g.pre_parts) {
            s1 += t[k].x;
            s2 += t[k].y;
          }
        const float mean = s1 * g.pre_inv_cnt;
        mr[lane] = make_float2(mean, rsqrtf(fmaxf(s2 * g.pre_inv_cnt - mean * mean, 0.f) + g.eps));
      }
    }
    __syncwarp();
    if (lane == 0) mbar_arrive(&B.stats[b]);
  }
}

// store warp (warp 2) of the EPI == 4 epilogue
template <int BN, int STAGES>
__device__ __forceinline__ void conv_gn_store_warp(const ConvParams& p, uint8_t* smem, uint8_t* gsm, const GnBars& B,
                                                   int tile0, int tile_step, int num_tiles, uint32_t rank) {
  using S = Conv2Smem<BN, STAGES, 4>;
  using GS = GnSmem<BN>;
  constexpr int kNS = BN / 64;
  constexpr int kNB = S::kOutBufs;
  uint8_t* ost0 = smem + STAGES * S::kStageBytes;
  const float2* s_em0 = reinterpret_cast<const float2*>(gsm + GS::kEm);
  const GnFuse& g = p.gn;
  const int lane = threadIdx.x & 31;
  const int hw = p.stats_hw;
  // the residual tile of tile t is TMA-loaded into its staging buffer (same box / swizzle as the store) once the
  // previous store from that buffer has read it; without a residual the same barrier just says "the buffer is free"
  auto stage = [&](int t, int ob) {
    if (t >= num_tiles) return;
    const int mp = t / p.n_tiles;
    const int nt = t - mp * p.n_tiles;
    const int mt2 = 2 * mp + (int)rank;
    if (g.has_res && mt2 < p.m_tiles) {
      int bb, yy;
      conv_tile_coords(p, mt2, bb, yy);
      const int rb = g.res_div > 0 ? (g.res_base + bb) / g.res_div : bb;
      uint8_t* dst = ost0 + ob * S::kOutBytes;
      mbar_expect_tx(B.res[ob], S::kOutBytes);
#pragma unroll 1
      for (int c2 = 0; c2 < kNS; ++c2)
        tma_load_4d(dst + c2 * (kBM * 128), &p.rmap, B.res[ob], nt * BN + c2 * 64, 0, yy, rb);
    } else {
      mbar_arrive(B.res[ob]);
    }
  };
  if (lane == 0) {
    stage(tile0, 0);
    if (kNB == 2) stage(tile0 + tile_step, 1);
  }
  int iter = 0;
  for (int tile = tile0; tile < num_tiles; tile += tile_step, ++iter) {
    const int ob = kNB == 2 ? (iter & 1) : 0;
    const int m_pair = tile / p.n_tiles;
    const int n_tile = tile - m_pair * p.n_tiles;
    const int m_tile = 2 * m_pair + (int)rank;
    if (m_tile >= p.m_tiles) break;
    int b0, y0;
    conv_tile_coords(p, m_tile, b0, y0);
    const int img0 = p.tiles_per_img > 0 ? m_tile / g.mt : m_tile * g.ipt;
    mbar_wait(&B.out[ob], (iter / kNB) & 1);
    if (g.emit && lane < g.ipt && img0 + lane < g.n_img) {
      const float2* s_em = s_em0 + ob * 32;
      const int r16 = hw >= kBM ? 8 : (hw >> 4);
      float s1 = 0.f, s2 = 0.f;
      for (int h2 = 0; h2 < kNS; ++h2)
        for (int r = lane * r16; r < (lane + 1) * r16; ++r) {
          s1 += s_em[h2 * 8 + r].x;
          s2 += s_em[h2 * 8 + r].y;
        }
      g.emit[(size_t)(img0 + lane) * g.emit_parts + (m_tile % g.mt) * p.n_tiles + n_tile] = make_float2(s1, s2);
    }
    __syncwarp();
    if (lane == 0) {
      uint8_t* ost = ost0 + ob * S::kOutBytes;
#pragma unroll 1
      for (int c2 = 0; c2 < kNS; ++c2)
        tma_store_4d(&p.omap[0], ost + c2 * (kBM * 128), n_tile * BN + c2 * 64, 0, y0, b0);
      tma_store_commit();
      // the next user of this buffer is tile iter + kNB: hand it over once this store has read the buffer (with two
      // buffers the math warps meanwhile work in the other one)
      const int nt = tile + kNB * tile_step;
      if (nt < num_tiles) {
        tma_store_wait_read0();
        stage(nt, ob);
      }
    }
    __syncwarp();
  }
  if (lane == 0) tma_store_wait_all();
}

// EPI: 0 = plain epilogue (the sweep), 1 = extras (ReLU / residual / hi-lo / fp32), 2 = GEGLU, 4 = GroupNorm fused
// Register split (setmaxnreg) of the clustered kernel at 384 and 512 threads: the control warpgroup (warps 0-3: the
// producer, and with EPI == 4 the store and statistics warps) drops to conv2_ctl_regs, the math warpgroups share the
// rest of the 64 K register file evenly: 224 per thread at 384 threads (208 with EPI == 4), 144 at 512 threads
// (BN = 192, EPI == 4).  Blocks of 256 threads already allow 255 registers per thread and keep that limit.
// Not every instantiation is spill-free (ptxas -v, spill store / load bytes): <192,4,4> 134 / 212,
// spread over the statistics warp at 80 and the math warps at 144; at 512 threads
// the four warpgroups average 128 registers, and moving registers between the roles moves the spills with them.
// <128,4,4> 60 / 112 (statistics warp and epilogue).
__host__ __device__ constexpr int conv2_threads(int BN, int EPI) { return EPI == 4 ? gn_threads(BN) : kConvThreads; }
__host__ __device__ constexpr int conv2_ctl_regs(int EPI) { return EPI == 4 ? 80 : 56; }
__host__ __device__ constexpr int conv2_launch_regs(int threads) { return 65536 / threads / 8 * 8; }
__host__ __device__ constexpr int conv2_math_regs(int threads, int EPI) {
  return (conv2_launch_regs(threads) * (threads / 128) - conv2_ctl_regs(EPI)) / (threads / 128 - 1) / 8 * 8;
}

template <int BN, int STAGES, int EPI>
__global__ void __cluster_dims__(2, 1, 1) __launch_bounds__(conv2_threads(BN, EPI), 1)
conv_tc2_kernel(const __grid_constant__ ConvParams p) {
  using S = Conv2Smem<BN, STAGES, EPI>;
  static_assert(BN % 64 == 0 && BN <= 256, "BN must be a multiple of 64");
  constexpr int kThreads = conv2_threads(BN, EPI);
  constexpr int kMathWarps = kThreads / 32 - 4;                        // warps 4.. run mainloop + epilogue
  constexpr bool kRegSplit = kThreads > 256;
  constexpr int kCtlRegs = conv2_ctl_regs(EPI);
  constexpr int kMathRegs = conv2_math_regs(kThreads, EPI);
  static_assert(!kRegSplit || (kMathRegs <= 256 && kCtlRegs + (kThreads / 128 - 1) * kMathRegs <=
                               conv2_launch_regs(kThreads) * (kThreads / 128)), "register split");

  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) &
                                             ~static_cast<uintptr_t>(1023));
  uint8_t* out_stage = smem + STAGES * S::kStageBytes;
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + S::kBarOffset);
  uint64_t* empty_bar = full_bar + STAGES;
  uint64_t* tempty_bar = empty_bar + STAGES;
  uint64_t* res_bar = tempty_bar + 1;                                 // EPI == 4: residual tile landed
  uint64_t* gn_bar = res_bar + 1;                                     // EPI == 4: part, stats[2], tabfree[2], out[2], res of buffer 1
  static_assert((2 * STAGES + 2 + 8) * 8 <= 256, "barrier block overflow");
  float* s_bias = reinterpret_cast<float*>(smem + S::kBiasOffset);
  float* s_acc = reinterpret_cast<float*>(smem);

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const uint32_t rank = cluster_ctarank();
  const int m_pairs = (p.m_tiles + 1) >> 1;
  const int num_tiles = m_pairs * p.n_tiles;          // pair tiles
  const int tile0 = cluster_id_x(), tile_step = num_clusters_x();

  if (warp == 0 && lane == 0) {
    for (int i = 0; i < p.n_amaps; ++i) prefetch_tmap(&p.amap[i]);
    prefetch_tmap(&p.bmap);
    for (int i = 0; i < p.n_par; ++i) prefetch_tmap(&p.omap[i]);
  }
  if (warp == 1 && lane == 0) {
    for (int s = 0; s < STAGES; ++s) {
      mbar_init(&full_bar[s], 1);
      mbar_init(&empty_bar[s], conv_mma_warps(kMathWarps / 4));
    }
    mbar_init(tempty_bar, kMathWarps);
    mbar_init(res_bar, 1);
    if constexpr (EPI == 4) {
      mbar_init(&gn_bar[0], gn_epi_warps(BN));                          // part
      mbar_init(&gn_bar[1], 1);                                         // stats[0]
      mbar_init(&gn_bar[2], 1);                                         // stats[1]
      mbar_init(&gn_bar[3], gn_epi_warps(BN));                          // tabfree[0]
      mbar_init(&gn_bar[4], gn_epi_warps(BN));                          // tabfree[1]
      mbar_init(&gn_bar[5], gn_epi_warps(BN));                          // out[0]
      mbar_init(&gn_bar[6], gn_epi_warps(BN));                          // out[1]
      mbar_init(&gn_bar[7], 1);                                         // res of staging buffer 1
    }
    fence_mbar_init();
  }
  __syncthreads();
  // Programmatic dependent launch: everything above (barrier init, descriptor prefetch) touched no global memory
  // and may overlap the tail of the previous kernel in the stream; from here on the kernel reads what that kernel
  // wrote.  The next kernel's CTAs may be scheduled as soon as this grid's CTAs retire.
  pdl_sync();
  auto gn_bars = [&] {                                                // EPI == 4
    GnBars B;
    B.full = full_bar; B.empty = empty_bar; B.tempty = tempty_bar; B.res[0] = res_bar; B.res[1] = &gn_bar[7];
    B.part = &gn_bar[0]; B.stats = &gn_bar[1]; B.tabfree = &gn_bar[3]; B.out = &gn_bar[5];
    return B;
  };
  uint8_t* gsm = smem + S::kGnOffset;

  // Each warpgroup sets its register limit once, before its warps take their roles (setmaxnreg is warpgroup-wide).
  if (warp < 4) {
    if constexpr (kRegSplit) setmaxnreg_dec<kCtlRegs>();
    if (warp == 0) {
    // ===================== TMA producer =====================
    int stage = 0;
    uint32_t phase = 0;
    int iter = 0;
    for (int tile = tile0; tile < num_tiles; tile += tile_step, ++iter) {
      const int m_pair = tile / p.n_tiles;
      const int n_tile = tile - m_pair * p.n_tiles;
      const int m_tile = 2 * m_pair + (int)rank;       // may be one past the end: TMA zero-fills
      const int par = n_tile / p.n_tiles_par;
      const int py = par >> 1, px = par & 1;
      int b0, y0;
      conv_tile_coords(p, m_tile, b0, y0);
      if (iter > 0) mbar_wait(tempty_bar, (iter - 1) & 1);     // the previous accumulator tile left the ring
      int kcol = 0;
      for (int s = 0; s < p.nseg; ++s) {
        const ConvSeg sg = p.seg[s];
        const CUtensorMap* am = &p.amap[sg.map];
        if (sg.wcol1) kcol = sg.wcol1 - 1;
        for (int ch = 0; ch < sg.nchunks; ++ch) {
          mbar_wait(&empty_bar[stage], phase ^ 1);
          if (elect_one()) {
            uint8_t* sa = smem + stage * S::kStageBytes;
            mbar_expect_tx(&full_bar[stage], S::kStageBytes);
            tma_load_4d(sa, am, &full_bar[stage], ch * kBK, sg.dx + px, y0 + sg.dy + py, b0);
            tma_load_2d(sa + S::kABytes, &p.bmap, &full_bar[stage], kcol, n_tile * BN);
          }
          kcol += kBK;
          if (++stage == STAGES) { stage = 0; phase ^= 1; }
        }
      }
    }
    } else if constexpr (EPI == 4) {
      // ===================== GroupNorm-fused epilogue: store warp 2, statistics warp 3 =====================
      const GnBars B = gn_bars();
      if (warp == 2) conv_gn_store_warp<BN, STAGES>(p, smem, gsm, B, tile0, tile_step, num_tiles, rank);
      else if (warp == 3) conv_gn_stats_warp<BN, STAGES>(p, gsm, B, tile0, tile_step, num_tiles, rank);
    }
  } else if constexpr (EPI == 4) {
    // ===================== mainloop + epilogue with GroupNorm fused, bookkeeping on warps 2 / 3 =====================
    if constexpr (kRegSplit) setmaxnreg_inc<kMathRegs>();
    if (warp >= 12) {                       // BN = 192: the third math warpgroup runs the epilogue only
      if constexpr (kMathWarps == 12) conv_gn_math_warps<BN, STAGES, false>(p, smem, gsm, gn_bars(), tile0, tile_step, num_tiles, rank);
    } else {
      conv_gn_math_warps<BN, STAGES, true>(p, smem, gsm, gn_bars(), tile0, tile_step, num_tiles, rank);
    }
  } else {
    // ===================== mainloop + epilogue (own 128 rows, 8 warps) =====================
    static_assert(kRegSplit, "the plain epilogues run 384 threads");
    setmaxnreg_inc<kMathRegs>();
    const int e = warp - 4;
    const int etid = threadIdx.x - 128;
    int kstage = 0;
    uint32_t kphase = 0;
    int obuf = 0;
    constexpr bool kPrefetchRes = EPI == 1 && BN <= 128;   // 32 registers; wider tiles load in place
    ResPrefetch<kPrefetchRes ? BN : 64> pre;
    if constexpr (kPrefetchRes) {
      if (tile0 < num_tiles) {     // operands of this CTA's first tile (residual convs have n_par == 1)
        const int mp0 = tile0 / p.n_tiles;
        pre.load(p, 2 * mp0 + (int)rank, (tile0 - mp0 * p.n_tiles) * BN, e, lane);
      }
    }
    for (int tile = tile0; tile < num_tiles; tile += tile_step) {
      const int m_pair = tile / p.n_tiles;
      const int n_tile = tile - m_pair * p.n_tiles;
      const int m_tile = 2 * m_pair + (int)rank;
      const int par = n_tile / p.n_tiles_par;
      const int n_chan0 = (n_tile - par * p.n_tiles_par) * BN;
      int b0, y0;
      conv_tile_coords(p, m_tile, b0, y0);
      if (etid < BN) s_bias[etid] = p.bias ? __ldg(p.bias + n_chan0 + etid) : 0.f;
      if constexpr (kPrefetchRes) {
        const int nt = tile + tile_step;
        const int nmp = nt / p.n_tiles;
        pre.next_m_tile = nt < num_tiles ? 2 * nmp + (int)rank : -1;
        pre.next_n_chan0 = (nt - nmp * p.n_tiles) * BN;
      }
      uint8_t* ost = out_stage + obuf * S::kOutBytes;
      if (etid == 0) {       // the store that last used this staging buffer has read it
        if constexpr (S::kOutBufs == 2) tma_store_wait_read1();
        else tma_store_wait_read0();
      }
      asm volatile("bar.sync 1, 256;" ::: "memory");
      conv_mma_tile<BN, 2, STAGES, S::kStageBytes, S::kABytes>(p, smem, full_bar, empty_bar, kstage, kphase, s_acc);
      if constexpr (EPI == 2)
        conv_epilogue_geglu(ost, s_bias, s_acc, e, lane);
      else if constexpr (kPrefetchRes)
        conv_epilogue_tile<BN, true>(p, ost, s_bias, s_acc, m_tile, n_chan0, e, lane, &pre, par);
      else if constexpr (EPI == 1)
        conv_epilogue_tile<BN, true>(p, ost, s_bias, s_acc, m_tile, n_chan0, e, lane, nullptr, par);
      else
        conv_epilogue_tile<BN, false>(p, ost, s_bias, s_acc, m_tile, n_chan0, e, lane);
      acc_release(tempty_bar, lane);
      fence_proxy_async_smem();
      asm volatile("bar.sync 1, 256;" ::: "memory");
      if (etid == 0) {
        if constexpr (EPI == 2) {
          tma_store_4d(&p.omap[0], ost, n_chan0 / 2, 0, y0, b0);
        } else {
#pragma unroll 1
          for (int cc = 0; cc < BN / 64; ++cc)
            tma_store_4d(&p.omap[par], ost + cc * (kBM * 128), n_chan0 + cc * 64, 0, y0, b0);
        }
        tma_store_commit();
      }
      obuf ^= S::kOutBufs - 1;
    }
    if (etid == 0) tma_store_wait_all();
  }
}

template <int BN, int STAGES, int EPI>
inline int launch_conv_tc2_t(const ConvParams& p, int num_sms, cudaStream_t stream) {
  using S = Conv2Smem<BN, STAGES, EPI>;
  // the shared-memory opt-in and the resident-cluster count are per device
  static int max_clusters_of[kMaxDevices];      // 0: not initialised on this device yet
  int dev = 0;
  NOPE_CUDA(cudaGetDevice(&dev));
  NOPE_CHECK(dev >= 0 && dev < kMaxDevices, "device index out of range");
  if (max_clusters_of[dev] == 0) {
    if (const char* e = getenv("NOPE_MBAR_HINT")) {
      const uint32_t v = (uint32_t)atoi(e);
      NOPE_CUDA(cudaMemcpyToSymbol(c_mbar_suspend_ns, &v, sizeof v));
    }
    NOPE_CUDA(cudaFuncSetAttribute(conv_tc2_kernel<BN, STAGES, EPI>,
                                   cudaFuncAttributeMaxDynamicSharedMemorySize, S::kTotal));
    int mc = num_sms / 2;
    if (EPI == 4) {
      // tiles of one image wait for each other: every cluster of the grid must be resident
      cudaLaunchConfig_t cfg;
      memset(&cfg, 0, sizeof cfg);
      cfg.gridDim = dim3(num_sms, 1, 1);
      cfg.blockDim = dim3(conv2_threads(BN, EPI), 1, 1);
      cfg.dynamicSmemBytes = S::kTotal;
      cudaLaunchAttribute at;
      at.id = cudaLaunchAttributeClusterDimension;
      at.val.clusterDim.x = 2; at.val.clusterDim.y = 1; at.val.clusterDim.z = 1;
      cfg.attrs = &at;
      cfg.numAttrs = 1;
      int n = 0;
      NOPE_CUDA(cudaOccupancyMaxActiveClusters(&n, conv_tc2_kernel<BN, STAGES, EPI>, &cfg));
      NOPE_CHECK(n >= 1, "conv_tc2_kernel: no resident cluster fits on this device");
      if (n < mc) mc = n;
    }
    max_clusters_of[dev] = mc;
  }
  const int pair_tiles = ((p.m_tiles + 1) / 2) * p.n_tiles;
  const int max_clusters = max_clusters_of[dev];
  const int clusters = pair_tiles < max_clusters ? pair_tiles : max_clusters;
  cudaLaunchConfig_t cfg;
  memset(&cfg, 0, sizeof cfg);
  cfg.gridDim = dim3(2 * clusters, 1, 1);
  cfg.blockDim = dim3(conv2_threads(BN, EPI), 1, 1);
  cfg.dynamicSmemBytes = S::kTotal;
  cfg.stream = stream;
  cudaLaunchAttribute at;
  at.id = cudaLaunchAttributeProgrammaticStreamSerialization;
  at.val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = &at;
  cfg.numAttrs = (pdl_mask() & 1) ? 1 : 0;
  NOPE_CUDA(cudaLaunchKernelEx(&cfg, conv_tc2_kernel<BN, STAGES, EPI>, p));
  return 0;
}

// GroupNorm-fused epilogue (GnFuse in p.gn)
inline int launch_conv_gn(const ConvParams& p, int bn, int num_sms, cudaStream_t stream) {
  if (p.n_par != 1 || p.geglu || conv_needs_extras(p) || p.stats)
    return fail("launch_conv_gn: the fused GroupNorm epilogue takes a plain convolution");
  // ring depths: the deepest ring that fits 227 KB of shared memory beside the staging buffers
  switch (bn) {
    case 192: return launch_conv_tc2_t<192, 4, 4>(p, num_sms, stream);
    case 128: return launch_conv_tc2_t<128, 4, 4>(p, num_sms, stream);
    case 64: return launch_conv_tc2_t<64, 7, 4>(p, num_sms, stream);
  }
  return fail("launch_conv_gn: unsupported BN");
}

inline int launch_conv_tc2(const ConvParams& p, int bn, int num_sms, cudaStream_t stream) {
  const bool ex = conv_needs_extras(p);
  if (p.geglu) {
    if (bn != 128 || ex || p.stats || p.n_par != 1) return fail("launch_conv_tc2: GEGLU epilogue needs BN = 128, no extras");
    return launch_conv_tc2_t<128, 5, 2>(p, num_sms, stream);
  }
  switch (bn) {
    // 256-wide tiles (LDM variant: every width is a multiple of 256): twice the MMA work per byte of A
    case 256:
      if (ex) return fail("launch_conv_tc2: epilogue extras need BN <= 192");
      return launch_conv_tc2_t<256, 3, 0>(p, num_sms, stream);
    case 192: return ex ? launch_conv_tc2_t<192, 4, 1>(p, num_sms, stream)
                        : launch_conv_tc2_t<192, 4, 0>(p, num_sms, stream);
    case 128: return ex ? launch_conv_tc2_t<128, 5, 1>(p, num_sms, stream)
                        : launch_conv_tc2_t<128, 5, 0>(p, num_sms, stream);
    case 64: return ex ? launch_conv_tc2_t<64, 8, 1>(p, num_sms, stream)
                       : launch_conv_tc2_t<64, 8, 0>(p, num_sms, stream);
  }
  return fail("launch_conv_tc2: unsupported BN");
}

}  // namespace nope
