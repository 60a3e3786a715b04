// nope_b200 -- implicit-GEMM convolution on wgmma tensor cores (sm_90a): the pieces the clustered
// kernel (conv_tc2_kernel, conv_tc2.cuh) is built from -- launch parameters (ConvParams, GnFuse), the
// wgmma mainloop of one tile (conv_mma_tile), the plain and GEGLU epilogues, and the tensor-map helpers.
//
// The convolution serves every GEMM-shaped op of the pose-conditioned UNet
// (reference: src/model/u_net/denoising_diffusion_pytorch/model_utils.py:240
//  conv3x3, :171 1x1-after-unshuffle, :269 res_conv, :373-374/:399-401 qkv and
//  to_out 1x1, :261-263 the pose projection Linear):
//
//   out[m, n] = bias[n] + sum_k A[m, k] * Wp[n, k]
//
// m enumerates output pixels of all batched hypotheses (NHWC, fp16), n output
// channels, k = (filter tap, source tensor, input channel).  A is never
// materialised: for each K-step of 64 channels the producer thread issues ONE
// 4-D TMA box load {64 ch, w_cnt, h_cnt, b_cnt} (= 128 pixels) from the NHWC
// activation tensor, shifted by the tap offset (dy, dx); out-of-image rows and
// columns are zero-filled by the TMA unit, which is exactly conv padding.  The
// box lands in shared memory as a 128-row x 128-byte K-major SWIZZLE_128B tile,
// the canonical wgmma operand layout.  Channel concatenation (skip
// connections, u_net.py:186-194) is two source tensor maps walked by the same K
// loop; pixel-unshuffle + 1x1 (HardDownsample) is four stride-2 tensor maps.
#pragma once
#include "common.cuh"
#include <cudaTypedefs.h>

#include <cstring>
#include <map>
#include <tuple>
#include <vector>

namespace nope {

constexpr int kBM = 128;         // pixels per tile (UMMA M)
constexpr int kBK = 64;          // channels per K-step (one 128-byte swizzle row)
constexpr int kMaxSeg = 64;      // 9 taps x 2 sources x 3 split-precision products
constexpr int kMaxAMaps = 8;     // 4 stride-2 lattices x (hi, lo)
constexpr int kConvThreads = 384;   // 4 control warps + 8 epilogue warps
constexpr int kEpiWarps = 8;

struct ConvSeg {
  int16_t map;      // index into amap[]
  int16_t dy, dx;   // tap offset in pixels
  int16_t nchunks;  // channels / 64 in this segment
  int32_t wcol1;    // 0: weight columns continue where the previous segment ended; else first column + 1
                    // (split precision re-reads the W_hi columns for the A_lo product)
};

// GroupNorm applied in the epilogue of the producing convolution (clustered kernel, EPI == 4):
//   y = [SiLU]((acc - mean) * rstd * gamma + beta) + pose_bias[img, c] + residual[pixel, c]
// (Block.forward / ResnetBlock.forward, model_utils.py:237-253, 271-279; PreNorm / to_out[1] of
// LinearAttention, model_utils.py:230, 401).  The statistics of an image are spread over the CTA
// tiles that hold its pixels (and, for groups wider than one tile, its channels): every such tile
// publishes its partial sums as {value, epoch} words (8-byte stores: value and tag arrive together,
// the low-latency flag protocol of NCCL's LL mode -- no fences, no atomics), then polls the
// `expected` slots of its sync group until all carry this launch's epoch (all tiles are resident:
// the kernel is persistent with one CTA per SM).  Partials are combined in slot order, so results
// do not depend on launch size or timing.
struct GnFuse {
  const float* gamma;    // [n_total]; G == 0: no normalisation (residual / pose-bias epilogue only)
  const float* beta;
  int G;                 // groups (0, 1 or 8)
  int cpg;               // channels per group
  int gpt;               // groups per N-tile            = max(1, BN / cpg)
  int tpg;               // N-tiles per group            = max(1, cpg / BN)
  int mt;                // M-tiles per image            = max(1, H*W / 128)
  int ipt;               // images per M-tile            = max(1, 128 / (H*W))
  int expected;          // tiles per sync group         = mt * tpg
  int hw_shift;          // log2(H*W)
  float inv_cnt;         // 1 / (H*W * cpg)
  float eps;
  int silu;
  const __half* pb;      // per-image channel bias added after the activation (pose projection) or nullptr
  int pb_stride, pb_off;
  int has_res;           // residual tile arrives through ConvParams::rmap (TMA) into the output staging
  int res_div, res_base; // res_div > 0: residual image index = (res_base + img) / res_div (hoisted prefix)
  int n_img;             // valid images
  uint2* xpart;          // [sync group][slot][ipt * gpt][2]: {sum, epoch}, {sum of squares, epoch}
  unsigned epoch;        // tag of this launch (unique per launch on the buffer, never 0)
  float2* emit;          // optional: GroupNorm(1, C) partial sums of the stored output,
  int emit_parts;        //   emit[img * emit_parts + (m_in_img * n_tiles + n_tile)], emit_parts = mt * n_tiles
  // split precision (activations carried as fp16 hi + lo): remainder of the output, [pixel][n_total],
  // and of the residual (same layout; the residual image mapping of res_div applies)
  __half* out_lo;
  const __half* res_lo;
  // Pre-norm fold (PreNorm(GroupNorm(1, C)) in front of a bias-free 1x1, model_utils.py:226-234, 399):
  //   W (gamma * (x - mean) * rstd + beta) = rstd * (W' x) - rstd * mean * w1 + wb,   W' = W diag(gamma),
  // W' is what the layer's packed weights hold, w1[c] = sum_k W'[c,k], wb[c] = sum_k W[c,k] beta[k].
  // (mean, rstd) of an input image come from the partial sums its producer emitted (GnFuse::emit layout).
  const float2* pre_stats;   // [img][pre_parts] or nullptr
  int pre_parts;
  float pre_inv_cnt;         // 1 / (H*W * Cin)
  const float* pre_w1;       // [n_total]
  const float* pre_wb;       // [n_total]
};

struct ConvParams {
  CUtensorMap amap[kMaxAMaps];
  int n_amaps;
  CUtensorMap bmap;     // weight box of the kernel's tile width (BN rows)
  CUtensorMap omap[4];  // one per output parity class when n_par == 4, else omap[0]
  CUtensorMap rmap;     // residual tensor (output geometry), EPI == 4 with gn.has_res
  GnFuse gn;            // EPI == 4
  const float* bias;  // [n_total] or nullptr
  // Sub-pixel ("parity") decomposition of nearest-x2-upsample + conv3x3 (HardUpsample,
  // model_utils.py:161-165): n_par == 4 makes n_tile enumerate (parity, channel tile); parity
  // (py, px) shifts every tap by (+py, +px), reads weight rows parity * n_per_par + ..., and
  // stores through omap[parity] (the stride-2 sub-lattice of the 2H x 2W output).
  int bf16;           // operands and the stored output are bf16 instead of fp16 (plain / GroupNorm-fused epilogues)
  int n_par;          // 1 or 4
  int n_tiles_par;    // channel tiles per parity (== n_tiles when n_par == 1)
  int src_w, src_hw;  // n_par == 4: width / pixels of one SOURCE image (out_lo addressing)
  // Optional epilogue extras (template encoder: folded BatchNorm = bias, ReLU, residual add and
  // fp32-accurate activations stored as an fp16 (hi, lo) pair).  All [pixel][n_total] row-major;
  // not available together with n_par == 4.
  int relu;
  const __half* res_hi;   // residual, high halves (nullptr: none)
  const __half* res_lo;   // residual, low halves (nullptr: residual is a single fp16 tensor)
  __half* out_lo;         // low halves of the output (omap receives the high halves)
  float* out_f32;         // fp32 output instead of the fp16 TMA store
  // GEGLU epilogue (ldm/attention.py:44-51; clustered kernel, BN = 128 only): every 128-column tile
  // holds 64 "x" channels followed by their 64 "gate" channels (rows permuted on the host);
  // the epilogue stores x * gelu(gate) as 64 fp16 channels at channel (n_tile * 64) of omap.
  int geglu;
  // optional GroupNorm partial statistics of the fp32 outputs (bias included), written
  // deterministically as stats[(img * parts + part) * n_oct + octet] = (sum, sum of squares)
  // over 32-pixel row segments x 8-channel octets; parts = max(1, H*W/32).
  float2* stats;
  int stats_hw;       // H*W of one output image
  int stats_noct;     // n_total / 8
  int n_total;        // output channels (row stride of res_* / out_lo / out_f32)
  int m_valid;        // n_img * H * W (rows beyond it are padding)
  int nseg;
  int ksteps;         // sum of nchunks
  int m_tiles, n_tiles;
  int tiles_per_img;  // H*W/128 when H*W >= 128, else 0
  int h_cnt, b_cnt;   // box rows per tile / images per tile
  ConvSeg seg[kMaxSeg];
};

__device__ __forceinline__ void conv_tile_coords(const ConvParams& p, int m_tile, int& b0,
                                                 int& y0) {
  if (p.tiles_per_img > 0) {
    b0 = m_tile / p.tiles_per_img;
    y0 = (m_tile - b0 * p.tiles_per_img) * p.h_cnt;
  } else {
    b0 = m_tile * p.b_cnt;
    y0 = 0;
  }
}

// Row stride (floats) of the fp32 accumulator tile in shared memory: 4 floats of padding keep the
// row-per-lane 16-byte reads of the epilogue free of bank conflicts.
__host__ __device__ constexpr int acc_ld(int BN) { return BN + 4; }

// Warps of a conv CTA that run the wgmma mainloop when NW warpgroups share a tile: two warpgroups split the tile by
// rows, a single one takes both row halves.  With NW == 3 the third warpgroup only joins the epilogue.
__host__ __device__ constexpr int conv_mma_warps(int NW) { return NW < 2 ? 4 * NW : 8; }

// K loop of one tile for one warpgroup: per 16-deep K step, NH m64nNk16 wgmmas, one per 64-row block of A starting at
// row block a_blk, each against the stage's whole N-row weight tile.  One wgmma group stays in flight while the
// previous stage is released.  The operand type is a template parameter, so the loop is one straight wgmma pipeline.
template <int N, int NH, int STAGES, int kStageBytes, int kABytes, bool BF>
__device__ __forceinline__ void conv_mma_loop(const ConvParams& p, const uint8_t* smem, uint64_t* full_bar,
                                              uint64_t* empty_bar, int& stage, uint32_t& phase, int a_blk,
                                              float (&d)[NH][N / 2]) {
  const int lane = threadIdx.x & 31;
  int prev = -1;
  for (int ks = 0; ks < p.ksteps; ++ks) {
    mbar_wait(&full_bar[stage], phase);
    const uint8_t* sa = smem + stage * kStageBytes;
    const uint64_t adesc = wg_desc_k(sa + a_blk * (64 * 128));
    const uint64_t bdesc = wg_desc_k(sa + kABytes);
    wgmma_fence();
#pragma unroll
    for (int k = 0; k < kBK / 16; ++k) {
      // advance 16 elements (32 B) along K inside the swizzle atom: +2 in the >>4 field; the next 64 rows are 8 KB on
      const uint32_t acc = (ks | k) != 0 ? 1u : 0u;
#pragma unroll
      for (int h = 0; h < NH; ++h) Wgmma<N, BF>::mma(d[h], adesc + 512 * h + 2 * k, bdesc + 2 * k, acc);
    }
    wgmma_commit();
    wgmma_wait<1>();            // the previous K-step's group has retired: its stage may be refilled
    if (prev >= 0 && lane == 0) mbar_arrive(&empty_bar[prev]);
    prev = stage;
    if (++stage == STAGES) { stage = 0; phase ^= 1; }
  }
  wgmma_wait<0>();
  if (prev >= 0 && lane == 0) mbar_arrive(&empty_bar[prev]);
}

// Mainloop of one 128 x BN tile, run by the NW warpgroups of threads [128, 128 + 128 NW).  With NW >= 2, warpgroup
// w in {0, 1} accumulates rows [64 w, 64 w + 64) x all BN columns in registers, one m64nBNk16 wgmma per 16-deep K
// step: per K step the tile's operands are read from shared memory once (A) and twice (B), where a split by
// columns reads A once per warpgroup and B once per row half.  With NW == 1 the warpgroup takes both row halves.
// The tile is then written as fp32 to s_acc, the front of the operand ring, in the [128][acc_ld(BN)] layout every
// epilogue reads.  The ring is idle by then (every stage of this tile has been consumed) and the producer refills it
// only after the epilogue has read the tile back (tempty barrier), so accumulator and operands share the memory.
template <int BN, int NW, int STAGES, int kStageBytes, int kABytes, bool MMA = true>
__device__ __forceinline__ void conv_mma_tile(const ConvParams& p, uint8_t* smem, uint64_t* full_bar,
                                              uint64_t* empty_bar, int& stage, uint32_t& phase, float* s_acc) {
  static_assert(NW >= 1 && NW <= 3 && BN % 64 == 0 && BN <= 256, "mainloop warpgroups / tile width");
  constexpr int NH = NW >= 2 ? 1 : 2;       // 64-row blocks per mainloop warpgroup
  const int wg = (threadIdx.x >> 7) - 1;
  static_assert(MMA || NW == 3, "only the third of three warpgroups skips the mainloop");
  if constexpr (MMA) {                      // NW == 3: warpgroup 2 (MMA = false) waits for the tile at the barriers
    float d[NH][BN / 2];
#pragma unroll
    for (int h = 0; h < NH; ++h)
#pragma unroll
      for (int i = 0; i < BN / 2; ++i) d[h][i] = 0.f;
    if (p.bf16) conv_mma_loop<BN, NH, STAGES, kStageBytes, kABytes, true>(p, smem, full_bar, empty_bar, stage, phase, wg, d);
    else conv_mma_loop<BN, NH, STAGES, kStageBytes, kABytes, false>(p, smem, full_bar, empty_bar, stage, phase, wg, d);
    asm volatile("barrier.sync 2, %0;" ::"n"(NW * 128) : "memory");    // no warpgroup still reads the ring
#pragma unroll
    for (int h = 0; h < NH; ++h) wg_store_acc64<BN>(s_acc, acc_ld(BN), 64 * (wg + h), d[h]);
  } else {
    asm volatile("barrier.sync 2, %0;" ::"n"(NW * 128) : "memory");
  }
  asm volatile("barrier.sync 2, %0;" ::"n"(NW * 128) : "memory");
}

// The epilogue has read the accumulator tile out of the ring: order its generic-proxy accesses before the
// producer's next TMA writes, then release the ring (one arrive per epilogue warp).
__device__ __forceinline__ void acc_release(uint64_t* tempty, int lane) {
  fence_proxy_async_smem();
  __syncwarp();
  if (lane == 0) mbar_arrive(tempty);
}

// Transposing butterfly: every lane holds 8 partial values; afterwards v[0] of lane l is the
// total over the kSeg lanes of its segment of value number `idx` (returned).  8+4+2(+1)
// shuffles instead of 8 x log2(kSeg); fixed combination order, so results are deterministic.
template <int kSeg>
__device__ __forceinline__ int butterfly8(float (&v)[8], int lane) {
  static_assert(kSeg == 16 || kSeg == 32, "segment must be 16 or 32 lanes");
  constexpr int m0 = kSeg / 2, m1 = kSeg / 4, m2 = kSeg / 8;
  {
    const bool up = (lane & m0) != 0;
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const float send = up ? v[i] : v[i + 4];
      const float keep = up ? v[i + 4] : v[i];
      v[i] = keep + __shfl_xor_sync(0xffffffffu, send, m0);
    }
  }
  {
    const bool up = (lane & m1) != 0;
#pragma unroll
    for (int i = 0; i < 2; ++i) {
      const float send = up ? v[i] : v[i + 2];
      const float keep = up ? v[i + 2] : v[i];
      v[i] = keep + __shfl_xor_sync(0xffffffffu, send, m1);
    }
  }
  {
    const bool up = (lane & m2) != 0;
    const float send = up ? v[0] : v[1];
    const float keep = up ? v[1] : v[0];
    v[0] = keep + __shfl_xor_sync(0xffffffffu, send, m2);
  }
#pragma unroll
  for (int m = m2 / 2; m > 0; m >>= 1) v[0] += __shfl_xor_sync(0xffffffffu, v[0], m);
  return ((lane & m0) ? 4 : 0) + ((lane & m1) ? 2 : 0) + ((lane & m2) ? 1 : 0);
}

// Epilogue of one 128 x BN accumulator tile, executed by the 8 epilogue warps of a CTA.
// Warp e reads accumulator rows 32*(e&3).. (its pixel rows) and the 32-column half (e>>2) of every
// 64-column sub-tile: +bias (from smem) -> GroupNorm partial sums -> fp16 -> swizzled staging.
// EXTRAS (compile time) enables ReLU / residual add / (hi, lo) split / fp32 output: the epilogue of
// the template encoder and of the LDM output convolution (clustered kernel only).  The sweep
// instantiates EXTRAS = false so its epilogue stays minimal (the extra predicates and registers
// cost ~10 % on the large convolutions when merely present).
// Residual operands (high halves) of a tile, software-pipelined ONE TILE AHEAD by the epilogue
// warps: while sub-tile cc of tile i is being combined, the loads of sub-tile cc of tile i+1 are
// already in flight (into the registers that sub-tile just vacated).  With the loads issued next to
// their use, their ~1-2 us latency sat in front of every tile of the short-K 1x1 layers.
template <int BN>
struct ResPrefetch {
  uint4 v[BN / 64][4];
  int next_m_tile, next_n_chan0;    // tile whose operands are fetched next; next_m_tile < 0: none
  __device__ __forceinline__ void load_sub(const ConvParams& p, int cc, int m_tile, int n_chan0, int e, int lane) {
    const int q = e & 3, hh = e >> 2;
    const int grow = m_tile * kBM + q * 32 + lane;
    if (p.res_hi && m_tile >= 0 && grow < p.m_valid) {
      const size_t roff = (size_t)grow * p.n_total + n_chan0 + cc * 64 + hh * 32;
#pragma unroll
      for (int j = 0; j < 4; ++j) v[cc][j] = *reinterpret_cast<const uint4*>(p.res_hi + roff + j * 8);
    }
  }
  __device__ __forceinline__ void load(const ConvParams& p, int m_tile, int n_chan0, int e, int lane) {
#pragma unroll
    for (int cc = 0; cc < BN / 64; ++cc) load_sub(p, cc, m_tile, n_chan0, e, lane);
  }
};

template <int BN, bool EXTRAS>
__device__ __forceinline__ void conv_epilogue_tile(const ConvParams& p, uint8_t* out_stage,
                                                   const float* s_bias, const float* s_acc, int m_tile,
                                                   int n_chan0, int e, int lane,
                                                   ResPrefetch<BN>* pre = nullptr, int par = 0) {
  const int q = e & 3, hh = e >> 2;
  const int row = q * 32 + lane;
  const float* a_row = s_acc + row * acc_ld(BN) + hh * 32;
  const int grow = m_tile * kBM + row;                                // linear pixel index
  const bool row_ok = grow < p.m_valid;
  size_t opix = (size_t)grow;                                         // output pixel (EXTRAS stores)
  if (EXTRAS && p.n_par == 4) {       // parity class (py, px) of the 2H x 2W output
    const int img = grow / p.src_hw, r = grow - img * p.src_hw;
    const int yy = r / p.src_w, xx = r - yy * p.src_w;
    opix = (size_t)img * 4 * p.src_hw + (size_t)(2 * yy + (par >> 1)) * (2 * p.src_w) + 2 * xx + (par & 1);
  }
  uint32_t v[32];
#pragma unroll
  for (int cc = 0; cc < BN / 64; ++cc) {
    acc_ld_32(a_row + cc * 64, v);
    const float* bs = s_bias + cc * 64 + hh * 32;
    uint8_t* srow = out_stage + cc * (kBM * 128) + row * 128;
    // residual operands of this sub-tile: all loads issued before the math
    uint4 rh[4], rl[4];
    if (EXTRAS && p.res_hi && row_ok) {
      const size_t roff = (size_t)grow * p.n_total + n_chan0 + cc * 64 + hh * 32;
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        rh[j] = pre ? pre->v[cc][j] : *reinterpret_cast<const uint4*>(p.res_hi + roff + j * 8);
        rl[j] = p.res_lo ? *reinterpret_cast<const uint4*>(p.res_lo + roff + j * 8) : make_uint4(0, 0, 0, 0);
      }
    }
    if (EXTRAS && pre) pre->load_sub(p, cc, pre->next_m_tile, pre->next_n_chan0, e, lane);   // next tile, same sub-tile
    float st[8];
#pragma unroll
    for (int j = 0; j < 4; ++j) {   // 4 x 16-byte chunks of 8 channels
      const float4 b0 = *reinterpret_cast<const float4*>(bs + j * 8);
      const float4 b1 = *reinterpret_cast<const float4*>(bs + j * 8 + 4);
      float f[8];
      f[0] = __uint_as_float(v[j * 8 + 0]) + b0.x;
      f[1] = __uint_as_float(v[j * 8 + 1]) + b0.y;
      f[2] = __uint_as_float(v[j * 8 + 2]) + b0.z;
      f[3] = __uint_as_float(v[j * 8 + 3]) + b0.w;
      f[4] = __uint_as_float(v[j * 8 + 4]) + b1.x;
      f[5] = __uint_as_float(v[j * 8 + 5]) + b1.y;
      f[6] = __uint_as_float(v[j * 8 + 6]) + b1.z;
      f[7] = __uint_as_float(v[j * 8 + 7]) + b1.w;
      if (EXTRAS) {
        const size_t goff = opix * p.n_total + n_chan0 + cc * 64 + hh * 32 + j * 8;
        if (p.res_hi && row_ok) {
          const __half2* h2 = reinterpret_cast<const __half2*>(&rh[j]);
          const __half2* l2 = reinterpret_cast<const __half2*>(&rl[j]);
#pragma unroll
          for (int q = 0; q < 4; ++q) {
            const float2 th = __half22float2(h2[q]), tl = __half22float2(l2[q]);
            f[2 * q] += th.x + tl.x;
            f[2 * q + 1] += th.y + tl.y;
          }
        }
        if (p.relu) {
#pragma unroll
          for (int i = 0; i < 8; ++i) f[i] = fmaxf(f[i], 0.f);
        }
        if (p.out_f32 && row_ok) {
          *reinterpret_cast<float4*>(p.out_f32 + goff) = make_float4(f[0], f[1], f[2], f[3]);
          *reinterpret_cast<float4*>(p.out_f32 + goff + 4) = make_float4(f[4], f[5], f[6], f[7]);
        }
        if (p.out_lo && row_ok) {
          float l[8];
#pragma unroll
          for (int i = 0; i < 8; ++i) l[i] = f[i] - __half2float(__float2half_rn(f[i]));
          *reinterpret_cast<uint4*>(p.out_lo + goff) =
              make_uint4(pack_half2(l[0], l[1]), pack_half2(l[2], l[3]), pack_half2(l[4], l[5]),
                         pack_half2(l[6], l[7]));
        }
      }
      float s = (f[0] + f[1]) + (f[2] + f[3]) + ((f[4] + f[5]) + (f[6] + f[7]));
      float q2 = f[0] * f[0];
#pragma unroll
      for (int i = 1; i < 8; ++i) q2 = fmaf(f[i], f[i], q2);
      st[2 * j] = s;
      st[2 * j + 1] = q2;
      const int phys = (hh * 4 + j) ^ (row & 7);   // SWIZZLE_128B: chunk index XOR (row mod 8)
      const bool bf = p.bf16 != 0;
      *reinterpret_cast<uint4*>(srow + phys * 16) =
          make_uint4(pack2(f[0], f[1], bf), pack2(f[2], f[3], bf), pack2(f[4], f[5], bf), pack2(f[6], f[7], bf));
    }
    if (p.stats) {
      const bool small = p.stats_hw < 32;            // 4x4 images: two per warp
      const int idx = small ? butterfly8<16>(st, lane) : butterfly8<32>(st, lane);
      const int seg = small ? 16 : 32;
      const int gp = m_tile * kBM + (row & ~(seg - 1));
      const bool writer = small ? ((lane & 1) == 0) : ((lane & 3) == 0);
      if (writer && gp < p.m_valid) {
        const int img = gp / p.stats_hw;
        const int parts = small ? 1 : p.stats_hw >> 5;
        const int part = small ? 0 : (gp - img * p.stats_hw) >> 5;
        float* dst = reinterpret_cast<float*>(p.stats + ((size_t)img * parts + part) * p.stats_noct +
                                              (n_chan0 + cc * 64 + hh * 32) / 8);
        dst[idx] = st[0];                            // idx = octet * 2 + {sum, sum of squares}
      }
    }
  }
}

// x * Phi(x), Phi from erf by Abramowitz-Stegun 7.1.26 (|error| <= 1.5e-7, far below the fp16
// rounding of the result): one MUFU.RCP + one MUFU.EX2 + 8 FMA-pipe instructions instead of
// erff's ~30 -- the GEGLU epilogue is bound by exactly this.
__device__ __forceinline__ float gelu_erf_fast(float g) {
  const float z = fabsf(g) * 0.70710678118654752f;
  const float t = __fdividef(1.f, fmaf(0.3275911f, z, 1.f));
  float poly = fmaf(t, 1.061405429f, -1.453152027f);
  poly = fmaf(poly, t, 1.421413741f);
  poly = fmaf(poly, t, -0.284496736f);
  poly = fmaf(poly, t, 0.254829592f);
  poly *= t;
  float e;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(e) : "f"(-z * z * 1.4426950408889634f));
  const float erf_abs = fmaf(-poly, e, 1.f);                 // erf(|g| / sqrt 2)
  const float phi = 0.5f * (1.f + copysignf(erf_abs, g));
  return g * phi;
}

// GEGLU epilogue of one 128 x 128 accumulator tile: columns 0..63 = x, 64..127 = gate.
// Warp e owns pixel rows 32*(e&3).. and the 32-column half (e>>2) of BOTH halves, so
// x * gelu(gate) needs no exchange.  erf-GELU (F.gelu's default) through gelu_erf_fast.
__device__ __forceinline__ void conv_epilogue_geglu(uint8_t* out_stage, const float* s_bias, const float* s_acc,
                                                    int e, int lane) {
  const int q = e & 3, hh = e >> 2;
  const int row = q * 32 + lane;
  const float* a_row = s_acc + row * acc_ld(128) + hh * 32;
  uint32_t vx[32], vg[32];
  acc_ld_32(a_row, vx);
  acc_ld_32(a_row + 64, vg);
  const float* bx = s_bias + hh * 32;
  const float* bg = s_bias + 64 + hh * 32;
  uint8_t* srow = out_stage + row * 128;
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    float f[8];
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      const float x = __uint_as_float(vx[j * 8 + i]) + bx[j * 8 + i];
      const float g = __uint_as_float(vg[j * 8 + i]) + bg[j * 8 + i];
      f[i] = x * gelu_erf_fast(g);
    }
    const int phys = (hh * 4 + j) ^ (row & 7);
    *reinterpret_cast<uint4*>(srow + phys * 16) =
        make_uint4(pack_half2(f[0], f[1]), pack_half2(f[2], f[3]), pack_half2(f[4], f[5]),
                   pack_half2(f[6], f[7]));
  }
}

// ----------------------------------------------------------------------------
// host side: tensor maps + launch
// ----------------------------------------------------------------------------
inline PFN_cuTensorMapEncodeTiled_v12000 get_encode_fn() {
  static PFN_cuTensorMapEncodeTiled_v12000 fn = nullptr;
  if (!fn) {
    void* ptr = nullptr;
    cudaDriverEntryPointQueryResult qres;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &ptr, cudaEnableDefault, &qres) ==
            cudaSuccess &&
        qres == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<PFN_cuTensorMapEncodeTiled_v12000>(ptr);
  }
  return fn;
}

// fp16 tensor map, rank 2..4, 128-byte swizzle, zero fill out of bounds.
// dims/box are innermost-first; strides_bytes[i] is the byte stride of dim i+1.
inline int make_tmap_f16(CUtensorMap* out, const void* base, int rank, const uint64_t* dims,
                         const uint64_t* strides_bytes, const uint32_t* box) {
  auto fn = get_encode_fn();
  if (!fn) return fail("cuTensorMapEncodeTiled driver entry point not available");
  cuuint64_t gdim[5], gstr[5];
  cuuint32_t bx[5], es[5];
  for (int i = 0; i < rank; ++i) { gdim[i] = dims[i]; bx[i] = box[i]; es[i] = 1; }
  for (int i = 0; i < rank - 1; ++i) gstr[i] = strides_bytes[i];
  CUresult r = fn(out, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, rank, const_cast<void*>(base), gdim, gstr,
                  bx, es, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B,
                  CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    char buf[256];
    snprintf(buf, sizeof buf,
             "cuTensorMapEncodeTiled failed (%d): rank %d dims [%llu %llu %llu %llu] box [%u %u %u %u]",
             (int)r, rank, (unsigned long long)dims[0], (unsigned long long)(rank > 1 ? dims[1] : 0),
             (unsigned long long)(rank > 2 ? dims[2] : 0), (unsigned long long)(rank > 3 ? dims[3] : 0),
             box[0], rank > 1 ? box[1] : 0, rank > 2 ? box[2] : 0, rank > 3 ? box[3] : 0);
    return fail(buf);
  }
  return 0;
}

// Tile geometry of an NHWC tensor with H x W pixels per image: 128 pixels per tile.
struct TileGeom {
  int W, H, w_cnt, h_cnt, b_cnt, tiles_per_img;
};
inline int make_geom(int H, int W, TileGeom* g) {
  g->W = W; g->H = H; g->w_cnt = W;
  if (W > kBM || kBM % W != 0) return fail("conv geometry: W must divide 128");
  const int hw = H * W;
  if (hw >= kBM) {
    if (hw % kBM != 0) return fail("conv geometry: H*W must be a multiple of 128");
    g->h_cnt = kBM / W; g->b_cnt = 1; g->tiles_per_img = hw / kBM;
  } else {
    if (kBM % hw != 0) return fail("conv geometry: H*W must divide 128");
    g->h_cnt = H; g->b_cnt = kBM / hw; g->tiles_per_img = 0;
  }
  return 0;
}
inline int geom_m_tiles(const TileGeom& g, int n_img) {
  return g.tiles_per_img > 0 ? n_img * g.tiles_per_img : (n_img + g.b_cnt - 1) / g.b_cnt;
}

// NHWC activation map [B, H, W, C] (contiguous), box = one 128-pixel tile x 64 channels.
inline int make_act_map(CUtensorMap* m, const void* base, int cap_img, int C, const TileGeom& g) {
  uint64_t dims[4] = {(uint64_t)C, (uint64_t)g.W, (uint64_t)g.H, (uint64_t)cap_img};
  uint64_t str[3] = {(uint64_t)C * 2, (uint64_t)g.W * C * 2, (uint64_t)g.H * g.W * C * 2};
  uint32_t box[4] = {64, (uint32_t)g.w_cnt, (uint32_t)g.h_cnt, (uint32_t)g.b_cnt};
  return make_tmap_f16(m, base, 4, dims, str, box);
}
// Stride-2 sub-lattice (p1, p2) of an NHWC tensor with 2H x 2W pixels: the input of a
// pixel-unshuffle + 1x1 conv seen from the H x W output geometry `g`.
inline int make_unshuffle_map(CUtensorMap* m, const void* base, int cap_img, int C,
                              const TileGeom& g, int p1, int p2) {
  const int W2 = g.W * 2, H2 = g.H * 2;
  const uint8_t* b = static_cast<const uint8_t*>(base) + ((size_t)p1 * W2 + p2) * C * 2;
  uint64_t dims[4] = {(uint64_t)C, (uint64_t)g.W, (uint64_t)g.H, (uint64_t)cap_img};
  uint64_t str[3] = {(uint64_t)2 * C * 2, (uint64_t)2 * W2 * C * 2, (uint64_t)H2 * W2 * C * 2};
  uint32_t box[4] = {64, (uint32_t)g.w_cnt, (uint32_t)g.h_cnt, (uint32_t)g.b_cnt};
  return make_tmap_f16(m, b, 4, dims, str, box);
}
// Packed weights [n_total, k_total] fp16, K-major.
inline int make_weight_map(CUtensorMap* m, const void* base, int n_total, int k_total, int bn) {
  uint64_t dims[2] = {(uint64_t)k_total, (uint64_t)n_total};
  uint64_t str[1] = {(uint64_t)k_total * 2};
  uint32_t box[2] = {64, (uint32_t)bn};
  return make_tmap_f16(m, base, 2, dims, str, box);
}
// 3-D fp16 tensor map with 128-byte swizzle (the LDM attention's operands).
inline int make_tmap3_f16(CUtensorMap* m, const void* base, uint64_t d0, uint64_t d1, uint64_t d2,
                          uint32_t b0, uint32_t b1) {
  uint64_t dims[3] = {d0, d1, d2};
  uint64_t str[2] = {d0 * 2, d0 * d1 * 2};
  uint32_t box[3] = {b0, b1, 1};
  return make_tmap_f16(m, base, 3, dims, str, box);
}

inline int pick_bn(int n_total) {
  if (n_total % 192 == 0) return 192;
  if (n_total % 128 == 0) return 128;
  if (n_total % 64 == 0) return 64;
  return 0;
}

inline bool conv_needs_extras(const ConvParams& p) {
  return p.relu || p.res_hi || p.out_lo || p.out_f32;
}

// Tensor maps of activation buffers, encoded once per (base, image capacity, lattice, C, H, W).  lattice < 0: the
// plain NHWC map of geometry g (make_act_map); 0..3: the stride-2 sub-lattice (lattice >> 1, lattice & 1) of a
// 2H x 2W tensor seen from g (make_unshuffle_map).  get3: the 3-D maps of make_tmap3_f16, once per (base, dims).
// Call clear() whenever the buffers are reallocated.
class TmapCache {
 public:
  int get(const CUtensorMap** out, const void* base, int cap_img, int C, const TileGeom& g, int lattice) {
    const auto key = std::make_tuple(base, cap_img, lattice, C, g.H, g.W);
    auto it = maps_.find(key);
    if (it == maps_.end()) {
      CUtensorMap m;
      const int rc = lattice < 0 ? make_act_map(&m, base, cap_img, C, g)
                                 : make_unshuffle_map(&m, base, cap_img, C, g, lattice >> 1, lattice & 1);
      if (rc) return -1;
      it = maps_.emplace(key, m).first;
    }
    *out = &it->second;
    return 0;
  }
  int get3(const CUtensorMap** out, const void* base, int d0, int d1, int d2, int b0, int b1) {
    const auto key = std::make_tuple(base, d0, d1, d2);
    auto it = maps3_.find(key);
    if (it == maps3_.end()) {
      CUtensorMap m;
      if (make_tmap3_f16(&m, base, d0, d1, d2, b0, b1)) return -1;
      it = maps3_.emplace(key, m).first;
    }
    *out = &it->second;
    return 0;
  }
  void clear() { maps_.clear(); maps3_.clear(); }

 private:
  std::map<std::tuple<const void*, int, int, int, int, int>, CUtensorMap> maps_;
  std::map<std::tuple<const void*, int, int, int>, CUtensorMap> maps3_;
};

// One filter tap: activation lattice (0 for a plain map) and pixel offset.
struct ConvTap {
  int lat, dy, dx;
};
// Tap (oy, ox) of a stride-2 convolution seen from its output geometry: input pixel (2y + oy, 2x + ox) lies on the
// stride-2 sub-lattice (oy & 1, ox & 1) at offset ((oy - (oy & 1)) / 2, (ox - (ox & 1)) / 2).  Pixel-unshuffle +
// 1x1 is the case oy, ox in {0, 1}.
inline ConvTap stride2_tap(int oy, int ox) {
  const int p1 = oy & 1, p2 = ox & 1;
  return ConvTap{p1 * 2 + p2, (oy - p1) / 2, (ox - p2) / 2};
}
// The k x k taps, row-major, of a convolution whose first tap reads input pixel (y + oy0, x + ox0) at stride 1 or
// (2y + oy0, 2x + ox0) at stride 2.
inline std::vector<ConvTap> conv_taps(int k, int stride, int oy0, int ox0) {
  std::vector<ConvTap> taps;
  for (int ky = 0; ky < k; ++ky)
    for (int kx = 0; kx < k; ++kx)
      taps.push_back(stride == 1 ? ConvTap{0, oy0 + ky, ox0 + kx} : stride2_tap(oy0 + ky, ox0 + kx));
  return taps;
}

// A convolution layer of any engine.  Its weights are K-major fp16 rows, one per output channel (cout is padded to a
// multiple of 64 with zero rows; the folded upsample has 4 cout rows, parity * cout + o): [W_hi (K) | W_lo (K)] when
// the layer has a W_lo plane (the fp16 remainders W - fp16(W)), W_hi alone otherwise (bf16 in the UNet's bf16 mode).
// The K columns of a plane are (tap, input channel) over the layer's taps, then any extra columns: a 1x1 shortcut or
// skip, an identity residual.
struct ConvLayer {
  int cin = 0, cout = 0, K = 0, bn = 0;
  bool wlo = false;                          // a W_lo plane follows at column K
  int k = 1, stride = 1, oy0 = 0, ox0 = 0;   // the taps: conv_taps(k, stride, oy0, ox0)
  bool up = false;                           // nearest-x2 upsample + 3x3 folded into four 2x2 parity kernels (n_par 4)
  __half* w = nullptr;
  float* bias = nullptr;                     // [cout] or nullptr
  CUtensorMap wmap;                          // weight box of bn rows
  // UNet: pre-norm folded into this (bias-free 1x1) layer: weights hold W diag(gamma); see GnFuse::pre_*
  float* pre_w1 = nullptr;
  float* pre_wb = nullptr;
  // LDM
  int skip_c = 0;        // channels of a folded 1x1 skip_connection / identity residual (extra K columns)
  int k_alg = 0;         // K without identity-residual columns (algorithmic FLOP count)
  bool geglu = false;    // rows permuted to (64 x | 64 gate) tiles; the epilogue emits x * gelu(gate)

  int rows() const { return up ? 4 * cout : cout; }
  int row_len() const { return wlo ? 2 * K : K; }
  std::vector<ConvTap> taps() const { return conv_taps(k, stride, oy0, ox0); }
};
// A layer of the given taps (conv_taps) and upsample fold, its other fields unset.
inline ConvLayer conv_shape(int k, int stride, int oy0, int ox0, bool up = false) {
  ConvLayer L;
  L.k = k;
  L.stride = stride;
  L.oy0 = oy0;
  L.ox0 = ox0;
  L.up = up;
  return L;
}
// The shapes the UNet and LDM engines share: 3x3 pad 1, 1x1, pixel-unshuffle + 1x1 (HardDownsample: a 2x2 stride-2
// convolution), nearest-x2 upsample + 3x3 folded into 2x2 kernels over the source, 3x3 stride 2 pad 1.
inline ConvLayer conv3x3() { return conv_shape(3, 1, -1, -1); }
inline ConvLayer conv1x1() { return conv_shape(1, 1, 0, 0); }
inline ConvLayer conv_unshuffle() { return conv_shape(2, 2, 0, 0); }
inline ConvLayer conv_upsample3x3() { return conv_shape(2, 1, -1, -1, true); }
inline ConvLayer conv3x3_s2() { return conv_shape(3, 2, -1, -1); }

// One input of a convolution as its K segments read it: its channels and the maps of its hi and lo halves for each
// lattice a tap names (lo[0] < 0: the input carries no lo).
struct ConvSrc {
  int C = 0;
  int hi[4] = {0, 0, 0, 0};
  int lo[4] = {-1, -1, -1, -1};
};

// Builds the ConvParams of one launch.  The engine adds its activation maps and, in its accumulation order, the
// K segments, then sets its epilogue fields around finish(), which fills everything that follows from the geometry,
// the layer and the output.  A map that cannot be encoded or a segment past kMaxSeg is remembered and returned by
// finish(), so no launch is made from a half-built block.
struct ConvBuilder {
  ConvParams p;
  TmapCache& maps;
  const TileGeom g;      // tile geometry: the output's, the source's for the folded upsample
  const int cap_img;     // images the activation buffers hold
  int err = 0;

  ConvBuilder(TmapCache& m, const TileGeom& geom, int cap) : maps(m), g(geom), cap_img(cap) {
    memset(&p, 0, sizeof p);
  }
  // appends the map of `base` (lattice as TmapCache::get) and returns its index
  int map(const void* base, int C, int lattice = -1) {
    const CUtensorMap* m = nullptr;
    if (p.n_amaps >= kMaxAMaps) err = fail("conv: activation map table overflow");
    else if (maps.get(&m, base, cap_img, C, g, lattice)) err = -1;
    if (err) return 0;
    p.amap[p.n_amaps] = *m;
    return p.n_amaps++;
  }
  // the input (hi, lo) of C channels (lo == nullptr: none): its plain map, or with lattices == 4 its four stride-2
  // sub-lattices
  ConvSrc src(const void* hi, const void* lo, int C, int lattices = 1) {
    ConvSrc s;
    s.C = C;
    for (int l = 0; l < lattices; ++l) s.hi[l] = map(hi, C, lattices == 4 ? l : -1);
    if (lo)
      for (int l = 0; l < lattices; ++l) s.lo[l] = map(lo, C, lattices == 4 ? l : -1);
    return s;
  }
  // appends a segment of nch 64-channel chunks (wcol1 as ConvSeg::wcol1)
  void seg(int map, int dy, int dx, int nch, int wcol1 = 0) {
    if (p.nseg >= kMaxSeg) {
      err = fail("conv: segment table overflow");
      return;
    }
    p.seg[p.nseg++] = ConvSeg{(int16_t)map, (int16_t)dy, (int16_t)dx, (int16_t)nch, wcol1};
    p.ksteps += nch;
  }
  // Appends the K segments of `taps` over the inputs `src` (a tap's lat picks each input's maps), whose W_hi columns
  // start at `col` in (tap, input, channel) order, and returns the column after them.  Per tap, over its inputs:
  // A_hi W_hi, then A_hi W_lo from the W_lo plane at column wlo_col (0: no W_lo plane), then A_lo W_hi for the inputs
  // that carry lo.
  int segs(const std::vector<ConvTap>& taps, const std::vector<ConvSrc>& src, int col, int wlo_col) {
    for (const ConvTap& t : taps) {
      int c = col;
      for (const ConvSrc& s : src) {
        seg(s.hi[t.lat], t.dy, t.dx, s.C / 64, c + 1);
        c += s.C;
      }
      if (wlo_col) {
        c = col;
        for (const ConvSrc& s : src) {
          seg(s.hi[t.lat], t.dy, t.dx, s.C / 64, wlo_col + c + 1);
          c += s.C;
        }
      }
      c = col;
      for (const ConvSrc& s : src) {
        if (s.lo[0] >= 0) seg(s.lo[t.lat], t.dy, t.dx, s.C / 64, c + 1);
        c += s.C;
      }
      col = c;
    }
    return col;
  }
  // n_par == 4: the folded upsample, whose output `out` (out_C channels) has 2H x 2W pixels and is stored through
  // its four parity sub-lattices
  int finish(const ConvLayer& L, const void* out, int out_C, int n_img, int n_par) {
    if (err) return err;
    for (int i = p.n_amaps; i < kMaxAMaps; ++i) p.amap[i] = p.amap[0];   // never read: any valid descriptor
    p.bmap = L.wmap;
    const CUtensorMap* m = nullptr;
    for (int t = 0; t < 4; ++t) {   // n_par == 1: omap[0] is the store map, the others copies of it
      if ((t == 0 || n_par == 4) && maps.get(&m, out, cap_img, out_C, g, n_par == 4 ? t : -1)) return -1;
      p.omap[t] = *m;
    }
    p.bias = L.bias;
    p.n_par = n_par;
    p.src_w = g.W;
    p.src_hw = g.H * g.W;
    p.stats_hw = n_par * g.H * g.W;
    p.stats_noct = L.cout / 8;
    p.n_total = L.cout;
    p.m_valid = n_img * g.H * g.W;     // rows of the GEMM (source pixels for the folded upsample)
    p.m_tiles = geom_m_tiles(g, n_img);
    p.n_tiles_par = L.cout / L.bn;
    p.n_tiles = p.n_tiles_par * n_par;
    p.tiles_per_img = g.tiles_per_img;
    p.h_cnt = g.h_cnt;
    p.b_cnt = g.b_cnt;
    return 0;
  }
};

}  // namespace nope
