// nope_b200 -- template encoder on the wgmma convolution kernel, fp32-accurate.
//
// Reference: FeatureExtractor.encode_image (src/model/encoder/template.py:47-53) =
// ResNet-50 without max-pool, layer4 at stride 1 (src/model/encoder/resnet.py:93-152),
// eval-mode BatchNorm, then ReLU -> 1x1(2048->256) -> ReLU -> 1x1(256->D).
//
// The latents feed the score directly, so they must match the reference's fp32 path far
// better than fp16 (TF32 / fp16 cuDNN are 2-3e-3 off, measured).  fp32 accuracy on fp16 tensor
// cores comes from split precision: every activation and weight is an fp16 pair
// (hi = fp16(x), lo = fp16(x - hi), 22 significant bits) and each convolution accumulates the
// three products A_hi W_hi + A_hi W_lo + A_lo W_hi in the fp32 accumulator -- for the
// implicit-GEMM kernel that is simply three K-segments per filter tap over two activation
// tensor maps.  BatchNorm is folded into the weights / bias in double precision on the host;
// ReLU, the bottleneck's residual add and the (hi, lo) split of the output run in the conv
// epilogue.  Stride-2 convolutions read the four stride-2 sub-lattices of their input through
// TMA maps (same trick as HardDownsample).  65 GFLOP per image in fp32 terms, 195 executed.
//
// precision 1 (nope_encoder_set_option, DESIGN.md section 22) is the opt-in single-fp16 mode: every weight is one
// fp16 value (BatchNorm still folded in double first), every stored activation one fp16 tensor (lo = nullptr, never
// allocated, written or read), one K-segment per tap; the stem's arithmetic and the accumulation stay fp32.
#pragma once
#include "conv_tc2.cuh"
#include "engine.cuh"
#include "kernels.cuh"

#include <cmath>
#include <map>
#include <string>
#include <vector>

namespace nope {

// stem: conv 7x7 stride 2 pad 3 (3 -> 64) + folded BN + ReLU, fp32 direct, -> (hi, lo) NHWC (out_lo nullptr: hi only).
// Block = 64 output channels x 4 pixels.  w: [64][3][7][7] folded, fp32.
__global__ void __launch_bounds__(256)
enc_stem_kernel(const float* __restrict__ x, const float* __restrict__ w, const float* __restrict__ bias,
                __half* __restrict__ out_hi, __half* __restrict__ out_lo, int B, int Hin, int Win) {
  __shared__ float s_w[64 * 147];
  for (int i = threadIdx.x; i < 64 * 147; i += 256) s_w[i] = w[i];
  __syncthreads();
  const int Ho = Hin / 2, Wo = Win / 2;
  const int o = threadIdx.x & 63;
  // 32-bit pixel arithmetic (B <= 32 images of a chunk), so no 64-bit division routine is called
  const int pix = blockIdx.x * 4 + (threadIdx.x >> 6);
  if (pix >= B * Ho * Wo) return;
  const int px = pix % Wo, py = (pix / Wo) % Ho, b = pix / (Wo * Ho);
  float acc = bias[o];
  for (int c = 0; c < 3; ++c)
    for (int ky = 0; ky < 7; ++ky) {
      const int yy = 2 * py + ky - 3;
      if (yy < 0 || yy >= Hin) continue;
      const float* xr = x + (size_t)((b * 3 + c) * Hin + yy) * Win;
      const float* wr = s_w + o * 147 + (c * 7 + ky) * 7;
#pragma unroll
      for (int kx = 0; kx < 7; ++kx) {
        const int xx = 2 * px + kx - 3;
        if (xx >= 0 && xx < Win) acc = fmaf(xr[xx], wr[kx], acc);
      }
    }
  acc = fmaxf(acc, 0.f);
  const __half hi = __float2half_rn(acc);
  out_hi[(size_t)pix * 64 + o] = hi;
  if (out_lo) out_lo[(size_t)pix * 64 + o] = __float2half_rn(acc - __half2float(hi));
}

// In-plane rotation of the query crops (DESIGN.md section 11): rotated copy a of image b is
// I_a(x, y) = I(c + R2(alpha_a) ((x, y) - c)), c = ((W - 1) / 2, (H - 1) / 2), R2 = [[cos, -sin], [sin, cos]],
// bilinear, taps outside the image read -1 (black in the model's [-1, 1] range).  One thread per output pixel
// (all three channels); grid (ceil(H * W / 256), pairs): blockIdx.y is the pair p = pair0 + blockIdx.y = b * A + a,
// and out is pair-major from pair0: [pairs, 3, H, W].  32-bit index arithmetic (H * W and B * A fit an int), so
// no 64-bit division routine is called.  Every product and sum is rounded on its own, in the order
// oracle/inplane_oracle.py restates: source coordinates, floor, fractions, the two row lerps, the column lerp.  At
// quarter turns of a square image the fractions are 0 and the copy is an exact permutation.
// The per-pixel body shared by both rotation kernels: pixel i = y * W + x of the copy of image src [3, H, W] rotated
// by (c, s), written to dst[0], dst[hw], dst[2 hw].
__device__ __forceinline__ void inplane_rotate_pixel(const float* __restrict__ src, float c, float s, int H, int W,
                                                     int i, float* __restrict__ dst) {
  const long long hw = (long long)H * W;
  const int x = i % W, y = i / W;
  const float cx = __fmul_rn((float)(W - 1), 0.5f), cy = __fmul_rn((float)(H - 1), 0.5f);
  const float dx = __fsub_rn((float)x, cx), dy = __fsub_rn((float)y, cy);
  const float sx = __fadd_rn(__fsub_rn(__fmul_rn(c, dx), __fmul_rn(s, dy)), cx);
  const float sy = __fadd_rn(__fadd_rn(__fmul_rn(s, dx), __fmul_rn(c, dy)), cy);
  const float x0 = floorf(sx), y0 = floorf(sy);
  const float fx = __fsub_rn(sx, x0), fy = __fsub_rn(sy, y0);
  const int ix = (int)x0, iy = (int)y0;
  const bool in_x0 = ix >= 0 && ix < W, in_x1 = ix + 1 >= 0 && ix + 1 < W;
  const bool in_y0 = iy >= 0 && iy < H, in_y1 = iy + 1 >= 0 && iy + 1 < H;
#pragma unroll
  for (int ch = 0; ch < 3; ++ch) {
    const float* plane = src + ch * hw;
    const float v00 = in_y0 && in_x0 ? plane[(long long)iy * W + ix] : -1.f;
    const float v01 = in_y0 && in_x1 ? plane[(long long)iy * W + ix + 1] : -1.f;
    const float v10 = in_y1 && in_x0 ? plane[(long long)(iy + 1) * W + ix] : -1.f;
    const float v11 = in_y1 && in_x1 ? plane[(long long)(iy + 1) * W + ix + 1] : -1.f;
    const float top = __fadd_rn(v00, __fmul_rn(fx, __fsub_rn(v01, v00)));
    const float bot = __fadd_rn(v10, __fmul_rn(fx, __fsub_rn(v11, v10)));
    dst[ch * hw] = __fadd_rn(top, __fmul_rn(fy, __fsub_rn(bot, top)));
  }
}

__global__ void __launch_bounds__(256)
inplane_rotate_kernel(const float* __restrict__ img, const float* __restrict__ cossin, int A, int H, int W, int pair0,
                      float* __restrict__ out) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  const int hw_i = H * W;
  if (i >= hw_i) return;
  const long long hw = hw_i;
  const int p = pair0 + (int)blockIdx.y;
  const int a = p % A, b = p / A;
  inplane_rotate_pixel(img + (long long)b * 3 * hw, cossin[2 * a], cossin[2 * a + 1], H, W, i,
                       out + (long long)blockIdx.y * 3 * hw + i);
}

// Rotated copies of arbitrary (image, roll) pairs (DESIGN.md section 14): pair p = pair0 + blockIdx.y rotates image
// image_idx[p] of img [B, 3, H, W] by (cossin[2p], cossin[2p + 1]) into out [pairs, 3, H, W] (pair-major from pair0),
// with the per-pixel body of inplane_rotate_kernel, so a pair holding table entry a equals copy a bit for bit.  An
// image index outside [0, B) gives a copy that is -1 everywhere.
__global__ void __launch_bounds__(256)
inplane_rotate_pairs_kernel(const float* __restrict__ img, int B, const int* __restrict__ image_idx,
                            const float* __restrict__ cossin, int H, int W, int pair0, float* __restrict__ out) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  const int hw_i = H * W;
  if (i >= hw_i) return;
  const long long hw = hw_i;
  const int p = pair0 + (int)blockIdx.y;
  const int b = image_idx[p];
  float* dst = out + (long long)blockIdx.y * 3 * hw + i;
  if (b < 0 || b >= B) {
#pragma unroll
    for (int ch = 0; ch < 3; ++ch) dst[ch * hw] = -1.f;
    return;
  }
  inplane_rotate_pixel(img + (long long)b * 3 * hw, cossin[2 * p], cossin[2 * p + 1], H, W, i, dst);
}

// [n_pix][ld] fp32 (first D columns valid) -> NCHW fp32 [B, D, hw]
__global__ void enc_extract_kernel(const float* __restrict__ x, float* __restrict__ out, int B, int D,
                                   int hw, int ld) {
  const long long total = (long long)B * D * hw;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const int p = (int)(i % hw), d = (int)((i / hw) % D), b = (int)(i / ((long long)hw * D));
    out[i] = x[((long long)b * hw + p) * ld + d];
  }
}

struct EncConv {
  int cin = 0, cout = 0, cout_real = 0, k = 1, stride = 1, K = 0, bn = 0;
  __half* w = nullptr;   // [cout][taps][3][cin] fp16: (W_hi | W_lo | W_hi) per tap; fp16 mode [cout][taps][cin]
  float* bias = nullptr;
  CUtensorMap wmap;
};

struct ActPair {
  __half* hi = nullptr;
  __half* lo = nullptr;   // nullptr: a single fp16 tensor
};
// the pair at element offset o of a (hi, lo) pair, keeping a null lo null
inline ActPair act_at(const ActPair& a, size_t o) { return ActPair{a.hi + o, a.lo ? a.lo + o : nullptr}; }

// the number of fp16 products per filter tap of a convolution: 3 in split precision (A_hi W_hi, A_hi W_lo,
// A_lo W_hi), 1 in the single-fp16 mode
inline int tap_products(int precision) { return precision == 0 ? 3 : 1; }

}  // namespace nope

struct nope_encoder {
  static constexpr const char* kName = "encoder";
  int D = 8, device = 0, num_sms = 132;
  int precision = 0;                  // 0: split (hi, lo) operands; 1: single fp16 (set before finalize)
  bool finalized = false;
  nope::StagedWeights staged;
  std::map<std::string, nope::EncConv> convs;
  float *stem_w = nullptr, *stem_b = nullptr;
  nope::DeviceAllocs mem;             // weights, rot_stage
  int cap = 0;
  nope::ActPair buf[5];
  float* proj_out = nullptr;
  nope::DeviceAllocs ws_mem;          // workspace for cap images (ensure_workspace)
  std::map<std::tuple<const void*, int, int, int, int>, CUtensorMap> tmaps;
  int64_t launches = 0;
  static constexpr int kChunk = 32;   // images per encode() call: the workspace holds this many
  float* rot_stage = nullptr;         // kChunk rotated 256x256 crops (25 MB), allocated by the first encode_inplane

  // ---------------------------------------------------------------- schema (resnet.py:93-133)
  void expect_bn(const std::string& p, int c) {
    for (const char* s : {".weight", ".bias", ".running_mean", ".running_var"}) staged.expect(p + s, {c});
  }
  void build_schema() {
    staged.expect("backbone.conv1.weight", {64, 3, 7, 7});
    expect_bn("backbone.bn1", 64);
    int inplanes = 64;
    const int planes[4] = {64, 128, 256, 512}, blocks[4] = {3, 4, 6, 3}, strides[4] = {1, 2, 2, 1};
    for (int li = 0; li < 4; ++li)
      for (int b = 0; b < blocks[li]; ++b) {
        const std::string p = "backbone.layer" + std::to_string(li + 1) + "." + std::to_string(b);
        staged.expect(p + ".conv1.weight", {planes[li], inplanes, 1, 1});
        expect_bn(p + ".bn1", planes[li]);
        staged.expect(p + ".conv2.weight", {planes[li], planes[li], 3, 3});
        expect_bn(p + ".bn2", planes[li]);
        staged.expect(p + ".conv3.weight", {planes[li] * 4, planes[li], 1, 1});
        expect_bn(p + ".bn3", planes[li] * 4);
        if (b == 0 && (strides[li] != 1 || inplanes != planes[li] * 4)) {
          staged.expect(p + ".downsample.0.weight", {planes[li] * 4, inplanes, 1, 1});
          expect_bn(p + ".downsample.1", planes[li] * 4);
        }
        inplanes = planes[li] * 4;
      }
    staged.expect("projector.1.weight", {256, 2048, 1, 1});
    staged.expect("projector.3.weight", {D, 256, 1, 1});
  }

  // ---------------------------------------------------------------- weights
  // fold eval-mode BN (eps 1e-5) into the conv in double, split into fp16 (hi, lo), pack; fp16 mode: hi only
  int make_conv(const std::string& name, const std::string& wkey, const std::string& bnkey, int stride) {
    using namespace nope;
    const HostTensor& W = staged.at(wkey);
    EncConv L;
    L.cout_real = (int)W.shape[0];
    L.cin = (int)W.shape[1];
    L.k = (int)W.shape[2];
    L.stride = stride;
    L.cout = (L.cout_real + 63) / 64 * 64;
    const int taps = L.k * L.k;
    const int prods = tap_products(precision);
    L.K = taps * prods * L.cin;
    NOPE_CHECK(L.cin % 64 == 0, wkey + ": input channels must be a multiple of 64");
    L.bn = pick_bn(L.cout);
    std::vector<double> scale(L.cout_real, 1.0), shift(L.cout_real, 0.0);
    if (!bnkey.empty()) {
      const auto &g = staged.at(bnkey + ".weight").data, &b = staged.at(bnkey + ".bias").data,
                 &m = staged.at(bnkey + ".running_mean").data, &v = staged.at(bnkey + ".running_var").data;
      for (int o = 0; o < L.cout_real; ++o) {
        scale[o] = (double)g[o] / std::sqrt((double)v[o] + 1e-5);
        shift[o] = (double)b[o] - (double)m[o] * scale[o];
      }
    }
    std::vector<__half> packed((size_t)L.cout * L.K, __float2half_rn(0.f));
    for (int o = 0; o < L.cout_real; ++o)
      for (int c = 0; c < L.cin; ++c)
        for (int t = 0; t < taps; ++t) {
          const float wf = (float)((double)W.data[((size_t)o * L.cin + c) * taps + t] * scale[o]);
          const __half hi = __float2half_rn(wf);
          const __half lo = __float2half_rn(wf - __half2float(hi));
          __half* dst = &packed[(size_t)o * L.K + (size_t)t * prods * L.cin];
          dst[c] = hi;
          if (prods == 1) continue;
          dst[L.cin + c] = lo;
          dst[2 * L.cin + c] = hi;
        }
    std::vector<float> bias(L.cout, 0.f);
    for (int o = 0; o < L.cout_real; ++o) bias[o] = (float)shift[o];
    if (mem.upload(&L.w, packed) || mem.upload(&L.bias, bias)) return -1;
    if (make_weight_map(&L.wmap, L.w, L.cout, L.K, L.bn)) return -1;
    convs[name] = L;
    return 0;
  }

  // packs the staged weights (nope::engine_finalize: every schema key is present, device selected)
  int finalize() {
    {  // stem: fold bn1 into conv1, keep fp32
      const auto& W = staged.at("backbone.conv1.weight").data;
      const auto &g = staged.at("backbone.bn1.weight").data, &b = staged.at("backbone.bn1.bias").data,
                 &m = staged.at("backbone.bn1.running_mean").data, &v = staged.at("backbone.bn1.running_var").data;
      std::vector<float> w(64 * 147), bias(64);
      for (int o = 0; o < 64; ++o) {
        const double s = (double)g[o] / std::sqrt((double)v[o] + 1e-5);
        for (int i = 0; i < 147; ++i) w[o * 147 + i] = (float)((double)W[o * 147 + i] * s);
        bias[o] = (float)((double)b[o] - (double)m[o] * s);
      }
      if (mem.upload(&stem_w, w) || mem.upload(&stem_b, bias)) return -1;
    }
    const int blocks[4] = {3, 4, 6, 3}, strides[4] = {1, 2, 2, 1};
    for (int li = 0; li < 4; ++li)
      for (int b = 0; b < blocks[li]; ++b) {
        const std::string p = "backbone.layer" + std::to_string(li + 1) + "." + std::to_string(b);
        const int st = b == 0 ? strides[li] : 1;
        if (make_conv(p + ".conv1", p + ".conv1.weight", p + ".bn1", 1)) return -1;
        if (make_conv(p + ".conv2", p + ".conv2.weight", p + ".bn2", st)) return -1;   // resnet.py:62
        if (make_conv(p + ".conv3", p + ".conv3.weight", p + ".bn3", 1)) return -1;
        if (staged.has(p + ".downsample.0.weight"))
          if (make_conv(p + ".down", p + ".downsample.0.weight", p + ".downsample.1", st)) return -1;
      }
    if (make_conv("projector.1", "projector.1.weight", "", 1)) return -1;
    return make_conv("projector.3", "projector.3.weight", "", 1);
  }

  // ---------------------------------------------------------------- workspace / maps
  int ensure_workspace(int B) {
    if (B <= cap) return 0;
    NOPE_CUDA(cudaDeviceSynchronize());
    ws_mem.release();
    tmaps.clear();
    cap = B;
    const size_t n = (size_t)cap * 128 * 128 * 256;     // largest activation: layer1 output
    for (auto& b : buf)
      if (ws_mem.alloc(&b.hi, n) || (precision == 0 && ws_mem.alloc(&b.lo, n))) return -1;
    return ws_mem.alloc(&proj_out, (size_t)cap * 1024 * 64);
  }
  int get_map(const CUtensorMap** out, const void* base, int C, const nope::TileGeom& g, int kind) {
    using namespace nope;
    auto key = std::make_tuple(base, kind + 1, C, g.H, g.W);
    auto it = tmaps.find(key);
    if (it == tmaps.end()) {
      CUtensorMap m;
      const int rc = kind < 0 ? make_act_map(&m, base, cap, C, g)
                              : make_unshuffle_map(&m, base, cap, C, g, kind >> 1, kind & 1);
      if (rc) return -1;
      it = tmaps.emplace(key, m).first;
    }
    *out = &it->second;
    return 0;
  }

  // out = [relu](conv(in) + bias [+ res]); Hin = input side; returns output side in *Hout
  int conv(const nope::EncConv& L, const nope::ActPair& in, int Hin, const nope::ActPair& out, int n_img,
           bool relu, const nope::ActPair* res, float* out_f32, cudaStream_t st) {
    using namespace nope;
    const int Ho = Hin / L.stride;
    TileGeom g;
    if (make_geom(Ho, Ho, &g)) return -1;
    ConvParams p;
    memset(&p, 0, sizeof p);
    const CUtensorMap* m = nullptr;
    int nseg = 0, ksteps = 0;
    const int nch = L.cin / 64;
    const bool split = precision == 0;   // fp16 mode: the hi maps only, one segment per tap
    if (L.stride == 1) {
      if (get_map(&m, in.hi, L.cin, g, -1)) return -1;
      p.amap[0] = *m;
      if (split) {
        if (get_map(&m, in.lo, L.cin, g, -1)) return -1;
        p.amap[1] = *m;
      }
      p.n_amaps = split ? 2 : 1;
    } else {
      for (int t = 0; t < 4; ++t) {
        if (get_map(&m, in.hi, L.cin, g, t)) return -1;
        p.amap[t] = *m;
        if (!split) continue;
        if (get_map(&m, in.lo, L.cin, g, t)) return -1;
        p.amap[4 + t] = *m;
      }
      p.n_amaps = split ? 8 : 4;
    }
    for (int ky = 0; ky < L.k; ++ky)
      for (int kx = 0; kx < L.k; ++kx) {
        int mh, ml, dy, dx;
        if (L.stride == 1) {
          mh = 0; ml = 1;
          dy = L.k == 3 ? ky - 1 : 0;
          dx = L.k == 3 ? kx - 1 : 0;
        } else {
          // in(2y + ky - pad, 2x + kx - pad) on the stride-2 lattices: odd offsets live on lattice 1
          const int oy = L.k == 3 ? ky - 1 : 0, ox = L.k == 3 ? kx - 1 : 0;
          const int p1 = oy & 1, p2 = ox & 1;
          dy = (oy - p1) / 2;
          dx = (ox - p2) / 2;
          mh = p1 * 2 + p2;
          ml = 4 + mh;
        }
        p.seg[nseg++] = ConvSeg{(int16_t)mh, (int16_t)dy, (int16_t)dx, (int16_t)nch};   // A_hi W_hi
        ksteps += nch;
        if (!split) continue;
        p.seg[nseg++] = ConvSeg{(int16_t)mh, (int16_t)dy, (int16_t)dx, (int16_t)nch};   // A_hi W_lo
        p.seg[nseg++] = ConvSeg{(int16_t)ml, (int16_t)dy, (int16_t)dx, (int16_t)nch};   // A_lo W_hi
        ksteps += 2 * nch;
      }
    NOPE_CHECK(nseg <= kMaxSeg && ksteps * 64 == L.K, "encoder conv: segment table");
    p.bmap = L.wmap;
    if (get_map(&m, out.hi, L.cout, g, -1)) return -1;
    for (int t = 0; t < 4; ++t) p.omap[t] = *m;
    p.bias = L.bias;
    p.stats = nullptr;
    p.stats_hw = Ho * Ho;
    p.stats_noct = L.cout / 8;
    p.n_total = L.cout;
    p.m_valid = n_img * Ho * Ho;
    p.nseg = nseg;
    p.ksteps = ksteps;
    p.m_tiles = geom_m_tiles(g, n_img);
    p.n_par = 1;
    p.n_tiles_par = L.cout / L.bn;
    p.n_tiles = p.n_tiles_par;
    p.tiles_per_img = g.tiles_per_img;
    p.h_cnt = g.h_cnt;
    p.b_cnt = g.b_cnt;
    p.relu = relu ? 1 : 0;
    p.res_hi = res ? res->hi : nullptr;
    p.res_lo = res ? res->lo : nullptr;
    p.out_lo = out_f32 ? nullptr : out.lo;
    p.out_f32 = out_f32;
    ++launches;
    return launch_conv_tc2(p, L.bn, num_sms, st);
  }

  // stem: images [B, 3, 256, 256] -> buf[0] (128 x 128 x 64)
  int stem(const float* images, int B, cudaStream_t st) {
    const long long npix = (long long)B * 128 * 128;
    nope::enc_stem_kernel<<<(unsigned)((npix + 3) / 4), 256, 0, st>>>(images, stem_w, stem_b, buf[0].hi, buf[0].lo,
                                                                      B, 256, 256);
    NOPE_CUDA(cudaGetLastError());
    ++launches;
    return 0;
  }

  // bottleneck p (conv2 / downsample stride stv) on buf[cur] of side H -> buf[cur] (the new cur), side H / stv
  int bottleneck(const std::string& p, int stv, int H, int B, int& cur, cudaStream_t st) {
    using namespace nope;
    // free buffers: the four that are not `cur`
    int f[4], nf = 0;
    for (int i = 0; i < 5; ++i)
      if (i != cur) f[nf++] = i;
    const ActPair &x = buf[cur], &a = buf[f[0]], &bb = buf[f[1]], &r = buf[f[2]], &o = buf[f[3]];
    if (conv(convs.at(p + ".conv1"), x, H, a, B, true, nullptr, nullptr, st)) return -1;
    if (conv(convs.at(p + ".conv2"), a, H, bb, B, true, nullptr, nullptr, st)) return -1;
    const int Ho = H / stv;
    const ActPair* res = &x;
    auto it = convs.find(p + ".down");
    if (it != convs.end()) {
      if (conv(it->second, x, H, r, B, false, nullptr, nullptr, st)) return -1;
      res = &r;
    }
    if (conv(convs.at(p + ".conv3"), bb, Ho, o, B, true, res, nullptr, st)) return -1;
    cur = f[3];
    return 0;
  }

  // projector (template.py:34-39) on buf[cur] of side H: ReLU (idempotent on the post-ReLU backbone output) ->
  // 1x1 2048->256 -> ReLU -> 1x1 256->D (no bias, no BN) -> out [B, D, H, H] fp32 NCHW
  int projector(int cur, int H, int B, float* out, cudaStream_t st) {
    using namespace nope;
    const int nxt = (cur + 1) % 5;
    if (conv(convs.at("projector.1"), buf[cur], H, buf[nxt], B, true, nullptr, nullptr, st)) return -1;
    const int nx2 = (cur + 2) % 5;
    if (conv(convs.at("projector.3"), buf[nxt], H, buf[nx2], B, false, nullptr, proj_out, st)) return -1;
    enc_extract_kernel<<<ew_grid((long long)B * D * H * H), 256, 0, st>>>(proj_out, out, B, D, H * H,
                                                                          convs.at("projector.3").cout);
    NOPE_CUDA(cudaGetLastError());
    ++launches;
    return 0;
  }

  static constexpr int kBlocks[4] = {3, 4, 6, 3}, kStrides[4] = {1, 2, 2, 1};
  static std::string block_name(int li, int b) {
    return "backbone.layer" + std::to_string(li + 1) + "." + std::to_string(b);
  }

  int encode(const float* images, int B, float* out, cudaStream_t st) {
    if (ensure_workspace(B)) return -1;
    launches = 0;
    if (stem(images, B, st)) return -1;
    int H = 128, cur = 0;   // buf[cur] holds the block input
    for (int li = 0; li < 4; ++li)
      for (int b = 0; b < kBlocks[li]; ++b) {
        const int stv = b == 0 ? kStrides[li] : 1;
        if (bottleneck(block_name(li, b), stv, H, B, cur, st)) return -1;
        H /= stv;
      }
    return projector(cur, H, B, out, st);
  }

  // Runs one module on its own (nope_encoder_run_block): "stem" on images [n, 3, 256, 256], a bottleneck
  // "backbone.layer<l>.<b>" or "projector" on x [n, C, H, H] fp32 NCHW, staged as (hi, lo) into the block's input
  // buffer -> out fp32 NCHW: hi + lo of the block's output pair, the projector's fp32 output.  *Co, *Ho: its shape.
  int run_block(const std::string& name, const float* x, int C, int H, int n, float* out, int64_t cap_floats,
                cudaStream_t st) {
    using namespace nope;
    NOPE_CHECK(n >= 1 && n <= kChunk, "run_block: n must be in [1, " + std::to_string(kChunk) + "]");
    int Ci = 0, Hi = 0, Co = 0, Ho = 0, stv = 1;
    if (name == "stem") {
      Ci = 3, Hi = 256, Co = 64, Ho = 128;
    } else if (name == "projector") {
      Ci = 2048, Hi = 32, Co = D, Ho = 32;
    } else {
      int h = 128;
      for (int li = 0; li < 4 && !Ci; ++li)
        for (int b = 0; b < kBlocks[li]; ++b) {
          const int s = b == 0 ? kStrides[li] : 1;
          if (name == block_name(li, b)) {
            Ci = convs.at(name + ".conv1").cin, Hi = h, Co = convs.at(name + ".conv3").cout, Ho = h / s, stv = s;
            break;
          }
          h /= s;
        }
      NOPE_CHECK(Ci, "run_block: unknown encoder module " + name);
    }
    NOPE_CHECK(C == Ci && H == Hi, "run_block: " + name + " takes [n, " + std::to_string(Ci) + ", " +
                                       std::to_string(Hi) + ", " + std::to_string(Hi) + "] inputs, got C = " +
                                       std::to_string(C) + ", H = " + std::to_string(H));
    NOPE_CHECK(cap_floats >= (int64_t)n * Co * Ho * Ho, "run_block: output buffer too small");
    if (ensure_workspace(n)) return -1;
    launches = 0;
    if (name == "stem") {
      if (stem(x, n, st)) return -1;
      to_nchw_pair(buf[0], out, n, Co, Ho, st);
    } else {
      nchw_f32_to_nhwc_f16_kernel<<<ew_grid((long long)n * C * H * H), 256, 0, st>>>(x, buf[0].hi, n, C, H * H,
                                                                                     buf[0].lo);
      NOPE_CUDA(cudaGetLastError());
      int cur = 0;
      if (name == "projector") {
        if (projector(cur, H, n, out, st)) return -1;
      } else {
        if (bottleneck(name, stv, H, n, cur, st)) return -1;
        to_nchw_pair(buf[cur], out, n, Co, Ho, st);
      }
    }
    NOPE_CUDA(cudaGetLastError());
    NOPE_CUDA(cudaStreamSynchronize(st));
    return 0;
  }
  static void to_nchw_pair(const nope::ActPair& a, float* out, int n, int C, int H, cudaStream_t st) {
    nope::nhwc_f16_to_nchw_f32_kernel<<<nope::ew_grid((long long)n * C * H * H), 256, 0, st>>>(a.hi, out, n, C, H * H,
                                                                                               a.lo);
  }

  // images [B, 3, 256, 256] x angles cossin [A, 2] -> out [B, A, D, 32, 32]: the (image, angle) pairs in b-major
  // order, kChunk at a time, each chunk rotated into rot_stage and encoded from there, so the [B, A, 3, 256, 256]
  // rotated batch never exists.  The chunks are those nope_encoder_encode makes of that batch.
  int encode_inplane(const float* images, int B, const float* cossin, int A, float* out, cudaStream_t st) {
    using namespace nope;
    constexpr long long kImg = 3LL * 256 * 256;
    if (!rot_stage && mem.alloc(&rot_stage, kChunk * kImg)) return -1;
    NOPE_CHECK((int64_t)B * A <= INT32_MAX, "too many (image, angle) pairs");
    const int pairs = B * A;
    int64_t total = 0;
    for (int lo = 0; lo < pairs; lo += kChunk) {
      const int n = pairs - lo < kChunk ? pairs - lo : kChunk;
      inplane_rotate_kernel<<<dim3(256 * 256 / 256, n), 256, 0, st>>>(images, cossin, A, 256, 256, lo, rot_stage);
      NOPE_CUDA(cudaGetLastError());
      if (encode(rot_stage, n, out + (size_t)lo * D * 32 * 32, st)) return -1;
      total += launches + 1;
    }
    launches = total;
    return 0;
  }

  // images [B, 3, 256, 256] x pairs (image_idx [P], cossin [P, 2]) -> out [P, D, 32, 32]: the pairs in order, kChunk
  // at a time through rot_stage, so the result equals nope_encoder_encode of the materialised [P, 3, 256, 256] batch.
  int encode_rotated(const float* images, int B, const int* image_idx, const float* cossin, int P, float* out,
                     cudaStream_t st) {
    using namespace nope;
    constexpr long long kImg = 3LL * 256 * 256;
    if (!rot_stage && mem.alloc(&rot_stage, kChunk * kImg)) return -1;
    int64_t total = 0;
    for (int lo = 0; lo < P; lo += kChunk) {
      const int n = P - lo < kChunk ? P - lo : kChunk;
      inplane_rotate_pairs_kernel<<<dim3(256 * 256 / 256, n), 256, 0, st>>>(images, B, image_idx, cossin, 256, 256,
                                                                             lo, rot_stage);
      NOPE_CUDA(cudaGetLastError());
      if (encode(rot_stage, n, out + (size_t)lo * D * 32 * 32, st)) return -1;
      total += launches + 1;
    }
    launches = total;
    return 0;
  }
};
