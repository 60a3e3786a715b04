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
// The sample of pixel (x, y) of the copy rotated by (c, s): top-left tap (ix, iy) and fractions (fx, fy).
// inplane_rotate_pixel and latent_visibility_kernel both sample through it.
__device__ __forceinline__ void inplane_sample(float c, float s, int H, int W, int x, int y, int& ix, int& iy,
                                               float& fx, float& fy) {
  const float cx = __fmul_rn((float)(W - 1), 0.5f), cy = __fmul_rn((float)(H - 1), 0.5f);
  const float dx = __fsub_rn((float)x, cx), dy = __fsub_rn((float)y, cy);
  const float sx = __fadd_rn(__fsub_rn(__fmul_rn(c, dx), __fmul_rn(s, dy)), cx);
  const float sy = __fadd_rn(__fadd_rn(__fmul_rn(s, dx), __fmul_rn(c, dy)), cy);
  const float x0 = floorf(sx), y0 = floorf(sy);
  fx = __fsub_rn(sx, x0);
  fy = __fsub_rn(sy, y0);
  ix = (int)x0;
  iy = (int)y0;
}

__device__ __forceinline__ void inplane_rotate_pixel(const float* __restrict__ src, float c, float s, int H, int W,
                                                     int i, float* __restrict__ dst) {
  const long long hw = (long long)H * W;
  const int x = i % W, y = i / W;
  int ix, iy;
  float fx, fy;
  inplane_sample(c, s, H, W, x, y, ix, iy, fx, fy);
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

// Latent visibility of rolled copies (DESIGN.md section 27).  Pair p rolls crop-space mask image_idx[p] of hidden
// [B, S, S] (uint8, non-zero = may be hidden) by (cossin[2p], cossin[2p + 1]) with inplane_rotate_pixel's sample:
// pixel (x, y) of the copy is hidden when one of its taps (ix, iy), (ix + 1, iy) if fx > 0, (ix, iy + 1) if fy > 0,
// (ix + 1, iy + 1) if both, lies inside the image and is hidden.  Latent pixel (i, j) of out [P, 32, 32] is 0 when
// its 8 x 8 block holds a hidden pixel, otherwise 1.  An image index outside [0, B) gives an all-visible row.  One
// CTA of 1024 threads per pair, thread (i, j) samples its block's 64 pixels (stopping at the first hidden one).
// S = 8 * 32.
constexpr int kVisSide = 32;                 // latent side of every visible map
constexpr int kVisThreads = kVisSide * kVisSide;

__global__ void __launch_bounds__(kVisThreads)
latent_visibility_kernel(const uint8_t* __restrict__ hidden, int B, int S, const int* __restrict__ image_idx,
                         const float* __restrict__ cossin, uint8_t* __restrict__ out) {
  const int p = blockIdx.x, t = threadIdx.x;
  const int li = t / kVisSide, lj = t - li * kVisSide;
  const int b = image_idx[p];
  uint8_t* o = out + (size_t)p * kVisThreads;
  if (b < 0 || b >= B) {
    o[t] = 1;
    return;
  }
  const float c = cossin[2 * p], s = cossin[2 * p + 1];
  const uint8_t* hb = hidden + (size_t)b * S * S;
  const int blk = S / kVisSide;
  bool any = false;
  for (int dy = 0; dy < blk && !any; ++dy)
    for (int dx = 0; dx < blk; ++dx) {
      int ix, iy;
      float fx, fy;
      inplane_sample(c, s, S, S, lj * blk + dx, li * blk + dy, ix, iy, fx, fy);
      const bool x0 = ix >= 0 && ix < S, y0 = iy >= 0 && iy < S;
      const bool x1 = fx > 0.f && ix + 1 >= 0 && ix + 1 < S, y1 = fy > 0.f && iy + 1 >= 0 && iy + 1 < S;
      const int r0 = iy * S + ix;          // read only where the tap lies inside the image
      any |= (y0 && x0 && __ldg(hb + r0)) || (y0 && x1 && __ldg(hb + r0 + 1)) ||
             (y1 && x0 && __ldg(hb + r0 + S)) || (y1 && x1 && __ldg(hb + r0 + S + 1));
      if (any) break;
    }
  o[t] = any ? 0 : 1;
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

struct ActPair {
  __half* hi = nullptr;
  __half* lo = nullptr;   // nullptr: a single fp16 tensor
};
// the pair at element offset o of a (hi, lo) pair, keeping a null lo null
inline ActPair act_at(const ActPair& a, size_t o) { return ActPair{a.hi + o, a.lo ? a.lo + o : nullptr}; }

// What the template encoder and the VAE engines share: the handle's state, the convolution layers, their packing and
// their launch.  Every activation buffer holds `cap` images.
struct ImageEngine {
  int device = 0, num_sms = 132;
  int precision = 0;                  // 0: split (hi, lo) operands; 1: single fp16 (set before finalize)
  bool finalized = false;
  StagedWeights staged;
  std::map<std::string, ConvLayer> convs;
  DeviceAllocs mem;
  TmapCache tmaps;
  int64_t launches = 0;
  int cap = 0;                        // images the workspace holds

  // L's taps, W [cout_real][cin][taps] and bias [cout_real] in float64 (any folding done), optional 1x1 shortcut
  // Ws [cout_real][cin_sc] in the extra K columns -> convs[name].  Split precision packs the W_lo plane; cout is padded
  // to 64 with zero rows.
  int pack_conv(const std::string& name, ConvLayer L, int cout_real, int cin, const std::vector<double>& W,
                const std::vector<double>& bias, int cin_sc = 0, const std::vector<double>* Ws = nullptr) {
    const int taps = L.k * L.k;
    L.cin = cin;
    L.cout = (cout_real + 63) / 64 * 64;
    L.K = taps * cin + cin_sc;
    L.wlo = precision == 0;
    NOPE_CHECK(cin % 64 == 0 && cin_sc % 64 == 0, name + ": input channels must be a multiple of 64");
    const std::vector<float> w(W.begin(), W.end());
    std::vector<float> ws;
    if (Ws) ws.assign(Ws->begin(), Ws->end());
    std::vector<float> b(L.cout, 0.f);
    for (int o = 0; o < cout_real; ++o) b[o] = (float)bias[o];
    std::vector<WeightBlock> blocks{{w.data(), cout_real, cin, taps, 0, 0}};
    if (cin_sc) blocks.push_back({ws.data(), cout_real, cin_sc, 1, 0, taps * cin});
    if (pack_conv_layer(mem, L, blocks, b)) return -1;
    convs[name] = L;
    return 0;
  }

  // out = [relu](conv(taps over the input pairs `in`) [+ 1x1 shortcut over the pair sc] + bias [+ res]); output
  // H x H.  in: (hi, lo) base pointers of each input pair with their lattice (-1: plain NHWC of side H); a tap's lat
  // is the index of its input pair; fp16 mode: the hi maps only.  K order: per tap A_hi W_hi, A_hi W_lo, A_lo W_hi,
  // then the shortcut's segments.
  int conv(const ConvLayer& L, const std::vector<std::pair<ActPair, int>>& in, const std::vector<ConvTap>& taps,
           const ActPair* sc, int H, int n, bool relu, const ActPair* res, __half* out_hi, __half* out_lo,
           float* out_f32, cudaStream_t st) {
    TileGeom g;
    if (make_geom(H, H, &g)) return -1;
    NOPE_CHECK(in.size() + (sc ? 1 : 0) <= (size_t)kMaxAMaps / 2, "conv: too many input maps");
    ConvBuilder b(tmaps, g, cap);
    ConvParams& p = b.p;
    ConvSrc src;
    src.C = L.cin;
    for (size_t i = 0; i < in.size(); ++i) {
      src.hi[i] = b.map(in[i].first.hi, L.cin, in[i].second);
      if (in[i].first.lo) src.lo[i] = b.map(in[i].first.lo, L.cin, in[i].second);
    }
    const int wlo_col = L.wlo ? L.K : 0;
    int col = b.segs(taps, {src}, 0, wlo_col);
    // the shortcut's channels are the W_hi columns past the taps
    if (sc) col = b.segs({ConvTap{0, 0, 0}}, {b.src(sc->hi, sc->lo, L.K - col)}, col, wlo_col);
    if (b.finish(L, out_hi, L.cout, n, 1)) return -1;
    NOPE_CHECK(col == L.K && p.ksteps * 64 == (L.wlo ? 3 : 1) * L.K, "conv: segment table");
    p.relu = relu ? 1 : 0;
    p.res_hi = res ? res->hi : nullptr;
    p.res_lo = res ? res->lo : nullptr;
    p.out_lo = out_lo;
    p.out_f32 = out_f32;
    ++launches;
    return launch_conv_tc2(p, L.bn, num_sms, st);
  }
};

}  // namespace nope

struct nope_encoder : nope::ImageEngine {
  static constexpr const char* kName = "encoder";
  enum { kStem, kBottleneck, kProjector };
  int D = 8;
  std::vector<nope::ImageModule> plan;
  float *stem_w = nullptr, *stem_b = nullptr;
  nope::ActPair buf[5];
  float* proj_out = nullptr;
  nope::WorkspaceSlab ws;
  static constexpr int kChunk = 32;   // images per encode() call: the workspace holds this many
  float* rot_stage = nullptr;         // kChunk rotated 256x256 crops (25 MB), allocated by the first rotated encode
  size_t out_floats() const { return (size_t)D * 32 * 32; }   // per encoded image

  // ---------------------------------------------------------------- plan + schema (resnet.py:93-133)
  // the stem, the 16 bottlenecks "backbone.layer<l>.<b>" (conv2 and the downsample at stride Hi / Ho) and the projector
  void build_plan() {
    plan = {{"stem", kStem, 3, 256, 64, 128}};
    const int planes[4] = {64, 128, 256, 512}, blocks[4] = {3, 4, 6, 3}, strides[4] = {1, 2, 2, 1};
    int cin = 64, H = 128;
    for (int li = 0; li < 4; ++li)
      for (int b = 0; b < blocks[li]; ++b) {
        const int s = b == 0 ? strides[li] : 1;   // resnet.py:62
        plan.push_back({"backbone.layer" + std::to_string(li + 1) + "." + std::to_string(b), kBottleneck, cin, H,
                        planes[li] * 4, H / s});
        cin = planes[li] * 4;
        H /= s;
      }
    plan.push_back({"projector", kProjector, 2048, 32, D, 32});
  }
  // a bottleneck that changes the side or the channels has a downsample on its shortcut
  static bool has_down(const nope::ImageModule& m) { return m.Ci != m.Co || m.Hi != m.Ho; }

  void expect_bn(const std::string& p, int c) {
    for (const char* s : {".weight", ".bias", ".running_mean", ".running_var"}) staged.expect(p + s, {c});
  }
  void build_schema() {
    for (const nope::ImageModule& m : plan) {
      const std::string& p = m.name;
      if (m.kind == kStem) {
        staged.expect("backbone.conv1.weight", {64, 3, 7, 7});
        expect_bn("backbone.bn1", 64);
      } else if (m.kind == kBottleneck) {
        const int planes = m.Co / 4;
        staged.expect(p + ".conv1.weight", {planes, m.Ci, 1, 1});
        expect_bn(p + ".bn1", planes);
        staged.expect(p + ".conv2.weight", {planes, planes, 3, 3});
        expect_bn(p + ".bn2", planes);
        staged.expect(p + ".conv3.weight", {m.Co, planes, 1, 1});
        expect_bn(p + ".bn3", m.Co);
        if (has_down(m)) {
          staged.expect(p + ".downsample.0.weight", {m.Co, m.Ci, 1, 1});
          expect_bn(p + ".downsample.1", m.Co);
        }
      } else {
        staged.expect("projector.1.weight", {256, 2048, 1, 1});
        staged.expect("projector.3.weight", {D, 256, 1, 1});
      }
    }
  }

  // ---------------------------------------------------------------- weights
  // fold eval-mode BN (eps 1e-5) into the conv in double, then pack_conv (a 1x1 or 3x3 pad-1 convolution at input
  // stride 1 or 2); bnkey empty: no BN, no bias
  int make_conv(const std::string& name, const std::string& wkey, const std::string& bnkey, int stride = 1) {
    const nope::HostTensor& W = staged.at(wkey);
    const int cout = (int)W.shape[0], cin = (int)W.shape[1], k = (int)W.shape[2], taps = k * k;
    std::vector<double> scale(cout, 1.0), shift(cout, 0.0);
    if (!bnkey.empty()) {
      const auto &g = staged.at(bnkey + ".weight").data, &b = staged.at(bnkey + ".bias").data,
                 &m = staged.at(bnkey + ".running_mean").data, &v = staged.at(bnkey + ".running_var").data;
      for (int o = 0; o < cout; ++o) {
        scale[o] = (double)g[o] / std::sqrt((double)v[o] + 1e-5);
        shift[o] = (double)b[o] - (double)m[o] * scale[o];
      }
    }
    std::vector<double> w(W.data.size());
    for (size_t i = 0; i < w.size(); ++i) w[i] = (double)W.data[i] * scale[i / ((size_t)cin * taps)];
    return pack_conv(name, nope::conv_shape(k, stride, -(k / 2), -(k / 2)), cout, cin, w, shift);
  }

  // packs the staged weights (nope::engine_finalize: every schema key is present, device selected)
  int finalize() {
    for (const nope::ImageModule& m : plan) {
      const std::string& p = m.name;
      if (m.kind == kStem) {  // fold bn1 into conv1, keep fp32
        const auto& W = staged.at("backbone.conv1.weight").data;
        const auto &g = staged.at("backbone.bn1.weight").data, &b = staged.at("backbone.bn1.bias").data,
                   &mu = staged.at("backbone.bn1.running_mean").data, &v = staged.at("backbone.bn1.running_var").data;
        std::vector<float> w(64 * 147), bias(64);
        for (int o = 0; o < 64; ++o) {
          const double s = (double)g[o] / std::sqrt((double)v[o] + 1e-5);
          for (int i = 0; i < 147; ++i) w[o * 147 + i] = (float)((double)W[o * 147 + i] * s);
          bias[o] = (float)((double)b[o] - (double)mu[o] * s);
        }
        if (mem.upload(&stem_w, w) || mem.upload(&stem_b, bias)) return -1;
      } else if (m.kind == kBottleneck) {
        const int s = m.Hi / m.Ho;
        if (make_conv(p + ".conv1", p + ".conv1.weight", p + ".bn1") ||
            make_conv(p + ".conv2", p + ".conv2.weight", p + ".bn2", s) ||
            make_conv(p + ".conv3", p + ".conv3.weight", p + ".bn3") ||
            (has_down(m) && make_conv(p + ".down", p + ".downsample.0.weight", p + ".downsample.1", s)))
          return -1;
      } else if (make_conv("projector.1", "projector.1.weight", "") ||
                 make_conv("projector.3", "projector.3.weight", "")) {
        return -1;
      }
    }
    return 0;
  }

  // ---------------------------------------------------------------- workspace
  size_t layout(nope::Bump& b, int c) {
    const size_t n = (size_t)c * 128 * 128 * 256;     // largest activation: layer1 output
    for (auto& a : buf) {
      b.take(&a.hi, n);
      if (precision == 0) b.take(&a.lo, n);
    }
    b.take(&proj_out, (size_t)c * 1024 * 64);
    return b.off;
  }
  int ensure_workspace(int B) { return B <= cap ? 0 : nope::grow_workspace(this, std::tie(cap), nullptr, B); }

  // out = [relu](conv(in) + bias [+ res]) of layer L over an input of side Hin; a stride-2 convolution reads its input
  // as its four stride-2 sub-lattices (same trick as HardDownsample).  out_f32: the fp32 output instead of out's lo
  // half.
  int conv_at(const nope::ConvLayer& L, const nope::ActPair& in, int Hin, const nope::ActPair& out, int n, bool relu,
              const nope::ActPair* res, float* out_f32, cudaStream_t st) {
    using namespace nope;
    std::vector<std::pair<ActPair, int>> src;
    for (int t = 0; t < (L.stride == 1 ? 1 : 4); ++t) src.push_back({in, L.stride == 1 ? -1 : t});
    return conv(L, src, L.taps(), nullptr, Hin / L.stride, n, relu, res, out.hi, out_f32 ? nullptr : out.lo, out_f32,
                st);
  }

  // bottleneck m on buf[cur] -> buf[cur] (the new cur)
  int bottleneck(const nope::ImageModule& m, int n, int& cur, cudaStream_t st) {
    using namespace nope;
    // free buffers: the four that are not `cur`
    int f[4], nf = 0;
    for (int i = 0; i < 5; ++i)
      if (i != cur) f[nf++] = i;
    const ActPair &x = buf[cur], &a = buf[f[0]], &bb = buf[f[1]], &r = buf[f[2]], &o = buf[f[3]];
    if (conv_at(convs.at(m.name + ".conv1"), x, m.Hi, a, n, true, nullptr, nullptr, st)) return -1;
    if (conv_at(convs.at(m.name + ".conv2"), a, m.Hi, bb, n, true, nullptr, nullptr, st)) return -1;
    const ActPair* res = &x;
    if (has_down(m)) {
      if (conv_at(convs.at(m.name + ".down"), x, m.Hi, r, n, false, nullptr, nullptr, st)) return -1;
      res = &r;
    }
    if (conv_at(convs.at(m.name + ".conv3"), bb, m.Ho, o, n, true, res, nullptr, st)) return -1;
    cur = f[3];
    return 0;
  }

  // projector (template.py:34-39) on buf[cur] of side H: ReLU (idempotent on the post-ReLU backbone output) ->
  // 1x1 2048->256 -> ReLU -> 1x1 256->D (no bias, no BN) -> out [B, D, H, H] fp32 NCHW
  int projector(int cur, int H, int B, float* out, cudaStream_t st) {
    using namespace nope;
    const int nxt = (cur + 1) % 5;
    if (conv_at(convs.at("projector.1"), buf[cur], H, buf[nxt], B, true, nullptr, nullptr, st)) return -1;
    const int nx2 = (cur + 2) % 5;
    if (conv_at(convs.at("projector.3"), buf[nxt], H, buf[nx2], B, false, nullptr, proj_out, st)) return -1;
    enc_extract_kernel<<<ew_grid((long long)B * D * H * H), 256, 0, st>>>(proj_out, out, B, D, H * H,
                                                                          convs.at("projector.3").cout);
    NOPE_CUDA(cudaGetLastError());
    ++launches;
    return 0;
  }

  // module m of n images: the stem on images [n, 3, 256, 256] -> buf[0]; a bottleneck on buf[cur] -> buf[cur] (the
  // new cur); the projector on buf[cur] -> out [n, D, 32, 32]
  int run(const nope::ImageModule& m, int n, int& cur, const float* images, float* out, cudaStream_t st) {
    if (m.kind == kBottleneck) return bottleneck(m, n, cur, st);
    if (m.kind == kProjector) return projector(cur, m.Hi, n, out, st);
    const long long npix = (long long)n * 128 * 128;   // stem: 7x7 stride 2, 256 -> 128
    nope::enc_stem_kernel<<<(unsigned)((npix + 3) / 4), 256, 0, st>>>(images, stem_w, stem_b, buf[0].hi, buf[0].lo,
                                                                      n, 256, 256);
    NOPE_CUDA(cudaGetLastError());
    ++launches;
    cur = 0;
    return 0;
  }

  int encode(const float* images, int B, float* out, cudaStream_t st) {
    if (ensure_workspace(B)) return -1;
    launches = 0;
    int cur = 0;
    for (const nope::ImageModule& m : plan)
      if (run(m, B, cur, images, out, st)) return -1;
    return 0;
  }

  // Runs one module on its own (nope_encoder_run_block): "stem" on images [n, 3, 256, 256], a bottleneck
  // "backbone.layer<l>.<b>" or "projector" on x [n, C, H, H] fp32 NCHW, staged as (hi, lo) into the block's input
  // buffer -> out fp32 NCHW: hi + lo of the block's output pair, the projector's fp32 output.
  int run_block(const std::string& name, const float* x, int C, int H, int n, float* out, int64_t cap_floats,
                cudaStream_t st) {
    using namespace nope;
    const ImageModule* m = find_module(plan, name);
    NOPE_CHECK(m, "run_block: unknown encoder module " + name);
    if (check_block(*m, kChunk, C, H, n, cap_floats)) return -1;
    if (ensure_workspace(n)) return -1;
    launches = 0;
    if (m->kind != kStem) {
      nchw_f32_to_nhwc_f16_kernel<<<ew_grid((long long)n * C * H * H), 256, 0, st>>>(x, buf[0].hi, n, C, H * H,
                                                                                     buf[0].lo);
      NOPE_CUDA(cudaGetLastError());
    }
    int cur = 0;
    if (run(*m, n, cur, x, out, st)) return -1;
    if (m->kind != kProjector)
      nhwc_f16_to_nchw_f32_kernel<<<ew_grid((long long)n * m->Co * m->Ho * m->Ho), 256, 0, st>>>(
          buf[cur].hi, out, n, m->Co, m->Ho * m->Ho, buf[cur].lo);
    NOPE_CUDA(cudaGetLastError());
    NOPE_CUDA(cudaStreamSynchronize(st));
    return 0;
  }
};
