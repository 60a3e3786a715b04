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
#pragma once
#include "conv_tc2.cuh"
#include "kernels.cuh"

#include <cmath>
#include <map>
#include <string>
#include <vector>

namespace nope {

// stem: conv 7x7 stride 2 pad 3 (3 -> 64) + folded BN + ReLU, fp32 direct, -> (hi, lo) NHWC.
// Block = 64 output channels x 4 pixels.  w: [64][3][7][7] folded, fp32.
__global__ void __launch_bounds__(256)
enc_stem_kernel(const float* __restrict__ x, const float* __restrict__ w, const float* __restrict__ bias,
                __half* __restrict__ out_hi, __half* __restrict__ out_lo, int B, int Hin, int Win) {
  __shared__ float s_w[64 * 147];
  for (int i = threadIdx.x; i < 64 * 147; i += 256) s_w[i] = w[i];
  __syncthreads();
  const int Ho = Hin / 2, Wo = Win / 2;
  const int o = threadIdx.x & 63;
  const long long pix = (long long)blockIdx.x * 4 + (threadIdx.x >> 6);
  if (pix >= (long long)B * Ho * Wo) return;
  const int px = (int)(pix % Wo), py = (int)((pix / Wo) % Ho), b = (int)(pix / ((long long)Wo * Ho));
  float acc = bias[o];
  for (int c = 0; c < 3; ++c)
    for (int ky = 0; ky < 7; ++ky) {
      const int yy = 2 * py + ky - 3;
      if (yy < 0 || yy >= Hin) continue;
      const float* xr = x + (((long long)b * 3 + c) * Hin + yy) * Win;
      const float* wr = s_w + o * 147 + (c * 7 + ky) * 7;
#pragma unroll
      for (int kx = 0; kx < 7; ++kx) {
        const int xx = 2 * px + kx - 3;
        if (xx >= 0 && xx < Win) acc = fmaf(xr[xx], wr[kx], acc);
      }
    }
  acc = fmaxf(acc, 0.f);
  const __half hi = __float2half_rn(acc);
  out_hi[pix * 64 + o] = hi;
  out_lo[pix * 64 + o] = __float2half_rn(acc - __half2float(hi));
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
  __half* w = nullptr;   // [cout][taps][3][cin] fp16: (W_hi | W_lo | W_hi) per tap
  float* bias = nullptr;
  CUtensorMap wmap;
};

struct ActPair {
  __half* hi = nullptr;
  __half* lo = nullptr;
};

}  // namespace nope

struct nope_encoder {
  int D = 8, device = 0, num_sms = 132;
  bool finalized = false;
  std::map<std::string, std::pair<std::vector<int64_t>, std::vector<float>>> host;
  std::map<std::string, std::vector<int64_t>> expected;
  std::map<std::string, nope::EncConv> convs;
  float *stem_w = nullptr, *stem_b = nullptr;
  std::vector<void*> owned;
  int cap = 0;
  nope::ActPair buf[5];
  float* proj_out = nullptr;
  std::vector<void*> ws_owned;
  std::map<std::tuple<const void*, int, int, int, int>, CUtensorMap> tmaps;
  int64_t launches = 0;

  ~nope_encoder() {
    for (void* p : owned) cudaFree(p);
    for (void* p : ws_owned) cudaFree(p);
  }

  // ---------------------------------------------------------------- schema (resnet.py:93-133)
  void expect_bn(const std::string& p, int c) {
    for (const char* s : {".weight", ".bias", ".running_mean", ".running_var"}) expected[p + s] = {c};
  }
  void build_schema() {
    expected["backbone.conv1.weight"] = {64, 3, 7, 7};
    expect_bn("backbone.bn1", 64);
    int inplanes = 64;
    const int planes[4] = {64, 128, 256, 512}, blocks[4] = {3, 4, 6, 3}, strides[4] = {1, 2, 2, 1};
    for (int li = 0; li < 4; ++li)
      for (int b = 0; b < blocks[li]; ++b) {
        const std::string p = "backbone.layer" + std::to_string(li + 1) + "." + std::to_string(b);
        expected[p + ".conv1.weight"] = {planes[li], inplanes, 1, 1};
        expect_bn(p + ".bn1", planes[li]);
        expected[p + ".conv2.weight"] = {planes[li], planes[li], 3, 3};
        expect_bn(p + ".bn2", planes[li]);
        expected[p + ".conv3.weight"] = {planes[li] * 4, planes[li], 1, 1};
        expect_bn(p + ".bn3", planes[li] * 4);
        if (b == 0 && (strides[li] != 1 || inplanes != planes[li] * 4)) {
          expected[p + ".downsample.0.weight"] = {planes[li] * 4, inplanes, 1, 1};
          expect_bn(p + ".downsample.1", planes[li] * 4);
        }
        inplanes = planes[li] * 4;
      }
    expected["projector.1.weight"] = {256, 2048, 1, 1};
    expected["projector.3.weight"] = {D, 256, 1, 1};
  }

  // ---------------------------------------------------------------- weights
  // fold eval-mode BN (eps 1e-5) into the conv in double, split into fp16 (hi, lo), pack
  int make_conv(const std::string& name, const std::string& wkey, const std::string& bnkey, int stride) {
    using namespace nope;
    const auto& W = host.at(wkey);
    EncConv L;
    L.cout_real = (int)W.first[0];
    L.cin = (int)W.first[1];
    L.k = (int)W.first[2];
    L.stride = stride;
    L.cout = (L.cout_real + 63) / 64 * 64;
    const int taps = L.k * L.k;
    L.K = taps * 3 * L.cin;
    NOPE_CHECK(L.cin % 64 == 0, wkey + ": input channels must be a multiple of 64");
    L.bn = pick_bn(L.cout);
    std::vector<double> scale(L.cout_real, 1.0), shift(L.cout_real, 0.0);
    if (!bnkey.empty()) {
      const auto &g = host.at(bnkey + ".weight").second, &b = host.at(bnkey + ".bias").second,
                 &m = host.at(bnkey + ".running_mean").second, &v = host.at(bnkey + ".running_var").second;
      for (int o = 0; o < L.cout_real; ++o) {
        scale[o] = (double)g[o] / std::sqrt((double)v[o] + 1e-5);
        shift[o] = (double)b[o] - (double)m[o] * scale[o];
      }
    }
    std::vector<__half> packed((size_t)L.cout * L.K, __float2half_rn(0.f));
    for (int o = 0; o < L.cout_real; ++o)
      for (int c = 0; c < L.cin; ++c)
        for (int t = 0; t < taps; ++t) {
          const float wf = (float)((double)W.second[((size_t)o * L.cin + c) * taps + t] * scale[o]);
          const __half hi = __float2half_rn(wf);
          const __half lo = __float2half_rn(wf - __half2float(hi));
          __half* dst = &packed[(size_t)o * L.K + (size_t)t * 3 * L.cin];
          dst[c] = hi;
          dst[L.cin + c] = lo;
          dst[2 * L.cin + c] = hi;
        }
    NOPE_CUDA(cudaMalloc(reinterpret_cast<void**>(&L.w), packed.size() * sizeof(__half)));
    owned.push_back(L.w);
    NOPE_CUDA(cudaMemcpy(L.w, packed.data(), packed.size() * sizeof(__half), cudaMemcpyHostToDevice));
    std::vector<float> bias(L.cout, 0.f);
    for (int o = 0; o < L.cout_real; ++o) bias[o] = (float)shift[o];
    NOPE_CUDA(cudaMalloc(reinterpret_cast<void**>(&L.bias), bias.size() * sizeof(float)));
    owned.push_back(L.bias);
    NOPE_CUDA(cudaMemcpy(L.bias, bias.data(), bias.size() * sizeof(float), cudaMemcpyHostToDevice));
    if (make_weight_map(&L.wmap, L.w, L.cout, L.K, L.bn)) return -1;
    convs[name] = L;
    return 0;
  }

  int finalize() {
    using namespace nope;
    NOPE_CHECK(!finalized, "already finalized");
    for (const auto& kv : expected) NOPE_CHECK(host.count(kv.first), "state_dict is missing " + kv.first);
    NOPE_CUDA(cudaSetDevice(device));
    {  // stem: fold bn1 into conv1, keep fp32
      const auto& W = host.at("backbone.conv1.weight").second;
      const auto &g = host.at("backbone.bn1.weight").second, &b = host.at("backbone.bn1.bias").second,
                 &m = host.at("backbone.bn1.running_mean").second, &v = host.at("backbone.bn1.running_var").second;
      std::vector<float> w(64 * 147), bias(64);
      for (int o = 0; o < 64; ++o) {
        const double s = (double)g[o] / std::sqrt((double)v[o] + 1e-5);
        for (int i = 0; i < 147; ++i) w[o * 147 + i] = (float)((double)W[o * 147 + i] * s);
        bias[o] = (float)((double)b[o] - (double)m[o] * s);
      }
      NOPE_CUDA(cudaMalloc(reinterpret_cast<void**>(&stem_w), w.size() * 4));
      NOPE_CUDA(cudaMalloc(reinterpret_cast<void**>(&stem_b), bias.size() * 4));
      owned.push_back(stem_w);
      owned.push_back(stem_b);
      NOPE_CUDA(cudaMemcpy(stem_w, w.data(), w.size() * 4, cudaMemcpyHostToDevice));
      NOPE_CUDA(cudaMemcpy(stem_b, bias.data(), bias.size() * 4, cudaMemcpyHostToDevice));
    }
    const int blocks[4] = {3, 4, 6, 3}, strides[4] = {1, 2, 2, 1};
    for (int li = 0; li < 4; ++li)
      for (int b = 0; b < blocks[li]; ++b) {
        const std::string p = "backbone.layer" + std::to_string(li + 1) + "." + std::to_string(b);
        const int st = b == 0 ? strides[li] : 1;
        if (make_conv(p + ".conv1", p + ".conv1.weight", p + ".bn1", 1)) return -1;
        if (make_conv(p + ".conv2", p + ".conv2.weight", p + ".bn2", st)) return -1;   // resnet.py:62
        if (make_conv(p + ".conv3", p + ".conv3.weight", p + ".bn3", 1)) return -1;
        if (host.count(p + ".downsample.0.weight"))
          if (make_conv(p + ".down", p + ".downsample.0.weight", p + ".downsample.1", st)) return -1;
      }
    if (make_conv("projector.1", "projector.1.weight", "", 1)) return -1;
    if (make_conv("projector.3", "projector.3.weight", "", 1)) return -1;
    host.clear();
    finalized = true;
    return 0;
  }

  // ---------------------------------------------------------------- workspace / maps
  int ensure_workspace(int B) {
    if (B <= cap) return 0;
    NOPE_CUDA(cudaDeviceSynchronize());
    for (void* p : ws_owned) cudaFree(p);
    ws_owned.clear();
    tmaps.clear();
    cap = B;
    const size_t n = (size_t)cap * 128 * 128 * 256;     // largest activation: layer1 output
    for (auto& b : buf) {
      NOPE_CUDA(cudaMalloc(reinterpret_cast<void**>(&b.hi), n * sizeof(__half)));
      ws_owned.push_back(b.hi);
      NOPE_CUDA(cudaMalloc(reinterpret_cast<void**>(&b.lo), n * sizeof(__half)));
      ws_owned.push_back(b.lo);
    }
    NOPE_CUDA(cudaMalloc(reinterpret_cast<void**>(&proj_out), (size_t)cap * 1024 * 64 * sizeof(float)));
    ws_owned.push_back(proj_out);
    return 0;
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
    if (L.stride == 1) {
      if (get_map(&m, in.hi, L.cin, g, -1)) return -1;
      p.amap[0] = *m;
      if (get_map(&m, in.lo, L.cin, g, -1)) return -1;
      p.amap[1] = *m;
      p.n_amaps = 2;
    } else {
      for (int t = 0; t < 4; ++t) {
        if (get_map(&m, in.hi, L.cin, g, t)) return -1;
        p.amap[t] = *m;
        if (get_map(&m, in.lo, L.cin, g, t)) return -1;
        p.amap[4 + t] = *m;
      }
      p.n_amaps = 8;
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
        p.seg[nseg++] = ConvSeg{(int16_t)mh, (int16_t)dy, (int16_t)dx, (int16_t)nch};   // A_hi W_lo
        p.seg[nseg++] = ConvSeg{(int16_t)ml, (int16_t)dy, (int16_t)dx, (int16_t)nch};   // A_lo W_hi
        ksteps += 3 * nch;
      }
    NOPE_CHECK(nseg <= kMaxSeg && ksteps * 64 == L.K, "encoder conv: segment table");
    p.bmap2 = L.wmap;
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

  int encode(const float* images, int B, float* out, cudaStream_t st) {
    using namespace nope;
    if (ensure_workspace(B)) return -1;
    launches = 0;
    int H = 128;
    {
      const long long npix = (long long)B * H * H;
      enc_stem_kernel<<<(unsigned)((npix + 3) / 4), 256, 0, st>>>(images, stem_w, stem_b, buf[0].hi, buf[0].lo,
                                                                  B, 256, 256);
      NOPE_CUDA(cudaGetLastError());
      ++launches;
    }
    int cur = 0;   // buf[cur] holds the block input
    const int blocks[4] = {3, 4, 6, 3}, strides[4] = {1, 2, 2, 1};
    for (int li = 0; li < 4; ++li)
      for (int b = 0; b < blocks[li]; ++b) {
        const std::string p = "backbone.layer" + std::to_string(li + 1) + "." + std::to_string(b);
        const int stv = b == 0 ? strides[li] : 1;
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
        H = Ho;
      }
    // projector (template.py:34-39): ReLU (idempotent on the post-ReLU backbone output) ->
    // 1x1 2048->256 -> ReLU -> 1x1 256->D (no bias, no BN)
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
};
