// nope_b200 -- engine of the pose-conditioned UNet (include/nope_b200.h, nope_unet_*).
//
// The engine owns the repacked UNet weights, a per-chunk activation workspace and the
// layer schedule of UNet.forward (reference:
// src/model/u_net/denoising_diffusion_pytorch/u_net.py:160-198), batched over all pose
// hypotheses of a chunk.  Host code is plain C++; kernels live in conv_tc2.cuh (convolution, with
// conv_tc.cuh) / kernels.cuh / linattn_tc.cuh.
#pragma once
#include "conv_tc2.cuh"
#include "engine.cuh"
#include "kernels.cuh"
#include "linattn_tc.cuh"
#include "rank.cuh"

#include <algorithm>
#include <cstring>
#include <map>
#include <string>
#include <vector>

namespace nope {

constexpr int kHeadsHidden = 128;  // 4 heads x 32 (model_utils.py:368,394)

struct NormLayer {
  float* gamma = nullptr;
  float* beta = nullptr;
  int C = 0, G = 1;
};

// NHWC fp16 activation [n_img, S, S, C]; `lo` carries the fp16 remainder x - fp16(x) in the
// split-precision mode (nullptr otherwise)
struct Act {
  __half* hi = nullptr;
  __half* lo = nullptr;
  int C = 0;
  Act() {}
  Act(__half* h, int c, __half* l = nullptr) : hi(h), lo(l), C(c) {}
};

// what the fused epilogue applies after the convolution (ResnetBlock / Block / to_out)
struct GnSpec {
  const NormLayer* norm = nullptr;   // nullptr: no normalisation
  bool silu = false;
  int pb_offset = -1;                // pose-projection columns of this block, -1: none
  Act res;                           // residual (hi == nullptr: none)
  int res_div = 0, res_base = 0;     // residual image = (res_base + img) / res_div (hoisted prefix)
  float2* emit = nullptr;            // GroupNorm(1) partial sums of the output for a following pre-norm
  const float2* pre_stats = nullptr; // folded pre-norm: partial sums of the INPUT images ([img][pre_parts])
  int pre_parts = 0;
};

struct UNetEngine {
  static constexpr const char* kName = "UNet";
  int dim = 0, Cl = 0, S0 = 0, rot_dim = 6, cemb = 0, device = 0, num_sms = 132;
  int dims[5] = {0, 0, 0, 0, 0};
  bool finalized = false;
  // 0: fp16 operands; 1: exact weights (W_hi + W_lo K-segments, 2x the MMA work); 2: split precision
  // (exact weights + activations carried as hi + lo: A_hi W_hi + A_hi W_lo + A_lo W_hi, 3x);
  // 3: bf16 operands and activations (8-bit mantissa: its own, looser tolerance)
  int precision = 0;
  int metric = 0;            // NOPE_METRIC_* of the fused scoring
  float occ_threshold = 0.2f;
  int chunk = 642;
  int64_t launches = 0;

  StagedWeights staged;

  std::map<std::string, ConvLayer> convs;
  std::map<std::string, NormLayer> norms;
  std::map<std::string, int> pb_off;
  int P = 0;  // total pose-projection width
  ConvLayer poseproj;
  float *pose_w = nullptr, *pose_b = nullptr, *init_w = nullptr, *init_b = nullptr,
        *final_w = nullptr, *final_b = nullptr;
  DeviceAllocs mem;  // every weight buffer

  // workspace: one slab, either caller-provided (nope_unet_set_workspace) or owned
  int cap = 0, cap_ref = 0, scores_cap = 0;
  WorkspaceSlab ws;
  bool ws_fresh = false;            // counters not zeroed yet
  Act sk[4][2];
  Act TB, TC, TD, XA, XB, RB;
  __half *cs = nullptr, *pb = nullptr;
  Act x0, g1;                       // per-reference pre-stage
  float2* SB = nullptr;           // GroupNorm(1) partial sums a fused epilogue emits for the next pre-norm
  uint2* xpart = nullptr;         // fused GroupNorm: cross-tile partial sums, {value, epoch} words
  size_t xpart_words = 0;
  unsigned gn_epoch = 0;          // tag of the last fused launch that exchanged partial sums
  int* ref_of = nullptr;
  float* score_partial = nullptr;
  float* sim_buf = nullptr;

  TmapCache tmaps;

  // per-launch profile of the convolution kernel: records carry shape (GEMM resolution, mode (prof_mode), Cout, K)
  LaunchProfile prof;
  DebugTap dtap;

  bool split() const { return precision == 2 || precision == 4; }
  // precision 4: the residual stream, skip tensors and resampled maps keep their (hi, lo) pair, the tensor INSIDE a
  // ResnetBlock (block1's output h, consumed only by block2's convolution) is a single fp16 value -- block2 runs two
  // products per tap instead of three.  CPU budget (tools/precision_sim.py): h alone costs 4.3e-4 on the embeddings.
  bool h_lo() const { return precision == 2; }
  bool bf() const { return precision == 3; }     // bf16 storage (BASELINE configs[2]); fp16 otherwise

  // ------------------------------------------------------------------ schema
  void expect(const std::string& k, std::vector<int64_t> s) { staged.expect(k, std::move(s)); }
  void expect_resblock(const std::string& p, int cin, int cout, bool mlp = true) {
    if (mlp) {
      expect(p + ".mlp.1.weight", {cout, cemb});
      expect(p + ".mlp.1.bias", {cout});
    }
    expect(p + ".block1.proj.weight", {cout, cin, 3, 3});
    expect(p + ".block1.proj.bias", {cout});
    expect(p + ".block1.norm.weight", {cout});
    expect(p + ".block1.norm.bias", {cout});
    expect(p + ".block2.proj.weight", {cout, cout, 3, 3});
    expect(p + ".block2.proj.bias", {cout});
    expect(p + ".block2.norm.weight", {cout});
    expect(p + ".block2.norm.bias", {cout});
    if (cin != cout) {
      expect(p + ".res_conv.weight", {cout, cin, 1, 1});
      expect(p + ".res_conv.bias", {cout});
    }
  }
  void expect_linattn(const std::string& p, int d) {
    expect(p + ".fn.fn.to_qkv.weight", {3 * kHeadsHidden, d, 1, 1});
    expect(p + ".fn.fn.to_out.0.weight", {d, kHeadsHidden, 1, 1});
    expect(p + ".fn.fn.to_out.0.bias", {d});
    expect(p + ".fn.fn.to_out.1.weight", {d});
    expect(p + ".fn.fn.to_out.1.bias", {d});
    expect(p + ".fn.norm.weight", {d});
    expect(p + ".fn.norm.bias", {d});
  }
  // state_dict schema of the reference UNet (u_net.py:27-158), encoder excluded.
  void build_schema() {
    expect("pose_mlp.0.weight", {cemb, rot_dim});
    expect("pose_mlp.0.bias", {cemb});
    expect("init_conv.weight", {dim, Cl, 3, 3});
    expect("init_conv.bias", {dim});
    for (int i = 0; i < 4; ++i) {
      const int din = dims[i], dout = dims[i + 1];
      const std::string p = "downs." + std::to_string(i);
      expect_resblock(p + ".0", din, din);
      expect_resblock(p + ".1", din, din);
      expect_linattn(p + ".2", din);
      if (i < 3) {
        expect(p + ".3.1.weight", {dout, din * 4, 1, 1});
        expect(p + ".3.1.bias", {dout});
      } else {
        expect(p + ".3.weight", {dout, din, 3, 3});
        expect(p + ".3.bias", {dout});
      }
    }
    const int mid = dims[4];
    expect("mid_attn.fn.fn.to_qkv.weight", {3 * kHeadsHidden, mid, 1, 1});
    expect("mid_attn.fn.fn.to_out.weight", {mid, kHeadsHidden, 1, 1});
    expect("mid_attn.fn.fn.to_out.bias", {mid});
    expect("mid_attn.fn.norm.weight", {mid});
    expect("mid_attn.fn.norm.bias", {mid});
    expect_resblock("mid_block1", mid, mid);
    expect_resblock("mid_block2", mid, mid);
    for (int j = 0; j < 4; ++j) {
      const int din = dims[3 - j], dout = dims[4 - j];
      const std::string p = "ups." + std::to_string(j);
      expect_resblock(p + ".0", dout + din, dout);
      expect_resblock(p + ".1", dout + din, dout);
      expect_linattn(p + ".2", dout);
      if (j < 3) {
        expect(p + ".3.1.weight", {din, dout, 3, 3});
        expect(p + ".3.1.bias", {din});
      } else {
        expect(p + ".3.weight", {din, dout, 3, 3});
        expect(p + ".3.bias", {din});
      }
    }
    expect_resblock("final_res_block", 2 * dim, dim);
    expect_resblock("final_conv.0", dim, dim);  // owns an unused mlp.1 (u_net.py:154-157)
    expect("final_conv.1.weight", {Cl, dim, 1, 1});
    expect("final_conv.1.bias", {Cl});
  }

  // ------------------------------------------------------------------ weights
  int upload_f32(const std::string& key, float** out) { return mem.upload(out, staged.at(key).data); }
  // the code of L's shape in the profile's mode column (tools/conv_class_table.py reads it): 0 3x3, 1 1x1,
  // 2 unshuffle, 3 folded upsample -- the mode ints of nope_op_conv*
  static int prof_mode(const ConvLayer& L) { return L.up ? 3 : L.stride == 2 ? 2 : L.k == 3 ? 0 : 1; }

  // pack one conv weight (+ bias) into a layer of the given shape (an unshuffle weight's input channel index is
  // c * 4 + tap; an upsample's 3x3 kernel is folded into four 2x2 parity kernels).  The exact-weight precisions
  // (1, 2, 4) add the W_lo plane: rows are [W_hi (K) | W_lo (K)].
  int make_conv(const std::string& name, const std::string& wkey, const std::string& bkey, ConvLayer L) {
    const HostTensor& W = staged.at(wkey);
    const auto& sh = W.shape;
    const int taps = L.k * L.k;
    L.cout = (int)sh[0];
    L.cin = L.stride == 2 ? (int)sh[1] / 4 : (int)sh[1];
    L.K = L.cin * taps;
    L.wlo = precision == 1 || precision == 2 || precision == 4;
    NOPE_CHECK(L.cin % 64 == 0, wkey + ": input channels must be a multiple of 64");
    NOPE_CHECK(pick_bn(L.cout) != 0, wkey + ": output channels must be a multiple of 64");
    NOPE_CHECK(!L.up || (sh.size() == 4 && sh[2] == 3 && sh[3] == 3), wkey + ": expected a 3x3 kernel");
    if (pack_conv_layer(mem, L, {{W.data.data(), L.cout, L.cin, taps, 0, 0}},
                        bkey.empty() ? std::vector<float>() : staged.at(bkey).data, bf()))
      return -1;
    convs[name] = L;
    return 0;
  }
  int make_norm(const std::string& name, const std::string& prefix, int G) {
    NormLayer n;
    n.C = (int)staged.at(prefix + ".weight").shape[0];
    n.G = G;
    NOPE_CHECK(n.C % (8 * G) == 0, prefix + ": channels per group must be a multiple of 8");
    if (upload_f32(prefix + ".weight", &n.gamma)) return -1;
    if (upload_f32(prefix + ".bias", &n.beta)) return -1;
    norms[name] = n;
    return 0;
  }
  int make_resblock(const std::string& p) {
    if (make_conv(p + ".block1", p + ".block1.proj.weight", p + ".block1.proj.bias", conv3x3())) return -1;
    if (make_conv(p + ".block2", p + ".block2.proj.weight", p + ".block2.proj.bias", conv3x3())) return -1;
    if (make_norm(p + ".norm1", p + ".block1.norm", 8)) return -1;
    if (make_norm(p + ".norm2", p + ".block2.norm", 8)) return -1;
    if (staged.has(p + ".res_conv.weight"))
      if (make_conv(p + ".res", p + ".res_conv.weight", p + ".res_conv.bias", conv1x1())) return -1;
    return 0;
  }
  // to_qkv with the PreNorm GroupNorm(1) folded in (model_utils.py:226-234, 399): packed weights
  // W' = W diag(gamma); w1[c] = sum_k W'[c,k] over the values the tensor core actually multiplies
  // (fp16 hi, + lo in the exact-weight modes); wb[c] = sum_k W[c,k] beta[k].
  int make_qkv_folded(const std::string& name, const std::string& wkey, const std::string& nprefix) {
    const HostTensor& W = staged.at(wkey);
    const std::vector<float>& gm = staged.at(nprefix + ".weight").data;
    const std::vector<float>& bt = staged.at(nprefix + ".bias").data;
    const int rows = (int)W.shape[0], cin = (int)W.shape[1];
    HostTensor Wf;
    Wf.shape = W.shape;
    Wf.data.resize(W.data.size());
    std::vector<float> w1(rows), wb(rows);
    for (int o = 0; o < rows; ++o) {
      double s1 = 0.0, sb = 0.0;
      for (int k = 0; k < cin; ++k) {
        const float w = W.data[(size_t)o * cin + k];
        const float wf = w * gm[k];
        Wf.data[(size_t)o * cin + k] = wf;
        if (precision == 3) {
          uint32_t u;
          std::memcpy(&u, &wf, 4);
          u = (u + 0x7fffu + ((u >> 16) & 1u)) & 0xffff0000u;        // round to nearest even bf16
          float r;
          std::memcpy(&r, &u, 4);
          s1 += (double)r;
        } else {
          const __half hi = __float2half_rn(wf);
          s1 += (double)__half2float(hi);
          if (precision >= 1) s1 += (double)__half2float(__float2half_rn(wf - __half2float(hi)));
        }
        sb += (double)w * (double)bt[k];
      }
      w1[o] = (float)s1;
      wb[o] = (float)sb;
    }
    const std::string tmpkey = "__folded." + name;
    staged.put(tmpkey, std::move(Wf));
    if (make_conv(name, tmpkey, "", conv1x1())) return -1;
    ConvLayer& L = convs[name];
    return mem.upload(&L.pre_w1, w1) || mem.upload(&L.pre_wb, wb) ? -1 : 0;
  }
  int make_linattn(const std::string& p) {
    if (make_qkv_folded(p + ".qkvf", p + ".fn.fn.to_qkv.weight", p + ".fn.norm")) return -1;
    if (make_conv(p + ".out", p + ".fn.fn.to_out.0.weight", p + ".fn.fn.to_out.0.bias", conv1x1())) return -1;
    if (make_norm(p + ".outnorm", p + ".fn.fn.to_out.1", 1)) return -1;
    return 0;
  }
  // concatenate the 19 pose projections (model_utils.py:261-263) into one [P, cemb] GEMM
  int make_poseproj() {
    std::vector<std::string> blocks;
    for (int i = 0; i < 4; ++i)
      for (int b = 0; b < 2; ++b) blocks.push_back("downs." + std::to_string(i) + "." + std::to_string(b));
    blocks.push_back("mid_block1");
    blocks.push_back("mid_block2");
    for (int j = 0; j < 4; ++j)
      for (int b = 0; b < 2; ++b) blocks.push_back("ups." + std::to_string(j) + "." + std::to_string(b));
    blocks.push_back("final_res_block");
    std::vector<float> w, bias;
    P = 0;
    for (const auto& b : blocks) {
      const HostTensor& hw = staged.at(b + ".mlp.1.weight");
      const HostTensor& hb = staged.at(b + ".mlp.1.bias");
      pb_off[b] = P;
      P += (int)hw.shape[0];
      w.insert(w.end(), hw.data.begin(), hw.data.end());
      bias.insert(bias.end(), hb.data.begin(), hb.data.end());
    }
    HostTensor tw;
    tw.shape = {P, cemb, 1, 1};
    tw.data = std::move(w);
    HostTensor tb;
    tb.shape = {P};
    tb.data = std::move(bias);
    staged.put("__poseproj.weight", std::move(tw));
    staged.put("__poseproj.bias", std::move(tb));
    if (make_conv("__poseproj", "__poseproj.weight", "__poseproj.bias", conv1x1())) return -1;
    poseproj = convs["__poseproj"];
    return 0;
  }

  // packs the staged weights (engine_finalize: every schema key is present, device selected)
  int finalize() {
    if (upload_f32("pose_mlp.0.weight", &pose_w) || upload_f32("pose_mlp.0.bias", &pose_b) ||
        upload_f32("init_conv.weight", &init_w) || upload_f32("init_conv.bias", &init_b) ||
        upload_f32("final_conv.1.weight", &final_w) || upload_f32("final_conv.1.bias", &final_b))
      return -1;
    for (int i = 0; i < 4; ++i) {
      const std::string p = "downs." + std::to_string(i);
      if (make_resblock(p + ".0") || make_resblock(p + ".1") || make_linattn(p + ".2")) return -1;
      if (i < 3) {
        if (make_conv(p + ".3", p + ".3.1.weight", p + ".3.1.bias", conv_unshuffle())) return -1;
      } else {
        if (make_conv(p + ".3", p + ".3.weight", p + ".3.bias", conv3x3())) return -1;
      }
    }
    if (make_resblock("mid_block1") || make_resblock("mid_block2")) return -1;
    if (make_qkv_folded("mid_attn.qkvf", "mid_attn.fn.fn.to_qkv.weight", "mid_attn.fn.norm")) return -1;
    if (make_conv("mid_attn.out", "mid_attn.fn.fn.to_out.weight", "mid_attn.fn.fn.to_out.bias", conv1x1()))
      return -1;
    for (int j = 0; j < 4; ++j) {
      const std::string p = "ups." + std::to_string(j);
      if (make_resblock(p + ".0") || make_resblock(p + ".1") || make_linattn(p + ".2")) return -1;
      if (j < 3) {
        if (make_conv(p + ".3", p + ".3.1.weight", p + ".3.1.bias", conv_upsample3x3())) return -1;
      } else {
        if (make_conv(p + ".3", p + ".3.weight", p + ".3.bias", conv3x3())) return -1;
      }
    }
    if (make_resblock("final_res_block") || make_resblock("final_conv.0")) return -1;
    return make_poseproj();
  }

  // ------------------------------------------------------------------ workspace
  // One slab carved by a bump allocator: ~4.7 MB per hypothesis at u_net_dim 192 (8.6 MB in the split-precision
  // modes), nearly all of it the 8 skip tensors, 3 temporaries of 786 KB and 3 feature maps of 393 KB.
  // layout(b) assigns every buffer for capacities (c hypotheses, r references).
  void take_act(Bump& b, Act* a, size_t n, int C, bool with_lo) {
    if (b.base) {
      a->C = C;
      a->lo = nullptr;
    }
    b.take(&a->hi, n);
    if (with_lo) b.take(&a->lo, n);
  }
  size_t layout(Bump& b, int c_hyp, int c_ref, int n_total_scores) {
    const size_t c = (size_t)c_hyp, r = (size_t)c_ref;
    const bool lo = precision == 2 || precision == 4;
    // temporaries hold the widest full-resolution tensor: a concat-conv output (<= 2*dim
    // channels) or the attention qkv tensor (3 x 128 channels, independent of dim)
    const size_t big = (size_t)S0 * S0 * std::max(dim * 2, 3 * kHeadsHidden);
    const size_t xsz = (size_t)S0 * S0 * dim;      // one full-resolution feature map
    for (int i = 0; i < 4; ++i) {
      const int s = S0 >> i;
      for (int k = 0; k < 2; ++k) take_act(b, &sk[i][k], c * s * s * dims[i], dims[i], lo);
    }
    take_act(b, &TB, c * big, 0, lo);
    take_act(b, &TC, c * big, 0, lo);
    take_act(b, &TD, c * big, 0, false);
    take_act(b, &XA, c * xsz, 0, lo);
    take_act(b, &XB, c * xsz, 0, lo);
    take_act(b, &RB, c * xsz, dim, lo);
    b.take(&cs, c * cemb);
    b.take(&pb, c * (size_t)P);
    take_act(b, &x0, r * xsz, dim, lo);
    take_act(b, &g1, r * xsz, dim, lo);
    const size_t m = std::max(c, r);
    b.take(&ref_of, m);
    b.take(&SB, m * 8);
    // <= 64 (slot, image, group) entries of two {value, epoch} words per image
    if (b.base) xpart_words = (m + 8) * 64 * 2;
    b.take(&xpart, (m + 8) * 64 * 2);
    b.take(&score_partial, (size_t)n_total_scores * nslab() * kScoreParts);
    b.take(&sim_buf, (size_t)n_total_scores);
    return b.off;
  }
  size_t workspace_bytes(int c_hyp, int c_ref, int n_scores) {
    Bump b;
    return layout(b, c_hyp, c_ref, n_scores) + 256;
  }
  // no allocation when the slab fits (always, with a caller-provided one); otherwise the engine grows its own slab
  // (device synchronisation + cudaMalloc on growth only)
  int ensure_workspace(int need_cap, int need_ref, int need_scores, cudaStream_t st) {
    if (need_cap > cap || need_ref > cap_ref || need_scores > scores_cap) {
      NOPE_CHECK(!ws.external, "the caller-provided workspace is too small for this sweep "
                               "(nope_unet_workspace_bytes / nope_unet_set_workspace)");
      if (adopt(nullptr, std::max(cap, need_cap), std::max(cap_ref, need_ref), std::max(scores_cap, need_scores)))
        return -1;
    }
    // the tile-sync words of a fresh slab carry epoch 0, which no launch uses
    if (ws_fresh) {
      NOPE_CUDA(cudaMemsetAsync(xpart, 0, xpart_words * sizeof(uint2), st));
      ws_fresh = false;
    }
    return 0;
  }
  // the workspace in `external` (a caller's buffer), or in a slab of the engine's own when null
  int adopt(void* external, int c, int r, int sc) {
    if (grow_workspace(this, std::tie(cap, cap_ref, scores_cap), external, c, r, sc)) return -1;
    ws_fresh = true;
    return 0;
  }
  int set_workspace(void* ptr, size_t bytes, int c, int r, int sc) {
    NOPE_CHECK(ptr && c >= 1 && r >= 1, "bad workspace arguments");
    NOPE_CHECK(bytes >= workspace_bytes(c, r, sc), "workspace buffer smaller than nope_unet_workspace_bytes");
    return adopt(ptr, c, r, sc);
  }

  // ------------------------------------------------------------------ op launchers
  // out[n_img, So, So, cout] = conv(L, in0 (++ in1)).  The K loop walks, per filter tap and source
  // tensor, up to three products: A_hi W_hi, A_hi W_lo (layers with a W_lo plane), A_lo W_hi (sources that
  // carry a remainder).  `gs` selects the fused GroupNorm epilogue; `stats` (plain epilogue only) receives the
  // GroupNorm partial sums of the output in the ConvParams::stats layout (nope_op_conv_gn checks them).
  int conv(const ConvLayer& L, const Act& in0, const Act& in1, const Act& out, int So, int n_img, int cap_img,
           cudaStream_t st, const GnSpec* gs = nullptr, float2* stats = nullptr) {
    const int c0 = in0.C, c1 = in1.hi ? in1.C : 0;
    NOPE_CHECK(c0 + c1 == L.cin, "conv: channel mismatch");
    NOPE_CHECK(!L.up || (in1.hi == nullptr && So % 2 == 0), "upsample conv takes one source");
    NOPE_CHECK(L.stride == 1 || in1.hi == nullptr, "unshuffle conv takes one source");
    ++launches;
    // the folded upsample's So is the OUTPUT side (2x the source side); tiles and input maps use the source geometry
    const int Sg = L.up ? So / 2 : So;
    TileGeom g;
    if (make_geom(Sg, Sg, &g)) return -1;
    ConvBuilder b(tmaps, g, cap_img);
    ConvParams& p = b.p;
    std::vector<ConvSrc> src{b.src(in0.hi, in0.lo, c0, L.stride == 2 ? 4 : 1)};
    if (in1.hi) src.push_back(b.src(in1.hi, in1.lo, c1));
    b.segs(L.taps(), src, 0, L.wlo ? L.K : 0);
    if (b.finish(L, out.hi, L.cout, n_img, L.up ? 4 : 1)) return -1;
    p.bf16 = bf() ? 1 : 0;
    p.stats = stats;
    NOPE_CHECK(!(stats && L.up), "fused statistics are not available on the upsample conv");
    if (gs) {
      NOPE_CHECK(!L.up && !stats, "fused GroupNorm epilogue: no upsample, no plain statistics");
      GnFuse& f = p.gn;
      const int hw = So * So;
      f.G = gs->norm ? gs->norm->G : 0;
      if (gs->norm) {
        NOPE_CHECK(gs->norm->C == L.cout, "fused GroupNorm: channel mismatch");
        f.gamma = gs->norm->gamma;
        f.beta = gs->norm->beta;
        f.cpg = L.cout / f.G;
        NOPE_CHECK(f.cpg % 8 == 0 && (f.cpg >= L.bn ? f.cpg % L.bn == 0 : L.bn % f.cpg == 0),
                   "fused GroupNorm: groups must tile the channel tiles");
      } else {
        f.cpg = L.cout;
      }
      f.gpt = std::max(1, L.bn / f.cpg);
      f.tpg = std::max(1, f.cpg / L.bn);
      f.mt = std::max(1, g.tiles_per_img);
      f.ipt = g.tiles_per_img > 0 ? 1 : g.b_cnt;
      f.expected = f.G > 0 ? f.mt * f.tpg : 1;
      int sh = 0;
      while ((1 << sh) < hw) ++sh;
      NOPE_CHECK((1 << sh) == hw, "fused GroupNorm: H*W must be a power of two");
      f.hw_shift = sh;
      f.inv_cnt = 1.0f / ((float)hw * (float)f.cpg);
      f.eps = 1e-5f;
      f.silu = gs->silu ? 1 : 0;
      f.pb = gs->pb_offset >= 0 ? pb : nullptr;
      f.pb_stride = P;
      f.pb_off = std::max(gs->pb_offset, 0);
      f.n_img = n_img;
      if (gs->res.hi) {
        NOPE_CHECK(gs->res.C == L.cout, "fused residual: channel mismatch");
        NOPE_CHECK(gs->res_div == 0 || g.tiles_per_img > 0, "residual image mapping needs >= 128-pixel images");
        const CUtensorMap* m = nullptr;
        if (tmaps.get(&m, gs->res.hi, gs->res_div > 0 ? cap_ref : cap_img, L.cout, g, -1)) return -1;
        p.rmap = *m;
        f.has_res = 1;
        f.res_lo = gs->res.lo;
      } else {
        p.rmap = p.omap[0];
      }
      f.res_div = gs->res_div;
      f.res_base = gs->res_base;
      if (gs->pre_stats) {
        NOPE_CHECK(!gs->norm && L.pre_w1 && L.pre_wb && L.k == 1 && L.stride == 1 && !L.bias,
                   "pre-norm fold: bias-free 1x1 layer with folded weights");
        f.pre_stats = gs->pre_stats;
        f.pre_parts = gs->pre_parts;
        f.pre_inv_cnt = 1.0f / ((float)hw * (float)L.cin);
        f.pre_w1 = L.pre_w1;
        f.pre_wb = L.pre_wb;
      }
      f.out_lo = out.lo;
      f.emit = gs->emit;
      f.emit_parts = f.mt * p.n_tiles;
      NOPE_CHECK(f.ipt * f.gpt <= 64 && f.ipt <= 8, "fused GroupNorm: tile holds too many (image, group) pairs");
      if (f.expected > 1) {
        const size_t n_sg = (size_t)(p.m_tiles / f.mt + 1) * (p.n_tiles / f.tpg);
        NOPE_CHECK(xpart && f.expected * f.ipt * f.gpt * 2 <= 256, "fused GroupNorm: sync group too large");
        NOPE_CHECK(n_sg * f.expected * f.ipt * f.gpt * 2 <= xpart_words, "fused GroupNorm: partial-sum buffer too small");
        f.xpart = xpart;
        if (++gn_epoch == 0) ++gn_epoch;     // 0 is the tag of a fresh buffer
        f.epoch = gn_epoch;
      }
    } else if (out.lo) {
      p.out_lo = out.lo;                // extras epilogue writes the remainder
    }
    auto launch = [&]() {
      return gs ? launch_conv_gn(p, L.bn, num_sms, st) : launch_conv_tc2(p, L.bn, num_sms, st);
    };
    if (prof.begin(st)) return -1;
    const int rc = launch();
    // executed FLOPs: the folded upsample runs 4 parity GEMMs of K = 4 Cin over the source-resolution pixels;
    // the split-precision modes execute 2x / 3x the K-steps of the fp16 mode
    const double px = 2.0 * (double)n_img * So * So * (double)L.cout;
    if (prof.end(st, {px * (double)p.ksteps * 64.0, px * (double)L.K, 0, make_int4(So, prof_mode(L), L.cout, L.K)}))
      return -1;
    return rc;
  }

  // partial sums per image emitted by the fused epilogue: one per (M-tile of the image, N-tile)
  static int fused_emit_parts(int S, int C) {
    return std::max(1, S * S / kBM) * (C / pick_bn(C));
  }

  int tap(const char* name, const Act& buf, int C, int S, int n, cudaStream_t st) {
    return dtap.capture(name, buf.hi, buf.lo, bf(), C, S, n, st);
  }

  // ResnetBlock.forward (model_utils.py:271-279) on NHWC fp16:
  // conv1 [GN8 + SiLU + pose bias] -> h ; (res_conv) ; conv2 [GN8 + SiLU + residual] -> out:
  // two or three launches, no tensor is written un-normalised.  `emit_g1` makes conv2's epilogue also
  // emit the GroupNorm(1, C) statistics of the block output into SB for a following attention pre-norm.
  int resblock(const std::string& p, const Act& in0, const Act& in1, const Act& out, int S, int n, bool pose,
               cudaStream_t st, bool emit_g1 = false, int res_div = 0, int res_base = 0, const Act* hoisted_h = nullptr) {
    const ConvLayer& b1 = convs.at(p + ".block1");
    const ConvLayer& b2 = convs.at(p + ".block2");
    const int co = b1.cout;
    auto it = convs.find(p + ".res");
    Act h(TB.hi, co, h_lo() ? TB.lo : nullptr);
    if (hoisted_h) {
      h = *hoisted_h;
      if (!h_lo()) h.lo = nullptr;
    } else {
      GnSpec s1;
      s1.norm = &norms.at(p + ".norm1");
      s1.silu = true;
      s1.pb_offset = pose ? pb_off.at(p) : -1;
      if (conv(b1, in0, in1, h, S, n, cap, st, &s1)) return -1;
    }
    GnSpec s2;
    s2.norm = &norms.at(p + ".norm2");
    s2.silu = true;
    if (it != convs.end()) {
      Act r(TC.hi, co, split() ? TC.lo : nullptr);
      // plain epilogue: routing this 1x1 through the GroupNorm-fused role split measured 8 % slower
      if (conv(it->second, in0, in1, r, S, n, cap, st)) return -1;
      s2.res = r;
    } else {
      NOPE_CHECK(in1.hi == nullptr && in0.C == co, "resblock: identity residual needs Cin == Cout");
      s2.res = in0;
      s2.res_div = res_div;
      s2.res_base = res_base;
    }
    s2.emit = emit_g1 ? SB : nullptr;
    return conv(b2, h, Act(), out, S, n, cap, st, &s2);
  }

  // Residual(PreNorm(LinearAttention)) (model_utils.py:393-418).  x's GroupNorm(1) statistics
  // were emitted into SB by the producer of x; to_out[1] (GroupNorm(1)) + the residual add run in the
  // to_out convolution's epilogue.
  int linattn(const std::string& p, const Act& x, const Act& out, int C, int S, int n, cudaStream_t st) {
    // pre-norm folded into to_qkv: x is read once, un-normalised, by the 1x1 itself
    GnSpec sq;
    sq.pre_stats = SB;
    sq.pre_parts = fused_emit_parts(S, C);
    if (conv(convs.at(p + ".qkvf"), x, Act(), Act(TD.hi, 3 * kHeadsHidden), S, n, cap, st, &sq)) return -1;
    if (S * S >= kBM) {
      if (launch_linattn_tc(TD.hi, TC.hi, n, S * S, num_sms, st, bf())) return -1;
    } else {
      NOPE_CUDA(launch_pdl(linattn_kernel, dim3(4, n), dim3(kLinAttnThreads), 0, st, TD.hi, TC.hi, S * S, bf()));
    }
    ++launches;
    // to_out (K = 128: two K-steps per tile) + GroupNorm(1) + residual in one kernel.  This takes the same time as
    // the plain convolution plus one normalisation pass (18.80 vs 18.71 ms over the step under ncu), and it never
    // rounds the un-normalised output to 16 bits (full-size configs[2] scores: 0.99e-3 vs 1.06e-3)
    GnSpec so;
    so.norm = &norms.at(p + ".outnorm");
    so.res = x;
    return conv(convs.at(p + ".out"), Act(TC.hi, kHeadsHidden), Act(), out, S, n, cap, st, &so);
  }

  // Residual(PreNorm(Attention)) (model_utils.py:367-390)
  int midattn(const Act& x, const Act& out, int C, int S, int n, cudaStream_t st) {
    NOPE_CHECK(S * S <= 32, "bottleneck attention supports at most 32 tokens");
    GnSpec sq;
    sq.pre_stats = SB;
    sq.pre_parts = fused_emit_parts(S, C);
    if (conv(convs.at("mid_attn.qkvf"), x, Act(), Act(TD.hi, 3 * kHeadsHidden), S, n, cap, st, &sq)) return -1;
    NOPE_CUDA(launch_pdl(midattn_kernel, dim3(n), dim3(128), 0, st, TD.hi, TC.hi, S * S, bf()));
    ++launches;
    GnSpec so;                 // no normalisation: out = to_out(attn) + x
    so.res = x;
    return conv(convs.at("mid_attn.out"), Act(TC.hi, kHeadsHidden), Act(), out, S, n, cap, st, &so);
  }

  // pose-independent prefix, once per reference image: x0 = init_conv(ref),
  // g1 = SiLU(GN(downs.0.0.block1.proj(x0)))   (u_net.py:161; model_utils.py:272)
  int prestage(const float* ref_feat, int B, cudaStream_t st) {
    init_conv_kernel<<<ew_grid((long long)B * S0 * S0 * dim), 256, 0, st>>>(ref_feat, init_w, init_b, x0.hi,
                                                                            B, Cl, S0, S0, dim, split() ? x0.lo : nullptr, bf());
    NOPE_CUDA(cudaGetLastError());
    ++launches;
    const Act xin(x0.hi, dim, split() ? x0.lo : nullptr);
    GnSpec s;
    s.norm = &norms.at("downs.0.0.norm1");
    s.silu = true;
    return conv(convs.at("downs.0.0.block1"), xin, Act(), Act(g1.hi, dim, h_lo() ? g1.lo : nullptr), S0, B,
                cap_ref, st, &s);
  }

  // UNet.forward for hypotheses [hyp0, hyp0 + n) of the flattened (b, pose) list
  // query_feat [B, Q, Cl, hw]; score_part [B * N, Q, nslab, kScoreParts]; vis (optional) [B, Q, hw] visible maps
  int forward_chunk(const float* poses, int hyp0, int n, int N, const float* query_feat,
                    float* out_emb, float* score_part, cudaStream_t st, int Q = 1, const uint8_t* vis = nullptr) {
    const bool sp = split();
    auto A = [&](const Act& buf, int C) { return Act(buf.hi, C, sp ? buf.lo : nullptr); };
    ref_of_kernel<<<(n + 255) / 256, 256, 0, st>>>(ref_of, hyp0, N, n);
    ++launches;
    // pose embedding + all 19 pose projections in one GEMM
    NOPE_CUDA(launch_pdl(pose_embed_kernel, dim3(n), dim3(256), 0, st, poses + (size_t)hyp0 * rot_dim, pose_w, pose_b,
                         cs, n, rot_dim, cemb, bf()));
    ++launches;
    if (conv_pose(n, st)) return -1;

    // r (= init_conv output) and the hoisted block1 output, broadcast per hypothesis
    const int hw0 = S0 * S0;
    NOPE_CUDA(launch_pdl(bcast_add_kernel, dim3(ew_grid((long long)hw0 * dim / 8 / 4), n), dim3(256), 0, st, x0.hi, ref_of,
                         nullptr, 0, 0, RB.hi, n, hw0, dim, sp ? x0.lo : nullptr, sp ? RB.lo : nullptr, bf()));
    NOPE_CUDA(launch_pdl(bcast_add_kernel, dim3(ew_grid((long long)hw0 * dim / 8 / 4), n), dim3(256), 0, st, g1.hi, ref_of,
                         pb, P, pb_off.at("downs.0.0"), TB.hi, n, hw0, dim, h_lo() ? g1.lo : nullptr,
                         h_lo() ? TB.lo : nullptr, bf()));
    launches += 2;
    if (tap("init_conv", A(RB, dim), dim, S0, n, st)) return -1;

    // ---- downs
    Act cur;
    int S = S0;
    for (int i = 0; i < 4; ++i) {
      const int C = dims[i];
      const std::string p = "downs." + std::to_string(i);
      const Act s0 = A(sk[i][0], C), s1 = A(sk[i][1], C);
      if (i == 0) {
        // block 0 with its block1 half hoisted: TB already holds SiLU(GN(conv(x0))) + pose bias
        const Act h = A(TB, C);
        if (resblock(p + ".0", A(x0, C), Act(), s0, S, n, true, st, false, N, hyp0, &h)) return -1;
      } else {
        if (resblock(p + ".0", cur, Act(), s0, S, n, true, st)) return -1;
      }
      if (tap((p + ".0").c_str(), s0, C, S, n, st)) return -1;
      if (resblock(p + ".1", s0, Act(), A(XA, C), S, n, true, st, true)) return -1;
      if (tap((p + ".1").c_str(), A(XA, C), C, S, n, st)) return -1;
      if (linattn(p + ".2", A(XA, C), s1, C, S, n, st)) return -1;
      if (tap((p + ".2").c_str(), s1, C, S, n, st)) return -1;
      if (i < 3) S >>= 1;
      if (conv(convs.at(p + ".3"), s1, Act(), A(XB, dims[i + 1]), S, n, cap, st)) return -1;
      if (tap((p + ".3").c_str(), A(XB, dims[i + 1]), dims[i + 1], S, n, st)) return -1;
      cur = A(XB, dims[i + 1]);
    }
    // ---- mid, twice with shared weights (u_net.py:177-183)
    const int Cm = dims[4];
    Act xa = XA, xb = XB;
    for (int rep = 0; rep < 2; ++rep) {
      if (resblock("mid_block1", A(xb, Cm), Act(), A(xa, Cm), S, n, true, st, true)) return -1;
      if (midattn(A(xa, Cm), A(xb, Cm), Cm, S, n, st)) return -1;
      if (resblock("mid_block2", A(xb, Cm), Act(), A(xa, Cm), S, n, true, st)) return -1;
      if (tap(rep == 0 ? "mid.0" : "mid.1", A(xa, Cm), Cm, S, n, st)) return -1;
      std::swap(xa, xb);
    }
    Act curb = xb, othb = xa;     // buffers (channel counts vary per level)
    // ---- ups
    int ccur = Cm;
    for (int j = 0; j < 4; ++j) {
      const int din = dims[3 - j], dout = dims[4 - j];
      const std::string p = "ups." + std::to_string(j);
      if (resblock(p + ".0", A(curb, dout), A(sk[3 - j][1], din), A(othb, dout), S, n, true, st)) return -1;
      std::swap(curb, othb);
      if (tap((p + ".0").c_str(), A(curb, dout), dout, S, n, st)) return -1;
      if (resblock(p + ".1", A(curb, dout), A(sk[3 - j][0], din), A(othb, dout), S, n, true, st, true)) return -1;
      std::swap(curb, othb);
      if (linattn(p + ".2", A(curb, dout), A(othb, dout), dout, S, n, st)) return -1;
      std::swap(curb, othb);
      if (tap((p + ".2").c_str(), A(curb, dout), dout, S, n, st)) return -1;
      if (j < 3) S <<= 1;   // folded nearest-x2 + conv3x3: reads `cur` at S/2, writes `oth` at S
      if (conv(convs.at(p + ".3"), A(curb, dout), Act(), A(othb, din), S, n, cap, st)) return -1;
      std::swap(curb, othb);
      ccur = din;
      if (tap((p + ".3").c_str(), A(curb, din), din, S, n, st)) return -1;
    }
    // ---- head
    if (resblock("final_res_block", A(curb, ccur), A(RB, dim), A(othb, dim), S, n, true, st)) return -1;
    std::swap(curb, othb);
    if (tap("final_res_block", A(curb, dim), dim, S, n, st)) return -1;
    if (resblock("final_conv.0", A(curb, dim), Act(), A(othb, dim), S, n, false, st)) return -1;
    std::swap(curb, othb);
    if (tap("final_conv.0", A(curb, dim), dim, S, n, st)) return -1;
    const int hw = S * S;
    const int nslab = (hw + kFinalPix - 1) / kFinalPix;
    NOPE_CUDA(launch_pdl(vis ? final_conv_score_kernel<true> : final_conv_score_kernel<false>, dim3(nslab, n),
                         dim3(kFinalThreads), (size_t)kMaxLatent * dim * sizeof(float),
                         st, curb.hi, final_w, final_b, out_emb ? out_emb + (size_t)hyp0 * Cl * hw : nullptr, query_feat,
                         ref_of, score_part ? score_part + (size_t)hyp0 * Q * nslab * kScoreParts : nullptr, hw, dim,
                         Cl, sp ? curb.lo : nullptr, metric, occ_threshold, bf(), Q, vis));
    ++launches;
    return 0;
  }

  int conv_pose(int n, cudaStream_t st) {
    // pb[n, P] = cs[n, cemb] @ Wp^T + bp : the 1x1 "image" geometry of the conv kernel
    return conv(poseproj, Act(cs, cemb), Act(), Act(pb, P), 1, n, cap, st);
  }

  // score slabs per (hypothesis, query) of final_conv_score_kernel, each of kScoreParts partials
  int nslab() const { return (S0 * S0 + kFinalPix - 1) / kFinalPix; }
  // similarities (sim [B * Q, N]) and top-k of every (reference, query) row from the score partials
  int rank(const float* part, float* sim, int B, int N, int Q, int k, float* topv, int64_t* topi, int64_t idx_base,
           cudaStream_t st, const uint8_t* vis = nullptr) {
    NOPE_CUDA(launch_pdl(vis ? sim_topk_kernel<true> : sim_topk_kernel<false>, dim3(B * Q), dim3(256), 0, st, part,
                         nslab(), sim, N, k, topv, reinterpret_cast<long long*>(topi), (long long)idx_base, kScoreParts,
                         metric, S0 * S0, Q, vis));
    return 0;
  }
};

}  // namespace nope

// the C ABI's handle (include/nope_b200.h)
struct nope_unet : nope::UNetEngine {};
