// nope_b200 -- engine of the LDM-variant pose-conditioned UNet (SURVEY.md section 8 row f2).
//
// Reference: UNetModelPose.forward (src/model/u_net/ldm/adapt_openaimodel.py:127-158) over the
// module list UNetModel.__init__ builds (ldm/openaimodel.py:543-726) for
// configs/model/vae_cin_ldm.yaml:2-31: model_channels 256, channel_mult (1, 2, 4), 2 ResBlocks per
// level, a SpatialTransformer (heads = C / 32, depth 1, context_dim 512) after every ResBlock,
// injecting_condition_twice = false (emb = 0), context = pose_mlp(pose) as ONE token.
//
// Batched over all pose hypotheses of a chunk, NHWC fp16:
//   ResBlock          GN32+SiLU (two-source: the skip concat is never materialised before the norm)
//                     -> conv3x3 (+ emb bias) -> GN32+SiLU (statistics from the conv epilogue)
//                     -> conv3x3 with the 1x1 skip_connection (or the identity skip) folded in
//                        as extra K segments
//   SpatialTransformer GN32 (statistics from the ResBlock's last epilogue) -> proj_in -> LN ->
//                     q|k|v GEMM -> wgmma attention -> to_out (+x) -> [+cross term, LN] ->
//                     GEGLU feed-forward (+x) -> proj_out (+x_in)
//   Downsample        conv3x3 stride 2 through the four stride-2 TMA lattices of its input
//   Upsample          nearest-x2 + conv3x3 folded into four 2x2 parity kernels
//   out               GN32+SiLU -> conv3x3 (256 -> 4, padded to a 64-channel tile, fp32 store) -> l2 score
// Every GEMM-shaped op runs on conv_tc2_kernel.
#pragma once
#include "conv_tc2.cuh"
#include "engine.cuh"
#include "kernels.cuh"
#include "ldm_kernels.cuh"
#include "rank.cuh"

#include <algorithm>
#include <cmath>
#include <cstring>
#include <map>
#include <memory>
#include <string>
#include <tuple>
#include <vector>

namespace nope {

struct LdmNorm {
  float* gamma = nullptr;
  float* beta = nullptr;
  int C = 0;
};
struct LdmBlock {      // one entry of input_blocks / output_blocks
  int kind = 0;        // 0: input conv, 1: ResBlock + SpatialTransformer, 2: Downsample
  int cin = 0, cout = 0, skip_c = 0;
  bool up = false;
};

}  // namespace nope

struct nope_ldm {
  using HostTensor = nope::HostTensor;
  static constexpr const char* kName = "LDM";
  int mc = 256, ctx = 512, Cl = 4, S0 = 32, rot_dim = 6, device = 0, num_sms = 132;
  int nres = 2;
  std::vector<int> mult{1, 2, 4};
  bool finalized = false;
  bool hoist = true;        // pose-independent prefix once per reference (prestage)
  int precision = 0;        // 0: fp16 weights; 1: exact weights -- every layer has a W_lo plane and the K loop
                            // walks its segment list twice (A W_hi + A W_lo), 2x the MMA work (set before finalize)
  int chunk = 256;
  int64_t launches = 0;

  std::vector<nope::LdmBlock> inp, outp;
  int mid_ch = 0;

  nope::StagedWeights staged;
  std::map<std::string, nope::ConvLayer> convs;
  std::map<std::string, nope::LdmNorm> norms;
  std::map<std::string, int> cb_off;   // transformer prefix -> offset in the cross-term vector
  int cb_width = 0;
  float *cross_w = nullptr, *cross_b = nullptr;      // [cb_width][6], [cb_width]
  float *in_w = nullptr, *in_b = nullptr;
  nope::DeviceAllocs mem;                      // weights

  // workspace (per chunk of `cap` hypotheses; `cap_ref` reference latents; `scores_cap` scored triples)
  int cap = 0, cap_ref = 0, scores_cap = 0;
  std::vector<__half*> HS;                     // skip stack, one buffer per input block (sized by build_plan)
  __half *XA = nullptr, *XB = nullptr, *XC = nullptr, *R = nullptr, *T1 = nullptr, *T2 = nullptr,
         *T3 = nullptr, *XN = nullptr, *PI = nullptr, *PJ = nullptr, *QKV = nullptr,
         *Vt = nullptr, *AO = nullptr, *GG = nullptr, *x0ref = nullptr, *Rref = nullptr, *Pref = nullptr;
  float2 *S_in = nullptr, *S_mid = nullptr, *S_out = nullptr;
  float* cb = nullptr;
  float* OF = nullptr;                          // out[2] result, fp32 [cap * S0 * S0][64]
  int* ref_of = nullptr;
  float* score_partial = nullptr;
  float* sim_buf = nullptr;
  nope::WorkspaceSlab ws;
  nope::TmapCache tmaps;

  // per-launch profile: record kind 0 = convolution / GEMM, 1 = attention
  nope::LaunchProfile prof;
  nope::DebugTap dtap;

  // ------------------------------------------------------------------ plan + schema
  void build_plan() {
    using nope::LdmBlock;
    inp.clear();
    outp.clear();
    std::vector<int> chans;
    inp.push_back(LdmBlock{0, Cl, mc, 0, false});
    chans.push_back(mc);
    int ch = mc;
    for (size_t level = 0; level < mult.size(); ++level) {
      for (int r = 0; r < nres; ++r) {
        inp.push_back(LdmBlock{1, ch, mult[level] * mc, 0, false});
        ch = mult[level] * mc;
        chans.push_back(ch);
      }
      if (level + 1 != mult.size()) {
        inp.push_back(LdmBlock{2, ch, ch, 0, false});
        chans.push_back(ch);
      }
    }
    mid_ch = ch;
    HS.assign(inp.size(), nullptr);
    for (int level = (int)mult.size() - 1; level >= 0; --level)
      for (int i = 0; i <= nres; ++i) {
        const int ich = chans.back();
        chans.pop_back();
        outp.push_back(LdmBlock{1, ch + ich, mc * mult[level], ich, level > 0 && i == nres});
        ch = mc * mult[level];
      }
  }
  void expect(const std::string& k, std::vector<int64_t> s) { staged.expect(k, std::move(s)); }
  void expect_res(const std::string& p, int cin, int cout) {
    const int temb = 4 * mc;
    expect(p + ".in_layers.0.weight", {cin});
    expect(p + ".in_layers.0.bias", {cin});
    expect(p + ".in_layers.2.weight", {cout, cin, 3, 3});
    expect(p + ".in_layers.2.bias", {cout});
    expect(p + ".emb_layers.1.weight", {cout, temb});
    expect(p + ".emb_layers.1.bias", {cout});
    expect(p + ".out_layers.0.weight", {cout});
    expect(p + ".out_layers.0.bias", {cout});
    expect(p + ".out_layers.3.weight", {cout, cout, 3, 3});
    expect(p + ".out_layers.3.bias", {cout});
    if (cin != cout) {
      expect(p + ".skip_connection.weight", {cout, cin, 1, 1});
      expect(p + ".skip_connection.bias", {cout});
    }
  }
  void expect_st(const std::string& p, int c) {
    expect(p + ".norm.weight", {c});
    expect(p + ".norm.bias", {c});
    expect(p + ".proj_in.weight", {c, c, 1, 1});
    expect(p + ".proj_in.bias", {c});
    const std::string t = p + ".transformer_blocks.0";
    for (int a = 1; a <= 2; ++a) {
      const std::string q = t + ".attn" + std::to_string(a);
      const int kd = a == 1 ? c : ctx;
      expect(q + ".to_q.weight", {c, c});
      expect(q + ".to_k.weight", {c, kd});
      expect(q + ".to_v.weight", {c, kd});
      expect(q + ".to_out.0.weight", {c, c});
      expect(q + ".to_out.0.bias", {c});
    }
    expect(t + ".ff.net.0.proj.weight", {8 * c, c});
    expect(t + ".ff.net.0.proj.bias", {8 * c});
    expect(t + ".ff.net.2.weight", {c, 4 * c});
    expect(t + ".ff.net.2.bias", {c});
    for (int n = 1; n <= 3; ++n) {
      expect(t + ".norm" + std::to_string(n) + ".weight", {c});
      expect(t + ".norm" + std::to_string(n) + ".bias", {c});
    }
    expect(p + ".proj_out.weight", {c, c, 1, 1});
    expect(p + ".proj_out.bias", {c});
  }
  // state_dict schema of UNetModelPose without the encoder (628 tensors for the default config)
  void build_schema() {
    const int temb = 4 * mc;
    expect("time_embed.0.weight", {temb, mc});     // in the state_dict, unused by forward
    expect("time_embed.0.bias", {temb});
    expect("time_embed.2.weight", {temb, temb});
    expect("time_embed.2.bias", {temb});
    for (size_t i = 0; i < inp.size(); ++i) {
      const std::string p = "input_blocks." + std::to_string(i);
      const auto& b = inp[i];
      if (b.kind == 0) {
        expect(p + ".0.weight", {mc, Cl, 3, 3});
        expect(p + ".0.bias", {mc});
      } else if (b.kind == 1) {
        expect_res(p + ".0", b.cin, b.cout);
        expect_st(p + ".1", b.cout);
      } else {
        expect(p + ".0.op.weight", {b.cout, b.cin, 3, 3});
        expect(p + ".0.op.bias", {b.cout});
      }
    }
    expect_res("middle_block.0", mid_ch, mid_ch);
    expect_st("middle_block.1", mid_ch);
    expect_res("middle_block.2", mid_ch, mid_ch);
    for (size_t i = 0; i < outp.size(); ++i) {
      const std::string p = "output_blocks." + std::to_string(i);
      const auto& b = outp[i];
      expect_res(p + ".0", b.cin, b.cout);
      expect_st(p + ".1", b.cout);
      if (b.up) {
        expect(p + ".2.conv.weight", {b.cout, b.cout, 3, 3});
        expect(p + ".2.conv.bias", {b.cout});
      }
    }
    expect("out.0.weight", {mc});
    expect("out.0.bias", {mc});
    expect("out.2.weight", {Cl, mc, 3, 3});
    expect("out.2.bias", {Cl});
    expect("pose_mlp.0.weight", {ctx, rot_dim});
    expect("pose_mlp.0.bias", {ctx});
  }

  // accepted for schema compatibility, never read (nope_ldm_load_tensor keeps their shapes only): emb = 0
  // (adapt_openaimodel.py:143-146) and the one-token cross-attention does not depend on its queries / keys
  static bool never_read(const char* key) {
    return std::strncmp(key, "time_embed.", 11) == 0 || std::strstr(key, ".emb_layers.1.weight") ||
           std::strstr(key, ".attn2.to_q.") || std::strstr(key, ".attn2.to_k.") || std::strstr(key, ".norm2.");
  }

  // ------------------------------------------------------------------ weights
  const HostTensor& H(const std::string& k) const { return staged.at(k); }
  // packs layer L (shape, cin, cout, K and the LDM fields set) from its weight blocks -> convs[name]
  int add_conv(const std::string& name, nope::ConvLayer L, const std::vector<nope::WeightBlock>& blocks,
               const std::vector<float>& bias) {
    using namespace nope;
    if (L.k_alg == 0) L.k_alg = L.K;
    L.wlo = precision != 0;
    L.bn = (!L.geglu && L.cout % 256 == 0) ? 256 : pick_bn(L.cout);
    NOPE_CHECK(L.bn != 0 && L.K % 64 == 0, name + ": channel counts must be multiples of 64");
    if (pack_conv_layer(mem, L, blocks, bias)) return -1;
    convs[name] = L;
    return 0;
  }
  // plain convolution / linear layer of the given shape.  extra_bias (optional) is added to the bias.
  int make_conv(const std::string& name, const std::string& wkey, const std::string& bkey, nope::ConvLayer L,
                const std::string& extra_bias = "") {
    const HostTensor& W = H(wkey);
    L.cout = (int)W.shape[0];
    L.cin = (int)W.shape[1];
    const int taps = L.k * L.k;
    L.K = L.cin * taps;
    std::vector<float> bias;
    if (!bkey.empty()) {
      bias = H(bkey).data;
      if (!extra_bias.empty()) {
        const auto& e = H(extra_bias).data;
        for (size_t i = 0; i < bias.size(); ++i) bias[i] += e[i];
      }
    }
    return add_conv(name, L, {{W.data.data(), L.cout, L.cin, taps, 0, 0}}, bias);
  }
  // [c][c] identity as a host "weight": a residual add rides in the GEMM as one more K-segment
  // (out = W x + I r).  The product of an fp16 value with 1.0 is exact and accumulates in fp32, so
  // this is the same arithmetic as adding r in the epilogue -- but r arrives through TMA like any
  // other operand instead of through per-row global loads in the epilogue (which stalled the short
  // 1x1 layers on long-scoreboard waits), the plain epilogue and the 256-wide tiles apply, and the
  // extra MMAs land on a tensor pipe that idles in these layers anyway.
  static HostTensor identity(int c) {
    HostTensor t;
    t.shape = {c, c};
    t.data.assign((size_t)c * c, 0.f);
    for (int i = 0; i < c; ++i) t.data[(size_t)i * c + i] = 1.f;
    return t;
  }
  // linear layer (1x1) whose output gets a residual of `cout` channels added
  int make_lin_res(const std::string& name, const std::string& wkey, const std::string& bkey) {
    const HostTensor& W = H(wkey);
    nope::ConvLayer L = nope::conv1x1();
    L.cout = (int)W.shape[0];
    L.cin = (int)W.shape[1];
    L.skip_c = L.cout;
    L.K = L.cin + L.skip_c;
    L.k_alg = L.cin;
    const HostTensor I = identity(L.cout);
    return add_conv(name, L, {{W.data.data(), L.cout, L.cin, 1, 0, 0}, {I.data.data(), L.cout, L.cout, 1, 0, L.cin}},
                    H(bkey).data);
  }
  int make_norm(const std::string& name, const std::string& prefix) {
    nope::LdmNorm n;
    n.C = (int)H(prefix + ".weight").shape[0];
    NOPE_CHECK(n.C % 256 == 0 && n.C <= nope::kLdmMaxC, prefix + ": GroupNorm(32) needs C % 256 == 0, C <= 2048");
    if (mem.upload(&n.gamma, H(prefix + ".weight").data) || mem.upload(&n.beta, H(prefix + ".bias").data)) return -1;
    norms[name] = n;
    return 0;
  }
  int make_res(const std::string& p) {
    // ResBlock (ldm/openaimodel.py:217-286).  emb = 0, so emb_layers(emb) = Linear(SiLU(0)) =
    // emb_layers.1.bias: folded into the first convolution's bias.
    if (make_norm(p + ".n1", p + ".in_layers.0") || make_norm(p + ".n2", p + ".out_layers.0")) return -1;
    if (make_conv(p + ".c1", p + ".in_layers.2.weight", p + ".in_layers.2.bias", nope::conv3x3(),
                  p + ".emb_layers.1.bias"))
      return -1;
    const HostTensor& W2 = H(p + ".out_layers.3.weight");
    nope::ConvLayer L = nope::conv3x3();
    L.cout = (int)W2.shape[0];
    L.cin = (int)W2.shape[1];
    std::vector<float> bias = H(p + ".out_layers.3.bias").data;
    const bool has_skip = staged.has(p + ".skip_connection.weight");
    if (has_skip) {
      // skip_connection (1x1 on the block input) rides in the same GEMM: extra K columns
      const HostTensor& Ws = H(p + ".skip_connection.weight");
      L.skip_c = (int)Ws.shape[1];
      const auto& bs = H(p + ".skip_connection.bias").data;
      for (size_t i = 0; i < bias.size(); ++i) bias[i] += bs[i];
    }
    const bool id_skip = !has_skip;      // identity skip as an identity K-segment
    if (id_skip) L.skip_c = L.cout;
    L.K = 9 * L.cin + L.skip_c;
    if (id_skip) L.k_alg = 9 * L.cin;
    // the skip's weights follow the 3x3's in the extra K columns
    const HostTensor I = id_skip ? identity(L.cout) : HostTensor();
    const float* ws = has_skip ? H(p + ".skip_connection.weight").data.data() : I.data.data();
    return add_conv(p + ".c2", L, {{W2.data.data(), L.cout, L.cin, 9, 0, 0}, {ws, L.cout, L.skip_c, 1, 0, 9 * L.cin}},
                    bias);
  }
  int make_st(const std::string& p) {
    const std::string t = p + ".transformer_blocks.0";
    const int c = (int)H(p + ".norm.weight").shape[0];
    if (make_norm(p + ".norm", p + ".norm")) return -1;
    if (make_conv(p + ".proj_in", p + ".proj_in.weight", p + ".proj_in.bias", nope::conv1x1())) return -1;
    if (make_lin_res(p + ".proj_out", p + ".proj_out.weight", p + ".proj_out.bias")) return -1;
    if (make_lin_res(p + ".to_out", t + ".attn1.to_out.0.weight", t + ".attn1.to_out.0.bias")) return -1;
    {  // the feed-forward projection with GEGLU fused into the epilogue: tile t of 128 rows =
       // x rows 64t..64t+63 followed by gate rows inner+64t..inner+64t+63
      const HostTensor& W = H(t + ".ff.net.0.proj.weight");
      const auto& b = H(t + ".ff.net.0.proj.bias").data;
      const int inner = 4 * c;
      HostTensor Wp;
      Wp.shape = W.shape;
      Wp.data.resize(W.data.size());
      std::vector<float> bp(2 * inner);
      for (int tl = 0; tl < inner / 64; ++tl)
        for (int half = 0; half < 2; ++half)
          for (int j = 0; j < 64; ++j) {
            const int src = half * inner + tl * 64 + j, dst = tl * 128 + half * 64 + j;
            std::copy(W.data.begin() + (size_t)src * c, W.data.begin() + (size_t)(src + 1) * c,
                      Wp.data.begin() + (size_t)dst * c);
            bp[dst] = b[src];
          }
      nope::ConvLayer L = nope::conv1x1();
      L.cin = c;
      L.cout = 2 * inner;
      L.K = c;
      L.geglu = true;
      if (add_conv(p + ".ff1g", L, {{Wp.data.data(), 2 * inner, c, 1, 0, 0}}, bp)) return -1;
      NOPE_CHECK(convs.at(p + ".ff1g").bn == 128, "GEGLU projection must tile by 128");
    }
    if (make_lin_res(p + ".ff2", t + ".ff.net.2.weight", t + ".ff.net.2.bias")) return -1;
    {  // q | k | v of the self-attention as one GEMM (no bias, ldm/attention.py:160-162)
      nope::ConvLayer L = nope::conv1x1();
      L.cin = c;
      L.cout = 3 * c;
      L.K = c;
      if (add_conv(p + ".qkv", L,
                   {{H(t + ".attn1.to_q.weight").data.data(), c, c, 1, 0, 0},
                    {H(t + ".attn1.to_k.weight").data.data(), c, c, 1, c, 0},
                    {H(t + ".attn1.to_v.weight").data.data(), c, c, 1, 2 * c, 0}},
                   {}))
        return -1;
    }
    for (int n = 1; n <= 3; n += 2) {   // norm2 only feeds attn2's queries, which cancel (see below)
      nope::LdmNorm ln;
      ln.C = c;
      if (mem.upload(&ln.gamma, H(t + ".norm" + std::to_string(n) + ".weight").data) ||
          mem.upload(&ln.beta, H(t + ".norm" + std::to_string(n) + ".bias").data))
        return -1;
      norms[p + ".ln" + std::to_string(n)] = ln;
    }
    cb_off[p] = cb_width;
    cb_width += c;
    return 0;
  }
  // Cross-attention with a one-token context (ldm/attention.py:170-195): softmax over a single
  // key is 1, so attn2(.) = to_out(to_v(pose_mlp(pose))) -- linear in the pose.  Fold
  // Wc = Wo Wv Wp and bc = Wo Wv bp + bo in double, for all transformer blocks at once.
  int make_cross() {
    std::vector<float> Wc((size_t)cb_width * rot_dim), bc(cb_width);
    const auto& Wp = H("pose_mlp.0.weight").data;   // [ctx][6]
    const auto& bp = H("pose_mlp.0.bias").data;
    for (const auto& kv : cb_off) {
      const std::string t = kv.first + ".transformer_blocks.0.attn2";
      const auto& Wv = H(t + ".to_v.weight").data;       // [c][ctx]
      const auto& Wo = H(t + ".to_out.0.weight").data;   // [c][c]
      const auto& bo = H(t + ".to_out.0.bias").data;
      const int c = (int)bo.size();
      std::vector<double> A((size_t)c * (rot_dim + 1), 0.0);   // Wv [Wp | bp]
      for (int i = 0; i < c; ++i)
        for (int k = 0; k < ctx; ++k) {
          const double w = Wv[(size_t)i * ctx + k];
          for (int r = 0; r < rot_dim; ++r) A[(size_t)i * (rot_dim + 1) + r] += w * Wp[(size_t)k * rot_dim + r];
          A[(size_t)i * (rot_dim + 1) + rot_dim] += w * bp[k];
        }
      for (int o = 0; o < c; ++o) {
        std::vector<double> acc(rot_dim + 1, 0.0);
        for (int i = 0; i < c; ++i) {
          const double w = Wo[(size_t)o * c + i];
          for (int r = 0; r <= rot_dim; ++r) acc[r] += w * A[(size_t)i * (rot_dim + 1) + r];
        }
        for (int r = 0; r < rot_dim; ++r) Wc[(size_t)(kv.second + o) * rot_dim + r] = (float)acc[r];
        bc[kv.second + o] = (float)(acc[rot_dim] + bo[o]);
      }
    }
    return mem.upload(&cross_w, Wc) || mem.upload(&cross_b, bc) ? -1 : 0;
  }

  // packs the staged weights (nope::engine_finalize: every schema key is present, device selected)
  int finalize() {
    if (mem.upload(&in_w, H("input_blocks.0.0.weight").data) || mem.upload(&in_b, H("input_blocks.0.0.bias").data))
      return -1;
    {  // out[2]: Cl output channels padded to one 64-wide tile of the tensor-core kernel
      HostTensor W;
      W.shape = {64, mc, 3, 3};
      W.data.assign((size_t)64 * mc * 9, 0.f);
      const auto& w = H("out.2.weight").data;
      std::copy(w.begin(), w.end(), W.data.begin());
      std::vector<float> bias(64, 0.f);
      std::copy(H("out.2.bias").data.begin(), H("out.2.bias").data.end(), bias.begin());
      nope::ConvLayer L = nope::conv3x3();
      L.cout = 64;
      L.cin = mc;
      L.K = 9 * mc;
      if (add_conv("out.2", L, {{W.data.data(), 64, mc, 9, 0, 0}}, bias)) return -1;
    }
    for (size_t i = 1; i < inp.size(); ++i) {
      const std::string p = "input_blocks." + std::to_string(i);
      if (inp[i].kind == 1) {
        if (make_res(p + ".0") || make_st(p + ".1")) return -1;
      } else {
        if (make_conv(p + ".0.op", p + ".0.op.weight", p + ".0.op.bias", nope::conv3x3_s2())) return -1;
      }
    }
    if (make_res("middle_block.0") || make_st("middle_block.1") || make_res("middle_block.2")) return -1;
    for (size_t i = 0; i < outp.size(); ++i) {
      const std::string p = "output_blocks." + std::to_string(i);
      if (make_res(p + ".0") || make_st(p + ".1")) return -1;
      if (outp[i].up && make_conv(p + ".2.conv", p + ".2.conv.weight", p + ".2.conv.bias", nope::conv_upsample3x3()))
        return -1;
    }
    if (make_norm("out.0", "out.0")) return -1;
    return make_cross();
  }

  // ------------------------------------------------------------------ workspace
  // layout(b) places every buffer for capacities (c hypotheses, r references, n_scores (reference, query, pose)
  // triples of score partials and similarity scratch)
  size_t layout(nope::Bump& b, int c_hyp, int c_ref, int n_scores) {
    const size_t c = (size_t)c_hyp, r = (size_t)c_ref;
    const size_t u = (size_t)S0 * S0 * mc;        // one full-resolution base-width map
    int S = S0;
    for (size_t i = 0; i < inp.size(); ++i) {
      if (inp[i].kind == 2) S /= 2;
      b.take(&HS[i], c * S * S * inp[i].cout);
    }
    // widest tensors: block outputs <= 2u (512 ch at 32^2 after the last upsample), ResBlock
    // inputs <= 3u (768 ch at 32^2), q|k|v 3u, V^T 1u, GEGLU output 4u
    for (__half** t : {&XA, &XB, &XC}) b.take(t, c * 2 * u);
    b.take(&R, c * u);
    b.take(&T1, c * 3 * u);
    for (__half** t : {&T2, &T3, &XN, &PI, &PJ}) b.take(t, c * u);
    b.take(&QKV, c * 3 * u);
    for (__half** t : {&Vt, &AO}) b.take(t, c * u);
    b.take(&GG, c * 4 * u);
    for (__half** t : {&x0ref, &Rref, &Pref}) b.take(t, r * u);
    const size_t sts = (size_t)32 * 256;   // parts (<= 32) x octets (<= 256) per image
    for (float2** t : {&S_in, &S_mid, &S_out}) b.take(t, c * sts);
    b.take(&cb, c * (size_t)cb_width);
    b.take(&ref_of, c);
    b.take(&OF, c * S0 * S0 * 64);
    b.take(&score_partial, (size_t)n_scores * nslab());
    b.take(&sim_buf, (size_t)n_scores);
    return b.off;
  }
  // Sizes the workspace for `need_cap` hypotheses, `need_ref` references and `need_scores` scored triples.  It grows
  // on demand only (a device synchronisation and cudaMalloc then).
  int ensure_workspace(int need_cap, int need_ref, int need_scores, cudaStream_t) {
    if (need_cap <= cap && need_ref <= cap_ref && need_scores <= scores_cap) return 0;
    return nope::grow_workspace(this, std::tie(cap, cap_ref, scores_cap), nullptr, std::max(cap, need_cap),
                                std::max(cap_ref, need_ref), std::max(scores_cap, need_scores));
  }

  // ------------------------------------------------------------------ op launchers
  // out[n_img, So, So, cout] = conv(L, in) [+ 1x1 skip or identity residual over cat(sk0, sk1)] + bias
  int conv(const nope::ConvLayer& L, const __half* in, __half* out, int So, int n_img, cudaStream_t st,
           float2* stats = nullptr, const __half* sk0 = nullptr, int skc0 = 0,
           const __half* sk1 = nullptr, int skc1 = 0, float* out_f32 = nullptr) {
    using namespace nope;
    NOPE_CHECK(skc0 + skc1 == L.skip_c, "conv: skip channel mismatch");
    NOPE_CHECK(!L.skip_c || (!L.up && L.stride == 1 && sk0 && skc0 % 64 == 0 && skc1 % 64 == 0),
               "conv: bad skip sources");
    NOPE_CHECK(!(stats && L.up), "upsample conv has no fused statistics");
    ++launches;
    TileGeom g;
    if (make_geom(L.up ? So / 2 : So, L.up ? So / 2 : So, &g)) return -1;
    ConvBuilder b(tmaps, g, cap);
    ConvParams& p = b.p;
    // a stride-2 convolution reads the four stride-2 lattices of its 2So x 2So input
    int col = b.segs(L.taps(), {b.src(in, nullptr, L.cin, L.stride == 2 ? 4 : 1)}, 0, 0);
    if (L.skip_c) {
      std::vector<ConvSrc> sk{b.src(sk0, nullptr, skc0)};
      if (sk1) sk.push_back(b.src(sk1, nullptr, skc1));
      col = b.segs({ConvTap{0, 0, 0}}, sk, col, 0);
    }
    NOPE_CHECK(col == L.K, "conv: K mismatch");
    // exact weights: the same segments again over the W_lo plane
    for (int i = 0, n = L.wlo ? p.nseg : 0; i < n; ++i) {
      const ConvSeg s = p.seg[i];
      b.seg(s.map, s.dy, s.dx, s.nchunks, s.wcol1 + L.K);
    }
    if (b.finish(L, out, L.geglu ? L.cout / 2 : L.cout, n_img, L.up ? 4 : 1)) return -1;
    p.geglu = L.geglu ? 1 : 0;
    p.out_f32 = out_f32;
    p.stats = stats;
    if (prof.begin(st)) return -1;
    const int rc = launch_conv_tc2(p, L.bn, num_sms, st);
    // executed FLOPs (the folded upsample runs 4 parity GEMMs of K = 4 Cin over the source pixels)
    const double fl = 2.0 * (double)n_img * g.H * g.W * (double)L.rows() * (double)L.k_alg;
    if (prof.end(st, {fl, fl, 0})) return -1;
    return rc;
  }

  static int parts_of(int S) { return S * S < 32 ? 1 : S * S / 32; }

  int stats(const __half* x0, int C0, const __half* x1, int C1, int S, int n, float2* dst, cudaStream_t st) {
    nope::ldm_stats_kernel<<<dim3(parts_of(S), n), 256, 0, st>>>(x0, C0, x1, C1, dst, S * S);
    NOPE_CUDA(cudaGetLastError());
    ++launches;
    return 0;
  }
  int gn(const nope::LdmNorm& N, const __half* x0, int C0, const __half* x1, int C1, const float2* stt, int S,
         int n, __half* y, bool silu, float eps, cudaStream_t st) {
    using namespace nope;
    NOPE_CHECK(N.C == C0 + C1, "gn: channel mismatch");
    LdmGnArgs a;
    a.x0 = x0; a.x1 = x1; a.y = y; a.stats = stt; a.gamma = N.gamma; a.beta = N.beta;
    a.C0 = C0; a.C1 = C1; a.st_parts = parts_of(S); a.hw = S * S;
    a.pps = a.hw >= 64 ? 64 : a.hw;
    a.eps = eps;
    const dim3 grid(a.hw / a.pps, n);
    if (silu) ldm_gn_apply_kernel<true><<<grid, 256, 0, st>>>(a);
    else ldm_gn_apply_kernel<false><<<grid, 256, 0, st>>>(a);
    NOPE_CUDA(cudaGetLastError());
    ++launches;
    return 0;
  }
  int ln(const nope::LdmNorm& N, const __half* x, __half* xout, const float* cbp, __half* y, int C, int S, int n,
         cudaStream_t st, const int* src_img = nullptr) {
    using namespace nope;
    const long long ntok = (long long)n * S * S;
    const int tpw = 1024 / C;                               // tokens per warp (ldm_ln_kernel)
    const unsigned grid = (unsigned)((ntok + 8 * tpw - 1) / (8 * tpw));
    switch (C) {
      case 256: ldm_ln_kernel<1><<<grid, 256, 0, st>>>(x, xout, cbp, cb_width, N.gamma, N.beta, y, ntok, S * S, src_img); break;
      case 512: ldm_ln_kernel<2><<<grid, 256, 0, st>>>(x, xout, cbp, cb_width, N.gamma, N.beta, y, ntok, S * S, src_img); break;
      case 1024: ldm_ln_kernel<4><<<grid, 256, 0, st>>>(x, xout, cbp, cb_width, N.gamma, N.beta, y, ntok, S * S, src_img); break;
      default: return fail("LayerNorm: channels must be 256, 512 or 1024");
    }
    NOPE_CUDA(cudaGetLastError());
    ++launches;
    return 0;
  }
  // self-attention core on qkv [n, ntok, 3C] -> out [n, ntok, C]; vt [n, ntok, C] holds V^T
  int attention(const __half* qkv, __half* vt, __half* out, int C, int ntok, int n, cudaStream_t st) {
    using namespace nope;
    const int Hh = C / 32;
    NOPE_CHECK(ntok % 64 == 0 && C % 64 == 0, "attention: tokens and channels must be multiples of 64");
    ldm_attn_prep_kernel<<<dim3(ntok / 64, n), 256, 0, st>>>(qkv, vt, ntok, C);
    NOPE_CUDA(cudaGetLastError());
    const float sl2e = 0.17677669529663687f * 1.4426950408889634f;   // 32^-1/2 * log2(e)
    const dim3 grid((unsigned)(n * Hh) * (unsigned)((ntok + 127) / 128));
    if (prof.begin(st)) return -1;
    static bool attr_set[kMaxDevices];     // the shared-memory opt-in is per device
    int dev = 0;
    NOPE_CUDA(cudaGetDevice(&dev));
    NOPE_CHECK(dev >= 0 && dev < kMaxDevices, "device index out of range");
    if (!attr_set[dev]) {
      NOPE_CUDA(cudaFuncSetAttribute(ldm_attn_tc_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kAttnSmem));
      attr_set[dev] = true;
    }
    AttnParams p;
    const CUtensorMap* m = nullptr;
    if (tmaps.get3(&m, qkv, 3 * C, ntok, n, 64, 128)) return -1;
    p.qkmap = *m;
    if (tmaps.get3(&m, vt, ntok, 32, n * Hh, 64, 32)) return -1;
    p.vmap = *m;
    p.out = out; p.n = ntok; p.H = Hh; p.C = C; p.scale_log2e = sl2e;
    ldm_attn_tc_kernel<<<grid, 128, kAttnSmem, st>>>(p);
    NOPE_CUDA(cudaGetLastError());
    const double fl = 4.0 * (double)n * ntok * (double)ntok * C;
    if (prof.end(st, {fl, fl, 1})) return -1;
    launches += 2;
    return 0;
  }

  int tap(const std::string& name, const __half* buf, int C, int S, int n, cudaStream_t st) {
    return dtap.capture(name.c_str(), buf, nullptr, false, C, S, n, st);
  }

  // ResBlock._forward (ldm/openaimodel.py:265-286) on cat(x0, x1).  Leaves the GroupNorm
  // statistics of `out` in S_out (conv epilogue) for a following SpatialTransformer.norm.
  int resblock(const std::string& p, const __half* x0, int C0, const __half* x1, int C1, __half* out, int S, int n,
               cudaStream_t st) {
    const nope::ConvLayer& c1 = convs.at(p + ".c1");
    const nope::ConvLayer& c2 = convs.at(p + ".c2");
    NOPE_CHECK(c1.cin == C0 + C1, "resblock: channel mismatch");
    if (stats(x0, C0, x1, C1, S, n, S_in, st)) return -1;
    if (gn(norms.at(p + ".n1"), x0, C0, x1, C1, S_in, S, n, T1, true, 1e-5f, st)) return -1;
    if (conv(c1, T1, T2, S, n, st, S_mid)) return -1;
    if (gn(norms.at(p + ".n2"), T2, c1.cout, nullptr, 0, S_mid, S, n, T3, true, 1e-5f, st)) return -1;
    return conv(c2, T3, out, S, n, st, S_out, x0, C0, x1, C1);
  }

  // SpatialTransformer.forward (ldm/attention.py:264-277) with one BasicTransformerBlock
  // (:229-233), in two halves.  st_pre: norm, proj_in, x = attn1(norm1(x)) + x -> `xs`; nothing in
  // it depends on the pose.  x_in's GroupNorm statistics must be in S_out.
  int st_pre(const std::string& p, const __half* x_in, __half* xs, int C, int S, int n, cudaStream_t st) {
    if (gn(norms.at(p + ".norm"), x_in, C, nullptr, 0, S_out, S, n, XN, false, 1e-6f, st)) return -1;
    if (conv(convs.at(p + ".proj_in"), XN, PI, S, n, st)) return -1;
    if (ln(norms.at(p + ".ln1"), PI, nullptr, nullptr, XN, C, S, n, st)) return -1;
    if (conv(convs.at(p + ".qkv"), XN, QKV, S, n, st)) return -1;
    if (attention(QKV, Vt, AO, C, S * S, n, st)) return -1;
    return conv(convs.at(p + ".to_out"), AO, xs, S, n, st, nullptr, PI, C);
  }
  // st_post: x = attn2(norm2(x), context) + x -- the one-token cross-attention is the
  // per-hypothesis vector cb (see make_cross), added by the LayerNorm kernel, which also applies
  // norm3 -- then x = ff(norm3(x)) + x (GEGLU) and proj_out(x) + x_in.  `xs` may hold one image
  // per reference (src_img maps hypothesis -> image); x_in and out are per hypothesis.
  int st_post(const std::string& p, const __half* xs, const int* src_img, const __half* x_in, __half* out, int C,
              int S, int n, const float* cbp, cudaStream_t st) {
    if (ln(norms.at(p + ".ln3"), xs, PJ, cbp + cb_off.at(p), XN, C, S, n, st, src_img)) return -1;
    if (conv(convs.at(p + ".ff1g"), XN, GG, S, n, st)) return -1;   // GEGLU in the projection's epilogue
    if (conv(convs.at(p + ".ff2"), GG, PI, S, n, st, nullptr, PJ, C)) return -1;
    return conv(convs.at(p + ".proj_out"), PI, out, S, n, st, nullptr, x_in, C);
  }
  int transformer(const std::string& p, const __half* x_in, __half* out, int C, int S, int n, const float* cbp,
                  cudaStream_t st) {
    if (st_pre(p, x_in, PJ, C, S, n, st)) return -1;
    return st_post(p, PJ, nullptr, x_in, out, C, S, n, cbp, st);
  }

  int cross_terms(const float* poses, int n, cudaStream_t st) {
    nope::ldm_cross_kernel<<<n, 256, 0, st>>>(poses, cross_w, cross_b, cb, n, rot_dim, cb_width);
    NOPE_CUDA(cudaGetLastError());
    ++launches;
    return 0;
  }

  // Pose-independent prefix, once per reference latent: input_blocks.0, the ResBlock of
  // input_blocks.1 and its transformer up to (and including) the self-attention -- the pose only
  // enters at the first cross-attention.  Leaves x0ref (conv), Rref (ResBlock output) and Pref
  // (x after attn1), one image per reference.
  int prestage(const float* ref_lat, int B, cudaStream_t st) {
    nope::init_conv_kernel<<<nope::ew_grid((long long)B * S0 * S0 * mc), 256, 0, st>>>(ref_lat, in_w, in_b, x0ref, B,
                                                                                     Cl, S0, S0, mc);
    NOPE_CUDA(cudaGetLastError());
    ++launches;
    if (!hoist) return 0;
    const size_t u = (size_t)S0 * S0 * mc;
    for (int b0 = 0; b0 < B; b0 += cap) {       // the temporaries hold `cap` images
      const int nb = std::min(cap, B - b0);
      if (resblock("input_blocks.1.0", x0ref + b0 * u, mc, nullptr, 0, Rref + b0 * u, S0, nb, st)) return -1;
      if (st_pre("input_blocks.1.1", Rref + b0 * u, Pref + b0 * u, mc, S0, nb, st)) return -1;
    }
    return 0;
  }

  // UNetModelPose.forward for hypotheses [hyp0, hyp0 + n) of the flattened (b, pose) list
  // query [B, Q, Cl, hw]; score_part [B * N, Q, nslab]; vis (optional) [B, Q, hw] visible maps
  int forward_chunk(const float* poses, int hyp0, int n, int N, const float* query, float* out_emb,
                    float* score_part, cudaStream_t st, int Q = 1, const uint8_t* vis = nullptr) {
    using namespace nope;
    ref_of_kernel<<<(n + 255) / 256, 256, 0, st>>>(ref_of, hyp0, N, n);
    ++launches;
    if (cross_terms(poses + (size_t)hyp0 * rot_dim, n, st)) return -1;
    int S = S0;
    bcast_add_kernel<<<dim3(ew_grid((long long)S * S * mc / 8 / 4), n), 256, 0, st>>>(x0ref, ref_of, nullptr, 0, 0, HS[0], n,
                                                                           S * S, mc);
    NOPE_CUDA(cudaGetLastError());
    ++launches;
    if (tap("input_blocks.0", HS[0], mc, S, n, st)) return -1;
    const __half* cur = HS[0];
    int C = mc;
    for (size_t i = 1; i < inp.size(); ++i) {
      const std::string p = "input_blocks." + std::to_string(i);
      const auto& b = inp[i];
      if (b.kind == 1 && i == 1 && hoist) {
        // prefix computed per reference in prestage(): broadcast the ResBlock output (the
        // transformer's residual) and enter the transformer at the cross-attention
        bcast_add_kernel<<<dim3(ew_grid((long long)S * S * mc / 8 / 4), n), 256, 0, st>>>(Rref, ref_of, nullptr, 0, 0, R, n,
                                                                               S * S, mc);
        NOPE_CUDA(cudaGetLastError());
        ++launches;
        if (tap(p + ".0", R, b.cout, S, n, st)) return -1;
        if (st_post(p + ".1", Pref, ref_of, R, HS[i], b.cout, S, n, cb, st)) return -1;
      } else if (b.kind == 1) {
        if (resblock(p + ".0", cur, C, nullptr, 0, R, S, n, st)) return -1;
        if (tap(p + ".0", R, b.cout, S, n, st)) return -1;
        if (transformer(p + ".1", R, HS[i], b.cout, S, n, cb, st)) return -1;
      } else {
        S /= 2;
        if (conv(convs.at(p + ".0.op"), cur, HS[i], S, n, st)) return -1;
      }
      C = b.cout;
      cur = HS[i];
      if (tap(p, cur, C, S, n, st)) return -1;
    }
    if (resblock("middle_block.0", cur, C, nullptr, 0, R, S, n, st)) return -1;
    if (tap("middle_block.0", R, C, S, n, st)) return -1;
    if (transformer("middle_block.1", R, XA, C, S, n, cb, st)) return -1;
    if (tap("middle_block.1", XA, C, S, n, st)) return -1;
    if (resblock("middle_block.2", XA, C, nullptr, 0, XB, S, n, st)) return -1;
    if (tap("middle_block", XB, C, S, n, st)) return -1;
    __half* curw = XB;
    __half* oth = XA;
    int skip_i = (int)inp.size() - 1;
    for (size_t i = 0; i < outp.size(); ++i, --skip_i) {
      const std::string p = "output_blocks." + std::to_string(i);
      const auto& b = outp[i];
      if (resblock(p + ".0", curw, C, HS[skip_i], b.skip_c, R, S, n, st)) return -1;
      if (tap(p + ".0", R, b.cout, S, n, st)) return -1;
      C = b.cout;
      if (b.up) {
        if (transformer(p + ".1", R, XC, C, S, n, cb, st)) return -1;
        if (tap(p + ".1", XC, C, S, n, st)) return -1;
        S *= 2;
        if (conv(convs.at(p + ".2.conv"), XC, oth, S, n, st)) return -1;
      } else {
        if (transformer(p + ".1", R, oth, C, S, n, cb, st)) return -1;
        if (tap(p + ".1", oth, C, S, n, st)) return -1;
      }
      std::swap(curw, oth);
      if (tap(p, curw, C, S, n, st)) return -1;
    }
    // out: GroupNorm32 + SiLU, then conv3x3 -> Cl fused with the score
    if (stats(curw, C, nullptr, 0, S, n, S_in, st)) return -1;
    if (gn(norms.at("out.0"), curw, C, nullptr, 0, S_in, S, n, T1, true, 1e-5f, st)) return -1;
    const int hw = S * S;
    const int nslab = (hw + kFinalThreads - 1) / kFinalThreads;
    if (conv(convs.at("out.2"), T1, T2, S, n, st, nullptr, nullptr, 0, nullptr, 0, OF)) return -1;
    (vis ? ldm_score_kernel<true> : ldm_score_kernel<false>)<<<dim3(nslab, n), kFinalThreads, 0, st>>>(
        OF, out_emb ? out_emb + (size_t)hyp0 * Cl * hw : nullptr, query, ref_of,
        score_part ? score_part + (size_t)hyp0 * Q * nslab : nullptr, hw, Cl, Q, vis);
    NOPE_CUDA(cudaGetLastError());
    ++launches;
    return 0;
  }

  // score slabs per (hypothesis, query) of ldm_score_kernel
  int nslab() const { return (S0 * S0 + nope::kFinalThreads - 1) / nope::kFinalThreads; }
  // similarities (sim [B * Q, N]) and top-k of every (reference, query) row from the score partials
  int rank(const float* part, float* sim, int B, int N, int Q, int k, float* topv, int64_t* topi, int64_t idx_base,
           cudaStream_t st, const uint8_t* vis = nullptr) {
    if (vis)
      nope::sim_topk_kernel<true><<<B * Q, 256, 0, st>>>(part, nslab(), sim, N, k, topv,
                                                         reinterpret_cast<long long*>(topi), (long long)idx_base, 1, 0,
                                                         S0 * S0, Q, vis);
    else
      nope::sim_topk_kernel<<<B * Q, 256, 0, st>>>(part, nslab(), sim, N, k, topv, reinterpret_cast<long long*>(topi),
                                                   (long long)idx_base, 1, 0, 1, Q);
    NOPE_CUDA(cudaGetLastError());
    return 0;
  }
};
