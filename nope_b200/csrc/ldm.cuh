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
//                     -> conv3x3 with the 1x1 skip_connection folded in as extra K segments
//                        (or the identity skip added in the epilogue)
//   SpatialTransformer GN32 (statistics from the ResBlock's last epilogue) -> proj_in -> LN ->
//                     q|k|v GEMM -> wgmma attention -> to_out (+x) -> [+cross term, LN] ->
//                     GEGLU feed-forward (+x) -> proj_out (+x_in)
//   Downsample        conv3x3 stride 2 through the four stride-2 TMA lattices of its input
//   Upsample          nearest-x2 + conv3x3 folded into four 2x2 parity kernels
//   out               GN32+SiLU -> conv3x3 (256 -> 4, padded to a 64-channel tile, fp32 store) -> l2 score
// Every GEMM-shaped op runs on conv_tc2_kernel / conv_tc_kernel.
#pragma once
#include "conv_tc2.cuh"
#include "kernels.cuh"
#include "ldm_kernels.cuh"

#include <algorithm>
#include <cmath>
#include <map>
#include <memory>
#include <string>
#include <tuple>
#include <vector>

namespace nope {

struct LdmConv {
  int mode = 0;   // 0: 3x3 pad 1, 1: 1x1 / linear, 3: nearest-x2 + 3x3 (folded), 4: 3x3 stride 2 pad 1
  int cin = 0, cout = 0, K = 0;
  int bn = 0;              // tile width of the clustered kernel (up to 256)
  int bn1 = 0;             // tile width of the 1-CTA kernel (up to 192)
  int skip_c = 0;          // channels of a folded 1x1 skip_connection / identity residual (extra K columns)
  int k_alg = 0;           // K without identity-residual columns (algorithmic FLOP count)
  bool geglu = false;      // rows permuted to (64 x | 64 gate) tiles; the epilogue emits x * gelu(gate)
  __half* w = nullptr;     // [rows][K] fp16
  float* bias = nullptr;
  CUtensorMap wmap, wmap2;      // weight boxes of bn1 / bn rows
};
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

__global__ void ldm_ref_of_kernel(int* r, int h0, int N, int n) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) r[i] = (h0 + i) / N;
}

}  // namespace nope

struct nope_ldm {
  using HostT = std::pair<std::vector<int64_t>, std::vector<float>>;
  int mc = 256, ctx = 512, Cl = 4, S0 = 32, rot_dim = 6, device = 0, num_sms = 132;
  int nres = 2;
  std::vector<int> mult{1, 2, 4};
  bool finalized = false;
  int conv_impl = 2;   // 2: clustered wgmma kernel (default), 0: single-CTA wgmma kernel
  int attn_impl = 0;   // 0: wgmma attention, 1: CUDA-core twin
  bool fold_residual = true;   // residual adds as identity K-segments of the GEMM (set before finalize)
  bool wide_tiles = true;   // 256-channel tiles on the clustered kernel where Cout % 256 == 0 (set before finalize)
  bool hoist = true;        // pose-independent prefix once per reference (prestage)
  bool fuse_geglu = true;   // GEGLU in the projection's epilogue (clustered kernel); false: separate kernel
  int precision = 0;        // 0: fp16 weights; 1: exact weights -- every packed row is [W_hi | W_lo] and the K loop
                            // walks its segment list twice (A W_hi + A W_lo), 2x the MMA work (set before finalize)
  int kp(int K) const { return precision ? 2 * K : K; }
  int chunk = 256;
  int64_t launches = 0;

  std::vector<nope::LdmBlock> inp, outp;
  int mid_ch = 0;

  std::map<std::string, HostT> host;
  std::map<std::string, std::vector<int64_t>> expected;
  std::map<std::string, nope::LdmConv> convs;
  std::map<std::string, nope::LdmNorm> norms;
  std::map<std::string, int> cb_off;   // transformer prefix -> offset in the cross-term vector
  int cb_width = 0;
  float *cross_w = nullptr, *cross_b = nullptr;      // [cb_width][6], [cb_width]
  float *in_w = nullptr, *in_b = nullptr;
  std::vector<void*> owned;

  // workspace (per chunk of `cap` hypotheses; `cap_ref` reference latents)
  int cap = 0, cap_ref = 0;
  std::vector<__half*> HS;                     // skip stack, one buffer per input block
  __half *XA = nullptr, *XB = nullptr, *XC = nullptr, *R = nullptr, *T1 = nullptr, *T2 = nullptr,
         *T3 = nullptr, *XN = nullptr, *PI = nullptr, *PJ = nullptr, *QKV = nullptr,
         *Vt = nullptr, *AO = nullptr, *FF = nullptr, *GG = nullptr, *x0ref = nullptr, *Rref = nullptr, *Pref = nullptr;
  float2 *S_in = nullptr, *S_mid = nullptr, *S_out = nullptr;
  float* cb = nullptr;
  float* OF = nullptr;                          // out[2] result, fp32 [cap * S0 * S0][64]
  int* ref_of = nullptr;
  float* score_partial = nullptr;
  size_t score_partial_cap = 0;
  float* sim_buf = nullptr;
  size_t sim_buf_cap = 0;
  std::vector<void*> ws_owned;
  std::map<std::tuple<const void*, int, int, int, int>, CUtensorMap> tmaps;
  std::map<std::tuple<const void*, int, int, int>, CUtensorMap> tmaps3;

  // per-launch CUDA-event profile (bench.py roofline): kind 0 = convolution / GEMM, 1 = attention
  bool profile = false;
  std::vector<cudaEvent_t> prof_ev;
  std::vector<double> prof_flops;
  std::vector<int> prof_kind;
  int prof_begin(cudaStream_t st) {
    cudaEvent_t e0;
    NOPE_CUDA(cudaEventCreate(&e0));
    NOPE_CUDA(cudaEventRecord(e0, st));
    prof_ev.push_back(e0);
    return 0;
  }
  int prof_end(cudaStream_t st, double flops, int kind) {
    cudaEvent_t e1;
    NOPE_CUDA(cudaEventCreate(&e1));
    NOPE_CUDA(cudaEventRecord(e1, st));
    prof_ev.push_back(e1);
    prof_flops.push_back(flops);
    prof_kind.push_back(kind);
    return 0;
  }

  // debug tap
  std::string tap_name;
  float* tap_out = nullptr;
  int64_t tap_cap = 0;
  int tap_C = 0, tap_S = 0;
  bool tap_hit = false;

  ~nope_ldm() {
    for (void* p : owned) cudaFree(p);
    for (void* p : ws_owned) cudaFree(p);
    if (score_partial) cudaFree(score_partial);
    if (sim_buf) cudaFree(sim_buf);
    for (cudaEvent_t e : prof_ev) cudaEventDestroy(e);
  }

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
    for (int level = (int)mult.size() - 1; level >= 0; --level)
      for (int i = 0; i <= nres; ++i) {
        const int ich = chans.back();
        chans.pop_back();
        outp.push_back(LdmBlock{1, ch + ich, mc * mult[level], ich, level > 0 && i == nres});
        ch = mc * mult[level];
      }
  }
  void expect(const std::string& k, std::vector<int64_t> s) { expected[k] = std::move(s); }
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

  // ------------------------------------------------------------------ weights
  int upload(const std::vector<float>& v, float** out) {
    NOPE_CUDA(cudaMalloc(reinterpret_cast<void**>(out), std::max<size_t>(v.size(), 1) * sizeof(float)));
    owned.push_back(*out);
    NOPE_CUDA(cudaMemcpy(*out, v.data(), v.size() * sizeof(float), cudaMemcpyHostToDevice));
    return 0;
  }
  const HostT& H(const std::string& k) const { return host.at(k); }
  // dst[(row_off + o) * K + col_off + t * cin + c] = fp16(src[o][c][t])
  int pack_into(__half* dst, int K, int row_off, int col_off, const HostT& t, int cout, int cin, int taps,
                bool fold_up = false) {
    using namespace nope;
    float *tmp = nullptr, *folded = nullptr;
    const size_t n = t.second.size();
    NOPE_CHECK(n == (size_t)cout * cin * (fold_up ? 9 : taps), "pack_into: size mismatch");
    NOPE_CUDA(cudaMalloc(reinterpret_cast<void**>(&tmp), n * sizeof(float)));
    NOPE_CUDA(cudaMemcpy(tmp, t.second.data(), n * sizeof(float), cudaMemcpyHostToDevice));
    const float* src = tmp;
    int rows = cout;
    if (fold_up) {
      NOPE_CUDA(cudaMalloc(reinterpret_cast<void**>(&folded), (size_t)4 * cout * cin * 4 * sizeof(float)));
      fold_upconv_kernel<<<ew_grid((long long)4 * cout * cin), 256>>>(tmp, folded, cout, cin);
      NOPE_CUDA(cudaGetLastError());
      src = folded;
      rows = 4 * cout;
    }
    pack_weight_kernel<<<ew_grid((long long)rows * cin * taps), 256>>>(
        src, dst + (size_t)row_off * kp(K), rows, cin, taps, kp(K), col_off, precision ? K : 0);
    NOPE_CUDA(cudaGetLastError());
    NOPE_CUDA(cudaDeviceSynchronize());
    NOPE_CUDA(cudaFree(tmp));
    if (folded) NOPE_CUDA(cudaFree(folded));
    return 0;
  }
  int finish_conv(const std::string& name, nope::LdmConv& L, int rows, const std::vector<float>& bias) {
    using namespace nope;
    if (L.k_alg == 0) L.k_alg = L.K;
    L.bn1 = pick_bn(L.cout);
    L.bn = (!L.geglu && L.cout % 256 == 0 && wide_tiles) ? 256 : L.bn1;
    NOPE_CHECK(L.bn != 0 && L.K % 64 == 0, name + ": channel counts must be multiples of 64");
    if (!bias.empty() && upload(bias, &L.bias)) return -1;
    if (make_weight_map(&L.wmap, L.w, rows, kp(L.K), L.bn1)) return -1;
    if (make_weight_map(&L.wmap2, L.w, rows, kp(L.K), L.bn)) return -1;
    convs[name] = L;
    return 0;
  }
  int alloc_w(nope::LdmConv& L, int rows) {
    NOPE_CUDA(cudaMalloc(reinterpret_cast<void**>(&L.w), (size_t)rows * kp(L.K) * sizeof(__half)));
    owned.push_back(L.w);
    return 0;
  }
  // plain convolution / linear layer.  extra_bias (optional) is added to the bias.
  int make_conv(const std::string& name, const std::string& wkey, const std::string& bkey, int mode,
                const std::string& extra_bias = "") {
    const HostT& W = H(wkey);
    nope::LdmConv L;
    L.mode = mode;
    L.cout = (int)W.first[0];
    L.cin = (int)W.first[1];
    const int taps = mode == 1 ? 1 : (mode == 3 ? 4 : 9);
    L.K = L.cin * taps;
    const int rows = mode == 3 ? 4 * L.cout : L.cout;
    if (alloc_w(L, rows)) return -1;
    if (pack_into(L.w, L.K, 0, 0, W, L.cout, L.cin, taps, mode == 3)) return -1;
    std::vector<float> bias;
    if (!bkey.empty()) {
      bias = H(bkey).second;
      if (!extra_bias.empty()) {
        const auto& e = H(extra_bias).second;
        for (size_t i = 0; i < bias.size(); ++i) bias[i] += e[i];
      }
    }
    return finish_conv(name, L, rows, bias);
  }
  // [c][c] identity as a host "weight": a residual add rides in the GEMM as one more K-segment
  // (out = W x + I r).  The product of an fp16 value with 1.0 is exact and accumulates in fp32, so
  // this is the same arithmetic as adding r in the epilogue -- but r arrives through TMA like any
  // other operand instead of through per-row global loads in the epilogue (which stalled the short
  // 1x1 layers on long-scoreboard waits), the plain epilogue and the 256-wide tiles apply, and the
  // extra MMAs land on a tensor pipe that idles in these layers anyway.
  static HostT identity(int c) {
    HostT t;
    t.first = {c, c};
    t.second.assign((size_t)c * c, 0.f);
    for (int i = 0; i < c; ++i) t.second[(size_t)i * c + i] = 1.f;
    return t;
  }
  // linear layer (1x1) whose output gets a residual of `cout` channels added
  int make_lin_res(const std::string& name, const std::string& wkey, const std::string& bkey) {
    if (!fold_residual) return make_conv(name, wkey, bkey, 1);
    const HostT& W = H(wkey);
    nope::LdmConv L;
    L.mode = 1;
    L.cout = (int)W.first[0];
    L.cin = (int)W.first[1];
    L.skip_c = L.cout;
    L.K = L.cin + L.skip_c;
    L.k_alg = L.cin;
    if (alloc_w(L, L.cout)) return -1;
    if (pack_into(L.w, L.K, 0, 0, W, L.cout, L.cin, 1) || pack_into(L.w, L.K, 0, L.cin, identity(L.cout), L.cout, L.cout, 1))
      return -1;
    return finish_conv(name, L, L.cout, H(bkey).second);
  }
  int make_norm(const std::string& name, const std::string& prefix) {
    nope::LdmNorm n;
    n.C = (int)H(prefix + ".weight").first[0];
    NOPE_CHECK(n.C % 256 == 0 && n.C <= nope::kLdmMaxC, prefix + ": GroupNorm(32) needs C % 256 == 0, C <= 2048");
    if (upload(H(prefix + ".weight").second, &n.gamma) || upload(H(prefix + ".bias").second, &n.beta)) return -1;
    norms[name] = n;
    return 0;
  }
  int make_res(const std::string& p) {
    // ResBlock (ldm/openaimodel.py:217-286).  emb = 0, so emb_layers(emb) = Linear(SiLU(0)) =
    // emb_layers.1.bias: folded into the first convolution's bias.
    if (make_norm(p + ".n1", p + ".in_layers.0") || make_norm(p + ".n2", p + ".out_layers.0")) return -1;
    if (make_conv(p + ".c1", p + ".in_layers.2.weight", p + ".in_layers.2.bias", 0, p + ".emb_layers.1.bias"))
      return -1;
    const HostT& W2 = H(p + ".out_layers.3.weight");
    nope::LdmConv L;
    L.mode = 0;
    L.cout = (int)W2.first[0];
    L.cin = (int)W2.first[1];
    std::vector<float> bias = H(p + ".out_layers.3.bias").second;
    const bool has_skip = host.count(p + ".skip_connection.weight") != 0;
    if (has_skip) {
      // skip_connection (1x1 on the block input) rides in the same GEMM: extra K columns
      const HostT& Ws = H(p + ".skip_connection.weight");
      L.skip_c = (int)Ws.first[1];
      const auto& bs = H(p + ".skip_connection.bias").second;
      for (size_t i = 0; i < bias.size(); ++i) bias[i] += bs[i];
    }
    const bool id_skip = !has_skip && fold_residual;      // identity skip as an identity K-segment
    if (id_skip) L.skip_c = L.cout;
    L.K = 9 * L.cin + L.skip_c;
    if (id_skip) L.k_alg = 9 * L.cin;
    if (alloc_w(L, L.cout)) return -1;
    if (pack_into(L.w, L.K, 0, 0, W2, L.cout, L.cin, 9)) return -1;
    if (has_skip && pack_into(L.w, L.K, 0, 9 * L.cin, H(p + ".skip_connection.weight"), L.cout, L.skip_c, 1))
      return -1;
    if (id_skip && pack_into(L.w, L.K, 0, 9 * L.cin, identity(L.cout), L.cout, L.cout, 1)) return -1;
    return finish_conv(p + ".c2", L, L.cout, bias);
  }
  int make_st(const std::string& p) {
    const std::string t = p + ".transformer_blocks.0";
    const int c = (int)H(p + ".norm.weight").first[0];
    if (make_norm(p + ".norm", p + ".norm")) return -1;
    if (make_conv(p + ".proj_in", p + ".proj_in.weight", p + ".proj_in.bias", 1)) return -1;
    if (make_lin_res(p + ".proj_out", p + ".proj_out.weight", p + ".proj_out.bias")) return -1;
    if (make_lin_res(p + ".to_out", t + ".attn1.to_out.0.weight", t + ".attn1.to_out.0.bias")) return -1;
    if (make_conv(p + ".ff1", t + ".ff.net.0.proj.weight", t + ".ff.net.0.proj.bias", 1)) return -1;
    {  // the same projection with GEGLU fused into the epilogue (clustered kernel): tile t of 128 rows =
       // x rows 64t..64t+63 followed by gate rows inner+64t..inner+64t+63
      const HostT& W = H(t + ".ff.net.0.proj.weight");
      const auto& b = H(t + ".ff.net.0.proj.bias").second;
      const int inner = 4 * c;
      HostT Wp;
      Wp.first = W.first;
      Wp.second.resize(W.second.size());
      std::vector<float> bp(2 * inner);
      for (int tl = 0; tl < inner / 64; ++tl)
        for (int half = 0; half < 2; ++half)
          for (int j = 0; j < 64; ++j) {
            const int src = half * inner + tl * 64 + j, dst = tl * 128 + half * 64 + j;
            std::copy(W.second.begin() + (size_t)src * c, W.second.begin() + (size_t)(src + 1) * c,
                      Wp.second.begin() + (size_t)dst * c);
            bp[dst] = b[src];
          }
      nope::LdmConv L;
      L.mode = 1;
      L.cin = c;
      L.cout = 2 * inner;
      L.K = c;
      L.geglu = true;
      if (alloc_w(L, 2 * inner) || pack_into(L.w, c, 0, 0, Wp, 2 * inner, c, 1) ||
          finish_conv(p + ".ff1g", L, 2 * inner, bp))
        return -1;
      NOPE_CHECK(convs.at(p + ".ff1g").bn == 128, "GEGLU projection must tile by 128");
    }
    if (make_lin_res(p + ".ff2", t + ".ff.net.2.weight", t + ".ff.net.2.bias")) return -1;
    {  // q | k | v of the self-attention as one GEMM (no bias, ldm/attention.py:160-162)
      nope::LdmConv L;
      L.mode = 1;
      L.cin = c;
      L.cout = 3 * c;
      L.K = c;
      if (alloc_w(L, 3 * c)) return -1;
      if (pack_into(L.w, c, 0, 0, H(t + ".attn1.to_q.weight"), c, c, 1) ||
          pack_into(L.w, c, c, 0, H(t + ".attn1.to_k.weight"), c, c, 1) ||
          pack_into(L.w, c, 2 * c, 0, H(t + ".attn1.to_v.weight"), c, c, 1))
        return -1;
      if (finish_conv(p + ".qkv", L, 3 * c, {})) return -1;
    }
    for (int n = 1; n <= 3; n += 2) {   // norm2 only feeds attn2's queries, which cancel (see below)
      nope::LdmNorm ln;
      ln.C = c;
      if (upload(H(t + ".norm" + std::to_string(n) + ".weight").second, &ln.gamma) ||
          upload(H(t + ".norm" + std::to_string(n) + ".bias").second, &ln.beta))
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
    const auto& Wp = H("pose_mlp.0.weight").second;   // [ctx][6]
    const auto& bp = H("pose_mlp.0.bias").second;
    for (const auto& kv : cb_off) {
      const std::string t = kv.first + ".transformer_blocks.0.attn2";
      const auto& Wv = H(t + ".to_v.weight").second;       // [c][ctx]
      const auto& Wo = H(t + ".to_out.0.weight").second;   // [c][c]
      const auto& bo = H(t + ".to_out.0.bias").second;
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
    return upload(Wc, &cross_w) || upload(bc, &cross_b) ? -1 : 0;
  }

  int finalize() {
    NOPE_CHECK(!finalized, "already finalized");
    for (const auto& kv : expected) NOPE_CHECK(host.count(kv.first), "state_dict is missing " + kv.first);
    NOPE_CUDA(cudaSetDevice(device));
    if (upload(H("input_blocks.0.0.weight").second, &in_w) || upload(H("input_blocks.0.0.bias").second, &in_b))
      return -1;
    {  // out[2]: Cl output channels padded to one 64-wide tile of the tensor-core kernel
      HostT W;
      W.first = {64, mc, 3, 3};
      W.second.assign((size_t)64 * mc * 9, 0.f);
      const auto& w = H("out.2.weight").second;
      std::copy(w.begin(), w.end(), W.second.begin());
      std::vector<float> bias(64, 0.f);
      std::copy(H("out.2.bias").second.begin(), H("out.2.bias").second.end(), bias.begin());
      nope::LdmConv L;
      L.mode = 0;
      L.cout = 64;
      L.cin = mc;
      L.K = 9 * mc;
      if (alloc_w(L, 64) || pack_into(L.w, L.K, 0, 0, W, 64, mc, 9) || finish_conv("out.2", L, 64, bias)) return -1;
    }
    for (size_t i = 1; i < inp.size(); ++i) {
      const std::string p = "input_blocks." + std::to_string(i);
      if (inp[i].kind == 1) {
        if (make_res(p + ".0") || make_st(p + ".1")) return -1;
      } else {
        if (make_conv(p + ".0.op", p + ".0.op.weight", p + ".0.op.bias", 4)) return -1;
      }
    }
    if (make_res("middle_block.0") || make_st("middle_block.1") || make_res("middle_block.2")) return -1;
    for (size_t i = 0; i < outp.size(); ++i) {
      const std::string p = "output_blocks." + std::to_string(i);
      if (make_res(p + ".0") || make_st(p + ".1")) return -1;
      if (outp[i].up && make_conv(p + ".2.conv", p + ".2.conv.weight", p + ".2.conv.bias", 3)) return -1;
    }
    if (make_norm("out.0", "out.0")) return -1;
    if (make_cross()) return -1;
    host.clear();
    finalized = true;
    return 0;
  }

  // ------------------------------------------------------------------ workspace
  int ws_half(__half** p, size_t n) {
    NOPE_CUDA(cudaMalloc(reinterpret_cast<void**>(p), n * sizeof(__half)));
    ws_owned.push_back(*p);
    return 0;
  }
  template <typename T> int ws_any(T** p, size_t n) {
    NOPE_CUDA(cudaMalloc(reinterpret_cast<void**>(p), n * sizeof(T)));
    ws_owned.push_back(*p);
    return 0;
  }
  int ensure_workspace(int need_cap, int need_ref) {
    if (need_cap <= cap && need_ref <= cap_ref) return 0;
    NOPE_CUDA(cudaDeviceSynchronize());
    for (void* p : ws_owned) cudaFree(p);
    ws_owned.clear();
    tmaps.clear();
    tmaps3.clear();
    cap = std::max(cap, need_cap);
    cap_ref = std::max(cap_ref, need_ref);
    const size_t c = (size_t)cap;
    const size_t u = (size_t)S0 * S0 * mc;        // one full-resolution base-width map
    HS.assign(inp.size(), nullptr);
    {
      int S = S0;
      for (size_t i = 0; i < inp.size(); ++i) {
        if (inp[i].kind == 2) S /= 2;
        if (ws_half(&HS[i], c * S * S * inp[i].cout)) return -1;
      }
    }
    // widest tensors: block outputs <= 2u (512 ch at 32^2 after the last upsample), ResBlock
    // inputs <= 3u (768 ch at 32^2), q|k|v 3u, V^T 1u, GEGLU input 8u, output 4u
    if (ws_half(&XA, c * 2 * u) || ws_half(&XB, c * 2 * u) || ws_half(&XC, c * 2 * u) || ws_half(&R, c * u) ||
        ws_half(&T1, c * 3 * u) || ws_half(&T2, c * u) || ws_half(&T3, c * u) || ws_half(&XN, c * u) ||
        ws_half(&PI, c * u) || ws_half(&PJ, c * u) || ws_half(&QKV, c * 3 * u) || ws_half(&Vt, c * u) || ws_half(&AO, c * u) || ws_half(&FF, c * 8 * u) ||
        ws_half(&GG, c * 4 * u) || ws_half(&x0ref, (size_t)cap_ref * u) || ws_half(&Rref, (size_t)cap_ref * u) ||
        ws_half(&Pref, (size_t)cap_ref * u))
      return -1;
    const size_t st = (size_t)32 * 256;   // parts (<= 32) x octets (<= 256) per image
    if (ws_any(&S_in, c * st) || ws_any(&S_mid, c * st) || ws_any(&S_out, c * st)) return -1;
    if (ws_any(&cb, c * (size_t)cb_width) || ws_any(&ref_of, c) || ws_any(&OF, c * S0 * S0 * 64)) return -1;
    return 0;
  }

  // ------------------------------------------------------------------ tensor maps
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

  // ------------------------------------------------------------------ op launchers
  // out[n_img, So, So, cout] = conv(L, in) [+ 1x1 skip over cat(sk0, sk1)] + bias [+ res]
  int conv(const nope::LdmConv& L, const __half* in, __half* out, int So, int n_img, cudaStream_t st,
           float2* stats = nullptr, const __half* res = nullptr, const __half* sk0 = nullptr, int skc0 = 0,
           const __half* sk1 = nullptr, int skc1 = 0, float* out_f32 = nullptr) {
    using namespace nope;
    NOPE_CHECK(skc0 + skc1 == L.skip_c, "conv: skip channel mismatch");
    ++launches;
    TileGeom g;
    if (make_geom(L.mode == 3 ? So / 2 : So, L.mode == 3 ? So / 2 : So, &g)) return -1;
    ConvParams p;
    memset(&p, 0, sizeof p);
    const CUtensorMap* m = nullptr;
    int nseg = 0, ksteps = 0, nmaps = 0;
    const int nch = L.cin / 64;
    p.n_par = 1;
    if (L.mode == 3) {
      if (get_map(&m, in, L.cin, g, -1)) return -1;
      p.amap[nmaps++] = *m;
      for (int a = 0; a < 2; ++a)
        for (int b = 0; b < 2; ++b) {
          p.seg[nseg++] = ConvSeg{0, (int16_t)(a - 1), (int16_t)(b - 1), (int16_t)nch};
          ksteps += nch;
        }
      p.n_par = 4;
    } else if (L.mode == 4) {
      // in(2y + ky - 1, 2x + kx - 1) on the four stride-2 lattices of the 2So x 2So input
      for (int t = 0; t < 4; ++t) {
        if (get_map(&m, in, L.cin, g, t)) return -1;
        p.amap[nmaps++] = *m;
      }
      for (int ky = 0; ky < 3; ++ky)
        for (int kx = 0; kx < 3; ++kx) {
          const int oy = ky - 1, ox = kx - 1;
          const int p1 = oy & 1, p2 = ox & 1;
          p.seg[nseg++] = ConvSeg{(int16_t)(p1 * 2 + p2), (int16_t)((oy - p1) / 2), (int16_t)((ox - p2) / 2),
                                  (int16_t)nch};
          ksteps += nch;
        }
    } else {
      if (get_map(&m, in, L.cin, g, -1)) return -1;
      p.amap[nmaps++] = *m;
      const int taps = L.mode == 0 ? 9 : 1;
      for (int t = 0; t < taps; ++t) {
        p.seg[nseg++] = ConvSeg{0, (int16_t)(L.mode == 0 ? t / 3 - 1 : 0), (int16_t)(L.mode == 0 ? t % 3 - 1 : 0),
                                (int16_t)nch};
        ksteps += nch;
      }
    }
    if (L.skip_c) {
      NOPE_CHECK((L.mode == 0 || L.mode == 1) && sk0 && skc0 % 64 == 0 && skc1 % 64 == 0, "conv: bad skip sources");
      if (get_map(&m, sk0, skc0, g, -1)) return -1;
      p.amap[nmaps] = *m;
      p.seg[nseg++] = ConvSeg{(int16_t)nmaps, 0, 0, (int16_t)(skc0 / 64)};
      ksteps += skc0 / 64;
      ++nmaps;
      if (sk1) {
        if (get_map(&m, sk1, skc1, g, -1)) return -1;
        p.amap[nmaps] = *m;
        p.seg[nseg++] = ConvSeg{(int16_t)nmaps, 0, 0, (int16_t)(skc1 / 64)};
        ksteps += skc1 / 64;
        ++nmaps;
      }
    }
    p.n_amaps = nmaps;
    for (int t = nmaps; t < kMaxAMaps; ++t) p.amap[t] = p.amap[0];
    p.bmap = L.wmap;
    p.bmap2 = L.wmap2;
    if (L.mode == 3) {
      for (int t = 0; t < 4; ++t) {
        if (get_map(&m, out, L.cout, g, t)) return -1;
        p.omap[t] = *m;
      }
    } else {
      if (get_map(&m, out, L.geglu ? L.cout / 2 : L.cout, g, -1)) return -1;
      for (int t = 0; t < 4; ++t) p.omap[t] = *m;
    }
    p.geglu = L.geglu ? 1 : 0;
    p.bias = L.bias;
    p.res_hi = res;
    p.out_f32 = out_f32;
    p.stats = stats;
    p.stats_hw = So * So;
    p.stats_noct = L.cout / 8;
    p.n_total = L.cout;
    p.m_valid = n_img * g.H * g.W;
    p.nseg = nseg;
    p.ksteps = ksteps;
    p.m_tiles = geom_m_tiles(g, n_img);
    const int bn = conv_impl == 2 ? L.bn : L.bn1;
    p.n_tiles_par = L.cout / bn;
    p.n_tiles = p.n_tiles_par * p.n_par;
    p.tiles_per_img = g.tiles_per_img;
    p.h_cnt = g.h_cnt;
    p.b_cnt = g.b_cnt;
    NOPE_CHECK(ksteps * 64 == L.K, "conv: K mismatch");
    if (precision) {
      // exact weights: the same segments again over the W_lo columns (weight columns simply continue past K)
      NOPE_CHECK(2 * nseg <= kMaxSeg, "conv: segment table overflow");
      for (int i = 0; i < nseg; ++i) p.seg[nseg + i] = p.seg[i];
      nseg *= 2;
      ksteps *= 2;
    }
    NOPE_CHECK(nseg <= kMaxSeg, "conv: segment table overflow");
    p.nseg = nseg;
    p.ksteps = ksteps;
    NOPE_CHECK(!((stats || res) && L.mode == 3), "upsample conv has no fused statistics / residual");
    if (profile && prof_begin(st)) return -1;
    const int rc = conv_impl == 2 ? launch_conv_tc2(p, bn, num_sms, st) : launch_conv_tc(p, bn, num_sms, st);
    // executed FLOPs (the folded upsample runs 4 parity GEMMs of K = 4 Cin over the source pixels)
    if (profile && prof_end(st, 2.0 * (double)n_img * g.H * g.W * (double)(L.mode == 3 ? 4 * L.cout : L.cout) * (double)L.k_alg, 0))
      return -1;
    return rc;
  }

  // out = L(in) + res: residual as an identity K-segment (fold_residual) or in the epilogue
  int lin_res(const nope::LdmConv& L, const __half* in, __half* out, const __half* res, int C, int S, int n,
              cudaStream_t st) {
    if (L.skip_c) return conv(L, in, out, S, n, st, nullptr, nullptr, res, C);
    return conv(L, in, out, S, n, st, nullptr, res);
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
  int get_map3(const CUtensorMap** out, const void* base, int d0, int d1, int d2, int b0, int b1) {
    auto key = std::make_tuple(base, d0, d1, d2);
    auto it = tmaps3.find(key);
    if (it == tmaps3.end()) {
      CUtensorMap m;
      if (nope::make_tmap3_f16(&m, base, d0, d1, d2, b0, b1)) return -1;
      it = tmaps3.emplace(key, m).first;
    }
    *out = &it->second;
    return 0;
  }
  // self-attention core on qkv [n, ntok, 3C] -> out [n, ntok, C]
  int attention(const __half* qkv, __half* out, int C, int ntok, int n, cudaStream_t st) {
    using namespace nope;
    const int Hh = C / 32;
    NOPE_CHECK(ntok % 64 == 0 && C % 64 == 0, "attention: tokens and channels must be multiples of 64");
    ldm_attn_prep_kernel<<<dim3(ntok / 64, n), 256, 0, st>>>(qkv, Vt, ntok, C);
    NOPE_CUDA(cudaGetLastError());
    const float sl2e = 0.17677669529663687f * 1.4426950408889634f;   // 32^-1/2 * log2(e)
    const dim3 grid((unsigned)(n * Hh) * (unsigned)((ntok + 127) / 128));
    if (profile && prof_begin(st)) return -1;
    if (attn_impl == 1) {
      ldm_attn_simt_kernel<<<grid, 128, 0, st>>>(qkv, Vt, out, ntok, Hh, C, sl2e);
    } else {
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
      if (get_map3(&m, qkv, 3 * C, ntok, n, 64, 128)) return -1;
      p.qkmap = *m;
      if (get_map3(&m, Vt, ntok, 32, n * Hh, 64, 32)) return -1;
      p.vmap = *m;
      p.out = out; p.n = ntok; p.H = Hh; p.C = C; p.scale_log2e = sl2e;
      ldm_attn_tc_kernel<<<grid, 128, kAttnSmem, st>>>(p);
    }
    NOPE_CUDA(cudaGetLastError());
    if (profile && prof_end(st, 4.0 * (double)n * ntok * (double)ntok * C, 1)) return -1;
    launches += 2;
    return 0;
  }

  int tap(const std::string& name, const __half* buf, int C, int S, int n, cudaStream_t st) {
    if (tap_out == nullptr || tap_name != name || tap_hit) return 0;
    NOPE_CHECK((int64_t)n * C * S * S <= tap_cap, "debug tap: output buffer too small");
    nope::nhwc_f16_to_nchw_f32_kernel<<<nope::ew_grid((long long)n * C * S * S), 256, 0, st>>>(buf, tap_out, n, C, S * S);
    NOPE_CUDA(cudaGetLastError());
    tap_C = C; tap_S = S; tap_hit = true;
    return 0;
  }

  // ResBlock._forward (ldm/openaimodel.py:265-286) on cat(x0, x1).  Leaves the GroupNorm
  // statistics of `out` in S_out (conv epilogue) for a following SpatialTransformer.norm.
  int resblock(const std::string& p, const __half* x0, int C0, const __half* x1, int C1, __half* out, int S, int n,
               cudaStream_t st) {
    const nope::LdmConv& c1 = convs.at(p + ".c1");
    const nope::LdmConv& c2 = convs.at(p + ".c2");
    NOPE_CHECK(c1.cin == C0 + C1, "resblock: channel mismatch");
    if (stats(x0, C0, x1, C1, S, n, S_in, st)) return -1;
    if (gn(norms.at(p + ".n1"), x0, C0, x1, C1, S_in, S, n, T1, true, 1e-5f, st)) return -1;
    if (conv(c1, T1, T2, S, n, st, S_mid)) return -1;
    if (gn(norms.at(p + ".n2"), T2, c1.cout, nullptr, 0, S_mid, S, n, T3, true, 1e-5f, st)) return -1;
    if (c2.skip_c) return conv(c2, T3, out, S, n, st, S_out, nullptr, x0, C0, x1, C1);
    NOPE_CHECK(x1 == nullptr && C0 == c2.cout, "resblock: identity skip needs Cin == Cout");
    return conv(c2, T3, out, S, n, st, S_out, x0);    // epilogue add (fold_residual off)
  }

  // SpatialTransformer.forward (ldm/attention.py:264-277) with one BasicTransformerBlock
  // (:229-233), in two halves.  st_pre: norm, proj_in, x = attn1(norm1(x)) + x -> `xs`; nothing in
  // it depends on the pose.  x_in's GroupNorm statistics must be in S_out.
  int st_pre(const std::string& p, const __half* x_in, __half* xs, int C, int S, int n, cudaStream_t st) {
    if (gn(norms.at(p + ".norm"), x_in, C, nullptr, 0, S_out, S, n, XN, false, 1e-6f, st)) return -1;
    if (conv(convs.at(p + ".proj_in"), XN, PI, S, n, st)) return -1;
    if (ln(norms.at(p + ".ln1"), PI, nullptr, nullptr, XN, C, S, n, st)) return -1;
    if (conv(convs.at(p + ".qkv"), XN, QKV, S, n, st)) return -1;
    if (attention(QKV, AO, C, S * S, n, st)) return -1;
    return lin_res(convs.at(p + ".to_out"), AO, xs, PI, C, S, n, st);
  }
  // st_post: x = attn2(norm2(x), context) + x -- the one-token cross-attention is the
  // per-hypothesis vector cb (see make_cross), added by the LayerNorm kernel, which also applies
  // norm3 -- then x = ff(norm3(x)) + x (GEGLU) and proj_out(x) + x_in.  `xs` may hold one image
  // per reference (src_img maps hypothesis -> image); x_in and out are per hypothesis.
  int st_post(const std::string& p, const __half* xs, const int* src_img, const __half* x_in, __half* out, int C,
              int S, int n, const float* cbp, cudaStream_t st) {
    if (ln(norms.at(p + ".ln3"), xs, PJ, cbp + cb_off.at(p), XN, C, S, n, st, src_img)) return -1;
    // GEGLU: fused into the projection's epilogue on the clustered kernel
    if (conv_impl == 2 && fuse_geglu) {
      if (conv(convs.at(p + ".ff1g"), XN, GG, S, n, st)) return -1;
    } else {
      if (conv(convs.at(p + ".ff1"), XN, FF, S, n, st)) return -1;
      nope::ldm_geglu_kernel<<<nope::ew_grid((long long)n * S * S * C / 2), 256, 0, st>>>(FF, GG, (long long)n * S * S,
                                                                                        4 * C);
      NOPE_CUDA(cudaGetLastError());
      ++launches;
    }
    if (lin_res(convs.at(p + ".ff2"), GG, PI, PJ, C, S, n, st)) return -1;
    return lin_res(convs.at(p + ".proj_out"), PI, out, x_in, C, S, n, st);
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
  int forward_chunk(const float* poses, int hyp0, int n, int N, const float* query, float* out_emb,
                    float* score_part, cudaStream_t st) {
    using namespace nope;
    ldm_ref_of_kernel<<<(n + 255) / 256, 256, 0, st>>>(ref_of, hyp0, N, n);
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
    if (conv(convs.at("out.2"), T1, T2, S, n, st, nullptr, nullptr, nullptr, 0, nullptr, 0, OF)) return -1;
    ldm_score_kernel<<<dim3(nslab, n), kFinalThreads, 0, st>>>(
        OF, out_emb ? out_emb + (size_t)hyp0 * Cl * hw : nullptr, query, ref_of,
        score_part ? score_part + (size_t)hyp0 * nslab : nullptr, hw, Cl);
    NOPE_CUDA(cudaGetLastError());
    ++launches;
    return 0;
  }
};
