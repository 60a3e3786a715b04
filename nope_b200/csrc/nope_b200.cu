// nope_b200 -- the C ABI (include/nope_b200.h) over the engines (unet.cuh, encoder.cuh, vae.cuh, ldm.cuh) and the
// stand-alone kernels, with the launch-scoped helpers its entry points use.  Host code is plain C++.
#include "../../include/nope_b200.h"

#include <algorithm>
#include <climits>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <functional>
#include <map>
#include <memory>
#include <string>
#include <tuple>
#include <type_traits>
#include <vector>

#include "common.cuh"
#include "engine.cuh"
#include "conv_tc.cuh"
#include "conv_tc2.cuh"
#include "kernels.cuh"
#include "rank.cuh"
#include "linattn_tc.cuh"
#include "unet.cuh"
#include "encoder.cuh"
#include "vae.cuh"
#include "ldm.cuh"
#include "render.cuh"
#include "pose_error.cuh"
#include "crop.cuh"
#include "translation.cuh"
#include "depth_refine.cuh"
#include "contour_refine.cuh"
#include "distinct.cuh"
#include "track.cuh"

using namespace nope;

namespace {

constexpr int kAbiVersion = 3;

int to_nhwc(const float* x, __half** out, DeviceAllocs& s, int n, int C, int hw, cudaStream_t st,
            __half** out_lo = nullptr) {
  if (s.alloc(out, (size_t)n * C * hw)) return -1;
  if (out_lo && s.alloc(out_lo, (size_t)n * C * hw)) return -1;
  nchw_f32_to_nhwc_f16_kernel<<<ew_grid((long long)n * C * hw), 256, 0, st>>>(x, *out, n, C, hw,
                                                                              out_lo ? *out_lo : nullptr);
  NOPE_CUDA(cudaGetLastError());
  return 0;
}
int to_nchw(const __half* x, float* out, int n, int C, int hw, cudaStream_t st, const __half* x_lo = nullptr) {
  nhwc_f16_to_nchw_f32_kernel<<<ew_grid((long long)n * C * hw), 256, 0, st>>>(x, out, n, C, hw, x_lo);
  NOPE_CUDA(cudaGetLastError());
  return 0;
}

// A launcher's stream-ordered scratch: every field is declared with add(), each aligned to 256 bytes, then alloc()
// makes one cudaMallocAsync, points the fields into it and copies in those declared with a HOST source (pageable,
// staged at once: no host synchronisation).  The block is freed in stream order, after the kernels that use it, when
// the arena goes out of scope.
class ScratchArena {
 public:
  explicit ScratchArena(cudaStream_t st) : st_(st) {}
  ScratchArena(const ScratchArena&) = delete;
  ScratchArena& operator=(const ScratchArena&) = delete;
  ~ScratchArena() {
    if (base_) cudaFreeAsync(base_, st_);
  }
  template <typename T> void add(T** field, size_t count, const std::remove_const_t<T>* host = nullptr) {
    bytes_ = (bytes_ + kAlign - 1) & ~(kAlign - 1);
    fields_.push_back({[field](char* p) { *field = reinterpret_cast<T*>(p); }, bytes_, host, sizeof(T) * count});
    bytes_ += sizeof(T) * count;
  }
  int alloc() {
    NOPE_CUDA(cudaMallocAsync(reinterpret_cast<void**>(&base_), std::max<size_t>(bytes_, 1), st_));
    for (const Field& f : fields_) {
      f.point(base_ + f.offset);
      if (f.host) NOPE_CUDA(cudaMemcpyAsync(base_ + f.offset, f.host, f.bytes, cudaMemcpyHostToDevice, st_));
    }
    return 0;
  }

 private:
  struct Field {
    std::function<void(char*)> point;
    size_t offset;
    const void* host;
    size_t bytes;
  };
  static constexpr size_t kAlign = 256;
  cudaStream_t st_;
  char* base_ = nullptr;
  size_t bytes_ = 0;
  std::vector<Field> fields_;
};

// HOST intrinsics K [F, 4] (fx, fy, cx, cy): checked (finite, fx and fy non-zero) and declared as an arena field that
// alloc() copies in
int stage_host_intrinsics(ScratchArena& arena, const double** dev, const double* K, int F) {
  for (int f = 0; f < F; ++f) {
    const double* k = K + 4 * (size_t)f;
    NOPE_CHECK(std::isfinite(k[0]) && std::isfinite(k[1]) && std::isfinite(k[2]) && std::isfinite(k[3]),
               "intrinsics must be finite");
    NOPE_CHECK(k[0] != 0.0 && k[1] != 0.0, "fx and fy must be non-zero");
  }
  arena.add(dev, 4 * (size_t)F, K);
  return 0;
}

// nope_score_topk_grouped and, with a visible map [R, HW], nope_score_topk_visible: the argument checks, one CTA per
// (template n, group g) scoring slot slots[g]'s template n against the group's rows, then with k > 0 the joint top-k
// over (row a, template n) of every A consecutive rows (sim viewed as [R / A, A * N]).
int score_grouped(const float* query_feat, const float* emb, int R, int O, int N, int C, int HW, const int32_t* slots,
                  const int32_t* row_off, int G, int A, const uint8_t* visible, int metric, float occlusion_threshold,
                  int k, float* out_sim, float* out_topv, int64_t* out_topi, void* stream) {
  NOPE_CHECK(query_feat && emb && slots && row_off && out_sim, "null argument");
  NOPE_CHECK(R >= 1 && O >= 1 && N >= 1 && C >= 1 && HW >= 1, "bad arguments");
  NOPE_CHECK(G >= 1 && G <= 65535, "G (row groups) must be in [1, 65535]");
  NOPE_CHECK(A >= 1 && R % A == 0, "R (query rows) must be a multiple of A (rows per search row) >= 1");
  NOPE_CHECK(O <= 65535 && (int64_t)R * N <= INT32_MAX, "too many templates or (query, template) pairs");
  NOPE_CHECK(!visible || (int64_t)R * HW <= INT32_MAX, "R * HW (visible map entries) exceeds 2^31 - 1");
  NOPE_CHECK(metric == NOPE_METRIC_L2 || metric == NOPE_METRIC_COSINE || metric == NOPE_METRIC_COSINE_OCC,
             "unknown similarity metric (l2, cosine and cosine_occlusion exist)");
  NOPE_CHECK(k >= 0 && k <= kMaxTopK && (int64_t)k <= (int64_t)A * N, "k must be in [0, min(64, A * N)]");
  NOPE_CHECK(k == 0 || (out_topv && out_topi), "top-k outputs missing");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  if (visible)
    score_kernel<true><<<dim3(N, G), 256, 0, st>>>(query_feat, emb, out_sim, N, C, HW, metric, occlusion_threshold, 0,
                                                   slots, row_off, visible);
  else
    score_kernel<<<dim3(N, G), 256, 0, st>>>(query_feat, emb, out_sim, N, C, HW, metric, occlusion_threshold, 0,
                                             slots, row_off);
  NOPE_CUDA(cudaGetLastError());
  if (k > 0) {
    sim_topk_kernel<<<R / A, 256, 0, st>>>(nullptr, 0, out_sim, A * N, k, out_topv,
                                           reinterpret_cast<long long*>(out_topi), 0LL);
    NOPE_CUDA(cudaGetLastError());
  }
  return 0;
}
}  // namespace

// =============================================================================
// C ABI
// =============================================================================
extern "C" {

const char* nope_last_error(void) { return last_error().c_str(); }
int nope_abi_version(void) { return kAbiVersion; }
const char* nope_build_arch(void) { return "sm_90a"; }

int nope_unet_create(nope_unet_t** out, int u_net_dim, int latent_ch, int latent_hw, int device) {
  NOPE_CHECK(out != nullptr, "null out pointer");
  NOPE_CHECK(u_net_dim > 0 && u_net_dim % 64 == 0, "u_net_dim must be a positive multiple of 64");
  NOPE_CHECK(latent_ch >= 1 && latent_ch <= kMaxLatent, "latent_ch must be in [1, 8]");
  NOPE_CHECK(latent_hw == 32, "latent_hw must be 32 (256x256 images) in this build");
  auto u = std::make_unique<nope_unet>();
  if (open_device(device, &u->num_sms)) return -1;
  u->dim = u_net_dim;
  u->Cl = latent_ch;
  u->S0 = latent_hw;
  u->cemb = 4 * u_net_dim;
  u->device = device;
  const int mults[4] = {1, 2, 4, 8};
  u->dims[0] = u_net_dim;
  for (int i = 0; i < 4; ++i) u->dims[i + 1] = u_net_dim * mults[i];
  u->build_schema();
  *out = u.release();
  return 0;
}

void nope_unet_destroy(nope_unet_t* u) { delete u; }

int nope_unet_load_tensor(nope_unet_t* u, const char* key, const float* data, const int64_t* shape,
                          int ndim) {
  return engine_load_tensor(u, key, data, shape, ndim);
}

int nope_unet_finalize(nope_unet_t* u) { return engine_finalize(u); }

int nope_unet_set_chunk(nope_unet_t* u, int hyps) {
  NOPE_CHECK(u && hyps >= 1 && hyps <= 4096, "chunk must be in [1, 4096]");
  u->chunk = hyps;
  return 0;
}
int nope_unet_set_option(nope_unet_t* u, const char* name, int value) {
  NOPE_CHECK(u && name, "null argument");
  if (std::strcmp(name, "precision") == 0) {
    NOPE_CHECK(!u->finalized, "precision must be set before nope_unet_finalize");
    NOPE_CHECK(value >= 0 && value <= 4, "precision must be 0 (fp16), 1 (exact weights), 2 (split), 3 (bf16) or 4 (split, fp16 inside ResnetBlocks)");
    u->precision = value;
    return 0;
  }
  return fail(std::string("unknown option: ") + name);
}
int64_t nope_unet_last_launch_count(const nope_unet_t* u) { return u ? u->launches : 0; }

int64_t nope_unet_workspace_bytes(nope_unet_t* u, int hyps, int refs, int scores) {
  if (!u || !u->finalized || hyps < 1 || refs < 1 || scores < 0) {
    fail("nope_unet_workspace_bytes: finalized engine, hyps >= 1, refs >= 1 required");
    return -1;
  }
  return (int64_t)u->workspace_bytes(hyps, refs, scores);
}
int nope_unet_set_workspace(nope_unet_t* u, void* ptr, int64_t bytes, int hyps, int refs, int scores) {
  NOPE_CHECK(u && u->finalized, "engine not finalized");
  NOPE_CUDA(cudaSetDevice(u->device));
  return u->set_workspace(ptr, (size_t)bytes, hyps, refs, scores);
}

int nope_unet_profile(nope_unet_t* u, int enable) {
  NOPE_CHECK(u, "null engine");
  u->prof.reset(enable != 0);
  return 0;
}

int nope_unet_profile_read(nope_unet_t* u, double* conv_ms, double* conv_flops, double* conv_alg_flops,
                           int64_t* conv_launches, double* max_launch_tflops) {
  NOPE_CHECK(u && conv_ms && conv_flops && conv_launches, "null argument");
  NOPE_CUDA(cudaDeviceSynchronize());
  const LaunchProfile& pr = u->prof;
  double ms = 0.0, fl = 0.0, alg = 0.0, best = 0.0;
  for (size_t i = 0; i < pr.rec.size(); ++i) {
    float t = 0.f;
    if (pr.ms(i, &t)) return -1;
    ms += t;
    fl += pr.rec[i].flops;
    alg += pr.rec[i].alg_flops;
    if (t > 0.f) best = std::max(best, pr.rec[i].flops / (t * 1e-3) / 1e12);
  }
  if (const char* path = std::getenv("NOPE_PROF_DUMP")) {     // development aid: per-launch table
    if (FILE* f = std::fopen(path, "a")) {
      std::fprintf(f, "# launch,ms,executed_gflop,algorithmic_gflop,res,mode,cout,k\n");
      for (size_t i = 0; i < pr.rec.size(); ++i) {
        float t = 0.f;
        pr.ms(i, &t);
        const int4 sh = pr.rec[i].shape;
        std::fprintf(f, "%zu,%.4f,%.3f,%.3f,%d,%d,%d,%d\n", i, t, pr.rec[i].flops / 1e9, pr.rec[i].alg_flops / 1e9,
                     sh.x, sh.y, sh.z, sh.w);
      }
      std::fclose(f);
    }
  }
  *conv_ms = ms;
  *conv_flops = fl;
  if (conv_alg_flops) *conv_alg_flops = alg;
  *conv_launches = (int64_t)pr.rec.size();
  if (max_launch_tflops) *max_launch_tflops = best;
  return 0;
}

int nope_unet_sweep_multi(nope_unet_t* u, const float* ref_feat, const float* poses, int B, int N,
                          const float* query_feat, int Q, float* out_emb, float* out_sim, int k, float* out_topv,
                          int64_t* out_topi, int64_t idx_base, void* stream) {
  return engine_sweep(u, ref_feat, poses, B, N, query_feat, Q, out_emb, out_sim, k, out_topv, out_topi, idx_base,
                      stream);
}

int nope_unet_set_metric(nope_unet_t* u, int metric, float occlusion_threshold) {
  NOPE_CHECK(u, "null engine");
  NOPE_CHECK(metric == NOPE_METRIC_L2 || metric == NOPE_METRIC_COSINE || metric == NOPE_METRIC_COSINE_OCC,
             "unknown similarity metric (l2, cosine and cosine_occlusion exist)");
  u->metric = metric;
  u->occ_threshold = occlusion_threshold;
  return 0;
}

int nope_score_topk_multi(const float* query_feat, const float* emb, int B, int Q, int Bt, int N, int C, int HW,
                          int metric, float occlusion_threshold, int k, float* out_sim, float* out_topv,
                          int64_t* out_topi, int64_t idx_base, void* stream) {
  NOPE_CHECK(query_feat && emb && out_sim, "null argument");
  NOPE_CHECK(B >= 1 && N >= 1 && C >= 1 && HW >= 1, "bad arguments");
  NOPE_CHECK(Q >= 1, "Q (queries per batch row) must be >= 1");
  NOPE_CHECK(Bt == 1 || Bt == B, "template batch Bt must be 1 or B");
  NOPE_CHECK(Bt <= 65535 && (int64_t)B * Q * N <= INT32_MAX, "too many templates or (query, template) pairs");
  NOPE_CHECK(metric == NOPE_METRIC_L2 || metric == NOPE_METRIC_COSINE || metric == NOPE_METRIC_COSINE_OCC,
             "unknown similarity metric (l2, cosine and cosine_occlusion exist)");
  NOPE_CHECK(k >= 0 && k <= N && k <= kMaxTopK, "k must be in [0, min(N, 64)]");
  NOPE_CHECK(k == 0 || (out_topv && out_topi), "top-k outputs missing");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  // query rows [B * Q] in order; template batch t serves rows [t * rows, (t + 1) * rows)
  const int rows = B * Q / Bt;
  score_kernel<<<dim3(N, Bt), 256, 0, st>>>(query_feat, emb, out_sim, N, C, HW, metric, occlusion_threshold, rows);
  NOPE_CUDA(cudaGetLastError());
  if (k > 0) {
    sim_topk_kernel<<<B * Q, 256, 0, st>>>(nullptr, 0, out_sim, N, k, out_topv,
                                           reinterpret_cast<long long*>(out_topi), (long long)idx_base);
    NOPE_CUDA(cudaGetLastError());
  }
  return 0;
}

int nope_score_topk_grouped(const float* query_feat, const float* emb, int R, int O, int N, int C, int HW,
                            const int32_t* slots, const int32_t* row_off, int G, int A, int metric,
                            float occlusion_threshold, int k, float* out_sim, float* out_topv, int64_t* out_topi,
                            void* stream) {
  return score_grouped(query_feat, emb, R, O, N, C, HW, slots, row_off, G, A, nullptr, metric, occlusion_threshold, k,
                       out_sim, out_topv, out_topi, stream);
}

int nope_topk(float* sim, int B, int N, int k, float* out_topv, int64_t* out_topi, int64_t idx_base,
              void* stream) {
  NOPE_CHECK(sim && out_topv && out_topi, "null argument");
  NOPE_CHECK(k >= 1 && k <= N && k <= kMaxTopK, "k must be in [1, min(N, 64)]");
  sim_topk_kernel<<<B, 256, 0, static_cast<cudaStream_t>(stream)>>>(
      nullptr, 0, sim, N, k, out_topv, reinterpret_cast<long long*>(out_topi), (long long)idx_base);
  NOPE_CUDA(cudaGetLastError());
  return 0;
}

int nope_pose_cells_expand(const int64_t* top_idx, int R, int keep, const int32_t* cells, int n_coarse, int F,
                           const float* poses, int B, int Q, int n_fine, int M, int32_t* out_cand, float* out_poses,
                           void* stream) {
  NOPE_CHECK(top_idx && cells && poses && out_cand && out_poses, "null argument");
  NOPE_CHECK(keep >= 1 && keep <= kMaxTopK, "keep must be in [1, 64]");
  NOPE_CHECK(n_coarse >= 1 && F >= 1 && n_fine >= 1 && B >= 1 && Q >= 1, "bad arguments");
  NOPE_CHECK(R >= 1 && (int64_t)B * Q == R, "R (rows) must equal B * Q");
  NOPE_CHECK((int64_t)M >= (int64_t)keep * F, "M must be at least keep * F (the largest union of keep cells)");
  pose_cells_expand_kernel<<<R, 256, 0, static_cast<cudaStream_t>(stream)>>>(
      reinterpret_cast<const long long*>(top_idx), keep, cells, n_coarse, F, poses, Q, n_fine, M, out_cand, out_poses);
  NOPE_CUDA(cudaGetLastError());
  return 0;
}

int nope_pose_cells_rank(const float* sim, const int32_t* cand, int R, int M, int n_fine, int k, float* out_sim,
                         float* out_topv, int64_t* out_topi, void* stream) {
  NOPE_CHECK(sim && cand && out_topv && out_topi, "null argument");
  NOPE_CHECK(k >= 1 && k <= kMaxTopK, "k must be in [1, 64]");
  NOPE_CHECK(R >= 1 && M >= 1 && n_fine >= 1, "bad arguments");
  pose_cells_rank_kernel<<<R, 256, 0, static_cast<cudaStream_t>(stream)>>>(
      sim, cand, M, n_fine, k, out_sim, out_topv, reinterpret_cast<long long*>(out_topi));
  NOPE_CUDA(cudaGetLastError());
  return 0;
}

int nope_pose_refine_propose(const float* D, const int32_t* seed, int R, int keep, const float* all_relativeR, int B,
                             int Q, int N, const float* stencil, float* out_D, int32_t* out_seed, float* out_rel,
                             float* out_poses, void* stream) {
  NOPE_CHECK(D && seed && all_relativeR && stencil && out_D && out_seed && out_rel && out_poses, "null argument");
  NOPE_CHECK(keep >= 1 && keep <= kMaxTopK, "keep must be in [1, 64]");
  NOPE_CHECK(B >= 1 && Q >= 1 && N >= 1, "bad arguments");
  NOPE_CHECK(R >= 1 && (int64_t)B * Q == R, "R (rows) must equal B * Q");
  pose_refine_propose_kernel<<<R, 256, 0, static_cast<cudaStream_t>(stream)>>>(
      D, seed, keep, all_relativeR, Q, N, stencil, out_D, out_seed, out_rel, out_poses);
  NOPE_CUDA(cudaGetLastError());
  return 0;
}

int nope_pose_refine_select(const float* sim, const float* cand_D, const int32_t* cand_seed, const float* cand_rel,
                            int R, int M, int k, float trace_threshold, float* out_D, int32_t* out_seed,
                            float* out_score, float* out_rel, void* stream) {
  NOPE_CHECK(sim && cand_D && cand_seed && cand_rel && out_D && out_seed && out_score, "null argument");
  NOPE_CHECK(k >= 1 && k <= kMaxTopK, "k must be in [1, 64]");
  NOPE_CHECK(M >= 1 && M <= kRefineMaxM, "M (candidates per row) must be in [1, 64 * 27]");
  NOPE_CHECK(k <= M, "k must not exceed M (candidates per row)");
  NOPE_CHECK(R >= 1, "bad arguments");
  pose_refine_select_kernel<<<R, 256, 0, static_cast<cudaStream_t>(stream)>>>(
      sim, cand_D, cand_seed, cand_rel, M, k, trace_threshold, out_D, out_seed, out_score, out_rel);
  NOPE_CUDA(cudaGetLastError());
  return 0;
}

int nope_pose_refine_inplane_propose(const float* D, const int32_t* seed, const float* cossin, int R, int keep,
                                     const float* all_relativeR, int B, int Q, int N, const float* stencil,
                                     float roll_cos, float roll_sin, float* out_D, int32_t* out_seed, float* out_rel,
                                     float* out_poses, float* out_cossin, void* stream) {
  NOPE_CHECK(D && seed && cossin && all_relativeR && stencil && out_D && out_seed && out_rel && out_poses &&
                 out_cossin, "null argument");
  NOPE_CHECK(keep >= 1 && keep <= kInplaneMaxKeep, "keep must be in [1, 16]");
  NOPE_CHECK(B >= 1 && Q >= 1 && N >= 1, "bad arguments");
  NOPE_CHECK(R >= 1 && (int64_t)B * Q == R, "R (rows) must equal B * Q");
  pose_refine_inplane_propose_kernel<<<R, 256, 0, static_cast<cudaStream_t>(stream)>>>(
      D, seed, cossin, keep, all_relativeR, Q, N, stencil, roll_cos, roll_sin, out_D, out_seed, out_rel, out_poses,
      out_cossin);
  NOPE_CUDA(cudaGetLastError());
  return 0;
}

int nope_pose_refine_inplane_select(const float* sim, const float* cand_D, const int32_t* cand_seed,
                                    const float* cand_rel, const float* cand_cossin, int R, int keep, int k,
                                    float trace_threshold, float* out_D, int32_t* out_seed, float* out_cossin,
                                    int32_t* out_aslot, float* out_score, float* out_rel, void* stream) {
  NOPE_CHECK(sim && cand_D && cand_seed && cand_rel && cand_cossin && out_D && out_seed && out_cossin && out_aslot &&
                 out_score, "null argument");
  NOPE_CHECK(keep >= 1 && keep <= kInplaneMaxKeep, "keep must be in [1, 16]");
  NOPE_CHECK(k >= 1 && k <= kMaxTopK, "k must be in [1, 64]");
  NOPE_CHECK(k <= kInplaneXY * kInplaneRoll * keep * keep, "k must not exceed the 27 * keep^2 pairs per row");
  NOPE_CHECK(R >= 1, "bad arguments");
  pose_refine_inplane_select_kernel<<<R, 256, 0, static_cast<cudaStream_t>(stream)>>>(
      sim, cand_D, cand_seed, cand_rel, cand_cossin, keep, k, trace_threshold, out_D, out_seed, out_cossin, out_aslot,
      out_score, out_rel);
  NOPE_CUDA(cudaGetLastError());
  return 0;
}

int64_t nope_topk_pack_floats(int B, int k, int n_local_max, int want_sim) {
  if (B < 1 || k < 1 || n_local_max < 0) return -1;
  const int64_t kk = ((int64_t)B * k + 1) & ~(int64_t)1;
  // rounded up to 4 floats: records sit back to back in the gathered buffer and every record's int64 block must
  // stay 8-byte aligned (an odd length misaligned every second record: 10 248 poses on 8 GPUs = 16 + 1281 floats)
  return (kk + 2 * (int64_t)B * k + (want_sim ? (int64_t)B * n_local_max : 0) + 3) & ~(int64_t)3;
}

int nope_topk_merge(const float* gathered, int world, int64_t pack_floats, int B, int k, int N, int per,
                    int has_sim, float* out_sim, float* out_topv, int64_t* out_topi, void* stream) {
  NOPE_CHECK(gathered && out_topv && out_topi, "null argument");
  NOPE_CHECK(world >= 1 && B >= 1 && k >= 1 && k <= N && world * k <= 1024, "bad merge geometry (world * k <= 1024)");
  NOPE_CHECK(per >= 1 && (int64_t)per * world >= N, "per-rank pose count does not cover the grid");
  NOPE_CHECK(pack_floats >= nope_topk_pack_floats(B, k, has_sim ? per : 0, has_sim) - 3, "packed record too short");
  NOPE_CHECK(pack_floats % 2 == 0 && (reinterpret_cast<uintptr_t>(gathered) & 7) == 0,
             "packed records must be 8-byte aligned: use nope_topk_pack_floats for the record length");
  NOPE_CHECK(!has_sim || out_sim, "similarity output missing");
  topk_merge_kernel<<<B, 256, 0, static_cast<cudaStream_t>(stream)>>>(
      gathered, world, (long long)pack_floats, B, k, N, per, has_sim, out_sim, out_topv,
      reinterpret_cast<long long*>(out_topi));
  NOPE_CUDA(cudaGetLastError());
  return 0;
}

// ---------------------------------------------------------------------------------
// template encoder
// ---------------------------------------------------------------------------------
int nope_encoder_create(nope_encoder_t** out, int descriptor_size, int device) {
  NOPE_CHECK(out != nullptr, "null out pointer");
  NOPE_CHECK(descriptor_size >= 1 && descriptor_size <= 64, "descriptor_size must be in [1, 64]");
  auto e = std::make_unique<nope_encoder>();
  if (open_device(device, &e->num_sms)) return -1;
  e->D = descriptor_size;
  e->device = device;
  e->build_plan();
  e->build_schema();
  *out = e.release();
  return 0;
}

void nope_encoder_destroy(nope_encoder_t* e) { delete e; }

int nope_encoder_load_tensor(nope_encoder_t* e, const char* key, const float* data, const int64_t* shape,
                             int ndim) {
  return engine_load_tensor(e, key, data, shape, ndim);
}

int nope_encoder_finalize(nope_encoder_t* e) { return engine_finalize(e); }

// "precision" of the template encoder and the VAE encoder: the name and the value are checked before the handle, so
// every refusal happens before any CUDA call
extern "C++" template <class Engine>
int encoder_set_option(Engine* e, const char* name, int value) {
  NOPE_CHECK(name, "null option name");
  if (std::strcmp(name, "precision") != 0) return fail(std::string("unknown option: ") + name);
  NOPE_CHECK(value == 0 || value == 1, "precision must be 0 (split) or 1 (fp16)");
  NOPE_CHECK(e, "null engine");
  NOPE_CHECK(!e->finalized, "precision must be set before finalize");
  e->precision = value;
  return 0;
}
int nope_encoder_set_option(nope_encoder_t* e, const char* name, int value) {
  return encoder_set_option(e, name, value);
}

// The entry points of the image engines (template encoder, VAE encoder, VAE decoder) check their arguments, then the
// handle (image_engine_ready), so every refusal comes before any CUDA call.
extern "C++" template <class Engine>
int image_engine_ready(Engine* e) {
  NOPE_CHECK(e && e->finalized, std::string(Engine::kName) + " not finalized");
  NOPE_CUDA(cudaSetDevice(e->device));
  return 0;
}

// *_encode / *_decode: B inputs of in_per floats, any B, Engine::kChunk at a time through step
extern "C++" template <class Engine>
int engine_encode(Engine* e, int (Engine::*step)(const float*, int, float*, cudaStream_t), const char* what,
                  const float* in, size_t in_per, int B, float* out, void* stream) {
  NOPE_CHECK(in && out, std::string("null ") + what + " / out pointer");
  NOPE_CHECK(B >= 1, "B must be >= 1");
  if (image_engine_ready(e)) return -1;
  return per_chunk(e, step, in, in_per, B, out, e->out_floats(), stream);
}

// *_encode_inplane: images [B, 3, 256, 256] x angles cossin [A, 2] -> out [B, A, ...]: the (image, angle) pairs in
// b-major order, rotated a chunk at a time, so the [B, A, 3, 256, 256] rotated batch never exists.  The chunks are
// those *_encode makes of that batch.
extern "C++" template <class Engine>
int engine_encode_inplane(Engine* e, const float* images, int B, const float* cossin, int A, float* out,
                          void* stream) {
  NOPE_CHECK(images && cossin && out, "null images / cossin / out pointer");
  NOPE_CHECK(B >= 1, "B must be >= 1");
  NOPE_CHECK(A >= 1 && A <= 360, "A (in-plane angles) must be in [1, 360]");
  NOPE_CHECK((int64_t)B * A <= INT32_MAX, "too many (image, angle) pairs");
  if (image_engine_ready(e)) return -1;
  const cudaStream_t st = static_cast<cudaStream_t>(stream);
  return per_rotated_chunk(e, B * A, out, e->out_floats(), st, [&](int lo, int n) {
    inplane_rotate_kernel<<<dim3(256 * 256 / 256, n), 256, 0, st>>>(images, cossin, A, 256, 256, lo, e->rot_stage);
  });
}

// *_encode_rotated: images [B, 3, 256, 256] x pairs (image_idx [P], cossin [P, 2]) -> out [P, ...]: the pairs in
// order, rotated a chunk at a time, so the result equals *_encode of the materialised [P, 3, 256, 256] batch.
extern "C++" template <class Engine>
int engine_encode_rotated(Engine* e, const float* images, int B, const int32_t* image_idx, const float* cossin, int P,
                          float* out, void* stream) {
  NOPE_CHECK(images && image_idx && cossin && out, "null images / image_idx / cossin / out pointer");
  NOPE_CHECK(B >= 1, "B must be >= 1");
  NOPE_CHECK(P >= 1 && P <= INT32_MAX / 2, "P (pairs) must be in [1, 2^30)");
  if (image_engine_ready(e)) return -1;
  const cudaStream_t st = static_cast<cudaStream_t>(stream);
  return per_rotated_chunk(e, P, out, e->out_floats(), st, [&](int lo, int n) {
    inplane_rotate_pairs_kernel<<<dim3(256 * 256 / 256, n), 256, 0, st>>>(images, B, image_idx, cossin, 256, 256, lo,
                                                                           e->rot_stage);
  });
}

// *_run_block of the VAE encoder and decoder
extern "C++" template <class Engine>
int vae_run_block(Engine* e, const char* name, const float* x, int C, int H, int n, float* out, float* out_pair,
                  int64_t out_capacity_floats, void* stream) {
  NOPE_CHECK(name && x && out, "null name / x / out pointer");
  if (image_engine_ready(e)) return -1;
  return e->run_block(name, x, C, H, n, out, out_pair, out_capacity_floats, static_cast<cudaStream_t>(stream));
}

int nope_encoder_encode(nope_encoder_t* e, const float* images, int B, float* out, void* stream) {
  return engine_encode(e, &nope_encoder::encode, "images", images, 3 * 256 * 256, B, out, stream);
}

int nope_encoder_encode_inplane(nope_encoder_t* e, const float* images, int B, const float* cossin, int A, float* out,
                                void* stream) {
  return engine_encode_inplane(e, images, B, cossin, A, out, stream);
}

int nope_inplane_rotate(const float* images, int B, int H, int W, const float* cossin, int A, float* out,
                        void* stream) {
  NOPE_CHECK(images && cossin && out, "null images / cossin / out pointer");
  NOPE_CHECK(B >= 1, "B must be >= 1");
  NOPE_CHECK(H >= 1 && W >= 1, "H and W must be >= 1");
  NOPE_CHECK(A >= 1 && A <= 360, "A (in-plane angles) must be in [1, 360]");
  NOPE_CHECK((int64_t)H * W <= INT32_MAX - 255 && (int64_t)B * A <= INT32_MAX, "images too large or too many");
  const int pairs = B * A, hw = H * W;
  constexpr int kMaxGridY = 65535;
  for (int lo = 0; lo < pairs; lo += kMaxGridY) {
    const int n = pairs - lo < kMaxGridY ? pairs - lo : kMaxGridY;
    inplane_rotate_kernel<<<dim3((hw + 255) / 256, n), 256, 0, static_cast<cudaStream_t>(stream)>>>(
        images, cossin, A, H, W, lo, out + (size_t)lo * 3 * hw);
    NOPE_CUDA(cudaGetLastError());
  }
  return 0;
}

int nope_inplane_rotate_pairs(const float* images, int B, int H, int W, const int32_t* image_idx, const float* cossin,
                              int P, float* out, void* stream) {
  NOPE_CHECK(images && image_idx && cossin && out, "null images / image_idx / cossin / out pointer");
  NOPE_CHECK(B >= 1, "B must be >= 1");
  NOPE_CHECK(H >= 1 && W >= 1, "H and W must be >= 1");
  NOPE_CHECK(P >= 1 && P <= INT32_MAX / 2, "P (pairs) must be in [1, 2^30)");
  NOPE_CHECK((int64_t)H * W <= INT32_MAX - 255, "images too large");
  const int hw = H * W;
  constexpr int kMaxGridY = 65535;
  for (int lo = 0; lo < P; lo += kMaxGridY) {
    const int n = P - lo < kMaxGridY ? P - lo : kMaxGridY;
    inplane_rotate_pairs_kernel<<<dim3((hw + 255) / 256, n), 256, 0, static_cast<cudaStream_t>(stream)>>>(
        images, B, image_idx, cossin, H, W, lo, out + (size_t)lo * 3 * hw);
    NOPE_CUDA(cudaGetLastError());
  }
  return 0;
}

int nope_encoder_encode_rotated(nope_encoder_t* e, const float* images, int B, const int32_t* image_idx,
                                const float* cossin, int P, float* out, void* stream) {
  return engine_encode_rotated(e, images, B, image_idx, cossin, P, out, stream);
}

int64_t nope_encoder_last_launch_count(const nope_encoder_t* e) { return e ? e->launches : 0; }

int nope_encoder_run_block(nope_encoder_t* e, const char* name, const float* x, int C, int H, int n, float* out,
                           int64_t out_capacity_floats, void* stream) {
  NOPE_CHECK(name && x && out, "null name / x / out pointer");
  if (image_engine_ready(e)) return -1;
  return e->run_block(name, x, C, H, n, out, out_capacity_floats, static_cast<cudaStream_t>(stream));
}

// ---------------------------------------------------------------------------------
// Stable Diffusion VAE encoder (vae.cuh, DESIGN.md section 16)
// ---------------------------------------------------------------------------------
int nope_vae_create(nope_vae_t** out, int device) {
  NOPE_CHECK(out != nullptr, "null out pointer");
  auto v = std::make_unique<nope_vae>();
  if (open_device(device, &v->num_sms)) return -1;
  v->device = device;
  v->build_plan();
  v->build_schema();
  *out = v.release();
  return 0;
}

void nope_vae_destroy(nope_vae_t* v) { delete v; }

int nope_vae_load_tensor(nope_vae_t* v, const char* key, const float* data, const int64_t* shape, int ndim) {
  return engine_load_tensor(v, key, data, shape, ndim);
}

int nope_vae_finalize(nope_vae_t* v) { return engine_finalize(v); }
int nope_vae_set_option(nope_vae_t* v, const char* name, int value) { return encoder_set_option(v, name, value); }

int nope_vae_encode(nope_vae_t* v, const float* images, int B, float* out, void* stream) {
  return engine_encode(v, &nope_vae::encode, "images", images, 3 * 256 * 256, B, out, stream);
}

int nope_vae_encode_inplane(nope_vae_t* v, const float* images, int B, const float* cossin, int A, float* out,
                            void* stream) {
  return engine_encode_inplane(v, images, B, cossin, A, out, stream);
}

int nope_vae_encode_rotated(nope_vae_t* v, const float* images, int B, const int32_t* image_idx, const float* cossin,
                            int P, float* out, void* stream) {
  return engine_encode_rotated(v, images, B, image_idx, cossin, P, out, stream);
}

int64_t nope_vae_last_launch_count(const nope_vae_t* v) { return v ? v->launches : 0; }

int nope_vae_run_block(nope_vae_t* v, const char* name, const float* x, int C, int H, int n, float* out,
                       float* out_pair, int64_t out_capacity_floats, void* stream) {
  return vae_run_block(v, name, x, C, H, n, out, out_pair, out_capacity_floats, stream);
}

// ---------------------------------------------------------------------------------
// Stable Diffusion VAE decoder (vae.cuh, DESIGN.md section 17)
// ---------------------------------------------------------------------------------
int nope_vae_decoder_create(nope_vae_decoder_t** out, int device) {
  NOPE_CHECK(out != nullptr, "null out pointer");
  auto d = std::make_unique<nope_vae_decoder>();
  if (open_device(device, &d->num_sms)) return -1;
  d->device = device;
  d->build_plan();
  d->build_schema();
  *out = d.release();
  return 0;
}

void nope_vae_decoder_destroy(nope_vae_decoder_t* d) { delete d; }

int nope_vae_decoder_load_tensor(nope_vae_decoder_t* d, const char* key, const float* data, const int64_t* shape,
                                 int ndim) {
  return engine_load_tensor(d, key, data, shape, ndim);
}

int nope_vae_decoder_finalize(nope_vae_decoder_t* d) { return engine_finalize(d); }

int nope_vae_decoder_decode(nope_vae_decoder_t* d, const float* latents, int B, float* out, void* stream) {
  return engine_encode(d, &nope_vae_decoder::decode, "latents", latents, 4 * 32 * 32, B, out, stream);
}

int64_t nope_vae_decoder_last_launch_count(const nope_vae_decoder_t* d) { return d ? d->launches : 0; }

int nope_vae_decoder_run_block(nope_vae_decoder_t* d, const char* name, const float* x, int C, int H, int n,
                               float* out, float* out_pair, int64_t out_capacity_floats, void* stream) {
  return vae_run_block(d, name, x, C, H, n, out, out_pair, out_capacity_floats, stream);
}

// ---------------------------------------------------------------------------------
// T-LESS evaluation: depth rasterizer and VSD (render.cuh, DESIGN.md section 12)
// ---------------------------------------------------------------------------------
// The depth bits z [F, P, H, W] of a mesh under F frames x P poses [F, P, 4, 4]: filled with +inf, then one raster
// launch per frame with that frame's HOST intrinsics K [F, 4].  launch_depth_finish turns +inf into 0 afterwards.
static int render_frames(const float* vertices, int V, const int32_t* faces, int NF, const float* poses,
                         const double* K, int F, int P, float znear, int H, int W, unsigned* z, cudaStream_t st) {
  const long long hw = (long long)H * W, n = (long long)F * P * hw;
  depth_fill_kernel<<<ew_grid(n), 256, 0, st>>>(z, n);
  NOPE_CUDA(cudaGetLastError());
  for (int f = 0; f < F; ++f) {
    const double* kf = K + 4 * (size_t)f;
    depth_raster_kernel<<<dim3((NF + 7) / 8, P), 256, 0, st>>>(
        vertices, V, faces, NF, poses + 16 * (size_t)f * P, (float)kf[0], (float)kf[1], (float)kf[2], (float)kf[3],
        znear, H, W, z + (size_t)f * P * hw);
    NOPE_CUDA(cudaGetLastError());
  }
  return 0;
}

static int launch_depth_finish(unsigned* z, long long n, cudaStream_t st) {
  depth_finish_kernel<<<ew_grid(n), 256, 0, st>>>(z, n);
  NOPE_CUDA(cudaGetLastError());
  return 0;
}

int nope_render_depth(const float* vertices, int V, const int32_t* faces, int F, const float* poses, int P, float fx,
                      float fy, float cx, float cy, float znear, int H, int W, float* out, void* stream) {
  NOPE_CHECK(vertices && faces && poses && out, "null argument");
  NOPE_CHECK(V >= 1 && F >= 1 && P >= 1, "V, F and P must be >= 1");
  NOPE_CHECK(P <= 65535, "P must be <= 65535");
  NOPE_CHECK(H >= 1 && H <= kRenderMaxSide && W >= 1 && W <= kRenderMaxSide, "H and W must be in [1, 8192]");
  NOPE_CHECK(znear > 0.f, "znear must be > 0");
  NOPE_CHECK(std::isfinite(fx) && std::isfinite(fy) && std::isfinite(cx) && std::isfinite(cy) && std::isfinite(znear),
             "intrinsics and znear must be finite");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  unsigned* z = reinterpret_cast<unsigned*>(out);
  const double K[4] = {fx, fy, cx, cy};             // one frame; float -> double -> float is exact
  if (render_frames(vertices, V, faces, F, poses, K, 1, P, znear, H, W, z, st)) return -1;
  return launch_depth_finish(z, (long long)P * H * W, st);
}

int nope_vsd_error(const double* depth_test, const float* depth_gt, const float* depth_est, int F, int P, int H, int W,
                   const double* K, double delta, double tau, int cost_type, double* out, void* stream) {
  NOPE_CHECK(depth_test && depth_gt && depth_est && K && out, "null argument");
  NOPE_CHECK(F >= 1 && P >= 1, "F and P must be >= 1");
  NOPE_CHECK(F <= 65535 && P <= 65535, "F and P must be <= 65535");
  NOPE_CHECK(H >= 1 && H <= kRenderMaxSide && W >= 1 && W <= kRenderMaxSide, "H and W must be in [1, 8192]");
  NOPE_CHECK(cost_type == NOPE_VSD_STEP || cost_type == NOPE_VSD_TLINEAR, "unknown cost_type (0 step, 1 tlinear)");
  NOPE_CHECK(delta >= 0.0 && std::isfinite(delta), "delta must be finite and >= 0");
  NOPE_CHECK(tau > 0.0 && std::isfinite(tau), "tau must be finite and > 0");
  VsdTaus taus{};
  taus.v[0] = tau;
  // the visibility test compares float32 differences with delta in float32, as numpy does with a Python number
  vsd_kernel<1><<<dim3(kVsdCluster * P, F), kVsdThreads, 0, static_cast<cudaStream_t>(stream)>>>(
      depth_test, depth_gt, depth_est, P, H, W, K, (float)delta, taus, 1, cost_type, out);
  NOPE_CUDA(cudaGetLastError());
  return 0;
}

int nope_distinct_topk(const float* sim, int R, int N, const double* rot, int G_r, int Q, const double* sym_disc,
                       const int32_t* n_disc, const double* axis, int G, const int32_t* group, int k, double c_thr,
                       int64_t* idx_out, float* score_out, void* stream) {
  NOPE_CHECK(sim && rot && sym_disc && n_disc && axis && group && idx_out && score_out, "null argument");
  NOPE_CHECK(R >= 1 && N >= 1 && N <= (1 << 30), "R (rows) must be >= 1 and N (entries per row) in [1, 2^30]");
  NOPE_CHECK(G_r >= 1 && Q >= 1 && (G_r == 1 || (int64_t)G_r * Q == R),
             "G_r (rotation sets) must be 1 or R / Q, with Q >= 1");
  NOPE_CHECK(k >= 1 && k <= kMaxTopK, "k must be in [1, 64]");
  NOPE_CHECK(c_thr >= -1.0 && c_thr <= 3.0, "c_thr = 1 + 2 cos(theta) must be in [-1, 3]");
  NOPE_CHECK(G >= 1 && G <= 65536, "G (symmetry groups) must be in [1, 65536]");
  // HOST symmetry groups, checked and packed for one stream-ordered upload together with the row -> group table
  std::vector<DistinctGroup> packed((size_t)G);
  std::memset(packed.data(), 0, sizeof(DistinctGroup) * (size_t)G);
  int64_t off = 0;
  for (int g = 0; g < G; ++g) {
    const int n = n_disc[g];
    NOPE_CHECK(n >= 1 && n <= kDistinctMaxSym, "every group needs 1 to 32 discrete rotations");
    const double* d = sym_disc + 9 * off;
    for (int e = 0; e < 9 * n; ++e) NOPE_CHECK(std::isfinite(d[e]), "discrete symmetries must be finite");
    for (int e = 0; e < 9; ++e)
      NOPE_CHECK(d[e] == (e % 4 == 0 ? 1.0 : 0.0), "the first discrete rotation of every group must be the identity");
    std::memcpy(packed[g].d, d, sizeof(double) * 9 * n);
    packed[g].n = n;
    off += n;
    const double* a = axis + 3 * (size_t)g;
    NOPE_CHECK(std::isfinite(a[0]) && std::isfinite(a[1]) && std::isfinite(a[2]), "axes must be finite");
    const double a2 = a[0] * a[0] + a[1] * a[1] + a[2] * a[2];
    NOPE_CHECK(a2 == 0.0 || std::fabs(a2 - 1.0) <= 1e-12, "an axis must be a unit vector, or zero for none");
    std::memcpy(packed[g].axis, a, sizeof(double) * 3);
    packed[g].has_axis = a2 != 0.0;
  }
  for (int r = 0; r < R; ++r) NOPE_CHECK(group[r] >= 0 && group[r] < G, "group indices must be in [0, G)");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const int64_t nwords = ((int64_t)N + 31) / 32;
  ScratchArena arena(st);                               // groups, row -> group, and (large N) the removal masks
  const DistinctGroup* groups_d;
  const int* group_d;
  unsigned* masks = nullptr;
  arena.add(&groups_d, (size_t)G, packed.data());
  arena.add(&group_d, (size_t)R, group);
  if (nwords > kDistinctSmemWords) arena.add(&masks, (size_t)nwords * R);
  if (arena.alloc()) return -1;
  distinct_topk_kernel<<<R, kDistinctThreads, 0, st>>>(sim, N, rot, G_r, Q, groups_d, group_d, k, c_thr, masks,
                                                      reinterpret_cast<long long*>(idx_out), score_out);
  NOPE_CUDA(cudaGetLastError());
  return 0;
}

int nope_vsd_error_taus(const double* depth_test, const float* depth_gt, const float* depth_est, int F, int P, int H,
                        int W, const double* K, double delta, int cost_type, const double* taus, int T, double* out,
                        void* stream) {
  NOPE_CHECK(depth_test && depth_gt && depth_est && K && taus && out, "null argument");
  NOPE_CHECK(F >= 1 && P >= 1, "F and P must be >= 1");
  NOPE_CHECK(F <= 65535 && P <= 65535, "F and P must be <= 65535");
  NOPE_CHECK(H >= 1 && H <= kRenderMaxSide && W >= 1 && W <= kRenderMaxSide, "H and W must be in [1, 8192]");
  NOPE_CHECK(T >= 1 && T <= kVsdMaxTaus, "T (tolerances) must be in [1, 16]");
  NOPE_CHECK(cost_type == NOPE_VSD_STEP || cost_type == NOPE_VSD_TLINEAR, "unknown cost_type (0 step, 1 tlinear)");
  NOPE_CHECK(delta >= 0.0 && std::isfinite(delta), "delta must be finite and >= 0");
  VsdTaus tv{};
  for (int j = 0; j < T; ++j) {
    NOPE_CHECK(taus[j] > 0.0 && std::isfinite(taus[j]), "every tau must be finite and > 0");
    tv.v[j] = taus[j];
  }
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  ScratchArena arena(st);
  const double* kd;
  if (stage_host_intrinsics(arena, &kd, K, F) || arena.alloc()) return -1;
  const dim3 grid(kVsdCluster * P, F);
  if (T == 1)
    vsd_kernel<1><<<grid, kVsdThreads, 0, st>>>(depth_test, depth_gt, depth_est, P, H, W, kd, (float)delta, tv, T,
                                                 cost_type, out);
  else
    vsd_kernel<kVsdMaxTaus><<<grid, kVsdThreads, 0, st>>>(depth_test, depth_gt, depth_est, P, H, W, kd, (float)delta,
                                                           tv, T, cost_type, out);
  NOPE_CUDA(cudaGetLastError());
  return 0;
}

// ---------------------------------------------------------------------------------
// BOP pose errors: symmetry-aware MSSD / MSPD (pose_error.cuh, DESIGN.md section 15)
// ---------------------------------------------------------------------------------
int nope_pose_errors(const float* points, int V, const double* sym, int S, const double* gt, const double* est,
                     const double* K, int F, int P, double* out_mssd, double* out_mspd, void* stream) {
  NOPE_CHECK(points && sym && gt && est && K && out_mssd && out_mspd, "null argument");
  NOPE_CHECK(V >= 1 && S >= 1 && F >= 1 && P >= 1, "V, S, F and P must be >= 1");
  NOPE_CHECK(F <= 65535 && P <= 65535, "F and P must be <= 65535");
  NOPE_CHECK(S <= (1 << 24), "S must be <= 2^24");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  ScratchArena arena(st);
  const double* kd;
  if (stage_host_intrinsics(arena, &kd, K, F) || arena.alloc()) return -1;
  const int n = F * P;
  auto* om = reinterpret_cast<unsigned long long*>(out_mssd);
  auto* op = reinterpret_cast<unsigned long long*>(out_mspd);
  pose_error_fill_kernel<<<std::min((n + 255) / 256, 1024), 256, 0, st>>>(om, op, n);
  NOPE_CUDA(cudaGetLastError());
  pose_error_kernel<<<dim3((S + kPoseErrSyms - 1) / kPoseErrSyms, P, F), kPoseErrThreads, 0, st>>>(
      points, V, sym, S, gt, est, kd, P, om, op);
  NOPE_CUDA(cudaGetLastError());
  return 0;
}

// ---------------------------------------------------------------------------------
// pose fits from the frame: translation (translation.cuh, DESIGN.md section 18), depth ICP (depth_refine.cuh,
// section 19) and contour alignment (contour_refine.cuh, section 20)
// ---------------------------------------------------------------------------------
// The arguments the three fits share.  iters_max bounds iters (INT_MAX: no bound).  Null pointers, rho and tau differ
// between the fits and each launcher checks its own; the host K is checked where it is staged.
static int check_fit_args(int V, int NF, int F, int P, int H, int W, float znear, int iters, int iters_max) {
  NOPE_CHECK(V >= 1 && NF >= 1, "V and NF must be >= 1");
  NOPE_CHECK(F >= 1 && F <= 65535 && P >= 1 && P <= 65535, "F and P must be in [1, 65535]");
  NOPE_CHECK(H >= 1 && H <= kRenderMaxSide && W >= 1 && W <= kRenderMaxSide, "H and W must be in [1, 8192]");
  NOPE_CHECK(iters >= 0 && iters <= iters_max, "iters must be in [0, iters_max]");
  NOPE_CHECK(znear > 0.f && std::isfinite(znear), "znear must be finite and > 0");
  return 0;
}

// the refinements' rho > 0 and tau [iters + 1] > 0, all finite
static int check_rho_tau(double rho, const double* tau, int iters) {
  NOPE_CHECK(std::isfinite(rho) && rho > 0.0, "rho must be finite and > 0");
  for (int i = 0; i <= iters; ++i) NOPE_CHECK(std::isfinite(tau[i]) && tau[i] > 0.0, "tau must be finite and > 0");
  return 0;
}

// occluders [F, H, W] (nullable): the pixels where the object may be hidden count for neither the silhouette nor the
// mask (DESIGN.md section 24); null: every pixel counts
int nope_fit_translation_occluded(const float* vertices, int V, const int32_t* faces, int NF, const double* R,
                                  const double* t_init, const uint8_t* masks, const uint8_t* occluders,
                                  const double* K, int F, int P, int H, int W, float znear, int iters, float* depth,
                                  double* t_out, double* iou, int32_t* stats_out, void* stream) {
  NOPE_CHECK(vertices && faces && R && t_init && masks && K && depth && t_out && iou, "null argument");
  if (check_fit_args(V, NF, F, P, H, W, znear, iters, INT_MAX)) return -1;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  // stream-ordered scratch: K, the current translations, the float32 poses and the integer statistics
  const size_t n = (size_t)F * P;
  ScratchArena arena(st);
  const double* kd;
  double* t;
  float* poses;
  int *sil_stats, *mask_stats;
  if (stage_host_intrinsics(arena, &kd, K, F)) return -1;
  arena.add(&t, 3 * n);
  arena.add(&poses, 16 * n);
  arena.add(&sil_stats, kFitStats * n);
  arena.add(&mask_stats, kFitStats * (size_t)F);
  if (arena.alloc()) return -1;
  const int ew_blocks = ew_grid((long long)n);
  fit_init_kernel<<<ew_blocks, 256, 0, st>>>(R, t_init, F, P, t, poses, sil_stats, mask_stats);
  NOPE_CUDA(cudaGetLastError());
  const long long hw = (long long)H * W;
  const int stat_blocks = (int)((hw + kFitPixelsPerCta - 1) / kFitPixelsPerCta);
  fit_stats_kernel<false><<<dim3(stat_blocks, 1, F), kFitThreads, 0, st>>>(nullptr, masks, occluders, P, H, W,
                                                                          mask_stats);
  NOPE_CUDA(cudaGetLastError());
  unsigned* z = reinterpret_cast<unsigned*>(depth);
  for (int it = 0; it <= iters; ++it) {
    if (render_frames(vertices, V, faces, NF, poses, K, F, P, znear, H, W, z, st)) return -1;
    fit_stats_kernel<true><<<dim3(stat_blocks, P, F), kFitThreads, 0, st>>>(z, masks, occluders, P, H, W,
                                                                           sil_stats);
    NOPE_CUDA(cudaGetLastError());
    if (it < iters) {
      fit_update_kernel<<<ew_blocks, 256, 0, st>>>(R, kd, mask_stats, F, P, t, poses, sil_stats);
      NOPE_CUDA(cudaGetLastError());
    }
  }
  fit_final_kernel<<<ew_blocks, 256, 0, st>>>(t, mask_stats, sil_stats, F, P, t_out, iou, stats_out);
  NOPE_CUDA(cudaGetLastError());
  return launch_depth_finish(z, (long long)n * hw, st);      // depth holds render_depth at the returned t
}

int nope_refine_depth(const float* vertices, int V, const int32_t* faces, int NF, const double* R, const double* t_init,
                      const double* depth_sensor, const uint8_t* masks, const double* K, int F, int P, int H, int W,
                      double rho, const double* tau, int iters, float znear, float* depth, double* R_out,
                      double* t_out, double* fit_out, int64_t* sums_out, void* stream) {
  NOPE_CHECK(vertices && faces && R && t_init && depth_sensor && K && tau && depth && R_out && t_out && fit_out,
             "null argument");
  if (check_fit_args(V, NF, F, P, H, W, znear, iters, 1024) || check_rho_tau(rho, tau, iters)) return -1;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  // stream-ordered scratch: K, the current R and t, the integer sums, the float32 poses and n_valid
  const size_t n = (size_t)F * P;
  ScratchArena arena(st);
  const double* kd;
  double *Rc, *tc;
  unsigned long long* sums;
  float* poses;
  int* n_valid;
  if (stage_host_intrinsics(arena, &kd, K, F)) return -1;
  arena.add(&Rc, 9 * n);
  arena.add(&tc, 3 * n);
  arena.add(&sums, kIcpSums * n);
  arena.add(&poses, 16 * n);
  arena.add(&n_valid, (size_t)F);
  if (arena.alloc()) return -1;
  const int ew_blocks = ew_grid((long long)n);
  icp_init_kernel<<<ew_blocks, 256, 0, st>>>(R, t_init, F, P, Rc, tc, poses, sums, n_valid);
  NOPE_CUDA(cudaGetLastError());
  const long long hw = (long long)H * W;
  const int px_blocks = (int)((hw + kIcpPixelsPerCta - 1) / kIcpPixelsPerCta);
  icp_valid_kernel<<<dim3(px_blocks, 1, F), kIcpThreads, 0, st>>>(depth_sensor, masks, H, W, n_valid);
  NOPE_CUDA(cudaGetLastError());
  unsigned* z = reinterpret_cast<unsigned*>(depth);
  for (int it = 0; it <= iters; ++it) {
    if (render_frames(vertices, V, faces, NF, poses, K, F, P, znear, H, W, z, st)) return -1;
    icp_accumulate_kernel<<<dim3(px_blocks, P, F), kIcpThreads, 0, st>>>(z, depth_sensor, masks, kd, tc, P, H, W,
                                                                         tau[it], rho, sums);
    NOPE_CUDA(cudaGetLastError());
    if (it < iters) {
      icp_solve_kernel<<<ew_blocks, 256, 0, st>>>(F, P, tau[it], rho, Rc, tc, poses, sums);
      NOPE_CUDA(cudaGetLastError());
    }
  }
  icp_final_kernel<<<ew_blocks, 256, 0, st>>>(Rc, tc, sums, n_valid, F, P, tau[iters], R_out, t_out, fit_out,
                                              reinterpret_cast<long long*>(sums_out));
  NOPE_CUDA(cudaGetLastError());
  return launch_depth_finish(z, (long long)n * hw, st);      // depth holds render_depth at the returned pose
}

// phi [F, H, W] of masks [F, H, W] minus the nullable occluders [F, H, W] through the column pass into g [F, H, W] and
// the row pass
static int launch_mask_sdf(const uint8_t* masks, const uint8_t* occ, int F, int H, int W, unsigned* g, double* phi,
                           cudaStream_t st) {
  mask_sdf_cols_kernel<<<dim3((W + kSdfColThreads - 1) / kSdfColThreads, F), kSdfColThreads, 0, st>>>(masks, occ, H,
                                                                                                     W, g);
  NOPE_CUDA(cudaGetLastError());
  const int rows = mask_sdf_rows_per_cta(W);
  mask_sdf_rows_kernel<<<dim3((H + rows - 1) / rows, F), rows, sizeof(unsigned) * rows * W, st>>>(g, H, W, phi);
  NOPE_CUDA(cudaGetLastError());
  return 0;
}

int nope_mask_sdf(const uint8_t* masks, int F, int H, int W, double* sdf_out, void* stream) {
  NOPE_CHECK(masks && sdf_out, "null argument");
  NOPE_CHECK(F >= 1 && F <= 65535, "F must be in [1, 65535]");
  NOPE_CHECK(H >= 1 && H <= kRenderMaxSide && W >= 1 && W <= kRenderMaxSide, "H and W must be in [1, 8192]");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  ScratchArena arena(st);                                       // the column pass's distances
  unsigned* g;
  arena.add(&g, (size_t)F * H * W);
  if (arena.alloc()) return -1;
  return launch_mask_sdf(masks, nullptr, F, H, W, g, sdf_out, st);
}

// occluders [F, H, W] (nullable): phi and the mask statistics are those of the mask minus the occluders, and a contour
// pixel next to an occluder is not paired (DESIGN.md section 24); null: every pixel counts
int nope_refine_contour_occluded(const float* vertices, int V, const int32_t* faces, int NF, const double* R,
                                 const double* t_init, const uint8_t* masks, const uint8_t* occluders,
                                 const double* K, int F, int P, int H, int W, double rho, const double* tau, int iters,
                                 float znear, float* depth, double* R_out, double* t_out, double* fit_out,
                                 int64_t* sums_out, void* stream) {
  NOPE_CHECK(vertices && faces && R && t_init && masks && K && tau && depth && R_out && t_out && fit_out,
             "null argument");
  if (check_fit_args(V, NF, F, P, H, W, znear, iters, 1024) || check_rho_tau(rho, tau, iters)) return -1;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  // stream-ordered scratch: K, the current R and t, the integer sums, phi, the float32 poses, the column pass's
  // distances, the silhouette and mask statistics and n_contour
  const size_t n = (size_t)F * P, fhw = (size_t)F * H * W;
  ScratchArena arena(st);
  const double* kd;
  double *Rc, *tc, *phi;
  unsigned long long* sums;
  float* poses;
  unsigned* g;
  int *sil_stats, *mask_stats, *n_contour;
  if (stage_host_intrinsics(arena, &kd, K, F)) return -1;
  arena.add(&Rc, 9 * n);
  arena.add(&tc, 3 * n);
  arena.add(&sums, kIcpSums * n);
  arena.add(&phi, fhw);
  arena.add(&poses, 16 * n);
  arena.add(&g, fhw);
  arena.add(&sil_stats, kFitStats * n);
  arena.add(&mask_stats, kFitStats * (size_t)F);
  arena.add(&n_contour, n);
  if (arena.alloc()) return -1;
  const int ew_blocks = ew_grid((long long)n);
  contour_init_kernel<<<ew_blocks, 256, 0, st>>>(R, t_init, F, P, Rc, tc, poses, sums, n_contour, sil_stats,
                                                 mask_stats);
  NOPE_CUDA(cudaGetLastError());
  const long long hw = (long long)H * W;
  const int px_blocks = (int)((hw + kIcpPixelsPerCta - 1) / kIcpPixelsPerCta);
  const int stat_blocks = (int)((hw + kFitPixelsPerCta - 1) / kFitPixelsPerCta);
  fit_stats_kernel<false><<<dim3(stat_blocks, 1, F), kFitThreads, 0, st>>>(nullptr, masks, occluders, P, H, W,
                                                                          mask_stats);
  NOPE_CUDA(cudaGetLastError());
  if (launch_mask_sdf(masks, occluders, F, H, W, g, phi, st)) return -1;
  unsigned* z = reinterpret_cast<unsigned*>(depth);
  for (int it = 0; it <= iters; ++it) {
    if (render_frames(vertices, V, faces, NF, poses, K, F, P, znear, H, W, z, st)) return -1;
    contour_accumulate_kernel<<<dim3(px_blocks, P, F), kIcpThreads, 0, st>>>(z, phi, occluders, kd, tc, mask_stats, P,
                                                                             H, W, tau[it], rho, sums, n_contour);
    NOPE_CUDA(cudaGetLastError());
    if (it < iters) {
      contour_solve_kernel<<<ew_blocks, 256, 0, st>>>(F, P, hw, tau[it], rho, mask_stats, kd, Rc, tc, poses, sums,
                                                      n_contour);
      NOPE_CUDA(cudaGetLastError());
    }
  }
  fit_stats_kernel<true><<<dim3(stat_blocks, P, F), kFitThreads, 0, st>>>(z, masks, occluders, P, H, W, sil_stats);
  NOPE_CUDA(cudaGetLastError());
  contour_final_kernel<<<ew_blocks, 256, 0, st>>>(Rc, tc, sums, n_contour, mask_stats, sil_stats, F, P, hw,
                                                  tau[iters], R_out, t_out, fit_out,
                                                  reinterpret_cast<long long*>(sums_out));
  NOPE_CUDA(cudaGetLastError());
  return launch_depth_finish(z, (long long)n * hw, st);      // depth holds render_depth at the returned pose
}

// ---------------------------------------------------------------------------------
// full-frame crops: the virtual-bounding-box perspective warp (crop.cuh, DESIGN.md section 13)
// ---------------------------------------------------------------------------------
int nope_crop_frames(const uint8_t* frames, int F, int H, int W, int C, const uint8_t* masks, const int32_t* frame_idx,
                     const double* inv_maps, int B, int S, float* out, void* stream) {
  NOPE_CHECK(frames && inv_maps && out, "null argument");
  NOPE_CHECK(F >= 1 && B >= 1, "F and B must be >= 1");
  NOPE_CHECK(B <= 65535, "B must be <= 65535");
  NOPE_CHECK(H >= 1 && H <= kCropMaxSide && W >= 1 && W <= kCropMaxSide, "H and W must be in [1, 16384]");
  NOPE_CHECK(S >= 1 && S <= kCropMaxS, "S must be in [1, 4096]");
  NOPE_CHECK(C == 3 || C == 4, "C must be 3 (RGB) or 4 (RGBA)");
  NOPE_CHECK(!(masks && C == 4), "a mask with C = 4: the alpha channel is the mask");
  NOPE_CHECK(frame_idx || F == B, "without frame_idx F must equal B");
  const dim3 grid((S * S + kCropThreads - 1) / kCropThreads, B);
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  if (C == 3)
    crop_warp_kernel<3><<<grid, kCropThreads, 0, st>>>(frames, F, H, W, masks, frame_idx, inv_maps, S, out);
  else
    crop_warp_kernel<4><<<grid, kCropThreads, 0, st>>>(frames, F, H, W, masks, frame_idx, inv_maps, S, out);
  NOPE_CUDA(cudaGetLastError());
  return 0;
}

// the crop camera (crop.cuh, DESIGN.md section 23)
int nope_crop_camera(const double* pose, int F, int keep_inplane, double* Rv, void* stream) {
  NOPE_CHECK(pose && Rv, "null argument");
  NOPE_CHECK(F >= 1 && F <= kCropCamMax, "F must be in [1, 65535]");
  NOPE_CHECK(keep_inplane == 0 || keep_inplane == 1, "keep_inplane must be 0 or 1");
  for (int f = 0; f < F; ++f) {
    const double* p = pose + 16 * (size_t)f;
    // keep_inplane reads the translation only, the other mode the top three rows
    for (int i = 0; i < 12; ++i)
      NOPE_CHECK(std::isfinite(p[i]) || (keep_inplane && i % 4 != 3), "poses must be finite");
    NOPE_CHECK(!keep_inplane || p[11] > 0.0, "keep_inplane needs the object centre in front of the camera (Z > 0)");
  }
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  ScratchArena arena(st);
  const double* pd;
  arena.add(&pd, 16 * (size_t)F, pose);
  if (arena.alloc()) return -1;
  crop_camera_kernel<<<ew_grid(F), 256, 0, st>>>(pd, F, keep_inplane, Rv);
  NOPE_CUDA(cudaGetLastError());
  return 0;
}

int nope_crop_rotate(const double* Rv, int F, const double* R, int P, int to_camera, double* out, void* stream) {
  NOPE_CHECK(Rv && R && out, "null argument");
  NOPE_CHECK(F >= 1 && F <= kCropCamMax && P >= 1 && P <= kCropCamMax, "F and P must be in [1, 65535]");
  NOPE_CHECK(to_camera == 0 || to_camera == 1, "to_camera must be 0 or 1");
  const long long n = (long long)F * P;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  crop_rotate_kernel<<<ew_grid(n), 256, 0, st>>>(Rv, R, P, n, to_camera, out);
  NOPE_CUDA(cudaGetLastError());
  return 0;
}

// pose tracking: prior rotations to refinement centres (track.cuh, DESIGN.md section 26)
int nope_track_seeds(const double* Rc, int H, const double* T, int N, float* out_D, int32_t* out_seed,
                     float* out_cossin, void* stream) {
  NOPE_CHECK(Rc && T && out_D && out_seed && out_cossin, "null argument");
  NOPE_CHECK(H >= 1 && N >= 1, "H and N must be >= 1");
  track_seed_kernel<<<H, kTrackThreads, 0, static_cast<cudaStream_t>(stream)>>>(Rc, T, N, out_D, out_seed,
                                                                               out_cossin);
  NOPE_CUDA(cudaGetLastError());
  return 0;
}

// ---------------------------------------------------------------------------------
// per-op entry points
// ---------------------------------------------------------------------------------

namespace {
// What the per-op convolution entry points share: the argument checks, the inputs staged as NHWC fp16 (with their
// fp16 remainders at precision 2), the output buffer, the packed layer, and a UNet engine on the current device to
// launch through.
struct OpConv {
  DeviceAllocs s;
  nope_unet eng;
  ConvLayer L;
  Act in0, in1, out;

  int setup(int mode, int max_mode, int precision, const float* x0, int C0, const float* x1, int C1,
            const float* weight, const float* bias, int n_img, int H, int W, int Cout, cudaStream_t st) {
    NOPE_CHECK(x0 && weight, "null argument");
    NOPE_CHECK(mode >= 0 && mode <= max_mode, "mode must be 0.." + std::to_string(max_mode));
    NOPE_CHECK(H == W, "square images only");
    NOPE_CHECK(C0 % 64 == 0 && C1 % 64 == 0 && Cout % 64 == 0, "channels must be multiples of 64");
    const bool sp = precision == 2;
    // the layer shape of each mode (nope_unet::prof_mode is its inverse)
    const ConvLayer shapes[4] = {conv3x3(), conv1x1(), conv_unshuffle(), conv_upsample3x3()};
    L = shapes[mode];
    const int Hin = L.stride == 2 ? 2 * H : (L.up ? H / 2 : H);
    __half *a0 = nullptr, *a0l = nullptr, *a1 = nullptr, *a1l = nullptr, *o = nullptr, *ol = nullptr;
    if (to_nhwc(x0, &a0, s, n_img, C0, Hin * Hin, st, sp ? &a0l : nullptr)) return -1;
    if (x1 && to_nhwc(x1, &a1, s, n_img, C1, Hin * Hin, st, sp ? &a1l : nullptr)) return -1;
    in0 = Act(a0, C0, a0l);
    if (x1) in1 = Act(a1, C1, a1l);
    if (s.alloc(&o, (size_t)n_img * H * W * Cout) || (sp && s.alloc(&ol, (size_t)n_img * H * W * Cout))) return -1;
    out = Act(o, Cout, ol);
    L.cin = C0 + (x1 ? C1 : 0);
    L.cout = Cout;
    L.K = L.cin * L.k * L.k;
    L.wlo = precision >= 1;
    if (pack_conv_layer(s, L, {{weight, Cout, L.cin, L.k * L.k, 0, 0}}, {}, false, st)) return -1;
    L.bias = const_cast<float*>(bias);
    eng.precision = precision;
    NOPE_CUDA(cudaGetDevice(&eng.device));
    NOPE_CUDA(cudaDeviceGetAttribute(&eng.num_sms, cudaDevAttrMultiProcessorCount, eng.device));
    return 0;
  }
};
}  // namespace

int nope_op_conv(int mode, const float* x0, int C0, const float* x1, int C1, const float* weight, const float* bias,
                 float* out, int n_img, int H, int W, int Cout, void* stream) {
  NOPE_CHECK(out, "null argument");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  OpConv op;
  if (op.setup(mode, 3, 0, x0, C0, x1, C1, weight, bias, n_img, H, W, Cout, st)) return -1;
  if (op.eng.conv(op.L, op.in0, op.in1, op.out, H, n_img, n_img, st)) return -1;
  if (to_nchw(op.out.hi, out, n_img, Cout, H * W, st)) return -1;
  NOPE_CUDA(cudaStreamSynchronize(st));
  return 0;
}

int nope_op_conv_gn(int mode, const float* x0, int C0, const float* x1, int C1, const float* weight,
                    const float* bias, const float* gamma, const float* beta, int G, int silu, float* out, int n_img,
                    int H, int W, int Cout, void* stream) {
  NOPE_CHECK(gamma && beta && out, "null argument");
  NOPE_CHECK(G >= 1 && (Cout / 8) % G == 0, "groups must divide the 8-channel octets");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const int hw = H * W, parts = hw < 32 ? 1 : hw / 32, noct = Cout / 8;
  OpConv op;
  if (op.setup(mode, 2, 0, x0, C0, x1, C1, weight, bias, n_img, H, W, Cout, st)) return -1;
  float2* stats = nullptr;
  if (op.s.alloc(&stats, (size_t)n_img * parts * noct)) return -1;
  if (op.eng.conv(op.L, op.in0, op.in1, op.out, H, n_img, n_img, st, nullptr, stats)) return -1;
  // GroupNorm on the host, in double, from the epilogue's [img][parts][octet] partial sums alone: a group's sum and
  // sum of squares are the totals of its octets over all parts (the layout the LDM engine normalises from)
  std::vector<__half> ho((size_t)n_img * hw * Cout);
  std::vector<float2> hs((size_t)n_img * parts * noct);
  std::vector<float> hg(Cout), hb(Cout), y((size_t)n_img * Cout * hw);
  NOPE_CUDA(cudaStreamSynchronize(st));
  NOPE_CUDA(cudaMemcpy(ho.data(), op.out.hi, ho.size() * sizeof(__half), cudaMemcpyDeviceToHost));
  NOPE_CUDA(cudaMemcpy(hs.data(), stats, hs.size() * sizeof(float2), cudaMemcpyDeviceToHost));
  NOPE_CUDA(cudaMemcpy(hg.data(), gamma, Cout * sizeof(float), cudaMemcpyDeviceToHost));
  NOPE_CUDA(cudaMemcpy(hb.data(), beta, Cout * sizeof(float), cudaMemcpyDeviceToHost));
  const int opg = noct / G, cpg = Cout / G;
  const double cnt = (double)hw * cpg;
  for (int i = 0; i < n_img; ++i)
    for (int g = 0; g < G; ++g) {
      double sum = 0.0, sq = 0.0;
      for (int part = 0; part < parts; ++part)
        for (int oc = g * opg; oc < (g + 1) * opg; ++oc) {
          const float2 t = hs[((size_t)i * parts + part) * noct + oc];
          sum += t.x;
          sq += t.y;
        }
      const double mean = sum / cnt;
      const double rstd = 1.0 / std::sqrt(std::max(sq / cnt - mean * mean, 0.0) + 1e-5);
      for (int c = g * cpg; c < (g + 1) * cpg; ++c)
        for (int px = 0; px < hw; ++px) {
          double v = ((double)__half2float(ho[((size_t)i * hw + px) * Cout + c]) - mean) * rstd * hg[c] + hb[c];
          if (silu) v /= 1.0 + std::exp(-v);
          y[((size_t)i * Cout + c) * hw + px] = (float)v;
        }
    }
  NOPE_CUDA(cudaMemcpy(out, y.data(), y.size() * sizeof(float), cudaMemcpyHostToDevice));
  return 0;
}

// The sweep's fused layer: out = [SiLU](GroupNorm_G(conv(x) + bias)) + chan_bias[n, c] + residual, all in the
// epilogue of the CTA-pair kernel (GnFuse).  precision 0 / 1 / 2 as nope_unet_set_option("precision"); with 2 the
// inputs and the residual are split into fp16 (hi, lo) pairs and the output is the sum of its pair.
int nope_op_conv_gn_fused(int mode, int precision, const float* x0, int C0, const float* x1, int C1,
                          const float* weight, const float* bias, const float* gamma, const float* beta, int G,
                          int silu, const float* chan_bias, const float* residual, int res_div, float* out,
                          float* emit_out, int n_img, int H, int W, int Cout, void* stream) {
  NOPE_CHECK(out, "null argument");
  NOPE_CHECK(precision >= 0 && precision <= 2, "precision must be 0..2");
  NOPE_CHECK(G == 0 || (gamma && beta), "GroupNorm needs gamma / beta");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const int hw = H * W;
  OpConv op;
  if (op.setup(mode, 2, precision, x0, C0, x1, C1, weight, bias, n_img, H, W, Cout, st)) return -1;
  __half *r = nullptr, *rl = nullptr, *pbh = nullptr;
  const int n_res = residual ? (res_div > 0 ? (n_img + res_div - 1) / res_div : n_img) : 0;
  if (residual && to_nhwc(residual, &r, op.s, n_res, Cout, hw, st, precision == 2 ? &rl : nullptr)) return -1;
  if (chan_bias && to_nhwc(chan_bias, &pbh, op.s, n_img, Cout, 1, st)) return -1;
  if (op.eng.ensure_workspace(n_img, std::max(n_res, 1), 0, st)) return -1;
  op.eng.pb = pbh;
  op.eng.P = Cout;
  NormLayer N;
  N.C = Cout; N.G = std::max(G, 1);
  N.gamma = const_cast<float*>(gamma);
  N.beta = const_cast<float*>(beta);
  GnSpec gs;
  gs.norm = G > 0 ? &N : nullptr;
  gs.silu = silu != 0;
  gs.pb_offset = chan_bias ? 0 : -1;
  if (residual) gs.res = Act(r, Cout, rl);
  gs.res_div = residual ? res_div : 0;
  float2* em = nullptr;
  const int eparts = nope_unet::fused_emit_parts(H, Cout);
  if (emit_out) {
    if (op.s.alloc(&em, (size_t)n_img * eparts)) return -1;
    gs.emit = em;
  }
  if (op.eng.conv(op.L, op.in0, op.in1, op.out, H, n_img, n_img, st, &gs)) return -1;
  if (to_nchw(op.out.hi, out, n_img, Cout, hw, st, op.out.lo)) return -1;
  if (emit_out) {
    // fold the per-tile partials on the host side of the test: [n_img][eparts] -> [n_img][2]
    std::vector<float2> h((size_t)n_img * eparts);
    NOPE_CUDA(cudaStreamSynchronize(st));
    NOPE_CUDA(cudaMemcpy(h.data(), em, h.size() * sizeof(float2), cudaMemcpyDeviceToHost));
    std::vector<float> sums((size_t)n_img * 2, 0.f);
    for (int i = 0; i < n_img; ++i)
      for (int e2 = 0; e2 < eparts; ++e2) {
        sums[2 * i] += h[(size_t)i * eparts + e2].x;
        sums[2 * i + 1] += h[(size_t)i * eparts + e2].y;
      }
    NOPE_CUDA(cudaMemcpy(emit_out, sums.data(), sums.size() * sizeof(float), cudaMemcpyHostToDevice));
  }
  NOPE_CUDA(cudaStreamSynchronize(st));
  return 0;
}

int nope_op_linear_attention(int impl, const float* qkv, float* out, int n_img, int H, int W, void* stream) {
  NOPE_CHECK(qkv && out, "null argument");
  NOPE_CHECK(impl == 1 || (impl == 0 && (H * W) % kBM == 0), "impl 0 (tensor cores) needs H*W % 128 == 0; impl 1 = CUDA cores");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  DeviceAllocs s;
  __half *a = nullptr, *o = nullptr;
  if (to_nhwc(qkv, &a, s, n_img, 384, H * W, st) || s.alloc(&o, (size_t)n_img * 128 * H * W)) return -1;
  if (impl == 0) {
    cudaDeviceProp prop;
    int dev = 0;
    NOPE_CUDA(cudaGetDevice(&dev));
    NOPE_CUDA(cudaGetDeviceProperties(&prop, dev));
    if (launch_linattn_tc(a, o, n_img, H * W, prop.multiProcessorCount, st)) return -1;
  } else {
    linattn_kernel<<<dim3(4, n_img), kLinAttnThreads, 0, st>>>(a, o, H * W);
  }
  NOPE_CUDA(cudaGetLastError());
  if (to_nchw(o, out, n_img, 128, H * W, st)) return -1;
  NOPE_CUDA(cudaStreamSynchronize(st));
  return 0;
}

int nope_op_attention(const float* qkv, float* out, int n_img, int H, int W, void* stream) {
  NOPE_CHECK(qkv && out && H * W <= 32, "bad argument (H*W must be <= 32)");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  DeviceAllocs s;
  __half *a = nullptr, *o = nullptr;
  if (to_nhwc(qkv, &a, s, n_img, 384, H * W, st) || s.alloc(&o, (size_t)n_img * 128 * H * W)) return -1;
  midattn_kernel<<<n_img, 128, 0, st>>>(a, o, H * W);
  NOPE_CUDA(cudaGetLastError());
  if (to_nchw(o, out, n_img, 128, H * W, st)) return -1;
  NOPE_CUDA(cudaStreamSynchronize(st));
  return 0;
}

int nope_op_upsample2x(const float* x, float* out, int n_img, int C, int H, int W, void* stream) {
  NOPE_CHECK(x && out && C % 8 == 0 && H == W, "bad argument");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  DeviceAllocs s;
  __half *a = nullptr, *o = nullptr;
  if (to_nhwc(x, &a, s, n_img, C, H * W, st) || s.alloc(&o, (size_t)n_img * C * H * W * 4)) return -1;
  upsample2x_kernel<<<ew_grid((long long)n_img * 4 * H * W * C / 8), 256, 0, st>>>(a, o, n_img, H, W, C);
  NOPE_CUDA(cudaGetLastError());
  if (to_nchw(o, out, n_img, C, 4 * H * W, st)) return -1;
  NOPE_CUDA(cudaStreamSynchronize(st));
  return 0;
}

int nope_unet_debug_tap(nope_unet_t* u, const float* ref_feat, const float* poses, int N, const char* tap,
                        float* out, int64_t out_capacity_floats, int* out_C, int* out_H, void* stream) {
  return engine_debug_tap(u, ref_feat, poses, N, tap, out, out_capacity_floats, out_C, out_H, stream);
}

// ---------------------------------------------------------------------------------
// LDM variant
// ---------------------------------------------------------------------------------
int nope_ldm_create(nope_ldm_t** out, int model_channels, int context_dim, int latent_ch, int latent_hw,
                    int device) {
  NOPE_CHECK(out != nullptr, "null out pointer");
  NOPE_CHECK(model_channels > 0 && model_channels % 256 == 0 && model_channels <= 512,
             "model_channels must be 256 or 512 (GroupNorm(32) statistics ride on 8-channel octets)");
  NOPE_CHECK(context_dim >= 1, "context_dim must be positive");
  NOPE_CHECK(latent_ch >= 1 && latent_ch <= kMaxLatent, "latent_ch must be in [1, 8]");
  NOPE_CHECK(latent_hw == 32, "latent_hw must be 32 in this build");
  auto m = std::make_unique<nope_ldm>();
  if (open_device(device, &m->num_sms)) return -1;
  m->mc = model_channels;
  m->ctx = context_dim;
  m->Cl = latent_ch;
  m->S0 = latent_hw;
  m->device = device;
  m->build_plan();
  m->build_schema();
  *out = m.release();
  return 0;
}

void nope_ldm_destroy(nope_ldm_t* m) { delete m; }

int nope_ldm_load_tensor(nope_ldm_t* m, const char* key, const float* data, const int64_t* shape, int ndim) {
  return engine_load_tensor(m, key, data, shape, ndim, !(key && nope_ldm::never_read(key)));
}

int nope_ldm_finalize(nope_ldm_t* m) { return engine_finalize(m); }
int nope_ldm_set_chunk(nope_ldm_t* m, int hyps) {
  NOPE_CHECK(m && hyps >= 1 && hyps <= 2048, "chunk must be in [1, 2048]");
  m->chunk = hyps;
  return 0;
}
int nope_ldm_set_option(nope_ldm_t* m, const char* name, int value) {
  NOPE_CHECK(m && name, "null argument");
  if (std::strcmp(name, "hoist") == 0) { m->hoist = value != 0; return 0; }
  if (std::strcmp(name, "precision") == 0) {
    NOPE_CHECK(!m->finalized, "precision must be set before finalize");
    NOPE_CHECK(value == 0 || value == 1, "LDM precision: 0 (fp16 weights) or 1 (exact weights, W_hi + W_lo)");
    m->precision = value;
    return 0;
  }
  return fail(std::string("unknown option: ") + name);
}
int64_t nope_ldm_last_launch_count(const nope_ldm_t* m) { return m ? m->launches : 0; }

int nope_ldm_profile(nope_ldm_t* m, int enable) {
  NOPE_CHECK(m, "null engine");
  m->prof.reset(enable != 0);
  return 0;
}
int nope_ldm_profile_read(nope_ldm_t* m, double* ms, double* flops, int64_t* launches) {
  NOPE_CHECK(m && ms && flops && launches, "null argument");
  NOPE_CUDA(cudaDeviceSynchronize());
  for (int k = 0; k < 2; ++k) { ms[k] = 0.0; flops[k] = 0.0; launches[k] = 0; }
  for (size_t i = 0; i < m->prof.rec.size(); ++i) {
    float t = 0.f;
    if (m->prof.ms(i, &t)) return -1;
    const int k = m->prof.rec[i].kind;
    ms[k] += t;
    flops[k] += m->prof.rec[i].flops;
    launches[k] += 1;
  }
  return 0;
}

int nope_ldm_sweep_multi(nope_ldm_t* m, const float* ref_latent, const float* poses, int B, int N,
                         const float* query_latent, int Q, float* out_emb, float* out_sim, int k, float* out_topv,
                         int64_t* out_topi, int64_t idx_base, void* stream) {
  return engine_sweep(m, ref_latent, poses, B, N, query_latent, Q, out_emb, out_sim, k, out_topv, out_topi, idx_base,
                      stream);
}

int nope_ldm_debug_tap(nope_ldm_t* m, const float* ref_latent, const float* poses, int N, const char* tap,
                       float* out, int64_t out_capacity_floats, int* out_C, int* out_H, void* stream) {
  return engine_debug_tap(m, ref_latent, poses, N, tap, out, out_capacity_floats, out_C, out_H, stream);
}

int nope_ldm_run_block(nope_ldm_t* m, const char* name, const float* x0, int C0, const float* x1, int C1, int S,
                       int n, const float* poses, float* out, void* stream) {
  NOPE_CHECK(m && m->finalized && name && x0 && out && n >= 1, "bad argument");
  NOPE_CHECK(S == 8 || S == 16 || S == 32, "side must be 8, 16 or 32");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  NOPE_CUDA(cudaSetDevice(m->device));
  if (m->ensure_workspace(std::max(n, 1), 1, 0, st)) return -1;
  NOPE_CHECK(n <= m->cap, "run_block: n exceeds the workspace");
  const std::string nm = name;
  // stage the inputs in XA / XB (NHWC fp16); results land in XC
  nchw_f32_to_nhwc_f16_kernel<<<ew_grid((long long)n * C0 * S * S), 256, 0, st>>>(x0, m->XA, n, C0, S * S);
  if (x1) nchw_f32_to_nhwc_f16_kernel<<<ew_grid((long long)n * C1 * S * S), 256, 0, st>>>(x1, m->XB, n, C1, S * S);
  NOPE_CUDA(cudaGetLastError());
  int Co = 0, So = S;
  if (m->convs.count(nm + ".c1")) {
    if (m->resblock(nm, m->XA, C0, x1 ? m->XB : nullptr, x1 ? C1 : 0, m->XC, S, n, st)) return -1;
    Co = m->convs.at(nm + ".c2").cout;
  } else if (m->convs.count(nm + ".qkv")) {
    NOPE_CHECK(poses != nullptr && x1 == nullptr, "transformer block: poses required, one input");
    if (m->cross_terms(poses, n, st)) return -1;
    if (m->stats(m->XA, C0, nullptr, 0, S, n, m->S_out, st)) return -1;
    if (m->transformer(nm, m->XA, m->XC, C0, S, n, m->cb, st)) return -1;
    Co = C0;
  } else if (m->convs.count(nm)) {
    const ConvLayer& L = m->convs.at(nm);
    NOPE_CHECK(x1 == nullptr && L.cin == C0 && (L.up || L.stride == 2), "run_block: not a resample conv");
    So = L.up ? 2 * S : S / 2;
    if (m->conv(L, m->XA, m->XC, So, n, st)) return -1;
    Co = L.cout;
  } else {
    return fail(std::string("run_block: unknown module ") + nm);
  }
  nhwc_f16_to_nchw_f32_kernel<<<ew_grid((long long)n * Co * So * So), 256, 0, st>>>(m->XC, out, n, Co, So * So);
  NOPE_CUDA(cudaGetLastError());
  NOPE_CUDA(cudaStreamSynchronize(st));
  return 0;
}

int nope_op_mh_attention(const float* qkv, float* out, int n_img, int n_tok, int C, void* stream) {
  NOPE_CHECK(qkv && out && n_img >= 1 && n_tok >= 64 && n_tok % 64 == 0 && C % 64 == 0 && C >= 64,
             "bad arguments (n_tok and C must be multiples of 64)");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  DeviceAllocs s;
  nope_ldm e;    // launches the attention on the staging buffers in s
  const size_t tok = (size_t)n_img * n_tok;
  __half *q16 = nullptr, *vt = nullptr, *o16 = nullptr;
  if (s.alloc(&q16, tok * 3 * C) || s.alloc(&o16, tok * C) || s.alloc(&vt, tok * C)) return -1;
  // [n_img, n_tok, 3C] fp32 is already token-major: a plain fp32 -> fp16 cast ("NCHW" with hw = 1)
  nchw_f32_to_nhwc_f16_kernel<<<ew_grid((long long)tok * 3 * C), 256, 0, st>>>(qkv, q16, (int)tok, 3 * C, 1);
  NOPE_CUDA(cudaGetLastError());
  if (e.attention(q16, vt, o16, C, n_tok, n_img, st)) return -1;
  nhwc_f16_to_nchw_f32_kernel<<<ew_grid((long long)tok * C), 256, 0, st>>>(o16, out, (int)tok, C, 1);
  NOPE_CUDA(cudaGetLastError());
  NOPE_CUDA(cudaStreamSynchronize(st));
  return 0;
}

// ---------------------------------------------------------------------------------
// searches under occlusion: visible latent maps and the scores over them (DESIGN.md section 27)
// ---------------------------------------------------------------------------------
int nope_crop_hidden(const uint8_t* occluders, int H, int W, const double* inv_maps, int B, int S, uint8_t* out,
                     void* stream) {
  NOPE_CHECK(occluders && inv_maps && out, "null argument");
  NOPE_CHECK(B >= 1 && B <= 65535, "B must be in [1, 65535]");
  NOPE_CHECK(H >= 1 && H <= kCropMaxSide && W >= 1 && W <= kCropMaxSide, "H and W must be in [1, 16384]");
  NOPE_CHECK(S >= 8 && S % 8 == 0 && S / 8 == kVisSide, "S must be 8 * 32 = 256 (the latent grid is 32 x 32)");
  crop_hidden_kernel<<<dim3((S * S + kCropThreads - 1) / kCropThreads, B), kCropThreads, 0,
                       static_cast<cudaStream_t>(stream)>>>(occluders, H, W, inv_maps, S, out);
  NOPE_CUDA(cudaGetLastError());
  return 0;
}

int nope_latent_visibility(const uint8_t* hidden, int B, int S, const int32_t* image_idx, const float* cossin, int P,
                           uint8_t* out, void* stream) {
  NOPE_CHECK(hidden && image_idx && cossin && out, "null argument");
  NOPE_CHECK(B >= 1, "B must be >= 1");
  NOPE_CHECK(S >= 8 && S % 8 == 0 && S / 8 == kVisSide, "S must be 8 * 32 = 256 (the latent grid is 32 x 32)");
  NOPE_CHECK(P >= 1 && P <= INT32_MAX / 2, "P (pairs) must be in [1, 2^30)");
  latent_visibility_kernel<<<P, kVisThreads, 0, static_cast<cudaStream_t>(stream)>>>(hidden, B, S, image_idx, cossin,
                                                                                     out);
  NOPE_CUDA(cudaGetLastError());
  return 0;
}

int nope_unet_sweep_visible(nope_unet_t* u, const float* ref_feat, const float* poses, int B, int N,
                            const float* query_feat, int Q, const uint8_t* query_visible, float* out_emb,
                            float* out_sim, int k, float* out_topv, int64_t* out_topi, int64_t idx_base,
                            void* stream) {
  NOPE_CHECK(query_feat && query_visible, "null query or visible map");
  return engine_sweep(u, ref_feat, poses, B, N, query_feat, Q, out_emb, out_sim, k, out_topv, out_topi, idx_base,
                      stream, query_visible);
}

int nope_ldm_sweep_visible(nope_ldm_t* m, const float* ref_latent, const float* poses, int B, int N,
                           const float* query_latent, int Q, const uint8_t* query_visible, float* out_emb,
                           float* out_sim, int k, float* out_topv, int64_t* out_topi, int64_t idx_base,
                           void* stream) {
  NOPE_CHECK(query_latent && query_visible, "null query or visible map");
  return engine_sweep(m, ref_latent, poses, B, N, query_latent, Q, out_emb, out_sim, k, out_topv, out_topi, idx_base,
                      stream, query_visible);
}

int nope_score_topk_visible(const float* query_feat, const float* emb, int R, int O, int N, int C, int HW,
                            const int32_t* slots, const int32_t* row_off, int G, int A, const uint8_t* visible,
                            int metric, float occlusion_threshold, int k, float* out_sim, float* out_topv,
                            int64_t* out_topi, void* stream) {
  NOPE_CHECK(visible, "null visible map");
  return score_grouped(query_feat, emb, R, O, N, C, HW, slots, row_off, G, A, visible, metric, occlusion_threshold, k,
                       out_sim, out_topv, out_topi, stream);
}

}  // extern "C"
