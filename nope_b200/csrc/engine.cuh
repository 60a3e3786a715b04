// nope_b200 -- the host-side code every weight-holding engine (UNet, template encoder, VAE encoder, VAE decoder,
// LDM) shares: the state_dict schema and the host copies staged against it until finalize, the device allocations
// freed with the engine, the device check of every *_create, and the bodies of the *_load_tensor / *_finalize /
// per-chunk C-ABI entry points.  The two sweep engines (UNet, LDM) also share the sweep driver, the debug tap and the
// per-launch profile; the three image engines (template encoder, VAE encoder, VAE decoder) share the module entry of
// their plans and the run_block argument checks, and the two image encoders the rotated-encode loop.
//
// An engine E provides: `static constexpr const char* kName` (the name its errors carry), `bool finalized`,
// `int device`, `StagedWeights staged`, and `int finalize()` (packs the staged tensors; runs once every schema key
// is present, on E's device).
//
// A sweep engine (engine_sweep, engine_debug_tap) also provides `int chunk`, `int64_t launches`, `DebugTap dtap`,
// `float* score_partial` and `float* sim_buf`, and
//   int ensure_workspace(int hyps, int refs, int scores, cudaStream_t)  sizes the workspace (grow_workspace), score
//       partials and similarity scratch of `scores` (reference, query, pose) triples included, before a launch;
//   int prestage(const float* ref, int B, cudaStream_t)                  the pose-independent prefix per reference;
//   int forward_chunk(poses, hyp0, n, N, query, out_emb, score_part, cudaStream_t, int Q, const uint8_t* vis);
//   int rank(part, sim, B, N, Q, k, topv, topi, idx_base, cudaStream_t, vis) the similarities and top-k from the
//       partials; vis (nullable) [B, Q, hw] the rows' visible maps (DESIGN.md section 27).
// An image engine derives from ImageEngine (encoder.cuh), which holds `launches`, `mem` and the convolution
// layers, and provides `kChunk` and `std::vector<ImageModule> plan`, built in forward order when the handle is
// created; its schema, weight packing, forward pass and run_block all walk that plan.  An image encoder
// (per_rotated_chunk) also provides `float* rot_stage` and `int encode(const float*, int, float*, cudaStream_t)`.
#pragma once
#include <algorithm>
#include <map>
#include <string>
#include <tuple>
#include <vector>

#include "common.cuh"
#include "conv_tc.cuh"
#include "kernels.cuh"
#include "rank.cuh"

namespace nope {

struct HostTensor {
  std::vector<int64_t> shape;
  std::vector<float> data;
};

// The state_dict schema of one engine (key -> shape) and the host copies loaded against it.
class StagedWeights {
 public:
  void expect(const std::string& key, std::vector<int64_t> shape) { schema_[key] = std::move(shape); }

  // Checks key, rank and shape against the schema and stages a copy of data.  data == nullptr records the shape
  // only: a key the engine accepts for schema compatibility but never reads.
  int load(const char* engine, const char* key, const float* data, const int64_t* shape, int ndim) {
    auto it = schema_.find(key);
    if (it == schema_.end()) return fail(std::string(engine) + ": unexpected state_dict key '" + key + "'");
    const std::vector<int64_t> got(shape, shape + std::max(ndim, 0));
    if (ndim < 0 || got != it->second)
      return fail(std::string(engine) + (got.size() != it->second.size() ? ": rank" : ": shape") + " mismatch for '" +
                  key + "': expected " + str(it->second) + ", got " + str(got));
    HostTensor& t = host_[key];
    t.shape = got;
    size_t n = 1;
    for (int64_t d : got) n *= (size_t)d;
    if (data) t.data.assign(data, data + n);
    else t.data.clear();
    return 0;
  }
  // every schema key has been loaded
  int require_all(const char* engine) const {
    for (const auto& kv : schema_)
      if (!host_.count(kv.first)) return fail(std::string(engine) + ": state_dict is missing '" + kv.first + "'");
    return 0;
  }
  bool has(const std::string& key) const { return host_.count(key) != 0; }
  const HostTensor& at(const std::string& key) const { return host_.at(key); }
  // stages a tensor the engine derives from loaded ones (a folded or concatenated weight) under a private key
  void put(const std::string& key, HostTensor t) { host_[key] = std::move(t); }
  void clear() { host_.clear(); }

 private:
  static std::string str(const std::vector<int64_t>& s) {
    std::string r = "[";
    for (size_t i = 0; i < s.size(); ++i) r += (i ? ", " : "") + std::to_string(s[i]);
    return r + "]";
  }
  std::map<std::string, std::vector<int64_t>> schema_;
  std::map<std::string, HostTensor> host_;
};

// Device allocations owned by an engine or a call, freed by release() or with the owner.
class DeviceAllocs {
 public:
  DeviceAllocs() = default;
  DeviceAllocs(const DeviceAllocs&) = delete;
  DeviceAllocs& operator=(const DeviceAllocs&) = delete;
  ~DeviceAllocs() { release(); }

  // n elements; n == 0 still gets a distinct pointer
  template <typename T> int alloc(T** out, size_t n) {
    NOPE_CUDA(cudaMalloc(reinterpret_cast<void**>(out), std::max<size_t>(n, 1) * sizeof(T)));
    ptrs_.push_back(*out);
    return 0;
  }
  template <typename T> int upload(T** out, const T* src, size_t n) {
    if (alloc(out, n)) return -1;
    NOPE_CUDA(cudaMemcpy(*out, src, n * sizeof(T), cudaMemcpyHostToDevice));
    return 0;
  }
  template <typename T> int upload(T** out, const std::vector<T>& v) { return upload(out, v.data(), v.size()); }
  void release() {
    for (void* p : ptrs_) cudaFree(p);
    ptrs_.clear();
  }

 private:
  std::vector<void*> ptrs_;
};

// One block of a layer's weights: fp32 [rows][cin][taps] in host or device memory, placed at weight row `row` and
// W_hi column `col` (its remainders at column K + col of the W_lo plane).  For the folded upsample it is the
// [rows][cin][3][3] kernel, packed as 4 rows per output channel.
struct WeightBlock {
  const float* w;
  int rows, cin, taps, row, col;
};

// Packs layer L, whose shape (cin, cout, K, wlo, taps, up) is set, from its weight blocks with pack_conv_weight (bf16:
// the W_hi plane in bf16) into memory of `mem`; rows no block covers (the zero rows that pad cout) are zero.  Uploads
// bias (cout values; empty: none) and encodes the weight map of bn rows (bn 0: pick_bn(cout)).
inline int pack_conv_layer(DeviceAllocs& mem, ConvLayer& L, const std::vector<WeightBlock>& blocks,
                           const std::vector<float>& bias, bool bf16 = false, cudaStream_t st = 0) {
  if (!L.bn) L.bn = pick_bn(L.cout);
  const size_t n = (size_t)L.rows() * L.row_len();
  if (mem.alloc(&L.w, n)) return -1;
  NOPE_CUDA(cudaMemsetAsync(L.w, 0, n * sizeof(__half), st));
  for (const WeightBlock& b : blocks)
    if (pack_conv_weight(b.w, L.w + (size_t)b.row * L.row_len(), b.rows, b.cin, b.taps, L.up, L.row_len(), b.col,
                         L.wlo ? L.K : 0, bf16 ? 1 : 0, st))
      return -1;
  if (!bias.empty() && mem.upload(&L.bias, bias)) return -1;
  return make_weight_map(&L.wmap, L.w, L.rows(), L.row_len(), L.bn);
}

// bump allocator over one device slab (base == nullptr: size computation only)
struct Bump {
  uint8_t* base = nullptr;
  size_t off = 0;
  template <typename T> void take(T** out, size_t n) {
    off = (off + 255) & ~static_cast<size_t>(255);
    if (base) *out = reinterpret_cast<T*>(base + off);     // size-only passes leave the engine untouched
    off += n * sizeof(T);
  }
};

// The slab a sweep or image engine's workspace lives in: owned and freed with the engine, or a caller's buffer
// (`external`, nope_unet_set_workspace) that the engine never frees.
struct WorkspaceSlab {
  uint8_t* base = nullptr;
  bool external = false;
  WorkspaceSlab() = default;
  WorkspaceSlab(const WorkspaceSlab&) = delete;
  WorkspaceSlab& operator=(const WorkspaceSlab&) = delete;
  ~WorkspaceSlab() { release(); }
  void release() {
    if (base && !external) cudaFree(base);
    base = nullptr;
    external = false;
  }
};

// Moves the workspace of engine e to a new slab for the capacities c...  The engine provides `WorkspaceSlab ws`,
// `TmapCache tmaps` and `size_t layout(Bump&, c...)`, which places every workspace buffer and returns the bytes they
// span.  In order: a size pass; a device synchronisation, since launches may still use the old slab; the old slab
// released and the tensor maps keyed by its pointers dropped; the new slab, `external` (a caller's buffer of at least
// the size pass's bytes + 256) or one cudaMalloc; the assign pass; the capacity fields `caps` set to c...  After a
// failure they are 0 and the slab is null, so the next call grows again instead of running on freed buffers, and the
// runtime's last error is cleared so that later calls do not report it.
template <typename E, typename... C>
int grow_workspace(E* e, std::tuple<C&...> caps, void* external, C... c) {
  caps = std::tuple<C...>();
  Bump size;
  const size_t bytes = e->layout(size, c...);
  cudaError_t err = cudaDeviceSynchronize();
  e->ws.release();
  e->tmaps.clear();
  if (err == cudaSuccess && !external) err = cudaMalloc(reinterpret_cast<void**>(&e->ws.base), bytes);
  if (err != cudaSuccess) {
    e->ws.base = nullptr;
    cudaGetLastError();
    return fail(std::string(E::kName) + ": workspace of " + std::to_string(bytes) + " bytes: " +
                cudaGetErrorString(err));
  }
  if (external) {
    e->ws.base = static_cast<uint8_t*>(external);
    e->ws.external = true;
  }
  Bump b;
  b.base = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(e->ws.base) + 255) & ~static_cast<uintptr_t>(255));
  e->layout(b, c...);
  caps = std::tuple<C...>(c...);
  return 0;
}

// The check of every *_create: `device` exists and is an sm_90 part; its SM count goes to *num_sms.
inline int open_device(int device, int* num_sms) {
  int ndev = 0;
  NOPE_CUDA(cudaGetDeviceCount(&ndev));
  NOPE_CHECK(device >= 0 && device < ndev, "no such CUDA device");
  cudaDeviceProp prop;
  NOPE_CUDA(cudaGetDeviceProperties(&prop, device));
  NOPE_CHECK(prop.major == 9 && prop.minor == 0, "nope_b200 kernels are built for sm_90a (H100) only");
  *num_sms = prop.multiProcessorCount;
  return 0;
}

// *_load_tensor.  stage == false accepts the key with its shape and drops the data.
template <typename E>
int engine_load_tensor(E* e, const char* key, const float* data, const int64_t* shape, int ndim, bool stage = true) {
  NOPE_CHECK(e && key && data && shape, "null argument");
  if (e->finalized) return fail(std::string(E::kName) + ": already finalized, cannot load '" + key + "'");
  return e->staged.load(E::kName, key, stage ? data : nullptr, shape, ndim);
}

// *_finalize: packs the staged weights once every schema key is present, then frees the host copies.
template <typename E> int engine_finalize(E* e) {
  NOPE_CHECK(e, "null engine");
  if (e->finalized) return fail(std::string(E::kName) + ": already finalized");
  if (e->staged.require_all(E::kName)) return -1;
  NOPE_CUDA(cudaSetDevice(e->device));
  if (e->finalize()) return -1;
  e->staged.clear();
  e->finalized = true;
  return 0;
}

// B items through step(in, n, out, stream) E::kChunk at a time (the engine's workspace holds that many); the
// engine's launch count becomes the sum over the chunks.
template <typename E>
int per_chunk(E* e, int (E::*step)(const float*, int, float*, cudaStream_t), const float* in, size_t in_per, int B,
              float* out, size_t out_per, void* stream) {
  const cudaStream_t st = static_cast<cudaStream_t>(stream);
  int64_t launches = 0;
  for (int lo = 0; lo < B; lo += E::kChunk) {
    const int n = std::min(E::kChunk, B - lo);
    const int rc = (e->*step)(in + (size_t)lo * in_per, n, out + (size_t)lo * out_per, st);
    if (rc != 0) return rc;
    launches += e->launches;
  }
  e->launches = launches;
  return 0;
}

// The argument rules of nope_unet_sweep_multi / nope_ldm_sweep_multi.
template <typename E>
int check_sweep(const E* e, const float* ref, const float* poses, int B, int N, const float* query, int Q,
                const float* out_sim, int k, const float* out_topv, const int64_t* out_topi) {
  NOPE_CHECK(e && e->finalized, "engine not finalized");
  NOPE_CHECK(ref && poses && B >= 1 && N >= 1, "bad arguments");
  NOPE_CHECK(Q >= 1, "Q (queries per reference) must be >= 1");
  NOPE_CHECK((int64_t)B * Q * N <= INT32_MAX, "B * Q * N exceeds the scored-triple limit (2^31 - 1)");
  NOPE_CHECK(!(out_sim || k > 0) || query, "scores / top-k need the query");
  NOPE_CHECK(k >= 0 && k <= N && k <= kMaxTopK, "k must be in [0, min(N, 64)]");
  NOPE_CHECK(k == 0 || (out_topv && out_topi), "top-k outputs missing");
  return 0;
}

// The debug tap of a sweep engine (nope_*_debug_tap): the first time forward_chunk passes the activation called
// `name`, capture() writes it to `out` as [n, C, S, S] fp32 and records its shape.
struct DebugTap {
  std::string name;
  float* out = nullptr;      // nullptr: no tap armed
  int64_t cap = 0;           // floats at out
  int C = 0, S = 0;
  bool hit = false;
  int capture(const char* at, const __half* hi, const __half* lo, bool bf16, int C_, int S_, int n, cudaStream_t st) {
    if (out == nullptr || name != at || hit) return 0;
    NOPE_CHECK((int64_t)n * C_ * S_ * S_ <= cap, "debug tap: output buffer too small");
    nhwc_f16_to_nchw_f32_kernel<<<ew_grid((long long)n * C_ * S_ * S_), 256, 0, st>>>(hi, out, n, C_, S_ * S_, lo,
                                                                                       bf16);
    NOPE_CUDA(cudaGetLastError());
    C = C_;
    S = S_;
    hit = true;
    return 0;
  }
};

// What one profiled launch computed: executed FLOPs, algorithmic FLOPs (those of the fp16 mode), and the engine's
// own launch kind and shape.
struct LaunchRecord {
  double flops = 0.0, alg_flops = 0.0;
  int kind = 0;
  int4 shape = {0, 0, 0, 0};
};

// CUDA-event times of an engine's heavy launches (bench.py's roofline): begin() and end() bracket one launch and do
// nothing while profiling is off.
struct LaunchProfile {
  bool on = false;
  std::vector<cudaEvent_t> ev;       // one (begin, end) pair per record
  std::vector<LaunchRecord> rec;

  LaunchProfile() = default;
  LaunchProfile(const LaunchProfile&) = delete;
  LaunchProfile& operator=(const LaunchProfile&) = delete;
  ~LaunchProfile() { reset(false); }
  void reset(bool enable) {
    for (cudaEvent_t e : ev) cudaEventDestroy(e);
    ev.clear();
    rec.clear();
    on = enable;
  }
  int begin(cudaStream_t st) { return on ? record(st) : 0; }
  int end(cudaStream_t st, const LaunchRecord& r) {
    if (!on) return 0;
    if (record(st)) return -1;
    rec.push_back(r);
    return 0;
  }
  // milliseconds of launch i (its events must have completed)
  int ms(size_t i, float* t) const {
    NOPE_CUDA(cudaEventElapsedTime(t, ev[2 * i], ev[2 * i + 1]));
    return 0;
  }

 private:
  int record(cudaStream_t st) {
    cudaEvent_t e;
    NOPE_CUDA(cudaEventCreate(&e));
    ev.push_back(e);
    NOPE_CUDA(cudaEventRecord(e, st));
    return 0;
  }
};

// nope_unet_sweep_multi / nope_ldm_sweep_multi: the B references' N poses in chunks of the engine's `chunk`
// hypotheses, each scored against its reference's Q queries, then ranked.  A sweep of a shape the engine has served
// before makes no allocation and no host synchronisation.  With vis (the *_sweep_visible entry points) each row
// scores only its visible latent pixels.
template <typename E>
int engine_sweep(E* e, const float* ref, const float* poses, int B, int N, const float* query, int Q, float* out_emb,
                 float* out_sim, int k, float* out_topv, int64_t* out_topi, int64_t idx_base, void* stream,
                 const uint8_t* vis = nullptr) {
  if (check_sweep(e, ref, poses, B, N, query, Q, out_sim, k, out_topv, out_topi)) return -1;
  const cudaStream_t st = static_cast<cudaStream_t>(stream);
  NOPE_CUDA(cudaSetDevice(e->device));
  e->launches = 0;
  const int total = B * N;
  const int cap = std::min(e->chunk, total);
  if (e->ensure_workspace(cap, B, query ? total * Q : 0, st)) return -1;
  float* part = query ? e->score_partial : nullptr;
  if (e->prestage(ref, B, st)) return -1;
  for (int h0 = 0; h0 < total; h0 += cap) {
    const int n = std::min(cap, total - h0);
    if (e->forward_chunk(poses, h0, n, N, query, out_emb, part, st, Q, vis)) return -1;
  }
  if (query && (out_sim || k > 0)) {
    if (e->rank(part, out_sim ? out_sim : e->sim_buf, B, N, Q, k, out_topv, out_topi, idx_base, st, vis)) return -1;
    ++e->launches;
  }
  return 0;
}

// nope_unet_debug_tap / nope_ldm_debug_tap: one reference's N <= chunk poses up to the activation called `name`,
// copied to out as [N, C, H, H] fp32.
template <typename E>
int engine_debug_tap(E* e, const float* ref, const float* poses, int N, const char* name, float* out,
                     int64_t out_capacity_floats, int* out_C, int* out_H, void* stream) {
  NOPE_CHECK(e && e->finalized && ref && poses && name && out, "bad argument");
  const cudaStream_t st = static_cast<cudaStream_t>(stream);
  NOPE_CHECK(N <= e->chunk, "debug tap: N must fit one chunk");
  NOPE_CUDA(cudaSetDevice(e->device));
  if (e->ensure_workspace(N, 1, 0, st)) return -1;
  DebugTap& t = e->dtap;
  t.name = name;
  t.out = out;
  t.cap = out_capacity_floats;
  t.hit = false;
  int rc = e->prestage(ref, 1, st);
  if (!rc) rc = e->forward_chunk(poses, 0, N, N, nullptr, nullptr, nullptr, st, 1);
  t.out = nullptr;
  if (rc) return rc;
  NOPE_CUDA(cudaStreamSynchronize(st));
  NOPE_CHECK(t.hit, std::string("unknown tap name: ") + name);
  if (out_C) *out_C = t.C;
  if (out_H) *out_H = t.S;
  return 0;
}

// P rotated 256 x 256 images through E::encode, E::kChunk at a time: rotate(lo, n) launches the rotation of pairs
// [lo, lo + n) into rot_stage (allocated on first use), whose encodings go to out rows [lo, lo + n) of out_per floats.
// The launch count is each chunk's plus its rotation.
template <typename E, typename Rotate>
int per_rotated_chunk(E* e, int P, float* out, size_t out_per, cudaStream_t st, Rotate rotate) {
  if (!e->rot_stage && e->mem.alloc(&e->rot_stage, (size_t)E::kChunk * 3 * 256 * 256)) return -1;
  int64_t launches = 0;
  for (int lo = 0; lo < P; lo += E::kChunk) {
    const int n = std::min(E::kChunk, P - lo);
    rotate(lo, n);
    NOPE_CUDA(cudaGetLastError());
    if (e->encode(e->rot_stage, n, out + (size_t)lo * out_per, st)) return -1;
    launches += e->launches + 1;
  }
  e->launches = launches;
  return 0;
}

// One module of an image engine's plan: the name *_run_block takes, the engine's kind of module, and its input
// [Ci, Hi, Hi] and output [Co, Ho, Ho] per image.  The plan lists the modules in forward order.
struct ImageModule {
  std::string name;
  int kind, Ci, Hi, Co, Ho;
};
inline const ImageModule* find_module(const std::vector<ImageModule>& plan, const std::string& name) {
  for (const ImageModule& m : plan)
    if (m.name == name) return &m;
  return nullptr;
}

// The checks every *_run_block of an image engine makes of its arguments against module m.
inline int check_block(const ImageModule& m, int chunk, int C, int H, int n, int64_t cap_floats) {
  NOPE_CHECK(n >= 1 && n <= chunk, "run_block: n must be in [1, " + std::to_string(chunk) + "]");
  NOPE_CHECK(C == m.Ci && H == m.Hi, "run_block: " + m.name + " takes [n, " + std::to_string(m.Ci) + ", " +
                                         std::to_string(m.Hi) + ", " + std::to_string(m.Hi) + "] inputs, got C = " +
                                         std::to_string(C) + ", H = " + std::to_string(H));
  NOPE_CHECK(cap_floats >= (int64_t)n * m.Co * m.Ho * m.Ho, "run_block: output buffer too small");
  return 0;
}

}  // namespace nope
