// nope_b200 -- the host-side lifecycle every weight-holding engine (UNet, template encoder, VAE encoder, VAE decoder,
// LDM) shares: the state_dict schema and the host copies staged against it until finalize, the device allocations
// freed with the engine, the device check of every *_create, and the bodies of the *_load_tensor / *_finalize /
// per-chunk C-ABI entry points.
//
// An engine E provides: `static constexpr const char* kName` (the name its errors carry), `bool finalized`,
// `int device`, `StagedWeights staged`, and `int finalize()` (packs the staged tensors; runs once every schema key
// is present, on E's device).
#pragma once
#include <algorithm>
#include <map>
#include <string>
#include <vector>

#include "common.cuh"

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

// Device allocations owned by an engine, freed by release() or with the owner.
class DeviceAllocs {
 public:
  DeviceAllocs() = default;
  DeviceAllocs(const DeviceAllocs&) = delete;
  DeviceAllocs& operator=(const DeviceAllocs&) = delete;
  ~DeviceAllocs() { release(); }

  template <typename T> int alloc(T** out, size_t n) {
    NOPE_CUDA(cudaMalloc(reinterpret_cast<void**>(out), n * sizeof(T)));
    ptrs_.push_back(*out);
    return 0;
  }
  template <typename T> int upload(T** out, const T* src, size_t n) {
    if (alloc(out, std::max<size_t>(n, 1))) return -1;
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
  NOPE_CHECK(k >= 0 && k <= N && k <= 64, "k must be in [0, min(N, 64)]");
  NOPE_CHECK(k == 0 || (out_topv && out_topi), "top-k outputs missing");
  return 0;
}

}  // namespace nope
