// nope_b200 -- shared device helpers: error plumbing, mbarrier / TMA / wgmma
// PTX wrappers for sm_90a.  Everything here is hand-written inline PTX; no
// CUTLASS/CuTe types are used.
#pragma once
#include <cuda.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <string>

#include "wgmma.cuh"

namespace nope {

constexpr int kMaxDevices = 64;   // per-device launch state (shared-memory opt-in, resident clusters)

// ----------------------------------------------------------------------------
// host-side error plumbing (C-ABI returns int codes; message kept thread-local)
// ----------------------------------------------------------------------------
inline std::string& last_error() {
  static thread_local std::string e;
  return e;
}
inline int fail(const std::string& msg) {
  last_error() = msg;
  return -1;
}
#define NOPE_CUDA(expr)                                                          \
  do {                                                                           \
    cudaError_t _e = (expr);                                                     \
    if (_e != cudaSuccess)                                                       \
      return ::nope::fail(std::string(#expr) + ": " + cudaGetErrorString(_e));   \
  } while (0)
#define NOPE_CHECK(cond, msg)                                                    \
  do {                                                                           \
    if (!(cond)) return ::nope::fail(std::string("check failed: ") + #cond + " -- " + (msg)); \
  } while (0)

// ----------------------------------------------------------------------------
// device helpers
// ----------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}

__device__ __forceinline__ bool elect_one() {
  uint32_t pred = 0;
  asm volatile(
      "{\n\t.reg .pred P;\n\t"
      "elect.sync _|P, 0xffffffff;\n\t"
      "selp.u32 %0, 1, 0, P;\n\t}\n"
      : "=r"(pred));
  return pred != 0;
}

// ---- mbarrier ---------------------------------------------------------------
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void fence_mbar_init() {
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)),
               "r"(bytes)
               : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
// suspend-time hint of try_wait: the thread sleeps in hardware until the phase completes or this many ns pass (the
// default limit is a few tens of ns: the wait loops of the idle roles then issue an instruction stream of their own
// -- 60 % of all instructions of the fused-epilogue convolution were PHASECHK / clock / compare / branch)
constexpr uint32_t kMbarSuspendNs = 20000;
__constant__ uint32_t c_mbar_suspend_ns = kMbarSuspendNs;      // NOPE_MBAR_HINT overrides it (A/B measurements)
__device__ __forceinline__ bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n\t.reg .pred P;\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 P, [%1], %2, %3;\n\t"
      "selp.u32 %0, 1, 0, P;\n\t}\n"
      : "=r"(ok)
      : "r"(smem_u32(bar)), "r"(parity), "r"(c_mbar_suspend_ns)
      : "memory");
  return ok != 0;
}
// Bounded wait: a protocol bug traps (surfaces as a CUDA error) instead of
// hanging the GPU.  ~4 s at 2 GHz.  No printf: a function call anywhere in a kernel makes
// ptxas retire every wgmma before issuing the next one, which serialises the mainloop.
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  if (mbar_try_wait(bar, parity)) return;
  const long long t0 = clock64();
  while (!mbar_try_wait(bar, parity))
    if (clock64() - t0 > 8000000000LL) __trap();
}

// ---- async proxy fences / TMA ------------------------------------------------
__device__ __forceinline__ void fence_proxy_async_smem() {
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}
__device__ __forceinline__ void prefetch_tmap(const CUtensorMap* m) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(m)) : "memory");
}
__device__ __forceinline__ void tma_load_2d(void* dst, const CUtensorMap* m, uint64_t* bar,
                                            int c0, int c1) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes"
      " [%0], [%1, {%3, %4}], [%2];"
      ::"r"(smem_u32(dst)), "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0),
      "r"(c1)
      : "memory");
}
__device__ __forceinline__ void tma_load_4d(void* dst, const CUtensorMap* m, uint64_t* bar,
                                            int c0, int c1, int c2, int c3) {
  asm volatile(
      "cp.async.bulk.tensor.4d.shared::cluster.global.mbarrier::complete_tx::bytes"
      " [%0], [%1, {%3, %4, %5, %6}], [%2];"
      ::"r"(smem_u32(dst)), "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0),
      "r"(c1), "r"(c2), "r"(c3)
      : "memory");
}
__device__ __forceinline__ void tma_load_3d(void* dst, const CUtensorMap* m, uint64_t* bar, int c0,
                                            int c1, int c2) {
  asm volatile(
      "cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes"
      " [%0], [%1, {%3, %4, %5}], [%2];"
      ::"r"(smem_u32(dst)), "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0),
      "r"(c1), "r"(c2)
      : "memory");
}
__device__ __forceinline__ void tma_store_3d(const CUtensorMap* m, const void* src, int c0, int c1, int c2) {
  asm volatile("cp.async.bulk.tensor.3d.global.shared::cta.bulk_group [%0, {%2, %3, %4}], [%1];"
               ::"l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(src)), "r"(c0), "r"(c1), "r"(c2)
               : "memory");
}
__device__ __forceinline__ void tma_store_4d(const CUtensorMap* m, const void* src, int c0,
                                             int c1, int c2, int c3) {
  asm volatile(
      "cp.async.bulk.tensor.4d.global.shared::cta.bulk_group [%0, {%2, %3, %4, %5}], [%1];"
      ::"l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(src)), "r"(c0), "r"(c1), "r"(c2),
      "r"(c3)
      : "memory");
}
__device__ __forceinline__ void tma_store_commit() {
  asm volatile("cp.async.bulk.commit_group;" ::: "memory");
}
__device__ __forceinline__ void tma_store_wait_read0() {
  asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory");
}
// at most one bulk group still reading its shared-memory source (double-buffered staging)
__device__ __forceinline__ void tma_store_wait_read1() {
  asm volatile("cp.async.bulk.wait_group.read 1;" ::: "memory");
}
__device__ __forceinline__ void tma_store_wait_all() {
  asm volatile("cp.async.bulk.wait_group 0;" ::: "memory");
}

// x * sigmoid(x) with the fast divide (MUFU.RCP + FMUL, <= 2 ulp): the IEEE '/' expands to a
// ~10-instruction Newton sequence, which made the GroupNorm+SiLU pass issue-bound.
__device__ __forceinline__ float silu_f(float x) { return __fdividef(x, 1.0f + __expf(-x)); }

// 16-bit storage of activations / weights: fp16 (default) or bf16 (engine precision "bf16",
// BASELINE configs[2]).  Pointers stay `__half*` (opaque 16-bit lanes); `bf` selects the conversion.
__device__ __forceinline__ uint32_t pack2(float a, float b, bool bf) {
  uint32_t r;
  if (bf) {
    asm("cvt.rn.bf16x2.f32 %0, %1, %2;" : "=r"(r) : "f"(b), "f"(a));       // {hi, lo} = {b, a}
  } else {
    __half2 h = __floats2half2_rn(a, b);
    r = *reinterpret_cast<uint32_t*>(&h);
  }
  return r;
}
__device__ __forceinline__ float2 unpack2(uint32_t u, bool bf) {
  if (bf) return make_float2(__uint_as_float(u << 16), __uint_as_float(u & 0xffff0000u));
  return __half22float2(*reinterpret_cast<__half2*>(&u));
}
__device__ __forceinline__ float ld16(const __half* p, bool bf) {
  const unsigned short u = *reinterpret_cast<const unsigned short*>(p);
  return bf ? __uint_as_float(static_cast<uint32_t>(u) << 16) : __half2float(*p);
}
__device__ __forceinline__ void st16(__half* p, float v, bool bf) {
  if (bf) *reinterpret_cast<unsigned short*>(p) = static_cast<unsigned short>(pack2(v, 0.f, true) & 0xffffu);
  else *p = __float2half_rn(v);
}

__device__ __forceinline__ uint32_t pack_half2(float a, float b) {
  __half2 h = __floats2half2_rn(a, b);
  return *reinterpret_cast<uint32_t*>(&h);
}
__device__ __forceinline__ float2 unpack_half2(uint32_t u) {
  return __half22float2(*reinterpret_cast<__half2*>(&u));
}


// ---------------------------------------------------------------------------------
// Programmatic dependent launch.  A kernel launched through launch_pdl() may be scheduled while its
// predecessor in the stream is still draining: its CTAs take the SMs the predecessor's CTAs leave, run
// whatever precedes pdl_sync() (nothing that touches global memory) and block there until the predecessor
// has completed and its writes are visible.  EVERY kernel launched this way must call pdl_sync() before its
// first global access; called from a kernel launched with plain stream ordering it is a no-op.
// NOPE_PDL (bit mask, see pdl_mask) switches the attribute off for A/B measurements.
// ---------------------------------------------------------------------------------
__device__ __forceinline__ void pdl_sync() {
  asm volatile("griddepcontrol.wait;" ::: "memory");
  asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
}
// NOPE_PDL: bit 0 = the convolution kernels, bit 1 = every other kernel of the chain (default 3)
inline int pdl_mask() {
  static const int m = [] {
    const char* e = getenv("NOPE_PDL");
    return e ? atoi(e) : 3;
  }();
  return m;
}
template <typename... KArgs, typename... Args>
inline cudaError_t launch_pdl(void (*kern)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t st,
                              Args&&... args) {
  cudaLaunchConfig_t cfg;
  memset(&cfg, 0, sizeof cfg);
  cfg.gridDim = grid;
  cfg.blockDim = block;
  cfg.dynamicSmemBytes = smem;
  cfg.stream = st;
  cudaLaunchAttribute at;
  at.id = cudaLaunchAttributeProgrammaticStreamSerialization;
  at.val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = &at;
  cfg.numAttrs = (pdl_mask() & 2) ? 1 : 0;
  return cudaLaunchKernelEx(&cfg, kern, static_cast<KArgs>(args)...);
}

}  // namespace nope
