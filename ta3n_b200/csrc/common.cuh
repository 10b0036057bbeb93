// common.cuh -- error plumbing, launch accounting and small device helpers shared by every
// translation unit of libta3n_sm90.so.
#pragma once

#include <cuda_runtime.h>
#include <stdarg.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <atomic>
#include <mutex>
#include <string>
#include <vector>

#include "../../include/ta3n_b200.h"

namespace ta3n {

// ---- error state ---------------------------------------------------------------------------
inline char* last_error_buf() {
  static thread_local char buf[512] = {0};
  return buf;
}

inline int fail(int code, const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(last_error_buf(), 512, fmt, ap);
  va_end(ap);
  return code;
}

#define TA3N_REQUIRE(cond, msg)                                                         \
  do {                                                                                   \
    if (!(cond)) return ::ta3n::fail(TA3N_ERR_INVALID, "%s: requirement failed: " msg " (line %d)", \
                                     __func__, (int)__LINE__);                           \
  } while (0)

#define TA3N_CUDA(expr)                                                                  \
  do {                                                                                   \
    cudaError_t _e = (expr);                                                             \
    if (_e != cudaSuccess)                                                               \
      return ::ta3n::fail(TA3N_ERR_CUDA, "CUDA error %s at line %d", cudaGetErrorString(_e), \
                          (int)__LINE__);                                                \
  } while (0)

#define TA3N_TRY(expr)                 \
  do {                                 \
    int _rc = (expr);                  \
    if (_rc != TA3N_OK) return _rc;    \
  } while (0)

// ---- launch accounting (bench.py reports gpu_launches from this) ----------------------------
inline std::atomic<uint64_t>& launch_counter() {
  static std::atomic<uint64_t> n{0};
  return n;
}

// ---- optional per-launch timing (CUDA events on the launching stream; eager mode only) --------
// bench.py switches this on for a separate pass to attribute device time to each call site.
struct TimingRegistry {
  struct Rec {
    const char* label;
    cudaEvent_t a, b;
  };
  std::mutex mu;
  std::atomic<bool> enabled{false};
  std::vector<Rec> recs;
};
inline TimingRegistry& timing() {
  static TimingRegistry t;
  return t;
}
struct PendingTimer {
  bool active = false;
  cudaEvent_t stop = nullptr;
  cudaStream_t stream = nullptr;
};
inline PendingTimer& pending_timer() {
  static thread_local PendingTimer p;
  return p;
}

// call right before a kernel launch
inline void pre_launch(const char* label, cudaStream_t stream) {
  TimingRegistry& t = timing();
  if (!t.enabled.load(std::memory_order_relaxed)) return;
  static const bool log_launches = []() {      // TA3N_LAUNCH_LOG=1: call-site label of every launch, in order, on stderr
    const char* e = getenv("TA3N_LAUNCH_LOG");
    return e && e[0] == '1';
  }();
  if (log_launches) fprintf(stderr, "ta3n-launch %s\n", label);
  TimingRegistry::Rec r;
  r.label = label;
  if (cudaEventCreate(&r.a) != cudaSuccess || cudaEventCreate(&r.b) != cudaSuccess) return;
  cudaEventRecord(r.a, stream);
  {
    std::lock_guard<std::mutex> g(t.mu);
    t.recs.push_back(r);
  }
  PendingTimer& p = pending_timer();
  p.active = true;
  p.stop = r.b;
  p.stream = stream;
}

inline int after_launch() {
  launch_counter().fetch_add(1, std::memory_order_relaxed);
  PendingTimer& p = pending_timer();
  if (p.active) {
    cudaEventRecord(p.stop, p.stream);
    p.active = false;
  }
  cudaError_t e = cudaGetLastError();  // launch-configuration errors only; never synchronises
  if (e != cudaSuccess) return fail(TA3N_ERR_CUDA, "kernel launch failed: %s", cudaGetErrorString(e));
  return TA3N_OK;
}

inline std::atomic<int>& gemm_engine() {
  static std::atomic<int> e{TA3N_GEMM_TF32X3_TCGEN05};   // the product engine; 'fp32' is the exact parity engine
  return e;
}

// ---- kernel launch with programmatic dependent launch (PDL) ---------------------------------------
// Every kernel starts with pdl_wait() (griddepcontrol.wait: the previous kernel in the stream has completed
// and its writes are visible) after whatever set-up needs no device data, then allows ITS dependents to be
// scheduled.  With the launch attribute below, kernel k+1's CTAs are placed on idle SMs and run their
// prologue (parameter staging, barrier init) while kernel k is still computing -- the
// step is a chain of ~26 short, mostly sub-wave kernels, so launch latency and prologues are on the
// critical path.  TA3N_PDL=0 disables the attribute (the device-side instructions are then no-ops).
inline bool pdl_enabled() {
  static const bool on = []() {
    const char* e = getenv("TA3N_PDL");
    return !(e && e[0] == '0');
  }();
  return on;
}

template <typename... KArgs, typename... Args>
inline void launch_kernel(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t stream,
                          Args&&... args) {
  cudaLaunchConfig_t cfg;
  memset(&cfg, 0, sizeof(cfg));
  cfg.gridDim = grid;
  cfg.blockDim = block;
  cfg.dynamicSmemBytes = smem;
  cfg.stream = stream;
  cudaLaunchAttribute attr[1];
  if (pdl_enabled()) {
    attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = attr;
    cfg.numAttrs = 1;
  }
  cudaLaunchKernelEx(&cfg, kernel, static_cast<KArgs>(args)...);   // errors surface in after_launch()
}

// ---- workspace carving ----------------------------------------------------------------------
struct Arena {
  char* base;
  size_t size;
  size_t used;
  Arena(void* p, size_t n) : base(static_cast<char*>(p)), size(n), used(0) {}
  static size_t round(size_t n) { return (n + 255) & ~size_t(255); }
  // returns nullptr when exhausted (caller checks via ok())
  float* floats(size_t n) {
    size_t bytes = round(n * sizeof(float));
    if (base == nullptr || used + bytes > size) return nullptr;   // caller decides whether that is fatal
    float* p = reinterpret_cast<float*>(base + used);
    used += bytes;
    return p;
  }
  bool ok() const { return used <= size; }
};

// ---- device helpers -------------------------------------------------------------------------
#ifdef __CUDACC__
__device__ __forceinline__ void pdl_wait() {
  asm volatile("griddepcontrol.wait;" ::: "memory");
  asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
}
#endif
__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// Counter-based keep decision for dropout: a stateless 64-bit mix of (seed, step, element).
// Recomputable in backward from the same triple, so no mask has to be stored.
__device__ __forceinline__ uint64_t mix64(uint64_t z) {
  z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
  z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
  return z ^ (z >> 31);
}

// One 64-bit hash serves FOUR consecutive elements (idx >> 2), 16 bits each: the mixing is ~60 integer instructions,
// and evaluated per element it was the largest part of the shared layer's tile epilogue (4 us of 11).  The dropout
// probability is therefore quantised to 1/65536 (0.5 is exact).
__device__ __forceinline__ uint64_t rng_hash4(uint64_t seed, uint64_t step, uint64_t idx4) {
  return mix64(mix64(seed + 0x9E3779B97F4A7C15ull * (step + 1)) ^ (idx4 * 0xD6E8FEB86659FD93ull));
}
__device__ __forceinline__ uint32_t rng_threshold(float p) { return (uint32_t)(p * 65536.0f + 0.5f); }
__device__ __forceinline__ bool rng_keep_bits(uint64_t h, int lane4, uint32_t thr) {
  return (uint32_t)((h >> (16 * lane4)) & 0xFFFFu) >= thr;
}
__device__ __forceinline__ bool rng_keep(uint64_t seed, uint64_t step, uint64_t idx, float p) {
  return rng_keep_bits(rng_hash4(seed, step, idx >> 2), (int)(idx & 3u), rng_threshold(p));
}

// softmax over two logits -> q0,q1, entropy E and w = 1 - E   (models.py:351-357)
struct Attn2 {
  float q0, q1, lq0, lq1, ent, w;
};
__device__ __forceinline__ Attn2 attn_from_logits(float p0, float p1) {
  Attn2 a;
  float mx = fmaxf(p0, p1);
  float e0 = expf(p0 - mx), e1 = expf(p1 - mx);
  float s = e0 + e1;
  float ls = logf(s);
  a.lq0 = p0 - mx - ls;
  a.lq1 = p1 - mx - ls;
  a.q0 = e0 / s;
  a.q1 = e1 / s;
  a.ent = -(a.q0 * a.lq0 + a.q1 * a.lq1);
  a.w = 1.0f - a.ent;
  return a;
}

}  // namespace ta3n
