// Host-side plumbing shared by the library's translation units: the error status and text, the launch macro with its counter,
// per-kernel profile and debug aids, and the per-device kernel configuration.  Internal: not part of the C ABI.
#pragma once
#include "../../include/pf_b200.h"

#include <cuda_runtime.h>
#include <nvtx3/nvToolsExt.h>

#include <atomic>
#include <cstdlib>
#include <vector>

namespace pf {

// ----------------------------------------------------------------------------------------------- errors
// Records the message that pf_last_error returns (per thread) and returns code.
int fail(int code, const char* fmt, ...);
extern std::atomic<long long> g_launches;   // pf_kernel_launch_count
#define CU(expr)                                                                                    \
  do {                                                                                              \
    cudaError_t e__ = (expr);                                                                       \
    if (e__ != cudaSuccess) return pf::fail(PF_ERR_CUDA, "%s: %s (%s:%d)", #expr, cudaGetErrorString(e__), __FILE__, __LINE__); \
  } while (0)
// PF_SYNC_DEBUG=1 in the environment: synchronise after every launch so that a device fault is reported at the launch that
// caused it (debugging aid; never set in production)
extern char g_crumb[96];   // name of the last debug tap taken (breadcrumb for the error text)
inline bool sync_debug() {
  static int v = -1;
  if (v < 0) v = getenv("PF_SYNC_DEBUG") ? 1 : 0;
  return v == 1;
}
// pf_profile_kernels_*: a CUDA-event pair around EVERY launch of the forward graph (in-pipeline time per kernel, bench.py's
// "per_kernel" table).  Off by default: the event records cost a few percent, so bench.py uses a separate pass for it.
// The state lives in the engine; the launch macro reaches it through a thread-local pointer that pf_forward sets for the
// duration of the call (operator entry points run with it unset).
struct KernelProf {
  bool on = false;
  cudaStream_t st = nullptr;
  std::vector<cudaEvent_t> pool;
  size_t used = 0;
  struct Rec { const char* expr; cudaEvent_t a, b; };
  std::vector<Rec> recs;
  cudaEvent_t next() { return used < pool.size() ? pool[used++] : nullptr; }
};
extern thread_local KernelProf* tl_kp;
#define LAUNCHED(expr)                                                                              \
  do {                                                                                              \
    pf::KernelProf* kp__ = pf::tl_kp;                                                               \
    cudaEvent_t ka__ = (kp__ && kp__->on) ? kp__->next() : nullptr;                                 \
    if (ka__) cudaEventRecord(ka__, kp__->st);                                                      \
    cudaError_t e__ = (expr);                                                                       \
    pf::g_launches.fetch_add(1, std::memory_order_relaxed);                                         \
    if (ka__) {                                                                                     \
      cudaEvent_t kb__ = kp__->next();                                                              \
      if (kb__) { cudaEventRecord(kb__, kp__->st); kp__->recs.push_back({#expr, ka__, kb__}); }     \
    }                                                                                               \
    if (e__ == cudaSuccess && pf::sync_debug()) e__ = cudaDeviceSynchronize();                      \
    if (e__ != cudaSuccess) return pf::fail(PF_ERR_CUDA, "%s: %s (%s:%d, after tap '%s')", #expr, cudaGetErrorString(e__), __FILE__, __LINE__, pf::g_crumb); \
  } while (0)
// NVTX range per section of the forward graph (visible in Nsight Systems / ncu --nvtx; a few ns when no tool is attached)
struct NvtxRange {
  explicit NvtxRange(const char* name) { nvtxRangePushA(name); }
  ~NvtxRange() { nvtxRangePop(); }
};
#define TRY(expr)                \
  do {                           \
    int r__ = (expr);            \
    if (r__ != PF_OK) return r__; \
  } while (0)

// The opt-in for more than 48 KB of dynamic shared memory is a per-device attribute of each kernel: set for every kernel of the
// library on every device an engine (or an operator entry point) uses, once per device and thread-safe.
int configure_device(int device);
int configure_current_device();

}  // namespace pf
