// Shared host/device helpers for libyolact_b200.so (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <cuda_bf16.h>
#include <stdint.h>
#include <stdio.h>
#include <stdarg.h>
#include <atomic>

#include "../../include/yolact_b200.h"

namespace yb {

// ---- error plumbing -------------------------------------------------------------------------
void set_error(const char* fmt, ...);
extern std::atomic<uint64_t> g_launches;
inline void count_launch(uint64_t n = 1) { g_launches.fetch_add(n, std::memory_order_relaxed); }

#define YB_CHECK_CUDA(expr)                                                                  \
  do {                                                                                       \
    cudaError_t _e = (expr);                                                                 \
    if (_e != cudaSuccess) {                                                                 \
      ::yb::set_error("%s:%d: %s failed: %s", __FILE__, __LINE__, #expr, cudaGetErrorString(_e)); \
      return YB_ERR_CUDA;                                                                    \
    }                                                                                        \
  } while (0)

#define YB_REQUIRE(cond, code, ...)                                                          \
  do {                                                                                       \
    if (!(cond)) {                                                                           \
      ::yb::set_error(__VA_ARGS__);                                                          \
      return (code);                                                                         \
    }                                                                                        \
  } while (0)

#define YB_CHECK_LAUNCH()                                                                    \
  do {                                                                                       \
    ::yb::count_launch();                                                                    \
    cudaError_t _e = cudaGetLastError();                                                     \
    if (_e != cudaSuccess) {                                                                 \
      ::yb::set_error("%s:%d: kernel launch failed: %s", __FILE__, __LINE__, cudaGetErrorString(_e)); \
      return YB_ERR_CUDA;                                                                    \
    }                                                                                        \
  } while (0)

#define YB_PROPAGATE(expr)                                                                   \
  do {                                                                                       \
    int _s = (expr);                                                                         \
    if (_s != YB_OK) return _s;                                                              \
  } while (0)

// SMs of an H100 SXM: sizes the grids of the grid-stride utility kernels (any grid size is correct)
constexpr int kSmCount = 132;

static inline size_t align_up(size_t x, size_t a) { return (x + a - 1) / a * a; }
static inline int ceil_div(int a, int b) { return (a + b - 1) / b; }

// ---- page-locked staging of host tables --------------------------------------------------------
// Copies host tables into device memory on `st` through a small ring of library-owned page-locked slots.  A copy from
// pageable memory may wait for the work already queued on the stream; from page-locked memory it is queued like a kernel,
// so a caller can submit batches ahead of the device.  A slot is reused only after the copy that last read it has run, so
// the host blocks only when it is a whole ring of calls ahead of the stream.  The caller's tables may be freed on return.
// Part i is written at byte parts[i].offset of the `bytes` copied to device_dst.
struct StagePart {
  const void* src;
  size_t bytes;
  size_t offset;
};
int stage_tables(void* device_dst, size_t bytes, const StagePart* parts, int n_parts, cudaStream_t st);

// ---- device helpers --------------------------------------------------------------------------
#ifdef __CUDACC__
__device__ __forceinline__ uint32_t float_to_ordered(float f) {
  // monotone map float -> uint32 (ascending); -0 canonicalised to +0
  f = f + 0.0f;
  uint32_t u = __float_as_uint(f);
  return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
__device__ __forceinline__ float ordered_to_float(uint32_t u) {
  return __uint_as_float((u & 0x80000000u) ? (u & 0x7fffffffu) : ~u);
}
// epilogue activation: 0 none, 1 ReLU, 2 exact GELU (torch.nn.GELU default: 0.5 x (1 + erf(x / sqrt 2)))
__device__ __forceinline__ float apply_act(float v, int act) {
  if (act == 1) return fmaxf(v, 0.f);
  if (act == 2) return 0.5f * v * (1.f + erff(v * 0.70710678118654752f));
  return v;
}
__device__ __forceinline__ int lane_id() { return threadIdx.x & 31; }
__device__ __forceinline__ int warp_id() { return threadIdx.x >> 5; }
#endif

}  // namespace yb
