// Error plumbing, version and device queries for libyolact_b200.so.
#include "common.cuh"
#include <string.h>
#include <mutex>

namespace yb {
static thread_local char g_err[512] = "";
std::atomic<uint64_t> g_launches{0};

void set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}

namespace {
struct StagingSlot {
  void* host = nullptr;
  size_t cap = 0;
  cudaEvent_t done = nullptr;
  int device = -1;
};
constexpr int kStagingSlots = 4;
std::mutex g_staging_mu;
StagingSlot g_staging[kStagingSlots];
int g_staging_next = 0;
}  // namespace

int stage_tables(void* device_dst, size_t bytes, const StagePart* parts, int n_parts, cudaStream_t st) {
  if (bytes == 0) return YB_OK;
  int device = 0;
  YB_CHECK_CUDA(cudaGetDevice(&device));
  std::lock_guard<std::mutex> lock(g_staging_mu);
  StagingSlot& s = g_staging[g_staging_next];
  g_staging_next = (g_staging_next + 1) % kStagingSlots;
  if (s.done) {
    YB_CHECK_CUDA(cudaEventSynchronize(s.done));
    if (s.device != device) {
      YB_CHECK_CUDA(cudaEventDestroy(s.done));
      s.done = nullptr;
    }
  }
  if (!s.done) {
    YB_CHECK_CUDA(cudaEventCreateWithFlags(&s.done, cudaEventDisableTiming));
    s.device = device;
  }
  if (s.cap < bytes) {
    if (s.host) YB_CHECK_CUDA(cudaFreeHost(s.host));
    s.host = nullptr;
    s.cap = 0;
    YB_CHECK_CUDA(cudaHostAlloc(&s.host, bytes, cudaHostAllocPortable));
    s.cap = bytes;
  }
  for (int i = 0; i < n_parts; ++i)
    if (parts[i].bytes) memcpy((char*)s.host + parts[i].offset, parts[i].src, parts[i].bytes);
  YB_CHECK_CUDA(cudaMemcpyAsync(device_dst, s.host, bytes, cudaMemcpyHostToDevice, st));
  YB_CHECK_CUDA(cudaEventRecord(s.done, st));
  return YB_OK;
}
}  // namespace yb

extern "C" int yb_version(void) { return YB_VERSION; }
extern "C" const char* yb_last_error(void) { return yb::g_err; }
extern "C" uint64_t yb_launch_count(void) { return yb::g_launches.load(); }

extern "C" int yb_device_info(int* sm_count, int* cc_major, int* cc_minor) {
  int dev = 0;
  YB_CHECK_CUDA(cudaGetDevice(&dev));
  cudaDeviceProp prop;
  YB_CHECK_CUDA(cudaGetDeviceProperties(&prop, dev));
  if (sm_count) *sm_count = prop.multiProcessorCount;
  if (cc_major) *cc_major = prop.major;
  if (cc_minor) *cc_minor = prop.minor;
  return YB_OK;
}
