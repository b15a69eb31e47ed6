// Mask output stage on the GPU (SURVEY.md 8(f) rank 2): what follows after_nms in the reference's evaluation loop --
//   bit-packed masks        1 bit / pixel instead of the reference's float32 {0,1} (utils/output_utils.py:222-231: 123 MB / image
//                           at 100 x 480 x 640 fp32 -> 3.8 MB), written directly by the mask assembly (masks.cu, mask_format 2)
//   mask_iou / box_iou      utils/box_utils.py:189-200 / :8-37 as used by prep_metrics (utils/common_utils.py:174-183): pairwise
//                           IoU of prediction and ground-truth masks by AND + popcount over the packed words
//   RLE                     the run lengths pycocotools.mask.encode produces from np.asfortranarray(mask) (utils/common_utils.py:88-96):
//                           column-major runs starting with a run of zeros; the ASCII compression of the counts is host work
// All HBM-bound streaming kernels: every packed word is read once per use.
#include "common.cuh"
#include "iou.cuh"

#include <stdint.h>

namespace yb {

// ---- pack {0,1} masks (uint8 or float32, [n][h][w]) into row-major bit words [n][h][ceil(w/32)], bit (x & 31) of word x >> 5 ----
template <typename T>
__global__ void __launch_bounds__(256) k_pack_bits(const T* __restrict__ m, int h, int w, int words, uint32_t* __restrict__ out) {
  const int wi = blockIdx.x * 256 + threadIdx.x, y = blockIdx.y, n = blockIdx.z;
  if (wi >= words) return;
  const T* row = m + ((size_t)n * h + y) * w + wi * 32;
  uint32_t v = 0;
  const int cnt = min(32, w - wi * 32);
  for (int b = 0; b < cnt; ++b) v |= (row[b] > (T)0.5f ? 1u : 0u) << b;
  out[((size_t)n * h + y) * words + wi] = v;
}

// ---- pairwise mask IoU: out[i][j] = |a_i & b_j| / (|a_i| + |b_j| - |a_i & b_j|), the reference's float division (NaN for 0/0) ----
__global__ void __launch_bounds__(256) k_mask_iou_bits(const uint32_t* __restrict__ a, const uint32_t* __restrict__ b, int m, long long words,
                                                       float* __restrict__ out) {
  const int i = blockIdx.y, j = blockIdx.x;
  const uint32_t* pa = a + (size_t)i * words;
  const uint32_t* pb = b + (size_t)j * words;
  unsigned inter = 0, ca = 0, cb = 0;
  for (long long k = threadIdx.x; k < words; k += 256) {
    mask_counts_add(pa[k], pb[k], inter, ca, cb);
  }
  __shared__ unsigned s[3][256];
  s[0][threadIdx.x] = inter; s[1][threadIdx.x] = ca; s[2][threadIdx.x] = cb;
  __syncthreads();
  for (int off = 128; off > 0; off >>= 1) {
    if (threadIdx.x < off) { s[0][threadIdx.x] += s[0][threadIdx.x + off]; s[1][threadIdx.x] += s[1][threadIdx.x + off]; s[2][threadIdx.x] += s[2][threadIdx.x + off]; }
    __syncthreads();
  }
  if (threadIdx.x == 0) out[(size_t)i * m + j] = mask_iou_from_counts(s[0][0], s[1][0], s[2][0]);
}

// ---- pairwise box IoU (utils/box_utils.py:8-37, separately rounded operations) ----
__global__ void k_box_iou(const float* __restrict__ a, int n, const float* __restrict__ b, int m, float* __restrict__ out) {
  const int t = blockIdx.x * 256 + threadIdx.x;
  if (t >= n * m) return;
  const int i = t / m, j = t - i * m;
  out[t] = box_iou_rn(reinterpret_cast<const float4*>(a)[i], reinterpret_cast<const float4*>(b)[j]);
}

// ---- COCO run-length encoding of packed masks: column-major scan (x outer, y inner), first run counts zeros ----
// One block per mask.  Pass 1 counts the value changes inside every column (a change at position p starts a new run), a block
// scan turns them into offsets, pass 2 writes the start positions, pass 3 turns starts into lengths in place.
constexpr int kRleMaxW = 4096;

__device__ __forceinline__ uint32_t bit_at(const uint32_t* __restrict__ m, int words, int y, int x) { return (m[(size_t)y * words + (x >> 5)] >> (x & 31)) & 1u; }

__global__ void __launch_bounds__(256) k_mask_rle(const uint32_t* __restrict__ bits, int h, int w, int words, uint32_t* __restrict__ counts, int max_runs,
                                                  int32_t* __restrict__ nruns) {
  __shared__ int col[kRleMaxW + 1];
  __shared__ int part[257];
  const int n = blockIdx.x;
  const uint32_t* m = bits + (size_t)n * h * words;
  uint32_t* out = counts + (size_t)n * max_runs;
  for (int x = threadIdx.x; x < w; x += 256) {
    uint32_t prev = x == 0 ? 0u : bit_at(m, words, h - 1, x - 1);
    int c = 0;
    for (int y = 0; y < h; ++y) { const uint32_t v = bit_at(m, words, y, x); c += v != prev; prev = v; }
    col[x] = c;
  }
  __syncthreads();
  // exclusive scan over columns: per-thread chunks, then the 256 partial sums
  const int per = (w + 255) / 256, x0 = threadIdx.x * per, x1 = min(x0 + per, w);
  int sum = 0;
  for (int x = x0; x < x1; ++x) sum += col[x];
  part[threadIdx.x] = sum;
  __syncthreads();
  if (threadIdx.x == 0) { int acc = 0; for (int i = 0; i < 256; ++i) { const int v = part[i]; part[i] = acc; acc += v; } part[256] = acc; }
  __syncthreads();
  int acc = part[threadIdx.x];
  for (int x = x0; x < x1; ++x) { const int v = col[x]; col[x] = acc; acc += v; }
  __syncthreads();
  const int total = part[256] + 1;                                   // runs = changes + 1 (the leading run of zeros may be empty)
  if (threadIdx.x == 0) nruns[n] = total <= max_runs ? total : -total;
  if (total > max_runs) return;
  // pass 2: start positions; out[i] (i >= 1) = position of the i-th change
  for (int x = threadIdx.x; x < w; x += 256) {
    uint32_t prev = x == 0 ? 0u : bit_at(m, words, h - 1, x - 1);
    int idx = col[x] + 1;
    for (int y = 0; y < h; ++y) { const uint32_t v = bit_at(m, words, y, x); if (v != prev) out[idx++] = (uint32_t)(x * h + y); prev = v; }
  }
  if (threadIdx.x == 0) out[0] = 0;
  __syncthreads();
  // pass 3: lengths, chunk by chunk in increasing order (a chunk reads its starts and the next one's first before anything is overwritten)
  const uint32_t hw = (uint32_t)h * (uint32_t)w;
  for (int base = 0; base < total; base += 256) {
    const int i = base + threadIdx.x;
    uint32_t s0 = 0, s1 = 0;
    if (i < total) { s0 = out[i]; s1 = i + 1 < total ? out[i + 1] : hw; }
    __syncthreads();
    if (i < total) out[i] = s1 - s0;
    __syncthreads();
  }
}

}  // namespace yb

using namespace yb;

extern "C" int yb_pack_mask_bits(const void* masks, int is_f32, int n, int h, int w, uint32_t* out, void* stream) {
  YB_REQUIRE(n >= 0 && h > 0 && w > 0, YB_ERR_INVALID, "yb_pack_mask_bits: n=%d h=%d w=%d", n, h, w);
  if (n == 0) return YB_OK;
  YB_REQUIRE(masks && out, YB_ERR_INVALID, "yb_pack_mask_bits: NULL argument");
  YB_REQUIRE(n <= 65535 && h <= 65535, YB_ERR_UNSUPPORTED, "yb_pack_mask_bits: n/h exceed grid limits");
  const int words = (w + 31) / 32;
  dim3 grid(ceil_div(words, 256), h, n);
  if (is_f32) k_pack_bits<float><<<grid, 256, 0, (cudaStream_t)stream>>>((const float*)masks, h, w, words, out);
  else k_pack_bits<uint8_t><<<grid, 256, 0, (cudaStream_t)stream>>>((const uint8_t*)masks, h, w, words, out);
  YB_CHECK_LAUNCH();
  return YB_OK;
}

extern "C" int yb_mask_iou_bits(const uint32_t* a, int n, const uint32_t* b, int m, int64_t words, float* out, void* stream) {
  YB_REQUIRE(n >= 0 && m >= 0 && words > 0, YB_ERR_INVALID, "yb_mask_iou_bits: n=%d m=%d", n, m);
  if (n == 0 || m == 0) return YB_OK;
  YB_REQUIRE(a && b && out, YB_ERR_INVALID, "yb_mask_iou_bits: NULL argument");
  YB_REQUIRE(n <= 65535, YB_ERR_UNSUPPORTED, "yb_mask_iou_bits: n=%d", n);
  k_mask_iou_bits<<<dim3(m, n), 256, 0, (cudaStream_t)stream>>>(a, b, m, words, out);
  YB_CHECK_LAUNCH();
  return YB_OK;
}

extern "C" int yb_box_iou(const float* a, int n, const float* b, int m, float* out, void* stream) {
  YB_REQUIRE(n >= 0 && m >= 0, YB_ERR_INVALID, "yb_box_iou: n=%d m=%d", n, m);
  if (n == 0 || m == 0) return YB_OK;
  YB_REQUIRE(a && b && out, YB_ERR_INVALID, "yb_box_iou: NULL argument");
  k_box_iou<<<ceil_div(n * m, 256), 256, 0, (cudaStream_t)stream>>>(a, n, b, m, out);
  YB_CHECK_LAUNCH();
  return YB_OK;
}

extern "C" int yb_mask_rle(const uint32_t* bits, int n, int h, int w, uint32_t* counts, int max_runs, int32_t* nruns, void* stream) {
  YB_REQUIRE(n >= 0 && h > 0 && w > 0 && max_runs >= 2, YB_ERR_INVALID, "yb_mask_rle: n=%d h=%d w=%d max_runs=%d", n, h, w, max_runs);
  if (n == 0) return YB_OK;
  YB_REQUIRE(bits && counts && nruns, YB_ERR_INVALID, "yb_mask_rle: NULL argument");
  YB_REQUIRE(w <= kRleMaxW, YB_ERR_UNSUPPORTED, "yb_mask_rle: width %d > %d", w, kRleMaxW);
  k_mask_rle<<<n, 256, 0, (cudaStream_t)stream>>>(bits, h, w, (w + 31) / 32, counts, max_runs, nruns);
  YB_CHECK_LAUNCH();
  return YB_OK;
}
