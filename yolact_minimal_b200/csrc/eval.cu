// Evaluation stage: box and mask mAP on the GPU (utils/common_utils.py:107-255, driven by eval.py:35-69,:106).
//   k_eval_match  one block per image: same-class IoUs (iou.cuh, the arithmetic of k_box_iou / k_mask_iou_bits), then one warp
//                 per (IoU type, threshold) runs prep_metrics' greedy loop in detection order and sets the detection's tp bit;
//                 the image's records are appended at (running count + prefix of earlier images' counts)
//   k_eval_keys   (class, descending score) sort keys of the records; CUB's stable radix sort keeps record order on ties
//   k_eval_ap     one block per (type, threshold, class): APDataObject.get_ap in float64
// Exactness: every IoU is the reference's fp32 value; the threshold test is in double (iou.item() > x / 100); precision and
// recall are the same double divisions; the 101 samples are summed in the reference's order with the compensation of Python's
// sum() (CPython >= 3.12).
#include "common.cuh"
#include "iou.cuh"

#include <cub/device/device_radix_sort.cuh>
#include <stdint.h>

#include <algorithm>

namespace yb {

constexpr int kMatchThreads = 512;   // 16 warps; warp w runs the (type, threshold) slots w and w + 16
constexpr int kMaxDet = 256;         // yb_detect's max_det limit
constexpr int kApThreads = 256;
constexpr int kApBars = 101;         // recall samples 0.00, 0.01, ..., 1.00

struct EvalState {
  unsigned long long nrec;           // records appended so far
  unsigned int ticket;               // blocks of the current k_eval_match launch that are done (reset by the last one)
  unsigned int flags;                // 1: capacity exceeded, 2: an image's ranges lie outside the buffers
  // followed by num_gt[num_classes], seen[num_classes] (uint32)
};

__host__ __device__ inline unsigned* state_num_gt(void* s) { return reinterpret_cast<unsigned*>(reinterpret_cast<char*>(s) + sizeof(EvalState)); }
__host__ __device__ inline unsigned* state_seen(void* s, int C) { return state_num_gt(s) + C; }

struct MatchArgs {
  yb_eval_params p;
  int batch, max_det;
  const int32_t* count; const int32_t* cls; const float* score; const int32_t* box_px;
  const uint32_t* det_masks; const int64_t* det_mask_off; long long det_mask_words;
  const int32_t* img_hw;
  const float* gt; const int32_t* gt_offset; long long total_gt;
  const uint32_t* gt_masks; const int64_t* gt_mask_off; long long gt_mask_words;
  float* rec_score; int32_t* rec_cls; uint32_t* rec_tp; long long capacity;
  EvalState* state;
  float* iou_box; float* iou_mask;   // [max_det * total_gt]: image b's [n][g] matrix at max_det * gt_offset[b]
  uint32_t* used;                    // [total_gt]: bit s = gt already matched in slot s
};

__device__ __forceinline__ int clamp_count(int c, int D) { return c < 0 ? 0 : (c > D ? D : c); }
__device__ __forceinline__ int gt_class(const float* gt, long long r) { return __float2int_rz(__ldg(gt + r * 5 + 4)); }   // gt[:, 4].int()

__device__ long long block_sum_ll(long long v, long long* red) {
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  if (lane_id() == 0) red[warp_id()] = v;
  __syncthreads();
  long long s = 0;
  for (int i = 0; i < (int)(blockDim.x >> 5); ++i) s += red[i];
  __syncthreads();
  return s;
}

__global__ void __launch_bounds__(kMatchThreads) k_eval_match(const MatchArgs a) {
  __shared__ uint32_t tp[kMaxDet];
  __shared__ long long red[kMatchThreads / 32];
  __shared__ unsigned long long s_base;
  const int b = blockIdx.x, D = a.max_det, C = a.p.num_classes, T = a.p.num_thr;
  if (threadIdx.x == 0) s_base = *reinterpret_cast<volatile unsigned long long*>(&a.state->nrec);
  long long pre = 0;
  for (int j = threadIdx.x; j < b; j += kMatchThreads) pre += clamp_count(a.count[j], D);
  pre = block_sum_ll(pre, red);                                   // also publishes s_base
  const long long base = (long long)s_base + pre;
  const int n = clamp_count(a.count[b], D);
  unsigned* num_gt = state_num_gt(a.state);
  unsigned* seen = state_seen(a.state, C);

  if (n > 0) {
    const long long g0 = a.gt_offset[b], g1 = a.gt_offset[b + 1];
    const int h = a.img_hw[2 * b], w = a.img_hw[2 * b + 1];
    const long long words = (long long)h * ((w + 31) >> 5);
    const long long doff = a.det_mask_off[b], dend = a.det_mask_off[b + 1], goff = a.gt_mask_off[b], gend = a.gt_mask_off[b + 1];
    // the image's masks must have its geometry: at least count[b] detection masks and exactly one mask per gt row
    const bool ok = h > 0 && w > 0 && 0 <= g0 && g0 <= g1 && g1 <= a.total_gt && 0 <= doff && doff <= dend && dend <= a.det_mask_words &&
                    n * words <= dend - doff && 0 <= goff && goff <= gend && gend <= a.gt_mask_words && (g1 - g0) * words == gend - goff;
    const int g = ok ? (int)(g1 - g0) : 0;
    if (!ok && threadIdx.x == 0) atomicOr(&a.state->flags, 2u);
    for (int i = threadIdx.x; i < n; i += kMatchThreads) tp[i] = 0;
    if (ok) {
      for (int j = threadIdx.x; j < g; j += kMatchThreads) {
        a.used[g0 + j] = 0;
        const int c = gt_class(a.gt, g0 + j);
        if (c >= 0 && c < C) { atomicAdd(&num_gt[c], 1u); seen[c] = 1u; }
      }
      for (int i = threadIdx.x; i < n; i += kMatchThreads) {
        const int c = a.cls[(long long)b * D + i];
        if (c >= 0 && c < C) seen[c] = 1u;
      }
      // ---- IoUs of the same-class pairs, one warp per pair ----
      const uint32_t* dm = a.det_masks + doff;
      const uint32_t* gm = a.gt_masks + goff;
      float* ib = a.iou_box + (long long)D * g0;
      float* im = a.iou_mask + (long long)D * g0;
      const float fw = (float)w, fh = (float)h;
      for (int pair = warp_id(); pair < n * g; pair += kMatchThreads / 32) {
        const int i = pair / g, j = pair - i * g;
        if (a.cls[(long long)b * D + i] != gt_class(a.gt, g0 + j)) continue;
        const uint32_t* pa = dm + i * words;
        const uint32_t* pb = gm + j * words;
        unsigned inter = 0, ca = 0, cb = 0;
        for (long long k = lane_id(); k < words; k += 32) mask_counts_add(__ldg(pa + k), __ldg(pb + k), inter, ca, cb);
        for (int o = 16; o > 0; o >>= 1) {
          inter += __shfl_xor_sync(0xffffffffu, inter, o);
          ca += __shfl_xor_sync(0xffffffffu, ca, o);
          cb += __shfl_xor_sync(0xffffffffu, cb, o);
        }
        if (lane_id() == 0) {
          const int32_t* bp = a.box_px + ((long long)b * D + i) * 4;
          const float* gr = a.gt + (g0 + j) * 5;
          // prep_metrics: gt x scaled by width, y by height in fp32 (:175-177); the int pixel boxes converted to float (:183)
          const float4 p = make_float4((float)bp[0], (float)bp[1], (float)bp[2], (float)bp[3]);
          const float4 q = make_float4(__fmul_rn(gr[0], fw), __fmul_rn(gr[1], fh), __fmul_rn(gr[2], fw), __fmul_rn(gr[3], fh));
          ib[i * g + j] = box_iou_rn(p, q);
          im[i * g + j] = mask_iou_from_counts(inter, ca, cb);
        }
      }
    }
    __syncthreads();
    // ---- greedy matching (common_utils.py:185-216): warp per (type, threshold) slot, detections in order ----
    if (ok) {
      const uint32_t* used = a.used + g0;
      for (int s = warp_id(); s < 2 * T; s += kMatchThreads / 32) {
        const double thr = a.p.thr[s % T];
        const float* iou = (s < T ? a.iou_box : a.iou_mask) + (long long)D * g0;
        for (int i = 0; i < n; ++i) {
          const int ci = a.cls[(long long)b * D + i];
          if (ci < 0 || ci >= C) continue;                        // uniform across the warp
          float bv = 0.f;
          int bj = -1;
          for (int j = lane_id(); j < g; j += 32) {   // increasing j per lane: the strict > keeps the earliest of equal IoUs
            if (gt_class(a.gt, g0 + j) != ci || ((__ldcg(used + j) >> s) & 1u)) continue;
            const float v = iou[i * g + j];
            if ((double)v > thr && (bj < 0 || v > bv)) { bv = v; bj = j; }   // NaN fails the double comparison
          }
          for (int o = 16; o > 0; o >>= 1) {
            const float ov = __shfl_xor_sync(0xffffffffu, bv, o);
            const int oj = __shfl_xor_sync(0xffffffffu, bj, o);
            if (oj >= 0 && (bj < 0 || ov > bv || (ov == bv && oj < bj))) { bv = ov; bj = oj; }
          }
          if (lane_id() == 0 && bj >= 0) {
            atomicOr(a.used + g0 + bj, 1u << s);
            atomicOr(&tp[i], 1u << s);
          }
          __syncwarp();
        }
      }
    }
    __syncthreads();
    for (int i = threadIdx.x; i < n; i += kMatchThreads) {
      const long long r = base + i;
      if (r >= a.capacity) { atomicOr(&a.state->flags, 1u); continue; }
      const int c = a.cls[(long long)b * D + i];
      a.rec_score[r] = a.score[(long long)b * D + i];
      a.rec_cls[r] = ok && c >= 0 && c < C ? c : -1;
      a.rec_tp[r] = tp[i];
    }
  }
  // the last block to finish advances the record count (every block has read it by then)
  __syncthreads();
  if (threadIdx.x == 0) {
    __threadfence();
    if (atomicAdd(&a.state->ticket, 1u) == gridDim.x - 1) {
      long long total = 0;
      for (int j = 0; j < a.batch; ++j) total += clamp_count(a.count[j], D);
      a.state->nrec = s_base + (unsigned long long)total;
      a.state->ticket = 0;
      __threadfence();
    }
  }
}

// ---- sort keys: class in the high word, descending score below it; invalid / unused records sort last (class = C) ----
__global__ void k_eval_keys(const float* __restrict__ score, const int32_t* __restrict__ cls, const uint32_t* __restrict__ tp, long long n,
                            const EvalState* __restrict__ st, int C, unsigned long long* __restrict__ keys, uint32_t* __restrict__ vals) {
  const long long nrec = (long long)st->nrec;
  for (long long r = blockIdx.x * (long long)blockDim.x + threadIdx.x; r < n; r += (long long)gridDim.x * blockDim.x) {
    const int c = r < nrec ? cls[r] : -1;
    if (c >= 0 && c < C) {
      keys[r] = ((unsigned long long)c << 32) | (unsigned long long)(~float_to_ordered(score[r]));
      vals[r] = tp[r];
    } else {
      keys[r] = (unsigned long long)C << 32;
      vals[r] = 0;
    }
  }
}

__device__ long long lower_bound_u64(const unsigned long long* k, long long n, unsigned long long v) {
  long long lo = 0, hi = n;
  while (lo < hi) { const long long mid = (lo + hi) >> 1; if (k[mid] < v) lo = mid + 1; else hi = mid; }
  return lo;
}

// ---- APDataObject.get_ap (common_utils.py:123-171) for one (slot, class) ----
// With nt_k true positives among the first k+1 records, precision_k = nt_k / (k+1) and recall_k = nt_k / num_gt.  The sample at
// recall x/100 is searchsorted(recalls, x/100, 'left') = the position of the m(x)-th true positive, where m(x) is the least m with
// m / num_gt >= x/100 in double (position 0 when m(x) = 0; past the end, value 0, when m(x) exceeds the true positives).  The
// smoothed precision there is the max of precision over the suffix, and precision only rises at true positives, so it is the max
// of m / (pos_m + 1) over the true positives m >= m(x).  Each true positive m lands in bucket max{x : m(x) <= m}; a suffix max
// over the 101 buckets gives every sample.
__global__ void __launch_bounds__(kApThreads) k_eval_ap(const unsigned long long* __restrict__ keys, const uint32_t* __restrict__ vals,
                                                        long long n, const EvalState* __restrict__ st, int C, int T,
                                                        double* __restrict__ ap, uint8_t* __restrict__ nonempty) {
  __shared__ int mx[kApBars];
  __shared__ unsigned long long bmax[kApBars];
  __shared__ int wsum[kApThreads / 32];
  __shared__ long long seg[2];
  const int c = blockIdx.x, s = blockIdx.y;
  const unsigned* num_gt = state_num_gt(const_cast<EvalState*>(st));
  const unsigned ng = num_gt[c];
  if (s == 0 && threadIdx.x == 0) nonempty[c] = state_seen(const_cast<EvalState*>(st), C)[c] ? 1 : 0;
  double* out = ap + (size_t)s * C + c;
  if (ng == 0) { if (threadIdx.x == 0) *out = 0.0; return; }
  if (threadIdx.x < kApBars) {
    const int x = threadIdx.x;
    const double xd = (double)x / 100.0, g = (double)ng;
    long long m = (long long)ceil((double)x * g / 100.0);
    while (m > 0 && (double)(m - 1) / g >= xd) --m;
    while ((double)m / g < xd) ++m;
    mx[x] = (int)m;
    bmax[x] = 0ull;
  }
  if (threadIdx.x == 0) seg[0] = lower_bound_u64(keys, n, (unsigned long long)c << 32);
  if (threadIdx.x == 1) seg[1] = lower_bound_u64(keys, n, (unsigned long long)(c + 1) << 32);
  __syncthreads();
  const long long lo = seg[0], hi = seg[1];
  int carry = 0;
  for (long long k0 = lo; k0 < hi; k0 += kApThreads) {
    const long long k = k0 + threadIdx.x;
    const int t = k < hi ? (int)((vals[k] >> s) & 1u) : 0;
    int incl = t;                                                  // inclusive block scan of the tp flags
    for (int o = 1; o < 32; o <<= 1) { const int v = __shfl_up_sync(0xffffffffu, incl, o); if (lane_id() >= o) incl += v; }
    if (lane_id() == 31) wsum[warp_id()] = incl;
    __syncthreads();
    int wpre = 0, chunk = 0;
    for (int i = 0; i < kApThreads / 32; ++i) { if (i < warp_id()) wpre += wsum[i]; chunk += wsum[i]; }
    if (t) {
      const int m = carry + wpre + incl;                           // this record is the m-th true positive
      const double prec = (double)m / (double)(k - lo + 1);
      int l = 0, r = kApBars - 1;                                  // largest x with mx[x] <= m (mx[0] = 0)
      while (l < r) { const int mid = (l + r + 1) >> 1; if (mx[mid] <= m) l = mid; else r = mid - 1; }
      atomicMax(&bmax[l], (unsigned long long)__double_as_longlong(prec));   // non-negative doubles order like their bits
    }
    carry += chunk;
    __syncthreads();
  }
  if (threadIdx.x == 0) {
    double run = 0.0;
    for (int x = kApBars - 1; x >= 0; --x) {                       // bucket maxima -> the samples y(x), in place
      run = fmax(run, __longlong_as_double((long long)bmax[x]));
      bmax[x] = (unsigned long long)__double_as_longlong(mx[x] <= carry ? run : 0.0);
    }
    // sum(y_range) / len(y_range): Python's sum() of floats is Neumaier-compensated (CPython >= 3.12), in list order
    double sum = 0.0, comp = 0.0;
    for (int x = 0; x < kApBars; ++x) {
      const double v = __longlong_as_double((long long)bmax[x]);
      const double t = __dadd_rn(sum, v);
      comp = __dadd_rn(comp, fabs(sum) >= fabs(v) ? __dadd_rn(__dsub_rn(sum, t), v) : __dadd_rn(__dsub_rn(v, t), sum));
      sum = t;
    }
    if (comp != 0.0 && isfinite(comp)) sum = __dadd_rn(sum, comp);
    *out = __ddiv_rn(sum, (double)kApBars);
  }
}

static int key_end_bit(int C) {
  int bits = 0;
  while ((1u << bits) <= (unsigned)C) ++bits;                     // the sentinel class C must fit too
  return 32 + bits;
}

static size_t ap_sort_temp_bytes(long long n, int C) {
  size_t temp = 0;
  cub::DeviceRadixSort::SortPairs(nullptr, temp, (const unsigned long long*)nullptr, (unsigned long long*)nullptr,
                                  (const uint32_t*)nullptr, (uint32_t*)nullptr, (int)n, 0, key_end_bit(C));
  return temp;
}

static bool params_ok(const yb_eval_params* p) {
  return p && p->num_classes > 0 && p->num_thr >= 1 && p->num_thr <= YB_EVAL_MAX_THR;
}

}  // namespace yb

using namespace yb;

extern "C" size_t yb_eval_state_bytes(const yb_eval_params* p) {
  if (!params_ok(p)) return 0;
  return sizeof(EvalState) + 2 * sizeof(unsigned) * (size_t)p->num_classes;
}

extern "C" size_t yb_eval_match_workspace_bytes(int batch, int max_det, int64_t total_gt, const yb_eval_params* p) {
  if (!params_ok(p) || batch < 0 || max_det < 0 || total_gt < 0) return 0;
  const size_t iou = align_up(sizeof(float) * (size_t)max_det * (size_t)total_gt, 256);
  return 2 * iou + align_up(sizeof(uint32_t) * (size_t)total_gt, 256) + 256;
}

extern "C" size_t yb_eval_ap_workspace_bytes(int64_t num_records, const yb_eval_params* p) {
  if (!params_ok(p) || num_records < 0 || num_records > INT32_MAX) return 0;
  const size_t n = (size_t)num_records;
  return 2 * align_up(8 * n, 256) + 2 * align_up(4 * n, 256) + align_up(ap_sort_temp_bytes((long long)n, p->num_classes), 256) + 256;
}

extern "C" int yb_eval_match(const yb_eval_params* p, int batch, int max_det, const int32_t* count, const int32_t* cls, const float* score,
                             const int32_t* box_px, const uint32_t* det_masks, const int64_t* det_mask_off, int64_t det_mask_words,
                             const int32_t* img_hw, const float* gt, const int32_t* gt_offset, int64_t total_gt, const uint32_t* gt_masks,
                             const int64_t* gt_mask_off, int64_t gt_mask_words, float* rec_score, int32_t* rec_cls, uint32_t* rec_tp,
                             int64_t capacity, void* state, void* workspace, size_t workspace_bytes, void* stream) {
  YB_REQUIRE(p, YB_ERR_INVALID, "yb_eval_match: NULL params");
  YB_REQUIRE(p->num_thr >= 1 && p->num_thr <= YB_EVAL_MAX_THR, YB_ERR_UNSUPPORTED, "yb_eval_match: num_thr=%d (1..%d)", p->num_thr, YB_EVAL_MAX_THR);
  YB_REQUIRE(p->num_classes > 0, YB_ERR_INVALID, "yb_eval_match: num_classes=%d", p->num_classes);
  YB_REQUIRE(batch >= 0 && max_det >= 0 && total_gt >= 0 && capacity >= 0 && det_mask_words >= 0 && gt_mask_words >= 0, YB_ERR_INVALID,
             "yb_eval_match: negative size (batch=%d max_det=%d total_gt=%lld)", batch, max_det, (long long)total_gt);
  YB_REQUIRE(max_det <= kMaxDet, YB_ERR_UNSUPPORTED, "yb_eval_match: max_det=%d > %d", max_det, kMaxDet);
  if (batch == 0) return YB_OK;
  YB_REQUIRE(count && cls && score && box_px && det_mask_off && img_hw && gt_offset && gt_mask_off && rec_score && rec_cls && rec_tp && state &&
             workspace, YB_ERR_INVALID, "yb_eval_match: NULL argument");
  YB_REQUIRE((det_masks || det_mask_words == 0) && (gt_masks || gt_mask_words == 0) && (gt || total_gt == 0), YB_ERR_INVALID,
             "yb_eval_match: NULL mask / gt buffer");
  YB_REQUIRE(workspace_bytes >= yb_eval_match_workspace_bytes(batch, max_det, total_gt, p), YB_ERR_INVALID,
             "yb_eval_match: workspace %zu < %zu bytes", workspace_bytes, yb_eval_match_workspace_bytes(batch, max_det, total_gt, p));
  MatchArgs a;
  a.p = *p; a.batch = batch; a.max_det = max_det;
  a.count = count; a.cls = cls; a.score = score; a.box_px = box_px;
  a.det_masks = det_masks; a.det_mask_off = det_mask_off; a.det_mask_words = det_mask_words; a.img_hw = img_hw;
  a.gt = gt; a.gt_offset = gt_offset; a.total_gt = total_gt;
  a.gt_masks = gt_masks; a.gt_mask_off = gt_mask_off; a.gt_mask_words = gt_mask_words;
  a.rec_score = rec_score; a.rec_cls = rec_cls; a.rec_tp = rec_tp; a.capacity = capacity;
  a.state = reinterpret_cast<EvalState*>(state);
  char* ws = reinterpret_cast<char*>(align_up(reinterpret_cast<size_t>(workspace), 256));
  const size_t iou = align_up(sizeof(float) * (size_t)max_det * (size_t)total_gt, 256);
  a.iou_box = reinterpret_cast<float*>(ws);
  a.iou_mask = reinterpret_cast<float*>(ws + iou);
  a.used = reinterpret_cast<uint32_t*>(ws + 2 * iou);
  k_eval_match<<<batch, kMatchThreads, 0, (cudaStream_t)stream>>>(a);
  YB_CHECK_LAUNCH();
  return YB_OK;
}

extern "C" int yb_eval_ap(const yb_eval_params* p, const float* rec_score, const int32_t* rec_cls, const uint32_t* rec_tp, int64_t num_records,
                          const void* state, void* workspace, size_t workspace_bytes, double* ap, uint8_t* nonempty, void* stream) {
  YB_REQUIRE(p, YB_ERR_INVALID, "yb_eval_ap: NULL params");
  YB_REQUIRE(p->num_thr >= 1 && p->num_thr <= YB_EVAL_MAX_THR, YB_ERR_UNSUPPORTED, "yb_eval_ap: num_thr=%d (1..%d)", p->num_thr, YB_EVAL_MAX_THR);
  YB_REQUIRE(p->num_classes > 0, YB_ERR_INVALID, "yb_eval_ap: num_classes=%d", p->num_classes);
  YB_REQUIRE(num_records >= 0 && num_records <= INT32_MAX, YB_ERR_UNSUPPORTED, "yb_eval_ap: num_records=%lld", (long long)num_records);
  YB_REQUIRE(state && workspace && ap && nonempty && (num_records == 0 || (rec_score && rec_cls && rec_tp)), YB_ERR_INVALID,
             "yb_eval_ap: NULL argument");
  YB_REQUIRE(workspace_bytes >= yb_eval_ap_workspace_bytes(num_records, p), YB_ERR_INVALID, "yb_eval_ap: workspace %zu < %zu bytes",
             workspace_bytes, yb_eval_ap_workspace_bytes(num_records, p));
  const int C = p->num_classes, T = p->num_thr;
  const size_t n = (size_t)num_records;
  cudaStream_t st = (cudaStream_t)stream;
  char* ws = reinterpret_cast<char*>(align_up(reinterpret_cast<size_t>(workspace), 256));
  unsigned long long* keys_in = reinterpret_cast<unsigned long long*>(ws);
  unsigned long long* keys_out = reinterpret_cast<unsigned long long*>(ws + align_up(8 * n, 256));
  uint32_t* vals_in = reinterpret_cast<uint32_t*>(ws + 2 * align_up(8 * n, 256));
  uint32_t* vals_out = reinterpret_cast<uint32_t*>(ws + 2 * align_up(8 * n, 256) + align_up(4 * n, 256));
  void* temp = ws + 2 * align_up(8 * n, 256) + 2 * align_up(4 * n, 256);
  const EvalState* es = reinterpret_cast<const EvalState*>(state);
  if (n > 0) {
    const unsigned grid = (unsigned)std::min<size_t>((n + 255) / 256, 8 * kSmCount);
    k_eval_keys<<<grid, 256, 0, st>>>(rec_score, rec_cls, rec_tp, (long long)n, es, C, keys_in, vals_in);
    YB_CHECK_LAUNCH();
    size_t temp_bytes = ap_sort_temp_bytes((long long)n, C);
    YB_CHECK_CUDA(cub::DeviceRadixSort::SortPairs(temp, temp_bytes, keys_in, keys_out, vals_in, vals_out, (int)n, 0, key_end_bit(C), st));
    count_launch();                                                 // the radix sort, counted as one launch
  }
  k_eval_ap<<<dim3(C, 2 * T), kApThreads, 0, st>>>(keys_out, vals_out, (long long)n, es, C, T, ap, nonempty);
  YB_CHECK_LAUNCH();
  return YB_OK;
}
