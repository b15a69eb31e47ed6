// COCO's own mAP on the GPU: pycocotools' COCOeval (default Params, 'bbox' and 'segm') over the detections of the batched
// evaluation loop, bit-identical to its float64 precision / recall arrays (DESIGN.md, COCO mAP on the GPU).
//   k_cocoeval_match   one block per image: the detections the result JSON would hold, their rank within (image, class), double
//                      IoUs against the same-class gts, then warp w = (type, area range) runs COCOeval's greedy matching at the
//                      10 IoU thresholds for the detections in score order; one record per kept detection is appended at the
//                      running count plus the earlier images' counts (no host sync)
//   k_cocoeval_keys    sort keys (class, descending score, image rank); CUB's stable radix sort keeps the in-image order on ties
//   k_cocoeval_gather  the sorted records' rank and slot bits, structure of arrays
//   k_cocoeval_ap      one block per (type, threshold, class, area range, maxDets): the tp / fp scan and the 101 samples
#include "common.cuh"
#include "iou.cuh"

#include <cub/device/device_radix_sort.cuh>
#include <stdint.h>

#include <algorithm>

namespace yb {
namespace {

constexpr int kThreads = 256;        // k_cocoeval_match: 8 warps, warp w matches slot group (type w / 4, area w % 4)
constexpr int kMaxDet = 256;         // yb_detect's max_det limit; also bounds the rank (int16) and max_dets[2]
constexpr int kGroups = 8;           // (type, area range) pairs: the words of yb_cocoeval_record::bits
constexpr int T = YB_COCOEVAL_THR, R = YB_COCOEVAL_REC, A = YB_COCOEVAL_AREAS, M = YB_COCOEVAL_MAXDETS;
constexpr int kApThreads = 256;

struct CocoState {
  unsigned long long nrec;           // records appended so far
  unsigned int ticket;               // blocks of the current k_cocoeval_match launch that are done (reset by the last one)
  unsigned int flags;                // 1: capacity exceeded, 2: an image's ranges lie outside the buffers, 4: image rank out of range
};

struct MatchArgs {
  yb_cocoeval_params p;
  int batch, max_det;
  const int32_t* count; const int32_t* cls; const float* score; const int32_t* box_px;
  const uint32_t* det_masks; const int64_t* det_mask_off; long long det_mask_words;
  const int32_t* img_hw; const int32_t* img_rank;
  const int32_t* gt_cls; const double* gt_box; const double* gt_area; const int32_t* gt_crowd; const int32_t* gt_offset;
  long long total_gt;
  const uint32_t* gt_masks; const int64_t* gt_mask_off; long long gt_mask_words;
  yb_cocoeval_record* rec; long long capacity;
  CocoState* state;
  double* iou_box; double* iou_mask;  // [max_det * total_gt]: image b's [n][g] matrix at max_det * gt_offset[b]
  uint32_t* used;                     // [total_gt][8]: word (type, area), bit t = gt matched at threshold t
};

__device__ __forceinline__ int clamp_count(int c, int D) { return c < 0 ? 0 : (c > D ? D : c); }

__device__ long long block_sum(long long v, long long* red) {
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  if (lane_id() == 0) red[warp_id()] = v;
  __syncthreads();
  long long s = 0;
  for (int i = 0; i < (int)(blockDim.x >> 5); ++i) s += red[i];
  __syncthreads();
  return s;
}

// (nonignored, iou, index) ordered lexicographically: COCOeval's loop ends on the non-ignored gt of the largest IoU, the later
// of equal IoUs (its test is `iou < best: continue`), and reaches the ignored gts only when no non-ignored one qualifies
__device__ __forceinline__ bool better(int nig, double v, int j, int bnig, double bv, int bj) {
  return bj < 0 || (j >= 0 && (nig > bnig || (nig == bnig && (v > bv || (v == bv && j > bj)))));
}

__global__ void __launch_bounds__(kThreads) k_cocoeval_match(const MatchArgs a) {
  __shared__ int s_cls[kMaxDet];          // class of a detection the JSON would hold, else -1
  __shared__ uint32_t s_key[kMaxDet];     // float_to_ordered(score): a total order, equal for equal scores
  __shared__ int s_rank[kMaxDet];         // rank within (image, class); -1 when not kept
  __shared__ int s_ngt[kMaxDet];          // same-class gts of the image
  __shared__ int s_order[kMaxDet];        // kept detections by descending score, ties by index
  __shared__ unsigned s_pix[kMaxDet];     // mask pixel count (the segm area)
  __shared__ uint32_t s_bits[kMaxDet][kGroups];
  __shared__ long long red[kThreads / 32];
  __shared__ unsigned long long s_base;
  __shared__ int s_kept;
  const int b = blockIdx.x, D = a.max_det, K = a.p.num_classes;
  if (threadIdx.x == 0) {
    s_base = *reinterpret_cast<volatile unsigned long long*>(&a.state->nrec);
    s_kept = 0;
  }
  long long pre = 0;
  for (int j = threadIdx.x; j < b; j += kThreads) pre += clamp_count(a.count[j], D);
  pre = block_sum(pre, red);                                       // also publishes s_base
  const long long base = (long long)s_base + pre;
  const int n = clamp_count(a.count[b], D);

  if (n > 0) {
    const long long g0 = a.gt_offset[b], g1 = a.gt_offset[b + 1];
    const int h = a.img_hw[2 * b], w = a.img_hw[2 * b + 1];
    const long long words = (long long)h * ((w + 31) >> 5);
    const long long doff = a.det_mask_off[b], dend = a.det_mask_off[b + 1], goff = a.gt_mask_off[b], gend = a.gt_mask_off[b + 1];
    const bool ok = h > 0 && w > 0 && 0 <= g0 && g0 <= g1 && g1 <= a.total_gt && 0 <= doff && doff <= dend && dend <= a.det_mask_words &&
                    n * words <= dend - doff && 0 <= goff && goff <= gend && gend <= a.gt_mask_words && (g1 - g0) * words == gend - goff;
    const int img = a.img_rank[b];
    const bool img_ok = img >= 0 && img < a.p.num_images;
    if (threadIdx.x == 0 && !ok) atomicOr(&a.state->flags, 2u);
    if (threadIdx.x == 0 && !img_ok) atomicOr(&a.state->flags, 4u);
    const int g = ok ? (int)(g1 - g0) : 0;
    // ---- the detections eval.py writes to the JSON: class in range and (y2-y1)*(x2-x1) > 0 ----
    for (int i = threadIdx.x; i < n; i += kThreads) {
      const long long r = (long long)b * D + i;
      const int c = a.cls[r];
      const int32_t* bp = a.box_px + r * 4;
      const long long area = (long long)(bp[3] - bp[1]) * (long long)(bp[2] - bp[0]);
      s_cls[i] = ok && img_ok && c >= 0 && c < K && area > 0 ? c : -1;
      s_key[i] = float_to_ordered(a.score[r]);
    }
    for (int j = threadIdx.x; j < g * kGroups; j += kThreads) a.used[g0 * kGroups + j] = 0u;
    __syncthreads();
    // ---- rank within (image, class): descending score, ties by detection order; the first max_dets[2] are kept ----
    for (int i = threadIdx.x; i < n; i += kThreads) {
      int rank = -1, ngt = 0;
      const int c = s_cls[i];
      if (c >= 0) {
        const uint32_t k = s_key[i];
        rank = 0;
        for (int j = 0; j < n; ++j) rank += s_cls[j] == c && (s_key[j] > k || (s_key[j] == k && j < i));
        if (rank >= a.p.max_dets[M - 1]) rank = -1;
        for (int j = 0; j < g; ++j) ngt += __ldg(a.gt_cls + g0 + j) == c;
      }
      s_rank[i] = rank;
      s_ngt[i] = ngt;
    }
    __syncthreads();
    for (int i = threadIdx.x; i < n; i += kThreads) {
      if (s_rank[i] < 0) continue;
      const uint32_t k = s_key[i];
      int pos = 0;
      for (int j = 0; j < n; ++j) pos += s_rank[j] >= 0 && (s_key[j] > k || (s_key[j] == k && j < i));
      s_order[pos] = i;
      atomicAdd(&s_kept, 1);
    }
    __syncthreads();
    const int kept = s_kept;
    // ---- mask pixel counts of the kept detections, and the IoUs of their same-class pairs (one warp each) ----
    const uint32_t* dm = a.det_masks + doff;
    const uint32_t* gm = a.gt_masks + goff;
    for (int p = warp_id(); p < kept; p += kThreads / 32) {
      const int i = s_order[p];
      const uint32_t* pa = dm + i * words;
      unsigned c = 0;
      for (long long k = lane_id(); k < words; k += 32) c += __popc(__ldg(pa + k));
      for (int o = 16; o > 0; o >>= 1) c += __shfl_xor_sync(0xffffffffu, c, o);
      if (lane_id() == 0) s_pix[i] = c;
    }
    double* ib = a.iou_box + (long long)D * g0;
    double* im = a.iou_mask + (long long)D * g0;
    for (int pair = warp_id(); pair < n * g; pair += kThreads / 32) {
      const int i = pair / g, j = pair - i * g;
      if (s_rank[i] < 0 || s_cls[i] != __ldg(a.gt_cls + g0 + j)) continue;
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
        // the JSON's bbox: x1, y1, x2 - x1, y2 - y1 of the int32 pixel box (the 0.1-px rounding is the identity on integers)
        const double4 d = make_double4((double)bp[0], (double)bp[1], (double)(bp[2] - bp[0]), (double)(bp[3] - bp[1]));
        const double* gb = a.gt_box + (g0 + j) * 4;
        const bool crowd = a.gt_crowd[g0 + j] != 0;
        ib[i * g + j] = coco_box_iou(d, make_double4(gb[0], gb[1], gb[2], gb[3]), crowd);
        im[i * g + j] = coco_mask_iou(inter, ca, cb, crowd);
      }
    }
    __syncthreads();
    // ---- greedy matching: warp (type, area) over the kept detections in score order, every threshold ----
    {
      const int grp = warp_id(), type = grp >> 2, area = grp & 3;
      const double lo = a.p.area_rng[area][0], hi = a.p.area_rng[area][1];
      const double* iou = type ? im : ib;
      uint32_t* used = a.used + g0 * kGroups + grp;                 // used[j * kGroups]: only lane j % 32 touches it
      for (int p = 0; p < kept; ++p) {
        const int i = s_order[p], c = s_cls[i];
        const int32_t* bp = a.box_px + ((long long)b * D + i) * 4;
        const double darea = type ? (double)s_pix[i] : __dmul_rn((double)(bp[2] - bp[0]), (double)(bp[3] - bp[1]));
        const bool outside = darea < lo || darea > hi;
        uint32_t word = 0;
        for (int t = 0; t < T; ++t) {
          int bj = -1, bnig = 0;
          double bv = 0.0;
          if (s_ngt[i] > 0) {                                        // uniform across the warp
            const double thr = fmin(a.p.iou_thr[t], 1.0 - 1e-10);
            for (int j = lane_id(); j < g; j += 32) {
              const long long r = g0 + j;
              if (__ldg(a.gt_cls + r) != c) continue;
              const bool crowd = __ldg(a.gt_crowd + r) != 0;
              if (!crowd && ((used[j * kGroups] >> t) & 1u)) continue;
              const double v = iou[i * g + j];
              if (v < thr) continue;
              const double ga = __ldg(a.gt_area + r);
              const int nig = !(crowd || ga < lo || ga > hi);
              if (better(nig, v, j, bnig, bv, bj)) { bnig = nig; bv = v; bj = j; }
            }
            for (int o = 16; o > 0; o >>= 1) {
              const int on = __shfl_xor_sync(0xffffffffu, bnig, o);
              const double ov = __shfl_xor_sync(0xffffffffu, bv, o);
              const int oj = __shfl_xor_sync(0xffffffffu, bj, o);
              if (oj >= 0 && better(on, ov, oj, bnig, bv, bj)) { bnig = on; bv = ov; bj = oj; }
            }
          }
          if (bj >= 0) {
            word |= (1u << t) | (bnig ? 0u : 1u << (16 + t));       // a matched detection takes its gt's ignore flag
            if (lane_id() == (bj & 31)) used[bj * kGroups] |= 1u << t;
          } else if (outside) {
            word |= 1u << (16 + t);                                  // unmatched and outside the area range
          }
        }
        if (lane_id() == 0) s_bits[p][grp] = word;
      }
    }
    __syncthreads();
    // ---- the image's region: kept detections in score order, then records of class -1 ----
    for (int p = threadIdx.x; p < n; p += kThreads) {
      const long long r = base + p;
      if (r >= a.capacity) { atomicOr(&a.state->flags, 1u); continue; }
      yb_cocoeval_record out;
      if (p < kept) {
        const int i = s_order[p];
        out.score = a.score[(long long)b * D + i];
        out.cls = s_cls[i];
        out.img = img;
        out.det = (int16_t)i;
        out.rank = (int16_t)s_rank[i];
        for (int q = 0; q < kGroups; ++q) out.bits[q] = s_bits[p][q];
      } else {
        out.score = 0.f; out.cls = -1; out.img = 0; out.det = -1; out.rank = -1;
        for (int q = 0; q < kGroups; ++q) out.bits[q] = 0u;
      }
      a.rec[r] = out;
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

// ---- sort keys: class | ~ordered(score) | image rank, from the high bits down; invalid / unused records sort last (class = K) ----
__global__ void k_cocoeval_keys(const yb_cocoeval_record* __restrict__ rec, long long n, const CocoState* __restrict__ st, int K,
                                int img_bits, unsigned long long* __restrict__ keys, uint32_t* __restrict__ vals) {
  const long long nrec = (long long)st->nrec;
  const int shift = 32 + img_bits;
  for (long long r = blockIdx.x * (long long)blockDim.x + threadIdx.x; r < n; r += (long long)gridDim.x * blockDim.x) {
    const int c = r < nrec ? rec[r].cls : -1;
    keys[r] = c >= 0 && c < K ? ((unsigned long long)c << shift) | ((unsigned long long)(~float_to_ordered(rec[r].score)) << img_bits) |
                                    (unsigned long long)(uint32_t)rec[r].img
                              : (unsigned long long)K << shift;
    vals[r] = (uint32_t)r;
  }
}

__global__ void k_cocoeval_gather(const yb_cocoeval_record* __restrict__ rec, const uint32_t* __restrict__ order, long long n,
                                  int16_t* __restrict__ rank, uint32_t* __restrict__ bits) {
  for (long long k = blockIdx.x * (long long)blockDim.x + threadIdx.x; k < n; k += (long long)gridDim.x * blockDim.x) {
    const yb_cocoeval_record& r = rec[order[k]];
    rank[k] = r.rank;
    for (int q = 0; q < kGroups; ++q) bits[q * n + k] = r.bits[q];
  }
}

__device__ long long lower_bound_u64(const unsigned long long* k, long long n, unsigned long long v) {
  long long lo = 0, hi = n;
  while (lo < hi) { const long long mid = (lo + hi) >> 1; if (k[mid] < v) lo = mid + 1; else hi = mid; }
  return lo;
}

// ---- COCOeval.accumulate for one (type, threshold, class, area range, maxDets) ----
// The records of the class in sorted order, minus those ranked >= maxDets in their image and the ignored ones (they repeat their
// predecessor's precision and recall, or add a 0 before the first detection that counts).  With m true positives among the first
// N counted records, precision = m / ((N - m) + m + eps) and recall = m / npig in double.  The sample at rec_thr[x] is the
// precision's suffix maximum from the m(x)-th true positive, m(x) the least m with m / npig >= rec_thr[x] (from the first record
// when m(x) = 0; 0 when m(x) exceeds the true positives); the suffix maximum is attained at a true positive, so each true positive
// goes to bucket max{x : m(x) <= m} and a suffix maximum over the 101 buckets gives every sample (DESIGN.md, section 8).
__global__ void __launch_bounds__(kApThreads) k_cocoeval_ap(const yb_cocoeval_params p, const unsigned long long* __restrict__ keys,
                                                            const int16_t* __restrict__ rank, const uint32_t* __restrict__ bits,
                                                            long long n, int shift, const int64_t* __restrict__ npig,
                                                            double* __restrict__ precision, double* __restrict__ recall) {
  __shared__ int mx[R];
  __shared__ unsigned long long bmax[R];
  __shared__ unsigned long long wsum[kApThreads / 32];
  __shared__ long long seg[2];
  const int K = p.num_classes, k = blockIdx.x, area = blockIdx.y / M, m = blockIdx.y % M, type = blockIdx.z / T, t = blockIdx.z % T;
  const long long ng = npig[k * A + area];
  double* prec = precision + ((long long)(type * T + t) * R * K + k) * (A * M) + area * M + m;   // stride K * A * M over x
  double* rc = recall + ((long long)(type * T + t) * K + k) * (A * M) + area * M + m;
  const long long stride = (long long)K * A * M;
  if (ng <= 0) {                                                    // COCOeval leaves the entry at -1
    for (int x = threadIdx.x; x < R; x += kApThreads) prec[x * stride] = -1.0;
    if (threadIdx.x == 0) *rc = -1.0;
    return;
  }
  if (threadIdx.x < R) {
    const int x = threadIdx.x;
    const double xd = p.rec_thr[x], g = (double)ng;
    long long mm = (long long)ceil(xd * g);
    if (mm < 0) mm = 0;
    while (mm > 0 && (double)(mm - 1) / g >= xd) --mm;
    while ((double)mm / g < xd) ++mm;
    mx[x] = (int)std::min<long long>(mm, 0x7fffffffLL);
    bmax[x] = 0ull;
  }
  if (threadIdx.x == 0) seg[0] = lower_bound_u64(keys, n, (unsigned long long)k << shift);
  if (threadIdx.x == 1) seg[1] = lower_bound_u64(keys, n, (unsigned long long)(k + 1) << shift);
  __syncthreads();
  const long long lo = seg[0], hi = seg[1];
  const int max_det = p.max_dets[m];
  const uint32_t* word = bits + (long long)(type * A + area) * n;
  unsigned long long carry = 0;                                     // (true positives << 32) | counted records so far
  for (long long k0 = lo; k0 < hi; k0 += kApThreads) {
    const long long q = k0 + threadIdx.x;
    bool counted = false, tp = false;
    if (q < hi) {
      const uint32_t wd = word[q];
      counted = rank[q] < max_det && !((wd >> (16 + t)) & 1u);
      tp = counted && ((wd >> t) & 1u);
    }
    unsigned long long incl = (counted ? 1ull : 0ull) | (tp ? 1ull << 32 : 0ull);
    for (int o = 1; o < 32; o <<= 1) { const unsigned long long v = __shfl_up_sync(0xffffffffu, incl, o); if (lane_id() >= o) incl += v; }
    if (lane_id() == 31) wsum[warp_id()] = incl;
    __syncthreads();
    unsigned long long wpre = 0, chunk = 0;
    for (int i = 0; i < kApThreads / 32; ++i) { if (i < warp_id()) wpre += wsum[i]; chunk += wsum[i]; }
    if (tp) {
      const unsigned long long c = carry + wpre + incl;
      const long long mt = (long long)(c >> 32), nt = (long long)(c & 0xffffffffull);
      const double pr = __ddiv_rn((double)mt, __dadd_rn(__dadd_rn((double)(nt - mt), (double)mt), 2.220446049250313e-16));
      int l = 0, r = R - 1;                                         // largest x with mx[x] <= mt (mx[0] = 0)
      while (l < r) { const int mid = (l + r + 1) >> 1; if (mx[mid] <= mt) l = mid; else r = mid - 1; }
      atomicMax(&bmax[l], (unsigned long long)__double_as_longlong(pr));   // non-negative doubles order like their bits
    }
    carry += chunk;
    __syncthreads();
  }
  const long long tps = (long long)(carry >> 32);
  if (threadIdx.x == 0) {
    double run = 0.0;
    for (int x = R - 1; x >= 0; --x) {
      run = fmax(run, __longlong_as_double((long long)bmax[x]));
      prec[x * stride] = mx[x] <= tps ? run : 0.0;
    }
    *rc = __ddiv_rn((double)tps, (double)ng);
  }
}

int bits_for(long long v) {                                         // bits to hold 0 .. v
  int b = 0;
  while (b < 63 && (1ll << b) <= v) ++b;
  return b;
}

bool params_ok(const yb_cocoeval_params* p) {
  return p && p->num_classes > 0 && p->num_images > 0 && 1 <= p->max_dets[0] && p->max_dets[0] <= p->max_dets[1] &&
         p->max_dets[1] <= p->max_dets[2] && p->max_dets[2] <= kMaxDet;
}

size_t sort_temp_bytes(long long n, int end_bit) {
  size_t temp = 0;
  cub::DeviceRadixSort::SortPairs(nullptr, temp, (const unsigned long long*)nullptr, (unsigned long long*)nullptr,
                                  (const uint32_t*)nullptr, (uint32_t*)nullptr, (int)n, 0, end_bit);
  return temp;
}

}  // namespace
}  // namespace yb

using namespace yb;

extern "C" size_t yb_cocoeval_state_bytes(void) { return sizeof(CocoState); }

extern "C" size_t yb_cocoeval_match_workspace_bytes(int batch, int max_det, int64_t total_gt) {
  if (batch < 0 || max_det < 0 || total_gt < 0) return 0;
  const size_t iou = align_up(sizeof(double) * (size_t)max_det * (size_t)total_gt, 256);
  return 2 * iou + align_up(sizeof(uint32_t) * kGroups * (size_t)total_gt, 256) + 256;
}

extern "C" size_t yb_cocoeval_accumulate_workspace_bytes(int64_t num_records) {
  if (num_records < 0 || num_records > INT32_MAX) return 0;
  const size_t n = (size_t)num_records;
  return 2 * align_up(8 * n, 256) + 2 * align_up(4 * n, 256) + align_up(2 * n, 256) + align_up(4 * kGroups * n, 256) +
         align_up(sort_temp_bytes((long long)n, 64), 256) + 256;
}

extern "C" int yb_cocoeval_match(const yb_cocoeval_params* p, int batch, int max_det, const int32_t* count, const int32_t* cls,
                                 const float* score, const int32_t* box_px, const uint32_t* det_masks, const int64_t* det_mask_off,
                                 int64_t det_mask_words, const int32_t* img_hw, const int32_t* img_rank, const int32_t* gt_cls,
                                 const double* gt_box, const double* gt_area, const int32_t* gt_crowd, const int32_t* gt_offset,
                                 int64_t total_gt, const uint32_t* gt_masks, const int64_t* gt_mask_off, int64_t gt_mask_words,
                                 yb_cocoeval_record* records, int64_t capacity, void* state, void* workspace, size_t workspace_bytes,
                                 void* stream) {
  YB_REQUIRE(params_ok(p), YB_ERR_INVALID, "yb_cocoeval_match: bad params (num_classes, num_images > 0; 1 <= max_dets ascending <= %d)",
             kMaxDet);
  YB_REQUIRE(batch >= 0 && max_det >= 0 && total_gt >= 0 && capacity >= 0 && det_mask_words >= 0 && gt_mask_words >= 0, YB_ERR_INVALID,
             "yb_cocoeval_match: negative size (batch=%d max_det=%d total_gt=%lld)", batch, max_det, (long long)total_gt);
  YB_REQUIRE(max_det <= kMaxDet, YB_ERR_UNSUPPORTED, "yb_cocoeval_match: max_det=%d > %d", max_det, kMaxDet);
  if (batch == 0) return YB_OK;
  YB_REQUIRE(count && cls && score && box_px && det_mask_off && img_hw && img_rank && gt_offset && gt_mask_off && records && state &&
             workspace, YB_ERR_INVALID, "yb_cocoeval_match: NULL argument");
  YB_REQUIRE((det_masks || det_mask_words == 0) && (gt_masks || gt_mask_words == 0) &&
             ((gt_cls && gt_box && gt_area && gt_crowd) || total_gt == 0), YB_ERR_INVALID, "yb_cocoeval_match: NULL mask / gt buffer");
  YB_REQUIRE(workspace_bytes >= yb_cocoeval_match_workspace_bytes(batch, max_det, total_gt), YB_ERR_INVALID,
             "yb_cocoeval_match: workspace %zu < %zu bytes", workspace_bytes, yb_cocoeval_match_workspace_bytes(batch, max_det, total_gt));
  MatchArgs a;
  a.p = *p; a.batch = batch; a.max_det = max_det;
  a.count = count; a.cls = cls; a.score = score; a.box_px = box_px;
  a.det_masks = det_masks; a.det_mask_off = det_mask_off; a.det_mask_words = det_mask_words;
  a.img_hw = img_hw; a.img_rank = img_rank;
  a.gt_cls = gt_cls; a.gt_box = gt_box; a.gt_area = gt_area; a.gt_crowd = gt_crowd; a.gt_offset = gt_offset; a.total_gt = total_gt;
  a.gt_masks = gt_masks; a.gt_mask_off = gt_mask_off; a.gt_mask_words = gt_mask_words;
  a.rec = records; a.capacity = capacity;
  a.state = reinterpret_cast<CocoState*>(state);
  char* ws = reinterpret_cast<char*>(align_up(reinterpret_cast<size_t>(workspace), 256));
  const size_t iou = align_up(sizeof(double) * (size_t)max_det * (size_t)total_gt, 256);
  a.iou_box = reinterpret_cast<double*>(ws);
  a.iou_mask = reinterpret_cast<double*>(ws + iou);
  a.used = reinterpret_cast<uint32_t*>(ws + 2 * iou);
  k_cocoeval_match<<<batch, kThreads, 0, (cudaStream_t)stream>>>(a);
  YB_CHECK_LAUNCH();
  return YB_OK;
}

extern "C" int yb_cocoeval_accumulate(const yb_cocoeval_params* p, const yb_cocoeval_record* records, int64_t num_records, const void* state,
                                      const int64_t* npig, void* workspace, size_t workspace_bytes, double* precision, double* recall,
                                      void* stream) {
  YB_REQUIRE(params_ok(p), YB_ERR_INVALID, "yb_cocoeval_accumulate: bad params (num_classes, num_images > 0; 1 <= max_dets ascending <= %d)",
             kMaxDet);
  YB_REQUIRE(num_records >= 0 && num_records <= INT32_MAX, YB_ERR_UNSUPPORTED, "yb_cocoeval_accumulate: num_records=%lld",
             (long long)num_records);
  const int K = p->num_classes, img_bits = std::max(1, bits_for((long long)p->num_images - 1)), cls_bits = bits_for(K);
  YB_REQUIRE(img_bits + cls_bits <= 32, YB_ERR_UNSUPPORTED,
             "yb_cocoeval_accumulate: %d classes and %d images do not fit the 64-bit sort key (bits(classes) + bits(images - 1) <= 32)",
             K, p->num_images);
  YB_REQUIRE(state && npig && workspace && precision && recall && (num_records == 0 || records), YB_ERR_INVALID,
             "yb_cocoeval_accumulate: NULL argument");
  YB_REQUIRE(workspace_bytes >= yb_cocoeval_accumulate_workspace_bytes(num_records), YB_ERR_INVALID,
             "yb_cocoeval_accumulate: workspace %zu < %zu bytes", workspace_bytes, yb_cocoeval_accumulate_workspace_bytes(num_records));
  const size_t n = (size_t)num_records;
  const int shift = 32 + img_bits, end_bit = shift + cls_bits;
  cudaStream_t st = (cudaStream_t)stream;
  char* ws = reinterpret_cast<char*>(align_up(reinterpret_cast<size_t>(workspace), 256));
  unsigned long long* keys_in = reinterpret_cast<unsigned long long*>(ws);
  ws += align_up(8 * n, 256);
  unsigned long long* keys_out = reinterpret_cast<unsigned long long*>(ws);
  ws += align_up(8 * n, 256);
  uint32_t* vals_in = reinterpret_cast<uint32_t*>(ws);
  ws += align_up(4 * n, 256);
  uint32_t* vals_out = reinterpret_cast<uint32_t*>(ws);
  ws += align_up(4 * n, 256);
  int16_t* rank = reinterpret_cast<int16_t*>(ws);
  ws += align_up(2 * n, 256);
  uint32_t* bits = reinterpret_cast<uint32_t*>(ws);
  ws += align_up(4 * kGroups * n, 256);
  const CocoState* cs = reinterpret_cast<const CocoState*>(state);
  if (n > 0) {
    const unsigned grid = (unsigned)std::min<size_t>((n + 255) / 256, 8 * kSmCount);
    k_cocoeval_keys<<<grid, 256, 0, st>>>(records, (long long)n, cs, K, img_bits, keys_in, vals_in);
    YB_CHECK_LAUNCH();
    size_t temp_bytes = sort_temp_bytes((long long)n, end_bit);
    YB_REQUIRE(temp_bytes <= align_up(sort_temp_bytes((long long)n, 64), 256), YB_ERR_INVALID, "yb_cocoeval_accumulate: sort scratch");
    YB_CHECK_CUDA(cub::DeviceRadixSort::SortPairs(ws, temp_bytes, keys_in, keys_out, vals_in, vals_out, (int)n, 0, end_bit, st));
    count_launch();                                                 // the radix sort, counted as one launch
    k_cocoeval_gather<<<grid, 256, 0, st>>>(records, vals_out, (long long)n, rank, bits);
    YB_CHECK_LAUNCH();
  }
  k_cocoeval_ap<<<dim3(K, A * M, 2 * T), kApThreads, 0, st>>>(*p, keys_out, rank, bits, (long long)n, shift, npig, precision, recall);
  YB_CHECK_LAUNCH();
  return YB_OK;
}
