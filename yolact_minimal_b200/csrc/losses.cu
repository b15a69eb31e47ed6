// Fused training targets and losses with their gradients (SURVEY.md 8 rows a12 / f3), batched over images:
//   match + encode        utils/box_utils.py:57-83,:104-114     k_match_anchor / k_match_gt / k_match_finalize
//   OHEM mining           modules/yolact.py:205-225             k_logit_max / k_ohem_mark / k_ohem_select
//   category + box loss   modules/yolact.py:227-239             k_cls_box_loss
//   lincomb mask loss     modules/yolact.py:241-291             k_downsample_masks / k_mask_select / k_mask_loss
//   semantic seg loss     modules/yolact.py:293-313             k_semantic_loss
// The reference runs these as per-image Python loops over ATen ops; here every stage is one launch over the whole batch and the
// gradient w.r.t. each network output is produced in the same pass as the loss.  fp32 throughout; the float operations that
// decide a LABEL (IoU, thresholds) are separately rounded in the reference's order (no FMA contraction) so that labels and
// matched indices equal the reference's bit for bit.
#include "train.cuh"

#include <math.h>
#include <stdint.h>

namespace yb {
namespace {

constexpr int kMaxGt = kLossMaxGt;       // ground-truth instances per image held in shared memory

struct LossWs {                          // carved out of the caller's workspace
  float* best_iou;        // [B,A]
  int32_t* best_gt;       // [B,A]
  int32_t* gt_anchor;     // [B,kMaxGt]
  int32_t* labels;        // [B,A]   >0 fg class+1, 0 bg, -1 neutral
  float* offsets;         // [B,A,4]
  float* matched;         // [B,A,4]
  uint32_t* mark;         // [B,A]   OHEM mark as an ascending key (float_to_ordered)
  uint8_t* neg;           // [B,A]
  int32_t* num_pos;       // [B] + total at [B]
  uint32_t* logit_max;    // [1] ordered-uint max of all class logits
  double* acc;            // [4] loss accumulators (sums before normalisation)
  uint8_t* ds_mask;       // [total_gt, P, P] binarised down-sampled gt masks
  int32_t* sel;           // [B, masks_to_train] selected positive anchors
  int32_t* sel_count;     // [B] selected, [B..2B) all positives of the image
};

__device__ __forceinline__ float iou_rn(float ax1, float ay1, float ax2, float ay2, float bx1, float by1, float bx2, float by2) {
  // utils/box_utils.py:28-36, each operation rounded separately
  const float iw = fmaxf(__fsub_rn(fminf(ax2, bx2), fmaxf(ax1, bx1)), 0.f);
  const float ih = fmaxf(__fsub_rn(fminf(ay2, by2), fmaxf(ay1, by1)), 0.f);
  const float inter = __fmul_rn(iw, ih);
  const float aa = __fmul_rn(__fsub_rn(ax2, ax1), __fsub_rn(ay2, ay1));
  const float ab = __fmul_rn(__fsub_rn(bx2, bx1), __fsub_rn(by2, by1));
  return __fdiv_rn(inter, __fsub_rn(__fadd_rn(aa, ab), inter));
}

__device__ __forceinline__ void anchor_corners(const float* a, float& x1, float& y1, float& x2, float& y2) {
  // box_utils.py:59: (cx - w/2, cy - h/2, cx + w/2, cy + h/2)
  const float hw = __fdiv_rn(a[2], 2.f), hh = __fdiv_rn(a[3], 2.f);
  x1 = __fsub_rn(a[0], hw); y1 = __fsub_rn(a[1], hh); x2 = __fadd_rn(a[0], hw); y2 = __fadd_rn(a[1], hh);
}

// ---- match: best gt per anchor (first maximum) ----
__global__ void __launch_bounds__(256) k_match_anchor(const float* __restrict__ anchors, const float* __restrict__ gt, const int32_t* __restrict__ gt_off,
                                                      int A, float* __restrict__ best_iou, int32_t* __restrict__ best_gt) {
  __shared__ float sg[kMaxGt * 4];
  const int b = blockIdx.y, g0 = gt_off[b], n = gt_off[b + 1] - g0;
  for (int i = threadIdx.x; i < n * 4; i += 256) sg[i] = gt[(size_t)(g0 + (i >> 2)) * 5 + (i & 3)];
  __syncthreads();
  const int a = blockIdx.x * 256 + threadIdx.x;
  if (a >= A) return;
  float x1, y1, x2, y2;
  anchor_corners(anchors + (size_t)a * 4, x1, y1, x2, y2);
  float bi = -INFINITY; int bj = 0;
  for (int j = 0; j < n; ++j) {
    const float v = iou_rn(sg[j * 4], sg[j * 4 + 1], sg[j * 4 + 2], sg[j * 4 + 3], x1, y1, x2, y2);
    if (v > bi) { bi = v; bj = j; }
  }
  best_iou[(size_t)b * A + a] = bi;
  best_gt[(size_t)b * A + a] = bj;
}

// ---- match: best anchor per gt (first maximum over anchors) ----
__global__ void __launch_bounds__(256) k_match_gt(const float* __restrict__ anchors, const float* __restrict__ gt, const int32_t* __restrict__ gt_off,
                                                  int A, int32_t* __restrict__ gt_anchor) {
  const int b = blockIdx.y, g0 = gt_off[b], n = gt_off[b + 1] - g0, j = blockIdx.x;
  if (j >= n) return;
  const float* g = gt + (size_t)(g0 + j) * 5;
  const float gx1 = g[0], gy1 = g[1], gx2 = g[2], gy2 = g[3];
  float bi = -INFINITY; int ba = 0x7fffffff;
  for (int a = threadIdx.x; a < A; a += 256) {
    float x1, y1, x2, y2;
    anchor_corners(anchors + (size_t)a * 4, x1, y1, x2, y2);
    const float v = iou_rn(gx1, gy1, gx2, gy2, x1, y1, x2, y2);
    if (v > bi) { bi = v; ba = a; }                                   // ascending a within the thread: first maximum
  }
  __shared__ float si[256];
  __shared__ int sa[256];
  si[threadIdx.x] = bi; sa[threadIdx.x] = ba;
  __syncthreads();
  for (int off = 128; off > 0; off >>= 1) {
    if (threadIdx.x < off) {
      const float o = si[threadIdx.x + off]; const int oa = sa[threadIdx.x + off];
      if (o > si[threadIdx.x] || (o == si[threadIdx.x] && oa < sa[threadIdx.x])) { si[threadIdx.x] = o; sa[threadIdx.x] = oa; }
    }
    __syncthreads();
  }
  if (threadIdx.x == 0) gt_anchor[b * kMaxGt + j] = sa[0] == 0x7fffffff ? 0 : sa[0];
}

// ---- match: forced pairs (sequential, a later gt wins a shared anchor), labels, matched boxes, SSD offsets ----
__global__ void __launch_bounds__(256) k_match_finalize(const float* __restrict__ anchors, const float* __restrict__ gt, const int32_t* __restrict__ gt_off,
                                                        int A, int B, float pos_thr, float neg_thr, float* __restrict__ best_iou,
                                                        int32_t* __restrict__ best_gt, const int32_t* __restrict__ gt_anchor, int32_t* __restrict__ labels,
                                                        float* __restrict__ offsets, float* __restrict__ matched, int32_t* __restrict__ num_pos) {
  const int b = blockIdx.x, g0 = gt_off[b], n = gt_off[b + 1] - g0;
  if (threadIdx.x == 0) {
    for (int j = 0; j < n; ++j) best_iou[(size_t)b * A + gt_anchor[b * kMaxGt + j]] = 2.f;       // index_fill_ first (box_utils.py:69)
    for (int j = 0; j < n; ++j) best_gt[(size_t)b * A + gt_anchor[b * kMaxGt + j]] = j;           // then the sequential loop (:72-73)
  }
  __syncthreads();
  int cnt = 0;
  for (int a = threadIdx.x; a < A; a += 256) {
    const size_t i = (size_t)b * A + a;
    const int j = best_gt[i];
    const float* g = gt + (size_t)(g0 + j) * 5;         // read only when n > 0: an empty last image's g0 is one row past the buffer
    const float iou = best_iou[i];
    int lab = 0;
    if (n > 0) {
      lab = (int)g[4] + 1;
      if (iou < pos_thr) lab = -1;
      if (iou < neg_thr) lab = 0;
    }
    labels[i] = lab;
    cnt += lab > 0;
    const float* an = anchors + (size_t)a * 4;
    float m[4] = {0.f, 0.f, 0.f, 0.f}, o[4] = {0.f, 0.f, 0.f, 0.f};
    if (n > 0) {
      m[0] = g[0]; m[1] = g[1]; m[2] = g[2]; m[3] = g[3];
      // encode (box_utils.py:104-114): ((x1+x2)/2 - cx) / (0.1 w),  log((x2-x1)/w) / 0.2
      o[0] = __fdiv_rn(__fsub_rn(__fdiv_rn(__fadd_rn(m[0], m[2]), 2.f), an[0]), __fmul_rn(0.1f, an[2]));
      o[1] = __fdiv_rn(__fsub_rn(__fdiv_rn(__fadd_rn(m[1], m[3]), 2.f), an[1]), __fmul_rn(0.1f, an[3]));
      o[2] = __fdiv_rn(logf(__fdiv_rn(__fsub_rn(m[2], m[0]), an[2])), 0.2f);
      o[3] = __fdiv_rn(logf(__fdiv_rn(__fsub_rn(m[3], m[1]), an[3])), 0.2f);
    }
#pragma unroll
    for (int q = 0; q < 4; ++q) { matched[i * 4 + q] = m[q]; offsets[i * 4 + q] = o[q]; }
  }
  __shared__ int sc[256];
  sc[threadIdx.x] = cnt;
  __syncthreads();
  for (int off = 128; off > 0; off >>= 1) { if (threadIdx.x < off) sc[threadIdx.x] += sc[threadIdx.x + off]; __syncthreads(); }
  if (threadIdx.x == 0) { num_pos[b] = sc[0]; atomicAdd(&num_pos[B], sc[0]); }
}

// ---- OHEM: global logit maximum (yolact.py:209), hardness mark per anchor ----
__global__ void __launch_bounds__(256) k_logit_max(const float* __restrict__ x, long long n, uint32_t* __restrict__ out) {
  float m = -INFINITY;
  for (long long i = blockIdx.x * 256LL + threadIdx.x; i < n; i += (long long)gridDim.x * 256) m = fmaxf(m, x[i]);
#pragma unroll
  for (int off = 16; off > 0; off >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, off));
  if ((threadIdx.x & 31) == 0) atomicMax(out, float_to_ordered(m));
}

__global__ void __launch_bounds__(256) k_ohem_mark(const float* __restrict__ cls, const int32_t* __restrict__ labels, const uint32_t* __restrict__ logit_max,
                                                   long long rows, int NC, uint32_t* __restrict__ mark) {
  const int lane = threadIdx.x & 31;
  const long long r = blockIdx.x * 8LL + (threadIdx.x >> 5);
  if (r >= rows) return;
  const float gm = ordered_to_float(*logit_max);
  const float* x = cls + r * NC;
  float s = 0.f;
  for (int c = lane; c < NC; c += 32) s += expf(x[c] - gm);
#pragma unroll
  for (int off = 16; off > 0; off >>= 1) s += __shfl_xor_sync(0xffffffffu, s, off);
  // positives and neutrals are filtered out (:213-214).  The true mark is >= 0, but its fp32 value is not: when class 0 holds the
  // row's maximum and gm is large, it rounds to -ulp(gm).  The ordered key sorts such a mark below the zeroed rows, as torch.sort does.
  if (lane == 0) mark[r] = float_to_ordered(labels[r] != 0 ? 0.f : (logf(s) + gm) - x[0]);
}

// k-th largest of n uint32 keys by 4 radix passes over shared histograms; returns the key value
__device__ uint32_t block_kth_largest(const uint32_t* __restrict__ keys, int n, int k, uint32_t* hist /*[256]*/, uint32_t* bc /*[2]*/) {
  uint32_t prefix = 0, mask = 0;
  int remaining = k;
  for (int shift = 24; shift >= 0; shift -= 8) {
    for (int i = threadIdx.x; i < 256; i += blockDim.x) hist[i] = 0;
    __syncthreads();
    for (int i = threadIdx.x; i < n; i += blockDim.x) {
      const uint32_t v = keys[i];
      if ((v & mask) == prefix) atomicAdd(&hist[(v >> shift) & 255u], 1u);
    }
    __syncthreads();
    if (threadIdx.x == 0) {
      int acc = 0, d = 255;
      for (; d > 0; --d) { if (acc + (int)hist[d] >= remaining) break; acc += (int)hist[d]; }
      bc[0] = (uint32_t)d; bc[1] = (uint32_t)(remaining - acc);
    }
    __syncthreads();
    prefix |= bc[0] << shift; mask |= 255u << shift; remaining = (int)bc[1];
    __syncthreads();
  }
  return prefix;
}

// per image: the num_neg = min(3 * num_pos, A - 1) anchors with the largest marks; ties by ascending anchor index (a stable
// descending sort, yolact.py:216-220); positives / neutrals are cleared afterwards (:223-224)
__global__ void __launch_bounds__(1024) k_ohem_select(const uint32_t* __restrict__ mark, const int32_t* __restrict__ labels, const int32_t* __restrict__ num_pos,
                                                      int A, int ratio, uint8_t* __restrict__ neg) {
  __shared__ uint32_t hist[256];
  __shared__ uint32_t bc[2];
  __shared__ int scan[1024];
  const int b = blockIdx.x;
  const uint32_t* keys = mark + (size_t)b * A;
  int k = ratio * num_pos[b];
  if (k > A - 1) k = A - 1;
  if (k <= 0) { for (int a = threadIdx.x; a < A; a += blockDim.x) neg[(size_t)b * A + a] = 0; return; }
  const uint32_t thr = block_kth_largest(keys, A, k, hist, bc);
  // count strictly greater, then hand the remaining slots to the == thr entries in index order
  int gt_cnt = 0;
  const int per = (A + blockDim.x - 1) / blockDim.x, a0 = threadIdx.x * per, a1 = min(a0 + per, A);
  int eq = 0;
  for (int a = a0; a < a1; ++a) { gt_cnt += keys[a] > thr; eq += keys[a] == thr; }
  scan[threadIdx.x] = gt_cnt;
  __syncthreads();
  for (int off = 512; off > 0; off >>= 1) { if (threadIdx.x < off) scan[threadIdx.x] += scan[threadIdx.x + off]; __syncthreads(); }
  const int total_gt = scan[0];
  __syncthreads();
  scan[threadIdx.x] = eq;
  __syncthreads();
  for (int off = 1; off < 1024; off <<= 1) {                         // inclusive Hillis-Steele scan of the per-thread == counts
    const int v = threadIdx.x >= off ? scan[threadIdx.x - off] : 0;
    __syncthreads();
    scan[threadIdx.x] += v;
    __syncthreads();
  }
  int eq_before = scan[threadIdx.x] - eq;
  const int eq_take = k - total_gt;
  for (int a = a0; a < a1; ++a) {
    bool sel = keys[a] > thr;
    if (keys[a] == thr) { sel = eq_before < eq_take; ++eq_before; }
    neg[(size_t)b * A + a] = (sel && labels[(size_t)b * A + a] == 0) ? 1 : 0;
  }
}

// ---- category loss (cross entropy over positives + mined negatives) and box loss (smooth L1 over positives) with gradients ----
__global__ void __launch_bounds__(256) k_cls_box_loss(const float* __restrict__ cls, const float* __restrict__ box, const int32_t* __restrict__ labels,
                                                      const uint8_t* __restrict__ neg, const float* __restrict__ offsets, const int32_t* __restrict__ num_pos,
                                                      long long rows, int NC, int B, const float* __restrict__ gsd, float gs_cls, float gs_box, double* __restrict__ acc,
                                                      float* __restrict__ d_cls, float* __restrict__ d_box) {
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  const long long r = blockIdx.x * 8LL + w;
  __shared__ float sl[8][2];
  float lc = 0.f, lb = 0.f;
  if (r < rows) {
    const int lab = labels[r];
    const bool chosen = lab > 0 || neg[r];
    const float npos = (float)max(num_pos[B], 1);
    const float* x = cls + r * NC;
    if (chosen) {
      float mx = -INFINITY;
      for (int c = lane; c < NC; c += 32) mx = fmaxf(mx, x[c]);
#pragma unroll
      for (int off = 16; off > 0; off >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, off));
      float s = 0.f;
      for (int c = lane; c < NC; c += 32) s += expf(x[c] - mx);
#pragma unroll
      for (int off = 16; off > 0; off >>= 1) s += __shfl_xor_sync(0xffffffffu, s, off);
      const float lse = logf(s) + mx;
      const int tgt = lab > 0 ? lab : 0;
      if (lane == 0) lc = lse - x[tgt];
      if (d_cls) {
        const float g = gs_cls * (gsd ? gsd[0] : 1.f) / npos;
        for (int c = lane; c < NC; c += 32) d_cls[r * NC + c] = g * (expf(x[c] - lse) - (c == tgt ? 1.f : 0.f));
      }
    } else if (d_cls) {
      for (int c = lane; c < NC; c += 32) d_cls[r * NC + c] = 0.f;
    }
    if (lane < 4) {
      float g = 0.f;
      if (lab > 0) {
        const float d = box[r * 4 + lane] - offsets[r * 4 + lane];
        const float ad = fabsf(d);
        lb = ad < 1.f ? 0.5f * d * d : ad - 0.5f;
        g = (ad < 1.f ? d : (d > 0.f ? 1.f : -1.f)) * gs_box * (gsd ? gsd[1] : 1.f) / npos;
      }
      if (d_box) d_box[r * 4 + lane] = g;
    }
    lb += __shfl_xor_sync(0xffffffffu, lb, 1);
    lb += __shfl_xor_sync(0xffffffffu, lb, 2);
  }
  if (lane == 0) { sl[w][0] = lc; sl[w][1] = lb; }
  __syncthreads();
  if (threadIdx.x == 0) {
    double a = 0, c = 0;
    for (int i = 0; i < 8; ++i) { a += sl[i][0]; c += sl[i][1]; }
    if (a != 0) atomicAdd(&acc[0], a);
    if (c != 0) atomicAdd(&acc[1], c);
  }
}

// ---- gt masks: bilinear down-sampling (align_corners=False, F.interpolate size=...) + binarisation (> 0.5) ----
__device__ __forceinline__ float bilinear_at(const float* __restrict__ m, int S, int out, int oy, int ox) {
  const float scale = (float)S / (float)out;
  const float sy = fmaxf(scale * ((float)oy + 0.5f) - 0.5f, 0.f), sx = fmaxf(scale * ((float)ox + 0.5f) - 0.5f, 0.f);
  const int y0 = min((int)sy, S - 1), x0 = min((int)sx, S - 1);
  const int y1 = min(y0 + 1, S - 1), x1 = min(x0 + 1, S - 1);
  const float ly1 = sy - (float)y0, ly0 = 1.f - ly1, lx1 = sx - (float)x0, lx0 = 1.f - lx1;
  return ly0 * (lx0 * m[(size_t)y0 * S + x0] + lx1 * m[(size_t)y0 * S + x1]) + ly1 * (lx0 * m[(size_t)y1 * S + x0] + lx1 * m[(size_t)y1 * S + x1]);
}

__global__ void __launch_bounds__(256) k_downsample_masks(const float* __restrict__ masks, const int32_t* __restrict__ gt_off, int B, int S, int P,
                                                          uint8_t* __restrict__ out) {
  const int j = blockIdx.y, i = blockIdx.x * 256 + threadIdx.x;
  if (i >= P * P || j >= gt_off[B]) return;                  // (the grid may be sized for a capacity: CUDA-graph replay)
  out[(size_t)j * P * P + i] = bilinear_at(masks + (size_t)j * S * S, S, P, i / P, i % P) > 0.5f ? 1 : 0;
}

// ---- positives of an image, in anchor order; more than `limit` -> a uniformly random subset of `limit` (yolact.py:261-268) ----
__global__ void __launch_bounds__(1024) k_mask_select(const int32_t* __restrict__ labels, int A, int limit, uint32_t seed_value, const uint32_t* __restrict__ seed_dev,
                                                      uint32_t* __restrict__ keys_ws /*[B,A]*/,
                                                      int32_t* __restrict__ sel, int32_t* __restrict__ sel_count, int B) {
  __shared__ uint32_t hist[256];
  __shared__ uint32_t bc[2];
  __shared__ int scan[1024];
  const int b = blockIdx.x;
  const uint32_t seed = seed_dev ? *seed_dev : seed_value;
  const int32_t* lab = labels + (size_t)b * A;
  uint32_t* keys = keys_ws + (size_t)b * A;
  const int per = (A + blockDim.x - 1) / blockDim.x, a0 = threadIdx.x * per, a1 = min(a0 + per, A);
  int cnt = 0;
  for (int a = a0; a < a1; ++a) {
    const bool pos = lab[a] > 0;
    cnt += pos;
    keys[a] = pos ? (hash32(seed ^ hash32((uint32_t)(b * A + a))) | 1u) : 0u;     // positives get a non-zero random key
  }
  scan[threadIdx.x] = cnt;
  __syncthreads();
  for (int off = 1; off < 1024; off <<= 1) {
    const int v = threadIdx.x >= off ? scan[threadIdx.x - off] : 0;
    __syncthreads();
    scan[threadIdx.x] += v;
    __syncthreads();
  }
  const int total = scan[1023];
  int before = scan[threadIdx.x] - cnt;
  __syncthreads();
  if (threadIdx.x == 0) { sel_count[b] = min(total, limit); sel_count[B + b] = total; }
  if (total <= limit) {
    for (int a = a0; a < a1; ++a) if (lab[a] > 0) sel[b * limit + before++] = a;
    return;
  }
  const uint32_t thr = block_kth_largest(keys, A, limit, hist, bc);   // keys are distinct with overwhelming probability; ties resolved below
  int g = 0, e = 0;
  for (int a = a0; a < a1; ++a) { g += keys[a] > thr; e += keys[a] == thr; }
  scan[threadIdx.x] = g;
  __syncthreads();
  for (int off = 1; off < 1024; off <<= 1) { const int v = threadIdx.x >= off ? scan[threadIdx.x - off] : 0; __syncthreads(); scan[threadIdx.x] += v; __syncthreads(); }
  const int total_g = scan[1023];
  int g_before = scan[threadIdx.x] - g;
  __syncthreads();
  scan[threadIdx.x] = e;
  __syncthreads();
  for (int off = 1; off < 1024; off <<= 1) { const int v = threadIdx.x >= off ? scan[threadIdx.x - off] : 0; __syncthreads(); scan[threadIdx.x] += v; __syncthreads(); }
  int e_before = scan[threadIdx.x] - e;
  for (int a = a0; a < a1; ++a) {
    if (keys[a] > thr) sel[b * limit + g_before++] = a;
    else if (keys[a] == thr) { if (e_before < limit - total_g) sel[b * limit + total_g + e_before] = a; ++e_before; }
  }
}

// ---- lincomb mask loss: sigmoid(proto @ coef^T), crop to the matched gt box (+1 px), BCE / box area; d_proto, d_coef ----
constexpr int kMaskPix = 128;            // pixels per block (one per thread)
constexpr int kMaxSel = 128;             // >= masks_to_train

__global__ void __launch_bounds__(kMaskPix) k_mask_loss(const float* __restrict__ proto, const float* __restrict__ coef, const float* __restrict__ matched,
                                                         const int32_t* __restrict__ best_gt, const int32_t* __restrict__ gt_off,
                                                         const uint8_t* __restrict__ ds_mask, const int32_t* __restrict__ sel,
                                                         const int32_t* __restrict__ sel_count, const int32_t* __restrict__ num_pos, int B, int A, int P, int K,
                                                         int limit, const float* __restrict__ gsd, float gs, double* __restrict__ acc, float* __restrict__ d_proto, float* __restrict__ d_coef) {
  extern __shared__ float sm[];
  float* s_coef = sm;                                  // [n][K]
  float* s_box = s_coef + kMaxSel * 32;                // [n][4]: x1, x2, y1, y2 of the crop (float)
  float* s_w = s_box + kMaxSel * 4;                    // [n] weight 1 / area * old / n
  int* s_gt = reinterpret_cast<int*>(s_w + kMaxSel);   // [n] global gt index
  int* s_a = s_gt + kMaxSel;                           // [n] anchor
  const int b = blockIdx.y, n = sel_count[b], n_all = sel_count[B + b];
  const int pix = blockIdx.x * kMaskPix + threadIdx.x;
  const bool live = pix < P * P;
  for (int i = threadIdx.x; i < n; i += kMaskPix) {
    const int a = sel[b * limit + i];
    const size_t r = (size_t)b * A + a;
    const float bx1 = matched[r * 4], by1 = matched[r * 4 + 1], bx2 = matched[r * 4 + 2], by2 = matched[r * 4 + 3];
    // sanitize_coordinates (box_utils.py:117-132) with padding 1 on the P x P grid
    const float xa = bx1 * (float)P, xb = bx2 * (float)P, ya = by1 * (float)P, yb_ = by2 * (float)P;
    s_box[i * 4 + 0] = fmaxf(fminf(xa, xb) - 1.f, 0.f); s_box[i * 4 + 1] = fminf(fmaxf(xa, xb) + 1.f, (float)P);
    s_box[i * 4 + 2] = fmaxf(fminf(ya, yb_) - 1.f, 0.f); s_box[i * 4 + 3] = fminf(fmaxf(ya, yb_) + 1.f, (float)P);
    const float area = (bx2 - bx1) * (by2 - by1);
    s_w[i] = (1.f / area) * (n_all > n ? (float)n_all / (float)n : 1.f);
    s_gt[i] = gt_off[b] + best_gt[r];
    s_a[i] = a;
    for (int k = 0; k < 32; ++k) s_coef[i * 32 + k] = k < K ? coef[r * K + k] : 0.f;
  }
  __syncthreads();
  float pr[32], dp[32];
#pragma unroll
  for (int k = 0; k < 32; ++k) { pr[k] = 0.f; dp[k] = 0.f; }
  const int py = live ? pix / P : 0, px = live ? pix - py * P : 0;
  if (live) {
    const float* p = proto + ((size_t)b * P * P + pix) * K;
#pragma unroll
    for (int k = 0; k < 32; ++k) if (k < K) pr[k] = p[k];
  }
  const float npos = (float)max(num_pos[B], 1);
  const float gscale = gs * (gsd ? gsd[2] : 1.f) / ((float)P * (float)P * npos);
  float loss = 0.f;
  const int lane = threadIdx.x & 31;
  for (int i = 0; i < n; ++i) {
    const bool inside = live && (float)px >= s_box[i * 4] && (float)px < s_box[i * 4 + 1] && (float)py >= s_box[i * 4 + 2] && (float)py < s_box[i * 4 + 3];
    const float t = live ? (float)ds_mask[(size_t)s_gt[i] * P * P + pix] : 0.f;
    const bool work = inside || t > 0.f;
    if (__ballot_sync(0xffffffffu, work) == 0u) continue;
    float g = 0.f;
    if (inside) {
      float z = 0.f;
#pragma unroll
      for (int k = 0; k < 32; ++k) z = fmaf(pr[k], s_coef[i * 32 + k], z);
      const float p = 1.f / (1.f + expf(-z));
      const float lp = fmaxf(logf(p), -100.f), lq = fmaxf(logf(1.f - p), -100.f);        // torch clamps the logs at -100
      loss += s_w[i] * -(t * lp + (1.f - t) * lq);
      // torch's chain: BCE backward (p - t) / max(p (1 - p), 1e-12), then sigmoid backward * p (1 - p).  The two cancel unless the
      // clamp bites: a saturated wrong prediction (p rounds to 0 or 1) then gets a vanishing gradient, as in the reference.
      g = s_w[i] * (p - t) * gscale;
      const float pq = p * (1.f - p);
      if (pq < 1e-12f) g = g / 1e-12f * pq;
#pragma unroll
      for (int k = 0; k < 32; ++k) dp[k] = fmaf(g, s_coef[i * 32 + k], dp[k]);
    } else if (t > 0.f) {
      loss += s_w[i] * 100.f * t;                                    // pred = 0 outside the crop: -t * max(log 0, -100)
    }
    if (d_coef && __ballot_sync(0xffffffffu, inside) != 0u) {
      const size_t r = ((size_t)b * A + s_a[i]) * K;
      for (int k = 0; k < K; ++k) {
        float v = g * pr[k];
#pragma unroll
        for (int off = 16; off > 0; off >>= 1) v += __shfl_xor_sync(0xffffffffu, v, off);
        if (lane == 0 && v != 0.f) atomicAdd(&d_coef[r + k], v);
      }
    }
  }
  if (d_proto && live) {
    float* o = d_proto + ((size_t)b * P * P + pix) * K;
#pragma unroll
    for (int k = 0; k < 32; ++k) if (k < K) o[k] = dp[k];
  }
#pragma unroll
  for (int off = 16; off > 0; off >>= 1) loss += __shfl_xor_sync(0xffffffffu, loss, off);
  if (lane == 0 && loss != 0.f) atomicAdd(&acc[2], (double)loss);
}

// ---- semantic segmentation loss: per-class max of the down-sampled gt masks as target, BCE with logits ----
__global__ void __launch_bounds__(128) k_semantic_loss(const float* __restrict__ seg, int ld, const float* __restrict__ gt, const int32_t* __restrict__ gt_off,
                                                       const float* __restrict__ masks, int S, int Hs, int NCs, const float* __restrict__ gsd, float gs0, double* __restrict__ acc,
                                                       float* __restrict__ d_seg) {
  const float gs = gs0 * (gsd ? gsd[3] : 1.f);
  const int b = blockIdx.y, pix = blockIdx.x * 128 + threadIdx.x;
  float loss = 0.f;
  if (pix < Hs * Hs) {
    const int g0 = gt_off[b], n = gt_off[b + 1] - g0;
    uint32_t bits[4] = {0u, 0u, 0u, 0u};                              // up to 128 classes
    const int oy = pix / Hs, ox = pix - oy * Hs;
    for (int j = 0; j < n; ++j) {
      if (bilinear_at(masks + (size_t)(g0 + j) * S * S, S, Hs, oy, ox) > 0.5f) {
        const int c = (int)gt[(size_t)(g0 + j) * 5 + 4];
        if (c >= 0 && c < 128) bits[c >> 5] |= 1u << (c & 31);
      }
    }
    const float* x = seg + ((size_t)b * Hs * Hs + pix) * ld;
    float* dx = d_seg ? d_seg + ((size_t)b * Hs * Hs + pix) * ld : nullptr;
    for (int c = 0; c < NCs; ++c) {
      const float v = x[c], t = (float)((bits[c >> 5] >> (c & 31)) & 1u);
      loss += fmaxf(v, 0.f) - v * t + log1pf(expf(-fabsf(v)));
      if (dx) dx[c] = gs * (1.f / (1.f + expf(-v)) - t);
    }
    if (dx) for (int c = NCs; c < ld; ++c) dx[c] = 0.f;
  }
#pragma unroll
  for (int off = 16; off > 0; off >>= 1) loss += __shfl_xor_sync(0xffffffffu, loss, off);
  if ((threadIdx.x & 31) == 0 && loss != 0.f) atomicAdd(&acc[3], (double)loss);
}

__global__ void k_finalize_losses(const double* __restrict__ acc, const int32_t* __restrict__ num_pos, int B, int P, int Hs, float ca, float ba, float ma, float sa,
                                  float* __restrict__ losses) {
  const double npos = (double)num_pos[B];
  losses[0] = (float)(ca * acc[0] / npos);
  losses[1] = (float)(ba * acc[1] / npos);
  losses[2] = (float)(ma * acc[2] / P / P / npos);
  losses[3] = (float)(sa * acc[3] / Hs / Hs / B);
}

__global__ void k_copy_debug(const int32_t* __restrict__ labels, const int32_t* __restrict__ best_gt, const float* __restrict__ offsets, const uint8_t* __restrict__ neg,
                             long long rows, int32_t* o_labels, int32_t* o_idx, float* o_offsets, uint8_t* o_neg) {
  for (long long i = blockIdx.x * 256LL + threadIdx.x; i < rows; i += (long long)gridDim.x * 256) {
    if (o_labels) o_labels[i] = labels[i];
    if (o_idx) o_idx[i] = best_gt[i];
    if (o_neg) o_neg[i] = neg[i];
    if (o_offsets) for (int q = 0; q < 4; ++q) o_offsets[i * 4 + q] = offsets[i * 4 + q];
  }
}

size_t carve(LossWs* w, char* base, const yb_loss_params& p, int total_gt) {
  size_t o = 0;
  auto take = [&](size_t bytes) { char* r = base ? base + o : nullptr; o += align_up(bytes, 256); return r; };
  const size_t BA = (size_t)p.batch * p.num_anchors;
  w->best_iou = (float*)take(BA * 4); w->best_gt = (int32_t*)take(BA * 4);
  w->gt_anchor = (int32_t*)take((size_t)p.batch * kMaxGt * 4);
  w->labels = (int32_t*)take(BA * 4); w->offsets = (float*)take(BA * 16); w->matched = (float*)take(BA * 16);
  w->mark = (uint32_t*)take(BA * 4); w->neg = (uint8_t*)take(BA);
  w->num_pos = (int32_t*)take((size_t)(p.batch + 1) * 4); w->logit_max = (uint32_t*)take(4); w->acc = (double*)take(4 * 8);
  w->ds_mask = (uint8_t*)take((size_t)(total_gt > 0 ? total_gt : 1) * p.proto_size * p.proto_size);
  w->sel = (int32_t*)take((size_t)p.batch * p.masks_to_train * 4); w->sel_count = (int32_t*)take((size_t)p.batch * 2 * 4);
  return o;
}

}  // namespace
}  // namespace yb

using namespace yb;

extern "C" size_t yb_losses_workspace_bytes(const yb_loss_params* p, int total_gt) {
  if (!p) return 0;
  LossWs w;
  return carve(&w, nullptr, *p, total_gt);
}

namespace yb {
// total_gt / max_gt_per_image only size grids and the workspace (the kernels read the real counts from gt_offset), so a caller that
// replays this launch sequence from a CUDA graph passes CAPACITIES here and the seed through device memory (seed_dev).
int losses_impl(const yb_loss_params* p, const float* cls, const float* box, const float* coef, const float* proto, const float* seg, int ld_seg,
                const float* anchors, const float* gt, const int32_t* gt_offset, const float* gt_masks, int total_gt, int max_gt_per_image,
                uint32_t seed, const uint32_t* seed_dev, const float* grad_scale, float* losses, float* d_cls, float* d_box, float* d_coef, float* d_proto,
                float* d_seg, int32_t* dbg_labels, int32_t* dbg_matched_idx, float* dbg_offsets, uint8_t* dbg_neg, void* workspace, size_t workspace_bytes,
                void* stream) {
  YB_REQUIRE(p && cls && box && coef && proto && seg && anchors && gt && gt_offset && gt_masks && losses && workspace, YB_ERR_INVALID, "yb_losses: NULL argument");
  YB_REQUIRE(p->batch >= 1 && p->num_anchors >= 1 && p->num_classes >= 2 && p->num_classes <= YB_MAX_CLASSES, YB_ERR_INVALID, "yb_losses: batch=%d anchors=%d classes=%d",
             p->batch, p->num_anchors, p->num_classes);
  YB_REQUIRE(p->coef_dim >= 1 && p->coef_dim <= 32, YB_ERR_UNSUPPORTED, "yb_losses: coef_dim=%d (<= 32)", p->coef_dim);
  YB_REQUIRE(p->masks_to_train >= 1 && p->masks_to_train <= kMaxSel, YB_ERR_UNSUPPORTED, "yb_losses: masks_to_train=%d (<= %d)", p->masks_to_train, kMaxSel);
  YB_REQUIRE(max_gt_per_image >= 0 && max_gt_per_image <= kMaxGt, YB_ERR_UNSUPPORTED, "yb_losses: %d ground-truth instances in one image (<= %d)", max_gt_per_image, kMaxGt);
  YB_REQUIRE(ld_seg >= p->num_classes - 1, YB_ERR_INVALID, "yb_losses: ld_seg=%d", ld_seg);
  LossWs w;
  const size_t need = carve(&w, (char*)workspace, *p, total_gt);
  YB_REQUIRE(workspace_bytes >= need, YB_ERR_INVALID, "yb_losses: workspace %zu < %zu bytes", workspace_bytes, need);
  cudaStream_t s = (cudaStream_t)stream;
  const int B = p->batch, A = p->num_anchors, NC = p->num_classes, K = p->coef_dim, P = p->proto_size, Hs = p->seg_size, S = p->mask_size;
  const long long rows = (long long)B * A;
  YB_CHECK_CUDA(cudaMemsetAsync(w.num_pos, 0, (size_t)(B + 1) * 4, s));
  YB_CHECK_CUDA(cudaMemsetAsync(w.acc, 0, 4 * 8, s));
  YB_CHECK_CUDA(cudaMemsetAsync(w.logit_max, 0, 4, s));
  YB_CHECK_CUDA(cudaMemsetAsync(w.gt_anchor, 0, (size_t)B * kMaxGt * 4, s));
  k_match_anchor<<<dim3(ceil_div(A, 256), B), 256, 0, s>>>(anchors, gt, gt_offset, A, w.best_iou, w.best_gt);
  YB_CHECK_LAUNCH();
  if (max_gt_per_image > 0) {
    k_match_gt<<<dim3(max_gt_per_image, B), 256, 0, s>>>(anchors, gt, gt_offset, A, w.gt_anchor);
    YB_CHECK_LAUNCH();
  }
  k_match_finalize<<<B, 256, 0, s>>>(anchors, gt, gt_offset, A, B, p->pos_iou_thr, p->neg_iou_thr, w.best_iou, w.best_gt, w.gt_anchor, w.labels, w.offsets,
                                     w.matched, w.num_pos);
  YB_CHECK_LAUNCH();
  k_logit_max<<<kSmCount * 4, 256, 0, s>>>(cls, rows * NC, w.logit_max);
  YB_CHECK_LAUNCH();
  k_ohem_mark<<<(unsigned)((rows + 7) / 8), 256, 0, s>>>(cls, w.labels, w.logit_max, rows, NC, w.mark);
  YB_CHECK_LAUNCH();
  k_ohem_select<<<B, 1024, 0, s>>>(w.mark, w.labels, w.num_pos, A, p->neg_pos_ratio, w.neg);
  YB_CHECK_LAUNCH();
  k_cls_box_loss<<<(unsigned)((rows + 7) / 8), 256, 0, s>>>(cls, box, w.labels, w.neg, w.offsets, w.num_pos, rows, NC, B, grad_scale, p->conf_alpha,
                                                            p->bbox_alpha, w.acc, d_cls, d_box);
  YB_CHECK_LAUNCH();
  if (total_gt > 0) {
    k_downsample_masks<<<dim3(ceil_div(P * P, 256), total_gt), 256, 0, s>>>(gt_masks, gt_offset, B, S, P, w.ds_mask);
    YB_CHECK_LAUNCH();
  }
  // the OHEM mark buffer is free again: reuse it for the random subset keys
  k_mask_select<<<B, 1024, 0, s>>>(w.labels, A, p->masks_to_train, seed, seed_dev, w.mark, w.sel, w.sel_count, B);
  YB_CHECK_LAUNCH();
  if (d_coef) YB_CHECK_CUDA(cudaMemsetAsync(d_coef, 0, (size_t)rows * K * 4, s));
  {
    const size_t smem = (size_t)(kMaxSel * 32 + kMaxSel * 4 + kMaxSel) * 4 + (size_t)kMaxSel * 2 * 4;
    k_mask_loss<<<dim3(ceil_div(P * P, kMaskPix), B), kMaskPix, smem, s>>>(proto, coef, w.matched, w.best_gt, gt_offset, w.ds_mask, w.sel, w.sel_count, w.num_pos,
                                                                            B, A, P, K, p->masks_to_train, grad_scale, p->mask_alpha, w.acc, d_proto, d_coef);
    YB_CHECK_LAUNCH();
  }
  k_semantic_loss<<<dim3(ceil_div(Hs * Hs, 128), B), 128, 0, s>>>(seg, ld_seg, gt, gt_offset, gt_masks, S, Hs, NC - 1, grad_scale,
                                                                   p->semantic_alpha / ((float)Hs * Hs * B), w.acc, d_seg);
  YB_CHECK_LAUNCH();
  k_finalize_losses<<<1, 1, 0, s>>>(w.acc, w.num_pos, B, P, Hs, p->conf_alpha, p->bbox_alpha, p->mask_alpha, p->semantic_alpha, losses);
  YB_CHECK_LAUNCH();
  if (dbg_labels || dbg_matched_idx || dbg_offsets || dbg_neg) {
    k_copy_debug<<<kSmCount, 256, 0, s>>>(w.labels, w.best_gt, w.offsets, w.neg, rows, dbg_labels, dbg_matched_idx, dbg_offsets, dbg_neg);
    YB_CHECK_LAUNCH();
  }
  return YB_OK;
}
}  // namespace yb

extern "C" int yb_losses(const yb_loss_params* p, const float* cls, const float* box, const float* coef, const float* proto, const float* seg, int ld_seg,
                         const float* anchors, const float* gt, const int32_t* gt_offset, const float* gt_masks, int total_gt, int max_gt_per_image,
                         uint32_t seed, const float* grad_scale, float* losses, float* d_cls, float* d_box, float* d_coef, float* d_proto, float* d_seg,
                         int32_t* dbg_labels, int32_t* dbg_matched_idx, float* dbg_offsets, uint8_t* dbg_neg, void* workspace, size_t workspace_bytes,
                         void* stream) {
  return yb::losses_impl(p, cls, box, coef, proto, seg, ld_seg, anchors, gt, gt_offset, gt_masks, total_gt, max_gt_per_image, seed, nullptr, grad_scale, losses,
                         d_cls, d_box, d_coef, d_proto, d_seg, dbg_labels, dbg_matched_idx, dbg_offsets, dbg_neg, workspace, workspace_bytes, stream);
}
