// Post-process chain on the GPU: score filter + SSD decode -> per-class Fast-NMS (or greedy hard
// NMS) -> cross-class top-k.  Replaces the reference's utils/output_utils.py:126-163 (nms),
// :11-43 (fast_nms), :84-123 (traditional_nms), utils/box_utils.py:8-37 (box_iou) and
// cython_nms.pyx:24-74.  Every float op that decides an index is a separately rounded fp32 op
// (__f*_rn, no FMA contraction) in the reference's order -- see DESIGN.md "index exactness".
//
// Data flow (per image b, A anchors, C classes incl. background, C1 = C-1):
//   phase 0  k_sample_cuts     grid (8, B): per-class score cuts from 1024 sampled anchors (Fast-NMS only)
//   phase 1  k_filter_decode   grid (ceil(A/128), B): streams cls[b] once (coalesced, the only
//            HBM-heavy step: A*C*4 bytes), keeps anchors whose fg max > thr, decodes their
//            boxes, and appends every (candidate, class) score that reaches the class's cut to the
//            class's candidate list (Fast-NMS; ~3 top_k entries per class instead of the whole
//            [C1][n] transposed score matrix of round 1, which cost 2.6x the algorithmic DRAM
//            traffic), or writes the transposed matrix scoreT[b][c][slot] (traditional NMS).
//   phase 2  k_class_fast_nms  grid (C1, B): radix-select the top_k scores of the class's list,
//            bitonic-sort them (score desc, anchor asc), k x k IoU upper triangle, keep rule.
//            (k_class_hard_nms is the traditional_nms alternative.)
//   phase 3  k_final_topk      grid (B): select max_det best of the <= C1*max_det survivors,
//            gather boxes / coefficient rows, write fixed-size detection records.
#include "common.cuh"
#include <math.h>
#include <stdlib.h>

namespace yb {

constexpr int kP1Anchors = 128;   // anchors per phase-1 tile
constexpr int kThreads = 256;
constexpr int kSortCap = 256;     // top_k, max_det <= 256
constexpr unsigned kFull = 0xffffffffu;
constexpr int kListCap = 2048;   // entries per (image, class) candidate list == the compact capacity of the per-class kernel
constexpr int kSamples = 512;     // sampled anchors per image (32 per warp of the sampling block)
constexpr int kStage = 16;        // per-class staging slots of a phase-1 tile before one global append per class

struct DetectWs {
  int* cand_count;    // [B]
  int* cand_anchor;   // [B][A]
  float4* cand_box;   // [B][A]   decoded, clipped corner boxes
  float* scoreT;      // [B][C1][A]
  int* cls_cnt;       // [B][C1]
  float* cls_score;   // [B][C1][KC]
  int* cls_anchor;    // [B][C1][KC]
  int* cls_slot;      // [B][C1][KC]
  int KC;
  // Fast-NMS path: per-class candidate lists instead of the transposed score matrix
  uint32_t* cut;      // [B][C1]   ordered-key threshold below which a class score cannot reach the class's top_k (0 = take all)
  int* list_cnt;      // [B][C1]   entries appended (may exceed kListCap: the list overflowed -> exact fallback)
  uint2* list;        // [B][C1][kListCap]  (ordered score key, candidate slot)
};

static size_t carve(DetectWs* w, char* base, int B, int A, int C1, int KC, bool traditional) {
  size_t off = 0;
  auto take = [&](size_t bytes) { size_t o = off; off = align_up(off + bytes, 256); return base ? base + o : (char*)nullptr; };
  w->cand_count = (int*)take(sizeof(int) * B);
  w->cand_anchor = (int*)take(sizeof(int) * (size_t)B * A);
  w->cand_box = (float4*)take(sizeof(float4) * (size_t)B * A);
  w->scoreT = (float*)take(traditional ? sizeof(float) * (size_t)B * C1 * A : 16);
  w->cls_cnt = (int*)take(sizeof(int) * (size_t)B * C1);
  w->cls_score = (float*)take(sizeof(float) * (size_t)B * C1 * KC);
  w->cls_anchor = (int*)take(sizeof(int) * (size_t)B * C1 * KC);
  w->cls_slot = (int*)take(sizeof(int) * (size_t)B * C1 * KC);
  w->KC = KC;
  w->cut = (uint32_t*)take(sizeof(uint32_t) * (size_t)B * C1);
  w->list_cnt = (int*)take(sizeof(int) * (size_t)B * C1);
  w->list = (uint2*)take(traditional ? 16 : sizeof(uint2) * (size_t)B * C1 * kListCap);
  return off;
}

// --------------------------------------------------------------------------------------------
// exact fp32 helpers
// --------------------------------------------------------------------------------------------
__device__ __forceinline__ float clip01(float x) { return x < 0.f ? 0.f : (x > 1.f ? 1.f : x); }  // NaN stays NaN

// utils/output_utils.py:148-153
__device__ __forceinline__ float4 decode_box(float4 b, float4 a, int no_clip) {
  float cx = __fadd_rn(a.x, __fmul_rn(__fmul_rn(b.x, 0.1f), a.z));
  float cy = __fadd_rn(a.y, __fmul_rn(__fmul_rn(b.y, 0.1f), a.w));
  // correctly-rounded fp32 exp (fp64 exp rounded once) -- matches oracle/postprocess_np.exp_f32
  float ew = (float)exp((double)__fmul_rn(b.z, 0.2f));
  float eh = (float)exp((double)__fmul_rn(b.w, 0.2f));
  float w = __fmul_rn(a.z, ew);
  float h = __fmul_rn(a.w, eh);
  float x1 = __fsub_rn(cx, __fmul_rn(w, 0.5f));
  float y1 = __fsub_rn(cy, __fmul_rn(h, 0.5f));
  float x2 = __fadd_rn(w, x1);
  float y2 = __fadd_rn(h, y1);
  if (no_clip) return make_float4(x1, y1, x2, y2);                 // the numpy twin nms_numpy has no clip (output_utils.py:186-190)
  return make_float4(clip01(x1), clip01(y1), clip01(x2), clip01(y2));
}

// utils/box_utils.py:28-36
__device__ __forceinline__ float iou_exact(float4 a, float4 b) {
  float w = __fsub_rn(fminf(a.z, b.z), fmaxf(a.x, b.x));
  float h = __fsub_rn(fminf(a.w, b.w), fmaxf(a.y, b.y));
  w = w < 0.f ? 0.f : w;
  h = h < 0.f ? 0.f : h;
  float inter = __fmul_rn(w, h);
  float area_a = __fmul_rn(__fsub_rn(a.z, a.x), __fsub_rn(a.w, a.y));
  float area_b = __fmul_rn(__fsub_rn(b.z, b.x), __fsub_rn(b.w, b.y));
  return __fdiv_rn(inter, __fsub_rn(__fadd_rn(area_a, area_b), inter));
}

// cython_nms.pyx:31, :63-70 ('+1' pixel convention)
__device__ __forceinline__ float area_plus1(float4 b) {
  return __fmul_rn(__fadd_rn(__fsub_rn(b.z, b.x), 1.f), __fadd_rn(__fsub_rn(b.w, b.y), 1.f));
}
__device__ __forceinline__ float ovr_plus1(float4 a, float area_a, float4 b, float area_b) {
  float xx1 = a.x >= b.x ? a.x : b.x, yy1 = a.y >= b.y ? a.y : b.y;
  float xx2 = a.z <= b.z ? a.z : b.z, yy2 = a.w <= b.w ? a.w : b.w;
  float w = __fadd_rn(__fsub_rn(xx2, xx1), 1.f), h = __fadd_rn(__fsub_rn(yy2, yy1), 1.f);
  w = 0.f >= w ? 0.f : w;
  h = 0.f >= h ? 0.f : h;
  float inter = __fmul_rn(w, h);
  return __fdiv_rn(inter, __fsub_rn(__fadd_rn(area_a, area_b), inter));
}

// --------------------------------------------------------------------------------------------
// phase 0 (Fast-NMS): per-class score cuts from a sample of the image's anchors.
// Only the top_k scores of a class row can matter (output_utils.py:12-14), so phase 1 appends an (anchor, class) score to the
// class's candidate list only if it is >= a per-class cut -- instead of materialising the whole [C1][n] transposed score matrix
// (2.6x the algorithmic DRAM traffic in round 1).  The cut comes from kSamples strided anchors: candidate samples are histogrammed
// per class; the cut is the lower edge of the bin where the sampled rank reaches ~3 top_k * (samples / anchors).  Exactness does not depend on the estimate: the per-class kernel takes the list only if it holds >= top_k entries and
// did not overflow (then the true top_k are all in it), otherwise it selects over the class column of `cls` itself.
// The histogram is LINEAR over each class's own sampled [min, max] key range (256 bins): score distributions that sit inside one
// binary octave (an untrained head: every class score ~ 1/81) still get a usable cut.
// --------------------------------------------------------------------------------------------
constexpr int kCutBins = 256;

// One warp per 32 sampled anchors, lane l owning classes l, l + 32, l + 64, ...: a sampled row is read with coalesced loads, the
// candidate test is a warp reduction, and every lane keeps the running min / max of ITS classes in registers (the first version
// gave each thread one sampled row and funnelled 80 min / max / histogram updates per thread through shared-memory atomics: 90 us).
__global__ void __launch_bounds__(kSamples)
k_sample_cuts(const float* __restrict__ cls, int A, int C, float score_thr, int top_k, DetectWs ws) {
  extern __shared__ int s_hist[];                         // [C1][kCutBins]
  __shared__ uint32_t s_lo[128], s_hi[128];               // per-class range of the sampled candidates' score keys (C1 <= 128 on this path)
  __shared__ int s_cnt;
  const int b = blockIdx.x, tid = threadIdx.x, C1 = C - 1, lane = tid & 31, w = tid >> 5;
  for (int i = tid; i < C1 * kCutBins; i += kSamples) s_hist[i] = 0;
  for (int c = tid; c < C1; c += kSamples) { s_lo[c] = 0xFFFFFFFFu; s_hi[c] = 0u; }
  if (tid == 0) s_cnt = 0;
  __syncthreads();
  constexpr int kCpl = 4;                                 // classes per lane (C1 <= 128)
  uint32_t lo[kCpl], hi[kCpl];
#pragma unroll
  for (int j = 0; j < kCpl; ++j) { lo[j] = 0xFFFFFFFFu; hi[j] = 0u; }
  uint32_t cand_mask = 0u;                                // bit k: sample w*32 + k is a candidate (output_utils.py:140-143)
  const float* base = cls + (size_t)b * A * C;
  constexpr int kGrp = 8;                                 // rows requested together: the loop is bound by load latency (~1 us per row from HBM)
  for (int k0 = 0; k0 < 32; k0 += kGrp) {
    float v[kGrp][kCpl];
#pragma unroll
    for (int g = 0; g < kGrp; ++g) {
      const long long a = ((long long)(w * 32 + k0 + g) * A) / kSamples;
      const float* row = base + (size_t)a * C + 1;
#pragma unroll
      for (int j = 0; j < kCpl; ++j) v[g][j] = (lane + 32 * j) < C1 ? __ldg(row + lane + 32 * j) : -INFINITY;
    }
#pragma unroll
    for (int g = 0; g < kGrp; ++g) {
      float m = -INFINITY; bool nan = false;
#pragma unroll
      for (int j = 0; j < kCpl; ++j) { nan |= (v[g][j] != v[g][j]); m = v[g][j] > m ? v[g][j] : m; }
#pragma unroll
      for (int off = 16; off > 0; off >>= 1) { const float o = __shfl_xor_sync(kFull, m, off); m = o > m ? o : m; }
      const bool cand = !__any_sync(kFull, nan) && m > score_thr;
      if (cand) {
        cand_mask |= 1u << (k0 + g);
#pragma unroll
        for (int j = 0; j < kCpl; ++j)
          if (lane + 32 * j < C1) { const uint32_t key = float_to_ordered(v[g][j]); lo[j] = min(lo[j], key); hi[j] = max(hi[j], key); }
      }
    }
  }
  if (cand_mask) {
#pragma unroll
    for (int j = 0; j < kCpl; ++j)
      if (lane + 32 * j < C1) { atomicMin(&s_lo[lane + 32 * j], lo[j]); atomicMax(&s_hi[lane + 32 * j], hi[j]); }
    if (lane == 0) atomicAdd(&s_cnt, __popc(cand_mask));
  }
  __syncthreads();
#pragma unroll
  for (int j = 0; j < kCpl; ++j) {                        // this lane's classes: range of the histogram
    const int c = lane + 32 * j;
    lo[j] = c < C1 ? s_lo[c] : 0u;
    hi[j] = c < C1 ? s_hi[c] : 0u;
  }
  for (int k0 = 0; k0 < 32; k0 += kGrp) {
    if (!((cand_mask >> k0) & ((1u << kGrp) - 1u))) continue;    // warp-uniform
    float v[kGrp][kCpl];
#pragma unroll
    for (int g = 0; g < kGrp; ++g) {
      const long long a = ((long long)(w * 32 + k0 + g) * A) / kSamples;
      const float* row = base + (size_t)a * C + 1;
#pragma unroll
      for (int j = 0; j < kCpl; ++j) v[g][j] = (lane + 32 * j) < C1 ? __ldg(row + lane + 32 * j) : 0.f;
    }
#pragma unroll
    for (int g = 0; g < kGrp; ++g) {
      if (!((cand_mask >> (k0 + g)) & 1u)) continue;
#pragma unroll
      for (int j = 0; j < kCpl; ++j) {
        const int c = lane + 32 * j;
        if (c < C1) {
          const uint32_t key = float_to_ordered(v[g][j]);
          const unsigned long long range = (unsigned long long)(hi[j] - lo[j]) + 1ull;
          atomicAdd(&s_hist[c * kCutBins + (int)((((unsigned long long)(key - lo[j])) << 8) / range)], 1);
        }
      }
    }
  }
  __syncthreads();
  const double est_n = (double)s_cnt * A / kSamples;      // estimated number of candidates of the image
  for (int c = w; c < C1; c += kSamples / 32) {           // one warp per class: lane l sums bins 8l .. 8l+7, suffix-scanned from the top
    uint32_t cut = 0u;
    if (est_n > 0.6 * kListCap) {                         // otherwise every candidate fits the list: take all
      const int want = (int)(3.0 * top_k * kSamples / A) + 6;      // sampled rank of ~3 top_k survivors, + margin
      int loc[8], sum = 0;
#pragma unroll
      for (int q = 0; q < 8; ++q) { loc[q] = s_hist[c * kCutBins + 255 - (lane * 8 + q)]; sum += loc[q]; }   // lane 0 holds the TOP 8 bins
      int incl = sum;
#pragma unroll
      for (int off = 1; off < 32; off <<= 1) { const int t = __shfl_up_sync(kFull, incl, off); if (lane >= off) incl += t; }
      const int excl = incl - sum;
      int bin = -1;
      if (excl < want && want <= incl) {
        int run = excl;
#pragma unroll
        for (int q = 0; q < 8; ++q) {
          run += loc[q];
          if (run >= want) { bin = 255 - (lane * 8 + q); break; }
        }
      }
      const unsigned found = __ballot_sync(kFull, bin >= 0);
      if (found) {
        bin = __shfl_sync(kFull, bin, __ffs(found) - 1);
        if (bin > 0) {                                    // bin 0 = the whole range: no cut
          const uint32_t l0 = s_lo[c];
          const unsigned long long range = (unsigned long long)(s_hi[c] - l0) + 1ull;
          cut = l0 + (uint32_t)(((unsigned long long)bin * range + 255ull) >> 8);   // smallest key of that bin
        }
      }
    }
    if (lane == 0) ws.cut[(size_t)b * C1 + c] = cut;
  }
}

// --------------------------------------------------------------------------------------------
// phase 1: filter + decode + (traditional: transpose | Fast-NMS: per-class candidate lists)
// --------------------------------------------------------------------------------------------
template <bool LISTS>
__global__ void __launch_bounds__(kThreads)
k_filter_decode(const float* __restrict__ cls, const float* __restrict__ box, const float* __restrict__ anchors,
                int A, int C, float score_thr, int no_clip, DetectWs ws) {
  extern __shared__ float tile[];                 // [kP1Anchors * C]
  __shared__ int s_kept[kP1Anchors];
  __shared__ int s_local[kP1Anchors];              // slot of the anchor inside this tile's kept list, -1 = not a candidate
  __shared__ int s_warp_cnt[kThreads / 32];
  __shared__ int s_warp_off[kThreads / 32];
  __shared__ int s_base, s_total;

  const int b = blockIdx.y, a0 = blockIdx.x * kP1Anchors;
  const int na = min(kP1Anchors, A - a0);
  const int tid = threadIdx.x, C1 = C - 1;

  const float* src = cls + ((size_t)b * A + a0) * C;
  const int nelem = na * C;
  {  // streamed once, 16 bytes per load where the tile's first element allows it (scalar head / tail: C is odd, A arbitrary)
    const int head = min(nelem, (int)((4 - ((((size_t)b * A + a0) * C) & 3)) & 3));
    const int nvec = (nelem - head) >> 2;
    if (tid < head) tile[tid] = __ldcs(src + tid);
    const float4* src4 = reinterpret_cast<const float4*>(src + head);
    for (int i = tid; i < nvec; i += kThreads) {
      const float4 v = __ldcs(src4 + i);
      if (head == 0) reinterpret_cast<float4*>(tile)[i] = v;
      else { float* t = tile + head + 4 * i; t[0] = v.x; t[1] = v.y; t[2] = v.z; t[3] = v.w; }
    }
    for (int i = head + 4 * nvec + tid; i < nelem; i += kThreads) tile[i] = __ldcs(src + i);
  }
  __syncthreads();

  // two threads per anchor: even/odd class columns (bank-conflict-free for odd C)
  const int la = tid >> 1, half = tid & 1;
  float m = -INFINITY;
  bool has_nan = false;
  if (la < na) {
    const float* row = tile + la * C;
    for (int c = 1 + half; c < C; c += 2) {
      float v = row[c];
      has_nan |= (v != v);
      m = v > m ? v : m;
    }
  }
  float mo = __shfl_xor_sync(kFull, m, 1);
  bool no = __shfl_xor_sync(kFull, (int)has_nan, 1) != 0;
  m = mo > m ? mo : m;
  has_nan |= no;
  // torch.max propagates NaN and NaN > thr is False (output_utils.py:140-143)
  const bool keep = (la < na) && (half == 0) && !has_nan && (m > score_thr);

  const unsigned bal = __ballot_sync(kFull, keep);
  const int w = tid >> 5, lane = tid & 31;
  if (lane == 0) s_warp_cnt[w] = __popc(bal);
  __syncthreads();
  if (tid == 0) {
    int tot = 0;
    for (int i = 0; i < kThreads / 32; ++i) { s_warp_off[i] = tot; tot += s_warp_cnt[i]; }
    s_total = tot;
    s_base = tot ? atomicAdd(&ws.cand_count[b], tot) : 0;
  }
  __syncthreads();
  const int total = s_total, base = s_base;
  if (total == 0) return;
  if (half == 0 && la < kP1Anchors) s_local[la] = -1;
  __syncwarp();
  if (keep) {
    const int local = s_warp_off[w] + __popc(bal & ((1u << lane) - 1u));
    s_kept[local] = la;
    s_local[la] = local;
    const int a = a0 + la;
    const size_t slot = (size_t)b * A + base + local;
    ws.cand_anchor[slot] = a;
    const float4 bb = __ldg(reinterpret_cast<const float4*>(box) + (size_t)b * A + a);
    const float4 an = __ldg(reinterpret_cast<const float4*>(anchors) + a);
    ws.cand_box[slot] = decode_box(bb, an, no_clip);
  }
  __syncthreads();
  if (!LISTS) {
    // class-major write: warp w takes classes w, w+8, ...; lanes run over the kept anchors
    float* dst = ws.scoreT + (size_t)b * C1 * A + base;
    for (int c = w; c < C1; c += kThreads / 32) {
      float* drow = dst + (size_t)c * A;
      for (int j = lane; j < total; j += 32) drow[j] = tile[s_kept[j] * C + c + 1];
    }
    return;
  }
  // per-class candidate lists.  The two threads of a kept anchor walk its even / odd classes; a score that reaches the class's cut
  // (a few per cent of them) is staged in shared memory, and each class is flushed to its global list with ONE atomic per tile.
  __shared__ int s_ccnt[128];                          // C1 <= 128 on this path
  __shared__ uint32_t s_cut[128];
  uint2* s_stage = reinterpret_cast<uint2*>(tile + (size_t)kP1Anchors * C + (((size_t)kP1Anchors * C) & 1));   // [C1][kStage], behind the tile (8-byte aligned)
  for (int c = tid; c < C1; c += kThreads) { s_ccnt[c] = 0; s_cut[c] = ws.cut[(size_t)b * C1 + c]; }
  __syncthreads();
  if (la < na && s_local[la] >= 0) {                   // kept anchor (both threads of the pair)
    const uint32_t slot = (uint32_t)(base + s_local[la]);
    const float* row = tile + la * C;
    for (int c = 1 + half; c < C; c += 2) {
      const uint32_t key = float_to_ordered(row[c]);
      if (key >= s_cut[c - 1]) {
        const int pos = atomicAdd(&s_ccnt[c - 1], 1);
        if (pos < kStage) s_stage[(c - 1) * kStage + pos] = make_uint2(key, slot);
        else {                                           // tile-local overflow (cut 0 on a dense tile): append directly
          const int g = atomicAdd(&ws.list_cnt[(size_t)b * C1 + c - 1], 1);
          if (g < kListCap) ws.list[((size_t)b * C1 + c - 1) * kListCap + g] = make_uint2(key, slot);
        }
      }
    }
  }
  __syncthreads();
  // flush: one global atomic per class with staged entries, ALL issued at once (thread c reserves class c's range; a warp that
  // reserves and writes class after class pays one global round trip per class, which dominated this kernel), then the copies
  __shared__ int s_gbase[128];
  for (int c = tid; c < C1; c += kThreads) {
    const int cnt = min(s_ccnt[c], kStage);
    s_gbase[c] = cnt ? atomicAdd(&ws.list_cnt[(size_t)b * C1 + c], cnt) : 0;
  }
  __syncthreads();
  for (int e = tid; e < C1 * kStage; e += kThreads) {
    const int c = e / kStage, i = e - c * kStage;
    if (i < min(s_ccnt[c], kStage) && s_gbase[c] + i < kListCap) ws.list[((size_t)b * C1 + c) * kListCap + s_gbase[c] + i] = s_stage[e];
  }
}

// --------------------------------------------------------------------------------------------
// block-wide radix select: threshold of the kk-th LARGEST value among valid elements
// --------------------------------------------------------------------------------------------
struct SelectResult { uint32_t thresh; int need_eq; int cnt_eq; };

template <class F>
__device__ SelectResult block_select_kth_largest(int n, int kk, F value, int* hist /*[256]*/, int* s_tmp /*[4]*/) {
  uint32_t desired = 0, mask = 0;
  int cnt_eq = 0;
  const int tid = threadIdx.x, nt = blockDim.x;
  for (int shift = 24; shift >= 0; shift -= 8) {
    for (int i = tid; i < 256; i += nt) hist[i] = 0;
    __syncthreads();
    for (int i = tid; i < n; i += nt) {
      uint32_t v;
      if (value(i, v) && (v & mask) == desired) atomicAdd(&hist[(v >> shift) & 255u], 1);
    }
    __syncthreads();
    if (tid < 32) {
      int loc[8], sum = 0;
#pragma unroll
      for (int q = 0; q < 8; ++q) { loc[q] = hist[255 - (tid * 8 + q)]; sum += loc[q]; }
      int incl = sum;
#pragma unroll
      for (int off = 1; off < 32; off <<= 1) {
        int t = __shfl_up_sync(kFull, incl, off);
        if (tid >= off) incl += t;
      }
      const int excl = incl - sum;
      if (excl < kk && kk <= incl) {
        int run = excl;
#pragma unroll
        for (int q = 0; q < 8; ++q) {
          if (run + loc[q] >= kk) { s_tmp[0] = 255 - (tid * 8 + q); s_tmp[1] = kk - run; s_tmp[2] = loc[q]; break; }
          run += loc[q];
        }
      }
    }
    __syncthreads();
    const int bin = s_tmp[0];
    kk = s_tmp[1];
    cnt_eq = s_tmp[2];
    desired |= (uint32_t)bin << shift;
    mask |= 0xFFu << shift;
    __syncthreads();
  }
  return {desired, kk, cnt_eq};
}

// 256-element bitonic sort, ascending by 64-bit key, with a 32-bit payload
__device__ void bitonic_sort_256(unsigned long long* key, int* val) {
  const int tid = threadIdx.x;
  for (int size = 2; size <= kSortCap; size <<= 1) {
    for (int stride = size >> 1; stride > 0; stride >>= 1) {
      __syncthreads();
      const int p = tid ^ stride;
      if (p > tid && tid < kSortCap) {
        const bool asc = (tid & size) == 0;
        unsigned long long a = key[tid], b = key[p];
        if ((a > b) == asc) {
          key[tid] = b; key[p] = a;
          int t = val[tid]; val[tid] = val[p]; val[p] = t;
        }
      }
    }
  }
  __syncthreads();
}

// --------------------------------------------------------------------------------------------
// phase 2 (Fast-NMS): one block per (class, image)   utils/output_utils.py:11-31
//   stage 1  load the class's candidate list written by phase 1 (every candidate whose class score reaches the sampled cut,
//            phase 0) into shared memory; if the list cannot be trusted to hold the class's top_k (fewer than top_k entries,
//            or it overflowed kListCap) the exact selection runs over the class column of `cls` instead (rare)
//   stage 2  exact top_k of the compact list: 8-bit radix select, tie-break on anchor index,
//            bitonic sort of the <= 256 winners by (score desc, anchor asc)
//   stage 3  k x k IoU upper triangle, keep rule, ordered compaction of the survivors
// --------------------------------------------------------------------------------------------
constexpr int kCompactCap = kListCap;

__device__ void bitonic_sort_256_desc_u32(uint32_t* key) {
  const int tid = threadIdx.x;
  for (int size = 2; size <= 256; size <<= 1) {
    for (int stride = size >> 1; stride > 0; stride >>= 1) {
      __syncthreads();
      const int p = tid ^ stride;
      if (p > tid) {
        const bool desc = (tid & size) == 0;
        const uint32_t a = key[tid], b = key[p];
        if ((a < b) == desc) { key[tid] = b; key[p] = a; }
      }
    }
  }
  __syncthreads();
}

// IoU(a,b) <= thr with the reference's fp32 rounding (utils/box_utils.py:28-36): a 2-instruction
// reciprocal estimate decides unless it lands within 4e-6 of the threshold, where the exactly
// rounded division is used.
__device__ __forceinline__ bool iou_le(float4 a, float area_a, float4 b, float area_b, float thr) {
  float w = __fsub_rn(fminf(a.z, b.z), fmaxf(a.x, b.x));
  float h = __fsub_rn(fminf(a.w, b.w), fmaxf(a.y, b.y));
  w = w < 0.f ? 0.f : w;
  h = h < 0.f ? 0.f : h;
  const float inter = __fmul_rn(w, h);
  const float uni = __fsub_rn(__fadd_rn(area_a, area_b), inter);
  const float q = __fdividef(inter, uni);            // MUFU.RCP + FMUL, <= 2 ulp
  if (q != q) return false;                          // 0/0 (two zero-area boxes): NaN <= thr is false, exactly as the IEEE quotient
  if (fabsf(q - thr) > 4e-6f) return q <= thr;
  return __fdiv_rn(inter, uni) <= thr;
}

__global__ void __launch_bounds__(kThreads)
k_class_fast_nms(const float* __restrict__ cls, int A, int C1, int top_k, float iou_thr, DetectWs ws) {
  __shared__ uint32_t s_ckey[kCompactCap];         // compact candidates: ordered score keys
  __shared__ int s_cidx[kCompactCap];              //                    : slot in the candidate list
  __shared__ unsigned long long s_sort[kSortCap];
  __shared__ int s_slot[kSortCap];
  __shared__ float4 s_box[kSortCap];
  __shared__ float s_area[kSortCap];
  __shared__ int s_hist[256];
  __shared__ int s_tmp[4];
  __shared__ int s_cnt, s_m;
  __shared__ int s_wcnt[kThreads / 32];
  __shared__ int s_keep[kSortCap];

  const int c = blockIdx.x, b = blockIdx.y, tid = threadIdx.x, lane = tid & 31;
  const int n = ws.cand_count[b];
  int* out_cnt = ws.cls_cnt + (size_t)b * C1 + c;
  if (n == 0) { if (tid == 0) *out_cnt = 0; return; }
  const int k = min(top_k, n);
  const int* canchor = ws.cand_anchor + (size_t)b * A;
  if (tid == 0) { s_cnt = 0; s_m = 0; }

  // ---- stage 1: the class's candidate list (phase 1), or -- when the list cannot hold the top_k for sure -- the class column ----
  const int lcnt = ws.list_cnt[(size_t)b * C1 + c];
  const bool full_scan = lcnt < k || lcnt > kListCap;      // cut too high / list overflowed (rare): exact selection over all candidates
  int m = full_scan ? n : lcnt;
  if (!full_scan) {
    const uint2* lst = ws.list + ((size_t)b * C1 + c) * kListCap;
    for (int i = tid; i < m; i += kThreads) { const uint2 e = lst[i]; s_ckey[i] = e.x; s_cidx[i] = (int)e.y; }
  }
  __syncthreads();
  const float* col = cls + (size_t)b * A * (C1 + 1) + c + 1;
  auto key_of = [&](int i) -> uint32_t { return full_scan ? float_to_ordered(__ldg(col + (size_t)canchor[i] * (C1 + 1))) : s_ckey[i]; };
  auto slot_of = [&](int i) -> int { return full_scan ? i : s_cidx[i]; };

  // ---- stage 2: exact top-k by (score desc, anchor asc) ----------------------------------------
  // Fast path (the usual case): ONE histogram pass over 256 linear bins of [min key, max key] finds the bin holding the k-th
  // score; everything above it is in, the few elements of that bin are ranked exactly among themselves (score desc, anchor asc).
  // The byte-wise radix select below needs 4+ passes whose first ones pile every key of a class onto two or three bins
  // (shared-memory atomics on one address serialise); it stays as the fallback for heavy ties / the full-column scan.
  bool selected = false;
  if (m > k && !full_scan) {
    uint32_t lo = 0xFFFFFFFFu, hi = 0u;
    for (int i = tid; i < m; i += kThreads) { const uint32_t v = s_ckey[i]; lo = min(lo, v); hi = max(hi, v); }
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) { lo = min(lo, __shfl_xor_sync(kFull, lo, off)); hi = max(hi, __shfl_xor_sync(kFull, hi, off)); }
    uint32_t* s_red = reinterpret_cast<uint32_t*>(s_area);            // [16] scratch (s_area is written only in stage 3)
    if (lane == 0) { s_red[tid >> 5] = lo; s_red[8 + (tid >> 5)] = hi; }
    for (int i = tid; i < 256; i += kThreads) s_hist[i] = 0;
    __syncthreads();
    lo = s_red[0]; hi = s_red[8];
#pragma unroll
    for (int q = 1; q < kThreads / 32; ++q) { lo = min(lo, s_red[q]); hi = max(hi, s_red[8 + q]); }
    const unsigned long long range = (unsigned long long)(hi - lo) + 1ull;
    auto bin_of = [&](uint32_t v) -> int { return (int)((((unsigned long long)(v - lo)) << 8) / range); };
    for (int i = tid; i < m; i += kThreads) atomicAdd(&s_hist[bin_of(s_ckey[i])], 1);
    __syncthreads();
    if (tid < 32) {                                                    // warp 0: bin of the k-th largest, count above it
      int loc[8], sum = 0;
#pragma unroll
      for (int q = 0; q < 8; ++q) { loc[q] = s_hist[255 - (tid * 8 + q)]; sum += loc[q]; }
      int incl = sum;
#pragma unroll
      for (int off = 1; off < 32; off <<= 1) { const int t2 = __shfl_up_sync(kFull, incl, off); if (tid >= off) incl += t2; }
      const int excl = incl - sum;
      if (excl < k && k <= incl) {
        int run = excl;
#pragma unroll
        for (int q = 0; q < 8; ++q) {
          if (run + loc[q] >= k) { s_tmp[0] = 255 - (tid * 8 + q); s_tmp[1] = k - run; s_tmp[2] = loc[q]; break; }
          run += loc[q];
        }
      }
    }
    __syncthreads();
    const int bstar = s_tmp[0], need = s_tmp[1], e = s_tmp[2];
    if (e <= kSortCap) {
      unsigned long long* s_bkey = reinterpret_cast<unsigned long long*>(s_box);       // [256] boundary-bin elements (s_box is written in stage 3)
      int* s_bslot = reinterpret_cast<int*>(s_bkey + kSortCap);                         // [256]
      for (int i = tid; i < m; i += kThreads) {
        const uint32_t key = s_ckey[i];
        const int bn = bin_of(key);
        if (bn < bstar) continue;
        const int slot = s_cidx[i];
        const unsigned long long comp = ((unsigned long long)(~key) << 32) | (uint32_t)canchor[slot];
        if (bn > bstar) { const int pos = atomicAdd(&s_cnt, 1); s_sort[pos] = comp; s_slot[pos] = slot; }
        else { const int q = atomicAdd(&s_m, 1); s_bkey[q] = comp; s_bslot[q] = slot; }
      }
      __syncthreads();
      if (tid < e) {                                                   // exact rank inside the boundary bin (smaller composite = better)
        const unsigned long long mine = s_bkey[tid];
        int rank = 0;
        for (int j = 0; j < e; ++j) rank += s_bkey[j] < mine ? 1 : 0;
        if (rank < need) { const int pos = atomicAdd(&s_cnt, 1); s_sort[pos] = mine; s_slot[pos] = s_bslot[tid]; }
      }
      selected = true;
    }
    __syncthreads();
  }
  if (selected) {
    // winners are in s_sort / s_slot
  } else if (m > k) {
    SelectResult r = block_select_kth_largest(m, k, [&](int i, uint32_t& v) { v = key_of(i); return true; }, s_hist, s_tmp);
    uint32_t anchor_max = 0xFFFFFFFFu;   // take ties with anchor <= anchor_max
    if (r.cnt_eq > r.need_eq) {
      // exact score ties at the cut: the reference's stable sort keeps the lowest candidate
      // indices (== lowest anchors).  Select the need_eq smallest anchors among the ties.
      const uint32_t T = r.thresh;
      SelectResult r2 = block_select_kth_largest(
          m, r.need_eq, [&](int i, uint32_t& v) { v = ~(uint32_t)canchor[slot_of(i)]; return key_of(i) == T; }, s_hist, s_tmp);
      anchor_max = ~r2.thresh;
    }
    for (int i = tid; i < m; i += kThreads) {
      const uint32_t key = key_of(i);
      if (key >= r.thresh) {
        const int slot = slot_of(i);
        const uint32_t anc = (uint32_t)canchor[slot];
        if (key > r.thresh || anc <= anchor_max) {
          const int pos = atomicAdd(&s_cnt, 1);
          if (pos < kSortCap) { s_sort[pos] = ((unsigned long long)(~key) << 32) | anc; s_slot[pos] = slot; }
        }
      }
    }
  } else {
    for (int i = tid; i < m; i += kThreads) {
      const int slot = slot_of(i);
      s_sort[i] = ((unsigned long long)(~key_of(i)) << 32) | (uint32_t)canchor[slot];
      s_slot[i] = slot;
    }
  }
  __syncthreads();
  {  // sort the k winners by (score desc, anchor asc): the 64-bit keys are distinct, so an element's sorted position is the number of
     // smaller keys -- one pass of broadcast shared-memory reads instead of the 36 barrier steps of a 256-element bitonic network
    unsigned long long mykey = 0ull; int myslot = -1, rank = 0;
    if (tid < k) {
      mykey = s_sort[tid]; myslot = s_slot[tid];
      for (int j = 0; j < k; ++j) rank += s_sort[j] < mykey ? 1 : 0;
    }
    __syncthreads();
    if (tid < k) { s_sort[rank] = mykey; s_slot[rank] = myslot; }
    __syncthreads();
  }

  // ---- stage 3: Fast-NMS keep rule ----------------------------------------------------------------
  const float4* cbox = ws.cand_box + (size_t)b * A;
  if (tid < k) {
    const float4 bx = cbox[s_slot[tid]];
    s_box[tid] = bx;
    s_area[tid] = __fmul_rn(__fsub_rn(bx.z, bx.x), __fsub_rn(bx.w, bx.y));
  }
  // keep_j = (0 <= thr) && all_{i<j} IoU(i,j) <= thr   (NaN compares false -> dropped;
  // the triu'd matrix contributes the 0 -- output_utils.py:21-26).
  if (tid < kSortCap) s_keep[tid] = (tid < k && 0.f <= iou_thr) ? 1 : 0;
  __syncthreads();
  for (int idx = tid; idx < k * 4; idx += kThreads) {          // 4 threads per column j, rows interleaved
    const int sub = idx & 3, j = idx >> 2;
    const float4 bj = s_box[j];
    const float aj = s_area[j];
    bool ok = true;
    for (int i = sub; i < j && ok; i += 4) ok = iou_le(s_box[i], s_area[i], bj, aj, iou_thr);
    if (!ok) s_keep[j] = 0;
  }
  __syncthreads();
  const bool keep = tid < k && s_keep[tid] != 0;
  const unsigned bal = __ballot_sync(kFull, keep);
  const int w = tid >> 5;
  if (lane == 0) s_wcnt[w] = __popc(bal);
  __syncthreads();
  int off = 0, tot = 0;
  for (int i = 0; i < kThreads / 32; ++i) { if (i < w) off += s_wcnt[i]; tot += s_wcnt[i]; }
  if (keep) {
    const int r = off + __popc(bal & ((1u << lane) - 1u));
    const size_t o = ((size_t)b * C1 + c) * ws.KC + r;
    const unsigned long long sk = s_sort[tid];
    ws.cls_score[o] = ordered_to_float(~(uint32_t)(sk >> 32));
    ws.cls_anchor[o] = (int)(uint32_t)sk;
    ws.cls_slot[o] = s_slot[tid];
  }
  if (tid == 0) *out_cnt = tot;
}

// --------------------------------------------------------------------------------------------
// phase 2 (traditional): greedy per-class NMS in pixel coords   output_utils.py:84-113 +
// cython_nms.pyx:24-74.  Survivors are found in descending score order (ties: larger anchor
// first), but the cross-class ranking (output_utils.py:115-117, k_final_topk) breaks ties by
// ascending anchor.  So the class keeps the max_keep best survivors by (score desc, anchor asc):
// the first max_keep in greedy order, except that the group tied at the max_keep-th score must
// hold the SMALLEST tied anchors.  After max_keep survivors the loop runs on while the winner ties
// with that score; each such winner has a smaller anchor than every stored one of the group and
// replaces the group's oldest (= largest-anchor) entry, so at most max_keep entries are stored.
// --------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(kThreads)
k_class_hard_nms(int A, int C1, float score_thr, float iou_thr, float img_size, int max_keep, DetectWs ws) {
  extern __shared__ float s_sc[];                  // [n] live scores (-inf = removed)
  __shared__ float s_best[kThreads / 32];
  __shared__ int s_besti[kThreads / 32];
  __shared__ int s_win;
  const int c = blockIdx.x, b = blockIdx.y, tid = threadIdx.x, lane = tid & 31, w = tid >> 5;
  const int n = ws.cand_count[b];
  const float* row = ws.scoreT + ((size_t)b * C1 + c) * A;
  const int* canchor = ws.cand_anchor + (size_t)b * A;
  const float4* cbox = ws.cand_box + (size_t)b * A;
  for (int i = tid; i < n; i += kThreads) { float s = row[i]; s_sc[i] = (s > score_thr) ? s : -INFINITY; }
  __syncthreads();
  int kept = 0;                                    // stored survivors (<= max_keep)
  float run_score = -INFINITY;                     // thread 0: score of the last stored survivor,
  int run_start = 0, replaced = 0;                 //   first slot holding it, tied winners past max_keep
  while (true) {
    // argmax (score desc, ties: larger anchor first == reversed stable ascending argsort)
    float best = -INFINITY; int besti = -1; int besta = -1;
    for (int i = tid; i < n; i += kThreads) {
      float s = s_sc[i];
      if (s > best || (s == best && s > -INFINITY && canchor[i] > besta)) { best = s; besti = i; besta = canchor[i]; }
    }
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) {
      float ob = __shfl_xor_sync(kFull, best, off);
      int oi = __shfl_xor_sync(kFull, besti, off);
      int oa = __shfl_xor_sync(kFull, besta, off);
      if (ob > best || (ob == best && oa > besta)) { best = ob; besti = oi; besta = oa; }
    }
    if (lane == 0) { s_best[w] = best; s_besti[w] = besti; }
    __syncthreads();
    if (tid == 0) {
      float bb = -INFINITY; int bi = -1, ba = -1;
      for (int i = 0; i < kThreads / 32; ++i) {
        int ii = s_besti[i];
        if (ii < 0) continue;
        int aa = canchor[ii];
        if (s_best[i] > bb || (s_best[i] == bb && aa > ba)) { bb = s_best[i]; bi = ii; ba = aa; }
      }
      int win = (bb > -INFINITY) ? bi : -1, slot = kept;
      if (win >= 0 && kept < max_keep) {
        if (bb != run_score) { run_score = bb; run_start = kept; }
      } else if (win >= 0 && bb == run_score) {     // tied with the max_keep-th survivor: replace the group's largest anchor
        slot = run_start + replaced % (max_keep - run_start);
        ++replaced;
      } else {
        win = -1;                                  // below the cut (or none left): no later survivor can rank in
      }
      s_win = win;
      if (win >= 0) {
        const size_t o = ((size_t)b * C1 + c) * ws.KC + slot;
        ws.cls_score[o] = bb; ws.cls_anchor[o] = ba; ws.cls_slot[o] = bi;
      }
    }
    __syncthreads();
    const int win = s_win;
    if (win < 0) break;
    if (kept < max_keep) ++kept;
    float4 bw = cbox[win];
    bw = make_float4(__fmul_rn(bw.x, img_size), __fmul_rn(bw.y, img_size), __fmul_rn(bw.z, img_size), __fmul_rn(bw.w, img_size));
    const float aw = area_plus1(bw);
    for (int i = tid; i < n; i += kThreads) {
      if (i == win) { s_sc[i] = -INFINITY; continue; }
      if (s_sc[i] > -INFINITY) {
        float4 bi = cbox[i];
        bi = make_float4(__fmul_rn(bi.x, img_size), __fmul_rn(bi.y, img_size), __fmul_rn(bi.z, img_size), __fmul_rn(bi.w, img_size));
        if (ovr_plus1(bw, aw, bi, area_plus1(bi)) >= iou_thr) s_sc[i] = -INFINITY;
      }
    }
    __syncthreads();
  }
  if (tid == 0) ws.cls_cnt[(size_t)b * C1 + c] = kept;
}

// --------------------------------------------------------------------------------------------
// phase 3: cross-class top max_det   utils/output_utils.py:33-41 / :115-123
// --------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(kThreads)
k_final_topk(const float* __restrict__ coef, int A, int C1, int max_det, int coef_dim, int traditional, float img_size,
             DetectWs ws, int32_t* out_count, int32_t* out_class, int32_t* out_anchor, float* out_score,
             float* out_box, float* out_coef) {
  extern __shared__ int s_ccnt[];                  // [C1] min(cls_cnt, max_det), then [C1*max_det] keys, [C1*max_det] tie keys
  __shared__ unsigned long long s_sort[kSortCap];
  __shared__ int s_idx[kSortCap];
  __shared__ int s_hist[256];
  __shared__ int s_tmp[4];
  __shared__ int s_cnt, s_total;
  const int b = blockIdx.x, tid = threadIdx.x;
  const int KC = ws.KC;
  const bool have = ws.cand_count[b] > 0;
  if (tid == 0) { s_cnt = 0; s_total = 0; }
  __syncthreads();
  int loc = 0;
  for (int c = tid; c < C1; c += kThreads) {
    int v = have ? min(ws.cls_cnt[(size_t)b * C1 + c], max_det) : 0;
    s_ccnt[c] = v; loc += v;
  }
  if (loc) atomicAdd(&s_total, loc);
  __syncthreads();
  const int total = s_total;
  const int d = min(total, max_det);
  const int dense = C1 * max_det;
  const float* cscore = ws.cls_score + (size_t)b * C1 * KC;
  const int* canchor = ws.cls_anchor + (size_t)b * C1 * KC;
  // stage the (score key, tie key) of every surviving candidate in shared memory once; key 0 = empty slot
  uint32_t* s_key = reinterpret_cast<uint32_t*>(s_ccnt + ((C1 + 3) & ~3));
  uint32_t* s_sec = s_key + dense;
  for (int i = tid; i < dense; i += kThreads) {
    const int c = i / max_det, r = i - c * max_det;
    uint32_t key = 0, sec = 0xFFFFFFFFu;
    if (r < s_ccnt[c]) {
      key = float_to_ordered(cscore[c * KC + r]);
      sec = (uint32_t)c * (uint32_t)A + (uint32_t)canchor[c * KC + r];   // class-major, anchor-ascending tie order
    }
    s_key[i] = key; s_sec[i] = sec;
  }
  __syncthreads();
  auto valid_key = [&](int i, uint32_t& key, uint32_t& sec) -> bool {
    key = s_key[i]; sec = s_sec[i];
    return key != 0u;
  };
  if (total > d) {
    SelectResult r = block_select_kth_largest(dense, d, [&](int i, uint32_t& v) { uint32_t s; return valid_key(i, v, s); }, s_hist, s_tmp);
    uint32_t sec_max = 0xFFFFFFFFu;
    if (r.cnt_eq > r.need_eq) {
      const uint32_t T = r.thresh;
      SelectResult r2 = block_select_kth_largest(
          dense, r.need_eq, [&](int i, uint32_t& v) { uint32_t k2, s; if (!valid_key(i, k2, s)) return false; v = ~s; return k2 == T; },
          s_hist, s_tmp);
      sec_max = ~r2.thresh;
    }
    for (int i = tid; i < dense; i += kThreads) {
      uint32_t key, sec;
      if (valid_key(i, key, sec) && (key > r.thresh || (key == r.thresh && sec <= sec_max))) {
        const int pos = atomicAdd(&s_cnt, 1);
        if (pos < kSortCap) { s_sort[pos] = ((unsigned long long)(~key) << 32) | sec; s_idx[pos] = i; }
      }
    }
  } else {
    for (int i = tid; i < dense; i += kThreads) {
      uint32_t key, sec;
      if (valid_key(i, key, sec)) {
        const int pos = atomicAdd(&s_cnt, 1);
        if (pos < kSortCap) { s_sort[pos] = ((unsigned long long)(~key) << 32) | sec; s_idx[pos] = i; }
      }
    }
  }
  __syncthreads();
  for (int i = d + tid; i < kSortCap; i += kThreads) { s_sort[i] = ~0ull; s_idx[i] = -1; }
  bitonic_sort_256(s_sort, s_idx);

  if (tid == 0) out_count[b] = d;
  const float4* cbox = ws.cand_box + (size_t)b * A;
  for (int j = tid; j < max_det; j += kThreads) {
    const size_t o = (size_t)b * max_det + j;
    if (j < d) {
      const int i = s_idx[j];
      const int c = i / max_det, r = i - c * max_det;
      out_class[o] = c;
      out_anchor[o] = canchor[c * KC + r];
      out_score[o] = cscore[c * KC + r];
      float4 bx = cbox[ws.cls_slot[(size_t)b * C1 * KC + c * KC + r]];
      if (traditional) {   // output_utils.py:90,:123  (boxes * img_size) / img_size
        bx = make_float4(__fdiv_rn(__fmul_rn(bx.x, img_size), img_size), __fdiv_rn(__fmul_rn(bx.y, img_size), img_size),
                         __fdiv_rn(__fmul_rn(bx.z, img_size), img_size), __fdiv_rn(__fmul_rn(bx.w, img_size), img_size));
      }
      reinterpret_cast<float4*>(out_box)[o] = bx;
    } else {
      out_class[o] = 0; out_anchor[o] = 0; out_score[o] = 0.f;
      reinterpret_cast<float4*>(out_box)[o] = make_float4(0.f, 0.f, 0.f, 0.f);
    }
  }
  if (out_coef) {
    for (int e = tid; e < max_det * coef_dim; e += kThreads) {
      const int j = e / coef_dim, q = e - j * coef_dim;
      float v = 0.f;
      if (j < d) {
        const int i = s_idx[j];
        const int c = i / max_det, r = i - c * max_det;
        v = __ldg(coef + ((size_t)b * A + canchor[c * KC + r]) * coef_dim + q);
      }
      out_coef[((size_t)b * max_det + j) * coef_dim + q] = v;
    }
  }
}

// --------------------------------------------------------------------------------------------
// standalone greedy NMS (cython_nms.pyx:24-74): one block, argmax-iterate
// --------------------------------------------------------------------------------------------
constexpr int kHardThreads = 1024;
__global__ void __launch_bounds__(kHardThreads)
k_hard_nms(const float* __restrict__ dets, int n, float thresh, uint8_t* keep /* 2 = undecided */) {
  __shared__ float s_best[kHardThreads / 32];
  __shared__ int s_besti[kHardThreads / 32];
  __shared__ int s_win;
  const int tid = threadIdx.x, lane = tid & 31, w = tid >> 5;
  for (int i = tid; i < n; i += kHardThreads) keep[i] = 2;
  __syncthreads();
  while (true) {
    float best = -INFINITY; int besti = -1;
    for (int i = tid; i < n; i += kHardThreads) {
      if (keep[i] != 2) continue;
      const float s = dets[i * 5 + 4];
      // descending score, ties: larger original index first (reversed stable argsort)
      if (besti < 0 || s > best || (s == best && i > besti)) { best = s; besti = i; }
    }
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) {
      float ob = __shfl_xor_sync(kFull, best, off);
      int oi = __shfl_xor_sync(kFull, besti, off);
      if (oi >= 0 && (besti < 0 || ob > best || (ob == best && oi > besti))) { best = ob; besti = oi; }
    }
    if (lane == 0) { s_best[w] = best; s_besti[w] = besti; }
    __syncthreads();
    if (tid == 0) {
      float bb = -INFINITY; int bi = -1;
      for (int i = 0; i < kHardThreads / 32; ++i) {
        if (s_besti[i] < 0) continue;
        if (bi < 0 || s_best[i] > bb || (s_best[i] == bb && s_besti[i] > bi)) { bb = s_best[i]; bi = s_besti[i]; }
      }
      s_win = bi;
    }
    __syncthreads();
    const int win = s_win;
    if (win < 0) break;
    const float4 bw = make_float4(dets[win * 5], dets[win * 5 + 1], dets[win * 5 + 2], dets[win * 5 + 3]);
    const float aw = area_plus1(bw);
    for (int i = tid; i < n; i += kHardThreads) {
      if (i == win) { keep[i] = 1; continue; }
      if (keep[i] != 2) continue;
      const float4 bi = make_float4(dets[i * 5], dets[i * 5 + 1], dets[i * 5 + 2], dets[i * 5 + 3]);
      if (ovr_plus1(bw, aw, bi, area_plus1(bi)) >= thresh) keep[i] = 0;
    }
    __syncthreads();
  }
}

}  // namespace yb

// ================================================================================================
// C ABI
// ================================================================================================
using namespace yb;

// k_final_topk's dynamic shared memory: [C1] counts, then [C1 * max_det] keys and as many tie keys
static size_t final_topk_smem(int C1, int max_det) {
  return (size_t)((C1 + 3) & ~3) * sizeof(int) + (size_t)2 * C1 * max_det * sizeof(uint32_t);
}

// every refusal happens here or before the first launch of yb_detect: a refused call writes nothing
static int check_params(const yb_detect_params* p, int batch, int A) {
  YB_REQUIRE(p != nullptr, YB_ERR_INVALID, "yb_detect: params is NULL");
  YB_REQUIRE(batch > 0 && A > 0, YB_ERR_INVALID, "yb_detect: batch=%d num_anchors=%d", batch, A);
  YB_REQUIRE(p->num_classes >= 2, YB_ERR_INVALID, "yb_detect: num_classes=%d", p->num_classes);
  YB_REQUIRE(p->top_k >= 1 && p->top_k <= kSortCap, YB_ERR_UNSUPPORTED, "yb_detect: top_k=%d outside [1,%d]", p->top_k, kSortCap);
  YB_REQUIRE(p->max_det >= 1 && p->max_det <= kSortCap, YB_ERR_UNSUPPORTED, "yb_detect: max_det=%d outside [1,%d]", p->max_det, kSortCap);
  YB_REQUIRE(p->coef_dim >= 0, YB_ERR_INVALID, "yb_detect: coef_dim=%d", p->coef_dim);
  YB_REQUIRE((double)(p->num_classes - 1) * A < 4294967296.0, YB_ERR_UNSUPPORTED, "yb_detect: (C-1)*A overflows 32 bits");
  YB_REQUIRE(p->num_classes <= YB_MAX_CLASSES, YB_ERR_UNSUPPORTED, "yb_detect: num_classes=%d > %d", p->num_classes, YB_MAX_CLASSES);
  YB_REQUIRE(final_topk_smem(p->num_classes - 1, p->max_det) <= 200 * 1024, YB_ERR_UNSUPPORTED,
             "yb_detect: (C-1)*max_det = %d too large for the final top-k stage", (p->num_classes - 1) * p->max_det);
  return YB_OK;
}

extern "C" size_t yb_detect_workspace_bytes(int batch, int num_anchors, const yb_detect_params* p) {
  if (!p || batch <= 0 || num_anchors <= 0) return 0;
  DetectWs w;
  return carve(&w, nullptr, batch, num_anchors, p->num_classes - 1, p->top_k > p->max_det ? p->top_k : p->max_det, p->traditional != 0);
}

extern "C" int yb_detect(const float* cls, const float* box, const float* coef, const float* anchors,
                         int batch, int num_anchors, const yb_detect_params* p,
                         void* workspace, size_t workspace_bytes,
                         int32_t* out_count, int32_t* out_class, int32_t* out_anchor,
                         float* out_score, float* out_box, float* out_coef, void* stream_) {
  YB_PROPAGATE(check_params(p, batch, num_anchors));
  YB_REQUIRE(cls && box && anchors && workspace && out_count && out_class && out_anchor && out_score && out_box,
             YB_ERR_INVALID, "yb_detect: NULL pointer argument");
  YB_REQUIRE(!out_coef || coef, YB_ERR_INVALID, "yb_detect: out_coef requested but coef is NULL");
  const int B = batch, A = num_anchors, C = p->num_classes, C1 = C - 1;
  const int KC = p->top_k > p->max_det ? p->top_k : p->max_det;
  DetectWs ws;
  const size_t need = carve(&ws, (char*)workspace, B, A, C1, KC, p->traditional != 0);
  YB_REQUIRE(workspace_bytes >= need, YB_ERR_INVALID, "yb_detect: workspace %zu < %zu bytes", workspace_bytes, need);
  if (p->traditional) {                                       // refused before anything is launched or written
    YB_REQUIRE(A <= 49152, YB_ERR_UNSUPPORTED, "yb_detect(traditional): num_anchors=%d > 49152", A);   // k_class_hard_nms: A scores in shared memory
    YB_REQUIRE(p->img_size > 0.f, YB_ERR_INVALID, "yb_detect(traditional): img_size must be > 0");
  }
  cudaStream_t stream = (cudaStream_t)stream_;

  YB_CHECK_CUDA(cudaMemsetAsync(ws.cand_count, 0, sizeof(int) * B, stream));
  {
    const size_t smem = (size_t)kP1Anchors * C * sizeof(float);
    dim3 grid(ceil_div(A, kP1Anchors), B);
    if (p->traditional) {
      YB_CHECK_CUDA(cudaFuncSetAttribute(k_filter_decode<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
      k_filter_decode<false><<<grid, kThreads, smem, stream>>>(cls, box, anchors, A, C, p->score_thr, p->no_clip, ws);
    } else {
      // cut [B][C1] | list_cnt [B][C1] are adjacent 256-byte aligned blocks: zero them (cut 0 = take all)
      YB_CHECK_CUDA(cudaMemsetAsync(ws.cut, 0, (size_t)((char*)ws.list - (char*)ws.cut), stream));
      if (A > kListCap) {                                     // small heads: every candidate fits its list, no sampling
        const size_t hs = (size_t)C1 * kCutBins * sizeof(int);
        YB_CHECK_CUDA(cudaFuncSetAttribute(k_sample_cuts, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)hs));
        k_sample_cuts<<<B, kSamples, hs, stream>>>(cls, A, C, p->score_thr, p->top_k, ws);
        YB_CHECK_LAUNCH();
      }
      // (a warp-per-32-anchors streaming form without the shared-memory tile was tried and measured 45 % slower: too few loads
      // in flight per warp; profiles/r2_postprocess_notes.txt)
      const size_t smem2 = smem + 8 + (size_t)C1 * kStage * sizeof(uint2);
      YB_CHECK_CUDA(cudaFuncSetAttribute(k_filter_decode<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem2));
      k_filter_decode<true><<<grid, kThreads, smem2, stream>>>(cls, box, anchors, A, C, p->score_thr, p->no_clip, ws);
    }
    YB_CHECK_LAUNCH();
  }
  if (!p->traditional) {
    k_class_fast_nms<<<dim3(C1, B), kThreads, 0, stream>>>(cls, A, C1, p->top_k, p->iou_thr, ws);
    YB_CHECK_LAUNCH();
  } else {
    const size_t smem = (size_t)A * sizeof(float);
    YB_CHECK_CUDA(cudaFuncSetAttribute(k_class_hard_nms, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    k_class_hard_nms<<<dim3(C1, B), kThreads, smem, stream>>>(A, C1, p->score_thr, p->iou_thr, p->img_size, p->max_det, ws);
    YB_CHECK_LAUNCH();
  }
  {
    const size_t smem = final_topk_smem(C1, p->max_det);
    YB_CHECK_CUDA(cudaFuncSetAttribute(k_final_topk, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    k_final_topk<<<B, kThreads, smem, stream>>>(coef, A, C1, p->max_det, p->coef_dim, p->traditional, p->img_size, ws,
                                                 out_count, out_class, out_anchor, out_score, out_box, out_coef);
    YB_CHECK_LAUNCH();
  }
  return YB_OK;
}

namespace {
struct DevBuf {
  void* p = nullptr;
  ~DevBuf() { if (p) cudaFree(p); }
  int alloc(size_t bytes) { YB_CHECK_CUDA(cudaMalloc(&p, bytes ? bytes : 1)); return YB_OK; }
};
}  // namespace

extern "C" int yb_detect_host(const float* cls, const float* box, const float* coef, const float* anchors,
                              int batch, int num_anchors, const yb_detect_params* p,
                              int32_t* out_count, int32_t* out_class, int32_t* out_anchor,
                              float* out_score, float* out_box, float* out_coef) {
  YB_PROPAGATE(check_params(p, batch, num_anchors));
  const size_t B = batch, A = num_anchors, C = p->num_classes, K = p->coef_dim, D = p->max_det;
  DevBuf dcls, dbox, dcoef, danc, dws, dcount, dclass, danchor, dscore, dobox, docoef;
  YB_PROPAGATE(dcls.alloc(B * A * C * 4)); YB_PROPAGATE(dbox.alloc(B * A * 16)); YB_PROPAGATE(danc.alloc(A * 16));
  const bool want_coef = out_coef && coef && K > 0;
  if (want_coef) { YB_PROPAGATE(dcoef.alloc(B * A * K * 4)); YB_PROPAGATE(docoef.alloc(B * D * K * 4)); }
  const size_t wsb = yb_detect_workspace_bytes(batch, num_anchors, p);
  YB_PROPAGATE(dws.alloc(wsb));
  YB_PROPAGATE(dcount.alloc(B * 4)); YB_PROPAGATE(dclass.alloc(B * D * 4)); YB_PROPAGATE(danchor.alloc(B * D * 4));
  YB_PROPAGATE(dscore.alloc(B * D * 4)); YB_PROPAGATE(dobox.alloc(B * D * 16));
  YB_CHECK_CUDA(cudaMemcpy(dcls.p, cls, B * A * C * 4, cudaMemcpyHostToDevice));
  YB_CHECK_CUDA(cudaMemcpy(dbox.p, box, B * A * 16, cudaMemcpyHostToDevice));
  YB_CHECK_CUDA(cudaMemcpy(danc.p, anchors, A * 16, cudaMemcpyHostToDevice));
  if (want_coef) YB_CHECK_CUDA(cudaMemcpy(dcoef.p, coef, B * A * K * 4, cudaMemcpyHostToDevice));
  YB_PROPAGATE(yb_detect((const float*)dcls.p, (const float*)dbox.p, (const float*)dcoef.p, (const float*)danc.p, batch,
                         num_anchors, p, dws.p, wsb, (int32_t*)dcount.p, (int32_t*)dclass.p, (int32_t*)danchor.p,
                         (float*)dscore.p, (float*)dobox.p, want_coef ? (float*)docoef.p : nullptr, nullptr));
  YB_CHECK_CUDA(cudaMemcpy(out_count, dcount.p, B * 4, cudaMemcpyDeviceToHost));
  YB_CHECK_CUDA(cudaMemcpy(out_class, dclass.p, B * D * 4, cudaMemcpyDeviceToHost));
  YB_CHECK_CUDA(cudaMemcpy(out_anchor, danchor.p, B * D * 4, cudaMemcpyDeviceToHost));
  YB_CHECK_CUDA(cudaMemcpy(out_score, dscore.p, B * D * 4, cudaMemcpyDeviceToHost));
  YB_CHECK_CUDA(cudaMemcpy(out_box, dobox.p, B * D * 16, cudaMemcpyDeviceToHost));
  if (want_coef) YB_CHECK_CUDA(cudaMemcpy(out_coef, docoef.p, B * D * K * 4, cudaMemcpyDeviceToHost));
  return YB_OK;
}

extern "C" int yb_hard_nms(const float* dets, int n, float thresh, uint8_t* out_keep, void* stream) {
  YB_REQUIRE(n >= 0, YB_ERR_INVALID, "yb_hard_nms: n=%d", n);
  if (n == 0) return YB_OK;
  YB_REQUIRE(dets && out_keep, YB_ERR_INVALID, "yb_hard_nms: NULL pointer argument");
  k_hard_nms<<<1, kHardThreads, 0, (cudaStream_t)stream>>>(dets, n, thresh, out_keep);
  YB_CHECK_LAUNCH();
  return YB_OK;
}

extern "C" int yb_hard_nms_host(const float* dets, int n, float thresh, uint8_t* out_keep) {
  YB_REQUIRE(n >= 0, YB_ERR_INVALID, "yb_hard_nms_host: n=%d", n);
  if (n == 0) return YB_OK;
  DevBuf d, k;
  YB_PROPAGATE(d.alloc((size_t)n * 20)); YB_PROPAGATE(k.alloc(n));
  YB_CHECK_CUDA(cudaMemcpy(d.p, dets, (size_t)n * 20, cudaMemcpyHostToDevice));
  YB_PROPAGATE(yb_hard_nms((const float*)d.p, n, thresh, (uint8_t*)k.p, nullptr));
  YB_CHECK_CUDA(cudaMemcpy(out_keep, k.p, n, cudaMemcpyDeviceToHost));
  return YB_OK;
}
