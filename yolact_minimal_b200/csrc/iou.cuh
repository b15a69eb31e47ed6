// Pairwise IoU arithmetic shared by the mask output stage (mask_ops.cu) and the evaluation stage (eval.cu): one definition, so
// the IoUs the evaluator matches on are bit-identical to what yb_box_iou / yb_mask_iou_bits return.
#pragma once
#include <stdint.h>

namespace yb {

// utils/box_utils.py:8-37 box_iou of two corner boxes (x1,y1,x2,y2): the reference's separately rounded fp32 operations
// (clamp(min=0) of the overlap, product areas, inter / (area_a + area_b - inter)); 0/0 = NaN
__device__ __forceinline__ float box_iou_rn(const float4 p, const float4 q) {
  const float iw = fmaxf(__fsub_rn(fminf(p.z, q.z), fmaxf(p.x, q.x)), 0.f);
  const float ih = fmaxf(__fsub_rn(fminf(p.w, q.w), fmaxf(p.y, q.y)), 0.f);
  const float inter = __fmul_rn(iw, ih);
  const float aa = __fmul_rn(__fsub_rn(p.z, p.x), __fsub_rn(p.w, p.y));
  const float ab = __fmul_rn(__fsub_rn(q.z, q.x), __fsub_rn(q.w, q.y));
  return __fdiv_rn(inter, __fsub_rn(__fadd_rn(aa, ab), inter));
}

// Popcounts of one word pair: |a & b|, |a|, |b| accumulate over the packed words of two masks
__device__ __forceinline__ void mask_counts_add(const uint32_t x, const uint32_t y, unsigned& inter, unsigned& ca, unsigned& cb) {
  inter += __popc(x & y); ca += __popc(x); cb += __popc(y);
}

// utils/box_utils.py:189-200 mask_iou from the pixel counts: the reference's fp32 matmul of {0,1} masks and its row sums are
// exact below 2^24 pixels, so inter / ((|a| + |b|) - inter) in separately rounded fp32 reproduces it (0/0 = NaN)
__device__ __forceinline__ float mask_iou_from_counts(const unsigned inter, const unsigned ca, const unsigned cb) {
  const float fi = (float)inter;
  return __fdiv_rn(fi, __fsub_rn(__fadd_rn((float)ca, (float)cb), fi));
}

}  // namespace yb
