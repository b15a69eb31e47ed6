// Training augmentation (utils/augmentations.py:230-252 train_aug) on the GPU, for a batch of host-drawn plans.
//
// train_aug's random draws depend only on shapes, boxes and labels, so the host planner
// (utils/augmentations.py: train_aug_plan) replays them and this kernel only moves pixels.  Each output pixel
// is a composite gather through the reference's stages, applied backwards:
//   to_train_size pad/crop (:192-209) -> cv2.resize INTER_LINEAR of the P x P square (:168-189) ->
//   pad_to_square (:138-165, image fill norm_mean, mask fill 0) -> crop (:80-124) -> mirror (:10-17) ->
//   photometric_distort (:62-77) of the source pixel, which is pointwise and so exact at fetch time.
// The resize follows OpenCV's resizeGeneric_ coordinates: fx = (float)((dx+0.5)*scale-0.5) in double with
// scale = 1/(dst/src); x taps clamped at the borders with weight 0 outside; y keeps its weights and clips the
// two source rows into the image.  Float images and padded (float) masks interpolate in float32; masks of an
// image that was square after the crop stay uint8 in the reference and use OpenCV's 11-bit fixed-point weights
// with the rounding of its vectorised vertical pass (VResizeLinearVec_32s8u).
#include "common.cuh"
#include <float.h>
#include <math.h>

namespace yb {

constexpr int kAugThreads = 256;

struct AugTap {
  int s0, s1;     // source coordinate of each tap in the un-mirrored image; -1 = square-pad fill
  float a0, a1;   // float weights
  int i0, i1;     // 11-bit fixed-point weights
};

// One axis of the composite map: output coordinate o (0..S-1) -> taps in the source image.  Returns false when o
// lies in to_train_size's pad border (the output there is the fill).
__device__ __forceinline__ bool aug_axis(int o, int S, int rs, int train_off, int P, int pad_off, int crop_off, int crop_len,
                                         int flip_len, bool y_rule, AugTap& t) {
  const int r = rs < S ? o - train_off : o + train_off;
  if (r < 0 || r >= rs) return false;
  const double scale = 1.0 / ((double)rs / (double)P);
  float f = (float)(((double)r + 0.5) * scale - 0.5);
  int s = (int)floorf(f);
  f -= (float)s;
  int s0, s1;
  if (y_rule) {
    s0 = min(max(s, 0), P - 1);
    s1 = min(max(s + 1, 0), P - 1);
  } else {
    if (s < 0) { s = 0; f = 0.f; }
    if (s >= P - 1) { s = P - 1; f = 0.f; }
    s0 = s;
    s1 = min(s + 1, P - 1);
  }
  t.a0 = 1.f - f;
  t.a1 = f;
  t.i0 = __float2int_rn(t.a0 * 2048.f);
  t.i1 = __float2int_rn(t.a1 * 2048.f);
  auto to_src = [&](int p) {
    const int q = p - pad_off;
    if (q < 0 || q >= crop_len) return -1;
    const int m = q + crop_off;
    return flip_len > 0 ? flip_len - 1 - m : m;
  };
  t.s0 = to_src(s0);
  t.s1 = to_src(s1);
  return true;
}

// cv2.cvtColor(COLOR_BGR2HSV) on float32 (H in [0,360), S = diff/(V+eps), V = max)
__device__ __forceinline__ void aug_bgr2hsv(float b, float g, float r, float& h, float& s, float& v) {
  float vmin = r;
  v = r;
  if (v < g) v = g;
  if (v < b) v = b;
  if (vmin > g) vmin = g;
  if (vmin > b) vmin = b;
  float diff = v - vmin;
  s = diff / (fabsf(v) + FLT_EPSILON);
  diff = 60.f / (diff + FLT_EPSILON);
  if (v == r) h = (g - b) * diff;
  else if (v == g) h = (b - r) * diff + 120.f;
  else h = (r - g) * diff + 240.f;
  if (h < 0.f) h += 360.f;
}

// cv2.cvtColor(COLOR_HSV2BGR) on float32; with S > 1 the outputs go negative (clipped by the caller)
__device__ __forceinline__ void aug_hsv2bgr(float h, float s, float v, float& b, float& g, float& r) {
  if (s == 0.f) { b = g = r = v; return; }
  h *= 6.f / 360.f;
  if (h >= 6.f) h -= 6.f;     // fmod(h, 6): exact here, the caller's h is in [0, 360] so h < 12
  int sector = (int)floorf(h);
  h -= (float)sector;
  if ((unsigned)sector >= 6u) { sector = 0; h = 0.f; }
  const float t0 = v, t1 = v * (1.f - s), t2 = v * (1.f - s * h), t3 = v * (1.f - s * (1.f - h));
  // OpenCV's sector table {b,g,r} = {1,3,0} {1,0,2} {3,0,1} {0,2,1} {0,1,3} {2,1,0}, as a switch (no local-memory table)
  switch (sector) {
    case 0: b = t1; g = t3; r = t0; break;
    case 1: b = t1; g = t0; r = t2; break;
    case 2: b = t3; g = t0; r = t1; break;
    case 3: b = t0; g = t2; r = t1; break;
    case 4: b = t0; g = t1; r = t3; break;
    default: b = t2; g = t1; r = t0; break;
  }
}

__device__ __forceinline__ float clip255(float x) { return fminf(fmaxf(x, 0.f), 255.f); }

// photometric_distort of one source pixel (float32 throughout, the scalars rounded to float32 as numpy does)
__device__ __forceinline__ void aug_photometric(const yb_train_aug_item& it, const uint8_t* px, float out[3]) {
  float c[3] = {(float)px[0], (float)px[1], (float)px[2]};
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    if (it.brightness_on) c[k] = clip255(c[k] + it.brightness_delta);
    if (it.contrast_on) c[k] = clip255(c[k] * it.contrast_alpha);
  }
  float h, s, v;
  aug_bgr2hsv(c[0], c[1], c[2], h, s, v);
  s *= it.saturation_scale;
  h += it.hue_delta;
  if (h > 360.f) h -= 360.f;
  if (h < 0.f) h += 360.f;
  aug_hsv2bgr(h, s, v, out[0], out[1], out[2]);
#pragma unroll
  for (int k = 0; k < 3; ++k) out[k] = clip255(out[k]);
}

// grid: (ceil(S*S / kAugThreads), n_items).  One thread per output pixel: the taps are built once and reused for the
// three channels and every surviving mask of the image.
__global__ void __launch_bounds__(kAugThreads) k_train_aug(const uint8_t* __restrict__ src, const yb_train_aug_item* __restrict__ items,
                                                          const int32_t* __restrict__ keep, int S, float* __restrict__ out_img,
                                                          float* __restrict__ out_masks) {
  const yb_train_aug_item it = items[blockIdx.y];
  const int total = S * S;
  const int i = blockIdx.x * kAugThreads + threadIdx.x;
  if (i >= total) return;
  const int oy = i / S, ox = i - oy * S;
  AugTap tx, ty;
  const bool inside = aug_axis(ox, S, it.resize, it.train_x, it.square, it.pad_x, it.crop_x, it.crop_w, it.mirror ? it.w : 0, false, tx) &&
                      aug_axis(oy, S, it.resize, it.train_y, it.square, it.pad_y, it.crop_y, it.crop_h, 0, true, ty);
  const float mean[3] = {103.94f, 116.78f, 123.68f}, stdv[3] = {57.38f, 57.12f, 58.40f};
  float* img = out_img + (size_t)blockIdx.y * 3 * total + i;
  float* msk = out_masks + (size_t)it.out_mask * total + i;
  if (!inside) {
#pragma unroll
    for (int c = 0; c < 3; ++c) img[(size_t)c * total] = 0.f;     // (norm_mean - mean) / std
    for (int k = 0; k < it.num_keep; ++k) msk[(size_t)k * total] = 0.f;
    return;
  }
  // image: four photometric taps, bilinear per channel (x first, as cv2's horizontal pass)
  const uint8_t* im = src + it.img_off;
  float p[4][3];
  const int ys[2] = {ty.s0, ty.s1}, xs[2] = {tx.s0, tx.s1};
#pragma unroll
  for (int a = 0; a < 2; ++a)
#pragma unroll
    for (int b = 0; b < 2; ++b) {
      float* q = p[a * 2 + b];
      if (ys[a] < 0 || xs[b] < 0) {
        q[0] = mean[0]; q[1] = mean[1]; q[2] = mean[2];
      } else {
        aug_photometric(it, im + ((size_t)ys[a] * it.w + xs[b]) * 3, q);
      }
    }
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    const float r0 = p[0][c] * tx.a0 + p[1][c] * tx.a1;
    const float r1 = p[2][c] * tx.a0 + p[3][c] * tx.a1;
    const float v = r0 * ty.a0 + r1 * ty.a1;
    img[(size_t)(2 - c) * total] = (v - mean[c]) / stdv[c];
  }
  // masks: same taps, 0 outside the crop
  const size_t plane = (size_t)it.h * it.w;
  const bool ok[4] = {ty.s0 >= 0 && tx.s0 >= 0, ty.s0 >= 0 && tx.s1 >= 0, ty.s1 >= 0 && tx.s0 >= 0, ty.s1 >= 0 && tx.s1 >= 0};
  const size_t off[4] = {(size_t)ty.s0 * it.w + tx.s0, (size_t)ty.s0 * it.w + tx.s1, (size_t)ty.s1 * it.w + tx.s0, (size_t)ty.s1 * it.w + tx.s1};
  const int32_t* kp = keep + it.keep_begin;
  for (int k = 0; k < it.num_keep; ++k) {
    const uint8_t* m = src + it.mask_off + (size_t)kp[k] * plane;
    int v[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) v[j] = ok[j] ? (int)m[off[j]] : 0;
    float o;
    if (it.mask_u8) {
      const int h0 = v[0] * tx.i0 + v[1] * tx.i1, h1 = v[2] * tx.i0 + v[3] * tx.i1;
      const int t = (((h0 >> 4) * ty.i0) >> 16) + (((h1 >> 4) * ty.i1) >> 16);
      o = (float)min(max((t + 2) >> 2, 0), 255);
    } else {
      const float r0 = (float)v[0] * tx.a0 + (float)v[1] * tx.a1;
      const float r1 = (float)v[2] * tx.a0 + (float)v[3] * tx.a1;
      o = r0 * ty.a0 + r1 * ty.a1;
    }
    msk[(size_t)k * total] = o;
  }
}

}  // namespace yb

namespace {
size_t aug_items_bytes(int n_items) { return yb::align_up((size_t)n_items * sizeof(yb_train_aug_item), 256); }
}  // namespace

extern "C" size_t yb_train_aug_workspace_bytes(int n_items, int64_t n_keep) {
  if (n_items < 0 || n_keep < 0) return 0;
  return aug_items_bytes(n_items) + yb::align_up((size_t)n_keep * sizeof(int32_t), 256);
}

extern "C" int yb_train_aug(const uint8_t* src, int64_t src_bytes, const yb_train_aug_item* items, int n_items, const int32_t* keep,
                            int img_size, void* workspace, size_t workspace_bytes, float* out_img, float* out_masks, void* stream) {
  YB_REQUIRE(src && items && out_img && workspace, YB_ERR_INVALID, "yb_train_aug: NULL pointer argument");
  YB_REQUIRE(src_bytes > 0 && n_items > 0 && n_items <= 65535, YB_ERR_INVALID, "yb_train_aug: src_bytes=%lld n_items=%d",
             (long long)src_bytes, n_items);
  YB_REQUIRE(img_size > 0 && img_size <= 4096, YB_ERR_INVALID, "yb_train_aug: img_size=%d", img_size);
  const int S = img_size;
  int64_t n_keep = 0;
  for (int i = 0; i < n_items; ++i) {
    const yb_train_aug_item& t = items[i];
    YB_REQUIRE(t.h > 0 && t.w > 0 && t.h <= 16384 && t.w <= 16384 && t.num_masks >= 0, YB_ERR_INVALID,
               "yb_train_aug: item %d: h=%d w=%d num_masks=%d", i, t.h, t.w, t.num_masks);
    const int64_t plane = (int64_t)t.h * t.w;
    YB_REQUIRE(t.img_off >= 0 && t.img_off <= src_bytes - plane * 3, YB_ERR_INVALID,
               "yb_train_aug: item %d: image [%lld, +%lld) outside src (%lld bytes)", i, (long long)t.img_off, (long long)(plane * 3),
               (long long)src_bytes);
    YB_REQUIRE(t.mask_off >= 0 && t.mask_off <= src_bytes - plane * t.num_masks, YB_ERR_INVALID,
               "yb_train_aug: item %d: masks [%lld, +%lld) outside src (%lld bytes)", i, (long long)t.mask_off,
               (long long)(plane * t.num_masks), (long long)src_bytes);
    YB_REQUIRE((t.brightness_on | t.contrast_on | t.mirror | t.mask_u8) >= 0 && t.brightness_on <= 1 && t.contrast_on <= 1 &&
                   t.mirror <= 1 && t.mask_u8 <= 1,
               YB_ERR_INVALID, "yb_train_aug: item %d: flags must be 0 or 1", i);
    YB_REQUIRE(t.crop_w > 0 && t.crop_h > 0 && t.crop_x >= 0 && t.crop_y >= 0 && t.crop_x <= t.w - t.crop_w && t.crop_y <= t.h - t.crop_h,
               YB_ERR_INVALID, "yb_train_aug: item %d: crop (%d,%d,%d,%d) outside %dx%d", i, t.crop_x, t.crop_y, t.crop_w, t.crop_h, t.h, t.w);
    YB_REQUIRE(t.square == (t.crop_w > t.crop_h ? t.crop_w : t.crop_h) && t.pad_x >= 0 && t.pad_y >= 0 && t.pad_x <= t.square - t.crop_w &&
                   t.pad_y <= t.square - t.crop_h,
               YB_ERR_INVALID, "yb_train_aug: item %d: square %d pad (%d,%d) for a %dx%d crop", i, t.square, t.pad_x, t.pad_y, t.crop_h, t.crop_w);
    const int span = t.resize < S ? S - t.resize : t.resize - S;
    YB_REQUIRE(t.resize > 0 && t.resize <= 16384 && t.train_x >= 0 && t.train_y >= 0 && t.train_x <= span && t.train_y <= span,
               YB_ERR_INVALID, "yb_train_aug: item %d: resize %d train offset (%d,%d) at img_size %d", i, t.resize, t.train_x, t.train_y, S);
    YB_REQUIRE(t.num_keep >= 0 && t.out_mask == n_keep && t.keep_begin == n_keep, YB_ERR_INVALID,
               "yb_train_aug: item %d: out_mask=%d keep_begin=%d num_keep=%d, expected dense rows from %lld", i, t.out_mask, t.keep_begin,
               t.num_keep, (long long)n_keep);
    YB_REQUIRE(t.num_keep == 0 || keep, YB_ERR_INVALID, "yb_train_aug: NULL keep table");
    for (int k = 0; k < t.num_keep; ++k)
      YB_REQUIRE(keep[n_keep + k] >= 0 && keep[n_keep + k] < t.num_masks, YB_ERR_INVALID,
                 "yb_train_aug: item %d: keep[%lld]=%d outside its %d masks", i, (long long)(n_keep + k), keep[n_keep + k], t.num_masks);
    n_keep += t.num_keep;
    YB_REQUIRE(n_keep <= INT32_MAX, YB_ERR_INVALID, "yb_train_aug: too many output masks");
  }
  YB_REQUIRE(n_keep == 0 || out_masks, YB_ERR_INVALID, "yb_train_aug: NULL out_masks with %lld output masks", (long long)n_keep);
  YB_REQUIRE(workspace_bytes >= yb_train_aug_workspace_bytes(n_items, n_keep), YB_ERR_INVALID,
             "yb_train_aug: workspace %zu bytes < %zu", workspace_bytes, yb_train_aug_workspace_bytes(n_items, n_keep));
  cudaStream_t st = (cudaStream_t)stream;
  yb_train_aug_item* d_items = (yb_train_aug_item*)workspace;
  int32_t* d_keep = (int32_t*)((char*)workspace + aug_items_bytes(n_items));
  const yb::StagePart parts[2] = {{items, (size_t)n_items * sizeof(yb_train_aug_item), 0},
                                   {keep, (size_t)n_keep * sizeof(int32_t), aug_items_bytes(n_items)}};
  YB_PROPAGATE(yb::stage_tables(workspace, aug_items_bytes(n_items) + (size_t)n_keep * sizeof(int32_t), parts, 2, st));
  dim3 grid(yb::ceil_div(S * S, yb::kAugThreads), n_items);
  yb::k_train_aug<<<grid, yb::kAugThreads, 0, st>>>(src, d_items, d_keep, S, out_img, out_masks);
  YB_CHECK_LAUNCH();
  return YB_OK;
}
