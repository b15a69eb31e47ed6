// Detection drawing on the GPU -- the pixel work of utils/output_utils.py:308-369 (draw_img):
//   semantic = (sum_i m_i * (ids_i + 1)) mod num_colors          (numpy floor modulo; m_i in {0,1})
//   overlay  = rint(0.4f * palette[semantic] + 0.6f * img)        k_draw_masks<.., kOutBlend>   (cv2.addWeighted(.., 0.4, .., 0.6, 0))
//   total_obj = semantic != 0 ? img : 255                         k_draw_masks<.., kOutMatte>   (cfg.cutout)
//   crop_i   = (m_i != 0 ? img : 255)[y1:y2, x1:x2]               k_draw_cutout                 (cfg.cutout)
// Masks come in the three layouts after_nms writes (yb_mask_assemble's codes): 0 uint8, 1 float32 [n,h,w], 2 bit-packed words
// [n,h,ceil(w/32)].  A block owns a kDrawTileW x kDrawTileH pixel tile.  Phase 1 reduces the n masks to the tile's semantic
// indices in shared memory, reading the masks coalesced (4 pixels per thread for bytes / floats, one 32-pixel word per thread for
// bits).  Phase 2 streams the tile's image bytes in order, so the image is read and written with fully used sectors.
// The same kernel draws a batch (yb_draw_masks_batch): blockIdx.z is the image, its geometry comes from a device table, and a
// DEVICE count limits image b to its first min(count[b], n) masks; an image with count <= 0 is copied unchanged.
//
// k_draw_lincomb is utils/output_utils.py:276-305 (draw_lincomb, the cfg.save_lincomb view) for detection 0 of each image: the
// 32 prototypes, ordered by |coef| descending (ties: lower channel first), each divided by its maximum and scaled by its
// coefficient, tiled 4 x 8 and mapped through COLORMAP_WINTER.
#include "common.cuh"
#include <vector>

namespace yb {

constexpr int kDrawThreads = 128;
constexpr int kDrawTileW = 256;            // pixels: 8 packed words, 64 threads x 4 pixels
constexpr int kDrawTileH = 16;             // rows: 16 x 8 words = one word per thread
constexpr int kDrawMaxDet = 4096;
constexpr int kDrawMaxColors = 1024;
constexpr int kCutoutBlocks = 64;
enum { kMaskU8 = 0, kMaskF32 = 1, kMaskBits = 2 };
enum { kOutBlend = 0, kOutMatte = 1 };
constexpr int kLincombK = 32, kLincombRows = 4, kLincombCols = 8;
constexpr int kLincombThreads = 256;

// where image blockIdx.z lies: img_off bytes into the image / output buffers, mask_off elements into the masks
struct DrawImage {
  int64_t img_off, mask_off;
  int h, w;
};

static_assert(kDrawTileW / 32 * kDrawTileH == kDrawThreads, "bits: one word per thread");
static_assert(kDrawTileW / 4 * 2 == kDrawThreads, "bytes / floats: two rows of 4-pixel groups per pass");

__device__ __forceinline__ int floor_mod(long long v, int m) {
  const long long r = v % m;
  return (int)(r < 0 ? r + m : r);
}

// dynamic shared memory: uint16 sem[tile] | int32 wgt[n] | uint8 palette[3 * num_colors]
// wgt_i = (ids_i + 1) mod num_colors, so the per-pixel sums stay below n * num_colors < 2^22 and sum mod num_colors is the
// reference's int64 sum mod num_colors.
// imgs == nullptr: one image described by `one` (yb_draw_masks).  Otherwise image blockIdx.z is imgs[blockIdx.z], its ids are
// ids[z * n ..], and count (DEVICE, may be nullptr) caps its masks; the grid covers the largest image, other blocks exit.
template <int FMT, int OUT>
__global__ void __launch_bounds__(kDrawThreads)
k_draw_masks(const uint8_t* __restrict__ img_base, const DrawImage* __restrict__ imgs, DrawImage one, const void* __restrict__ mask_base,
             int n_max, const int32_t* __restrict__ ids_base, const int32_t* __restrict__ count, const uint8_t* __restrict__ palette,
             int nc, uint8_t* __restrict__ out_base) {
  extern __shared__ __align__(16) unsigned char s_raw[];
  const int z = blockIdx.z;
  const DrawImage g = imgs ? imgs[z] : one;
  const int h = g.h, w = g.w;
  const int x0 = blockIdx.x * kDrawTileW, y0 = blockIdx.y * kDrawTileH;
  if (x0 >= w || y0 >= h) return;
  int n = n_max;
  bool copy = false;                                          // count[z] <= 0: nothing to draw, the image is copied unchanged
  if (count) {
    const int c = count[z];
    copy = c <= 0;
    n = copy ? 0 : min(c, n_max);
  }
  const uint8_t* img = img_base + g.img_off;
  uint8_t* out = out_base + g.img_off;
  const int32_t* ids = ids_base + (size_t)z * n_max;
  const void* masks = FMT == kMaskBits  ? static_cast<const void*>(static_cast<const uint32_t*>(mask_base) + g.mask_off)
                      : FMT == kMaskF32 ? static_cast<const void*>(static_cast<const float*>(mask_base) + g.mask_off)
                                        : static_cast<const void*>(static_cast<const uint8_t*>(mask_base) + g.mask_off);
  uint16_t* s_sem = reinterpret_cast<uint16_t*>(s_raw);
  int* s_wgt = reinterpret_cast<int*>(s_raw + kDrawTileW * kDrawTileH * sizeof(uint16_t));
  uint8_t* s_pal = reinterpret_cast<uint8_t*>(s_wgt + n_max);
  const int tid = threadIdx.x;
  for (int i = tid; i < n; i += kDrawThreads) s_wgt[i] = floor_mod((long long)ids[i] + 1, nc);
  if (OUT == kOutBlend && !copy)
    for (int i = tid; i < 3 * nc; i += kDrawThreads) s_pal[i] = palette[i];
  __syncthreads();

  const size_t plane = (size_t)h * w;
  if (copy) {
  } else if (FMT == kMaskBits) {
    const int words = (w + 31) >> 5;
    const int row = tid >> 3, wi = (x0 >> 5) + (tid & 7), y = y0 + row;
    if (y < h && wi < words) {
      int acc[32];
#pragma unroll
      for (int b = 0; b < 32; ++b) acc[b] = 0;
      const uint32_t* src = static_cast<const uint32_t*>(masks) + (size_t)y * words + wi;
      const size_t stride = (size_t)h * words;
#pragma unroll 4
      for (int i = 0; i < n; ++i) {
        const uint32_t m = __ldg(src + i * stride);
        if (m) {
          const int wt = s_wgt[i];
#pragma unroll
          for (int b = 0; b < 32; ++b) acc[b] += (m >> b & 1u) ? wt : 0;
        }
      }
      const int base = row * kDrawTileW + (tid & 7) * 32;
#pragma unroll
      for (int b = 0; b < 32; ++b) s_sem[base + b] = (uint16_t)(acc[b] % nc);
    }
  } else {
    const int g = tid & 63, xs = x0 + 4 * g;
    for (int row = tid >> 6; row < kDrawTileH; row += 2) {
      const int y = y0 + row;
      if (y >= h || xs >= w) continue;
      int acc[4] = {0, 0, 0, 0};
      const size_t p = (size_t)y * w + xs;
      if ((w & 3) == 0) {                                     // 4-pixel groups are 16 B (float) / 4 B (uint8) aligned
#pragma unroll 4
        for (int i = 0; i < n; ++i) {
          const int wt = s_wgt[i];
          if (FMT == kMaskF32) {
            const float4 v = __ldg(reinterpret_cast<const float4*>(static_cast<const float*>(masks) + i * plane + p));
            acc[0] += v.x != 0.f ? wt : 0; acc[1] += v.y != 0.f ? wt : 0; acc[2] += v.z != 0.f ? wt : 0; acc[3] += v.w != 0.f ? wt : 0;
          } else {
            const uchar4 v = __ldg(reinterpret_cast<const uchar4*>(static_cast<const uint8_t*>(masks) + i * plane + p));
            acc[0] += v.x ? wt : 0; acc[1] += v.y ? wt : 0; acc[2] += v.z ? wt : 0; acc[3] += v.w ? wt : 0;
          }
        }
      } else {
        const int cnt = min(4, w - xs);
        for (int i = 0; i < n; ++i) {
          const int wt = s_wgt[i];
#pragma unroll
          for (int k = 0; k < 4; ++k) {
            if (k < cnt) {
              const bool on = FMT == kMaskF32 ? __ldg(static_cast<const float*>(masks) + i * plane + p + k) != 0.f
                                              : __ldg(static_cast<const uint8_t*>(masks) + i * plane + p + k) != 0;
              acc[k] += on ? wt : 0;
            }
          }
        }
      }
#pragma unroll
      for (int k = 0; k < 4; ++k) s_sem[row * kDrawTileW + 4 * g + k] = (uint16_t)(acc[k] % nc);
    }
  }
  __syncthreads();

  // phase 2: the tile's image bytes in order, 3 per pixel (BGR); byte b of a row belongs to pixel b / 3, channel b % 3
  const int tw = min(kDrawTileW, w - x0), th = min(kDrawTileH, h - y0), rb = 3 * tw;
  for (int e = tid; e < th * rb; e += kDrawThreads) {
    const int row = e / rb, b = e - row * rb, px = b / 3, ch = b - 3 * px;
    const size_t o = ((size_t)(y0 + row) * w + x0) * 3 + b;
    const int s = s_sem[row * kDrawTileW + px];
    const uint8_t v = img[o];
    if (copy)
      out[o] = v;
    else if (OUT == kOutBlend)   // cv2.addWeighted(color, 0.4, img, 0.6, 0) on uint8: each product rounded to fp32, sum rounded to nearest
      out[o] = (uint8_t)__float2int_rn(__fadd_rn(__fmul_rn(0.4f, (float)s_pal[3 * s + ch]), __fmul_rn(0.6f, (float)v)));
    else
      out[o] = s != 0 ? v : (uint8_t)255;
  }
}

__device__ __forceinline__ bool mask_on(const void* masks, int fmt, int i, int y, int x, int h, int w) {
  if (fmt == kMaskBits) {
    const int words = (w + 31) >> 5;
    return (__ldg(static_cast<const uint32_t*>(masks) + ((size_t)i * h + y) * words + (x >> 5)) >> (x & 31)) & 1u;
  }
  const size_t p = ((size_t)i * h + y) * w + x;
  return fmt == kMaskF32 ? __ldg(static_cast<const float*>(masks) + p) != 0.f : __ldg(static_cast<const uint8_t*>(masks) + p) != 0;
}

// one crop per blockIdx.y, its pixels grid-strided over blockIdx.x; crop i = rows [y1,y2) x cols [x1,x2) of the image, written
// row-major as [y2-y1, x2-x1, 3] at out + off[i].  A crop outside the image, or whose byte range does not hold exactly its pixels,
// is not written.
__global__ void __launch_bounds__(kDrawThreads)
k_draw_cutout(const uint8_t* __restrict__ img, int h, int w, const void* __restrict__ masks, int fmt,
              const int32_t* __restrict__ yyxx, const int64_t* __restrict__ off, uint8_t* __restrict__ out) {
  const int i = blockIdx.y;
  const int y1 = yyxx[4 * i], y2 = yyxx[4 * i + 1], x1 = yyxx[4 * i + 2], x2 = yyxx[4 * i + 3];
  if (!(0 <= y1 && y1 <= y2 && y2 <= h && 0 <= x1 && x1 <= x2 && x2 <= w)) return;
  const int cw = x2 - x1;
  const long long area = (long long)(y2 - y1) * cw;
  if (off[i] < 0 || off[i + 1] - off[i] != 3 * area) return;
  uint8_t* dst = out + off[i];
  for (long long q = (long long)blockIdx.x * kDrawThreads + threadIdx.x; q < area; q += (long long)gridDim.x * kDrawThreads) {
    const int cy = (int)(q / cw), cx = (int)(q - (long long)cy * cw), y = y1 + cy, x = x1 + cx;
    const bool on = mask_on(masks, fmt, i, y, x, h, w);
    const uint8_t* s = img + ((size_t)y * w + x) * 3;
#pragma unroll
    for (int c = 0; c < 3; ++c) dst[3 * q + c] = on ? s[c] : (uint8_t)255;
  }
}

template <int OUT>
static int launch_draw(const uint8_t* img, int h, int w, const void* masks, int fmt, int n, const int32_t* ids, const uint8_t* palette,
                       int nc, uint8_t* out, cudaStream_t stream) {
  const dim3 grid(ceil_div(w, kDrawTileW), ceil_div(h, kDrawTileH));
  const size_t smem = kDrawTileW * kDrawTileH * sizeof(uint16_t) + (size_t)n * sizeof(int) + (OUT == kOutBlend ? 3 * nc : 0);
  const DrawImage one{0, 0, h, w};
  if (fmt == kMaskBits)
    k_draw_masks<kMaskBits, OUT><<<grid, kDrawThreads, smem, stream>>>(img, nullptr, one, masks, n, ids, nullptr, palette, nc, out);
  else if (fmt == kMaskF32)
    k_draw_masks<kMaskF32, OUT><<<grid, kDrawThreads, smem, stream>>>(img, nullptr, one, masks, n, ids, nullptr, palette, nc, out);
  else
    k_draw_masks<kMaskU8, OUT><<<grid, kDrawThreads, smem, stream>>>(img, nullptr, one, masks, n, ids, nullptr, palette, nc, out);
  YB_CHECK_LAUNCH();
  return YB_OK;
}

// NaN-propagating max, as torch.max
__device__ __forceinline__ float nan_max(float a, float b) { return (a != a || a > b) ? a : b; }

// |coef| order key: NaN after every number (numpy's argsort puts NaN last), then descending magnitude
__device__ __forceinline__ bool lincomb_before(float a, int ia, float b, int ib) {
  const bool na = a != a, nb = b != b;
  if (na != nb) return nb;
  if (!na && a != b) return a > b;
  return ia < ib;
}

// one block per (cell, image): cell i = 8r + c shows channel order[i] of image blockIdx.y's detection 0 at rows [rP, rP+P), cols
// [cP, cP+P) of its [4P, 8P, 3] output
__global__ void __launch_bounds__(kLincombThreads)
k_draw_lincomb(const float* __restrict__ proto, const float* __restrict__ coef, const int32_t* __restrict__ count, int D, int P,
               const uint8_t* __restrict__ lut, uint8_t* __restrict__ out) {
  const int cell = blockIdx.x, b = blockIdx.y, tid = threadIdx.x;
  if (count && count[b] <= 0) return;
  __shared__ int s_ch;
  __shared__ float s_red[kLincombThreads / 32];
  __shared__ uint8_t s_lut[256 * 3];
  const float* cf = coef + (size_t)b * D * kLincombK;                   // detection 0
  if (tid < kLincombK) {
    const float a = fabsf(cf[tid]);
    int rank = 0;
    for (int j = 0; j < kLincombK; ++j) rank += j != tid && lincomb_before(fabsf(cf[j]), j, a, tid);
    if (rank == cell) s_ch = tid;
  }
  for (int i = tid; i < 256 * 3; i += kLincombThreads) s_lut[i] = lut[i];
  __syncthreads();
  const int ch = s_ch;
  const int PP = P * P;
  const float* pr = proto + (size_t)b * PP * kLincombK + ch;
  float m = -INFINITY;
  for (int q = tid; q < PP; q += kLincombThreads) m = nan_max(m, pr[(size_t)q * kLincombK]);
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) m = nan_max(m, __shfl_xor_sync(0xffffffffu, m, o));
  if ((tid & 31) == 0) s_red[tid >> 5] = m;
  __syncthreads();
  m = s_red[0];
#pragma unroll
  for (int k = 1; k < kLincombThreads / 32; ++k) m = nan_max(m, s_red[k]);
  const float c = cf[ch];
  const int r0 = (cell / kLincombCols) * P, c0 = (cell % kLincombCols) * P;
  const size_t row_bytes = (size_t)kLincombCols * P * 3;
  uint8_t* dst = out + (size_t)b * kLincombRows * P * row_bytes;
  for (int q = tid; q < PP * 3; q += kLincombThreads) {             // output bytes of the cell, row by row
    const int y = q / (3 * P), rem = q - y * 3 * P, x = rem / 3, k = rem - 3 * x;
    const float v = __fmul_rn(__fdiv_rn(pr[((size_t)y * P + x) * kLincombK], m), c);
    // ((arr + 1) * 127.5).astype('uint8') on x86-64: truncation to int32 (NaN and out-of-range give INT_MIN), low byte kept
    const double u = ((double)v + 1.0) * 127.5;
    const int t = (u > -2147483649.0 && u < 2147483648.0) ? (int)u : INT_MIN;
    dst[(size_t)(r0 + y) * row_bytes + (size_t)(c0 + x) * 3 + k] = s_lut[3 * (t & 255) + k];
  }
}

static int check_draw_args(const char* fn, const uint8_t* img, int h, int w, const void* masks, int fmt, int n, const int32_t* ids,
                           int nc) {
  YB_REQUIRE(img, YB_ERR_INVALID, "%s: NULL image", fn);
  YB_REQUIRE(h > 0 && w > 0 && h <= 65535 * kDrawTileH && w <= (1 << 24), YB_ERR_INVALID, "%s: bad image size h=%d w=%d", fn, h, w);
  YB_REQUIRE(fmt >= kMaskU8 && fmt <= kMaskBits, YB_ERR_INVALID, "%s: mask_fmt=%d (0 uint8, 1 float32, 2 bits)", fn, fmt);
  YB_REQUIRE(n >= 0 && n <= kDrawMaxDet, YB_ERR_UNSUPPORTED, "%s: n=%d (0 .. %d masks)", fn, n, kDrawMaxDet);
  YB_REQUIRE(n == 0 || (masks && ids), YB_ERR_INVALID, "%s: NULL masks / ids", fn);
  YB_REQUIRE(((uintptr_t)masks & (fmt == kMaskF32 ? 15 : 3)) == 0, YB_ERR_INVALID, "%s: masks not %d-byte aligned", fn,
             fmt == kMaskF32 ? 16 : 4);
  YB_REQUIRE(nc >= 1 && nc <= kDrawMaxColors, YB_ERR_INVALID, "%s: num_colors=%d (1 .. %d)", fn, nc, kDrawMaxColors);
  return YB_OK;
}

}  // namespace yb

using namespace yb;

extern "C" int yb_draw_masks(const uint8_t* img_bgr, int h, int w, const void* masks, int mask_fmt, int n, const int32_t* ids,
                             const uint8_t* palette, int num_colors, uint8_t* out_bgr, void* stream) {
  YB_PROPAGATE(check_draw_args("yb_draw_masks", img_bgr, h, w, masks, mask_fmt, n, ids, num_colors));
  YB_REQUIRE(palette && out_bgr, YB_ERR_INVALID, "yb_draw_masks: NULL palette / output");
  return launch_draw<kOutBlend>(img_bgr, h, w, masks, mask_fmt, n, ids, palette, num_colors, out_bgr, (cudaStream_t)stream);
}

extern "C" int yb_draw_cutout(const uint8_t* img_bgr, int h, int w, const void* masks, int mask_fmt, int n, const int32_t* ids,
                              int num_colors, const int32_t* crop_yyxx, const int64_t* crop_off, uint8_t* out_total,
                              uint8_t* out_crops, void* stream) {
  YB_PROPAGATE(check_draw_args("yb_draw_cutout", img_bgr, h, w, masks, mask_fmt, n, ids, num_colors));
  YB_REQUIRE(out_total, YB_ERR_INVALID, "yb_draw_cutout: NULL total_obj output");
  YB_REQUIRE(n == 0 || (crop_yyxx && crop_off && out_crops), YB_ERR_INVALID, "yb_draw_cutout: NULL crop table / output");
  cudaStream_t st = (cudaStream_t)stream;
  YB_PROPAGATE(launch_draw<kOutMatte>(img_bgr, h, w, masks, mask_fmt, n, ids, nullptr, num_colors, out_total, st));
  if (n == 0) return YB_OK;
  // blocks per crop: enough for a crop of the whole image to fill the GPU a few times over; the rest grid-strides
  const size_t hw = (size_t)h * w;
  const int bx = hw >= (size_t)kCutoutBlocks * kDrawThreads ? kCutoutBlocks : ceil_div((int)hw, kDrawThreads);
  k_draw_cutout<<<dim3(bx, n), kDrawThreads, 0, st>>>(img_bgr, h, w, masks, mask_fmt, crop_yyxx, crop_off, out_crops);
  YB_CHECK_LAUNCH();
  return YB_OK;
}

extern "C" size_t yb_draw_masks_batch_workspace_bytes(int batch) {
  return batch <= 0 ? 0 : align_up((size_t)batch * sizeof(DrawImage), 256);
}

extern "C" int yb_draw_masks_batch(const uint8_t* src, int64_t src_bytes, const yb_val_aug_item* items, int batch, const uint32_t* masks,
                                   const int64_t* mask_off, int64_t mask_words, int max_det, const int32_t* ids, const int32_t* count,
                                   const uint8_t* palette, int num_colors, void* workspace, size_t workspace_bytes, uint8_t* out,
                                   void* stream) {
  YB_REQUIRE(src && items && masks && mask_off && ids && count && palette && workspace && out, YB_ERR_INVALID,
             "yb_draw_masks_batch: NULL pointer argument");
  YB_REQUIRE(src_bytes > 0 && batch > 0 && batch <= 65535 && mask_words >= 0, YB_ERR_INVALID,
             "yb_draw_masks_batch: src_bytes=%lld batch=%d mask_words=%lld", (long long)src_bytes, batch, (long long)mask_words);
  YB_REQUIRE(max_det >= 1 && max_det <= kDrawMaxDet, YB_ERR_UNSUPPORTED, "yb_draw_masks_batch: max_det=%d (1 .. %d)", max_det, kDrawMaxDet);
  YB_REQUIRE(num_colors >= 1 && num_colors <= kDrawMaxColors, YB_ERR_INVALID, "yb_draw_masks_batch: num_colors=%d (1 .. %d)", num_colors,
             kDrawMaxColors);
  YB_REQUIRE(((uintptr_t)masks & 3) == 0, YB_ERR_INVALID, "yb_draw_masks_batch: masks not 4-byte aligned");
  YB_REQUIRE(out + src_bytes <= src || src + src_bytes <= out, YB_ERR_INVALID, "yb_draw_masks_batch: out overlaps src");
  YB_REQUIRE(workspace_bytes >= yb_draw_masks_batch_workspace_bytes(batch), YB_ERR_INVALID, "yb_draw_masks_batch: workspace %zu bytes < %zu",
             workspace_bytes, yb_draw_masks_batch_workspace_bytes(batch));
  std::vector<DrawImage> imgs(batch);
  int max_h = 0, max_w = 0;
  YB_REQUIRE(mask_off[0] >= 0, YB_ERR_INVALID, "yb_draw_masks_batch: mask_off[0]=%lld", (long long)mask_off[0]);
  for (int b = 0; b < batch; ++b) {
    const yb_val_aug_item& t = items[b];
    YB_REQUIRE(t.h > 0 && t.w > 0 && t.h <= 65535 * kDrawTileH && t.w <= (1 << 24), YB_ERR_INVALID, "yb_draw_masks_batch: item %d: h=%d w=%d",
               b, t.h, t.w);
    const int64_t bytes = (int64_t)t.h * t.w * 3;
    YB_REQUIRE(t.img_off >= 0 && t.img_off <= src_bytes - bytes, YB_ERR_INVALID,
               "yb_draw_masks_batch: item %d: image [%lld, +%lld) outside src (%lld bytes)", b, (long long)t.img_off, (long long)bytes,
               (long long)src_bytes);
    const int64_t need = (int64_t)max_det * t.h * ((t.w + 31) / 32);
    YB_REQUIRE(mask_off[b + 1] >= 0 && mask_off[b] <= mask_off[b + 1] - need, YB_ERR_INVALID,
               "yb_draw_masks_batch: image %d (%dx%d, %d masks) needs %lld words from mask_off %lld, the next image starts at %lld", b,
               t.h, t.w, max_det, (long long)need, (long long)mask_off[b], (long long)mask_off[b + 1]);
    imgs[b] = DrawImage{t.img_off, mask_off[b], t.h, t.w};
    max_h = max(max_h, t.h);
    max_w = max(max_w, t.w);
  }
  YB_REQUIRE(mask_off[batch] <= mask_words, YB_ERR_INVALID, "yb_draw_masks_batch: mask_off[%d]=%lld beyond the %lld mask words", batch,
             (long long)mask_off[batch], (long long)mask_words);
  cudaStream_t st = (cudaStream_t)stream;
  const StagePart part{imgs.data(), (size_t)batch * sizeof(DrawImage), 0};
  YB_PROPAGATE(stage_tables(workspace, part.bytes, &part, 1, st));
  const dim3 grid(ceil_div(max_w, kDrawTileW), ceil_div(max_h, kDrawTileH), batch);
  const size_t smem = kDrawTileW * kDrawTileH * sizeof(uint16_t) + (size_t)max_det * sizeof(int) + 3 * num_colors;
  k_draw_masks<kMaskBits, kOutBlend><<<grid, kDrawThreads, smem, st>>>(src, (const DrawImage*)workspace, DrawImage{}, masks, max_det, ids,
                                                                        count, palette, num_colors, out);
  YB_CHECK_LAUNCH();
  return YB_OK;
}

extern "C" int yb_draw_lincomb(const float* proto, const float* coef, const int32_t* count, int batch, int max_det, int proto_size,
                               int coef_dim, const uint8_t* lut, uint8_t* out, void* stream) {
  YB_REQUIRE(proto && coef && lut && out, YB_ERR_INVALID, "yb_draw_lincomb: NULL pointer argument");
  YB_REQUIRE(coef_dim == kLincombK, YB_ERR_UNSUPPORTED, "yb_draw_lincomb: coef_dim=%d (the 4 x 8 grid needs 32)", coef_dim);
  YB_REQUIRE(batch > 0 && batch <= 65535 && max_det > 0 && proto_size > 0 && proto_size <= 4096, YB_ERR_INVALID,
             "yb_draw_lincomb: batch=%d max_det=%d P=%d", batch, max_det, proto_size);
  k_draw_lincomb<<<dim3(kLincombRows * kLincombCols, batch), kLincombThreads, 0, (cudaStream_t)stream>>>(proto, coef, count, max_det,
                                                                                                          proto_size, lut, out);
  YB_CHECK_LAUNCH();
  return YB_OK;
}
