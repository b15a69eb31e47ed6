// Detection drawing on the GPU -- the pixel work of utils/output_utils.py:308-369 (draw_img):
//   semantic = (sum_i m_i * (ids_i + 1)) mod num_colors          (numpy floor modulo; m_i in {0,1})
//   overlay  = rint(0.4f * palette[semantic] + 0.6f * img)        k_draw_masks<.., kOutBlend>   (cv2.addWeighted(.., 0.4, .., 0.6, 0))
//   total_obj = semantic != 0 ? img : 255                         k_draw_masks<.., kOutMatte>   (cfg.cutout)
//   crop_i   = (m_i != 0 ? img : 255)[y1:y2, x1:x2]               k_draw_cutout                 (cfg.cutout)
// Masks come in the three layouts after_nms writes (yb_mask_assemble's codes): 0 uint8, 1 float32 [n,h,w], 2 bit-packed words
// [n,h,ceil(w/32)].  A block owns a kDrawTileW x kDrawTileH pixel tile.  Phase 1 reduces the n masks to the tile's semantic
// indices in shared memory, reading the masks coalesced (4 pixels per thread for bytes / floats, one 32-pixel word per thread for
// bits).  Phase 2 streams the tile's image bytes in order, so the image is read and written with fully used sectors.
#include "common.cuh"

namespace yb {

constexpr int kDrawThreads = 128;
constexpr int kDrawTileW = 256;            // pixels: 8 packed words, 64 threads x 4 pixels
constexpr int kDrawTileH = 16;             // rows: 16 x 8 words = one word per thread
constexpr int kDrawMaxDet = 4096;
constexpr int kDrawMaxColors = 1024;
constexpr int kCutoutBlocks = 64;
enum { kMaskU8 = 0, kMaskF32 = 1, kMaskBits = 2 };
enum { kOutBlend = 0, kOutMatte = 1 };

static_assert(kDrawTileW / 32 * kDrawTileH == kDrawThreads, "bits: one word per thread");
static_assert(kDrawTileW / 4 * 2 == kDrawThreads, "bytes / floats: two rows of 4-pixel groups per pass");

__device__ __forceinline__ int floor_mod(long long v, int m) {
  const long long r = v % m;
  return (int)(r < 0 ? r + m : r);
}

// dynamic shared memory: uint16 sem[tile] | int32 wgt[n] | uint8 palette[3 * num_colors]
// wgt_i = (ids_i + 1) mod num_colors, so the per-pixel sums stay below n * num_colors < 2^22 and sum mod num_colors is the
// reference's int64 sum mod num_colors.
template <int FMT, int OUT>
__global__ void __launch_bounds__(kDrawThreads)
k_draw_masks(const uint8_t* __restrict__ img, int h, int w, const void* __restrict__ masks, int n, const int32_t* __restrict__ ids,
             const uint8_t* __restrict__ palette, int nc, uint8_t* __restrict__ out) {
  extern __shared__ __align__(16) unsigned char s_raw[];
  uint16_t* s_sem = reinterpret_cast<uint16_t*>(s_raw);
  int* s_wgt = reinterpret_cast<int*>(s_raw + kDrawTileW * kDrawTileH * sizeof(uint16_t));
  uint8_t* s_pal = reinterpret_cast<uint8_t*>(s_wgt + n);
  const int tid = threadIdx.x;
  for (int i = tid; i < n; i += kDrawThreads) s_wgt[i] = floor_mod((long long)ids[i] + 1, nc);
  if (OUT == kOutBlend)
    for (int i = tid; i < 3 * nc; i += kDrawThreads) s_pal[i] = palette[i];
  __syncthreads();

  const int x0 = blockIdx.x * kDrawTileW, y0 = blockIdx.y * kDrawTileH;
  const size_t plane = (size_t)h * w;
  if (FMT == kMaskBits) {
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
    if (OUT == kOutBlend)   // cv2.addWeighted(color, 0.4, img, 0.6, 0) on uint8: each product rounded to fp32, sum rounded to nearest
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
  if (fmt == kMaskBits) k_draw_masks<kMaskBits, OUT><<<grid, kDrawThreads, smem, stream>>>(img, h, w, masks, n, ids, palette, nc, out);
  else if (fmt == kMaskF32) k_draw_masks<kMaskF32, OUT><<<grid, kDrawThreads, smem, stream>>>(img, h, w, masks, n, ids, palette, nc, out);
  else k_draw_masks<kMaskU8, OUT><<<grid, kDrawThreads, smem, stream>>>(img, h, w, masks, n, ids, palette, nc, out);
  YB_CHECK_LAUNCH();
  return YB_OK;
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
