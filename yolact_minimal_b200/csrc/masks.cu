// Mask assembly on the GPU.  Replaces utils/output_utils.py:217-231 (after_nms) and
// utils/box_utils.py:117-132,:147-168 (sanitize_coordinates, crop):
//   low  = crop(sigmoid(proto[P,P,K] @ coef[d,K]^T))            k_mask_lowres   -> ws[d,P,P]
//   mask = bilinear(low -> max(h,w)^2, align_corners=False) > 0.5, sliced to h x w   k_mask_resize
//   boxes_px = int32(trunc(box * max(h,w)))
// Both kernels are HBM/L2 streaming kernels: proto is read once per 16-detection group (from
// L2 after the first), the full-resolution mask is written once, coalesced along x.
// The same kernels run a batch (yb_mask_assemble_batch): blockIdx.z (k_boxes_px: blockIdx.y) is the image, and a DEVICE count
// per image turns the blocks of detections at or past it into early exits.  A single-image call passes count = NULL.
#include "common.cuh"
#include <math.h>
#include <vector>

namespace yb {

constexpr int kMaskThreads = 256;
constexpr int kDetGroup = 16;      // detections per lowres thread (registers hold 16 accumulators)
constexpr int kMaxK = 64;

// one image of a batch: first output word of its masks, size
struct MaskImage {
  int64_t off;
  int32_t h, w;
};

// detections of image `img` to assemble: the device count (clamped to [0, d]) or all d
__device__ __forceinline__ int live_dets(const int32_t* count, int img, int d) { return count ? min(max(count[img], 0), d) : d; }

// proto pixel per thread; blockIdx.y = detection group, blockIdx.z = image (proto [P,P,K], coef [d,K], box [d,4], low [d,P,P] each)
__global__ void __launch_bounds__(kMaskThreads)
k_mask_lowres(const float* __restrict__ proto, const float* __restrict__ coef, const float* __restrict__ box,
              const int32_t* __restrict__ count, int d, int P, int K, int crop, float* __restrict__ low) {
  __shared__ float s_coef[kDetGroup][kMaxK];
  __shared__ float s_x1[kDetGroup], s_x2[kDetGroup], s_y1[kDetGroup], s_y2[kDetGroup];
  const int img = blockIdx.z;
  const int n = live_dets(count, img, d);
  const int g0 = blockIdx.y * kDetGroup;
  if (g0 >= n) return;
  const int ng = min(kDetGroup, n - g0);
  const int tid = threadIdx.x;
  proto += (size_t)img * P * P * K;
  coef += (size_t)img * d * K;
  box += (size_t)img * d * 4;
  low += (size_t)img * d * P * P;
  for (int e = tid; e < ng * K; e += kMaskThreads) s_coef[e / K][e % K] = coef[(size_t)(g0 + e / K) * K + e % K];
  if (tid < ng) {
    // sanitize_coordinates (box_utils.py:124-132), padding = 1, float compares, no rounding
    const float4 b = reinterpret_cast<const float4*>(box)[g0 + tid];
    const float fp = (float)P;
    float xa = __fmul_rn(b.x, fp), xb = __fmul_rn(b.z, fp), ya = __fmul_rn(b.y, fp), yb_ = __fmul_rn(b.w, fp);
    float x1 = fminf(xa, xb), x2 = fmaxf(xa, xb), y1 = fminf(ya, yb_), y2 = fmaxf(ya, yb_);
    x1 = __fsub_rn(x1, 1.f); x1 = x1 < 0.f ? 0.f : x1;
    y1 = __fsub_rn(y1, 1.f); y1 = y1 < 0.f ? 0.f : y1;
    x2 = __fadd_rn(x2, 1.f); x2 = x2 > fp ? fp : x2;
    y2 = __fadd_rn(y2, 1.f); y2 = y2 > fp ? fp : y2;
    s_x1[tid] = x1; s_x2[tid] = x2; s_y1[tid] = y1; s_y2[tid] = y2;
  }
  __syncthreads();
  const int pix = blockIdx.x * kMaskThreads + tid;
  if (pix >= P * P) return;
  const int y = pix / P, x = pix - y * P;
  float acc[kDetGroup];
#pragma unroll
  for (int g = 0; g < kDetGroup; ++g) acc[g] = 0.f;
  const float* pp = proto + (size_t)pix * K;
  for (int k0 = 0; k0 < K; k0 += 4) {
    const float4 pv = *reinterpret_cast<const float4*>(pp + k0);
#pragma unroll
    for (int g = 0; g < kDetGroup; ++g) {
      acc[g] = fmaf(pv.x, s_coef[g][k0], acc[g]);
      acc[g] = fmaf(pv.y, s_coef[g][k0 + 1], acc[g]);
      acc[g] = fmaf(pv.z, s_coef[g][k0 + 2], acc[g]);
      acc[g] = fmaf(pv.w, s_coef[g][k0 + 3], acc[g]);
    }
  }
  const float fx = (float)x, fy = (float)y;
#pragma unroll
  for (int g = 0; g < kDetGroup; ++g) {
    if (g < ng) {
      float v = __fdiv_rn(1.f, __fadd_rn(1.f, expf(-acc[g])));
      if (crop) {
        const bool in = (fx >= s_x1[g]) && (fx < s_x2[g]) && (fy >= s_y1[g]) && (fy < s_y2[g]);
        v = in ? v : 0.f;
      }
      low[((size_t)(g0 + g) * P + y) * P + x] = v;
    }
  }
}

// ATen upsample_bilinear2d (align_corners=False) source index, fp32 arithmetic
__device__ __forceinline__ void bilinear_src(int dst, float scale, int in_size, int& i0, int& i1, float& l0, float& l1) {
  float src = __fsub_rn(__fmul_rn(scale, __fadd_rn((float)dst, 0.5f)), 0.5f);
  src = src < 0.f ? 0.f : src;
  i0 = min((int)src, in_size - 1);
  i1 = min(i0 + 1, in_size - 1);
  l1 = __fsub_rn(src, (float)i0);
  l0 = __fsub_rn(1.f, l1);
}

// One thread = a 4 x 4 patch of output pixels: the four column interpolations (index pair + weights) are computed once and reused
// for four rows, each row leaves as one 16-byte float4 / 4-byte uchar4 store when the row pitch allows it.  (One pixel per thread
// was launch / index bound -- 144k blocks, ~50 instructions per pixel, 137 us for 100 masks of 480 x 640 where the bytes take 20 us;
// four pixels of one row per thread: 81 us.)  Per-pixel arithmetic is unchanged (ATen's order, separately rounded).
constexpr int kMaskRows = 4;

template <typename OutT>
__global__ void __launch_bounds__(kMaskThreads)
k_mask_resize(const float* __restrict__ low, int d, int P, int ori, int img_h, int img_w, OutT* __restrict__ out) {
  const int det = blockIdx.y;
  const int nq = (img_w + 3) >> 2;                                     // pixel quads per row
  const int q = blockIdx.x * kMaskThreads + threadIdx.x;
  if (q >= nq * ((img_h + kMaskRows - 1) / kMaskRows)) return;
  const int rg = q / nq, ox0 = (q - rg * nq) * 4;
  const float scale = __fdiv_rn((float)P, (float)ori);
  int x0[4], x1[4]; float lx0[4], lx1[4];
#pragma unroll
  for (int i = 0; i < 4; ++i) bilinear_src(min(ox0 + i, img_w - 1), scale, P, x0[i], x1[i], lx0[i], lx1[i]);
  const float* src = low + (size_t)det * P * P;
#pragma unroll
  for (int r = 0; r < kMaskRows; ++r) {
    const int oy = rg * kMaskRows + r;
    if (oy >= img_h) break;
    int y0, y1; float ly0, ly1;
    bilinear_src(oy, scale, P, y0, y1, ly0, ly1);
    const float* r0 = src + (size_t)y0 * P;
    const float* r1 = src + (size_t)y1 * P;
    OutT o[4];
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      // ATen: w_y0 * (w_x0 * v00 + w_x1 * v01) + w_y1 * (w_x0 * v10 + w_x1 * v11)
      const float top = __fadd_rn(__fmul_rn(lx0[i], r0[x0[i]]), __fmul_rn(lx1[i], r0[x1[i]]));
      const float bot = __fadd_rn(__fmul_rn(lx0[i], r1[x0[i]]), __fmul_rn(lx1[i], r1[x1[i]]));
      const float v = __fadd_rn(__fmul_rn(ly0, top), __fmul_rn(ly1, bot));
      o[i] = (OutT)(v > 0.5f ? 1 : 0);
    }
    OutT* dst = out + ((size_t)det * img_h + oy) * img_w + ox0;
    if ((img_w & 3) == 0) {
      if (sizeof(OutT) == 4) *reinterpret_cast<float4*>(dst) = make_float4((float)o[0], (float)o[1], (float)o[2], (float)o[3]);
      else *reinterpret_cast<uchar4*>(dst) = make_uchar4((unsigned char)o[0], (unsigned char)o[1], (unsigned char)o[2], (unsigned char)o[3]);
    } else {
#pragma unroll
      for (int i = 0; i < 4; ++i) if (ox0 + i < img_w) dst[i] = o[i];
    }
  }
}

// bit-packed output: one thread = one 32-pixel word of kMaskRows consecutive output rows (1 bit / pixel: 32x less HBM write traffic
// than float32 masks); the column interpolation of a pixel is computed once for the four rows.  blockIdx.z = image: its geometry
// comes from imgs[blockIdx.z] (batch) or `one` (imgs = NULL), its masks start at word `off` of out; low holds d masks per image.
__global__ void __launch_bounds__(kMaskThreads)
k_mask_resize_bits(const float* __restrict__ low, int P, int d, const int32_t* __restrict__ count, const MaskImage* __restrict__ imgs,
                   MaskImage one, uint32_t* __restrict__ out) {
  const int img = blockIdx.z, det = blockIdx.y, q = blockIdx.x * kMaskThreads + threadIdx.x;   // (row group, word) flattened: rows are only ~20 words wide
  if (det >= live_dets(count, img, d)) return;
  const MaskImage g = imgs ? imgs[img] : one;
  const int img_h = g.h, img_w = g.w, words = (img_w + 31) / 32, ori = img_h > img_w ? img_h : img_w;
  if (q >= words * ((img_h + kMaskRows - 1) / kMaskRows)) return;
  out += g.off;
  const int rg = q / words, wi = q - rg * words;
  const float scale = __fdiv_rn((float)P, (float)ori);
  const float* src = low + ((size_t)img * d + det) * P * P;
  const float* r0[kMaskRows]; const float* r1[kMaskRows];
  float ly0[kMaskRows], ly1[kMaskRows];
  uint32_t v[kMaskRows];
#pragma unroll
  for (int r = 0; r < kMaskRows; ++r) {
    int y0, y1;
    bilinear_src(min(rg * kMaskRows + r, img_h - 1), scale, P, y0, y1, ly0[r], ly1[r]);
    r0[r] = src + (size_t)y0 * P; r1[r] = src + (size_t)y1 * P;
    v[r] = 0u;
  }
  const int cnt = min(32, img_w - wi * 32);
  for (int b = 0; b < cnt; ++b) {
    int x0, x1; float lx0, lx1;
    bilinear_src(wi * 32 + b, scale, P, x0, x1, lx0, lx1);
#pragma unroll
    for (int r = 0; r < kMaskRows; ++r) {
      const float top = __fadd_rn(__fmul_rn(lx0, r0[r][x0]), __fmul_rn(lx1, r0[r][x1]));
      const float bot = __fadd_rn(__fmul_rn(lx0, r1[r][x0]), __fmul_rn(lx1, r1[r][x1]));
      v[r] |= (__fadd_rn(__fmul_rn(ly0[r], top), __fmul_rn(ly1[r], bot)) > 0.5f ? 1u : 0u) << b;
    }
  }
#pragma unroll
  for (int r = 0; r < kMaskRows; ++r) {
    const int oy = rg * kMaskRows + r;
    if (oy < img_h) out[((size_t)det * img_h + oy) * words + wi] = v[r];
  }
}

// blockIdx.y = image (n4 values each); with imgs, ori = max(h, w) of the image, and rows at or past its count are the zero box
__global__ void k_boxes_px(const float* __restrict__ box, int n4, const int32_t* __restrict__ count, const MaskImage* __restrict__ imgs,
                           float ori, int32_t* __restrict__ out) {
  const int img = blockIdx.y, i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n4) return;
  if (imgs) ori = (float)max(imgs[img].h, imgs[img].w);
  const size_t e = (size_t)img * n4 + i;
  out[e] = i / 4 < live_dets(count, img, n4 / 4) ? (int32_t)__fmul_rn(box[e], ori) : 0;      // .int() truncates toward zero
}

}  // namespace yb

using namespace yb;

extern "C" size_t yb_mask_workspace_bytes(int num_det, int proto_size) {
  if (num_det <= 0 || proto_size <= 0) return 0;
  return (size_t)num_det * proto_size * proto_size * sizeof(float);
}

extern "C" int yb_mask_assemble(const float* proto, const float* coef, const float* box, int num_det,
                                int proto_size, int coef_dim, int img_h, int img_w, int crop, int mask_f32,
                                void* workspace, size_t workspace_bytes, void* out_mask, int32_t* out_box_px,
                                void* stream_) {
  YB_REQUIRE(num_det >= 0, YB_ERR_INVALID, "yb_mask_assemble: num_det=%d", num_det);
  if (num_det == 0) return YB_OK;
  YB_REQUIRE(proto && coef && box && workspace && out_mask && out_box_px, YB_ERR_INVALID, "yb_mask_assemble: NULL pointer argument");
  YB_REQUIRE(proto_size > 0 && img_h > 0 && img_w > 0, YB_ERR_INVALID, "yb_mask_assemble: bad sizes P=%d h=%d w=%d", proto_size, img_h, img_w);
  YB_REQUIRE(coef_dim > 0 && coef_dim <= kMaxK && coef_dim % 4 == 0, YB_ERR_UNSUPPORTED, "yb_mask_assemble: coef_dim=%d (need multiple of 4, <= %d)", coef_dim, kMaxK);
  YB_REQUIRE(workspace_bytes >= yb_mask_workspace_bytes(num_det, proto_size), YB_ERR_INVALID, "yb_mask_assemble: workspace too small");
  YB_REQUIRE(num_det <= 65535 && img_h <= 65535, YB_ERR_UNSUPPORTED, "yb_mask_assemble: num_det/img_h exceed grid limits");
  cudaStream_t stream = (cudaStream_t)stream_;
  const int P = proto_size, ori = img_h > img_w ? img_h : img_w;
  float* low = (float*)workspace;
  k_mask_lowres<<<dim3(ceil_div(P * P, kMaskThreads), ceil_div(num_det, kDetGroup)), kMaskThreads, 0, stream>>>(
      proto, coef, box, nullptr, num_det, P, coef_dim, crop, low);
  YB_CHECK_LAUNCH();
  dim3 grid(ceil_div(((img_w + 3) / 4) * ((img_h + kMaskRows - 1) / kMaskRows), kMaskThreads), num_det);
  if (mask_f32 == 2) {
    const int words = (img_w + 31) / 32;
    k_mask_resize_bits<<<dim3(ceil_div(words * ((img_h + kMaskRows - 1) / kMaskRows), kMaskThreads), num_det), kMaskThreads, 0, stream>>>(
        low, P, num_det, nullptr, nullptr, MaskImage{0, img_h, img_w}, (uint32_t*)out_mask);
  } else if (mask_f32 == 1) k_mask_resize<float><<<grid, kMaskThreads, 0, stream>>>(low, num_det, P, ori, img_h, img_w, (float*)out_mask);
  else k_mask_resize<uint8_t><<<grid, kMaskThreads, 0, stream>>>(low, num_det, P, ori, img_h, img_w, (uint8_t*)out_mask);
  YB_CHECK_LAUNCH();
  k_boxes_px<<<ceil_div(num_det * 4, 128), 128, 0, stream>>>(box, num_det * 4, nullptr, nullptr, (float)ori, out_box_px);
  YB_CHECK_LAUNCH();
  return YB_OK;
}

namespace {
size_t batch_low_bytes(int batch, int max_det, int P) { return yb::align_up((size_t)batch * max_det * P * P * sizeof(float), 256); }
}  // namespace

extern "C" size_t yb_mask_assemble_batch_workspace_bytes(int batch, int max_det, int proto_size) {
  if (batch <= 0 || max_det <= 0 || proto_size <= 0) return 0;
  return batch_low_bytes(batch, max_det, proto_size) + yb::align_up((size_t)batch * sizeof(MaskImage), 256);
}

extern "C" int yb_mask_assemble_batch(const float* proto, const float* coef, const float* box, const int32_t* count, int batch,
                                      int max_det, int proto_size, int coef_dim, const int32_t* img_hw, const int64_t* mask_off,
                                      int64_t mask_words, int crop, void* workspace, size_t workspace_bytes, uint32_t* out_mask,
                                      int32_t* out_box_px, void* stream_) {
  YB_REQUIRE(proto && coef && box && count && img_hw && mask_off && workspace && out_mask && out_box_px, YB_ERR_INVALID,
             "yb_mask_assemble_batch: NULL pointer argument");
  YB_REQUIRE(batch > 0 && batch <= 65535 && max_det > 0 && max_det <= 65535 && proto_size > 0 && mask_words >= 0, YB_ERR_INVALID,
             "yb_mask_assemble_batch: batch=%d max_det=%d P=%d mask_words=%lld", batch, max_det, proto_size, (long long)mask_words);
  YB_REQUIRE(coef_dim > 0 && coef_dim <= kMaxK && coef_dim % 4 == 0, YB_ERR_UNSUPPORTED,
             "yb_mask_assemble_batch: coef_dim=%d (need multiple of 4, <= %d)", coef_dim, kMaxK);
  YB_REQUIRE(workspace_bytes >= yb_mask_assemble_batch_workspace_bytes(batch, max_det, proto_size), YB_ERR_INVALID,
             "yb_mask_assemble_batch: workspace %zu bytes < %zu", workspace_bytes,
             yb_mask_assemble_batch_workspace_bytes(batch, max_det, proto_size));
  std::vector<MaskImage> imgs(batch);
  int max_q = 0;
  YB_REQUIRE(mask_off[0] >= 0, YB_ERR_INVALID, "yb_mask_assemble_batch: mask_off[0]=%lld", (long long)mask_off[0]);
  for (int b = 0; b < batch; ++b) {
    const int h = img_hw[2 * b], w = img_hw[2 * b + 1];
    YB_REQUIRE(h > 0 && w > 0 && h <= 65535 && w <= 65535, YB_ERR_INVALID, "yb_mask_assemble_batch: image %d is %dx%d", b, h, w);
    const int words = (w + 31) / 32;
    const int64_t need = (int64_t)max_det * h * words;
    YB_REQUIRE(mask_off[b + 1] >= 0 && mask_off[b] <= mask_off[b + 1] - need, YB_ERR_INVALID,
               "yb_mask_assemble_batch: image %d (%dx%d, %d detections) needs %lld words from mask_off %lld, the next image starts at %lld",
               b, h, w, max_det, (long long)need, (long long)mask_off[b], (long long)mask_off[b + 1]);
    imgs[b] = MaskImage{mask_off[b], h, w};
    max_q = max(max_q, words * ((h + kMaskRows - 1) / kMaskRows));
  }
  YB_REQUIRE(mask_off[batch] <= mask_words, YB_ERR_INVALID, "yb_mask_assemble_batch: mask_off[%d]=%lld beyond the %lld output words", batch,
             (long long)mask_off[batch], (long long)mask_words);
  cudaStream_t stream = (cudaStream_t)stream_;
  const int P = proto_size, D = max_det;
  float* low = (float*)workspace;
  MaskImage* d_imgs = (MaskImage*)((char*)workspace + batch_low_bytes(batch, D, P));
  const yb::StagePart part{imgs.data(), (size_t)batch * sizeof(MaskImage), 0};
  YB_PROPAGATE(yb::stage_tables(d_imgs, part.bytes, &part, 1, stream));
  k_mask_lowres<<<dim3(ceil_div(P * P, kMaskThreads), ceil_div(D, kDetGroup), batch), kMaskThreads, 0, stream>>>(
      proto, coef, box, count, D, P, coef_dim, crop, low);
  YB_CHECK_LAUNCH();
  k_mask_resize_bits<<<dim3(ceil_div(max_q, kMaskThreads), D, batch), kMaskThreads, 0, stream>>>(low, P, D, count, d_imgs, MaskImage{},
                                                                                                   out_mask);
  YB_CHECK_LAUNCH();
  k_boxes_px<<<dim3(ceil_div(D * 4, 128), batch), 128, 0, stream>>>(box, D * 4, count, d_imgs, 0.f, out_box_px);
  YB_CHECK_LAUNCH();
  return YB_OK;
}

// ================================================================================================
// Pre-process (SURVEY.md 8(f) rank 1): the reference's val_aug on the GPU --
// utils/augmentations.py:219-227: uint8 BGR HWC -> float32, pad to square at the top-left with the
// BGR mean (:138-165), bilinear resize to S x S with OpenCV's INTER_LINEAR coordinate rule
// (fx = (dx+0.5)*scale-0.5, clamped taps), (x-mean)/std, BGR->RGB, CHW (:212-216).  One kernel,
// one read of the uint8 image, one write of the network input (4x less H2D than fp32 images).
// k_val_aug does one image; k_val_aug_batch a batch of images of any sizes packed in one buffer (grid: pixel tiles x image).
// Both compute each output pixel with val_aug_pixel, so image b of a batch equals yb_val_aug on image b bit for bit.
// ================================================================================================
namespace yb {
// output pixel i (of S*S) of one image: out = the image's [3,S,S] planes
__device__ __forceinline__ void val_aug_pixel(const uint8_t* __restrict__ img, int h, int w, int S, int i, float* __restrict__ out) {
  const int P = h > w ? h : w;
  const double scale = (double)P / (double)S;
  const float mean[3] = {103.94f, 116.78f, 123.68f}, stdv[3] = {57.38f, 57.12f, 58.40f};
  const int total = S * S;
  const int dy = i / S, dx = i - dy * S;
  float fx = (float)(((double)dx + 0.5) * scale - 0.5), fy = (float)(((double)dy + 0.5) * scale - 0.5);
  int sx = (int)floorf(fx), sy = (int)floorf(fy);
  fx -= (float)sx; fy -= (float)sy;
  if (sx < 0) { sx = 0; fx = 0.f; }
  if (sx >= P - 1) { sx = P - 1; fx = 0.f; }
  if (sy < 0) { sy = 0; fy = 0.f; }
  if (sy >= P - 1) { sy = P - 1; fy = 0.f; }
  const int sx1 = min(sx + 1, P - 1), sy1 = min(sy + 1, P - 1);
#pragma unroll
  for (int c = 0; c < 3; ++c) {                      // c indexes BGR; output channel is 2 - c (RGB)
    auto px = [&](int y, int x) -> float { return (y < h && x < w) ? (float)img[((size_t)y * w + x) * 3 + c] : mean[c]; };
    const float r0 = px(sy, sx) * (1.f - fx) + px(sy, sx1) * fx;
    const float r1 = px(sy1, sx) * (1.f - fx) + px(sy1, sx1) * fx;
    const float v = r0 * (1.f - fy) + r1 * fy;
    out[(size_t)(2 - c) * total + i] = (v - mean[c]) / stdv[c];
  }
}

__global__ void __launch_bounds__(256) k_val_aug(const uint8_t* __restrict__ img, int h, int w, int S, float* __restrict__ out) {
  const int total = S * S;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < total; i += gridDim.x * blockDim.x) val_aug_pixel(img, h, w, S, i, out);
}

__global__ void __launch_bounds__(256) k_val_aug_batch(const uint8_t* __restrict__ src, const yb_val_aug_item* __restrict__ items, int S,
                                                       float* __restrict__ out) {
  const yb_val_aug_item it = items[blockIdx.y];
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < S * S) val_aug_pixel(src + it.img_off, it.h, it.w, S, i, out + (size_t)blockIdx.y * 3 * S * S);
}
}  // namespace yb

extern "C" int yb_val_aug(const uint8_t* img_bgr, int h, int w, int img_size, float* out, void* stream) {
  YB_REQUIRE(img_bgr && out, YB_ERR_INVALID, "yb_val_aug: NULL pointer argument");
  YB_REQUIRE(h > 0 && w > 0 && img_size > 0 && img_size <= 8192, YB_ERR_INVALID, "yb_val_aug: h=%d w=%d img_size=%d", h, w, img_size);
  const int total = img_size * img_size;
  yb::k_val_aug<<<yb::ceil_div(total, 256), 256, 0, (cudaStream_t)stream>>>(img_bgr, h, w, img_size, out);
  YB_CHECK_LAUNCH();
  return YB_OK;
}

namespace {
size_t val_items_bytes(int n_items) { return yb::align_up((size_t)n_items * sizeof(yb_val_aug_item), 256); }
}  // namespace

extern "C" size_t yb_val_aug_batch_workspace_bytes(int n_items) { return n_items < 0 ? 0 : val_items_bytes(n_items); }

extern "C" int yb_val_aug_batch(const uint8_t* src, int64_t src_bytes, const yb_val_aug_item* items, int n_items, int img_size,
                                void* workspace, size_t workspace_bytes, float* out, void* stream) {
  YB_REQUIRE(src && items && workspace && out, YB_ERR_INVALID, "yb_val_aug_batch: NULL pointer argument");
  YB_REQUIRE(src_bytes > 0 && n_items > 0 && n_items <= 65535, YB_ERR_INVALID, "yb_val_aug_batch: src_bytes=%lld n_items=%d",
             (long long)src_bytes, n_items);
  YB_REQUIRE(img_size > 0 && img_size <= 8192, YB_ERR_INVALID, "yb_val_aug_batch: img_size=%d", img_size);
  for (int i = 0; i < n_items; ++i) {
    const yb_val_aug_item& t = items[i];
    YB_REQUIRE(t.h > 0 && t.w > 0 && t.h <= 65535 && t.w <= 65535, YB_ERR_INVALID, "yb_val_aug_batch: item %d: h=%d w=%d", i, t.h, t.w);
    const int64_t bytes = (int64_t)t.h * t.w * 3;
    YB_REQUIRE(t.img_off >= 0 && t.img_off <= src_bytes - bytes, YB_ERR_INVALID,
               "yb_val_aug_batch: item %d: image [%lld, +%lld) outside src (%lld bytes)", i, (long long)t.img_off, (long long)bytes,
               (long long)src_bytes);
  }
  YB_REQUIRE(workspace_bytes >= val_items_bytes(n_items), YB_ERR_INVALID, "yb_val_aug_batch: workspace %zu bytes < %zu", workspace_bytes,
             val_items_bytes(n_items));
  cudaStream_t st = (cudaStream_t)stream;
  const yb::StagePart part{items, (size_t)n_items * sizeof(yb_val_aug_item), 0};
  YB_PROPAGATE(yb::stage_tables(workspace, part.bytes, &part, 1, st));
  const int S = img_size;
  yb::k_val_aug_batch<<<dim3(yb::ceil_div(S * S, 256), n_items), 256, 0, st>>>(src, (const yb_val_aug_item*)workspace, S, out);
  YB_CHECK_LAUNCH();
  return YB_OK;
}
