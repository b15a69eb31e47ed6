// Baseline JPEG encoding of a batch of uint8 BGR images, byte for byte the file cv2.imencode('.jpg', img, [IMWRITE_JPEG_QUALITY, q])
// writes (libjpeg-turbo with cv2's defaults: 4:2:0, ISLOW DCT, Annex K Huffman tables, no restart markers).  oracle/jpeg_np.py
// states every rule in numpy; the kernels follow it step by step in the same integer arithmetic.
//
// Five launches, no host synchronisation:
//   k_jpeg_blocks  one CTA per (16x16 MCU, image): libjpeg's fixed-point RGB -> YCbCr, h2v2 downsampling with the 1, 2 bias,
//                  edge replication, ISLOW FDCT, reciprocal quantization, zigzag.  Writes int16 coefficient blocks in scan order
//                  (Y0 Y1 Y2 Y3 Cb Cr per MCU), the dummy blocks of a partial last MCU included.
//   k_jpeg_bits    one warp per block: the block's code length (DC difference against the previous block of its component).
//   k_jpeg_scan    one CTA per image: exclusive scan of the code lengths -> each block's bit offset; zeroes the words a block
//                  shares with its neighbours, so k_jpeg_emit needs no memset.
//   k_jpeg_emit    one warp per block: assembles its codes in shared memory, stores its interior words and ORs the two words it may
//                  share with the neighbouring blocks.
//   k_jpeg_stuff   one CTA per image: header (only SOF0's height and width vary), the bitstream padded with 1-bits, a 0x00 after
//                  every 0xFF byte, EOI; writes the file's length.
#include "common.cuh"

#include <cub/block/block_scan.cuh>
#include <vector>

namespace yb {
namespace {

constexpr int kJpegHeaderBytes = 623;     // SOI, APP0, 2 DQT, SOF0, 4 DHT, SOS
constexpr int kJpegSofOffset = 158;       // first byte of the SOF0 marker in the header
constexpr int kBlockMaxBits = 1664;       // >= 20 (DC) + 63 * 26 (AC): 52 words per block
constexpr int kBlockWords = kBlockMaxBits / 32;
constexpr int kBlocksThreads = 128;
constexpr int kWarpThreads = 256;         // k_jpeg_bits / k_jpeg_emit: 8 blocks per CTA
constexpr int kScanThreads = 512;
constexpr int kStuffThreads = 512;
constexpr int kStuffWords = 4;            // bitstream words per thread per iteration

struct JpegImage {
  int64_t img_off;     // byte offset of the image in src
  int64_t out_off;     // byte offset of the file in out
  int64_t blk0;        // first block in the coefficient array
  int64_t word0;       // first word of the image's bitstream
  int64_t mcu0;        // first MCU of the image over the batch
  int32_t h, w, mx, my, bx, by;
};
static_assert(sizeof(JpegImage) % sizeof(int64_t) == 0, "find_image strides over JpegImage in int64 steps");

// Tables every image shares.  Quantization per jcdctmgr.c compute_reciprocal (16-bit DCTELEM) in natural order, the Huffman codes
// per jchuff.c jpeg_make_c_derived_tbl: tables 0 DC luma, 1 AC luma, 2 DC chroma, 3 AC chroma.
struct JpegTables {
  uint16_t recip[2][64];
  uint16_t corr[2][64];
  uint8_t shift[2][64];
  uint16_t code[4][256];
  uint8_t size[4][256];
  uint8_t header[kJpegHeaderBytes + 1];
};

__constant__ uint8_t c_zigzag[64] = {0,  1,  8,  16, 9,  2,  3,  10, 17, 24, 32, 25, 18, 11, 4,  5,  12, 19, 26, 33, 40, 48,
                                     41, 34, 27, 20, 13, 6,  7,  14, 21, 28, 35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23,
                                     30, 37, 44, 51, 58, 59, 52, 45, 38, 31, 39, 46, 53, 60, 61, 54, 47, 55, 62, 63};

__device__ __forceinline__ int find_image(const int64_t* starts, int n, int64_t x, int stride) {
  // last image i with starts[i * stride] <= x (starts ascending)
  int lo = 0, hi = n - 1;
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (starts[(int64_t)mid * stride] <= x) lo = mid; else hi = mid - 1;
  }
  return lo;
}

// ---- blocks: colour, downsampling, FDCT, quantization -------------------------------------------------------------------------
constexpr int kFix0299 = 19595, kFix0587 = 38470, kFix0114 = 7471, kFix0168 = 11059, kFix0331 = 21709, kFix05 = 32768,
              kFix0418 = 27439, kFix0081 = 5329;
constexpr int kOneHalf = 1 << 15, kCbCrOffset = 128 << 16;

// One 1-D pass of jpeg_fdct_islow over d[0], d[s], ..., d[7 s]
template <bool kFirst>
__device__ __forceinline__ void fdct_pass(int* d, int s) {
  constexpr int n = kFirst ? 11 : 15;         // CONST_BITS -/+ PASS1_BITS
  const int t0 = d[0] + d[7 * s], t7 = d[0] - d[7 * s];
  const int t1 = d[s] + d[6 * s], t6 = d[s] - d[6 * s];
  const int t2 = d[2 * s] + d[5 * s], t5 = d[2 * s] - d[5 * s];
  const int t3 = d[3 * s] + d[4 * s], t4 = d[3 * s] - d[4 * s];
  const int t10 = t0 + t3, t13 = t0 - t3, t11 = t1 + t2, t12 = t1 - t2;
  if (kFirst) {
    d[0] = (t10 + t11) * 4;
    d[4 * s] = (t10 - t11) * 4;
  } else {
    d[0] = (t10 + t11 + 2) >> 2;
    d[4 * s] = (t10 - t11 + 2) >> 2;
  }
  constexpr int r = 1 << (n - 1);
  int z1 = (t12 + t13) * 4433;
  d[2 * s] = (z1 + t13 * 6270 + r) >> n;
  d[6 * s] = (z1 - t12 * 15137 + r) >> n;
  z1 = t4 + t7;
  int z2 = t5 + t6, z3 = t4 + t6, z4 = t5 + t7;
  const int z5 = (z3 + z4) * 9633;
  z1 *= -7373;
  z2 *= -20995;
  z3 = z3 * -16069 + z5;
  z4 = z4 * -3196 + z5;
  d[7 * s] = (t4 * 2446 + z1 + z3 + r) >> n;
  d[5 * s] = (t5 * 16819 + z2 + z4 + r) >> n;
  d[3 * s] = (t6 * 25172 + z2 + z3 + r) >> n;
  d[s] = (t7 * 12299 + z1 + z4 + r) >> n;
}

__global__ void __launch_bounds__(kBlocksThreads) k_jpeg_blocks(const uint8_t* __restrict__ src, const JpegImage* __restrict__ imgs,
                                                                const JpegTables* __restrict__ tab, int n, int16_t* __restrict__ coef) {
  __shared__ int s_cb[16][17], s_cr[16][17];
  __shared__ int s_blk[6][64];                 // level-shifted samples, then DCT output (natural order)
  __shared__ int16_t s_q[6][64];               // quantized, natural order
  const int t = threadIdx.x;
  const int i = find_image(&imgs[0].mcu0, n, blockIdx.x, sizeof(JpegImage) / sizeof(int64_t));
  const JpegImage im = imgs[i];
  const int64_t m = blockIdx.x - im.mcu0;
  const int mcu_x = (int)(m % im.mx), mcu_y = (int)(m / im.mx);
  const uint8_t* img = src + im.img_off;
  for (int p = t; p < 256; p += kBlocksThreads) {
    const int r = p >> 4, c = p & 15;
    const int y = min(mcu_y * 16 + r, im.h - 1), x = min(mcu_x * 16 + c, im.w - 1);
    const uint8_t* px = img + ((int64_t)y * im.w + x) * 3;
    const int B = px[0], G = px[1], R = px[2];
    const int Y = (kFix0299 * R + kFix0587 * G + kFix0114 * B + kOneHalf) >> 16;
    s_blk[(r >> 3) * 2 + (c >> 3)][(r & 7) * 8 + (c & 7)] = Y - 128;
    s_cb[r][c] = (-kFix0168 * R - kFix0331 * G + kFix05 * B + kCbCrOffset + kOneHalf - 1) >> 16;
    s_cr[r][c] = (kFix05 * R - kFix0418 * G - kFix0081 * B + kCbCrOffset + kOneHalf - 1) >> 16;
  }
  __syncthreads();
  {
    // h2v2: rows beyond the last chroma row repeat it (the colour buffer's bottom row was replicated to an even count first)
    const int last = (im.h + 1) / 2 - 1 - mcu_y * 8;
    const int r2 = (t >> 3) & 7, c2 = t & 7, comp = t >> 6;    // threads 0..63 Cb, 64..127 Cr
    const int rr = 2 * min(r2, last);
    int(*s)[17] = comp ? s_cr : s_cb;
    const int v = (s[rr][2 * c2] + s[rr][2 * c2 + 1] + s[rr + 1][2 * c2] + s[rr + 1][2 * c2 + 1] + 1 + (c2 & 1)) >> 2;
    s_blk[4 + comp][r2 * 8 + c2] = v - 128;
  }
  __syncthreads();
  if (t < 48) fdct_pass<true>(&s_blk[t >> 3][(t & 7) * 8], 1);
  __syncthreads();
  if (t < 48) fdct_pass<false>(&s_blk[t >> 3][t & 7], 8);
  __syncthreads();
  for (int e = t; e < 384; e += kBlocksThreads) {
    const int b = e >> 6, k = e & 63, q = b >= 4;
    const int v = s_blk[b][k];
    const uint32_t mag = ((uint32_t)(v < 0 ? -v : v) + tab->corr[q][k]) * tab->recip[q][k] >> tab->shift[q][k];
    s_q[b][k] = (int16_t)(v < 0 ? -(int)mag : (int)mag);
  }
  __syncthreads();
  // dummy blocks (jccoefct.c): zero AC; DC of the block to the left (right edge) or of the MCU's block 1 (bottom edge)
  const bool right = 2 * mcu_x + 1 >= im.bx, bottom = 2 * mcu_y + 1 >= im.by;
  const int dc1 = right ? s_q[0][0] : s_q[1][0];
  int16_t* out = coef + (im.blk0 + m * 6) * 64;
  for (int e = t; e < 384; e += kBlocksThreads) {
    const int b = e >> 6, k = e & 63;
    int v = s_q[b][c_zigzag[k]];
    if (b >= 2 && b < 4 && bottom) v = k ? 0 : dc1;
    else if ((b == 1 || b == 3) && right) v = k ? 0 : s_q[b - 1][0];
    out[e] = (int16_t)v;
  }
}

// ---- entropy coding ------------------------------------------------------------------------------------------------------------
__device__ __forceinline__ int magnitude_bits(int v) { return v ? 32 - __clz(v < 0 ? -v : v) : 0; }

struct BlockRef {
  const int16_t* blk;
  int image;
  int prev;            // previous block of the same component relative to this one (0: none)
  int chroma;
};

__device__ __forceinline__ BlockRef block_ref(const JpegImage* imgs, int n, const int16_t* coef, int64_t g) {
  const int i = find_image(&imgs[0].blk0, n, g, sizeof(JpegImage) / sizeof(int64_t));
  const int64_t l = g - imgs[i].blk0;
  const int b = (int)(l % 6);
  int prev = 0;
  if (b >= 1 && b <= 3) prev = 1;
  else if (l >= 6) prev = b == 0 ? 3 : 6;
  return BlockRef{coef + g * 64, i, prev, b >= 4};
}

// The codes of coefficient k (zigzag) of a block whose nonzero mask is `nz`, as one MSB-first value of `len` bits: the DC
// difference (k = 0), or the ZRLs before an AC coefficient and its code.  len = 0 for a zero AC coefficient.
__device__ __forceinline__ uint64_t coef_codes(const JpegTables* tab, int chroma, int k, int v, int dc_pred, uint64_t nz, int* len) {
  const int t = chroma * 2;
  if (k == 0) {
    const int diff = v - dc_pred, s = magnitude_bits(diff);
    *len = tab->size[t][s] + s;
    return ((uint64_t)tab->code[t][s] << s) | ((uint32_t)(diff < 0 ? diff - 1 : diff) & ((1u << s) - 1));
  }
  if (!v) {
    *len = 0;
    return 0;
  }
  const uint64_t below = nz & ((1ull << k) - 1) & ~1ull;
  const int prev = below ? 63 - __clzll(below) : 0;
  int run = k - prev - 1;
  const int s = magnitude_bits(v);
  uint64_t bits = 0;
  int n = 0;
  const int zsize = tab->size[t + 1][0xF0], zcode = tab->code[t + 1][0xF0];
  for (; run >= 16; run -= 16) {
    bits = (bits << zsize) | zcode;
    n += zsize;
  }
  const int sym = (run << 4) | s, csize = tab->size[t + 1][sym];
  bits = (bits << csize) | tab->code[t + 1][sym];
  bits = (bits << s) | ((uint32_t)(v < 0 ? v - 1 : v) & ((1u << s) - 1));
  *len = n + csize + s;
  return bits;
}

// Loads coefficients `lane` and `lane + 32` of a block and its nonzero mask; DC prediction from the previous block of the component.
__device__ __forceinline__ void load_block(const BlockRef& r, int lane, int* v0, int* v1, int* pred, uint64_t* nz) {
  *v0 = r.blk[lane];
  *v1 = r.blk[lane + 32];
  *pred = r.prev ? r.blk[-64 * r.prev] : 0;
  *nz = (uint64_t)__ballot_sync(~0u, *v0 != 0) | ((uint64_t)__ballot_sync(~0u, *v1 != 0) << 32);
}

__device__ __forceinline__ int eob_bits(const JpegTables* tab, int chroma, uint64_t nz) {
  return (nz >> 63) ? 0 : tab->size[chroma * 2 + 1][0];
}

__global__ void __launch_bounds__(kWarpThreads) k_jpeg_bits(const JpegImage* __restrict__ imgs, const JpegTables* __restrict__ tab, int n,
                                                            const int16_t* __restrict__ coef, int64_t total_blocks,
                                                            uint32_t* __restrict__ blen) {
  const int64_t g = (int64_t)blockIdx.x * (kWarpThreads / 32) + warp_id();
  if (g >= total_blocks) return;
  const int lane = lane_id();
  const BlockRef r = block_ref(imgs, n, coef, g);
  int v0, v1, pred, l0, l1;
  uint64_t nz;
  load_block(r, lane, &v0, &v1, &pred, &nz);
  coef_codes(tab, r.chroma, lane, v0, pred, nz, &l0);
  coef_codes(tab, r.chroma, lane + 32, v1, pred, nz, &l1);
  int len = l0 + l1;
#pragma unroll
  for (int o = 16; o; o >>= 1) len += __shfl_xor_sync(~0u, len, o);
  if (lane == 0) blen[g] = len + eob_bits(tab, r.chroma, nz);
}

__global__ void __launch_bounds__(kScanThreads) k_jpeg_scan(const JpegImage* __restrict__ imgs, const uint32_t* __restrict__ blen,
                                                            uint64_t* __restrict__ boff, uint64_t* __restrict__ img_bits,
                                                            uint32_t* __restrict__ bits) {
  using Scan = cub::BlockScan<uint64_t, kScanThreads>;
  __shared__ typename Scan::TempStorage tmp;
  const JpegImage im = imgs[blockIdx.x];
  const int64_t nb = (int64_t)im.mx * im.my * 6;
  uint64_t carry = 0;
  for (int64_t a = 0; a < nb; a += kScanThreads) {
    const int64_t j = a + threadIdx.x;
    const uint64_t len = j < nb ? blen[im.blk0 + j] : 0;
    uint64_t off, total;
    Scan(tmp).ExclusiveSum(len, off, total);
    __syncthreads();
    if (j < nb) {
      off += carry;
      boff[im.blk0 + j] = off;
      // the words k_jpeg_emit ORs into: the first and the last of the block
      bits[im.word0 + (int64_t)(off >> 5)] = 0;
      bits[im.word0 + (int64_t)((off + len - 1) >> 5)] = 0;
    }
    carry += total;
  }
  if (threadIdx.x == 0) img_bits[blockIdx.x] = carry;
}

__global__ void __launch_bounds__(kWarpThreads) k_jpeg_emit(const JpegImage* __restrict__ imgs, const JpegTables* __restrict__ tab, int n,
                                                            const int16_t* __restrict__ coef, int64_t total_blocks,
                                                            const uint32_t* __restrict__ blen, const uint64_t* __restrict__ boff,
                                                            uint32_t* __restrict__ bits) {
  __shared__ uint32_t s_words[kWarpThreads / 32][kBlockWords + 2];
  const int64_t g = (int64_t)blockIdx.x * (kWarpThreads / 32) + warp_id();
  if (g >= total_blocks) return;
  const int lane = lane_id();
  uint32_t* sw = s_words[warp_id()];
  for (int w = lane; w < kBlockWords + 2; w += 32) sw[w] = 0;
  const BlockRef r = block_ref(imgs, n, coef, g);
  int v0, v1, pred, l0, l1;
  uint64_t nz;
  load_block(r, lane, &v0, &v1, &pred, &nz);
  const uint64_t c0 = coef_codes(tab, r.chroma, lane, v0, pred, nz, &l0);
  const uint64_t c1 = coef_codes(tab, r.chroma, lane + 32, v1, pred, nz, &l1);
  const uint64_t off = boff[g];
  const int phase = (int)(off & 31);
  // bit positions within the staged words: coefficients 0..31, then 32..63, then EOB
  int p0 = l0, p1 = l1;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const int a = __shfl_up_sync(~0u, p0, o), b = __shfl_up_sync(~0u, p1, o);
    if (lane >= o) p0 += a, p1 += b;
  }
  const int tot0 = __shfl_sync(~0u, p0, 31), tot1 = __shfl_sync(~0u, p1, 31);
  __syncwarp();
  auto put = [&](uint64_t v, int len, int pos) {     // OR `len` bits of v at bit pos (MSB-first) of the staged words
    while (len > 0) {
      const int w = pos >> 5, room = 32 - (pos & 31), take = min(room, len);
      const uint32_t chunk = (uint32_t)(v >> (len - take)) & (take == 32 ? ~0u : ((1u << take) - 1));
      atomicOr(&sw[w], chunk << (room - take));
      pos += take;
      len -= take;
    }
  };
  if (l0) put(c0, l0, phase + p0 - l0);
  if (l1) put(c1, l1, phase + tot0 + p1 - l1);
  const int eob = eob_bits(tab, r.chroma, nz);
  if (lane == 0 && eob) put(tab->code[r.chroma * 2 + 1][0], eob, phase + tot0 + tot1);
  __syncwarp();
  const int len = (int)blen[g];
  const int nw = (phase + len + 31) >> 5;
  uint32_t* dst = bits + imgs[r.image].word0 + (int64_t)(off >> 5);
  for (int w = lane; w < nw; w += 32) {
    if (w == 0 || w == nw - 1) atomicOr(&dst[w], sw[w]);     // may be shared with the neighbouring block
    else dst[w] = sw[w];
  }
}

__global__ void __launch_bounds__(kStuffThreads) k_jpeg_stuff(const JpegImage* __restrict__ imgs, const JpegTables* __restrict__ tab,
                                                              const uint64_t* __restrict__ img_bits, const uint32_t* __restrict__ bits,
                                                              uint8_t* __restrict__ out, int64_t* __restrict__ out_len) {
  using Scan = cub::BlockScan<int, kStuffThreads>;
  __shared__ typename Scan::TempStorage tmp;
  const JpegImage im = imgs[blockIdx.x];
  uint8_t* dst = out + im.out_off;
  for (int j = threadIdx.x; j < kJpegHeaderBytes; j += kStuffThreads) {
    uint8_t v = tab->header[j];
    const int f = j - kJpegSofOffset;
    if (f == 5) v = (uint8_t)(im.h >> 8);
    else if (f == 6) v = (uint8_t)im.h;
    else if (f == 7) v = (uint8_t)(im.w >> 8);
    else if (f == 8) v = (uint8_t)im.w;
    dst[j] = v;
  }
  const uint64_t nbits = img_bits[blockIdx.x];
  const int64_t nbytes = (int64_t)((nbits + 7) >> 3);
  const uint32_t* srcw = bits + im.word0;
  int64_t o = kJpegHeaderBytes;
  for (int64_t a = 0; a < nbytes; a += kStuffThreads * kStuffWords * 4) {
    const int64_t b0 = a + (int64_t)threadIdx.x * kStuffWords * 4;
    uint8_t by[kStuffWords * 4];
    int nff = 0, nown = 0;
#pragma unroll
    for (int q = 0; q < kStuffWords; ++q) {
      const int64_t bq = b0 + q * 4;
      const uint32_t w = bq < nbytes ? srcw[bq >> 2] : 0;
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        const int64_t j = bq + k;
        uint32_t v = (w >> (24 - 8 * k)) & 0xFF;
        if (j == nbytes - 1 && (nbits & 7)) v |= 0xFFu >> (nbits & 7);     // pad the last byte with 1-bits
        by[q * 4 + k] = (uint8_t)v;
        if (j < nbytes) {
          ++nown;
          nff += v == 0xFF;
        }
      }
    }
    int pos, total;
    Scan(tmp).ExclusiveSum(nown + nff, pos, total);
    __syncthreads();
    uint8_t* d = dst + o + pos;
#pragma unroll
    for (int k = 0; k < kStuffWords * 4; ++k) {
      if (k < nown) {
        *d++ = by[k];
        if (by[k] == 0xFF) *d++ = 0;
      }
    }
    o += total;
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    dst[o] = 0xFF;
    dst[o + 1] = 0xD9;
    out_len[blockIdx.x] = o + 2;
  }
}

// ---- host --------------------------------------------------------------------------------------------------------------------
const uint8_t kBaseLuma[64] = {16, 11, 10, 16, 24,  40,  51,  61,  12, 12, 14, 19, 26,  58,  60,  55,  14, 13, 16, 24,  40, 57,
                               69, 56, 14, 17, 22,  29,  51,  87,  80, 62, 18, 22, 37,  56,  68,  109, 103, 77, 24, 35, 55, 64,
                               81, 104, 113, 92, 49, 64, 78, 87, 103, 121, 120, 101, 72, 92, 95, 98, 112, 100, 103, 99};
const uint8_t kBaseChroma[64] = {17, 18, 24, 47, 99, 99, 99, 99, 18, 21, 26, 66, 99, 99, 99, 99, 24, 26, 56, 99, 99, 99,
                                 99, 99, 47, 66, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99,
                                 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99};
const uint8_t kZigzag[64] = {0,  1,  8,  16, 9,  2,  3,  10, 17, 24, 32, 25, 18, 11, 4,  5,  12, 19, 26, 33, 40, 48,
                             41, 34, 27, 20, 13, 6,  7,  14, 21, 28, 35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23,
                             30, 37, 44, 51, 58, 59, 52, 45, 38, 31, 39, 46, 53, 60, 61, 54, 47, 55, 62, 63};
// Annex K.3 - K.6: code-length counts and symbols of DC luma, AC luma, DC chroma, AC chroma
const uint8_t kHuffBits[4][16] = {{0, 1, 5, 1, 1, 1, 1, 1, 1, 0, 0, 0, 0, 0, 0, 0},
                                  {0, 2, 1, 3, 3, 2, 4, 3, 5, 5, 4, 4, 0, 0, 1, 0x7d},
                                  {0, 3, 1, 1, 1, 1, 1, 1, 1, 1, 1, 0, 0, 0, 0, 0},
                                  {0, 2, 1, 2, 4, 4, 3, 4, 7, 5, 4, 4, 0, 1, 2, 0x77}};
const uint8_t kDcVals[12] = {0, 1, 2, 3, 4, 5, 6, 7, 8, 9, 10, 11};
const uint8_t kAcLumaVals[162] = {
    0x01, 0x02, 0x03, 0x00, 0x04, 0x11, 0x05, 0x12, 0x21, 0x31, 0x41, 0x06, 0x13, 0x51, 0x61, 0x07, 0x22, 0x71, 0x14, 0x32, 0x81,
    0x91, 0xa1, 0x08, 0x23, 0x42, 0xb1, 0xc1, 0x15, 0x52, 0xd1, 0xf0, 0x24, 0x33, 0x62, 0x72, 0x82, 0x09, 0x0a, 0x16, 0x17, 0x18,
    0x19, 0x1a, 0x25, 0x26, 0x27, 0x28, 0x29, 0x2a, 0x34, 0x35, 0x36, 0x37, 0x38, 0x39, 0x3a, 0x43, 0x44, 0x45, 0x46, 0x47, 0x48,
    0x49, 0x4a, 0x53, 0x54, 0x55, 0x56, 0x57, 0x58, 0x59, 0x5a, 0x63, 0x64, 0x65, 0x66, 0x67, 0x68, 0x69, 0x6a, 0x73, 0x74, 0x75,
    0x76, 0x77, 0x78, 0x79, 0x7a, 0x83, 0x84, 0x85, 0x86, 0x87, 0x88, 0x89, 0x8a, 0x92, 0x93, 0x94, 0x95, 0x96, 0x97, 0x98, 0x99,
    0x9a, 0xa2, 0xa3, 0xa4, 0xa5, 0xa6, 0xa7, 0xa8, 0xa9, 0xaa, 0xb2, 0xb3, 0xb4, 0xb5, 0xb6, 0xb7, 0xb8, 0xb9, 0xba, 0xc2, 0xc3,
    0xc4, 0xc5, 0xc6, 0xc7, 0xc8, 0xc9, 0xca, 0xd2, 0xd3, 0xd4, 0xd5, 0xd6, 0xd7, 0xd8, 0xd9, 0xda, 0xe1, 0xe2, 0xe3, 0xe4, 0xe5,
    0xe6, 0xe7, 0xe8, 0xe9, 0xea, 0xf1, 0xf2, 0xf3, 0xf4, 0xf5, 0xf6, 0xf7, 0xf8, 0xf9, 0xfa};
const uint8_t kAcChromaVals[162] = {
    0x00, 0x01, 0x02, 0x03, 0x11, 0x04, 0x05, 0x21, 0x31, 0x06, 0x12, 0x41, 0x51, 0x07, 0x61, 0x71, 0x13, 0x22, 0x32, 0x81, 0x08,
    0x14, 0x42, 0x91, 0xa1, 0xb1, 0xc1, 0x09, 0x23, 0x33, 0x52, 0xf0, 0x15, 0x62, 0x72, 0xd1, 0x0a, 0x16, 0x24, 0x34, 0xe1, 0x25,
    0xf1, 0x17, 0x18, 0x19, 0x1a, 0x26, 0x27, 0x28, 0x29, 0x2a, 0x35, 0x36, 0x37, 0x38, 0x39, 0x3a, 0x43, 0x44, 0x45, 0x46, 0x47,
    0x48, 0x49, 0x4a, 0x53, 0x54, 0x55, 0x56, 0x57, 0x58, 0x59, 0x5a, 0x63, 0x64, 0x65, 0x66, 0x67, 0x68, 0x69, 0x6a, 0x73, 0x74,
    0x75, 0x76, 0x77, 0x78, 0x79, 0x7a, 0x82, 0x83, 0x84, 0x85, 0x86, 0x87, 0x88, 0x89, 0x8a, 0x92, 0x93, 0x94, 0x95, 0x96, 0x97,
    0x98, 0x99, 0x9a, 0xa2, 0xa3, 0xa4, 0xa5, 0xa6, 0xa7, 0xa8, 0xa9, 0xaa, 0xb2, 0xb3, 0xb4, 0xb5, 0xb6, 0xb7, 0xb8, 0xb9, 0xba,
    0xc2, 0xc3, 0xc4, 0xc5, 0xc6, 0xc7, 0xc8, 0xc9, 0xca, 0xd2, 0xd3, 0xd4, 0xd5, 0xd6, 0xd7, 0xd8, 0xd9, 0xda, 0xe2, 0xe3, 0xe4,
    0xe5, 0xe6, 0xe7, 0xe8, 0xe9, 0xea, 0xf2, 0xf3, 0xf4, 0xf5, 0xf6, 0xf7, 0xf8, 0xf9, 0xfa};

void make_tables(int quality, JpegTables* t) {
  memset(t, 0, sizeof(*t));
  const int scale = quality < 50 ? 5000 / quality : 200 - 2 * quality;        // jpeg_quality_scaling
  uint8_t qt[2][64];
  for (int c = 0; c < 2; ++c)
    for (int k = 0; k < 64; ++k) {
      const long v = ((long)(c ? kBaseChroma : kBaseLuma)[k] * scale + 50) / 100;
      qt[c][k] = (uint8_t)(v < 1 ? 1 : v > 255 ? 255 : v);                   // force_baseline
      // compute_reciprocal, 16-bit DCTELEM
      const uint32_t d = (uint32_t)qt[c][k] << 3;
      int b = 31 - __builtin_clz(d), r = 16 + b;
      uint64_t fq = (1ull << r) / d;
      const uint64_t fr = (1ull << r) % d;
      uint32_t corr = d / 2;
      if (fr == 0) {
        fq >>= 1;
        --r;
      } else if (fr <= d / 2) {
        ++corr;
      } else {
        ++fq;
      }
      t->recip[c][k] = (uint16_t)fq;
      t->corr[c][k] = (uint16_t)corr;
      t->shift[c][k] = (uint8_t)r;
    }
  const uint8_t* vals[4] = {kDcVals, kAcLumaVals, kDcVals, kAcChromaVals};
  const int nvals[4] = {12, 162, 12, 162};
  for (int h = 0; h < 4; ++h) {       // jpeg_make_c_derived_tbl: canonical codes
    int code = 0, k = 0;
    for (int len = 1; len <= 16; ++len) {
      for (int j = 0; j < kHuffBits[h][len - 1]; ++j, ++k, ++code) {
        t->code[h][vals[h][k]] = (uint16_t)code;
        t->size[h][vals[h][k]] = (uint8_t)len;
      }
      code <<= 1;
    }
  }
  uint8_t* p = t->header;
  const uint8_t app0[20] = {0xFF, 0xD8, 0xFF, 0xE0, 0x00, 0x10, 'J', 'F', 'I', 'F', 0, 1, 1, 0, 0, 1, 0, 1, 0, 0};
  memcpy(p, app0, 20);
  p += 20;
  for (int c = 0; c < 2; ++c) {
    const uint8_t dqt[5] = {0xFF, 0xDB, 0x00, 0x43, (uint8_t)c};
    memcpy(p, dqt, 5);
    p += 5;
    for (int k = 0; k < 64; ++k) *p++ = qt[c][kZigzag[k]];
  }
  const uint8_t sof[19] = {0xFF, 0xC0, 0x00, 0x11, 8, 0, 0, 0, 0, 3, 1, 0x22, 0, 2, 0x11, 1, 3, 0x11, 1};
  memcpy(p, sof, 19);
  p += 19;
  const uint8_t cls_id[4] = {0x00, 0x10, 0x01, 0x11};
  for (int h = 0; h < 4; ++h) {
    const int len = 2 + 1 + 16 + nvals[h];
    const uint8_t dht[5] = {0xFF, 0xC4, (uint8_t)(len >> 8), (uint8_t)len, cls_id[h]};
    memcpy(p, dht, 5);
    p += 5;
    memcpy(p, kHuffBits[h], 16);
    p += 16;
    memcpy(p, vals[h], nvals[h]);
    p += nvals[h];
  }
  const uint8_t sos[14] = {0xFF, 0xDA, 0x00, 0x0C, 3, 1, 0x00, 2, 0x11, 3, 0x11, 0, 63, 0};
  memcpy(p, sos, 14);
}

int64_t image_blocks(int h, int w) { return (int64_t)((w + 15) / 16) * ((h + 15) / 16) * 6; }

struct JpegLayout {
  size_t tables, coef, blen, boff, img_bits, bits, total;
};

JpegLayout jpeg_layout(int n, int64_t blocks, int64_t words) {
  JpegLayout l;
  size_t o = 0;
  l.tables = o;
  o = align_up(o + (size_t)n * sizeof(JpegImage) + sizeof(JpegTables), 256);
  l.coef = o;
  o = align_up(o + (size_t)blocks * 64 * sizeof(int16_t), 256);
  l.blen = o;
  o = align_up(o + (size_t)blocks * sizeof(uint32_t), 256);
  l.boff = o;
  o = align_up(o + (size_t)blocks * sizeof(uint64_t), 256);
  l.img_bits = o;
  o = align_up(o + (size_t)n * sizeof(uint64_t), 256);
  l.bits = o;
  o = align_up(o + (size_t)words * sizeof(uint32_t), 256);
  l.total = o;
  return l;
}

bool valid_size(int h, int w) { return h >= 1 && w >= 1 && h <= 65535 && w <= 65535; }

}  // namespace
}  // namespace yb

using namespace yb;

extern "C" int64_t yb_jpeg_encode_bound(int h, int w) {
  if (!valid_size(h, w)) return -1;
  return kJpegHeaderBytes + 2 * image_blocks(h, w) * (kBlockMaxBits / 8) + 2;
}

extern "C" size_t yb_jpeg_encode_workspace_bytes(const yb_val_aug_item* items, int n) {
  if (!items || n <= 0) return 0;
  int64_t blocks = 0;
  for (int i = 0; i < n; ++i) {
    if (!valid_size(items[i].h, items[i].w)) return 0;
    blocks += image_blocks(items[i].h, items[i].w);
  }
  return jpeg_layout(n, blocks, blocks * kBlockWords + n).total;
}

extern "C" int yb_jpeg_encode_batch(const uint8_t* src, int64_t src_bytes, const yb_val_aug_item* items, int n, int quality,
                                    void* workspace, size_t workspace_bytes, uint8_t* out, const int64_t* out_off, int64_t* out_len,
                                    void* stream) {
  YB_REQUIRE(src && items && workspace && out && out_off && out_len, YB_ERR_INVALID, "yb_jpeg_encode_batch: NULL pointer argument");
  YB_REQUIRE(n >= 1 && n <= 65535 && src_bytes > 0, YB_ERR_INVALID, "yb_jpeg_encode_batch: n=%d src_bytes=%lld", n, (long long)src_bytes);
  YB_REQUIRE(quality >= 1 && quality <= 100, YB_ERR_INVALID, "yb_jpeg_encode_batch: quality=%d (1 .. 100)", quality);
  YB_REQUIRE(out_off[0] >= 0, YB_ERR_INVALID, "yb_jpeg_encode_batch: out_off[0]=%lld", (long long)out_off[0]);
  std::vector<JpegImage> imgs(n);
  int64_t blocks = 0, words = 0, mcus = 0;
  for (int i = 0; i < n; ++i) {
    const yb_val_aug_item& t = items[i];
    YB_REQUIRE(valid_size(t.h, t.w), YB_ERR_INVALID, "yb_jpeg_encode_batch: item %d: h=%d w=%d (1 .. 65535)", i, t.h, t.w);
    const int64_t bytes = (int64_t)t.h * t.w * 3;
    YB_REQUIRE(t.img_off >= 0 && t.img_off <= src_bytes - bytes, YB_ERR_INVALID,
               "yb_jpeg_encode_batch: item %d: image [%lld, +%lld) outside src (%lld bytes)", i, (long long)t.img_off, (long long)bytes,
               (long long)src_bytes);
    const int64_t bound = yb_jpeg_encode_bound(t.h, t.w);
    YB_REQUIRE(out_off[i + 1] >= 0 && out_off[i] <= out_off[i + 1] - bound, YB_ERR_INVALID,
               "yb_jpeg_encode_batch: image %d (%dx%d) needs %lld bytes from out_off %lld, the next image starts at %lld", i, t.h, t.w,
               (long long)bound, (long long)out_off[i], (long long)out_off[i + 1]);
    const int mx = (t.w + 15) / 16, my = (t.h + 15) / 16;
    imgs[i] = JpegImage{t.img_off, out_off[i], blocks, words, mcus, t.h, t.w, mx, my, (t.w + 7) / 8, (t.h + 7) / 8};
    blocks += image_blocks(t.h, t.w);
    words += image_blocks(t.h, t.w) * kBlockWords + 1;
    mcus += (int64_t)mx * my;
  }
  YB_REQUIRE(out + out_off[n] <= src || src + src_bytes <= out + out_off[0], YB_ERR_INVALID, "yb_jpeg_encode_batch: out overlaps src");
  YB_REQUIRE(mcus < INT32_MAX && (blocks + 7) / 8 < INT32_MAX, YB_ERR_UNSUPPORTED, "yb_jpeg_encode_batch: %lld MCUs in one batch",
             (long long)mcus);
  const JpegLayout l = jpeg_layout(n, blocks, words);
  YB_REQUIRE(workspace_bytes >= l.total, YB_ERR_INVALID, "yb_jpeg_encode_batch: workspace %zu bytes < %zu", workspace_bytes, l.total);
  JpegTables tables;
  make_tables(quality, &tables);
  cudaStream_t st = (cudaStream_t)stream;
  char* ws = (char*)workspace;
  const size_t img_bytes = (size_t)n * sizeof(JpegImage);
  const StagePart parts[2] = {{imgs.data(), img_bytes, 0}, {&tables, sizeof(JpegTables), img_bytes}};
  YB_PROPAGATE(stage_tables(ws + l.tables, img_bytes + sizeof(JpegTables), parts, 2, st));
  const JpegImage* d_imgs = (const JpegImage*)(ws + l.tables);
  const JpegTables* d_tab = (const JpegTables*)(ws + l.tables + img_bytes);
  int16_t* coef = (int16_t*)(ws + l.coef);
  uint32_t* blen = (uint32_t*)(ws + l.blen);
  uint64_t* boff = (uint64_t*)(ws + l.boff);
  uint64_t* img_bits = (uint64_t*)(ws + l.img_bits);
  uint32_t* bits = (uint32_t*)(ws + l.bits);
  const int warp_grid = (int)((blocks + kWarpThreads / 32 - 1) / (kWarpThreads / 32));
  k_jpeg_blocks<<<(unsigned)mcus, kBlocksThreads, 0, st>>>(src, d_imgs, d_tab, n, coef);
  YB_CHECK_LAUNCH();
  k_jpeg_bits<<<warp_grid, kWarpThreads, 0, st>>>(d_imgs, d_tab, n, coef, blocks, blen);
  YB_CHECK_LAUNCH();
  k_jpeg_scan<<<n, kScanThreads, 0, st>>>(d_imgs, blen, boff, img_bits, bits);
  YB_CHECK_LAUNCH();
  k_jpeg_emit<<<warp_grid, kWarpThreads, 0, st>>>(d_imgs, d_tab, n, coef, blocks, blen, boff, bits);
  YB_CHECK_LAUNCH();
  k_jpeg_stuff<<<n, kStuffThreads, 0, st>>>(d_imgs, d_tab, img_bits, bits, out, out_len);
  YB_CHECK_LAUNCH();
  return YB_OK;
}
