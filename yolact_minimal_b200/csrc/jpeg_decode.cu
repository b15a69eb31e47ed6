// Baseline JPEG decoding of a batch of files, pixel for pixel what cv2.imread returns (libjpeg-turbo: ISLOW IDCT, fancy
// upsampling, BGR output, the EXIF orientation applied as OpenCV applies it).  oracle/jpeg_decode_np.py states every rule in
// numpy; the kernels follow it in the same integer arithmetic.
//
// The host parses every header (yb_jpeg_header is the only parser of the format) and stages the per-file tables; then five
// launches, no host synchronisation:
//   k_jpeg_destuff   one CTA per file: scan-and-compact of the entropy-coded bytes -- a 0x00 after 0xFF and the restart markers
//                    dropped -- into a word-aligned stream; records where each restart interval starts.
//   k_jpeg_huffman   one CTA per file: the self-synchronising decode of Weissenberger & Schmidt.  Each interval is cut into
//                    1024-bit subsequences; thread j decodes subsequence j from its start state to its first codeword boundary
//                    past its end, and a changed end state becomes subsequence j+1's start state for the next round, until no
//                    start state changes (the first subsequence of an interval starts from the true state, so the fixpoint is the
//                    sequential decode).  The blocks whose DC code starts in each subsequence are counted as it decodes; an
//                    exclusive scan gives every subsequence its first block, and a last pass writes the quantized coefficients
//                    (DC differences) in block order into the zeroed coefficient buffer.
//   k_jpeg_dc        one CTA per (file, component): segmented scan of the DC differences, restarting at every interval.
//   k_jpeg_idct      8 threads per block: dequantization, jidctint.c's ISLOW IDCT, the range limit; component planes at their
//                    own resolution.
//   k_jpeg_color     one thread per output pixel: fancy upsampling from the chroma planes, YCbCr -> BGR, the orientation map.
#include "common.cuh"

#include <cub/block/block_reduce.cuh>
#include <cub/block/block_scan.cuh>
#include <string.h>
#include <vector>

namespace yb {
namespace {

constexpr int kSubBits = 1024;          // bits per subsequence
constexpr int kDestuffThreads = 512;
constexpr int kDestuffBytes = 16;       // bytes per thread per iteration
constexpr int kHuffThreads = 512;
constexpr int kDcThreads = 512;
constexpr int kIdctBlocks = 32;         // blocks per CTA of k_jpeg_idct (8 threads each)
constexpr int kColorThreads = 256;
constexpr int kStreamPad = 16;          // zero bytes after a file's destuffed stream

enum DecodeStatus { kOk = 0, kBadRestarts = 1, kBadCode = 2, kRunPast63 = 3, kTooFewBlocks = 4 };

// One Huffman table: codes of up to 9 bits by lookup ((length << 8) | symbol, 0 if longer), longer ones by jdhuff.c's
// canonical maxcode / valoffset.
struct DecTable {
  uint16_t lut[512];
  int32_t maxcode[18];                  // largest code of each length, -1 if none; maxcode[17] sentinel
  int32_t valoff[18];                   // symbol index of code c of length l: c + valoff[l]
  uint8_t vals[256];
};

struct DecTables {
  DecTable t[6];                        // DC, AC of component 0, 1, 2
  uint16_t q[3][64];                    // quantization, natural order
};

struct DecImage {
  int64_t scan_off;                     // first entropy-coded byte in src
  int64_t scan_end;                     // end of the file in src
  int64_t stream_off;                   // destuffed stream in the workspace (bytes, 4-aligned)
  int64_t out_off;                      // BGR output in out
  int64_t blk0;                         // first block in the coefficient buffer
  int64_t pix0;                         // first output pixel over the batch
  int64_t plane_off[3];
  int64_t int0;                         // first entry of the interval-start table (n_int + 1 entries)
  int64_t sub0;                         // first subsequence slot
  int32_t sub_cap;                      // subsequence slots
  int32_t h, w, orient;                 // frame size, EXIF orientation
  int32_t ncomp, hs, vs;                // luma sampling (1x1 for grayscale)
  int32_t mx, my, bpm;                  // MCU grid, blocks per MCU
  int32_t ri, n_int;                    // restart interval (MCUs), intervals
  int32_t pw[3], ph[3];                 // plane sizes (block grid x 8)
};
static_assert(sizeof(DecImage) % sizeof(int64_t) == 0, "find_image strides over DecImage in int64 steps");

// zigzag position of natural (row-major) coefficient k
__constant__ uint8_t c_unzig[64] = {0,  1,  5,  6,  14, 15, 27, 28, 2,  4,  7,  13, 16, 26, 29, 42, 3,  8,  12, 17, 25, 30,
                                    41, 43, 9,  11, 18, 24, 31, 40, 44, 53, 10, 19, 23, 32, 39, 45, 52, 54, 20, 22, 33, 38,
                                    46, 51, 55, 60, 21, 34, 37, 47, 50, 56, 59, 61, 35, 36, 48, 49, 57, 58, 62, 63};

__device__ __forceinline__ int find_item(const int64_t* starts, int n, int64_t x, int stride) {
  int lo = 0, hi = n - 1;
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (starts[(int64_t)mid * stride] <= x) lo = mid; else hi = mid - 1;
  }
  return lo;
}

constexpr int kImgStride = sizeof(DecImage) / sizeof(int64_t);

// ---- destuff ---------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(kDestuffThreads) k_jpeg_destuff(const uint8_t* __restrict__ src, const DecImage* __restrict__ imgs,
                                                                  uint8_t* __restrict__ stream, int32_t* __restrict__ int_start,
                                                                  int32_t* __restrict__ status) {
  using Scan = cub::BlockScan<uint64_t, kDestuffThreads>;
  using Reduce = cub::BlockReduce<int64_t, kDestuffThreads>;
  __shared__ typename Scan::TempStorage tmp;
  __shared__ typename Reduce::TempStorage rtmp;
  __shared__ int64_t s_term;
  const DecImage im = imgs[blockIdx.x];
  const uint8_t* b = src + im.scan_off;
  const int64_t n = im.scan_end - im.scan_off;
  uint8_t* dst = stream + im.stream_off;
  int32_t* starts = int_start + im.int0;
  int64_t kept = 0, rsts = 0;
  for (int64_t a = 0; a < n; a += (int64_t)kDestuffThreads * kDestuffBytes) {
    const int64_t i0 = a + (int64_t)threadIdx.x * kDestuffBytes;
    // the first marker other than RSTn (or a 0xFF at the last byte) ends the entropy-coded data
    int64_t term = INT64_MAX;
    for (int k = 0; k < kDestuffBytes; ++k) {
      const int64_t i = i0 + k;
      if (i >= n) break;
      if (b[i] == 0xFF) {
        const int nx = i + 1 < n ? b[i + 1] : -1;
        if (!(nx == 0x00 || (nx >= 0xD0 && nx <= 0xD7) || nx == 0xFF)) {
          term = i;
          break;
        }
      }
    }
    term = Reduce(rtmp).Reduce(term, cub::Min());
    if (threadIdx.x == 0) s_term = term;
    __syncthreads();
    term = s_term;
    uint32_t keep_mask = 0, rst_mask = 0;
    int nk = 0, nr = 0;
    for (int k = 0; k < kDestuffBytes; ++k) {
      const int64_t i = i0 + k;
      if (i >= n || i >= term) break;
      const uint8_t v = b[i];
      const int pv = i > 0 ? b[i - 1] : -1;
      bool keep = true;
      if (v == 0xFF) {
        const uint8_t nx = i + 1 < n ? b[i + 1] : 0;
        if (nx != 0x00) keep = false;                             // a fill byte or the 0xFF of RSTn
        if (nx >= 0xD0 && nx <= 0xD7) {
          rst_mask |= 1u << k;
          ++nr;
        }
      } else if (pv == 0xFF && (v == 0x00 || (v >= 0xD0 && v <= 0xD7))) {
        keep = false;                                             // stuffed zero, or the RSTn byte
      }
      if (keep) {
        keep_mask |= 1u << k;
        ++nk;
      }
    }
    uint64_t pos, total;
    Scan(tmp).ExclusiveSum(((uint64_t)nr << 32) | (uint64_t)nk, pos, total);
    int64_t o = kept + (int64_t)(pos & 0xFFFFFFFFu), r = rsts + (int64_t)(pos >> 32);
    for (int k = 0; k < kDestuffBytes; ++k) {
      if (rst_mask >> k & 1) {
        if (r + 1 < im.n_int) starts[r + 1] = (int32_t)o;
        ++r;
      }
      if (keep_mask >> k & 1) dst[o++] = b[i0 + k];
    }
    kept += (int64_t)(total & 0xFFFFFFFFu);
    rsts += (int64_t)(total >> 32);
    __syncthreads();
    if (term != INT64_MAX) break;
  }
  for (int k = threadIdx.x; k < kStreamPad + 4; k += kDestuffThreads) dst[kept + k] = 0;
  if (threadIdx.x == 0) {
    starts[0] = 0;
    starts[im.n_int] = (int32_t)kept;
    status[blockIdx.x] = rsts + 1 == im.n_int ? kOk : kBadRestarts;
  }
}

// ---- Huffman decode --------------------------------------------------------------------------------------------------------
// Decoder state at a codeword boundary: bit offset in the file's stream, block within the MCU, next coefficient (0: DC).
__device__ __forceinline__ uint64_t pack_state(uint32_t p, int c, int z) { return (uint64_t)p << 16 | (uint64_t)c << 8 | (uint64_t)z; }

struct Bits {
  const uint32_t* w;                    // the stream as big-endian words
  __device__ __forceinline__ uint32_t peek32(uint32_t p) const {
    const uint32_t i = p >> 5;
    const uint64_t v = (uint64_t)__byte_perm(w[i], 0, 0x0123) << 32 | __byte_perm(w[i + 1], 0, 0x0123);
    return (uint32_t)((v << (p & 31)) >> 32);
  }
};

// Decodes one symbol from the 32 bits at the read position; *len = 0 for an invalid code.
__device__ __forceinline__ int huff_symbol(const DecTable& t, uint32_t top, int* len) {
  const int e = t.lut[top >> 23];
  if (e) {
    *len = e >> 8;
    return e & 0xFF;
  }
  for (int l = 10; l <= 16; ++l) {
    const int32_t code = (int32_t)(top >> (32 - l));
    if (code <= t.maxcode[l]) {
      *len = l;
      return t.vals[(code + t.valoff[l]) & 0xFF];
    }
  }
  *len = 0;
  return 0;
}

__device__ __forceinline__ int extend(uint32_t v, int s) { return s && v < (1u << (s - 1)) ? (int)v - (1 << s) + 1 : (int)v; }

// Decodes from `state` to the first codeword boundary at or past end_bit.  Counts the blocks whose DC code starts here.
// kWrite: writes the coefficients (DC differences) of block first_blk + k (k-th block started here; first_blk - 1 for a block
// in progress at the start) while its index is below blk_end, and returns the first error met in such a block in *err.
template <bool kWrite>
__device__ uint64_t decode_sub(const Bits& bits, const DecTable* tabs, int bpm, int hv, uint64_t state, uint32_t end_bit, int* count,
                               int16_t* coef, int64_t first_blk, int64_t blk_end, int* err) {
  uint32_t p = (uint32_t)(state >> 16);
  int c = (int)(state >> 8) & 0xFF, z = (int)state & 0xFF;
  int n = 0;
  int64_t cur = first_blk - 1;
  for (int guard = 0; p < end_bit && guard < 4 * kSubBits; ++guard) {
    const int comp = c < hv ? 0 : c - hv + 1;
    const uint32_t top = bits.peek32(p);
    int len;
    if (z == 0) {
      const int s = huff_symbol(tabs[2 * comp], top, &len);
      ++n;
      ++cur;
      if (!len) {                      // invalid code: skip 16 bits (only a corrupt stream meets one on the true chain)
        if (kWrite && cur < blk_end && !*err) *err = kBadCode;
        p += 16;
        z = 64;
      } else {
        const int ss = s & 15;
        if (kWrite && cur < blk_end) coef[cur * 64] = (int16_t)extend(ss ? (top << len) >> (32 - ss) : 0, ss);
        p += len + ss;
        z = 1;
      }
    } else {
      const int rs = huff_symbol(tabs[2 * comp + 1], top, &len);
      if (!len) {
        if (kWrite && cur < blk_end && !*err) *err = kBadCode;
        p += 16;
        z = 64;
      } else {
        const int r = rs >> 4, s = rs & 15;
        p += len;
        if (s == 0) {
          z = r == 15 ? z + 16 : 64;
        } else {
          z += r;
          if (z > 63) {
            if (kWrite && cur < blk_end && !*err) *err = kRunPast63;
            z = 64;
          } else {
            if (kWrite && cur < blk_end) coef[cur * 64 + z] = (int16_t)extend((top << len) >> (32 - s), s);
            ++z;
          }
          p += s;
        }
      }
    }
    if (z >= 64) {
      z = 0;
      c = c + 1 == bpm ? 0 : c + 1;
    }
  }
  *count = n;
  return pack_state(p, c, z);
}

struct SubArrays {
  uint64_t* start;                      // start state
  uint64_t* end;                        // state at the first codeword boundary past the subsequence
  uint32_t* end_bit;                    // bit the subsequence ends at
  int32_t* interval;
  int32_t* count;                       // blocks whose DC code starts in it
  int32_t* first;                       // exclusive scan of count
  int32_t* int_sub;                     // first subsequence of each interval (n_int + 1)
};

__global__ void __launch_bounds__(kHuffThreads) k_jpeg_huffman(const DecImage* __restrict__ imgs, const DecTables* __restrict__ tabs,
                                                               const uint8_t* __restrict__ stream, const int32_t* __restrict__ int_start,
                                                               SubArrays sa, int16_t* __restrict__ coef, int32_t* __restrict__ status,
                                                               int32_t* __restrict__ rounds_out) {
  using Scan = cub::BlockScan<int, kHuffThreads>;
  __shared__ typename Scan::TempStorage tmp;
  __shared__ DecTable s_tab[6];
  __shared__ int s_flag, s_err;
  const int img = blockIdx.x;
  const DecImage im = imgs[img];
  const int t = threadIdx.x;
  if (status[img] != kOk) {            // restart markers missing or extra: the interval table is not usable
    if (t == 0) rounds_out[img] = 0;
    return;
  }
  {
    const uint32_t* s = (const uint32_t*)tabs[img].t;
    uint32_t* d = (uint32_t*)s_tab;
    for (int k = t; k < (int)(sizeof(s_tab) / 4); k += kHuffThreads) d[k] = s[k];
  }
  const int32_t* starts = int_start + im.int0;
  const int64_t s0 = im.sub0;
  uint64_t* st = sa.start + s0;
  uint64_t* en = sa.end + s0;
  uint32_t* eb = sa.end_bit + s0;
  int32_t* iv = sa.interval + s0;
  int32_t* cnt = sa.count + s0;
  int32_t* first = sa.first + s0;
  int32_t* isub = sa.int_sub + im.int0;
  // subsequences of each interval: max(1, ceil(bits / 1024))
  int carry = 0;
  for (int a = 0; a < im.n_int; a += kHuffThreads) {
    const int k = a + t;
    int ns = 0;
    if (k < im.n_int) {
      const int64_t bits = 8ll * (starts[k + 1] - starts[k]);
      ns = bits <= 0 ? 1 : (int)((bits + kSubBits - 1) / kSubBits);
    }
    int o, total;
    Scan(tmp).ExclusiveSum(ns, o, total);
    __syncthreads();
    if (k < im.n_int) isub[k] = carry + o;
    carry += total;
  }
  const int nsub = min(carry, im.sub_cap);
  if (t == 0) isub[im.n_int] = nsub;
  __syncthreads();
  for (int j = t; j < nsub; j += kHuffThreads) {
    int lo = 0, hi = im.n_int - 1;
    while (lo < hi) {
      const int mid = (lo + hi + 1) >> 1;
      if (isub[mid] <= j) lo = mid; else hi = mid - 1;
    }
    const uint32_t b0 = 8u * (uint32_t)starts[lo], b1 = 8u * (uint32_t)starts[lo + 1];
    const uint32_t beg = b0 + (uint32_t)(j - isub[lo]) * kSubBits;
    iv[j] = lo;
    eb[j] = min(beg + kSubBits, b1);
    st[j] = pack_state(beg, 0, 0);       // true for the first subsequence of an interval, a guess for the others
  }
  __syncthreads();
  const Bits bits{(const uint32_t*)(stream + im.stream_off)};
  const int hv = im.ncomp == 1 ? 1 : im.hs * im.vs;
  int dummy = 0;
  // round 0 decodes every subsequence; each later round redecodes the ones whose start state changed
  for (int j = t; j < nsub; j += kHuffThreads)
    en[j] = decode_sub<false>(bits, s_tab, im.bpm, hv, st[j], eb[j], &cnt[j], nullptr, 0, 0, &dummy);
  int rounds = 1;
  for (; rounds <= nsub; ++rounds) {
    if (t == 0) s_flag = 0;
    __syncthreads();
    bool any = false;
    for (int j = t; j < nsub; j += kHuffThreads) {
      if (j > 0 && iv[j - 1] == iv[j] && en[j - 1] != st[j]) {
        st[j] = en[j - 1];
        cnt[j] = -1;                    // marks the subsequence to redecode
        any = true;
      }
    }
    if (any) s_flag = 1;
    __syncthreads();
    if (!s_flag) break;
    for (int j = t; j < nsub; j += kHuffThreads)
      if (cnt[j] < 0) en[j] = decode_sub<false>(bits, s_tab, im.bpm, hv, st[j], eb[j], &cnt[j], nullptr, 0, 0, &dummy);
    __syncthreads();
  }
  // first block of every subsequence, relative to its interval's first subsequence
  carry = 0;
  for (int a = 0; a < nsub; a += kHuffThreads) {
    const int j = a + t;
    int o, total;
    Scan(tmp).ExclusiveSum(j < nsub ? cnt[j] : 0, o, total);
    __syncthreads();
    if (j < nsub) first[j] = carry + o;
    carry += total;
  }
  if (t == 0) {
    s_err = 0;
    rounds_out[img] = rounds;
  }
  const int64_t nblk = (int64_t)im.mx * im.my * im.bpm;
  int16_t* cf = coef + im.blk0 * 64;
  for (int64_t e = t; e < nblk * 32; e += kHuffThreads) ((uint32_t*)cf)[e] = 0;
  __syncthreads();
  // every interval must hold its MCUs; the blocks decoded past them (from the padding bits) are dropped
  for (int k = t; k < im.n_int; k += kHuffThreads) {
    const int j0 = isub[k], j1 = isub[k + 1];
    const int got = (j1 < nsub ? first[j1] : carry) - first[j0];
    const int64_t mcus = min((int64_t)im.ri, (int64_t)im.mx * im.my - (int64_t)k * im.ri);
    if (j0 >= j1 || got < mcus * im.bpm) atomicCAS(&s_err, 0, kTooFewBlocks);
  }
  for (int j = t; j < nsub; j += kHuffThreads) {
    const int k = iv[j];
    const int64_t blk_first = (int64_t)k * im.ri * im.bpm;
    const int64_t blk_end = min(nblk, blk_first + (int64_t)im.ri * im.bpm);
    int n, err = 0;
    decode_sub<true>(bits, s_tab, im.bpm, hv, st[j], eb[j], &n, cf, blk_first + first[j] - first[isub[k]], blk_end, &err);
    if (err) atomicCAS(&s_err, 0, err);
  }
  __syncthreads();
  if (t == 0 && s_err) status[img] = s_err;
}

// ---- DC prediction ---------------------------------------------------------------------------------------------------------
struct SegSum {
  int v;
  int reset;                            // this element starts a segment
};
struct SegOp {
  __device__ __forceinline__ SegSum operator()(const SegSum& a, const SegSum& b) const {
    return SegSum{b.reset ? b.v : a.v + b.v, a.reset | b.reset};
  }
};

__global__ void __launch_bounds__(kDcThreads) k_jpeg_dc(const DecImage* __restrict__ imgs, int16_t* __restrict__ coef) {
  using Scan = cub::BlockScan<SegSum, kDcThreads>;
  __shared__ typename Scan::TempStorage tmp;
  __shared__ int s_carry;
  const DecImage im = imgs[blockIdx.x / 3];
  const int comp = blockIdx.x % 3;
  if (comp >= im.ncomp) return;
  const int per = im.ncomp == 1 ? 1 : comp == 0 ? im.hs * im.vs : 1;       // blocks of this component per MCU
  const int before = comp == 0 ? 0 : im.hs * im.vs + comp - 1;
  const int64_t nmcu = (int64_t)im.mx * im.my;
  const int64_t n = nmcu * per;
  int16_t* cf = coef + im.blk0 * 64;
  int carry = 0;
  for (int64_t a = 0; a < n; a += kDcThreads) {
    const int64_t j = a + threadIdx.x;
    int16_t* dc = nullptr;
    SegSum x{0, 0};
    if (j < n) {
      const int64_t m = j / per;
      dc = cf + (m * im.bpm + before + j % per) * 64;
      x = SegSum{*dc, (j % per == 0 && m % im.ri == 0) ? 1 : 0};
    }
    if (threadIdx.x == 0 && !x.reset) x.v += carry;
    SegSum y;
    Scan(tmp).InclusiveScan(x, y, SegOp());
    __syncthreads();
    if (dc) *dc = (int16_t)y.v;
    if (threadIdx.x == kDcThreads - 1) s_carry = y.v;
    __syncthreads();
    carry = s_carry;
    __syncthreads();
  }
}

// ---- IDCT ------------------------------------------------------------------------------------------------------------------
constexpr int kF0298 = 2446, kF0390 = 3196, kF0541 = 4433, kF0765 = 6270, kF0899 = 7373, kF1175 = 9633, kF1501 = 12299,
              kF1847 = 15137, kF1961 = 16069, kF2053 = 16819, kF2562 = 20995, kF3072 = 25172;

// jpeg_idct_islow's even and odd parts over d[0..7]; o[k] the sums before the descale.  64-bit, as jidctint.c's JLONG: exact for
// any int16 coefficient times any 16-bit quantizer.
using Long = long long;
__device__ __forceinline__ void idct_1d(const Long* d, Long* o) {
  Long z1 = (d[2] + d[6]) * kF0541;
  const Long tmp2 = z1 - d[6] * kF1847, tmp3 = z1 + d[2] * kF0765;
  const Long tmp0 = (d[0] + d[4]) * 8192, tmp1 = (d[0] - d[4]) * 8192;
  const Long t10 = tmp0 + tmp3, t13 = tmp0 - tmp3, t11 = tmp1 + tmp2, t12 = tmp1 - tmp2;
  Long o0 = d[7], o1 = d[5], o2 = d[3], o3 = d[1];
  z1 = o0 + o3;
  Long z2 = o1 + o2, z3 = o0 + o2, z4 = o1 + o3;
  const Long z5 = (z3 + z4) * kF1175;
  o0 *= kF0298;
  o1 *= kF2053;
  o2 *= kF3072;
  o3 *= kF1501;
  z1 *= -kF0899;
  z2 *= -kF2562;
  z3 = z3 * -kF1961 + z5;
  z4 = z4 * -kF0390 + z5;
  o0 += z1 + z3;
  o1 += z2 + z4;
  o2 += z2 + z3;
  o3 += z1 + z4;
  o[0] = t10 + o3;
  o[7] = t10 - o3;
  o[1] = t11 + o2;
  o[6] = t11 - o2;
  o[2] = t12 + o1;
  o[5] = t12 - o1;
  o[3] = t13 + o0;
  o[4] = t13 - o0;
}

__device__ __forceinline__ uint8_t range_limit(int x) {
  const int y = ((x + 512) & 1023) - 512 + 128;
  return (uint8_t)min(max(y, 0), 255);
}

__global__ void __launch_bounds__(kIdctBlocks * 8) k_jpeg_idct(const DecImage* __restrict__ imgs, const DecTables* __restrict__ tabs,
                                                               int n, const int16_t* __restrict__ coef, int64_t total_blocks,
                                                               uint8_t* __restrict__ planes) {
  __shared__ int s_ws[kIdctBlocks][8][9];
  const int lb = threadIdx.x >> 3, r = threadIdx.x & 7;
  const int64_t g = (int64_t)blockIdx.x * kIdctBlocks + lb;
  const bool live = g < total_blocks;
  const int i = live ? find_item(&imgs[0].blk0, n, g, kImgStride) : 0;
  const DecImage& im = imgs[i];
  int comp = 0, bx = 0, by = 0;
  if (live) {
    const int64_t l = g - im.blk0;
    if (im.ncomp == 1) {
      bx = (int)(l % im.mx);
      by = (int)(l / im.mx);
    } else {
      const int64_t m = l / im.bpm;
      const int k = (int)(l % im.bpm), hv = im.hs * im.vs;
      const int mx = (int)(m % im.mx), my = (int)(m / im.mx);
      if (k < hv) {
        bx = mx * im.hs + k % im.hs;
        by = my * im.vs + k / im.hs;
      } else {
        comp = k - hv + 1;
        bx = mx;
        by = my;
      }
    }
  }
  const int16_t* blk = coef + g * 64;
  const uint16_t* q = tabs[i].q[comp];
  // pass 1: column r; coefficients are in zigzag order
  if (live) {
    Long d[8], o[8];
#pragma unroll
    for (int k = 0; k < 8; ++k) d[k] = (Long)blk[c_unzig[k * 8 + r]] * (Long)q[k * 8 + r];
    idct_1d(d, o);
#pragma unroll
    for (int k = 0; k < 8; ++k) s_ws[lb][k][r] = (int)((o[k] + (1 << 10)) >> 11);     // jidctint.c's int workspace
  }
  __syncthreads();
  if (!live) return;
  Long d[8], o[8];
#pragma unroll
  for (int k = 0; k < 8; ++k) d[k] = s_ws[lb][r][k];
  idct_1d(d, o);
  uint8_t* dst = planes + im.plane_off[comp] + (int64_t)(by * 8 + r) * im.pw[comp] + bx * 8;
  uint32_t lo = 0, hi = 0;
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    lo |= (uint32_t)range_limit((int)((o[k] + (1 << 17)) >> 18)) << (8 * k);
    hi |= (uint32_t)range_limit((int)((o[k + 4] + (1 << 17)) >> 18)) << (8 * k);
  }
  *(uint2*)dst = make_uint2(lo, hi);
}

// ---- upsampling, colour, orientation ---------------------------------------------------------------------------------------
// Chroma sample at luma (y, x) of a plane downsampled fh x fv (jdsample.c fancy upsampling; plain replication for widths <= 2).
__device__ __forceinline__ int chroma_at(const uint8_t* p, int pw, int dw, int dh, int fh, int fv, int y, int x) {
  if (fh == 1) return p[(int64_t)y * pw + x];
  const int i = x >> 1;
  if (fv == 1) {
    const uint8_t* row = p + (int64_t)y * pw;
    if (dw <= 2) return row[i];
    if ((x & 1) == 0) return i == 0 ? row[0] : (3 * row[i] + row[i - 1] + 1) >> 2;
    return i == dw - 1 ? row[i] : (3 * row[i] + row[i + 1] + 2) >> 2;
  }
  const int rr = y >> 1;
  if (dw <= 2) return p[(int64_t)rr * pw + i];
  const int ro = (y & 1) ? min(rr + 1, dh - 1) : max(rr - 1, 0);
  const uint8_t* a = p + (int64_t)rr * pw;
  const uint8_t* b = p + (int64_t)ro * pw;
  auto cs = [&](int c) { return 3 * a[c] + b[c]; };
  if ((x & 1) == 0) return i == 0 ? (4 * cs(0) + 8) >> 4 : (3 * cs(i) + cs(i - 1) + 8) >> 4;
  return i == dw - 1 ? (4 * cs(i) + 7) >> 4 : (3 * cs(i) + cs(i + 1) + 7) >> 4;
}

__global__ void __launch_bounds__(kColorThreads) k_jpeg_color(const DecImage* __restrict__ imgs, int n, int64_t total_pix,
                                                              const uint8_t* __restrict__ planes, uint8_t* __restrict__ out) {
  const int64_t g = (int64_t)blockIdx.x * kColorThreads + threadIdx.x;
  if (g >= total_pix) return;
  const DecImage& im = imgs[find_item(&imgs[0].pix0, n, g, kImgStride)];
  const int64_t l = g - im.pix0;
  const bool swap = im.orient >= 5;
  const int ow = swap ? im.h : im.w;
  const int oy = (int)(l / ow), ox = (int)(l % ow);
  // OpenCV's ExifTransform: transpose for 5 .. 8, then the flips
  int ty = oy, tx = ox;
  const int th = swap ? im.w : im.h, tw = ow;
  const int o = im.orient;
  if (o == 3 || o == 4 || o == 7 || o == 8) ty = th - 1 - ty;
  if (o == 2 || o == 3 || o == 6 || o == 7) tx = tw - 1 - tx;
  const int y = swap ? tx : ty, x = swap ? ty : tx;
  const int Y = planes[im.plane_off[0] + (int64_t)y * im.pw[0] + x];
  uint8_t* px = out + im.out_off + l * 3;
  if (im.ncomp == 1) {
    px[0] = px[1] = px[2] = (uint8_t)Y;
    return;
  }
  const int dw = (im.w * 1 + im.hs - 1) / im.hs, dh = (im.h + im.vs - 1) / im.vs;
  const int cb = chroma_at(planes + im.plane_off[1], im.pw[1], dw, dh, im.hs, im.vs, y, x) - 128;
  const int cr = chroma_at(planes + im.plane_off[2], im.pw[2], dw, dh, im.hs, im.vs, y, x) - 128;
  const int R = Y + ((91881 * cr + 32768) >> 16);
  const int G = Y + ((-22554 * cb + 32768 - 46802 * cr) >> 16);
  const int B = Y + ((116130 * cb + 32768) >> 16);
  px[0] = (uint8_t)min(max(B, 0), 255);
  px[1] = (uint8_t)min(max(G, 0), 255);
  px[2] = (uint8_t)min(max(R, 0), 255);
}

// ---- host: header parse ----------------------------------------------------------------------------------------------------
const uint8_t kZigzag[64] = {0,  1,  8,  16, 9,  2,  3,  10, 17, 24, 32, 25, 18, 11, 4,  5,  12, 19, 26, 33, 40, 48,
                             41, 34, 27, 20, 13, 6,  7,  14, 21, 28, 35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23,
                             30, 37, 44, 51, 58, 59, 52, 45, 38, 31, 39, 46, 53, 60, 61, 54, 47, 55, 62, 63};

struct Header {
  int h = 0, w = 0, orient = 1, ri = 0, ncomp = 0;
  int cid[3], hs[3], vs[3], tq[3], td[3], ta[3];
  bool qdef[4] = {}, hdef[2][4] = {};
  uint16_t q[4][64];
  uint8_t hbits[2][4][16], hvals[2][4][256];
  int64_t scan_off = 0;
};

int rd16(const uint8_t* p) { return p[0] << 8 | p[1]; }

int exif_orientation(const uint8_t* seg, int64_t n) {
  if (n < 14 || memcmp(seg, "Exif\0\0", 6) != 0) return 1;
  const uint8_t* t = seg + 6;
  const int64_t tn = n - 6;
  bool le;
  if (t[0] == 'I' && t[1] == 'I') le = true;
  else if (t[0] == 'M' && t[1] == 'M') le = false;
  else return 1;
  auto rd = [&](int64_t o, int k) -> uint32_t {
    uint32_t v = 0;
    for (int i = 0; i < k; ++i) v |= (uint32_t)t[o + i] << (8 * (le ? i : k - 1 - i));
    return v;
  };
  const int64_t ifd = rd(4, 4);
  if (ifd + 2 > tn) return 1;
  const int cnt = (int)rd(ifd, 2);
  for (int e = 0; e < cnt; ++e) {
    const int64_t o = ifd + 2 + 12ll * e;
    if (o + 12 > tn) break;
    if (rd(o, 2) == 0x0112 && rd(o + 2, 2) == 3) {
      const int v = (int)rd(o + 8, 2);
      return v >= 1 && v <= 8 ? v : 1;
    }
  }
  return 1;
}

#define HDR_FAIL(code, ...)  \
  do {                       \
    set_error(__VA_ARGS__);  \
    return (code);           \
  } while (0)

// jdhuff.c jpeg_make_d_derived_tbl's checks of a table a scan uses: every length's codes fit in that many bits with the all-ones
// code left free (canonical code < 1 << length after the last code of each length), and DC symbols are at most 15.
bool valid_table(const uint8_t* counts, const uint8_t* vals, bool dc) {
  int last = 0, n = 0;
  for (int l = 1; l <= 16; ++l)
    if (counts[l - 1]) last = l;
  int64_t code = 0;
  for (int l = 1; l <= last; ++l) {
    code += counts[l - 1];
    n += counts[l - 1];
    if (code >= (1ll << l)) return false;
    code <<= 1;
  }
  if (dc)
    for (int i = 0; i < n; ++i)
      if (vals[i] > 15) return false;
  return true;
}

int parse_header(const uint8_t* d, int64_t len, Header* hd) {
  if (!d || len < 4 || d[0] != 0xFF || d[1] != 0xD8) HDR_FAIL(YB_ERR_INVALID, "yb_jpeg_header: no SOI");
  bool seen_exif = false, seen_sof = false;
  int64_t o = 2;
  for (;;) {
    if (o >= len || d[o] != 0xFF) HDR_FAIL(YB_ERR_INVALID, "yb_jpeg_header: no marker at byte %lld", (long long)o);
    while (o < len && d[o] == 0xFF) ++o;
    if (o + 2 >= len) HDR_FAIL(YB_ERR_INVALID, "yb_jpeg_header: truncated header");
    const int m = d[o++];
    if (m == 0x01 || (m >= 0xD0 && m <= 0xD9)) HDR_FAIL(YB_ERR_INVALID, "yb_jpeg_header: marker 0x%02x before SOS", m);
    const int n = rd16(d + o);
    if (n < 2 || o + n > len) HDR_FAIL(YB_ERR_INVALID, "yb_jpeg_header: segment 0x%02x past the end of the file", m);
    const uint8_t* seg = d + o + 2;
    const int sn = n - 2;
    if (m == 0xE1 && !seen_exif && sn >= 6 && memcmp(seg, "Exif\0\0", 6) == 0) {
      seen_exif = true;
      hd->orient = exif_orientation(seg, sn);
    } else if (m == 0xEE && sn >= 5 && memcmp(seg, "Adobe", 5) == 0) {
      HDR_FAIL(YB_ERR_UNSUPPORTED, "yb_jpeg_header: Adobe APP14 (colour transform)");
    } else if (m == 0xDB) {
      for (int p = 0; p < sn;) {
        const int pq = seg[p] >> 4, tq = seg[p] & 15, size = pq ? 128 : 64;
        if (pq > 1 || tq > 3 || p + 1 + size > sn) HDR_FAIL(YB_ERR_INVALID, "yb_jpeg_header: bad DQT");
        for (int k = 0; k < 64; ++k) hd->q[tq][kZigzag[k]] = pq ? (uint16_t)rd16(seg + p + 1 + 2 * k) : seg[p + 1 + k];
        hd->qdef[tq] = true;
        p += 1 + size;
      }
    } else if (m == 0xC4) {
      for (int p = 0; p < sn;) {
        if (p + 17 > sn) HDR_FAIL(YB_ERR_INVALID, "yb_jpeg_header: bad DHT");
        const int tc = seg[p] >> 4, th = seg[p] & 15;
        int nv = 0;
        for (int k = 0; k < 16; ++k) nv += seg[p + 1 + k];
        if (tc > 1 || th > 3 || nv > 256 || p + 17 + nv > sn) HDR_FAIL(YB_ERR_INVALID, "yb_jpeg_header: bad DHT");
        memcpy(hd->hbits[tc][th], seg + p + 1, 16);
        memcpy(hd->hvals[tc][th], seg + p + 17, nv);
        hd->hdef[tc][th] = true;
        p += 17 + nv;
      }
    } else if (m == 0xDD) {
      if (n != 4) HDR_FAIL(YB_ERR_INVALID, "yb_jpeg_header: bad DRI");
      hd->ri = rd16(seg);
    } else if (m == 0xC0 || m == 0xC1) {
      if (seen_sof || sn < 6) HDR_FAIL(YB_ERR_INVALID, "yb_jpeg_header: bad SOF");
      seen_sof = true;
      const int nf = seg[5];
      if (nf == 0 || sn != 6 + 3 * nf) HDR_FAIL(YB_ERR_INVALID, "yb_jpeg_header: bad SOF");
      if (seg[0] != 8) HDR_FAIL(YB_ERR_UNSUPPORTED, "yb_jpeg_header: %d-bit samples", seg[0]);
      hd->h = rd16(seg + 1);
      hd->w = rd16(seg + 3);
      if (!hd->h || !hd->w) HDR_FAIL(YB_ERR_UNSUPPORTED, "yb_jpeg_header: height or width 0 (DNL)");
      if (nf != 1 && nf != 3) HDR_FAIL(YB_ERR_UNSUPPORTED, "yb_jpeg_header: %d components", nf);
      hd->ncomp = nf;
      for (int i = 0; i < nf; ++i) {
        hd->cid[i] = seg[6 + 3 * i];
        hd->hs[i] = seg[7 + 3 * i] >> 4;
        hd->vs[i] = seg[7 + 3 * i] & 15;
        hd->tq[i] = seg[8 + 3 * i];
        if (hd->hs[i] < 1 || hd->hs[i] > 4 || hd->vs[i] < 1 || hd->vs[i] > 4 || hd->tq[i] > 3)
          HDR_FAIL(YB_ERR_INVALID, "yb_jpeg_header: bad component %d", i);
      }
    } else if ((m >= 0xC2 && m <= 0xCF && m != 0xC4 && m != 0xC8)) {
      HDR_FAIL(YB_ERR_UNSUPPORTED, "yb_jpeg_header: SOF 0x%02x (progressive, lossless or arithmetic)", m);
    } else if (m == 0xDA) {
      if (!seen_sof) HDR_FAIL(YB_ERR_INVALID, "yb_jpeg_header: SOS before SOF");
      const int ns = sn > 0 ? seg[0] : 0;
      if (sn != 4 + 2 * ns) HDR_FAIL(YB_ERR_INVALID, "yb_jpeg_header: bad SOS");
      if (ns != hd->ncomp) HDR_FAIL(YB_ERR_UNSUPPORTED, "yb_jpeg_header: a scan of %d of %d components (multi-scan)", ns, hd->ncomp);
      for (int i = 0; i < ns; ++i) {
        if (seg[1 + 2 * i] != hd->cid[i]) HDR_FAIL(YB_ERR_UNSUPPORTED, "yb_jpeg_header: scan components not in frame order");
        hd->td[i] = seg[2 + 2 * i] >> 4;
        hd->ta[i] = seg[2 + 2 * i] & 15;
      }
      if (seg[1 + 2 * ns] != 0 || seg[2 + 2 * ns] != 63 || seg[3 + 2 * ns] != 0)
        HDR_FAIL(YB_ERR_UNSUPPORTED, "yb_jpeg_header: spectral selection or successive approximation");
      hd->scan_off = o + n;
      if (hd->ncomp == 3) {
        const bool luma_ok = (hd->hs[0] == 1 && hd->vs[0] == 1) || (hd->hs[0] == 2 && hd->vs[0] == 1) || (hd->hs[0] == 2 && hd->vs[0] == 2);
        if (!luma_ok || hd->hs[1] != 1 || hd->vs[1] != 1 || hd->hs[2] != 1 || hd->vs[2] != 1)
          HDR_FAIL(YB_ERR_UNSUPPORTED, "yb_jpeg_header: sampling %dx%d,%dx%d,%dx%d", hd->hs[0], hd->vs[0], hd->hs[1], hd->vs[1], hd->hs[2],
                   hd->vs[2]);
        if (hd->cid[0] == 82 && hd->cid[1] == 71 && hd->cid[2] == 66) HDR_FAIL(YB_ERR_UNSUPPORTED, "yb_jpeg_header: RGB components");
      }
      for (int i = 0; i < hd->ncomp; ++i)
        if (!hd->qdef[hd->tq[i]] || hd->td[i] > 3 || hd->ta[i] > 3 || !hd->hdef[0][hd->td[i]] || !hd->hdef[1][hd->ta[i]])
          HDR_FAIL(YB_ERR_INVALID, "yb_jpeg_header: a table the scan uses is not defined");
      for (int i = 0; i < hd->ncomp; ++i)
        if (!valid_table(hd->hbits[0][hd->td[i]], hd->hvals[0][hd->td[i]], true) ||
            !valid_table(hd->hbits[1][hd->ta[i]], hd->hvals[1][hd->ta[i]], false))
          HDR_FAIL(YB_ERR_INVALID, "yb_jpeg_header: a Huffman table the scan uses is invalid (over-subscribed code lengths or a DC "
                                   "symbol above 15)");
      return YB_OK;
    }
    o += n;
  }
}

// The table must have passed valid_table: every code then fits its length, so the lookup writes stay inside lut[512].
void make_table(const uint8_t* counts, const uint8_t* vals, DecTable* t) {
  memset(t, 0, sizeof(*t));
  int code = 0, k = 0;
  for (int l = 1; l <= 16; ++l) {
    t->valoff[l] = k - code;
    for (int j = 0; j < counts[l - 1]; ++j, ++k, ++code) {
      if (l <= 9)
        for (int f = 0; f < 1 << (9 - l); ++f) t->lut[(code << (9 - l)) | f] = (uint16_t)(l << 8 | vals[k]);
    }
    t->maxcode[l] = counts[l - 1] ? code - 1 : -1;
    code <<= 1;
  }
  t->maxcode[17] = INT32_MAX;
  memcpy(t->vals, vals, k);
}

struct Geometry {
  int mx, my, bpm, nint, pw[3], ph[3];
  int64_t blocks, plane_bytes;
};

Geometry geometry(const Header& hd) {
  Geometry g{};
  if (hd.ncomp == 1) {
    g.mx = (hd.w + 7) / 8;
    g.my = (hd.h + 7) / 8;
    g.bpm = 1;
    g.pw[0] = g.mx * 8;
    g.ph[0] = g.my * 8;
  } else {
    g.mx = (hd.w + 8 * hd.hs[0] - 1) / (8 * hd.hs[0]);
    g.my = (hd.h + 8 * hd.vs[0] - 1) / (8 * hd.vs[0]);
    g.bpm = hd.hs[0] * hd.vs[0] + 2;
    g.pw[0] = g.mx * hd.hs[0] * 8;
    g.ph[0] = g.my * hd.vs[0] * 8;
    g.pw[1] = g.pw[2] = g.mx * 8;
    g.ph[1] = g.ph[2] = g.my * 8;
  }
  const int64_t nmcu = (int64_t)g.mx * g.my;
  const int64_t ri = hd.ri ? hd.ri : nmcu;
  g.nint = (int)((nmcu + ri - 1) / ri);
  g.blocks = nmcu * g.bpm;
  g.plane_bytes = 0;
  for (int c = 0; c < hd.ncomp; ++c) g.plane_bytes += align_up((size_t)g.pw[c] * g.ph[c], 16);
  return g;
}

struct DecLayout {
  size_t rounds, tables, stream, int_start, int_sub, sub_start, sub_end, sub_bit, sub_int, sub_cnt, sub_first, coef, planes, total;
};

struct BatchPlan {
  int64_t stream_bytes = 0, intervals = 0, subs = 0, blocks = 0, plane_bytes = 0;
};

DecLayout dec_layout(int n, const BatchPlan& b) {
  DecLayout l;
  size_t o = 0;
  auto take = [&](size_t bytes) {
    const size_t at = o;
    o = align_up(o + bytes, 256);
    return at;
  };
  l.rounds = take((size_t)n * sizeof(int32_t));
  l.tables = take((size_t)n * (sizeof(DecImage) + sizeof(DecTables)));
  l.stream = take((size_t)b.stream_bytes);
  l.int_start = take((size_t)b.intervals * sizeof(int32_t));
  l.int_sub = take((size_t)b.intervals * sizeof(int32_t));
  l.sub_start = take((size_t)b.subs * sizeof(uint64_t));
  l.sub_end = take((size_t)b.subs * sizeof(uint64_t));
  l.sub_bit = take((size_t)b.subs * sizeof(uint32_t));
  l.sub_int = take((size_t)b.subs * sizeof(int32_t));
  l.sub_cnt = take((size_t)b.subs * sizeof(int32_t));
  l.sub_first = take((size_t)b.subs * sizeof(int32_t));
  l.coef = take((size_t)b.blocks * 64 * sizeof(int16_t));
  l.planes = take((size_t)b.plane_bytes);
  l.total = o;
  return l;
}

// Per-file sizes of the workspace: the stream and subsequences are bounded by the entropy-coded byte count
void plan_file(const Header& hd, int64_t file_len, const Geometry& g, BatchPlan* b) {
  const int64_t scan = file_len - hd.scan_off;
  b->stream_bytes += align_up((size_t)scan + kStreamPad + 8, 16);
  b->intervals += g.nint + 1;
  b->subs += (scan * 8 + kSubBits - 1) / kSubBits + g.nint;
  b->blocks += g.blocks;
  b->plane_bytes += g.plane_bytes;
}

constexpr int64_t kMaxScanBytes = (1ll << 28) - 64;       // bit offsets within a file's stream fit in 31 bits

}  // namespace
}  // namespace yb

using namespace yb;

extern "C" int yb_jpeg_header(const uint8_t* data, int64_t len, int32_t* h, int32_t* w) {
  Header hd;
  YB_PROPAGATE(parse_header(data, len, &hd));
  const bool swap = hd.orient >= 5;
  if (h) *h = swap ? hd.w : hd.h;
  if (w) *w = swap ? hd.h : hd.w;
  return YB_OK;
}

extern "C" size_t yb_jpeg_decode_workspace_bytes(const uint8_t* src_host, const int64_t* src_off, int n) {
  if (!src_host || !src_off || n <= 0) return 0;
  BatchPlan b;
  for (int i = 0; i < n; ++i) {
    Header hd;
    const int64_t len = src_off[i + 1] - src_off[i];
    if (src_off[i] < 0 || len <= 0 || parse_header(src_host + src_off[i], len, &hd) != YB_OK) return 0;
    plan_file(hd, len, geometry(hd), &b);
  }
  return dec_layout(n, b).total;
}

extern "C" int yb_jpeg_decode_batch(const uint8_t* src_host, const uint8_t* src_dev, const int64_t* src_off, int n,
                                    const yb_val_aug_item* items, uint8_t* out, int64_t out_bytes, void* workspace,
                                    size_t workspace_bytes, int32_t* status, void* stream) {
  YB_REQUIRE(src_host && src_dev && src_off && items && out && workspace && status, YB_ERR_INVALID,
             "yb_jpeg_decode_batch: NULL pointer argument");
  YB_REQUIRE(n >= 1 && n <= 65535 && out_bytes > 0, YB_ERR_INVALID, "yb_jpeg_decode_batch: n=%d out_bytes=%lld", n, (long long)out_bytes);
  YB_REQUIRE(src_off[0] >= 0, YB_ERR_INVALID, "yb_jpeg_decode_batch: src_off[0]=%lld", (long long)src_off[0]);
  std::vector<DecImage> imgs(n);
  std::vector<DecTables> tabs(n);
  BatchPlan b;
  int64_t pix = 0;
  for (int i = 0; i < n; ++i) {
    const int64_t len = src_off[i + 1] - src_off[i];
    YB_REQUIRE(len > 0, YB_ERR_INVALID, "yb_jpeg_decode_batch: file %d: src_off %lld .. %lld", i, (long long)src_off[i],
               (long long)src_off[i + 1]);
    Header hd;
    const int s = parse_header(src_host + src_off[i], len, &hd);
    if (s != YB_OK) {
      char msg[400];
      snprintf(msg, sizeof(msg), "%s", yb_last_error());
      set_error("yb_jpeg_decode_batch: file %d: %s", i, msg);
      return s;
    }
    YB_REQUIRE(len - hd.scan_off <= kMaxScanBytes, YB_ERR_UNSUPPORTED, "yb_jpeg_decode_batch: file %d: %lld entropy-coded bytes", i,
               (long long)(len - hd.scan_off));
    const bool swap = hd.orient >= 5;
    const int oh = swap ? hd.w : hd.h, ow = swap ? hd.h : hd.w;
    const yb_val_aug_item& t = items[i];
    YB_REQUIRE(t.h == oh && t.w == ow, YB_ERR_INVALID, "yb_jpeg_decode_batch: file %d decodes to %dx%d, its item says %dx%d", i, oh, ow,
               t.h, t.w);
    const int64_t bytes = (int64_t)oh * ow * 3;
    YB_REQUIRE(t.img_off >= 0 && t.img_off <= out_bytes - bytes, YB_ERR_INVALID,
               "yb_jpeg_decode_batch: item %d: image [%lld, +%lld) outside out (%lld bytes)", i, (long long)t.img_off, (long long)bytes,
               (long long)out_bytes);
    const Geometry g = geometry(hd);
    DecImage& im = imgs[i];
    memset(&im, 0, sizeof(im));
    im.scan_off = src_off[i] + hd.scan_off;
    im.scan_end = src_off[i + 1];
    im.stream_off = b.stream_bytes;
    im.out_off = t.img_off;
    im.blk0 = b.blocks;
    im.pix0 = pix;
    int64_t po = b.plane_bytes;
    for (int c = 0; c < hd.ncomp; ++c) {
      im.plane_off[c] = po;
      im.pw[c] = g.pw[c];
      im.ph[c] = g.ph[c];
      po += align_up((size_t)g.pw[c] * g.ph[c], 16);
    }
    im.int0 = b.intervals;
    im.sub0 = b.subs;
    im.sub_cap = (int32_t)(((len - hd.scan_off) * 8 + kSubBits - 1) / kSubBits + g.nint);
    im.h = hd.h;
    im.w = hd.w;
    im.orient = hd.orient;
    im.ncomp = hd.ncomp;
    im.hs = hd.ncomp == 1 ? 1 : hd.hs[0];
    im.vs = hd.ncomp == 1 ? 1 : hd.vs[0];
    im.mx = g.mx;
    im.my = g.my;
    im.bpm = g.bpm;
    im.ri = hd.ri ? hd.ri : g.mx * g.my;
    im.n_int = g.nint;
    DecTables& tb = tabs[i];
    memset(&tb, 0, sizeof(tb));
    for (int c = 0; c < hd.ncomp; ++c) {
      make_table(hd.hbits[0][hd.td[c]], hd.hvals[0][hd.td[c]], &tb.t[2 * c]);
      make_table(hd.hbits[1][hd.ta[c]], hd.hvals[1][hd.ta[c]], &tb.t[2 * c + 1]);
      memcpy(tb.q[c], hd.q[hd.tq[c]], sizeof(tb.q[c]));
    }
    plan_file(hd, len, g, &b);
    pix += (int64_t)oh * ow;
  }
  for (int i = 0; i < n; ++i)
    for (int j = i + 1; j < n; ++j) {
      const int64_t ai = items[i].img_off, bi = ai + (int64_t)items[i].h * items[i].w * 3;
      const int64_t aj = items[j].img_off, bj = aj + (int64_t)items[j].h * items[j].w * 3;
      YB_REQUIRE(bi <= aj || bj <= ai, YB_ERR_INVALID, "yb_jpeg_decode_batch: output slots %d and %d overlap", i, j);
    }
  YB_REQUIRE(b.subs < INT32_MAX && (b.blocks + kIdctBlocks - 1) / kIdctBlocks < INT32_MAX &&
                 (pix + kColorThreads - 1) / kColorThreads < INT32_MAX,
             YB_ERR_UNSUPPORTED, "yb_jpeg_decode_batch: batch too large");
  const DecLayout l = dec_layout(n, b);
  YB_REQUIRE(workspace_bytes >= l.total, YB_ERR_INVALID, "yb_jpeg_decode_batch: workspace %zu bytes < %zu", workspace_bytes, l.total);
  cudaStream_t st = (cudaStream_t)stream;
  char* ws = (char*)workspace;
  const size_t img_bytes = (size_t)n * sizeof(DecImage), tab_bytes = (size_t)n * sizeof(DecTables);
  const StagePart parts[2] = {{imgs.data(), img_bytes, 0}, {tabs.data(), tab_bytes, img_bytes}};
  YB_PROPAGATE(stage_tables(ws + l.tables, img_bytes + tab_bytes, parts, 2, st));
  const DecImage* d_imgs = (const DecImage*)(ws + l.tables);
  const DecTables* d_tabs = (const DecTables*)(ws + l.tables + img_bytes);
  uint8_t* d_stream = (uint8_t*)(ws + l.stream);
  int32_t* d_int = (int32_t*)(ws + l.int_start);
  SubArrays sa{(uint64_t*)(ws + l.sub_start), (uint64_t*)(ws + l.sub_end), (uint32_t*)(ws + l.sub_bit), (int32_t*)(ws + l.sub_int),
               (int32_t*)(ws + l.sub_cnt),   (int32_t*)(ws + l.sub_first), (int32_t*)(ws + l.int_sub)};
  int16_t* coef = (int16_t*)(ws + l.coef);
  uint8_t* planes = (uint8_t*)(ws + l.planes);
  k_jpeg_destuff<<<n, kDestuffThreads, 0, st>>>(src_dev, d_imgs, d_stream, d_int, status);
  YB_CHECK_LAUNCH();
  k_jpeg_huffman<<<n, kHuffThreads, 0, st>>>(d_imgs, d_tabs, d_stream, d_int, sa, coef, status, (int32_t*)(ws + l.rounds));
  YB_CHECK_LAUNCH();
  k_jpeg_dc<<<3 * n, kDcThreads, 0, st>>>(d_imgs, coef);
  YB_CHECK_LAUNCH();
  k_jpeg_idct<<<(unsigned)((b.blocks + kIdctBlocks - 1) / kIdctBlocks), kIdctBlocks * 8, 0, st>>>(d_imgs, d_tabs, n, coef, b.blocks, planes);
  YB_CHECK_LAUNCH();
  k_jpeg_color<<<(unsigned)((pix + kColorThreads - 1) / kColorThreads), kColorThreads, 0, st>>>(d_imgs, n, pix, planes, out);
  YB_CHECK_LAUNCH();
  return YB_OK;
}
