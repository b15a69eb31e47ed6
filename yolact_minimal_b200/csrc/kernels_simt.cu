// CUDA-core kernels of the forward: the fp32 parity-mode convolution (also the on-device
// reference for the wgmma path), the stem, and the memory-bound glue layers (max-pool, parity
// split for stride-2 convs, FPN upsample+add, protonet upsample, head softmax/tanh scatter).
// All activations use the haloed NHWC layout described in layers.cuh.
#include "layers.cuh"
#include <mutex>
#include "vecio.cuh"
#include <math.h>
#include <algorithm>

namespace yb {

__device__ __forceinline__ bool is_halo(long long m, const Geom& g, int& n, int& y, int& x) {
  const int plane = g.plane();
  n = (int)(m / plane);
  const int pos = (int)(m - (long long)n * plane);
  y = pos / g.Wp();
  x = pos - y * g.Wp();
  return y == 0 || y == g.H + 1 || x == 0 || x == g.W + 1;
}

// ------------------------------------------------------------------------------------------------
// implicit-GEMM convolution on CUDA cores (fp32 accumulate).  64x64 tile, BK=16, 4x4 per thread.
// ------------------------------------------------------------------------------------------------
constexpr int SBM = 64, SBN = 64, SBK = 16;

template <typename T>
__global__ void __launch_bounds__(256) k_conv_simt(ConvArgs a, long long M) {
  __shared__ float As[SBK][SBM + 4];
  __shared__ float Bs[SBK][SBN + 4];
  const int tid = threadIdx.x;
  const long long m0 = (long long)blockIdx.x * SBM;
  const int n0 = blockIdx.y * SBN;
  const int tx = tid & 15, ty = tid >> 4;
  const int lr = tid >> 2, lk = (tid & 3) * 4;         // loader: row lr, k offset lk..lk+3
  const T* in = (const T*)a.in;
  const T* w = (const T*)a.weight;
  const int Ktot = a.ntaps * a.Cin_pad;
  float acc[4][4];
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;

  for (int t = 0; t < a.ntaps; ++t) {
    const long long arow = m0 + lr + a.tap_shift[t];
    const bool a_ok = (m0 + lr < M) && arow >= 0 && arow < a.in_rows;
    const T* ap = in + arow * a.Cin + lk;
    const T* bp = w + (long long)(n0 + lr) * Ktot + (long long)t * a.Cin_pad + lk;
    for (int k0 = 0; k0 < a.Cin_pad; k0 += SBK) {
      float av[4] = {0.f, 0.f, 0.f, 0.f}, bv[4];
      if (a_ok && k0 + lk < a.Cin) {
#pragma unroll
        for (int q = 0; q < 4; ++q) av[q] = Act<T>::ld(ap + k0 + q);
      }
#pragma unroll
      for (int q = 0; q < 4; ++q) bv[q] = Act<T>::ld(bp + k0 + q);
      __syncthreads();
#pragma unroll
      for (int q = 0; q < 4; ++q) { As[lk + q][lr] = av[q]; Bs[lk + q][lr] = bv[q]; }
      __syncthreads();
#pragma unroll
      for (int k = 0; k < SBK; ++k) {
        const float4 af = *reinterpret_cast<const float4*>(&As[k][ty * 4]);
        const float4 bf = *reinterpret_cast<const float4*>(&Bs[k][tx * 4]);
        const float ar[4] = {af.x, af.y, af.z, af.w}, br[4] = {bf.x, bf.y, bf.z, bf.w};
#pragma unroll
        for (int i = 0; i < 4; ++i)
#pragma unroll
          for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(ar[i], br[j], acc[i][j]);
      }
    }
  }
  // epilogue
  const T* res = (const T*)a.residual;
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const long long m = m0 + ty * 4 + i;
    if (m >= M) continue;
    int n, y, x;
    const bool halo = is_halo(m, a.g, n, y, x);
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int c = n0 + tx * 4 + j;
      if (c >= a.Cout_pad) continue;
      float v = acc[i][j] + a.bias[c];
      if (a.out_mode == 0) {
        if (c >= a.Cout) continue;
        if (res) v += Act<T>::ld(res + m * a.Cout + c);
        v = apply_act(v, a.relu);
        Act<T>::st((T*)a.out + m * a.Cout + c, halo ? 0.f : v);
      } else if (!halo) {
        v = apply_act(v, a.relu);
        const long long r = ((long long)n * a.g.H + (y - 1)) * a.g.W + (x - 1);
        ((float*)a.out)[r * a.Cout_pad + c] = v;
      }
    }
  }
}

int launch_conv_simt(const ConvArgs& a, cudaStream_t s) {
  const long long M = (long long)a.B * a.g.plane();
  dim3 grid((unsigned)((M + SBM - 1) / SBM), (unsigned)ceil_div(a.Cout_pad, SBN));
  YB_REQUIRE(a.Cin % 4 == 0 && a.Cin_pad % SBK == 0, YB_ERR_UNSUPPORTED, "conv_simt: Cin=%d / Cin_pad=%d", a.Cin, a.Cin_pad);
  YB_DISPATCH_DT(a.act_dt, (k_conv_simt<T><<<grid, 256, 0, s>>>(a, M)));
  YB_CHECK_LAUNCH();
  return YB_OK;
}

// ------------------------------------------------------------------------------------------------
// stem: conv 7x7 s2 p3 (3->64) + folded BN + ReLU, NCHW fp32 image -> haloed NHWC.
// One thread = one output pixel x 64 channels; 16x16 pixel tile per block.
// ------------------------------------------------------------------------------------------------
constexpr int ST = 16;                       // tile side (output pixels)
constexpr int SP = ST * 2 + 5;               // input patch side (37)

template <typename T>
__global__ void __launch_bounds__(256) k_stem(const float* __restrict__ img, const float* __restrict__ w,
                                              const float* __restrict__ bias, T* __restrict__ out, int S, int H1) {
  extern __shared__ float sm[];
  float* s_w = sm;                           // [7*7*3][64]
  float* s_in = sm + 147 * 64;               // [3][SP][SP+1]
  const int tid = threadIdx.x, b = blockIdx.z;
  const int oy0 = blockIdx.y * ST, ox0 = blockIdx.x * ST;
  for (int i = tid; i < 147 * 64; i += 256) s_w[i] = w[i];
  const int iy0 = oy0 * 2 - 3, ix0 = ox0 * 2 - 3;
  for (int i = tid; i < 3 * SP * SP; i += 256) {
    const int c = i / (SP * SP), r = (i / SP) % SP, q = i % SP;
    const int iy = iy0 + r, ix = ix0 + q;
    float v = 0.f;
    if (iy >= 0 && iy < S && ix >= 0 && ix < S) v = img[(((size_t)b * 3 + c) * S + iy) * S + ix];
    s_in[(c * SP + r) * (SP + 1) + q] = v;
  }
  __syncthreads();
  const int py = tid / ST, px = tid % ST;
  const int oy = oy0 + py, ox = ox0 + px;
  float acc[64];
#pragma unroll
  for (int c = 0; c < 64; ++c) acc[c] = 0.f;
  for (int r = 0; r < 7; ++r)
    for (int q = 0; q < 7; ++q)
#pragma unroll
      for (int ci = 0; ci < 3; ++ci) {
        const float v = s_in[(ci * SP + py * 2 + r) * (SP + 1) + px * 2 + q];
        const float4* wp = reinterpret_cast<const float4*>(s_w + ((r * 7 + q) * 3 + ci) * 64);
#pragma unroll
        for (int c4 = 0; c4 < 16; ++c4) {
          const float4 ww = wp[c4];
          acc[c4 * 4 + 0] = fmaf(v, ww.x, acc[c4 * 4 + 0]);
          acc[c4 * 4 + 1] = fmaf(v, ww.y, acc[c4 * 4 + 1]);
          acc[c4 * 4 + 2] = fmaf(v, ww.z, acc[c4 * 4 + 2]);
          acc[c4 * 4 + 3] = fmaf(v, ww.w, acc[c4 * 4 + 3]);
        }
      }
  if (oy < H1 && ox < H1) {
    T* o = out + (((size_t)b * (H1 + 2) + oy + 1) * (H1 + 2) + ox + 1) * 64;
#pragma unroll
    for (int c = 0; c < 64; ++c) Act<T>::st(o + c, fmaxf(acc[c] + bias[c], 0.f));
  }
}

// ------------------------------------------------------------------------------------------------
// stem, 16-bit modes: space-to-depth repack.  The 7x7 stride-2 convolution over 3 channels equals a 4x4
// stride-1 convolution over the 12 channels (py, px, ci) of the 2x2 space-to-depth image (one all-zero tap
// row/column pads 7 to 8).  This kernel writes that image, 16-bit, channels padded 12 -> 16, on the SAME
// haloed pixel grid as the stem output:  s2d[b][Y][X][(py*2+px)*3+ci] = img[b][ci][2Y+py-4][2X+px-4]
// (zero outside the image), so tap (dy, dx) of output pixel m is pixel m + (dy-1)*Wp - 1 + dx.  The four dx
// taps of one dy are 64 CONTIGUOUS elements starting at that pixel: with WIDE=false the tensor-core kernel
// reads them through a tensor map whose rows overlap (row stride 16 elements, row length 64); WIDE=true
// materialises the four pixels per row ([pixel][64]) for drivers that refuse an overlapping map.
// ------------------------------------------------------------------------------------------------
template <typename T, bool WIDE>
__global__ void __launch_bounds__(160) k_stem_s2d(const float* __restrict__ img, T* __restrict__ out, int S, int Hp) {
  const int X = blockIdx.x * 160 + threadIdx.x, Y = blockIdx.y, b = blockIdx.z;
  if (X >= Hp) return;
  constexpr int NP = WIDE ? 4 : 1;
  T* dst = out + (((size_t)b * Hp + Y) * Hp + X) * (16 * NP);
#pragma unroll
  for (int d = 0; d < NP; ++d) {
    float v[16];
#pragma unroll
    for (int c = 0; c < 16; ++c) v[c] = 0.f;
    const int ix0 = 2 * (X + d) - 4;
    if (X + d < Hp) {
#pragma unroll
      for (int py = 0; py < 2; ++py) {
        const int iy = 2 * Y + py - 4;
        if (iy < 0 || iy >= S) continue;
#pragma unroll
        for (int ci = 0; ci < 3; ++ci) {
          const float* row = img + (((size_t)b * 3 + ci) * S + iy) * S;
          if (ix0 >= 0 && ix0 < S) v[(py * 2 + 0) * 3 + ci] = __ldg(row + ix0);
          if (ix0 + 1 >= 0 && ix0 + 1 < S) v[(py * 2 + 1) * 3 + ci] = __ldg(row + ix0 + 1);
        }
      }
    }
    VecIO<T>::store(dst + d * 16, v);
    VecIO<T>::store(dst + d * 16 + 8, v + 8);
  }
}

int launch_stem_s2d(const float* img, void* out, int dt, int wide, int B, int S, int H1, cudaStream_t s) {
  YB_REQUIRE(dt != DT_F32, YB_ERR_INVALID, "stem_s2d is for the 16-bit modes");
  const int Hp = H1 + 2;
  dim3 grid(ceil_div(Hp, 160), Hp, B);
  if (dt == DT_BF16) {
    if (wide) k_stem_s2d<__nv_bfloat16, true><<<grid, 160, 0, s>>>(img, (__nv_bfloat16*)out, S, Hp);
    else k_stem_s2d<__nv_bfloat16, false><<<grid, 160, 0, s>>>(img, (__nv_bfloat16*)out, S, Hp);
  } else {
    if (wide) k_stem_s2d<__half, true><<<grid, 160, 0, s>>>(img, (__half*)out, S, Hp);
    else k_stem_s2d<__half, false><<<grid, 160, 0, s>>>(img, (__half*)out, S, Hp);
  }
  YB_CHECK_LAUNCH();
  return YB_OK;
}

template <typename T>
__global__ void k_zero_halo(T* __restrict__ t, int B, int C, int H) {
  // zero the 1-pixel frame of a haloed tensor [B][H+2][H+2][C]
  const int Hp = H + 2;
  const long long total = (long long)B * (4 * Hp - 4) * C;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int c = (int)(i % C);
    long long r = i / C;
    const int e = (int)(r % (4 * Hp - 4));
    const int b = (int)(r / (4 * Hp - 4));
    int y, x;
    if (e < Hp) { y = 0; x = e; }
    else if (e < 2 * Hp) { y = Hp - 1; x = e - Hp; }
    else if (e < 3 * Hp - 2) { y = e - 2 * Hp + 1; x = 0; }
    else { y = e - (3 * Hp - 2) + 1; x = Hp - 1; }
    Act<T>::st(t + (((size_t)b * Hp + y) * Hp + x) * C + c, 0.f);
  }
}

int launch_stem(const float* img, const float* w, const float* bias, void* out, int out_dt, int B, int S, int H1,
                cudaStream_t s) {
  const size_t smem = (147 * 64 + 3 * SP * (SP + 1)) * sizeof(float);
  dim3 grid(ceil_div(H1, ST), ceil_div(H1, ST), B);
  cudaError_t attr = cudaSuccess;
  YB_DISPATCH_DT(out_dt, attr = cudaFuncSetAttribute(k_stem<T>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
                 if (attr == cudaSuccess) k_stem<T><<<grid, 256, smem, s>>>(img, w, bias, (T*)out, S, H1));
  YB_CHECK_CUDA(attr);
  YB_CHECK_LAUNCH();
  YB_DISPATCH_DT(out_dt, (k_zero_halo<T><<<kSmCount, 256, 0, s>>>((T*)out, B, 64, H1)));
  YB_CHECK_LAUNCH();
  return YB_OK;
}

// ------------------------------------------------------------------------------------------------
// max-pool 3x3 s2 p1 on post-ReLU data (zero halo == -inf padding because everything is >= 0)
// ------------------------------------------------------------------------------------------------
// Elementwise kernels use a (x*channel-vectors, y, image) launch geometry: no 64-bit index arithmetic
// (the first versions spent ~75 % of their issue slots on long-long div/mod).
// max of two 16-byte vectors in their own type: the maximum of representable values is representable, so the packed 16-bit
// compare gives the same bits as converting to fp32 and back (without the 24 conversions per load)
template <typename T> __device__ __forceinline__ uint4 vmax16(uint4 a, uint4 b);
template <> __device__ __forceinline__ uint4 vmax16<float>(uint4 a, uint4 b) {
  return make_uint4(__float_as_uint(fmaxf(__uint_as_float(a.x), __uint_as_float(b.x))), __float_as_uint(fmaxf(__uint_as_float(a.y), __uint_as_float(b.y))),
                    __float_as_uint(fmaxf(__uint_as_float(a.z), __uint_as_float(b.z))), __float_as_uint(fmaxf(__uint_as_float(a.w), __uint_as_float(b.w))));
}
template <> __device__ __forceinline__ uint4 vmax16<__half>(uint4 a, uint4 b) {
  uint4 r;
  const __half2* x = reinterpret_cast<const __half2*>(&a); const __half2* y = reinterpret_cast<const __half2*>(&b);
  __half2* o = reinterpret_cast<__half2*>(&r);
#pragma unroll
  for (int i = 0; i < 4; ++i) o[i] = __hmax2(x[i], y[i]);
  return r;
}
template <> __device__ __forceinline__ uint4 vmax16<__nv_bfloat16>(uint4 a, uint4 b) {
  uint4 r;
  const __nv_bfloat162* x = reinterpret_cast<const __nv_bfloat162*>(&a); const __nv_bfloat162* y = reinterpret_cast<const __nv_bfloat162*>(&b);
  __nv_bfloat162* o = reinterpret_cast<__nv_bfloat162*>(&r);
#pragma unroll
  for (int i = 0; i < 4; ++i) o[i] = __hmax2(x[i], y[i]);
  return r;
}

template <typename T>
__global__ void __launch_bounds__(256) k_maxpool(const T* __restrict__ in, T* __restrict__ out, int C, int Hin, int Hout) {
  constexpr int N = VecIO<T>::N;
  const int Hpi = Hin + 2, Hpo = Hout + 2, CV = C / N;
  const int t = blockIdx.x * 256 + threadIdx.x;
  if (t >= Hpo * CV) return;
  const int xp = t / CV, cv = t - xp * CV, yp = blockIdx.y, b = blockIdx.z;
  uint4 m = make_uint4(0u, 0u, 0u, 0u);                      // +0.0 in every type: the inputs are post-ReLU
  if (yp >= 1 && yp <= Hout && xp >= 1 && xp <= Hout) {
    const int y = yp - 1, x = xp - 1;                      // window rows 2y-1..2y+1 -> haloed 2y..2y+2
    uint4 v[9];
#pragma unroll
    for (int dy = 0; dy < 3; ++dy)
#pragma unroll
      for (int dx = 0; dx < 3; ++dx)
        v[dy * 3 + dx] = __ldg(reinterpret_cast<const uint4*>(in + (((size_t)b * Hpi + 2 * y + dy) * Hpi + 2 * x + dx) * C + cv * N));
#pragma unroll
    for (int i = 0; i < 9; ++i) m = vmax16<T>(m, v[i]);
  }
  *reinterpret_cast<uint4*>(out + (((size_t)b * Hpo + yp) * Hpo + xp) * C + cv * N) = m;
}

int launch_maxpool(const void* in, void* out, int dt, int B, int C, int Hin, int Hout, cudaStream_t s) {
  const int cv = C / (dt == DT_F32 ? 4 : 8);
  dim3 grid(ceil_div((Hout + 2) * cv, 256), Hout + 2, B);
  YB_DISPATCH_DT(dt, (k_maxpool<T><<<grid, 256, 0, s>>>((const T*)in, (T*)out, C, Hin, Hout)));
  YB_CHECK_LAUNCH();
  return YB_OK;
}

// ------------------------------------------------------------------------------------------------
// parity split for stride-2 convs: plane (p,q)[y'][x'] = X[2y'+p][2x'+q] (0 outside), y' in
// [-1, Hout], stored with the OUTPUT's haloed geometry.  nplanes = 4 (3x3 s2) or 1 (1x1 s2).
// ------------------------------------------------------------------------------------------------
// A pure copy: 16 raw bytes per thread (8 sixteen-bit or 4 fp32 channels), no conversion (the first version went through
// VecIO's float unpack / clamp / repack and was instruction-issue bound at 76 %: profiles/r2_glue_kernels.txt).
template <typename T>
__global__ void __launch_bounds__(256) k_phase_split(const T* __restrict__ in, T* __restrict__ out, int B, int C, int Hin, int Hout,
                                                     long long plane_stride_rows) {
  constexpr int N = VecIO<T>::N;
  constexpr int kPx = 4;                                               // output pixels per thread: four independent 16-byte loads in flight
  const int Hpi = Hin + 2, Hpo = Hout + 2, CV = C / N;
  const int nq = (Hpo + kPx - 1) / kPx;
  const int t = blockIdx.x * 256 + threadIdx.x;
  if (t >= nq * CV) return;
  const int xq = t / CV, cv = t - xq * CV, yp = blockIdx.y;
  const int pl = blockIdx.z / B, b = blockIdx.z - pl * B;
  const int p = pl >> 1, q = pl & 1;
  const int iy = 2 * (yp - 1) + p;
  const bool row_ok = iy >= 0 && iy < Hin;
  const T* irow = in + (((size_t)b * Hpi + iy + 1) * Hpi + 1) * C + cv * N;
  T* orow = out + ((size_t)pl * plane_stride_rows + ((size_t)b * Hpo + yp) * Hpo) * C + cv * N;
  uint4 v[kPx];
#pragma unroll
  for (int i = 0; i < kPx; ++i) {
    const int xp = xq * kPx + i, ix = 2 * (xp - 1) + q;
    v[i] = make_uint4(0u, 0u, 0u, 0u);
    if (row_ok && xp < Hpo && ix >= 0 && ix < Hin) v[i] = __ldg(reinterpret_cast<const uint4*>(irow + (size_t)ix * C));
  }
#pragma unroll
  for (int i = 0; i < kPx; ++i) {
    const int xp = xq * kPx + i;
    if (xp < Hpo) *reinterpret_cast<uint4*>(orow + (size_t)xp * C) = v[i];
  }
}

int launch_phase_split(const void* in, void* out, int dt, int B, int C, int Hin, int Hout, int nplanes,
                       long long plane_stride_rows, cudaStream_t s) {
  const int cv = C / (dt == DT_F32 ? 4 : 8);
  dim3 grid(ceil_div(((Hout + 2 + 3) / 4) * cv, 256), Hout + 2, B * nplanes);
  YB_DISPATCH_DT(dt, (k_phase_split<T><<<grid, 256, 0, s>>>((const T*)in, (T*)out, B, C, Hin, Hout, plane_stride_rows)));
  YB_CHECK_LAUNCH();
  return YB_OK;
}

// ------------------------------------------------------------------------------------------------
// FPN top-down: fine += bilinear(coarse -> fine size), align_corners=False (modules/yolact.py:74-80)
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ void src_index(int dst, float scale, bool align, int in_size, int& i0, int& i1, float& l0, float& l1) {
  float src = align ? scale * (float)dst : fmaxf(scale * ((float)dst + 0.5f) - 0.5f, 0.f);
  i0 = min((int)src, in_size - 1);
  i1 = min(i0 + 1, in_size - 1);
  l1 = src - (float)i0;
  l0 = 1.f - l1;
}

template <typename T, bool kAdd, bool kAlign>
__global__ void __launch_bounds__(256) k_bilinear(const T* __restrict__ src, T* __restrict__ dst, int C, int Hs, int Hd, float scale) {
  constexpr int N = VecIO<T>::N;
  const int Hps = Hs + 2, Hpd = Hd + 2, CV = C / N;
  const int t = blockIdx.x * 256 + threadIdx.x;
  if (t >= Hpd * CV) return;
  const int xp = t / CV, cv = t - xp * CV, yp = blockIdx.y, b = blockIdx.z;
  T* d = dst + (((size_t)b * Hpd + yp) * Hpd + xp) * C + cv * N;
  const bool halo = yp == 0 || yp == Hd + 1 || xp == 0 || xp == Hd + 1;
  float v[N];
  if (halo) {
    if (!kAdd) {
#pragma unroll
      for (int e = 0; e < N; ++e) v[e] = 0.f;
      VecIO<T>::store(d, v);
    }
    return;
  }
  int y0, y1, x0, x1; float ly0, ly1, lx0, lx1;
  src_index(yp - 1, scale, kAlign, Hs, y0, y1, ly0, ly1);
  src_index(xp - 1, scale, kAlign, Hs, x0, x1, lx0, lx1);
  const T* sb = src + (size_t)b * Hps * Hps * C + cv * N;
  float v00[N], v01[N], v10[N], v11[N];
  VecIO<T>::load(sb + ((size_t)(y0 + 1) * Hps + x0 + 1) * C, v00);
  VecIO<T>::load(sb + ((size_t)(y0 + 1) * Hps + x1 + 1) * C, v01);
  VecIO<T>::load(sb + ((size_t)(y1 + 1) * Hps + x0 + 1) * C, v10);
  VecIO<T>::load(sb + ((size_t)(y1 + 1) * Hps + x1 + 1) * C, v11);
  if (kAdd) VecIO<T>::load(d, v);
#pragma unroll
  for (int e = 0; e < N; ++e) {
    const float tt = ly0 * (lx0 * v00[e] + lx1 * v01[e]) + ly1 * (lx0 * v10[e] + lx1 * v11[e]);
    v[e] = kAdd ? v[e] + tt : tt;
  }
  VecIO<T>::store(d, v);
}

int launch_upsample_add(const void* coarse, void* fine, int dt, int B, int C, int Hc, int Hf, cudaStream_t s) {
  const int cv = C / (dt == DT_F32 ? 4 : 8);
  dim3 grid(ceil_div((Hf + 2) * cv, 256), Hf + 2, B);
  const float scale = (float)Hc / (float)Hf;
  YB_DISPATCH_DT(dt, (k_bilinear<T, true, false><<<grid, 256, 0, s>>>((const T*)coarse, (T*)fine, C, Hc, Hf, scale)));
  YB_CHECK_LAUNCH();
  return YB_OK;
}

// protonet: bilinear x2, align_corners=True (modules/yolact.py:43,:51).
// One block per 4 x 16 tile of (haloed) output pixels, all C channels, in two phases: (1) the vertical interpolation runs once per
// (output row, source column) -- <= 4 x 10 per tile -- into an fp32 shared-memory buffer; (2) every output is one horizontal
// interpolation of two of those.  k_bilinear (four 16-byte gathers, 32 conversions
// and both interpolations per 16-byte output) spent 250 instructions per output vector and was issue-bound at 81 % with the DRAM
// pipe at 25 % (profiles/r2_glue_kernels.txt); this form needs ~60.  Interpolation weights are those of k_bilinear / torch; the
// vertical-first order changes fp32 rounding only.
constexpr int kUpTY = 4, kUpTX = 16, kUpSX = 10;                        // output tile, source columns it can touch

template <typename T>
__global__ void __launch_bounds__(256) k_upsample2x_tile(const T* __restrict__ src, T* __restrict__ dst, int C, int Hs, int Hd, float scale) {
  constexpr int N = VecIO<T>::N;
  extern __shared__ __align__(16) uint8_t s_up[];
  float* sv = reinterpret_cast<float*>(s_up);                          // [kUpTY][kUpSX][C] vertically interpolated, fp32
  __shared__ int s_y0[kUpTY], s_y1[kUpTY], s_x0[kUpTX], s_x1[kUpTX];
  __shared__ float s_ly0[kUpTY], s_ly1[kUpTY], s_lx0[kUpTX], s_lx1[kUpTX];
  const int Hps = Hs + 2, Hpd = Hd + 2, CV = C / N;                    // 256 % CV == 0 (checked by the launcher)
  const int ty0 = blockIdx.y * kUpTY, tx0 = blockIdx.x * kUpTX, b = blockIdx.z;
  // valid (non-halo) output range of the tile, in haloed coordinates
  const int vy0 = max(ty0, 1), vy1 = min(ty0 + kUpTY - 1, Hd), vx0 = max(tx0, 1), vx1 = min(tx0 + kUpTX - 1, Hd);
  int sx0 = 0, nx = 0;
  if (vy0 <= vy1 && vx0 <= vx1) {
    int i0, i1; float l0, l1;
    src_index(vx0 - 1, scale, true, Hs, sx0, i1, l0, l1);
    src_index(vx1 - 1, scale, true, Hs, i0, i1, l0, l1); nx = i1 - sx0 + 1;
  }
  if (threadIdx.x < kUpTY) {                                           // per-row / per-column source indices (patch-relative) and weights
    const int oy = ty0 + (int)threadIdx.x;
    int y0 = -1, y1 = -1; float l0 = 0.f, l1 = 0.f;
    if (oy >= 1 && oy <= Hd) src_index(oy - 1, scale, true, Hs, y0, y1, l0, l1);      // absolute source rows
    s_y0[threadIdx.x] = y0; s_y1[threadIdx.x] = y1; s_ly0[threadIdx.x] = l0; s_ly1[threadIdx.x] = l1;
  } else if (threadIdx.x >= 32 && threadIdx.x < 32 + kUpTX) {
    const int k = (int)threadIdx.x - 32, ox = tx0 + k;
    int x0 = -1, x1 = -1; float l0 = 0.f, l1 = 0.f;
    if (ox >= 1 && ox <= Hd) { src_index(ox - 1, scale, true, Hs, x0, x1, l0, l1); x0 -= sx0; x1 -= sx0; }
    s_x0[k] = x0; s_x1[k] = x1; s_lx0[k] = l0; s_lx1[k] = l1;
  }
  const int cv = (int)threadIdx.x % CV, sub = (int)threadIdx.x / CV, nsub = 256 / CV;   // nsub >= 8 (launcher: CV <= 32)
  const T* sb = src + (size_t)b * Hps * Hps * C + cv * N;
  __syncthreads();
  {                                                                    // (1) vertical interpolation, once per (output row, source column):
    constexpr int kIt = (kUpTY * kUpSX + 7) / 8;                       //     all loads of a thread's <= 5 entries are issued before the first use
    uint4 ra[kIt], rc[kIt];
    int slot[kIt];
#pragma unroll
    for (int it = 0; it < kIt; ++it) {
      const int e = sub + it * nsub;
      slot[it] = -1;
      if (e < kUpTY * nx) {
        const int r = e / nx, j = e - r * nx;
        const int y0 = s_y0[r];
        if (y0 >= 0) {
          slot[it] = r * kUpSX + j;
          ra[it] = __ldg(reinterpret_cast<const uint4*>(sb + ((size_t)(y0 + 1) * Hps + sx0 + j + 1) * C));
          rc[it] = __ldg(reinterpret_cast<const uint4*>(sb + ((size_t)(s_y1[r] + 1) * Hps + sx0 + j + 1) * C));
        }
      }
    }
#pragma unroll
    for (int it = 0; it < kIt; ++it) {
      if (slot[it] < 0) continue;
      const int r = slot[it] / kUpSX;
      float a[N], c[N], v[N];
      VecIO<T>::load(reinterpret_cast<const T*>(&ra[it]), a);
      VecIO<T>::load(reinterpret_cast<const T*>(&rc[it]), c);
      const float l0 = s_ly0[r], l1 = s_ly1[r];
#pragma unroll
      for (int q = 0; q < N; ++q) v[q] = l0 * a[q] + l1 * c[q];
      float* o = sv + (size_t)slot[it] * C + cv * 4;                   // [slot][N/4 planes][CV] float4: lanes touch consecutive 16-byte words
#pragma unroll
      for (int q = 0; q < N; q += 4) *reinterpret_cast<float4*>(o + (q / 4) * (CV * 4)) = make_float4(v[q], v[q + 1], v[q + 2], v[q + 3]);
    }
  }
  __syncthreads();
  for (int e = sub; e < kUpTY * kUpTX; e += nsub) {                    // (2) horizontal interpolation + store
    const int r = e / kUpTX, k = e % kUpTX, oy = ty0 + r, ox = tx0 + k;
    if (oy >= Hpd || ox >= Hpd) continue;
    T* d = dst + (((size_t)b * Hpd + oy) * Hpd + ox) * C + cv * N;
    float v[N];
    const int x0 = s_x0[k];
    if (x0 < 0 || s_y0[r] < 0) {                                       // halo
#pragma unroll
      for (int q = 0; q < N; ++q) v[q] = 0.f;
    } else {
      const float* p0 = sv + ((size_t)(r * kUpSX + x0)) * C + cv * 4;
      const float* p1 = sv + ((size_t)(r * kUpSX + s_x1[k])) * C + cv * 4;
      const float l0 = s_lx0[k], l1 = s_lx1[k];
#pragma unroll
      for (int q = 0; q < N; q += 4) {
        const float4 f0 = *reinterpret_cast<const float4*>(p0 + (q / 4) * (CV * 4)), f1 = *reinterpret_cast<const float4*>(p1 + (q / 4) * (CV * 4));
        v[q] = l0 * f0.x + l1 * f1.x; v[q + 1] = l0 * f0.y + l1 * f1.y; v[q + 2] = l0 * f0.z + l1 * f1.z; v[q + 3] = l0 * f0.w + l1 * f1.w;
      }
    }
    VecIO<T>::store(d, v);
  }
}

int launch_upsample2x_ac(const void* in, void* out, int dt, int B, int C, int Hin, cudaStream_t s) {
  const int Hout = 2 * Hin;
  const float scale = Hout > 1 ? (float)(Hin - 1) / (float)(Hout - 1) : 0.f;
  const int cv = C / (dt == DT_F32 ? 4 : 8);
  const size_t smem = (size_t)kUpTY * kUpSX * C * 4;
  if (dt != DT_F32 && smem <= 100 * 1024 && C % 8 == 0 && 256 % cv == 0 && cv <= 32) {
    {  // function attributes are per device: set once for the device this launch runs on
      static std::mutex mu;
      static bool done[64] = {};
      int dev = 0;
      YB_CHECK_CUDA(cudaGetDevice(&dev));
      std::lock_guard<std::mutex> lock(mu);
      if (dev >= 0 && dev < 64 && !done[dev]) {
        YB_CHECK_CUDA(cudaFuncSetAttribute(k_upsample2x_tile<__half>, cudaFuncAttributeMaxDynamicSharedMemorySize, 100 * 1024));
        YB_CHECK_CUDA(cudaFuncSetAttribute(k_upsample2x_tile<__nv_bfloat16>, cudaFuncAttributeMaxDynamicSharedMemorySize, 100 * 1024));
        done[dev] = true;
      }
    }
    dim3 grid(ceil_div(Hout + 2, kUpTX), ceil_div(Hout + 2, kUpTY), B);
    if (dt == DT_F16) k_upsample2x_tile<__half><<<grid, 256, smem, s>>>((const __half*)in, (__half*)out, C, Hin, Hout, scale);
    else k_upsample2x_tile<__nv_bfloat16><<<grid, 256, smem, s>>>((const __nv_bfloat16*)in, (__nv_bfloat16*)out, C, Hin, Hout, scale);
  } else {
    dim3 grid(ceil_div((Hout + 2) * cv, 256), Hout + 2, B);
    YB_DISPATCH_DT(dt, (k_bilinear<T, false, true><<<grid, 256, 0, s>>>((const T*)in, (T*)out, C, Hin, Hout, scale)));
  }
  YB_CHECK_LAUNCH();
  return YB_OK;
}

// ------------------------------------------------------------------------------------------------
// head epilogue: per (image, pixel) -- one warp -- softmax over the class logits of its anchors, copy
// the box regression, tanh the mask coefficients, written in the reference's
// [B, A, C] / [B, A, 4] / [B, A, K] layout (modules/yolact.py:26-31,:155-163).
// head row layout: [conf: R*C | box: R*4 | coef: R*K | pad]
// ------------------------------------------------------------------------------------------------
// One warp per pixel: the pixel's head row (R*NC + R*4 + R*K <= ld floats, 16-byte aligned) is read with 128-bit loads into the
// warp's shared-memory slice, the R softmaxes / tanh run from there, and the results leave as the pixel's R consecutive anchor rows --
// contiguous runs of R*NC, R*4 and R*K floats in the outputs.  (The first version gave each warp one (pixel, anchor) item and read
// its 81 + 4 + 32 values with partially filled, misaligned loads: 2.9 TB/s; profiles/r2_glue_kernels.txt.)
constexpr int kHeadWarps = 8;
constexpr int kHeadLogitsPerLane = (YB_MAX_CLASSES + 31) / 32;          // class c is lane c % 32's logit c / 32

__global__ void __launch_bounds__(kHeadWarps * 32) k_head_finalize(const float* __restrict__ head, int ld, int HW, int R, int NC, int K,
                                                                   int anchor_offset, int A_total, float* __restrict__ cls,
                                                                   float* __restrict__ box, float* __restrict__ coef) {
  extern __shared__ float s_head[];                                    // [kHeadWarps][ld]
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  const int pix = blockIdx.x * kHeadWarps + w;
  if (pix >= HW) return;
  const int b = blockIdx.y;
  float* sr = s_head + (size_t)w * ld;
  const float4* row4 = reinterpret_cast<const float4*>(head + ((size_t)b * HW + pix) * ld);
  const int used4 = (R * (NC + 4 + K) + 3) >> 2;
  for (int i = lane; i < used4; i += 32) reinterpret_cast<float4*>(sr)[i] = __ldg(row4 + i);
  __syncwarp();
  const size_t arow = (size_t)b * A_total + anchor_offset + (size_t)pix * R;   // first of the pixel's R anchors
  for (int a = 0; a < R; ++a) {
    float lg[kHeadLogitsPerLane], mx = -INFINITY;
#pragma unroll
    for (int i = 0; i < kHeadLogitsPerLane; ++i) {
      const int c = lane + 32 * i;
      lg[i] = c < NC ? sr[a * NC + c] : -INFINITY;
      mx = fmaxf(mx, lg[i]);
    }
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, off));
    float ex[kHeadLogitsPerLane], sum = 0.f;
#pragma unroll
    for (int i = 0; i < kHeadLogitsPerLane; ++i) { ex[i] = (lane + 32 * i) < NC ? __expf(lg[i] - mx) : 0.f; sum += ex[i]; }
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, off);
    const float inv = 1.f / sum;
    __syncwarp();                                                      // every lane has read this anchor's logits
#pragma unroll
    for (int i = 0; i < kHeadLogitsPerLane; ++i) { const int c = lane + 32 * i; if (c < NC) sr[a * NC + c] = ex[i] * inv; }
  }
  __syncwarp();
  float* co = cls + arow * NC;
  for (int i = lane; i < R * NC; i += 32) co[i] = sr[i];
  if (lane < R * 4) box[arow * 4 + lane] = sr[R * NC + lane];
  float* ko = coef + arow * K;
  for (int i = lane; i < R * K; i += 32) ko[i] = tanhf(sr[R * NC + R * 4 + i]);
}

int launch_head_finalize(const float* head, int ld, int B, int HW, int R, int NC, int K, int anchor_offset, int A_total,
                         float* cls, float* box, float* coef, cudaStream_t s) {
  YB_REQUIRE(NC <= YB_MAX_CLASSES && K <= 64 && R * 4 <= 32, YB_ERR_UNSUPPORTED, "head_finalize: num_classes=%d > %d, coef_dim=%d > 64 or %d ratios",
             NC, YB_MAX_CLASSES, K, R);
  YB_REQUIRE(ld % 4 == 0 && R * (NC + 4 + K) <= ld && (size_t)kHeadWarps * ld * 4 <= 48 * 1024, YB_ERR_UNSUPPORTED, "head_finalize: row stride %d", ld);
  dim3 grid(ceil_div(HW, kHeadWarps), B);
  k_head_finalize<<<grid, kHeadWarps * 32, (size_t)kHeadWarps * ld * 4, s>>>(head, ld, HW, R, NC, K, anchor_offset, A_total, cls, box, coef);
  YB_CHECK_LAUNCH();
  return YB_OK;
}

// ------------------------------------------------------------------------------------------------
// debug tap: haloed NHWC -> dense NCHW fp32
// ------------------------------------------------------------------------------------------------
template <typename T>
__global__ void k_read_act(const T* __restrict__ in, int B, int C, int H, float* __restrict__ out) {
  const int Hp = H + 2;
  const long long total = (long long)B * C * H * H;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int x = (int)(i % H);
    long long r = i / H;
    const int y = (int)(r % H); r /= H;
    const int c = (int)(r % C);
    const int b = (int)(r / C);
    out[i] = Act<T>::ld(in + (((size_t)b * Hp + y + 1) * Hp + x + 1) * C + c);
  }
}

template <typename T>
__global__ void k_write_act(const float* __restrict__ in, int B, int C, int H, T* __restrict__ out) {
  const int Hp = H + 2;
  const long long total = (long long)B * Hp * Hp * C;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int c = (int)(i % C);
    long long r = i / C;
    const int xp = (int)(r % Hp); r /= Hp;
    const int yp = (int)(r % Hp);
    const int b = (int)(r / Hp);
    float v = 0.f;
    if (yp >= 1 && yp <= H && xp >= 1 && xp <= H) v = in[(((size_t)b * C + c) * H + yp - 1) * H + xp - 1];
    Act<T>::st(out + i, v);
  }
}

int launch_write_activation(const float* in_nchw, int dt, int B, int C, int H, void* out, cudaStream_t s) {
  const long long total = (long long)B * C * (H + 2) * (H + 2);
  const int blocks = (int)std::min<long long>((total + 255) / 256, (long long)kSmCount * 16);
  YB_DISPATCH_DT(dt, (k_write_act<T><<<blocks, 256, 0, s>>>(in_nchw, B, C, H, (T*)out)));
  YB_CHECK_LAUNCH();
  return YB_OK;
}

int launch_read_activation(const void* in, int dt, int B, int C, int H, float* out, cudaStream_t s) {
  const long long total = (long long)B * C * H * H;
  const int blocks = (int)std::min<long long>((total + 255) / 256, (long long)kSmCount * 16);
  YB_DISPATCH_DT(dt, (k_read_act<T><<<blocks, 256, 0, s>>>((const T*)in, B, C, H, out)));
  YB_CHECK_LAUNCH();
  return YB_OK;
}

}  // namespace yb
