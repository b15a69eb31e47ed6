// CUDA-core kernels of the TRAINING path (SURVEY.md 8 row a12): everything around the wgmma convolutions / GEMMs --
// weight packing from the fp32 master parameters, batch-statistics BatchNorm forward / backward (modules/resnet.py:20-40 in
// train mode), transposes feeding the weight-gradient GEMM, and the backward passes of the memory-bound glue layers
// (max-pool, bilinear up-sampling, ReLU, stride-2 parity planes, head scatter).  16-bit activations in the haloed NHWC layout
// of layers.cuh; statistics, parameters and parameter gradients in fp32.
#include "train.cuh"
#include "vecio.cuh"

#include <math.h>

namespace yb {

#define YB_DISPATCH16(dt, ...)                                           \
  do {                                                                   \
    if ((dt) == DT_BF16) { using T = __nv_bfloat16; __VA_ARGS__; }       \
    else { using T = __half; __VA_ARGS__; }                              \
  } while (0)

// ------------------------------------------------------------------------------------------------
// weight packing, batched over a descriptor table: fp32 [Cout][Cin][k][k]  ->
//   forward operand   wf[(row0+co) * ldf + t * Cin_pad + ci]          (K-major rows = output channels)
//   dgrad operand     wb[ci * ldb + tapslot[t] * CoutT_pad + row0+co] (K-major rows = input channels; taps regrouped by parity
//                                                                      plane for stride-2 convs so that each plane's taps are contiguous)
// ------------------------------------------------------------------------------------------------
template <typename T>
__global__ void __launch_bounds__(256) k_pack_weights(const PackDesc* __restrict__ descs) {
  const PackDesc d = descs[blockIdx.y];
  const int k2 = d.k * d.k;
  const long long total = (long long)d.Cout * d.Cin * k2;
  T* wf = (T*)d.dst_fwd;
  T* wb = (T*)d.dst_bwd;
  for (long long i = blockIdx.x * 256LL + threadIdx.x; i < total; i += (long long)gridDim.x * 256) {
    const int t = (int)(i % k2);
    const long long r = i / k2;
    const int ci = (int)(r % d.Cin), co = (int)(r / d.Cin);
    const float v = d.src[i];
    if (wf) Act<T>::st(wf + (long long)(d.row0 + co) * d.ldf + (long long)t * d.Cin_pad + ci, v);
    if (wb) Act<T>::st(wb + (long long)ci * d.ldb + (long long)d.tapslot[t] * d.CoutT_pad + d.row0 + co, v);
  }
}

int launch_pack_weights(const PackDesc* d_descs, int n, int dt, cudaStream_t s) {
  if (n == 0) return YB_OK;
  dim3 grid(32, n);
  YB_DISPATCH16(dt, (k_pack_weights<T><<<grid, 256, 0, s>>>(d_descs)));
  YB_CHECK_LAUNCH();
  return YB_OK;
}

// stem: fp32 [64][3][7][7] -> 16-bit [64][256], k = dy*64 + dx*16 + (py*2+px)*3 + ci (the space-to-depth 4x4 form, net.cu)
template <typename T>
__global__ void k_pack_stem(const float* __restrict__ src, T* __restrict__ dst) {
  const int i = blockIdx.x * 256 + threadIdx.x;
  if (i >= 64 * 256) return;
  const int co = i >> 8, k = i & 255;
  const int dy = k >> 6, dx = (k >> 4) & 3, e = k & 15;
  float v = 0.f;
  if (e < 12) {
    const int pp = e / 3, ci = e - pp * 3, py = pp >> 1, px = pp & 1;
    const int r = 2 * dy + py - 1, q = 2 * dx + px - 1;
    if (r >= 0 && q >= 0) v = src[((co * 3 + ci) * 7 + r) * 7 + q];
  }
  Act<T>::st(dst + i, v);
}

int launch_pack_stem(const float* src, void* dst, int dt, cudaStream_t s) {
  YB_DISPATCH16(dt, (k_pack_stem<T><<<64, 256, 0, s>>>(src, (T*)dst)));
  YB_CHECK_LAUNCH();
  return YB_OK;
}

// inverse for the gradient: packed fp32 [64][16 taps (dy,dx)][16] -> += / = grad [64][3][7][7]
__global__ void k_unpack_stem_grad(float* __restrict__ g, float* __restrict__ dst, float scale) {
  const int i = blockIdx.x * 256 + threadIdx.x;
  if (i >= 64 * 147) return;
  const int q = i % 7, r = (i / 7) % 7, ci = (i / 49) % 3, co = i / 147;
  const int dy = (r + 1) >> 1, py = (r + 1) & 1, dx = (q + 1) >> 1, px = (q + 1) & 1;
  float* src = g + co * 256 + (dy * 4 + dx) * 16 + (py * 2 + px) * 3 + ci;
  dst[i] = scale * *src;
  *src = 0.f;
}

int launch_unpack_stem_grad(float* g, float* dst, float scale, cudaStream_t s) {
  k_unpack_stem_grad<<<ceil_div(64 * 147, 256), 256, 0, s>>>(g, dst, scale);
  YB_CHECK_LAUNCH();
  return YB_OK;
}

// packed weight gradients fp32 [Cout_total][taps][Cin_pad] -> parameter gradient [Cout][Cin][k][k] (batched); the packed buffer is
// cleared behind the read: it is the atomically accumulated output of the split-K weight-gradient GEMMs
__global__ void __launch_bounds__(256) k_unpack_wgrad(const UnpackDesc* __restrict__ descs) {
  const UnpackDesc d = descs[blockIdx.y];
  const int k2 = d.k * d.k;
  const long long total = (long long)d.Cout * d.Cin * k2;
  for (long long i = blockIdx.x * 256LL + threadIdx.x; i < total; i += (long long)gridDim.x * 256) {
    const int t = (int)(i % k2);
    const long long r = i / k2;
    const int ci = (int)(r % d.Cin), co = (int)(r / d.Cin);
    float* src = const_cast<float*>(d.src) + (long long)(d.row0 + co) * d.ld + (long long)t * d.Cin_pad + ci;
    d.dst[i] = d.scale * *src;
    *src = 0.f;                                                    // the split-K GEMMs of the next backward pass accumulate from zero
  }
}

int launch_unpack_wgrad(const UnpackDesc* d_descs, int n, cudaStream_t s) {
  if (n == 0) return YB_OK;
  dim3 grid(32, n);
  k_unpack_wgrad<<<grid, 256, 0, s>>>(d_descs);
  YB_CHECK_LAUNCH();
  return YB_OK;
}

// ------------------------------------------------------------------------------------------------
// per-channel column sums of a [rows][C] 16-bit matrix:  sums[c] += sum_r x,  sums[C + c] += sum_r x^2   (bias gradients use the
// first half only).  Halo rows are zero and contribute nothing.
// BN statistics (kPivot, x haloed [B][Hp][Hp][C]): the sums are taken of d = x - p, p = the channel's first interior value (stored
// to sums[2C + c]), so that  var = sum d^2 / N - (sum d / N)^2  does not cancel when |mean| >> std (the plain one-pass
// sum x^2 / N - mean^2 loses (mean / std)^2 of its fp32 precision).  Halo rows are summed unshifted: zero, as before.
// ------------------------------------------------------------------------------------------------
template <typename T, bool kPivot>
__global__ void __launch_bounds__(256) k_colstats(const T* __restrict__ x, long long rows, int C, int rows_per_block, float* __restrict__ sums, int Hp) {
  extern __shared__ float sh[];                                   // [2][Cb]
  const int CV = C >> 3;                                          // 8-channel vectors per row
  const int cvb = CV < 256 ? CV : 256;                            // vectors per block
  const int rl = 256 / cvb;                                       // row lanes
  const int cv = blockIdx.x * cvb + (threadIdx.x % cvb), lane = threadIdx.x / cvb;
  const int Cb = cvb * 8;
  for (int i = threadIdx.x; i < 2 * Cb; i += 256) sh[i] = 0.f;
  __syncthreads();
  float s1[8], s2[8];
#pragma unroll
  for (int e = 0; e < 8; ++e) { s1[e] = 0.f; s2[e] = 0.f; }
  const long long r0 = (long long)blockIdx.y * rows_per_block;
  const long long r1 = r0 + rows_per_block < rows ? r0 + rows_per_block : rows;
  if (cv < CV && lane < rl) {
    float p[8];
#pragma unroll
    for (int e = 0; e < 8; ++e) p[e] = 0.f;
    if (kPivot) {
      VecIO<T>::load(x + (long long)(Hp + 1) * C + cv * 8, p);
      if (blockIdx.y == 0 && lane == 0) {
#pragma unroll
        for (int e = 0; e < 8; ++e) sums[2 * C + cv * 8 + e] = p[e];
      }
    }
    const unsigned plane = (unsigned)Hp * (unsigned)Hp;
    for (long long r = r0 + lane; r < r1; r += rl) {
      float v[8];
      VecIO<T>::load(x + r * C + cv * 8, v);
      bool halo = true;
      if (kPivot) {
        const unsigned rr = (unsigned)r % plane, yp = rr / (unsigned)Hp, xp = rr - yp * (unsigned)Hp;
        halo = yp == 0 || xp == 0 || yp == (unsigned)Hp - 1 || xp == (unsigned)Hp - 1;
      }
#pragma unroll
      for (int e = 0; e < 8; ++e) {
        const float d = halo ? v[e] : v[e] - p[e];
        s1[e] += d; s2[e] = fmaf(d, d, s2[e]);
      }
    }
    const int lc = (threadIdx.x % cvb) * 8;
#pragma unroll
    for (int e = 0; e < 8; ++e) { atomicAdd(&sh[lc + e], s1[e]); atomicAdd(&sh[Cb + lc + e], s2[e]); }
  }
  __syncthreads();
  for (int i = threadIdx.x; i < Cb; i += 256) {
    const int c = blockIdx.x * Cb + i;
    if (c < C) { atomicAdd(&sums[c], sh[i]); atomicAdd(&sums[C + c], sh[Cb + i]); }
  }
}

int launch_colstats(const void* x, int dt, long long rows, int C, float* sums, cudaStream_t s, int pivot_Hp) {
  YB_REQUIRE(C % 8 == 0, YB_ERR_UNSUPPORTED, "colstats: C=%d", C);
  YB_REQUIRE(rows < (1LL << 32), YB_ERR_UNSUPPORTED, "colstats: %lld rows", rows);
  const int CV = C / 8, cvb = CV < 256 ? CV : 256;
  const int bx = ceil_div(CV, cvb);
  long long want = (long long)kSmCount * 8 / bx;
  if (want < 1) want = 1;
  int rpb = (int)((rows + want - 1) / want);
  if (rpb < 64) rpb = 64;
  dim3 grid(bx, (unsigned)((rows + rpb - 1) / rpb));
  if (pivot_Hp > 0) YB_DISPATCH16(dt, (k_colstats<T, true><<<grid, 256, 2 * cvb * 8 * sizeof(float), s>>>((const T*)x, rows, C, rpb, sums, pivot_Hp)));
  else YB_DISPATCH16(dt, (k_colstats<T, false><<<grid, 256, 2 * cvb * 8 * sizeof(float), s>>>((const T*)x, rows, C, rpb, sums, 0)));
  YB_CHECK_LAUNCH();
  return YB_OK;
}

// batch statistics (pivot-shifted sums of launch_colstats(.., pivot_Hp): [sum d | sum d^2 | pivot]) -> affine (scale, shift),
// saved (mean, invstd), running-stat update (torch: momentum 0.1, unbiased variance)
__global__ void k_bn_finalize(const float* __restrict__ sums, int C, double count, const float* __restrict__ gamma, const float* __restrict__ beta,
                              float* __restrict__ run_mean, float* __restrict__ run_var, float momentum, float eps,
                              float* __restrict__ scale, float* __restrict__ shift, float* __restrict__ mean, float* __restrict__ invstd) {
  const int c = blockIdx.x * 256 + threadIdx.x;
  if (c >= C) return;
  const double md = (double)sums[c] / count;
  const double m = (double)sums[2 * C + c] + md;
  double var = (double)sums[C + c] / count - md * md;
  if (var < 0) var = 0;
  const float is = (float)(1.0 / sqrt(var + (double)eps));
  mean[c] = (float)m; invstd[c] = is;
  const float sc = gamma[c] * is;
  scale[c] = sc; shift[c] = beta[c] - (float)m * sc;
  if (run_mean) {
    run_mean[c] = (1.f - momentum) * run_mean[c] + momentum * (float)m;
    run_var[c] = (1.f - momentum) * run_var[c] + momentum * (float)(var * count / (count > 1 ? count - 1 : 1));
  }
}

int launch_bn_finalize(const float* sums, int C, double count, const float* gamma, const float* beta, float* run_mean, float* run_var,
                       float momentum, float eps, float* scale, float* shift, float* mean, float* invstd, cudaStream_t s) {
  k_bn_finalize<<<ceil_div(C, 256), 256, 0, s>>>(sums, C, count, gamma, beta, run_mean, run_var, momentum, eps, scale, shift, mean, invstd);
  YB_CHECK_LAUNCH();
  return YB_OK;
}

// z = act(y * scale + shift [+ res]); halo rows / columns are written as zero
template <typename T>
__global__ void __launch_bounds__(256) k_bn_apply(const T* __restrict__ y, T* __restrict__ z, const T* __restrict__ res, const float* __restrict__ scale,
                                                  const float* __restrict__ shift, int relu, int C, int H) {
  const int Hp = H + 2, CV = C >> 3;
  const int t = blockIdx.x * 256 + threadIdx.x;
  if (t >= Hp * CV) return;
  const int xp = t / CV, cv = t - xp * CV, yp = blockIdx.y, b = blockIdx.z;
  const size_t off = (((size_t)b * Hp + yp) * Hp + xp) * C + cv * 8;
  float v[8];
  if (yp == 0 || yp == H + 1 || xp == 0 || xp == H + 1) {
#pragma unroll
    for (int e = 0; e < 8; ++e) v[e] = 0.f;
  } else {
    VecIO<T>::load(y + off, v);
    float r[8];
    if (res) VecIO<T>::load(res + off, r);
#pragma unroll
    for (int e = 0; e < 8; ++e) {
      float q = fmaf(v[e], scale[cv * 8 + e], shift[cv * 8 + e]);
      if (res) q += r[e];
      v[e] = relu ? fmaxf(q, 0.f) : q;
    }
  }
  VecIO<T>::store(z + off, v);
}

int launch_bn_apply(const void* y, void* z, const void* res, const float* scale, const float* shift, int relu, int dt, int B, int C, int H,
                    cudaStream_t s) {
  dim3 grid(ceil_div((H + 2) * (C / 8), 256), H + 2, B);
  YB_DISPATCH16(dt, (k_bn_apply<T><<<grid, 256, 0, s>>>((const T*)y, (T*)z, (const T*)res, scale, shift, relu, C, H)));
  YB_CHECK_LAUNCH();
  return YB_OK;
}

// backward, pass 1:  g = dz * [z > 0];  sums[c] += sum g,  sums[C + c] += sum g * xhat,  xhat = (y - mean) * invstd
template <typename T>
__global__ void __launch_bounds__(256) k_bn_bwd_reduce(const T* __restrict__ y, const T* __restrict__ dz, const T* __restrict__ z, int relu,
                                                       const float* __restrict__ mean, const float* __restrict__ invstd, long long rows, int C,
                                                       int rows_per_block, float* __restrict__ sums) {
  extern __shared__ float sh[];
  const int CV = C >> 3;
  const int cvb = CV < 256 ? CV : 256;
  const int rl = 256 / cvb;
  const int cv = blockIdx.x * cvb + (threadIdx.x % cvb), lane = threadIdx.x / cvb;
  const int Cb = cvb * 8;
  for (int i = threadIdx.x; i < 2 * Cb; i += 256) sh[i] = 0.f;
  __syncthreads();
  float s1[8], s2[8];
#pragma unroll
  for (int e = 0; e < 8; ++e) { s1[e] = 0.f; s2[e] = 0.f; }
  const long long r0 = (long long)blockIdx.y * rows_per_block;
  const long long r1 = r0 + rows_per_block < rows ? r0 + rows_per_block : rows;
  if (cv < CV && lane < rl) {
    float mu[8], is[8];
#pragma unroll
    for (int e = 0; e < 8; ++e) { mu[e] = mean[cv * 8 + e]; is[e] = invstd[cv * 8 + e]; }
    for (long long r = r0 + lane; r < r1; r += rl) {
      float g[8], yy[8], zz[8];
      VecIO<T>::load(dz + r * C + cv * 8, g);
      VecIO<T>::load(y + r * C + cv * 8, yy);
      if (relu) VecIO<T>::load(z + r * C + cv * 8, zz);
#pragma unroll
      for (int e = 0; e < 8; ++e) {
        const float ge = (relu && !(zz[e] > 0.f)) ? 0.f : g[e];       // halo rows: dz == 0
        s1[e] += ge; s2[e] = fmaf(ge, (yy[e] - mu[e]) * is[e], s2[e]);
      }
    }
    const int lc = (threadIdx.x % cvb) * 8;
#pragma unroll
    for (int e = 0; e < 8; ++e) { atomicAdd(&sh[lc + e], s1[e]); atomicAdd(&sh[Cb + lc + e], s2[e]); }
  }
  __syncthreads();
  for (int i = threadIdx.x; i < Cb; i += 256) {
    const int c = blockIdx.x * Cb + i;
    if (c < C) { atomicAdd(&sums[c], sh[i]); atomicAdd(&sums[C + c], sh[Cb + i]); }
  }
}

int launch_bn_bwd_reduce(const void* y, const void* dz, const void* z, int relu, const float* mean, const float* invstd, int dt, long long rows,
                         int C, float* sums, cudaStream_t s) {
  const int CV = C / 8, cvb = CV < 256 ? CV : 256;
  const int bx = ceil_div(CV, cvb);
  long long want = (long long)kSmCount * 8 / bx;
  if (want < 1) want = 1;
  int rpb = (int)((rows + want - 1) / want);
  if (rpb < 64) rpb = 64;
  dim3 grid(bx, (unsigned)((rows + rpb - 1) / rpb));
  YB_DISPATCH16(dt, (k_bn_bwd_reduce<T><<<grid, 256, 2 * cvb * 8 * sizeof(float), s>>>((const T*)y, (const T*)dz, (const T*)z, relu, mean, invstd, rows, C,
                                                                                      rpb, sums)));
  YB_CHECK_LAUNCH();
  return YB_OK;
}

// backward, pass 2:  dy = gamma * invstd * (g - sum_g / N - xhat * sum_gx / N);  dres = g (the residual branch's gradient);
// the (0,0,0) halo threads also publish dgamma = sum_gx, dbeta = sum_g
template <typename T>
__global__ void __launch_bounds__(256) k_bn_bwd_apply(const T* __restrict__ y, const T* __restrict__ dz, const T* __restrict__ z, int relu,
                                                      const float* __restrict__ mean, const float* __restrict__ invstd, const float* __restrict__ gamma,
                                                      const float* __restrict__ sums, float inv_count, T* __restrict__ dy, T* __restrict__ dres,
                                                      float* __restrict__ dgamma, float* __restrict__ dbeta, float gscale, int C, int H) {
  const int Hp = H + 2, CV = C >> 3;
  const int t = blockIdx.x * 256 + threadIdx.x;
  if (t >= Hp * CV) return;
  const int xp = t / CV, cv = t - xp * CV, yp = blockIdx.y, b = blockIdx.z;
  const size_t off = (((size_t)b * Hp + yp) * Hp + xp) * C + cv * 8;
  float o[8], gr[8];
  if (yp == 0 || yp == H + 1 || xp == 0 || xp == H + 1) {
#pragma unroll
    for (int e = 0; e < 8; ++e) { o[e] = 0.f; gr[e] = 0.f; }
    if (yp == 0 && xp == 0 && b == 0) {
#pragma unroll
      for (int e = 0; e < 8; ++e) { dbeta[cv * 8 + e] = gscale * sums[cv * 8 + e]; dgamma[cv * 8 + e] = gscale * sums[C + cv * 8 + e]; }
    }
  } else {
    float g[8], yy[8], zz[8];
    VecIO<T>::load(dz + off, g);
    VecIO<T>::load(y + off, yy);
    if (relu) VecIO<T>::load(z + off, zz);
#pragma unroll
    for (int e = 0; e < 8; ++e) {
      const int c = cv * 8 + e;
      const float ge = (relu && !(zz[e] > 0.f)) ? 0.f : g[e];
      const float xh = (yy[e] - mean[c]) * invstd[c];
      o[e] = gamma[c] * invstd[c] * (ge - sums[c] * inv_count - xh * sums[C + c] * inv_count);
      gr[e] = ge;
    }
  }
  VecIO<T>::store(dy + off, o);
  if (dres) VecIO<T>::store(dres + off, gr);
}

int launch_bn_bwd_apply(const void* y, const void* dz, const void* z, int relu, const float* mean, const float* invstd, const float* gamma,
                        const float* sums, double count, void* dy, void* dres, float* dgamma, float* dbeta, float gscale, int dt, int B, int C, int H,
                        cudaStream_t s) {
  dim3 grid(ceil_div((H + 2) * (C / 8), 256), H + 2, B);
  YB_DISPATCH16(dt, (k_bn_bwd_apply<T><<<grid, 256, 0, s>>>((const T*)y, (const T*)dz, (const T*)z, relu, mean, invstd, gamma, sums, (float)(1.0 / count),
                                                            (T*)dy, (T*)dres, dgamma, dbeta, gscale, C, H)));
  YB_CHECK_LAUNCH();
  return YB_OK;
}

// ------------------------------------------------------------------------------------------------
// transpose a 16-bit [rows][C] matrix into [C][ld] (K-major operands of the weight-gradient GEMM: K = pixels)
// ------------------------------------------------------------------------------------------------
template <typename T>
__global__ void __launch_bounds__(256) k_transpose16(const T* __restrict__ in, int ld_in, T* __restrict__ out, long long rows, int C, long long ld) {
  __shared__ uint16_t tile[64][66];
  const long long r0 = (long long)blockIdx.x * 64;
  const int c0 = blockIdx.y * 64;
  const uint16_t* src = reinterpret_cast<const uint16_t*>(in);
  uint16_t* dst = reinterpret_cast<uint16_t*>(out);
  for (int i = threadIdx.x; i < 64 * 64; i += 256) {
    const int r = i >> 6, c = i & 63;
    uint16_t v = 0;
    if (r0 + r < rows && c0 + c < C) v = src[(r0 + r) * ld_in + c0 + c];
    tile[r][c] = v;
  }
  __syncthreads();
  for (int i = threadIdx.x; i < 64 * 64; i += 256) {
    const int c = i >> 6, r = i & 63;
    if (c0 + c < C && r0 + r < rows) dst[(long long)(c0 + c) * ld + r0 + r] = tile[r][c];
  }
}

int launch_transpose16(const void* in, int ld_in, void* out, int dt, long long rows, int C, long long ld, cudaStream_t s) {
  dim3 grid((unsigned)((rows + 63) / 64), ceil_div(C, 64));
  YB_DISPATCH16(dt, (k_transpose16<T><<<grid, 256, 0, s>>>((const T*)in, ld_in, (T*)out, rows, C, ld)));
  YB_CHECK_LAUNCH();
  return YB_OK;
}

// ------------------------------------------------------------------------------------------------
// element-wise backward helpers on flat 16-bit tensors (n % 8 == 0)
// ------------------------------------------------------------------------------------------------
template <typename T>
__global__ void __launch_bounds__(256) k_relu_bwd(T* __restrict__ dz, const T* __restrict__ z, long long nvec) {
  for (long long i = blockIdx.x * 256LL + threadIdx.x; i < nvec; i += (long long)gridDim.x * 256) {
    float g[8], zz[8];
    VecIO<T>::load(dz + i * 8, g);
    VecIO<T>::load(z + i * 8, zz);
#pragma unroll
    for (int e = 0; e < 8; ++e) g[e] = zz[e] > 0.f ? g[e] : 0.f;
    VecIO<T>::store(dz + i * 8, g);
  }
}

int launch_relu_bwd(void* dz, const void* z, int dt, long long n, cudaStream_t s) {
  const long long nvec = n / 8;
  const int blocks = (int)((nvec + 255) / 256 < kSmCount * 8 ? (nvec + 255) / 256 : kSmCount * 8);
  YB_DISPATCH16(dt, (k_relu_bwd<T><<<blocks > 0 ? blocks : 1, 256, 0, s>>>((T*)dz, (const T*)z, nvec)));
  YB_CHECK_LAUNCH();
  return YB_OK;
}

template <typename T>
__global__ void __launch_bounds__(256) k_add16(T* __restrict__ a, const T* __restrict__ b, long long nvec) {
  for (long long i = blockIdx.x * 256LL + threadIdx.x; i < nvec; i += (long long)gridDim.x * 256) {
    float x[8], y[8];
    VecIO<T>::load(a + i * 8, x);
    VecIO<T>::load(b + i * 8, y);
#pragma unroll
    for (int e = 0; e < 8; ++e) x[e] += y[e];
    VecIO<T>::store(a + i * 8, x);
  }
}

int launch_add16(void* a, const void* b, int dt, long long n, cudaStream_t s) {
  const long long nvec = n / 8;
  const int blocks = (int)((nvec + 255) / 256 < kSmCount * 8 ? (nvec + 255) / 256 : kSmCount * 8);
  YB_DISPATCH16(dt, (k_add16<T><<<blocks > 0 ? blocks : 1, 256, 0, s>>>((T*)a, (const T*)b, nvec)));
  YB_CHECK_LAUNCH();
  return YB_OK;
}

// ------------------------------------------------------------------------------------------------
// max-pool 3x3 s2 p1 backward (gather form): an input pixel receives dy of every window whose FIRST maximum (row-major scan over
// the in-bounds window, strict >: the element torch's max_pool2d records) it is.
// ------------------------------------------------------------------------------------------------
template <typename T>
__global__ void __launch_bounds__(256) k_maxpool_bwd(const T* __restrict__ x, const T* __restrict__ dy, T* __restrict__ dx, int C, int Hin, int Hout) {
  const int Hpi = Hin + 2, Hpo = Hout + 2, CV = C >> 3;
  const int t = blockIdx.x * 256 + threadIdx.x;
  if (t >= Hpi * CV) return;
  const int xp = t / CV, cv = t - xp * CV, yp = blockIdx.y, b = blockIdx.z;
  float acc[8];
#pragma unroll
  for (int e = 0; e < 8; ++e) acc[e] = 0.f;
  if (yp >= 1 && yp <= Hin && xp >= 1 && xp <= Hin) {
    const int iy = yp - 1, ix = xp - 1;
    const T* xb = x + (size_t)b * Hpi * Hpi * C + cv * 8;
    // windows covering row iy: 2*oy-1 <= iy <= 2*oy+1  ->  oy in [ceil((iy-1)/2), floor((iy+1)/2)] = [iy/2, (iy+1)/2]
    const int oya = iy / 2, oyb = (iy + 1) / 2;
    const int oxa = ix / 2, oxb = (ix + 1) / 2;
    for (int oy = oya; oy <= oyb && oy < Hout; ++oy)
      for (int ox = oxa; ox <= oxb && ox < Hout; ++ox) {
        float best[8]; int by[8], bx[8];
#pragma unroll
        for (int e = 0; e < 8; ++e) { best[e] = -INFINITY; by[e] = -1; bx[e] = -1; }
        for (int dy_ = 0; dy_ < 3; ++dy_) {
          const int wy = 2 * oy - 1 + dy_;
          if (wy < 0 || wy >= Hin) continue;
          for (int dx_ = 0; dx_ < 3; ++dx_) {
            const int wx = 2 * ox - 1 + dx_;
            if (wx < 0 || wx >= Hin) continue;
            float v[8];
            VecIO<T>::load(xb + ((size_t)(wy + 1) * Hpi + wx + 1) * C, v);
#pragma unroll
            for (int e = 0; e < 8; ++e) if (v[e] > best[e]) { best[e] = v[e]; by[e] = wy; bx[e] = wx; }
          }
        }
        float g[8];
        VecIO<T>::load(dy + (((size_t)b * Hpo + oy + 1) * Hpo + ox + 1) * C + cv * 8, g);
#pragma unroll
        for (int e = 0; e < 8; ++e) if (by[e] == iy && bx[e] == ix) acc[e] += g[e];
      }
  }
  VecIO<T>::store(dx + (((size_t)b * Hpi + yp) * Hpi + xp) * C + cv * 8, acc);
}

int launch_maxpool_bwd(const void* x, const void* dy, void* dx, int dt, int B, int C, int Hin, int Hout, cudaStream_t s) {
  dim3 grid(ceil_div((Hin + 2) * (C / 8), 256), Hin + 2, B);
  YB_DISPATCH16(dt, (k_maxpool_bwd<T><<<grid, 256, 0, s>>>((const T*)x, (const T*)dy, (T*)dx, C, Hin, Hout)));
  YB_CHECK_LAUNCH();
  return YB_OK;
}

// ------------------------------------------------------------------------------------------------
// bilinear up-sampling backward (transpose of k_bilinear, kernels_simt.cu), gather form over the COARSE grid:
//   dcoarse[iy][ix] (+)= sum over fine (jy, jx) of wy(jy -> iy) * wx(jx -> ix) * dfine[jy][jx]
// with the forward's own index / weight arithmetic (src_index) so that the weights match bit for bit.
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ void src_index_t(int dst, float scale, bool align, int in_size, int& i0, int& i1, float& l0, float& l1) {
  float src = align ? scale * (float)dst : fmaxf(scale * ((float)dst + 0.5f) - 0.5f, 0.f);
  i0 = min((int)src, in_size - 1);
  i1 = min(i0 + 1, in_size - 1);
  l1 = src - (float)i0;
  l0 = 1.f - l1;
}

template <typename T, bool kAlign, bool kAccum>
__global__ void __launch_bounds__(256) k_bilinear_bwd(const T* __restrict__ dfine, T* __restrict__ dcoarse, int C, int Hc, int Hf, float scale) {
  const int Hpc = Hc + 2, Hpf = Hf + 2, CV = C >> 3;
  const int t = blockIdx.x * 256 + threadIdx.x;
  if (t >= Hpc * CV) return;
  const int xp = t / CV, cv = t - xp * CV, yp = blockIdx.y, b = blockIdx.z;
  T* d = dcoarse + (((size_t)b * Hpc + yp) * Hpc + xp) * C + cv * 8;
  float acc[8];
#pragma unroll
  for (int e = 0; e < 8; ++e) acc[e] = 0.f;
  const bool halo = yp == 0 || yp == Hc + 1 || xp == 0 || xp == Hc + 1;
  if (!halo) {
    const int iy = yp - 1, ix = xp - 1;
    const float inv = 1.f / scale;
    int jy0 = (int)floorf(((float)iy - 1.f) * inv) - 2, jy1 = (int)ceilf(((float)iy + 1.f) * inv) + 2;
    int jx0 = (int)floorf(((float)ix - 1.f) * inv) - 2, jx1 = (int)ceilf(((float)ix + 1.f) * inv) + 2;
    jy0 = max(jy0, 0); jx0 = max(jx0, 0); jy1 = min(jy1, Hf - 1); jx1 = min(jx1, Hf - 1);
    const T* fb = dfine + (size_t)b * Hpf * Hpf * C + cv * 8;
    for (int jy = jy0; jy <= jy1; ++jy) {
      int a0, a1; float l0, l1;
      src_index_t(jy, scale, kAlign, Hc, a0, a1, l0, l1);
      const float wy = (a0 == iy ? l0 : 0.f) + (a1 == iy ? l1 : 0.f);
      if (wy == 0.f) continue;
      for (int jx = jx0; jx <= jx1; ++jx) {
        int c0, c1; float m0, m1;
        src_index_t(jx, scale, kAlign, Hc, c0, c1, m0, m1);
        const float wx = (c0 == ix ? m0 : 0.f) + (c1 == ix ? m1 : 0.f);
        if (wx == 0.f) continue;
        float g[8];
        VecIO<T>::load(fb + ((size_t)(jy + 1) * Hpf + jx + 1) * C, g);
        const float w = wy * wx;
#pragma unroll
        for (int e = 0; e < 8; ++e) acc[e] = fmaf(w, g[e], acc[e]);
      }
    }
    if (kAccum) {
      float o[8];
      VecIO<T>::load(d, o);
#pragma unroll
      for (int e = 0; e < 8; ++e) acc[e] += o[e];
    }
  }
  VecIO<T>::store(d, acc);
}

int launch_bilinear_bwd(const void* dfine, void* dcoarse, int dt, int B, int C, int Hc, int Hf, int align_corners, int accumulate, cudaStream_t s) {
  dim3 grid(ceil_div((Hc + 2) * (C / 8), 256), Hc + 2, B);
  const float scale = align_corners ? (Hf > 1 ? (float)(Hc - 1) / (float)(Hf - 1) : 0.f) : (float)Hc / (float)Hf;
  if (align_corners) {
    if (accumulate) YB_DISPATCH16(dt, (k_bilinear_bwd<T, true, true><<<grid, 256, 0, s>>>((const T*)dfine, (T*)dcoarse, C, Hc, Hf, scale)));
    else YB_DISPATCH16(dt, (k_bilinear_bwd<T, true, false><<<grid, 256, 0, s>>>((const T*)dfine, (T*)dcoarse, C, Hc, Hf, scale)));
  } else {
    if (accumulate) YB_DISPATCH16(dt, (k_bilinear_bwd<T, false, true><<<grid, 256, 0, s>>>((const T*)dfine, (T*)dcoarse, C, Hc, Hf, scale)));
    else YB_DISPATCH16(dt, (k_bilinear_bwd<T, false, false><<<grid, 256, 0, s>>>((const T*)dfine, (T*)dcoarse, C, Hc, Hf, scale)));
  }
  YB_CHECK_LAUNCH();
  return YB_OK;
}

// ------------------------------------------------------------------------------------------------
// stride-2 dgrad: gradient parity planes (output geometry) -> gradient of the conv input (inverse of k_phase_split)
// ------------------------------------------------------------------------------------------------
template <typename T>
__global__ void __launch_bounds__(256) k_phase_merge(const T* __restrict__ planes, T* __restrict__ dx, int C, int Hin, int Hout, int nplanes,
                                                     long long plane_stride_rows) {
  const int Hpi = Hin + 2, Hpo = Hout + 2, CV = C >> 3;
  const int t = blockIdx.x * 256 + threadIdx.x;
  if (t >= Hpi * CV) return;
  const int xp = t / CV, cv = t - xp * CV, yp = blockIdx.y, b = blockIdx.z;
  float v[8];
#pragma unroll
  for (int e = 0; e < 8; ++e) v[e] = 0.f;
  if (yp >= 1 && yp <= Hin && xp >= 1 && xp <= Hin) {
    const int iy = yp - 1, ix = xp - 1;
    const int p = iy & 1, q = ix & 1, pl = p * 2 + q;
    if (pl < nplanes) {
      const int py = (iy - p) / 2 + 1, px = (ix - q) / 2 + 1;          // haloed plane coordinates
      VecIO<T>::load(planes + ((size_t)pl * plane_stride_rows + ((size_t)b * Hpo + py) * Hpo + px) * C + cv * 8, v);
    }
  }
  VecIO<T>::store(dx + (((size_t)b * Hpi + yp) * Hpi + xp) * C + cv * 8, v);
}

int launch_phase_merge(const void* planes, void* dx, int dt, int B, int C, int Hin, int Hout, int nplanes, long long plane_stride_rows, cudaStream_t s) {
  dim3 grid(ceil_div((Hin + 2) * (C / 8), 256), Hin + 2, B);
  YB_DISPATCH16(dt, (k_phase_merge<T><<<grid, 256, 0, s>>>((const T*)planes, (T*)dx, C, Hin, Hout, nplanes, plane_stride_rows)));
  YB_CHECK_LAUNCH();
  return YB_OK;
}

// ------------------------------------------------------------------------------------------------
// dense fp32 [B*H*W][lds] (first C columns) -> haloed 16-bit [B][H+2][W+2][C], optionally masked by [act > 0] (ReLU backward) and
// scaled; halo zero.  Feeds the gradients of the fp32 network outputs (prototypes, segmentation logits) into the dgrad / wgrad convs.
// ------------------------------------------------------------------------------------------------
template <typename T>
__global__ void __launch_bounds__(256) k_dense_to_haloed(const float* __restrict__ src, const float* __restrict__ act, int lds, int Csrc, T* __restrict__ dst, int C, int H) {
  const int Hp = H + 2, CV = C >> 3;
  const int t = blockIdx.x * 256 + threadIdx.x;
  if (t >= Hp * CV) return;
  const int xp = t / CV, cv = t - xp * CV, yp = blockIdx.y, b = blockIdx.z;
  float v[8];
#pragma unroll
  for (int e = 0; e < 8; ++e) v[e] = 0.f;
  if (yp >= 1 && yp <= H && xp >= 1 && xp <= H) {
    const size_t r = ((size_t)b * H + yp - 1) * H + xp - 1;
#pragma unroll
    for (int e = 0; e < 8; ++e) {
      const int c = cv * 8 + e;
      if (c >= Csrc) continue;                                      // zero padding columns
      const float g = src[r * lds + c];
      v[e] = (act && !(act[r * lds + c] > 0.f)) ? 0.f : g;
    }
  }
  VecIO<T>::store(dst + (((size_t)b * Hp + yp) * Hp + xp) * C + cv * 8, v);
}

int launch_dense_to_haloed(const float* src, const float* act, int lds, int Csrc, void* dst, int dt, int B, int C, int H, cudaStream_t s) {
  dim3 grid(ceil_div((H + 2) * (C / 8), 256), H + 2, B);
  YB_DISPATCH16(dt, (k_dense_to_haloed<T><<<grid, 256, 0, s>>>(src, act, lds, Csrc, (T*)dst, C, H)));
  YB_CHECK_LAUNCH();
  return YB_OK;
}

// ------------------------------------------------------------------------------------------------
// prediction head, training: raw class logits / box regressions / tanh coefficients scattered to [B, A, .] (no softmax:
// modules/yolact.py:159-161), and the reverse scatter of their gradients into the fused head conv's haloed 16-bit dY
// (columns: conf R*NC | box R*4 | coef R*K | zero pad; dcoef is taken w.r.t. the tanh OUTPUT and multiplied by 1 - tanh^2 here).
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) k_head_train(const float* __restrict__ head, int ld, int HW, int R, int NC, int K, int anchor_offset, int A_total,
                                                    float* __restrict__ cls, float* __restrict__ box, float* __restrict__ coef) {
  const int lane = threadIdx.x & 31;
  const int wi = blockIdx.x * 8 + (threadIdx.x >> 5);
  if (wi >= HW * R) return;
  const int b = blockIdx.y;
  const int pix = wi / R, a = wi - pix * R;
  const float* row = head + ((size_t)b * HW + pix) * ld;
  const size_t arow = (size_t)b * A_total + anchor_offset + (size_t)pix * R + a;
  for (int c = lane; c < NC; c += 32) cls[arow * NC + c] = row[a * NC + c];
  if (lane < 4) box[arow * 4 + lane] = row[R * NC + a * 4 + lane];
  for (int k = lane; k < K; k += 32) coef[arow * K + k] = tanhf(row[R * NC + R * 4 + a * K + k]);
}

int launch_head_train(const float* head, int ld, int B, int HW, int R, int NC, int K, int anchor_offset, int A_total, float* cls, float* box,
                      float* coef, cudaStream_t s) {
  dim3 grid(ceil_div(HW * R, 8), B);
  k_head_train<<<grid, 256, 0, s>>>(head, ld, HW, R, NC, K, anchor_offset, A_total, cls, box, coef);
  YB_CHECK_LAUNCH();
  return YB_OK;
}

template <typename T>
__global__ void __launch_bounds__(256) k_head_grad(const float* __restrict__ dcls, const float* __restrict__ dbox, const float* __restrict__ dcoef,
                                                   const float* __restrict__ coef, int H, int R, int NC, int K, int anchor_offset, int A_total,
                                                   int ldo, T* __restrict__ out) {
  const int Hp = H + 2;
  const int t = blockIdx.x * 256 + threadIdx.x;
  if (t >= Hp * ldo) return;
  const int xp = t / ldo, col = t - xp * ldo, yp = blockIdx.y, b = blockIdx.z;
  float v = 0.f;
  if (yp >= 1 && yp <= H && xp >= 1 && xp <= H) {
    const int pix = (yp - 1) * H + xp - 1;
    const size_t a0 = (size_t)b * A_total + anchor_offset + (size_t)pix * R;
    if (col < R * NC) { const int a = col / NC; v = dcls[(a0 + a) * NC + col - a * NC]; }
    else if (col < R * NC + R * 4) { const int c = col - R * NC, a = c >> 2; v = dbox[(a0 + a) * 4 + (c & 3)]; }
    else if (col < R * (NC + 4 + K)) {
      const int c = col - R * NC - R * 4, a = c / K, k = c - a * K;
      const float th = coef[(a0 + a) * K + k];
      v = dcoef[(a0 + a) * K + k] * (1.f - th * th);
    }
  }
  Act<T>::st(out + (((size_t)b * Hp + yp) * Hp + xp) * ldo + col, v);
}

int launch_head_grad(const float* dcls, const float* dbox, const float* dcoef, const float* coef, int dt, int B, int H, int R, int NC, int K,
                     int anchor_offset, int A_total, int ldo, void* out, cudaStream_t s) {
  dim3 grid(ceil_div((H + 2) * ldo, 256), H + 2, B);
  YB_DISPATCH16(dt, (k_head_grad<T><<<grid, 256, 0, s>>>(dcls, dbox, dcoef, coef, H, R, NC, K, anchor_offset, A_total, ldo, (T*)out)));
  YB_CHECK_LAUNCH();
  return YB_OK;
}

// fp32 vector helpers for the small parameter gradients (biases): dst[i] = scale * src[i]
__global__ void k_scale_copy(const float* __restrict__ src, float* __restrict__ dst, int n, float scale) {
  const int i = blockIdx.x * 256 + threadIdx.x;
  if (i < n) dst[i] = scale * src[i];
}

int launch_scale_copy(const float* src, float* dst, int n, float scale, cudaStream_t s) {
  k_scale_copy<<<ceil_div(n, 256), 256, 0, s>>>(src, dst, n, scale);
  YB_CHECK_LAUNCH();
  return YB_OK;
}

}  // namespace yb
