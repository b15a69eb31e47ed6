// CUDA-core kernels of the Swin-T TRAINING path (modules/swin_transformer.py:62-80, :172-325, :419-518 in train mode; the backward
// passes are derived here -- the reference gets them from torch autograd).  The linear layers are not here: they run as 1x1
// convolutions (forward, dgrad, weight-gradient GEMM, bias sums) on the wgmma kernels of the training engine (train.cu).
//
// Every activation lives on the haloed NHWC token grid of layers.cuh ([B][H+2][H+2][C], 16-bit, halo rows zero).  A kernel that
// produces an activation or a gradient leaves the halo rows at zero, so the weight-gradient GEMMs and bias sums, which run over
// every row, see only the real tokens.  Statistics, softmax, parameters and parameter gradients are fp32; parameter gradients are
// reduced per block and added with atomics to the engine's per-pass zeroed arena.
#include "train.cuh"
#include "vecio.cuh"

#include <math.h>

namespace yb {

#define YB_DISPATCH16(dt, ...)                                           \
  do {                                                                   \
    if ((dt) == DT_BF16) { using T = __nv_bfloat16; __VA_ARGS__; }       \
    else { using T = __half; __VA_ARGS__; }                              \
  } while (0)

namespace {

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

__device__ __forceinline__ bool is_halo(long long row, int H) {
  const int Hp = H + 2;
  const int ti = (int)(row % ((long long)Hp * Hp)), yp = ti / Hp, xp = ti - yp * Hp;
  return yp == 0 || yp == H + 1 || xp == 0 || xp == H + 1;
}

int grid_for(long long units, int per_block) {
  const long long g = (units + per_block - 1) / per_block;
  return (int)(g < kSmCount * 8 ? (g < 1 ? 1 : g) : kSmCount * 8);
}

}  // namespace

// ------------------------------------------------------------------------------------------------
// LayerNorm forward (train): y = (x - mean) * rstd * g + b per token, mean and rstd stored in fp32 for the backward pass.
// One warp per token, two-pass statistics in fp32.  X is the input's element type (fp32 for the patch embedding's conv output).
// ------------------------------------------------------------------------------------------------
template <typename X, typename T>
__global__ void __launch_bounds__(256) k_ln_fwd(const X* __restrict__ x, T* __restrict__ y, const float* __restrict__ g, const float* __restrict__ be,
                                                float* __restrict__ mean, float* __restrict__ rstd, long long rows, int C, int H) {
  const int lane = threadIdx.x & 31;
  for (long long r = (long long)blockIdx.x * 8 + (threadIdx.x >> 5); r < rows; r += (long long)gridDim.x * 8) {
    if (is_halo(r, H)) continue;                                    // halo rows stay zero (the buffer is zeroed once)
    const X* xr = x + r * C;
    float s = 0.f;
    for (int c = lane; c < C; c += 32) s += Act<X>::ld(xr + c);
    const float mu = warp_sum(s) / (float)C;
    float v = 0.f;
    for (int c = lane; c < C; c += 32) { const float d = Act<X>::ld(xr + c) - mu; v += d * d; }
    const float rs = rsqrtf(warp_sum(v) / (float)C + 1e-5f);
    for (int c = lane; c < C; c += 32) Act<T>::st(y + r * C + c, (Act<X>::ld(xr + c) - mu) * rs * g[c] + be[c]);
    if (lane == 0) { mean[r] = mu; rstd[r] = rs; }
  }
}

int launch_ln_fwd(const void* x, int x_f32, void* y, const float* g, const float* be, float* mean, float* rstd, int dt, int B, int C, int H,
                  cudaStream_t s) {
  const long long rows = (long long)B * (H + 2) * (H + 2);
  const int grid = grid_for(rows, 8);
  if (x_f32) YB_DISPATCH16(dt, (k_ln_fwd<float, T><<<grid, 256, 0, s>>>((const float*)x, (T*)y, g, be, mean, rstd, rows, C, H)));
  else YB_DISPATCH16(dt, (k_ln_fwd<T, T><<<grid, 256, 0, s>>>((const T*)x, (T*)y, g, be, mean, rstd, rows, C, H)));
  YB_CHECK_LAUNCH();
  return YB_OK;
}

// ------------------------------------------------------------------------------------------------
// LayerNorm backward: xh = (x - mean) * rstd, dxh = dy * g,
//   dx = rstd * (dxh - mean(dxh) - xh * mean(dxh * xh))   (written, or added to dx when accumulate)
//   dgb[c] += sum dy * xh,  dgb[C + c] += sum dy          (per-block shared sums, then one atomic per channel and block)
// ------------------------------------------------------------------------------------------------
template <typename X, typename T>
__global__ void __launch_bounds__(256) k_ln_bwd(const X* __restrict__ x, const T* __restrict__ dy, const float* __restrict__ g,
                                                const float* __restrict__ mean, const float* __restrict__ rstd, X* __restrict__ dx, int accumulate,
                                                float* __restrict__ dgb, long long rows, int C, int H) {
  extern __shared__ float sh[];                                     // [2C]
  for (int i = threadIdx.x; i < 2 * C; i += 256) sh[i] = 0.f;
  __syncthreads();
  const int lane = threadIdx.x & 31;
  for (long long r = (long long)blockIdx.x * 8 + (threadIdx.x >> 5); r < rows; r += (long long)gridDim.x * 8) {
    if (is_halo(r, H)) continue;
    const X* xr = x + r * C;
    const T* dr = dy + r * C;
    const float mu = mean[r], rs = rstd[r];
    float a = 0.f, b = 0.f;
    for (int c = lane; c < C; c += 32) {
      const float xh = (Act<X>::ld(xr + c) - mu) * rs, d = Act<T>::ld(dr + c), dxh = d * g[c];
      a += dxh; b += dxh * xh;
      atomicAdd(&sh[c], d * xh); atomicAdd(&sh[C + c], d);
    }
    a = warp_sum(a) / (float)C; b = warp_sum(b) / (float)C;
    for (int c = lane; c < C; c += 32) {
      const float xh = (Act<X>::ld(xr + c) - mu) * rs, dxh = Act<T>::ld(dr + c) * g[c];
      float v = rs * (dxh - a - xh * b);
      if (accumulate) v += Act<X>::ld(dx + r * C + c);
      Act<X>::st(dx + r * C + c, v);
    }
  }
  __syncthreads();
  for (int i = threadIdx.x; i < 2 * C; i += 256) atomicAdd(dgb + i, sh[i]);
}

int launch_ln_bwd(const void* x, int x_f32, const void* dy, const float* g, const float* mean, const float* rstd, void* dx, int accumulate, float* dgb,
                  int dt, int B, int C, int H, cudaStream_t s) {
  YB_REQUIRE(C <= 2048, YB_ERR_UNSUPPORTED, "ln_bwd: C=%d", C);
  const long long rows = (long long)B * (H + 2) * (H + 2);
  const int grid = grid_for(rows, 64);                              // 8 tokens per block pass, a few passes per block
  const size_t smem = (size_t)2 * C * 4;
  if (x_f32) YB_DISPATCH16(dt, (k_ln_bwd<float, T><<<grid, 256, smem, s>>>((const float*)x, (const T*)dy, g, mean, rstd, (float*)dx, accumulate, dgb, rows, C, H)));
  else YB_DISPATCH16(dt, (k_ln_bwd<T, T><<<grid, 256, smem, s>>>((const T*)x, (const T*)dy, g, mean, rstd, (T*)dx, accumulate, dgb, rows, C, H)));
  YB_CHECK_LAUNCH();
  return YB_OK;
}

// ------------------------------------------------------------------------------------------------
// Patch embedding conv 4x4 stride 4, 3 -> 96 channels, bias, zero padding past the image edge (modules/swin_transformer.py:419-433),
// fp32 output on the haloed grid (the LayerNorm after it reads fp32).  One warp per token, lane l owns channels l, l+32, l+64.
// w is the parameter as bound: [96][3][4][4], i.e. [96][48] with k = ci*16 + r*4 + q.
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) k_pe_conv(const float* __restrict__ img, const float* __restrict__ w, const float* __restrict__ bias,
                                                 float* __restrict__ out, int B, int S, int Hg) {
  __shared__ float s_w[48 * 96];                                    // [k][co]
  for (int i = threadIdx.x; i < 48 * 96; i += 256) s_w[(i % 48) * 96 + i / 48] = w[i];
  __syncthreads();
  const int lane = threadIdx.x & 31, Hp = Hg + 2;
  const long long rows = (long long)B * Hp * Hp;
  for (long long r = (long long)blockIdx.x * 8 + (threadIdx.x >> 5); r < rows; r += (long long)gridDim.x * 8) {
    if (is_halo(r, Hg)) continue;
    const int b = (int)(r / ((long long)Hp * Hp)), ti = (int)(r % ((long long)Hp * Hp)), yp = ti / Hp, xp = ti - yp * Hp;
    const int y0 = (yp - 1) * 4, x0 = (xp - 1) * 4;
    float a0 = bias[lane], a1 = bias[lane + 32], a2 = bias[lane + 64];
    float in0, in1 = 0.f;
    {
      const int k = lane, ci = k >> 4, rr = (k >> 2) & 3, q = k & 3;
      in0 = (y0 + rr < S && x0 + q < S) ? img[(((size_t)b * 3 + ci) * S + y0 + rr) * S + x0 + q] : 0.f;
      if (lane < 16) {
        const int k2 = lane + 32, c2 = k2 >> 4, r2 = (k2 >> 2) & 3, q2 = k2 & 3;
        in1 = (y0 + r2 < S && x0 + q2 < S) ? img[(((size_t)b * 3 + c2) * S + y0 + r2) * S + x0 + q2] : 0.f;
      }
    }
#pragma unroll
    for (int k = 0; k < 48; ++k) {
      const float v = __shfl_sync(0xffffffffu, k < 32 ? in0 : in1, k & 31);
      a0 = fmaf(v, s_w[k * 96 + lane], a0);
      a1 = fmaf(v, s_w[k * 96 + lane + 32], a1);
      a2 = fmaf(v, s_w[k * 96 + lane + 64], a2);
    }
    float* o = out + r * 96;
    o[lane] = a0; o[lane + 32] = a1; o[lane + 64] = a2;
  }
}

int launch_pe_conv(const float* img, const float* w, const float* bias, float* out, int B, int S, int Hg, cudaStream_t s) {
  k_pe_conv<<<grid_for((long long)B * (Hg + 2) * (Hg + 2), 8), 256, 0, s>>>(img, w, bias, out, B, S, Hg);
  YB_CHECK_LAUNCH();
  return YB_OK;
}

// Patch embedding weight / bias gradient: dW[co][k] += sum_tok dY[tok][co] * patch[tok][k], db[co] += sum_tok dY[tok][co] (no image
// gradient).  A block stages 32 tokens' dY and patches in shared memory; thread t owns the 18 (co, k) pairs t + 256 i.
constexpr int PE_TILE = 32;
__global__ void __launch_bounds__(256) k_pe_wgrad(const float* __restrict__ img, const float* __restrict__ dy, float* __restrict__ dw /*[96*48]*/,
                                                  float* __restrict__ db /*[96]*/, int B, int S, int Hg) {
  __shared__ float s_dy[PE_TILE][96], s_p[PE_TILE][48];
  float acc[18], accb = 0.f;
#pragma unroll
  for (int i = 0; i < 18; ++i) acc[i] = 0.f;
  const long long tokens = (long long)B * Hg * Hg;
  const int Hp = Hg + 2;
  for (long long t0 = (long long)blockIdx.x * PE_TILE; t0 < tokens; t0 += (long long)gridDim.x * PE_TILE) {
    __syncthreads();
    for (int i = threadIdx.x; i < PE_TILE * 96; i += 256) {
      const int tt = i / 96, co = i - tt * 96;
      const long long tok = t0 + tt;
      float v = 0.f;
      if (tok < tokens) {
        const int b = (int)(tok / ((long long)Hg * Hg)), p = (int)(tok % ((long long)Hg * Hg)), yy = p / Hg, xx = p - yy * Hg;
        v = dy[(((long long)b * Hp + yy + 1) * Hp + xx + 1) * 96 + co];
      }
      s_dy[tt][co] = v;
    }
    for (int i = threadIdx.x; i < PE_TILE * 48; i += 256) {
      const int tt = i / 48, k = i - tt * 48;
      const long long tok = t0 + tt;
      float v = 0.f;
      if (tok < tokens) {
        const int b = (int)(tok / ((long long)Hg * Hg)), p = (int)(tok % ((long long)Hg * Hg)), yy = p / Hg, xx = p - yy * Hg;
        const int ci = k >> 4, r = (k >> 2) & 3, q = k & 3, iy = yy * 4 + r, ix = xx * 4 + q;
        if (iy < S && ix < S) v = img[(((size_t)b * 3 + ci) * S + iy) * S + ix];
      }
      s_p[tt][k] = v;
    }
    __syncthreads();
#pragma unroll
    for (int i = 0; i < 18; ++i) {
      const int idx = threadIdx.x + 256 * i, co = idx / 48, k = idx - co * 48;
      float a = acc[i];
      for (int tt = 0; tt < PE_TILE; ++tt) a = fmaf(s_dy[tt][co], s_p[tt][k], a);
      acc[i] = a;
    }
    if (threadIdx.x < 96)
      for (int tt = 0; tt < PE_TILE; ++tt) accb += s_dy[tt][threadIdx.x];
  }
#pragma unroll
  for (int i = 0; i < 18; ++i) atomicAdd(dw + threadIdx.x + 256 * i, acc[i]);
  if (threadIdx.x < 96) atomicAdd(db + threadIdx.x, accb);
}

int launch_pe_wgrad(const float* img, const float* dy, float* dw, float* db, int B, int S, int Hg, cudaStream_t s) {
  k_pe_wgrad<<<grid_for((long long)B * Hg * Hg, 4 * PE_TILE), 256, 0, s>>>(img, dy, dw, db, B, S, Hg);
  YB_CHECK_LAUNCH();
  return YB_OK;
}

// ------------------------------------------------------------------------------------------------
// (Shifted-)window attention, train forward and backward (modules/swin_transformer.py:172-200, :234-289, mask :369-387).
// One block per (window, head, image), thread i = window token i.  Window tokens are addressed as k_window_attention does: rolled
// frame -> original (padded-grid) coordinates by index arithmetic, region ids for the -100 mask.  Grid padding tokens (the grid is
// padded to a multiple of 7 AFTER norm1 and BEFORE qkv, :246-253) have qkv == the qkv bias and take part as keys and values.
//   forward   out[row][head*32 + d] for real tokens, lse[row * nH + head] = log-sum-exp of the token's scores
//   backward  recomputes P from Q, K and the log-sum-exp;  D_i = sum_j P_ij dP_ij,  dP = dO V^T,  dS = P o (dP - D),
//             dQ = scale dS K,  dK = scale dS^T Q,  dV = P^T dO  into dqkv (rows of real tokens);  the padding tokens' dK / dV go to
//             the qkv bias gradient (dbias, atomics);  the relative-position table gradient is reduced in shared memory per block
// ------------------------------------------------------------------------------------------------
constexpr int WS = 7, WT = 49, HD = 32;
constexpr float kAttnScale = 0.17677669529663687f;                  // 32^-0.5

__device__ __forceinline__ void window_tokens(int win, int b, int H, int shift, int* s_row, int* s_reg) {
  const int Hpad = (H + WS - 1) / WS * WS, nW = Hpad / WS, Hp = H + 2;
  const int wy = win / nW, wx = win - wy * nW;
  for (int t = threadIdx.x; t < WT; t += blockDim.x) {
    const int iy = t / WS, ix = t - iy * WS;
    const int ys = wy * WS + iy, xs = wx * WS + ix;
    const int yo = (ys + shift) % Hpad, xo = (xs + shift) % Hpad;
    s_row[t] = (yo < H && xo < H) ? ((b * Hp + yo + 1) * Hp + xo + 1) : -1;
    const int ry = ys < Hpad - WS ? 0 : (ys < Hpad - shift ? 1 : 2), rx = xs < Hpad - WS ? 0 : (xs < Hpad - shift ? 1 : 2);
    s_reg[t] = ry * 3 + rx;
  }
}

__device__ __forceinline__ int rel_idx(int i, int j) {
  const int iy = i / WS, ix = i - iy * WS, jy = j / WS, jx = j - jy * WS;
  return (iy - jy + WS - 1) * (2 * WS - 1) + (ix - jx + WS - 1);
}

template <typename T>
__device__ __forceinline__ void load_qkv_window(const T* qkv, const float* qkv_bias, const int* s_row, int C, int head, float (*s_q)[HD],
                                                float (*s_k)[HD], float (*s_v)[HD]) {
  const int C3 = 3 * C;
  for (int e = threadIdx.x; e < WT * HD; e += blockDim.x) {
    const int t = e / HD, d = e - t * HD, row = s_row[t];
    const int c = head * HD + d;
    if (row >= 0) {
      const T* p = qkv + (size_t)row * C3;
      if (s_q) s_q[t][d] = Act<T>::ld(p + c);
      s_k[t][d] = Act<T>::ld(p + C + c); s_v[t][d] = Act<T>::ld(p + 2 * C + c);
    } else {
      if (s_q) s_q[t][d] = qkv_bias[c];
      s_k[t][d] = qkv_bias[C + c]; s_v[t][d] = qkv_bias[2 * C + c];
    }
  }
}

template <typename T>
__global__ void __launch_bounds__(64) k_wattn_fwd(const T* __restrict__ qkv, const float* __restrict__ qkv_bias, const float* __restrict__ table,
                                                  T* __restrict__ out, float* __restrict__ lse, int H, int C, int nH, int shift) {
  __shared__ __align__(16) float s_k[WT][HD], s_v[WT][HD];
  __shared__ int s_row[WT], s_reg[WT];
  const int head = blockIdx.y, b = blockIdx.z, tid = threadIdx.x;
  window_tokens(blockIdx.x, b, H, shift, s_row, s_reg);
  __syncthreads();
  load_qkv_window<T>(qkv, qkv_bias, s_row, C, head, nullptr, s_k, s_v);
  __syncthreads();
  if (tid >= WT) return;
  const int row = s_row[tid];
  if (row < 0) return;                                              // padding tokens are cropped away (:283)
  float q[HD];
#pragma unroll
  for (int d = 0; d < HD; ++d) q[d] = Act<T>::ld(qkv + (size_t)row * 3 * C + head * HD + d) * kAttnScale;
  float sc[WT], mx = -INFINITY;
#pragma unroll
  for (int j = 0; j < WT; ++j) {
    float a = 0.f;
#pragma unroll
    for (int d = 0; d < HD; ++d) a = fmaf(q[d], s_k[j][d], a);
    a += table[rel_idx(tid, j) * nH + head];
    if (shift > 0 && s_reg[j] != s_reg[tid]) a += -100.f;
    sc[j] = a;
    mx = fmaxf(mx, a);
  }
  float sum = 0.f;
#pragma unroll
  for (int j = 0; j < WT; ++j) { sc[j] = expf(sc[j] - mx); sum += sc[j]; }
  const float inv = 1.f / sum;
  float o[HD];
#pragma unroll
  for (int d = 0; d < HD; ++d) o[d] = 0.f;
#pragma unroll
  for (int j = 0; j < WT; ++j) {
    const float p = sc[j] * inv;
#pragma unroll
    for (int d = 0; d < HD; ++d) o[d] = fmaf(p, s_v[j][d], o[d]);
  }
#pragma unroll
  for (int d = 0; d < HD; ++d) Act<T>::st(out + (size_t)row * C + head * HD + d, o[d]);
  lse[(size_t)row * nH + head] = mx + logf(sum);
}

template <typename T>
__global__ void __launch_bounds__(64) k_wattn_bwd(const T* __restrict__ qkv, const float* __restrict__ qkv_bias, const float* __restrict__ table,
                                                  const T* __restrict__ dout, const float* __restrict__ lse, T* __restrict__ dqkv,
                                                  float* __restrict__ dtable, float* __restrict__ dbias, int H, int C, int nH, int shift) {
  __shared__ float s_q[WT][HD], s_k[WT][HD], s_v[WT][HD], s_do[WT][HD];
  __shared__ float s_p[WT][WT], s_ds[WT][WT];
  __shared__ float s_tab[169];
  __shared__ int s_row[WT], s_reg[WT];
  const int head = blockIdx.y, b = blockIdx.z, tid = threadIdx.x, C3 = 3 * C;
  window_tokens(blockIdx.x, b, H, shift, s_row, s_reg);
  for (int i = tid; i < 169; i += 64) s_tab[i] = 0.f;
  __syncthreads();
  load_qkv_window<T>(qkv, qkv_bias, s_row, C, head, s_q, s_k, s_v);
  for (int e = tid; e < WT * HD; e += 64) {
    const int t = e / HD, d = e - t * HD, row = s_row[t];
    s_do[t][d] = row >= 0 ? Act<T>::ld(dout + (size_t)row * C + head * HD + d) : 0.f;
  }
  __syncthreads();
  if (tid < WT) {
    const int i = tid, row = s_row[i];
    if (row < 0) {                                                  // a cropped padding query: no output, no gradient
      for (int j = 0; j < WT; ++j) { s_p[i][j] = 0.f; s_ds[i][j] = 0.f; }
    } else {
      const float l = lse[(size_t)row * nH + head];
      float D = 0.f;
      for (int j = 0; j < WT; ++j) {
        float a = 0.f, dp = 0.f;
#pragma unroll
        for (int d = 0; d < HD; ++d) { a = fmaf(s_q[i][d] * kAttnScale, s_k[j][d], a); dp = fmaf(s_do[i][d], s_v[j][d], dp); }
        a += table[rel_idx(i, j) * nH + head];
        if (shift > 0 && s_reg[j] != s_reg[i]) a += -100.f;
        const float p = expf(a - l);
        s_p[i][j] = p; s_ds[i][j] = dp;
        D = fmaf(p, dp, D);
      }
      float dq[HD];
#pragma unroll
      for (int d = 0; d < HD; ++d) dq[d] = 0.f;
      for (int j = 0; j < WT; ++j) {
        const float ds = s_p[i][j] * (s_ds[i][j] - D);
        s_ds[i][j] = ds;
        atomicAdd(&s_tab[rel_idx(i, j)], ds);
#pragma unroll
        for (int d = 0; d < HD; ++d) dq[d] = fmaf(ds, s_k[j][d], dq[d]);
      }
#pragma unroll
      for (int d = 0; d < HD; ++d) Act<T>::st(dqkv + (size_t)row * C3 + head * HD + d, dq[d] * kAttnScale);
    }
  }
  __syncthreads();
  if (tid < WT) {
    const int j = tid, row = s_row[j];
    float dk[HD], dv[HD];
#pragma unroll
    for (int d = 0; d < HD; ++d) { dk[d] = 0.f; dv[d] = 0.f; }
    for (int i = 0; i < WT; ++i) {
      const float p = s_p[i][j], ds = s_ds[i][j];
#pragma unroll
      for (int d = 0; d < HD; ++d) { dv[d] = fmaf(p, s_do[i][d], dv[d]); dk[d] = fmaf(ds, s_q[i][d], dk[d]); }
    }
    if (row >= 0) {
#pragma unroll
      for (int d = 0; d < HD; ++d) {
        Act<T>::st(dqkv + (size_t)row * C3 + C + head * HD + d, dk[d] * kAttnScale);
        Act<T>::st(dqkv + (size_t)row * C3 + 2 * C + head * HD + d, dv[d]);
      }
    } else {                                                        // padding key / value = the qkv bias: its gradient
#pragma unroll
      for (int d = 0; d < HD; ++d) {
        atomicAdd(dbias + C + head * HD + d, dk[d] * kAttnScale);
        atomicAdd(dbias + 2 * C + head * HD + d, dv[d]);
      }
    }
  }
  for (int i = tid; i < 169; i += 64) atomicAdd(dtable + i * nH + head, s_tab[i]);
}

int launch_wattn_fwd(const void* qkv, const float* qkv_bias, const float* table, void* out, float* lse, int dt, int B, int H, int C, int nH, int shift,
                     cudaStream_t s) {
  YB_REQUIRE(C == nH * HD, YB_ERR_UNSUPPORTED, "wattn_fwd: head_dim must be 32 (C=%d heads=%d)", C, nH);
  const int nW = (H + WS - 1) / WS;
  dim3 grid(nW * nW, nH, B);
  YB_DISPATCH16(dt, (k_wattn_fwd<T><<<grid, 64, 0, s>>>((const T*)qkv, qkv_bias, table, (T*)out, lse, H, C, nH, shift)));
  YB_CHECK_LAUNCH();
  return YB_OK;
}

int launch_wattn_bwd(const void* qkv, const float* qkv_bias, const float* table, const void* dout, const float* lse, void* dqkv, float* dtable,
                     float* dbias, int dt, int B, int H, int C, int nH, int shift, cudaStream_t s) {
  YB_REQUIRE(C == nH * HD, YB_ERR_UNSUPPORTED, "wattn_bwd: head_dim must be 32 (C=%d heads=%d)", C, nH);
  const int nW = (H + WS - 1) / WS;
  dim3 grid(nW * nW, nH, B);
  YB_DISPATCH16(dt, (k_wattn_bwd<T><<<grid, 64, 0, s>>>((const T*)qkv, qkv_bias, table, (const T*)dout, lse, (T*)dqkv, dtable, dbias, H, C, nH, shift)));
  YB_CHECK_LAUNCH();
  return YB_OK;
}

// ------------------------------------------------------------------------------------------------
// exact-erf GELU on the stored pre-activation (fc1's output): forward y = h Phi(h), backward dh = dy (Phi(h) + h phi(h))
// ------------------------------------------------------------------------------------------------
template <typename T>
__global__ void k_gelu_fwd(const T* __restrict__ h, T* __restrict__ y, long long n) {
  for (long long i = blockIdx.x * 256LL + threadIdx.x; i < n; i += (long long)gridDim.x * 256) {
    const float v = Act<T>::ld(h + i);
    Act<T>::st(y + i, 0.5f * v * (1.f + erff(v * 0.70710678118654752f)));
  }
}

template <typename T>
__global__ void k_gelu_bwd(const T* __restrict__ h, const T* __restrict__ dy, T* __restrict__ dh, long long n) {
  for (long long i = blockIdx.x * 256LL + threadIdx.x; i < n; i += (long long)gridDim.x * 256) {
    const float v = Act<T>::ld(h + i);
    const float cdf = 0.5f * (1.f + erff(v * 0.70710678118654752f)), pdf = 0.39894228040143268f * expf(-0.5f * v * v);
    Act<T>::st(dh + i, Act<T>::ld(dy + i) * (cdf + v * pdf));
  }
}

int launch_gelu_fwd(const void* h, void* y, int dt, long long n, cudaStream_t s) {
  YB_DISPATCH16(dt, (k_gelu_fwd<T><<<grid_for(n, 256 * 4), 256, 0, s>>>((const T*)h, (T*)y, n)));
  YB_CHECK_LAUNCH();
  return YB_OK;
}

int launch_gelu_bwd(const void* h, const void* dy, void* dh, int dt, long long n, cudaStream_t s) {
  YB_DISPATCH16(dt, (k_gelu_bwd<T><<<grid_for(n, 256 * 4), 256, 0, s>>>((const T*)h, (const T*)dy, (T*)dh, n)));
  YB_CHECK_LAUNCH();
  return YB_OK;
}

// ------------------------------------------------------------------------------------------------
// Patch merging gather (modules/swin_transformer.py:299-325): output token (y, x) = [x0 | x1 | x2 | x3] with parts (0,0), (1,0),
// (0,1), (1,1) = input tokens (2y + (part & 1), 2x + (part >> 1)), zero beyond an odd edge.  The LayerNorm(4C) after it is
// k_ln_fwd.  The backward is the inverse gather over the input tokens: no atomics; the padding positions receive nothing.
// ------------------------------------------------------------------------------------------------
template <typename T>
__global__ void k_merge_fwd(const T* __restrict__ in, T* __restrict__ out, int B, int C, int Hin, int Hout) {
  const int Hpi = Hin + 2, Hpo = Hout + 2, C4 = 4 * C;
  const long long n = (long long)B * Hout * Hout * C4;
  for (long long i = blockIdx.x * 256LL + threadIdx.x; i < n; i += (long long)gridDim.x * 256) {
    const int c4 = (int)(i % C4);
    const long long tok = i / C4;
    const int b = (int)(tok / ((long long)Hout * Hout)), p = (int)(tok % ((long long)Hout * Hout)), y = p / Hout, x = p - y * Hout;
    const int part = c4 / C, c = c4 - part * C, iy = 2 * y + (part & 1), ix = 2 * x + (part >> 1);
    const float v = (iy < Hin && ix < Hin) ? Act<T>::ld(in + (((long long)b * Hpi + iy + 1) * Hpi + ix + 1) * C + c) : 0.f;
    Act<T>::st(out + (((long long)b * Hpo + y + 1) * Hpo + x + 1) * C4 + c4, v);
  }
}

template <typename T>
__global__ void k_merge_bwd(const T* __restrict__ dout, T* __restrict__ dx, int accumulate, int B, int C, int Hin, int Hout) {
  const int Hpi = Hin + 2, Hpo = Hout + 2, C4 = 4 * C;
  const long long n = (long long)B * Hin * Hin * C;
  for (long long i = blockIdx.x * 256LL + threadIdx.x; i < n; i += (long long)gridDim.x * 256) {
    const int c = (int)(i % C);
    const long long tok = i / C;
    const int b = (int)(tok / ((long long)Hin * Hin)), p = (int)(tok % ((long long)Hin * Hin)), iy = p / Hin, ix = p - iy * Hin;
    const int part = (iy & 1) + 2 * (ix & 1);
    const long long di = (((long long)b * Hpi + iy + 1) * Hpi + ix + 1) * C + c;
    float v = Act<T>::ld(dout + (((long long)b * Hpo + (iy >> 1) + 1) * Hpo + (ix >> 1) + 1) * C4 + part * C + c);
    if (accumulate) v += Act<T>::ld(dx + di);
    Act<T>::st(dx + di, v);
  }
}

int launch_merge_fwd(const void* in, void* out, int dt, int B, int C, int Hin, int Hout, cudaStream_t s) {
  YB_DISPATCH16(dt, (k_merge_fwd<T><<<grid_for((long long)B * Hout * Hout * 4 * C, 256 * 4), 256, 0, s>>>((const T*)in, (T*)out, B, C, Hin, Hout)));
  YB_CHECK_LAUNCH();
  return YB_OK;
}

int launch_merge_bwd(const void* dout, void* dx, int accumulate, int dt, int B, int C, int Hin, int Hout, cudaStream_t s) {
  YB_DISPATCH16(dt, (k_merge_bwd<T><<<grid_for((long long)B * Hin * Hin * C, 256 * 4), 256, 0, s>>>((const T*)dout, (T*)dx, accumulate, B, C, Hin, Hout)));
  YB_CHECK_LAUNCH();
  return YB_OK;
}

// ------------------------------------------------------------------------------------------------
// Stochastic depth (modules/swin_transformer.py:62-80, rates :464).  Block i (of kSwinBlocks, over all stages) drops each branch
// with p_i = 0.2 i / 11; per image and branch the mask is floor(keep + U), U uniform in [0, 1) from a counter hash of the step's
// seed (in device memory: a replayed graph draws anew).  The salt keeps these draws apart from the mask subset's (losses.cu).
// masks: [B][kSwinBlocks][2] (attention, MLP).  Distribution-equal to the reference's torch.rand, not stream-equal.
// ------------------------------------------------------------------------------------------------
__global__ void k_drop_path_masks(const uint32_t* __restrict__ seed_dev, float* __restrict__ masks, int B) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= B * kSwinBlocks * 2) return;
  const int blk = (i / 2) % kSwinBlocks;
  const float keep = 1.f - swin_drop_rate(blk);
  const uint32_t u = hash32(seed_dev[0] ^ hash32(0x5d2f1a97u + (uint32_t)i));
  masks[i] = floorf(keep + (float)(u >> 8) * (1.f / 16777216.f));
}

int launch_drop_path_masks(const uint32_t* seed_dev, float* masks, int B, cudaStream_t s) {
  k_drop_path_masks<<<ceil_div(B * kSwinBlocks * 2, 128), 128, 0, s>>>(seed_dev, masks, B);
  YB_CHECK_LAUNCH();
  return YB_OK;
}

// residual with the branch's mask: out = x + m / keep * y  (per image; the halo rows of x and y are zero, so are out's);
// backward: dx (+)= dout, dy = m / keep * dout
template <typename T>
__global__ void k_drop_residual(const T* __restrict__ x, const T* __restrict__ y, T* __restrict__ out, const float* __restrict__ masks, int mi,
                                float inv_keep, long long per_img, long long n) {
  for (long long i = blockIdx.x * 256LL + threadIdx.x; i < n; i += (long long)gridDim.x * 256) {
    const float m = masks[(i / per_img) * kSwinBlocks * 2 + mi] * inv_keep;
    Act<T>::st(out + i, Act<T>::ld(x + i) + m * Act<T>::ld(y + i));
  }
}

template <typename T>
__global__ void k_drop_residual_bwd(const T* __restrict__ dout, T* __restrict__ dx, int accumulate, T* __restrict__ dy, const float* __restrict__ masks,
                                    int mi, float inv_keep, long long per_img, long long n) {
  for (long long i = blockIdx.x * 256LL + threadIdx.x; i < n; i += (long long)gridDim.x * 256) {
    const float m = masks[(i / per_img) * kSwinBlocks * 2 + mi] * inv_keep, d = Act<T>::ld(dout + i);
    Act<T>::st(dx + i, accumulate ? Act<T>::ld(dx + i) + d : d);
    Act<T>::st(dy + i, m * d);
  }
}

int launch_drop_residual(const void* x, const void* y, void* out, const float* masks, int blk, int branch, int dt, int B, long long per_img,
                         cudaStream_t s) {
  const long long n = (long long)B * per_img;
  const float inv_keep = 1.f / (1.f - swin_drop_rate(blk));
  YB_DISPATCH16(dt, (k_drop_residual<T><<<grid_for(n, 256 * 4), 256, 0, s>>>((const T*)x, (const T*)y, (T*)out, masks, blk * 2 + branch, inv_keep, per_img, n)));
  YB_CHECK_LAUNCH();
  return YB_OK;
}

int launch_drop_residual_bwd(const void* dout, void* dx, int accumulate, void* dy, const float* masks, int blk, int branch, int dt, int B,
                             long long per_img, cudaStream_t s) {
  const long long n = (long long)B * per_img;
  const float inv_keep = 1.f / (1.f - swin_drop_rate(blk));
  YB_DISPATCH16(dt, (k_drop_residual_bwd<T><<<grid_for(n, 256 * 4), 256, 0, s>>>((const T*)dout, (T*)dx, accumulate, (T*)dy, masks, blk * 2 + branch,
                                                                                   inv_keep, per_img, n)));
  YB_CHECK_LAUNCH();
  return YB_OK;
}

}  // namespace yb
