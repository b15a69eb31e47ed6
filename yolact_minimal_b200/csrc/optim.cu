// The optimizer step of the training loop as one launch over every parameter: torch's foreach SGD (momentum, L2 weight decay) and
// AdamW (decoupled weight decay) on CUDA, restated element by element.  Each torch foreach kernel rounds its result to fp32 and
// stores it; the fused kernel keeps the same roundings with explicit _rn intrinsics, so nvcc cannot contract two of torch's
// separate kernels into one FMA.  Where one torch kernel computes `a + s * b` (foreach add with alpha, lerp, addcmul, addcdiv),
// torch's nvcc build contracts it to fma(s, b, a), and so does this file (DESIGN.md §13).
//
// Layout: the gradient is one flat fp32 buffer, the parameters concatenated in the order given to yb_optim_create.  The
// optimizer's state mirrors it tensor by tensor, but each tensor's state starts at the same 16-byte phase as the parameter, so
// parameter and state are read and written with float4 accesses together; the gradient is read as float4 wherever its own
// offset allows it and as four scalars elsewhere.  The few elements before the parameter's first 16-byte boundary and after its
// last one are scalar.  Nothing outside [p, p + count) of each parameter is touched.
#include "common.cuh"

#include <math.h>
#include <algorithm>
#include <vector>

struct yb_optim {
  int kind = 0;
  double momentum = 0, weight_decay = 0, beta1 = 0, beta2 = 0, eps = 0;
  int device = 0;
  int64_t total = 0;                   // gradient elements
  int64_t step = 0;                    // steps taken (torch's state['step'])
  int num_chunks = 0;
  float* state0 = nullptr;             // SGD momentum buffer | AdamW exp_avg
  float* state1 = nullptr;             // AdamW exp_avg_sq
  void* chunks = nullptr;              // OptimChunk[num_chunks] (device)
  std::vector<int64_t> soffs, counts;  // per parameter: state offset, elements
};

namespace yb {

struct OptimChunk {
  float* p;                            // first parameter element of the chunk
  int64_t g;                           // its offset in the flat gradient
  int64_t s;                           // its offset in the state buffers
  int n;                               // elements
  int pad_;
};
constexpr int kOptimChunk = 4096;      // elements per CTA: 4 float4 per thread of 256
constexpr int kOptimThreads = 256;

struct OptimScalars {                  // computed on the host in double, as torch computes them, and rounded to fp32 once
  float wd, momentum, neg_lr;          // SGD
  float decay, w1, beta2, c2, bc2_sqrt, eps, step_size;   // AdamW
  float grad_scale;
  int first, use_wd;
};

template <int KIND>
__device__ __forceinline__ void optim_elem(float& p, float g, float& m, float& v, const OptimScalars& c) {
  g = __fmul_rn(g, c.grad_scale);
  if (KIND == YB_OPTIM_SGD) {
    if (c.use_wd) g = __fmaf_rn(c.wd, p, g);                              // _foreach_add(grads, params, alpha=wd)
    m = c.first ? g : __fadd_rn(__fmul_rn(m, c.momentum), g);            // clone | _foreach_mul_ then _foreach_add_(alpha=1)
    p = __fmaf_rn(c.neg_lr, m, p);                                      // _foreach_add_(params, bufs, alpha=-lr)
  } else {
    p = __fmul_rn(p, c.decay);                                          // _foreach_mul_(params, 1 - lr * wd)
    m = __fmaf_rn(c.w1, __fsub_rn(g, m), m);                             // _foreach_lerp_(exp_avgs, grads, 1 - beta1), weight < 0.5
    v = __fmaf_rn(c.c2, __fmul_rn(g, g), __fmul_rn(v, c.beta2));         // _foreach_mul_(beta2), _foreach_addcmul_(g, g, 1 - beta2)
    const float d = __fadd_rn(__fdiv_rn(__fsqrt_rn(v), c.bc2_sqrt), c.eps);   // sqrt, _foreach_div_(bc2_sqrt), _foreach_add_(eps)
    p = __fmaf_rn(c.step_size, __fdiv_rn(m, d), p);                     // _foreach_addcdiv_(params, exp_avgs, denom, step_size)
  }
}

template <int KIND>
__global__ void __launch_bounds__(kOptimThreads) k_optim_step(const OptimChunk* __restrict__ chunks, const float* __restrict__ grad,
                                                              float* __restrict__ s0, float* __restrict__ s1, OptimScalars c) {
  const OptimChunk ck = chunks[blockIdx.x];
  float* p = ck.p;
  const float* g = grad + ck.g;
  float* m = s0 + ck.s;
  float* v = KIND == YB_OPTIM_ADAMW ? s1 + ck.s : m;
  const int head = min(ck.n, (int)(((16 - ((uintptr_t)p & 15)) & 15) >> 2));
  const int nq = (ck.n - head) >> 2;
  const int tail = head + 4 * nq;
  const int t = threadIdx.x;
  if (t < head || (t >= 4 && t - 4 < ck.n - tail)) {                     // threads 0-2: head, 4-6: tail
    const int i = t < head ? t : tail + t - 4;
    float pv = p[i], mv = m[i], vv = KIND == YB_OPTIM_ADAMW ? v[i] : 0.f;
    optim_elem<KIND>(pv, g[i], mv, vv, c);
    p[i] = pv; m[i] = mv;
    if (KIND == YB_OPTIM_ADAMW) v[i] = vv;
  }
  const bool g_vec = ((uintptr_t)(g + head) & 15) == 0;
  for (int q = t; q < nq; q += kOptimThreads) {
    const int i = head + 4 * q;
    float4 pv = *reinterpret_cast<const float4*>(p + i);
    float4 mv = *reinterpret_cast<const float4*>(m + i);
    float4 vv = KIND == YB_OPTIM_ADAMW ? *reinterpret_cast<const float4*>(v + i) : make_float4(0.f, 0.f, 0.f, 0.f);
    const float4 gv = g_vec ? __ldg(reinterpret_cast<const float4*>(g + i)) : make_float4(__ldg(g + i), __ldg(g + i + 1), __ldg(g + i + 2), __ldg(g + i + 3));
    optim_elem<KIND>(pv.x, gv.x, mv.x, vv.x, c);
    optim_elem<KIND>(pv.y, gv.y, mv.y, vv.y, c);
    optim_elem<KIND>(pv.z, gv.z, mv.z, vv.z, c);
    optim_elem<KIND>(pv.w, gv.w, mv.w, vv.w, c);
    *reinterpret_cast<float4*>(p + i) = pv;
    *reinterpret_cast<float4*>(m + i) = mv;
    if (KIND == YB_OPTIM_ADAMW) *reinterpret_cast<float4*>(v + i) = vv;
  }
}

}  // namespace yb

using namespace yb;

extern "C" {

YB_API void yb_optim_destroy(yb_optim* o) {
  if (!o) return;
  int prev = 0;
  cudaGetDevice(&prev);
  cudaSetDevice(o->device);
  cudaFree(o->state0);
  cudaFree(o->state1);
  cudaFree(o->chunks);
  cudaSetDevice(prev);
  delete o;
}

YB_API int yb_optim_create(const yb_optim_params* hp, int n, float* const* params_device, const int64_t* counts, yb_optim** out) {
  YB_REQUIRE(hp && params_device && counts && out && n > 0, YB_ERR_INVALID, "yb_optim_create: null argument or no parameters");
  *out = nullptr;
  YB_REQUIRE(hp->kind == YB_OPTIM_SGD || hp->kind == YB_OPTIM_ADAMW, YB_ERR_INVALID, "yb_optim_create: unknown kind %d", hp->kind);
  YB_REQUIRE(hp->weight_decay >= 0, YB_ERR_INVALID, "yb_optim_create: weight_decay %g < 0", hp->weight_decay);
  if (hp->kind == YB_OPTIM_SGD) {
    YB_REQUIRE(hp->momentum > 0 && hp->dampening == 0, YB_ERR_UNSUPPORTED,
               "yb_optim_create: SGD needs momentum > 0 and dampening 0 (got %g, %g)", hp->momentum, hp->dampening);
  } else {
    // beta1 > 0.5 keeps the lerp weight 1 - beta1 below 0.5, the branch of torch's lerp the kernel restates
    YB_REQUIRE(hp->beta1 > 0.5 && hp->beta1 < 1 && hp->beta2 >= 0 && hp->beta2 < 1 && hp->eps >= 0, YB_ERR_UNSUPPORTED,
               "yb_optim_create: AdamW needs 0.5 < beta1 < 1, 0 <= beta2 < 1 and eps >= 0 (got %g, %g, %g)", hp->beta1, hp->beta2,
               hp->eps);
  }
  std::vector<OptimChunk> chunks;
  std::vector<int64_t> o_soffs, o_counts;
  int64_t goff = 0, soff = 0;
  for (int i = 0; i < n; ++i) {
    float* p = params_device[i];
    const int64_t cnt = counts[i];
    YB_REQUIRE(p && cnt > 0, YB_ERR_INVALID, "yb_optim_create: parameter %d is null or empty", i);
    YB_REQUIRE(((uintptr_t)p & 3) == 0, YB_ERR_INVALID, "yb_optim_create: parameter %d is not 4-byte aligned", i);
    const int phase = (int)(((uintptr_t)p >> 2) & 3);                    // the state starts at the parameter's 16-byte phase
    soff += (phase - soff % 4 + 4) % 4;
    const int64_t head = std::min<int64_t>(cnt, (4 - phase) % 4);
    for (int64_t a = 0; a < cnt;) {
      const int64_t len = std::min<int64_t>(cnt - a, a == 0 ? head + kOptimChunk : kOptimChunk);
      chunks.push_back(OptimChunk{p + a, goff + a, soff + a, (int)len, 0});
      a += len;
    }
    o_soffs.push_back(soff);
    o_counts.push_back(cnt);
    goff += cnt;
    soff += cnt;
  }
  YB_REQUIRE(chunks.size() < (1u << 31), YB_ERR_UNSUPPORTED, "yb_optim_create: too many parameters");
  yb_optim* o = new yb_optim();
  o->kind = hp->kind;
  o->momentum = hp->momentum;
  o->weight_decay = hp->weight_decay;
  o->beta1 = hp->beta1;
  o->beta2 = hp->beta2;
  o->eps = hp->eps;
  o->total = goff;
  o->num_chunks = (int)chunks.size();
  o->soffs = std::move(o_soffs);
  o->counts = std::move(o_counts);
  cudaError_t e = cudaGetDevice(&o->device);
  const size_t sbytes = (size_t)(soff + 4) * sizeof(float);
  if (e == cudaSuccess) e = cudaMalloc((void**)&o->state0, sbytes);
  if (e == cudaSuccess && o->kind == YB_OPTIM_ADAMW) e = cudaMalloc((void**)&o->state1, sbytes);
  if (e == cudaSuccess) e = cudaMalloc(&o->chunks, chunks.size() * sizeof(OptimChunk));
  if (e == cudaSuccess) e = cudaMemset(o->state0, 0, sbytes);
  if (e == cudaSuccess && o->state1) e = cudaMemset(o->state1, 0, sbytes);
  if (e == cudaSuccess) e = cudaMemcpy(o->chunks, chunks.data(), chunks.size() * sizeof(OptimChunk), cudaMemcpyHostToDevice);
  if (e != cudaSuccess) {
    set_error("yb_optim_create: %s", cudaGetErrorString(e));
    yb_optim_destroy(o);
    return YB_ERR_CUDA;
  }
  *out = o;
  return YB_OK;
}

YB_API int yb_optim_step(yb_optim* o, const float* grad_flat, double lr, float grad_scale, void* stream) {
  YB_REQUIRE(o && grad_flat, YB_ERR_INVALID, "yb_optim_step: null argument");
  YB_REQUIRE(((uintptr_t)grad_flat & 3) == 0, YB_ERR_INVALID, "yb_optim_step: grad_flat is not 4-byte aligned");
  int dev = 0;
  YB_CHECK_CUDA(cudaGetDevice(&dev));
  YB_REQUIRE(dev == o->device, YB_ERR_INVALID, "yb_optim_step: created on device %d, current device is %d", o->device, dev);
  const int64_t t = ++o->step;
  OptimScalars c{};
  c.grad_scale = grad_scale;
  c.first = t == 1;
  c.use_wd = o->weight_decay != 0;
  c.wd = (float)o->weight_decay;
  c.momentum = (float)o->momentum;
  c.neg_lr = (float)(-lr);
  // torch/optim/adam.py, _multi_tensor_adam without capturable: Python floats (double), each scalar rounded to fp32 by its kernel
  c.decay = (float)(1.0 - lr * o->weight_decay);
  c.w1 = (float)(1.0 - o->beta1);
  c.beta2 = (float)o->beta2;
  c.c2 = (float)(1.0 - o->beta2);
  c.bc2_sqrt = (float)pow(1.0 - pow(o->beta2, (double)t), 0.5);
  c.eps = (float)o->eps;
  c.step_size = (float)((lr / (1.0 - pow(o->beta1, (double)t))) * -1.0);
  cudaStream_t s = (cudaStream_t)stream;
  const OptimChunk* ch = (const OptimChunk*)o->chunks;
  if (o->kind == YB_OPTIM_SGD)
    k_optim_step<YB_OPTIM_SGD><<<o->num_chunks, kOptimThreads, 0, s>>>(ch, grad_flat, o->state0, o->state1, c);
  else
    k_optim_step<YB_OPTIM_ADAMW><<<o->num_chunks, kOptimThreads, 0, s>>>(ch, grad_flat, o->state0, o->state1, c);
  YB_CHECK_LAUNCH();
  return YB_OK;
}

YB_API int yb_optim_read_state(const yb_optim* o, int which, float* out, int64_t out_count, void* stream) {
  YB_REQUIRE(o && out, YB_ERR_INVALID, "yb_optim_read_state: null argument");
  YB_REQUIRE(which == 0 || (which == 1 && o->kind == YB_OPTIM_ADAMW), YB_ERR_INVALID, "yb_optim_read_state: no state %d", which);
  YB_REQUIRE(out_count == o->total, YB_ERR_INVALID, "yb_optim_read_state: out has %lld elements, the gradient %lld",
             (long long)out_count, (long long)o->total);
  const float* src = which == 0 ? o->state0 : o->state1;
  int64_t goff = 0;
  for (size_t i = 0; i < o->counts.size(); ++i) {
    YB_CHECK_CUDA(cudaMemcpyAsync(out + goff, src + o->soffs[i], o->counts[i] * sizeof(float), cudaMemcpyDeviceToDevice,
                                  (cudaStream_t)stream));
    goff += o->counts[i];
  }
  return YB_OK;
}

YB_API int64_t yb_optim_num_elements(const yb_optim* o) { return o ? o->total : -1; }

}  // extern "C"
