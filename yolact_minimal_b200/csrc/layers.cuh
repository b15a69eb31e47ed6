// Layer-level launchers shared by net.cu, kernels_simt.cu and conv_tc.cu.
//
// Activation layout ("haloed NHWC"): a tensor with logical shape [B, C, H, W] is stored as
// [B, H+2, W+2, C] with a ZERO one-pixel halo, i.e. as a row-major matrix of
// M = B*(H+2)*(W+2) rows by C columns.  In this layout every convolution tap of a stride-1
// 3x3 / 1x1 convolution is a constant ROW SHIFT of that matrix (dy*(W+2) + dx), so each conv
// is a plain GEMM  out[M, Cout] = sum_taps  in[M + shift_t, Cin] * Wt[Cin, Cout]  whose A
// operand is loaded by 2D TMA tiles at a shifted row coordinate (out-of-range rows are
// zero-filled by TMA).  Stride-2 convolutions first split their input into 4 parity planes
// with the OUTPUT geometry (k_phase_split), after which they are again constant row shifts.
// Every producer writes zeros into the halo rows/columns of its output.
#pragma once
#include "common.cuh"
#include <cuda_fp16.h>

namespace yb {

enum DType { DT_F32 = 0, DT_BF16 = 1, DT_F16 = 2 };
static inline size_t dtype_size(int dt) { return dt == DT_F32 ? 4 : 2; }

struct Geom {          // geometry of a haloed tensor
  int H, W;            // valid extent
  __host__ __device__ int Hp() const { return H + 2; }
  __host__ __device__ int Wp() const { return W + 2; }
  __host__ __device__ int plane() const { return Hp() * Wp(); }
};

constexpr int kMaxTaps = 9;

struct ConvArgs {
  const void* in;        // haloed NHWC activations (dtype act_dt); for stride-2: parity planes
  const void* weight;    // packed [Cout_pad][ntaps*Cin], act_dt (fp32 or bf16), BN folded
  const float* bias;     // [Cout_pad]
  const void* residual;  // haloed NHWC (act_dt) with Cout channels, or nullptr
  void* out;             // see out_mode
  int act_dt;            // DType of in / residual / (out when out_mode == 0)
  int B;                 // images in this call
  Geom g;                // geometry of the OUTPUT (== input geometry for stride 1 / parity planes)
  int Cin, Cout, Cout_pad;
  int Cin_pad;           // per-tap K stride of the packed weights (Cin rounded up to 64; A columns beyond Cin read as 0)
  int ntaps;
  int tap_shift[kMaxTaps];   // row shift into `in` per tap (includes parity-plane offsets)
  int relu;              // activation: 0 none, 1 ReLU, 2 exact (erf) GELU
  int out_mode;          // 0: haloed NHWC act_dt, halo zeroed;  1: dense fp32 [B*H*W][Cout] (halo rows skipped)
  long long in_rows;     // total rows addressable in `in` (for bounds checks)
  int in_row_stride;     // tensor-core path: elements between consecutive rows of `in` (0 = Cin; < Cin = overlapping rows, stem)
  long long w_ld;        // tensor-core path: elements between consecutive rows of `weight` (0 = ntaps*Cin_pad; larger = a tap subset of a wider matrix)
};

// run `expr` with type alias T bound to the C++ type of DType dt
#define YB_DISPATCH_DT(dt, ...)                                   \
  do {                                                            \
    if ((dt) == DT_F32) { using T = float; __VA_ARGS__; }         \
    else if ((dt) == DT_BF16) { using T = __nv_bfloat16; __VA_ARGS__; } \
    else { using T = __half; __VA_ARGS__; }                       \
  } while (0)

int launch_conv_simt(const ConvArgs& a, cudaStream_t s);

// conv_tc.cu: wgmma path (bf16 or fp16 operands, fp32 accumulation).  `plan` is an opaque per-layer object holding the TMA
// descriptors; created once at finalize time.
struct TcPlan;
int tc_plan_create(const ConvArgs& a_maxbatch, int max_batch, TcPlan** out);
void tc_plan_destroy(TcPlan* p);
int launch_conv_tc(const TcPlan* p, const ConvArgs& a, cudaStream_t s);
bool tc_supported(const ConvArgs& a);

// plain GEMM over a long K on the wgmma kernel (weight gradients):  out[M][ntaps*Nper] (+)= sum_k A[M][k] * B[k + shift_tap][Nper], fp32 out.
// A (the TRANSPOSED output gradient) is K-major [M][lda]; B (the activations as they are: [Kb pixel rows][ldb channels]) is read MN-major,
// tap t at pixel row k + shift[t] (rows outside [0, Kb) read as zero) -- a row shift, because TMA wants 16-byte aligned inner coordinates.
struct GemmArgs {
  const void* a; const void* b; float* out;
  int act_dt, M, Nper, K, lda, ldb, ntaps, accumulate;
  int splits;              // split-K pieces per output tile (needs accumulate = 1 and a zeroed / accumulating `out`); 0 / 1 = none
  long long Kb;            // addressable columns of b
  int shift[16];
};
int tc_plan_create_gemm(const GemmArgs& g, TcPlan** out);
int launch_gemm_tc(const TcPlan* p, const GemmArgs& g, cudaStream_t s);

// Fused tail of one ResNet bottleneck and head of the next (modules/resnet.py:20-40):
//   xo = relu(W3 * t2 + b3 + x)            1x1 Cin -> Cexp, residual x, written out (the next block's residual / the stage output)
//   t1 = relu(W1 * xo + b1)                1x1 Cexp -> Cout of the NEXT block, fed from shared memory: xo is never re-read from HBM
// Cout = Cin between the stride-1 blocks of a stage; Cout = 2 Cin when the next block opens the next stage (its conv1 runs at this
// block's resolution, its stride-2 conv2 and downsample read xo / t1 from HBM).
// All four tensors are haloed NHWC with the same geometry; weights are the packed K-major matrices of the two convolutions.
// First block of a stage (Cd > 0): the residual branch is itself a 1x1 convolution of the block input xd (Cd channels, same geometry);
// it is folded into the first GEMM -- w3 is then [Cexp][Cin + Cd] (conv3 | downsample weights side by side), b3 the summed biases, x unused.
struct BneckArgs {
  const void* t2; const void* x; const void* w3; const void* w1;
  const void* xd; int Cd;
  const float* b3; const float* b1;
  void* xo; void* t1;
  int act_dt, B, Cin, Cexp, Cout;
  Geom g;
};
struct BnPlan;
bool bneck_supported(int act_dt, int Cin, int Cexp, int Cout);
int bneck_plan_create(const BneckArgs& a_maxbatch, int max_batch, BnPlan** out);
void bneck_plan_destroy(BnPlan* p);
int launch_bneck_tc(const BnPlan* p, const BneckArgs& a, cudaStream_t s);

int launch_stem(const float* img_nchw, const float* w /*[7][7][3][64]*/, const float* bias, void* out, int out_dt,
                int B, int S, int H1, cudaStream_t s);
int launch_stem_s2d(const float* img_nchw, void* out /*[B][(H1+2)^2][16 | 64]*/, int dt, int wide, int B, int S, int H1, cudaStream_t s);
bool tc_overlapping_rows_ok();   // can the driver encode a tensor map whose rows overlap (row stride < row length)?
int launch_maxpool(const void* in, void* out, int dt, int B, int C, int Hin, int Hout, cudaStream_t s);
int launch_phase_split(const void* in, void* out, int dt, int B, int C, int Hin, int Hout, int nplanes,
                       long long plane_stride_rows, cudaStream_t s);
int launch_upsample_add(const void* coarse, void* fine, int dt, int B, int C, int Hc, int Hf, cudaStream_t s);
int launch_upsample2x_ac(const void* in, void* out, int dt, int B, int C, int Hin, cudaStream_t s);
int launch_head_finalize(const float* head /*[B*H*W][ld]*/, int ld, int B, int HW, int num_ratios, int num_classes,
                         int coef_dim, int anchor_offset, int A_total, float* cls, float* box, float* coef,
                         cudaStream_t s);
int launch_write_activation(const float* in_nchw, int dt, int B, int C, int H, void* out, cudaStream_t s);
int launch_patch_embed(const float* img, const float* w /*[48][96]*/, const float* bias, const float* g, const float* be, void* out,
                       int dt, int B, int S, int Hg, cudaStream_t s);
int launch_layernorm(const void* in, void* out, const float* g, const float* be, int dt, int B, int C, int H, cudaStream_t s);
int launch_patch_merge_ln(const void* in, void* out, const float* g, const float* be, int dt, int B, int C, int Hin, int Hout,
                          cudaStream_t s);
int launch_window_attention(const void* qkv, const float* qkv_bias, const float* table, void* out, int dt, int B, int H, int C, int nH,
                            int shift, cudaStream_t s);
int launch_read_activation(const void* in, int dt, int B, int C, int H, float* out_nchw, cudaStream_t s);

}  // namespace yb
