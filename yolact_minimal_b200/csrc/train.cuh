// Launchers of the training path (train_kernels.cu, losses.cu) shared with the training engine (train.cu).
#pragma once
#include "layers.cuh"

namespace yb {

// ---- weight packing / gradient unpacking (batched over descriptor tables that live in device memory) ----
struct PackDesc {
  const float* src;        // fp32 master parameter [Cout][Cin][k][k]
  void* dst_fwd;           // forward operand  [rows][ldf]:   (row0+co, t*Cin_pad + ci)            (may be NULL)
  void* dst_bwd;           // dgrad operand    [Cin][ldb]:    (ci, tapslot[t]*CoutT_pad + row0+co)  (may be NULL)
  int Cout, Cin, k, Cin_pad, CoutT_pad, row0;
  long long ldf, ldb;
  int tapslot[9];
};
struct UnpackDesc {
  const float* src;        // packed gradient fp32 [rows][ld]
  float* dst;              // parameter gradient [Cout][Cin][k][k]
  int Cout, Cin, k, Cin_pad, row0;
  long long ld;
  float scale;
};
int launch_pack_weights(const PackDesc* d_descs, int n, int dt, cudaStream_t s);
int launch_pack_stem(const float* src, void* dst, int dt, cudaStream_t s);
int launch_unpack_stem_grad(float* g, float* dst, float scale, cudaStream_t s);
int launch_unpack_wgrad(const UnpackDesc* d_descs, int n, cudaStream_t s);

// ---- batch-statistics BatchNorm ----
int launch_colstats(const void* x, int dt, long long rows, int C, float* sums /*[2C], pre-zeroed*/, cudaStream_t s,
                    int pivot_Hp = 0 /* > 0: BN statistics of a haloed [B][Hp][Hp][C] tensor, sums [3C] (k_bn_finalize) */);
int launch_bn_finalize(const float* sums, int C, double count, const float* gamma, const float* beta, float* run_mean, float* run_var,
                       float momentum, float eps, float* scale, float* shift, float* mean, float* invstd, cudaStream_t s);
int launch_bn_apply(const void* y, void* z, const void* res, const float* scale, const float* shift, int relu, int dt, int B, int C, int H,
                    cudaStream_t s);
int launch_bn_bwd_reduce(const void* y, const void* dz, const void* z, int relu, const float* mean, const float* invstd, int dt, long long rows,
                         int C, float* sums /*[2C], pre-zeroed*/, cudaStream_t s);
int launch_bn_bwd_apply(const void* y, const void* dz, const void* z, int relu, const float* mean, const float* invstd, const float* gamma,
                        const float* sums, double count, void* dy, void* dres, float* dgamma, float* dbeta, float gscale, int dt, int B, int C, int H,
                        cudaStream_t s);

// ---- data movement / element-wise backward ----
int launch_transpose16(const void* in, int ld_in, void* out, int dt, long long rows, int C, long long ld, cudaStream_t s);
int launch_relu_bwd(void* dz, const void* z, int dt, long long n, cudaStream_t s);
int launch_add16(void* a, const void* b, int dt, long long n, cudaStream_t s);
int launch_maxpool_bwd(const void* x, const void* dy, void* dx, int dt, int B, int C, int Hin, int Hout, cudaStream_t s);
int launch_bilinear_bwd(const void* dfine, void* dcoarse, int dt, int B, int C, int Hc, int Hf, int align_corners, int accumulate, cudaStream_t s);
int launch_phase_merge(const void* planes, void* dx, int dt, int B, int C, int Hin, int Hout, int nplanes, long long plane_stride_rows, cudaStream_t s);
int launch_dense_to_haloed(const float* src, const float* act, int lds, int Csrc, void* dst, int dt, int B, int C, int H, cudaStream_t s);
int launch_head_train(const float* head, int ld, int B, int HW, int R, int NC, int K, int anchor_offset, int A_total, float* cls, float* box,
                      float* coef, cudaStream_t s);
int launch_head_grad(const float* dcls, const float* dbox, const float* dcoef, const float* coef, int dt, int B, int H, int R, int NC, int K,
                     int anchor_offset, int A_total, int ldo, void* out, cudaStream_t s);
int launch_scale_copy(const float* src, float* dst, int n, float scale, cudaStream_t s);

// counter hash of the device-side random draws (mask subset in losses.cu, stochastic depth in swin_train.cu)
__device__ __forceinline__ uint32_t hash32(uint32_t x) { x ^= x >> 16; x *= 0x7feb352du; x ^= x >> 15; x *= 0x846ca68bu; x ^= x >> 16; return x; }

// ---- Swin-T training (swin_train.cu): 16-bit haloed token grids, fp32 statistics; dgb / dtable / dw / db / dbias accumulate ----
constexpr int kSwinBlocks = 12;                                    // blocks over the four stages (2 + 2 + 6 + 2)
__host__ __device__ inline float swin_drop_rate(int blk) { return 0.2f * (float)blk / (float)(kSwinBlocks - 1); }   // linspace(0, 0.2, 12)
int launch_ln_fwd(const void* x, int x_f32, void* y, const float* g, const float* be, float* mean, float* rstd, int dt, int B, int C, int H,
                  cudaStream_t s);
int launch_ln_bwd(const void* x, int x_f32, const void* dy, const float* g, const float* mean, const float* rstd, void* dx, int accumulate,
                  float* dgb /*[2C]: dgamma | dbeta*/, int dt, int B, int C, int H, cudaStream_t s);
int launch_pe_conv(const float* img, const float* w, const float* bias, float* out /*fp32 haloed [..][96]*/, int B, int S, int Hg, cudaStream_t s);
int launch_pe_wgrad(const float* img, const float* dy, float* dw /*[96*48]*/, float* db /*[96]*/, int B, int S, int Hg, cudaStream_t s);
int launch_wattn_fwd(const void* qkv, const float* qkv_bias, const float* table, void* out, float* lse /*[rows][nH]*/, int dt, int B, int H, int C,
                     int nH, int shift, cudaStream_t s);
int launch_wattn_bwd(const void* qkv, const float* qkv_bias, const float* table, const void* dout, const float* lse, void* dqkv, float* dtable,
                     float* dbias /*[3C]*/, int dt, int B, int H, int C, int nH, int shift, cudaStream_t s);
int launch_gelu_fwd(const void* h, void* y, int dt, long long n, cudaStream_t s);
int launch_gelu_bwd(const void* h, const void* dy, void* dh, int dt, long long n, cudaStream_t s);
int launch_merge_fwd(const void* in, void* out, int dt, int B, int C, int Hin, int Hout, cudaStream_t s);
int launch_merge_bwd(const void* dout, void* dx, int accumulate, int dt, int B, int C, int Hin, int Hout, cudaStream_t s);
int launch_drop_path_masks(const uint32_t* seed_dev, float* masks /*[B][kSwinBlocks][2]*/, int B, cudaStream_t s);
int launch_drop_residual(const void* x, const void* y, void* out, const float* masks, int blk, int branch, int dt, int B, long long per_img,
                         cudaStream_t s);
int launch_drop_residual_bwd(const void* dout, void* dx, int accumulate, void* dy, const float* masks, int blk, int branch, int dt, int B,
                             long long per_img, cudaStream_t s);


// losses.cu: yb_losses with the seed in device memory; total_gt / max_gt_per_image only size grids and the workspace (graph replay)
constexpr int kLossMaxGt = 256;
int losses_impl(const yb_loss_params* p, const float* cls, const float* box, const float* coef, const float* proto, const float* seg, int ld_seg,
                const float* anchors, const float* gt, const int32_t* gt_offset, const float* gt_masks, int total_gt, int max_gt_per_image,
                uint32_t seed, const uint32_t* seed_dev, const float* grad_scale, float* losses, float* d_cls, float* d_box, float* d_coef, float* d_proto,
                float* d_seg, int32_t* dbg_labels, int32_t* dbg_matched_idx, float* dbg_offsets, uint8_t* dbg_neg, void* workspace, size_t workspace_bytes,
                void* stream);

}  // namespace yb
