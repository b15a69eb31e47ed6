// Training engine (SURVEY.md 8 row a12): Yolact.forward in training mode and its backward pass for the ResNet and Swin-T backbones,
// restated as two flat launch lists over persistent buffers (modules/resnet.py:20-98, modules/swin_transformer.py:436-518,
// modules/yolact.py:12-161 forward; the backward is derived here -- the reference gets it from torch autograd).  Swin-T's linear
// layers are 1x1 convs on the kernels below; its LayerNorm / attention / GELU / merge / stochastic-depth kernels are swin_train.cu.
//
//   forward   conv (wgmma, 16-bit operands, fp32 accumulate, raw output) -> batch statistics -> affine + ReLU (+ residual);
//             FPN / ProtoNet / heads as in inference but with raw logits; targets + the four losses (losses.cu)
//   backward  per conv: bias gradient (column sums), weight gradient = GEMM over the pixel dimension of the TRANSPOSED
//             activations and output gradients on the same wgmma kernel (tc_plan_create_gemm), input gradient = the same
//             implicit-GEMM conv kernel with the transposed, tap-reversed weights (stride 2: one conv per parity plane +
//             k_phase_merge); BatchNorm / ReLU / max-pool / bilinear backward on CUDA cores (train_kernels.cu)
//
// The program is built ONCE per engine (fixed batch): every buffer, TMA descriptor and launch closure is created up front, a
// step replays the two lists.  Parameters are never copied: yb_train_bind stores the caller's device pointers (fp32 master
// weights and their gradient buffers); each forward re-packs the 16-bit operand copies from them in one batched launch.
#include "arch.cuh"
#include "train.cuh"

#include <stdlib.h>
#include <string.h>
#include <functional>
#include <map>
#include <memory>
#include <string>
#include <vector>

using namespace yb;

namespace {

struct TT {                       // an activation tensor of the training graph
  std::string name;
  void* data = nullptr;           // haloed NHWC 16-bit [B*planes][H+2][H+2][C]  (or dense fp32 [B*H*H][ld] when dense)
  void* grad = nullptr;           // same geometry, Cg channels
  void* tr = nullptr;             // transposed data [C][ldT] (weight-gradient operand), filled lazily in the backward pass
  int C = 0, Cg = 0, H = 0, planes = 1, ld = 0;
  bool dense = false, grad_set = false, tr_done = false, needs_grad = true;
  long long rows = 0;             // B * planes * (H+2)^2
  long long ldT = 0;
};

struct BoundTensor {
  std::string name;
  int64_t count;
  int kind;                       // 0 parameter, 1 buffer
  float* data = nullptr;
  float* grad = nullptr;
};

struct ConvRec {                  // one convolution's parameters (possibly used at several places: the shared prediction head)
  std::string wname, bname;
  std::vector<std::string> cat;   // fused head: conf | box | coef
  int Cin = 0, Cout = 0, Cout_pad = 0, k = 1, stride = 1, Cin_pad = 0, CoutT_pad = 0;
  void* wf = nullptr;             // forward operand [ceil64(Cout_pad)][k2*Cin_pad]
  void* wb = nullptr;             // dgrad operand   [ceil64(Cin)][k2*CoutT_pad], taps regrouped (tapslot)
  float* bias = nullptr;          // forward bias pointer ([Cout_pad] fp32): bound parameter, packed buffer (cat) or zeros
  float* bias_cat = nullptr;
  float* dWp = nullptr;           // packed weight gradient fp32 [Cout_pad][k2*Cin_pad]
  float* bsum = nullptr;          // bias-gradient column sums [2*Cg]
  bool wgrad_set = false, needs_dgrad_w = true;
  int bias_idx = -1;              // bound-tensor index of the bias parameter (resolved at launch time: bindings come after build)
  int tapslot[9];
  int plane_slot0[4];
};

typedef std::function<int(cudaStream_t)> Launch;

}  // namespace

struct yb_train {
  yb_net_config cfg{};
  int B = 0, dt = DT_BF16, S = 0;
  int A = 0, P = 0, Hs = 0;
  int level_size[5]{}, level_off[5]{};
  std::vector<BoundTensor> bound;
  std::map<std::string, int> bidx;
  std::vector<std::unique_ptr<TT>> tensors;
  std::map<std::string, TT*> by_name;
  std::vector<std::unique_ptr<ConvRec>> convs;
  std::vector<void*> allocs;
  std::vector<TcPlan*> plans;
  std::vector<Launch> fwd, bwd, bwd_tail;
  std::vector<std::string> fwd_what, bwd_what;     // debug labels (YOLACT_B200_TRAIN_DEBUG=1 synchronises after every launch)
  std::string cur_label;
  std::vector<std::function<int()>> bwd_builders;     // run in reverse op order when the program is finalised
  std::vector<PackDesc> pack_descs;
  std::vector<UnpackDesc> unpack_descs;
  PackDesc* d_pack = nullptr; UnpackDesc* d_unpack = nullptr;
  float* stats = nullptr; size_t stats_floats = 0, stats_cap = 0;    // zeroed at the start of forward and of backward
  float* zeros = nullptr;                                              // [4096] zero bias
  float* drop_masks = nullptr;                                         // Swin: stochastic-depth masks of the step [B][kSwinBlocks][2]
  bool built = false, descs_dirty = true;
  std::vector<float> anchors;
  float* d_anchors = nullptr;
  // network outputs / loss plumbing
  float *d_img = nullptr, *cls = nullptr, *box = nullptr, *coef = nullptr, *proto = nullptr, *seg = nullptr;
  float *g_cls = nullptr, *g_box = nullptr, *g_coef = nullptr, *g_proto = nullptr, *g_seg = nullptr;
  int ld_seg = 0;
  void* loss_ws = nullptr; size_t loss_ws_bytes = 0;
  // per-step state read by the closures
  const float* cur_gt = nullptr;
  yb_train_hparams hp{};
  float* d_losses_scratch = nullptr;
  // graph-stable copies of the per-step inputs, and the captured forward / backward launch lists
  float* p_gt = nullptr; int32_t* p_gt_off = nullptr; float* p_masks = nullptr; int mask_cap = 0;
  float *p_loss_grad = nullptr, *p_losses = nullptr; uint32_t* p_seed = nullptr;
  uint32_t seed_host = 0;
  cudaGraphExec_t g_fwd = nullptr, g_bwd = nullptr;
  cudaStream_t gstream = nullptr;                                     // the graphs are captured and replayed here (the caller's stream may be the
  cudaEvent_t ev_in = nullptr, ev_out = nullptr;                      // legacy default stream, which cannot be captured), fenced by two events
  bool use_graphs = true;
  yb_train_hparams g_hp{};
  uint64_t launches_fwd = 0, launches_bwd = 0;

  int add_bound(const std::string& n, int64_t count, int kind) {
    BoundTensor b; b.name = n; b.count = count; b.kind = kind;
    bidx[n] = (int)bound.size();
    bound.push_back(b);
    return (int)bound.size() - 1;
  }
  BoundTensor& bt(const std::string& n) { return bound[bidx.at(n)]; }
};

namespace {

#define FWD_PUSH(...) do { t->fwd_what.push_back(t->cur_label + " @" + std::to_string(__LINE__)); t->fwd.push_back(__VA_ARGS__); } while (0)
#define BWD_PUSH(...) do { t->bwd_what.push_back(t->cur_label + " @" + std::to_string(__LINE__)); t->bwd.push_back(__VA_ARGS__); } while (0)

int dev_alloc(yb_train* t, void** p, size_t bytes) {
  YB_CHECK_CUDA(cudaMalloc(p, bytes ? bytes : 16));
  YB_CHECK_CUDA(cudaMemset(*p, 0, bytes ? bytes : 16));
  t->allocs.push_back(*p);
  return YB_OK;
}

float* stats_take(yb_train* t, size_t n) {       // offsets into the per-step zeroed fp32 arena (resolved after allocation)
  const size_t o = t->stats_floats;
  t->stats_floats += (n + 63) / 64 * 64;
  return reinterpret_cast<float*>(o * sizeof(float));     // an OFFSET until finalize_stats() rebases it
}

TT* new_tensor(yb_train* t, const std::string& name, int C, int H, int planes = 1, bool dense = false, int ld = 0) {
  std::unique_ptr<TT> u(new TT());
  u->name = name; u->C = C; u->Cg = C; u->H = H; u->planes = planes; u->dense = dense; u->ld = ld;
  u->rows = (long long)t->B * planes * (H + 2) * (H + 2);
  TT* r = u.get();
  t->tensors.push_back(std::move(u));
  if (!name.empty()) t->by_name[name] = r;
  return r;
}

int alloc_data(yb_train* t, TT* x, long long pad_rows = 0) {
  if (x->dense) return dev_alloc(t, &x->data, (size_t)t->B * x->H * x->H * x->ld * 4);
  return dev_alloc(t, &x->data, (size_t)(x->rows + pad_rows) * x->C * 2);
}

int ensure_grad(yb_train* t, TT* x) {
  if (x->grad) return YB_OK;
  return dev_alloc(t, &x->grad, (size_t)x->rows * x->Cg * 2);
}

// ---- convolution records ----
ConvRec* new_conv(yb_train* t, const std::string& prefix, int Cin, int Cout, int k, int stride, bool bias) {
  std::unique_ptr<ConvRec> u(new ConvRec());
  u->wname = prefix + ".weight"; u->bname = bias ? prefix + ".bias" : "";
  u->Cin = Cin; u->Cout = Cout; u->Cout_pad = (Cout + 15) / 16 * 16; u->k = k; u->stride = stride;
  u->Cin_pad = (Cin + 63) / 64 * 64; u->CoutT_pad = (u->Cout_pad + 63) / 64 * 64;
  t->add_bound(u->wname, (int64_t)Cout * Cin * k * k, 0);
  if (bias) t->add_bound(u->bname, Cout, 0);
  ConvRec* r = u.get();
  t->convs.push_back(std::move(u));
  return r;
}

void conv_tap_layout(ConvRec* c) {
  const int k2 = c->k * c->k;
  for (int i = 0; i < 4; ++i) c->plane_slot0[i] = 0;
  if (c->stride == 1 || c->k == 1) {
    for (int tt = 0; tt < k2; ++tt) c->tapslot[tt] = k2 - 1 - tt;          // reversed taps: dgrad shifts == forward shifts
  } else {                                                                  // 3x3 stride 2: each plane's taps, in dgrad shift order
    int slot = 0;
    for (int pl = 0; pl < 4; ++pl) {
      int taps[4];
      c->plane_slot0[pl] = slot;
      const int n = parity_plane_taps(pl, taps);
      for (int i = 0; i < n; ++i) c->tapslot[taps[i]] = slot++;
    }
  }
}

int alloc_conv(yb_train* t, ConvRec* c, bool needs_dgrad) {
  const int k2 = c->k * c->k;
  conv_tap_layout(c);
  c->needs_dgrad_w = needs_dgrad;
  YB_PROPAGATE(dev_alloc(t, &c->wf, (size_t)((c->Cout_pad + 63) / 64 * 64) * k2 * c->Cin_pad * 2));
  if (needs_dgrad) YB_PROPAGATE(dev_alloc(t, &c->wb, (size_t)((c->Cin + 63) / 64 * 64) * k2 * c->CoutT_pad * 2));
  YB_PROPAGATE(dev_alloc(t, (void**)&c->dWp, (size_t)c->Cout_pad * k2 * c->Cin_pad * 4));
  return YB_OK;
}

void add_pack_descs(yb_train* t, ConvRec* c) {
  const int k2 = c->k * c->k;
  auto one = [&](const std::string& wname, int cout, int row0) {
    PackDesc d; memset(&d, 0, sizeof(d));
    d.src = reinterpret_cast<const float*>((uintptr_t)t->bidx.at(wname));       // an INDEX until resolve_descs()
    d.dst_fwd = c->wf; d.dst_bwd = c->needs_dgrad_w ? c->wb : nullptr;
    d.Cout = cout; d.Cin = c->Cin; d.k = c->k; d.Cin_pad = c->Cin_pad; d.CoutT_pad = c->CoutT_pad; d.row0 = row0;
    d.ldf = (long long)k2 * c->Cin_pad; d.ldb = (long long)k2 * c->CoutT_pad;
    for (int i = 0; i < 9; ++i) d.tapslot[i] = i < k2 ? c->tapslot[i] : 0;
    t->pack_descs.push_back(d);
    UnpackDesc u; memset(&u, 0, sizeof(u));
    u.src = c->dWp; u.dst = reinterpret_cast<float*>((uintptr_t)t->bidx.at(wname));
    u.Cout = cout; u.Cin = c->Cin; u.k = c->k; u.Cin_pad = c->Cin_pad; u.row0 = row0; u.ld = (long long)k2 * c->Cin_pad; u.scale = 1.f;
    t->unpack_descs.push_back(u);
  };
  if (c->cat.empty()) one(c->wname, c->Cout, 0);
  else {
    int row = 0;
    for (const auto& n : c->cat) {
      const int cout = (int)t->bt(n + ".bias").count;
      one(n + ".weight", cout, row);
      row += cout;
    }
  }
}

// ---- forward conv op + its backward ----
// x: input (haloed, planes == 1); returns y (raw conv output + bias, optional fused ReLU; haloed 16-bit, or dense fp32 [B*Ho*Ho][Cout_pad])
int op_conv(yb_train* t, TT* x, ConvRec* c, int relu, bool out_dense, const std::string& yname, TT** out, TT* y_given = nullptr) {
  const int B = t->B, Hin = x->H, Hout = out_size(Hin, c->stride), Wp = Hout + 2;
  t->cur_label = "conv " + yname;
  const long long plane_rows = (long long)B * Wp * Wp;
  TT* src = x;
  if (c->stride == 2) {
    const int planes = c->k == 3 ? 4 : 1;
    src = new_tensor(t, yname + ".planes", c->Cin, Hout, planes);
    YB_PROPAGATE(alloc_data(t, src));
    void* xin = x->data; void* pout = src->data;
    const int dt = t->dt, Cin = c->Cin;
    FWD_PUSH([=](cudaStream_t s) { return launch_phase_split(xin, pout, dt, B, Cin, Hin, Hout, planes, plane_rows, s); });
  }
  TT* y = y_given;
  if (!y) {
    y = out_dense ? new_tensor(t, yname, c->Cout, Hout, 1, true, c->Cout_pad) : new_tensor(t, yname, c->Cout_pad, Hout);
    YB_PROPAGATE(alloc_data(t, y));
  }
  if (out_dense) y->Cg = c->Cout_pad < 64 ? 64 : c->Cout_pad;       // gradient operand width (K of the dgrad GEMM), >= one TMA box
  ConvArgs a; memset(&a, 0, sizeof(a));
  a.in = src->data; a.weight = c->wf; a.bias = c->bias; a.residual = nullptr; a.out = y->data;
  a.act_dt = t->dt; a.B = B; a.g.H = Hout; a.g.W = Hout;
  a.Cin = c->Cin; a.Cin_pad = c->Cin_pad; a.Cout = out_dense ? c->Cout : c->Cout_pad; a.Cout_pad = c->Cout_pad;
  a.relu = relu; a.out_mode = out_dense ? 1 : 0;
  a.ntaps = conv_taps(c->k, c->stride, Wp, plane_rows, a.tap_shift);
  a.in_rows = src->rows;
  YB_REQUIRE(tc_supported(a), YB_ERR_UNSUPPORTED, "train: conv %s (Cin=%d Cout=%d) not supported by the wgmma kernel", c->wname.c_str(), c->Cin, c->Cout);
  TcPlan* pl = nullptr;
  YB_PROPAGATE(tc_plan_create(a, B, &pl));
  t->plans.push_back(pl);
  const int bias_idx = c->bias_idx;
  FWD_PUSH([=](cudaStream_t s) {
    ConvArgs aa = a;
    if (bias_idx >= 0) aa.bias = t->bound[bias_idx].data;
    return launch_conv_tc(pl, aa, s);
  });

  // ---------------- backward (built later, in reverse op order) ----------------
  t->bwd_builders.push_back([=]() -> int {
    const int dt = t->dt;
    t->cur_label = "conv-bwd " + y->name;
    YB_REQUIRE(y->grad != nullptr && y->grad_set, YB_ERR_STATE, "train: conv output %s has no gradient", y->name.c_str());
    const int Cg = y->Cg;                                            // channels of dY (== Cout_pad except padded small outputs)
    void* dy = y->grad;
    const long long rows_y = plane_rows;                             // rows of y / dY
    if (relu == 1 && !out_dense) {                                   // z = relu(conv + b): dY = dz * [z > 0]   (dense outputs are masked by their producer)
      void* z = y->data;
      const long long n = rows_y * Cg;
      BWD_PUSH([=](cudaStream_t s) { return launch_relu_bwd(dy, z, dt, n, s); });
    }
    // bias gradient
    if (!c->bname.empty() || !c->cat.empty()) {
      float* bs = c->bsum;                                           // offset into the per-step zeroed statistics arena
      BWD_PUSH([=](cudaStream_t s) { return launch_colstats(dy, dt, rows_y, Cg, (float*)((char*)t->stats + (size_t)bs), s); });
    }
    // weight gradient: dW[co][tap][ci] = sum_m dY[m][co] * X[m + shift_tap][ci]
    {
      const long long ldT = (rows_y + 7) / 8 * 8;
      void* dyT = nullptr;
      YB_PROPAGATE(dev_alloc(t, &dyT, (size_t)c->Cout_pad * ldT * 2));
      const int Mrows = c->Cout_pad;
      BWD_PUSH([=](cudaStream_t s) { return launch_transpose16(dy, Cg, dyT, dt, rows_y, Mrows, ldT, s); });
      GemmArgs g; memset(&g, 0, sizeof(g));
      g.a = dyT; g.b = src->data; g.out = c->dWp; g.act_dt = dt; g.M = c->Cout_pad; g.Nper = c->Cin_pad; g.K = (int)rows_y; g.lda = (int)ldT; g.ldb = src->C;
      g.Kb = src->rows; g.accumulate = 1;                           // dWp is zero at the start of a backward pass (cleared by the unpack kernel)
      g.ntaps = conv_taps(c->k, c->stride, Wp, plane_rows, g.shift);
      {  // split-K: a weight gradient has few output tiles and a long K (the pixels); cut K so that ~2 waves of CTAs are busy
        const int bn = c->Cin_pad % 256 == 0 ? 256 : (c->Cin_pad % 128 == 0 ? 128 : 64);
        const int tiles = ((c->Cout_pad + 127) / 128) * g.ntaps * (c->Cin_pad / bn);
        const int kb_total = (int)((rows_y + 63) / 64);
        int sms = 0;
        YB_PROPAGATE(yb_device_info(&sms, nullptr, nullptr));
        int splits = (2 * sms + tiles - 1) / tiles;
        if (splits > kb_total / 4) splits = kb_total / 4;
        g.splits = splits < 1 ? 1 : splits;
        if (getenv("YOLACT_B200_TRAIN_NO_SPLITK")) g.splits = 1;              // tooling: A/B
      }
      TcPlan* gp = nullptr;
      YB_PROPAGATE(tc_plan_create_gemm(g, &gp));
      t->plans.push_back(gp);
      BWD_PUSH([=](cudaStream_t s) { return launch_gemm_tc(gp, g, s); });
      c->wgrad_set = true;
    }
    // input gradient
    if (x->needs_grad) {
      YB_PROPAGATE(ensure_grad(t, x));
      if (c->stride == 1) {
        ConvArgs d; memset(&d, 0, sizeof(d));
        d.in = dy; d.weight = c->wb; d.bias = t->zeros; d.residual = x->grad_set ? x->grad : nullptr; d.out = x->grad;
        d.act_dt = dt; d.B = B; d.g.H = Hout; d.g.W = Hout; d.Cin = Cg; d.Cin_pad = c->CoutT_pad; d.Cout = c->Cin; d.Cout_pad = c->Cin;
        d.relu = 0; d.out_mode = 0; d.in_rows = rows_y;
        d.ntaps = conv_taps(c->k, c->stride, Wp, plane_rows, d.tap_shift);
        YB_REQUIRE(tc_supported(d), YB_ERR_UNSUPPORTED, "train: dgrad of %s not supported", c->wname.c_str());
        TcPlan* dp = nullptr;
        YB_PROPAGATE(tc_plan_create(d, B, &dp));
        t->plans.push_back(dp);
        BWD_PUSH([=](cudaStream_t s) { return launch_conv_tc(dp, d, s); });
      } else {
        const int planes = src->planes;
        void* dplanes = nullptr;
        YB_PROPAGATE(dev_alloc(t, &dplanes, (size_t)src->rows * c->Cin * 2));
        for (int pl_i = 0; pl_i < planes; ++pl_i) {
          ConvArgs d; memset(&d, 0, sizeof(d));
          d.in = dy; d.weight = (char*)c->wb + (size_t)c->plane_slot0[pl_i] * c->CoutT_pad * 2; d.w_ld = (long long)c->k * c->k * c->CoutT_pad;
          d.bias = t->zeros; d.residual = nullptr; d.out = (char*)dplanes + (size_t)pl_i * plane_rows * c->Cin * 2;
          d.act_dt = dt; d.B = B; d.g.H = Hout; d.g.W = Hout; d.Cin = Cg; d.Cin_pad = c->CoutT_pad; d.Cout = c->Cin; d.Cout_pad = c->Cin;
          d.relu = 0; d.out_mode = 0; d.in_rows = rows_y;
          int taps[4];
          d.ntaps = c->k == 1 ? 1 : parity_plane_taps(pl_i, taps, Wp, d.tap_shift);
          YB_REQUIRE(tc_supported(d), YB_ERR_UNSUPPORTED, "train: stride-2 dgrad of %s not supported", c->wname.c_str());
          TcPlan* dp = nullptr;
          YB_PROPAGATE(tc_plan_create(d, B, &dp));
          t->plans.push_back(dp);
          BWD_PUSH([=](cudaStream_t s) { return launch_conv_tc(dp, d, s); });
        }
        const int Cin = c->Cin;
        if (!x->grad_set) {
          void* xg = x->grad;
          BWD_PUSH([=](cudaStream_t s) { return launch_phase_merge(dplanes, xg, dt, B, Cin, Hin, Hout, planes, plane_rows, s); });
        } else {
          void* tmp = nullptr;
          YB_PROPAGATE(dev_alloc(t, &tmp, (size_t)x->rows * x->C * 2));
          void* xg = x->grad; const long long n = x->rows * x->C;
          BWD_PUSH([=](cudaStream_t s) { return launch_phase_merge(dplanes, tmp, dt, B, Cin, Hin, Hout, planes, plane_rows, s); });
          BWD_PUSH([=](cudaStream_t s) { return launch_add16(xg, tmp, dt, n, s); });
        }
      }
      x->grad_set = true;
    }
    return YB_OK;
  });
  *out = y;
  return YB_OK;
}

// ---- batch-norm (+ residual, + ReLU) ----
int op_bn(yb_train* t, TT* y, const std::string& bn, int relu, TT* res, const std::string& zname, TT** out) {
  const int B = t->B, C = y->C, H = y->H, dt = t->dt;
  t->cur_label = "bn " + zname;
  for (const char* sfx : {".weight", ".bias"}) t->add_bound(bn + sfx, C, 0);
  for (const char* sfx : {".running_mean", ".running_var"}) t->add_bound(bn + sfx, C, 1);
  TT* z = new_tensor(t, zname, C, H);
  YB_PROPAGATE(alloc_data(t, z));
  float* sums = stats_take(t, 3 * C);                             // sum d | sum d^2 | pivot  (d = y - pivot: k_colstats)
  float* aff = nullptr;                                            // scale | shift | mean | invstd
  YB_PROPAGATE(dev_alloc(t, (void**)&aff, (size_t)4 * C * 4));
  const int ig = t->bidx.at(bn + ".weight"), ib = t->bidx.at(bn + ".bias"), im = t->bidx.at(bn + ".running_mean"), iv = t->bidx.at(bn + ".running_var");
  const double count = (double)B * H * H;
  const long long rows = y->rows;
  void* yd = y->data; void* zd = z->data; void* rd = res ? res->data : nullptr;
  FWD_PUSH([=](cudaStream_t s) { return launch_colstats(yd, dt, rows, C, (float*)((char*)t->stats + (size_t)sums), s, H + 2); });
  FWD_PUSH([=](cudaStream_t s) {
    return launch_bn_finalize((float*)((char*)t->stats + (size_t)sums), C, count, t->bound[ig].data, t->bound[ib].data, t->bound[im].data, t->bound[iv].data,
                              t->hp.bn_momentum, t->hp.bn_eps, aff, aff + C, aff + 2 * C, aff + 3 * C, s);
  });
  FWD_PUSH([=](cudaStream_t s) { return launch_bn_apply(yd, zd, rd, aff, aff + C, relu, dt, B, C, H, s); });

  float* bsums = stats_take(t, 2 * C);
  t->bwd_builders.push_back([=]() -> int {
    t->cur_label = "bn-bwd " + z->name;
    YB_REQUIRE(z->grad != nullptr && z->grad_set, YB_ERR_STATE, "train: bn output %s has no gradient", z->name.c_str());
    YB_PROPAGATE(ensure_grad(t, y));
    void* dz = z->grad; void* dyp = y->grad;
    void* dres = nullptr; void* tmp = nullptr;
    if (res && res->needs_grad) {
      YB_PROPAGATE(ensure_grad(t, res));
      if (!res->grad_set) dres = res->grad;
      else { YB_PROPAGATE(dev_alloc(t, &tmp, (size_t)res->rows * res->C * 2)); dres = tmp; }
    }
    BWD_PUSH([=](cudaStream_t s) {
      return launch_bn_bwd_reduce(yd, dz, zd, relu, aff + 2 * C, aff + 3 * C, dt, rows, C, (float*)((char*)t->stats + (size_t)bsums), s);
    });
    BWD_PUSH([=](cudaStream_t s) {
      return launch_bn_bwd_apply(yd, dz, zd, relu, aff + 2 * C, aff + 3 * C, t->bound[ig].data, (float*)((char*)t->stats + (size_t)bsums), count, dyp, dres,
                                 t->bound[ig].grad, t->bound[ib].grad, 1.f, dt, B, C, H, s);
    });
    if (tmp) {
      void* rg = res->grad; const long long n = res->rows * res->C;
      BWD_PUSH([=](cudaStream_t s) { return launch_add16(rg, tmp, dt, n, s); });
    }
    if (res && res->needs_grad) res->grad_set = true;
    y->grad_set = true;
    return YB_OK;
  });
  *out = z;
  return YB_OK;
}

// ---- Swin-T ops (swin_train.cu kernels; the linear layers are op_conv with k = 1) ----
// a linear layer of the reference (nn.Linear): a 1x1 conv record with the parameter's own names
int swin_linear(yb_train* t, const std::string& prefix, int Cin, int Cout, bool bias, std::vector<ConvRec*>* all, ConvRec** out) {
  ConvRec* c = new_conv(t, prefix, Cin, Cout, 1, 1, bias);
  c->bias = t->zeros;
  if (bias) { c->bias_idx = t->bidx.at(c->bname); c->bsum = stats_take(t, 2 * (size_t)(c->Cout_pad < 64 ? 64 : c->Cout_pad)); }
  YB_PROPAGATE(alloc_conv(t, c, true));
  all->push_back(c);
  *out = c;
  return YB_OK;
}

// copies a parameter gradient reduced in the statistics arena to the bound gradient buffer at the end of the backward pass
void tail_copy(yb_train* t, float* arena_off, const std::string& name, int n) {
  const int ib = t->bidx.at(name);
  t->bwd_tail.push_back([=](cudaStream_t s) { return launch_scale_copy((float*)((char*)t->stats + (size_t)arena_off), t->bound[ib].grad, n, 1.f, s); });
}

// LayerNorm `prm` over the channels of x (per-token mean / rstd kept for the backward pass)
int op_ln(yb_train* t, TT* x, const std::string& prm, const std::string& yname, TT** out) {
  const int B = t->B, C = x->C, H = x->H, dt = t->dt;
  t->cur_label = "ln " + yname;
  t->add_bound(prm + ".weight", C, 0); t->add_bound(prm + ".bias", C, 0);
  const int ig = t->bidx.at(prm + ".weight"), ib = t->bidx.at(prm + ".bias");
  TT* y = new_tensor(t, yname, C, H);
  YB_PROPAGATE(alloc_data(t, y));
  const long long rows = x->rows;
  float* st = nullptr;                                             // mean | rstd per token row
  YB_PROPAGATE(dev_alloc(t, (void**)&st, (size_t)2 * rows * 4));
  void* xd = x->data; void* yd = y->data;
  FWD_PUSH([=](cudaStream_t s) { return launch_ln_fwd(xd, 0, yd, t->bound[ig].data, t->bound[ib].data, st, st + rows, dt, B, C, H, s); });
  float* dgb = stats_take(t, 2 * (size_t)C);
  tail_copy(t, dgb, prm + ".weight", C);
  tail_copy(t, dgb + C, prm + ".bias", C);
  t->bwd_builders.push_back([=]() -> int {
    t->cur_label = "ln-bwd " + y->name;
    YB_REQUIRE(y->grad && y->grad_set, YB_ERR_STATE, "train: LayerNorm output %s has no gradient", y->name.c_str());
    YB_PROPAGATE(ensure_grad(t, x));
    void* dy = y->grad; void* dx = x->grad; const int acc = x->grad_set ? 1 : 0;
    BWD_PUSH([=](cudaStream_t s) {
      return launch_ln_bwd(xd, 0, dy, t->bound[ig].data, st, st + rows, dx, acc, (float*)((char*)t->stats + (size_t)dgb), dt, B, C, H, s);
    });
    x->grad_set = true;
    return YB_OK;
  });
  *out = y;
  return YB_OK;
}

// x + m / keep * y with block `blk`'s mask of `branch` (0 attention, 1 MLP)
int op_drop_residual(yb_train* t, TT* x, TT* y, int blk, int branch, const std::string& zname, TT** out) {
  const int B = t->B, dt = t->dt;
  t->cur_label = "residual " + zname;
  YB_REQUIRE(x->C == y->C && x->H == y->H, YB_ERR_INVALID, "train: residual %s: shapes differ", zname.c_str());
  TT* z = new_tensor(t, zname, x->C, x->H);
  YB_PROPAGATE(alloc_data(t, z));
  const long long per_img = (long long)(x->H + 2) * (x->H + 2) * x->C;
  void* xd = x->data; void* yd = y->data; void* zd = z->data;
  FWD_PUSH([=](cudaStream_t s) { return launch_drop_residual(xd, yd, zd, t->drop_masks, blk, branch, dt, B, per_img, s); });
  t->bwd_builders.push_back([=]() -> int {
    t->cur_label = "residual-bwd " + z->name;
    YB_REQUIRE(z->grad && z->grad_set && !y->grad_set, YB_ERR_STATE, "train: residual %s: gradient state", z->name.c_str());
    YB_PROPAGATE(ensure_grad(t, x)); YB_PROPAGATE(ensure_grad(t, y));
    void* dz = z->grad; void* dx = x->grad; void* dy = y->grad; const int acc = x->grad_set ? 1 : 0;
    BWD_PUSH([=](cudaStream_t s) { return launch_drop_residual_bwd(dz, dx, acc, dy, t->drop_masks, blk, branch, dt, B, per_img, s); });
    x->grad_set = true; y->grad_set = true;
    return YB_OK;
  });
  *out = z;
  return YB_OK;
}

// (shifted-)window attention over the qkv linear's output (its only consumer)
int op_attn(yb_train* t, TT* qkv, ConvRec* cq, const std::string& p, int heads, int shift, TT** out) {
  const int B = t->B, dt = t->dt, C = qkv->C / 3, H = qkv->H;
  t->cur_label = "attn " + p;
  YB_REQUIRE(qkv->C == 3 * C && cq->Cout_pad == 3 * C, YB_ERR_INVALID, "train: attention %s: qkv width %d", p.c_str(), qkv->C);
  const std::string tname = p + ".attn.relative_position_bias_table";
  t->add_bound(tname, 169 * heads, 0);
  const int iq = cq->bias_idx, it = t->bidx.at(tname);
  TT* o = new_tensor(t, p + ".attn", C, H);
  YB_PROPAGATE(alloc_data(t, o));
  float* lse = nullptr;
  YB_PROPAGATE(dev_alloc(t, (void**)&lse, (size_t)qkv->rows * heads * 4));
  void* qd = qkv->data; void* od = o->data;
  FWD_PUSH([=](cudaStream_t s) { return launch_wattn_fwd(qd, t->bound[iq].data, t->bound[it].data, od, lse, dt, B, H, C, heads, shift, s); });
  float* dtab = stats_take(t, 169 * (size_t)heads);
  tail_copy(t, dtab, tname, 169 * heads);
  float* dbias = cq->bsum;                                         // the qkv bias sums: the padding tokens' dK / dV land there too
  t->bwd_builders.push_back([=]() -> int {
    t->cur_label = "attn-bwd " + o->name;
    YB_REQUIRE(o->grad && o->grad_set && !qkv->grad_set, YB_ERR_STATE, "train: attention %s: gradient state", o->name.c_str());
    YB_PROPAGATE(ensure_grad(t, qkv));
    void* dout = o->grad; void* dq = qkv->grad;
    BWD_PUSH([=](cudaStream_t s) {
      return launch_wattn_bwd(qd, t->bound[iq].data, t->bound[it].data, dout, lse, dq, (float*)((char*)t->stats + (size_t)dtab),
                              (float*)((char*)t->stats + (size_t)dbias), dt, B, H, C, heads, shift, s);
    });
    qkv->grad_set = true;
    return YB_OK;
  });
  *out = o;
  return YB_OK;
}

// exact-erf GELU of fc1's stored pre-activation (its only consumer)
int op_gelu(yb_train* t, TT* h, const std::string& gname, TT** out) {
  const int dt = t->dt;
  t->cur_label = "gelu " + gname;
  TT* g = new_tensor(t, gname, h->C, h->H);
  YB_PROPAGATE(alloc_data(t, g));
  const long long n = h->rows * h->C;
  void* hd = h->data; void* gd = g->data;
  FWD_PUSH([=](cudaStream_t s) { return launch_gelu_fwd(hd, gd, dt, n, s); });
  t->bwd_builders.push_back([=]() -> int {
    YB_REQUIRE(g->grad && g->grad_set && !h->grad_set, YB_ERR_STATE, "train: GELU %s: gradient state", g->name.c_str());
    YB_PROPAGATE(ensure_grad(t, h));
    void* dg = g->grad; void* dh = h->grad;
    BWD_PUSH([=](cudaStream_t s) { return launch_gelu_bwd(hd, dg, dh, dt, n, s); });
    h->grad_set = true;
    return YB_OK;
  });
  *out = g;
  return YB_OK;
}

// patch-merging gather [x0 | x1 | x2 | x3] (the LayerNorm and the reduction follow as op_ln / op_conv)
int op_merge(yb_train* t, TT* x, const std::string& mname, TT** out) {
  const int B = t->B, dt = t->dt, C = x->C, Hin = x->H, Hout = (Hin + 1) / 2;
  t->cur_label = "merge " + mname;
  TT* m = new_tensor(t, mname, 4 * C, Hout);
  YB_PROPAGATE(alloc_data(t, m));
  void* xd = x->data; void* md = m->data;
  FWD_PUSH([=](cudaStream_t s) { return launch_merge_fwd(xd, md, dt, B, C, Hin, Hout, s); });
  t->bwd_builders.push_back([=]() -> int {
    YB_REQUIRE(m->grad && m->grad_set, YB_ERR_STATE, "train: patch merge %s has no gradient", m->name.c_str());
    YB_PROPAGATE(ensure_grad(t, x));
    void* dm = m->grad; void* dx = x->grad; const int acc = x->grad_set ? 1 : 0;
    BWD_PUSH([=](cudaStream_t s) { return launch_merge_bwd(dm, dx, acc, dt, B, C, Hin, Hout, s); });
    x->grad_set = true;
    return YB_OK;
  });
  *out = m;
  return YB_OK;
}

// Swin-T backbone (modules/swin_transformer.py:436-518, as net.cu's depth-0 program): patch embedding, 4 stages of (shifted-)window
// blocks with stochastic depth, patch merging; couts[1..3] = backbone.norm1..3 (tensors "c3", "c4", "c5")
int build_swin(yb_train* t, std::vector<ConvRec*>* all, TT** couts) {
  const int B = t->B, S = t->S, dt = t->dt, Hg = stem_sizes(S).Hg;
  YB_PROPAGATE(dev_alloc(t, (void**)&t->drop_masks, (size_t)B * kSwinBlocks * 2 * 4));
  {
    float* masks = t->drop_masks;
    t->cur_label = "drop-path masks";
    FWD_PUSH([=](cudaStream_t s) { return launch_drop_path_masks(t->p_seed, masks, B, s); });
  }
  // ---- patch embedding: conv 4x4 / 4 (fp32 output) + LayerNorm; backward: LayerNorm, then the conv's weight and bias gradient ----
  const std::string pe = "backbone.patch_embed";
  t->add_bound(pe + ".proj.weight", 96 * 48, 0); t->add_bound(pe + ".proj.bias", 96, 0);
  t->add_bound(pe + ".norm.weight", 96, 0); t->add_bound(pe + ".norm.bias", 96, 0);
  TT* x = new_tensor(t, "patch_embed", 96, Hg);
  YB_PROPAGATE(alloc_data(t, x));
  {
    t->cur_label = "patch embed";
    const long long rows = x->rows;
    float *raw = nullptr, *draw = nullptr, *st = nullptr;
    YB_PROPAGATE(dev_alloc(t, (void**)&raw, (size_t)rows * 96 * 4));
    YB_PROPAGATE(dev_alloc(t, (void**)&draw, (size_t)rows * 96 * 4));
    YB_PROPAGATE(dev_alloc(t, (void**)&st, (size_t)2 * rows * 4));
    const int iw = t->bidx.at(pe + ".proj.weight"), ib = t->bidx.at(pe + ".proj.bias"), ig = t->bidx.at(pe + ".norm.weight"),
              ibe = t->bidx.at(pe + ".norm.bias");
    float* img = t->d_img; void* xd = x->data;
    FWD_PUSH([=](cudaStream_t s) { return launch_pe_conv(img, t->bound[iw].data, t->bound[ib].data, raw, B, S, Hg, s); });
    FWD_PUSH([=](cudaStream_t s) { return launch_ln_fwd(raw, 1, xd, t->bound[ig].data, t->bound[ibe].data, st, st + rows, dt, B, 96, Hg, s); });
    float* dgb = stats_take(t, 2 * 96);
    float* dwb = stats_take(t, 96 * 48 + 96);
    tail_copy(t, dgb, pe + ".norm.weight", 96); tail_copy(t, dgb + 96, pe + ".norm.bias", 96);
    tail_copy(t, dwb, pe + ".proj.weight", 96 * 48); tail_copy(t, dwb + 96 * 48, pe + ".proj.bias", 96);
    TT* xx = x;
    t->bwd_builders.push_back([=]() -> int {
      t->cur_label = "patch embed bwd";
      YB_REQUIRE(xx->grad && xx->grad_set, YB_ERR_STATE, "train: patch embedding has no gradient");
      void* dy = xx->grad;
      BWD_PUSH([=](cudaStream_t s) {
        return launch_ln_bwd(raw, 1, dy, t->bound[ig].data, st, st + rows, draw, 0, (float*)((char*)t->stats + (size_t)dgb), dt, B, 96, Hg, s);
      });
      BWD_PUSH([=](cudaStream_t s) {
        float* w = (float*)((char*)t->stats + (size_t)dwb);
        return launch_pe_wgrad(img, draw, w, w + 96 * 48, B, S, Hg, s);
      });
      return YB_OK;
    });
  }
  // ---- stages ----
  int blk = 0;
  for (int st = 0; st < 4; ++st) {
    const int C = 96 << st;
    for (int b = 0; b < kSwinDepths[st]; ++b, ++blk) {
      const std::string p = "backbone.layers." + std::to_string(st) + ".blocks." + std::to_string(b);
      TT *t1, *qkv, *att, *y, *x1, *t2, *h, *g, *y2;
      ConvRec *cq, *cp, *c1, *c2;
      YB_PROPAGATE(op_ln(t, x, p + ".norm1", p + ".norm1", &t1));
      YB_PROPAGATE(swin_linear(t, p + ".attn.qkv", C, 3 * C, true, all, &cq));
      YB_PROPAGATE(op_conv(t, t1, cq, 0, false, p + ".attn.qkv", &qkv));
      YB_PROPAGATE(op_attn(t, qkv, cq, p, kSwinHeads[st], (b % 2) ? 3 : 0, &att));
      YB_PROPAGATE(swin_linear(t, p + ".attn.proj", C, C, true, all, &cp));
      YB_PROPAGATE(op_conv(t, att, cp, 0, false, p + ".attn.proj", &y));
      YB_PROPAGATE(op_drop_residual(t, x, y, blk, 0, p + ".x1", &x1));
      YB_PROPAGATE(op_ln(t, x1, p + ".norm2", p + ".norm2", &t2));
      YB_PROPAGATE(swin_linear(t, p + ".mlp.fc1", C, 4 * C, true, all, &c1));
      YB_PROPAGATE(op_conv(t, t2, c1, 0, false, p + ".mlp.fc1", &h));
      YB_PROPAGATE(op_gelu(t, h, p + ".mlp.gelu", &g));
      YB_PROPAGATE(swin_linear(t, p + ".mlp.fc2", 4 * C, C, true, all, &c2));
      YB_PROPAGATE(op_conv(t, g, c2, 0, false, p + ".mlp.fc2", &y2));
      YB_PROPAGATE(op_drop_residual(t, x1, y2, blk, 1, p + ".out", &x));
    }
    if (st > 0) YB_PROPAGATE(op_ln(t, x, "backbone.norm" + std::to_string(st), "c" + std::to_string(st + 2), &couts[st]));
    if (st < 3) {
      const std::string p = "backbone.layers." + std::to_string(st) + ".downsample";
      TT *mg, *mn;
      ConvRec* cr;
      YB_PROPAGATE(op_merge(t, x, p + ".merge", &mg));
      YB_PROPAGATE(op_ln(t, mg, p + ".norm", p + ".norm", &mn));
      YB_PROPAGATE(swin_linear(t, p + ".reduction", 4 * C, 2 * C, false, all, &cr));
      YB_PROPAGATE(op_conv(t, mn, cr, 0, false, p + ".reduction", &x));
    }
  }
  return YB_OK;
}

int build(yb_train* t) {
  const yb_net_config& cfg = t->cfg;
  const int B = t->B, S = cfg.img_size, dt = t->dt;
  t->S = S;
  YB_PROPAGATE(dev_alloc(t, (void**)&t->zeros, 4096 * 4));
  YB_PROPAGATE(dev_alloc(t, (void**)&t->d_img, (size_t)B * 3 * S * S * 4));
  TT* couts[4] = {nullptr, nullptr, nullptr, nullptr};
  std::vector<ConvRec*> all_convs;
  if (cfg.depth == 0) {
    YB_PROPAGATE(build_swin(t, &all_convs, couts));
  } else {

  // ---------------- stem: space-to-depth image -> 4-tap K=64 conv -> BN -> ReLU -> max-pool ----------------
  const StemSizes ss = stem_sizes(S);
  const int H1 = ss.H1, H2 = ss.H2, Wp1 = H1 + 2;
  t->add_bound("backbone.conv1.weight", 64 * 3 * 7 * 7, 0);
  TT* s2d = new_tensor(t, "stem.s2d", 64, H1);            // 4 pixels x 16 channels per row (materialised: rows are self-contained)
  YB_PROPAGATE(alloc_data(t, s2d));
  s2d->needs_grad = false;
  void* w16 = nullptr;
  YB_PROPAGATE(dev_alloc(t, &w16, 64 * 256 * 2));
  TT* sy = new_tensor(t, "stem.y", 64, H1);
  YB_PROPAGATE(alloc_data(t, sy));
  {
    void* s2dd = s2d->data; float* img = t->d_img;
    FWD_PUSH([=](cudaStream_t s) { return launch_stem_s2d(img, s2dd, dt, 1, B, S, H1, s); });
    const int iw = t->bidx.at("backbone.conv1.weight");
    FWD_PUSH([=](cudaStream_t s) { return launch_pack_stem(t->bound[iw].data, w16, dt, s); });
    ConvArgs a; memset(&a, 0, sizeof(a));
    a.in = s2d->data; a.weight = w16; a.bias = t->zeros; a.out = sy->data; a.act_dt = dt; a.B = B; a.g.H = H1; a.g.W = H1;
    a.Cin = 64; a.Cin_pad = 64; a.Cout = 64; a.Cout_pad = 64; a.ntaps = 4; a.relu = 0; a.out_mode = 0;
    stem_taps(Wp1, a.tap_shift);
    a.in_rows = s2d->rows;
    TcPlan* pl = nullptr;
    YB_PROPAGATE(tc_plan_create(a, B, &pl));
    t->plans.push_back(pl);
    FWD_PUSH([=](cudaStream_t s) { return launch_conv_tc(pl, a, s); });
    // backward: weight gradient only (the image needs no gradient): 16 taps (dy, dx) of 16 channels each
    float* dW16 = nullptr;
    YB_PROPAGATE(dev_alloc(t, (void**)&dW16, 64 * 256 * 4));
    t->bwd_builders.push_back([=]() -> int {
      YB_REQUIRE(sy->grad && sy->grad_set, YB_ERR_STATE, "train: stem output has no gradient");
      const long long rows = sy->rows, ldT = (rows + 7) / 8 * 8;
      void* dyT = nullptr;
      YB_PROPAGATE(dev_alloc(t, &dyT, (size_t)64 * ldT * 2));
      void* dy = sy->grad;
      BWD_PUSH([=](cudaStream_t s) { return launch_transpose16(dy, 64, dyT, dt, rows, 64, ldT, s); });
      GemmArgs g; memset(&g, 0, sizeof(g));
      g.a = dyT; g.b = s2dd; g.out = dW16; g.act_dt = dt; g.M = 64; g.Nper = 64; g.K = (int)rows; g.lda = (int)ldT; g.ldb = 64; g.Kb = rows; g.ntaps = 4;
      g.accumulate = 1; g.splits = 74;                              // 4 output tiles, K = every pixel of the batch: split-K
      stem_taps(Wp1, g.shift);                                      // out [64][dy*64 + dx*16 + e]: the packed stem layout
      TcPlan* gp = nullptr;
      YB_PROPAGATE(tc_plan_create_gemm(g, &gp));
      t->plans.push_back(gp);
      BWD_PUSH([=](cudaStream_t s) { return launch_gemm_tc(gp, g, s); });
      BWD_PUSH([=](cudaStream_t s) { return launch_unpack_stem_grad(dW16, t->bound[iw].grad, 1.f, s); });
      return YB_OK;
    });
  }
  TT* sz = nullptr;
  YB_PROPAGATE(op_bn(t, sy, "backbone.bn1", 1, nullptr, "stem.z", &sz));
  TT* x = new_tensor(t, "pool", 64, H2);
  YB_PROPAGATE(alloc_data(t, x));
  {
    void* in = sz->data; void* out = x->data;
    FWD_PUSH([=](cudaStream_t s) { return launch_maxpool(in, out, dt, B, 64, H1, H2, s); });
    TT* xx = x;
    t->bwd_builders.push_back([=]() -> int {
      YB_REQUIRE(xx->grad && xx->grad_set, YB_ERR_STATE, "train: pool output has no gradient");
      YB_PROPAGATE(ensure_grad(t, sz));
      void* dy = xx->grad; void* dx = sz->grad;
      BWD_PUSH([=](cudaStream_t s) { return launch_maxpool_bwd(in, dy, dx, dt, B, 64, H1, H2, s); });
      sz->grad_set = true;
      return YB_OK;
    });
  }

  // ---------------- bottleneck stages (modules/resnet.py:46-98) ----------------
  const int* nblk = resnet_blocks(cfg.depth);
  int inpl = 64;
  for (int st = 0; st < 4; ++st) {
    const int planes = 64 << st;
    for (int b = 0; b < nblk[st]; ++b) {
      const int stride = (b == 0 && st > 0) ? 2 : 1;
      const std::string p = "backbone.layers." + std::to_string(st) + "." + std::to_string(b);
      ConvRec* c1 = new_conv(t, p + ".conv1", inpl, planes, 1, 1, false);
      ConvRec* c2 = new_conv(t, p + ".conv2", planes, planes, 3, stride, false);
      ConvRec* c3 = new_conv(t, p + ".conv3", planes, planes * 4, 1, 1, false);
      for (ConvRec* c : {c1, c2, c3}) { c->bias = t->zeros; YB_PROPAGATE(alloc_conv(t, c, true)); all_convs.push_back(c); }
      TT *y1, *z1, *y2, *z2, *y3, *z3, *r = x;
      YB_PROPAGATE(op_conv(t, x, c1, 0, false, p + ".conv1.y", &y1));
      YB_PROPAGATE(op_bn(t, y1, p + ".bn1", 1, nullptr, p + ".bn1.z", &z1));
      YB_PROPAGATE(op_conv(t, z1, c2, 0, false, p + ".conv2.y", &y2));
      YB_PROPAGATE(op_bn(t, y2, p + ".bn2", 1, nullptr, p + ".bn2.z", &z2));
      if (b == 0) {
        ConvRec* cd = new_conv(t, p + ".downsample.0", inpl, planes * 4, 1, stride, false);
        cd->bias = t->zeros;
        YB_PROPAGATE(alloc_conv(t, cd, true));
        all_convs.push_back(cd);
        TT *yd, *zd;
        YB_PROPAGATE(op_conv(t, x, cd, 0, false, p + ".downsample.y", &yd));
        YB_PROPAGATE(op_bn(t, yd, p + ".downsample.1", 0, nullptr, p + ".downsample.z", &zd));
        r = zd;
      }
      YB_PROPAGATE(op_conv(t, z2, c3, 0, false, p + ".conv3.y", &y3));
      YB_PROPAGATE(op_bn(t, y3, p + ".bn3", 1, r, p + ".out", &z3));
      x = z3;
      inpl = planes * 4;
    }
    couts[st] = x;
  }
  t->by_name["c2"] = couts[0]; t->by_name["c3"] = couts[1]; t->by_name["c4"] = couts[2]; t->by_name["c5"] = couts[3];
  }

  // ---------------- FPN (modules/yolact.py:57-89) ----------------
  const int fin[3] = {couts[1]->C, couts[2]->C, couts[3]->C};
  ConvRec *lat[3], *pred[3], *down[2];
  auto biased = [&](const std::string& prefix, int Cin, int Cout, int k, int stride, ConvRec** out) -> int {
    ConvRec* c = new_conv(t, prefix, Cin, Cout, k, stride, true);
    c->bias = t->zeros; c->bias_idx = t->bidx.at(c->bname);
    YB_PROPAGATE(alloc_conv(t, c, true));
    c->bsum = stats_take(t, 2 * (size_t)(c->Cout_pad < 64 ? 64 : c->Cout_pad));
    all_convs.push_back(c);
    *out = c;
    return YB_OK;
  };
  for (int i = 0; i < 3; ++i) YB_PROPAGATE(biased("fpn.lat_layers." + std::to_string(i), fin[i], 256, 1, 1, &lat[i]));
  for (int i = 0; i < 3; ++i) YB_PROPAGATE(biased("fpn.pred_layers." + std::to_string(i) + ".0", 256, 256, 3, 1, &pred[i]));
  for (int i = 0; i < 2; ++i) YB_PROPAGATE(biased("fpn.downsample_layers." + std::to_string(i) + ".0", 256, 256, 3, 2, &down[i]));
  auto upadd = [&](TT* coarse, TT* fine) {
    void* cd = coarse->data; void* fd = fine->data; const int Hc = coarse->H, Hf = fine->H;
    FWD_PUSH([=](cudaStream_t s) { return launch_upsample_add(cd, fd, dt, B, 256, Hc, Hf, s); });
    t->bwd_builders.push_back([=]() -> int {
      YB_REQUIRE(fine->grad && fine->grad_set, YB_ERR_STATE, "train: FPN level %s has no gradient", fine->name.c_str());
      YB_PROPAGATE(ensure_grad(t, coarse));
      void* df = fine->grad; void* dc = coarse->grad; const int acc = coarse->grad_set ? 1 : 0;
      BWD_PUSH([=](cudaStream_t s) { return launch_bilinear_bwd(df, dc, dt, B, 256, Hc, Hf, 0, acc, s); });
      coarse->grad_set = true;
      return YB_OK;
    });
  };
  TT *p5_1, *p4_1, *p3_1, *lv[5];
  YB_PROPAGATE(op_conv(t, couts[3], lat[2], 0, false, "p5_1", &p5_1));
  YB_PROPAGATE(op_conv(t, couts[2], lat[1], 0, false, "p4_1", &p4_1));
  upadd(p5_1, p4_1);
  YB_PROPAGATE(op_conv(t, couts[1], lat[0], 0, false, "p3_1", &p3_1));
  upadd(p4_1, p3_1);
  YB_PROPAGATE(op_conv(t, p5_1, pred[2], 1, false, "p5", &lv[2]));
  YB_PROPAGATE(op_conv(t, p4_1, pred[1], 1, false, "p4", &lv[1]));
  YB_PROPAGATE(op_conv(t, p3_1, pred[0], 1, false, "p3", &lv[0]));
  YB_PROPAGATE(op_conv(t, lv[2], down[0], 1, false, "p6", &lv[3]));
  YB_PROPAGATE(op_conv(t, lv[3], down[1], 1, false, "p7", &lv[4]));

  // ---------------- ProtoNet (modules/yolact.py:34-53) ----------------
  const int K = cfg.coef_dim, NC = cfg.num_classes, R = cfg.num_ratios;
  TT* q = lv[0];
  for (int i : {0, 2, 4}) {
    ConvRec* c; TT* o;
    YB_PROPAGATE(biased("proto_net.proto1." + std::to_string(i), 256, 256, 3, 1, &c));
    YB_PROPAGATE(op_conv(t, q, c, 1, false, "proto1." + std::to_string(i), &o));
    q = o;
  }
  TT* up = new_tensor(t, "proto.up", 256, 2 * q->H);
  YB_PROPAGATE(alloc_data(t, up));
  {
    void* in = q->data; void* out = up->data; const int Hin = q->H; TT* qq = q;
    FWD_PUSH([=](cudaStream_t s) { return launch_upsample2x_ac(in, out, dt, B, 256, Hin, s); });
    t->bwd_builders.push_back([=]() -> int {
      YB_REQUIRE(up->grad && up->grad_set, YB_ERR_STATE, "train: proto up-sample has no gradient");
      YB_PROPAGATE(ensure_grad(t, qq));
      void* df = up->grad; void* dc = qq->grad; const int acc = qq->grad_set ? 1 : 0;
      BWD_PUSH([=](cudaStream_t s) { return launch_bilinear_bwd(df, dc, dt, B, 256, Hin, 2 * Hin, 1, acc, s); });
      qq->grad_set = true;
      return YB_OK;
    });
  }
  ConvRec *pc0, *pc2;
  TT *pq, *protoT;
  YB_PROPAGATE(biased("proto_net.proto2.0", 256, 256, 3, 1, &pc0));
  YB_PROPAGATE(op_conv(t, up, pc0, 1, false, "proto2.0", &pq));
  YB_PROPAGATE(biased("proto_net.proto2.2", 256, K, 1, 1, &pc2));
  YB_PROPAGATE(op_conv(t, pq, pc2, 1, true, "proto", &protoT));
  t->P = protoT->H; t->proto = (float*)protoT->data;
  YB_PROPAGATE(dev_alloc(t, (void**)&t->g_proto, (size_t)B * t->P * t->P * K * 4));

  // ---------------- prediction head (shared over 5 levels) + semantic segmentation conv ----------------
  ConvRec* upf;
  YB_PROPAGATE(biased("prediction_layers.upfeature.0", 256, 256, 3, 1, &upf));
  std::unique_ptr<ConvRec> hu(new ConvRec());
  ConvRec* hc = hu.get();
  t->convs.push_back(std::move(hu));
  const HeadLayout hl = head_layout(cfg);
  hc->Cin = 256; hc->Cin_pad = 256; hc->k = 3; hc->stride = 1; hc->Cout = hl.Cout; hc->Cout_pad = hl.Cout_pad;
  hc->CoutT_pad = (hc->Cout_pad + 63) / 64 * 64;
  hc->cat = hl.cat;
  for (const auto& p : hl.params) t->add_bound(p.first, p.second, 0);
  YB_PROPAGATE(alloc_conv(t, hc, true));
  YB_PROPAGATE(dev_alloc(t, (void**)&hc->bias_cat, (size_t)hc->Cout_pad * 4));
  hc->bias = hc->bias_cat;
  hc->bsum = stats_take(t, 2 * (size_t)hc->Cout_pad);
  all_convs.push_back(hc);
  {
    int row = 0;
    for (const auto& n : hc->cat) {
      const int ib = t->bidx.at(n + ".bias"), cnt = (int)t->bound[ib].count;
      float* dst = hc->bias_cat + row;
      FWD_PUSH([=](cudaStream_t s) { return launch_scale_copy(t->bound[ib].data, dst, cnt, 1.f, s); });
      row += cnt;
    }
  }
  for (int l = 0; l < 5; ++l) t->level_size[l] = lv[l]->H;
  t->A = level_offsets(t->level_size, R, t->level_off);
  const size_t BA = (size_t)B * t->A;
  YB_PROPAGATE(dev_alloc(t, (void**)&t->cls, BA * NC * 4)); YB_PROPAGATE(dev_alloc(t, (void**)&t->box, BA * 16)); YB_PROPAGATE(dev_alloc(t, (void**)&t->coef, BA * K * 4));
  YB_PROPAGATE(dev_alloc(t, (void**)&t->g_cls, BA * NC * 4)); YB_PROPAGATE(dev_alloc(t, (void**)&t->g_box, BA * 16)); YB_PROPAGATE(dev_alloc(t, (void**)&t->g_coef, BA * K * 4));
  for (int l = 0; l < 5; ++l) {
    TT *f, *h;
    YB_PROPAGATE(op_conv(t, lv[l], upf, 1, false, "head.f" + std::to_string(l), &f));
    // the head's dY is built from the loss gradients right before the conv's backward runs: register that builder AFTER op_conv's
    // (builders run in reverse), so insert a placeholder order: op_conv(head) first, then the scatter builder
    YB_PROPAGATE(op_conv(t, f, hc, 0, true, "head.h" + std::to_string(l), &h));
    {
      const float* hd = (const float*)h->data; const int ld = hc->Cout_pad, HW = lv[l]->H * lv[l]->H, aoff = t->level_off[l], A = t->A, Hl = lv[l]->H;
      float *cls = t->cls, *box = t->box, *coef = t->coef;
      FWD_PUSH([=](cudaStream_t s) { return launch_head_train(hd, ld, B, HW, R, NC, K, aoff, A, cls, box, coef, s); });
      TT* hh = h;
      t->bwd_builders.push_back([=]() -> int {
        YB_PROPAGATE(ensure_grad(t, hh));
        void* g = hh->grad; const int ldo = hh->Cg;
        float *gc = t->g_cls, *gb = t->g_box, *gk = t->g_coef;
        BWD_PUSH([=](cudaStream_t s) { return launch_head_grad(gc, gb, gk, coef, dt, B, Hl, R, NC, K, aoff, A, ldo, g, s); });
        hh->grad_set = true;
        return YB_OK;
      });
    }
  }
  ConvRec* sc;
  TT* segT;
  YB_PROPAGATE(biased("semantic_seg_conv", 256, NC - 1, 1, 1, &sc));
  YB_PROPAGATE(op_conv(t, lv[0], sc, 0, true, "seg", &segT));
  t->Hs = segT->H; t->seg = (float*)segT->data; t->ld_seg = sc->Cout_pad;
  YB_PROPAGATE(dev_alloc(t, (void**)&t->g_seg, (size_t)B * t->Hs * t->Hs * t->ld_seg * 4));
  {
    TT* ss = segT; TT* pp = protoT;
    t->bwd_builders.push_back([=]() -> int {
      YB_PROPAGATE(ensure_grad(t, ss)); YB_PROPAGATE(ensure_grad(t, pp));
      void* gs = ss->grad; void* gp = pp->grad; const int Cs = ss->Cg, Cp = pp->Cg, Hs = t->Hs, P = t->P, lds = t->ld_seg;
      float *dseg = t->g_seg, *dproto = t->g_proto, *proto = t->proto;
      BWD_PUSH([=](cudaStream_t s) { return launch_dense_to_haloed(dseg, nullptr, lds, NC - 1, gs, dt, B, Cs, Hs, s); });
      BWD_PUSH([=](cudaStream_t s) { return launch_dense_to_haloed(dproto, proto, K, K, gp, dt, B, Cp, P, s); });
      ss->grad_set = true; pp->grad_set = true;
      return YB_OK;
    });
  }

  // the builders above were registered in forward order EXCEPT that a dense output's gradient scatter must run BEFORE its conv's
  // backward: they were registered after the conv (so they run first in the reversed order) -- as required.
  t->anchors = default_anchors(cfg, t->level_size);
  YB_PROPAGATE(dev_alloc(t, (void**)&t->d_anchors, t->anchors.size() * 4));
  YB_CHECK_CUDA(cudaMemcpy(t->d_anchors, t->anchors.data(), t->anchors.size() * 4, cudaMemcpyHostToDevice));
  YB_PROPAGATE(dev_alloc(t, (void**)&t->d_losses_scratch, 16));

  // ---------------- backward program: run the builders in reverse op order ----------------
  for (size_t i = t->bwd_builders.size(); i-- > 0;) YB_PROPAGATE(t->bwd_builders[i]());
  // bias gradients and the packed weight gradients -> the bound gradient buffers
  for (ConvRec* c : all_convs) {
    if (!c->bname.empty()) {
      const int ib = t->bidx.at(c->bname), cnt = c->Cout; float* bs = c->bsum;
      t->bwd_tail.push_back([=](cudaStream_t s) { return launch_scale_copy((float*)((char*)t->stats + (size_t)bs), t->bound[ib].grad, cnt, 1.f, s); });
    } else if (!c->cat.empty()) {
      int row = 0;
      for (const auto& n : c->cat) {
        const int ib = t->bidx.at(n + ".bias"), cnt = (int)t->bound[ib].count; float* bs = c->bsum; const int r0 = row;
        t->bwd_tail.push_back([=](cudaStream_t s) { return launch_scale_copy((float*)((char*)t->stats + (size_t)bs) + r0, t->bound[ib].grad, cnt, 1.f, s); });
        row += cnt;
      }
    }
    add_pack_descs(t, c);
  }
  // the per-step zeroed statistics arena
  YB_PROPAGATE(dev_alloc(t, (void**)&t->stats, t->stats_floats * 4 + 256));
  YB_PROPAGATE(dev_alloc(t, (void**)&t->d_pack, t->pack_descs.size() * sizeof(PackDesc)));
  YB_PROPAGATE(dev_alloc(t, (void**)&t->d_unpack, t->unpack_descs.size() * sizeof(UnpackDesc)));
  // loss workspace (re-grown on demand in forward when a batch brings more ground truth)
  t->built = true;
  return YB_OK;
}

int resolve_descs(yb_train* t) {
  // parameters may be re-bound between steps: resolve the descriptor tables from the current bindings
  std::vector<PackDesc> pd = t->pack_descs;
  for (auto& d : pd) d.src = t->bound[(int)(uintptr_t)d.src].data;
  std::vector<UnpackDesc> ud = t->unpack_descs;
  for (auto& u : ud) u.dst = t->bound[(int)(uintptr_t)u.dst].grad;
  YB_CHECK_CUDA(cudaMemcpy(t->d_pack, pd.data(), pd.size() * sizeof(PackDesc), cudaMemcpyHostToDevice));
  YB_CHECK_CUDA(cudaMemcpy(t->d_unpack, ud.data(), ud.size() * sizeof(UnpackDesc), cudaMemcpyHostToDevice));
  return YB_OK;
}

}  // namespace

// ================================================================================================
extern "C" int yb_train_create(const yb_net_config* cfg, int batch, int precision, yb_train** out) {
  YB_REQUIRE(cfg && out, YB_ERR_INVALID, "yb_train_create: NULL argument");
  YB_REQUIRE(cfg->depth == 50 || cfg->depth == 101 || cfg->depth == 0, YB_ERR_UNSUPPORTED,
             "yb_train_create: depth=%d (the training engine covers ResNet-50 / 101 and Swin-T, depth 0)", cfg->depth);
  YB_REQUIRE(batch >= 1 && batch <= 256, YB_ERR_INVALID, "yb_train_create: batch=%d", batch);
  YB_REQUIRE(precision == YB_PREC_BF16 || precision == YB_PREC_FP16, YB_ERR_UNSUPPORTED, "yb_train_create: precision=%d (bf16 or fp16 operands)", precision);
  YB_REQUIRE(cfg->coef_dim == 32 && cfg->num_ratios >= 1 && cfg->num_ratios <= 3 && cfg->num_classes >= 2 && cfg->num_classes <= YB_MAX_CLASSES, YB_ERR_UNSUPPORTED,
             "yb_train_create: coef_dim=%d num_ratios=%d num_classes=%d", cfg->coef_dim, cfg->num_ratios, cfg->num_classes);
  int cc_major = 0;
  YB_PROPAGATE(yb_device_info(nullptr, &cc_major, nullptr));
  YB_REQUIRE(cc_major == 9, YB_ERR_UNSUPPORTED, "yb_train_create: this library is built for sm_90a only (device cc major %d)", cc_major);
  yb_train* t = new yb_train();
  t->cfg = *cfg; t->B = batch; t->dt = precision == YB_PREC_BF16 ? DT_BF16 : DT_F16;
  t->hp.bn_momentum = 0.1f; t->hp.bn_eps = 1e-5f;
  const int st = build(t);
  if (st != YB_OK) { yb_train_destroy(t); return st; }
  *out = t;
  return YB_OK;
}

extern "C" void yb_train_destroy(yb_train* t) {
  if (!t) return;
  if (t->g_fwd) cudaGraphExecDestroy(t->g_fwd);
  if (t->g_bwd) cudaGraphExecDestroy(t->g_bwd);
  if (t->ev_in) cudaEventDestroy(t->ev_in);
  if (t->ev_out) cudaEventDestroy(t->ev_out);
  if (t->gstream) cudaStreamDestroy(t->gstream);
  for (TcPlan* p : t->plans) tc_plan_destroy(p);
  for (void* p : t->allocs) cudaFree(p);
  if (t->loss_ws) cudaFree(t->loss_ws);
  if (t->p_masks) cudaFree(t->p_masks);
  delete t;
}

extern "C" int yb_train_num_tensors(const yb_train* t) { return t ? (int)t->bound.size() : 0; }

extern "C" int yb_train_tensor_info(const yb_train* t, int i, const char** name, int64_t* count, int* kind) {
  YB_REQUIRE(t && i >= 0 && i < (int)t->bound.size(), YB_ERR_INVALID, "yb_train_tensor_info: index %d", i);
  if (name) *name = t->bound[i].name.c_str();
  if (count) *count = t->bound[i].count;
  if (kind) *kind = t->bound[i].kind;
  return YB_OK;
}

extern "C" int yb_train_bind(yb_train* t, const char* name, float* data, float* grad) {
  YB_REQUIRE(t && name && data, YB_ERR_INVALID, "yb_train_bind: NULL argument");
  auto it = t->bidx.find(name);
  YB_REQUIRE(it != t->bidx.end(), YB_ERR_INVALID, "yb_train_bind: unexpected tensor '%s'", name);
  BoundTensor& b = t->bound[it->second];
  YB_REQUIRE(b.kind == 1 || grad != nullptr, YB_ERR_INVALID, "yb_train_bind: parameter '%s' needs a gradient buffer", name);
  b.data = data; b.grad = grad;
  t->descs_dirty = true;
  return YB_OK;
}

extern "C" int yb_train_set_anchors(yb_train* t, const float* anchors_host, int n) {
  YB_REQUIRE(t && anchors_host && n == t->A, YB_ERR_INVALID, "yb_train_set_anchors: %d anchors, the network has %d", n, t ? t->A : 0);
  t->anchors.assign(anchors_host, anchors_host + (size_t)n * 4);
  YB_CHECK_CUDA(cudaMemcpy(t->d_anchors, t->anchors.data(), t->anchors.size() * 4, cudaMemcpyHostToDevice));
  return YB_OK;
}

namespace {
void drop_graphs(yb_train* t) {
  if (t->g_fwd) cudaGraphExecDestroy(t->g_fwd);
  if (t->g_bwd) cudaGraphExecDestroy(t->g_bwd);
  t->g_fwd = t->g_bwd = nullptr;
}

yb_loss_params loss_params(const yb_train* t) {
  yb_loss_params p; memset(&p, 0, sizeof(p));
  p.batch = t->B; p.num_anchors = t->A; p.num_classes = t->cfg.num_classes; p.coef_dim = t->cfg.coef_dim; p.proto_size = t->P; p.seg_size = t->Hs;
  p.mask_size = t->S; p.pos_iou_thr = t->hp.pos_iou_thr; p.neg_iou_thr = t->hp.neg_iou_thr; p.neg_pos_ratio = t->hp.neg_pos_ratio;
  p.masks_to_train = t->hp.masks_to_train; p.conf_alpha = t->hp.conf_alpha; p.bbox_alpha = t->hp.bbox_alpha; p.mask_alpha = t->hp.mask_alpha;
  p.semantic_alpha = t->hp.semantic_alpha;
  return p;
}

// grids and workspace are sized for the CAPACITY of the target buffers (the kernels read the real counts from p_gt_off), so the
// same launch sequence can be replayed from a CUDA graph whatever the step's ground truth is
int run_losses(yb_train* t, bool with_grads, cudaStream_t s) {
  const yb_loss_params p = loss_params(t);
  return losses_impl(&p, t->cls, t->box, t->coef, t->proto, t->seg, t->ld_seg, t->d_anchors, t->p_gt, t->p_gt_off, t->p_masks, t->mask_cap, kLossMaxGt, 0,
                     t->p_seed, with_grads ? t->p_loss_grad : nullptr, with_grads ? t->d_losses_scratch : t->p_losses, with_grads ? t->g_cls : nullptr,
                     with_grads ? t->g_box : nullptr, with_grads ? t->g_coef : nullptr, with_grads ? t->g_proto : nullptr, with_grads ? t->g_seg : nullptr,
                     nullptr, nullptr, nullptr, nullptr, t->loss_ws, t->loss_ws_bytes, s);
}

int ensure_target_capacity(yb_train* t, int total_gt, cudaStream_t s) {
  if (!t->p_gt) {
    YB_PROPAGATE(dev_alloc(t, (void**)&t->p_gt, (size_t)t->B * kLossMaxGt * 5 * 4));
    YB_PROPAGATE(dev_alloc(t, (void**)&t->p_gt_off, (size_t)(t->B + 1) * 4));
    YB_PROPAGATE(dev_alloc(t, (void**)&t->p_loss_grad, 16)); YB_PROPAGATE(dev_alloc(t, (void**)&t->p_losses, 16)); YB_PROPAGATE(dev_alloc(t, (void**)&t->p_seed, 16));
  }
  if (total_gt > t->mask_cap) {
    YB_CHECK_CUDA(cudaStreamSynchronize(s));
    drop_graphs(t);
    if (t->p_masks) cudaFree(t->p_masks);
    if (t->loss_ws) cudaFree(t->loss_ws);
    t->p_masks = nullptr; t->loss_ws = nullptr;
    t->mask_cap = total_gt < 16 ? 32 : 2 * total_gt;
    YB_CHECK_CUDA(cudaMalloc(&t->p_masks, (size_t)t->mask_cap * t->S * t->S * 4));
    const yb_loss_params p = loss_params(t);
    t->loss_ws_bytes = yb_losses_workspace_bytes(&p, t->mask_cap);
    YB_CHECK_CUDA(cudaMalloc(&t->loss_ws, t->loss_ws_bytes));
  }
  return YB_OK;
}

int forward_list(yb_train* t, cudaStream_t s) {
  static const bool dbg = getenv("YOLACT_B200_TRAIN_DEBUG") != nullptr;
  YB_CHECK_CUDA(cudaMemsetAsync(t->stats, 0, t->stats_floats * 4, s));
  YB_PROPAGATE(launch_pack_weights(t->d_pack, (int)t->pack_descs.size(), t->dt, s));
  for (size_t i = 0; i < t->fwd.size(); ++i) {
    YB_PROPAGATE(t->fwd[i](s));
    if (dbg) { cudaError_t e = cudaStreamSynchronize(s); YB_REQUIRE(e == cudaSuccess, YB_ERR_CUDA, "train debug: forward launch %zu (%s): %s", i, t->fwd_what[i].c_str(), cudaGetErrorString(e)); }
  }
  YB_PROPAGATE(run_losses(t, false, s));
  if (dbg) { cudaError_t e = cudaStreamSynchronize(s); YB_REQUIRE(e == cudaSuccess, YB_ERR_CUDA, "train debug: losses: %s", cudaGetErrorString(e)); }
  return YB_OK;
}

int backward_list(yb_train* t, cudaStream_t s) {
  static const bool dbg = getenv("YOLACT_B200_TRAIN_DEBUG") != nullptr;
  YB_CHECK_CUDA(cudaMemsetAsync(t->stats, 0, t->stats_floats * 4, s));    // BN reductions / bias sums of this pass start from zero
  YB_PROPAGATE(run_losses(t, true, s));
  if (dbg) { cudaError_t e = cudaStreamSynchronize(s); YB_REQUIRE(e == cudaSuccess, YB_ERR_CUDA, "train debug: loss gradients: %s", cudaGetErrorString(e)); }
  for (size_t i = 0; i < t->bwd.size(); ++i) {
    YB_PROPAGATE(t->bwd[i](s));
    if (dbg) { cudaError_t e = cudaStreamSynchronize(s); YB_REQUIRE(e == cudaSuccess, YB_ERR_CUDA, "train debug: backward launch %zu (%s): %s", i, t->bwd_what[i].c_str(), cudaGetErrorString(e)); }
  }
  for (auto& f : t->bwd_tail) YB_PROPAGATE(f(s));
  YB_PROPAGATE(launch_unpack_wgrad(t->d_unpack, (int)t->unpack_descs.size(), s));
  return YB_OK;
}

// replay `list` from a CUDA graph (captured on first use) on the engine's own stream, ordered after / before the caller's stream by
// events; any capture problem falls back to plain launches on the caller's stream for good
int run_graphed(yb_train* t, cudaGraphExec_t* exec, int (*list)(yb_train*, cudaStream_t), cudaStream_t s, uint64_t* launches) {
  static const bool off = getenv("YOLACT_B200_TRAIN_NO_GRAPH") != nullptr || getenv("YOLACT_B200_TRAIN_DEBUG") != nullptr;
  const uint64_t l0 = yb_launch_count();
  if (off || !t->use_graphs) { const int st = list(t, s); *launches = yb_launch_count() - l0; return st; }
  if (!t->gstream) {
    if (cudaStreamCreateWithFlags(&t->gstream, cudaStreamNonBlocking) != cudaSuccess || cudaEventCreateWithFlags(&t->ev_in, cudaEventDisableTiming) != cudaSuccess ||
        cudaEventCreateWithFlags(&t->ev_out, cudaEventDisableTiming) != cudaSuccess) {
      cudaGetLastError(); t->use_graphs = false;
      return run_graphed(t, exec, list, s, launches);
    }
  }
  YB_CHECK_CUDA(cudaEventRecord(t->ev_in, s));
  YB_CHECK_CUDA(cudaStreamWaitEvent(t->gstream, t->ev_in, 0));
  if (!*exec) {
    cudaGraph_t graph = nullptr;
    bool ok = cudaStreamBeginCapture(t->gstream, cudaStreamCaptureModeThreadLocal) == cudaSuccess;
    int st = YB_OK;
    if (ok) {
      st = list(t, t->gstream);
      ok = cudaStreamEndCapture(t->gstream, &graph) == cudaSuccess && st == YB_OK && graph != nullptr;
    }
    if (ok) ok = cudaGraphInstantiate(exec, graph, 0) == cudaSuccess;
    if (graph) cudaGraphDestroy(graph);
    if (!ok) {
      cudaGetLastError();
      *exec = nullptr; t->use_graphs = false;
      if (st != YB_OK) return st;
      return run_graphed(t, exec, list, s, launches);             // plain launches on the caller's stream
    }
    *launches = yb_launch_count() - l0;                            // kernels per replay
  }
  YB_CHECK_CUDA(cudaGraphLaunch(*exec, t->gstream));
  count_launch(*launches);
  YB_CHECK_CUDA(cudaEventRecord(t->ev_out, t->gstream));
  YB_CHECK_CUDA(cudaStreamWaitEvent(s, t->ev_out, 0));
  return YB_OK;
}
}  // namespace

extern "C" int yb_train_forward(yb_train* t, const float* img, const float* gt, const int32_t* gt_offset, const float* gt_masks, int total_gt,
                                int max_gt_per_image, const yb_train_hparams* hp, uint32_t seed, float* losses, void* stream) {
  YB_REQUIRE(t && img && gt && gt_offset && gt_masks && hp && losses, YB_ERR_INVALID, "yb_train_forward: NULL argument");
  YB_REQUIRE(t->built, YB_ERR_STATE, "yb_train_forward: engine not built");
  for (const auto& b : t->bound) YB_REQUIRE(b.data != nullptr, YB_ERR_STATE, "yb_train_forward: tensor '%s' was never bound", b.name.c_str());
  YB_REQUIRE(hp->masks_to_train >= 1 && hp->neg_pos_ratio >= 1, YB_ERR_INVALID, "yb_train_forward: hparams");
  cudaStream_t s = (cudaStream_t)stream;
  YB_REQUIRE(total_gt >= 1 && total_gt <= t->B * kLossMaxGt && max_gt_per_image <= kLossMaxGt, YB_ERR_UNSUPPORTED,
             "yb_train_forward: %d ground-truth instances (max %d per image)", total_gt, kLossMaxGt);
  if (memcmp(&t->g_hp, hp, sizeof(*hp)) != 0) { drop_graphs(t); t->g_hp = *hp; }       // hyper-parameters are baked into the captured launches
  t->hp = *hp;
  if (t->descs_dirty) { YB_PROPAGATE(resolve_descs(t)); t->descs_dirty = false; drop_graphs(t); }   // so are the bound pointers
  YB_PROPAGATE(ensure_target_capacity(t, total_gt, s));
  t->cur_gt = gt;                                                    // (marks "forward was called"; the kernels read the copies below)
  t->seed_host = seed;
  YB_CHECK_CUDA(cudaMemcpyAsync(t->d_img, img, (size_t)t->B * 3 * t->S * t->S * 4, cudaMemcpyDeviceToDevice, s));
  YB_CHECK_CUDA(cudaMemcpyAsync(t->p_gt, gt, (size_t)total_gt * 5 * 4, cudaMemcpyDeviceToDevice, s));
  YB_CHECK_CUDA(cudaMemcpyAsync(t->p_gt_off, gt_offset, (size_t)(t->B + 1) * 4, cudaMemcpyDeviceToDevice, s));
  YB_CHECK_CUDA(cudaMemcpyAsync(t->p_masks, gt_masks, (size_t)total_gt * t->S * t->S * 4, cudaMemcpyDeviceToDevice, s));
  YB_CHECK_CUDA(cudaMemcpyAsync(t->p_seed, &t->seed_host, 4, cudaMemcpyHostToDevice, s));
  YB_PROPAGATE(run_graphed(t, &t->g_fwd, forward_list, s, &t->launches_fwd));
  YB_CHECK_CUDA(cudaMemcpyAsync(losses, t->p_losses, 16, cudaMemcpyDeviceToDevice, s));
  return YB_OK;
}

extern "C" int yb_train_backward(yb_train* t, const float* loss_grad, void* stream) {
  YB_REQUIRE(t, YB_ERR_INVALID, "yb_train_backward: NULL argument");
  YB_REQUIRE(t->cur_gt != nullptr, YB_ERR_STATE, "yb_train_backward: call yb_train_forward first");
  cudaStream_t s = (cudaStream_t)stream;
  if (loss_grad) YB_CHECK_CUDA(cudaMemcpyAsync(t->p_loss_grad, loss_grad, 16, cudaMemcpyDeviceToDevice, s));
  else { const float one[4] = {1.f, 1.f, 1.f, 1.f}; YB_CHECK_CUDA(cudaMemcpyAsync(t->p_loss_grad, one, 16, cudaMemcpyHostToDevice, s)); }
  YB_PROPAGATE(run_graphed(t, &t->g_bwd, backward_list, s, &t->launches_bwd));
  return YB_OK;
}

extern "C" uint64_t yb_train_launches_per_step(const yb_train* t) { return t ? t->launches_fwd + t->launches_bwd : 0; }

extern "C" int yb_train_read(yb_train* t, const char* name, int grad, float* out, int64_t out_count, int* C, int* H, void* stream) {
  YB_REQUIRE(t && name, YB_ERR_INVALID, "yb_train_read: NULL argument");
  {  // the network outputs the losses consume (dense fp32): "out.cls" [B,A,C], "out.box" [B,A,4], "out.coef" [B,A,K], "out.proto"
     // [B,P,P,K], "out.seg" [B,Hs,Hs,ld]; Swin-T: the step's stochastic-depth masks "out.drop_path" [B,12,2] -- C / H report the last
     // two extents
    const std::string n(name);
    const float* src = nullptr; int64_t cnt = 0; int c = 0, h = 0;
    if (n == "out.cls") { src = t->cls; c = t->cfg.num_classes; h = t->A; cnt = (int64_t)t->B * t->A * c; }
    else if (n == "out.box") { src = t->box; c = 4; h = t->A; cnt = (int64_t)t->B * t->A * 4; }
    else if (n == "out.coef") { src = t->coef; c = t->cfg.coef_dim; h = t->A; cnt = (int64_t)t->B * t->A * c; }
    else if (n == "out.proto") { src = t->proto; c = t->cfg.coef_dim; h = t->P; cnt = (int64_t)t->B * t->P * t->P * c; }
    else if (n == "out.seg") { src = t->seg; c = t->ld_seg; h = t->Hs; cnt = (int64_t)t->B * t->Hs * t->Hs * c; }
    else if (n == "out.drop_path" && t->drop_masks) { src = t->drop_masks; c = 2; h = kSwinBlocks; cnt = (int64_t)t->B * kSwinBlocks * 2; }
    if (src) {
      YB_REQUIRE(!grad, YB_ERR_UNSUPPORTED, "yb_train_read: '%s' has no readable gradient", name);
      if (C) *C = c;
      if (H) *H = h;
      if (!out) return YB_OK;
      YB_REQUIRE(out_count >= cnt, YB_ERR_INVALID, "yb_train_read: output too small");
      YB_CHECK_CUDA(cudaMemcpyAsync(out, src, (size_t)cnt * 4, cudaMemcpyDeviceToDevice, (cudaStream_t)stream));
      return YB_OK;
    }
  }
  auto it = t->by_name.find(name);
  YB_REQUIRE(it != t->by_name.end(), YB_ERR_INVALID, "yb_train_read: unknown tensor '%s'", name);
  const TT* x = it->second;
  YB_REQUIRE(!x->dense && x->planes == 1, YB_ERR_UNSUPPORTED, "yb_train_read: '%s' is not a haloed activation", name);
  const int Cc = grad ? x->Cg : x->C;
  if (C) *C = Cc;
  if (H) *H = x->H;
  if (!out) return YB_OK;
  const void* src = grad ? x->grad : x->data;
  YB_REQUIRE(src != nullptr, YB_ERR_STATE, "yb_train_read: '%s' has no %s", name, grad ? "gradient" : "data");
  YB_REQUIRE(out_count >= (int64_t)t->B * Cc * x->H * x->H, YB_ERR_INVALID, "yb_train_read: output too small");
  return launch_read_activation(src, t->dt, t->B, Cc, x->H, out, (cudaStream_t)stream);
}
