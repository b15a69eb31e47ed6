// Host side of the network: parameter table with the reference's state-dict names, BN folding
// and weight packing, the flat layer program (modules/resnet.py:86-98 + modules/yolact.py:73-89,
// :49-53, :26-31, :141-164 restated as a list of GEMM-shaped convs on haloed NHWC tensors),
// a liveness-based activation arena, and the yb_net_* C ABI.
#include "arch.cuh"
#include "layers.cuh"

#include <math.h>
#include <stdlib.h>
#include <string.h>
#include <algorithm>
#include <map>
#include <memory>
#include <string>
#include <vector>

using namespace yb;

namespace {

struct Param {
  std::string name;
  int64_t count;
  std::vector<float> data;
  bool set = false;
};

struct ActBuf {
  int C = 0, H = 0;            // logical channels / valid side (square feature maps)
  int planes = 1;              // >1 for parity-split tensors
  int dt = DT_F32;
  size_t bytes = 0;            // for max_batch
  int first = 0, last = 0;     // op indices (liveness)
  int slot = -1;
  bool dense_f32 = false;      // dense [B*H*W][C] fp32 scratch (head outputs)
  int pad_rows = 0;            // extra pixel rows allocated behind the last image (stem space-to-depth image, see OP_STEM)
};

enum OpKind { OP_STEM, OP_POOL, OP_SPLIT, OP_CONV, OP_UPADD, OP_UP2X, OP_HEADFIN, OP_PATCH_EMBED, OP_LN, OP_ATTN, OP_MERGE_LN, OP_BNECK };
enum ExtOut { EXT_NONE = 0, EXT_PROTO = 1 };

struct ConvW {                 // one packed convolution
  std::string wname, bname, bnname;   // weight / bias / batch-norm prefix ("" if absent)
  std::vector<std::string> cat;        // head: concatenated convs (conf|box|coef)
  int Cin = 0, Cin_pad = 0, Cout = 0, Cout_pad = 0, k = 1;
  void* d_w = nullptr;         // packed [Cout_alloc][k*k*Cin] in act dtype
  float* d_b = nullptr;        // [Cout_alloc]
};

struct Op {
  OpKind kind;
  int in = -1, out = -1, res = -1;
  int conv = -1;               // index into convs
  int stride = 1, relu = 0, out_mode = 0, ext = EXT_NONE;
  int level = 0;               // head level
  int aux = -1;                // extra scratch activation (stem: space-to-depth image)
  std::string p0, p1, p2;      // Swin ops: parameter names (LayerNorm weight/bias; attention: qkv bias, rel-pos table)
  int heads = 0, shift = 0;    // attention
  TcPlan* tc = nullptr;
  // OP_BNECK (fuse_bottlenecks): conv3 (`conv`, in, res -> out) of one bottleneck chained into conv1 (`conv2`, out -> out2) of the next
  int conv2 = -1, out2 = -1;
  BnPlan* bn = nullptr;
  // ... and, for the first block of a stage, the 1x1 downsample convolution (`convd`, in2 -> the residual) folded into the first GEMM:
  // weights of conv3 and downsample side by side along K (`d_wcat`), biases summed (`d_bcat`); no residual tensor exists any more
  int convd = -1, in2 = -1;
  void* d_wcat = nullptr;
  float* d_bcat = nullptr;
};

}  // namespace

struct yb_net {
  yb_net_config cfg{};
  std::vector<Param> params;
  std::map<std::string, int> pidx;
  std::vector<ActBuf> acts;
  std::vector<ConvW> convs;
  std::vector<Op> ops;                      // the program that runs (finalize: ops_base with the fusable pairs merged)
  std::vector<Op> ops_base;                 // one op per reference layer, as build_program wrote it
  std::map<std::string, int> taps;          // debug taps: name -> act
  std::vector<void*> slots;
  std::vector<size_t> slot_bytes;
  bool finalized = false;
  int max_batch = 0, precision = 0, act_dt = DT_F32;
  int H1 = 0, H2 = 0;
  int level_size[5]{}, level_off[5]{};
  int A = 0, P = 0;
  std::vector<float> anchors;               // [A,4]
  float* d_anchors = nullptr;
  float* d_stem_w = nullptr;                // [7][7][3][64]
  float* d_stem_b = nullptr;
  std::map<std::string, float*> d_vec;      // Swin: LayerNorm / attention parameters on the device (fp32)
  float* d_pe_w = nullptr;                  // Swin patch embedding weights [48][96]
  void* d_stem_w16 = nullptr;               // 16-bit modes: [64][256] GEMM weights (k = dy*64 + dx*16 + (py*2+px)*3+ci)
  int stem_wide = 0;                        // s2d rows materialised 4 pixels wide (driver refused overlapping tensor-map rows)
  float* d_stem_b16 = nullptr;
  ConvArgs stem_args{};
  // scratch for yb_net_detect_host
  float *d_img = nullptr, *d_cls = nullptr, *d_box = nullptr, *d_coef = nullptr, *d_proto = nullptr;
  void* d_ws = nullptr; size_t ws_bytes = 0;
  int32_t *d_cnt = nullptr, *d_ocls = nullptr, *d_oanc = nullptr; float *d_osc = nullptr, *d_obox = nullptr, *d_ocoef = nullptr;
  int host_batch = 0; int host_maxdet = 0;
  cudaStream_t own_stream = nullptr;
  // pipelined host entry points: 2 slots of staging input + pinned result buffers
  struct Slot {
    float* d_stage = nullptr;                 // [B,3,S,S] staging copy target (copy stream)
    void* h_res = nullptr;                    // pinned: count | class | anchor | score | box | coef
    cudaEvent_t h2d = nullptr, done = nullptr;
    int batch = 0, max_det = 0, busy = 0;
  } slot[2];
  cudaStream_t copy_stream = nullptr;
  int next_ticket = 0;
  bool profiling = false;
  // CUDA graphs of (forward + post-process) for the host-buffer entry point, keyed by batch + params
  struct HostGraph { cudaGraphExec_t exec; uint64_t launches; };
  std::map<std::string, HostGraph> host_graphs;
  void drop_graphs() { for (auto& kv : host_graphs) cudaGraphExecDestroy(kv.second.exec); host_graphs.clear(); }
  std::vector<std::vector<cudaEvent_t>> prof_sets;   // one event list per profiled forward
  std::vector<int> prof_batch;

  int add_param(const std::string& n, int64_t count) {
    Param p; p.name = n; p.count = count;
    pidx[n] = (int)params.size();
    params.push_back(std::move(p));
    return (int)params.size() - 1;
  }
  const std::vector<float>& P_(const std::string& n) const { return params[pidx.at(n)].data; }
};

namespace {

int new_act(yb_net* net, int C, int H, int planes = 1, bool dense_f32 = false) {
  ActBuf a; a.C = C; a.H = H; a.planes = planes; a.dense_f32 = dense_f32;
  net->acts.push_back(a);
  return (int)net->acts.size() - 1;
}

int new_conv(yb_net* net, const std::string& wname, const std::string& bname, const std::string& bnname, int Cin, int Cout, int k) {
  ConvW c; c.wname = wname; c.bname = bname; c.bnname = bnname; c.Cin = Cin; c.Cin_pad = (Cin + 63) / 64 * 64; c.Cout = Cout; c.Cout_pad = Cout; c.k = k;
  net->add_param(wname, (int64_t)Cout * Cin * k * k);
  if (!bname.empty()) net->add_param(bname, Cout);
  if (!bnname.empty()) {
    for (const char* s : {".weight", ".bias", ".running_mean", ".running_var"}) net->add_param(bnname + s, Cout);
  }
  net->convs.push_back(c);
  return (int)net->convs.size() - 1;
}

// appends [split +] conv; returns output act
int add_conv(yb_net* net, int in, int conv, int stride, int relu, int res = -1, int out_mode = 0, int ext = EXT_NONE, int out_act = -1) {
  const ConvW& c = net->convs[conv];
  const int Hin = net->acts[in].H;
  const int Hout = out_size(Hin, stride);
  int src = in;
  if (stride == 2) {
    const int planes = c.k == 3 ? 4 : 1;
    src = new_act(net, c.Cin, Hout, planes);
    Op sp; sp.kind = OP_SPLIT; sp.in = in; sp.out = src;
    net->ops.push_back(sp);
  }
  int out = out_act;
  if (out < 0 && ext == EXT_NONE) out = new_act(net, out_mode == 1 ? c.Cout_pad : c.Cout, Hout, 1, out_mode == 1);
  Op op; op.kind = OP_CONV; op.in = src; op.out = out; op.res = res; op.conv = conv; op.stride = stride; op.relu = relu;
  op.out_mode = out_mode; op.ext = ext;
  net->ops.push_back(op);
  return out;
}

void build_program(yb_net* net) {
  const yb_net_config& cfg = net->cfg;
  const StemSizes ss = stem_sizes(cfg.img_size);
  net->H1 = ss.H1; net->H2 = ss.H2;
  int couts[4] = {-1, -1, -1, -1};
  int fin[3] = {512, 1024, 2048};
  if (cfg.depth == 0) {
    // ---------------- Swin-T backbone (modules/swin_transformer.py:436-518) ----------------
    fin[0] = 192; fin[1] = 384; fin[2] = 768;
    net->H1 = ss.Hg;
    net->add_param("backbone.patch_embed.proj.weight", 96 * 3 * 4 * 4);
    net->add_param("backbone.patch_embed.proj.bias", 96);
    net->add_param("backbone.patch_embed.norm.weight", 96);
    net->add_param("backbone.patch_embed.norm.bias", 96);
    int x = new_act(net, 96, ss.Hg);
    { Op o; o.kind = OP_PATCH_EMBED; o.out = x; net->ops.push_back(o); }
    auto add_ln = [&](int in, const std::string& name, int C) {
      net->add_param(name + ".weight", C); net->add_param(name + ".bias", C);
      const int out = new_act(net, C, net->acts[in].H);
      Op o; o.kind = OP_LN; o.in = in; o.out = out; o.p0 = name + ".weight"; o.p1 = name + ".bias";
      net->ops.push_back(o);
      return out;
    };
    for (int s = 0; s < 4; ++s) {
      const int C = 96 << s;
      for (int b = 0; b < kSwinDepths[s]; ++b) {
        const std::string p = "backbone.layers." + std::to_string(s) + ".blocks." + std::to_string(b);
        const int t1 = add_ln(x, p + ".norm1", C);
        net->add_param(p + ".attn.relative_position_bias_table", 169 * kSwinHeads[s]);
        const int cq = new_conv(net, p + ".attn.qkv.weight", p + ".attn.qkv.bias", "", C, 3 * C, 1);
        const int cp = new_conv(net, p + ".attn.proj.weight", p + ".attn.proj.bias", "", C, C, 1);
        const int qkv = add_conv(net, t1, cq, 1, 0);
        const int att = new_act(net, C, net->acts[x].H);
        { Op o; o.kind = OP_ATTN; o.in = qkv; o.out = att; o.p0 = p + ".attn.qkv.bias"; o.p1 = p + ".attn.relative_position_bias_table";
          o.heads = kSwinHeads[s]; o.shift = (b % 2) ? 3 : 0; net->ops.push_back(o); }
        x = add_conv(net, att, cp, 1, 0, x);                         // x + proj(attn)
        const int t2 = add_ln(x, p + ".norm2", C);
        const int c1 = new_conv(net, p + ".mlp.fc1.weight", p + ".mlp.fc1.bias", "", C, 4 * C, 1);
        const int c2 = new_conv(net, p + ".mlp.fc2.weight", p + ".mlp.fc2.bias", "", 4 * C, C, 1);
        const int h = add_conv(net, t2, c1, 1, 2);                   // GELU
        x = add_conv(net, h, c2, 1, 0, x);                           // x + fc2(gelu(fc1(norm2 x)))
      }
      if (s > 0) couts[s] = add_ln(x, "backbone.norm" + std::to_string(s), C);
      if (s < 3) {
        const std::string p = "backbone.layers." + std::to_string(s) + ".downsample";
        const int Hin = net->acts[x].H, Hout = (Hin + 1) / 2;
        net->add_param(p + ".norm.weight", 4 * C); net->add_param(p + ".norm.bias", 4 * C);
        const int mg = new_act(net, 4 * C, Hout);
        { Op o; o.kind = OP_MERGE_LN; o.in = x; o.out = mg; o.p0 = p + ".norm.weight"; o.p1 = p + ".norm.bias"; net->ops.push_back(o); }
        x = add_conv(net, mg, new_conv(net, p + ".reduction.weight", "", "", 4 * C, 2 * C, 1), 1, 0);
      }
    }
    net->taps["c3"] = couts[1]; net->taps["c4"] = couts[2]; net->taps["c5"] = couts[3];
  } else {
  // stem (direct kernel; parameters registered by hand)
  net->add_param("backbone.conv1.weight", 64 * 3 * 7 * 7);
  for (const char* s : {".weight", ".bias", ".running_mean", ".running_var"}) net->add_param(std::string("backbone.bn1") + s, 64);
  const int stem = new_act(net, 64, net->H1);
  // 16-bit modes: space-to-depth repack of the image (kernels_simt.cu k_stem_s2d), 16 channels per pixel; the
  // wgmma kernel then runs the stem as a 4-tap K=64 convolution over it.  YOLACT_B200_STEM_WIDE=1 forces the
  // 64-channel materialised form that is otherwise only the fallback when the overlapping tensor map is refused.
  net->stem_wide = (getenv("YOLACT_B200_STEM_WIDE") || !tc_overlapping_rows_ok()) ? 1 : 0;
  const int stem_cols = new_act(net, net->stem_wide ? 64 : 16, net->H1);
  // The 4-tap stem reads TWO pixel rows below an output row (dy = 3) and, through the overlapping tensor map, up to 3 pixels past
  // a row: for the last image of a batch that is one pixel row (+4 pixels) BEHIND the image, which must read as zero.  The buffer
  // carries that many spare rows and yb_net_forward zeroes them behind the batch's last image on every call (with fewer images
  // than max_batch the region belongs to the next image slot and holds stale data; the arena slot is shared with other tensors).
  net->acts[stem_cols].pad_rows = net->H1 + 2 + 4;
  { Op o; o.kind = OP_STEM; o.out = stem; o.aux = stem_cols; net->ops.push_back(o); }
  int x = new_act(net, 64, net->H2);
  { Op o; o.kind = OP_POOL; o.in = stem; o.out = x; net->ops.push_back(o); }

  const int* nblk = resnet_blocks(cfg.depth);
  int inpl = 64;
  for (int s = 0; s < 4; ++s) {
    const int planes = 64 << s;
    for (int b = 0; b < nblk[s]; ++b) {
      const int stride = (b == 0 && s > 0) ? 2 : 1;
      const std::string p = "backbone.layers." + std::to_string(s) + "." + std::to_string(b);
      const int c1 = new_conv(net, p + ".conv1.weight", "", p + ".bn1", inpl, planes, 1);
      const int c2 = new_conv(net, p + ".conv2.weight", "", p + ".bn2", planes, planes, 3);
      const int c3 = new_conv(net, p + ".conv3.weight", "", p + ".bn3", planes, planes * 4, 1);
      int r = x;
      int cd = -1;
      if (b == 0) cd = new_conv(net, p + ".downsample.0.weight", "", p + ".downsample.1", inpl, planes * 4, 1);
      const int t1 = add_conv(net, x, c1, 1, 1);
      const int t2 = add_conv(net, t1, c2, stride, 1);
      if (b == 0) r = add_conv(net, x, cd, stride, 0);
      x = add_conv(net, t2, c3, 1, 1, r);
      inpl = planes * 4;
    }
    couts[s] = x;
  }
  net->taps["c2"] = couts[0]; net->taps["c3"] = couts[1]; net->taps["c4"] = couts[2]; net->taps["c5"] = couts[3];
  }

  // FPN (modules/yolact.py:73-89)
  int lat[3], pred[3];
  for (int i = 0; i < 3; ++i) {
    const std::string n = "fpn.lat_layers." + std::to_string(i);
    lat[i] = new_conv(net, n + ".weight", n + ".bias", "", fin[i], 256, 1);
  }
  for (int i = 0; i < 3; ++i) {
    const std::string n = "fpn.pred_layers." + std::to_string(i) + ".0";
    pred[i] = new_conv(net, n + ".weight", n + ".bias", "", 256, 256, 3);
  }
  int down[2];
  for (int i = 0; i < 2; ++i) {
    const std::string n = "fpn.downsample_layers." + std::to_string(i) + ".0";
    down[i] = new_conv(net, n + ".weight", n + ".bias", "", 256, 256, 3);
  }
  const int p5_1 = add_conv(net, couts[3], lat[2], 1, 0);
  const int p4_1 = add_conv(net, couts[2], lat[1], 1, 0);
  { Op o; o.kind = OP_UPADD; o.in = p5_1; o.out = p4_1; net->ops.push_back(o); }
  const int p3_1 = add_conv(net, couts[1], lat[0], 1, 0);
  { Op o; o.kind = OP_UPADD; o.in = p4_1; o.out = p3_1; net->ops.push_back(o); }
  int lv[5];
  lv[2] = add_conv(net, p5_1, pred[2], 1, 1);
  lv[1] = add_conv(net, p4_1, pred[1], 1, 1);
  lv[0] = add_conv(net, p3_1, pred[0], 1, 1);
  lv[3] = add_conv(net, lv[2], down[0], 2, 1);
  lv[4] = add_conv(net, lv[3], down[1], 2, 1);
  const char* lvn[5] = {"p3", "p4", "p5", "p6", "p7"};
  for (int i = 0; i < 5; ++i) net->taps[lvn[i]] = lv[i];

  // ProtoNet (modules/yolact.py:34-53)
  int t = lv[0];
  for (int i : {0, 2, 4}) {
    const std::string n = "proto_net.proto1." + std::to_string(i);
    t = add_conv(net, t, new_conv(net, n + ".weight", n + ".bias", "", 256, 256, 3), 1, 1);
  }
  const int up = new_act(net, 256, 2 * net->acts[t].H);
  { Op o; o.kind = OP_UP2X; o.in = t; o.out = up; net->ops.push_back(o); }
  t = add_conv(net, up, new_conv(net, "proto_net.proto2.0.weight", "proto_net.proto2.0.bias", "", 256, 256, 3), 1, 1);
  net->P = net->acts[t].H;
  add_conv(net, t, new_conv(net, "proto_net.proto2.2.weight", "proto_net.proto2.2.bias", "", 256, cfg.coef_dim, 1), 1, 1, -1, 1, EXT_PROTO);

  // prediction heads, shared weights over 5 levels (modules/yolact.py:12-31,:149-157)
  const int upf = new_conv(net, "prediction_layers.upfeature.0.weight", "prediction_layers.upfeature.0.bias", "", 256, 256, 3);
  const HeadLayout hl = head_layout(cfg);
  ConvW hc; hc.Cin = 256; hc.Cin_pad = 256; hc.k = 3; hc.Cout = hl.Cout; hc.Cout_pad = hl.Cout_pad; hc.cat = hl.cat;
  for (const auto& p : hl.params) net->add_param(p.first, p.second);
  net->convs.push_back(hc);
  const int head = (int)net->convs.size() - 1;
  for (int l = 0; l < 5; ++l) {
    net->level_size[l] = net->acts[lv[l]].H;
    const int f = add_conv(net, lv[l], upf, 1, 1);
    const int h = add_conv(net, f, head, 1, 0, -1, 1);
    Op o; o.kind = OP_HEADFIN; o.in = h; o.level = l; net->ops.push_back(o);
  }
  net->A = level_offsets(net->level_size, cfg.num_ratios, net->level_off);
  net->anchors = default_anchors(cfg, net->level_size);
}

// 16-bit modes: merge [1x1 Cin->Cexp + residual + ReLU] followed by [1x1 Cexp->Cout + ReLU] (conv3 of a bottleneck and conv1 of the
// next, modules/resnet.py:20-40) into one OP_BNECK where k_bneck_tc supports the widths (bneck_supported: within layer1 / 2 / 3, and
// layer1 -> layer2 / layer2 -> layer3, where the next block's conv1 still runs at this resolution)
void fuse_bottlenecks(yb_net* net) {
  if (net->act_dt == DT_F32 || getenv("YOLACT_B200_NO_TC")) return;
  std::vector<Op> merged;
  for (size_t i = 0; i < net->ops.size(); ++i) {
    const Op& a = net->ops[i];
    if (i + 1 < net->ops.size() && a.kind == OP_CONV && net->ops[i + 1].kind == OP_CONV) {
      const Op& b = net->ops[i + 1];
      const ConvW& ca = net->convs[a.conv];
      const ConvW& cb = net->convs[b.conv];
      const bool ok = ca.k == 1 && cb.k == 1 && a.stride == 1 && b.stride == 1 && a.res >= 0 && b.res < 0 && a.relu == 1 && b.relu == 1 &&
                      a.out_mode == 0 && b.out_mode == 0 && a.ext == EXT_NONE && b.ext == EXT_NONE && b.in == a.out && ca.cat.empty() &&
                      cb.cat.empty() && ca.Cout == cb.Cin && ca.Cin == ca.Cin_pad && cb.Cin == cb.Cin_pad && ca.Cout == ca.Cout_pad &&
                      cb.Cout == cb.Cout_pad && bneck_supported(net->act_dt, ca.Cin, ca.Cout, cb.Cout);
      if (ok) {
        Op f = a;
        f.kind = OP_BNECK; f.conv2 = b.conv; f.out2 = b.out;
        merged.push_back(f);
        ++i;
        continue;
      }
    }
    merged.push_back(a);
  }
  // first block of a stage whose residual branch is a stride-1 1x1 convolution of the block input (layer1): fold it into GEMM A
  // when the concatenated K still fits the resident A tile (two k-blocks)
  std::vector<Op> folded;
  for (size_t i = 0; i < merged.size(); ++i) {
    Op f = merged[i];
    if (f.kind == OP_BNECK && !folded.empty() && !getenv("YOLACT_B200_NO_FUSE_DOWN")) {
      const Op& d = folded.back();
      if (d.kind == OP_CONV && d.out == f.res && d.stride == 1 && d.relu == 0 && d.res < 0 && d.out_mode == 0 && d.ext == EXT_NONE) {
        const ConvW& cd = net->convs[d.conv];
        const ConvW& c3 = net->convs[f.conv];
        if (cd.k == 1 && cd.cat.empty() && cd.Cin == cd.Cin_pad && cd.Cout == c3.Cout && (c3.Cin + cd.Cin) / 64 <= 2 && net->acts[d.in].H == net->acts[f.in].H) {
          f.convd = d.conv; f.in2 = d.in; f.res = -1;
          folded.pop_back();                                         // the downsample launch and its output tensor are gone
        }
      }
    }
    folded.push_back(f);
  }
  net->ops.swap(folded);
}

void bneck_args(const yb_net* net, const Op& o, int B, BneckArgs* a) {
  const ConvW& c3 = net->convs[o.conv];
  const ConvW& c1 = net->convs[o.conv2];
  memset(a, 0, sizeof(*a));
  a->t2 = net->slots[net->acts[o.in].slot];
  if (o.convd >= 0) { a->xd = net->slots[net->acts[o.in2].slot]; a->Cd = net->convs[o.convd].Cin; }
  else a->x = net->slots[net->acts[o.res].slot];
  a->xo = net->slots[net->acts[o.out].slot]; a->t1 = net->slots[net->acts[o.out2].slot];
  a->w3 = o.convd >= 0 ? o.d_wcat : c3.d_w; a->b3 = o.convd >= 0 ? o.d_bcat : c3.d_b; a->w1 = c1.d_w; a->b1 = c1.d_b;
  a->act_dt = net->act_dt; a->B = B; a->Cin = c3.Cin; a->Cexp = c3.Cout; a->Cout = c1.Cout;
  a->g.H = net->acts[o.in].H; a->g.W = a->g.H;
}

// liveness + slot assignment
void plan_memory(yb_net* net) {
  auto& acts = net->acts;
  for (auto& a : acts) { a.first = 1 << 30; a.last = -1; }
  for (int i = 0; i < (int)net->ops.size(); ++i) {
    const Op& o = net->ops[i];
    for (int t : {o.in, o.out, o.res, o.aux, o.out2, o.in2}) {
      if (t < 0) continue;
      acts[t].first = acts[t].first < i ? acts[t].first : i;
      acts[t].last = acts[t].last > i ? acts[t].last : i;
    }
  }
  for (auto& kv : net->taps) acts[kv.second].last = 1 << 30;     // keep debug taps alive
  const size_t esz = dtype_size(net->act_dt);
  for (auto& a : acts) {
    a.dt = a.dense_f32 ? DT_F32 : net->act_dt;
    const size_t rows = a.dense_f32 ? (size_t)net->max_batch * a.H * a.H : (size_t)net->max_batch * (a.H + 2) * (a.H + 2) * a.planes;
    a.bytes = align_up((rows + a.pad_rows) * a.C * (a.dense_f32 ? 4 : esz), 1024);
  }
  std::vector<int> slot_free_at;                                   // op index after which the slot is free
  net->slot_bytes.clear();
  std::vector<int> order(acts.size());
  for (size_t i = 0; i < acts.size(); ++i) order[i] = (int)i;
  std::stable_sort(order.begin(), order.end(), [&](int x, int y) { return acts[x].first < acts[y].first; });
  for (int ai : order) {
    ActBuf& a = acts[ai];
    if (a.last < 0) continue;
    // best fit: the smallest free slot that is large enough, else the largest free slot (grown)
    int best = -1;
    for (size_t s = 0; s < slot_free_at.size(); ++s) {
      if (slot_free_at[s] >= a.first) continue;
      if (best < 0) { best = (int)s; continue; }
      const size_t sb = net->slot_bytes[s], bb = net->slot_bytes[best];
      const bool s_fits = sb >= a.bytes, b_fits = bb >= a.bytes;
      if ((s_fits && (!b_fits || sb < bb)) || (!s_fits && !b_fits && sb > bb)) best = (int)s;
    }
    if (best < 0) { slot_free_at.push_back(a.last); net->slot_bytes.push_back(a.bytes); a.slot = (int)slot_free_at.size() - 1; }
    else { a.slot = best; slot_free_at[best] = a.last; if (net->slot_bytes[best] < a.bytes) net->slot_bytes[best] = a.bytes; }
  }
}

int upload(const void* host, size_t bytes, void** dev) {
  YB_CHECK_CUDA(cudaMalloc(dev, bytes));
  YB_CHECK_CUDA(cudaMemcpy(*dev, host, bytes, cudaMemcpyHostToDevice));
  return YB_OK;
}

// fold BN (eval) into scale/shift: y = conv(x)*s + t
void bn_fold(const yb_net* net, const std::string& bn, int C, std::vector<float>& s, std::vector<float>& t) {
  const auto& g = net->P_(bn + ".weight"); const auto& b = net->P_(bn + ".bias");
  const auto& m = net->P_(bn + ".running_mean"); const auto& v = net->P_(bn + ".running_var");
  s.resize(C); t.resize(C);
  for (int c = 0; c < C; ++c) {
    const float sc = g[c] / sqrtf(v[c] + 1e-5f);
    s[c] = sc; t[c] = b[c] - m[c] * sc;
  }
}

int pack_conv(yb_net* net, ConvW& c) {
  const int k2 = c.k * c.k, Ktot = k2 * c.Cin_pad;
  const int Cout_alloc = (c.Cout_pad + 63) / 64 * 64;
  std::vector<float> w((size_t)Cout_alloc * Ktot, 0.f), bias(Cout_alloc, 0.f);
  auto pack_one = [&](const std::vector<float>& src, int cout, int row0, const std::vector<float>* scale) {
    // src [cout][Cin][k][k] -> w[row0+co][(r*k+s)*Cin + ci]
    for (int co = 0; co < cout; ++co)
      for (int ci = 0; ci < c.Cin; ++ci)
        for (int t = 0; t < k2; ++t)
          w[(size_t)(row0 + co) * Ktot + (size_t)t * c.Cin_pad + ci] = src[((size_t)co * c.Cin + ci) * k2 + t] * (scale ? (*scale)[co] : 1.f);
  };
  if (c.cat.empty()) {
    std::vector<float> s, t;
    if (!c.bnname.empty()) bn_fold(net, c.bnname, c.Cout, s, t);
    pack_one(net->P_(c.wname), c.Cout, 0, c.bnname.empty() ? nullptr : &s);
    for (int co = 0; co < c.Cout; ++co) {
      float b = c.bname.empty() ? 0.f : net->P_(c.bname)[co];
      bias[co] = c.bnname.empty() ? b : b * s[co] + t[co];
    }
  } else {
    int row = 0;
    for (const auto& n : c.cat) {
      const auto& ww = net->P_(n + ".weight"); const auto& bb = net->P_(n + ".bias");
      const int cout = (int)bb.size();
      pack_one(ww, cout, row, nullptr);
      for (int co = 0; co < cout; ++co) bias[row + co] = bb[co];
      row += cout;
    }
  }
  if (net->act_dt == DT_F32) {
    YB_PROPAGATE(upload(w.data(), w.size() * 4, &c.d_w));
  } else if (net->act_dt == DT_BF16) {
    std::vector<__nv_bfloat16> wb(w.size());
    for (size_t i = 0; i < w.size(); ++i) wb[i] = __float2bfloat16_rn(w[i]);
    YB_PROPAGATE(upload(wb.data(), wb.size() * 2, &c.d_w));
  } else {
    std::vector<__half> wb(w.size());
    for (size_t i = 0; i < w.size(); ++i) wb[i] = __float2half_rn(w[i]);
    YB_PROPAGATE(upload(wb.data(), wb.size() * 2, &c.d_w));
  }
  YB_PROPAGATE(upload(bias.data(), bias.size() * 4, (void**)&c.d_b));
  return YB_OK;
}

void* act_ptr(const yb_net* net, int a) { return net->slots[net->acts[a].slot]; }

// fill ConvArgs for op at batch B
void conv_args(const yb_net* net, const Op& o, int B, ConvArgs* a, void* ext_out) {
  const ConvW& c = net->convs[o.conv];
  const ActBuf& in = net->acts[o.in];
  memset(a, 0, sizeof(*a));
  a->in = act_ptr(net, o.in);
  a->weight = c.d_w; a->bias = c.d_b;
  a->residual = o.res >= 0 ? act_ptr(net, o.res) : nullptr;
  a->out = o.ext != EXT_NONE ? ext_out : act_ptr(net, o.out);
  a->act_dt = net->act_dt; a->B = B;
  a->g.H = in.H; a->g.W = in.H;
  a->Cin = c.Cin; a->Cin_pad = c.Cin_pad; a->Cout = c.Cout; a->Cout_pad = c.Cout_pad;
  a->relu = o.relu; a->out_mode = o.out_mode;
  const int Wp = in.H + 2;
  const long long plane_rows = (long long)net->max_batch * Wp * Wp;      // parity planes sit at max-batch strides
  a->in_rows = o.stride == 1 ? (long long)B * Wp * Wp : plane_rows * in.planes;
  a->ntaps = conv_taps(c.k, o.stride, Wp, plane_rows, a->tap_shift);
}

}  // namespace

// ================================================================================================
// C ABI
// ================================================================================================
extern "C" int yb_net_create(const yb_net_config* cfg, yb_net** out) {
  YB_REQUIRE(cfg && out, YB_ERR_INVALID, "yb_net_create: NULL argument");
  YB_REQUIRE(cfg->depth == 50 || cfg->depth == 101 || cfg->depth == 0, YB_ERR_UNSUPPORTED, "yb_net_create: depth=%d (50, 101, or 0 = Swin-T)", cfg->depth);
  YB_REQUIRE(cfg->img_size >= 64 && cfg->img_size <= 4096, YB_ERR_INVALID, "yb_net_create: img_size=%d", cfg->img_size);
  YB_REQUIRE(cfg->num_classes >= 2 && cfg->num_ratios >= 1 && cfg->num_ratios <= 3, YB_ERR_INVALID, "yb_net_create: num_classes=%d num_ratios=%d", cfg->num_classes, cfg->num_ratios);
  YB_REQUIRE(cfg->num_classes <= YB_MAX_CLASSES, YB_ERR_UNSUPPORTED, "yb_net_create: num_classes=%d > %d", cfg->num_classes, YB_MAX_CLASSES);
  YB_REQUIRE(cfg->coef_dim > 0 && cfg->coef_dim % 4 == 0 && cfg->coef_dim <= 64, YB_ERR_UNSUPPORTED, "yb_net_create: coef_dim=%d", cfg->coef_dim);
  yb_net* net = new yb_net();
  net->cfg = *cfg;
  build_program(net);
  net->ops_base = net->ops;
  *out = net;
  return YB_OK;
}

extern "C" void yb_net_destroy(yb_net* net) {
  if (!net) return;
  for (void* p : net->slots) cudaFree(p);
  for (auto& c : net->convs) { cudaFree(c.d_w); cudaFree(c.d_b); }
  for (auto& o : net->ops) { tc_plan_destroy(o.tc); bneck_plan_destroy(o.bn); cudaFree(o.d_wcat); cudaFree(o.d_bcat); }
  for (auto& kv : net->d_vec) cudaFree(kv.second);
  cudaFree(net->d_pe_w);
  for (void* p : {(void*)net->d_anchors, (void*)net->d_stem_w, (void*)net->d_stem_b, net->d_stem_w16, (void*)net->d_stem_b16, (void*)net->d_img, (void*)net->d_cls,
                  (void*)net->d_box, (void*)net->d_coef, (void*)net->d_proto, net->d_ws, (void*)net->d_cnt, (void*)net->d_ocls,
                  (void*)net->d_oanc, (void*)net->d_osc, (void*)net->d_obox, (void*)net->d_ocoef})
    cudaFree(p);
  net->drop_graphs();
  for (auto& sl : net->slot) { cudaFree(sl.d_stage); if (sl.h_res) cudaFreeHost(sl.h_res); if (sl.h2d) cudaEventDestroy(sl.h2d); if (sl.done) cudaEventDestroy(sl.done); }
  if (net->copy_stream) cudaStreamDestroy(net->copy_stream);
  if (net->own_stream) cudaStreamDestroy(net->own_stream);
  delete net;
}

extern "C" int yb_net_num_params(const yb_net* net) { return net ? (int)net->params.size() : 0; }

extern "C" int yb_net_param_info(const yb_net* net, int i, const char** name, int64_t* count) {
  YB_REQUIRE(net && i >= 0 && i < (int)net->params.size(), YB_ERR_INVALID, "yb_net_param_info: index %d", i);
  if (name) *name = net->params[i].name.c_str();
  if (count) *count = net->params[i].count;
  return YB_OK;
}

extern "C" int yb_net_set_param(yb_net* net, const char* name, const float* data, int64_t count) {
  YB_REQUIRE(net && name && data, YB_ERR_INVALID, "yb_net_set_param: NULL argument");
  auto it = net->pidx.find(name);
  YB_REQUIRE(it != net->pidx.end(), YB_ERR_INVALID, "yb_net_set_param: unexpected parameter '%s'", name);
  Param& p = net->params[it->second];
  YB_REQUIRE(p.count == count, YB_ERR_INVALID, "yb_net_set_param: '%s' has %lld elements, expected %lld", name, (long long)count, (long long)p.count);
  p.data.assign(data, data + count);
  p.set = true;
  net->finalized = false;
  return YB_OK;
}

extern "C" int yb_net_finalize(yb_net* net, int max_batch, int precision) {
  YB_REQUIRE(net, YB_ERR_INVALID, "yb_net_finalize: NULL net");
  YB_REQUIRE(max_batch >= 1 && max_batch <= 4096, YB_ERR_INVALID, "yb_net_finalize: max_batch=%d", max_batch);
  YB_REQUIRE(precision == YB_PREC_FP32 || precision == YB_PREC_BF16 || precision == YB_PREC_FP16, YB_ERR_INVALID, "yb_net_finalize: precision=%d", precision);
  for (const auto& p : net->params)
    YB_REQUIRE(p.set, YB_ERR_STATE, "yb_net_finalize: parameter '%s' was never set (strict load)", p.name.c_str());
  int cc_major = 0;
  YB_PROPAGATE(yb_device_info(nullptr, &cc_major, nullptr));
  YB_REQUIRE(cc_major == 9, YB_ERR_UNSUPPORTED, "yb_net_finalize: this library is built for sm_90a only (device cc major %d)", cc_major);
  // release a previous finalisation
  net->drop_graphs();
  for (void* p : net->slots) cudaFree(p);
  net->slots.clear();
  for (auto& c : net->convs) { cudaFree(c.d_w); cudaFree(c.d_b); c.d_w = nullptr; c.d_b = nullptr; }
  for (auto& o : net->ops) { tc_plan_destroy(o.tc); bneck_plan_destroy(o.bn); cudaFree(o.d_wcat); cudaFree(o.d_bcat); }
  net->ops = net->ops_base;
  cudaFree(net->d_anchors); cudaFree(net->d_stem_w); cudaFree(net->d_stem_b); cudaFree(net->d_stem_w16); cudaFree(net->d_stem_b16);
  net->d_anchors = net->d_stem_w = net->d_stem_b = net->d_stem_b16 = nullptr; net->d_stem_w16 = nullptr;

  net->max_batch = max_batch; net->precision = precision;
  net->act_dt = precision == YB_PREC_BF16 ? DT_BF16 : (precision == YB_PREC_FP16 ? DT_F16 : DT_F32);
  fuse_bottlenecks(net);
  plan_memory(net);
  net->slots.resize(net->slot_bytes.size(), nullptr);
  for (size_t s = 0; s < net->slot_bytes.size(); ++s) {
    YB_CHECK_CUDA(cudaMalloc(&net->slots[s], net->slot_bytes[s]));
    YB_CHECK_CUDA(cudaMemset(net->slots[s], 0, net->slot_bytes[s]));
  }
  for (auto& c : net->convs) YB_PROPAGATE(pack_conv(net, c));
  for (auto& kv : net->d_vec) cudaFree(kv.second);
  net->d_vec.clear();
  cudaFree(net->d_pe_w); net->d_pe_w = nullptr;
  if (net->cfg.depth == 0) {
    // Swin: LayerNorm / attention vectors as they are; patch-embed weights [96][3][4][4] -> [48][96]
    for (const Op& o : net->ops)
      for (const std::string* nm : {&o.p0, &o.p1})
        if (!nm->empty() && !net->d_vec.count(*nm)) { float* d = nullptr; const auto& v = net->P_(*nm); YB_PROPAGATE(upload(v.data(), v.size() * 4, (void**)&d)); net->d_vec[*nm] = d; }
    for (const char* nm : {"backbone.patch_embed.proj.bias", "backbone.patch_embed.norm.weight", "backbone.patch_embed.norm.bias"}) {
      float* d = nullptr; const auto& v = net->P_(nm); YB_PROPAGATE(upload(v.data(), v.size() * 4, (void**)&d)); net->d_vec[nm] = d;
    }
    const auto& src = net->P_("backbone.patch_embed.proj.weight");
    std::vector<float> w(48 * 96);
    for (int co = 0; co < 96; ++co) for (int k = 0; k < 48; ++k) w[k * 96 + co] = src[co * 48 + k];
    YB_PROPAGATE(upload(w.data(), w.size() * 4, (void**)&net->d_pe_w));
  } else {  // stem: [64][3][7][7] * bn scale -> [7][7][3][64]
    std::vector<float> s, t, w(147 * 64);
    bn_fold(net, "backbone.bn1", 64, s, t);
    const auto& src = net->P_("backbone.conv1.weight");
    for (int co = 0; co < 64; ++co)
      for (int ci = 0; ci < 3; ++ci)
        for (int r = 0; r < 7; ++r)
          for (int q = 0; q < 7; ++q) w[((r * 7 + q) * 3 + ci) * 64 + co] = src[((co * 3 + ci) * 7 + r) * 7 + q] * s[co];
    YB_PROPAGATE(upload(w.data(), w.size() * 4, (void**)&net->d_stem_w));
    YB_PROPAGATE(upload(t.data(), t.size() * 4, (void**)&net->d_stem_b));
  }
  YB_PROPAGATE(upload(net->anchors.data(), net->anchors.size() * 4, (void**)&net->d_anchors));
  // tensor-core plans (16-bit operand modes)
  if (net->act_dt != DT_F32 && !getenv("YOLACT_B200_NO_TC")) {
    if (net->cfg.depth != 0) {  // stem as a 4-tap (dy) K=64 (dx x 16 ch) GEMM over the space-to-depth image
      std::vector<float> sc, sh, w((size_t)64 * 256, 0.f);
      bn_fold(net, "backbone.bn1", 64, sc, sh);
      const auto& src = net->P_("backbone.conv1.weight");
      for (int co = 0; co < 64; ++co)
        for (int dy = 0; dy < 4; ++dy)
          for (int dx = 0; dx < 4; ++dx)
            for (int py = 0; py < 2; ++py)
              for (int px = 0; px < 2; ++px) {
                const int r = 2 * dy + py - 1, q = 2 * dx + px - 1;      // 7x7 tap; -1 = the zero pad tap
                if (r < 0 || q < 0) continue;
                for (int ci = 0; ci < 3; ++ci)
                  w[(size_t)co * 256 + dy * 64 + dx * 16 + (py * 2 + px) * 3 + ci] = src[((size_t)co * 3 + ci) * 49 + r * 7 + q] * sc[co];
              }
      if (net->act_dt == DT_BF16) { std::vector<__nv_bfloat16> t(w.size()); for (size_t i = 0; i < w.size(); ++i) t[i] = __float2bfloat16_rn(w[i]); YB_PROPAGATE(upload(t.data(), t.size() * 2, &net->d_stem_w16)); }
      else { std::vector<__half> t(w.size()); for (size_t i = 0; i < w.size(); ++i) t[i] = __float2half_rn(w[i]); YB_PROPAGATE(upload(t.data(), t.size() * 2, &net->d_stem_w16)); }
      YB_PROPAGATE(upload(sh.data(), sh.size() * 4, (void**)&net->d_stem_b16));
      Op& so = net->ops[0];
      ConvArgs& a = net->stem_args;
      memset(&a, 0, sizeof(a));
      a.in = act_ptr(net, so.aux); a.weight = net->d_stem_w16; a.bias = net->d_stem_b16; a.out = act_ptr(net, so.out);
      a.act_dt = net->act_dt; a.B = max_batch; a.g.H = net->H1; a.g.W = net->H1; a.Cin = 64; a.Cin_pad = 64; a.Cout = 64; a.Cout_pad = 64;
      a.ntaps = 4; a.relu = 1; a.out_mode = 0;
      stem_taps(net->H1 + 2, a.tap_shift);
      a.in_rows = (long long)max_batch * (net->H1 + 2) * (net->H1 + 2);
      if (!net->stem_wide) a.in_row_stride = 16;                      // rows overlap: row p = pixels p .. p+3 (3 spare pixels exist: pad_rows)
      YB_PROPAGATE(tc_plan_create(a, max_batch, &so.tc));
    }
    for (auto& o : net->ops) {
      if (o.kind == OP_BNECK) {
        if (o.convd >= 0) {                                          // [Cexp][Cmid | Cd] 16-bit weights (both already BN-folded and rounded), b3 + bd
          const ConvW& c3 = net->convs[o.conv];
          const ConvW& cd = net->convs[o.convd];
          const size_t esz = dtype_size(net->act_dt), ldc = (size_t)(c3.Cin + cd.Cin) * esz;
          YB_CHECK_CUDA(cudaMalloc(&o.d_wcat, (size_t)c3.Cout * ldc));
          YB_CHECK_CUDA(cudaMemcpy2D(o.d_wcat, ldc, c3.d_w, (size_t)c3.Cin * esz, (size_t)c3.Cin * esz, c3.Cout, cudaMemcpyDeviceToDevice));
          YB_CHECK_CUDA(cudaMemcpy2D((char*)o.d_wcat + (size_t)c3.Cin * esz, ldc, cd.d_w, (size_t)cd.Cin * esz, (size_t)cd.Cin * esz, c3.Cout, cudaMemcpyDeviceToDevice));
          std::vector<float> b3(c3.Cout), bd(c3.Cout);
          YB_CHECK_CUDA(cudaMemcpy(b3.data(), c3.d_b, b3.size() * 4, cudaMemcpyDeviceToHost));
          YB_CHECK_CUDA(cudaMemcpy(bd.data(), cd.d_b, bd.size() * 4, cudaMemcpyDeviceToHost));
          for (size_t i = 0; i < b3.size(); ++i) b3[i] += bd[i];
          YB_PROPAGATE(upload(b3.data(), b3.size() * 4, (void**)&o.d_bcat));
        }
        BneckArgs b;
        bneck_args(net, o, max_batch, &b);
        YB_PROPAGATE(bneck_plan_create(b, max_batch, &o.bn));
        continue;
      }
      if (o.kind != OP_CONV) continue;
      ConvArgs a;
      static float dummy;
      conv_args(net, o, max_batch, &a, &dummy);
      if (tc_supported(a)) YB_PROPAGATE(tc_plan_create(a, max_batch, &o.tc));
    }
  }
  net->finalized = true;
  return YB_OK;
}

extern "C" int yb_net_num_anchors(const yb_net* net) { return net ? net->A : 0; }
extern "C" int yb_net_proto_size(const yb_net* net) { return net ? net->P : 0; }
extern "C" const float* yb_net_anchors_device(const yb_net* net) { return net ? net->d_anchors : nullptr; }
extern "C" int yb_net_anchors_host(const yb_net* net, float* out) {
  YB_REQUIRE(net && out, YB_ERR_INVALID, "yb_net_anchors_host: NULL argument");
  memcpy(out, net->anchors.data(), net->anchors.size() * 4);
  return YB_OK;
}

extern "C" int yb_net_set_anchors(yb_net* net, const float* anchors_host, int num_anchors) {
  YB_REQUIRE(net && anchors_host, YB_ERR_INVALID, "yb_net_set_anchors: NULL argument");
  YB_REQUIRE(num_anchors == net->A, YB_ERR_INVALID, "yb_net_set_anchors: %d anchors, the network has %d", num_anchors, net->A);
  net->anchors.assign(anchors_host, anchors_host + (size_t)net->A * 4);
  if (net->d_anchors) YB_CHECK_CUDA(cudaMemcpy(net->d_anchors, net->anchors.data(), net->anchors.size() * 4, cudaMemcpyHostToDevice));
  return YB_OK;
}

namespace {

// ops [first, last) of the program; per-op profiling events only for a whole forward
int forward_ops(yb_net* net, const float* img, int batch, int first, int last, float* cls, float* box, float* coef, float* proto,
                cudaStream_t s) {
  const yb_net_config& cfg = net->cfg;
  std::vector<cudaEvent_t>* evs = nullptr;
  if (net->profiling && net->prof_sets.size() < 512 && first == 0 && last == (int)net->ops.size()) {
    net->prof_sets.emplace_back(net->ops.size() + 1);
    net->prof_batch.push_back(batch);
    evs = &net->prof_sets.back();
    for (auto& e : *evs) YB_CHECK_CUDA(cudaEventCreate(&e));
    YB_CHECK_CUDA(cudaEventRecord((*evs)[0], s));
  }
  for (int op_index = first + 1; op_index <= last; ++op_index) {
    const Op& o = net->ops[op_index - 1];
    switch (o.kind) {
      case OP_STEM:
        if (o.tc) {
          YB_PROPAGATE(launch_stem_s2d(img, act_ptr(net, o.aux), net->act_dt, net->stem_wide, batch, cfg.img_size, net->H1, s));
          {  // zero the pixel row (+4 pixels) behind the batch's last image: the dy = 3 taps of its bottom row land there
            const size_t px = (size_t)(net->stem_wide ? 64 : 16) * dtype_size(net->act_dt), Wp1 = (size_t)net->H1 + 2;
            YB_CHECK_CUDA(cudaMemsetAsync((char*)act_ptr(net, o.aux) + (size_t)batch * Wp1 * Wp1 * px, 0, (Wp1 + 4) * px, s));
          }
          ConvArgs a = net->stem_args;
          a.B = batch;
          YB_PROPAGATE(launch_conv_tc(o.tc, a, s));
        } else {
          YB_PROPAGATE(launch_stem(img, net->d_stem_w, net->d_stem_b, act_ptr(net, o.out), net->act_dt, batch, cfg.img_size, net->H1, s));
        }
        break;
      case OP_POOL:
        YB_PROPAGATE(launch_maxpool(act_ptr(net, o.in), act_ptr(net, o.out), net->act_dt, batch, 64, net->H1, net->H2, s));
        break;
      case OP_SPLIT: {
        const ActBuf& out = net->acts[o.out];
        const long long plane_rows = (long long)net->max_batch * (out.H + 2) * (out.H + 2);
        YB_PROPAGATE(launch_phase_split(act_ptr(net, o.in), act_ptr(net, o.out), net->act_dt, batch, out.C, net->acts[o.in].H, out.H,
                                        out.planes, plane_rows, s));
        break;
      }
      case OP_CONV: {
        ConvArgs a;
        conv_args(net, o, batch, &a, proto);
        if (o.tc) YB_PROPAGATE(launch_conv_tc(o.tc, a, s));
        else YB_PROPAGATE(launch_conv_simt(a, s));
        break;
      }
      case OP_BNECK: {
        BneckArgs b;
        bneck_args(net, o, batch, &b);
        YB_PROPAGATE(launch_bneck_tc(o.bn, b, s));
        break;
      }
      case OP_UPADD:
        YB_PROPAGATE(launch_upsample_add(act_ptr(net, o.in), act_ptr(net, o.out), net->act_dt, batch, 256, net->acts[o.in].H,
                                         net->acts[o.out].H, s));
        break;
      case OP_UP2X:
        YB_PROPAGATE(launch_upsample2x_ac(act_ptr(net, o.in), act_ptr(net, o.out), net->act_dt, batch, 256, net->acts[o.in].H, s));
        break;
      case OP_PATCH_EMBED:
        YB_PROPAGATE(launch_patch_embed(img, net->d_pe_w, net->d_vec.at("backbone.patch_embed.proj.bias"),
                                        net->d_vec.at("backbone.patch_embed.norm.weight"), net->d_vec.at("backbone.patch_embed.norm.bias"),
                                        act_ptr(net, o.out), net->act_dt, batch, cfg.img_size, net->acts[o.out].H, s));
        break;
      case OP_LN:
        YB_PROPAGATE(launch_layernorm(act_ptr(net, o.in), act_ptr(net, o.out), net->d_vec.at(o.p0), net->d_vec.at(o.p1), net->act_dt, batch,
                                      net->acts[o.in].C, net->acts[o.in].H, s));
        break;
      case OP_ATTN:
        YB_PROPAGATE(launch_window_attention(act_ptr(net, o.in), net->d_vec.at(o.p0), net->d_vec.at(o.p1), act_ptr(net, o.out), net->act_dt,
                                             batch, net->acts[o.out].H, net->acts[o.out].C, o.heads, o.shift, s));
        break;
      case OP_MERGE_LN:
        YB_PROPAGATE(launch_patch_merge_ln(act_ptr(net, o.in), act_ptr(net, o.out), net->d_vec.at(o.p0), net->d_vec.at(o.p1), net->act_dt,
                                           batch, net->acts[o.in].C, net->acts[o.in].H, net->acts[o.out].H, s));
        break;
      case OP_HEADFIN: {
        const ActBuf& h = net->acts[o.in];
        YB_PROPAGATE(launch_head_finalize((const float*)act_ptr(net, o.in), h.C, batch, h.H * h.H, cfg.num_ratios, cfg.num_classes,
                                          cfg.coef_dim, net->level_off[o.level], net->A, cls, box, coef, s));
        break;
      }
    }
    if (evs) YB_CHECK_CUDA(cudaEventRecord((*evs)[op_index], s));
  }
  return YB_OK;
}

}  // namespace

extern "C" int yb_net_forward(yb_net* net, const float* img, int batch, float* cls, float* box, float* coef, float* proto,
                              void* stream_) {
  YB_REQUIRE(net && img && cls && box && coef && proto, YB_ERR_INVALID, "yb_net_forward: NULL argument");
  YB_REQUIRE(net->finalized, YB_ERR_STATE, "yb_net_forward: call yb_net_finalize first");
  YB_REQUIRE(batch >= 1 && batch <= net->max_batch, YB_ERR_INVALID, "yb_net_forward: batch=%d outside [1,%d]", batch, net->max_batch);
  return forward_ops(net, img, batch, 0, (int)net->ops.size(), cls, box, coef, proto, (cudaStream_t)stream_);
}

extern "C" int yb_net_forward_range(yb_net* net, const float* img, int batch, int first, int last, float* cls, float* box, float* coef,
                                    float* proto, void* stream_) {
  YB_REQUIRE(net && img && cls && box && coef && proto, YB_ERR_INVALID, "yb_net_forward_range: NULL argument");
  YB_REQUIRE(net->finalized, YB_ERR_STATE, "yb_net_forward_range: call yb_net_finalize first");
  YB_REQUIRE(batch >= 1 && batch <= net->max_batch, YB_ERR_INVALID, "yb_net_forward_range: batch=%d outside [1,%d]", batch, net->max_batch);
  YB_REQUIRE(first >= 0 && first <= last && last <= (int)net->ops.size(), YB_ERR_INVALID, "yb_net_forward_range: ops [%d,%d) of %d", first,
             last, (int)net->ops.size());
  return forward_ops(net, img, batch, first, last, cls, box, coef, proto, (cudaStream_t)stream_);
}

extern "C" int yb_net_set_profiling(yb_net* net, int enable) {
  YB_REQUIRE(net, YB_ERR_INVALID, "yb_net_set_profiling: NULL net");
  net->profiling = enable != 0;
  return YB_OK;
}

extern "C" int yb_net_profile(yb_net* net, yb_prof_entry* out, int max_entries, int* num_entries) {
  YB_REQUIRE(net && out && num_entries, YB_ERR_INVALID, "yb_net_profile: NULL argument");
  static const char* kNames[] = {"conv_tc", "conv_simt", "stem", "maxpool", "phase_split", "upsample_add", "upsample2x", "head_finalize",
                                 "patch_embed", "layernorm", "window_attention", "patch_merge_ln", "bneck_tc"};
  const int NK = 13;
  YB_REQUIRE(max_entries >= NK, YB_ERR_INVALID, "yb_net_profile: need room for %d entries", NK);
  for (int i = 0; i < NK; ++i) { memset(&out[i], 0, sizeof(out[i])); strncpy(out[i].name, kNames[i], sizeof(out[i].name) - 1); }
  const size_t esz = dtype_size(net->act_dt);
  FILE* dump = nullptr;
  if (const char* path = getenv("YOLACT_B200_PROFILE_DUMP")) dump = fopen(path, "w");
  if (dump) fprintf(dump, "forward,op,kind,tc,cin,cout,k,stride,h_out,batch,ms,gflop,res,out_mode\n");
  for (size_t f = 0; f < net->prof_sets.size(); ++f) {
    auto& evs = net->prof_sets[f];
    const double B = net->prof_batch[f];
    YB_CHECK_CUDA(cudaEventSynchronize(evs.back()));
    for (size_t i = 0; i < net->ops.size(); ++i) {
      const Op& o = net->ops[i];
      float ms = 0.f;
      YB_CHECK_CUDA(cudaEventElapsedTime(&ms, evs[i], evs[i + 1]));
      int k = 0; double flops = 0, bytes = 0;
      switch (o.kind) {
        case OP_CONV: {
          const ConvW& c = net->convs[o.conv];
          const double Ho = net->acts[o.in].H, px = B * Ho * Ho;
          k = o.tc ? 0 : 1;
          flops = 2.0 * px * c.Cout * c.Cin * c.k * c.k;
          bytes = px * c.Cin * esz * (o.stride == 2 && c.k == 3 ? 4 : 1) + (double)c.Cout * c.Cin * c.k * c.k * esz +
                  px * c.Cout * (o.out_mode == 1 ? 4 : esz) + (o.res >= 0 ? px * c.Cout * esz : 0);
          break;
        }
        case OP_BNECK: {                                               // both convolutions; x' written once and never re-read
          const ConvW& c3 = net->convs[o.conv];
          const double Cin = c3.Cin, Cexp = c3.Cout, Cout = net->convs[o.conv2].Cout;
          const double Ho = net->acts[o.in].H, px = B * Ho * Ho;
          k = 12;
          flops = 2.0 * px * Cexp * (Cin + Cout);
          bytes = px * esz * (Cin + 2.0 * Cexp + Cout) + Cexp * (Cin + Cout) * esz;   // t2, x read; x', t1 written; W3, W1
          if (o.convd >= 0) {                                          // + the folded downsample conv; its output / the residual read do not exist
            const double Cd = net->convs[o.convd].Cin;
            flops += 2.0 * px * c3.Cout * Cd;
            bytes += px * esz * (Cd - c3.Cout) + c3.Cout * Cd * esz;
          }
          break;
        }
        case OP_STEM: k = 2; flops = 2.0 * B * net->H1 * net->H1 * 64 * 147; bytes = B * 3.0 * net->cfg.img_size * net->cfg.img_size * 4 + B * net->H1 * net->H1 * 64.0 * esz; break;
        case OP_POOL: k = 3; bytes = B * 64.0 * esz * ((double)net->H1 * net->H1 + (double)net->H2 * net->H2); break;
        case OP_SPLIT: { k = 4; const ActBuf& a = net->acts[o.out]; bytes = 2.0 * B * a.H * a.H * a.planes * a.C * esz; break; }
        case OP_UPADD: { k = 5; const ActBuf& a = net->acts[o.out]; bytes = 2.25 * B * a.H * a.H * a.C * esz; break; }
        case OP_UP2X: { k = 6; const ActBuf& a = net->acts[o.out]; bytes = 1.25 * B * a.H * a.H * a.C * esz; break; }
        case OP_HEADFIN: { k = 7; const ActBuf& a = net->acts[o.in]; bytes = 2.0 * B * a.H * a.H * a.C * 4; break; }
        case OP_PATCH_EMBED: { k = 8; const ActBuf& a = net->acts[o.out]; flops = 2.0 * B * a.H * a.H * 96 * 48; bytes = B * 3.0 * net->cfg.img_size * net->cfg.img_size * 4 + B * a.H * a.H * 96.0 * esz; break; }
        case OP_LN: { k = 9; const ActBuf& a = net->acts[o.out]; bytes = 2.0 * B * a.H * a.H * a.C * esz; break; }
        case OP_ATTN: { k = 10; const ActBuf& a = net->acts[o.out]; const double nw = ((a.H + 6) / 7) * ((a.H + 6) / 7);
                        flops = B * nw * o.heads * 4.0 * 49 * 49 * 32; bytes = 4.0 * B * a.H * a.H * a.C * esz; break; }
        case OP_MERGE_LN: { k = 11; const ActBuf& a = net->acts[o.out]; bytes = 2.0 * B * a.H * a.H * a.C * esz; break; }
      }
      if (dump) {
        const ConvW* c = (o.kind == OP_CONV || o.kind == OP_BNECK) ? &net->convs[o.conv] : nullptr;
        fprintf(dump, "%zu,%zu,%d,%d,%d,%d,%d,%d,%d,%d,%.5f,%.4f,%d,%d\n", f, i, (int)o.kind, o.tc ? 1 : 0, c ? c->Cin : 0, c ? c->Cout_pad : 0,
                c ? c->k : 0, o.stride, c ? net->acts[o.in].H : 0, (int)B, ms, flops * 1e-9, o.res >= 0 ? 1 : 0, o.out_mode);
      }
      out[k].launches += (o.kind == OP_STEM ? 2 : 1);
      out[k].ms += ms; out[k].flops += flops; out[k].bytes += bytes;
    }
    for (int i = 0; i < NK; ++i) out[i].forwards += 1;
    for (auto& e : evs) cudaEventDestroy(e);
  }
  if (dump) fclose(dump);
  net->prof_sets.clear(); net->prof_batch.clear();
  *num_entries = NK;
  return YB_OK;
}

extern "C" int yb_net_read_activation(yb_net* net, const char* name, int batch, float* out, int64_t out_count, int* C, int* H,
                                      int* W, void* stream) {
  YB_REQUIRE(net && name, YB_ERR_INVALID, "yb_net_read_activation: NULL argument");
  YB_REQUIRE(net->finalized, YB_ERR_STATE, "yb_net_read_activation: net not finalized");
  auto it = net->taps.find(name);
  YB_REQUIRE(it != net->taps.end(), YB_ERR_INVALID, "yb_net_read_activation: unknown tap '%s'", name);
  const ActBuf& a = net->acts[it->second];
  if (C) *C = a.C;
  if (H) *H = a.H;
  if (W) *W = a.H;
  if (!out) return YB_OK;
  YB_REQUIRE(out_count >= (int64_t)batch * a.C * a.H * a.H, YB_ERR_INVALID, "yb_net_read_activation: output too small");
  return launch_read_activation(act_ptr(net, it->second), a.dt, batch, a.C, a.H, out, (cudaStream_t)stream);
}

// ---- debug: the program op by op -----------------------------------------------------------------
static_assert((int)OP_STEM == YB_OP_STEM && (int)OP_CONV == YB_OP_CONV && (int)OP_HEADFIN == YB_OP_HEADFIN && (int)OP_ATTN == YB_OP_ATTN &&
              (int)OP_BNECK == YB_OP_BNECK, "yb_op_kind mirrors OpKind");

extern "C" int yb_net_num_ops(const yb_net* net) { return net ? (int)net->ops.size() : 0; }
extern "C" int yb_net_num_acts(const yb_net* net) { return net ? (int)net->acts.size() : 0; }

extern "C" int yb_net_op_info(const yb_net* net, int i, yb_op_info* out) {
  YB_REQUIRE(net && out, YB_ERR_INVALID, "yb_net_op_info: NULL argument");
  YB_REQUIRE(net->finalized, YB_ERR_STATE, "yb_net_op_info: net not finalized");
  YB_REQUIRE(i >= 0 && i < (int)net->ops.size(), YB_ERR_INVALID, "yb_net_op_info: op %d of %d", i, (int)net->ops.size());
  const Op& o = net->ops[i];
  memset(out, 0, sizeof(*out));
  out->kind = (int)o.kind;
  out->in = o.in; out->out = o.out; out->res = o.res; out->aux = o.aux; out->in2 = o.in2; out->out2 = o.out2;
  out->stride = o.stride; out->relu = o.relu; out->heads = o.heads; out->shift = o.shift; out->level = o.level;
  out->convd = o.convd >= 0 ? 1 : 0;
  out->out_mode = o.out_mode; out->ext_proto = o.ext == EXT_PROTO ? 1 : 0;
  out->anchor_offset = o.kind == OP_HEADFIN ? net->level_off[o.level] : 0;
  static const char* kNone = "";
  out->w0 = out->b0 = out->bn0 = out->w1 = out->bn1 = out->wd = out->bnd = kNone;
  out->p0 = o.p0.c_str(); out->p1 = o.p1.c_str();
  if (o.conv >= 0) {
    const ConvW& c = net->convs[o.conv];
    out->k = c.k; out->cin = c.Cin; out->cout = c.Cout; out->cout_pad = c.Cout_pad;
    out->w0 = c.wname.c_str(); out->b0 = c.bname.c_str(); out->bn0 = c.bnname.c_str();
  }
  if (o.conv2 >= 0) { out->w1 = net->convs[o.conv2].wname.c_str(); out->bn1 = net->convs[o.conv2].bnname.c_str(); }
  if (o.convd >= 0) { out->wd = net->convs[o.convd].wname.c_str(); out->bnd = net->convs[o.convd].bnname.c_str(); }
  return YB_OK;
}

extern "C" int yb_net_act_info(const yb_net* net, int act, yb_act_info* out) {
  YB_REQUIRE(net && out, YB_ERR_INVALID, "yb_net_act_info: NULL argument");
  YB_REQUIRE(net->finalized, YB_ERR_STATE, "yb_net_act_info: net not finalized");
  YB_REQUIRE(act >= 0 && act < (int)net->acts.size(), YB_ERR_INVALID, "yb_net_act_info: act %d of %d", act, (int)net->acts.size());
  const ActBuf& a = net->acts[act];
  memset(out, 0, sizeof(*out));
  out->C = a.C; out->H = a.H; out->planes = a.planes; out->dtype = a.dt; out->dense = a.dense_f32 ? 1 : 0; out->pad_rows = a.pad_rows;
  out->plane_rows = (int64_t)net->max_batch * (a.H + 2) * (a.H + 2);
  return YB_OK;
}

extern "C" int yb_net_read_act_raw(yb_net* net, int act, int batch, void* dst, size_t bytes, void* stream) {
  YB_REQUIRE(net && dst, YB_ERR_INVALID, "yb_net_read_act_raw: NULL argument");
  YB_REQUIRE(net->finalized, YB_ERR_STATE, "yb_net_read_act_raw: net not finalized");
  YB_REQUIRE(act >= 0 && act < (int)net->acts.size(), YB_ERR_INVALID, "yb_net_read_act_raw: act %d of %d", act, (int)net->acts.size());
  YB_REQUIRE(batch >= 1 && batch <= net->max_batch, YB_ERR_INVALID, "yb_net_read_act_raw: batch=%d outside [1,%d]", batch, net->max_batch);
  const ActBuf& a = net->acts[act];
  YB_REQUIRE(a.slot >= 0, YB_ERR_STATE, "yb_net_read_act_raw: act %d is never used", act);
  cudaStream_t s = (cudaStream_t)stream;
  const char* src = (const char*)act_ptr(net, act);
  if (a.dense_f32) {
    const size_t n = (size_t)batch * a.H * a.H * a.C * 4;
    YB_REQUIRE(bytes == n, YB_ERR_INVALID, "yb_net_read_act_raw: %zu bytes, act %d has %zu", bytes, act, n);
    YB_CHECK_CUDA(cudaMemcpyAsync(dst, src, n, cudaMemcpyDeviceToDevice, s));
    return YB_OK;
  }
  const size_t row = (size_t)a.C * dtype_size(a.dt), img_rows = (size_t)(a.H + 2) * (a.H + 2);
  const size_t part = (size_t)batch * img_rows * row, pitch = (size_t)net->max_batch * img_rows * row;
  const size_t n = part * a.planes + (size_t)a.pad_rows * row;
  YB_REQUIRE(bytes == n, YB_ERR_INVALID, "yb_net_read_act_raw: %zu bytes, act %d has %zu", bytes, act, n);
  YB_CHECK_CUDA(cudaMemcpy2DAsync(dst, part, src, pitch, part, a.planes, cudaMemcpyDeviceToDevice, s));
  if (a.pad_rows) YB_CHECK_CUDA(cudaMemcpyAsync((char*)dst + part * a.planes, src + part, (size_t)a.pad_rows * row, cudaMemcpyDeviceToDevice, s));
  return YB_OK;
}

extern "C" int yb_net_read_op_weights(yb_net* net, int op, int which, void* w, size_t w_bytes, float* b, size_t b_bytes, int* rows, int* cols,
                                      void* stream) {
  YB_REQUIRE(net && rows && cols, YB_ERR_INVALID, "yb_net_read_op_weights: NULL argument");
  YB_REQUIRE(net->finalized, YB_ERR_STATE, "yb_net_read_op_weights: net not finalized");
  YB_REQUIRE(op >= 0 && op < (int)net->ops.size(), YB_ERR_INVALID, "yb_net_read_op_weights: op %d of %d", op, (int)net->ops.size());
  const Op& o = net->ops[op];
  const void* dw = nullptr; const float* db = nullptr;
  if (o.kind == OP_STEM && which == 0) {
    YB_REQUIRE(o.tc, YB_ERR_UNSUPPORTED, "yb_net_read_op_weights: the stem runs on its fp32 kernel");
    dw = net->d_stem_w16; db = net->d_stem_b16; *rows = 64; *cols = 256;
  } else if ((o.kind == OP_CONV || o.kind == OP_BNECK) && which == 0) {
    const ConvW& c = net->convs[o.conv];
    if (o.convd >= 0) { dw = o.d_wcat; db = o.d_bcat; *rows = c.Cout; *cols = c.Cin + net->convs[o.convd].Cin; }
    else { dw = c.d_w; db = c.d_b; *rows = (c.Cout_pad + 63) / 64 * 64; *cols = c.k * c.k * c.Cin_pad; }
  } else if (o.kind == OP_BNECK && which == 1) {
    const ConvW& c = net->convs[o.conv2];
    dw = c.d_w; db = c.d_b; *rows = (c.Cout_pad + 63) / 64 * 64; *cols = c.k * c.k * c.Cin_pad;
  } else {
    YB_REQUIRE(false, YB_ERR_INVALID, "yb_net_read_op_weights: op %d (kind %d) has no GEMM %d", op, (int)o.kind, which);
  }
  if (!w && !b) return YB_OK;
  const size_t nw = (size_t)*rows * *cols * dtype_size(net->act_dt), nb = (size_t)*rows * 4;
  YB_REQUIRE(w && b && w_bytes == nw && b_bytes == nb, YB_ERR_INVALID, "yb_net_read_op_weights: buffers of %zu / %zu bytes, need %zu / %zu",
             w_bytes, b_bytes, nw, nb);
  YB_CHECK_CUDA(cudaMemcpyAsync(w, dw, nw, cudaMemcpyDeviceToDevice, (cudaStream_t)stream));
  YB_CHECK_CUDA(cudaMemcpyAsync(b, db, nb, cudaMemcpyDeviceToDevice, (cudaStream_t)stream));
  return YB_OK;
}

extern "C" const float* yb_net_last_proto(const yb_net* net) { return net ? net->d_proto : nullptr; }

namespace {

int ensure_host_scratch(yb_net* net, const yb_detect_params* p) {
  const size_t B = net->max_batch, A = net->A, C = net->cfg.num_classes, K = net->cfg.coef_dim, S = net->cfg.img_size, P = net->P;
  if (!net->own_stream) YB_CHECK_CUDA(cudaStreamCreateWithFlags(&net->own_stream, cudaStreamNonBlocking));
  if (net->host_batch == (int)B && net->host_maxdet >= p->max_det) return YB_OK;
  net->drop_graphs();
  for (void* q : {(void*)net->d_img, (void*)net->d_cls, (void*)net->d_box, (void*)net->d_coef, (void*)net->d_proto, net->d_ws,
                  (void*)net->d_cnt, (void*)net->d_ocls, (void*)net->d_oanc, (void*)net->d_osc, (void*)net->d_obox, (void*)net->d_ocoef})
    cudaFree(q);
  YB_CHECK_CUDA(cudaMalloc(&net->d_img, B * 3 * S * S * 4));
  YB_CHECK_CUDA(cudaMalloc(&net->d_cls, B * A * C * 4));
  YB_CHECK_CUDA(cudaMalloc(&net->d_box, B * A * 16));
  YB_CHECK_CUDA(cudaMalloc(&net->d_coef, B * A * K * 4));
  YB_CHECK_CUDA(cudaMalloc(&net->d_proto, B * P * P * K * 4));
  yb_detect_params pm = *p;
  pm.top_k = 256; pm.max_det = 256;
  net->ws_bytes = yb_detect_workspace_bytes((int)B, (int)A, &pm);
  YB_CHECK_CUDA(cudaMalloc(&net->d_ws, net->ws_bytes));
  YB_CHECK_CUDA(cudaMalloc(&net->d_cnt, B * 4));
  YB_CHECK_CUDA(cudaMalloc(&net->d_ocls, B * 256 * 4));
  YB_CHECK_CUDA(cudaMalloc(&net->d_oanc, B * 256 * 4));
  YB_CHECK_CUDA(cudaMalloc(&net->d_osc, B * 256 * 4));
  YB_CHECK_CUDA(cudaMalloc(&net->d_obox, B * 256 * 16));
  YB_CHECK_CUDA(cudaMalloc(&net->d_ocoef, B * 256 * K * 4));
  net->host_batch = (int)B; net->host_maxdet = 256;
  return YB_OK;
}

int check_host_call(yb_net* net, int batch, const yb_detect_params* p, const char* who) {
  YB_REQUIRE(net->finalized, YB_ERR_STATE, "%s: call yb_net_finalize first", who);
  YB_REQUIRE(batch >= 1 && batch <= net->max_batch, YB_ERR_INVALID, "%s: batch=%d outside [1,%d]", who, batch, net->max_batch);
  YB_REQUIRE(p->num_classes == net->cfg.num_classes && p->coef_dim == net->cfg.coef_dim, YB_ERR_INVALID,
             "%s: params do not match the network (classes %d/%d, coef %d/%d)", who, p->num_classes, net->cfg.num_classes, p->coef_dim,
             net->cfg.coef_dim);
  return YB_OK;
}

// forward + post-process of net->d_img on stream s (captured into a CUDA graph per (batch, params))
// `img`: device image batch the forward reads (net->d_img, or a submission slot's staging buffer: one graph per buffer)
int run_device_pipeline(yb_net* net, const float* img, int batch, const yb_detect_params* p, bool want_coef, cudaStream_t s) {
  auto run = [&]() -> int {
    YB_PROPAGATE(yb_net_forward(net, img, batch, net->d_cls, net->d_box, net->d_coef, net->d_proto, s));
    YB_PROPAGATE(yb_detect(net->d_cls, net->d_box, net->d_coef, net->d_anchors, batch, net->A, p, net->d_ws, net->ws_bytes, net->d_cnt,
                           net->d_ocls, net->d_oanc, net->d_osc, net->d_obox, want_coef ? net->d_ocoef : nullptr, s));
    return YB_OK;
  };
  if (net->profiling || getenv("YOLACT_B200_NO_GRAPH")) return run();
  // ~150 kernel launches per call: capture once per (batch, params), replay afterwards
  std::string key((const char*)p, sizeof(*p));
  key += std::to_string(batch) + (want_coef ? "c" : "n") + std::to_string((unsigned long long)(uintptr_t)img);
  auto it = net->host_graphs.find(key);
  if (it == net->host_graphs.end()) {
    YB_PROPAGATE(run());                                         // warm run: lazy one-time setup stays outside the capture
    YB_CHECK_CUDA(cudaStreamSynchronize(s));
    const uint64_t l0 = g_launches.load();
    YB_CHECK_CUDA(cudaStreamBeginCapture(s, cudaStreamCaptureModeThreadLocal));
    const int st = run();
    cudaGraph_t graph = nullptr;
    cudaError_t ce = cudaStreamEndCapture(s, &graph);
    if (st != YB_OK) { if (graph) cudaGraphDestroy(graph); return st; }
    YB_CHECK_CUDA(ce);
    yb_net::HostGraph hg{nullptr, g_launches.load() - l0};
    ce = cudaGraphInstantiate(&hg.exec, graph, 0);
    cudaGraphDestroy(graph);
    YB_CHECK_CUDA(ce);
    it = net->host_graphs.emplace(key, hg).first;
  }
  YB_CHECK_CUDA(cudaGraphLaunch(it->second.exec, s));
  count_launch(it->second.launches);
  return YB_OK;
}

}  // namespace

extern "C" int yb_net_detect_host(yb_net* net, const float* img_host, int batch, const yb_detect_params* p,
                                  int32_t* out_count, int32_t* out_class, int32_t* out_anchor, float* out_score,
                                  float* out_box, float* out_coef) {
  YB_REQUIRE(net && img_host && p && out_count && out_class && out_anchor && out_score && out_box, YB_ERR_INVALID,
             "yb_net_detect_host: NULL argument");
  YB_PROPAGATE(check_host_call(net, batch, p, "yb_net_detect_host"));
  YB_PROPAGATE(ensure_host_scratch(net, p));
  const size_t K = net->cfg.coef_dim, S = net->cfg.img_size, D = p->max_det, b = batch;
  cudaStream_t s = net->own_stream;
  YB_CHECK_CUDA(cudaMemcpyAsync(net->d_img, img_host, b * 3 * S * S * 4, cudaMemcpyHostToDevice, s));
  YB_PROPAGATE(run_device_pipeline(net, net->d_img, batch, p, out_coef != nullptr, s));
  YB_CHECK_CUDA(cudaMemcpyAsync(out_count, net->d_cnt, b * 4, cudaMemcpyDeviceToHost, s));
  YB_CHECK_CUDA(cudaMemcpyAsync(out_class, net->d_ocls, b * D * 4, cudaMemcpyDeviceToHost, s));
  YB_CHECK_CUDA(cudaMemcpyAsync(out_anchor, net->d_oanc, b * D * 4, cudaMemcpyDeviceToHost, s));
  YB_CHECK_CUDA(cudaMemcpyAsync(out_score, net->d_osc, b * D * 4, cudaMemcpyDeviceToHost, s));
  YB_CHECK_CUDA(cudaMemcpyAsync(out_box, net->d_obox, b * D * 16, cudaMemcpyDeviceToHost, s));
  if (out_coef) YB_CHECK_CUDA(cudaMemcpyAsync(out_coef, net->d_ocoef, b * D * K * 4, cudaMemcpyDeviceToHost, s));
  YB_CHECK_CUDA(cudaStreamSynchronize(s));
  return YB_OK;
}

extern "C" int yb_net_submit_host(yb_net* net, const float* img_host, int batch, const yb_detect_params* p, int* ticket) {
  YB_REQUIRE(net && img_host && p && ticket, YB_ERR_INVALID, "yb_net_submit_host: NULL argument");
  YB_PROPAGATE(check_host_call(net, batch, p, "yb_net_submit_host"));
  YB_PROPAGATE(ensure_host_scratch(net, p));
  const size_t K = net->cfg.coef_dim, S = net->cfg.img_size, D = p->max_det, b = batch, B = net->max_batch;
  if (!net->copy_stream) YB_CHECK_CUDA(cudaStreamCreateWithFlags(&net->copy_stream, cudaStreamNonBlocking));
  const int t = net->next_ticket;
  yb_net::Slot& sl = net->slot[t & 1];
  YB_REQUIRE(!sl.busy, YB_ERR_STATE, "yb_net_submit_host: two submissions already in flight (collect ticket %d first)", t - 2);
  if (!sl.d_stage) {
    YB_CHECK_CUDA(cudaMalloc(&sl.d_stage, B * 3 * S * S * 4));
    YB_CHECK_CUDA(cudaMallocHost(&sl.h_res, B * (4 + 256 * (4 + 4 + 4 + 16 + K * 4))));
    YB_CHECK_CUDA(cudaEventCreateWithFlags(&sl.h2d, cudaEventDisableTiming));
    YB_CHECK_CUDA(cudaEventCreateWithFlags(&sl.done, cudaEventDisableTiming));
  }
  // copy stream: H2D into the slot's staging buffer (overlaps the previous submission's compute)
  YB_CHECK_CUDA(cudaMemcpyAsync(sl.d_stage, img_host, b * 3 * S * S * 4, cudaMemcpyHostToDevice, net->copy_stream));
  YB_CHECK_CUDA(cudaEventRecord(sl.h2d, net->copy_stream));
  cudaStream_t s = net->own_stream;
  YB_CHECK_CUDA(cudaStreamWaitEvent(s, sl.h2d, 0));
  YB_PROPAGATE(run_device_pipeline(net, sl.d_stage, batch, p, true, s));     // the forward reads the slot's staging buffer directly
  char* h = (char*)sl.h_res;
  YB_CHECK_CUDA(cudaMemcpyAsync(h, net->d_cnt, b * 4, cudaMemcpyDeviceToHost, s)); h += B * 4;
  YB_CHECK_CUDA(cudaMemcpyAsync(h, net->d_ocls, b * D * 4, cudaMemcpyDeviceToHost, s)); h += B * 256 * 4;
  YB_CHECK_CUDA(cudaMemcpyAsync(h, net->d_oanc, b * D * 4, cudaMemcpyDeviceToHost, s)); h += B * 256 * 4;
  YB_CHECK_CUDA(cudaMemcpyAsync(h, net->d_osc, b * D * 4, cudaMemcpyDeviceToHost, s)); h += B * 256 * 4;
  YB_CHECK_CUDA(cudaMemcpyAsync(h, net->d_obox, b * D * 16, cudaMemcpyDeviceToHost, s)); h += B * 256 * 16;
  YB_CHECK_CUDA(cudaMemcpyAsync(h, net->d_ocoef, b * D * K * 4, cudaMemcpyDeviceToHost, s));
  YB_CHECK_CUDA(cudaEventRecord(sl.done, s));
  sl.batch = batch; sl.max_det = (int)D; sl.busy = 1;
  *ticket = t;
  net->next_ticket = t + 1;
  return YB_OK;
}

extern "C" int yb_net_collect_host(yb_net* net, int ticket, int32_t* out_count, int32_t* out_class, int32_t* out_anchor,
                                   float* out_score, float* out_box, float* out_coef) {
  YB_REQUIRE(net && out_count && out_class && out_anchor && out_score && out_box, YB_ERR_INVALID, "yb_net_collect_host: NULL argument");
  YB_REQUIRE(ticket >= 0 && ticket < net->next_ticket && ticket >= net->next_ticket - 2, YB_ERR_INVALID, "yb_net_collect_host: bad ticket %d", ticket);
  yb_net::Slot& sl = net->slot[ticket & 1];
  YB_REQUIRE(sl.busy, YB_ERR_STATE, "yb_net_collect_host: ticket %d already collected", ticket);
  YB_CHECK_CUDA(cudaEventSynchronize(sl.done));
  const size_t K = net->cfg.coef_dim, D = sl.max_det, b = sl.batch, B = net->max_batch;
  const char* h = (const char*)sl.h_res;
  memcpy(out_count, h, b * 4); h += B * 4;
  memcpy(out_class, h, b * D * 4); h += B * 256 * 4;
  memcpy(out_anchor, h, b * D * 4); h += B * 256 * 4;
  memcpy(out_score, h, b * D * 4); h += B * 256 * 4;
  memcpy(out_box, h, b * D * 16); h += B * 256 * 16;
  if (out_coef) memcpy(out_coef, h, b * D * K * 4);
  sl.busy = 0;
  return YB_OK;
}

// ---- standalone conv layer (tests) ---------------------------------------------------------------
namespace {
struct Scratch {
  std::vector<void*> ptrs;
  ~Scratch() { for (void* p : ptrs) cudaFree(p); }
  int alloc(void** p, size_t bytes) { YB_CHECK_CUDA(cudaMalloc(p, bytes)); YB_CHECK_CUDA(cudaMemset(*p, 0, bytes)); ptrs.push_back(*p); return YB_OK; }
};
}  // namespace

extern "C" int yb_conv2d(const float* x, int batch, int cin, int h, const float* w, const float* bias, int cout, int k,
                         int stride, int relu, const float* residual, int precision, int use_tc, float* out) {
  YB_REQUIRE(x && w && out, YB_ERR_INVALID, "yb_conv2d: NULL argument");
  YB_REQUIRE((k == 1 || k == 3) && (stride == 1 || stride == 2), YB_ERR_UNSUPPORTED, "yb_conv2d: k=%d stride=%d", k, stride);
  YB_REQUIRE(cin % 8 == 0 && cout >= 1 && batch >= 1 && h >= 1, YB_ERR_UNSUPPORTED, "yb_conv2d: cin=%d cout=%d", cin, cout);
  const int cin_pad = (cin + 63) / 64 * 64;
  YB_REQUIRE(precision >= 0 && precision <= 2, YB_ERR_INVALID, "yb_conv2d: precision=%d", precision);
  const int dt = precision == YB_PREC_BF16 ? DT_BF16 : (precision == YB_PREC_FP16 ? DT_F16 : DT_F32);
  const size_t esz = dtype_size(dt);
  const int ho = out_size(h, stride);
  const int planes = stride == 2 ? (k == 3 ? 4 : 1) : 1;
  const int cout_pad = (cout + 15) / 16 * 16, cout_alloc = (cout_pad + 63) / 64 * 64;
  const int k2 = k * k, Ktot = k2 * cin_pad;
  Scratch sc;
  void *d_in = nullptr, *d_split = nullptr, *d_out = nullptr, *d_res = nullptr, *d_w = nullptr; float* d_b = nullptr;
  const size_t in_rows = (size_t)batch * (h + 2) * (h + 2), out_rows = (size_t)batch * (ho + 2) * (ho + 2);
  YB_PROPAGATE(sc.alloc(&d_in, in_rows * cin * esz));
  YB_PROPAGATE(sc.alloc(&d_out, out_rows * cout_pad * esz));
  YB_PROPAGATE(launch_write_activation(x, dt, batch, cin, h, d_in, nullptr));
  if (stride == 2) {
    YB_PROPAGATE(sc.alloc(&d_split, out_rows * planes * cin * esz));
    YB_PROPAGATE(launch_phase_split(d_in, d_split, dt, batch, cin, h, ho, planes, (long long)out_rows, nullptr));
  }
  if (residual) {
    YB_PROPAGATE(sc.alloc(&d_res, out_rows * cout * esz));
    YB_PROPAGATE(launch_write_activation(residual, dt, batch, cout, ho, d_res, nullptr));
  }
  std::vector<float> wp((size_t)cout_alloc * Ktot, 0.f), bp(cout_alloc, 0.f);
  for (int co = 0; co < cout; ++co) {
    for (int ci = 0; ci < cin; ++ci)
      for (int t = 0; t < k2; ++t) wp[(size_t)co * Ktot + (size_t)t * cin_pad + ci] = w[((size_t)co * cin + ci) * k2 + t];
    bp[co] = bias ? bias[co] : 0.f;
  }
  YB_PROPAGATE(sc.alloc(&d_w, wp.size() * esz));
  if (dt == DT_F32) YB_CHECK_CUDA(cudaMemcpy(d_w, wp.data(), wp.size() * 4, cudaMemcpyHostToDevice));
  else if (dt == DT_BF16) { std::vector<__nv_bfloat16> t(wp.size()); for (size_t i = 0; i < wp.size(); ++i) t[i] = __float2bfloat16_rn(wp[i]); YB_CHECK_CUDA(cudaMemcpy(d_w, t.data(), t.size() * 2, cudaMemcpyHostToDevice)); }
  else { std::vector<__half> t(wp.size()); for (size_t i = 0; i < wp.size(); ++i) t[i] = __float2half_rn(wp[i]); YB_CHECK_CUDA(cudaMemcpy(d_w, t.data(), t.size() * 2, cudaMemcpyHostToDevice)); }
  YB_PROPAGATE(sc.alloc((void**)&d_b, bp.size() * 4));
  YB_CHECK_CUDA(cudaMemcpy(d_b, bp.data(), bp.size() * 4, cudaMemcpyHostToDevice));

  ConvArgs a;
  memset(&a, 0, sizeof(a));
  a.in = stride == 2 ? d_split : d_in; a.weight = d_w; a.bias = d_b; a.residual = d_res; a.out = d_out;
  a.act_dt = dt; a.B = batch; a.g.H = ho; a.g.W = ho; a.Cin = cin; a.Cin_pad = cin_pad; a.Cout = cout; a.Cout_pad = cout; a.relu = relu; a.out_mode = 0;
  YB_REQUIRE(cout % 16 == 0 || !use_tc, YB_ERR_UNSUPPORTED, "yb_conv2d: tc path needs cout %% 16 == 0");
  a.ntaps = conv_taps(k, stride, ho + 2, (long long)out_rows, a.tap_shift);
  a.in_rows = (long long)out_rows * planes;
  if (use_tc) {
    YB_REQUIRE(tc_supported(a), YB_ERR_UNSUPPORTED, "yb_conv2d: shape/precision not supported by the wgmma kernel");
    TcPlan* pl = nullptr;
    YB_PROPAGATE(tc_plan_create(a, batch, &pl));
    int st = launch_conv_tc(pl, a, nullptr);
    if (const char* reps_env = getenv("YOLACT_B200_CONV_REPS")) {        // tooling: time repeated launches with CUDA events
      const int reps = atoi(reps_env);
      cudaEvent_t e0, e1;
      cudaEventCreate(&e0); cudaEventCreate(&e1);
      cudaDeviceSynchronize();
      cudaEventRecord(e0, nullptr);
      for (int i = 0; i < reps && st == YB_OK; ++i) st = launch_conv_tc(pl, a, nullptr);
      cudaEventRecord(e1, nullptr);
      cudaEventSynchronize(e1);
      float ms = 0.f;
      cudaEventElapsedTime(&ms, e0, e1);
      const double us = 1e3 * ms / (reps > 0 ? reps : 1);
      const double flops = 2.0 * batch * ho * ho * (double)cout * cin * k2;
      fprintf(stderr, "[yb_conv2d] B=%d Cin=%d H=%d Cout=%d k=%d s=%d res=%d: %.1f us/launch, %.0f TFLOP/s\n", batch, cin, h, cout, k,
              stride, residual ? 1 : 0, us, flops / us * 1e-6);
      cudaEventDestroy(e0); cudaEventDestroy(e1);
    }
    cudaError_t e = cudaDeviceSynchronize();
    tc_plan_destroy(pl);
    YB_PROPAGATE(st);
    YB_CHECK_CUDA(e);
  } else {
    YB_PROPAGATE(launch_conv_simt(a, nullptr));
  }
  YB_PROPAGATE(launch_read_activation(d_out, dt, batch, cout, ho, out, nullptr));
  YB_CHECK_CUDA(cudaDeviceSynchronize());
  return YB_OK;
}
