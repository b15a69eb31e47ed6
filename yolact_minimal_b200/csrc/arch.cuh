// The YOLACT network's shape, stated once for its two host-side builders: the inference program (net.cu) and the training
// engine (train.cu).
#pragma once
#include <math.h>
#include <string>
#include <utility>
#include <vector>

#include "../../include/yolact_b200.h"

namespace yb {

// ---- stage tables (modules/resnet.py:86-98, modules/swin_transformer.py:436-518) ----
inline const int* resnet_blocks(int depth) {             // bottleneck blocks per stage of ResNet-50 / 101
  static const int b50[4] = {3, 4, 6, 3}, b101[4] = {3, 4, 23, 3};
  return depth == 50 ? b50 : b101;
}
constexpr int kSwinDepths[4] = {2, 2, 6, 2};             // Swin-T blocks per stage
constexpr int kSwinHeads[4] = {3, 6, 12, 24};            // Swin-T attention heads per stage

// ---- feature sizes ----
// output side of a convolution (k 1 or 3, padding k / 2) or of the stem's 3x3 max-pool (padding 1)
inline int out_size(int H, int stride) { return stride == 2 ? (H - 1) / 2 + 1 : H; }

struct StemSizes {
  int H1, H2;   // ResNet: sides of the stride-2 7x7 stem convolution's output and of the stride-2 max-pool's
  int Hg;       // Swin-T: side of the 4x4 patch grid (a partial last patch is zero-padded)
};
inline StemSizes stem_sizes(int S) { return {out_size(S, 2), out_size(out_size(S, 2), 2), (S + 3) / 4}; }

// anchors are ordered [level][row][column][ratio]: each level's first anchor, and the total count A
inline int level_offsets(const int level_size[5], int num_ratios, int level_off[5]) {
  int A = 0;
  for (int l = 0; l < 5; ++l) { level_off[l] = A; A += level_size[l] * level_size[l] * num_ratios; }
  return A;
}

// ---- convolution taps over haloed NHWC tensors (layers.cuh) ----
// A stride-2 3x3 convolution reads its input split into four parity planes with the OUTPUT geometry (k_phase_split): tap (r, s)
// reads plane (r != 1)*2 + (s != 1) at pixel offset (dy, dx).
struct ParityTap { int plane, dy, dx; };
inline ParityTap parity_tap(int r, int s) { return {(r != 1) * 2 + (s != 1), r == 0 ? -1 : 0, s == 0 ? -1 : 0}; }

// Row shift into the input of each tap r*k + s of a (k, stride) convolution, k = 1 or 3; Wp = output side + 2, plane_rows = rows
// between parity planes.  Returns the number of taps.
inline int conv_taps(int k, int stride, int Wp, long long plane_rows, int* shift) {
  if (k == 1) { shift[0] = 0; return 1; }
  for (int r = 0; r < 3; ++r)
    for (int s = 0; s < 3; ++s) {
      const ParityTap p = parity_tap(r, s);
      shift[r * 3 + s] = stride == 1 ? (r - 1) * Wp + (s - 1) : (int)(p.plane * plane_rows) + p.dy * Wp + p.dx;
    }
  return 9;
}

// The input gradient of a stride-2 3x3 convolution is one convolution of dY per parity plane, over the plane's taps at negated
// offsets: lists plane `plane`'s taps (r*3 + s) in ascending order of their row shift -(dy*Wp + dx), stored to `shift` if given.
inline int parity_plane_taps(int plane, int* taps, int Wp = 0, int* shift = nullptr) {
  int n = 0;
  for (int sdy = 0; sdy <= 1; ++sdy)
    for (int sdx = 0; sdx <= 1; ++sdx)
      for (int t = 0; t < 9; ++t) {
        const ParityTap p = parity_tap(t / 3, t % 3);
        if (p.plane == plane && -p.dy == sdy && -p.dx == sdx) { if (shift) shift[n] = sdy * Wp + sdx; taps[n++] = t; }
      }
  return n;
}

// The ResNet stem runs as a 4-tap convolution over the space-to-depth image (k_stem_s2d, side H1, Wp1 = H1 + 2): tap dy reads
// 4 pixels x 16 channels starting at row offset dy - 1 and column offset -1.
inline void stem_taps(int Wp1, int* shift) { for (int dy = 0; dy < 4; ++dy) shift[dy] = (dy - 1) * Wp1 - 1; }

// ---- the fused prediction head (modules/yolact.py:12-31) ----
// conf_layer | bbox_layer | coef_layer.0 concatenated along the output channels: one 3x3 convolution over 256 channels
struct HeadLayout {
  std::vector<std::string> cat;                          // parameter prefixes, in output-channel order
  std::vector<std::pair<std::string, int64_t>> params;   // their weights and biases, in the reference's parameter order
  int Cout, Cout_pad;                                    // R*(NC + 4 + K), and rounded up to 16
};
inline HeadLayout head_layout(const yb_net_config& cfg) {
  const int R = cfg.num_ratios, Cout = R * (cfg.num_classes + 4 + cfg.coef_dim);
  const std::string conf = "prediction_layers.conf_layer", bbox = "prediction_layers.bbox_layer", coef = "prediction_layers.coef_layer.0";
  HeadLayout h{{conf, bbox, coef}, {}, Cout, (Cout + 15) / 16 * 16};
  for (const auto& p : {std::make_pair(bbox, R * 4), std::make_pair(conf, R * cfg.num_classes), std::make_pair(coef, R * cfg.coef_dim)}) {
    h.params.push_back({p.first + ".weight", (int64_t)p.second * 256 * 9});
    h.params.push_back({p.first + ".bias", p.second});
  }
  return h;
}

// ---- default anchors (utils/box_utils.py:86-101, modules/yolact.py:111-114): float64, rounded once; [A][4] cx, cy, w, h ----
inline std::vector<float> default_anchors(const yb_net_config& cfg, const int level_size[5]) {
  const int S = cfg.img_size;
  const double ars[3] = {1.0, 0.5, 2.0};
  std::vector<float> a;
  for (int l = 0; l < 5; ++l) {
    const int size = level_size[l];
    const double scale = (double)(int)((double)S / 544.0 * (double)(24 << l));
    for (int j = 0; j < size; ++j)
      for (int i = 0; i < size; ++i)
        for (int r = 0; r < cfg.num_ratios; ++r) {
          const double ar = sqrt(ars[r % 3]);
          a.insert(a.end(), {(float)((i + 0.5) / size), (float)((j + 0.5) / size), (float)(scale * ar / S), (float)(scale / ar / S)});
        }
  }
  return a;
}

}  // namespace yb
