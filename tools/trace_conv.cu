// Per-tile timeline of the tensor-core convolution k_conv_tc: one stride-1 launch at a given shape (default: the layer3 3×3
// convolutions of res101 at 550×550, B = 64: 35×35 valid pixels, 256 -> 256 channels), traced with %globaltimer stamps that the
// trace build of conv_tc.cu (YB_CONV_TRACE) writes per CTA, consumer warpgroup and tile.  Prints the mean time per tile spent in
// each step (waiting for the first k-block, the MMAs, the epilogue arithmetic, the last segment's store, and the gap to the next
// tile), the distribution of the CTAs' exit times relative to the launch's earliest CTA start (the tail of the last round of
// tiles), and the launch time with the trace off (CUDA events, 20 launches).  Operands are seeded uniform values; only the timing
// is of interest.
//   nvcc -gencode arch=compute_90a,code=sm_90a -O3 -std=c++17 --expt-relaxed-constexpr -diag-suppress 68 -DYB_CONV_TRACE \
//        -o trace_conv tools/trace_conv.cu yolact_minimal_b200/csrc/common.cu
//   ./trace_conv [B H Cin Cout k residual]        e.g. 64 35 256 256 3 0 (layer3), 64 138 256 256 3 0 (proto), 64 138 64 64 3 0 (layer1)
#include "../yolact_minimal_b200/csrc/conv_tc.cu"

#include <cuda_fp16.h>
#include <algorithm>
#include <vector>

using namespace yb;

static void* dev_fill(size_t n, float scale, uint32_t seed, bool half) {
  uint32_t s = seed * 2654435761u + 1u;
  auto next = [&] { s = s * 1664525u + 1013904223u; return ((s >> 8) * (1.f / 16777216.f) * 2.f - 1.f) * scale; };
  void* d = nullptr;
  if (half) {
    std::vector<__half> h(n);
    for (auto& v : h) v = __float2half(next());
    cudaMalloc(&d, n * 2);
    cudaMemcpy(d, h.data(), n * 2, cudaMemcpyHostToDevice);
  } else {
    std::vector<float> h(n);
    for (auto& v : h) v = next();
    cudaMalloc(&d, n * 4);
    cudaMemcpy(d, h.data(), n * 4, cudaMemcpyHostToDevice);
  }
  return d;
}

int main(int argc, char** argv) {
  const int B = argc > 1 ? atoi(argv[1]) : 64, H = argc > 2 ? atoi(argv[2]) : 35;
  const int Cin = argc > 3 ? atoi(argv[3]) : 256, Cout = argc > 4 ? atoi(argv[4]) : 256;
  const int k = argc > 5 ? atoi(argv[5]) : 3, res = argc > 6 ? atoi(argv[6]) : 0;
  cudaDeviceProp prop;
  cudaGetDeviceProperties(&prop, 0);
  ConvArgs a;
  memset(&a, 0, sizeof(a));
  a.g.H = a.g.W = H;
  const size_t rows = (size_t)B * a.g.plane();
  a.act_dt = DT_F16; a.B = B; a.Cin = Cin; a.Cin_pad = (Cin + 63) / 64 * 64; a.Cout = a.Cout_pad = Cout;
  a.ntaps = k * k;
  for (int t = 0; t < a.ntaps; ++t) a.tap_shift[t] = k == 1 ? 0 : (t / 3 - 1) * a.g.Wp() + (t % 3 - 1);
  a.relu = 1; a.out_mode = 0; a.in_rows = (long long)rows;
  a.in = dev_fill(rows * Cin, 1.f, 1, true);
  a.weight = dev_fill((size_t)Cout * a.ntaps * a.Cin_pad, 0.03f, 2, true);
  a.bias = (const float*)dev_fill(Cout, 0.1f, 3, false);
  a.residual = res ? dev_fill(rows * Cout, 1.f, 4, true) : nullptr;
  cudaMalloc(&a.out, rows * Cout * 2);
  TcPlan* pl = nullptr;
  if (tc_plan_create(a, B, &pl) != YB_OK) { fprintf(stderr, "tc_plan_create: %s\n", yb_last_error()); return 1; }

  for (int r = 0; r < 5; ++r) launch_conv_tc(pl, a, 0);
  cudaEvent_t e0, e1;
  cudaEventCreate(&e0); cudaEventCreate(&e1);
  const int reps = 20;
  cudaEventRecord(e0);
  for (int r = 0; r < reps; ++r) launch_conv_tc(pl, a, 0);
  cudaEventRecord(e1);
  cudaEventSynchronize(e1);
  float ms = 0.f;
  cudaEventElapsedTime(&ms, e0, e1);

  const size_t n = (size_t)CT_TRACE_CTAS * 3 + (size_t)CT_TRACE_CTAS * 2 * CT_TRACE_TILES * CT_TRACE_SLOTS;
  unsigned long long* dtr = nullptr;
  cudaMalloc(&dtr, n * 8);
  cudaMemset(dtr, 0, n * 8);
  conv_trace_buf = dtr;
  launch_conv_tc(pl, a, 0);
  conv_trace_buf = nullptr;
  if (cudaDeviceSynchronize() != cudaSuccess) { fprintf(stderr, "launch failed: %s\n", cudaGetErrorString(cudaGetLastError())); return 1; }
  std::vector<unsigned long long> tr(n);
  cudaMemcpy(tr.data(), dtr, n * 8, cudaMemcpyDeviceToHost);

  int grid = 0;
  unsigned long long t0 = ~0ull;
  for (int cta = 0; cta < CT_TRACE_CTAS && tr[(size_t)cta * 3]; ++cta, ++grid) t0 = std::min(t0, tr[(size_t)cta * 3]);
  std::vector<double> exits;
  for (int cta = 0; cta < grid; ++cta) exits.push_back((double)(std::max(tr[(size_t)cta * 3 + 1], tr[(size_t)cta * 3 + 2]) - t0) * 1e-3);
  std::sort(exits.begin(), exits.end());
  auto quant = [&](double q) { return exits[std::min(exits.size() - 1, (size_t)(q * (exits.size() - 1) + 0.5))]; };
  double busy = 0.0;                                                // SM-microseconds the launch's CTAs ran, against grid x the last exit
  for (int cta = 0; cta < grid; ++cta) busy += exits[cta] - (double)(tr[(size_t)cta * 3] - t0) * 1e-3;

  // per tile: the first k-block's wait, the MMAs (first wait to last drain), the epilogue arithmetic, the last segment's
  // barrier and store issue, and the gap to this warpgroup's next tile (its producer lookahead and residual wait)
  const char* names[] = {"first wait", "MMA", "epilogue", "last store", "to next tile"};
  double sum[5] = {}, tile_ns = 0.0;
  int tiles = 0, gaps = 0;
  const unsigned long long* T = &tr[(size_t)CT_TRACE_CTAS * 3];
  for (int cta = 0; cta < grid; ++cta)
    for (int wg = 0; wg < 2; ++wg)
      for (int i = 0; i < CT_TRACE_TILES; ++i) {
        const unsigned long long* s = T + ((size_t)(cta * 2 + wg) * CT_TRACE_TILES + i) * CT_TRACE_SLOTS;
        if (!s[0]) break;
        for (int j = 0; j < 4; ++j) sum[j] += (double)(s[j + 1] - s[j]);
        tile_ns += (double)(s[4] - s[0]);
        ++tiles;
        if (i + 1 < CT_TRACE_TILES && s[CT_TRACE_SLOTS]) { sum[4] += (double)(s[CT_TRACE_SLOTS] - s[4]); ++gaps; }
      }
  if (!tiles) { fprintf(stderr, "no tiles traced\n"); return 1; }
  printf("{\"gpu\": \"%s\", \"B\": %d, \"H\": %d, \"Cin\": %d, \"Cout\": %d, \"k\": %d, \"residual\": %d, \"BN\": %d, \"stages\": %d, "
         "\"grid\": %d, \"ms_per_launch\": %.4f, \"tile_us\": %.2f", prop.name, B, H, Cin, Cout, k, res, pl->BN, pl->stages, grid, ms / reps,
         tile_ns / tiles * 1e-3);
  for (int j = 0; j < 4; ++j) printf(", \"%s_us\": %.2f", names[j], sum[j] / tiles * 1e-3);
  printf(", \"%s_us\": %.2f", names[4], gaps ? sum[4] / gaps * 1e-3 : 0.0);
  printf(", \"exit_us\": [%.1f, %.1f, %.1f, %.1f, %.1f], \"sm_busy\": %.3f}\n", quant(0), quant(0.25), quant(0.5), quant(0.75), quant(1),
         busy / (grid * exits.back()));
  printf("per tile (mean over %d tile-warpgroups): %.2f us\n", tiles, tile_ns / tiles * 1e-3);
  for (int j = 0; j < 5; ++j) printf("  %-13s %7.2f us\n", names[j], (j < 4 ? sum[j] / tiles : gaps ? sum[j] / gaps : 0.0) * 1e-3);
  printf("CTA exit after the first CTA start (us): min %.1f  p25 %.1f  p50 %.1f  p75 %.1f  max %.1f; SMs busy %.1f%% of grid x last exit\n",
         quant(0), quant(0.25), quant(0.5), quant(0.75), quant(1), 100.0 * busy / (grid * exits.back()));
  return 0;
}
