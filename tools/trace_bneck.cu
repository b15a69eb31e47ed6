// Per-tile timeline of the fused bottleneck kernel k_bneck_tc: one launch at a given shape (default: the layer3 blocks of
// res101 at 550×550, B = 64: 35×35 valid pixels, Cin = Cout = 256, Cexp = 1024), traced with %globaltimer stamps that the
// trace build of conv_tc.cu (YB_BNECK_TRACE) writes per CTA, consumer warpgroup and tile.  Prints the mean time per tile spent
// in each step of the chunk loop, summed over the chunks, and the launch time with the trace off (CUDA events, 20 launches).
// Operands are seeded uniform values; only the timing is of interest.
//   nvcc -gencode arch=compute_90a,code=sm_90a -O3 -std=c++17 --expt-relaxed-constexpr -diag-suppress 68 -DYB_BNECK_TRACE \
//        -o trace_bneck tools/trace_bneck.cu yolact_minimal_b200/csrc/common.cu
//   ./trace_bneck [B H Cin Cout]
#include "../yolact_minimal_b200/csrc/conv_tc.cu"

#include <cuda_fp16.h>
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
  const int Cin = argc > 3 ? atoi(argv[3]) : 256, Cout = argc > 4 ? atoi(argv[4]) : 256, Cexp = 4 * Cin;
  cudaDeviceProp prop;
  cudaGetDeviceProperties(&prop, 0);
  BneckArgs a = {};
  a.g.H = a.g.W = H;
  const size_t rows = (size_t)B * a.g.plane();
  a.t2 = dev_fill(rows * Cin, 1.f, 1, true);
  a.x = dev_fill(rows * Cexp, 1.f, 2, true);
  a.w3 = dev_fill((size_t)Cexp * Cin, 0.06f, 3, true);
  a.w1 = dev_fill((size_t)Cout * Cexp, 0.03f, 4, true);
  a.b3 = (const float*)dev_fill(Cexp, 0.1f, 5, false);
  a.b1 = (const float*)dev_fill(Cout, 0.1f, 6, false);
  cudaMalloc(&a.xo, rows * Cexp * 2);
  cudaMalloc(&a.t1, rows * Cout * 2);
  a.act_dt = DT_F16; a.B = B; a.Cin = Cin; a.Cexp = Cexp; a.Cout = Cout;
  BnPlan* pl = nullptr;
  if (bneck_plan_create(a, B, &pl) != YB_OK) { fprintf(stderr, "bneck_plan_create: %s\n", yb_last_error()); return 1; }
  const int m_tiles = (int)((rows + TC_BM - 1) / TC_BM), grid = m_tiles < pl->sms ? m_tiles : pl->sms, nch = Cexp / 128;

  for (int k = 0; k < 5; ++k) launch_bneck_tc(pl, a, 0);
  cudaEvent_t e0, e1;
  cudaEventCreate(&e0); cudaEventCreate(&e1);
  const int reps = 20;
  cudaEventRecord(e0);
  for (int k = 0; k < reps; ++k) launch_bneck_tc(pl, a, 0);
  cudaEventRecord(e1);
  cudaEventSynchronize(e1);
  float ms = 0.f;
  cudaEventElapsedTime(&ms, e0, e1);

  const size_t n = (size_t)grid * 2 * BN_TRACE_TILES * BN_TRACE_SLOTS;
  unsigned long long* dtr = nullptr;
  cudaMalloc(&dtr, n * 8);
  cudaMemset(dtr, 0, n * 8);
  bn_trace_buf = dtr;
  launch_bneck_tc(pl, a, 0);
  bn_trace_buf = nullptr;
  if (cudaDeviceSynchronize() != cudaSuccess) { fprintf(stderr, "launch failed: %s\n", cudaGetErrorString(cudaGetLastError())); return 1; }
  std::vector<unsigned long long> tr(n);
  cudaMemcpy(tr.data(), dtr, n * 8, cudaMemcpyDeviceToHost);

  // per tile, summed over its chunks: issue A (from the previous B's issue, or the tile start), drain A, wait for x, E, issue B;
  // then drain the last B, and the t1 epilogue
  const char* names[] = {"A issue", "A drain", "x_full wait", "E", "B issue", "last B drain", "t1 epilogue"};
  double sum[7] = {}, tile_ns = 0.0;
  unsigned long long t_min = ~0ull, t_max = 0;
  int tiles = 0;
  for (int cta = 0; cta < grid; ++cta)
    for (int wg = 0; wg < 2; ++wg)
      for (int i = 0; i < BN_TRACE_TILES && cta + i * grid < m_tiles; ++i) {
        const unsigned long long* s = &tr[((size_t)(cta * 2 + wg) * BN_TRACE_TILES + i) * BN_TRACE_SLOTS];
        for (int c = 0; c < nch; ++c) {
          const unsigned long long prev = c == 0 ? s[0] : s[5 * c];
          const unsigned long long* e = s + 1 + 5 * c;
          sum[0] += (double)(e[0] - prev); sum[1] += (double)(e[1] - e[0]); sum[2] += (double)(e[2] - e[1]);
          sum[3] += (double)(e[3] - e[2]); sum[4] += (double)(e[4] - e[3]);
        }
        sum[5] += (double)(s[BN_TRACE_T1] - s[5 * nch]);
        sum[6] += (double)(s[BN_TRACE_T1 + 1] - s[BN_TRACE_T1]);
        tile_ns += (double)(s[BN_TRACE_T1 + 1] - s[0]);
        t_min = s[0] < t_min ? s[0] : t_min;
        t_max = s[BN_TRACE_T1 + 1] > t_max ? s[BN_TRACE_T1 + 1] : t_max;
        ++tiles;
      }
  printf("{\"gpu\": \"%s\", \"B\": %d, \"H\": %d, \"Cin\": %d, \"Cexp\": %d, \"Cout\": %d, \"m_tiles\": %d, \"grid\": %d, "
         "\"ms_per_launch\": %.4f, \"traced_span_us\": %.1f, \"tile_us\": %.2f", prop.name, B, H, Cin, Cexp, Cout, m_tiles, grid,
         ms / reps, (t_max - t_min) * 1e-3, tile_ns / tiles * 1e-3);
  for (int k = 0; k < 7; ++k) printf(", \"%s_us\": %.2f", names[k], sum[k] / tiles * 1e-3);
  printf("}\n");
  printf("per tile (mean over %d tile-warpgroups): %.2f us\n", tiles, tile_ns / tiles * 1e-3);
  for (int k = 0; k < 7; ++k) printf("  %-12s %7.2f us  %5.1f%%\n", names[k], sum[k] / tiles * 1e-3, 100.0 * sum[k] / tile_ns);
  return 0;
}
