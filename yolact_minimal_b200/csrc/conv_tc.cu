// wgmma implicit-GEMM convolution for sm_90a (fp16 / bf16 operands, fp32 accumulation in registers).
//
//   out[M, Cout] = epilogue( sum_{tap} A[M + shift_tap, Cin] * W_tap[Cin, Cout] )
//
// on the haloed NHWC layout of layers.cuh, where every convolution tap is a constant row shift
// of the activation matrix.  Persistent, warp-specialised CTA of three warpgroups (384 threads, 1 CTA / SM):
//   warpgroup 0   TMA producer (one thread): per k-block one 128x64 A tile (row coordinate m0 + shift_tap,
//                 out-of-range rows zero-filled by TMA = the conv padding) and one BNx64 weight tile, both
//                 128B-swizzled, into a ring of shared-memory stages (mbarrier full / empty)
//   warpgroups 1, 2  consumers: each owns 64 rows of the 128 x BN tile and issues wgmma.m64nBNk16 over the
//                 staged operands, one k-block in flight while the previous one retires; then the epilogue
//                 (+ folded-BN bias, + residual, ReLU / GELU, clamp / pack, halo zeroing, or dense fp32 rows)
//                 through shared memory, see "staged epilogue" below
// Tiles are scheduled round-robin over the persistent grid, the N tiles of one M tile adjacent so the A tile
// is shared through L2.  The tile width BN is a template parameter (wgmma encodes N in the instruction).
// Launches use programmatic dependent launch: the prologue (barrier set-up, descriptor prefetch) overlaps the
// previous kernel's tail; every role passes griddep_wait() before it touches activations.
//
// Staged epilogue (convolutions; the weight-gradient GEMM stores its fp32 fragments directly).  Each consumer warpgroup owns two
// 8 KiB staging buffers and writes its 64 x BN result one column segment at a time, alternating between them:
//   16-bit haloed output   segments of 64 columns (a 32- and a 16-column segment finish a width that is not a multiple of 64), in
//                          the layout of a TMA box of [64 rows][w columns] with the swizzle of its 2w-byte rows (128, 64 or 32 B),
//                          so the fragment's 4-byte stores are bank-conflict free; one thread then stores the box with
//                          cp.async.bulk.tensor.  The map ends at the launch's last row: rows >= M are never written.  Halo rows
//                          are staged as zero.  With a residual, the same box of the residual is loaded into the buffer by TMA one
//                          segment ahead; the epilogue reads it and writes the result in place.
//   dense fp32 output      segments of 32 columns ([64 rows][128 B], 16-byte chunks swizzled by row); after a warpgroup barrier the
//                          128 threads copy the valid rows out with 16-byte stores, a 128-byte row segment per 8 threads.
// A buffer is written again only after the store that read it has finished reading (cp.async.bulk.wait_group.read before the
// warpgroup barrier that precedes the next segment's store), so the consumers go straight on to the next tile's MMAs.
//
// Launch forms, selected per plan (tc_plan_create):
//   pair      cluster of two CTAs on adjacent 128-row tiles of one N tile; each CTA loads half of every weight tile and multicasts
//             it to both shared memories (TMA .multicast::cluster), the stage is recycled once the consumers of BOTH CTAs release it
//
// Environment switches (tooling / A-B runs only): YOLACT_B200_PAIR=1, YOLACT_B200_NO_PDL, YOLACT_B200_BN=<n>.
#include "layers.cuh"
#include "wgmma.cuh"

#include <cuda.h>
#include <cuda_fp16.h>
#include <stdlib.h>
#include <string.h>
#include <mutex>
#include <type_traits>

namespace yb {

constexpr int TC_BM = 128;
constexpr int TC_BK = 64;                          // 16-bit elements = 128 bytes = one swizzle row
constexpr int TC_THREADS = 384;                    // producer warpgroup + 2 consumer warpgroups
constexpr uint32_t TC_A_STAGE = TC_BM * TC_BK * 2;   // 16 KiB
constexpr int TC_MAX_STAGES = 8;
constexpr size_t TC_SMEM_MAX = 227 * 1024;
constexpr uint32_t TC_STG_BYTES = 64 * 128;        // one staging buffer: 64 rows x 128 B
constexpr uint32_t TC_STG_TOTAL = 4 * TC_STG_BYTES;  // two per consumer warpgroup

struct TcParams {
  long long M;            // rows to produce (B * plane)
  int m_tiles, n_tiles;
  int kb_per_tap;         // Cin_pad / 64
  int ntaps;
  int tap_shift[kMaxTaps];
  int stages;
  int pair;               // cluster of two CTAs on adjacent 128-row tiles of the same N tile: each loads half of the weight tile and
                          // multicasts it to both, halving the L2 -> shared-memory weight traffic per MMA
  int Cout, Cout_pad, relu, out_mode;
  int gemm;               // plain GEMM over long K (weight gradients): out[M x taps*Nper] (+)= A[M x K] * B_tap[K x Nper], B read
                          // MN-major; N tile n -> tap n / gemm_ntile_tap, B columns (n % gemm_ntile_tap) * BN, B rows k + gemm_shift[tap]
  int gemm_ntile_tap;     // N tiles per tap
  int gemm_shift[16];     // per-tap row shift of the B operand
  int accumulate;         // out_mode 2: out += result (shared weights: one launch per use; split-K partial tiles)
  int gemm_splits;        // split-K: the K range of every output tile is cut into gemm_splits pieces of gemm_kb_split k-blocks, one
  int gemm_kb_split;      // scheduling unit each; the partial tiles are added to `out` with atomics (out is zeroed by the caller)
  Geom g;
  const float* bias;
  int residual;           // out_mode 0: + the residual, loaded into the staging buffers by TMA (TcMaps::res)
  void* out;
#ifdef YB_CONV_TRACE
  unsigned long long* trace;
#endif
};

// Trace build (tools/trace_conv.cu; the library never defines YB_CONV_TRACE): thread 0 of each consumer warpgroup writes
// %globaltimer stamps for the launch that conv_trace_buf points at.  Per CTA (up to CT_TRACE_CTAS): trace[cta * 3] its start
// (thread 0, before the barrier set-up), trace[cta * 3 + 1 + warpgroup] the warpgroup's exit (its stores complete).  Per tile, at
// trace[CT_TRACE_CTAS * 3 + ((cta * 2 + warpgroup) * CT_TRACE_TILES + tile) * CT_TRACE_SLOTS + slot]: 0 k-loop start; 1 first
// full-barrier wait done; 2 last MMA drained; 3 epilogue arithmetic done (the last segment staged); 4 last store issued.
#ifdef YB_CONV_TRACE
constexpr int CT_TRACE_CTAS = 1024, CT_TRACE_TILES = 96, CT_TRACE_SLOTS = 5;
unsigned long long* conv_trace_buf = nullptr;
__device__ __forceinline__ unsigned long long ct_now() {
  unsigned long long ns;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(ns));
  return ns;
}
#define CT_TRACE(slot)                                                                                                     \
  do {                                                                                                                     \
    if (p.trace && t == 0 && i < CT_TRACE_TILES)                                                                           \
      p.trace[CT_TRACE_CTAS * 3 + (((size_t)blockIdx.x * 2 + c) * CT_TRACE_TILES + i) * CT_TRACE_SLOTS + (slot)] = ct_now(); \
  } while (0)
#define CT_TRACE_CTA(k)                                                                                                    \
  do {                                                                                                                     \
    if (p.trace) p.trace[(size_t)blockIdx.x * 3 + (k)] = ct_now();                                                        \
  } while (0)
#else
#define CT_TRACE(slot) do { } while (0)
#define CT_TRACE_CTA(k) do { } while (0)
#endif

// the staged epilogue's TMA maps, one per segment width (index 0: 64, 1: 32, 2: 16 columns; unused widths hold a placeholder)
struct TcMaps {
  CUtensorMap res[3];      // the residual, boxes of [64 rows][w columns]
  CUtensorMap out[3];      // the 16-bit output, the same boxes; the map ends at the launch's last row
};

struct TcPlan {
  CUtensorMap tmA, tmB;
  CUtensorMap tmRes[3];    // TcMaps::res, encoded once for the max-batch rows
  int BN, stages, pair;
  int sms;                 // SM count of the device the plan was created on
  int gemm;                // plain-GEMM plan (tc_plan_create_gemm)
  size_t smem_bytes;
};

// ---- PTX wrappers ------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "WAIT_LOOP:\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n\t"
      "@p bra WAIT_DONE;\n\t"
      "bra WAIT_LOOP;\n\t"
      "WAIT_DONE:\n\t}" ::"r"(smem_u32(bar)), "r"(parity)
      : "memory");
}
__device__ __forceinline__ void tma_load_2d(void* dst, const CUtensorMap* map, int c0, int c1, uint64_t* bar) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];" ::"r"(smem_u32(dst)),
      "l"(map), "r"(smem_u32(bar)), "r"(c0), "r"(c1)
      : "memory");
}
// pair form (cluster of two CTAs): one TMA load written to the same offset in every CTA of `mask`, its bytes counted on the
// barrier at the same offset in each
__device__ __forceinline__ void tma_load_2d_multicast(void* dst, const CUtensorMap* map, int c0, int c1, uint64_t* bar, uint16_t mask) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes.multicast::cluster [%0], [%1, {%3, %4}], [%2], %5;"
      ::"r"(smem_u32(dst)), "l"(map), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "h"(mask)
      : "memory");
}
__device__ __forceinline__ uint32_t cluster_ctarank() { uint32_t r; asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r)); return r; }
__device__ __forceinline__ void cluster_sync_all() {
  asm volatile("barrier.cluster.arrive.release.aligned;" ::: "memory");
  asm volatile("barrier.cluster.wait.acquire.aligned;" ::: "memory");
}
// shared::cluster address of the same shared-memory offset in CTA `rank` of the cluster
__device__ __forceinline__ uint32_t map_to_rank(uint32_t saddr, uint32_t rank) {
  uint32_t r; asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(r) : "r"(saddr), "r"(rank)); return r;
}
__device__ __forceinline__ void mbar_arrive_cluster(uint32_t cluster_addr) {
  asm volatile("mbarrier.arrive.release.cluster.shared::cluster.b64 _, [%0];" ::"r"(cluster_addr) : "memory");
}
__device__ __forceinline__ void fence_async_smem() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
__device__ __forceinline__ void named_barrier_sync(int id, int threads) { asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(threads) : "memory"); }
__device__ __forceinline__ uint32_t lds32(uint32_t a) { uint32_t v; asm volatile("ld.shared.b32 %0, [%1];" : "=r"(v) : "r"(a) : "memory"); return v; }
__device__ __forceinline__ void sts32(uint32_t a, uint32_t v) { asm volatile("st.shared.b32 [%0], %1;" ::"r"(a), "r"(v) : "memory"); }
__device__ __forceinline__ void sts64(uint32_t a, float x, float y) { asm volatile("st.shared.v2.f32 [%0], {%1, %2};" ::"r"(a), "f"(x), "f"(y) : "memory"); }
__device__ __forceinline__ float2 lds64(uint32_t a) {
  float2 v;
  asm volatile("ld.shared.v2.f32 {%0, %1}, [%2];" : "=f"(v.x), "=f"(v.y) : "r"(a) : "memory");
  return v;
}
__device__ __forceinline__ float4 lds128(uint32_t a) {
  float4 v;
  asm volatile("ld.shared.v4.f32 {%0, %1, %2, %3}, [%4];" : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "r"(a) : "memory");
  return v;
}
// non-tensor bulk copy global -> shared (16-byte aligned, a multiple of 16 bytes), its bytes counted on `bar`
__device__ __forceinline__ void bulk_load(void* dst, const void* src, uint32_t bytes, uint64_t* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(smem_u32(dst)), "l"(src),
               "r"(bytes), "r"(smem_u32(bar))
               : "memory");
}
__device__ __forceinline__ void tma_store_2d(const CUtensorMap* map, const void* src, int c0, int c1) {
  asm volatile("cp.async.bulk.tensor.2d.global.shared::cta.bulk_group [%0, {%2, %3}], [%1];" ::"l"(map), "r"(smem_u32(src)), "r"(c0), "r"(c1)
               : "memory");
}
__device__ __forceinline__ void bulk_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
__device__ __forceinline__ void bulk_wait_read0() { asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory"); }
__device__ __forceinline__ void bulk_wait0() { asm volatile("cp.async.bulk.wait_group 0;" ::: "memory"); }
// programmatic dependent launch: let the next grid's CTAs start their prologue / block until the previous grid's
// memory is complete and visible (both are no-ops for a launch without the programmatic-serialization attribute)
__device__ __forceinline__ void griddep_launch_dependents() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }
__device__ __forceinline__ void griddep_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }

__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N> __device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
// keep the compiler from moving accumulator reads / writes across the asynchronous MMAs
template <int R> __device__ __forceinline__ void acc_fence(float* d) {
#pragma unroll
  for (int i = 0; i < R; ++i) asm volatile("" : "+f"(d[i])::"memory");
}

// 128B-swizzled operand tile, K-major: rows of 128 bytes (64 k), 8-row groups 1024 bytes apart
__device__ __forceinline__ uint64_t gmma_desc(uint32_t saddr) {
  uint64_t d = 0;
  d |= (uint64_t)((saddr & 0x3FFFFu) >> 4);          // start address
  d |= (uint64_t)1 << 16;                             // leading byte offset (unused for swizzled K-major)
  d |= (uint64_t)(1024 >> 4) << 32;                   // stride byte offset: between 8-row groups
  d |= (uint64_t)1 << 62;                             // SWIZZLE_128B
  return d;
}
// 128B-swizzled operand tile, MN-major (the weight-gradient GEMM's B operand, read straight from the [pixels][channels] activations):
// BN/64 TMA boxes of [64 k-rows][64 channels] (8 KiB each); a row of 128 bytes holds 64 consecutive N elements of one k,
// 8 k-rows form a 1 KiB swizzle atom (stride byte offset), the next 64-element N chunk is the next box (leading byte offset 8192).
__device__ __forceinline__ uint64_t gmma_desc_mn(uint32_t saddr) {
  uint64_t d = 0;
  d |= (uint64_t)((saddr & 0x3FFFFu) >> 4);
  d |= (uint64_t)(8192 >> 4) << 16;
  d |= (uint64_t)(1024 >> 4) << 32;
  d |= (uint64_t)1 << 62;
  return d;
}

template <bool F16> __device__ __forceinline__ uint32_t pack2(float a, float b) {
  if (F16) {
    __half2 v = __floats2half2_rn(fminf(fmaxf(a, -65504.f), 65504.f), fminf(fmaxf(b, -65504.f), 65504.f));
    return *reinterpret_cast<uint32_t*>(&v);
  } else {
    __nv_bfloat162 v = __floats2bfloat162_rn(a, b);
    return *reinterpret_cast<uint32_t*>(&v);
  }
}
template <bool F16> __device__ __forceinline__ float2 unpack2(uint32_t u) {
  if (F16) return __half22float2(*reinterpret_cast<const __half2*>(&u));
  return __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&u));
}

// CTA-local iteration i -> tile coordinates: round-robin over the grid, the N tiles of one M tile adjacent.  Pair form: the
// scheduling unit is the cluster of two CTAs; p.m_tiles counts 256-row pair tiles and the CTA takes the 128-row half of its rank.
__device__ __forceinline__ bool tile_at(const TcParams& p, int i, int& m_tile, int& n_tile) {
  const int unit = p.pair ? (int)(blockIdx.x >> 1) : (int)blockIdx.x;
  const int units = p.pair ? (int)(gridDim.x >> 1) : (int)gridDim.x;
  int tile = unit + i * units;
  if (p.gemm) {                                                    // split-K: the split index is recovered by kb_range()
    if (tile >= p.m_tiles * p.n_tiles * p.gemm_splits) return false;
    tile %= p.m_tiles * p.n_tiles;
  } else if (tile >= p.m_tiles * p.n_tiles) return false;
  m_tile = tile / p.n_tiles;
  n_tile = tile - m_tile * p.n_tiles;
  if (p.pair) m_tile = 2 * m_tile + (int)cluster_ctarank();
  return true;
}

// k-block range [kb0, kb1) of CTA-local iteration i (all k-blocks of all taps for a convolution)
__device__ __forceinline__ void kb_range(const TcParams& p, int i, int& kb0, int& kb1) {
  if (!p.gemm) { kb0 = 0; kb1 = p.ntaps * p.kb_per_tap; return; }
  const int split = ((int)blockIdx.x + i * (int)gridDim.x) / (p.m_tiles * p.n_tiles);
  kb0 = split * p.gemm_kb_split;
  kb1 = min(kb0 + p.gemm_kb_split, p.kb_per_tap);
}

// Column segments of a BN-wide tile in the staged epilogue.  16-bit output: 64 columns each, then at most one of 32 and one of 16
// (176 = 64 + 64 + 32 + 16).  fp32 output: 32 columns each, the last one 16 when BN is an odd multiple of 16.
template <int BN> struct Segs16 {
  static constexpr int n64 = BN / 64, rem = BN % 64;
  static constexpr int count = n64 + (rem >= 32 ? 1 : 0) + (rem % 32 != 0 ? 1 : 0);
  static constexpr int width(int s) { return s < n64 ? 64 : (s == n64 && rem >= 32) ? 32 : 16; }
  static constexpr int base(int s) { return s < n64 ? 64 * s : 64 * n64 + (s == n64 || rem < 32 ? 0 : 32); }
  static constexpr int of(int col) { return col < 64 * n64 ? col / 64 : (rem >= 32 && col < 64 * n64 + 32) ? n64 : count - 1; }
};
// TcMaps index of a segment width
__host__ __device__ constexpr int seg_map(int w) { return w == 64 ? 0 : w == 32 ? 1 : 2; }

// Byte offset of 16-bit element cc of row r in a TMA box of [64 rows][w columns] with the swizzle of its 2w-byte rows: the 16-byte
// chunk index is XORed with address bits 7.. (SWIZZLE_128B / 64B / 32B).  A warp's fragment stores of one column pair cover eight
// rows; the XOR puts them in distinct banks.
__device__ __forceinline__ uint32_t stg_off16(int r, int cc, int w) {
  const int rb = r * 2 * w;
  return (uint32_t)(rb + ((((cc >> 3) ^ (rb >> 7)) & (w / 8 - 1)) << 4) + (cc & 7) * 2);
}
// fp32 staging: row r at r * 128 B, 16-byte chunk (cc / 4) ^ (r % 8)
__device__ __forceinline__ uint32_t stg_off32(int r, int cc) { return (uint32_t)(r * 128 + ((((cc >> 2) ^ r) & 7) << 4) + (cc & 3) * 4); }

template <bool F16, bool MNB, int BN>
__global__ void __launch_bounds__(TC_THREADS, 1)
k_conv_tc(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB, const __grid_constant__ TcMaps maps,
          const TcParams p) {
  constexpr uint32_t B_STAGE = (uint32_t)BN * TC_BK * 2;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = (uint8_t*)(((uintptr_t)smem_raw + 1023) & ~(uintptr_t)1023);     // SWIZZLE_128B needs 1024B alignment
  uint8_t* sA = smem;                                                               // [stages][128 rows x 128 B]
  uint8_t* sB = smem + (size_t)p.stages * TC_A_STAGE;                               // [stages][BN rows x 128 B] (MN-major: BN/64 boxes)
  uint8_t* sStg = sB + (size_t)p.stages * B_STAGE;                                  // convolutions: [2 warpgroups][2 buffers][8 KiB]
  uint64_t* full = reinterpret_cast<uint64_t*>(sStg + (MNB ? 0u : TC_STG_TOTAL));
  uint64_t* empty = full + TC_MAX_STAGES;
  uint64_t* res_full = empty + TC_MAX_STAGES;                                       // [2 warpgroups][2 buffers]: the residual box landed

  const int wg = threadIdx.x >> 7;
  const uint32_t rank = p.pair ? cluster_ctarank() : 0u;
  if (threadIdx.x == 0) {
    CT_TRACE_CTA(0);
    asm volatile("prefetch.tensormap [%0];" ::"l"(&tmA) : "memory");
    asm volatile("prefetch.tensormap [%0];" ::"l"(&tmB) : "memory");
    // empty: one arrive per consumer warp -- of both CTAs in the pair form, whose weight half lands in both shared memories
    for (int i = 0; i < TC_MAX_STAGES; ++i) { mbar_init(&full[i], 1); mbar_init(&empty[i], p.pair ? 16 : 8); }
    for (int i = 0; i < 4; ++i) mbar_init(&res_full[i], 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  if (p.pair) cluster_sync_all(); else __syncthreads();            // pair: the peer's barriers are initialised too
  griddep_launch_dependents();

  // the producer warpgroup needs few registers: the consumers take them (BN = 256: 128 accumulators and the staged epilogue)
  if (wg == 0) {
    // ================= TMA producer =================
    asm volatile("setmaxnreg.dec.sync.aligned.u32 40;" ::: "memory");
    if (threadIdx.x == 0) {
      griddep_wait();
      int stage = 0; uint32_t phase = 0;
      int m_tile, n_tile;
      const uint32_t b_half = B_STAGE / 2;                         // pair: this CTA loads weight rows rank*BN/2 .. and multicasts them
      for (int i = 0; tile_at(p, i, m_tile, n_tile); ++i) {
        const int m0 = m_tile * TC_BM;
        int n0 = n_tile * BN, brow0 = 0;
        if (MNB) {                                                 // B tile: columns of the tap's operand, rows shifted by the tap
          const int tap = n_tile / p.gemm_ntile_tap;
          n0 = (n_tile - tap * p.gemm_ntile_tap) * BN;
          brow0 = p.gemm_shift[tap];
        }
        int kb0, kb1;
        kb_range(p, i, kb0, kb1);
        for (int kb = kb0; kb < kb1; ++kb) {
          const int t = kb / p.kb_per_tap, kin = kb - t * p.kb_per_tap;
          mbar_wait(&empty[stage], phase ^ 1);
          mbar_expect_tx(&full[stage], TC_A_STAGE + B_STAGE);
          tma_load_2d(sA + (size_t)stage * TC_A_STAGE, &tmA, kin * TC_BK, m0 + p.tap_shift[t], &full[stage]);
          if (MNB) {                                               // BN/64 boxes [64 k-rows][64 channels] at k-row kb*64 + tap shift
#pragma unroll
            for (int j = 0; j < BN / 64; ++j)
              tma_load_2d(sB + (size_t)stage * B_STAGE + (size_t)j * 8192, &tmB, n0 + j * 64, kb * TC_BK + brow0, &full[stage]);
          } else if (p.pair) {
            tma_load_2d_multicast(sB + (size_t)stage * B_STAGE + rank * b_half, &tmB, kb * TC_BK, n0 + (int)rank * (BN / 2), &full[stage], 3);
          } else {
            tma_load_2d(sB + (size_t)stage * B_STAGE, &tmB, kb * TC_BK, n0, &full[stage]);
          }
          if (++stage == p.stages) { stage = 0; phase ^= 1; }
        }
      }
    }
  } else {
    // ================= consumers: warpgroup c owns rows 64c .. 64c+63 of every tile =================
    asm volatile("setmaxnreg.inc.sync.aligned.u32 232;" ::: "memory");
    const int c = wg - 1;
    const int t = threadIdx.x & 127, warp = t >> 5, lane = t & 31;
    const bool signal = lane == 0;
    uint32_t peer_empty = 0;
    if (p.pair) peer_empty = map_to_rank(smem_u32(empty), rank ^ 1u);
    auto release = [&](int s) {                                    // this warp is done with stage s (in both CTAs for the pair form)
      if (!signal) return;
      mbar_arrive(&empty[s]);
      if (p.pair) mbar_arrive_cluster(peer_empty + (uint32_t)s * 8u);
    };
    griddep_wait();
    float acc[BN / 2];
    int stage = 0; uint32_t phase = 0;
    int m_tile, n_tile;
    uint8_t* stg = sStg + (size_t)c * 2 * TC_STG_BYTES;             // this warpgroup's two staging buffers
    uint32_t q = 0;                                                 // segments staged so far: buffer q & 1
    // the residual box of 16-bit segment s of tile (mt, nt) into the buffer of segment qq (thread 0 of the warpgroup)
    auto load_res = [&](uint32_t qq, int mt, int nt, int s) {
      const int w = Segs16<BN>::width(s);
      uint64_t* bar = &res_full[2 * c + (qq & 1)];
      mbar_expect_tx(bar, 64u * 2u * (uint32_t)w);
      tma_load_2d(stg + (qq & 1) * TC_STG_BYTES, &maps.res[seg_map(w)], nt * BN + Segs16<BN>::base(s), mt * TC_BM + c * 64, bar);
    };
    if (!MNB && p.residual && t == 0 && tile_at(p, 0, m_tile, n_tile)) load_res(0, m_tile, n_tile, 0);
    for (int i = 0; tile_at(p, i, m_tile, n_tile); ++i) {
      int kb0, kb1;
      kb_range(p, i, kb0, kb1);
      const int nmain = kb1 - kb0;
      int prev = -1;
      CT_TRACE(0);
      for (int s = 0; s < nmain; ++s) {
        mbar_wait(&full[stage], phase);
        if (s == 0) CT_TRACE(1);
        const uint64_t da = gmma_desc(smem_u32(sA + (size_t)stage * TC_A_STAGE + (size_t)c * (TC_A_STAGE / 2)));
        const uint32_t b_addr = smem_u32(sB + (size_t)stage * B_STAGE);
        const uint64_t db = MNB ? gmma_desc_mn(b_addr) : gmma_desc(b_addr);
        acc_fence<BN / 2>(acc);
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < TC_BK / 16; ++k)
          // 16 k = 32 bytes along a K-major swizzle row (+2 in the address field), or 16 k-rows = 2 KiB of an MN-major tile (+128)
          wgmma_tile<BN, F16, MNB ? 1 : 0>(acc, da + (uint64_t)(k * 2), db + (uint64_t)k * (MNB ? 128u : 2u), (s | k) != 0 ? 1u : 0u);
        wgmma_commit();
        wgmma_wait<1>();                                           // the previous k-block's MMAs have retired: release its stage
        acc_fence<BN / 2>(acc);
        if (prev >= 0) release(prev);
        prev = stage;
        if (++stage == p.stages) { stage = 0; phase ^= 1; }
      }
      wgmma_wait<0>();
      acc_fence<BN / 2>(acc);
      if (prev >= 0) release(prev);
      CT_TRACE(2);

      // ---- epilogue: this thread's fragment holds rows r and r + 8 of the warpgroup's 64, columns 8j + 2 (lane % 4) + {0, 1} ----
      const int n0 = n_tile * BN;                                  // gemm: N tile n of tap t is column t * Nper + (n % gemm_ntile_tap) * BN
      const int row0 = m_tile * TC_BM + c * 64;
      const int r0 = warp * 16 + (lane >> 2);
      if constexpr (MNB) {                                         // weight-gradient GEMM: plain fp32 [M][Cout_pad], stored or added
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const long long m = (long long)row0 + r0 + 8 * h;
          if (m >= p.M) continue;
#pragma unroll
          for (int j = 0; j < BN / 8; ++j) {
            float2* o = reinterpret_cast<float2*>((float*)p.out + m * p.Cout_pad + n0 + 8 * j + 2 * (lane & 3));
            const float2 v = make_float2(acc[4 * j + 2 * h], acc[4 * j + 2 * h + 1]);
            if (p.accumulate) atomicAdd(o, v);
            else *o = v;
          }
        }
      } else if (p.out_mode == 0) {
        // ---- 16-bit haloed rows: staged per segment, stored by TMA ----
        bool zero[2];                                              // halo rows are zero (rows >= M too; the store clips them)
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const long long m = (long long)row0 + r0 + 8 * h;
          zero[h] = true;
          if (m < p.M) {
            const int pos = (int)(m % p.g.plane());
            const int y = pos / p.g.Wp(), x = pos - y * p.g.Wp();
            zero[h] = y == 0 || y == p.g.H + 1 || x == 0 || x == p.g.W + 1;
          }
        }
        const float2* bias = reinterpret_cast<const float2*>(p.bias + n0) + (lane & 3);
        // the loop for one activation and residual setting (compile-time ACT / RES): the per-value arithmetic is straight-line code
        auto stage_tile = [&](auto act_c, auto res_c) {
          constexpr int ACT = decltype(act_c)::value;
          constexpr bool RES = decltype(res_c)::value;
#pragma unroll
        for (int j = 0; j < BN / 8; ++j) {                         // j is a compile-time index: the segment arithmetic folds away
          const int s = Segs16<BN>::of(8 * j), w = Segs16<BN>::width(s), sb = Segs16<BN>::base(s);
          uint8_t* buf = stg + (q & 1) * TC_STG_BYTES;
          if (RES && 8 * j == sb) mbar_wait(&res_full[2 * c + (q & 1)], (q >> 1) & 1);
          const float2 b = __ldg(bias + 4 * j);
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            const uint32_t a = smem_u32(buf) + stg_off16(r0 + 8 * h, 8 * j - sb + 2 * (lane & 3), w);
            float v0 = b.x + acc[4 * j + 2 * h], v1 = b.y + acc[4 * j + 2 * h + 1];
            if (RES) {
              const float2 rr = unpack2<F16>(lds32(a));
              v0 += rr.x; v1 += rr.y;
            }
            const uint32_t pk = pack2<F16>(apply_act(v0, ACT), apply_act(v1, ACT));
            sts32(a, zero[h] ? 0u : pk);
          }
          if (8 * j + 8 == sb + w) {                               // the segment is complete
            if (8 * j + 8 == BN) CT_TRACE(3);
            fence_async_smem();
            if (t == 0) bulk_wait_read0();                         // the previous segment's store has read the other buffer
            named_barrier_sync(1 + c, 128);
            if (t == 0) {
              tma_store_2d(&maps.out[seg_map(w)], buf, n0 + sb, row0);
              bulk_commit();
              if (RES) {                                           // the next segment's residual box, into the other buffer
                int mt, nt;
                if (s + 1 < Segs16<BN>::count) load_res(q + 1, m_tile, n_tile, s + 1);
                else if (tile_at(p, i + 1, mt, nt)) load_res(q + 1, mt, nt, 0);
              }
            }
            ++q;
          }
        }
        };
        using F = std::false_type;
        using T = std::true_type;
        using A0 = std::integral_constant<int, 0>;
        using A1 = std::integral_constant<int, 1>;
        using A2 = std::integral_constant<int, 2>;
        if (p.residual) {
          if (p.relu == 1) stage_tile(A1{}, T{}); else if (p.relu == 2) stage_tile(A2{}, T{}); else stage_tile(A0{}, T{});
        } else {
          if (p.relu == 1) stage_tile(A1{}, F{}); else if (p.relu == 2) stage_tile(A2{}, F{}); else stage_tile(A0{}, F{});
        }
      } else {
        // ---- dense fp32 rows (halo rows skipped): staged per segment, copied out with 16-byte stores ----
        // thread t copies 16-byte chunk t % 8 of rows t / 8 + 16k; drow: their dense rows, -1 for halo rows and rows >= M
        long long drow[4];
#pragma unroll
        for (int k = 0; k < 4; ++k) {
          const long long m = (long long)row0 + (t >> 3) + 16 * k;
          drow[k] = -1;
          if (m < p.M) {
            const int plane = p.g.plane();
            const int img = (int)(m / plane);
            const int pos = (int)(m - (long long)img * plane);
            const int y = pos / p.g.Wp(), x = pos - y * p.g.Wp();
            if (!(y == 0 || y == p.g.H + 1 || x == 0 || x == p.g.W + 1)) drow[k] = ((long long)img * p.g.H + (y - 1)) * p.g.W + (x - 1);
          }
        }
        const float2* bias = reinterpret_cast<const float2*>(p.bias + n0) + (lane & 3);
        auto stage_tile = [&](auto act_c) {                        // as above: one loop per activation
          constexpr int ACT = decltype(act_c)::value;
#pragma unroll
        for (int j = 0; j < BN / 8; ++j) {
          const int sb = (8 * j) / 32 * 32, w = BN - sb < 32 ? BN - sb : 32;
          const uint32_t buf = smem_u32(stg + (q & 1) * TC_STG_BYTES);
          const float2 b = __ldg(bias + 4 * j);
#pragma unroll
          for (int h = 0; h < 2; ++h)
            sts64(buf + stg_off32(r0 + 8 * h, 8 * j - sb + 2 * (lane & 3)), apply_act(b.x + acc[4 * j + 2 * h], ACT),
                  apply_act(b.y + acc[4 * j + 2 * h + 1], ACT));
          if (8 * j + 8 == sb + w) {
            if (8 * j + 8 == BN) CT_TRACE(3);
            // every thread has staged this segment and finished copying out the previous one from the other buffer
            named_barrier_sync(1 + c, 128);
            const int ch = t & 7;
            if (ch < w / 4) {
#pragma unroll
              for (int k = 0; k < 4; ++k)
                if (drow[k] >= 0)
                  *reinterpret_cast<float4*>((float*)p.out + drow[k] * p.Cout_pad + n0 + sb + 4 * ch) = lds128(buf + stg_off32((t >> 3) + 16 * k, 4 * ch));
            }
            ++q;
          }
        }
        };
        if (p.relu == 1) stage_tile(std::integral_constant<int, 1>{});
        else if (p.relu == 2) stage_tile(std::integral_constant<int, 2>{});
        else stage_tile(std::integral_constant<int, 0>{});
      }
      CT_TRACE(4);                                                 // 16-bit: after the last segment's TMA store was issued
    }
    if (!MNB && t == 0) bulk_wait0();                              // the TMA stores are complete before the CTA exits
    if (t == 0) CT_TRACE_CTA(1 + c);
  }
  if (p.pair) cluster_sync_all();                                  // neither CTA leaves while the peer may still signal its barriers
}

// =================================================================================================================
// Fused bottleneck tail + next head (layers.cuh BneckArgs), persistent, one 128-row tile at a time, the same three warpgroups:
//   for each 128-channel chunk c of the expanded width:
//     A(c):  accA  = t2 * W3_c^T                 (wgmma m64n128, K = Cin [+ Cd: the folded downsample branch])
//     E(c):  x'_c  = relu(accA + b3_c [+ x_c])   -> 16 bit, in shared memory in the 128B-swizzled A-operand layout -> xo (TMA store)
//     B(c):  accB += x'_c * W1_c^T               (wgmma m64nCout, K = 128)
//   t1 = relu(accB + b1) -> HBM.
// Cin is the t2 width (this block's conv3 input), Cout the t1 width (the next block's conv1 output): equal inside a stage, Cout =
// 2 Cin where the next block opens a stage (layer1 -> layer2: 64 -> 256 -> 128, layer2 -> layer3: 128 -> 512 -> 256).
// x' never makes a round trip through HBM before the next block's conv1.  The operand rounding points, the k order and the epilogue
// arithmetic are those of the two separate k_conv_tc launches, so the result is bit-identical to the unfused pair (the folded
// downsample branch skips one 16-bit rounding of the residual).  Both GEMMs' accumulators live in registers (64 + Cout / 2 per
// thread), so the consumers take 232 registers from the producer with setmaxnreg.
//
// Shared memory: the t2 tile (resident for the whole tile), two x buffers and a ring of weight slots in the order the consumers use
// them.  An x buffer is one chunk, [2 k-blocks][128 rows x 128 B] in the A-operand layout.  The producer loads the residual chunk x_c
// into it by TMA one chunk ahead; E(c) reads x_c and writes x'_c at the same swizzled address, so the buffer is in turn the residual,
// the A operand of B(c) and the source of the TMA store of xo (rows >= M are clipped by the store's tensor map).  A buffer is handed
// back to the producer once B(c) has retired and the store has read it.  Both GEMMs keep one k-block in flight and release a slot
// when it retires; B(c)'s last k-block retires under A(c+1).  Every slot is 16 KiB: one W3 k-block [128 rows][128 B], or one 128-row
// part of a W1 k-block ([min(Cout, 128) rows][128 B]; at Cout = 256 a W1 k-block is two parts, each the B operand of an m64n128 wgmma
// into its half of accB).  Small slots release early: a consumer warpgroup holds two (the group in flight and the one it issues),
// and the rest of the ring is the producer's lookahead.
// =================================================================================================================
struct BnParams {
  long long M;
  int m_tiles, Cexp, nch, kbA, kbT, has_res, slots;
  Geom g;
  const float* b3;
  const float* b1;
  void* t1;
#ifdef YB_BNECK_TRACE
  unsigned long long* trace;
#endif
};

// Trace build (tools/trace_bneck.cu; the library never defines YB_BNECK_TRACE): thread 0 of each consumer warpgroup writes
// %globaltimer stamps to trace[((cta * 2 + warpgroup) * BN_TRACE_TILES + tile) * BN_TRACE_SLOTS + slot] for the launch that
// bn_trace_buf points at.  Slots: 0 tile start; 1 + 5c + {0 A(c) issued, 1 A(c) drained, 2 x_full waited, 3 E(c) done, 4 B(c)
// issued}; BN_TRACE_T1 the t1 epilogue's start, BN_TRACE_T1 + 1 its end.
#ifdef YB_BNECK_TRACE
constexpr int BN_TRACE_TILES = 8, BN_TRACE_SLOTS = 44, BN_TRACE_T1 = 41;
unsigned long long* bn_trace_buf = nullptr;
#define BN_TRACE(slot)                                                                                                     \
  do {                                                                                                                     \
    if (p.trace && t == 0 && i < BN_TRACE_TILES) {                                                                         \
      unsigned long long ns_;                                                                                              \
      asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(ns_));                                                              \
      p.trace[(((size_t)blockIdx.x * 2 + cw) * BN_TRACE_TILES + i) * BN_TRACE_SLOTS + (slot)] = ns_;                      \
    }                                                                                                                      \
  } while (0)
#else
#define BN_TRACE(slot) do { } while (0)
#endif

constexpr uint32_t BN_X_BYTES = 2 * TC_A_STAGE;                  // one x buffer: 128 rows x 128 channels
constexpr uint32_t BN_B3_BYTES = 128 * 4;                        // b3 of one chunk, beside each x buffer
constexpr uint32_t BN_SLOT = TC_A_STAGE;                         // one ring slot: 128 rows x 128 B

template <bool F16, int COUT>
__global__ void __launch_bounds__(TC_THREADS, 1)
k_bneck_tc(const __grid_constant__ CUtensorMap tmT2, const __grid_constant__ CUtensorMap tmXd, const __grid_constant__ CUtensorMap tmW3,
           const __grid_constant__ CUtensorMap tmW1, const __grid_constant__ CUtensorMap tmX, const __grid_constant__ CUtensorMap tmXo,
           const BnParams p) {
  constexpr int W1R = COUT < 128 ? COUT : 128;                   // rows of one W1 part (one ring slot)
  constexpr int W1P = COUT / W1R;                                // W1 parts per k-block
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = (uint8_t*)(((uintptr_t)smem_raw + 1023) & ~(uintptr_t)1023);
  uint8_t* sT2 = smem;                                         // [kbA][128 rows x 128 B]
  uint8_t* sX = sT2 + (size_t)p.kbA * TC_A_STAGE;              // [2 buffers][2 k-blocks][128 rows x 128 B]
  uint8_t* sB3 = sX + 2 * BN_X_BYTES;                          // [2 buffers][128 floats]: b3 of the chunk in x buffer b
  uint8_t* sRing = sB3 + 2 * BN_B3_BYTES;                      // [slots][BN_SLOT]
  uint64_t* full = reinterpret_cast<uint64_t*>(sRing + (size_t)p.slots * BN_SLOT);
  uint64_t* empty = full + TC_MAX_STAGES;
  uint64_t* t2_full = empty + TC_MAX_STAGES;
  uint64_t* t2_empty = t2_full + 1;
  uint64_t* x_full = t2_empty + 1;                             // [2]
  uint64_t* x_empty = x_full + 2;                              // [2]

  const int wg = threadIdx.x >> 7;
  if (threadIdx.x == 0) {
    for (int i = 0; i < TC_MAX_STAGES; ++i) { mbar_init(&full[i], 1); mbar_init(&empty[i], 8); }
    mbar_init(t2_full, 1); mbar_init(t2_empty, 8);
    for (int i = 0; i < 2; ++i) { mbar_init(&x_full[i], 1); mbar_init(&x_empty[i], 8); }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();
  griddep_launch_dependents();

  if (wg == 0) {
    // ================= TMA producer =================
    asm volatile("setmaxnreg.dec.sync.aligned.u32 40;" ::: "memory");
    if (threadIdx.x == 0) {
      griddep_wait();
      int stage = 0; uint32_t phase = 0;
      int q = 0;                                                 // chunk count over all tiles: x buffer q & 1
      for (int i = 0, tile = (int)blockIdx.x; tile < p.m_tiles; ++i, tile += (int)gridDim.x) {
        const int row0 = tile * TC_BM;
        mbar_wait(t2_empty, (uint32_t)(i & 1) ^ 1u);                // the previous tile's A GEMMs have read the resident t2 tile
        mbar_expect_tx(t2_full, (uint32_t)p.kbA * TC_A_STAGE);
        for (int kb = 0; kb < p.kbA; ++kb)                          // t2's k-blocks, then the block input's (folded downsample)
          tma_load_2d(sT2 + (size_t)kb * TC_A_STAGE, kb < p.kbT ? &tmT2 : &tmXd, (kb < p.kbT ? kb : kb - p.kbT) * TC_BK, row0, t2_full);
        for (int c = 0; c < p.nch; ++c, ++q) {
          const int xb = q & 1;
          mbar_wait(&x_empty[xb], (uint32_t)((q >> 1) & 1) ^ 1u);   // B(q-2) has retired and xo's store has read the buffer
          // the chunk's b3 with it (folded branch: no residual, the buffer only holds x')
          mbar_expect_tx(&x_full[xb], (p.has_res ? BN_X_BYTES : 0u) + BN_B3_BYTES);
          bulk_load(sB3 + (size_t)xb * BN_B3_BYTES, p.b3 + c * 128, BN_B3_BYTES, &x_full[xb]);
          if (p.has_res)
            for (int kb = 0; kb < 2; ++kb)
              tma_load_2d(sX + (size_t)xb * BN_X_BYTES + (size_t)kb * TC_A_STAGE, &tmX, c * 128 + kb * TC_BK, row0, &x_full[xb]);
          for (int kb = 0; kb < p.kbA; ++kb) {                      // W3 rows c*128 .., k-block kb
            mbar_wait(&empty[stage], phase ^ 1);
            mbar_expect_tx(&full[stage], TC_A_STAGE);
            tma_load_2d(sRing + (size_t)stage * BN_SLOT, &tmW3, kb * TC_BK, c * 128, &full[stage]);
            if (++stage == p.slots) { stage = 0; phase ^= 1; }
          }
          for (int kb = 0; kb < 2 * W1P; ++kb) {                    // W1[part * W1R .., c*128 + (kb / W1P)*64 ..]
            mbar_wait(&empty[stage], phase ^ 1);
            mbar_expect_tx(&full[stage], (uint32_t)W1R * 128u);
            tma_load_2d(sRing + (size_t)stage * BN_SLOT, &tmW1, c * 128 + (kb / W1P) * TC_BK, (kb % W1P) * W1R, &full[stage]);
            if (++stage == p.slots) { stage = 0; phase ^= 1; }
          }
        }
      }
    }
  } else {
    // ================= consumers: warpgroup c owns rows 64c .. 64c+63 of every tile =================
    asm volatile("setmaxnreg.inc.sync.aligned.u32 232;" ::: "memory");
    const int cw = wg - 1;
    const int t = threadIdx.x & 127, warp = t >> 5, lane = t & 31;
    const bool signal = lane == 0;
    griddep_wait();
    float accA[64];
    float accB[COUT / 2];
    int stage = 0; uint32_t phase = 0;
    int prev = -1;                                               // ring slot whose MMAs are still in flight
    int xpend = -1;                                              // x buffer read by the in-flight B(c)
    auto release = [&](int s) { if (signal) mbar_arrive(&empty[s]); };
    auto release_x = [&](int b) {                                // B(c) has retired: hand the buffer back once xo's store has read it
      if (t == 0) bulk_wait_read0();
      if (signal) mbar_arrive(&x_empty[b]);
    };
    int q = 0;
    for (int i = 0, tile = (int)blockIdx.x; tile < p.m_tiles; ++i, tile += (int)gridDim.x) {
      BN_TRACE(0);
      long long m[2];
      bool valid[2], zero[2];
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        m[h] = (long long)tile * TC_BM + cw * 64 + warp * 16 + (lane >> 2) + 8 * h;
        valid[h] = m[h] < p.M;
        zero[h] = true;
        if (valid[h]) {
          const int pos = (int)(m[h] % p.g.plane());
          const int y = pos / p.g.Wp(), x = pos - y * p.g.Wp();
          zero[h] = y == 0 || y == p.g.H + 1 || x == 0 || x == p.g.W + 1;
        }
      }
      mbar_wait(t2_full, (uint32_t)(i & 1));
      for (int c = 0; c < p.nch; ++c, ++q) {
        const int xb = q & 1;
        // ---- A(c) ----
        for (int kb = 0; kb < p.kbA; ++kb) {
          mbar_wait(&full[stage], phase);
          const uint64_t da = gmma_desc(smem_u32(sT2 + (size_t)kb * TC_A_STAGE + (size_t)cw * (TC_A_STAGE / 2)));
          const uint64_t db = gmma_desc(smem_u32(sRing + (size_t)stage * BN_SLOT));
          acc_fence<64>(accA);
          wgmma_fence();
#pragma unroll
          for (int k = 0; k < TC_BK / 16; ++k)
            wgmma_n128<F16, 0>(accA, da + (uint64_t)(k * 2), db + (uint64_t)(k * 2), (kb | k) != 0 ? 1u : 0u);
          wgmma_commit();
          wgmma_wait<1>();                                         // the previous group (a W3 slot, or B(c-1)'s last k-block) has retired
          acc_fence<64>(accA);
          if (prev >= 0) release(prev);
          prev = stage;
          if (xpend >= 0) { release_x(xpend); xpend = -1; }
          if (++stage == p.slots) { stage = 0; phase ^= 1; }
        }
        BN_TRACE(1 + 5 * c);
        wgmma_wait<0>();
        acc_fence<64>(accA);
        BN_TRACE(2 + 5 * c);
        release(prev);
        prev = -1;
        if (c == p.nch - 1 && signal) mbar_arrive(t2_empty);
        // ---- E(c): rows r, r + 8 of this thread, columns c*128 + 8j + 2 (lane % 4) + {0, 1} ----
        mbar_wait(&x_full[xb], (uint32_t)((q >> 1) & 1));          // x_c and its b3 have landed (and the buffer is free)
        BN_TRACE(3 + 5 * c);
        const uint32_t sXw = smem_u32(sX + (size_t)xb * BN_X_BYTES + (size_t)cw * (TC_A_STAGE / 2));   // this warpgroup's 64 rows
        // b3 from shared memory: per column group a global load would miss the small L1 left beside the shared-memory carve-out and
        // wait out an L2 latency behind the previous group's shared-memory store
        const uint32_t b3 = smem_u32(sB3 + (size_t)xb * BN_B3_BYTES) + 8u * (lane & 3);
#pragma unroll
        for (int j = 0; j < 16; ++j) {
          const float2 b = lds64(b3 + 32u * j);                    // columns c*128 + 8j + 2 (lane % 4) + {0, 1}: shared by both rows
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            const int r = warp * 16 + (lane >> 2) + 8 * h;        // row in this warpgroup's 64-row slab
            // A-operand layout: k-block j / 8, 16-byte chunk (j % 8) ^ (r % 8) of row r, element pair 2 (lane % 4)
            const uint32_t a = sXw + (uint32_t)(j >> 3) * TC_A_STAGE + (uint32_t)r * 128u + ((uint32_t)((j & 7) ^ (r & 7)) << 4) + 4u * (lane & 3);
            float v0 = b.x + accA[4 * j + 2 * h], v1 = b.y + accA[4 * j + 2 * h + 1];
            if (p.has_res) {
              const float2 rr = unpack2<F16>(lds32(a));
              v0 += rr.x; v1 += rr.y;
            }
            const uint32_t pk = pack2<F16>(apply_act(v0, 1), apply_act(v1, 1));
            sts32(a, zero[h] ? 0u : pk);                           // halo rows (and rows >= M) are zero
          }
        }
        fence_async_smem();
        named_barrier_sync(1 + cw, 128);                           // the whole x' chunk of this warpgroup is staged
        BN_TRACE(4 + 5 * c);
        if (t == 0) {
          const int row = tile * TC_BM + cw * 64;
#pragma unroll
          for (int kb = 0; kb < 2; ++kb)
            tma_store_2d(&tmXo, sX + (size_t)xb * BN_X_BYTES + (size_t)kb * TC_A_STAGE + (size_t)cw * (TC_A_STAGE / 2), c * 128 + kb * TC_BK, row);
          bulk_commit();
        }
        // ---- B(c): k-block kb / W1P, W1 part kb % W1P -> columns (kb % W1P) * W1R .. of accB ----
#pragma unroll
        for (int kb = 0; kb < 2 * W1P; ++kb) {
          mbar_wait(&full[stage], phase);
          const uint64_t da = gmma_desc(sXw + (uint32_t)(kb / W1P) * TC_A_STAGE);
          const uint64_t db = gmma_desc(smem_u32(sRing + (size_t)stage * BN_SLOT));
          acc_fence<COUT / 2>(accB);
          wgmma_fence();
#pragma unroll
          for (int k = 0; k < TC_BK / 16; ++k)
            wgmma_tile<W1R, F16, 0>(accB + (kb % W1P) * (W1R / 2), da + (uint64_t)(k * 2), db + (uint64_t)(k * 2), (c | (kb / W1P) | k) != 0 ? 1u : 0u);
          wgmma_commit();
          wgmma_wait<1>();
          acc_fence<COUT / 2>(accB);
          if (prev >= 0) release(prev);
          prev = stage;
          if (++stage == p.slots) { stage = 0; phase ^= 1; }
        }
        BN_TRACE(5 + 5 * c);
        xpend = xb;
      }
      wgmma_wait<0>();
      acc_fence<COUT / 2>(accB);
      BN_TRACE(BN_TRACE_T1);
      release(prev);
      prev = -1;
      release_x(xpend);
      xpend = -1;
      // ---- t1 = relu(accB + b1), halo rows zero ----
      // Lane l of a quad holds 4 bytes of a row per column group j (words 4j + l).  One xor shuffle between lanes l and l ^ 1 gives
      // each lane 8 contiguous bytes of group 2g (even lanes) or 2g + 1 (odd lanes), so a quad stores a full 32-byte sector per row.
      const float2* b1 = reinterpret_cast<const float2*>(p.b1) + (lane & 3);
      const bool odd = lane & 1;
#pragma unroll
      for (int g = 0; g < COUT / 16; ++g) {
        const float2 ba = __ldg(b1 + 8 * g), bb = __ldg(b1 + 8 * g + 4);         // groups 2g, 2g + 1: shared by both rows
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          uint32_t v0 = pack2<F16>(apply_act(ba.x + accB[8 * g + 2 * h], 1), apply_act(ba.y + accB[8 * g + 2 * h + 1], 1));
          uint32_t v1 = pack2<F16>(apply_act(bb.x + accB[8 * g + 4 + 2 * h], 1), apply_act(bb.y + accB[8 * g + 4 + 2 * h + 1], 1));
          const uint32_t r = __shfl_xor_sync(0xffffffffu, odd ? v0 : v1, 1);
          if (odd) v0 = r; else v1 = r;
          if (valid[h])
            reinterpret_cast<uint2*>((uint16_t*)p.t1 + m[h] * COUT)[4 * g + 2 * (lane & 1) + ((lane >> 1) & 1)] = zero[h] ? make_uint2(0u, 0u) : make_uint2(v0, v1);
        }
      }
      BN_TRACE(BN_TRACE_T1 + 1);
    }
    if (t == 0) bulk_wait0();                                      // xo's stores are complete before the CTA exits
  }
}

// ---- host side -----------------------------------------------------------------------------------
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                  const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static EncodeTiledFn get_encode() {
  static EncodeTiledFn fn = nullptr;
  static std::once_flag once;
  std::call_once(once, [] {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess && q == cudaDriverEntryPointSuccess)
      fn = (EncodeTiledFn)p;
  });
  return fn;
}

// 2D map over a 16-bit [rows][inner] matrix; the swizzle spans a box row: 128 B for 64 elements, 64 B for 32, 32 B for 16
static int make_map(CUtensorMap* map, const void* base, uint64_t inner, uint64_t rows, uint32_t box_rows, bool f16,
                    uint32_t box_inner = TC_BK, uint64_t row_stride = 0) {
  EncodeTiledFn enc = get_encode();
  YB_REQUIRE(enc != nullptr, YB_ERR_CUDA, "cuTensorMapEncodeTiled entry point not available");
  const cuuint64_t dims[2] = {inner, rows};
  const cuuint64_t strides[1] = {(row_stride ? row_stride : inner) * 2};
  const cuuint32_t box[2] = {box_inner, box_rows};
  const cuuint32_t estr[2] = {1, 1};
  const CUtensorMapSwizzle swz = box_inner == 64 ? CU_TENSOR_MAP_SWIZZLE_128B : box_inner == 32 ? CU_TENSOR_MAP_SWIZZLE_64B : CU_TENSOR_MAP_SWIZZLE_32B;
  CUresult r = enc(map, f16 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT16 : CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, const_cast<void*>(base), dims, strides, box, estr,
                   CU_TENSOR_MAP_INTERLEAVE_NONE, swz, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  YB_REQUIRE(r == CUDA_SUCCESS, YB_ERR_CUDA, "cuTensorMapEncodeTiled failed (%d) inner=%llu rows=%llu box_rows=%u", (int)r,
             (unsigned long long)inner, (unsigned long long)rows, box_rows);
  return YB_OK;
}

bool tc_overlapping_rows_ok() {
  EncodeTiledFn enc = get_encode();
  if (!enc) return false;
  alignas(64) static CUtensorMap probe;
  const cuuint64_t dims[2] = {64, 4096};
  const cuuint64_t strides[1] = {32};
  const cuuint32_t box[2] = {64, 128};
  const cuuint32_t estr[2] = {1, 1};
  void* base = nullptr;
  if (cudaMalloc(&base, 4096 * 32 + 128) != cudaSuccess) { cudaGetLastError(); return false; }
  const CUresult r = enc(&probe, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2, base, dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                         CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  cudaFree(base);
  return r == CUDA_SUCCESS;
}

// call f(kernel) with the instantiation for (f16, MN-major B, BN)
template <class F> static cudaError_t with_kernel(bool f16, bool mnb, int bn, F&& f) {
#define YB_TC_CASE(N)                                                              \
  case N:                                                                          \
    return f16 ? f(k_conv_tc<true, false, N>) : f(k_conv_tc<false, false, N>);
#define YB_TC_CASE_MN(N)                                                           \
  case N:                                                                          \
    return f16 ? f(k_conv_tc<true, true, N>) : f(k_conv_tc<false, true, N>);
  if (mnb) {
    switch (bn) { YB_TC_CASE_MN(64) YB_TC_CASE_MN(128) YB_TC_CASE_MN(256) }
  } else {
    switch (bn) { YB_TC_CASE(16) YB_TC_CASE(32) YB_TC_CASE(64) YB_TC_CASE(96) YB_TC_CASE(128) YB_TC_CASE(176) YB_TC_CASE(192) YB_TC_CASE(256) }
  }
#undef YB_TC_CASE
#undef YB_TC_CASE_MN
  return cudaErrorInvalidValue;
}

// does the 16-bit staged epilogue of a BN-wide tile have a segment of width w (Segs16)?
static bool seg_width_used(int bn, int w) { return w == 64 ? bn >= 64 : w == 32 ? bn % 64 >= 32 : bn % 32 != 0; }

// the tile widths with a kernel instantiation (wgmma.cuh), widest first
static const int kTileWidths[] = {256, 192, 176, 128, 96, 64, 32, 16};

static int pick_bn(int cout_pad) {
  if (const char* e = getenv("YOLACT_B200_BN")) {                    // tooling
    const int v = atoi(e);
    for (int w : kTileWidths) if (w == v && cout_pad % v == 0) return v;
  }
  for (int w : kTileWidths) if (cout_pad % w == 0) return w;       // 1152 -> 192, 352 -> 176, 288 -> 96
  return 0;
}

bool tc_supported(const ConvArgs& a) {
  if (a.act_dt != DT_BF16 && a.act_dt != DT_F16) return false;
  if (a.Cin % 8 != 0 || a.Cin_pad % TC_BK != 0 || a.Cin_pad < a.Cin) return false;
  if (a.out_mode == 0 && a.Cout != a.Cout_pad) return false;
  return pick_bn(a.Cout_pad) != 0;
}

// per-device set-up and SM count; the kernel's dynamic shared-memory limit is raised for the plan's instantiation
static int tc_device_setup(bool f16, bool mnb, int bn, int* sms) {
  int dev = 0;
  YB_CHECK_CUDA(cudaGetDevice(&dev));
  // the instantiation's limit is the whole 227 KB: plans of different sizes share one instantiation
  YB_CHECK_CUDA(with_kernel(f16, mnb, bn, [&](auto k) { return cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)TC_SMEM_MAX); }));
  YB_CHECK_CUDA(cudaDeviceGetAttribute(sms, cudaDevAttrMultiProcessorCount, dev));
  YB_REQUIRE(*sms > 0, YB_ERR_CUDA, "cannot read the SM count");
  return YB_OK;
}

static void plan_stages(TcPlan* pl) {
  const size_t per_stage = TC_A_STAGE + (size_t)pl->BN * TC_BK * 2;
  const size_t fixed = 1024 /*align*/ + (2 * TC_MAX_STAGES + 4) * 8 /*barriers*/ + (pl->gemm ? 0 : TC_STG_TOTAL);
  int stages = (int)((TC_SMEM_MAX - fixed) / per_stage);
  pl->stages = stages > TC_MAX_STAGES ? TC_MAX_STAGES : stages;
  pl->smem_bytes = (size_t)pl->stages * per_stage + fixed;
}

int tc_plan_create(const ConvArgs& a, int max_batch, TcPlan** out) {
  YB_REQUIRE(tc_supported(a), YB_ERR_UNSUPPORTED, "tc_plan_create: unsupported conv Cin=%d Cout_pad=%d", a.Cin, a.Cout_pad);
  YB_REQUIRE(!a.residual || a.out_mode == 0, YB_ERR_UNSUPPORTED, "tc_plan_create: a residual needs the 16-bit haloed output");
  TcPlan* pl = new TcPlan();
  pl->gemm = 0;
  pl->BN = pick_bn(a.Cout_pad);
  // The pair form is selected with YOLACT_B200_PAIR=1 (A-B runs; it is checked at every test shape); the default is one CTA per tile.
  const char* e_pair = getenv("YOLACT_B200_PAIR");
  pl->pair = (e_pair && atoi(e_pair) != 0) ? 1 : 0;
  plan_stages(pl);
  const int Ktot = a.ntaps * a.Cin_pad;
  const int cout_alloc = (a.Cout_pad + 63) / 64 * 64;
  const bool f16 = a.act_dt == DT_F16;
  int s = make_map(&pl->tmA, a.in, (uint64_t)a.Cin, (uint64_t)a.in_rows, TC_BM, f16, TC_BK, (uint64_t)a.in_row_stride);
  if (s == YB_OK) s = make_map(&pl->tmB, a.weight, (uint64_t)Ktot, (uint64_t)cout_alloc, (uint32_t)(pl->pair ? pl->BN / 2 : pl->BN), f16, TC_BK,
                               (uint64_t)a.w_ld);
  for (int w : {64, 32, 16}) {                                     // the residual boxes of the tile's segment widths (placeholders otherwise)
    CUtensorMap* m = &pl->tmRes[seg_map(w)];
    *m = pl->tmA;
    if (s == YB_OK && a.residual && seg_width_used(pl->BN, w))
      s = make_map(m, a.residual, (uint64_t)a.Cout, (uint64_t)max_batch * a.g.plane(), 64, f16, (uint32_t)w);
  }
  if (s == YB_OK) s = tc_device_setup(f16, false, pl->BN, &pl->sms);
  if (s != YB_OK) { delete pl; return s; }
  *out = pl;
  return YB_OK;
}

void tc_plan_destroy(TcPlan* p) { delete p; }

static int launch(const TcPlan* pl, const TcParams& p, const TcMaps& maps, bool f16, int grid, cudaStream_t s) {
  static const bool pdl = getenv("YOLACT_B200_NO_PDL") == nullptr;
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3((unsigned)grid); cfg.blockDim = dim3(TC_THREADS); cfg.dynamicSmemBytes = pl->smem_bytes; cfg.stream = s;
  cudaLaunchAttribute attr[2];
  int na = 0;
  if (pdl) {
    attr[na].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[na].val.programmaticStreamSerializationAllowed = 1;
    ++na;
  }
  if (p.pair) {
    attr[na].id = cudaLaunchAttributeClusterDimension;
    attr[na].val.clusterDim.x = 2; attr[na].val.clusterDim.y = 1; attr[na].val.clusterDim.z = 1;
    ++na;
  }
  cfg.attrs = attr; cfg.numAttrs = na;
  YB_CHECK_CUDA(with_kernel(f16, pl->gemm != 0, pl->BN, [&](auto k) { return cudaLaunchKernelEx(&cfg, k, pl->tmA, pl->tmB, maps, p); }));
  YB_CHECK_LAUNCH();
  return YB_OK;
}

// ---- plain GEMM over long K on the same kernel (weight gradients; see TcParams::gemm) ---------------------------
int tc_plan_create_gemm(const GemmArgs& g, TcPlan** out) {
  YB_REQUIRE(g.act_dt == DT_BF16 || g.act_dt == DT_F16, YB_ERR_UNSUPPORTED, "tc_plan_create_gemm: 16-bit operands only");
  YB_REQUIRE(g.M >= 1 && g.K >= 1 && g.lda % 8 == 0 && g.ldb % 8 == 0 && g.ldb > g.Nper - 64 && g.ntaps >= 1 && g.ntaps <= 16, YB_ERR_INVALID,
             "tc_plan_create_gemm: M=%d K=%d lda=%d ldb=%d ntaps=%d", g.M, g.K, g.lda, g.ldb, g.ntaps);
  int bn = 0;
  if (g.Nper % 256 == 0) bn = 256;
  else if (g.Nper % 128 == 0) bn = 128;
  else if (g.Nper % 64 == 0) bn = 64;
  YB_REQUIRE(bn != 0, YB_ERR_UNSUPPORTED, "tc_plan_create_gemm: N per tap = %d is not a multiple of 64", g.Nper);
  TcPlan* pl = new TcPlan();
  pl->gemm = 1; pl->BN = bn;
  plan_stages(pl);
  const bool f16 = g.act_dt == DT_F16;
  int s = make_map(&pl->tmA, g.a, (uint64_t)g.K, (uint64_t)g.M, TC_BM, f16, TC_BK, (uint64_t)g.lda);
  // B is read MN-major straight from the [Kb pixels][ldb channels] activations: boxes of [64 k-rows][64 channels].  With fewer than
  // Nper channels (ldb = 96, Nper = 128: Swin-T stage 1) the TMA zero-fills the last box's missing channels.
  const uint64_t nb = (uint64_t)(g.ldb < g.Nper ? g.ldb : g.Nper);
  if (s == YB_OK) s = make_map(&pl->tmB, g.b, nb, (uint64_t)g.Kb, 64, f16, TC_BK, (uint64_t)g.ldb);
  if (s == YB_OK) s = tc_device_setup(f16, true, bn, &pl->sms);
  if (s != YB_OK) { delete pl; return s; }
  *out = pl;
  return YB_OK;
}

int launch_gemm_tc(const TcPlan* pl, const GemmArgs& g, cudaStream_t s) {
  YB_REQUIRE(pl && pl->gemm, YB_ERR_INVALID, "launch_gemm_tc: not a GEMM plan");
  TcParams p;
  memset(&p, 0, sizeof(p));
  p.M = g.M;
  p.m_tiles = (g.M + TC_BM - 1) / TC_BM;
  p.gemm = 1; p.gemm_ntile_tap = g.Nper / pl->BN;
  p.gemm_splits = g.splits > 0 ? g.splits : 1;
  p.n_tiles = g.ntaps * p.gemm_ntile_tap;
  p.kb_per_tap = (g.K + TC_BK - 1) / TC_BK;
  p.gemm_kb_split = (p.kb_per_tap + p.gemm_splits - 1) / p.gemm_splits;
  p.gemm_splits = (p.kb_per_tap + p.gemm_kb_split - 1) / p.gemm_kb_split;          // no empty split
  YB_REQUIRE(p.gemm_splits == 1 || g.accumulate, YB_ERR_INVALID, "launch_gemm_tc: split-K needs accumulate (atomic) output");
  p.ntaps = 1; p.tap_shift[0] = 0;
  for (int i = 0; i < g.ntaps; ++i) p.gemm_shift[i] = g.shift[i];
  p.stages = pl->stages;
  p.Cout = p.Cout_pad = g.ntaps * g.Nper; p.relu = 0; p.out_mode = 2; p.accumulate = g.accumulate;
  p.g.H = 1 << 20; p.g.W = 1 << 20;
  p.bias = nullptr; p.residual = 0; p.out = g.out;
  const int total = p.m_tiles * p.n_tiles * p.gemm_splits;
  TcMaps maps;                                                     // no staged epilogue: placeholders
  for (int k = 0; k < 3; ++k) maps.res[k] = maps.out[k] = pl->tmA;
  return launch(pl, p, maps, g.act_dt == DT_F16, total < pl->sms ? total : pl->sms, s);
}

int launch_conv_tc(const TcPlan* pl, const ConvArgs& a, cudaStream_t s) {
  TcParams p;
  memset(&p, 0, sizeof(p));
  p.M = (long long)a.B * a.g.plane();
  const int unit_rows = pl->pair ? 2 * TC_BM : TC_BM;
  p.m_tiles = (int)((p.M + unit_rows - 1) / unit_rows);            // tiles per scheduling unit (CTA or CTA pair)
  p.n_tiles = a.Cout_pad / pl->BN;
  p.pair = pl->pair;
  p.kb_per_tap = a.Cin_pad / TC_BK;
  p.ntaps = a.ntaps;
  for (int i = 0; i < kMaxTaps; ++i) p.tap_shift[i] = a.tap_shift[i];
  p.stages = pl->stages;
  p.Cout = a.Cout; p.Cout_pad = a.Cout_pad; p.relu = a.relu; p.out_mode = a.out_mode;
  p.g = a.g; p.bias = a.bias; p.out = a.out;
  p.residual = a.residual != nullptr;
  p.gemm = 0; p.gemm_ntile_tap = 1; p.gemm_splits = 1;
#ifdef YB_CONV_TRACE
  p.trace = conv_trace_buf;
#endif
  const int total = p.m_tiles * p.n_tiles;
  const int max_units = pl->pair ? pl->sms / 2 : pl->sms;
  const int units = total < max_units ? total : max_units;
  // 16-bit output: TMA store boxes of the tile's segment widths; the maps end at this launch's last row, so rows >= M stay untouched
  TcMaps maps;
  for (int w : {64, 32, 16}) {
    const int k = seg_map(w);
    maps.res[k] = pl->tmRes[k];
    maps.out[k] = pl->tmA;
    if (a.out_mode == 0 && seg_width_used(pl->BN, w))
      YB_PROPAGATE(make_map(&maps.out[k], a.out, (uint64_t)a.Cout, (uint64_t)p.M, 64, a.act_dt == DT_F16, (uint32_t)w));
  }
  return launch(pl, p, maps, a.act_dt == DT_F16, pl->pair ? 2 * units : units, s);
}

// ---- fused bottleneck tail (k_bneck_tc) ------------------------------------------------------------------------------
struct BnPlan {
  CUtensorMap tmT2, tmXd, tmW3, tmW1, tmX;                         // tmX: the residual, read by TMA in 128-row boxes
  int sms, Cin, Cout, Cd, slots;
  size_t smem_bytes;
};

template <class F> static cudaError_t with_bneck_kernel(bool f16, int cout, F&& f) {
  switch (cout) {
    case 64: return f16 ? f(k_bneck_tc<true, 64>) : f(k_bneck_tc<false, 64>);
    case 128: return f16 ? f(k_bneck_tc<true, 128>) : f(k_bneck_tc<false, 128>);
    case 256: return f16 ? f(k_bneck_tc<true, 256>) : f(k_bneck_tc<false, 256>);
  }
  return cudaErrorInvalidValue;
}

// (Cin, Cexp, Cout): the stride-1 blocks of layer1 / layer2 / layer3 (Cout = Cin) and the first blocks of layer2 / layer3 (Cout = 2 Cin).
// Not layer3 -> layer4 (256, 1024, 512): accB would need 256 registers per thread.
bool bneck_supported(int act_dt, int Cin, int Cexp, int Cout) {
  const bool widths = Cexp == 4 * Cin && (((Cin == 64 || Cin == 128 || Cin == 256) && Cout == Cin) || ((Cin == 64 || Cin == 128) && Cout == 2 * Cin));
  return (act_dt == DT_F16 || act_dt == DT_BF16) && widths && !getenv("YOLACT_B200_NO_FUSE");
}

int bneck_plan_create(const BneckArgs& a, int max_batch, BnPlan** out) {
  YB_REQUIRE(bneck_supported(a.act_dt, a.Cin, a.Cexp, a.Cout), YB_ERR_UNSUPPORTED, "bneck_plan_create: unsupported Cin=%d Cexp=%d Cout=%d", a.Cin,
             a.Cexp, a.Cout);
  YB_REQUIRE(a.Cd == 0 || (a.xd && a.Cd % 64 == 0 && (a.Cin + a.Cd) / 64 <= 4), YB_ERR_UNSUPPORTED, "bneck_plan_create: folded residual branch with Cd=%d", a.Cd);
  YB_REQUIRE(a.Cd != 0 || a.x, YB_ERR_INVALID, "bneck_plan_create: no residual");
  BnPlan* pl = new BnPlan();
  pl->Cin = a.Cin; pl->Cout = a.Cout; pl->Cd = a.Cd;
  const int kbA = (a.Cin + a.Cd) / 64;
  const size_t fixed = 1024 /*align*/ + (2 * TC_MAX_STAGES + 6) * 8 /*barriers*/ + (size_t)kbA * TC_A_STAGE + 2 * (BN_X_BYTES + BN_B3_BYTES);
  int slots = (int)((TC_SMEM_MAX - fixed) / BN_SLOT);
  pl->slots = slots > TC_MAX_STAGES ? TC_MAX_STAGES : slots;
  pl->smem_bytes = fixed + (size_t)pl->slots * BN_SLOT;
  const bool f16 = a.act_dt == DT_F16;
  const uint64_t rows = (uint64_t)max_batch * a.g.plane();
  int s = pl->slots >= 2 ? YB_OK : YB_ERR_UNSUPPORTED;
  if (s == YB_OK) s = make_map(&pl->tmT2, a.t2, (uint64_t)a.Cin, rows, TC_BM, f16);
  pl->tmXd = pl->tmT2;                                             // placeholder without a folded branch
  if (s == YB_OK && a.Cd) s = make_map(&pl->tmXd, a.xd, (uint64_t)a.Cd, rows, TC_BM, f16);
  pl->tmX = pl->tmT2;                                              // placeholder with a folded branch (no residual read)
  if (s == YB_OK && !a.Cd) s = make_map(&pl->tmX, a.x, (uint64_t)a.Cexp, rows, TC_BM, f16);
  if (s == YB_OK) s = make_map(&pl->tmW3, a.w3, (uint64_t)(a.Cin + a.Cd), (uint64_t)a.Cexp, 128, f16);
  if (s == YB_OK) s = make_map(&pl->tmW1, a.w1, (uint64_t)a.Cexp, (uint64_t)a.Cout, (uint32_t)(a.Cout < 128 ? a.Cout : 128), f16);
  int dev = 0;
  if (s == YB_OK && cudaGetDevice(&dev) != cudaSuccess) s = YB_ERR_CUDA;
  if (s == YB_OK && cudaDeviceGetAttribute(&pl->sms, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess) s = YB_ERR_CUDA;
  if (s == YB_OK && with_bneck_kernel(f16, a.Cout, [&](auto k) {
        return cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)TC_SMEM_MAX); }) != cudaSuccess) s = YB_ERR_CUDA;
  if (s != YB_OK) { delete pl; return s; }
  *out = pl;
  return YB_OK;
}

void bneck_plan_destroy(BnPlan* p) { delete p; }

int launch_bneck_tc(const BnPlan* pl, const BneckArgs& a, cudaStream_t s) {
  BnParams p;
  memset(&p, 0, sizeof(p));
  p.M = (long long)a.B * a.g.plane();
  p.m_tiles = (int)((p.M + TC_BM - 1) / TC_BM);
  p.Cexp = a.Cexp; p.nch = a.Cexp / 128; p.kbT = pl->Cin / 64; p.kbA = (pl->Cin + pl->Cd) / 64; p.has_res = pl->Cd ? 0 : 1;
  p.slots = pl->slots;
  p.g = a.g; p.b3 = a.b3; p.b1 = a.b1; p.t1 = a.t1;
#ifdef YB_BNECK_TRACE
  p.trace = bn_trace_buf;
#endif
  // xo is written by TMA stores of [64 rows x 64 channels]; the map ends at this launch's last row, so rows >= M stay untouched
  YB_REQUIRE(((uintptr_t)a.b3 & 15) == 0, YB_ERR_INVALID, "launch_bneck_tc: b3 is not 16-byte aligned (bulk copy)");
  CUtensorMap tmXo;
  YB_PROPAGATE(make_map(&tmXo, a.xo, (uint64_t)a.Cexp, (uint64_t)p.M, 64, a.act_dt == DT_F16));
  static const bool pdl = getenv("YOLACT_B200_NO_PDL") == nullptr;
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3((unsigned)(p.m_tiles < pl->sms ? p.m_tiles : pl->sms)); cfg.blockDim = dim3(TC_THREADS);
  cfg.dynamicSmemBytes = pl->smem_bytes; cfg.stream = s;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr; cfg.numAttrs = pdl ? 1 : 0;
  YB_CHECK_CUDA(with_bneck_kernel(a.act_dt == DT_F16, pl->Cout, [&](auto k) { return cudaLaunchKernelEx(&cfg, k, pl->tmT2, pl->tmXd, pl->tmW3, pl->tmW1, pl->tmX, tmXo, p); }));
  YB_CHECK_LAUNCH();
  return YB_OK;
}

}  // namespace yb
