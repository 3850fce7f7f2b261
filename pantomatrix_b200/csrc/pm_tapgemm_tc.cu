// Hopper tap-GEMM: Conv1d (stride 1, any taps / zero padding) and Linear on the sm_90a tensor cores (wgmma).
//
//   out[b,l,n] = act( bias[n] + sum_t sum_c A[b, l+t-pad, c] * W[t,n,c] + residual[b,l,n] )
//
// Operands are split-bf16 planes (x ~ p0 + p1 + p2, each plane bf16): nsplit 1 = plain bf16, 2 = bf16x3
// (p0*p0 + p0*p1 + p1*p0), 3 = bf16x6 (every product down to 2^-24): all products accumulate in fp32 registers, so
// the result has fp32-grade accuracy at tensor-core rates.
//
// Structure (one 128 x BN output tile per CTA, BN = 64 or 128 chosen per launch on the host, 384 threads):
//   warpgroup 0      producer, 40 registers per thread (setmaxnreg.dec) -
//                      warp 0: TMA (one elected lane): A box (64 ch x R rows x NB clips) per plane, with the tap shift
//                              folded into the row coordinate (im2col-free; padding rows are TMA zero fill), W box
//                              (64 ch x BN rows) per plane; 128B-swizzled K-major smem tiles; mbarrier ring.
//                              After the last k-block: the tile's fp32 residual (BN ch x R rows x NB clips) into
//                              ring slots the remaining MMAs no longer read
//                      warp 1: L2 prefetch of the next GEMM's weights; warp 2: the tile's bias into smem; warp 3
//                              exits at once
//   warpgroups 1-2   consumers, 232 registers per thread (setmaxnreg.inc) - consumer warpgroup g issues
//                      wgmma.m64nBNk16 for tile rows 64 g .. 64 g + 63 out of the shared operand stage into three
//                      BN / 2-register accumulators, then runs the epilogue: bias / residual (both from smem) /
//                      activation on its own fragment values in registers -> fp32 and/or split-plane tiles in smem
//                      in the TMA boxes' swizzled layout -> TMA stores by one thread.  Output views TMA cannot
//                      describe take the per-element store loop: registers -> staging tile -> global
// Contract and reference call sites: include/pm_emage.h (pm_tapgemm_tc).
#include <cuda.h>
#include <stdio.h>
#include <stdlib.h>

#include <cstring>
#include <type_traits>
#include "pm_common.cuh"
#include "../../include/pm_emage.h"


namespace {

constexpr int BM = 128;             // tile rows (two 64-row warpgroups)
constexpr int BK = 64;              // bf16 channels per k-block = one 128-byte swizzle row
constexpr int MMA_K = 16;
constexpr int A_TILE_BYTES = BM * BK * 2;           // 16 KB per plane
constexpr int PRODUCER_THREADS = 128;
constexpr int CONSUMER_THREADS = 256;
constexpr int NUM_THREADS = PRODUCER_THREADS + CONSUMER_THREADS;   // producer warpgroup + two consumer warpgroups
// The CTA is launched with 168 registers per thread (the most 384 threads get: 65536 / 384 rounded down to 8).  The
// producer hands 128 of every thread's registers back, and the consumers take them: three m64n128 accumulators are
// 192 registers per thread.  setmaxnreg.inc waits until the pool holds what it asks for, so the split must add up.
constexpr int PRODUCER_REGS = 40, CONSUMER_REGS = 232;
static_assert(PRODUCER_THREADS * PRODUCER_REGS + CONSUMER_THREADS * CONSUMER_REGS == (65536 / NUM_THREADS & ~7) * NUM_THREADS,
              "the setmaxnreg split must use exactly the launch's register pool");
constexpr int STAMP_WARP = PRODUCER_THREADS / 32;   // first consumer warp: writes the PM_TC_TIMING stamps
constexpr int MAX_STAGES = 8;
constexpr int RING_KB = 200;        // operand ring per CTA (one CTA per SM; 227 KB is the sm_90 limit)

struct TcParams {
  int taps, pad, nsplit, kblocks;   // kblocks = ceil(cin / 64)
  int rows_out, cout, batch;
  int R, NB;                        // tile = NB clips x R rows (R * NB == 128)
  int w_rows;                       // rows per tap in the packed weight tensor (>= cout, multiple of BN)
  const float* bias;
  const float* residual; long long r_bs; int ldr;
  int res_tma;                      // residual tile loaded by TMA (map_r) into the ring; else read per element
  int tma_out;                      // outputs written by TMA stores (map_o / map_p) from swizzled smem tiles; else
                                    // the per-element store loop
  int act, act_cols; float slope;
  float* out_f32; long long o_bs; int ldo;
  __nv_bfloat16* out_bf16; long long ob_ps, ob_bs; int ldob; int out_nsplit;
  int stages;
  int res_slot0, rot;               // residual tile's first physical ring slot; ring slot rotation (see the kernel)
  const uint8_t* prefetch; long long prefetch_bytes;   // next GEMM's weights: pulled into L2 while this one runs
  float acc_scale;   // fp16 operands: weights are packed scaled by a power of two, undone here (1 for bf16)
};

// Instrumented build only (-DPM_TC_TIMING, tools/gemm_timeline.py): per-CTA clock64 stamps of the kernel's phases.
#ifdef PM_TC_TIMING
__device__ unsigned long long pm_tc_stamps[4096 * 8];
#define PM_STAMP(i)                                                                                              \
  do {                                                                                                           \
    if ((threadIdx.x & 31) == 0) {                                                                               \
      const unsigned cta_ = (blockIdx.z * gridDim.y + blockIdx.y) * gridDim.x + blockIdx.x;                      \
      if (cta_ < 4096) pm_tc_stamps[cta_ * 8 + (i)] = (unsigned long long)clock64();                             \
    }                                                                                                            \
  } while (0)
#else
#define PM_STAMP(i) do {} while (0)
#endif

#include "pm_tc_ptx.cuh"   // PTX wrappers: mbarrier, TMA, wgmma

template <int BN, bool F16>
__device__ __forceinline__ void mma_k16(float (&d)[BN / 2], uint64_t a, uint64_t b) {
  static_assert(BN == 64 || BN == 128, "64- or 128-column tiles (see pm_tapgemm_tc)");
  if constexpr (BN == 64) wgmma_m64n64k16<!F16>(d, a, b);
  else wgmma_m64n128k16<!F16>(d, a, b);
}

// Three fp32 accumulators: two "main" ones that take the p0*p0 products of alternate k-iterations and one
// "correction" accumulator for every cross product.  The tensor core aligns and truncates addends to the
// accumulator's exponent, a biased error ~2^-25 |acc| per instruction; keeping the 2^-8-scaled cross terms apart and
// halving the chain length of the main sums keeps the result at fp32-FMA quality.  The epilogue adds the three.
template <int BN, bool F16, int NSPLIT>
__device__ __forceinline__ void mma_kblock(float (&main)[BN / 2], float (&corr)[BN / 2], uint64_t a0, uint64_t w0) {
  constexpr uint64_t A_PL = A_TILE_BYTES >> 4, W_PL = (BN * BK * 2) >> 4, K_ST = (MMA_K * 2) >> 4;   // descriptor units
  // cross products first (small -> large), into the correction accumulator
  if constexpr (NSPLIT == 3) {
#pragma unroll
    for (int k = 0; k < BK / MMA_K; ++k) mma_k16<BN, F16>(corr, a0 + k * K_ST, w0 + 2 * W_PL + k * K_ST);
#pragma unroll
    for (int k = 0; k < BK / MMA_K; ++k) mma_k16<BN, F16>(corr, a0 + A_PL + k * K_ST, w0 + W_PL + k * K_ST);
#pragma unroll
    for (int k = 0; k < BK / MMA_K; ++k) mma_k16<BN, F16>(corr, a0 + 2 * A_PL + k * K_ST, w0 + k * K_ST);
  }
  if constexpr (NSPLIT >= 2) {
#pragma unroll
    for (int k = 0; k < BK / MMA_K; ++k) mma_k16<BN, F16>(corr, a0 + k * K_ST, w0 + W_PL + k * K_ST);
#pragma unroll
    for (int k = 0; k < BK / MMA_K; ++k) mma_k16<BN, F16>(corr, a0 + A_PL + k * K_ST, w0 + k * K_ST);
  }
#pragma unroll
  for (int k = 0; k < BK / MMA_K; ++k) mma_k16<BN, F16>(main, a0 + k * K_ST, w0 + k * K_ST);
}

template <int BN, bool F16, int NSPLIT>
__global__ void __launch_bounds__(NUM_THREADS, 1) tapgemm_tc_kernel(const __grid_constant__ CUtensorMap map_a,
                                                                  const __grid_constant__ CUtensorMap map_w,
                                                                  const __grid_constant__ CUtensorMap map_r,
                                                                  const __grid_constant__ CUtensorMap map_o,
                                                                  const __grid_constant__ CUtensorMap map_p,
                                                                  const TcParams p) {
  constexpr int W_TILE_BYTES = BN * BK * 2;
  constexpr int NACC = BN / 2;                      // accumulator registers per thread (m64 x BN over 128 threads)
  constexpr int ST = BN + 8;                        // epilogue staging row stride (floats)
  constexpr int RES_BYTES = BM * BN * 4;            // fp32 residual tile, [NB clips][R rows][BN ch]

  extern __shared__ __align__(1024) uint8_t smem_raw[];
  // carve: [stages][nsplit A tiles][nsplit W tiles] (1024-aligned), then barriers, then the tile's BN bias values.
  // The epilogue reuses the ring: the staging tile at its start, the residual tile in its last RES_BYTES (launch()
  // checks that they do not overlap).
  // 1024-aligned by pointer arithmetic on smem_raw itself: a pointer that went through an integer is generic to the
  // compiler, and every epilogue access through it would be a generic ld / st instead of lds / sts
  uint8_t* tiles = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
  const int stage_bytes = p.nsplit * (A_TILE_BYTES + W_TILE_BYTES);
  const int ring_bytes = p.stages * stage_bytes > BM * ST * 4 ? p.stages * stage_bytes : BM * ST * 4;
  uint64_t* bars = reinterpret_cast<uint64_t*>(tiles + ring_bytes);
  uint64_t* full_bar = bars;                       // [MAX_STAGES]
  uint64_t* empty_bar = bars + MAX_STAGES;         // [MAX_STAGES]
  uint64_t* epi_bar = bars + 2 * MAX_STAGES;       // bias (and residual tile) in smem
  float* bias_s = reinterpret_cast<float*>(bars + 2 * MAX_STAGES + 2);

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (warp == STAMP_WARP) PM_STAMP(0);                          // kernel entry
  const int l0 = blockIdx.x * p.R;
  const int n0 = blockIdx.y * BN;
  const int b0 = blockIdx.z * p.NB;
  const int n_iter = p.taps * p.kblocks;
  // Ring slot s (barrier index) lives at physical slot (s + p.rot) % stages.  The residual tile takes the physical
  // slots p.res_slot0 .. stages - 1; the rotation puts the last k-block just below them, so they hold the oldest
  // k-blocks in flight and are handed back, and refilled with the residual, while the last k-blocks still compute.

  if (threadIdx.x == 0) {
    asm volatile("prefetch.tensormap [%0];" ::"l"(&map_a) : "memory");
    asm volatile("prefetch.tensormap [%0];" ::"l"(&map_w) : "memory");
    if (p.res_tma) asm volatile("prefetch.tensormap [%0];" ::"l"(&map_r) : "memory");
    if (p.tma_out && p.out_f32) asm volatile("prefetch.tensormap [%0];" ::"l"(&map_o) : "memory");
    if (p.tma_out && p.out_nsplit) asm volatile("prefetch.tensormap [%0];" ::"l"(&map_p) : "memory");
    for (int s = 0; s < p.stages; ++s) {
      mbar_init(smem_u32(&full_bar[s]), 1);
      mbar_init(smem_u32(&empty_bar[s]), 2);       // one arrival per consumer warpgroup
    }
    mbar_init(smem_u32(epi_bar), p.res_tma ? 2 : 1);   // warp 2's bias arrival (+ warp 0's residual transaction)
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();
  if (warp == STAMP_WARP) PM_STAMP(1);                          // prologue done (barriers, descriptors)

  if (warp < PRODUCER_THREADS / 32) {
    // ===== producer warpgroup =====
    setmaxnreg_dec<PRODUCER_REGS>();
    if (warp == 1 && lane == 0 && p.prefetch) {
      // Weights are read once per window and the per-window set (0.6-0.8 GB) does not fit the 50 MB L2, so every
      // GEMM would stream its W tiles from HBM at DRAM latency.  Each CTA instead prefetches its share of the NEXT
      // GEMM's weights into L2 (cp.async.bulk.prefetch.L2) while this one computes.
      const long long ncta = (long long)gridDim.x * gridDim.y * gridDim.z;
      const long long cta = ((long long)blockIdx.z * gridDim.y + blockIdx.y) * gridDim.x + blockIdx.x;
      long long share = ((p.prefetch_bytes + ncta - 1) / ncta + 127) & ~127LL;
      long long off = cta * share;
      long long end = off + share < p.prefetch_bytes ? off + share : p.prefetch_bytes;
      end &= ~15LL;
      for (; off < end; off += 16384) {
        const uint32_t n = (uint32_t)(end - off < 16384 ? end - off : 16384);
        asm volatile("cp.async.bulk.prefetch.L2.global [%0], %1;" ::"l"(p.prefetch + off), "r"(n) : "memory");
      }
    }
    if (warp == 2) {
      for (int c = lane; c < BN; c += 32) bias_s[c] = p.bias && n0 + c < p.cout ? __ldg(p.bias + n0 + c) : 0.f;
      __syncwarp();
      if (lane == 0) mbar_arrive(smem_u32(epi_bar));
    }
    if (warp != 0) return;
    // ----- warp 0: TMA -----
    const uint32_t tx = (uint32_t)stage_bytes;
    int s = 0, q = p.rot, tap = 0, kb = 0;
    uint32_t ph = 0;
    for (int it = 0; it < n_iter; ++it) {
      mbar_wait_fast(smem_u32(&empty_bar[s]), ph ^ 1u);       // whole warp waits (uniform control flow)
      if (elect_one()) {
        const uint32_t bar = smem_u32(&full_bar[s]);
        uint8_t* st = tiles + (size_t)q * stage_bytes;
        mbar_expect_tx(bar, tx);
        for (int pl = 0; pl < p.nsplit; ++pl) {
          tma_load_4d(smem_u32(st + pl * A_TILE_BYTES), &map_a, bar, kb * BK, l0 + tap - p.pad, b0, pl);
          tma_load_3d(smem_u32(st + p.nsplit * A_TILE_BYTES + pl * W_TILE_BYTES), &map_w, bar, kb * BK, tap * p.w_rows + n0, pl);
        }
      }
      __syncwarp();
      if (++s == p.stages) { s = 0; ph ^= 1u; }
      if (++q == p.stages) q = 0;
      if (++kb == p.kblocks) { kb = 0; ++tap; }
    }
    if (p.res_tma) {
      // the next stages - res_slot0 ring slots are the residual's physical slots: once their k-blocks are consumed
      // (or were never filled), load the residual tile over them
      for (int j = p.res_slot0; j < p.stages; ++j) {
        mbar_wait_fast(smem_u32(&empty_bar[s]), ph ^ 1u);
        if (++s == p.stages) { s = 0; ph ^= 1u; }
      }
      if (elect_one()) {
        // the store loop reads one [NB][R][BN] box; the TMA-store epilogue reads BN / 32 128B-swizzled
        // [NB][R][32] boxes (the layout of its output tile, conflict-free for the accumulator fragments)
        const uint32_t bar = smem_u32(epi_bar);
        mbar_expect_tx(bar, (uint32_t)RES_BYTES);
        const int nbox = p.tma_out ? BN / 32 : 1;
        for (int j = 0; j < nbox; ++j)
          tma_load_3d(smem_u32(tiles + ring_bytes - RES_BYTES + j * (RES_BYTES / nbox)), &map_r, bar, n0 + j * (BN / nbox), l0, b0);
      }
      __syncwarp();
    }
    return;                                        // the consumers' named barriers below do not count this warpgroup
  }

  // ===== consumer warpgroups =====
  setmaxnreg_inc<CONSUMER_REGS>();
  const int ct = threadIdx.x - PRODUCER_THREADS;    // consumer thread 0 .. 255
  const int wg = ct >> 7;                           // 0 / 1: tile rows 64 wg .. 64 wg + 63
  float acc0[NACC], acc1[NACC], accc[NACC];
#pragma unroll
  for (int i = 0; i < NACC; ++i) { acc0[i] = 0.f; acc1[i] = 0.f; accc[i] = 0.f; }
  {
    const uint32_t tiles_u32 = smem_u32(tiles);
    int s = 0, q = p.rot;
    uint32_t ph = 0;
    int prev = -1;                                  // stage whose MMAs are still in flight
    // one k-block: the even ones accumulate into acc0, the odd ones into acc1 (unrolled by two, so that every wgmma
    // names its accumulator statically)
    auto kblock = [&](float (&main)[NACC]) {
      mbar_wait_fast(smem_u32(&full_bar[s]), ph);
      if (prev < 0 && warp == STAMP_WARP) PM_STAMP(2);            // first operand stage landed
      const uint32_t a_base = tiles_u32 + (uint32_t)q * (uint32_t)stage_bytes + (uint32_t)wg * (64 * 128);
      const uint32_t w_base = tiles_u32 + (uint32_t)q * (uint32_t)stage_bytes + (uint32_t)(NSPLIT * A_TILE_BYTES);
      wgmma_fence();
      mma_kblock<BN, F16, NSPLIT>(main, accc, gmma_desc(GMMA_DESC_K_SW128, a_base), gmma_desc(GMMA_DESC_K_SW128, w_base));
      wgmma_commit();
      // at most one k-block in flight: the previous one has finished reading its stage, hand it back to the producer
      wgmma_wait<1>();
      if (prev >= 0 && ct % 128 == 0) mbar_arrive(smem_u32(&empty_bar[prev]));
      prev = s;
      if (++s == p.stages) { s = 0; ph ^= 1u; }
      if (++q == p.stages) q = 0;
    };
    int it = 0;
    for (; it + 1 < n_iter; it += 2) {
      kblock(acc0);
      kblock(acc1);
    }
    if (it < n_iter) kblock(acc0);
    if (warp == STAMP_WARP) PM_STAMP(3);                       // all MMAs issued
    wgmma_wait<0>();
    if (warp == STAMP_WARP) PM_STAMP(4);                       // accumulators complete
    wgmma_fence_regs(acc0);
    wgmma_fence_regs(acc1);
    wgmma_fence_regs(accc);
  }
  // every MMA of both warpgroups has read its operands: the ring becomes the epilogue's output / staging tile
  named_bar_sync(1, CONSUMER_THREADS);
  if (p.tma_out) {
    // ===== epilogue, TMA stores: each thread finishes its own fragment values in registers, writes them once into
    // the output tiles in the TMA boxes' 128B-swizzled layout, and one thread stores the tiles.  TMA clips at the
    // maps' bounds (ragged rows_out / cout / batch, clip tiles with R < 128).  Smem (ring start): fp32 tile
    // [BN / 32][BM][32 floats], then out_nsplit plane tiles [BN / 64][BM][64 halves]; the residual tile is
    // [BN / 32][BM][32 floats] in the ring's last RES_BYTES.  A 128B swizzle puts 16-byte chunk k of 128-byte row r
    // at chunk k ^ (r % 8), so the 8 rows of a fragment access hit 8 different chunks.  With both outputs the fp32
    // tile goes out first: the TMA engine reads it while the consumers split the planes.
    const int wq = warp & 3, t4 = lane & 3, sw = lane >> 2;       // sw = r % 8 for both rows of the thread
    const int r0 = wg * 64 + wq * 16 + sw;
    const float act_slope = p.act == PM_ACT_NONE ? 1.f : (p.act == PM_ACT_RELU ? 0.f : p.slope);
    const float* res_s = reinterpret_cast<const float*>(tiles + ring_bytes - RES_BYTES);
    // float offset of (row r, column c) in a [BN / 32][BM][32] swizzled tile; c = 8 i + 2 t4 (even)
    auto off32 = [&](int r, int i) { return (i >> 2) * (BM * 32) + r * 32 + (((2 * (i & 3) + (t4 >> 1)) ^ sw) << 2) + 2 * (t4 & 1); };
    mbar_wait_fast(smem_u32(epi_bar), 0);                        // bias (and residual tile) landed
    // (acc0 + acc1) + accc, x acc_scale, + bias, + residual, activation: the store loop's order, into acc0
#pragma unroll
    for (int i = 0; i < NACC / 4; ++i) {
      const int c = 8 * i + 2 * t4, n = n0 + c;
      const float2 bc = *reinterpret_cast<const float2*>(bias_s + c);   // both rows' columns
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int j = 4 * i + 2 * h;
        float v0 = acc0[j] + acc1[j], v1 = acc0[j + 1] + acc1[j + 1];
        v0 += accc[j];
        v1 += accc[j + 1];
        if constexpr (F16) { v0 = __fmul_rn(v0, p.acc_scale); v1 = __fmul_rn(v1, p.acc_scale); }   // not fused with + bias
        if (p.bias) { v0 += bc.x; v1 += bc.y; }
        if (p.residual) {
          const float2 t = *reinterpret_cast<const float2*>(res_s + off32(r0 + 8 * h, i));
          v0 += t.x; v1 += t.y;
        }
        // compare-select, NaN kept (see the store loop)
        acc0[j] = v0 < 0.f ? (n < p.act_cols ? act_slope : 1.f) * v0 : v0;
        acc0[j + 1] = v1 < 0.f ? (n + 1 < p.act_cols ? act_slope : 1.f) * v1 : v1;
      }
    }
    float* of_s = reinterpret_cast<float*>(tiles);
    uint8_t* pl_s = tiles + (p.out_f32 ? BM * BN * 4 : 0);
    constexpr int PLANE_BYTES = BM * BN * 2;
    if (p.out_f32) {
#pragma unroll
      for (int i = 0; i < NACC / 4; ++i)
#pragma unroll
        for (int h = 0; h < 2; ++h)
          *reinterpret_cast<float2*>(of_s + off32(r0 + 8 * h, i)) = make_float2(acc0[4 * i + 2 * h], acc0[4 * i + 2 * h + 1]);
      fence_proxy_async_smem();                                  // the tile's generic writes -> the TMA engine
      named_bar_sync(1, CONSUMER_THREADS);
      if (ct == 0) {
        for (int j = 0; j < BN / 32 && n0 + 32 * j < p.cout; ++j)
          tma_store_3d(&map_o, smem_u32(of_s + j * (BM * 32)), n0 + 32 * j, l0, b0);
        bulk_commit();
      }
    }
    // the plane count as a constant where it is the operand split (every engine call), else read at run time
    auto planes = [&](auto ons) {
      constexpr int ONS = decltype(ons)::value;
#pragma unroll
      for (int i = 0; i < NACC / 4; ++i)
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          uint32_t w[3];
          pm_split_pair_t<F16, ONS>(acc0[4 * i + 2 * h], acc0[4 * i + 2 * h + 1], p.out_nsplit, w);
          // byte offset of (row r, column c) in a [BN / 64][BM][64 halves] swizzled plane tile
          const int o = (i >> 3) * (BM * 128) + (r0 + 8 * h) * 128 + (((i & 7) ^ sw) << 4) + 4 * t4;
#pragma unroll
          for (int pl = 0; pl < 3; ++pl)
            if (pl < (ONS ? ONS : p.out_nsplit)) *reinterpret_cast<uint32_t*>(pl_s + pl * PLANE_BYTES + o) = w[pl];
        }
    };
    if (p.out_nsplit) {
      if (p.out_nsplit == NSPLIT) planes(std::integral_constant<int, NSPLIT>{});
      else planes(std::integral_constant<int, 0>{});
      fence_proxy_async_smem();
      named_bar_sync(1, CONSUMER_THREADS);
      if (ct == 0) {
        for (int pl = 0; pl < p.out_nsplit; ++pl)
          for (int j = 0; j < BN / 64 && n0 + 64 * j < p.cout; ++j)
            tma_store_4d(&map_p, smem_u32(pl_s + pl * PLANE_BYTES + j * (BM * 128)), n0 + 64 * j, l0, b0, pl);
        bulk_commit();
      }
    }
    if (warp == STAMP_WARP) PM_STAMP(5);                      // the stores issued
    if (ct == 0) bulk_wait_read0();                            // the tiles must stay until the TMA engine has read them
    if (warp == STAMP_WARP) PM_STAMP(6);                       // their shared-memory reads complete
    return;
  }
  {
    const int wq = warp & 3, t4 = lane & 3;
    const int r0 = wg * 64 + wq * 16 + (lane >> 2);
    float* stg = reinterpret_cast<float*>(tiles);
#pragma unroll
    for (int i = 0; i < NACC / 4; ++i) {
      const int c = 8 * i + 2 * t4;
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        float v0 = acc0[4 * i + 2 * h] + acc1[4 * i + 2 * h];
        float v1 = acc0[4 * i + 2 * h + 1] + acc1[4 * i + 2 * h + 1];
        v0 += accc[4 * i + 2 * h];
        v1 += accc[4 * i + 2 * h + 1];
        if constexpr (F16) { v0 *= p.acc_scale; v1 *= p.acc_scale; }       // undo the weight pre-scale (exact)
        *reinterpret_cast<float2*>(stg + (r0 + 8 * h) * ST + c) = make_float2(v0, v1);
      }
    }
  }
  named_bar_sync(1, CONSUMER_THREADS);

  // ===== epilogue: one float4 of one row per thread and round; consecutive threads cover a row (coalesced) =====
  const bool vec_f = p.out_f32 && ((p.ldo & 3) == 0) && ((reinterpret_cast<uintptr_t>(p.out_f32) & 15) == 0) && ((p.o_bs & 3) == 0);
  const bool vec_b = p.out_bf16 && ((p.ldob & 3) == 0) && ((reinterpret_cast<uintptr_t>(p.out_bf16) & 7) == 0) &&
                     ((p.ob_bs & 3) == 0) && ((p.ob_ps & 3) == 0);
  // the vector path reads the residual from the TMA-loaded tile; a residual TMA cannot describe is read per element
  const bool all_vec = (!p.out_f32 || vec_f) && (!p.residual || p.res_tma) && (!p.out_bf16 || vec_b);
  const float act_slope = p.act == PM_ACT_NONE ? 1.f : (p.act == PM_ACT_RELU ? 0.f : p.slope);
  const int r_shift = 31 - __clz(p.R);                           // R is a power of two
  constexpr int C4 = BN / 4;                                     // float4 columns per row
  const float* stg = reinterpret_cast<const float*>(tiles);
  const float* res_s = reinterpret_cast<const float*>(tiles + ring_bytes - RES_BYTES);
  mbar_wait_fast(smem_u32(epi_bar), 0);                          // bias (and residual tile) landed
  // Kept rolled: unrolled (all shared-memory reads first, then the stores) the EMAGE step ran at 294 k instead of
  // 325 k frames/s (bench.py, H100 80GB HBM3 at 700 W): the larger kernel costs more than the overlap gains.
#pragma unroll 1
  for (int item = ct; item < BM * C4; item += CONSUMER_THREADS) {
    const int rt = item / C4, c = (item % C4) * 4;
    const int b = b0 + (rt >> r_shift), l = l0 + (rt & (p.R - 1));
    const int n = n0 + c;
    if (b >= p.batch || l >= p.rows_out || n >= p.cout) continue;
    const float4 x4 = *reinterpret_cast<const float4*>(stg + rt * ST + c);
    // identity == leaky with slope 1: one branch-free (select) formula for none / relu / leaky / partial activation.
    // Compare-select, not fmaxf / fminf: those return the non-NaN operand and would turn the NaN an fp16 operand
    // overflow leaves into 0, hiding it from the host's overflow guard.
    const long long of = (long long)b * p.o_bs + (long long)l * p.ldo;
    const long long orr = (long long)b * p.r_bs + (long long)l * p.ldr;
    const PmPlanes P{p.out_bf16 ? p.out_bf16 + (long long)b * p.ob_bs + (long long)l * p.ldob : nullptr,
                     p.ob_ps, p.ldob, p.out_nsplit};
    if (all_vec && n + 4 <= p.cout) {
      float4 x = x4;
      if (p.bias) {
        const float4 t = *reinterpret_cast<const float4*>(bias_s + c);
        x.x += t.x; x.y += t.y; x.z += t.z; x.w += t.w;
      }
      if (p.residual) {
        const float4 t = *reinterpret_cast<const float4*>(res_s + rt * BN + c);
        x.x += t.x; x.y += t.y; x.z += t.z; x.w += t.w;
      }
      x.x = x.x < 0.f ? (n < p.act_cols ? act_slope : 1.f) * x.x : x.x;
      x.y = x.y < 0.f ? (n + 1 < p.act_cols ? act_slope : 1.f) * x.y : x.y;
      x.z = x.z < 0.f ? (n + 2 < p.act_cols ? act_slope : 1.f) * x.z : x.z;
      x.w = x.w < 0.f ? (n + 3 < p.act_cols ? act_slope : 1.f) * x.w : x.w;
      if (p.out_f32) *reinterpret_cast<float4*>(p.out_f32 + of + n) = x;
      if (P.ptr) pm_store_planes4_t<F16>(P, 0, n, x);
    } else {
      // ragged / unaligned tail: per element
      const float xs[4] = {x4.x, x4.y, x4.z, x4.w};
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        if (n + k >= p.cout) break;
        float y = xs[k];
        if (p.bias) y += bias_s[c + k];
        if (p.residual) y += p.residual[orr + n + k];
        y = y < 0.f ? (n + k < p.act_cols ? act_slope : 1.f) * y : y;
        if (p.out_f32) p.out_f32[of + n + k] = y;
        if (P.ptr) pm_store_planes_t<F16>(P, 0, n + k, y);
      }
    }
  }
  if (warp == STAMP_WARP) PM_STAMP(5);                         // this warp's share of the epilogue issued
#ifdef PM_TC_TIMING
  named_bar_sync(1, CONSUMER_THREADS);
#endif
  if (warp == STAMP_WARP) PM_STAMP(6);                         // all consumer warps done
}

// ---------------------------------------------------------------------------------------------------
// fp32 -> bf16 planes.  One CTA row-block per (clip, row tile): no per-element index arithmetic, 16-byte loads,
// 8-byte stores.  VEC path needs ch % 4 == 0 and 16-byte aligned rows.
template <bool VEC, bool F16>
__global__ void __launch_bounds__(256) split_bf16_kernel(const float* __restrict__ x, long long x_bs, int ldx, int rows,
                                                         int ch, __nv_bfloat16* __restrict__ out, long long o_ps,
                                                         long long o_bs, int ldo, int nsplit) {
  const int b = blockIdx.y;
  const float* __restrict__ xb = x + (long long)b * x_bs;
  __nv_bfloat16* __restrict__ ob = out + (long long)b * o_bs;
  if (VEC) {
    const int ch4 = ch >> 2;
    const long long total = (long long)rows * ch4;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
      const int r = (int)(i / ch4), c4 = (int)(i - (long long)r * ch4);
      const float4 v = *reinterpret_cast<const float4*>(xb + (long long)r * ldx + 4 * c4);
      const PmPlanes P{ob, o_ps, ldo, nsplit};
      pm_store_planes4_t<F16>(P, r, 4 * c4, v);
    }
  } else {
    const long long total = (long long)rows * ch;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
      const int r = (int)(i / ch), c = (int)(i - (long long)r * ch);
      const PmPlanes P{ob, o_ps, ldo, nsplit};
      pm_store_planes_t<F16>(P, r, c, xb[(long long)r * ldx + c]);
    }
  }
}

// ---------------------------------------------------------------------------------------------------
// The operand ring of an instance: as many stages of nsplit A and W tiles as fit RING_KB, at most MAX_STAGES.
constexpr int stage_bytes_of(int bn, int nsplit) { return nsplit * (A_TILE_BYTES + bn * BK * 2); }
constexpr int stages_of(int bn, int nsplit) {
  return RING_KB * 1024 / stage_bytes_of(bn, nsplit) < MAX_STAGES ? RING_KB * 1024 / stage_bytes_of(bn, nsplit) : MAX_STAGES;
}
constexpr int ring_bytes_of(int bn, int nsplit) { return stages_of(bn, nsplit) * stage_bytes_of(bn, nsplit); }
// Whether the TMA-store epilogue's tiles fit the ring: fp32 tile and out_nsplit plane tiles from its start, the
// residual tile at its end.
constexpr bool tma_out_fits(int bn, int nsplit, bool f32, int out_nsplit, bool residual) {
  return (f32 ? BM * bn * 4 : 0) + out_nsplit * BM * bn * 2 + (residual ? BM * bn * 4 : 0) <= ring_bytes_of(bn, nsplit);
}

template <int BN, bool F16, int NSPLIT>
int launch(const CUtensorMap& ma, const CUtensorMap& mw, const CUtensorMap& mr, const CUtensorMap& mo,
           const CUtensorMap& mp, TcParams& p, dim3 grid, cudaStream_t st) {
  constexpr int stage_bytes = stage_bytes_of(BN, NSPLIT);
  constexpr int stages = stages_of(BN, NSPLIT);
  static_assert(stages >= 2, "the operand ring needs two stages");
  // The store loop's staging tile (ring start) and residual tile (ring end) must not overlap, and the residual must
  // leave the slot below it to the last k-block.
  constexpr int staging = BM * (BN + 8) * 4, res_bytes = BM * BN * 4;
  static_assert(staging + res_bytes <= stages * stage_bytes && res_bytes <= (stages - 1) * stage_bytes,
                "staging and residual tiles must fit the ring side by side");
  // The TMA-store epilogue fits with the fp32 tile, two plane tiles and the residual (the fp16x3 engine's widest
  // call); three planes beside fp32 and a residual at BN = 128 take the store loop (pm_tapgemm_tc checks).
  static_assert(tma_out_fits(BN, NSPLIT, true, 2, true), "fp32, two plane and residual tiles must fit the ring");
  static_assert(BN * 4 * BM % 1024 == 0 && stage_bytes % 1024 == 0, "128B-swizzled TMA boxes need 1024-byte alignment");
  p.stages = stages;
  p.res_slot0 = (stages * stage_bytes - res_bytes) / stage_bytes;
  p.rot = (p.res_slot0 - 1 - (p.taps * p.kblocks - 1) % stages + stages) % stages;
  const size_t smem = (size_t)stages * stage_bytes + 1024 /*align slack*/ + (2 * MAX_STAGES + 2) * sizeof(uint64_t) + BN * sizeof(float);
  static unsigned long long configured = 0;       // per template instantiation, one bit per device
  if (pm_first_use_on_device(configured)) {
    cudaError_t e = cudaFuncSetAttribute(tapgemm_tc_kernel<BN, F16, NSPLIT>, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024);
    if (e != cudaSuccess) { configured = 0; return (int)e; }
  }
  tapgemm_tc_kernel<BN, F16, NSPLIT><<<grid, NUM_THREADS, smem, st>>>(ma, mw, mr, mo, mp, p);
  PM_LAUNCH_CHECK();
}

template <int BN>
int launch_fmt(const CUtensorMap* m, TcParams& p, dim3 grid, cudaStream_t st, bool f16) {
  if (f16) {
    if (p.nsplit == 1) return launch<BN, true, 1>(m[0], m[1], m[2], m[3], m[4], p, grid, st);
    if (p.nsplit == 2) return launch<BN, true, 2>(m[0], m[1], m[2], m[3], m[4], p, grid, st);
    return launch<BN, true, 3>(m[0], m[1], m[2], m[3], m[4], p, grid, st);
  }
  if (p.nsplit == 1) return launch<BN, false, 1>(m[0], m[1], m[2], m[3], m[4], p, grid, st);
  if (p.nsplit == 2) return launch<BN, false, 2>(m[0], m[1], m[2], m[3], m[4], p, grid, st);
  return launch<BN, false, 3>(m[0], m[1], m[2], m[3], m[4], p, grid, st);
}

// N tile of a launch: a pure function of the shape and the SM count, so a captured graph keeps its choice.
// One CTA per SM, so a launch runs in waves of `sms` tiles.  A 128-column tile halves the shared-memory operand reads
// per MAC and the per-tile fixed cost (barrier setup, pipeline fill, epilogue) per FLOP; it is chosen when the
// 64-column grid needs at least 1.4x as many waves.  So it is not chosen where both grids fit one wave (the 32-clip
// k = 3 convs of the motion encoder and the seed decode: 64 vs 32 CTAs, 10.5 vs 18.3 us at 128) and is everywhere
// else on the EMAGE step.  Alone, a 128-column tile costs about 1.7 64-column ones; in the step, the forked face /
// body / part branches fill partly used waves, and 1.4 measured best.  bench.py on one H100 80GB HBM3 at a 700 W
// power limit, fp16x3: ratio 1.0 (always 128) 299-300 k frames/s, 1.4 306 k, 1.7 293-294 k, 2.0 292 k, 64 only 283 k.
// tools/bench_gemm.py (fp16x3, fp32 out, us at BN = 64 / 128): 2048 x 768 <- 768 23.0 / 18.7; 2048 x 2304 <- 768
// 58.1 / 56.3; 2048 x 1536 <- 768 37.0 / 37.3; 2048 x 768 <- 1536 36.8 / 29.0; 8192 x 1536 <- 768 148.9 / 122.6;
// 32 x 300 conv k3 256 -> 256 36.5 / 36.1; 128 x 205 conv k15 128 -> 128 95.4 / 69.7.
int pick_bn(long long row_tiles, int cout, int w_rows, int sms) {
  if (cout <= 64 || w_rows % 128) return 64;
  const long long waves64 = (row_tiles * pm_cdiv(cout, 64) + sms - 1) / sms;
  const long long waves128 = (row_tiles * pm_cdiv(cout, 128) + sms - 1) / sms;
  return waves128 * 14 <= waves64 * 10 ? 128 : 64;
}

}  // namespace

extern "C" int pm_tapgemm_tc(const uint16_t* A, long long a_ps, long long a_bs, int lda, int batch, int rows_in, int cin,
                             const uint16_t* W, long long w_ps, int w_rows, int ldw, int taps, int pad, int nsplit,
                             const float* bias, int rows_out, int cout,
                             const float* residual, long long r_bs, int ldr,
                             int act, int act_cols, float slope, float acc_scale,
                             float* out_f32, long long o_bs, int ldo,
                             uint16_t* out_bf16, long long ob_ps, long long ob_bs, int ldob, int out_nsplit,
                             const void* prefetch, long long prefetch_bytes, void* stream) {
  PM_REQUIRE(A && W && (out_f32 || out_bf16));
  const int tile = (nsplit >> PM_TC_TILE_SHIFT) & 0xff;   // N tile override: 0 automatic, 1 = 64, 2 = 128 columns
  const bool store_loop = (nsplit & PM_TC_STORE_LOOP) != 0;   // force the per-element store loop (tests, A/B runs)
  PM_TAKE_FMT(nsplit, f16);                 // operand planes: bf16 (default) or fp16
  PM_TAKE_FMT(out_nsplit, out_f16);
  PM_REQUIRE(!out_bf16 || out_f16 == f16);  // emitted planes use the operand format
  PM_REQUIRE(f16 || acc_scale == 1.0f);
  PM_REQUIRE(!prefetch || (prefetch_bytes >= 0 && (reinterpret_cast<uintptr_t>(prefetch) & 15) == 0));
  PM_REQUIRE(batch > 0 && rows_in > 0 && rows_out > 0 && cin > 0 && cout > 0 && taps > 0);
  PM_REQUIRE(nsplit >= 1 && nsplit <= 3 && (!out_bf16 || (out_nsplit >= 1 && out_nsplit <= 3)));
  PM_REQUIRE(act >= PM_ACT_NONE && act <= PM_ACT_LEAKY);
  // TMA: 16-byte aligned base and strides
  PM_REQUIRE((reinterpret_cast<uintptr_t>(A) & 15) == 0 && (reinterpret_cast<uintptr_t>(W) & 15) == 0);
  PM_REQUIRE((lda & 7) == 0 && (ldw & 7) == 0 && lda >= cin && ldw >= cin && w_rows >= cout);
  PM_REQUIRE(batch == 1 || (a_bs & 7) == 0);
  PM_REQUIRE(nsplit == 1 || ((a_ps & 7) == 0 && (w_ps & 7) == 0));
  PM_REQUIRE(!out_f32 || ldo >= cout);
  PM_REQUIRE(!out_bf16 || ldob >= cout);
  PM_REQUIRE(!residual || ldr >= cout);

  int R = 128;
  if (rows_out <= 64 && batch > 1) { R = 16; while (R < rows_out) R <<= 1; }
  const int NB = 128 / R;
  PM_REQUIRE(tile <= 2 && w_rows % 64 == 0 && (tile != 2 || w_rows % 128 == 0));
  int BNsel = tile == 1 ? 64 : 128;
  if (tile == 0) {
    int dev = 0, sms = 0;
    cudaError_t e = cudaGetDevice(&dev);
    if (e == cudaSuccess) e = cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
    if (e != cudaSuccess) return (int)e;
    BNsel = pick_bn((long long)pm_cdiv(rows_out, R) * pm_cdiv(batch, NB), cout, w_rows, sms);
  }

  TcParams p;
  p.taps = taps; p.pad = pad; p.nsplit = nsplit; p.kblocks = (cin + BK - 1) / BK;
  p.rows_out = rows_out; p.cout = cout; p.batch = batch; p.R = R; p.NB = NB; p.w_rows = w_rows;
  p.bias = bias; p.residual = residual; p.r_bs = r_bs; p.ldr = ldr;
  p.act = act; p.act_cols = act_cols <= 0 ? cout : act_cols; p.slope = slope;
  p.out_f32 = out_f32; p.o_bs = o_bs; p.ldo = ldo;
  p.out_bf16 = reinterpret_cast<__nv_bfloat16*>(out_bf16); p.ob_ps = ob_ps; p.ob_bs = ob_bs; p.ldob = ldob;
  p.out_nsplit = out_bf16 ? out_nsplit : 0;
  p.stages = 0;
  p.prefetch = static_cast<const uint8_t*>(prefetch);
  p.prefetch_bytes = prefetch ? prefetch_bytes : 0;
  p.acc_scale = acc_scale;
  CUtensorMap m[5];   // A, W, residual, fp32 output, output planes
  std::memset(m, 0, sizeof(m));
  CUtensorMap &ma = m[0], &mw = m[1], &mr = m[2], &mo = m[3], &mp = m[4];
  {
    const long long bs_el = batch > 1 ? a_bs : (long long)rows_in * lda;
    const long long ps_el = nsplit > 1 ? a_ps : bs_el * batch;
    cuuint64_t dims[4] = {(cuuint64_t)cin, (cuuint64_t)rows_in, (cuuint64_t)batch, (cuuint64_t)nsplit};
    cuuint64_t strides[3] = {(cuuint64_t)lda * 2, (cuuint64_t)bs_el * 2, (cuuint64_t)ps_el * 2};
    cuuint32_t box[4] = {(cuuint32_t)BK, (cuuint32_t)R, (cuuint32_t)NB, 1};
    if (!encode_map(&ma, A, 4, dims, strides, box, f16)) return PM_EBADARG;
  }
  {
    const long long ps_el = nsplit > 1 ? w_ps : (long long)taps * w_rows * ldw;
    cuuint64_t dims[3] = {(cuuint64_t)cin, (cuuint64_t)taps * w_rows, (cuuint64_t)nsplit};
    cuuint64_t strides[2] = {(cuuint64_t)ldw * 2, (cuuint64_t)ps_el * 2};
    cuuint32_t box[3] = {(cuuint32_t)BK, (cuuint32_t)BNsel, 1};
    if (!encode_map(&mw, W, 3, dims, strides, box, f16)) return PM_EBADARG;
  }
  // The residual tile by TMA where it can describe the view (16-byte base and strides); the box is the output tile,
  // zero-filled past cout / rows_out / batch.  Any other view (or one the driver declines to encode) is read per
  // element in the store loop.
  const bool res_ok = residual && (reinterpret_cast<uintptr_t>(residual) & 15) == 0 && (ldr & 3) == 0 && (batch == 1 || (r_bs & 3) == 0);
  // The outputs by TMA stores where TMA can describe every output view (16-byte base and strides), the residual (if
  // any) is TMA-loaded and the tiles fit the ring.  Boxes of 32 fp32 / 64 plane elements (one 128-byte swizzle row)
  // x R rows x NB clips, clipped at cout / rows_out / batch; views at an offset (a window's rows, a column slice) are
  // just another base.  Every other case, or a view the driver declines to encode, keeps the per-element store loop.
  bool tma_out = !store_loop && (!residual || res_ok) && tma_out_fits(BNsel, nsplit, out_f32, p.out_nsplit, residual);
  if (tma_out && out_f32) {
    tma_out = (reinterpret_cast<uintptr_t>(out_f32) & 15) == 0 && (ldo & 3) == 0 && (batch == 1 || (o_bs & 3) == 0);
    const long long bs_el = batch > 1 ? o_bs : (long long)rows_out * ldo;
    cuuint64_t dims[3] = {(cuuint64_t)cout, (cuuint64_t)rows_out, (cuuint64_t)batch};
    cuuint64_t strides[2] = {(cuuint64_t)ldo * 4, (cuuint64_t)bs_el * 4};
    cuuint32_t box[3] = {32, (cuuint32_t)R, (cuuint32_t)NB};
    tma_out = tma_out && encode_tiled(&mo, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, CU_TENSOR_MAP_SWIZZLE_128B, out_f32, 3, dims, strides, box);
  }
  if (tma_out && out_bf16) {
    tma_out = (reinterpret_cast<uintptr_t>(out_bf16) & 15) == 0 && (ldob & 7) == 0 && (batch == 1 || (ob_bs & 7) == 0) &&
              (out_nsplit == 1 || (ob_ps & 7) == 0);
    const long long bs_el = batch > 1 ? ob_bs : (long long)rows_out * ldob;
    const long long ps_el = out_nsplit > 1 ? ob_ps : bs_el * batch;
    cuuint64_t dims[4] = {(cuuint64_t)cout, (cuuint64_t)rows_out, (cuuint64_t)batch, (cuuint64_t)out_nsplit};
    cuuint64_t strides[3] = {(cuuint64_t)ldob * 2, (cuuint64_t)bs_el * 2, (cuuint64_t)ps_el * 2};
    cuuint32_t box[4] = {64, (cuuint32_t)R, (cuuint32_t)NB, 1};
    tma_out = tma_out && encode_map(&mp, out_bf16, 4, dims, strides, box, f16);
  }
  // the TMA-store epilogue reads the residual in its output tile's layout: BN / 32 swizzled 32-column boxes
  p.res_tma = false;
  for (int swz = tma_out; res_ok && !p.res_tma && swz >= 0; --swz) {
    const long long bs_el = batch > 1 ? r_bs : (long long)rows_out * ldr;
    cuuint64_t dims[3] = {(cuuint64_t)cout, (cuuint64_t)rows_out, (cuuint64_t)batch};
    cuuint64_t strides[2] = {(cuuint64_t)ldr * 4, (cuuint64_t)bs_el * 4};
    cuuint32_t box[3] = {swz ? 32u : (cuuint32_t)BNsel, (cuuint32_t)R, (cuuint32_t)NB};
    p.res_tma = encode_tiled(&mr, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, swz ? CU_TENSOR_MAP_SWIZZLE_128B : CU_TENSOR_MAP_SWIZZLE_NONE,
                             residual, 3, dims, strides, box);
    if (!p.res_tma) tma_out = false;
  }
  p.tma_out = tma_out;
  dim3 grid(pm_cdiv(rows_out, R), pm_cdiv(cout, BNsel), pm_cdiv(batch, NB));
  PM_REQUIRE(grid.z <= 65535 && grid.y <= 65535);
  const cudaStream_t st = (cudaStream_t)stream;
  if (BNsel == 128) return launch_fmt<128>(m, p, grid, st, f16);
  return launch_fmt<64>(m, p, grid, st, f16);
}

#ifdef PM_TC_TIMING
extern "C" int pm_tc_timing_reset() {
  cudaError_t e = cudaDeviceSynchronize();
  if (e != cudaSuccess) return (int)e;
  void* d = nullptr;
  e = cudaGetSymbolAddress(&d, pm_tc_stamps);
  if (e != cudaSuccess) return (int)e;
  return (int)cudaMemset(d, 0, sizeof(unsigned long long) * 4096 * 8);
}
extern "C" int pm_tc_timing_read(unsigned long long* host) {
  cudaError_t e = cudaDeviceSynchronize();
  if (e != cudaSuccess) return (int)e;
  return (int)cudaMemcpyFromSymbol(host, pm_tc_stamps, sizeof(unsigned long long) * 4096 * 8);
}
#endif

extern "C" int pm_split_bf16(const float* x, long long x_bs, int ldx, int batch, int rows, int ch,
                             uint16_t* out, long long o_ps, long long o_bs, int ldo, int nsplit, void* stream) {
  PM_TAKE_FMT(nsplit, f16);
  PM_REQUIRE(x && out && batch >= 0 && rows >= 0 && ch > 0 && ldx >= ch && ldo >= ch && nsplit >= 1 && nsplit <= 3);
  if ((long long)batch * rows == 0) return PM_OK;
  PM_REQUIRE(batch <= 65535);
  const bool vec = (ch & 3) == 0 && (ldx & 3) == 0 && (x_bs & 3) == 0 && (ldo & 3) == 0 && (o_bs & 3) == 0 &&
                   (o_ps & 3) == 0 && (reinterpret_cast<uintptr_t>(x) & 15) == 0 && (reinterpret_cast<uintptr_t>(out) & 7) == 0;
  const long long work = (long long)rows * (vec ? ch / 4 : ch);
  long long gx = (work + 255) / 256;
  const long long cap = batch >= 132 * 4 ? 1 : (132 * 8 + batch - 1) / batch;
  if (gx > cap) gx = cap;
  dim3 grid((unsigned)gx, batch);
  __nv_bfloat16* o = reinterpret_cast<__nv_bfloat16*>(out);
  cudaStream_t st = (cudaStream_t)stream;
  if (f16) {
    if (vec) split_bf16_kernel<true, true><<<grid, 256, 0, st>>>(x, x_bs, ldx, rows, ch, o, o_ps, o_bs, ldo, nsplit);
    else split_bf16_kernel<false, true><<<grid, 256, 0, st>>>(x, x_bs, ldx, rows, ch, o, o_ps, o_bs, ldo, nsplit);
  } else {
    if (vec) split_bf16_kernel<true, false><<<grid, 256, 0, st>>>(x, x_bs, ldx, rows, ch, o, o_ps, o_bs, ldo, nsplit);
    else split_bf16_kernel<false, false><<<grid, 256, 0, st>>>(x, x_bs, ldx, rows, ch, o, o_ps, o_bs, ldo, nsplit);
  }
  PM_LAUNCH_CHECK();
}
