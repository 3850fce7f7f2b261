// VQ codebook lookup on the Hopper tensor cores (wgmma): exact fp32 argmin at HBM speed.
//
//   index[r] = argmin_k ( |z_r|^2 + |e_k|^2 - 2 z_r.e_k ),  first minimum wins   (M.py:60-65, P.py:158-164)
//
// 131 072 FLOP per 1 032-byte row is ~40x above the fp32-FMA ridge, so an exact SIMT kernel sits at a few per cent
// of HBM bandwidth (pm_vq.cu).  Here the 128 x 256 score matrix of a 128-row tile is one fp16 MMA chain per 64-row
// half (screen), and only the rows whose two best screened distances are closer than a RIGOROUS bound on the screen's
// error are re-scored in exact fp32 (same expression and tie rule as the SIMT kernel).  The emitted index is
// therefore the fp32 argmin for every row, while each row's 1 KB is read from HBM once.
//
// Persistent kernel, one CTA per SM, 384 threads:
//   warps 0-7   two consumer warpgroups - 16 x wgmma.m64n256k16 per tile (64 rows each) into 128 fp32 registers per
//                                         thread; screened distances d~ = e2[k] - 2 z.e (row scale folded into the FMA),
//                                         pass 1: minimum, pass 2: every k within tau of it; rows with more than one
//                                         candidate are re-scored in fp32 by the whole warp (8 lanes per candidate,
//                                         shuffle reduction)
//   warps 8-11  loaders - coalesced float4 loads of 8 full rows per warp and batch, per-row sum of squares by warp
//                         shuffle, power-of-two row scaling into the fp16 range, fp16 conversion into the 128B-swizzled
//                         K-major layout; they stage the next tile while the consumers run their epilogue
// The fp16 codebook (128 KB, scaled by a power of two) stays resident in shared memory for the CTA's lifetime.
//
// Screen error bound (DESIGN.md section 4): both operands are rounded to fp16 (relative 2^-11 each, values scaled
// by exact powers of two so neither overflow nor the subnormal range matters), products are exact, accumulation is
// fp32: |d~_k - d_k| <= 2 * 2^-10 * 1.01 * |z| |e_k| =: B.  If d_k* is the true minimum then d~_k* <= min d~ + 2B,
// so the candidate set {k : d~_k <= min d~ + 2B (+ fp32 slack)} always contains it.
#include "pm_common.cuh"
#include "pm_tc_ptx.cuh"
#include "../../include/pm_emage.h"

namespace {

constexpr int ED = 256;                 // e_dim
constexpr int NC = 256;                 // codes
constexpr int TM = 128;                 // rows per tile (two 64-row warpgroups)
constexpr int CONSUMER_WARPS = 8, LOAD_WARPS = 4;
constexpr int NTHREADS = 32 * (CONSUMER_WARPS + LOAD_WARPS);     // 384
constexpr int KB_A = TM * 128;          // bytes of one 64-channel k-block of the z tile (16 KB)
constexpr int KB_B = NC * 128;          // ... of the codebook (32 KB)
constexpr int MAXC = 8;                 // candidates kept per row (the screen's minimum included); more = "re-score every code"

// Instrumented build only (-DPM_VQ_TIMING, tools/vq_timeline.py): clock64 cycles CTA 0 spends per phase.
#ifdef PM_VQ_TIMING
__device__ unsigned long long pm_vq_stamps[16];
#define VQ_T(var) const long long var = clock64()
#define VQ_ADD(i, t0)                                                                                     \
  do {                                                                                                    \
    if (blockIdx.x == 0 && (threadIdx.x & 31) == 0) atomicAdd(&pm_vq_stamps[i], (unsigned long long)(clock64() - (t0))); \
  } while (0)
#define VQ_CNT(i, n)                                                                                      \
  do {                                                                                                    \
    if (blockIdx.x == 0 && (threadIdx.x & 31) == 0) atomicAdd(&pm_vq_stamps[i], (unsigned long long)(n)); \
  } while (0)
#else
#define VQ_T(var) do {} while (0)
#define VQ_ADD(i, t0) do {} while (0)
#define VQ_CNT(i, n) do {} while (0)
#endif

struct Smem {
  static constexpr int B = 0;                               // fp16 codebook, 4 k-blocks
  static constexpr int A = B + 4 * KB_B;                    // fp16 z tile, 4 k-blocks
  static constexpr int E2 = A + 4 * KB_A;                   // float[256]
  static constexpr int INFO = E2 + NC * 4;                  // float2[2 slots][TM]: (fma multiplier, tau)
  static constexpr int CAND = INFO + 2 * TM * 8;            // uint8[TM][MAXC]
  static constexpr int CNT = CAND + TM * MAXC;              // int[TM]: codes within tau per row
  static constexpr int BARS = CNT + TM * 4;                 // a_full, a_empty
  static constexpr int MISC = BARS + 2 * 8;                 // max |e_k|^2
  static constexpr int TOTAL = MISC + 16;
};

__device__ __forceinline__ uint32_t sw128(int row, int byte_in_row) {      // offset inside one k-block
  return (uint32_t)((row >> 3) * 1024 + (row & 7) * 128 + ((((byte_in_row >> 4) ^ (row & 7)) << 4) | (byte_in_row & 15)));
}
__device__ __forceinline__ void sts64(uint32_t addr, uint32_t a, uint32_t b) {
  asm volatile("st.shared.v2.b32 [%0], {%1, %2};" ::"r"(addr), "r"(a), "r"(b) : "memory");
}
__device__ __forceinline__ void sts8(uint32_t addr, uint32_t v) {
  asm volatile("st.shared.u8 [%0], %1;" ::"r"(addr), "r"(v) : "memory");
}
__device__ __forceinline__ uint32_t lds8(uint32_t addr) {
  uint32_t v;
  asm volatile("ld.shared.u8 %0, [%1];" : "=r"(v) : "r"(addr) : "memory");
  return v;
}
__device__ __forceinline__ float lds32f(uint32_t addr) {
  float v;
  asm volatile("ld.shared.f32 %0, [%1];" : "=f"(v) : "r"(addr) : "memory");
  return v;
}
__device__ __forceinline__ float2 lds64f(uint32_t addr) {
  float2 v;
  asm volatile("ld.shared.v2.f32 {%0, %1}, [%2];" : "=f"(v.x), "=f"(v.y) : "r"(addr) : "memory");
  return v;
}
__device__ __forceinline__ uint32_t pack_h2(float a, float b) {
  const __half2 h = __floats2half2_rn(a, b);
  return *reinterpret_cast<const uint32_t*>(&h);
}
// exact power of two 2^s as a float, s in [-126, 127]
__device__ __forceinline__ float pow2i(int s) { return __uint_as_float((uint32_t)(s + 127) << 23); }
// s such that m * 2^s lies in [2^13, 2^14) for a finite normal m > 0; 0 for zero / subnormal / non-finite m
__device__ __forceinline__ int scale_exp(float m) {
  const int ex = (int)(__float_as_uint(m) >> 23) & 0xFF;
  if (ex == 0 || ex == 255) return 0;
  int s = 140 - ex;
  return s < -100 ? -100 : (s > 100 ? 100 : s);
}

__global__ void __launch_bounds__(NTHREADS, 1) l2_argmin_tc_kernel(
    const float* __restrict__ z, long long rows, int rows_per_batch, long long z_bs, const float* __restrict__ codebook,
    const float* __restrict__ e2, long long* __restrict__ index) {
  // row g of the (batch, rows_per_batch, 256) view: z + (g / rows_per_batch) * z_bs + (g % rows_per_batch) * 256.
  // rows_per_batch == 0 marks one dense matrix (the host folds dense views into it): no division on the hot path,
  // and the strided case (a window's tail frames: a few hundred rows) divides in 32 bits.
  auto row_ptr = [&](long long g) -> const float* {
    if (rows_per_batch == 0) return z + g * ED;
    const unsigned gb = (unsigned)g / (unsigned)rows_per_batch, gl = (unsigned)g - gb * (unsigned)rows_per_batch;
    return z + (long long)gb * z_bs + (long long)gl * ED;
  };
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* sm = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  const uint32_t sm_u = smem_u32(sm);
  float* e2s = reinterpret_cast<float*>(sm + Smem::E2);
  const uint32_t e2s_u = sm_u + Smem::E2, info_u = sm_u + Smem::INFO, cands_u = sm_u + Smem::CAND;
  int* cnt = reinterpret_cast<int*>(sm + Smem::CNT);
  const uint32_t bars = sm_u + Smem::BARS;
  const uint32_t a_full = bars, a_empty = bars + 8;
  float* misc_f = reinterpret_cast<float*>(sm + Smem::MISC);       // [0] = max |e_k|^2

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const long long n_tiles = (rows + TM - 1) / TM;
  VQ_T(t_kernel);

  // ---- prologue: barriers, resident codebook ----
  if (tid == 0) {
    mbar_init(a_full, LOAD_WARPS);
    mbar_init(a_empty, 2);                           // one arrival per consumer warpgroup
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  if (warp == 0) {                       // max |e_k|^2 -> codebook scale and the error bound
    float m = 0.f;
    for (int k = lane; k < NC; k += 32) { const float v = __ldg(e2 + k); e2s[k] = v; m = fmaxf(m, v); }
    m = pm_warp_max(m);
    if (lane == 0) misc_f[0] = m;
  }
  __syncthreads();
  const float e2max = misc_f[0];
  const float emax = sqrtf(e2max);
  const int s_cb = scale_exp(emax);      // every |e_kd| <= emax, so the scaled codebook stays below 2^14
  {
    const float sc = pow2i(s_cb);
    for (int i = tid; i < NC * (ED / 4); i += NTHREADS) {
      const int k = i >> 6, c4 = i & 63;                              // code row, float4 index within it
      const float4 v = __ldg(reinterpret_cast<const float4*>(codebook) + i);
      const int kb = c4 >> 4, byte = (c4 & 15) * 8;
      sts64(sm_u + Smem::B + kb * KB_B + sw128(k, byte), pack_h2(v.x * sc, v.y * sc), pack_h2(v.z * sc, v.w * sc));
    }
  }
  fence_proxy_async_smem();
  __syncthreads();

  if (warp >= CONSUMER_WARPS) {
    // ===== loaders: warp lw stages tile rows 32 lw .. 32 lw + 31, eight rows per batch =====
    const int lw = warp - CONSUMER_WARPS;
    const float bound_c = 2.0f * 0.0009765625f * 1.02f * emax;        // B = bound_c * |z|  (2 * 2^-10 * 1.02 * |e|max)
    const float inv_cb = pow2i(-s_cb);
    //  - one row statistic only, sum of squares: the scale comes from |z| (>= every |z_d|), reduced by a halving
    //    butterfly (9 shuffles for 8 rows instead of 80) that leaves row j's total on lanes 4j..4j+3;
    //  - the owner lanes compute scale / multiplier / tau once, the scale is broadcast back with one shuffle per row;
    //  - the warp's 32 KB of the NEXT tile are pulled into L2 by one bulk prefetch a whole tile period ahead, so HBM
    //    stays busy during the convert phases and the demand loads hit L2.
    const bool dense = rows_per_batch == 0;
    auto batch_base = [&](long long tl, int q) { return z + (tl * TM + lw * 32 + q * 8) * ED; };
    int it = 0;
    for (long long tile = blockIdx.x; tile < n_tiles; tile += gridDim.x, ++it) {
      const long long r0 = tile * TM;
      const int slot = it & 1;
      const bool full = dense && r0 + TM <= rows;
      if (lane == 0) {
        const long long nt = tile + gridDim.x;
        if (dense && nt * TM + TM <= rows)
          asm volatile("cp.async.bulk.prefetch.L2.global [%0], %1;" ::"l"(batch_base(nt, 0)), "r"(32 * ED * 4) : "memory");
      }
#pragma unroll 1
      for (int q = 0; q < 4; ++q) {
        const int rb = lw * 32 + q * 8;
        VQ_T(t_ld);
        float4 v[8][2];
        if (full) {
          const float4* p = reinterpret_cast<const float4*>(batch_base(tile, q)) + lane;
#pragma unroll
          for (int j = 0; j < 8; ++j) {
            v[j][0] = ldg_stream4(p + j * (ED / 4));
            v[j][1] = ldg_stream4(p + j * (ED / 4) + 32);
          }
        } else {
#pragma unroll
          for (int j = 0; j < 8; ++j) {
            const long long g = r0 + rb + j;
            if (g < rows) {
              const float4* p = reinterpret_cast<const float4*>(row_ptr(g));
              v[j][0] = ldg_stream4(p + lane);
              v[j][1] = ldg_stream4(p + 32 + lane);
            } else {
              v[j][0] = v[j][1] = make_float4(0.f, 0.f, 0.f, 0.f);
            }
          }
        }
        float ss[8];
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          const float4 a = v[j][0], b = v[j][1];
          ss[j] = fmaf(a.x, a.x, fmaf(a.y, a.y, fmaf(a.z, a.z, fmaf(a.w, a.w, fmaf(b.x, b.x, fmaf(b.y, b.y, fmaf(b.z, b.z, b.w * b.w)))))));
        }
        // halving butterfly: after the xor-16 / 8 / 4 steps each lane holds ONE row's partial, then two full steps
        {
          const bool h16 = lane & 16, h8 = lane & 8, h4 = lane & 4;
#pragma unroll
          for (int i = 0; i < 4; ++i) {
            const float recv = __shfl_xor_sync(0xffffffffu, h16 ? ss[i] : ss[i + 4], 16);
            ss[i] = (h16 ? ss[i + 4] : ss[i]) + recv;
          }
#pragma unroll
          for (int i = 0; i < 2; ++i) {
            const float recv = __shfl_xor_sync(0xffffffffu, h8 ? ss[i] : ss[i + 2], 8);
            ss[i] = (h8 ? ss[i + 2] : ss[i]) + recv;
          }
          const float recv = __shfl_xor_sync(0xffffffffu, h4 ? ss[0] : ss[1], 4);
          ss[0] = (h4 ? ss[1] : ss[0]) + recv;
          ss[0] += __shfl_xor_sync(0xffffffffu, ss[0], 2);
          ss[0] += __shfl_xor_sync(0xffffffffu, ss[0], 1);
        }
        // this lane owns row (lane >> 2) & 7 of the batch: |z| < 2^(floor(e/2)+1) for |z|^2 = m 2^e, so scaling by
        // 2^(13 - floor(e/2)) keeps every element below 2^14 (no fp16 overflow whatever the data's scale)
        const float ss_own = ss[0];
        int s_own = 0;
        {
          const int ex = (int)(__float_as_uint(ss_own) >> 23) & 0xFF;
          if (ex != 0 && ex != 255) {
            s_own = 13 - ((ex - 127) >> 1);
            s_own = s_own < -100 ? -100 : (s_own > 100 ? 100 : s_own);
          }
        }
        const float sc_own = pow2i(s_own);
        if (lw == 0) VQ_ADD(0, t_ld);
        VQ_T(t_we);
        // the previous tile's MMAs must have read the A tile before it is overwritten
        if (q == 0) mbar_wait_relaxed<20>(a_empty, (uint32_t)(it & 1) ^ 1u);
        if (lw == 0) VQ_ADD(1, t_we);
        VQ_T(t_cv);
        if ((lane & 3) == 0) {
          // d~ = e2[k] + mult * acc ;  tau = 2 B + fp32 slack (covers the exact path's own rounding and flushes)
          const float mult = -2.0f * pow2i(-s_own) * inv_cb;
          const float tau = 2.0f * bound_c * sqrtf(ss_own) + 2.4e-7f * 16.f * (ss_own + e2max);
          sts64(info_u + (uint32_t)(slot * TM + rb + (lane >> 2)) * 8, __float_as_uint(mult), __float_as_uint(tau));
        }
        // lane holds channels 4*lane..+3 (k-block lane/16) and 128 + 4*lane..+3 (k-block 2 + lane/16)
        const uint32_t dst0 = sm_u + Smem::A + (lane >> 4) * KB_A + (uint32_t)((rb >> 3) * 1024);   // rb is a multiple of 8
#pragma unroll
        for (int j = 0; j < 8; ++j) {                      // row rb + j: 8-row group rb / 8, row j within it
          const float sc = __shfl_sync(0xffffffffu, sc_own, 4 * j);
          const uint32_t dst = dst0 + (uint32_t)(j * 128 + ((((lane & 15) >> 1) ^ j) << 4) + (lane & 1) * 8);
          sts64(dst, pack_h2(v[j][0].x * sc, v[j][0].y * sc), pack_h2(v[j][0].z * sc, v[j][0].w * sc));
          sts64(dst + 2 * KB_A, pack_h2(v[j][1].x * sc, v[j][1].y * sc), pack_h2(v[j][1].z * sc, v[j][1].w * sc));
        }
        if (lw == 0) VQ_ADD(2, t_cv);
      }
      fence_proxy_async_smem();
      __syncwarp();
      if (lane == 0) mbar_arrive(a_full);
    }
    return;
  }

  // ===== consumer warpgroup wg: screen of tile rows 64 wg .. 64 wg + 63 against all 256 codes, then the argmin =====
  const int wg = warp >> 2, t2 = 2 * (lane & 3);
  const int rloc = (warp & 3) * 16 + (lane >> 2);          // this thread's first row within the warpgroup (and + 8)
  const uint64_t b_desc = gmma_desc(GMMA_DESC_K_SW128, sm_u + Smem::B);
  const uint64_t a_desc = gmma_desc(GMMA_DESC_K_SW128, sm_u + Smem::A + wg * (64 * 128));
  int it = 0;
  for (long long tile = blockIdx.x; tile < n_tiles; tile += gridDim.x, ++it) {
    const int slot = it & 1;
    float acc[NC / 2];
#pragma unroll
    for (int i = 0; i < NC / 2; ++i) acc[i] = 0.f;
    VQ_T(t_m1);
    mbar_wait(a_full, (uint32_t)(it & 1));
    if (warp == 0) { VQ_ADD(4, t_m1); VQ_CNT(11, 1); }
    VQ_T(t_e1);
    wgmma_fence();
#pragma unroll
    for (int kb = 0; kb < 4; ++kb)
#pragma unroll
      for (int k = 0; k < 4; ++k)
        wgmma_m64n256k16<false>(acc, a_desc + (uint64_t)(kb * (KB_A >> 4) + k * 2), b_desc + (uint64_t)(kb * (KB_B >> 4) + k * 2));
    wgmma_commit();
    wgmma_wait<0>();
    wgmma_fence_regs(acc);
    float2 inf[2];
#pragma unroll
    for (int hr = 0; hr < 2; ++hr) inf[hr] = lds64f(info_u + (uint32_t)(slot * TM + wg * 64 + rloc + 8 * hr) * 8);
    // the A tile and this tile's row info have been read: the loaders may stage the next tile
    named_bar_sync(1 + wg, 128);
    if ((tid & 127) == 0) mbar_arrive(a_empty);

    // pass 1: minimum of the screened distances d~ = e2[k] + mult * acc (first index wins), per thread over its 64
    // columns in increasing order, then across the four lanes of the quad that share the row
    float m1[2] = {INFINITY, INFINITY};
    int k1[2] = {0, 0};
#pragma unroll
    for (int i = 0; i < NC / 8; ++i) {
      const float2 e = lds64f(e2s_u + (uint32_t)(8 * i + t2) * 4);
#pragma unroll
      for (int hr = 0; hr < 2; ++hr) {
        const float d0 = fmaf(inf[hr].x, acc[4 * i + 2 * hr], e.x), d1 = fmaf(inf[hr].x, acc[4 * i + 2 * hr + 1], e.y);
        if (d0 < m1[hr]) { m1[hr] = d0; k1[hr] = 8 * i + t2; }
        if (d1 < m1[hr]) { m1[hr] = d1; k1[hr] = 8 * i + t2 + 1; }
      }
    }
#pragma unroll
    for (int hr = 0; hr < 2; ++hr)
#pragma unroll
      for (int o = 1; o <= 2; o <<= 1) {
        const float om = __shfl_xor_sync(0xffffffffu, m1[hr], o);
        const int ok = __shfl_xor_sync(0xffffffffu, k1[hr], o);
        if (om < m1[hr] || (om == m1[hr] && ok < k1[hr])) { m1[hr] = om; k1[hr] = ok; }
      }
    if (warp == 0) VQ_ADD(7, t_e1);
    VQ_T(t_e2);
    // pass 2: every code within tau of the minimum (the minimum itself included), listed per row in shared memory
    const int row_w = (warp & 3) * 16 + (lane >> 2);         // row within this warp's 16 = lane >> 2 (+ 8)
    const int crow0 = wg * 64 + row_w;                       // candidate-list row of the first of this thread's rows
    if ((lane & 3) == 0) { cnt[crow0] = 0; cnt[crow0 + 8] = 0; }
    __syncwarp();
#pragma unroll
    for (int i = 0; i < NC / 8; ++i) {
      const float2 e = lds64f(e2s_u + (uint32_t)(8 * i + t2) * 4);
#pragma unroll
      for (int hr = 0; hr < 2; ++hr) {
        const float thr = m1[hr] + inf[hr].y;
#pragma unroll
        for (int u = 0; u < 2; ++u) {
          if (fmaf(inf[hr].x, acc[4 * i + 2 * hr + u], u ? e.y : e.x) <= thr) {
            const int n = atomicAdd(&cnt[crow0 + 8 * hr], 1);
            if (n < MAXC) sts8(cands_u + (uint32_t)((crow0 + 8 * hr) * MAXC + n), (uint32_t)(8 * i + t2 + u));
          }
        }
      }
    }
    __syncwarp();

    if (warp == 0) VQ_ADD(8, t_e2);
    VQ_T(t_e3);
    // ---- exact fp32 re-scoring of rows with more than one candidate: the whole warp per row, four candidates at a
    // time (8 lanes each: 32 elements per lane, xor-shuffle reduction - a fixed summation order) ----
    const long long gbase = tile * TM + wg * 64 + (warp & 3) * 16;     // global row of this warp's row 0
    // bit 4 r of the first ballot = row r of the warp, of the second = row r + 8: fold both into one 16-bit row mask
    unsigned rmask = 0;
    {
      const unsigned b0 = __ballot_sync(0xffffffffu, (lane & 3) == 0 && cnt[crow0] > 1 && gbase + (lane >> 2) < rows);
      const unsigned b1 = __ballot_sync(0xffffffffu, (lane & 3) == 0 && cnt[crow0 + 8] > 1 && gbase + (lane >> 2) + 8 < rows);
#pragma unroll
      for (int r = 0; r < 8; ++r) rmask |= (((b0 >> (4 * r)) & 1u) << r) | (((b1 >> (4 * r)) & 1u) << (r + 8));
    }
#ifdef PM_VQ_TIMING
    if (warp == 0) { VQ_CNT(12, __popc(rmask)); }
#endif
    const int grp = lane >> 3, gl = lane & 7;
    while (rmask) {
      const int r = __ffs(rmask) - 1;
      rmask &= rmask - 1;
      const int lrow = wg * 64 + (warp & 3) * 16 + r;          // candidate-list row
      const int nsrc = cnt[lrow];
      const bool all = nsrc > MAXC;                             // list overflowed: every code is a candidate
      const int ncand = all ? NC : nsrc;
      const float4* zr = reinterpret_cast<const float4*>(row_ptr(gbase + r));
      float4 zv[8];
#pragma unroll
      for (int i = 0; i < 8; ++i) zv[i] = __ldg(zr + gl + 8 * i);
      float z2 = 0.f;
#pragma unroll
      for (int i = 0; i < 8; ++i) z2 = fmaf(zv[i].x, zv[i].x, fmaf(zv[i].y, zv[i].y, fmaf(zv[i].z, zv[i].z, fmaf(zv[i].w, zv[i].w, z2))));
      z2 += __shfl_xor_sync(0xffffffffu, z2, 1);
      z2 += __shfl_xor_sync(0xffffffffu, z2, 2);
      z2 += __shfl_xor_sync(0xffffffffu, z2, 4);
      float best = INFINITY;
      int bk = NC;                                                     // NC = "nothing yet" (loses every tie)
      const uint32_t list = cands_u + (uint32_t)(lrow * MAXC);
#pragma unroll 1
      for (int base = 0; base < ncand; base += 4) {
        const int ci = base + grp;
        const bool valid = ci < ncand;
        const int c = all ? (ci & (NC - 1)) : (int)lds8(list + (valid ? ci : 0));
        const float4* er = reinterpret_cast<const float4*>(codebook + (long long)c * ED);
        float dot = 0.f;
#pragma unroll
        for (int i = 0; i < 8; ++i) {
          const float4 ev = __ldg(er + gl + 8 * i);
          dot = fmaf(zv[i].x, ev.x, fmaf(zv[i].y, ev.y, fmaf(zv[i].z, ev.z, fmaf(zv[i].w, ev.w, dot))));
        }
        dot += __shfl_xor_sync(0xffffffffu, dot, 1);
        dot += __shfl_xor_sync(0xffffffffu, dot, 2);
        dot += __shfl_xor_sync(0xffffffffu, dot, 4);
        float dd = __fsub_rn(__fadd_rn(z2, lds32f(e2s_u + (uint32_t)c * 4)), __fmul_rn(2.f, dot));   // the expression of M.py:64
        int cc = c;
        if (!valid) { dd = INFINITY; cc = NC; }
#pragma unroll
        for (int o = 8; o <= 16; o <<= 1) {                            // the other candidates of this round
          const float od = __shfl_xor_sync(0xffffffffu, dd, o);
          const int oc = __shfl_xor_sync(0xffffffffu, cc, o);
          if (od < dd || (od == dd && oc < cc)) { dd = od; cc = oc; }
        }
        if (dd < best || (dd == best && cc < bk)) { best = dd; bk = cc; }
      }
      // all-NaN rows keep the screen's answer (0, like torch.argmin)
      if (bk < NC && (lane >> 2) == (r & 7)) k1[r >> 3] = bk;
    }
    if ((lane & 3) == 0) {
#pragma unroll
      for (int hr = 0; hr < 2; ++hr) {
        const long long g = gbase + (lane >> 2) + 8 * hr;
        if (g < rows) index[g] = (long long)k1[hr];
      }
    }
    if (warp == 0) VQ_ADD(9, t_e3);
    __syncwarp();                     // candidate lists and counters are rewritten for the next tile
  }
  if (warp == 0) VQ_ADD(10, t_kernel);
}

constexpr size_t kSmem = Smem::TOTAL + 1024;

}  // namespace

extern "C" int pm_l2_argmin_tc(const float* z, long long rows, int rows_per_batch, long long z_bs,
                               const float* codebook, const float* e2,
                               int n_codes, int e_dim, long long* index, int max_ctas, void* stream) {
  PM_REQUIRE(z && codebook && e2 && index && rows >= 0);
  if (rows_per_batch <= 0 || z_bs == (long long)rows_per_batch * ED) { rows_per_batch = 0; z_bs = 0; }   // one dense (rows, 256) matrix
  PM_REQUIRE((z_bs & 3) == 0 && (rows_per_batch == 0 || rows < 0x7fffffffLL));
  if (e_dim != ED || n_codes != NC) return PM_EUNSUPPORTED;
  PM_REQUIRE((reinterpret_cast<uintptr_t>(z) & 15) == 0 && (reinterpret_cast<uintptr_t>(codebook) & 15) == 0);
  if (rows == 0) return PM_OK;
  int dev = 0, sms = 0;
  cudaError_t e = cudaGetDevice(&dev);
  if (e == cudaSuccess) e = cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
  if (e != cudaSuccess) return (int)e;
  static unsigned long long configured = 0;
  if (pm_first_use_on_device(configured)) {
    e = cudaFuncSetAttribute(l2_argmin_tc_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kSmem);
    if (e != cudaSuccess) { configured = 0; return (int)e; }
  }
  const long long tiles = (rows + TM - 1) / TM;
  long long grid = tiles < sms ? tiles : sms;
  if (max_ctas > 0 && grid > max_ctas) grid = max_ctas;
  l2_argmin_tc_kernel<<<(unsigned)grid, NTHREADS, kSmem, (cudaStream_t)stream>>>(z, rows, rows_per_batch, z_bs, codebook, e2, index);
  PM_LAUNCH_CHECK();
}

#ifdef PM_VQ_TIMING
extern "C" int pm_vq_timing_reset() {
  cudaError_t e = cudaDeviceSynchronize();
  if (e != cudaSuccess) return (int)e;
  void* d = nullptr;
  e = cudaGetSymbolAddress(&d, pm_vq_stamps);
  if (e != cudaSuccess) return (int)e;
  return (int)cudaMemset(d, 0, sizeof(unsigned long long) * 16);
}
extern "C" int pm_vq_timing_read(unsigned long long* host) {
  cudaError_t e = cudaDeviceSynchronize();
  if (e != cudaSuccess) return (int)e;
  return (int)cudaMemcpyFromSymbol(host, pm_vq_stamps, sizeof(unsigned long long) * 16);
}
#endif
