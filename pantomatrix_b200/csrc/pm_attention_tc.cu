// Multi-head attention core on the Hopper tensor cores (wgmma; T <= 64 tokens, head_dim 192, no masks): the whole
// 64 x 64 score tile of one (clip, head) is one warpgroup's register accumulator, softmax runs in registers, P goes
// back through shared memory as the A operand of the P.V product.  Contract: include/pm_emage.h (pm_attention_tc); replaces
// scaled_dot_product_attention inside nn.MultiheadAttention of every transformer layer (M.py:238-250).
//
// Operands are the two-plane fp16 activations of the fp16x3 engine (x = (p0 + p1) / 64, pm_common.cuh), written
// by the producing GEMM's epilogue, so Q, K, V arrive by TMA straight from the packed q|k|v projection output:
//   S  = Q K^T            3 products (p0 p0 + p0 p1 + p1 p0), wgmma m64n64k16, A and B K-major (dims contiguous)
//   P  = exp(S/sqrt(hd) - rowmax)   fp32 in registers (quad of threads = query row), split into two fp16 planes of 1024 P
//   O  = P V              3 products, wgmma m64n192k16, B = V as stored (keys x dims): MN-major descriptor
//   out = O / (rowsum * 64 * 1024)  -> fp32 and / or fp16 planes for the out-projection GEMM
// Accuracy is that of the GEMM engine (2^-22 relative per product), so the fp32 parity gates hold.
//
// One CTA per (clip, head), one warpgroup (128 threads): one elected thread issues the TMA loads, the warpgroup issues
// the MMAs, and each thread owns two query rows of the accumulators for softmax and epilogue.
#include "pm_common.cuh"
#include "pm_tc_ptx.cuh"
#include "../../include/pm_emage.h"

namespace {

constexpr int T = 64;                   // tokens per tile (queries and keys)
constexpr int HD = 192;                 // head dim
constexpr int KB = HD / 64;             // 64-column blocks per head
constexpr int BLK = T * 128;            // bytes of one 64 x 64 fp16 block (128-byte rows, 128B swizzle): 8 KB
constexpr int NTHREADS = 128;
constexpr float P_SCALE = 1024.f;       // probabilities are split as fp16 planes of 1024 * p (second plane stays normal)

struct Smem {
  static constexpr int Q = 0;                          // [2 planes][KB blocks]
  static constexpr int K = Q + 2 * KB * BLK;
  static constexpr int V = K + 2 * KB * BLK;
  static constexpr int P = V + 2 * KB * BLK;           // [2 planes] one block each
  static constexpr int BARS = P + 2 * BLK;             // qk_full[KB], v_full
  static constexpr int TOTAL = BARS + (KB + 1) * 8;
};

// Instrumented build only (-DPM_ATTN_TIMING, tools/bench_attention.py --timeline): clock64 stamps of CTA 0's phases.
#ifdef PM_ATTN_TIMING
__device__ unsigned long long pm_attn_stamps[16];
#define AT_STAMP(i) do { if (blockIdx.x == 0 && (threadIdx.x & 31) == 0) pm_attn_stamps[i] = (unsigned long long)clock64(); } while (0)
#else
#define AT_STAMP(i) do {} while (0)
#endif

struct AttnParams {
  int heads, tq, tk;
  int qc0, kc0, vc0;                    // first column of head 0 inside the Q / K / V plane tensors
  float scale;                          // 1 / (sqrt(hd) * 64 * 64): the operand planes hold 64 x
  float* out; int ldo;                  // fp32 (batch*tq, >= heads*hd) or null
  PmPlanes planes;                      // fp16 planes of the output or ptr == null
};

__global__ void __launch_bounds__(NTHREADS, 1) attention_tc_kernel(const __grid_constant__ CUtensorMap map_q,
                                                                   const __grid_constant__ CUtensorMap map_k,
                                                                   const __grid_constant__ CUtensorMap map_v,
                                                                   const AttnParams p) {
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* sm = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  const uint32_t sm_u = smem_u32(sm);
  const uint32_t bars = sm_u + Smem::BARS;
  const uint32_t qk_full = bars, v_full = bars + 8 * KB;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int b = blockIdx.x / p.heads, h = blockIdx.x % p.heads;
  if (warp == 0) AT_STAMP(0);                              // kernel entry

  if (threadIdx.x == 0) {
    for (int kb = 0; kb < KB; ++kb) mbar_init(qk_full + 8 * kb, 1);
    mbar_init(v_full, 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();
  if (warp == 0) AT_STAMP(1);                              // prologue done
  if (warp == 0) {
    // ===== TMA: one barrier per 64-column block, so the first MMAs start on a third of Q, K =====
    if (elect_one()) {
      asm volatile("prefetch.tensormap [%0];" ::"l"(&map_q) : "memory");
      asm volatile("prefetch.tensormap [%0];" ::"l"(&map_k) : "memory");
      asm volatile("prefetch.tensormap [%0];" ::"l"(&map_v) : "memory");
      for (int kb = 0; kb < KB; ++kb) {
        mbar_expect_tx(qk_full + 8 * kb, 4 * BLK);
        for (int pl = 0; pl < 2; ++pl) {
          tma_load_4d(sm_u + Smem::Q + (pl * KB + kb) * BLK, &map_q, qk_full + 8 * kb, p.qc0 + h * HD + kb * 64, 0, b, pl);
          tma_load_4d(sm_u + Smem::K + (pl * KB + kb) * BLK, &map_k, qk_full + 8 * kb, p.kc0 + h * HD + kb * 64, 0, b, pl);
        }
      }
      mbar_expect_tx(v_full, 2 * KB * BLK);
      for (int pl = 0; pl < 2; ++pl)
        for (int nb = 0; nb < KB; ++nb)
          tma_load_4d(sm_u + Smem::V + (pl * KB + nb) * BLK, &map_v, v_full, p.vc0 + h * HD + nb * 64, 0, b, pl);
    }
    __syncwarp();
  }

  // Fragment of this thread (pm_tc_ptx.cuh): query rows r0 = 16 warp + lane / 4 and r0 + 8; columns 8 i + 2 (lane % 4).
  const int r0 = warp * 16 + (lane >> 2), t2 = 2 * (lane & 3);
  // per block: cross products first (small), the main product last: (A plane, B plane) = (0,1), (1,0), (0,0)
  const int pa[3] = {0, 1, 0}, pb[3] = {1, 0, 0};

  // ---- S = Q K^T : A = Q, B = K, both K-major (dims contiguous), M = N = 64
  float sr[32];
#pragma unroll
  for (int i = 0; i < 32; ++i) sr[i] = 0.f;
#pragma unroll
  for (int kb = 0; kb < KB; ++kb) {
    mbar_wait(qk_full + 8 * kb, 0);
    if (warp == 0) AT_STAMP(8 + kb);                       // Q | K block kb landed
    wgmma_fence();
#pragma unroll
    for (int t = 0; t < 3; ++t)
#pragma unroll
      for (int k = 0; k < 4; ++k)
        wgmma_m64n64k16<false>(sr, gmma_desc(GMMA_DESC_K_SW128, sm_u + Smem::Q + (pa[t] * KB + kb) * BLK + 32 * k),
                               gmma_desc(GMMA_DESC_K_SW128, sm_u + Smem::K + (pb[t] * KB + kb) * BLK + 32 * k));
    wgmma_commit();
  }
  wgmma_wait<0>();
  wgmma_fence_regs(sr);
  if (warp == 0) AT_STAMP(2);                              // S complete

  // ---- softmax in registers.  exp(s - m) = 2^((s - m) log2 e): log2 e is folded into the scale and the exponential
  // is one MUFU.EX2 (2 ulp).  A row is spread over the four lanes of a quad: max and sum are reduced by two shuffles.
  float inv[2];
  {
    const float sl2 = p.scale * 1.4426950408889634f;
#pragma unroll
    for (int hr = 0; hr < 2; ++hr) {
      float m = -INFINITY;
#pragma unroll
      for (int i = 0; i < 8; ++i)
#pragma unroll
        for (int u = 0; u < 2; ++u) {
          const int j = 8 * i + t2 + u;
          const float v = j < p.tk ? sr[4 * i + 2 * hr + u] * sl2 : -INFINITY;
          sr[4 * i + 2 * hr + u] = v;
          m = fmaxf(m, v);
        }
      m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, 1));
      m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, 2));
      float sum = 0.f;
#pragma unroll
      for (int i = 0; i < 8; ++i)
#pragma unroll
        for (int u = 0; u < 2; ++u) {
          const int j = 8 * i + t2 + u;
          float e = 0.f;
          if (j < p.tk) asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(e) : "f"(sr[4 * i + 2 * hr + u] - m));
          sum += e;
          sr[4 * i + 2 * hr + u] = e * P_SCALE;
        }
      sum += __shfl_xor_sync(0xffffffffu, sum, 1);
      sum += __shfl_xor_sync(0xffffffffu, sum, 2);
      inv[hr] = 1.f / (sum * (P_SCALE * PM_F16_ACT_SCALE));
    }
    // P as two fp16 planes, K-major 128B-swizzled (query row = 128-byte row of 64 keys): the A operand of P V
#pragma unroll
    for (int hr = 0; hr < 2; ++hr) {
      const int row = r0 + 8 * hr;
      const uint32_t dst = sm_u + Smem::P + (row >> 3) * 1024 + (row & 7) * 128;
#pragma unroll
      for (int i = 0; i < 8; ++i) {        // keys 8 i + t2, + 1: one 4-byte pair inside 16-byte chunk i
        const float a0 = sr[4 * i + 2 * hr], a1 = sr[4 * i + 2 * hr + 1];
        const float f0 = pm_f16_head(a0), f1 = pm_f16_head(a1);       // exact in fp16: no conversion back (pm_common.cuh)
        const __half2 h0 = __floats2half2_rn(f0, f1);
        const __half2 h1 = __floats2half2_rn(a0 - f0, a1 - f1);
        const uint32_t off = (uint32_t)(((i ^ (row & 7)) << 4) + 2 * t2);
        asm volatile("st.shared.b32 [%0], %1;" ::"r"(dst + off), "r"(*reinterpret_cast<const uint32_t*>(&h0)) : "memory");
        asm volatile("st.shared.b32 [%0], %1;" ::"r"(dst + BLK + off), "r"(*reinterpret_cast<const uint32_t*>(&h1)) : "memory");
      }
    }
    fence_proxy_async_smem();
    __syncthreads();
    if (warp == 0) AT_STAMP(3);                            // softmax done, P stored
  }

  // ---- O = P V : B = V as stored, (keys x dims) = MN-major: 64-dim blocks 8 KB apart (LBO), 8-key groups 1 KB (SBO)
  float orr[96];
#pragma unroll
  for (int i = 0; i < 96; ++i) orr[i] = 0.f;
  mbar_wait(v_full, 0);
  wgmma_fence();
  {
    constexpr uint64_t DESC_MN = gmma_desc_mn_sw128(BLK);
#pragma unroll
    for (int t = 0; t < 3; ++t)
#pragma unroll
      for (int k = 0; k < 4; ++k)        // 16 keys per step: A advances 32 B inside the swizzled row, B by two 8-key groups
        wgmma_m64n192k16<false, 1>(orr, gmma_desc(GMMA_DESC_K_SW128, sm_u + Smem::P + pa[t] * BLK + 32 * k),
                                   gmma_desc(DESC_MN, sm_u + Smem::V + pb[t] * KB * BLK + 2048 * k));
  }
  wgmma_commit();
  wgmma_wait<0>();
  wgmma_fence_regs(orr);
  if (warp == 0) AT_STAMP(4);                              // O complete

  // ---- normalise and write straight from registers: 2 consecutive columns per store
  const bool pair_ok = p.planes.ptr && ((p.planes.ld & 1) == 0) && ((p.planes.ps & 1) == 0) &&
                       ((reinterpret_cast<uintptr_t>(p.planes.ptr) & 3) == 0);
#pragma unroll
  for (int hr = 0; hr < 2; ++hr) {
    const int row = r0 + 8 * hr;
    if (row >= p.tq) continue;
    const long long grow = (long long)b * p.tq + row;
    __half* const prow = reinterpret_cast<__half*>(p.planes.ptr) + grow * p.planes.ld + h * HD;
    float* const frow = p.out ? p.out + grow * p.ldo + h * HD : nullptr;
#pragma unroll
    for (int i = 0; i < HD / 8; ++i) {
      const int c = 8 * i + t2;
      const float x0 = orr[4 * i + 2 * hr] * inv[hr], x1 = orr[4 * i + 2 * hr + 1] * inv[hr];
      if (frow) *reinterpret_cast<float2*>(frow + c) = make_float2(x0, x1);
      if (p.planes.ptr) {
        if (pair_ok) {
          const float a0 = x0 * PM_F16_ACT_SCALE, a1 = x1 * PM_F16_ACT_SCALE;
          const float f0 = pm_f16_head(a0), f1 = pm_f16_head(a1);
          *reinterpret_cast<__half2*>(prow + c) = __floats2half2_rn(f0, f1);
          if (p.planes.nsplit > 1) *reinterpret_cast<__half2*>(prow + p.planes.ps + c) = __floats2half2_rn(a0 - f0, a1 - f1);
        } else {
          pm_store_planes_t<true>(p.planes, grow, h * HD + c, x0);
          pm_store_planes_t<true>(p.planes, grow, h * HD + c + 1, x1);
        }
      }
    }
  }
  if (warp == 0) AT_STAMP(5);                              // outputs written
#ifdef PM_ATTN_TIMING
  __syncthreads();
#endif
  if (warp == 0) AT_STAMP(7);                              // all warps done
}

constexpr size_t kSmem = Smem::TOTAL + 1024;

// (cols, rows of one clip, clips, planes) view of a two-plane fp16 activation; box = 64 cols x 64 rows of one clip
bool plane_map(CUtensorMap* m, const uint16_t* base, long long ps, long long bs, int ld, int cols, int rows, int batch) {
  cuuint64_t dims[4] = {(cuuint64_t)cols, (cuuint64_t)rows, (cuuint64_t)batch, 2};
  cuuint64_t strides[3] = {(cuuint64_t)ld * 2, (cuuint64_t)bs * 2, (cuuint64_t)ps * 2};
  cuuint32_t box[4] = {64, (cuuint32_t)T, 1, 1};
  return encode_map(m, base, 4, dims, strides, box, true);
}

}  // namespace

extern "C" int pm_attention_tc(const uint16_t* Q, long long q_ps, long long q_bs, int ldq, int q_cols, int q_col0,
                               const uint16_t* K, long long k_ps, long long k_bs, int ldk, int k_cols, int k_col0,
                               const uint16_t* V, long long v_ps, long long v_bs, int ldv, int v_cols, int v_col0,
                               float* O, int ldo, int batch, int heads, int tq, int tk, int head_dim,
                               uint16_t* planes, long long p_ps, int p_ld, int p_nsplit, void* stream) {
  PM_REQUIRE(Q && K && V && (O || planes) && batch >= 0 && heads > 0);
  PM_TAKE_FMT(p_nsplit, f16);
  PM_REQUIRE(!planes || (f16 && p_nsplit <= 2));           // fp16 planes in, (at most two) fp16 planes out
  PM_REQUIRE(pm_planes_ok(planes, p_ps, p_ld, p_nsplit, heads * head_dim, false));
  if (head_dim != HD || tq > T || tk > T || tq <= 0 || tk <= 0) return PM_EUNSUPPORTED;
  PM_REQUIRE(!O || (ldo & 3) == 0);
  // TMA: 16-byte aligned bases and strides; the head slices must lie inside the tensors
  for (const void* ptr : {(const void*)Q, (const void*)K, (const void*)V}) PM_REQUIRE((reinterpret_cast<uintptr_t>(ptr) & 15) == 0);
  PM_REQUIRE((ldq & 7) == 0 && (ldk & 7) == 0 && (ldv & 7) == 0 && (q_ps & 7) == 0 && (k_ps & 7) == 0 && (v_ps & 7) == 0);
  PM_REQUIRE(batch <= 1 || ((q_bs & 7) == 0 && (k_bs & 7) == 0 && (v_bs & 7) == 0));
  PM_REQUIRE(q_col0 >= 0 && k_col0 >= 0 && v_col0 >= 0 && q_col0 + heads * HD <= q_cols && k_col0 + heads * HD <= k_cols &&
             v_col0 + heads * HD <= v_cols && q_cols <= ldq && k_cols <= ldk && v_cols <= ldv);
  if (batch == 0) return PM_OK;
  CUtensorMap mq, mk, mv;
  if (!plane_map(&mq, Q, q_ps, q_bs, ldq, q_cols, tq, batch) || !plane_map(&mk, K, k_ps, k_bs, ldk, k_cols, tk, batch) ||
      !plane_map(&mv, V, v_ps, v_bs, ldv, v_cols, tk, batch))
    return PM_EBADARG;
  AttnParams p;
  p.heads = heads; p.tq = tq; p.tk = tk; p.qc0 = q_col0; p.kc0 = k_col0; p.vc0 = v_col0;
  p.scale = 1.0f / (sqrtf((float)head_dim) * PM_F16_ACT_SCALE * PM_F16_ACT_SCALE);
  p.out = O; p.ldo = ldo;
  p.planes = PmPlanes{reinterpret_cast<__nv_bfloat16*>(planes), p_ps, p_ld, p_nsplit};
  static unsigned long long configured = 0;
  if (pm_first_use_on_device(configured)) {
    cudaError_t e = cudaFuncSetAttribute(attention_tc_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kSmem);
    if (e != cudaSuccess) { configured = 0; return (int)e; }
  }
  attention_tc_kernel<<<batch * heads, NTHREADS, kSmem, (cudaStream_t)stream>>>(mq, mk, mv, p);
  PM_LAUNCH_CHECK();
}

#ifdef PM_ATTN_TIMING
extern "C" int pm_attn_timing_read(unsigned long long* host) {
  cudaError_t e = cudaDeviceSynchronize();
  if (e != cudaSuccess) return (int)e;
  return (int)cudaMemcpyFromSymbol(host, pm_attn_stamps, sizeof(unsigned long long) * 16);
}
#endif
