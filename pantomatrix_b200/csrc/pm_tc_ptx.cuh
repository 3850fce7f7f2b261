// PTX wrappers shared by the Hopper tensor-core kernels (tap-GEMM, VQ lookup, attention): mbarrier, TMA, wgmma and
// its shared-memory descriptors.  sm_90a.  Everything is static-inline: include from one .cu at a time.
#pragma once
#include <cuda.h>
#include <stdint.h>

// ---------------------------------------------------------------------------------------------------
// PTX wrappers
// ---------------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint32_t bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
// The watchdog's trap, out of line: a trap inlined into code after setmaxnreg.inc makes ptxas allocate that code at the
// launch's register limit instead of the raised one (the tap-GEMM consumers then spill their accumulators).
static __device__ __noinline__ void pm_watchdog_trap() { __trap(); }
// Bounded wait: a protocol bug must become a trap (an error the host sees), never a hung GPU.  The spin body is kept to
// the probe itself (try_wait suspends the thread for a hardware-defined slice): the watchdog clock is read only every
// 4096 probes.
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
  uint32_t spins = 0;
  long long t0 = 0;
  while (true) {
    uint32_t done;
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
        "selp.u32 %0, 1, 0, p;\n\t}"
        : "=r"(done) : "r"(bar), "r"(parity) : "memory");
    if (done) return;
    if ((++spins & 0xFFFu) == 0) {
      const long long t = clock64();
      if (t0 == 0) t0 = t;
      else if (t - t0 > 4000000000LL) pm_watchdog_trap();
    }
  }
}
// For waits that are expected to be long (a pipeline stage waiting for a slower one): back off between probes so that
// the waiting warps do not eat the issue slots of the working ones.
template <int SLEEP_NS = 40>
__device__ __forceinline__ void mbar_wait_relaxed(uint32_t bar, uint32_t parity) {
  uint32_t spins = 0;
  while (true) {
    uint32_t done;
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
        "selp.u32 %0, 1, 0, p;\n\t}"
        : "=r"(done) : "r"(bar), "r"(parity) : "memory");
    if (done) return;
    __nanosleep(SLEEP_NS);
    if (++spins > 50000000u) __trap();            // > 2 s: a protocol bug must become an error, never a hung GPU
  }
}
// Same, for the hot loops: first probe without touching the clock; the watchdog only runs while actually waiting.
__device__ __forceinline__ void mbar_wait_fast(uint32_t bar, uint32_t parity) {
  uint32_t done;
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
      "selp.u32 %0, 1, 0, p;\n\t}"
      : "=r"(done) : "r"(bar), "r"(parity) : "memory");
  if (!done) mbar_wait(bar, parity);
}
// One lane of a converged warp (PTX elect.sync): the canonical guard for TMA issue.  With warp-uniform control flow
// around it the compiler keeps descriptors and barrier addresses in uniform registers.
__device__ __forceinline__ bool elect_one() {
  uint32_t pred;
  asm volatile("{\n\t.reg .pred P1;\n\telect.sync _|P1, 0xffffffff;\n\tselp.u32 %0, 1, 0, P1;\n\t}" : "=r"(pred));
  return pred != 0;
}
__device__ __forceinline__ void tma_load_4d(uint32_t dst, const CUtensorMap* map, uint32_t bar, int c0, int c1, int c2, int c3) {
  asm volatile(
      "cp.async.bulk.tensor.4d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6}], [%2];"
      ::"r"(dst), "l"(map), "r"(bar), "r"(c0), "r"(c1), "r"(c2), "r"(c3) : "memory");
}
__device__ __forceinline__ void tma_load_3d(uint32_t dst, const CUtensorMap* map, uint32_t bar, int c0, int c1, int c2) {
  asm volatile(
      "cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5}], [%2];"
      ::"r"(dst), "l"(map), "r"(bar), "r"(c0), "r"(c1), "r"(c2) : "memory");
}
// TMA stores (smem -> global, clipped at the map's bounds), tracked per issuing thread as bulk async-groups
__device__ __forceinline__ void tma_store_3d(const CUtensorMap* map, uint32_t src, int c0, int c1, int c2) {
  asm volatile("cp.async.bulk.tensor.3d.global.shared::cta.bulk_group [%0, {%2, %3, %4}], [%1];"
               ::"l"(map), "r"(src), "r"(c0), "r"(c1), "r"(c2) : "memory");
}
__device__ __forceinline__ void tma_store_4d(const CUtensorMap* map, uint32_t src, int c0, int c1, int c2, int c3) {
  asm volatile("cp.async.bulk.tensor.4d.global.shared::cta.bulk_group [%0, {%2, %3, %4, %5}], [%1];"
               ::"l"(map), "r"(src), "r"(c0), "r"(c1), "r"(c2), "r"(c3) : "memory");
}
__device__ __forceinline__ void bulk_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
// this thread's bulk stores have finished reading shared memory (their global writes may still be in flight)
__device__ __forceinline__ void bulk_wait_read0() { asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory"); }
__device__ __forceinline__ void sts128(uint32_t addr, float a, float b, float c, float d) {
  asm volatile("st.shared.v4.f32 [%0], {%1, %2, %3, %4};" ::"r"(addr), "f"(a), "f"(b), "f"(c), "f"(d) : "memory");
}
__device__ __forceinline__ float4 lds128(uint32_t addr) {
  float4 v;
  asm volatile("ld.shared.v4.f32 {%0, %1, %2, %3}, [%4];" : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "r"(addr) : "memory");
  return v;
}
__device__ __forceinline__ void mbar_arrive(uint32_t bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}
// generic-proxy smem writes -> visible to the async proxy (TMA engine, wgmma operand reads)
__device__ __forceinline__ void fence_proxy_async_smem() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
// streaming 16-byte global load: read-only path, no L1 allocation (data is touched once)
__device__ __forceinline__ float4 ldg_stream4(const float4* p) {
  float4 v;
  asm volatile("ld.global.nc.L1::no_allocate.v4.f32 {%0, %1, %2, %3}, [%4];"
               : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "l"(p));
  return v;
}
// Warp-specialised register split (sm_90a): a whole warpgroup gives registers back to the CTA's pool or takes them
// from it.  Every warp of the warpgroup executes the same instruction; N is a multiple of 8 in [24, 256].
template <int N>
__device__ __forceinline__ void setmaxnreg_dec() { asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(N)); }
template <int N>
__device__ __forceinline__ void setmaxnreg_inc() { asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(N)); }
// named barrier over a subset of the CTA's warps (id 0 is __syncthreads)
__device__ __forceinline__ void named_bar_sync(uint32_t id, uint32_t threads) {
  asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(threads) : "memory");
}

// ---- wgmma (warpgroup MMA, sm_90a): D(64 x N, fp32 registers) += A(64 x 16, smem) * B(16 x N, smem) ----------------
// The accumulator fragment of thread t of the warpgroup: warp w = t / 32 owns rows 16 w + (t % 32) / 4 and that + 8;
// register 4 i + {0, 1} holds columns 8 i + 2 (t % 4) + {0, 1} of the first row, 4 i + {2, 3} the same columns of the
// second.  Accumulators are zeroed by the caller and always accumulated into (scale-d = 1).
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
// Keeps the compiler from moving accesses of an accumulator across wgmma issue / wait.
template <int R>
__device__ __forceinline__ void wgmma_fence_regs(float (&d)[R]) {
#pragma unroll
  for (int i = 0; i < R; ++i) asm volatile("" : "+f"(d[i])::"memory");
}
// Shared-memory matrix descriptor, 128-byte swizzle (layout type 1 in bits 62-63), start address >> 4 OR-ed in.
//   K-major operand: 8-row groups 1024 B apart (stride byte offset), leading byte offset unused (1).
//   MN-major operand: 64-element MN blocks LBO bytes apart, 8-row K groups 1024 B apart.
constexpr uint64_t GMMA_DESC_K_SW128 = (1ull << 62) | ((uint64_t)(1024 >> 4) << 32) | (1ull << 16);
constexpr uint64_t gmma_desc_mn_sw128(uint32_t lbo_bytes) {
  return (1ull << 62) | ((uint64_t)(1024 >> 4) << 32) | ((uint64_t)(lbo_bytes >> 4) << 16);
}
__device__ __forceinline__ uint64_t gmma_desc(uint64_t hi, uint32_t smem_addr) { return hi | (uint64_t)((smem_addr >> 4) & 0x3FFFu); }

#define PM_D8(i) "+f"(d[i]), "+f"(d[i + 1]), "+f"(d[i + 2]), "+f"(d[i + 3]), "+f"(d[i + 4]), "+f"(d[i + 5]), "+f"(d[i + 6]), "+f"(d[i + 7])
#define PM_WGMMA_N64(TY)                                                                                   \
  asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %34, 0;\n\t"                                           \
               "wgmma.mma_async.sync.aligned.m64n64k16.f32." TY "." TY " {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, %32, %33, p, 1, 1, 0, %35;\n\t}" \
               : PM_D8(0), PM_D8(8), PM_D8(16), PM_D8(24) \
               : "l"(da), "l"(db), "r"(1), "n"(TRANS_B))
template <bool BF16, int TRANS_B = 0>
__device__ __forceinline__ void wgmma_m64n64k16(float (&d)[32], uint64_t da, uint64_t db) {
  if constexpr (BF16) PM_WGMMA_N64("bf16");
  else PM_WGMMA_N64("f16");
}
#undef PM_WGMMA_N64
#define PM_WGMMA_N128(TY)                                                                                   \
  asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %66, 0;\n\t"                                           \
               "wgmma.mma_async.sync.aligned.m64n128k16.f32." TY "." TY " {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, %64, %65, p, 1, 1, 0, %67;\n\t}" \
               : PM_D8(0), PM_D8(8), PM_D8(16), PM_D8(24), PM_D8(32), PM_D8(40), PM_D8(48), PM_D8(56) \
               : "l"(da), "l"(db), "r"(1), "n"(TRANS_B))
template <bool BF16, int TRANS_B = 0>
__device__ __forceinline__ void wgmma_m64n128k16(float (&d)[64], uint64_t da, uint64_t db) {
  if constexpr (BF16) PM_WGMMA_N128("bf16");
  else PM_WGMMA_N128("f16");
}
#undef PM_WGMMA_N128
#define PM_WGMMA_N192(TY)                                                                                 \
  asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %98, 0;\n\t"                                           \
               "wgmma.mma_async.sync.aligned.m64n192k16.f32." TY "." TY " {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63, %64, %65, %66, %67, %68, %69, %70, %71, %72, %73, %74, %75, %76, %77, %78, %79, %80, %81, %82, %83, %84, %85, %86, %87, %88, %89, %90, %91, %92, %93, %94, %95}, %96, %97, p, 1, 1, 0, %99;\n\t}" \
               : PM_D8(0), PM_D8(8), PM_D8(16), PM_D8(24), PM_D8(32), PM_D8(40), PM_D8(48), PM_D8(56), PM_D8(64), PM_D8(72), PM_D8(80), PM_D8(88) \
               : "l"(da), "l"(db), "r"(1), "n"(TRANS_B))
template <bool BF16, int TRANS_B = 0>
__device__ __forceinline__ void wgmma_m64n192k16(float (&d)[96], uint64_t da, uint64_t db) {
  if constexpr (BF16) PM_WGMMA_N192("bf16");
  else PM_WGMMA_N192("f16");
}
#undef PM_WGMMA_N192
#define PM_WGMMA_N256(TY)                                                                                   \
  asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %130, 0;\n\t"                                           \
               "wgmma.mma_async.sync.aligned.m64n256k16.f32." TY "." TY " {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63, %64, %65, %66, %67, %68, %69, %70, %71, %72, %73, %74, %75, %76, %77, %78, %79, %80, %81, %82, %83, %84, %85, %86, %87, %88, %89, %90, %91, %92, %93, %94, %95, %96, %97, %98, %99, %100, %101, %102, %103, %104, %105, %106, %107, %108, %109, %110, %111, %112, %113, %114, %115, %116, %117, %118, %119, %120, %121, %122, %123, %124, %125, %126, %127}, %128, %129, p, 1, 1, 0, %131;\n\t}" \
               : PM_D8(0), PM_D8(8), PM_D8(16), PM_D8(24), PM_D8(32), PM_D8(40), PM_D8(48), PM_D8(56), PM_D8(64), PM_D8(72), PM_D8(80), PM_D8(88), PM_D8(96), PM_D8(104), PM_D8(112), PM_D8(120) \
               : "l"(da), "l"(db), "r"(1), "n"(TRANS_B))
template <bool BF16, int TRANS_B = 0>
__device__ __forceinline__ void wgmma_m64n256k16(float (&d)[128], uint64_t da, uint64_t db) {
  if constexpr (BF16) PM_WGMMA_N256("bf16");
  else PM_WGMMA_N256("f16");
}
#undef PM_WGMMA_N256
#undef PM_D8

// ---- host side: cuTensorMapEncodeTiled through the runtime's driver entry point (no -lcuda link dependency) ----
// Zero fill out of bounds.  encode_map: 2-byte elements (bf16 / fp16), 128-byte swizzle (wgmma operands).
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static inline EncodeTiledFn get_encode() {
  static EncodeTiledFn fn = nullptr;
  if (!fn) {
    void* sym = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &sym, cudaEnableDefault, &q) == cudaSuccess &&
        q == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<EncodeTiledFn>(sym);
  }
  return fn;
}

static inline bool encode_tiled(CUtensorMap* m, CUtensorMapDataType type, CUtensorMapSwizzle swizzle, const void* base,
                                int rank, const cuuint64_t* dims, const cuuint64_t* strides_bytes, const cuuint32_t* box) {
  EncodeTiledFn fn = get_encode();
  if (!fn) return false;
  cuuint32_t ones[5] = {1, 1, 1, 1, 1};
  return fn(m, type, (cuuint32_t)rank, const_cast<void*>(base), dims, strides_bytes, box, ones,
            CU_TENSOR_MAP_INTERLEAVE_NONE, swizzle, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
            CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
}

static inline bool encode_map(CUtensorMap* m, const void* base, int rank, const cuuint64_t* dims, const cuuint64_t* strides_bytes,
                const cuuint32_t* box, bool f16 = false) {
  return encode_tiled(m, f16 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT16 : CU_TENSOR_MAP_DATA_TYPE_BFLOAT16,
                      CU_TENSOR_MAP_SWIZZLE_128B, base, rank, dims, strides_bytes, box);
}

