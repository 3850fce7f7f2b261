// Shared helpers for the EMAGE hot-path kernels (sm_90a).
#pragma once
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#define PM_OK 0
#define PM_EBADARG (-1)
#define PM_EUNSUPPORTED (-2)

// Every entry point: validate -> launch -> return cudaGetLastError() (positive) or PM_E* (negative).
#define PM_LAUNCH_CHECK()                                  \
  do {                                                     \
    cudaError_t _e = cudaGetLastError();                   \
    return _e == cudaSuccess ? PM_OK : (int)_e;            \
  } while (0)

#define PM_REQUIRE(cond) \
  do {                   \
    if (!(cond)) return PM_EBADARG; \
  } while (0)

static inline int pm_cdiv(long long a, long long b) { return (int)((a + b - 1) / b); }

// cudaFuncSetAttribute(MaxDynamicSharedMemorySize) is per DEVICE: one bit per device ordinal, kept by each call site.
// True when the current device has not been configured through `mask` yet (idempotent, so a race only repeats the call).
static inline bool pm_first_use_on_device(unsigned long long& mask) {
  int d = 0;
  if (cudaGetDevice(&d) != cudaSuccess || d < 0 || d >= 64) return true;
  if ((mask >> d) & 1ull) return false;
  mask |= 1ull << d;
  return true;
}

enum PmAct { PM_ACT_NONE = 0, PM_ACT_RELU = 1, PM_ACT_LEAKY = 2 };

__device__ __forceinline__ float pm_act(float v, int act, float slope) {
  if (act == PM_ACT_RELU) return v > 0.f ? v : 0.f;
  if (act == PM_ACT_LEAKY) return v > 0.f ? v : v * slope;
  return v;
}

// ORs the nb (0..32) low bits of v, MSB first, into the big-endian bit stream at w at bit pos: stream byte i is byte i
// of the buffer in memory, so the words hold the stream in its own byte order.  atomicOr keeps it independent of
// the order in which threads write codes that share a word.
__device__ __forceinline__ void pm_put_bits(unsigned* w, long long pos, unsigned v, int nb) {
  if (nb == 0) return;
  const unsigned long long x = (unsigned long long)v << (64 - (int)(pos & 31) - nb);
  atomicOr(w + (pos >> 5), __byte_perm((unsigned)(x >> 32), 0, 0x0123));
  if ((unsigned)x) atomicOr(w + (pos >> 5) + 1, __byte_perm((unsigned)x, 0, 0x0123));
}

__device__ __forceinline__ float pm_warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

__device__ __forceinline__ float pm_warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

// ---- split planes (operands of the tensor-core engine): x ~ p0 + p1 + p2, each the running remainder rounded to
// nearest even; two fp16 activation planes start from the half-away head of pm_f16_head instead (include/pm_emage.h) ----
struct PmPlanes {
  __nv_bfloat16* ptr;   // plane 0, element (row 0, channel 0); nullptr = no plane output
  long long ps;         // plane stride (elements)
  int ld;               // row stride (elements)
  int nsplit;           // 1..3
};

__device__ __forceinline__ void pm_split3(float v, __nv_bfloat16 (&p)[3]) {
  p[0] = __float2bfloat16_rn(v);
  float r = v - __bfloat162float(p[0]);
  p[1] = __float2bfloat16_rn(r);
  r -= __bfloat162float(p[1]);
  p[2] = __float2bfloat16_rn(r);
}

// Plane element format.  bf16 (default) needs 3 planes / 6 products for an fp32-quality GEMM; IEEE fp16 reaches the
// same accuracy with 2 planes / 3 products (11-bit mantissas) as long as magnitudes stay below 65504 - an overflow
// turns into inf - inf = NaN in the consumer GEMM and is caught by the host.
// Callers select it with bit 8 of an `nsplit` argument of the C ABI.
#ifndef PM_FMT_F16
#define PM_FMT_F16 0x100
#endif
// fp16 activation planes hold PM_F16_ACT_SCALE * x.  The second plane of an element below 2^-3 would be an fp16
// subnormal (|p1| < 2^-14), which tensor cores may flush; the exact pre-scale moves that threshold to 2^-9 (absolute error <= 2^-21 per element) and the overflow threshold to 65504 / 64 = 1023.
// The packed weights' acc_scale carries the matching 1 / 64 (ops.PackedW), so GEMM results are unchanged.
#define PM_F16_ACT_SCALE 64.0f
// host side: strip the format bit of an `nsplit` ABI argument into a flag
#define PM_TAKE_FMT(nsplit_var, flag_var)                          \
  const bool flag_var = ((nsplit_var) & PM_FMT_F16) != 0;          \
  (nsplit_var) &= 0xff

// Two-plane fp16 split of v (already pre-scaled): plane 0 = v rounded to 11 significant bits, plane 1 = the remainder.
// Plane 0 is formed with integer ops on the fp32 bit pattern (add half an ulp of the 10-bit mantissa, clear the 13 low
// bits: round-half-away, exponent carry included) - the result is exactly representable in fp16, so its conversion is
// exact and the remainder v - f0 needs no conversion BACK from fp16.  Those back-conversions run at a fraction of the
// FP32 rate and would make every plane-writing epilogue conversion-bound.  (Below 2^-14 plane 0 would be an fp16 subnormal, which the
// tensor core flushes anyway.)
__device__ __forceinline__ float pm_f16_head(float v) {
  return __uint_as_float((__float_as_uint(v) + 0x00001000u) & 0xFFFFE000u);
}

// The split rule itself, in registers, for two values at once (two adjacent channels): w[pl] holds plane pl of x in
// its low and of y in its high 16 bits, for pl < nsplit.  fp16: both are pre-scaled by PM_F16_ACT_SCALE first, and
// two planes take the pm_f16_head head; otherwise each plane is the running remainder rounded to nearest even.
// Every plane writer goes through it (pm_store_planes*_t, the tap-GEMM's TMA-store epilogue).  Successive planes are
// peeled off a running remainder under a fully unrolled loop: no dynamically indexed temporaries (they would live in
// local memory).  The pre-scale is __fmul_rn so that no caller's code can contract it into a following subtraction.
// NS > 0 fixes the plane count at compile time (then `nsplit` is ignored); NS = 0 reads it from `nsplit`.
template <bool F16, int NS = 0>
__device__ __forceinline__ void pm_split_pair_t(float x, float y, int nsplit, uint32_t (&w)[3]) {
  if constexpr (NS > 0) nsplit = NS;
  if constexpr (F16) {
    x = __fmul_rn(x, PM_F16_ACT_SCALE);
    y = __fmul_rn(y, PM_F16_ACT_SCALE);
    if (nsplit == 2) {
      const float fx = pm_f16_head(x), fy = pm_f16_head(y);
      const __half2 a = __floats2half2_rn(fx, fy), b = __floats2half2_rn(x - fx, y - fy);   // a is exact
      w[0] = *reinterpret_cast<const uint32_t*>(&a);
      w[1] = *reinterpret_cast<const uint32_t*>(&b);
      return;
    }
#pragma unroll
    for (int pl = 0; pl < 3; ++pl) {
      if (pl < nsplit) {
        const __half2 h = __floats2half2_rn(x, y);
        w[pl] = *reinterpret_cast<const uint32_t*>(&h);
        x -= __low2float(h); y -= __high2float(h);
      }
    }
  } else {
#pragma unroll
    for (int pl = 0; pl < 3; ++pl) {
      if (pl < nsplit) {
        const __nv_bfloat162 h = __floats2bfloat162_rn(x, y);
        w[pl] = *reinterpret_cast<const uint32_t*>(&h);
        x -= __low2float(h); y -= __high2float(h);
      }
    }
  }
}

template <bool F16>
__device__ __forceinline__ void pm_store_planes_t(const PmPlanes& P, long long row, int c, float v) {
  uint16_t* o = reinterpret_cast<uint16_t*>(P.ptr) + row * P.ld + c;
  uint32_t w[3];
  pm_split_pair_t<F16>(v, 0.f, P.nsplit, w);
#pragma unroll
  for (int pl = 0; pl < 3; ++pl)
    if (pl < P.nsplit) o[(long long)pl * P.ps] = (uint16_t)w[pl];
}
__device__ __forceinline__ void pm_store_planes(const PmPlanes& P, long long row, int c, float v) {
  pm_store_planes_t<false>(P, row, c, v);
}

// 4 consecutive channels, c % 4 == 0, ld % 4 == 0, ps % 4 == 0, 8-byte aligned base
template <bool F16>
__device__ __forceinline__ void pm_store_planes4_t(const PmPlanes& P, long long row, int c, float4 v) {
  __nv_bfloat16* o = P.ptr + row * P.ld + c;
  uint32_t lo[3], hi[3];
  pm_split_pair_t<F16>(v.x, v.y, P.nsplit, lo);
  pm_split_pair_t<F16>(v.z, v.w, P.nsplit, hi);
#pragma unroll
  for (int pl = 0; pl < 3; ++pl)
    if (pl < P.nsplit) *reinterpret_cast<uint2*>(o + (long long)pl * P.ps) = make_uint2(lo[pl], hi[pl]);
}
__device__ __forceinline__ void pm_store_planes4(const PmPlanes& P, long long row, int c, float4 v) {
  pm_store_planes4_t<false>(P, row, c, v);
}

static inline bool pm_planes_ok(const void* ptr, long long ps, int ld, int nsplit, int ch, bool vec4) {
  if (!ptr) return true;
  if (nsplit < 1 || nsplit > 3 || ld < ch) return false;
  if (vec4 && ((ld & 3) || (ps & 3) || (reinterpret_cast<uintptr_t>(ptr) & 7))) return false;
  return true;
}
