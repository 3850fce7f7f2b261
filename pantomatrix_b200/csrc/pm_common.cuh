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

// ---- split-bf16 planes (operands of the tensor-core engine): x ~ p0 + p1 + p2, round-to-nearest each ----
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

// Successive planes are peeled off a running remainder: no dynamically indexed temporaries (they would live in
// local memory).
template <bool F16>
__device__ __forceinline__ void pm_store_planes_t(const PmPlanes& P, long long row, int c, float v) {
  if constexpr (F16) {
    __half* o = reinterpret_cast<__half*>(P.ptr) + row * P.ld + c;
    v *= PM_F16_ACT_SCALE;
    if (P.nsplit <= 2) {
      const float f0 = P.nsplit == 2 ? pm_f16_head(v) : v;
      o[0] = __float2half_rn(f0);
      if (P.nsplit == 2) o[P.ps] = __float2half_rn(v - f0);
    } else {
      for (int pl = 0; pl < P.nsplit; ++pl) {
        const __half h = __float2half_rn(v);
        o[(long long)pl * P.ps] = h;
        v -= __half2float(h);
      }
    }
  } else {
    __nv_bfloat16* o = P.ptr + row * P.ld + c;
    for (int pl = 0; pl < P.nsplit; ++pl) {
      const __nv_bfloat16 h = __float2bfloat16_rn(v);
      o[(long long)pl * P.ps] = h;
      v -= __bfloat162float(h);
    }
  }
}
__device__ __forceinline__ void pm_store_planes(const PmPlanes& P, long long row, int c, float v) {
  pm_store_planes_t<false>(P, row, c, v);
}

// 4 consecutive channels, c % 4 == 0, ld % 4 == 0, ps % 4 == 0, 8-byte aligned base
template <bool F16>
__device__ __forceinline__ void pm_store_planes4_t(const PmPlanes& P, long long row, int c, float4 v) {
  if constexpr (F16) {
    __half* o = reinterpret_cast<__half*>(P.ptr) + row * P.ld + c;
    v.x *= PM_F16_ACT_SCALE; v.y *= PM_F16_ACT_SCALE; v.z *= PM_F16_ACT_SCALE; v.w *= PM_F16_ACT_SCALE;
    if (P.nsplit == 2) {
      const float4 f = make_float4(pm_f16_head(v.x), pm_f16_head(v.y), pm_f16_head(v.z), pm_f16_head(v.w));
      const __half2 a0 = __floats2half2_rn(f.x, f.y), a1 = __floats2half2_rn(f.z, f.w);                       // exact
      const __half2 b0 = __floats2half2_rn(v.x - f.x, v.y - f.y), b1 = __floats2half2_rn(v.z - f.z, v.w - f.w);
      uint2 w0, w1;
      w0.x = *reinterpret_cast<const uint32_t*>(&a0); w0.y = *reinterpret_cast<const uint32_t*>(&a1);
      w1.x = *reinterpret_cast<const uint32_t*>(&b0); w1.y = *reinterpret_cast<const uint32_t*>(&b1);
      *reinterpret_cast<uint2*>(o) = w0;
      *reinterpret_cast<uint2*>(o + P.ps) = w1;
      return;
    }
    for (int pl = 0; pl < P.nsplit; ++pl) {
      const __half2 lo = __floats2half2_rn(v.x, v.y), hi = __floats2half2_rn(v.z, v.w);
      uint2 w;
      w.x = *reinterpret_cast<const uint32_t*>(&lo);
      w.y = *reinterpret_cast<const uint32_t*>(&hi);
      *reinterpret_cast<uint2*>(o + (long long)pl * P.ps) = w;
      v.x -= __low2float(lo); v.y -= __high2float(lo); v.z -= __low2float(hi); v.w -= __high2float(hi);
    }
  } else {
    __nv_bfloat16* o = P.ptr + row * P.ld + c;
    for (int pl = 0; pl < P.nsplit; ++pl) {
      const __nv_bfloat162 lo = __floats2bfloat162_rn(v.x, v.y), hi = __floats2bfloat162_rn(v.z, v.w);
      uint2 w;
      w.x = *reinterpret_cast<const uint32_t*>(&lo);
      w.y = *reinterpret_cast<const uint32_t*>(&hi);
      *reinterpret_cast<uint2*>(o + (long long)pl * P.ps) = w;
      v.x -= __low2float(lo); v.y -= __high2float(lo); v.z -= __low2float(hi); v.w -= __high2float(hi);
    }
  }
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
