// Audio front-end: PCM (int16 or fp32, interleaved channels) -> mono fp32 -> polyphase resampling, one launch.
//
// Output m of a clip is y[m] = sum_k h[k] * u[(m + n_pre_remove)*down - k], u = the mixed signal upsampled by zero
// insertion (scipy.signal.resample_poly / upfirdn, padtype='constant').  With t = (m + n_pre_remove)*down = q*up + p,
// only the taps k = p + up*j reach a nonzero u sample, the input sample q - j: output m visits the `taps` entries of
// phase p of the bank (bank[p*taps + j] = h[p + up*j], zero past the filter's end).
//
// Work split.  Outputs m and m + up share their phase, and their input windows lie `down` samples apart.  A tile covers
// up*G consecutive outputs; a warp takes one phase r and 32 of its G rows (outputs m0 + r + up*g), so the 32 lanes read
// the same tap in each step (one broadcast load through the read-only path) and shared-memory samples `down` apart
// (conflict-free for odd `down`).  The tile's input span (about G*down + taps samples) is converted, mixed down and
// staged in shared memory once.  G is chosen on the host so that the span fits; when even one row does not (reduced
// denominators beyond ~16 000), the kernel reads and mixes the input directly from global memory instead.  Every output
// is one thread's sequential FMA chain over its taps in a fixed order (oldest sample first), whatever the tile size,
// staging mode or batch position, so the result is deterministic and independent of the tiling.
#include "pm_common.cuh"
#include "../../include/pm_emage.h"

namespace {

constexpr int kThreads = 256;
constexpr int kMaxStage = 16384;             // staged samples per tile: 64 KB of shared memory
constexpr long long kTileOutputs = 4096;     // target outputs per tile

// Mono sample i of a clip: int16 -> v / 32768, channels summed in fp32 from +0.0 and divided by their count.  The
// association order is numpy's x.mean(axis=1) on an (n, channels) float32 array (the host path of audio_io): in channel
// order below 8 channels, numpy's 8-way pairwise block at exactly 8.  Explicit _rn intrinsics: no contraction, no fold
// of the +0.0 start (it turns -0.0 into +0.0, as numpy does).  C > 0: the channel count known at compile time (the
// common mono / stereo cases get straight-line loads); C == 0: `channels` at run time.
template <bool I16, int C>
__device__ __forceinline__ float pm_mix(const void* clip, long long i, int channels) {
  if constexpr (C > 0) channels = C;
  const long long e = i * channels;
  auto at = [&](int c) -> float {
    if constexpr (I16) return (float)__ldg(reinterpret_cast<const int16_t*>(clip) + e + c) * (1.0f / 32768.0f);
    else return __ldg(reinterpret_cast<const float*>(clip) + e + c);
  };
  if constexpr (C == 1) return __fadd_rn(0.0f, at(0));
  if constexpr (C == 2) return __fmul_rn(__fadd_rn(__fadd_rn(0.0f, at(0)), at(1)), 0.5f);   // == / 2, exactly
  if (channels == 1) return __fadd_rn(0.0f, at(0));
  float s;
  if (channels == 8) {
    s = __fadd_rn(__fadd_rn(__fadd_rn(at(0), at(1)), __fadd_rn(at(2), at(3))),
                  __fadd_rn(__fadd_rn(at(4), at(5)), __fadd_rn(at(6), at(7))));
    s = __fadd_rn(0.0f, s);
  } else {
    s = 0.0f;
    for (int c = 0; c < channels; ++c) s = __fadd_rn(s, at(c));
  }
  return __fdiv_rn(s, (float)channels);
}

template <bool I16, int C = 0>
__device__ __forceinline__ float pm_mix_or_zero(const void* clip, long long i, long long n_in, int channels) {
  return (i >= 0 && i < n_in) ? pm_mix<I16, C>(clip, i, channels) : 0.0f;
}

// stage[i - lo] = mono sample i for i in [lo, hi]: kStageUnroll independent loads in flight per thread.
constexpr int kStageUnroll = 8;
template <bool I16, int C>
__device__ __forceinline__ void pm_stage(float* stage, const void* clip, long long lo, long long hi, long long n_in,
                                         int channels) {
  for (long long base = lo + threadIdx.x; base <= hi; base += (long long)kThreads * kStageUnroll) {
    float v[kStageUnroll];
#pragma unroll
    for (int u = 0; u < kStageUnroll; ++u) v[u] = pm_mix_or_zero<I16, C>(clip, base + u * kThreads, n_in, channels);
#pragma unroll
    for (int u = 0; u < kStageUnroll; ++u)
      if (base + u * kThreads <= hi) stage[base + u * kThreads - lo] = v[u];
  }
}

template <bool I16, bool STAGED>
__global__ void __launch_bounds__(kThreads)
resample_poly_kernel(const void* __restrict__ pcm, long long in_bs, long long n_in, int channels,
                     const float* __restrict__ bank, int up, int down, int taps, long long n_pre_remove,
                     float* __restrict__ out, long long out_bs, long long n_out, int rows) {
  extern __shared__ float stage[];
  const int b = blockIdx.y;
  const void* clip = I16 ? (const void*)(reinterpret_cast<const int16_t*>(pcm) + b * in_bs)
                         : (const void*)(reinterpret_cast<const float*>(pcm) + b * in_bs);
  float* y = out + b * out_bs;
  const long long m0 = (long long)blockIdx.x * up * rows;
  const long long m_end = min(m0 + (long long)up * rows, n_out);
  // input span of the tile: the oldest sample of the first output .. the newest of the last
  const long long lo = (m0 + n_pre_remove) * down / up - (taps - 1);
  const long long hi = (m_end - 1 + n_pre_remove) * down / up;
  if constexpr (STAGED) {
    if (channels == 1) pm_stage<I16, 1>(stage, clip, lo, hi, n_in, channels);
    else if (channels == 2) pm_stage<I16, 2>(stage, clip, lo, hi, n_in, channels);
    else pm_stage<I16, 0>(stage, clip, lo, hi, n_in, channels);
    __syncthreads();
  }
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int groups = (rows + 31) >> 5;
  for (int unit = warp; unit < up * groups; unit += kThreads / 32) {
    const int r = unit / groups;
    const int g = (unit - r * groups) * 32 + lane;
    const long long m = m0 + r + (long long)up * g;
    if (g >= rows || m >= m_end) continue;
    const long long t = (m + n_pre_remove) * down;
    const long long q = t / up;
    const float* h = bank + (t - q * up) * taps;
    float acc = 0.0f;
    if constexpr (STAGED) {
      const float* x = stage + (q - lo);           // x[-j] = input sample q - j
#pragma unroll 4
      for (int j = taps - 1; j >= 0; --j) acc = fmaf(__ldg(h + j), x[-j], acc);
    } else {
      for (int j = taps - 1; j >= 0; --j) acc = fmaf(__ldg(h + j), pm_mix_or_zero<I16>(clip, q - j, n_in, channels), acc);
    }
    y[m] = acc;
  }
}

template <bool I16, bool STAGED>
int launch(const void* pcm, long long in_bs, int batch, long long n_in, int channels, const float* bank, int up,
           int down, int taps, long long n_pre_remove, float* out, long long out_bs, long long n_out, int rows,
           size_t smem, cudaStream_t st) {
  static unsigned long long configured = 0;
  auto kern = resample_poly_kernel<I16, STAGED>;
  if (STAGED && pm_first_use_on_device(configured)) {
    const cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, kMaxStage * 4);
    if (e != cudaSuccess) return (int)e;
  }
  const long long tiles = (n_out + (long long)up * rows - 1) / ((long long)up * rows);
  kern<<<dim3((unsigned)tiles, (unsigned)batch), kThreads, smem, st>>>(pcm, in_bs, n_in, channels, bank, up, down, taps,
                                                                       n_pre_remove, out, out_bs, n_out, rows);
  PM_LAUNCH_CHECK();
}

}  // namespace

extern "C" int pm_resample_poly_f32(const void* pcm, int is_int16, long long in_bs, int batch, long long n_in,
                                    int channels, const float* bank, int up, int down, int taps,
                                    long long n_pre_remove, float* out, long long out_bs, void* stream) {
  if (channels < 1 || channels > 8) return PM_EUNSUPPORTED;
  PM_REQUIRE(batch >= 0 && batch <= 65535 && n_in >= 0);
  PM_REQUIRE(up >= 1 && down >= 1 && taps >= 1 && n_pre_remove >= 0);
  PM_REQUIRE(is_int16 == 0 || is_int16 == 1);
  if (n_in == 0 || batch == 0) return PM_OK;              // nothing to write (empty tensors may have null pointers)
  PM_REQUIRE(pcm && bank && out);
  const long long n_out = (n_in * up + down - 1) / down;
  PM_REQUIRE(batch <= 1 || (in_bs >= n_in * channels && out_bs >= n_out));
  // rows per tile: about kTileOutputs outputs, a multiple of 32 where the staged span allows it
  long long rows = (kTileOutputs + up - 1) / up;
  rows = (rows + 31) / 32 * 32;
  const auto span = [&](long long g) { return g * down + taps + 1; };   // >= hi - lo + 1 of any tile of g rows
  while (rows > 32 && span(rows) > kMaxStage) rows -= 32;
  while (rows > 1 && span(rows) > kMaxStage) --rows;
  const bool staged = span(rows) <= kMaxStage;
  if (!staged) rows = 32;
  PM_REQUIRE((n_out + (long long)up * rows - 1) / ((long long)up * rows) <= 0x7fffffffLL);
  const size_t smem = staged ? (size_t)span(rows) * sizeof(float) : 0;
  cudaStream_t st = (cudaStream_t)stream;
  const int r = (int)rows;
  if (is_int16) {
    return staged ? launch<true, true>(pcm, in_bs, batch, n_in, channels, bank, up, down, taps, n_pre_remove, out, out_bs, n_out, r, smem, st)
                  : launch<true, false>(pcm, in_bs, batch, n_in, channels, bank, up, down, taps, n_pre_remove, out, out_bs, n_out, r, smem, st);
  }
  return staged ? launch<false, true>(pcm, in_bs, batch, n_in, channels, bank, up, down, taps, n_pre_remove, out, out_bs, n_out, r, smem, st)
                : launch<false, false>(pcm, in_bs, batch, n_in, channels, bank, up, down, taps, n_pre_remove, out, out_bs, n_out, r, smem, st);
}
