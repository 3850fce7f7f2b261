// Persistent bidirectional LSTM layer (CaMN / DisCo decoders, BASELINE configs[2],[3]).
// Replaces the cuDNN/ATen recurrence inside nn.LSTM (reference models/camn_audio/modeling_camn_audio.py:205-217,
// 264-271; models/disco_audio/modeling_disco_audio.py:212-216,255).  Contract: include/pm_emage.h.
//
// The input projections W_ih x + b for all time steps are one big tap-GEMM; this kernel runs the sequential part.
// One cooperative launch per layer (and per 64 clips).  CTA (dir, half, slot) owns 16 hidden units of one direction
// for one half (32 rows) of the batch and keeps their 64 rows of W_hh (fp32, 128 KB) in shared memory for all T
// steps.  Per step the CTA reloads h_{t-1} of its rows (written by the 32 CTAs of its group one step earlier, read
// with ld.global.cg), forms the gate pre-activations, updates its private cell states (registers), publishes h_t
// and meets its group at a global-memory barrier (release/acquire on a counter).
//
// The recurrent product is shared-memory-bandwidth bound, so it is register tiled: a thread accumulates an
// 8 gate-row x 8 batch-row block over one eighth of K (16 LDS.128 per 256 FMA; a quarter-warp always reads 128
// contiguous bytes), then the eight K-slices - adjacent lanes - are combined with a shuffle reduce-scatter that
// leaves each lane with the 8 gate rows (2 units x 4 gates) of ONE batch row, whose cell update it then performs.
#include "pm_common.cuh"
#include "../../include/pm_emage.h"

namespace {

constexpr int HID = 512;      // hidden size
constexpr int RB = 32;        // batch rows per CTA
constexpr int UPC = 16;       // hidden units per CTA
constexpr int G = HID / UPC;  // CTAs per (direction, batch half) group
constexpr int NT = 256;       // 8 unit pairs (warps) x 4 row groups x 8 K-slices

struct LstmParams {
  const float* xproj; long long x_bs; int ldx;   // (B, T, >= 2*4H): column dir*4H + gate*H + unit
  const float* whh;                              // (2, 4H, H)
  float* y; long long y_bs; int ldy;             // (B, T, >= 2H): forward h in [0,H), backward in [H,2H)
  unsigned int* barrier;                         // 2 * halves counters, zero at launch
  int B, T, halves;                              // halves = ceil(B / RB) <= 2
};

__device__ __forceinline__ float sigmoidf_(float x) { return 1.f / (1.f + expf(-x)); }

__global__ void __launch_bounds__(NT, 1) lstm_bidir_kernel(LstmParams p) {
  extern __shared__ float smem[];
  constexpr int H = HID;
  float* Ws = smem;                             // [4 * UPC][H]  rows ordered gate-major: gate * UPC + unit_local
  float* hs = Ws + 4 * UPC * H;                 // [RB][H]
  const int grp = blockIdx.x / G, slot = blockIdx.x % G;
  const int dir = grp / p.halves, half = grp % p.halves;
  const int tid = threadIdx.x;
  const int up = tid >> 5;                      // unit pair: local units 2*up, 2*up+1
  const int kq = tid & 7, bg = (tid >> 3) & 3;  // K-slice, group of 8 batch rows
  const int u0 = slot * UPC;                    // first global unit of this CTA
  const int row0 = half * RB;                   // first batch row of this CTA
  const int nrows = p.B - row0 < RB ? p.B - row0 : RB;

  // resident W_hh slice
  const float* W = p.whh + (long long)dir * 4 * H * H;
  for (int i = tid; i < 4 * UPC * (H / 4); i += NT) {
    const int r = i / (H / 4), k4 = i % (H / 4);
    const int gate = r / UPC, ul = r % UPC;
    *reinterpret_cast<float4*>(Ws + r * H + k4 * 4) =
        *reinterpret_cast<const float4*>(W + (long long)(gate * H + u0 + ul) * H + k4 * 4);
  }
  float c0 = 0.f, c1 = 0.f;                      // cell states: batch row `b`, units 2*up and 2*up+1
  const int bl = bg * 8 + kq;                    // the batch row (within this CTA) this lane finishes
  const bool active = bl < nrows;
  const long long b = row0 + bl;
  const float* xrow = p.xproj + b * p.x_bs + (long long)dir * 4 * H + u0 + 2 * up;
  float* yrow = p.y + b * p.y_bs + (long long)dir * H + u0 + 2 * up;
  const float* ybase = p.y + (long long)row0 * p.y_bs + dir * H;
  const float* wbase = Ws + (2 * up) * H + kq * 4;
  const float* hbase = hs + (bg * 8) * H + kq * 4;
  const bool s4 = kq & 4, s2 = kq & 2, s1 = kq & 1;
  __syncthreads();

  for (int s = 0; s < p.T; ++s) {
    const int t = dir == 0 ? s : p.T - 1 - s;
    const int tp = dir == 0 ? t - 1 : t + 1;    // time index holding h_{prev}
    // input projection of this lane's row (issued early: global latency overlaps the h load and the product)
    float x[8];                                  // [gate * 2 + unit]
#pragma unroll
    for (int r = 0; r < 8; ++r) x[r] = 0.f;
    if (active) {
      const float* xp = xrow + (long long)t * p.ldx;
#pragma unroll
      for (int g = 0; g < 4; ++g) { x[2 * g] = __ldg(xp + g * H); x[2 * g + 1] = __ldg(xp + g * H + 1); }
    }
    float pre[8];                                // gate pre-activations of row bl
    if (s > 0) {                                 // block-uniform
      // h_{prev} of this group's rows -> smem
#pragma unroll 4
      for (int i = tid; i < RB * (H / 4); i += NT) {
        const int r = i / (H / 4), k4 = i % (H / 4);
        float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
        if (r < nrows) v = __ldcg(reinterpret_cast<const float4*>(ybase + (long long)r * p.y_bs + (long long)tp * p.ldy + k4 * 4));
        *reinterpret_cast<float4*>(hs + r * H + k4 * 4) = v;
      }
      __syncthreads();
      float acc[8][8];                           // [gate * 2 + unit][batch row of the group]
#pragma unroll
      for (int r = 0; r < 8; ++r)
#pragma unroll
        for (int i = 0; i < 8; ++i) acc[r][i] = 0.f;
#pragma unroll 1
      for (int j = 0; j < H / 32; ++j) {         // K-slice kq takes the float4 columns kq, kq + 8, kq + 16, ...
        float4 w[8];
#pragma unroll
        for (int r = 0; r < 8; ++r) w[r] = *reinterpret_cast<const float4*>(wbase + ((r >> 1) * UPC + (r & 1)) * H + j * 32);
#pragma unroll
        for (int i = 0; i < 8; ++i) {
          const float4 h4 = *reinterpret_cast<const float4*>(hbase + i * H + j * 32);
#pragma unroll
          for (int r = 0; r < 8; ++r) {
            acc[r][i] = fmaf(h4.x, w[r].x, acc[r][i]); acc[r][i] = fmaf(h4.y, w[r].y, acc[r][i]);
            acc[r][i] = fmaf(h4.z, w[r].z, acc[r][i]); acc[r][i] = fmaf(h4.w, w[r].w, acc[r][i]);
          }
        }
      }
      // reduce-scatter over the 8 K-slices (lanes kq = 0..7): lane kq ends with the full sums of batch row kq
#pragma unroll
      for (int r = 0; r < 8; ++r) {
        float a4[4], a2[2];
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          const float keep = s4 ? acc[r][i + 4] : acc[r][i], send = s4 ? acc[r][i] : acc[r][i + 4];
          a4[i] = keep + __shfl_xor_sync(0xffffffffu, send, 4);
        }
#pragma unroll
        for (int i = 0; i < 2; ++i) {
          const float keep = s2 ? a4[i + 2] : a4[i], send = s2 ? a4[i] : a4[i + 2];
          a2[i] = keep + __shfl_xor_sync(0xffffffffu, send, 2);
        }
        const float keep = s1 ? a2[1] : a2[0], send = s1 ? a2[0] : a2[1];
        pre[r] = x[r] + (keep + __shfl_xor_sync(0xffffffffu, send, 1));
      }
    } else {
#pragma unroll
      for (int r = 0; r < 8; ++r) pre[r] = x[r];
    }
    if (active) {                                 // gates i, f, g, o -> c, h   (nn.LSTM equations)
      c0 = sigmoidf_(pre[2]) * c0 + sigmoidf_(pre[0]) * tanhf(pre[4]);
      c1 = sigmoidf_(pre[3]) * c1 + sigmoidf_(pre[1]) * tanhf(pre[5]);
      float* yo = yrow + (long long)t * p.ldy;
      __stcg(yo, sigmoidf_(pre[6]) * tanhf(c0));
      __stcg(yo + 1, sigmoidf_(pre[7]) * tanhf(c1));
    }
    // group barrier: every CTA of this (direction, batch half) has published h_t
    __threadfence();
    __syncthreads();
    if (tid == 0) {
      atomicAdd(p.barrier + grp, 1u);
      const unsigned int target = (unsigned int)(s + 1) * (unsigned int)G;
      const long long t0 = clock64();
      while (*reinterpret_cast<volatile unsigned int*>(p.barrier + grp) < target) {
        if (clock64() - t0 > 4000000000LL) __trap();          // never hang the GPU on a protocol bug
      }
      __threadfence();
    }
    __syncthreads();
  }
}

// Conditioning columns of the layer-0 input, one thread per output element: [speaker row | seed pose | seed flag].
// Output row r of a clip shows seed row j = r, or r - (t - seed_len) past the end of a shorter seed (the appended
// copy of its last t - seed_len rows); rows j < seed_frames carry (seed[j], 1), the others zeros.
__global__ void __launch_bounds__(256) lstm_cond_kernel(
    const float* __restrict__ spk, long long n_spk, int spk_dim, const long long* __restrict__ speaker_id,
    const float* __restrict__ seed, long long seed_bs, int seed_ld, int seed_len, int seed_frames, int pose_dims,
    float* __restrict__ out, long long o_bs, int ldo, int batch, int t) {
  const int cols = spk_dim + pose_dims + 1;
  const long long total = (long long)batch * t * cols;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const int c = (int)(i % cols);
    const long long bt = i / cols;
    const int r = (int)(bt % t);
    const long long b = bt / t;
    float v;
    if (c < spk_dim) {
      long long k = speaker_id[b];                 // clamped like pm_gather_rows_f32: never read outside the table
      k = k < 0 ? 0 : (k >= n_spk ? n_spk - 1 : k);
      v = spk[k * spk_dim + c];
    } else {
      const int j = r < seed_len ? r : r - (t - seed_len);
      const bool flagged = j < seed_frames;
      const int k = c - spk_dim;
      v = k == pose_dims ? (flagged ? 1.f : 0.f)
                         : (flagged && seed ? seed[b * seed_bs + (long long)j * seed_ld + k] : 0.f);
    }
    out[b * o_bs + (long long)r * ldo + c] = v;
  }
}

}  // namespace

extern "C" int pm_lstm_cond_f32(const float* spk, long long n_spk, int spk_dim, const long long* speaker_id,
                                const float* seed, long long seed_bs, int seed_ld, int seed_len, int seed_frames,
                                int pose_dims, float* out, long long o_bs, int ldo, int batch, int t, void* stream) {
  PM_REQUIRE(spk && speaker_id && out && n_spk > 0 && spk_dim >= 0 && pose_dims >= 0 && batch >= 0 && t >= 0);
  PM_REQUIRE(ldo >= spk_dim + pose_dims + 1 && seed_frames >= 0 && seed_len > 0 && t <= 2LL * seed_len);
  PM_REQUIRE(!seed || seed_ld >= pose_dims);
  if (seed_frames > seed_len) seed_frames = seed_len;
  const long long total = (long long)batch * t * (spk_dim + pose_dims + 1);
  if (total == 0) return PM_OK;
  long long g = (total + 255) / 256;
  if (g > 148 * 16) g = 148 * 16;
  lstm_cond_kernel<<<(unsigned)g, 256, 0, (cudaStream_t)stream>>>(spk, n_spk, spk_dim, speaker_id, seed, seed_bs, seed_ld,
                                                                 seed_len, seed_frames, pose_dims, out, o_bs, ldo, batch, t);
  PM_LAUNCH_CHECK();
}

extern "C" int pm_lstm_bidir_f32(const float* xproj, long long x_bs, int ldx, const float* whh,
                                 float* y, long long y_bs, int ldy, unsigned int* barrier,
                                 int batch, int t, int hidden, void* stream) {
  PM_REQUIRE(xproj && whh && y && barrier && batch > 0 && t > 0);
  if (hidden != HID) return PM_EUNSUPPORTED;
  PM_REQUIRE(ldx >= 8 * hidden && ldy >= 2 * hidden && (ldy & 3) == 0 && (y_bs & 3) == 0);
  PM_REQUIRE((reinterpret_cast<uintptr_t>(y) & 15) == 0 && (reinterpret_cast<uintptr_t>(whh) & 15) == 0);
  const size_t smem = (size_t)(4 * UPC + RB) * HID * sizeof(float);       // 192 KB
  static unsigned long long configured = 0;
  if (pm_first_use_on_device(configured)) {
    cudaError_t e = cudaFuncSetAttribute(lstm_bidir_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) { configured = 0; return (int)e; }
  }
  cudaStream_t st = (cudaStream_t)stream;
  for (int b0 = 0; b0 < batch; b0 += 2 * RB) {         // batch rows are independent: 64 clips (128 CTAs) per launch
    const int nb = batch - b0 < 2 * RB ? batch - b0 : 2 * RB;
    const int halves = (nb + RB - 1) / RB;
    cudaError_t e = cudaMemsetAsync(barrier, 0, 4 * sizeof(unsigned int), st);
    if (e != cudaSuccess) return (int)e;
    LstmParams p{xproj + (long long)b0 * x_bs, x_bs, ldx, whh, y + (long long)b0 * y_bs, y_bs, ldy, barrier, nb, t, halves};
    void* args[] = {&p};
    e = cudaLaunchCooperativeKernel((const void*)lstm_bidir_kernel, dim3(2 * halves * G), dim3(NT), args, smem, st);
    if (e != cudaSuccess) return (int)e;
  }
  return PM_OK;
}
