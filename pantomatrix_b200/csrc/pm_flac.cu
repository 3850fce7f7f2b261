// FLAC encoding of int16 / 24-bit int32 samples (pantomatrix_b200/flac.py): frames of 4096 samples by the rule of
// include/pm_emage.h and DESIGN.md section 13 (CONSTANT, FIXED 0..4 with partitioned Rice residuals or VERBATIM
// subframes, the exact minimum; stereo decorrelation by the smallest pair).  Two launches per call after the caller's
// memset of the output slots:
//   pm_flac_analyse  one CTA per (clip, frame, channel candidate): the best subframe's size and parameters, a record;
//   pm_flac_emit     one CTA per (clip, frame): channel assignment, header, subframes ORed into the slot, CRC-16.
// Every subframe's size is exact after the analysis, so the emit writes straight into the slot: no scratch copy.
// CPU restatement: oracle/flac_oracle.py.  Every byte depends only on the clip's samples, channels, bps and rate.
#include <cub/block/block_scan.cuh>

#include "pm_common.cuh"
#include "../../include/pm_emage.h"

namespace {

constexpr int BLOCK = 4096;               // samples per frame
constexpr int THREADS = 256;
constexpr int PER = BLOCK / THREADS;      // samples per thread in the emit's scan
constexpr int NK = 31;                    // Rice parameters 0..30
constexpr int KMAX0 = 14;                 // method 00: 4-bit parameters, 15 is the escape
constexpr int MAXP = 8;                   // partition orders 0..8
constexpr int REC = 66;                   // record: bits, type | order << 8 | p << 16 | method << 24, 256 k bytes
constexpr int CONSTANT = 0, FIXED = 1, VERBATIM = 2;

// Candidate c of a stereo frame: 0 L, 1 R, 2 S = L - R (bps + 1), 3 M = (L + R) >> 1; otherwise channel c.
template <typename T>
__device__ __forceinline__ bool load(int* x, const T* src, int bs, int ch, int cand, int bps) {
  bool bad = false;
  const int lim = 1 << (bps - 1);
  for (int i = threadIdx.x; i < bs; i += THREADS) {
    int v;
    if (ch == 2 && cand >= 2) {
      const int l = src[2 * i], r = src[2 * i + 1];
      bad |= l < -lim || l >= lim || r < -lim || r >= lim;
      v = cand == 2 ? l - r : (l + r) >> 1;
    } else {
      v = src[(long long)i * ch + cand];
      bad |= v < -lim || v >= lim;
    }
    x[i] = v;
  }
  return bad;
}

// FIXED predictor residual of order o at i >= o.
__device__ __forceinline__ int residual(const int* x, int i, int o) {
  switch (o) {
    case 0: return x[i];
    case 1: return x[i] - x[i - 1];
    case 2: return x[i] - 2 * x[i - 1] + x[i - 2];
    case 3: return x[i] - 3 * x[i - 1] + 3 * x[i - 2] - x[i - 3];
    default: return x[i] - 4 * x[i - 1] + 6 * x[i - 2] - 4 * x[i - 3] + x[i - 4];
  }
}

__device__ __forceinline__ unsigned zigzag(int e) { return ((unsigned)e << 1) ^ (unsigned)(e >> 31); }

// S[k] += the same sums held by the thread off lanes / threads away (a butterfly step).  Called by every thread.
__device__ __forceinline__ void xor_add(unsigned long long (&S)[NK], int off, unsigned long long (*xch)[NK]) {
  if (off < 32) {
#pragma unroll
    for (int k = 0; k < NK; ++k) S[k] += __shfl_xor_sync(0xffffffffu, S[k], off);
    return;
  }
  const int w = threadIdx.x >> 5;            // every lane of a warp holds the warp's sums by now
  if ((threadIdx.x & 31) == 0) {
#pragma unroll
    for (int k = 0; k < NK; ++k) xch[w][k] = S[k];
  }
  __syncthreads();
#pragma unroll
  for (int k = 0; k < NK; ++k) S[k] += xch[w ^ (off >> 5)][k];
  __syncthreads();
}

template <typename T>
__global__ void __launch_bounds__(THREADS) flac_analyse_kernel(const T* __restrict__ pcm, long long cs, int n, int ch,
                                                               int bps, int* __restrict__ rec) {
  __shared__ int x[BLOCK];
  __shared__ unsigned cost[2][512];                    // per (level p, partition j) at (1 << p) + j: bits, method 0/1
  __shared__ unsigned char kbest[2][512];
  __shared__ unsigned long long xch[THREADS / 32][NK];
  __shared__ unsigned long long tot[2][MAXP + 1];
  __shared__ unsigned char kord[5][256];
  __shared__ int ord_bits[5], ord_pm[5];
  const int nc = ch == 2 ? 4 : ch;
  const int frame = blockIdx.x / nc, cand = blockIdx.x % nc, t = threadIdx.x;
  const long long clip = blockIdx.y;
  const int start = frame * BLOCK, bs = min(BLOCK, n - start);
  int* r = rec + ((clip * (gridDim.x / nc) + frame) * nc + cand) * REC;
  const int bpsc = ch == 2 && cand == 2 ? bps + 1 : bps;
  if (__syncthreads_or(load(x, pcm + clip * cs + (long long)start * ch, bs, ch, cand, bps))) {
    if (t == 0) r[0] = -1;                              // a 24-bit sample out of range: the frame is not coded
    return;
  }
  bool diff = false;
  for (int i = t; i < bs; i += THREADS) diff |= x[i] != x[0];
  if (!__syncthreads_or(diff)) {
    if (t == 0) r[0] = 8 + bpsc, r[1] = CONSTANT;
    return;
  }
  const int pmax = min(MAXP, __ffs(bs) - 1);
  const int grp = THREADS >> pmax, s = bs >> pmax;      // threads per smallest partition, its samples
  const int j0 = t / grp, sub = t % grp;
  const int maxo = min(4, bs);
  for (int o = 0; o <= maxo; ++o) {
    unsigned long long S[NK];
#pragma unroll
    for (int k = 0; k < NK; ++k) S[k] = 0;
    for (int i = j0 * s + sub; i < (j0 + 1) * s; i += grp) {
      if (i < o) continue;
      const unsigned u = zigzag(residual(x, i, o));
#pragma unroll
      for (int k = 0; k < NK; ++k) S[k] += u >> k;
    }
    int off = 1;
    for (; off < grp; off <<= 1) xor_add(S, off, xch);
    for (int p = pmax; p >= 0; --p) {                   // here off == THREADS >> p: the level's group size
      if ((t & (off - 1)) == 0 && (bs >> p) >= o) {
        const int j = t / off;
        const unsigned long long count = (bs >> p) - (j == 0 ? o : 0);
        unsigned long long b0 = ~0ull, b1 = ~0ull;
        int k0 = 0, k1 = 0;
#pragma unroll
        for (int k = 0; k < NK; ++k) {
          const unsigned long long c = count * (k + 1) + S[k];
          if (k <= KMAX0 && c < b0) b0 = c, k0 = k;
          if (c < b1) b1 = c, k1 = k;
        }
        cost[0][(1 << p) + j] = (unsigned)b0 + 4, kbest[0][(1 << p) + j] = (unsigned char)k0;
        cost[1][(1 << p) + j] = (unsigned)b1 + 5, kbest[1][(1 << p) + j] = (unsigned char)k1;
      }
      if (p > 0) {
        xor_add(S, off, xch);
        off <<= 1;
      }
    }
    __syncthreads();
    const int warp = t >> 5, lane = t & 31;
    for (int p = warp; p <= pmax; p += THREADS / 32) {
      unsigned long long a = 0, b = 0;
      for (int j = lane; j < (1 << p); j += 32) a += cost[0][(1 << p) + j], b += cost[1][(1 << p) + j];
      for (int d = 16; d; d >>= 1) a += __shfl_xor_sync(0xffffffffu, a, d), b += __shfl_xor_sync(0xffffffffu, b, d);
      if (lane == 0) tot[0][p] = a, tot[1][p] = b;
    }
    __syncthreads();
    if (t == 0) {
      unsigned long long best = ~0ull;
      int bp = 0, bm = 0;
      for (int p = 0; p <= pmax; ++p) {
        if ((bs >> p) < o) continue;
        const int m = tot[1][p] < tot[0][p];
        const unsigned long long bits = 6 + tot[m][p];
        if (bits < best) best = bits, bp = p, bm = m;
      }
      ord_bits[o] = 8 + o * bpsc + (int)best;
      ord_pm[o] = bp | bm << 8;
    }
    __syncthreads();
    const int bp = ord_pm[o] & 0xff, bm = ord_pm[o] >> 8;
    for (int j = t; j < (1 << bp); j += THREADS) kord[o][j] = kbest[bm][(1 << bp) + j];
    __syncthreads();
  }
  __shared__ int pick;
  if (t == 0) {
    int bo = 0;
    for (int o = 1; o <= maxo; ++o)
      if (ord_bits[o] < ord_bits[bo]) bo = o;
    const int verbatim = 8 + bpsc * bs;
    if (ord_bits[bo] <= verbatim) {
      r[0] = ord_bits[bo];
      r[1] = FIXED | bo << 8 | (ord_pm[bo] & 0xff) << 16 | (ord_pm[bo] >> 8) << 24;
    } else {
      r[0] = verbatim, r[1] = VERBATIM;
    }
    pick = ord_bits[bo] <= verbatim ? bo : -1;
  }
  __syncthreads();
  if (pick >= 0) {
    unsigned char* kb = reinterpret_cast<unsigned char*>(r + 2);
    for (int j = t; j < (1 << (ord_pm[pick] & 0xff)); j += THREADS) kb[j] = kord[pick][j];
  }
}

// ORs the nb (0..32) low bits of v, MSB first, into the big-endian bit stream of the slot at bit pos.
__device__ __forceinline__ void put(unsigned* w, long long pos, unsigned v, int nb) {
  if (nb == 0) return;
  const unsigned long long x = (unsigned long long)v << (64 - (int)(pos & 31) - nb);
  atomicOr(w + (pos >> 5), __byte_perm((unsigned)(x >> 32), 0, 0x0123));
  if ((unsigned)x) atomicOr(w + (pos >> 5) + 1, __byte_perm((unsigned)x, 0, 0x0123));
}

// a b mod x^16 + x^15 + x^2 + 1 over GF(2).
__device__ unsigned gf_mul(unsigned a, unsigned b) {
  unsigned r = 0;
  for (int i = 15; i >= 0; --i) {
    r <<= 1;
    if (r & 0x10000) r ^= 0x18005;
    if (b >> i & 1) r ^= a;
  }
  return r;
}

__device__ unsigned x_pow(unsigned long long e) {     // x^e mod the CRC-16 polynomial
  unsigned r = 1, b = 2;
  for (; e; e >>= 1) {
    if (e & 1) r = gf_mul(r, b);
    b = gf_mul(b, b);
  }
  return r;
}

template <typename T>
__global__ void __launch_bounds__(THREADS) flac_emit_kernel(const T* __restrict__ pcm, long long cs, int n, int ch,
                                                            int bps, int rate, const int* __restrict__ rec,
                                                            unsigned char* __restrict__ data, long long cap,
                                                            long long* __restrict__ nbytes) {
  using Scan = cub::BlockScan<int, THREADS>;
  __shared__ typename Scan::TempStorage scan_tmp;
  __shared__ int x[BLOCK];
  __shared__ unsigned short tab[256];
  __shared__ int sub_cand[8], bad;
  __shared__ long long sub_off[9];
  __shared__ unsigned crc_part[THREADS / 32];
  const int nc = ch == 2 ? 4 : ch, t = threadIdx.x, frame = blockIdx.x;
  const long long clip = blockIdx.y, f = clip * gridDim.x + frame;
  const int start = frame * BLOCK, bs = min(BLOCK, n - start);
  const int* r0 = rec + f * nc * REC;
  unsigned* out = reinterpret_cast<unsigned*>(data + f * cap);
  {
    unsigned c = (unsigned)t << 8;
    for (int i = 0; i < 8; ++i) c = c & 0x8000 ? (c << 1) ^ 0x8005 : c << 1;
    tab[t] = (unsigned short)c;
  }
  const int nsub = ch;
  if (t == 0) {
    bad = 0;
    for (int c = 0; c < nc; ++c) bad |= r0[c * REC] < 0;
    int chan = ch - 1;
    for (int c = 0; c < ch; ++c) sub_cand[c] = c;
    if (ch == 2 && !bad) {
      const long long b[4] = {r0[0], r0[REC], r0[2 * REC], r0[3 * REC]};
      long long best = b[0] + b[1];
      if (b[0] + b[2] < best) best = b[0] + b[2], chan = 8, sub_cand[0] = 0, sub_cand[1] = 2;
      if (b[2] + b[1] < best) best = b[2] + b[1], chan = 9, sub_cand[0] = 2, sub_cand[1] = 1;
      if (b[3] + b[2] < best) best = b[3] + b[2], chan = 10, sub_cand[0] = 3, sub_cand[1] = 2;
    }
    unsigned char h[16];
    const int bcode = bs == BLOCK ? 12 : 7;
    int rcode;
    switch (rate) {
      case 8000: rcode = 4; break;
      case 16000: rcode = 5; break;
      case 22050: rcode = 6; break;
      case 24000: rcode = 7; break;
      case 32000: rcode = 8; break;
      case 44100: rcode = 9; break;
      case 48000: rcode = 10; break;
      default: rcode = rate % 1000 == 0 && rate / 1000 < 256 ? 12 : 13;
    }
    h[0] = 0xFF, h[1] = 0xF8, h[2] = (unsigned char)(bcode << 4 | rcode);
    h[3] = (unsigned char)(chan << 4 | (bps == 16 ? 4 : 6) << 1);
    int hl = 4;
    const unsigned fn = (unsigned)frame;
    if (fn < 0x80) {
      h[hl++] = (unsigned char)fn;
    } else {
      int nb = 2;
      while (fn >= 1u << (5 * nb + 1)) ++nb;
      h[hl++] = (unsigned char)((0xFF00 >> nb) & 0xFF | fn >> (6 * (nb - 1)));
      for (int i = nb - 2; i >= 0; --i) h[hl++] = (unsigned char)(0x80 | (fn >> (6 * i) & 0x3F));
    }
    if (bcode == 7) h[hl++] = (unsigned char)((bs - 1) >> 8), h[hl++] = (unsigned char)(bs - 1);
    if (rcode == 12) h[hl++] = (unsigned char)(rate / 1000);
    if (rcode == 13) h[hl++] = (unsigned char)(rate >> 8), h[hl++] = (unsigned char)rate;
    unsigned c8 = 0;
    for (int i = 0; i < hl; ++i) {
      c8 ^= h[i];
      for (int b = 0; b < 8; ++b) c8 = (c8 & 0x80 ? (c8 << 1) ^ 0x07 : c8 << 1) & 0xFF;
    }
    h[hl++] = (unsigned char)c8;
    if (!bad)
      for (int i = 0; i < hl; ++i) put(out, 8LL * i, h[i], 8);
    sub_off[0] = 8LL * hl;
    for (int c = 0; c < nsub; ++c) sub_off[c + 1] = sub_off[c] + r0[sub_cand[c] * REC];
  }
  __syncthreads();
  if (bad) {
    if (t == 0) nbytes[f] = -1;
    return;
  }
  const T* src = pcm + clip * cs + (long long)start * ch;
  for (int c = 0; c < nsub; ++c) {
    const int cand = sub_cand[c];
    const int* r = r0 + cand * REC;
    const int bpsc = ch == 2 && cand == 2 ? bps + 1 : bps;
    const unsigned mask = (1u << bpsc) - 1;
    load(x, src, bs, ch, cand, bps);
    __syncthreads();
    const long long pos = sub_off[c];
    const int type = r[1] & 0xff;
    if (type == CONSTANT) {
      if (t == 0) put(out, pos, 0, 8), put(out, pos + 8, (unsigned)x[0] & mask, bpsc);
    } else if (type == VERBATIM) {
      if (t == 0) put(out, pos, 2, 8);
      for (int i = t; i < bs; i += THREADS) put(out, pos + 8 + (long long)i * bpsc, (unsigned)x[i] & mask, bpsc);
    } else {
      const int o = r[1] >> 8 & 0xff, p = r[1] >> 16 & 0xff, m = r[1] >> 24;
      const unsigned char* kb = reinterpret_cast<const unsigned char*>(r + 2);
      const int plen = 4 + m, s = bs >> p;
      if (t == 0) {
        put(out, pos, (unsigned)(8 | o) << 1, 8);
        put(out, pos + 8 + o * bpsc, (unsigned)(m << 4 | p), 6);
        put(out, pos + 14 + o * bpsc, kb[0], plen);
      }
      if (t < o) put(out, pos + 8 + t * bpsc, (unsigned)x[t] & mask, bpsc);
      const int lo = max(t * PER, o), hi = min(t * PER + PER, bs);
      int len = 0;
      for (int i = lo; i < hi; ++i) {
        const int j = i / s, k = kb[j];
        len += (i % s == 0 && i > 0 ? plen : 0) + (int)(zigzag(residual(x, i, o)) >> k) + 1 + k;
      }
      int at;
      Scan(scan_tmp).ExclusiveSum(len, at);
      long long cur = pos + 14 + o * bpsc + plen + at;
      for (int i = lo; i < hi; ++i) {
        const int j = i / s, k = kb[j];
        if (i % s == 0 && i > 0) put(out, cur, k, plen), cur += plen;
        const unsigned u = zigzag(residual(x, i, o));
        put(out, cur + (u >> k), 1u << k | (u & ((1u << k) - 1)), k + 1);
        cur += (u >> k) + 1 + k;
      }
    }
    __syncthreads();
  }
  // CRC-16 over the frame: each thread's word-aligned chunk, moved to the end of the frame, XORed together
  const long long L = (sub_off[nsub] + 7) / 8;
  const long long chunk = ((L + THREADS - 1) / THREADS + 3) & ~3LL;
  const long long b0 = min(L, t * chunk), b1 = min(L, b0 + chunk);
  unsigned crc = 0;
  for (long long w = b0; w < b1; w += 4) {
    const unsigned word = __ldcg(out + (w >> 2));
    for (int i = 0; i < 4 && w + i < b1; ++i)
      crc = ((crc << 8) ^ tab[((crc >> 8) ^ (word >> (8 * i))) & 0xFF]) & 0xFFFF;
  }
  crc = b1 > b0 ? gf_mul(crc, x_pow(8 * (L - b1))) : 0;
  for (int d = 16; d; d >>= 1) crc ^= __shfl_xor_sync(0xffffffffu, crc, d);
  if ((t & 31) == 0) crc_part[t >> 5] = crc;
  __syncthreads();
  if (t == 0) {
    crc = crc_part[0];
    for (int w = 1; w < THREADS / 32; ++w) crc ^= crc_part[w];
    put(out, 8 * L, crc, 16);
    nbytes[f] = L + 2;
  }
}

long long frame_bound(int ch, int bps, int n) {        // 18 + ceil(C (8 + bps n) / 8)
  return 18 + ((long long)ch * (8 + (long long)bps * n) + 7) / 8;
}

bool args_ok(const void* pcm, long long cs, int batch, int n, int ch, int bps) {
  return pcm && batch >= 0 && batch <= 65535 && n >= 1 && ch >= 1 && ch <= 8 && (bps == 16 || bps == 24)
         && (batch <= 1 || cs >= (long long)n * ch);
}

}  // namespace

extern "C" int pm_flac_analyse(const void* pcm, long long clip_stride, int batch, int n, int channels, int bps,
                               int* rec, void* stream) {
  PM_REQUIRE(args_ok(pcm, clip_stride, batch, n, channels, bps) && rec);
  if (batch == 0) return PM_OK;
  const long long frames = (n + (long long)BLOCK - 1) / BLOCK;
  const long long blocks = frames * (channels == 2 ? 4 : channels);
  PM_REQUIRE(blocks < 0x7fffffffLL);
  const dim3 grid((unsigned)blocks, batch);
  if (bps == 16)
    flac_analyse_kernel<short><<<grid, THREADS, 0, (cudaStream_t)stream>>>(
        (const short*)pcm, clip_stride, n, channels, bps, rec);
  else
    flac_analyse_kernel<int><<<grid, THREADS, 0, (cudaStream_t)stream>>>(
        (const int*)pcm, clip_stride, n, channels, bps, rec);
  PM_LAUNCH_CHECK();
}

extern "C" int pm_flac_emit(const void* pcm, long long clip_stride, int batch, int n, int channels, int bps, int rate,
                            const int* rec, unsigned char* data, long long cap, long long* nbytes, void* stream) {
  PM_REQUIRE(args_ok(pcm, clip_stride, batch, n, channels, bps) && rec && data && nbytes && rate >= 1
             && rate <= 65535 && cap % 4 == 0 && cap >= frame_bound(channels, bps, n < BLOCK ? n : BLOCK)
             && ((unsigned long long)data & 3) == 0);
  if (batch == 0) return PM_OK;
  const long long frames = (n + (long long)BLOCK - 1) / BLOCK;
  const dim3 grid((unsigned)frames, batch);
  if (bps == 16)
    flac_emit_kernel<short><<<grid, THREADS, 0, (cudaStream_t)stream>>>(
        (const short*)pcm, clip_stride, n, channels, bps, rate, rec, data, cap, nbytes);
  else
    flac_emit_kernel<int><<<grid, THREADS, 0, (cudaStream_t)stream>>>(
        (const int*)pcm, clip_stride, n, channels, bps, rate, rec, data, cap, nbytes);
  PM_LAUNCH_CHECK();
}
