// H.264 encoding of RGB8 frames (pantomatrix_b200/video.py): one IDR access unit per frame by the rule of
// include/pm_emage.h and DESIGN.md section 12 (one I slice per macroblock row, Intra16x16 DC / Horizontal or I_PCM,
// CAVLC, deblocking off).  Two launches per call after the caller's memset of the output slots:
//   pm_h264_encode  one warp per (frame, macroblock row): the row's slice, emulation prevention applied, into its
//                   scratch slot, and the slice's size;
//   pm_h264_gather  one CTA per (frame, row): the slice's offset in the frame's sample, the copy, the frame's size.
// A warp stages its bits in shared memory in stream byte order (pm_put_bits, as FLAC writes its slots), so whole
// bytes leave the staging buffer as byte loads.
// CPU restatement: oracle/h264_oracle.py.  Every byte depends only on the frame, qp and its index parity.
#include <cub/block/block_reduce.cuh>

#include "pm_common.cuh"
#include "../../include/pm_emage.h"

namespace {

constexpr int WARPS = 4;                  // warps (slices) per CTA of pm_h264_encode
constexpr int MB_BITS_LIMIT = 3200;       // 128 + RawMbBits (A.3.1)
constexpr int SLICE_HEADER_BITS = 62;     // NAL header byte and the longest slice header
constexpr int STG_WORDS = 128;            // staging bits of one warp: header + one macroblock < 4096 bits
constexpr int GATHER_THREADS = 256;

// ---- CAVLC tables (ITU-T H.264 tables 9-5, 9-7, 9-8, 9-9a, 9-10): length << 8 | value ----
#define C(l, v) (unsigned short)((l) << 8 | (v))
__constant__ unsigned short CT[3][68] = {
    {C(1, 1), 0, 0, 0, C(6, 5), C(2, 1), 0, 0, C(8, 7), C(6, 4), C(3, 1), 0, C(9, 7), C(8, 6), C(7, 5), C(5, 3),
     C(10, 7), C(9, 6), C(8, 5), C(6, 3), C(11, 7), C(10, 6), C(9, 5), C(7, 4), C(13, 15), C(11, 6), C(10, 5), C(8, 4),
     C(13, 11), C(13, 14), C(11, 5), C(9, 4), C(13, 8), C(13, 10), C(13, 13), C(10, 4), C(14, 15), C(14, 14),
     C(13, 9), C(11, 4), C(14, 11), C(14, 10), C(14, 13), C(13, 12), C(15, 15), C(15, 14), C(14, 9), C(14, 12),
     C(15, 11), C(15, 10), C(15, 13), C(14, 8), C(16, 15), C(15, 1), C(15, 9), C(15, 12), C(16, 11), C(16, 14),
     C(16, 13), C(15, 8), C(16, 7), C(16, 10), C(16, 9), C(16, 12), C(16, 4), C(16, 6), C(16, 5), C(16, 8)},
    {C(2, 3), 0, 0, 0, C(6, 11), C(2, 2), 0, 0, C(6, 7), C(5, 7), C(3, 3), 0, C(7, 7), C(6, 10), C(6, 9), C(4, 5),
     C(8, 7), C(6, 6), C(6, 5), C(4, 4), C(8, 4), C(7, 6), C(7, 5), C(5, 6), C(9, 7), C(8, 6), C(8, 5), C(6, 8),
     C(11, 15), C(9, 6), C(9, 5), C(6, 4), C(11, 11), C(11, 14), C(11, 13), C(7, 4), C(12, 15), C(11, 10), C(11, 9),
     C(9, 4), C(12, 11), C(12, 14), C(12, 13), C(11, 12), C(12, 8), C(12, 10), C(12, 9), C(11, 8), C(13, 15),
     C(13, 14), C(13, 13), C(12, 12), C(13, 11), C(13, 10), C(13, 9), C(13, 12), C(13, 7), C(14, 11), C(13, 6),
     C(13, 8), C(14, 9), C(14, 8), C(14, 10), C(13, 1), C(14, 7), C(14, 6), C(14, 5), C(14, 4)},
    {C(4, 15), 0, 0, 0, C(6, 15), C(4, 14), 0, 0, C(6, 11), C(5, 15), C(4, 13), 0, C(6, 8), C(5, 12), C(5, 14),
     C(4, 12), C(7, 15), C(5, 10), C(5, 11), C(4, 11), C(7, 11), C(5, 8), C(5, 9), C(4, 10), C(7, 9), C(6, 14),
     C(6, 13), C(4, 9), C(7, 8), C(6, 10), C(6, 9), C(4, 8), C(8, 15), C(7, 14), C(7, 13), C(5, 13), C(8, 11),
     C(8, 14), C(7, 10), C(6, 12), C(9, 15), C(8, 10), C(8, 13), C(7, 12), C(9, 11), C(9, 14), C(8, 9), C(8, 12),
     C(9, 8), C(9, 10), C(9, 13), C(8, 8), C(10, 13), C(9, 7), C(9, 9), C(9, 12), C(10, 9), C(10, 12), C(10, 11),
     C(10, 10), C(10, 5), C(10, 8), C(10, 7), C(10, 6), C(10, 1), C(10, 4), C(10, 3), C(10, 2)}};
__constant__ unsigned short CDC_CT[20] = {C(2, 1), 0, 0, 0, C(6, 7), C(1, 1), 0, 0, C(6, 4), C(6, 6), C(3, 1), 0,
                                          C(6, 3), C(7, 3), C(7, 2), C(6, 5), C(6, 2), C(8, 3), C(8, 2), C(7, 0)};
__constant__ unsigned short TZ[15][16] = {
    {C(1, 1), C(3, 3), C(3, 2), C(4, 3), C(4, 2), C(5, 3), C(5, 2), C(6, 3), C(6, 2), C(7, 3), C(7, 2), C(8, 3),
     C(8, 2), C(9, 3), C(9, 2), C(9, 1)},
    {C(3, 7), C(3, 6), C(3, 5), C(3, 4), C(3, 3), C(4, 5), C(4, 4), C(4, 3), C(4, 2), C(5, 3), C(5, 2), C(6, 3),
     C(6, 2), C(6, 1), C(6, 0)},
    {C(4, 5), C(3, 7), C(3, 6), C(3, 5), C(4, 4), C(4, 3), C(3, 4), C(3, 3), C(4, 2), C(5, 3), C(5, 2), C(6, 1),
     C(5, 1), C(6, 0)},
    {C(5, 3), C(3, 7), C(4, 5), C(4, 4), C(3, 6), C(3, 5), C(3, 4), C(4, 3), C(3, 3), C(4, 2), C(5, 2), C(5, 1),
     C(5, 0)},
    {C(4, 5), C(4, 4), C(4, 3), C(3, 7), C(3, 6), C(3, 5), C(3, 4), C(3, 3), C(4, 2), C(5, 1), C(4, 1), C(5, 0)},
    {C(6, 1), C(5, 1), C(3, 7), C(3, 6), C(3, 5), C(3, 4), C(3, 3), C(3, 2), C(4, 1), C(3, 1), C(6, 0)},
    {C(6, 1), C(5, 1), C(3, 5), C(3, 4), C(3, 3), C(2, 3), C(3, 2), C(4, 1), C(3, 1), C(6, 0)},
    {C(6, 1), C(4, 1), C(5, 1), C(3, 3), C(2, 3), C(2, 2), C(3, 2), C(3, 1), C(6, 0)},
    {C(6, 1), C(6, 0), C(4, 1), C(2, 3), C(2, 2), C(3, 1), C(2, 1), C(5, 1)},
    {C(5, 1), C(5, 0), C(3, 1), C(2, 3), C(2, 2), C(2, 1), C(4, 1)},
    {C(4, 0), C(4, 1), C(3, 1), C(3, 2), C(1, 1), C(3, 3)},
    {C(4, 0), C(4, 1), C(2, 1), C(1, 1), C(3, 1)},
    {C(3, 0), C(3, 1), C(1, 1), C(2, 1)},
    {C(2, 0), C(2, 1), C(1, 1)},
    {C(1, 0), C(1, 1)}};
__constant__ unsigned short CDC_TZ[3][4] = {{C(1, 1), C(2, 1), C(3, 1), C(3, 0)}, {C(1, 1), C(2, 1), C(2, 0), 0},
                                            {C(1, 1), C(1, 0), 0, 0}};
__constant__ unsigned short RB[7][15] = {
    {C(1, 1), C(1, 0)},
    {C(1, 1), C(2, 1), C(2, 0)},
    {C(2, 3), C(2, 2), C(2, 1), C(2, 0)},
    {C(2, 3), C(2, 2), C(2, 1), C(3, 1), C(3, 0)},
    {C(2, 3), C(2, 2), C(3, 3), C(3, 2), C(3, 1), C(3, 0)},
    {C(2, 3), C(3, 0), C(3, 1), C(3, 3), C(3, 2), C(3, 5), C(3, 4)},
    {C(3, 7), C(3, 6), C(3, 5), C(3, 4), C(3, 3), C(3, 2), C(3, 1), C(4, 1), C(5, 1), C(6, 1), C(7, 1), C(8, 1),
     C(9, 1), C(10, 1), C(11, 1)}};
#undef C

// ---- transform and quantisation ----
__constant__ int ZZ[16] = {0, 1, 4, 8, 5, 2, 3, 6, 9, 12, 13, 10, 7, 11, 14, 15};   // scan index -> raster
__constant__ int MF[6][3] = {{13107, 5243, 8066}, {11916, 4660, 7490}, {10082, 4194, 6554},
                             {9362, 3647, 5825}, {8192, 3355, 5243}, {7282, 2893, 4559}};
__constant__ int VS[6][3] = {{10, 16, 13}, {11, 18, 14}, {13, 20, 16}, {14, 23, 18}, {16, 25, 20}, {18, 29, 23}};
__constant__ unsigned char QPC[52] = {0,  1,  2,  3,  4,  5,  6,  7,  8,  9,  10, 11, 12, 13, 14, 15, 16, 17,
                                      18, 19, 20, 21, 22, 23, 24, 25, 26, 27, 28, 29, 29, 30, 31, 32, 32, 33,
                                      34, 34, 35, 35, 36, 36, 37, 37, 37, 38, 38, 38, 39, 39, 39, 39};

__device__ __forceinline__ int pos_class(int raster) {
  const int r = raster >> 2, c = raster & 3;
  return ((r | c) & 1) == 0 ? 0 : ((r & c) & 1) ? 1 : 2;
}

// Bits of the warp's staging buffer, in stream byte order (pm_put_bits): stream byte i is byte i of the buffer, its
// bits MSB first.  WRITE false only counts them.
template <bool WRITE>
struct Bits {
  unsigned* stg;
  int pos;
  __device__ __forceinline__ void put(unsigned v, int n) {   // n <= 32, v < 2^n
    if (WRITE) pm_put_bits(stg, pos, v, n);
    pos += n;
  }
  __device__ __forceinline__ void code(unsigned short lv) { put(lv & 0xff, lv >> 8); }
  __device__ __forceinline__ void ue(unsigned k) {
    const int n = 32 - __clz(k + 1);
    put(k + 1, 2 * n - 1);
  }
  __device__ __forceinline__ void se(int k) { ue(k > 0 ? 2 * k - 1 : -2 * k); }
};

// CAVLC residual_block() of c[0, max_num) (scan order) with context nc (-1: chroma DC).  Returns false when a level
// needs a level_prefix above 15.
template <bool WRITE>
__device__ bool residual_block(Bits<WRITE>& b, const int* c, int max_num, int nc) {
  int total = 0, last = -1;
  for (int i = 0; i < max_num; ++i)
    if (c[i]) { ++total; last = i; }
  int t1 = 0;
  {
    int seen = 0;
    for (int i = last; i >= 0 && seen < 3 && t1 == seen; --i)
      if (c[i]) {
        ++seen;
        if (abs(c[i]) == 1) ++t1;
      }
  }
  if (nc == -1) b.code(CDC_CT[4 * total + t1]);
  else if (nc >= 8) b.put(total ? (unsigned)((total - 1) << 2 | t1) : 3u, 6);
  else b.code(CT[nc < 2 ? 0 : (nc < 4 ? 1 : 2)][4 * total + t1]);
  if (total == 0) return true;
  int suffix = (total > 10 && t1 < 3) ? 1 : 0;
  int k = 0;                                              // levels coded so far, highest frequency first
  for (int i = last; i >= 0; --i) {
    const int lv = c[i];
    if (!lv) continue;
    if (k < t1) b.put(lv < 0, 1);
    else {
      int code = lv > 0 ? 2 * lv - 2 : -2 * lv - 1;
      if (k == t1 && t1 < 3) code -= 2;
      int prefix, sfx, size;
      if (suffix == 0) {
        if (code < 14) { prefix = code; sfx = 0; size = 0; }
        else if (code < 30) { prefix = 14; sfx = code - 14; size = 4; }
        else { prefix = 15; sfx = code - 30; size = 12; }
      } else if (code < (15 << suffix)) {
        prefix = code >> suffix; sfx = code & ((1 << suffix) - 1); size = suffix;
      } else {
        prefix = 15; sfx = code - (15 << suffix); size = 12;
      }
      if (sfx >= 4096) return false;
      b.put(1, prefix + 1);
      b.put(sfx, size);
      if (suffix == 0) suffix = 1;
      if (abs(lv) > (3 << (suffix - 1)) && suffix < 6) ++suffix;
    }
    ++k;
  }
  if (total < max_num) {
    const int tz = last + 1 - total;
    if (nc == -1) b.code(CDC_TZ[total - 1][tz]);
    else b.code(TZ[total - 1][tz]);
    int left = tz, seen = 0;
    for (int i = last; i >= 0 && left > 0 && seen < total - 1; --i) {
      if (!c[i]) continue;
      int j = i - 1;
      while (j >= 0 && !c[j]) --j;
      const int run = i - 1 - j;
      b.code(RB[min(left, 7) - 1][run]);
      left -= run;
      ++seen;
    }
  }
  return true;
}

// 4x4 forward core transform of x (raster), in place: rows, then columns.
__device__ __forceinline__ void fdct(int* x) {
#pragma unroll
  for (int r = 0; r < 4; ++r) {
    int* p = x + 4 * r;
    const int s0 = p[0] + p[3], s1 = p[1] + p[2], d0 = p[0] - p[3], d1 = p[1] - p[2];
    p[0] = s0 + s1; p[2] = s0 - s1; p[1] = 2 * d0 + d1; p[3] = d0 - 2 * d1;
  }
#pragma unroll
  for (int c = 0; c < 4; ++c) {
    const int a = x[c], b = x[4 + c], e = x[8 + c], g = x[12 + c];
    const int s0 = a + g, s1 = b + e, d0 = a - g, d1 = b - e;
    x[c] = s0 + s1; x[8 + c] = s0 - s1; x[4 + c] = 2 * d0 + d1; x[12 + c] = d0 - 2 * d1;
  }
}

// 8.5.12.2: rows (horizontal) first, then columns, then (x + 32) >> 6.
__device__ __forceinline__ void idct(int* d) {
#pragma unroll
  for (int r = 0; r < 4; ++r) {
    int* p = d + 4 * r;
    const int e0 = p[0] + p[2], e1 = p[0] - p[2], e2 = (p[1] >> 1) - p[3], e3 = p[1] + (p[3] >> 1);
    p[0] = e0 + e3; p[1] = e1 + e2; p[2] = e1 - e2; p[3] = e0 - e3;
  }
#pragma unroll
  for (int c = 0; c < 4; ++c) {
    const int a = d[c], b = d[4 + c], e = d[8 + c], g = d[12 + c];
    const int e0 = a + e, e1 = a - e, e2 = (b >> 1) - g, e3 = b + (g >> 1);
    d[c] = (e0 + e3 + 32) >> 6; d[4 + c] = (e1 + e2 + 32) >> 6; d[8 + c] = (e1 - e2 + 32) >> 6;
    d[12 + c] = (e0 - e3 + 32) >> 6;
  }
}

__device__ __forceinline__ int quant(int w, int mf, int f, int qbits) {
  const int q = (abs(w) * mf + f) >> qbits;
  return w < 0 ? -q : q;
}

// One warp's state.  Units of a macroblock_layer(), in syntax order: 0 header, 1 luma DC, 2..17 luma AC by
// luma4x4BlkIdx, 18 / 19 chroma DC Cb / Cr, 20..27 chroma AC Cb 0..3, Cr 0..3; lev[u - 1] holds unit u's levels.
struct Warp {
  unsigned stg[STG_WORDS];
  int lev[27][16];
  int dcw[16], cdcw[2][4];                 // DC of each block's forward transform (raster)
  int dcy[16], dcc[2][4];                  // scaled DC (8.5.10, 8.5.11.1)
  int tc[24];                              // TotalCoeff of the AC blocks: luma raster 0..15, chroma 16 + 4 k + raster
  int ly[16], lc[2][8];                    // left neighbour: reconstructed right column
  int ny[16], nc[2][8];                    // this macroblock's Intra16x16 right column
  int lnz[8];                              // left neighbour's right blocks' TotalCoeff: luma rows, Cb rows, Cr rows
  unsigned char y[256], cb[64], cr[64];    // source samples
};

__device__ __forceinline__ unsigned stg_byte(const unsigned* stg, int i) {
  return reinterpret_cast<const unsigned char*>(stg)[i];
}

// Append staging bytes [0, nb) to out + at with emulation prevention; zrun: zero bytes ending the output so far
// (0..2).  32 bytes per step; inside a step each insertion is found in turn with ballots.  Returns the new `at`.
__device__ long long flush_bytes(const unsigned* stg, int nb, unsigned char* out, long long at, int& zrun, int lane) {
  for (int base = 0; base < nb; base += 32) {
    const int cnt = min(32, nb - base);
    const bool valid = lane < cnt;
    const unsigned b = valid ? stg_byte(stg, base + lane) : 0xffu;
    const unsigned z = __ballot_sync(0xffffffffu, valid && b == 0);
    const unsigned below = lane ? (0xffffffffu >> (32 - lane)) : 0u;
    int start = 0, carry = zrun;
    unsigned epb = 0;
    for (;;) {
      const unsigned nz = (~z | (start ? (0xffffffffu >> (32 - start)) : 0u)) & below;
      const int run = nz ? lane - 1 - (31 - __clz(nz)) : lane + carry;
      const unsigned cand = __ballot_sync(0xffffffffu, valid && lane >= start && b <= 3 && run >= 2);
      if (!cand) break;
      start = __ffs(cand) - 1;
      epb |= 1u << start;
      carry = 0;
    }
    const int shift = __popc(epb & (lane == 31 ? 0xffffffffu : ((2u << lane) - 1)));
    if (valid) {
      out[at + lane + shift] = (unsigned char)b;
      if ((epb >> lane) & 1) out[at + lane + shift - 1] = 3;
    }
    at += cnt + __popc(epb);
    // zero bytes ending this step's output
    const unsigned upto = cnt == 32 ? 0xffffffffu : ((1u << cnt) - 1);
    const unsigned nz = (~z | (start ? (0xffffffffu >> (32 - start)) : 0u)) & upto;
    zrun = min(2, nz ? cnt - 1 - (31 - __clz(nz)) : cnt + carry);
  }
  return at;
}

__device__ __forceinline__ int warp_sum(int v) {
#pragma unroll
  for (int o = 16; o; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

struct Job {
  const unsigned char* px;   // frame 0, pixel (0, 0)
  long long fs;              // frame stride (bytes)
  int n_frames, clip_len, h, w, qp;
  unsigned char* scratch;
  long long slice_cap;
  int* slice_bytes;
};

__device__ __forceinline__ void rgb(const unsigned char* p, int& r, int& g, int& b) { r = p[0]; g = p[1]; b = p[2]; }

__global__ void __launch_bounds__(32 * WARPS) h264_encode_kernel(Job J) {
  __shared__ Warp WS[WARPS];
  const int lane = threadIdx.x & 31;
  Warp& S = WS[threadIdx.x >> 5];
  const int mbw = J.w >> 4, mbh = J.h >> 4;
  const long long slice = (long long)blockIdx.x * WARPS + (threadIdx.x >> 5);
  if (slice >= (long long)J.n_frames * mbh) return;
  const long long f = slice / mbh;
  const int my = (int)(slice % mbh);
  const unsigned char* fr = J.px + f * J.fs;
  const int qp = J.qp, qpc = QPC[qp];
  unsigned char* out = J.scratch + slice * J.slice_cap;
  long long at = 4;                                      // the 4-byte length prefix goes first
  int zrun = 0;

  for (int i = lane; i < STG_WORDS; i += 32) S.stg[i] = 0;
  __syncwarp();
  int pend;                                              // bits in the staging buffer
  {
    Bits<true> b{S.stg, 0};
    if (lane == 0) {
      b.put(0x65, 8);                                    // nal_ref_idc 3, nal_unit_type 5 (IDR)
      b.ue((unsigned)(my * mbw));                        // first_mb_in_slice
      b.ue(7);                                           // slice_type I (every slice of the picture)
      b.ue(0);                                           // pic_parameter_set_id
      b.put(0, 4);                                       // frame_num
      b.ue((unsigned)((f % J.clip_len) & 1));            // idr_pic_id
      b.put(0, 2);                                       // no_output_of_prior_pics_flag, long_term_reference_flag
      b.se(qp - 26);                                     // slice_qp_delta
      b.ue(1);                                           // disable_deblocking_filter_idc
    }
    pend = __shfl_sync(0xffffffffu, b.pos, 0);
  }

  const int mf0 = MF[qp % 6][0], qbits = 15 + qp / 6, fq = (1 << qbits) / 3;
  const int cmf0 = MF[qpc % 6][0], cqbits = 15 + qpc / 6, cfq = (1 << cqbits) / 3;

  for (int mx = 0; mx < mbw; ++mx) {
    const bool have_left = mx > 0;
    // ---- source samples (colour rule) ----
    for (int p = lane; p < 256; p += 32) {
      int r, g, bb;
      rgb(fr + ((long long)(16 * my + (p >> 4)) * J.w + 16 * mx + (p & 15)) * 3, r, g, bb);
      S.y[p] = (unsigned char)(((66 * r + 129 * g + 25 * bb + 128) >> 8) + 16);
    }
    for (int p = lane; p < 64; p += 32) {
      const int yy = 16 * my + 2 * (p >> 3), xx = 16 * mx + 2 * (p & 7);
      int rs = 0, gs = 0, bs = 0;
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        int r, g, bb;
        rgb(fr + ((long long)(yy + (q >> 1)) * J.w + xx + (q & 1)) * 3, r, g, bb);
        rs += r; gs += g; bs += bb;
      }
      S.cb[p] = (unsigned char)(((-38 * rs - 74 * gs + 112 * bs + 512) >> 10) + 128);
      S.cr[p] = (unsigned char)(((112 * rs - 94 * gs - 18 * bs + 512) >> 10) + 128);
    }
    __syncwarp();
    // ---- prediction: DC, or Horizontal when its SAD is strictly lower ----
    int dc = 128;
    if (have_left) {
      int s = 0;
#pragma unroll
      for (int r = 0; r < 16; ++r) s += S.ly[r];
      dc = (s + 8) >> 4;
    }
    int sad_dc = 0, sad_h = 0;
    for (int p = lane; p < 256; p += 32) {
      sad_dc += abs((int)S.y[p] - dc);
      if (have_left) sad_h += abs((int)S.y[p] - S.ly[p >> 4]);
    }
    sad_dc = warp_sum(sad_dc);
    sad_h = warp_sum(sad_h);
    const bool use_h = have_left && sad_h < sad_dc;
    int cp[2][2];
#pragma unroll
    for (int k = 0; k < 2; ++k)
#pragma unroll
      for (int hy = 0; hy < 2; ++hy)
        cp[k][hy] = have_left ? (S.lc[k][4 * hy] + S.lc[k][4 * hy + 1] + S.lc[k][4 * hy + 2] + S.lc[k][4 * hy + 3]
                                 + 2) >> 2
                              : 128;
    // ---- forward transform and AC quantisation: lanes 0..15 luma blocks, 16..23 chroma blocks (raster) ----
    if (lane < 24) {
      const bool luma = lane < 16;
      const int k = luma ? 0 : (lane - 16) >> 2, bi = luma ? lane : (lane - 16) & 3;
      const int by = luma ? bi >> 2 : bi >> 1, bx = luma ? bi & 3 : bi & 1;
      int x[16];
#pragma unroll
      for (int i = 0; i < 16; ++i) {
        const int r = 4 * by + (i >> 2), c = 4 * bx + (i & 3);
        if (luma) x[i] = (int)S.y[16 * r + c] - (use_h ? S.ly[r] : dc);
        else x[i] = (int)(k ? S.cr : S.cb)[8 * r + c] - cp[k][by];
      }
      fdct(x);
      const int unit = luma ? 2 + ((by >> 1) << 3) + ((bx >> 1) << 2) + ((by & 1) << 1) + (bx & 1)
                            : 20 + 4 * k + bi;
      const int q = luma ? qp : qpc;
      const int qb = 15 + q / 6, fr3 = (1 << qb) / 3;
      int total = 0;
#pragma unroll
      for (int s = 1; s < 16; ++s) {
        const int rz = ZZ[s];
        const int l = quant(x[rz], MF[q % 6][pos_class(rz)], fr3, qb);
        S.lev[unit - 1][s - 1] = l;
        total += l != 0;
      }
      S.tc[lane] = total;
      if (luma) S.dcw[bi] = x[0];
      else S.cdcw[k][bi] = x[0];
    }
    __syncwarp();
    // ---- DC paths: lane 0 luma (4x4 Hadamard), lanes 1 / 2 chroma Cb / Cr (2x2 Hadamard) ----
    bool cdc_nz = false;
    if (lane == 0) {
      int d[16];
#pragma unroll
      for (int i = 0; i < 16; ++i) d[i] = S.dcw[i];
      // H d H with H = [[1,1,1,1],[1,1,-1,-1],[1,-1,-1,1],[1,-1,1,-1]]: columns, then rows (exact, so any order)
#pragma unroll
      for (int pass = 0; pass < 2; ++pass)
#pragma unroll
        for (int a = 0; a < 4; ++a) {
          const int st = pass ? 1 : 4, o = pass ? 4 * a : a;
          const int v0 = d[o], v1 = d[o + st], v2 = d[o + 2 * st], v3 = d[o + 3 * st];
          d[o] = v0 + v1 + v2 + v3; d[o + st] = v0 + v1 - v2 - v3;
          d[o + 2 * st] = v0 - v1 - v2 + v3; d[o + 3 * st] = v0 - v1 + v2 - v3;
        }
      int z[16];
#pragma unroll
      for (int i = 0; i < 16; ++i) {
        const int q = ((abs(d[i]) >> 1) * mf0 + 2 * fq) >> (qbits + 1);
        z[i] = d[i] < 0 ? -q : q;
      }
#pragma unroll
      for (int s = 0; s < 16; ++s) S.lev[0][s] = z[ZZ[s]];
      // 8.5.10: f = H z H, then scaled with LevelScale(qp % 6, 0, 0) = 16 v0
#pragma unroll
      for (int pass = 0; pass < 2; ++pass)
#pragma unroll
        for (int a = 0; a < 4; ++a) {
          const int st = pass ? 1 : 4, o = pass ? 4 * a : a;
          const int v0 = z[o], v1 = z[o + st], v2 = z[o + 2 * st], v3 = z[o + 3 * st];
          z[o] = v0 + v1 + v2 + v3; z[o + st] = v0 + v1 - v2 - v3;
          z[o + 2 * st] = v0 - v1 - v2 + v3; z[o + 3 * st] = v0 - v1 + v2 - v3;
        }
      const int ls = 16 * VS[qp % 6][0];
#pragma unroll
      for (int i = 0; i < 16; ++i)
        S.dcy[i] = qp >= 36 ? (z[i] * ls) << (qp / 6 - 6) : (z[i] * ls + (1 << (5 - qp / 6))) >> (6 - qp / 6);
    } else if (lane <= 2) {
      const int k = lane - 1;
      const int a = S.cdcw[k][0], b = S.cdcw[k][1], c = S.cdcw[k][2], e = S.cdcw[k][3];
      const int d[4] = {a + b + c + e, a - b + c - e, a + b - c - e, a - b - c + e};
      int z[4];
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        z[i] = quant(d[i], cmf0, 2 * cfq, cqbits + 1);
        S.lev[17 + k][i] = z[i];
        cdc_nz |= z[i] != 0;
      }
      const int g[4] = {z[0] + z[1] + z[2] + z[3], z[0] - z[1] + z[2] - z[3], z[0] + z[1] - z[2] - z[3],
                        z[0] - z[1] - z[2] + z[3]};
      const int ls = 16 * VS[qpc % 6][0];
#pragma unroll
      for (int i = 0; i < 4; ++i) S.dcc[k][i] = ((g[i] * ls) << (qpc / 6)) >> 5;
    }
    const bool cbp_l = __ballot_sync(0xffffffffu, lane < 16 && S.tc[lane] > 0) != 0;
    const bool ac_c = __ballot_sync(0xffffffffu, lane >= 16 && lane < 24 && S.tc[lane] > 0) != 0;
    const bool dc_c = __ballot_sync(0xffffffffu, cdc_nz) != 0;
    const int cbp_c = ac_c ? 2 : (dc_c ? 1 : 0);
    __syncwarp();
    // ---- reconstruction of the right column: luma blocks with bx = 3, chroma blocks with bx = 1 ----
    if ((lane < 16 && (lane & 3) == 3) || (lane >= 16 && lane < 24 && (lane & 1) == 1)) {
      const bool luma = lane < 16;
      const int k = luma ? 0 : (lane - 16) >> 2, bi = luma ? lane : (lane - 16) & 3;
      const int by = luma ? bi >> 2 : bi >> 1, bx = luma ? 3 : 1;
      const int unit = luma ? 2 + ((by >> 1) << 3) + ((bx >> 1) << 2) + ((by & 1) << 1) + (bx & 1)
                            : 20 + 4 * k + bi;
      const int q = luma ? qp : qpc;
      int d[16];
      d[0] = luma ? S.dcy[bi] : S.dcc[k][bi];
#pragma unroll
      for (int s = 1; s < 16; ++s) {
        const int rz = ZZ[s];
        const int c = S.lev[unit - 1][s - 1], ls = 16 * VS[q % 6][pos_class(rz)];
        d[rz] = q >= 24 ? (c * ls) << (q / 6 - 4) : (c * ls + (1 << (3 - q / 6))) >> (4 - q / 6);
      }
      idct(d);
#pragma unroll
      for (int r = 0; r < 4; ++r) {
        const int row = 4 * by + r;
        const int pred = luma ? (use_h ? S.ly[row] : dc) : cp[k][by];
        const int v = min(255, max(0, pred + d[4 * r + 3]));
        if (luma) S.ny[row] = v;
        else S.nc[k][row] = v;
      }
    }
    // ---- macroblock_layer() bits per unit, then the I_PCM decision ----
    auto unit_bits = [&](auto& b) -> bool {
      const int u = lane;
      if (u == 0) {
        b.ue((unsigned)(1 + (use_h ? 1 : 2) + 4 * cbp_c + (cbp_l ? 12 : 0)));
        b.ue(0);                                         // intra_chroma_pred_mode: DC
        b.se(0);                                         // mb_qp_delta
        return true;
      }
      if (u == 1) return residual_block(b, S.lev[0], 16, have_left ? S.lnz[0] : 0);
      if (u < 18) {
        if (!cbp_l) return true;
        const int blk = u - 2;
        const int by = ((blk >> 3) << 1) | ((blk >> 1) & 1), bx = (((blk >> 2) & 1) << 1) | (blk & 1);
        const bool ha = bx > 0 || have_left, hb = by > 0;
        const int na = bx > 0 ? S.tc[4 * by + bx - 1] : (have_left ? S.lnz[by] : 0);
        const int nb = hb ? S.tc[4 * (by - 1) + bx] : 0;
        const int nc = ha && hb ? (na + nb + 1) >> 1 : (ha ? na : nb);
        return residual_block(b, S.lev[u - 1], 15, nc);
      }
      if (u < 20) return cbp_c ? residual_block(b, S.lev[u - 1], 4, -1) : true;
      if (u < 28) {
        if (cbp_c != 2) return true;
        const int k = (u - 20) >> 2, bi = (u - 20) & 3, by = bi >> 1, bx = bi & 1;
        const bool ha = bx > 0 || have_left, hb = by > 0;
        const int na = bx > 0 ? S.tc[16 + 4 * k + 2 * by] : (have_left ? S.lnz[4 + 2 * k + by] : 0);
        const int nb = hb ? S.tc[16 + 4 * k + bx] : 0;
        const int nc = ha && hb ? (na + nb + 1) >> 1 : (ha ? na : nb);
        return residual_block(b, S.lev[u - 1], 15, nc);
      }
      return true;
    };
    Bits<false> cnt{nullptr, 0};
    const bool ok = unit_bits(cnt);
    int excl = cnt.pos;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const int v = __shfl_up_sync(0xffffffffu, excl, o);
      if (lane >= o) excl += v;
    }
    const int mb_bits = __shfl_sync(0xffffffffu, excl, 31);
    excl -= cnt.pos;
    const bool pcm = __ballot_sync(0xffffffffu, !ok) != 0 || mb_bits > MB_BITS_LIMIT;
    int end;
    if (!pcm) {
      Bits<true> b{S.stg, pend + excl};
      unit_bits(b);
      end = pend + mb_bits;
    } else {
      if (lane == 0) {
        Bits<true> b{S.stg, pend};
        b.ue(25);                                        // I_PCM, then pcm_alignment_zero_bits
      }
      const int at8 = (pend + 9 + 7) >> 3;
      __syncwarp();
      for (int i = lane; i < 384; i += 32) {
        const int j = at8 + i;
        const unsigned v = i < 256 ? S.y[i] : (i < 320 ? S.cb[i - 256] : S.cr[i - 320]);
        atomicOr(S.stg + (j >> 2), v << (8 * (j & 3)));
      }
      end = 8 * (at8 + 384);
    }
    __syncwarp();
    // ---- whole bytes out, the partial byte stays ----
    at = flush_bytes(S.stg, end >> 3, out, at, zrun, lane);
    const unsigned keep = (end & 7) ? stg_byte(S.stg, end >> 3) : 0u;
    __syncwarp();
    for (int i = lane; i <= (end >> 5) && i < STG_WORDS; i += 32) S.stg[i] = 0;
    __syncwarp();
    if (lane == 0) S.stg[0] = keep;
    pend = end & 7;
    // ---- the left neighbour of the next macroblock ----
    if (lane < 16) {
      const int k = lane >> 3, r = lane & 7;
      S.ly[lane] = pcm ? S.y[16 * lane + 15] : S.ny[lane];
      S.lc[k][r] = pcm ? (k ? S.cr : S.cb)[8 * r + 7] : S.nc[k][r];
    }
    if (lane < 8) {
      int v;
      if (pcm) v = 16;
      else if (lane < 4) v = S.tc[4 * lane + 3];
      else {
        const int k = (lane - 4) >> 1, by = (lane - 4) & 1;
        v = S.tc[16 + 4 * k + 2 * by + 1];
      }
      S.lnz[lane] = v;
    }
    __syncwarp();
  }
  // ---- rbsp_slice_trailing_bits, the last bytes, the length prefix ----
  if (lane == 0) {
    Bits<true> b{S.stg, pend};
    b.put(1, 1);
  }
  __syncwarp();
  at = flush_bytes(S.stg, (pend + 1 + 7) >> 3, out, at, zrun, lane);
  if (lane == 0) {
    const long long len = at - 4;
    out[0] = (unsigned char)(len >> 24); out[1] = (unsigned char)(len >> 16);
    out[2] = (unsigned char)(len >> 8); out[3] = (unsigned char)len;
    J.slice_bytes[slice] = (int)at;
  }
}

__global__ void __launch_bounds__(GATHER_THREADS) h264_gather_kernel(int mbh, const unsigned char* __restrict__ scratch,
                                                                     long long slice_cap,
                                                                     const int* __restrict__ slice_bytes,
                                                                     unsigned char* __restrict__ data, long long cap,
                                                                     long long* __restrict__ nbytes) {
  using Sum = cub::BlockReduce<long long, GATHER_THREADS>;
  __shared__ typename Sum::TempStorage tmp;
  __shared__ long long off_s;
  const long long f = blockIdx.y;
  const int r = blockIdx.x;
  const int* sz = slice_bytes + f * mbh;
  long long mine = 0;
  for (int i = threadIdx.x; i < r; i += GATHER_THREADS) mine += sz[i];
  const long long off = Sum(tmp).Sum(mine);
  if (threadIdx.x == 0) {
    off_s = off;
    if (r == mbh - 1) nbytes[f] = off + sz[r];
  }
  __syncthreads();
  const long long o = off_s;
  const unsigned char* src = scratch + (f * mbh + r) * slice_cap;
  unsigned char* dst = data + f * cap + o;
  for (int i = threadIdx.x; i < sz[r]; i += GATHER_THREADS) dst[i] = src[i];
}

long long slice_bound(int w) {
  const long long p = (SLICE_HEADER_BITS + (long long)MB_BITS_LIMIT * (w / 16) + 8 + 7) / 8;
  return 4 + p + p / 2;
}

bool shape_ok(int frames, int h, int w) {
  if (frames < 0 || h < 16 || w < 16 || h % 16 || w % 16) return false;
  const long long mbh = h / 16, mbw = w / 16;
  return mbh * mbw <= 36864 && mbh <= 543 && mbw <= 543;
}

}  // namespace

extern "C" int pm_h264_encode(const unsigned char* frames, long long f_fs, int n_frames, int clip_len, int h, int w,
                              int qp, unsigned char* scratch, long long slice_cap, int* slice_bytes, void* stream) {
  PM_REQUIRE(shape_ok(n_frames, h, w) && frames && scratch && slice_bytes && f_fs >= 3LL * w * h && clip_len >= 1
             && qp >= 0 && qp <= 51 && slice_cap >= slice_bound(w));
  const long long slices = (long long)n_frames * (h / 16);
  if (slices == 0) return PM_OK;
  PM_REQUIRE(slices / WARPS < 0x7fffffffLL);
  h264_encode_kernel<<<(unsigned)((slices + WARPS - 1) / WARPS), 32 * WARPS, 0, (cudaStream_t)stream>>>(
      Job{frames, f_fs, n_frames, clip_len, h, w, qp, scratch, slice_cap, slice_bytes});
  PM_LAUNCH_CHECK();
}

extern "C" int pm_h264_gather(int n_frames, int h, int w, const unsigned char* scratch, long long slice_cap,
                              const int* slice_bytes, unsigned char* data, long long cap, long long* nbytes,
                              void* stream) {
  PM_REQUIRE(shape_ok(n_frames, h, w) && scratch && slice_bytes && data && nbytes && slice_cap >= slice_bound(w)
             && cap >= (h / 16) * slice_bound(w));
  if (n_frames == 0) return PM_OK;
  PM_REQUIRE(n_frames <= 65535);
  h264_gather_kernel<<<dim3(h / 16, n_frames), GATHER_THREADS, 0, (cudaStream_t)stream>>>(
      h / 16, scratch, slice_cap, slice_bytes, data, cap, nbytes);
  PM_LAUNCH_CHECK();
}
