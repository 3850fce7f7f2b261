// H.264 encoding of RGB8 frames (pantomatrix_b200/video.py): one access unit per frame by the rule of
// include/pm_emage.h and DESIGN.md section 12 (one slice per macroblock row, Intra16x16 DC / Horizontal or I_PCM,
// CAVLC, deblocking off; with a keyframe interval gop > 1, P frames of P_Skip and zero-motion inter macroblocks
// between the IDR frames, or with a motion search range, quarter-pel vectors against the whole previous frame; with
// PM_H264_I4X4 in qp, Intra 4x4 (I_NxN) macroblocks beside Intra16x16 in I and P slices).  Two
// launches per call after the caller's memset of the output slots (pm_h264_encode_me: 2 gop - 1 encode launches,
// h264_search_kernel before each P frame's):
//   pm_h264_encode  one warp per (frame, macroblock row): the row's slice, emulation prevention applied, into its
//                   scratch slot, and the slice's size; pm_h264_encode_gop: one warp per (GOP, row), walking the
//                   GOP's frames in order;
//   pm_h264_gather  one CTA per (frame, row): the slice's offset in the frame's sample, the copy, the frame's size.
// A warp stages its bits in shared memory in stream byte order (pm_put_bits, as FLAC writes its slots), so whole
// bytes leave the staging buffer as byte loads.
// CPU restatement: oracle/h264_oracle.py for the intra rule, tests/h264_ref.py for P frames, motion and Intra 4x4.
// Every byte depends only on the frame (its GOP's frames), qp, gop, search, the
// Intra 4x4 switch and the parity of its index (t div gop).
#include <cub/block/block_reduce.cuh>

#include <type_traits>

#include "pm_common.cuh"
#include "../../include/pm_emage.h"

namespace {

constexpr int WARPS = 4;                  // warps (slices) per CTA of pm_h264_encode
constexpr int MB_BITS_LIMIT = 3200;       // 128 + RawMbBits (A.3.1)
constexpr int SLICE_HEADER_BITS = 62;     // NAL header byte and the slice header, as the gop = 1 bound counts it
constexpr int SLICE_HEADER_BITS_GOP = 70; // the longest slice header of either kind: IDR, last row, qp 0
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

// Table 9-4 (ChromaArrayType 1): codeNum of each coded_block_pattern of an Inter macroblock.
__constant__ unsigned char INTER_CODE[48] = {0,  2,  3,  7,  4,  8,  17, 13, 5,  18, 9,  14, 10, 15, 16, 11,
                                             1,  32, 33, 36, 34, 37, 44, 40, 35, 45, 38, 41, 39, 42, 43, 19,
                                             6,  24, 25, 20, 26, 21, 46, 28, 27, 47, 22, 29, 23, 30, 31, 12};

// The reference samples of a P frame's macroblock: the co-located samples of the previous reconstruction.
struct WarpRef {
  unsigned char ry[256], rc[2][64];
  __device__ __forceinline__ int ref(int k, int i) const { return k < 0 ? ry[i] : rc[k][i]; }
};
struct WarpNoRef {
  __device__ __forceinline__ int ref(int, int) const { return 0; }
};

// One warp's state.  Units of a macroblock_layer(), in syntax order: 0 header, 1 luma DC, 2..17 luma AC by
// luma4x4BlkIdx, 18 / 19 chroma DC Cb / Cr, 20..27 chroma AC Cb 0..3, Cr 0..3; lev[u - 1] holds unit u's levels.  An
// inter macroblock has no unit 1, and its luma units 2..17 hold all 16 levels of their block.
template <bool GOP>
struct Warp : std::conditional_t<GOP, WarpRef, WarpNoRef> {
  unsigned stg[STG_WORDS];
  int lev[27][16];
  int dcw[16], cdcw[2][4];                 // DC of each block's forward transform (raster)
  int dcy[16], dcc[2][4];                  // scaled DC (8.5.10, 8.5.11.1)
  int tc[24];                              // TotalCoeff of the AC blocks: luma raster 0..15, chroma 16 + 4 k + raster
  int ly[16], lc[2][8];                    // left neighbour: reconstructed right column
  int ny[16], nc[2][8];                    // this macroblock's reconstructed right column
  int lnz[8];                              // left neighbour's right blocks' TotalCoeff: luma rows, Cb rows, Cr rows
  unsigned char y[256], cb[64], cr[64];    // source samples
};
// The I4 instances' warp state: the I_NxN candidate beside the others.
template <bool GOP>
struct WarpI4 : Warp<GOP> {
  int lev4[16][16];                        // each block's 16 levels (luma4x4BlkIdx, scan order)
  int tc4[16];                             // each block's TotalCoeff (raster)
  int j4[18];                              // J of each (block of the step, mode)
  unsigned char rec4[256];                 // the candidate's luma reconstruction
  unsigned char m4[16], pm4[16];           // each block's mode and predIntra4x4PredMode (raster)
  unsigned char lm4[4];                    // the left macroblock's right blocks' modes; 2 when it is not I_NxN
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

__device__ __forceinline__ int ue_bits(unsigned k) { return 2 * (32 - __clz(k + 1)) - 1; }

struct Job {
  const unsigned char* px;   // frame 0, pixel (0, 0)
  long long fs;              // frame stride (bytes)
  int n_frames, clip_len, h, w, qp;
  unsigned char* scratch;
  long long slice_cap;
  int* slice_bytes;
  int gop, chains_per_clip;  // GOP: frames per GOP, GOPs per clip
  unsigned char* recon;      // GOP: one macroblock row's reconstruction per (chain, row), recon_stride apart; ME: two
  long long recon_stride;    // whole-frame reconstructions per chain (frame k in buffer k & 1), recon_stride apart
  int k, search;             // ME: the frame of each chain this launch codes (or searches), the search range
  short2* mv;                // ME: frame k's vector per (chain, macroblock), quarter-pel
};

// The kernel's three instances: every frame IDR; GOPs with zero motion, a warp walking its GOP's frames; GOPs with
// motion search, one launch per frame of the GOPs (h264_search_kernel before each P frame's).
enum Mode { INTRA, GOP_ZERO, GOP_ME };

__constant__ unsigned char LAMBDA[52] = {0,  0,  0,  0,  0,  0,  0,  1,  1,  1,  1,  1,  1,  1,  1,  1,  1,  2,
                                         2,  2,  2,  3,  3,  3,  4,  4,  5,  5,  6,  7,  7,  8,  9,  10, 12, 13,
                                         15, 17, 19, 21, 23, 26, 30, 33, 37, 42, 47, 53, 59, 66, 74, 83};

// Table 9-4 (ChromaArrayType 1): codeNum of each coded_block_pattern of an Intra_4x4 macroblock.
__constant__ unsigned char INTRA_CODE[48] = {3,  29, 30, 17, 31, 18, 37, 8,  32, 38, 19, 9,  20, 10, 11, 2,
                                             16, 33, 34, 21, 35, 22, 39, 4,  36, 40, 23, 5,  24, 6,  7,  1,
                                             41, 42, 43, 25, 44, 26, 46, 12, 45, 47, 27, 13, 28, 14, 15, 0};

// ---- Intra 4x4 (8.3.1.2) ----
// A block's neighbours as one edge E[0..12]: p[-1, 3..0], p[-1, -1], p[0..7, -1].  Each sample of modes 0, 1, 3..8 is
// kind << 4 | c: kind 0 E[c], 1 (E[c] + E[c + 1] + 1) >> 1, 2 (E[c - 1] + 2 E[c] + E[c + 1] + 2) >> 2 with the
// indices clamped to 0..12 (which gives Diagonal_Down_Left's (3, 3) and Horizontal_Up's zHU = 5); raster order.
__constant__ unsigned char PRED4[9][16] = {
    {0x05, 0x06, 0x07, 0x08, 0x05, 0x06, 0x07, 0x08, 0x05, 0x06, 0x07, 0x08, 0x05, 0x06, 0x07, 0x08},
    {0x03, 0x03, 0x03, 0x03, 0x02, 0x02, 0x02, 0x02, 0x01, 0x01, 0x01, 0x01, 0x00, 0x00, 0x00, 0x00},
    {0},
    {0x26, 0x27, 0x28, 0x29, 0x27, 0x28, 0x29, 0x2a, 0x28, 0x29, 0x2a, 0x2b, 0x29, 0x2a, 0x2b, 0x2c},
    {0x24, 0x25, 0x26, 0x27, 0x23, 0x24, 0x25, 0x26, 0x22, 0x23, 0x24, 0x25, 0x21, 0x22, 0x23, 0x24},
    {0x14, 0x15, 0x16, 0x17, 0x24, 0x25, 0x26, 0x27, 0x23, 0x14, 0x15, 0x16, 0x22, 0x24, 0x25, 0x26},
    {0x13, 0x24, 0x25, 0x26, 0x12, 0x23, 0x13, 0x24, 0x11, 0x22, 0x12, 0x23, 0x10, 0x21, 0x11, 0x22},
    {0x15, 0x16, 0x17, 0x18, 0x26, 0x27, 0x28, 0x29, 0x16, 0x17, 0x18, 0x19, 0x27, 0x28, 0x29, 0x2a},
    {0x12, 0x22, 0x11, 0x21, 0x11, 0x21, 0x10, 0x20, 0x10, 0x20, 0x00, 0x00, 0x00, 0x00, 0x00, 0x00}};
// The 10 wavefront steps of a macroblock's blocks (raster, -1 none): a block follows its left, above-left, above and
// above-right neighbours, so step bx + 2 by holds every block that can go.
__constant__ signed char WAVE[10][2] = {{0, -1}, {1, -1}, {2, 4}, {3, 5}, {6, 8}, {7, 9}, {10, 12}, {11, 13},
                                        {14, -1}, {15, -1}};
constexpr unsigned AR_AVAIL = 0x5750;      // raster blocks whose above-right block is coded before them (6.4.11.4)
// luma4x4BlkIdx -> raster block, and (being its own inverse) raster -> luma4x4BlkIdx
__constant__ unsigned char BLK_RASTER[16] = {0, 1, 4, 5, 2, 3, 6, 7, 8, 9, 12, 13, 10, 11, 14, 15};
__constant__ unsigned char SCAN_OF[16] = {0, 1, 5, 6, 2, 4, 7, 12, 3, 8, 11, 13, 9, 10, 14, 15};   // raster -> scan
constexpr int C_I4 = 6;                    // an I_NxN macroblock's J4 is charged C_I4 lambda(qp) more (pm_emage.h)

__device__ __forceinline__ int se_bits(int v) { return ue_bits(v > 0 ? 2 * v - 1 : -2 * v); }

__device__ __forceinline__ int clip255(int v) { return min(255, max(0, v)); }

// 8.4.2.2.1: the luma prediction sample at quarter-pel phase (fx, fy) of the integer sample G = at(0, 0); at(dx, dy)
// reads the reference at an offset from G (clipped to the frame by the caller).  b, h, m, s: the half-pel samples
// right of G, below G, below G's right neighbour and right of G's lower neighbour; j from unrounded intermediates;
// the quarter-pel samples are rounded averages of the two nearest.
template <class At>
__device__ __forceinline__ int luma_pred(const At& at, int fx, int fy) {
  auto tap = [](int a, int b, int c, int d, int e, int f) { return a - 5 * b + 20 * c + 20 * d - 5 * e + f; };
  auto row1 = [&](int r) { return tap(at(-2, r), at(-1, r), at(0, r), at(1, r), at(2, r), at(3, r)); };
  auto col1 = [&](int c) { return tap(at(c, -2), at(c, -1), at(c, 0), at(c, 1), at(c, 2), at(c, 3)); };
  auto half = [](int v) { return clip255((v + 16) >> 5); };
  if (fy == 0) {
    if (fx == 0) return at(0, 0);
    const int b = half(row1(0));
    return fx == 2 ? b : (b + at(fx >> 1, 0) + 1) >> 1;                      // a, b, c
  }
  if (fx == 0) {
    const int h = half(col1(0));
    return fy == 2 ? h : (h + at(0, fy >> 1) + 1) >> 1;                      // d, h, n
  }
  if (fx == 2 || fy == 2) {
    const int j = clip255((tap(row1(-2), row1(-1), row1(0), row1(1), row1(2), row1(3)) + 512) >> 10);
    if (fx == 2 && fy == 2) return j;
    const int o = fx == 2 ? half(row1(fy >> 1)) : half(col1(fx >> 1));      // f / q: b / s; i / k: h / m
    return (j + o + 1) >> 1;
  }
  return (half(row1(fy >> 1)) + half(col1(fx >> 1)) + 1) >> 1;              // e, g, p, r
}

// 8.4.2.2.2: the chroma prediction sample at eighth-pel phase (fx, fy) between A = at(0, 0), B, C, D.
template <class At>
__device__ __forceinline__ int chroma_pred(const At& at, int fx, int fy) {
  return ((8 - fx) * (8 - fy) * at(0, 0) + fx * (8 - fy) * at(1, 0) + (8 - fx) * fy * at(0, 1) + fx * fy * at(1, 1)
          + 32) >> 6;
}

__device__ __forceinline__ void rgb(const unsigned char* p, int& r, int& g, int& b) { r = p[0]; g = p[1]; b = p[2]; }

// One warp per (chain, macroblock row).  A chain is one frame (INTRA: every frame IDR) or one GOP of one clip.
// GOP_ZERO: the warp codes the row of each of the chain's frames in turn, the IDR frame first, and keeps the row's
// reconstruction in J.recon for the next frame's P slice.  GOP_ME: the warp codes the row of the chain's frame J.k
// only, against the whole reconstruction of frame k - 1, with the vectors h264_search_kernel chose, and writes frame
// k's reconstruction to the other buffer; kernel boundaries order the frames.  I4: each coded macroblock also gets
// the I_NxN candidate, its blocks in 10 wavefront steps (lanes per (block, mode) for the costs, one per block for the
// transform), the candidate's luma reconstruction in shared memory.
// (The I4 instances ask for one CTA per SM at least, which lets the GOP_ZERO one keep its state in registers; the bound
// is 0, no request, for the others.)
template <Mode MODE, bool I4>
__global__ void __launch_bounds__(32 * WARPS, I4 ? 1 : 0) h264_encode_kernel(Job J) {
  constexpr bool GOP = MODE != INTRA, ME = MODE == GOP_ME;
  using W = std::conditional_t<I4, WarpI4<GOP>, Warp<GOP>>;
  __shared__ W WS[WARPS];
  const int lane = threadIdx.x & 31;
  W& S = WS[threadIdx.x >> 5];
  const int mbw = J.w >> 4, mbh = J.h >> 4;
  const long long slice = (long long)blockIdx.x * WARPS + (threadIdx.x >> 5);
  const long long chains = GOP ? (long long)(J.n_frames / J.clip_len) * J.chains_per_clip : J.n_frames;
  if (slice >= chains * mbh) return;
  const long long chain = slice / mbh;
  const int my = (int)(slice % mbh);
  long long f0;                                          // the chain's first frame, at index t0 of its clip
  int t0, t1;
  if (GOP) {
    t0 = (int)(chain % J.chains_per_clip) * J.gop;
    t1 = min(t0 + J.gop, J.clip_len);
    f0 = chain / J.chains_per_clip * J.clip_len + t0;
  } else {
    f0 = chain;
    t0 = (int)(chain % J.clip_len);
    t1 = t0 + 1;
  }
  if (ME && t0 + J.k >= t1) return;                     // a last GOP shorter than gop
  // GOP_ZERO: the row's reconstruction (Y 16 x w, Cb, Cr 8 x w / 2), read and updated in place.  GOP_ME: frame k's
  // reconstruction (Y h x w, Cb, Cr h / 2 x w / 2) is written to rrow, frame k - 1's read from rref.
  const long long fsz = 3LL * J.h * J.w / 2;
  unsigned char* const rrow = ME ? J.recon + chain * J.recon_stride + (J.k & 1) * fsz
                                 : (GOP ? J.recon + slice * J.recon_stride : nullptr);
  const unsigned char* const rref = ME ? J.recon + chain * J.recon_stride + ((J.k + 1) & 1) * fsz : rrow;
  // offsets in rrow / rref of luma (row, col) and chroma k (row, col) of macroblock mx of the row
  auto yo = [&](int row, int mx, int col) -> long long {
    if constexpr (ME) return (long long)(16 * my + row) * J.w + 16 * mx + col;
    else return row * J.w + 16 * mx + col;
  };
  auto co = [&](int k, int row, int mx, int col) -> long long {
    if constexpr (ME)
      return (long long)J.h * J.w + k * ((long long)J.h * J.w >> 2) + (long long)(8 * my + row) * (J.w >> 1) + 8 * mx
             + col;
    else return 16 * J.w + k * 4 * J.w + row * (J.w >> 1) + 8 * mx + col;
  };
  const int qp = J.qp, qpc = QPC[qp];
  const int mf0 = MF[qp % 6][0], qbits = 15 + qp / 6, fq = (1 << qbits) / 3;
  const int cmf0 = MF[qpc % 6][0], cqbits = 15 + qpc / 6, cfq = (1 << cqbits) / 3;

  for (int t = ME ? t0 + J.k : t0; t < t1; ++t) {
    const long long f = f0 + (t - t0);
    const bool pf = GOP && t > t0;                       // a P frame: every frame of a GOP after its IDR frame
    const unsigned char* fr = J.px + f * J.fs;
    const long long row = GOP ? f * mbh + my : slice;    // this slice's index in scratch and slice_bytes
    unsigned char* out = J.scratch + row * J.slice_cap;
    long long at = 4;                                      // the 4-byte length prefix goes first
    int zrun = 0;

    for (int i = lane; i < STG_WORDS; i += 32) S.stg[i] = 0;
    __syncwarp();
    int pend;                                              // bits in the staging buffer
    {
      Bits<true> b{S.stg, 0};
      if (lane == 0) {
        if (pf) {
          b.put(0x41, 8);                                  // nal_ref_idc 2, nal_unit_type 1 (non-IDR)
          b.ue((unsigned)(my * mbw));                      // first_mb_in_slice
          b.ue(5);                                         // slice_type P (every slice of the picture)
          b.ue(0);                                         // pic_parameter_set_id
          b.put((t - t0) & 15, 4);                         // frame_num = (t mod gop) mod 16
          b.put(0, 3);                                     // num_ref_idx_active_override_flag,
                                                           // ref_pic_list_modification_flag_l0,
                                                           // adaptive_ref_pic_marking_mode_flag
        } else {
          b.put(0x65, 8);                                  // nal_ref_idc 3, nal_unit_type 5 (IDR)
          b.ue((unsigned)(my * mbw));                      // first_mb_in_slice
          b.ue(7);                                         // slice_type I (every slice of the picture)
          b.ue(0);                                         // pic_parameter_set_id
          b.put(0, 4);                                     // frame_num
          b.ue((unsigned)((GOP ? t / J.gop : t) & 1));               // idr_pic_id
          b.put(0, 2);                                     // no_output_of_prior_pics_flag, long_term_reference_flag
        }
        b.se(qp - 26);                                     // slice_qp_delta
        b.ue(1);                                           // disable_deblocking_filter_idc
      }
      pend = __shfl_sync(0xffffffffu, b.pos, 0);
    }
    int run = 0;                                           // P_Skip macroblocks since the last coded one
    short2 lmv = make_short2(0, 0);                        // ME: the vector predictor, the left P_L0_16x16's vector

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
      if constexpr (GOP) {
        if (pf) {
          // (the GOP_ZERO instance keeps its own address arithmetic: sharing yo / co costs it spills)
          for (int p = lane; p < 256; p += 32)
            S.ry[p] = ME ? rref[yo(p >> 4, mx, p & 15)] : rrow[(p >> 4) * J.w + 16 * mx + (p & 15)];
          for (int p = lane; p < 128; p += 32) {
            const int k = p >> 6, q = p & 63;
            S.rc[k][q] = ME ? rref[co(k, q >> 3, mx, q & 7)]
                            : rrow[16 * J.w + k * 4 * J.w + (q >> 3) * (J.w >> 1) + 8 * mx + (q & 7)];
          }
        }
      }
      __syncwarp();
      int dc = 128;
      bool use_h = false;
      // the chroma DC prediction of rows 4 hy .. 4 hy + 3 of component k
      auto cpred = [&](int k, int hy) {
        return have_left ? (S.lc[k][4 * hy] + S.lc[k][4 * hy + 1] + S.lc[k][4 * hy + 2] + S.lc[k][4 * hy + 3] + 2) >> 2
                         : 128;
      };
      // ---- forward transform and AC quantisation: lanes 0..15 luma blocks, 16..23 chroma blocks (raster); then the
      // DC paths: lane 0 luma (4x4 Hadamard, intra only), lanes 1 / 2 chroma Cb / Cr (2x2 Hadamard).  An inter
      // macroblock transforms source - reference, quantises all 16 luma levels, and rounds with f = 2^qbits / 6. ----
      auto transform = [&](bool inter) -> bool {
        if (lane < 24) {
          const bool luma = lane < 16;
          const int k = luma ? 0 : (lane - 16) >> 2, bi = luma ? lane : (lane - 16) & 3;
          const int by = luma ? bi >> 2 : bi >> 1, bx = luma ? bi & 3 : bi & 1;
          int x[16];
#pragma unroll
          for (int i = 0; i < 16; ++i) {
            const int r = 4 * by + (i >> 2), c = 4 * bx + (i & 3);
            if (luma) x[i] = (int)S.y[16 * r + c] - (inter ? S.ref(-1, 16 * r + c) : (use_h ? S.ly[r] : dc));
            else x[i] = (int)(k ? S.cr : S.cb)[8 * r + c] - (inter ? S.ref(k, 8 * r + c) : cpred(k, by));
          }
          fdct(x);
          const int unit = luma ? 2 + ((by >> 1) << 3) + ((bx >> 1) << 2) + ((by & 1) << 1) + (bx & 1)
                                : 20 + 4 * k + bi;
          const int q = luma ? qp : qpc;
          const int qb = 15 + q / 6, fr3 = (1 << qb) / (inter ? 6 : 3);
          const bool all16 = inter && luma;
          int total = 0;
#pragma unroll
          for (int s = 0; s < 16; ++s) {
            if (s == 0 && !all16) continue;
            const int rz = ZZ[s];
            const int l = quant(x[rz], MF[q % 6][pos_class(rz)], fr3, qb);
            S.lev[unit - 1][all16 ? s : s - 1] = l;
            total += l != 0;
          }
          S.tc[lane] = total;
          if (luma) S.dcw[bi] = x[0];
          else S.cdcw[k][bi] = x[0];
        }
        __syncwarp();
        bool cdc_nz = false;
        if (lane == 0 && !inter) {
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
        } else if (lane >= 1 && lane <= 2) {
          const int k = lane - 1;
          const int a = S.cdcw[k][0], b = S.cdcw[k][1], c = S.cdcw[k][2], e = S.cdcw[k][3];
          const int d[4] = {a + b + c + e, a - b + c - e, a + b - c - e, a - b - c + e};
          const int cf = inter ? (1 << cqbits) / 6 : cfq;
          int z[4];
#pragma unroll
          for (int i = 0; i < 4; ++i) {
            z[i] = quant(d[i], cmf0, 2 * cf, cqbits + 1);
            S.lev[17 + k][i] = z[i];
            cdc_nz |= z[i] != 0;
          }
          const int g[4] = {z[0] + z[1] + z[2] + z[3], z[0] - z[1] + z[2] - z[3], z[0] + z[1] - z[2] - z[3],
                            z[0] - z[1] - z[2] + z[3]};
          const int ls = 16 * VS[qpc % 6][0];
#pragma unroll
          for (int i = 0; i < 4; ++i) S.dcc[k][i] = ((g[i] * ls) << (qpc / 6)) >> 5;
        }
        return cdc_nz;
      };
      // ---- P frames: the zero-motion inter candidate; P_Skip when all its levels are zero ----
      bool cdc_nz = false;
      short2 mv = make_short2(0, 0);
      if (pf) {
        cdc_nz = transform(true);
        if (!__ballot_sync(0xffffffffu, (lane < 24 && S.tc[lane] > 0) || cdc_nz)) {
          ++run;
          if constexpr (ME) {                              // the reconstruction is the reference
            for (int p = lane; p < 256; p += 32) rrow[yo(p >> 4, mx, p & 15)] = S.ry[p];
            for (int p = lane; p < 128; p += 32) {
              const int k = p >> 6, q = p & 63;
              rrow[co(k, q >> 3, mx, q & 7)] = S.rc[k][q];
            }
            lmv = make_short2(0, 0);
          }
          // GOP_ZERO: the reconstruction is the reference, already in J.recon; the next macroblock's left neighbour
          if (lane < 16) {
            const int k = lane >> 3, r = lane & 7;
            S.ly[lane] = S.ref(-1, 16 * lane + 15);
            S.lc[k][r] = S.ref(k, 8 * r + 7);
          }
          if (lane < 8) S.lnz[lane] = 0;
          if constexpr (I4) {
            if (lane < 4) S.lm4[lane] = 2;
          }
          __syncwarp();
          continue;
        }
        if constexpr (ME) {                                // the inter candidate at the searched vector
          mv = J.mv[(chain * mbh + my) * mbw + mx];
          if (mv.x | mv.y) {
            __syncwarp();
            const int w = J.w, h = J.h;
            for (int p = lane; p < 256; p += 32) {
              const int xi = 16 * mx + (p & 15) + (mv.x >> 2), yi = 16 * my + (p >> 4) + (mv.y >> 2);
              S.ry[p] = (unsigned char)luma_pred([&](int dx, int dy) {
                return (int)rref[(long long)min(h - 1, max(0, yi + dy)) * w + min(w - 1, max(0, xi + dx))];
              }, mv.x & 3, mv.y & 3);
            }
            for (int p = lane; p < 128; p += 32) {
              const int k = p >> 6, q = p & 63;
              const int xi = 8 * mx + (q & 7) + (mv.x >> 3), yi = 8 * my + (q >> 3) + (mv.y >> 3);
              const unsigned char* pl = rref + (long long)h * w + k * ((long long)h * w >> 2);
              S.rc[k][q] = (unsigned char)chroma_pred([&](int dx, int dy) {
                return (int)pl[(long long)min((h >> 1) - 1, max(0, yi + dy)) * (w >> 1)
                               + min((w >> 1) - 1, max(0, xi + dx))];
              }, mv.x & 7, mv.y & 7);
            }
            __syncwarp();
            cdc_nz = transform(true);
          }
        }
      }
      // ---- Intra16x16 prediction: DC, or Horizontal when its SAD is strictly lower ----
      if (have_left) {
        int s = 0;
#pragma unroll
        for (int r = 0; r < 16; ++r) s += S.ly[r];
        dc = (s + 8) >> 4;
      }
      int sad_dc = 0, sad_h = 0, sad_p = 0;
      for (int p = lane; p < 256; p += 32) {
        sad_dc += abs((int)S.y[p] - dc);
        if (have_left) sad_h += abs((int)S.y[p] - S.ly[p >> 4]);
        if (pf) sad_p += abs((int)S.y[p] - S.ref(-1, p));
      }
      sad_dc = warp_sum(sad_dc);
      sad_h = warp_sum(sad_h);
      use_h = have_left && sad_h < sad_dc;
      int j_intra = 0;                                     // I4: the intra candidate's cost
      bool nxn = false;                                    // I4: the I_NxN candidate is the intra choice
      if constexpr (I4) {
        // ---- the I_NxN candidate: per wavefront step, lane 9 s + m costs mode m of the step's block s, then lane s
        // transforms, quantises and reconstructs block s by its lowest-J mode ----
        const int lam = LAMBDA[qp];
        int jsum = 0;
        for (int step = 0; step < 10; ++step) {
          const int slot = lane / 9, m = lane - 9 * slot;
          const int blk = slot < 2 ? WAVE[step][slot] : -1;
          const int bx = blk & 3, by = blk >> 2, X = 4 * bx, Y = 4 * by;
          const bool la = bx > 0 || have_left, ua = by > 0, ar = (AR_AVAIL >> blk) & 1;
          // E[c] of the block's edge (clamped to 0..12); only the samples its candidate modes read
          auto edge = [&](int c) -> int {
            c = min(12, max(0, c));
            if (c < 5) return bx ? S.rec4[(Y + 3 - c) * 16 + X - 1] : S.ly[Y + 3 - c];
            const int x = c > 8 && !ar ? 3 : c - 5;
            return S.rec4[(Y - 1) * 16 + X + x];
          };
          auto pred = [&](int mode, int i, int dc) -> int {
            if (mode == 2) return dc;
            const int t = PRED4[mode][i], c = t & 15;
            if (t >> 4 == 0) return edge(c);
            if (t >> 4 == 1) return (edge(c) + edge(c + 1) + 1) >> 1;
            return (edge(c - 1) + 2 * edge(c) + edge(c + 1) + 2) >> 2;
          };
          auto dc_of = [&]() -> int {
            int sa = 0, sl = 0;
#pragma unroll
            for (int i = 0; i < 4; ++i) {
              if (ua) sa += edge(5 + i);
              if (la) sl += edge(3 - i);
            }
            return la && ua ? (sa + sl + 4) >> 3 : (la ? (sl + 2) >> 2 : (ua ? (sa + 2) >> 2 : 128));
          };
          if (blk >= 0) {
            // 8.3.1.1: DC when the block to the left or above is not available; a left macroblock not I_NxN counts as 2
            const int pm = la && ua ? min(bx ? (int)S.m4[blk - 1] : (int)S.lm4[by], (int)S.m4[blk - 4]) : 2;
            const bool cand = m == 2 || (m == 0 || m == 3 || m == 7 ? ua : (m == 1 || m == 8 ? la : la && ua));
            int j = 0x7fffffff;
            if (cand) {
              const int dc = m == 2 ? dc_of() : 0;
              int sad = 0;
#pragma unroll 4
              for (int i = 0; i < 16; ++i) sad += abs((int)S.y[(Y + (i >> 2)) * 16 + X + (i & 3)] - pred(m, i, dc));
              j = sad + lam * (m == pm ? 1 : 4);
            }
            S.j4[lane] = j;
            if (m == 0) S.pm4[blk] = (unsigned char)pm;
          }
          __syncwarp();
          if (blk >= 0 && m == 0) {                        // lanes 0 and 9: the step's blocks
            int best = 0, bj = S.j4[lane];
#pragma unroll
            for (int k = 1; k < 9; ++k)
              if (S.j4[lane + k] < bj) { bj = S.j4[lane + k]; best = k; }
            jsum += bj;
            S.m4[blk] = (unsigned char)best;
            const int dc = best == 2 ? dc_of() : 0;
            int x[16];
#pragma unroll
            for (int i = 0; i < 16; ++i) x[i] = (int)S.y[(Y + (i >> 2)) * 16 + X + (i & 3)] - pred(best, i, dc);
            fdct(x);
            const int b16 = BLK_RASTER[blk];
            int total = 0;
#pragma unroll
            for (int i = 0; i < 16; ++i) {
              const int l = quant(x[i], MF[qp % 6][pos_class(i)], fq, qbits);
              S.lev4[b16][SCAN_OF[i]] = l;
              total += l != 0;
              const int ls = 16 * VS[qp % 6][pos_class(i)];
              x[i] = qp >= 24 ? (l * ls) << (qp / 6 - 4) : (l * ls + (1 << (3 - qp / 6))) >> (4 - qp / 6);
            }
            S.tc4[blk] = total;
            idct(x);
#pragma unroll
            for (int i = 0; i < 16; ++i)
              S.rec4[(Y + (i >> 2)) * 16 + X + (i & 3)] = (unsigned char)min(255, max(0, pred(best, i, dc) + x[i]));
          }
          __syncwarp();
        }
        const int j4 = warp_sum(jsum) + C_I4 * lam;
        nxn = j4 < (use_h ? sad_h : sad_dc);
        j_intra = nxn ? j4 : (use_h ? sad_h : sad_dc);
      }
      // inter when the inter candidate's luma SAD is at most the intra candidate's cost
      const bool inter = pf && warp_sum(sad_p) <= (I4 ? j_intra : (use_h ? sad_h : sad_dc));
      if (I4 && inter) nxn = false;
      if (!inter) cdc_nz = transform(false);
      if constexpr (I4) {
        if (nxn) {                                         // the I_NxN luma levels replace the Intra16x16 ones
          __syncwarp();
          if (lane < 16) {
            const int b16 = BLK_RASTER[lane];
#pragma unroll
            for (int s = 0; s < 16; ++s) S.lev[1 + b16][s] = S.lev4[b16][s];
            S.tc[lane] = S.tc4[lane];
          }
          __syncwarp();
        }
      }
      const bool cbp_l = __ballot_sync(0xffffffffu, lane < 16 && S.tc[lane] > 0) != 0;
      const bool ac_c = __ballot_sync(0xffffffffu, lane >= 16 && lane < 24 && S.tc[lane] > 0) != 0;
      const bool dc_c = __ballot_sync(0xffffffffu, cdc_nz) != 0;
      const int cbp_c = ac_c ? 2 : (dc_c ? 1 : 0);
      // an inter macroblock's CodedBlockPatternLuma: bit b8 when a 4x4 block of 8x8 block b8 has a level
      int cbp8 = 0;
      if (inter || (I4 && nxn))
        cbp8 = (int)__reduce_or_sync(0xffffffffu, lane < 16 && S.tc[lane] > 0
                                                      ? 1u << (((lane >> 3) << 1) | ((lane & 3) >> 1)) : 0u);
      __syncwarp();
      // ---- reconstruction: GOP every block into J.recon, else the right column (luma bx = 3, chroma bx = 1); an
      // I_NxN macroblock's luma is the candidate's ----
      if constexpr (I4) {
        if (nxn) {
          for (int p = lane; p < 256; p += 32) {
            const int v = S.rec4[p];
            if constexpr (ME) rrow[yo(p >> 4, mx, p & 15)] = (unsigned char)v;
            else if constexpr (GOP) rrow[(p >> 4) * J.w + 16 * mx + (p & 15)] = (unsigned char)v;
            if ((p & 15) == 15) S.ny[p >> 4] = v;
          }
        }
      }
      if ((GOP ? lane < 24 : ((lane < 16 && (lane & 3) == 3) || (lane >= 16 && lane < 24 && (lane & 1) == 1)))
          && !(I4 && nxn && lane < 16)) {
        const bool luma = lane < 16;
        const int k = luma ? 0 : (lane - 16) >> 2, bi = luma ? lane : (lane - 16) & 3;
        const int by = luma ? bi >> 2 : bi >> 1, bx = GOP ? (luma ? bi & 3 : bi & 1) : (luma ? 3 : 1);
        const int unit = luma ? 2 + ((by >> 1) << 3) + ((bx >> 1) << 2) + ((by & 1) << 1) + (bx & 1)
                              : 20 + 4 * k + bi;
        const int q = luma ? qp : qpc;
        const bool all16 = inter && luma;
        int d[16];
        d[0] = luma ? S.dcy[bi] : S.dcc[k][bi];
#pragma unroll
        for (int s = 0; s < 16; ++s) {
          if (s == 0 && !all16) continue;
          const int rz = ZZ[s];
          const int c = S.lev[unit - 1][all16 ? s : s - 1], ls = 16 * VS[q % 6][pos_class(rz)];
          d[rz] = q >= 24 ? (c * ls) << (q / 6 - 4) : (c * ls + (1 << (3 - q / 6))) >> (4 - q / 6);
        }
        idct(d);
        const bool right = bx == (luma ? 3 : 1);
        if constexpr (GOP) {
#pragma unroll
          for (int r = 0; r < 4; ++r)
#pragma unroll
            for (int c = 0; c < 4; ++c) {
              const int row = 4 * by + r, col = 4 * bx + c;
              const int pred = inter ? (luma ? S.ref(-1, 16 * row + col) : S.ref(k, 8 * row + col))
                                     : (luma ? (use_h ? S.ly[row] : dc) : cpred(k, by));
              const int v = min(255, max(0, pred + d[4 * r + c]));
              if constexpr (ME) {
                if (luma) rrow[yo(row, mx, col)] = (unsigned char)v;
                else rrow[co(k, row, mx, col)] = (unsigned char)v;
              } else {
                if (luma) rrow[row * J.w + 16 * mx + col] = (unsigned char)v;
                else rrow[16 * J.w + k * 4 * J.w + row * (J.w >> 1) + 8 * mx + col] = (unsigned char)v;
              }
              if (right && c == 3) {
                if (luma) S.ny[row] = v;
                else S.nc[k][row] = v;
              }
            }
        } else {
#pragma unroll
          for (int r = 0; r < 4; ++r) {
            const int row = 4 * by + r;
            const int pred = luma ? (use_h ? S.ly[row] : dc) : cpred(k, by);
            const int v = min(255, max(0, pred + d[4 * r + 3]));
            if (luma) S.ny[row] = v;
            else S.nc[k][row] = v;
          }
        }
      }
      // ---- macroblock_layer() bits per unit, then the I_PCM decision ----
      auto unit_bits = [&](auto& b) -> bool {
        const int u = lane;
        if (u == 0) {
          if (inter) {
            b.ue(0);                                       // mb_type P_L0_16x16
            b.se(ME ? mv.x - lmv.x : 0);                   // mvd_l0; GOP_ZERO: (0, 0), the predictor is (0, 0)
            b.se(ME ? mv.y - lmv.y : 0);
            b.ue(INTER_CODE[cbp8 | cbp_c << 4]);           // coded_block_pattern
            if (cbp8 | cbp_c) b.se(0);                     // mb_qp_delta
          } else if (I4 && nxn) {
            if constexpr (I4) {
              b.ue(pf ? 5 : 0);                            // mb_type I_NxN
              for (int k = 0; k < 16; ++k) {               // luma4x4BlkIdx order
                const int r = BLK_RASTER[k], m = S.m4[r], pm = S.pm4[r];
                if (m == pm) b.put(1, 1);                  // prev_intra4x4_pred_mode_flag
                else b.put((unsigned)(m < pm ? m : m - 1), 4);   // 0, rem_intra4x4_pred_mode
              }
              b.ue(0);                                     // intra_chroma_pred_mode: DC
              b.ue(INTRA_CODE[cbp8 | cbp_c << 4]);         // coded_block_pattern
              if (cbp8 | cbp_c) b.se(0);                   // mb_qp_delta
            }
          } else {
            b.ue((unsigned)((pf ? 5 : 0) + 1 + (use_h ? 1 : 2) + 4 * cbp_c + (cbp_l ? 12 : 0)));
            b.ue(0);                                       // intra_chroma_pred_mode: DC
            b.se(0);                                       // mb_qp_delta
          }
          return true;
        }
        if (u == 1) return inter || (I4 && nxn) || residual_block(b, S.lev[0], 16, have_left ? S.lnz[0] : 0);
        if (u < 18) {
          const int blk = u - 2;
          if (inter || (I4 && nxn) ? !((cbp8 >> (blk >> 2)) & 1) : !cbp_l) return true;
          const int by = ((blk >> 3) << 1) | ((blk >> 1) & 1), bx = (((blk >> 2) & 1) << 1) | (blk & 1);
          const bool ha = bx > 0 || have_left, hb = by > 0;
          const int na = bx > 0 ? S.tc[4 * by + bx - 1] : (have_left ? S.lnz[by] : 0);
          const int nb = hb ? S.tc[4 * (by - 1) + bx] : 0;
          const int nc = ha && hb ? (na + nb + 1) >> 1 : (ha ? na : nb);
          return residual_block(b, S.lev[u - 1], inter || (I4 && nxn) ? 16 : 15, nc);
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
      if (pf) {                                            // mb_skip_run before every coded macroblock
        if (lane == 0) {
          Bits<true> b{S.stg, pend};
          b.ue((unsigned)run);
        }
        pend += ue_bits((unsigned)run);
        run = 0;
      }
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
          b.ue(pf ? 30 : 25);                              // I_PCM, then pcm_alignment_zero_bits
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
      if constexpr (GOP) {
        if (pcm) {                                         // the reconstruction is the source
          for (int i = lane; i < 384; i += 32) {
            const int k = (i - 256) >> 6, q = (i - 256) & 63;
            if constexpr (ME) {
              if (i < 256) rrow[yo(i >> 4, mx, i & 15)] = S.y[i];
              else rrow[co(k, q >> 3, mx, q & 7)] = (k ? S.cr : S.cb)[q];
            } else {
              if (i < 256) rrow[(i >> 4) * J.w + 16 * mx + (i & 15)] = S.y[i];
              else rrow[16 * J.w + k * 4 * J.w + (q >> 3) * (J.w >> 1) + 8 * mx + (q & 7)] = (k ? S.cr : S.cb)[q];
            }
          }
        }
      }
      // ---- whole bytes out, the partial byte stays ----
      at = flush_bytes(S.stg, end >> 3, out, at, zrun, lane);
      const unsigned keep = (end & 7) ? stg_byte(S.stg, end >> 3) : 0u;
      __syncwarp();
      for (int i = lane; i <= (end >> 5) && i < STG_WORDS; i += 32) S.stg[i] = 0;
      __syncwarp();
      if (lane == 0) S.stg[0] = keep;
      pend = end & 7;
      // ---- the left neighbour of the next macroblock ----
      if constexpr (ME) lmv = inter && !pcm ? mv : make_short2(0, 0);
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
      if constexpr (I4) {
        if (lane < 4) S.lm4[lane] = nxn && !pcm ? S.m4[4 * lane + 3] : 2;
      }
      __syncwarp();
    }
    // ---- a trailing mb_skip_run, rbsp_slice_trailing_bits, the last bytes, the length prefix ----
    if (lane == 0) {
      Bits<true> b{S.stg, pend};
      if (run) b.ue((unsigned)run);
      b.put(1, 1);
    }
    if (run) pend += ue_bits((unsigned)run);
    __syncwarp();
    at = flush_bytes(S.stg, (pend + 1 + 7) >> 3, out, at, zrun, lane);
    if (lane == 0) {
      const long long len = at - 4;
      out[0] = (unsigned char)(len >> 24); out[1] = (unsigned char)(len >> 16);
      out[2] = (unsigned char)(len >> 8); out[3] = (unsigned char)len;
      J.slice_bytes[row] = (int)at;
    }
    if (!GOP || ME) break;                               // one frame per warp
    __syncwarp();
  }
}

// One CTA per (chain, macroblock) of frame J.k of every chain (k >= 1): the vector of the P_L0_16x16 candidate by the
// rule of include/pm_emage.h, into J.mv.  The reference window the search and the 6-tap filter read, clipped to the
// frame, is staged in shared memory.  Integer search: one thread per candidate, SADs four samples at a time; the
// argmin under the tie rule is a block-wide minimum of (J, |dx| + |dy|, dy, dx) keys.  Sub-pel refinement: one warp
// per neighbour, 8 neighbours per step.
constexpr int SEARCH_THREADS = 256;
constexpr int MAX_SEARCH = 32;
constexpr int WIN_PITCH = (16 + 2 * MAX_SEARCH + 6 + 3) & ~3;   // window row bytes (16 + 2 search + 6 used)

__global__ void __launch_bounds__(SEARCH_THREADS) h264_search_kernel(Job J) {
  __shared__ unsigned win[(16 + 2 * MAX_SEARCH + 6) * WIN_PITCH / 4];
  __shared__ unsigned src[64];
  __shared__ unsigned long long red[SEARCH_THREADS / 32];
  __shared__ int jn[8];
  const unsigned char* wb = reinterpret_cast<const unsigned char*>(win);
  const unsigned char* sb = reinterpret_cast<const unsigned char*>(src);
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int mbw = J.w >> 4, mbh = J.h >> 4;
  const long long chain = blockIdx.x / ((long long)mbw * mbh);
  const int my = (int)(blockIdx.x / mbw % mbh), mx = (int)(blockIdx.x % mbw);
  const int t0 = (int)(chain % J.chains_per_clip) * J.gop;
  if (t0 + J.k >= min(t0 + J.gop, J.clip_len)) return;
  const unsigned char* fr = J.px + (chain / J.chains_per_clip * J.clip_len + t0 + J.k) * J.fs;
  const unsigned char* ref = J.recon + chain * J.recon_stride + ((J.k + 1) & 1) * (3LL * J.h * J.w / 2);
  const int s = J.search, wn = 16 + 2 * s + 6, ox = 16 * mx - s - 3, oy = 16 * my - s - 3;
  {
    const unsigned char* p = fr + ((long long)(16 * my + (tid >> 4)) * J.w + 16 * mx + (tid & 15)) * 3;
    reinterpret_cast<unsigned char*>(src)[tid] =
        (unsigned char)(((66 * p[0] + 129 * p[1] + 25 * p[2] + 128) >> 8) + 16);
  }
  for (int i = tid; i < wn * wn; i += SEARCH_THREADS) {
    const int r = i / wn, c = i - r * wn;
    reinterpret_cast<unsigned char*>(win)[r * WIN_PITCH + c] =
        ref[(long long)min(J.h - 1, max(0, oy + r)) * J.w + min(J.w - 1, max(0, ox + c))];
  }
  __syncthreads();
  const int lam = LAMBDA[J.qp];
  // ---- integer search: every (dx, dy), |dx|, |dy| <= s, whose block lies inside the frame ----
  const int dx0 = max(-s, -16 * mx), dx1 = min(s, J.w - 16 - 16 * mx);
  const int dy0 = max(-s, -16 * my), dy1 = min(s, J.h - 16 - 16 * my);
  const int nx = dx1 - dx0 + 1, n = nx * (dy1 - dy0 + 1);
  unsigned long long best = ~0ull;
  for (int c = tid; c < n; c += SEARCH_THREADS) {
    const int dx = dx0 + c % nx, dy = dy0 + c / nx;
    const int x = 3 + s + dx, sh = 8 * (x & 3);
    const unsigned* row = win + ((3 + s + dy) * WIN_PITCH + (x & ~3)) / 4;
    unsigned sad = 0;
#pragma unroll 4
    for (int r = 0; r < 16; ++r, row += WIN_PITCH / 4) {
      unsigned a = row[0];
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const unsigned b = row[i + 1];
        sad = __vsadu4(__funnelshift_r(a, b, sh), src[4 * r + i]) + sad;
        a = b;
      }
    }
    const unsigned cost = sad + lam * (se_bits(4 * dx) + se_bits(4 * dy));
    const unsigned long long key = (unsigned long long)cost << 24 | (unsigned)(abs(dx) + abs(dy)) << 16
                                   | (unsigned)(dy + MAX_SEARCH) << 8 | (unsigned)(dx + MAX_SEARCH);
    best = min(best, key);
  }
#pragma unroll
  for (int o = 16; o; o >>= 1) best = min(best, __shfl_xor_sync(0xffffffffu, best, o));
  if (lane == 0) red[warp] = best;
  __syncthreads();
#pragma unroll
  for (int i = 0; i < SEARCH_THREADS / 32; ++i) best = min(best, red[i]);
  int mvx = 4 * ((int)(best & 0xff) - MAX_SEARCH), mvy = 4 * ((int)(best >> 8 & 0xff) - MAX_SEARCH);
  int cost = (int)(best >> 24);
  // ---- sub-pel refinement: the 8 neighbours at +-2, then at +-1, in raster order; strictly lower J replaces ----
  for (int step = 2; step >= 1; step >>= 1) {
    if (warp < 8) {
      const int nb = warp < 4 ? warp : warp + 1;                  // raster index around the centre (4)
      const int cx = mvx + (nb % 3 - 1) * step, cy = mvy + (nb / 3 - 1) * step;
      int sad = 0;
      for (int p = lane; p < 256; p += 32) {
        const unsigned char* g = wb + (3 + s + (p >> 4) + (cy >> 2)) * WIN_PITCH + 3 + s + (p & 15) + (cx >> 2);
        sad += abs((int)sb[p] - luma_pred([&](int dx, int dy) { return (int)g[dy * WIN_PITCH + dx]; }, cx & 3, cy & 3));
      }
      sad = warp_sum(sad);
      if (lane == 0) jn[warp] = sad + lam * (se_bits(cx) + se_bits(cy));
    }
    __syncthreads();
    int bi = -1;
#pragma unroll
    for (int i = 0; i < 8; ++i)
      if (jn[i] < cost) { cost = jn[i]; bi = i; }
    if (bi >= 0) {
      const int nb = bi < 4 ? bi : bi + 1;
      mvx += (nb % 3 - 1) * step;
      mvy += (nb / 3 - 1) * step;
    }
    __syncthreads();
  }
  if (tid == 0) J.mv[blockIdx.x] = make_short2((short)mvx, (short)mvy);
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

// gop > 1: the longest slice header of either kind, and at most 3201 bits per macroblock with its share of the
// mb_skip_run codes (include/pm_emage.h).
long long slice_bound_gop(int w) {
  const long long p = (SLICE_HEADER_BITS_GOP + (long long)(MB_BITS_LIMIT + 1) * (w / 16) + 8 + 7) / 8;
  return 4 + p + p / 2;
}

bool shape_ok(int frames, int h, int w) {
  if (frames < 0 || h < 16 || w < 16 || h % 16 || w % 16) return false;
  const long long mbh = h / 16, mbw = w / 16;
  return mbh * mbw <= 36864 && mbh <= 543 && mbw <= 543;
}

// qp's bits above the quantiser: PM_H264_I4X4 or nothing.
bool split_qp(int& qp, bool& i4) {
  i4 = (qp & PM_H264_I4X4) != 0;
  qp &= ~PM_H264_I4X4;
  return qp >= 0 && qp <= 51;
}

}  // namespace

extern "C" int pm_h264_encode(const unsigned char* frames, long long f_fs, int n_frames, int clip_len, int h, int w,
                              int qp, unsigned char* scratch, long long slice_cap, int* slice_bytes, void* stream) {
  bool i4;
  PM_REQUIRE(split_qp(qp, i4) && shape_ok(n_frames, h, w) && frames && scratch && slice_bytes && f_fs >= 3LL * w * h
             && clip_len >= 1 && slice_cap >= slice_bound(w));
  const long long slices = (long long)n_frames * (h / 16);
  if (slices == 0) return PM_OK;
  PM_REQUIRE(slices / WARPS < 0x7fffffffLL);
  const Job j{frames, f_fs, n_frames, clip_len, h, w, qp, scratch, slice_cap, slice_bytes, 1, 1, nullptr, 0};
  const unsigned grid = (unsigned)((slices + WARPS - 1) / WARPS);
  if (i4) h264_encode_kernel<INTRA, true><<<grid, 32 * WARPS, 0, (cudaStream_t)stream>>>(j);
  else h264_encode_kernel<INTRA, false><<<grid, 32 * WARPS, 0, (cudaStream_t)stream>>>(j);
  PM_LAUNCH_CHECK();
}

extern "C" int pm_h264_encode_gop(const unsigned char* frames, long long f_fs, int n_frames, int clip_len, int h,
                                  int w, int qp, unsigned char* scratch, long long slice_cap, int* slice_bytes,
                                  int gop, unsigned char* recon, long long recon_stride, void* stream) {
  PM_REQUIRE(gop >= 1);
  if (gop == 1) return pm_h264_encode(frames, f_fs, n_frames, clip_len, h, w, qp, scratch, slice_cap, slice_bytes,
                                      stream);
  bool i4;
  PM_REQUIRE(split_qp(qp, i4) && shape_ok(n_frames, h, w) && frames && scratch && slice_bytes && recon
             && f_fs >= 3LL * w * h && clip_len >= 1 && n_frames % clip_len == 0 && gop <= clip_len
             && slice_cap >= slice_bound_gop(w) && recon_stride >= 24LL * w);
  const int chains_per_clip = (int)(((long long)clip_len + gop - 1) / gop);
  const long long slices = (long long)(n_frames / clip_len) * chains_per_clip * (h / 16);
  if (slices == 0) return PM_OK;
  PM_REQUIRE(slices / WARPS < 0x7fffffffLL);
  const Job j{frames, f_fs, n_frames, clip_len, h, w, qp, scratch, slice_cap, slice_bytes, gop, chains_per_clip, recon,
              recon_stride};
  const unsigned grid = (unsigned)((slices + WARPS - 1) / WARPS);
  if (i4) h264_encode_kernel<GOP_ZERO, true><<<grid, 32 * WARPS, 0, (cudaStream_t)stream>>>(j);
  else h264_encode_kernel<GOP_ZERO, false><<<grid, 32 * WARPS, 0, (cudaStream_t)stream>>>(j);
  PM_LAUNCH_CHECK();
}

extern "C" int pm_h264_encode_me(const unsigned char* frames, long long f_fs, int n_frames, int clip_len, int h,
                                 int w, int qp, unsigned char* scratch, long long slice_cap, int* slice_bytes, int gop,
                                 unsigned char* recon, long long recon_stride, int search, short* mv,
                                 long long mv_len, void* stream) {
  bool i4;
  PM_REQUIRE(split_qp(qp, i4) && shape_ok(n_frames, h, w) && frames && scratch && slice_bytes && recon && mv
             && f_fs >= 3LL * w * h && clip_len >= 1 && n_frames % clip_len == 0 && gop >= 2 && gop <= clip_len
             && search >= 1 && search <= MAX_SEARCH && slice_cap >= slice_bound_gop(w) && recon_stride >= 3LL * h * w);
  const int chains_per_clip = (int)(((long long)clip_len + gop - 1) / gop);
  const long long chains = (long long)(n_frames / clip_len) * chains_per_clip, slices = chains * (h / 16);
  if (slices == 0) return PM_OK;
  const long long mbs = slices * (w / 16);
  PM_REQUIRE(mv_len >= mbs && reinterpret_cast<unsigned long long>(mv) % 4 == 0 && slices / WARPS < 0x7fffffffLL
             && mbs < 0x7fffffffLL);
  Job j{frames, f_fs, n_frames, clip_len, h, w, qp, scratch, slice_cap, slice_bytes, gop, chains_per_clip, recon,
        recon_stride, 0, search, reinterpret_cast<short2*>(mv)};
  const cudaStream_t st = (cudaStream_t)stream;
  const unsigned grid = (unsigned)((slices + WARPS - 1) / WARPS);
  for (j.k = 0; j.k < gop; ++j.k) {
    if (j.k) h264_search_kernel<<<(unsigned)mbs, SEARCH_THREADS, 0, st>>>(j);
    if (i4) h264_encode_kernel<GOP_ME, true><<<grid, 32 * WARPS, 0, st>>>(j);
    else h264_encode_kernel<GOP_ME, false><<<grid, 32 * WARPS, 0, st>>>(j);
  }
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
