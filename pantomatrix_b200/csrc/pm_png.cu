// PNG encoding of RGB8 frames (pantomatrix_b200/png.py): one file per frame by the rule of include/pm_emage.h and
// DESIGN.md section 11 (Sub filter, a greedy parse over fixed candidate distances, one fixed-Huffman deflate block).
// Four launches per call after the caller's memset of the output slots:
//   pm_png_count  one thread per (frame, row): parse the row, write its bit count and its Adler-32 partial sums;
//   pm_png_scan   one CTA per frame: row bit offsets, Adler-32, the header, the trailer and the frame's byte count;
//   pm_png_emit   one thread per (frame, row): parse the row again and OR its bits in at the row's offset;
//   pm_png_crc    one thread per 1 KiB block of IDAT: each block's CRC-32 shifted to the end of the chunk, XORed in.
// CPU restatement: oracle/png_oracle.py.  Every byte depends only on the frame, never on execution order.
#include <cub/block/block_reduce.cuh>
#include <cub/block/block_scan.cuh>

#include "pm_common.cuh"
#include "../../include/pm_emage.h"

namespace {

constexpr int MAX_MATCH = 258, MIN_MATCH = 3, WINDOW = 32768, NCAND = 15;
constexpr int DEFLATE_AT = 43;            // signature 8 + IHDR 25 + IDAT length and type 8 + zlib header 2
constexpr int IDAT_TYPE_AT = 37;          // the IDAT CRC covers bytes [37, crc position)
constexpr long long OVERHEAD = 63;        // + Adler 4 + IDAT CRC 4 + IEND 12
constexpr unsigned ADLER_MOD = 65521, ADLER_NMAX = 5552;   // NMAX: the most bytes before b can pass 2^32
constexpr unsigned CRC_POLY = 0xEDB88320u;
constexpr int CRC_BLOCK = 1024;
constexpr int SCAN_THREADS = 1024;

// The bound of pm_emage.h: ceil((3 + 9 H s + 7) / 8) + 63 bytes.
__host__ __device__ inline long long max_bytes(long long h, long long s) { return (9 * h * s + 17) / 8 + OVERHEAD; }

struct Frame {
  const unsigned char* px;   // frame 0, row 0
  long long fs;              // frame stride (bytes)
  int h, w, s;               // s = 3 w + 1
};

// Filtered byte at (row r, column c) of frame f's scanlines: 1 (Sub) at column 0, then raw[i] - raw[i - 3] mod 256.
__device__ __forceinline__ unsigned fbyte(const unsigned char* fr, int s, int r, int c) {
  if (c == 0) return 1u;
  const unsigned char* row = fr + (long long)r * (s - 1);
  const int i = c - 1;
  return (unsigned)(unsigned char)(row[i] - (i >= 3 ? row[i - 3] : 0));
}

// Candidate k of the list (1..9, 12, s, s-3, s+3, s-6, s+6).
__device__ __forceinline__ int candidate(int k, int s) {
  if (k < 9) return k + 1;
  switch (k) {
    case 9: return 12;
    case 10: return s;
    case 11: return s - 3;
    case 12: return s + 3;
    case 13: return s - 6;
    default: return s + 6;
  }
}

// Greedy match at (row r, column c), p = r s + c: the longest length over the valid candidates (0 when < 3) and the
// first distance that reaches it.
__device__ __forceinline__ int longest(const unsigned char* fr, int s, int r, int c, long long p, int& dist) {
  const int room = min(MAX_MATCH, s - c);
  int best = 0;
  dist = 0;
  if (room < MIN_MATCH) return 0;
  for (int k = 0; k < NCAND && best < room; ++k) {
    const int d = candidate(k, s);
    if (d < 1 || d > WINDOW || d > p) continue;
    int rq = r, cq = c - d;                       // the source (p - d) as (row, column)
    while (cq < 0) { cq += s; --rq; }
    // a candidate can only win with a longer match: test the byte that would make it longer first
    if (best >= MIN_MATCH) {
      int rb = rq, cb = cq + best;
      while (cb >= s) { cb -= s; ++rb; }
      if (fbyte(fr, s, rb, cb) != fbyte(fr, s, r, c + best)) continue;
    }
    int len = 0;
    while (len < room && fbyte(fr, s, rq, cq) == fbyte(fr, s, r, c + len)) {
      ++len;
      if (++cq == s) { cq = 0; ++rq; }
    }
    if (len > best) { best = len; dist = d; }
  }
  return best >= MIN_MATCH ? best : 0;
}

__device__ __forceinline__ unsigned rev(unsigned code, int n) { return __brev(code) >> (32 - n); }

// One token as (bits, count) of the LSB-first stream: fixed Huffman codes reversed, extra bits as they are.
__device__ __forceinline__ unsigned literal_code(unsigned v, int& n) {
  n = v < 144 ? 8 : 9;
  return v < 144 ? rev(0x30 + v, 8) : rev(0x190 + v - 144, 9);
}

__device__ __forceinline__ unsigned match_code(int len, int dist, int& n) {
  int idx, extra = 0, base;
  if (len == MAX_MATCH) { idx = 28; base = MAX_MATCH; }
  else if (len < 11) { idx = len - 3; base = len; }
  else {
    const int x = len - 3;
    extra = 29 - __clz(x);                                  // floor(log2 x) - 2
    idx = 4 * extra + 4 + ((x >> extra) & 3);
    base = 3 + ((4 + ((x >> extra) & 3)) << extra);
  }
  const int sym = 257 + idx;
  unsigned v = sym < 280 ? rev(sym - 256, 7) : rev(0xC0 + sym - 280, 8);
  n = sym < 280 ? 7 : 8;
  v |= (unsigned)(len - base) << n;
  n += extra;
  int dcode, dextra = 0, dbase;
  if (dist <= 4) { dcode = dist - 1; dbase = dist; }
  else {
    const int x = dist - 1;
    dextra = 30 - __clz(x);                                 // floor(log2 x) - 1
    dcode = 2 * dextra + 2 + ((x >> dextra) & 1);
    dbase = 1 + ((2 + ((x >> dextra) & 1)) << dextra);
  }
  v |= rev(dcode, 5) << n;
  n += 5;
  v |= (unsigned)(dist - dbase) << n;
  n += dextra;
  return v;
}

// Words of the output slot: bits at or past `start` (slot bit index) are ORed into 32-bit little-endian words, whose
// byte order is the stream's.  Only the first and the last word of a row are shared with its neighbours: those go
// through atomicOr, the rest are stored.
struct BitWriter {
  unsigned* words;
  long long word;
  unsigned long long acc;
  int nb;
  bool first;
  __device__ BitWriter(unsigned char* slot, long long start)
      : words(reinterpret_cast<unsigned*>(slot)), word(start >> 5), acc(0), nb((int)(start & 31)), first(true) {}
  __device__ __forceinline__ void put(unsigned v, int n) {
    acc |= (unsigned long long)v << nb;
    nb += n;
    while (nb >= 32) {
      if (first) atomicOr(words + word, (unsigned)acc);
      else words[word] = (unsigned)acc;
      first = false;
      ++word;
      acc >>= 32;
      nb -= 32;
    }
  }
  __device__ __forceinline__ void flush() {
    if (nb > 0) atomicOr(words + word, (unsigned)acc);
  }
};

// Parse row r of frame `fr`: the bit count, or (EMIT) write the bits from slot bit `start`.
template <bool EMIT>
__device__ long long parse_row(const unsigned char* fr, int s, int r, unsigned char* slot, long long start) {
  const long long p0 = (long long)r * s;
  long long bits = 0;
  BitWriter out(slot, start);
  for (int c = 0; c < s;) {
    int dist, n;
    const int len = longest(fr, s, r, c, p0 + c, dist);
    const unsigned v = len ? match_code(len, dist, n) : literal_code(fbyte(fr, s, r, c), n);
    if (EMIT) out.put(v, n);
    bits += n;
    c += len ? len : 1;
  }
  if (EMIT) out.flush();
  return bits;
}

__global__ void __launch_bounds__(128) png_count_kernel(Frame F, long long total, long long* __restrict__ row_bits,
                                                        unsigned long long* __restrict__ row_adler) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= total) return;
  const long long f = i / F.h;
  const int r = (int)(i % F.h);
  const unsigned char* fr = F.px + f * F.fs;
  row_bits[i] = parse_row<false>(fr, F.s, r, nullptr, 0);
  // Adler-32 partials of the row with a = 0 at its start: sum = sum x_i, wsum = sum (s - i) x_i, both mod 65521
  unsigned a = 0, b = 0;
  for (int c0 = 0; c0 < F.s; c0 += ADLER_NMAX) {
    for (int c = c0, c1 = min(F.s, c0 + (int)ADLER_NMAX); c < c1; ++c) {
      a += fbyte(fr, F.s, r, c);
      b += a;
    }
    a %= ADLER_MOD;
    b %= ADLER_MOD;
  }
  row_adler[i] = (unsigned long long)b << 32 | a;
}

// ---- CRC-32 (reflected, polynomial 0xEDB88320): byte table, and x^n mod P for the shifts ----
__device__ __forceinline__ unsigned crc_mul(unsigned a, unsigned b) {   // a b mod P, bit 31 = x^0
  unsigned p = 0;
  for (int k = 31; k >= 0; --k) {
    if (a & (1u << k)) p ^= b;
    b = (b & 1) ? (b >> 1) ^ CRC_POLY : b >> 1;
  }
  return p;
}

// x^(2^k) mod P for k = 0..31 (the sequence repeats with period 32): k = 0 is x^1, each entry the square of the last
__constant__ unsigned X2N[32] = {
    0x40000000, 0x20000000, 0x08000000, 0x00800000, 0x00008000, 0xedb88320, 0xb1e6b092, 0xa06a2517,
    0xed627dae, 0x88d14467, 0xd7bbfe6a, 0xec447f11, 0x8e7ea170, 0x6427800e, 0x4d47bae0, 0x09fe548f,
    0x83852d0f, 0x30362f1a, 0x7b5a9cc3, 0x31fec169, 0x9fec022a, 0x6c8dedc4, 0x15d6874d, 0x5fde7a4e,
    0xbad90e37, 0x2e4e5eef, 0x4eaba214, 0xa8a472c0, 0x429a969e, 0x148d302a, 0xc40ba6d0, 0xc4e22c3c};

struct CrcTables { unsigned byte[256]; unsigned x2n[32]; };

__device__ void crc_tables(CrcTables& T) {
  for (int i = threadIdx.x; i < 256; i += blockDim.x) {
    unsigned c = i;
    for (int k = 0; k < 8; ++k) c = (c & 1) ? (c >> 1) ^ CRC_POLY : c >> 1;
    T.byte[i] = c;
    if (i < 32) T.x2n[i] = X2N[i];
  }
  __syncthreads();
}

// c x^(8 n) mod P: a CRC register moved past n zero bytes.
__device__ __forceinline__ unsigned crc_shift(const CrcTables& T, unsigned c, unsigned long long n) {
  unsigned x = 1u << 31;                                   // x^0
  for (int k = 3; n; n >>= 1, ++k)
    if (n & 1) x = crc_mul(T.x2n[k & 31], x);
  return crc_mul(x, c);
}

__device__ __forceinline__ unsigned crc_bytes(const unsigned* table, unsigned c, const unsigned char* p, int n) {
  for (int i = 0; i < n; ++i) c = table[(c ^ p[i]) & 0xff] ^ (c >> 8);
  return c;
}

__device__ __forceinline__ void be32(unsigned char* p, unsigned v) {
  p[0] = v >> 24; p[1] = v >> 16; p[2] = v >> 8; p[3] = v;
}

__global__ void __launch_bounds__(SCAN_THREADS) png_scan_kernel(int h, int w, long long* __restrict__ row_bits,
                                                                const unsigned long long* __restrict__ row_adler,
                                                                unsigned char* __restrict__ data, long long cap,
                                                                long long* __restrict__ nbytes) {
  using Scan = cub::BlockScan<long long, SCAN_THREADS>;
  using Sum = cub::BlockReduce<unsigned long long, SCAN_THREADS>;
  __shared__ union { typename Scan::TempStorage scan; typename Sum::TempStorage sum; } tmp;
  __shared__ CrcTables T;
  __shared__ long long row_total;
  crc_tables(T);
  const long long f = blockIdx.x;
  const int s = 3 * w + 1;
  const long long n = (long long)h * s;
  long long* bits = row_bits + f * h;
  const unsigned long long* ad = row_adler + f * h;
  const int per = (h + SCAN_THREADS - 1) / SCAN_THREADS, r0 = min(h, (int)threadIdx.x * per), r1 = min(h, r0 + per);
  // Adler-32 of S from the rows: A = 1 + sum_r sum_r, B = n + sum_r (wsum_r + (n - (r + 1) s) sum_r), mod 65521
  long long mine = 0;
  unsigned long long a = 0, b = 0;
  for (int r = r0; r < r1; ++r) {
    mine += bits[r];
    const unsigned long long sum = ad[r] & 0xffffffffu, wsum = ad[r] >> 32;
    a = (a + sum) % ADLER_MOD;
    b = (b + wsum + (unsigned long long)((n - (long long)(r + 1) * s) % ADLER_MOD) * sum) % ADLER_MOD;
  }
  long long before;
  Scan(tmp.scan).ExclusiveSum(mine, before);
  for (int r = r0; r < r1; ++r) {                       // row bit counts become their slot bit offsets
    const long long nbits = bits[r];
    bits[r] = 8LL * DEFLATE_AT + 3 + before;
    before += nbits;
  }
  if (threadIdx.x == SCAN_THREADS - 1) row_total = before;   // the last thread ends at the sum of every row
  __syncthreads();
  const unsigned long long asum = Sum(tmp.sum).Sum(a);     // the reductions are valid in thread 0
  __syncthreads();
  const unsigned long long bsum = Sum(tmp.sum).Sum(b);
  if (threadIdx.x != 0) return;
  const long long deflate_bits = 3 + row_total + 7;        // block header, the rows, end-of-block (7 zero bits)
  const long long deflate_bytes = (deflate_bits + 7) / 8;
  const long long total = deflate_bytes + OVERHEAD;
  unsigned char* o = data + f * cap;
  const unsigned char sig[8] = {0x89, 'P', 'N', 'G', '\r', '\n', 0x1a, '\n'};
  for (int i = 0; i < 8; ++i) o[i] = sig[i];
  be32(o + 8, 13);
  const unsigned char ihdr[17] = {'I', 'H', 'D', 'R', (unsigned char)(w >> 24), (unsigned char)(w >> 16),
                                  (unsigned char)(w >> 8), (unsigned char)w, (unsigned char)(h >> 24),
                                  (unsigned char)(h >> 16), (unsigned char)(h >> 8), (unsigned char)h, 8, 2, 0, 0, 0};
  for (int i = 0; i < 17; ++i) o[12 + i] = ihdr[i];
  be32(o + 29, ~crc_bytes(T.byte, 0xffffffffu, ihdr, 17));
  const long long idat_len = 2 + deflate_bytes + 4;
  be32(o + 33, (unsigned)idat_len);
  o[37] = 'I'; o[38] = 'D'; o[39] = 'A'; o[40] = 'T';
  o[41] = 0x78; o[42] = 0x01;
  o[43] = 0x03;                                          // BFINAL = 1, BTYPE = 01, LSB first
  const unsigned adler = (unsigned)((((n % ADLER_MOD) + bsum) % ADLER_MOD) << 16 | ((1 + asum) % ADLER_MOD));
  unsigned char* tail = o + DEFLATE_AT + deflate_bytes;
  be32(tail, adler);
  // the IDAT CRC's part that does not depend on the data: the 0xffffffff start moved past the chunk, and the final
  // complement; pm_png_crc XORs in each block's register
  const long long msg = 4 + idat_len;
  be32(tail + 4, crc_shift(T, 0xffffffffu, (unsigned long long)msg) ^ 0xffffffffu);
  const unsigned char iend[12] = {0, 0, 0, 0, 'I', 'E', 'N', 'D', 0xae, 0x42, 0x60, 0x82};
  for (int i = 0; i < 12; ++i) tail[8 + i] = iend[i];
  nbytes[f] = total;
}

__global__ void __launch_bounds__(256) png_emit_kernel(Frame F, long long total, const long long* __restrict__ row_off,
                                                       unsigned char* __restrict__ data, long long cap) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= total) return;
  const long long f = i / F.h;
  parse_row<true>(F.px + f * F.fs, F.s, (int)(i % F.h), data + f * cap, row_off[i]);
}

__global__ void __launch_bounds__(256) png_crc_kernel(int frames, long long blocks, unsigned char* __restrict__ data,
                                                      long long cap, const long long* __restrict__ nbytes) {
  __shared__ CrcTables T;
  crc_tables(T);
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= frames * blocks) return;
  const long long f = i / blocks, b = i % blocks;
  const long long msg = nbytes[f] - OVERHEAD + 10;        // "IDAT" + zlib header + deflate + Adler
  const long long start = b * CRC_BLOCK;
  if (start >= msg) return;
  const int len = (int)min((long long)CRC_BLOCK, msg - start);
  unsigned char* o = data + f * cap;
  // this block's register from 0, moved to the end of the chunk: the CRC is linear, so the XOR of every block's
  // contribution and the data-independent part pm_png_scan wrote is the chunk's CRC, whatever the order
  const unsigned c = crc_shift(T, crc_bytes(T.byte, 0, o + IDAT_TYPE_AT + start, len),
                               (unsigned long long)(msg - start - len));
  const long long at = IDAT_TYPE_AT + msg;                // big-endian CRC bytes at [at, at + 4)
  unsigned* words = reinterpret_cast<unsigned*>(o);
  const unsigned long long be = (unsigned long long)__byte_perm(c, 0, 0x0123) << (8 * (at & 3));
  atomicXor(words + (at >> 2), (unsigned)be);
  if (be >> 32) atomicXor(words + (at >> 2) + 1, (unsigned)(be >> 32));
}

// Shapes every entry point accepts: a frame's bound within 2^31 bytes; slots of `cap` >= the bound, 4-byte multiples.
bool shape_ok(int frames, int h, int w) {
  return frames >= 0 && h >= 1 && w >= 1 && w <= (0x7fffffff - 1) / 3 && max_bytes(h, 3LL * w + 1) <= (1LL << 31);
}
bool slots_ok(const unsigned char* data, long long cap, int h, int w) {
  return data && cap >= max_bytes(h, 3LL * w + 1) && (cap & 3) == 0 && (reinterpret_cast<uintptr_t>(data) & 3) == 0;
}

inline unsigned blocks(long long n, int t) { return (unsigned)((n + t - 1) / t); }

}  // namespace

extern "C" int pm_png_count(const unsigned char* frames, long long f_fs, int n_frames, int h, int w, long long* row_bits,
                            unsigned long long* row_adler, void* stream) {
  PM_REQUIRE(shape_ok(n_frames, h, w) && frames && row_bits && row_adler && f_fs >= 3LL * w * h);
  const long long total = (long long)n_frames * h;
  if (total == 0) return PM_OK;
  PM_REQUIRE(total / 128 < 0x7fffffffLL);
  png_count_kernel<<<blocks(total, 128), 128, 0, (cudaStream_t)stream>>>(Frame{frames, f_fs, h, w, 3 * w + 1}, total,
                                                                         row_bits, row_adler);
  PM_LAUNCH_CHECK();
}

extern "C" int pm_png_scan(int n_frames, int h, int w, long long* row_bits, const unsigned long long* row_adler,
                           unsigned char* data, long long cap, long long* nbytes, void* stream) {
  PM_REQUIRE(shape_ok(n_frames, h, w) && slots_ok(data, cap, h, w) && row_bits && row_adler && nbytes);
  if (n_frames == 0) return PM_OK;
  png_scan_kernel<<<n_frames, SCAN_THREADS, 0, (cudaStream_t)stream>>>(h, w, row_bits, row_adler, data, cap, nbytes);
  PM_LAUNCH_CHECK();
}

extern "C" int pm_png_emit(const unsigned char* frames, long long f_fs, int n_frames, int h, int w,
                           const long long* row_off, unsigned char* data, long long cap, void* stream) {
  PM_REQUIRE(shape_ok(n_frames, h, w) && slots_ok(data, cap, h, w) && frames && row_off && f_fs >= 3LL * w * h);
  const long long total = (long long)n_frames * h;
  if (total == 0) return PM_OK;
  PM_REQUIRE(total / 256 < 0x7fffffffLL);
  png_emit_kernel<<<blocks(total, 256), 256, 0, (cudaStream_t)stream>>>(Frame{frames, f_fs, h, w, 3 * w + 1}, total,
                                                                        row_off, data, cap);
  PM_LAUNCH_CHECK();
}

extern "C" int pm_png_crc(int n_frames, int h, int w, unsigned char* data, long long cap, const long long* nbytes,
                          void* stream) {
  PM_REQUIRE(shape_ok(n_frames, h, w) && slots_ok(data, cap, h, w) && nbytes);
  // IDAT's CRC covers at most the bound less the 37 bytes before "IDAT", the CRC itself and the 12-byte IEND
  const long long nblk = (max_bytes(h, 3LL * w + 1) - 53 + CRC_BLOCK - 1) / CRC_BLOCK;
  const long long total = (long long)n_frames * nblk;
  if (total == 0) return PM_OK;
  PM_REQUIRE(total / 256 < 0x7fffffffLL);
  png_crc_kernel<<<blocks(total, 256), 256, 0, (cudaStream_t)stream>>>(n_frames, nblk, data, cap, nbytes);
  PM_LAUNCH_CHECK();
}
