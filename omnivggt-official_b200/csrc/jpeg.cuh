// Baseline JPEG decoding on the device, bit-identical to libjpeg-turbo's default decode as Pillow calls it.
//
// Host (no CUDA calls): plan_build walks the markers of every file, decides device or host (and why), builds the Huffman
// lookup tables, and writes the staging stream: [files][segments][Huffman tables][entropy data], the data unstuffed (FF 00 -> FF,
// RST markers removed) with one segment per restart interval, each 16-byte aligned and followed by >= 16 zero bytes so that no
// read of the decoder leaves the buffer.
//
// Device, one set of launches for the whole batch:
//   jpeg_sync_kernel      self-synchronising parallel Huffman decoding (Weissenberger & Schmidt, ICPP 2018): every segment is cut
//                         into subsequences of subseq_bits, one thread each.  A thread decodes from its predecessor's exit state
//                         (bit position, block within the MCU, coefficient index z) to the first symbol boundary at or past its
//                         end and publishes its own exit state and the number of DC symbols that start inside it.  The host
//                         repeats rounds until no exit state changes; the first subsequence of a segment starts exact, so the
//                         result is exact for every input (the worst case is serial, never wrong).
//   jpeg_count_scan_*     exclusive scan of the per-subsequence block counts: each block's ordinal within its segment.
//   jpeg_write_kernel     decodes again from the converged states and scatters the coefficients in natural order (a block
//                         belongs to the subsequence in which its DC symbol starts; that thread finishes it); DC differences
//                         go to coefficient 0.  Flags the file (status word) on a code not in the table, z past 63, too few
//                         blocks in a segment, or a block that runs past the segment's data.
//   jpeg_dc_*             segmented scan of the DC differences per component, reset at every restart marker (modulo 2^16,
//                         which is what storing libjpeg's int prediction into a 16-bit JCOEF keeps).
//   jpeg_idct_kernel      jidctint.c jpeg_idct_islow with dequantisation, into the component planes.  Exact only inside the
//                         range where libjpeg-turbo's C and SIMD IDCTs agree (ST_IDCT_RANGE below); a block outside it
//                         flags its file for Pillow.
//   jpeg_color_kernel     jdsample.c h2v1 / h2v2 fancy upsampling (plain replication when the chroma width is <= 2, as
//                         jinit_upsampler picks), jdcolor.c ycc_rgb_convert tables (SCALEBITS 16) -> uint8 RGB [h, w, 3];
//                         one component: the sample replicated three times (Pillow "L" -> "RGB").
// oracle/jpeg_oracle.py restates every step in numpy; tests/test_jpeg.py checks both against Pillow.
#pragma once
#include <cstdint>
#include <algorithm>
#include <atomic>
#include <cstring>
#include <new>
#include <thread>
#include <vector>
#include "arena.cuh"

namespace ovg {
namespace jpg {

constexpr int LUT_BITS = 9;
constexpr int MAX_BLK = 6;                       // blocks per MCU: luma 2 x 2 + Cb + Cr
constexpr int MIN_SUBSEQ_BITS = 32;              // > the longest symbol (16-bit code + 15 value bits)
constexpr int MAX_SUBSEQ_BITS = 1 << 16;
constexpr int DEFAULT_SUBSEQ_BITS = 512;
constexpr int SCAN_CHUNK = 1024;
constexpr int SEG_ALIGN = 16, SEG_PAD = 16;

// status bits of a device-decoded file (0: exact)
constexpr unsigned ST_BAD_CODE = 1, ST_Z_OVERFLOW = 2, ST_BLOCK_COUNT = 4, ST_ENDS_EARLY = 8, ST_IDCT_RANGE = 16;
// libjpeg-turbo's C islow IDCT (64-bit intermediates, masked range limit) and its SIMD versions (16-bit dequantisation and
// pairwise sums, pass-1 outputs saturated to int16, final samples clamped) agree only while the values stay in range.  A block
// whose dequantised coefficients or pass-1 outputs leave [-16383, 16383], or whose pass-2 results leave [-512, 511], flags its
// file, which is then decoded by Pillow.  Inside those bounds every 32-bit intermediate here is exact (the largest gain of an
// intermediate over its eight inputs is 61214, and 61214 * 16383 < 2^30), so both libjpeg-turbo paths give these samples.
constexpr int IDCT_IN_MAX = 16383, IDCT_OUT_MIN = -512, IDCT_OUT_MAX = 511;

struct Huff {                                    // jdhuff.c d_derived_tbl with a 9-bit lookahead
  uint16_t lut[1 << LUT_BITS];                   // (length << 8) | symbol for codes of <= 9 bits, 0 otherwise
  int32_t maxcode[18];                           // largest code of each length, -1 if none
  int32_t valoff[18];                            // symbol index = code + valoff[length]
  uint8_t val[256];
};

struct FileDev {
  int width, height, ncomp, gray;
  int hmax, vmax, mcux, mcuy;
  int nblk, restart;                             // blocks per MCU; MCUs per restart interval (all of them without DRI)
  int blk_comp[MAX_BLK], blk_sub[MAX_BLK];       // per block of the MCU: component and raster index within its h x v group
  int h[3], v[3];                                // sampling factors as the scan lays blocks out (1 x 1 for one component)
  int huff_dc[3], huff_ac[3];                    // index into the Huff array
  int out_index;                                 // position in the caller's file list (output pointer and status word)
  int pad_;
  long long coef_base[3];                        // first block of each component in the coefficient array (MCU-major order)
  long long plane_off[3];                        // byte offset of each component plane (width bw * 8, rows bh * 8)
  long long pix_base;                            // first output pixel of this file in the batch's pixel enumeration
  uint16_t quant[3][64];                         // natural order
};

struct SegDev {
  long long bit_start, nbits;                    // in the stream
  long long first_sub;                           // first subsequence of this segment
  int file, first_mcu, n_mcu, n_sub;
};

struct Params {
  const FileDev* files;
  const SegDev* segs;
  const Huff* huffs;
  const uint8_t* data;                           // stream base (bit positions are relative to it)
  int nfiles, nsegs;
  long long nsub, nblocks, npix;
  int subseq_bits;
  uint32_t* exits;                               // [nsub] packed exit state
  uint32_t* counts;                              // [nsub] DC symbols starting inside
  unsigned long long* pre;                       // [nsub] block ordinal prefix within the chunk
  unsigned long long* chunk;                     // [nsub chunks] exclusive chunk prefix
  int16_t* coef;                                 // [nblocks][64]
  int* dc_agg;                                   // [nblocks chunks] (value)
  int* dc_aggf;                                  // [nblocks chunks] (a segment head inside)
  uint8_t* dc_head;                              // [nblocks] a head at or before this block within its chunk
  uint8_t* planes;
  uint8_t* const* out;                           // [ncaller files]
  unsigned* status;                              // [ncaller files]
  int* changed;
};

// ------------------------------------------------------------------------------------------------------------- device
__device__ __forceinline__ uint32_t peek32(const uint8_t* data, long long pos) {
  const uint32_t* w = reinterpret_cast<const uint32_t*>(data) + (pos >> 5);
  const uint32_t a = __byte_perm(__ldg(w), 0, 0x0123), b = __byte_perm(__ldg(w + 1), 0, 0x0123);
  return __funnelshift_l(b, a, static_cast<unsigned>(pos & 31));
}

__constant__ uint8_t kNatural[64] = {0,  1,  8,  16, 9,  2,  3,  10, 17, 24, 32, 25, 18, 11, 4,  5,  12, 19, 26, 33, 40, 48,
                                     41, 34, 27, 20, 13, 6,  7,  14, 21, 28, 35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23,
                                     30, 37, 44, 51, 58, 59, 52, 45, 38, 31, 39, 46, 53, 60, 61, 54, 47, 55, 62, 63};

struct Sym {
  int len;      // bits consumed (code + value)
  int value;    // extended value
  int run_s;    // DC: s; AC: (r << 4) | s
  bool bad;
};

__device__ __forceinline__ Sym decode_symbol(const Huff* __restrict__ t, uint32_t bits, bool dc) {
  Sym r;
  const uint32_t e = t->lut[bits >> (32 - LUT_BITS)];
  int len, sym;
  r.bad = false;
  if (e) {
    len = e >> 8;
    sym = e & 255;
  } else {
    len = 0;
    sym = 0;
    for (int l = LUT_BITS + 1; l <= 16; ++l) {
      const int code = static_cast<int>(bits >> (32 - l));
      if (code <= t->maxcode[l]) {
        len = l;
        sym = t->val[code + t->valoff[l]];
        break;
      }
    }
    if (!len) {
      r.bad = true;
      r.len = 1;
      r.value = 0;
      r.run_s = 0;
      return r;
    }
  }
  const int s = dc ? sym : (sym & 15);
  int v = 0;
  if (s) {
    const uint32_t raw = (bits << len) >> (32 - s);       // len + s <= 31: inside the 32 peeked bits
    v = raw < (1u << (s - 1)) ? static_cast<int>(raw) - (1 << s) + 1 : static_cast<int>(raw);   // HUFF_EXTEND
  }
  r.len = len + s;
  r.value = v;
  r.run_s = sym;
  return r;
}

struct State {
  long long pos;
  int slot, z;
};

// One symbol of the state machine.  Returns the zigzag index of the coefficient it decoded (-1: none), with its value in *val;
// *err gets a status bit.  Deterministic for any state, so the sync rounds and the write pass agree.
__device__ __forceinline__ int step(const Params& p, const FileDev& f, State& s, int* val, unsigned* err, bool* block_end) {
  const int c = f.blk_comp[s.slot];
  const bool dc = s.z == 0;
  const Huff* t = p.huffs + (dc ? f.huff_dc[c] : f.huff_ac[c]);
  const Sym y = decode_symbol(t, peek32(p.data, s.pos), dc);
  s.pos += y.len;
  int idx = -1;
  *block_end = false;
  if (y.bad) {
    *err |= ST_BAD_CODE;
    *block_end = true;
  } else if (dc) {
    idx = 0;
    *val = y.value;
    s.z = 1;
  } else {
    const int r = y.run_s >> 4, sz = y.run_s & 15;
    if (sz) {
      s.z += r;
      if (s.z > 63) {
        *err |= ST_Z_OVERFLOW;
        *block_end = true;
      } else {
        idx = s.z;
        *val = y.value;
        if (++s.z == 64) *block_end = true;
      }
    } else if (r == 15) {
      s.z += 16;
      if (s.z > 64) *err |= ST_Z_OVERFLOW;
      if (s.z >= 64) *block_end = true;
    } else {
      *block_end = true;                                   // EOB
    }
  }
  if (*block_end) {
    s.z = 0;
    s.slot = s.slot + 1 == f.nblk ? 0 : s.slot + 1;
  }
  return idx;
}

__device__ __forceinline__ int find_seg(const Params& p, long long i) {
  int lo = 0, hi = p.nsegs - 1;
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (p.segs[mid].first_sub <= i) lo = mid; else hi = mid - 1;
  }
  return lo;
}

// start state of subsequence i (global), its end, and its segment
__device__ __forceinline__ void sub_bounds(const Params& p, long long i, const SegDev& sg, State* st, long long* end) {
  const long long j = i - sg.first_sub;
  const long long start = sg.bit_start + j * p.subseq_bits;
  const long long seg_end = sg.bit_start + sg.nbits;
  *end = start + p.subseq_bits < seg_end ? start + p.subseq_bits : seg_end;
  if (j == 0) {
    st->pos = start; st->slot = 0; st->z = 0;
  } else {
    const uint32_t e = *reinterpret_cast<volatile const uint32_t*>(p.exits + i - 1);
    st->pos = start + (e >> 10);
    st->slot = (e >> 6) & 15;
    st->z = e & 63;
  }
}

__global__ void __launch_bounds__(256) jpeg_sync_kernel(Params p) {
  const long long i = blockIdx.x * 256LL + threadIdx.x;
  if (i >= p.nsub) return;
  const SegDev sg = p.segs[find_seg(p, i)];
  const FileDev& f = p.files[sg.file];
  State s;
  long long end;
  sub_bounds(p, i, sg, &s, &end);
  uint32_t cnt = 0;
  unsigned err = 0;
  int val;
  bool be;
  while (s.pos < end) {
    cnt += s.z == 0;
    step(p, f, s, &val, &err, &be);
  }
  const uint32_t e = (static_cast<uint32_t>(s.pos - end) << 10) | (s.slot << 6) | s.z;
  volatile uint32_t* slot = p.exits + i;
  if (*slot != e) {
    *slot = e;
    atomicAdd(p.changed, 1);
  }
  p.counts[i] = cnt;
}

__device__ __forceinline__ unsigned long long block_excl_scan(unsigned long long x, unsigned long long* total) {
  __shared__ unsigned long long warp_sums[32];
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  unsigned long long inc = x;
  for (int o = 1; o < 32; o <<= 1) {
    const unsigned long long y = __shfl_up_sync(0xffffffffu, inc, o);
    if (lane >= o) inc += y;
  }
  if (lane == 31) warp_sums[wid] = inc;
  __syncthreads();
  if (wid == 0) {
    unsigned long long w = lane < (blockDim.x >> 5) ? warp_sums[lane] : 0;
    for (int o = 1; o < 32; o <<= 1) {
      const unsigned long long y = __shfl_up_sync(0xffffffffu, w, o);
      if (lane >= o) w += y;
    }
    warp_sums[lane] = w;
  }
  __syncthreads();
  const unsigned long long base = wid ? warp_sums[wid - 1] : 0;
  *total = warp_sums[(blockDim.x >> 5) - 1];
  __syncthreads();
  return base + inc - x;
}

__global__ void __launch_bounds__(SCAN_CHUNK) jpeg_count_scan_local_kernel(Params p) {
  const long long i = blockIdx.x * static_cast<long long>(SCAN_CHUNK) + threadIdx.x;
  unsigned long long total;
  const unsigned long long ex = block_excl_scan(i < p.nsub ? p.counts[i] : 0, &total);
  if (i < p.nsub) p.pre[i] = ex;
  if (threadIdx.x == 0) p.chunk[blockIdx.x] = total;
}

__global__ void __launch_bounds__(SCAN_CHUNK) jpeg_count_scan_chunks_kernel(unsigned long long* chunk, long long n) {
  unsigned long long carry = 0;
  for (long long b = 0; b < n; b += SCAN_CHUNK) {
    const long long i = b + threadIdx.x;
    unsigned long long total;
    const unsigned long long ex = block_excl_scan(i < n ? chunk[i] : 0, &total);
    if (i < n) chunk[i] = carry + ex;
    carry += total;
  }
}

__device__ __forceinline__ unsigned long long ordinal(const Params& p, long long i) {
  return p.pre[i] + p.chunk[i / SCAN_CHUNK];
}

__device__ __forceinline__ long long block_index(const FileDev& f, int mcu, int slot) {
  const int c = f.blk_comp[slot];
  return f.coef_base[c] + static_cast<long long>(mcu) * (f.h[c] * f.v[c]) + f.blk_sub[slot];
}

__global__ void __launch_bounds__(256) jpeg_write_kernel(Params p) {
  const long long i = blockIdx.x * 256LL + threadIdx.x;
  if (i >= p.nsub) return;
  const SegDev sg = p.segs[find_seg(p, i)];
  const FileDev& f = p.files[sg.file];
  State s;
  long long end;
  sub_bounds(p, i, sg, &s, &end);
  const long long seg_end = sg.bit_start + sg.nbits;
  const unsigned long long first = ordinal(p, sg.first_sub);
  unsigned long long k = ordinal(p, i) - first;
  const unsigned long long expected = static_cast<unsigned long long>(sg.n_mcu) * f.nblk;
  unsigned err = 0, ignored = 0;
  int val;
  bool be;
  while (s.z != 0 && s.pos < seg_end) step(p, f, s, &val, &ignored, &be);     // the tail of a block owned by a predecessor
  while (s.pos < end && k < expected) {
    const int mcu = sg.first_mcu + static_cast<int>(k / f.nblk);
    int16_t* blk = p.coef + block_index(f, mcu, s.slot) * 64;
    do {
      if (s.pos >= seg_end) {
        err |= ST_ENDS_EARLY;
        break;
      }
      const int idx = step(p, f, s, &val, &err, &be);
      if (idx >= 0) blk[kNatural[idx]] = static_cast<int16_t>(val);
    } while (!be);
    if (s.pos > seg_end) err |= ST_ENDS_EARLY;
    ++k;
  }
  if (i == sg.first_sub + sg.n_sub - 1 && ordinal(p, i) + p.counts[i] - first < expected) err |= ST_BLOCK_COUNT;
  if (err) atomicOr(p.status + f.out_index, err);
}

// ---- DC prediction: segmented inclusive scan over blocks in coefficient order; a head starts every (file, component) run
// and every restart interval.
__device__ __forceinline__ bool dc_head(const Params& p, long long g) {
  int lo = 0, hi = p.nfiles - 1;
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (p.files[mid].coef_base[0] <= g) lo = mid; else hi = mid - 1;
  }
  const FileDev& f = p.files[lo];
  int c = 0;
  while (c + 1 < f.ncomp && f.coef_base[c + 1] <= g) ++c;
  const long long local = g - f.coef_base[c];
  const int nb = f.h[c] * f.v[c];
  const long long mcu = local / nb;
  return local % nb == 0 && mcu % f.restart == 0;
}

struct DcPair {
  int v;
  int f;
};

__device__ __forceinline__ DcPair dc_combine(DcPair a, DcPair b) {
  return DcPair{b.f ? b.v : a.v + b.v, a.f | b.f};
}

__device__ __forceinline__ DcPair block_seg_scan(DcPair x, DcPair* total) {
  __shared__ int sv[32], sf[32];
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  DcPair inc = x;
  for (int o = 1; o < 32; o <<= 1) {
    DcPair y{__shfl_up_sync(0xffffffffu, inc.v, o), __shfl_up_sync(0xffffffffu, inc.f, o)};
    if (lane >= o) inc = dc_combine(y, inc);
  }
  if (lane == 31) { sv[wid] = inc.v; sf[wid] = inc.f; }
  __syncthreads();
  if (wid == 0) {
    DcPair w = lane < (blockDim.x >> 5) ? DcPair{sv[lane], sf[lane]} : DcPair{0, 0};
    for (int o = 1; o < 32; o <<= 1) {
      DcPair y{__shfl_up_sync(0xffffffffu, w.v, o), __shfl_up_sync(0xffffffffu, w.f, o)};
      if (lane >= o) w = dc_combine(y, w);
    }
    sv[lane] = w.v; sf[lane] = w.f;
  }
  __syncthreads();
  DcPair r = inc;
  if (wid) r = dc_combine(DcPair{sv[wid - 1], sf[wid - 1]}, inc);
  const int last = (blockDim.x >> 5) - 1;
  *total = DcPair{sv[last], sf[last]};
  __syncthreads();
  return r;
}

__global__ void __launch_bounds__(SCAN_CHUNK) jpeg_dc_local_kernel(Params p) {
  const long long g = blockIdx.x * static_cast<long long>(SCAN_CHUNK) + threadIdx.x;
  DcPair x{0, 0};
  if (g < p.nblocks) x = DcPair{p.coef[g * 64], dc_head(p, g) ? 1 : 0};
  DcPair total;
  const DcPair r = block_seg_scan(x, &total);
  if (g < p.nblocks) {
    p.coef[g * 64] = static_cast<int16_t>(r.v);
    p.dc_head[g] = static_cast<uint8_t>(r.f);
  }
  if (threadIdx.x == 0) { p.dc_agg[blockIdx.x] = total.v; p.dc_aggf[blockIdx.x] = total.f; }
}

// exclusive carry into every chunk (serial over chunks of 1024 aggregates, scanned in parallel)
__global__ void __launch_bounds__(SCAN_CHUNK) jpeg_dc_chunks_kernel(int* agg, int* aggf, long long n) {
  __shared__ int pv[SCAN_CHUNK], pf[SCAN_CHUNK];
  DcPair carry{0, 0};
  for (long long b = 0; b < n; b += SCAN_CHUNK) {
    const long long i = b + threadIdx.x;
    const DcPair x = i < n ? DcPair{agg[i], aggf[i]} : DcPair{0, 0};
    DcPair total;
    const DcPair inc = block_seg_scan(x, &total);
    pv[threadIdx.x] = inc.v; pf[threadIdx.x] = inc.f;
    __syncthreads();
    DcPair ex = carry;                                   // carry combined with everything before i in this round
    if (threadIdx.x) ex = dc_combine(carry, DcPair{pv[threadIdx.x - 1], pf[threadIdx.x - 1]});
    if (i < n) { agg[i] = ex.v; aggf[i] = ex.f; }
    carry = dc_combine(carry, total);
    __syncthreads();
  }
}

// ---- jidctint.c jpeg_idct_islow
constexpr int F0298 = 2446, F0390 = 3196, F0541 = 4433, F0765 = 6270, F0899 = 7373, F1175 = 9633, F1501 = 12299, F1847 = 15137,
              F1961 = 16069, F2053 = 16819, F2562 = 20995, F3072 = 25172;

template <int SHIFT>
__device__ __forceinline__ void idct_1d(const int x[8], int o[8]) {
  int z2 = x[2], z3 = x[6];
  int z1 = (z2 + z3) * F0541;
  const int tmp2 = z1 + z3 * -F1847;
  const int tmp3 = z1 + z2 * F0765;
  const int tmp0 = (x[0] + x[4]) * (1 << 13);
  const int tmp1 = (x[0] - x[4]) * (1 << 13);
  const int t10 = tmp0 + tmp3, t13 = tmp0 - tmp3, t11 = tmp1 + tmp2, t12 = tmp1 - tmp2;
  int a0 = x[7], a1 = x[5], a2 = x[3], a3 = x[1];
  z1 = a0 + a3; z2 = a1 + a2; z3 = a0 + a2;
  int z4 = a1 + a3;
  const int z5 = (z3 + z4) * F1175;
  a0 *= F0298; a1 *= F2053; a2 *= F3072; a3 *= F1501;
  z1 *= -F0899; z2 *= -F2562; z3 *= -F1961; z4 *= -F0390;
  z3 += z5; z4 += z5;
  a0 += z1 + z3; a1 += z2 + z4; a2 += z2 + z3; a3 += z1 + z4;
  constexpr int R = 1 << (SHIFT - 1);
  o[0] = (t10 + a3 + R) >> SHIFT; o[7] = (t10 - a3 + R) >> SHIFT;
  o[1] = (t11 + a2 + R) >> SHIFT; o[6] = (t11 - a2 + R) >> SHIFT;
  o[2] = (t12 + a1 + R) >> SHIFT; o[5] = (t12 - a1 + R) >> SHIFT;
  o[3] = (t13 + a0 + R) >> SHIFT; o[4] = (t13 - a0 + R) >> SHIFT;
}

__device__ __forceinline__ uint32_t range_limit(int x) {    // idct_table[x & RANGE_MASK]; a clamp on [-512, 511]
  const int v = x & 1023;
  return static_cast<uint32_t>(v < 128 ? v + 128 : v < 512 ? 255 : v < 896 ? 0 : v - 896);
}

__global__ void __launch_bounds__(128) jpeg_idct_kernel(Params p) {
  const long long g = blockIdx.x * 128LL + threadIdx.x;
  if (g >= p.nblocks) return;
  int lo = 0, hi = p.nfiles - 1;
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (p.files[mid].coef_base[0] <= g) lo = mid; else hi = mid - 1;
  }
  const FileDev& f = p.files[lo];
  int c = 0;
  while (c + 1 < f.ncomp && f.coef_base[c + 1] <= g) ++c;
  const uint16_t* q = f.quant[c];
  int16_t coef[64];
  const int4* src = reinterpret_cast<const int4*>(p.coef + g * 64);
#pragma unroll
  for (int k = 0; k < 8; ++k) *reinterpret_cast<int4*>(coef + 8 * k) = src[k];
  if (!p.dc_head[g]) coef[0] = static_cast<int16_t>(coef[0] + p.dc_agg[g / SCAN_CHUNK]);   // carry into the chunk
  int ws[64];
  bool out_of_range = false;
#pragma unroll
  for (int col = 0; col < 8; ++col) {
    int x[8], o[8];
#pragma unroll
    for (int r = 0; r < 8; ++r) {
      x[r] = coef[r * 8 + col] * static_cast<int>(q[r * 8 + col]);
      out_of_range |= x[r] < -IDCT_IN_MAX || x[r] > IDCT_IN_MAX;
    }
    idct_1d<13 - 2>(x, o);
#pragma unroll
    for (int r = 0; r < 8; ++r) {
      ws[r * 8 + col] = o[r];
      out_of_range |= o[r] < -IDCT_IN_MAX || o[r] > IDCT_IN_MAX;
    }
  }
  // block position in the component plane
  const long long local = g - f.coef_base[c];
  const int nb = f.h[c] * f.v[c];
  const long long mcu = local / nb;
  const int sub = static_cast<int>(local % nb);
  const int bx = static_cast<int>(mcu % f.mcux) * f.h[c] + sub % f.h[c];
  const int by = static_cast<int>(mcu / f.mcux) * f.v[c] + sub / f.h[c];
  const int pw = f.mcux * f.h[c] * 8;
  uint8_t* dst = p.planes + f.plane_off[c] + static_cast<long long>(by * 8) * pw + bx * 8;
#pragma unroll
  for (int r = 0; r < 8; ++r) {
    int o[8];
    idct_1d<13 + 2 + 3>(ws + r * 8, o);
#pragma unroll
    for (int k = 0; k < 8; ++k) out_of_range |= o[k] < IDCT_OUT_MIN || o[k] > IDCT_OUT_MAX;
    uint2 w;
    w.x = range_limit(o[0]) | (range_limit(o[1]) << 8) | (range_limit(o[2]) << 16) | (range_limit(o[3]) << 24);
    w.y = range_limit(o[4]) | (range_limit(o[5]) << 8) | (range_limit(o[6]) << 16) | (range_limit(o[7]) << 24);
    *reinterpret_cast<uint2*>(dst + static_cast<long long>(r) * pw) = w;
  }
  if (out_of_range) atomicOr(p.status + f.out_index, ST_IDCT_RANGE);
}

// ---- jdsample.c + jdcolor.c
__device__ __forceinline__ int chroma(const uint8_t* pl, int pw, int x, int y, int hm, int vm, int dw, int dh) {
  if (hm == 1) return pl[static_cast<long long>(y) * pw + x];
  if (dw <= 2) return pl[static_cast<long long>(y / vm) * pw + (x >> 1)];
  const int k = x >> 1;
  const int kp = k > 0 ? k - 1 : 0, kn = k + 1 < dw ? k + 1 : dw - 1;
  if (vm == 1) {                                          // h2v1_fancy_upsample
    const uint8_t* row = pl + static_cast<long long>(y) * pw;
    if (x == 0) return row[0];
    if (x == 2 * dw - 1) return row[dw - 1];
    return (x & 1) ? (3 * row[k] + row[kn] + 2) >> 2 : (3 * row[k] + row[kp] + 1) >> 2;
  }
  const int r = y >> 1;                                   // h2v2_fancy_upsample, edge rows repeated
  const int nbr = (y & 1) ? (r + 1 < dh ? r + 1 : dh - 1) : (r > 0 ? r - 1 : 0);
  const uint8_t* r0 = pl + static_cast<long long>(r) * pw;
  const uint8_t* r1 = pl + static_cast<long long>(nbr) * pw;
  const int sk = 3 * r0[k] + r1[k];
  if (x == 0) return (4 * sk + 8) >> 4;
  if (x == 2 * dw - 1) return (4 * sk + 7) >> 4;
  if (x & 1) return (3 * sk + 3 * r0[kn] + r1[kn] + 7) >> 4;
  return (3 * sk + 3 * r0[kp] + r1[kp] + 8) >> 4;
}

__device__ __forceinline__ uint8_t clamp255(int v) { return static_cast<uint8_t>(v < 0 ? 0 : v > 255 ? 255 : v); }

__global__ void __launch_bounds__(256) jpeg_color_kernel(Params p) {
  const long long t = blockIdx.x * 256LL + threadIdx.x;
  if (t >= p.npix) return;
  int lo = 0, hi = p.nfiles - 1;
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (p.files[mid].pix_base <= t) lo = mid; else hi = mid - 1;
  }
  const FileDev& f = p.files[lo];
  const long long px = t - f.pix_base;
  const int y = static_cast<int>(px / f.width), x = static_cast<int>(px % f.width);
  uint8_t* o = p.out[f.out_index] + px * 3;
  const int pw0 = f.mcux * f.h[0] * 8;
  const int Y = p.planes[f.plane_off[0] + static_cast<long long>(y) * pw0 + x];
  if (f.gray) {
    o[0] = o[1] = o[2] = static_cast<uint8_t>(Y);
    return;
  }
  const int pwc = f.mcux * 8;
  const int dw = (f.width + f.hmax - 1) / f.hmax, dh = (f.height + f.vmax - 1) / f.vmax;
  const int cb = chroma(p.planes + f.plane_off[1], pwc, x, y, f.hmax, f.vmax, dw, dh) - 128;
  const int cr = chroma(p.planes + f.plane_off[2], pwc, x, y, f.hmax, f.vmax, dw, dh) - 128;
  // build_ycc_rgb_table: FIX(1.40200) = 91881, FIX(1.77200) = 116130, FIX(0.71414) = 46802, FIX(0.34414) = 22554
  const int cr_r = (91881 * cr + 32768) >> 16;
  const int cb_b = (116130 * cb + 32768) >> 16;
  const int g = (-22554 * cb + 32768 + -46802 * cr) >> 16;
  o[0] = clamp255(Y + cr_r);
  o[1] = clamp255(Y + g);
  o[2] = clamp255(Y + cb_b);
}


// ------------------------------------------------------------------------------------------------------------- host plan
// routing reasons: OVG_JPEG_* in include/ovg.h, the same order as oracle/jpeg_oracle.py
enum Route { R_DEVICE, R_NOT_JPEG, R_TRUNCATED, R_PROCESS, R_PRECISION, R_COLOR, R_SAMPLING, R_SCANS, R_TABLES, R_MARKER,
             R_RESTART, R_SIZE };

struct HostSeg {
  long long byte_off, nbytes;                    // in the stream's data section
  const uint8_t* src;                            // unstuffed bytes, in Plan::file_data
  int file, first_mcu, n_mcu;
};

struct Plan {
  int subseq_bits = DEFAULT_SUBSEQ_BITS;
  std::vector<int> route, width, height, ncomp;
  std::vector<FileDev> files;                    // device-routed files
  std::vector<HostSeg> segs;
  std::vector<Huff> huffs;
  std::vector<std::vector<uint8_t>> file_data;   // unstuffed entropy data per device-routed file
  long long files_off = 0, segs_off = 0, huffs_off = 0, data_off = 0, stream_bytes = 0;
  long long nsub = 0, nblocks = 0, npix = 0, plane_bytes = 0;
  int rounds = 0;                                // sync rounds of the last decode
};

inline int be16(const uint8_t* d) { return (d[0] << 8) | d[1]; }

// jdhuff.c jpeg_make_d_derived_tbl; false where libjpeg would stop with an error
inline bool build_huff(const uint8_t* bits, const uint8_t* vals, bool dc, Huff* t) {
  std::memset(t, 0, sizeof(Huff));
  int code = 0, k = 0, total = 0;
  for (int l = 1; l <= 16; ++l) total += bits[l - 1];
  if (total > 256) return false;
  for (int l = 1; l <= 16; ++l) {
    t->valoff[l] = k - code;
    for (int i = 0; i < bits[l - 1]; ++i) {
      if (dc && vals[k] > 15) return false;
      if (l <= LUT_BITS)
        for (int j = code << (LUT_BITS - l); j < (code + 1) << (LUT_BITS - l); ++j)
          t->lut[j] = static_cast<uint16_t>((l << 8) | vals[k]);
      ++code;
      ++k;
    }
    if (code >= (1 << l)) return false;             // no code may be all ones
    t->maxcode[l] = bits[l - 1] ? code - 1 : -1;
    code <<= 1;
  }
  std::memcpy(t->val, vals, total);
  return true;
}

struct RawHuff {
  bool set = false;
  uint8_t bits[16];
  uint8_t vals[256];
};

struct Parsed {
  int route = R_NOT_JPEG;
  FileDev f;
  Huff h[6];
  std::vector<uint8_t> data;                     // unstuffed entropy data of all segments, back to back
  std::vector<long long> seg_end;                // end of each segment in `data`
};

// Parses one file into *out (route, frame, tables, unstuffed segments).
inline int parse_file(const uint8_t* d, long long n, Parsed* out) {
  static const int zigzag[64] = {0,  1,  8,  16, 9,  2,  3,  10, 17, 24, 32, 25, 18, 11, 4,  5,  12, 19, 26, 33, 40, 48,
                                 41, 34, 27, 20, 13, 6,  7,  14, 21, 28, 35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23,
                                 30, 37, 44, 51, 58, 59, 52, 45, 38, 31, 39, 46, 53, 60, 61, 54, 47, 55, 62, 63};
  FileDev* f = &out->f;
  Huff* hout = out->h;
  if (n < 4 || d[0] != 0xFF || d[1] != 0xD8) return R_NOT_JPEG;
  uint16_t quant[4][64];
  bool qset[4] = {false, false, false, false};
  RawHuff huff[2][4];
  bool jfif = false, adobe = false, sof = false;
  int transform = -1, restart = 0, width = 0, height = 0, nc = 0;
  int cid[4] = {0, 0, 0, 0}, ch[4] = {0, 0, 0, 0}, cv[4] = {0, 0, 0, 0}, ctq[4] = {0, 0, 0, 0};
  long long i = 2;
  for (;;) {
    if (i + 4 > n) return R_TRUNCATED;
    if (d[i] != 0xFF) return R_MARKER;
    while (i < n && d[i] == 0xFF) ++i;
    if (i + 3 > n) return R_TRUNCATED;
    const int m = d[i++];
    if (m == 0xD9) return R_SCANS;
    if ((m >= 0xD0 && m <= 0xD7) || m == 0x01) return R_MARKER;
    const int ln = be16(d + i);
    if (ln < 2 || i + ln > n) return R_TRUNCATED;
    const uint8_t* s = d + i + 2;
    const int sl = ln - 2;
    if (m == 0xE0 && sl >= 14 && std::memcmp(s, "JFIF\0", 5) == 0) {          // examine_app0: APP0_DATA_LEN bytes
      jfif = true;
    } else if (m == 0xEE && sl >= 12 && std::memcmp(s, "Adobe", 5) == 0) {
      adobe = true;
      transform = s[11];
    } else if ((m >= 0xE0 && m <= 0xEF) || m == 0xFE) {
    } else if (m == 0xDB) {                                             // get_dqt
      for (int k = 0; k < sl;) {
        const int pq = s[k] >> 4, tq = s[k] & 15, sz = pq ? 128 : 64;
        if (tq > 3 || k + 1 + sz > sl) return R_TABLES;
        for (int j = 0; j < 64; ++j) quant[tq][zigzag[j]] = pq ? be16(s + k + 1 + 2 * j) : s[k + 1 + j];
        qset[tq] = true;
        k += 1 + sz;
      }
    } else if (m == 0xC4) {                                             // get_dht
      for (int k = 0; k < sl;) {
        if (k + 17 > sl) return R_TABLES;
        const int tc = s[k] >> 4, th = s[k] & 15;
        int cnt = 0;
        for (int j = 0; j < 16; ++j) cnt += s[k + 1 + j];
        if (tc > 1 || th > 3 || cnt > 256 || k + 17 + cnt > sl) return R_TABLES;
        RawHuff& h = huff[tc][th];
        h.set = true;
        std::memcpy(h.bits, s + k + 1, 16);
        std::memcpy(h.vals, s + k + 17, cnt);
        k += 17 + cnt;
      }
    } else if (m == 0xDD) {                                             // get_dri
      if (ln != 4) return R_MARKER;
      restart = be16(s);
    } else if (m >= 0xC0 && m <= 0xCF && m != 0xC4 && m != 0xC8 && m != 0xCC) {   // get_sof
      if (sof) return R_MARKER;
      sof = true;
      if (m != 0xC0 && m != 0xC1) return R_PROCESS;
      if (sl < 6) return R_MARKER;
      if (s[0] != 8) return R_PRECISION;
      height = be16(s + 1);
      width = be16(s + 3);
      nc = s[5];
      if (sl != 6 + 3 * nc) return R_MARKER;
      for (int c = 0; c < nc && c < 4; ++c) {
        cid[c] = s[6 + 3 * c];
        ch[c] = s[7 + 3 * c] >> 4;
        cv[c] = s[7 + 3 * c] & 15;
        ctq[c] = s[8 + 3 * c];
      }
    } else if (m == 0xDA) {                                             // get_sos
      if (!sof) return R_MARKER;
      if (height == 0 || width == 0) return R_SIZE;
      if (nc == 3) {                                                    // jdapimin.c default_decompress_parms
        if (!jfif && adobe && transform == 0) return R_COLOR;
        if (!jfif && !adobe && ((cid[0] == 82 && cid[1] == 71 && cid[2] == 66) || (cid[0] == 1 && cid[1] == 0x22 && cid[2] == 0x23)))
          return R_COLOR;
        const bool y_ok = (ch[0] == 1 && cv[0] == 1) || (ch[0] == 2 && cv[0] == 1) || (ch[0] == 2 && cv[0] == 2);
        if (!y_ok || ch[1] != 1 || cv[1] != 1 || ch[2] != 1 || cv[2] != 1) return R_SAMPLING;
      } else if (nc == 1) {
        if (ch[0] < 1 || ch[0] > 4 || cv[0] < 1 || cv[0] > 4) return R_SAMPLING;
      } else {
        return R_COLOR;
      }
      const int ns = sl > 0 ? s[0] : -1;
      if (ns != nc || sl != 4 + 2 * ns) return R_SCANS;
      for (int c = 0; c < ns; ++c)
        if (s[1 + 2 * c] != cid[c]) return R_SCANS;
      if (s[1 + 2 * ns] != 0 || s[2 + 2 * ns] != 63 || s[3 + 2 * ns] != 0) return R_SCANS;
      for (int c = 0; c < ns; ++c) {
        const int dc = s[2 + 2 * c] >> 4, ac = s[2 + 2 * c] & 15;
        if (ctq[c] > 3 || !qset[ctq[c]] || dc > 3 || ac > 3 || !huff[0][dc].set || !huff[1][ac].set) return R_TABLES;
        if (!build_huff(huff[0][dc].bits, huff[0][dc].vals, true, hout + 2 * c) ||
            !build_huff(huff[1][ac].bits, huff[1][ac].vals, false, hout + 2 * c + 1))
          return R_TABLES;
        for (int j = 0; j < 64; ++j) f->quant[c][j] = quant[ctq[c]][j];
      }
      // frame geometry
      f->width = width; f->height = height; f->ncomp = nc; f->gray = nc == 1;
      if (nc == 1) {
        f->hmax = f->vmax = 1;
        f->h[0] = f->v[0] = 1;
        f->mcux = (width + 7) / 8;
        f->mcuy = (height + 7) / 8;
        f->nblk = 1;
        f->blk_comp[0] = 0; f->blk_sub[0] = 0;
      } else {
        f->hmax = ch[0]; f->vmax = cv[0];
        f->mcux = (width + 8 * f->hmax - 1) / (8 * f->hmax);
        f->mcuy = (height + 8 * f->vmax - 1) / (8 * f->vmax);
        int b = 0;
        for (int c = 0; c < 3; ++c) {
          f->h[c] = ch[c]; f->v[c] = cv[c];
          for (int j = 0; j < ch[c] * cv[c]; ++j) { f->blk_comp[b] = c; f->blk_sub[b] = j; ++b; }
        }
        f->nblk = b;
      }
      const long long nmcu = static_cast<long long>(f->mcux) * f->mcuy;
      f->restart = restart ? restart : static_cast<int>(nmcu);
      // entropy data: one memchr-driven pass, FF 00 -> FF, RST markers split the segments
      std::vector<int> rsts;
      long long p = i + ln;
      out->data.resize(n - p);
      uint8_t* w = out->data.data();
      long long wn = 0;
      for (;;) {
        const uint8_t* q = static_cast<const uint8_t*>(std::memchr(d + p, 0xFF, n - p));
        if (!q || q + 1 >= d + n) return R_TRUNCATED;
        const long long j = q - d;
        std::memcpy(w + wn, d + p, j - p);
        wn += j - p;
        const int mk = d[j + 1];
        if (mk == 0) {
          w[wn++] = 0xFF;
          p = j + 2;
        } else if (mk >= 0xD0 && mk <= 0xD7) {
          rsts.push_back(mk - 0xD0);
          out->seg_end.push_back(wn);
          p = j + 2;
        } else if (mk == 0xFF) {
          return R_TRUNCATED;
        } else {
          if (mk != 0xD9) return (mk == 0xDA || mk == 0xDC || (mk >= 0xC0 && mk <= 0xFE)) ? R_SCANS : R_MARKER;
          out->seg_end.push_back(wn);
          out->data.resize(wn);
          break;
        }
      }
      const long long want = restart ? (nmcu + restart - 1) / restart : 1;
      if (static_cast<long long>(out->seg_end.size()) != want) return R_RESTART;
      for (size_t k = 0; k < rsts.size(); ++k)
        if (rsts[k] != static_cast<int>(k % 8)) return R_RESTART;
      return R_DEVICE;
    } else {
      return R_MARKER;
    }
    i += ln;
  }
}

inline long long align_up(long long x, long long a) { return (x + a - 1) / a * a; }

// Fills *P.  Throws std::bad_alloc when memory runs out (also inside a worker thread); fewer threads are used when they
// cannot be started.
inline void plan_build(Plan* P, const uint8_t* const* bufs, const long long* nbytes, int n, int subseq_bits) {
  P->subseq_bits = subseq_bits ? subseq_bits : DEFAULT_SUBSEQ_BITS;
  P->route.assign(n, R_NOT_JPEG);
  P->width.assign(n, 0);
  P->height.assign(n, 0);
  P->ncomp.assign(n, 0);
  // files are independent: parse and unstuff them on several host threads
  std::vector<Parsed> parsed(n);
  std::atomic<int> next{0};
  std::atomic<bool> failed{false};
  auto work = [&] {
    for (int i; (i = next.fetch_add(1)) < n;) {
      try {
        std::memset(&parsed[i].f, 0, sizeof(FileDev));
        parsed[i].route = bufs[i] ? parse_file(bufs[i], nbytes[i], &parsed[i]) : R_NOT_JPEG;
      } catch (...) {
        failed = true;
      }
      if (parsed[i].route != R_DEVICE) {
        parsed[i].data = std::vector<uint8_t>();
        parsed[i].seg_end.clear();
      }
    }
  };
  const int nt = std::max(1, std::min<int>(n, static_cast<int>(std::thread::hardware_concurrency())));
  std::vector<std::thread> pool;
  try {
    pool.reserve(nt);
    for (int t = 1; t < nt; ++t) pool.emplace_back(work);
  } catch (...) {                                // run with the threads that did start
  }
  work();
  for (std::thread& t : pool) t.join();
  if (failed) throw std::bad_alloc();
  long long coef = 0, plane = 0, pix = 0, bytes = 0;
  for (int i = 0; i < n; ++i) {
    Parsed& q = parsed[i];
    P->route[i] = q.route;
    if (q.route != R_DEVICE) continue;
    FileDev f = q.f;
    P->width[i] = f.width;
    P->height[i] = f.height;
    P->ncomp[i] = f.ncomp;
    f.out_index = i;
    for (int c = 0; c < f.ncomp; ++c) {
      f.huff_dc[c] = static_cast<int>(P->huffs.size());
      P->huffs.push_back(q.h[2 * c]);
      f.huff_ac[c] = static_cast<int>(P->huffs.size());
      P->huffs.push_back(q.h[2 * c + 1]);
      const long long nb = static_cast<long long>(f.mcux) * f.mcuy * f.h[c] * f.v[c];
      f.coef_base[c] = coef;
      coef += nb;
      f.plane_off[c] = plane;
      plane = align_up(plane + nb * 64, 256);
    }
    f.pix_base = pix;
    pix += static_cast<long long>(f.width) * f.height;
    const int fi = static_cast<int>(P->files.size());
    const long long nmcu = static_cast<long long>(f.mcux) * f.mcuy;
    long long from = 0;
    for (size_t k = 0; k < q.seg_end.size(); ++k) {
      HostSeg s;
      s.byte_off = bytes;
      s.nbytes = q.seg_end[k] - from;
      s.src = q.data.data() + from;
      s.file = fi;
      s.first_mcu = static_cast<int>(k * f.restart);
      s.n_mcu = static_cast<int>(std::min<long long>(f.restart, nmcu - s.first_mcu));
      bytes = align_up(bytes + s.nbytes + SEG_PAD, SEG_ALIGN);
      from = q.seg_end[k];
      P->segs.push_back(s);
    }
    P->files.push_back(f);
    P->file_data.push_back(std::move(q.data));   // the vector's heap buffer (and the segments' src pointers) move along
  }
  P->nblocks = coef;
  P->plane_bytes = plane;
  P->npix = pix;
  long long nsub = 0;
  for (const HostSeg& s : P->segs) nsub += std::max<long long>(1, (8 * s.nbytes + P->subseq_bits - 1) / P->subseq_bits);
  P->nsub = nsub;
  P->files_off = 0;
  P->segs_off = align_up(P->files.size() * sizeof(FileDev), 256);
  P->huffs_off = align_up(P->segs_off + P->segs.size() * sizeof(SegDev), 256);
  P->data_off = align_up(P->huffs_off + P->huffs.size() * sizeof(Huff), 256);
  P->stream_bytes = P->data_off + bytes;
}

inline void plan_fill(const Plan* P, uint8_t* dst) {
  std::memset(dst, 0, P->data_off);
  if (!P->files.empty()) std::memcpy(dst + P->files_off, P->files.data(), P->files.size() * sizeof(FileDev));
  SegDev* sd = reinterpret_cast<SegDev*>(dst + P->segs_off);
  long long sub = 0;
  for (size_t k = 0; k < P->segs.size(); ++k) {
    const HostSeg& s = P->segs[k];
    SegDev g;
    g.bit_start = 8 * s.byte_off;
    g.nbits = 8 * s.nbytes;
    g.first_sub = sub;
    g.file = s.file;
    g.first_mcu = s.first_mcu;
    g.n_mcu = s.n_mcu;
    g.n_sub = static_cast<int>(std::max<long long>(1, (g.nbits + P->subseq_bits - 1) / P->subseq_bits));
    sub += g.n_sub;
    std::memcpy(sd + k, &g, sizeof(g));
  }
  if (!P->huffs.empty()) std::memcpy(dst + P->huffs_off, P->huffs.data(), P->huffs.size() * sizeof(Huff));
  for (size_t k = 0; k < P->segs.size(); ++k) {
    const HostSeg& s = P->segs[k];
    const long long end = k + 1 < P->segs.size() ? P->segs[k + 1].byte_off : P->stream_bytes - P->data_off;
    uint8_t* o = dst + P->data_off + s.byte_off;
    std::memcpy(o, s.src, s.nbytes);
    std::memset(o + s.nbytes, 0, end - s.nbytes - s.byte_off);
  }
}

struct Workspace {
  uint32_t* exits;
  uint32_t* counts;
  unsigned long long* pre;
  unsigned long long* chunk;
  int16_t* coef;
  int* dc_agg;
  int* dc_aggf;
  uint8_t* dc_head;
  uint8_t* planes;
  uint8_t** out;
  int* changed;
};

inline Workspace plan_layout(Arena& ar, const Plan* P, int nout) {
  Workspace w;
  auto take = [&](long long bytes) { return static_cast<uint8_t*>(ar.take(std::max<long long>(bytes, 1))); };
  const long long nsub_chunks = (P->nsub + SCAN_CHUNK - 1) / SCAN_CHUNK;
  const long long nblk_chunks = (P->nblocks + SCAN_CHUNK - 1) / SCAN_CHUNK;
  w.exits = reinterpret_cast<uint32_t*>(take(4 * P->nsub));
  w.counts = reinterpret_cast<uint32_t*>(take(4 * P->nsub));
  w.pre = reinterpret_cast<unsigned long long*>(take(8 * P->nsub));
  w.chunk = reinterpret_cast<unsigned long long*>(take(8 * nsub_chunks));
  w.coef = reinterpret_cast<int16_t*>(take(128 * P->nblocks));
  w.dc_agg = reinterpret_cast<int*>(take(4 * nblk_chunks));
  w.dc_aggf = reinterpret_cast<int*>(take(4 * nblk_chunks));
  w.dc_head = take(P->nblocks);
  w.planes = take(P->plane_bytes);
  w.out = reinterpret_cast<uint8_t**>(take(8LL * nout));
  w.changed = reinterpret_cast<int*>(take(4));
  return w;
}

}  // namespace jpg
}  // namespace ovg
