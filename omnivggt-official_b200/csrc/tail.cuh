// Fused DPT output tail (reference heads/dpt_head.py:242-260, heads/head_act.py:61-125):
//   bilinear resize (align_corners) of the output_conv1 map to the image size + UV position embedding
//   -> 3x3 conv 128 -> 32 -> ReLU -> 1x1 conv 32 -> outc -> exp / inverse-log / 1+exp  (fp32 NHWC predictions).
// The full-resolution 128-channel map (550 MB per head and 8 frames at 518^2) is never written: producer warps interpolate one
// image row of a 128-pixel column strip at a time straight into the swizzled shared-memory A operand of the tensor core.
//
// One CTA walks DOWN a strip, one input row per step.  An input row r contributes to the three output rows r-1, r, r+1 (kernel rows
// ky = 2, 1, 0), so ONE N = 96 wgmma per (kx, k-step) computes [W_ky=2 | W_ky=1 | W_ky=0] x row r: the A row block (136 x 64 halves)
// is read from shared memory once per kx instead of once per (ky, kx).  The three 32-column blocks of that product go into three
// register accumulators: output row r-1 is finished (and drained by the epilogue), the partial sums of rows r and r+1 move up.
//
// Roles (640 threads, one CTA per SM, 222 KB of shared memory):
//   warp 0        loads the 72 KB of weights once (TMA);
//   warps 1-3, 12-19 (352 threads) producers: one thread bulk-copies the strip's source rows into a 4-row ring two rows ahead of use,
//                 all of them blend vertically + horizontally (fp32) and write the swizzled A stage (2 stages);
//   warps 4-11    two consumer warpgroups, 64 strip pixels each: wgmma, then the epilogue on the finished row in registers:
//                 + bias + conv(position embedding) tables (the convolution is linear: its image under the 3x3 kernel separates into
//                 gx[row class][x] + gy[column class][y], tail_tables_kernel) -> ReLU -> 1x1 (quad shuffles) -> activations.
// Work items: (frame, strip, segment of rows) with two halo rows per segment, about three per SM.
#pragma once
#include "ptx.cuh"

namespace ovg {

struct TailParams {
  const uint16_t* src;  // [F, h+2, w+2, 128] zero-bordered 16-bit map (output_conv1)
  const float* gx;      // [3, W, 32] conv of the x half of the position embedding (tail_tables_kernel) or nullptr
  const float* gy;      // [3, H, 32] ... of the y half
  const float* bias;    // [32]
  const float* w2;      // [outc, 32]
  const float* b2;      // [outc]
  float* preds;         // [F, H, W, outc-1]
  float* conf;          // [F, H, W]
  int F, h, w, H, W;
  float sy, sx;
  int outc, head_act, f16;
  int n_strips, n_segs, seg_rows, n_items;
};

constexpr int FT_THREADS = 640;                 // warp 0: weights; warps 4-11: wgmma + epilogue; warps 1-3 and 12-19: producers
constexpr int FT_PROD_THREADS = 352;
constexpr int FT_PROD_GROUPS = FT_PROD_THREADS / 16;   // 22 groups of 16 channel vectors
constexpr int FT_IPT = 4;                       // consecutive source intervals per producer thread (22 x 4 >= 80)
constexpr int FT_A_KB_BYTES = 136 * 128;        // one K block (64 channels) of a row block: 17 swizzle atoms
constexpr int FT_A_STAGE = 2 * FT_A_KB_BYTES;
constexpr int FT_A_STAGES = 2;
constexpr int FT_A_ROWS = 130;                  // pixels x0-1 .. x0+128
constexpr int FT_B_TILE = 96 * 128;             // [96 x 64] weights of one (kx, K block): rows (ky = 2 | 1 | 0, oc)
constexpr int FT_B_BYTES = 6 * FT_B_TILE;
constexpr int FT_VBUF_PX = 80;                  // source pixels a strip spans
constexpr int FT_RING = 4;                      // source rows resident per CTA (two in use, two in flight)
constexpr int FT_RAW_ROW = FT_VBUF_PX * 256;    // one source row of the strip, 16-bit, 128 channels
constexpr int FT_ITAB_BYTES = FT_VBUF_PX * 4;      // per source pixel of the strip: first strip row it feeds | count << 16
constexpr int FT_W_BYTES = (32 + 4 * 32 + 4) * 4;  // bias | w2 | b2 of the epilogue (broadcast reads)
constexpr int FT_SMEM_BYTES = FT_A_STAGES * FT_A_STAGE + FT_B_BYTES + FT_RING * FT_RAW_ROW + FT_ITAB_BYTES + FT_W_BYTES + 1024 + 512;

__device__ __forceinline__ void ft_prod_sync() { asm volatile("bar.sync 1, 352;" ::: "memory"); }
__device__ __forceinline__ uint4 ft_lds128(uint32_t a) {
  uint4 r;
  asm volatile("ld.shared.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w) : "r"(a));
  return r;
}
__device__ __forceinline__ void ft_sts128(uint32_t a, uint4 v) {
  asm volatile("st.shared.v4.u32 [%0], {%1,%2,%3,%4};" ::"r"(a), "r"(v.x), "r"(v.y), "r"(v.z), "r"(v.w) : "memory");
}

// waits of the roles that are ahead of the pipeline most of the time: back off so the spin does not take issue slots from the producers
__device__ __forceinline__ void ft_wait_idle(uint64_t* bar, uint32_t parity) {
  if (mbar_try_wait(bar, parity)) return;
  long long t0 = clock64();
  uint32_t spins = 0;
  while (!mbar_try_wait(bar, parity)) {
    __nanosleep(40);
    if ((++spins & 0x3ff) == 0 && clock64() - t0 > 8000000000LL) __trap();
  }
}

// Epilogue of one finished output row y for this thread's two pixels (rows h = 0, 1 of its accumulator fragment) and eight
// channels (8 jj + fcol + c): + bias + position-embedding tables -> ReLU -> 1x1 conv (partial dots reduced over the quad of
// threads that share a pixel) -> activations; lane fcol / 2 == h writes pixel h.
__device__ __forceinline__ void ft_epilogue_row(const TailParams& p, const float* acc, const float* sw,
                                                const int y, const int f, const int (&X)[2], const int fcol, const int lane) {
  const int q = lane & 3;
  float res[2][4];
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const int Xc = X[h] < p.W ? X[h] : p.W - 1;
    float v[8];
#pragma unroll
    for (int jj = 0; jj < 4; ++jj)
#pragma unroll
      for (int c = 0; c < 2; ++c) v[2 * jj + c] = acc[4 * jj + 2 * h + c] + sw[8 * jj + fcol + c];
    if (p.gx) {
      const int xcls = Xc == 0 ? 0 : (Xc == p.W - 1 ? 2 : 1);
      const float* gy = p.gy + (static_cast<size_t>(xcls) * p.H + y) * 32 + fcol;
      const int ycls = y == 0 ? 0 : (y == p.H - 1 ? 2 : 1);
      const float* gx = p.gx + (static_cast<size_t>(ycls) * p.W + Xc) * 32 + fcol;   // interior rows: the same row for every y (L1)
#pragma unroll
      for (int jj = 0; jj < 4; ++jj) {
        const float2 t = __ldg(reinterpret_cast<const float2*>(gy + 8 * jj));
        const float2 u = __ldg(reinterpret_cast<const float2*>(gx + 8 * jj));
        v[2 * jj] += t.x + u.x;
        v[2 * jj + 1] += t.y + u.y;
      }
    }
#pragma unroll
    for (int o = 0; o < 4; ++o) {
      float a = 0.f;
#pragma unroll
      for (int jj = 0; jj < 4; ++jj)
#pragma unroll
        for (int c = 0; c < 2; ++c) a = fmaf(sw[32 + o * 32 + 8 * jj + fcol + c], fmaxf(v[2 * jj + c], 0.f), a);
      a += __shfl_xor_sync(0xffffffffu, a, 1);
      a += __shfl_xor_sync(0xffffffffu, a, 2);
      res[h][o] = a + sw[160 + o];
    }
  }
  if (q >= 2) return;
  if (X[q] >= p.W) return;                               // columns past the image
  const long long pix = (static_cast<long long>(f) * p.H + y) * p.W + X[q];
#pragma unroll
  for (int o = 0; o < 4; ++o) {
    if (o < p.outc) {
      const float a = res[q][o];
      if (o == p.outc - 1) {
        p.conf[pix] = 1.0f + expf(a);
      } else {
        p.preds[pix * (p.outc - 1) + o] = p.head_act == 0 ? expf(a) : copysignf(expm1f(fabsf(a)), a);
      }
    }
  }
}

template <bool F16>
__global__ void __launch_bounds__(FT_THREADS, 1)
fusedtail_kernel(const __grid_constant__ CUtensorMap tmB, const TailParams p) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* sA = smem;
  uint8_t* sB = sA + FT_A_STAGES * FT_A_STAGE;
  uint8_t* ring = sB + FT_B_BYTES;
  int* itab = reinterpret_cast<int*>(ring + FT_RING * FT_RAW_ROW);
  float* sw = reinterpret_cast<float*>(reinterpret_cast<uint8_t*>(itab) + FT_ITAB_BYTES);
  uint64_t* bars = reinterpret_cast<uint64_t*>(reinterpret_cast<uint8_t*>(sw) + FT_W_BYTES);
  uint64_t* a_full = bars;         // [2]  producers (11 warps) -> consumers
  uint64_t* a_empty = bars + 2;    // [2]  consumers (8 warps) -> producers
  uint64_t* bfull = bars + 4;
  uint64_t* r_full = bars + 5;     // [FT_RING] bulk copies of source rows

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmB);
    for (int i = 0; i < 2; ++i) {
      mbar_init(&a_full[i], FT_PROD_THREADS / 32);
      mbar_init(&a_empty[i], 8);
    }
    mbar_init(bfull, 1);
    for (int i = 0; i < FT_RING; ++i) mbar_init(&r_full[i], 1);
    fence_barrier_init();
  }
  if (threadIdx.x >= 128 && threadIdx.x < 128 + 32 + 4 * 32 + 4) {
    const int i = threadIdx.x - 128;
    sw[i] = i < 32 ? p.bias[i] : (i < 160 ? (i - 32 < p.outc * 32 ? p.w2[i - 32] : 0.f) : (i - 160 < p.outc ? p.b2[i - 160] : 0.f));
  }
  __syncthreads();
  // Registers: 96 per thread for every role (640 threads; no setmaxnreg).  The consumers hold 80 accumulator registers (this
  // row's product and the partial sums of the next two output rows), and ptxas spills about 180 B per thread at this budget.
  // Moving registers to the consumers does not remove that: the producers then need more than the 64-72 registers left for them
  // (ptxas ignores the split) or spill themselves at 80, and a 512-thread layout with 128 registers for everyone still spills.

#define OVG_FT_ITEM(item)                                        \
  const int seg = (item) % p.n_segs;                             \
  const int strip = ((item) / p.n_segs) % p.n_strips;            \
  const int f = (item) / (p.n_segs * p.n_strips);                \
  const int ya = seg * p.seg_rows;                               \
  const int yb = ya + p.seg_rows < p.H ? ya + p.seg_rows : p.H;  \
  const int x0 = strip * 128;

  if (warp == 0) {
    // ===================== weights (once) =====================
    if (lane == 0) {
      mbar_expect_tx(bfull, FT_B_BYTES);
      for (int kx = 0; kx < 3; ++kx)
        for (int kb = 0; kb < 2; ++kb)
          for (int s = 0; s < 3; ++s)        // slot s holds kernel row ky = 2 - s
            tma_load_2d(sB + (kx * 2 + kb) * FT_B_TILE + s * 4096, &tmB, bfull, ((2 - s) * 3 + kx) * 128 + kb * 64, 0);
    }
  } else if (warp >= 4 && warp < 12) {
    // ===================== wgmma + epilogue: 64 strip pixels per warpgroup =====================
    const int cw = (warp >> 2) - 1;
    const int prow = cw * 64 + (warp & 3) * 16 + (lane >> 2);   // strip pixels prow, prow + 8
    const int fcol = 2 * (lane & 3);
    mbar_wait_quiet(bfull, 0);
    int st = 0;
    uint32_t aph = 0;
    for (int item = blockIdx.x; item < p.n_items; item += gridDim.x) {
      OVG_FT_ITEM(item)
      const int X[2] = {x0 + prow, x0 + prow + 8};
      float p1[16], p2[16];                   // partial sums of output rows r and r + 1
#pragma unroll
      for (int i = 0; i < 16; ++i) p1[i] = p2[i] = 0.f;
      for (int r = ya - 1; r <= yb; ++r) {
        float d[48];
        if (r >= 0 && r < p.H) {
          mbar_wait_quiet(&a_full[st], aph);
          wgmma_fence();
#pragma unroll
          for (int kb = 0; kb < 2; ++kb) {
            const uint32_t a_atom = smem_u32(sA + st * FT_A_STAGE + kb * FT_A_KB_BYTES + cw * 64 * 128);
#pragma unroll
            for (int kx = 0; kx < 3; ++kx) {
              const uint64_t adesc = make_sw128_desc_rows(a_atom, kx);
              const uint64_t bdesc = make_sw128_desc(smem_u32(sB + (kx * 2 + kb) * FT_B_TILE));
#pragma unroll
              for (int k = 0; k < 4; ++k) wgmma_ss<96, F16>(d, adesc + 2 * k, bdesc + 2 * k, (kb | kx | k) != 0);
            }
          }
          wgmma_commit();
          wgmma_wait<0>();
          fence_regs<48>(d);
          __syncwarp();
          if (lane == 0) mbar_arrive(&a_empty[st]);
          if (++st == FT_A_STAGES) {
            st = 0;
            aph ^= 1;
          }
        } else {
#pragma unroll
          for (int i = 0; i < 48; ++i) d[i] = 0.f;   // zero padding above / below the image
        }
        // d = [ky = 2 -> row r-1 | ky = 1 -> row r | ky = 0 -> row r+1], 16 registers per 32-column block
#pragma unroll
        for (int i = 0; i < 16; ++i) {
          d[i] += p1[i];
          p1[i] = p2[i] + d[16 + i];
          p2[i] = d[32 + i];
        }
        const int y = r - 1;
        if (y >= ya && y < yb) ft_epilogue_row(p, d, sw, y, f, X, fcol, lane);
      }
    }
  } else {
    // ===================== producers (11 warps): interpolate one strip row into the swizzled A operand =====================
    // Source rows of the strip (<= 80 pixels x 128 channels, 16-bit) are bulk-copied (cp.async.bulk, one thread) into a ring of four
    // rows, two rows ahead of their first use, so no thread ever waits on a global load.  Thread (v, grp): 16-byte channel vector
    // v = 8 channels, FT_IPT consecutive source intervals [s, s+1).  Per image row it loads the texels of its FT_IPT + 1 source
    // pixels from both source rows once, blends them vertically (fp32), and emits the 1-2 strip pixels inside each interval
    // (itab): horizontal blend, pack to 16 bits, store with the 128-byte swizzle (row = pixel, chunk ^ (row & 7)).  The position
    // embedding is not added here: the convolution is linear, its image under the 3x3 kernel is a per-shape table that the
    // epilogue adds in fp32.
    const int ptid = warp < 4 ? (warp - 1) * 32 + lane : (warp - 9) * 32 + lane;      // 0 .. 351
    const int v = ptid & 15, grp = ptid >> 4;
    int st = 0, pcnt = 0;
    uint32_t eph = 0, loaded = 0;                       // `loaded`: source rows copied so far (ring slot = index % FT_RING)
    const int ws = p.w + 2;
    const uint32_t ring_s = smem_u32(ring) + v * 16, itab_s = smem_u32(itab);
    const uint32_t vsw = static_cast<uint32_t>(v & 7);
    for (int item = blockIdx.x; item < p.n_items; item += gridDim.x) {
      OVG_FT_ITEM(item)
      const int x_lo = x0 - 1 > 0 ? x0 - 1 : 0;
      const int x_hi = x0 + 128 < p.W - 1 ? x0 + 128 : p.W - 1;
      const int xs_lo = static_cast<int>(p.sx * x_lo);
      int xs_hi = static_cast<int>(p.sx * x_hi) + 1;
      if (xs_hi > p.w - 1) xs_hi = p.w - 1;
      const int ns = xs_hi - xs_lo + 1;
      // strip pixels of every source interval: X in [x_lo, x_hi] with floor(sx * X) == s, consecutive because sx <= 1
      if (ptid < FT_VBUF_PX) {
        int packed = 0;
        if (ptid < ns) {
          const int sabs = xs_lo + ptid;
          int Xg = static_cast<int>(static_cast<float>(sabs) / p.sx) - 2;
          if (Xg < x_lo) Xg = x_lo;
          while (Xg <= x_hi && static_cast<int>(p.sx * Xg) < sabs) ++Xg;
          int n = 0;
          while (Xg + n <= x_hi && static_cast<int>(p.sx * (Xg + n)) == sabs) ++n;
          packed = (Xg - (x0 - 1)) | (n << 16);
        }
        itab[ptid] = packed;                             // intervals past the strip: no pixels
      }
      const int r_first = ya - 1 > 0 ? ya - 1 : 0;
      const int r_last = yb < p.H - 1 ? yb : p.H - 1;
      const int zrow = p.W - x0 + 1;                     // strip row of the zero column right of the image
      const int y_first = static_cast<int>(p.sy * r_first);
      int y_end = static_cast<int>(p.sy * r_last) + 1;
      if (y_end > p.h - 1) y_end = p.h - 1;
      const uint32_t lbase = loaded;
      const uint32_t row_bytes = static_cast<uint32_t>(ns) * 256u;
      const uint16_t* fsrc = p.src + (static_cast<size_t>(f) * (p.h + 2) * ws + ws + 1 + xs_lo) * 128;   // source pixel (0, xs_lo)
      int next_y = y_first;
      auto copy_rows = [&](int upto) {                   // thread 0: bulk-copy source rows next_y .. min(upto, y_end)
        for (; next_y <= upto && next_y <= y_end; ++next_y) {
          const uint32_t l = lbase + static_cast<uint32_t>(next_y - y_first);
          uint64_t* bar = &r_full[l % FT_RING];
          mbar_expect_tx(bar, row_bytes);
          bulk_load_1d(ring + (l % FT_RING) * FT_RAW_ROW, fsrc + static_cast<size_t>(next_y) * ws * 128, row_bytes, bar);
        }
      };
      if (ptid == 0) copy_rows(y_first + FT_RING - 1);
      ft_prod_sync();                                    // itab visible; every thread is done with the previous item's rows
      // this thread's intervals: s = grp * FT_IPT + j; pixel offsets (bytes) of its FT_IPT + 1 source pixels, the last one clamped
      const int s_first = grp * FT_IPT;
      int pk[FT_IPT];
#pragma unroll
      for (int j = 0; j < FT_IPT; ++j) {
        uint32_t t;
        asm volatile("ld.shared.u32 %0, [%1];" : "=r"(t) : "r"(itab_s + (s_first + j < FT_VBUF_PX ? s_first + j : 0) * 4));
        pk[j] = s_first + j < ns ? static_cast<int>(t) : 0;
      }
      for (int r = r_first; r <= r_last; ++r, ++pcnt) {
        const float fy = p.sy * r;
        const int y0 = static_cast<int>(fy);
        const int y1 = y0 + (y0 < p.h - 1 ? 1 : 0);
        const float wy1 = fy - y0, wy0 = 1.f - wy1;
        const float2 wy0_2 = make_float2(wy0, wy0), wy1_2 = make_float2(wy1, wy1);
        const uint32_t l0 = lbase + static_cast<uint32_t>(y0 - y_first), l1 = lbase + static_cast<uint32_t>(y1 - y_first);
        mbar_wait_quiet(&r_full[l0 % FT_RING], (l0 / FT_RING) & 1);
        mbar_wait_quiet(&r_full[l1 % FT_RING], (l1 / FT_RING) & 1);
        const uint32_t ra = ring_s + (l0 % FT_RING) * FT_RAW_ROW, rb = ring_s + (l1 % FT_RING) * FT_RAW_ROW;
        mbar_wait_quiet(&a_empty[st], eph ^ 1);     // the MMAs that read this stage two rows ago have completed
        const uint32_t stage = smem_u32(sA) + st * FT_A_STAGE + (v >> 3) * FT_A_KB_BYTES;
        // zero columns left / right of the image (conv padding)
        if (x0 == 0 && grp == 20) ft_sts128(stage + (vsw << 4), make_uint4(0, 0, 0, 0));
        if (zrow < FT_A_ROWS && grp == 21) ft_sts128(stage + zrow * 128 + ((vsw ^ (zrow & 7)) << 4), make_uint4(0, 0, 0, 0));
        if (s_first < ns) {
          float2 va[4], vb[4];
          auto blend = [&](int s_, float2 (&o)[4]) {       // vertical blend of source pixel s_ (clamped to the strip)
            const int sc = s_ < ns ? s_ : ns - 1;
            const uint4 t0 = ft_lds128(ra + sc * 256), t1 = ft_lds128(rb + sc * 256);
            const uint32_t* p0 = &t0.x;
            const uint32_t* p1 = &t1.x;
#pragma unroll
            for (int k = 0; k < 4; ++k) o[k] = ffma2(wy1_2, unpack_h(p1[k], F16), fmul2(wy0_2, unpack_h(p0[k], F16)));
          };
          blend(s_first, va);
#pragma unroll
          for (int j = 0; j < FT_IPT; ++j) {
            blend(s_first + j + 1, vb);
            const int row0 = pk[j] & 0xffff, n = pk[j] >> 16;
            const float sbase = static_cast<float>(xs_lo + s_first + j);
            auto emit = [&](int row) {
              const float wx1 = p.sx * (x0 - 1 + row) - sbase, wx0 = 1.f - wx1;
              const float2 w0 = make_float2(wx0, wx0), w1 = make_float2(wx1, wx1);
              const float2 q0 = ffma2(w1, vb[0], fmul2(w0, va[0]));
              const float2 q1 = ffma2(w1, vb[1], fmul2(w0, va[1]));
              const float2 q2 = ffma2(w1, vb[2], fmul2(w0, va[2]));
              const float2 q3 = ffma2(w1, vb[3], fmul2(w0, va[3]));
              uint4 out;
              out.x = pack_h(q0.x, q0.y, F16);
              out.y = pack_h(q1.x, q1.y, F16);
              out.z = pack_h(q2.x, q2.y, F16);
              out.w = pack_h(q3.x, q3.y, F16);
              ft_sts128(stage + row * 128 + ((vsw ^ (row & 7)) << 4), out);
            };
            if (n > 0) emit(row0);
            if (n > 1) emit(row0 + 1);
            for (int k = 2; k < n; ++k) emit(row0 + k);      // upsampling factors above 2
#pragma unroll
            for (int k = 0; k < 4; ++k) va[k] = vb[k];
          }
        }
        fence_proxy_async();
        __syncwarp();
        if (lane == 0) mbar_arrive(&a_full[st]);
        if (++st == FT_A_STAGES) {
          st = 0;
          eph ^= 1;
        }
        ft_prod_sync();                              // every thread has read the source rows of image row r
        if (ptid == 0 && r < r_last) copy_rows(static_cast<int>(p.sy * (r + 1)) + FT_RING - 1);   // slots below y0(r+1) are free
      }
      loaded = lbase + static_cast<uint32_t>(y_end - y_first + 1);
    }
  }
#undef OVG_FT_ITEM
}

// Image of the UV position embedding (heads/dpt_head.py:249-250, separable: channels [0, 64) depend on x, [64, 128) on y) under
// the 3x3 convolution with zero padding, split by linearity:  conv(E)[y, x, oc] = gx[rc(y)][x][oc] + gy[cc(x)][y][oc], where the row
// class rc (0: y = 0, 1: interior, 2: y = H-1) selects the kernel rows that fall inside the image for the x part, and the column
// class cc likewise for the y part.  Weights are the 16-bit operands the MMA uses, widened to fp32.  Grid (max(W, H), 2) x 96.
struct TailTableParams {
  const float* tx;       // [W, 64]
  const float* ty;       // [H, 64]
  const uint16_t* w;     // [32, 9 * 128]  K order (ky, kx, c)
  float* gx;             // [3, W, 32]
  float* gy;             // [3, H, 32]
  int H, W, f16;
};
__global__ void __launch_bounds__(96) tail_tables_kernel(const TailTableParams p) {
  // block = one table position, thread = (class, output channel); 16-byte loads, four independent accumulators
  const int oc = threadIdx.x & 31, cls = threadIdx.x >> 5, part = blockIdx.y, pos = blockIdx.x;
  const int n = part == 0 ? p.W : p.H;
  if (pos >= n) return;
  const int lo = cls == 0 ? 1 : 0, hi = cls == 2 ? 1 : 2;              // kernel taps of the OTHER axis inside the image
  float acc[4] = {0.f, 0.f, 0.f, 0.f};
  for (int ks = 0; ks < 3; ++ks) {                                      // tap along the table's own axis
    const int q = pos + ks - 1;
    if (q < 0 || q >= n) continue;
    const float4* t4 = reinterpret_cast<const float4*>((part == 0 ? p.tx : p.ty) + static_cast<size_t>(q) * 64);
    for (int ko = lo; ko <= hi; ++ko) {
      const int ky = part == 0 ? ko : ks, kx = part == 0 ? ks : ko;
      const uint4* w4 = reinterpret_cast<const uint4*>(p.w + static_cast<size_t>(oc) * 9 * 128 + (ky * 3 + kx) * 128 + (part == 0 ? 0 : 64));
#pragma unroll
      for (int c8 = 0; c8 < 8; ++c8) {
        const uint4 wv = __ldg(w4 + c8);
        const float4 ta = __ldg(t4 + 2 * c8), tb = __ldg(t4 + 2 * c8 + 1);
        const float2 w0 = unpack_h(wv.x, p.f16), w1 = unpack_h(wv.y, p.f16), w2 = unpack_h(wv.z, p.f16), w3 = unpack_h(wv.w, p.f16);
        acc[0] = fmaf(ta.x, w0.x, acc[0]); acc[1] = fmaf(ta.y, w0.y, acc[1]);
        acc[2] = fmaf(ta.z, w1.x, acc[2]); acc[3] = fmaf(ta.w, w1.y, acc[3]);
        acc[0] = fmaf(tb.x, w2.x, acc[0]); acc[1] = fmaf(tb.y, w2.y, acc[1]);
        acc[2] = fmaf(tb.z, w3.x, acc[2]); acc[3] = fmaf(tb.w, w3.y, acc[3]);
      }
    }
  }
  (part == 0 ? p.gx : p.gy)[(static_cast<size_t>(cls) * n + pos) * 32 + oc] = (acc[0] + acc[1]) + (acc[2] + acc[3]);
}

}  // namespace ovg
