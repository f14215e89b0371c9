// Image ranking by camera distance (datasets/utils/image_ranking.py:9-140, compute_ranking): two launches per call.
//
//   - rank_prep_kernel (one CTA): the mean of |t| over the views as one fp64 reduction in a fixed order (each thread sums
//     views tid, tid + 256, ... in order, then a tree over the 256 partials), and the operands of every view packed as 12
//     doubles (R row-major, then t): t / mean rounded to the input dtype when normalizing, and everything rounded to fp32
//     when the output is fp32.
//   - rank_smem_kernel / rank_grid_kernel: row i of the distance matrix and its ranking.  The CTA evaluates d(i, j) for
//     every j in fp64 (each operation rounded on its own, the reference's order), rounds it once to the output dtype,
//     writes the dists row, maps each value to an ordered unsigned key and sorts (key, j) by a stable LSD radix sort of
//     8-bit digits, then writes the first k indices.  Ties keep index order, -0 sorts equal to +0 and NaN sorts last.
//     Up to RANK_CTA_VIEWS views the keys and indices sit in shared memory and one CTA runs per row; above, a persistent
//     grid of RANK_GRID_CTAS CTAs sorts its rows in a per-CTA scratch in the workspace.
//
// The sort: the digit histograms of all passes are counted while the keys are made.  Each pass scatters the keys tile by
// tile (RANK_THREADS keys per tile, in order): a key's destination is the offset of its digit (exclusive scan of the
// histogram plus the keys of that digit in earlier tiles), plus the keys of that digit in earlier warps of the tile, plus
// its rank among the lanes of its warp with the same digit (__match_any_sync).  Every position follows from counts alone,
// so the order never depends on timing, and a pass whose digit is the same for every key is skipped.
#pragma once

#include <cuda_runtime.h>

namespace ovg {

constexpr int RANK_THREADS = 512;
constexpr int RANK_WARPS = RANK_THREADS / 32;
constexpr int RANK_PREP_THREADS = 256;
constexpr int RANK_CTA_VIEWS = OVG_RANK_CTA_VIEWS;       // 8192 x 24 B (fp64 keys, both buffers) = 192 KB of shared memory
constexpr int RANK_GRID_CTAS = 256;                      // CTAs (and scratch rows) of the persistent grid
constexpr double RANK_DEG = 180.0 / 3.141592653589793;   // numpy's degrees: x * (180 / pi)

struct RankParams {
  const void* ext;              // extrinsics, element (v, r, c) at v s0 + r s1 + c s2
  long long s0, s1, s2;
  double* pose;                 // [N][12] operands: R row-major, then t
  unsigned char* scratch;       // grid path: [RANK_GRID_CTAS][scratch_stride] bytes
  long long scratch_stride;
  long long* ranking;           // [N][k]
  void* dists;                  // [N][N], fp32 or fp64
  double lambda;
  int N, k, in_f64, out_f64, normalize;
};

struct RankSmem {
  unsigned hist[8][256];                      // digit histograms of every pass
  unsigned short cnt[RANK_WARPS][256];        // keys per (warp, digit) of the current tile
  unsigned short off[RANK_WARPS][256];        // their exclusive offsets within the tile
  unsigned base[256];                         // per digit: destination of the tile's first key
  unsigned tot[256];                          // per digit: keys in the current tile
  unsigned wsum[256 / 32];
};

__device__ __forceinline__ double rank_in(const RankParams& p, long long v, int r, int c) {
  const long long o = v * p.s0 + r * p.s1 + c * p.s2;
  return p.in_f64 ? static_cast<const double*>(p.ext)[o] : static_cast<double>(static_cast<const float*>(p.ext)[o]);
}

__device__ __forceinline__ double rank_f32(double x) { return static_cast<double>(__double2float_rn(x)); }

__global__ void __launch_bounds__(RANK_PREP_THREADS) rank_prep_kernel(RankParams p) {
  __shared__ double acc[RANK_PREP_THREADS];
  double mean = 1.0;
  if (p.normalize) {
    double a = 0.0;
    for (int v = threadIdx.x; v < p.N; v += RANK_PREP_THREADS) {
      const double x = rank_in(p, v, 0, 3), y = rank_in(p, v, 1, 3), z = rank_in(p, v, 2, 3);
      a = __dadd_rn(a, __dsqrt_rn(__dadd_rn(__dadd_rn(__dmul_rn(x, x), __dmul_rn(y, y)), __dmul_rn(z, z))));
    }
    acc[threadIdx.x] = a;
    __syncthreads();
    for (int h = RANK_PREP_THREADS / 2; h > 0; h >>= 1) {
      if (threadIdx.x < h) acc[threadIdx.x] = __dadd_rn(acc[threadIdx.x], acc[threadIdx.x + h]);
      __syncthreads();
    }
    mean = __ddiv_rn(acc[0], static_cast<double>(p.N));
  }
  for (int v = threadIdx.x; v < p.N; v += RANK_PREP_THREADS) {
    double* q = p.pose + static_cast<long long>(v) * 12;
    for (int r = 0; r < 3; ++r) {
      for (int c = 0; c < 3; ++c) {
        const double x = rank_in(p, v, r, c);
        q[r * 3 + c] = p.out_f64 ? x : rank_f32(x);
      }
      double t = rank_in(p, v, r, 3);
      if (p.normalize) {                       // the reference divides in place, in the input's dtype
        t = __ddiv_rn(t, mean);
        if (!p.in_f64) t = rank_f32(t);
      }
      q[9 + r] = p.out_f64 ? t : rank_f32(t);
    }
  }
}

// d(i, j) from the packed operands a (view i) and b (view j): trace(R_i^T R_j) as the sum of the diagonal of the matrix
// product, each diagonal entry summed over k in order; then (trace - 1) / 2, clip (NaN stays NaN), arccos, degrees, / 180;
// plus lambda * sqrt((dx dx + dy dy) + dz dz), dx = t_i - t_j.
__device__ __forceinline__ double rank_dist(const double* a, const double* b, double lambda) {
  double m[3];
#pragma unroll
  for (int c = 0; c < 3; ++c)
    m[c] = __dadd_rn(__dadd_rn(__dmul_rn(a[c], b[c]), __dmul_rn(a[3 + c], b[3 + c])), __dmul_rn(a[6 + c], b[6 + c]));
  const double tr = __dadd_rn(__dadd_rn(m[0], m[1]), m[2]);
  double v = __dmul_rn(__dsub_rn(tr, 1.0), 0.5);
  v = v < -1.0 ? -1.0 : (v > 1.0 ? 1.0 : v);
  const double rot = __ddiv_rn(__dmul_rn(acos(v), RANK_DEG), 180.0);
  const double dx = __dsub_rn(a[9], b[9]), dy = __dsub_rn(a[10], b[10]), dz = __dsub_rn(a[11], b[11]);
  const double tn = __dsqrt_rn(__dadd_rn(__dadd_rn(__dmul_rn(dx, dx), __dmul_rn(dy, dy)), __dmul_rn(dz, dz)));
  return __dadd_rn(rot, __dmul_rn(lambda, tn));
}

// Ordered keys: unsigned order equals the float order, -0 maps to +0's key and every NaN to the largest key.
__device__ __forceinline__ unsigned rank_key(float x) {
  unsigned b = __float_as_uint(x);
  if (x != x) return 0xffffffffu;
  if (b == 0x80000000u) b = 0u;
  return (b & 0x80000000u) ? ~b : (b | 0x80000000u);
}

__device__ __forceinline__ unsigned long long rank_key(double x) {
  unsigned long long b = static_cast<unsigned long long>(__double_as_longlong(x));
  if (x != x) return ~0ull;
  if (b == 0x8000000000000000ull) b = 0ull;
  return (b & 0x8000000000000000ull) ? ~b : (b | 0x8000000000000000ull);
}

// Row i: dists, keys and the stable sort.  ka / ia and kb / ib: two buffers of N keys and indices (shared or global).
template <typename T, typename K>
__device__ __forceinline__ void rank_row(const RankParams& p, int i, K* ka, unsigned* ia, K* kb, unsigned* ib,
                                         RankSmem& s) {
  constexpr int P = sizeof(K);                            // 8-bit digit passes
  const int n = p.N;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const unsigned lt = (1u << lane) - 1u;
  __syncthreads();                                        // the previous row's last reads of the buffers and histograms
  for (int x = threadIdx.x; x < P * 256; x += RANK_THREADS) s.hist[x >> 8][x & 255] = 0u;
  for (int x = threadIdx.x; x < RANK_WARPS * 256; x += RANK_THREADS) s.cnt[x >> 8][x & 255] = 0;   // the scan keeps it zero
  double a[12];
#pragma unroll
  for (int c = 0; c < 12; ++c) a[c] = __ldg(p.pose + static_cast<long long>(i) * 12 + c);
  __syncthreads();

  T* drow = static_cast<T*>(p.dists) + static_cast<long long>(i) * n;
  for (int j0 = 0; j0 < n; j0 += RANK_THREADS) {          // whole tiles: every lane takes part in __match_any_sync
    const int j = j0 + threadIdx.x;
    const bool ok = j < n;
    K key = 0;
    if (ok) {
      double b[12];
      const double2* q = reinterpret_cast<const double2*>(p.pose + static_cast<long long>(j) * 12);
#pragma unroll
      for (int c = 0; c < 6; ++c) {
        const double2 w = __ldg(q + c);
        b[2 * c] = w.x;
        b[2 * c + 1] = w.y;
      }
      const T d = static_cast<T>(rank_dist(a, b, p.lambda));   // one rounding to the output dtype (nearest)
      drow[j] = d;
      key = rank_key(d);
      ka[j] = key;
      ia[j] = static_cast<unsigned>(j);
    }
#pragma unroll
    for (int q = 0; q < P; ++q) {
      const unsigned dg = ok ? static_cast<unsigned>(key >> (8 * q)) & 255u : 256u;
      const unsigned peers = __match_any_sync(0xffffffffu, dg);
      if (ok && (peers & lt) == 0u) atomicAdd(&s.hist[q][dg], static_cast<unsigned>(__popc(peers)));
    }
  }

  __syncthreads();                                        // the histograms are complete before the passes read them

  K* sk = ka; unsigned* si = ia; K* dk = kb; unsigned* di = ib;
  for (int q = 0; q < P; ++q) {
    // also orders the previous pass's scatter before this pass reads it and rewrites base / off
    if (__syncthreads_or(threadIdx.x < 256 && s.hist[q][threadIdx.x] == static_cast<unsigned>(n))) continue;
    unsigned c = 0, x = 0;
    if (threadIdx.x < 256) {                              // exclusive scan of the pass's histogram
      c = s.hist[q][threadIdx.x];
      x = c;
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        const unsigned y = __shfl_up_sync(0xffffffffu, x, o);
        if (lane >= o) x += y;
      }
      if (lane == 31) s.wsum[warp] = x;
    }
    __syncthreads();
    if (threadIdx.x < 256) {
      for (int w = 0; w < warp; ++w) x += s.wsum[w];
      s.base[threadIdx.x] = x - c;
      s.tot[threadIdx.x] = 0u;
    }
    for (int j0 = 0; j0 < n; j0 += RANK_THREADS) {
      const int j = j0 + threadIdx.x;
      const bool ok = j < n;
      K key = 0;
      unsigned idx = 0;
      if (ok) {
        key = sk[j];
        idx = si[j];
      }
      const unsigned dg = ok ? static_cast<unsigned>(key >> (8 * q)) & 255u : 256u;
      const unsigned peers = __match_any_sync(0xffffffffu, dg);
      const unsigned r = __popc(peers & lt);
      if (ok && r == 0u) s.cnt[warp][dg] = static_cast<unsigned short>(__popc(peers));
      __syncthreads();                                    // counts written; the previous tile's scatter is done
      if (threadIdx.x < 256) {
        const int d = threadIdx.x;
        unsigned run = 0;
#pragma unroll
        for (int w = 0; w < RANK_WARPS; ++w) {
          const unsigned cw = s.cnt[w][d];
          s.cnt[w][d] = 0;
          s.off[w][d] = static_cast<unsigned short>(run);
          run += cw;
        }
        s.base[d] += s.tot[d];                            // past the previous tile's keys of digit d
        s.tot[d] = run;
      }
      __syncthreads();
      if (ok) {
        const unsigned dst = s.base[dg] + s.off[warp][dg] + r;
        dk[dst] = key;
        di[dst] = idx;
      }
    }
    K* tk = sk; sk = dk; dk = tk;
    unsigned* ti = si; si = di; di = ti;
  }
  __syncthreads();
  long long* out = p.ranking + static_cast<long long>(i) * p.k;
  for (int c = threadIdx.x; c < p.k; c += RANK_THREADS) out[c] = static_cast<long long>(si[c]);
}

// One CTA per row; the row's two key / index buffers in dynamic shared memory (N (2 sizeof(K) + 8) bytes).
template <typename T, typename K>
__global__ void __launch_bounds__(RANK_THREADS) rank_smem_kernel(RankParams p) {
  extern __shared__ __align__(16) unsigned char rank_dyn[];
  __shared__ RankSmem s;
  K* ka = reinterpret_cast<K*>(rank_dyn);
  K* kb = ka + p.N;
  unsigned* ia = reinterpret_cast<unsigned*>(kb + p.N);
  unsigned* ib = ia + p.N;
  rank_row<T, K>(p, blockIdx.x, ka, ia, kb, ib, s);
}

// Persistent grid: CTA b sorts rows b, b + gridDim.x, ... in its own scratch_stride bytes of the workspace.
template <typename T, typename K>
__global__ void __launch_bounds__(RANK_THREADS) rank_grid_kernel(RankParams p) {
  __shared__ RankSmem s;
  K* ka = reinterpret_cast<K*>(p.scratch + blockIdx.x * p.scratch_stride);
  K* kb = ka + p.N;
  unsigned* ia = reinterpret_cast<unsigned*>(kb + p.N);
  unsigned* ib = ia + p.N;
  for (int i = blockIdx.x; i < p.N; i += gridDim.x) rank_row<T, K>(p, i, ka, ia, kb, ib, s);
}

}  // namespace ovg
