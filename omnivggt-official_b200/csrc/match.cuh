// Reciprocal nearest-neighbour matches between the point sets of several views (utils/geometry.py:435-451,
// find_reciprocal_matches: two cKDTree builds and two queries per pair on the host).
//   match_keep_* kernels     per-view ordered compaction of the kept points (compact.cuh: tile count / scan / gather)
//   match_hist_* kernels     per-view grid range: 0.1 % / 99.9 % quantiles per axis, coarse (fp32 key) then linear bins
//   match_cell_* kernels     uniform grid per view: cell of every point, counts, per-view scan of the cell starts
//   match_radix_* kernels    stable LSD radix sort of every view's points by cell (kept-index order inside a cell)
//   match_query_kernel       exact nearest neighbour of every point of view a among the points of view b, both directions of
//                            every pair in one launch
//   match_recip_count_kernel reciprocity nn1[nn2[j]] == j, tile counts of every pair
//   tile_scan_kernel         one scan over the pairs' tile counts, concatenated (compact.cuh)
//   match_counts_kernel      matches per pair
//   match_gather_kernel      ordered compaction of the matches
// Distances are fp64, d2 = ((dx * dx) + (dy * dy)) + dz * dz without contraction, as cKDTree computes them for 3-D data; among
// points at the same d2 the lowest index wins.  The grid only prunes: a cell or a whole shell of cells is skipped only when a
// lower bound on its d2 is strictly greater than the best d2 so far, so the result is the exact (d2, index) minimum over all
// points whatever the grid looks like; the grid's range and resolution only decide the speed.
#pragma once
#include "post.cuh"

namespace ovg {

constexpr int MATCH_BINS = 2048;                           // histogram bins per axis
constexpr int MATCH_MAX_DIM = 4096;                        // cells per axis
constexpr int MATCH_QUERY_THREADS = 128;

__host__ __device__ inline long long match_cells_cap(long long cap) { return 2 * cap + 64; }   // cells per view

struct MatchGrid {        // one view's grid; cell k along an axis holds lo + k h <= x < lo + (k + 1) h (up to rounding, see pad)
  double lo[3];
  double inv[3];          // cells per unit length; 0 on an axis with one cell
  double h[3];            // 1 / inv
  int dim[3];
  int n;                  // kept points of the view
};

struct MatchParams {
  const float* points;            // [V, cap, 3]
  const unsigned char* keep;      // [V, cap] or NULL (all kept)
  int V;
  long long cap;
  int tiles;                      // compaction tiles per view (compact_tiles(cap))
  unsigned int* flag;             // bit 0: a kept point is not finite
  unsigned int* view_tile_count;  // [V, tiles]
  unsigned int* view_tile_offset; // [V, tiles]
  MatchGrid* grid;                // [V]
  unsigned int* hist;             // [V, 3, MATCH_BINS]
  float* range0;                  // [V, 3, 2] coarse range of the linear histogram
  float4* pts;                    // [V, cap] compacted: x, y, z, pixel index (int bits)
  int* keys[2];                   // [V, cap] cell of each point, ping-pong buffers of the radix sort by cell
  float4* vals[2];                // [V, cap] x, y, z, kept index (int bits), sorted along with the keys
  float4* sorted;                 // = vals[passes % 2]: the points in cell order, by kept index inside a cell
  int rtiles;                     // radix-sort tiles of MATCH_RADIX_TILE points per view
  unsigned int* radix_off;        // [V, 256, rtiles] digit counts per tile, then their exclusive scan (digit-major)
  int* cell_count;                // [V, cells_cap]
  int* cell_start;                // [V, cells_cap + 1]
  long long cells_cap;
  // queries
  const int* pairs;               // [P, 2]
  int P;
  int* nn;                        // [2P, cap]: segment 2p = view i into view j, 2p + 1 = view j into view i
  int ptiles;                     // reciprocity tiles per pair (compact_tiles(cap))
  unsigned int* pair_tile_count;  // [P, ptiles]
  unsigned long long* pair_tile_offset;
  unsigned long long* total;
  long long* counts;              // [P + 1]: matches per pair, then the non-finite flag
};

// ---------------------------------------------------------------------------------------------------- compaction
__device__ __forceinline__ bool match_kept(const MatchParams& p, int v, long long i) {
  return i < p.cap && (p.keep == nullptr || p.keep[v * p.cap + i] != 0);
}

// grid (tiles, V): kept points per tile
__global__ void __launch_bounds__(COMPACT_THREADS) match_keep_count_kernel(const MatchParams p) {
  const int v = blockIdx.y;
  const long long base = static_cast<long long>(blockIdx.x) * COMPACT_TILE;
  unsigned int kept[1] = {0u};
  for (int it = 0; it < COMPACT_ITERS; ++it) kept[0] += match_kept(p, v, base + it * COMPACT_THREADS + threadIdx.x) ? 1u : 0u;
  const unsigned int s = tile_sum<1>(kept);
  if (threadIdx.x == 0) p.view_tile_count[v * p.tiles + blockIdx.x] = s;
}

// grid V, 1024 threads: exclusive scan of the view's tile counts, the view's kept count
__global__ void __launch_bounds__(1024) match_keep_scan_kernel(const MatchParams p) {
  const int v = blockIdx.x;
  const unsigned int n = block_exclusive_scan(p.view_tile_count + v * p.tiles, p.view_tile_offset + v * p.tiles, p.tiles);
  if (threadIdx.x == 0) p.grid[v].n = static_cast<int>(n);
}

// grid (tiles, V): kept point k of view v -> pts[v, k] = (x, y, z, pixel index), in pixel order
__global__ void __launch_bounds__(COMPACT_THREADS) match_keep_gather_kernel(const MatchParams p) {
  const int v = blockIdx.y;
  const long long base = static_cast<long long>(blockIdx.x) * COMPACT_TILE;
  unsigned int out = p.view_tile_offset[v * p.tiles + blockIdx.x];
  for (int it = 0; it < COMPACT_ITERS; ++it) {
    const long long i = base + it * COMPACT_THREADS + threadIdx.x;
    const bool keep[1] = {match_kept(p, v, i)};
    unsigned int rank[1], sum[1];
    chunk_ranks<1>(keep, rank, sum);
    if (keep[0]) {
      const unsigned int k = out + rank[0];
      const float* s = p.points + (v * p.cap + i) * 3;
      p.pts[v * p.cap + k] = make_float4(s[0], s[1], s[2], __int_as_float(static_cast<int>(i)));
    }
    out += sum[0];
  }
}

// ---------------------------------------------------------------------------------------------------- grid range
// Pass 0 bins the monotone fp32 key (sign, exponent, 2 mantissa bits: robust to any spread, 19 % resolution in magnitude);
// pass 1 bins linearly inside the coarse range found by pass 0 (values outside are clamped into the end bins).  The range is
// [lower edge of the bin holding rank n / 1000, upper edge of the bin holding rank n - 1 - n / 1000]: a few far outliers
// do not stretch the grid, they fall into the clamped boundary cells.
__device__ __forceinline__ int match_lin_bin(float x, float lo, float hi) {
  const float t = (x - lo) / (hi - lo) * static_cast<float>(MATCH_BINS);
  if (!(t >= 1.0f)) return 0;
  if (t >= static_cast<float>(MATCH_BINS - 1)) return MATCH_BINS - 1;
  return static_cast<int>(t);
}

// grid (blocks, V)
__global__ void __launch_bounds__(256) match_hist_kernel(const MatchParams p, int pass) {
  __shared__ unsigned int sh[3 * MATCH_BINS];
  for (int i = threadIdx.x; i < 3 * MATCH_BINS; i += blockDim.x) sh[i] = 0;
  __syncthreads();
  const int v = blockIdx.y;
  const int n = p.grid[v].n;
  const float* r0 = p.range0 + v * 6;
  bool bad = false;
  for (long long k = blockIdx.x * 256LL + threadIdx.x; k < n; k += 256LL * gridDim.x) {
    const float4 q = p.pts[v * p.cap + k];
    const float c[3] = {q.x, q.y, q.z};
#pragma unroll
    for (int a = 0; a < 3; ++a) {
      bad |= !isfinite(c[a]);
      const int b = pass == 0 ? static_cast<int>(f32_key(c[a]) >> 21) : match_lin_bin(c[a], r0[2 * a], r0[2 * a + 1]);
      atomicAdd(&sh[a * MATCH_BINS + b], 1u);
    }
  }
  if (pass == 0 && __syncthreads_or(bad) && threadIdx.x == 0) atomicOr(p.flag, 1u);
  __syncthreads();
  unsigned int* h = p.hist + v * 3 * MATCH_BINS;
  for (int i = threadIdx.x; i < 3 * MATCH_BINS; i += blockDim.x)
    if (sh[i]) atomicAdd(&h[i], sh[i]);
}

// grid V, 3 threads (one per axis): the ranked bins of the histogram, then the histogram is cleared for the next pass.
// pass 0 -> range0; pass 1 -> the grid: resolution ~2 cells per point over the axes of non-zero extent, capped per axis and in
// total (match_cells_cap).
__global__ void match_range_kernel(const MatchParams p, int pass) {
  __shared__ double ext[3];
  const int v = blockIdx.x, a = threadIdx.x;
  MatchGrid& g = p.grid[v];
  const int n = g.n;
  unsigned int* h = p.hist + (v * 3 + a) * MATCH_BINS;
  double lo = 0.0, hi = 0.0;
  if (a < 3 && n > 0) {
    const unsigned int r_lo = static_cast<unsigned int>(n / 1000), r_hi = static_cast<unsigned int>(n - 1 - n / 1000);
    int b_lo = -1, b_hi = -1;
    unsigned int s = 0;
    for (int b = 0; b < MATCH_BINS; ++b) {
      s += h[b];
      if (b_lo < 0 && s > r_lo) b_lo = b;
      if (b_hi < 0 && s > r_hi) b_hi = b;
    }
    if (pass == 0) {
      const float flo = key_f32(static_cast<uint32_t>(b_lo) << 21);
      const float fhi = key_f32((static_cast<uint32_t>(b_hi) << 21) | 0x1fffffu);
      p.range0[v * 6 + 2 * a] = flo;
      p.range0[v * 6 + 2 * a + 1] = fhi;
    } else {
      const double r0 = p.range0[v * 6 + 2 * a], r1 = p.range0[v * 6 + 2 * a + 1], w = (r1 - r0) / MATCH_BINS;
      lo = r0 + b_lo * w;
      hi = r0 + (b_hi + 1) * w;
    }
  }
  if (a < 3) for (int b = 0; b < MATCH_BINS; ++b) h[b] = 0;
  if (pass == 0) return;
  if (a < 3) {
    const double e = hi - lo;
    ext[a] = (isfinite(e) && e > 0.0) ? e : 0.0;
    g.lo[a] = isfinite(lo) ? lo : 0.0;
  }
  __syncthreads();
  if (a != 0) return;
  int k = 0;
  double vol = 1.0;
  for (int b = 0; b < 3; ++b)
    if (ext[b] > 0.0) { ++k; vol *= ext[b]; }
  long long dim[3] = {1, 1, 1};
  if (k > 0) {
    const double s = pow(2.0 * n / vol, 1.0 / k);
    for (int b = 0; b < 3; ++b)
      if (ext[b] > 0.0) {
        const double d = floor(ext[b] * s);
        dim[b] = d < 1.0 ? 1 : (d > MATCH_MAX_DIM ? MATCH_MAX_DIM : static_cast<long long>(d));
      }
    while (dim[0] * dim[1] * dim[2] > p.cells_cap) {
      const int m = dim[0] >= dim[1] ? (dim[0] >= dim[2] ? 0 : 2) : (dim[1] >= dim[2] ? 1 : 2);
      dim[m] = (dim[m] + 1) / 2;
    }
  }
  for (int b = 0; b < 3; ++b) {
    g.dim[b] = static_cast<int>(dim[b]);
    g.inv[b] = dim[b] > 1 ? static_cast<double>(dim[b]) / ext[b] : 0.0;
    g.h[b] = dim[b] > 1 ? 1.0 / g.inv[b] : 0.0;
  }
}

// ---------------------------------------------------------------------------------------------------- grid fill
// Cell coordinate along one axis: floor((x - lo) * inv) in fp64, clamped (NaN -> 0).  Points beyond the grid's range land in
// the boundary cells, which therefore extend to infinity.
__device__ __forceinline__ int match_cell_coord(float x, double lo, double inv, int dim) {
  const double t = __dmul_rn(__dsub_rn(static_cast<double>(x), lo), inv);
  if (!(t >= 1.0)) return 0;
  if (t >= static_cast<double>(dim - 1)) return dim - 1;
  return static_cast<int>(t);
}

__device__ __forceinline__ int match_cell(const MatchGrid& g, float x, float y, float z) {
  return (match_cell_coord(z, g.lo[2], g.inv[2], g.dim[2]) * g.dim[1] + match_cell_coord(y, g.lo[1], g.inv[1], g.dim[1])) *
             g.dim[0] + match_cell_coord(x, g.lo[0], g.inv[0], g.dim[0]);
}

// grid (blocks, V): the cell of every point and the cell counts; the radix sort's first keys / values (in kept-index order)
__global__ void __launch_bounds__(256) match_cell_count_kernel(const MatchParams p) {
  const int v = blockIdx.y;
  const MatchGrid g = p.grid[v];
  for (long long k = blockIdx.x * 256LL + threadIdx.x; k < g.n; k += 256LL * gridDim.x) {
    const float4 q = p.pts[v * p.cap + k];
    const int c = match_cell(g, q.x, q.y, q.z);
    p.keys[0][v * p.cap + k] = c;
    p.vals[0][v * p.cap + k] = make_float4(q.x, q.y, q.z, __int_as_float(static_cast<int>(k)));
    atomicAdd(&p.cell_count[v * p.cells_cap + c], 1);
  }
}

// grid V, 1024 threads: cell_start = exclusive scan of the view's cell counts, cell_start[cells] = n
__global__ void __launch_bounds__(1024) match_cell_scan_kernel(const MatchParams p) {
  const int v = blockIdx.x;
  const MatchGrid& g = p.grid[v];
  const long long cells = static_cast<long long>(g.dim[0]) * g.dim[1] * g.dim[2];
  int* start = p.cell_start + v * (p.cells_cap + 1);
  const int total = block_exclusive_scan(p.cell_count + v * p.cells_cap, start, cells);
  if (threadIdx.x == 0) start[cells] = total;
}

// Stable LSD radix sort of each view's points by cell, 8 bits per pass: a tile of MATCH_RADIX_TILE consecutive points counts its
// digits, a per-view scan over (digit, tile) gives every tile's first slot per digit, and the scatter ranks each point among the
// earlier points of its tile with the same digit (match_any within a warp, per-warp counts across warps).  No atomic decides a
// slot, so inside a cell the points stay in kept-index order.
constexpr int MATCH_RADIX_TILE = 256;

// grid (rtiles, V)
__global__ void __launch_bounds__(MATCH_RADIX_TILE) match_radix_count_kernel(const MatchParams p, int shift, int src) {
  __shared__ unsigned int h[256];
  h[threadIdx.x] = 0;
  __syncthreads();
  const int v = blockIdx.y;
  const long long k = static_cast<long long>(blockIdx.x) * MATCH_RADIX_TILE + threadIdx.x;
  if (k < p.grid[v].n) atomicAdd(&h[(p.keys[src][v * p.cap + k] >> shift) & 255], 1u);
  __syncthreads();
  p.radix_off[(static_cast<long long>(v) * 256 + threadIdx.x) * p.rtiles + blockIdx.x] = h[threadIdx.x];
}

// grid V, 1024 threads
__global__ void __launch_bounds__(1024) match_radix_scan_kernel(const MatchParams p) {
  unsigned int* off = p.radix_off + static_cast<long long>(blockIdx.x) * 256 * p.rtiles;
  block_exclusive_scan(off, off, 256LL * p.rtiles);
}

// grid (rtiles, V)
__global__ void __launch_bounds__(MATCH_RADIX_TILE) match_radix_scatter_kernel(const MatchParams p, int shift, int src) {
  __shared__ unsigned int wcnt[MATCH_RADIX_TILE / 32][256];
  for (int i = threadIdx.x; i < MATCH_RADIX_TILE / 32 * 256; i += MATCH_RADIX_TILE) (&wcnt[0][0])[i] = 0;
  __syncthreads();
  const int v = blockIdx.y;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const long long k = static_cast<long long>(blockIdx.x) * MATCH_RADIX_TILE + threadIdx.x;
  const bool valid = k < p.grid[v].n;
  int key = 0;
  float4 val = make_float4(0.f, 0.f, 0.f, 0.f);
  unsigned int d = 256;                                   // invalid lanes form their own group
  if (valid) {
    key = p.keys[src][v * p.cap + k];
    val = p.vals[src][v * p.cap + k];
    d = (static_cast<unsigned int>(key) >> shift) & 255;
  }
  const unsigned int same = __match_any_sync(0xffffffffu, d);
  const unsigned int rank_w = __popc(same & ((1u << lane) - 1u));
  if (valid && rank_w == 0) wcnt[warp][d] = __popc(same);
  __syncthreads();
  if (valid) {
    unsigned int r = rank_w;
    for (int w = 0; w < warp; ++w) r += wcnt[w][d];
    const long long slot = v * p.cap + p.radix_off[(static_cast<long long>(v) * 256 + d) * p.rtiles + blockIdx.x] + r;
    p.keys[src ^ 1][slot] = key;
    p.vals[src ^ 1][slot] = val;
  }
}

// ---------------------------------------------------------------------------------------------------- query
// Lower bounds.  A point x of cell k satisfies lo + k h - pad <= x (k > 0) and x < lo + (k + 1) h + pad (k < dim - 1); pad
// covers the rounding of the cell assignment and of the bound itself, relative to every magnitude involved (1e-9 against
// errors of a few 1e-16).  So the fp64 gap computed below never exceeds |q - x|, and the bound sum never exceeds the d2 the
// query computes for any point of the cell.
__device__ __forceinline__ double match_axis_gap(double q, double lo, double h, int k, int dim, double pad) {
  double g = 0.0;
  if (k > 0) g = fmax(g, (lo + k * h) - pad - q);                  // q below the cell
  if (k < dim - 1) g = fmax(g, q - (lo + (k + 1) * h) - pad);      // q above the cell
  return g;
}

__device__ __forceinline__ void match_visit(const float4* cell_pts, int b, int e, double qx, double qy, double qz, double& best,
                                            int& best_i) {
  for (int s = b; s < e; ++s) {
    const float4 t = cell_pts[s];
    const double dx = __dsub_rn(qx, static_cast<double>(t.x));
    const double dy = __dsub_rn(qy, static_cast<double>(t.y));
    const double dz = __dsub_rn(qz, static_cast<double>(t.z));
    const double d2 = __dadd_rn(__dadd_rn(__dmul_rn(dx, dx), __dmul_rn(dy, dy)), __dmul_rn(dz, dz));
    const int idx = __float_as_int(t.w);
    if (d2 < best || (d2 == best && idx < best_i)) {
      best = d2;
      best_i = idx;
    }
  }
}

// grid (ceil(cap / 128), 2P): segment 2p + d, query view a = (d ? j : i) into target view b = (d ? i : j).  One thread per query
// point: cells in Chebyshev shells r = 0, 1, ... around the query's cell; a cell is skipped when its bound is > best, and the
// search stops when every cell beyond the current box is farther than best (or there is none).  nn = -1 for an empty target
// and for a query without any candidate (NaN distances: the call's non-finite flag is set).
__global__ void __launch_bounds__(MATCH_QUERY_THREADS) match_query_kernel(const MatchParams p) {
  const int seg = blockIdx.y, pr = seg >> 1, dir = seg & 1;
  const int vi = p.pairs[2 * pr], vj = p.pairs[2 * pr + 1];
  if (vi < 0 || vi >= p.V || vj < 0 || vj >= p.V) return;
  const int va = dir ? vj : vi, vb = dir ? vi : vj;
  const int na = p.grid[va].n;
  const long long k = static_cast<long long>(blockIdx.x) * MATCH_QUERY_THREADS + threadIdx.x;
  if (k >= na) return;
  const MatchGrid& g = p.grid[vb];
  int* out = p.nn + static_cast<long long>(seg) * p.cap + k;
  if (g.n == 0) {
    *out = -1;
    return;
  }
  const float4 q = p.pts[va * p.cap + k];
  const double qc[3] = {static_cast<double>(q.x), static_cast<double>(q.y), static_cast<double>(q.z)};
  int dim[3], c[3];
  double lo[3], h[3], pad[3];
#pragma unroll
  for (int a = 0; a < 3; ++a) {
    dim[a] = g.dim[a];
    lo[a] = g.lo[a];
    h[a] = g.h[a];
    pad[a] = 1e-9 * (fabs(qc[a]) + fabs(lo[a]) + dim[a] * h[a]);
  }
  c[0] = match_cell_coord(q.x, lo[0], g.inv[0], dim[0]);
  c[1] = match_cell_coord(q.y, lo[1], g.inv[1], dim[1]);
  c[2] = match_cell_coord(q.z, lo[2], g.inv[2], dim[2]);
  const float4* pts = p.sorted + vb * p.cap;
  const int* start = p.cell_start + vb * (p.cells_cap + 1);
  double best = __longlong_as_double(0x7ff0000000000000LL);   // +inf
  int best_i = 0x7fffffff;
  for (int r = 0;; ++r) {
    const int z0 = max(c[2] - r, 0), z1 = min(c[2] + r, dim[2] - 1);
    const int y0 = max(c[1] - r, 0), y1 = min(c[1] + r, dim[1] - 1);
    const int x0 = max(c[0] - r, 0), x1 = min(c[0] + r, dim[0] - 1);
    for (int z = z0; z <= z1; ++z) {
      const double gz = match_axis_gap(qc[2], lo[2], h[2], z, dim[2], pad[2]);
      const double bz = gz * gz;
      if (bz > best) continue;
      const bool zface = z == c[2] - r || z == c[2] + r;
      for (int y = y0; y <= y1; ++y) {
        const double gy = match_axis_gap(qc[1], lo[1], h[1], y, dim[1], pad[1]);
        const double byz = bz + gy * gy;
        if (byz > best) continue;
        const bool face = zface || y == c[1] - r || y == c[1] + r;
        const int xstep = face ? 1 : 2 * r;             // inside the shell only the two x faces are new (r > 0 here)
        for (int x = face ? x0 : c[0] - r; x <= x1; x += xstep) {
          if (x < x0) continue;
          const double gx = match_axis_gap(qc[0], lo[0], h[0], x, dim[0], pad[0]);
          if (byz + gx * gx > best) continue;
          const int cell = (z * dim[1] + y) * dim[0] + x;
          match_visit(pts, start[cell], start[cell + 1], qc[0], qc[1], qc[2], best, best_i);
        }
      }
    }
    // every cell not yet visited lies beyond one face of the box [c - r, c + r] that is not a grid boundary
    double shell = __longlong_as_double(0x7ff0000000000000LL);
    bool more = false;
#pragma unroll
    for (int a = 0; a < 3; ++a) {
      if (c[a] - r > 0) {
        more = true;
        const double gap = fmax(0.0, qc[a] - (lo[a] + (c[a] - r) * h[a]) - pad[a]);
        shell = fmin(shell, gap * gap);
      }
      if (c[a] + r < dim[a] - 1) {
        more = true;
        const double gap = fmax(0.0, (lo[a] + (c[a] + r + 1) * h[a]) - pad[a] - qc[a]);
        shell = fmin(shell, gap * gap);
      }
    }
    if (!more || shell > best) break;
  }
  *out = best_i == 0x7fffffff ? -1 : best_i;     // no candidate: every d2 is NaN (a non-finite query or target)
}

// ---------------------------------------------------------------------------------------------------- reciprocity
// reciprocal_in_P2[jj] = nn1_in_P2[nn2_in_P1[jj]] == jj (geometry.py:448-449), jj over the kept points of view j
__device__ __forceinline__ bool match_recip(const MatchParams& p, int pr, long long jj, int* nn_i) {
  const int vi = p.pairs[2 * pr], vj = p.pairs[2 * pr + 1];
  if (vi < 0 || vi >= p.V || vj < 0 || vj >= p.V || jj >= p.grid[vj].n) return false;
  const int i = p.nn[(2LL * pr + 1) * p.cap + jj];
  *nn_i = i;
  return i >= 0 && i < p.grid[vi].n && p.nn[2LL * pr * p.cap + i] == jj;
}

// grid (ptiles, P)
__global__ void __launch_bounds__(COMPACT_THREADS) match_recip_count_kernel(const MatchParams p) {
  const int pr = blockIdx.y;
  const long long base = static_cast<long long>(blockIdx.x) * COMPACT_TILE;
  unsigned int kept[1] = {0u};
  for (int it = 0; it < COMPACT_ITERS; ++it) {
    int nn_i;
    kept[0] += match_recip(p, pr, base + it * COMPACT_THREADS + threadIdx.x, &nn_i) ? 1u : 0u;
  }
  const unsigned int s = tile_sum<1>(kept);
  if (threadIdx.x == 0) p.pair_tile_count[pr * p.ptiles + blockIdx.x] = s;
}

// one thread per pair, after the scan of the tile counts: matches of the pair; then the non-finite flag
__global__ void match_counts_kernel(const MatchParams p) {
  for (int pr = blockIdx.x * blockDim.x + threadIdx.x; pr <= p.P; pr += gridDim.x * blockDim.x) {
    if (pr == p.P) {
      p.counts[pr] = static_cast<long long>(*p.flag);
    } else {
      const unsigned long long a = p.pair_tile_offset[static_cast<long long>(pr) * p.ptiles];
      const unsigned long long b = pr + 1 < p.P ? p.pair_tile_offset[static_cast<long long>(pr + 1) * p.ptiles] : *p.total;
      p.counts[pr] = static_cast<long long>(b - a);
    }
  }
}

struct MatchOut {
  int W;                 // xy: pixel index -> (index % W, index / W)
  long long* xy_i;       // [total, 2] (scene outputs) or NULL
  long long* xy_j;
  int pair;              // per-query outputs of this pair (reciprocal_in_P2, nn2_in_P1), or -1
  unsigned char* recip;  // [n_j]
  long long* nn;         // [n_j]
};

// grid (ptiles, P): the matches of every pair in ascending jj, pairs in order (offsets from the scan of the tile counts)
__global__ void __launch_bounds__(COMPACT_THREADS) match_gather_kernel(const MatchParams p, const MatchOut o) {
  const int pr = blockIdx.y;
  const long long base = static_cast<long long>(blockIdx.x) * COMPACT_TILE;
  unsigned long long out = p.pair_tile_offset[static_cast<long long>(pr) * p.ptiles + blockIdx.x];
  const int vi = p.pairs[2 * pr], vj = p.pairs[2 * pr + 1];
  for (int it = 0; it < COMPACT_ITERS; ++it) {
    const long long jj = base + it * COMPACT_THREADS + threadIdx.x;
    int nn_i = -1;
    const bool keep[1] = {match_recip(p, pr, jj, &nn_i)};
    unsigned int rank[1], sum[1];
    chunk_ranks<1>(keep, rank, sum);
    if (keep[0]) {
      const unsigned long long k = out + rank[0];
      const long long pj = __float_as_int(p.pts[vj * p.cap + jj].w), pi = __float_as_int(p.pts[vi * p.cap + nn_i].w);
      o.xy_j[2 * k] = pj % o.W;
      o.xy_j[2 * k + 1] = pj / o.W;
      o.xy_i[2 * k] = pi % o.W;
      o.xy_i[2 * k + 1] = pi / o.W;
    }
    out += sum[0];
  }
}

// grid ceil(n_j / 256): reciprocal_in_P2 and nn2_in_P1 of one pair
__global__ void __launch_bounds__(256) match_pair_kernel(const MatchParams p, const MatchOut o) {
  const int vj = p.pairs[2 * o.pair + 1];
  const long long jj = blockIdx.x * 256LL + threadIdx.x;
  if (vj < 0 || vj >= p.V || jj >= p.grid[vj].n) return;
  int nn_i = -1;
  const bool r = match_recip(p, o.pair, jj, &nn_i);
  o.recip[jj] = r ? 1 : 0;
  o.nn[jj] = nn_i;
}

}  // namespace ovg
