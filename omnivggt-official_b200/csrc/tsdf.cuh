// Fused mesh of a scene's depth maps (no counterpart in the reference): TSDF integration into a voxel grid and marching cubes.
//   tsdf_fill_kernel / tsdf_select_init_kernel / tsdf_bounds_kernel
//                           per-axis 1st / 99th percentiles of the kept points by post.cuh's radix selection, with the
//                           ranks taken from the kept count on the device
//   tsdf_mark_kernel        bricks (8^3 voxels) that each kept pixel's surface band touches (Open3D's block allocation)
//   tsdf_integrate_kernel   one CTA per brick, one thread per voxel, every view in order: the mean truncated distance and colour
//   tsdf_count_kernel       per-brick vertex and triangle counts, scanned by tile_scan_kernel (compact.cuh)
//   tsdf_vertices_kernel / tsdf_triangles_kernel
//                           the vertices (with each owned edge's index) and the triangles, at the scanned offsets
// Every fp32 operation is an explicitly rounded intrinsic in the order oracle/tsdf_oracle.py restates, sums run in view order
// in one thread, and no atomic decides a value or a slot: the results are bit-identical from run to run.
#pragma once
#include "compact.cuh"
#include "post.cuh"

#define OVG_MC_STORAGE static __constant__ const
#include "mc_table.h"
#undef OVG_MC_STORAGE

namespace ovg {

constexpr int TSDF_BRICK = 8;
constexpr int TSDF_BRICK_VOXELS = TSDF_BRICK * TSDF_BRICK * TSDF_BRICK;
static_assert(TSDF_BRICK_VOXELS == 2 * COMPACT_THREADS, "a brick is two compaction chunks");

// ---------------------------------------------------------------------------------------------------------------- bounds
struct TsdfBoundsParams {
  const float* points;          // [n, 3]
  const unsigned char* mask;    // [n]
  long long n, ld;              // pixels, column stride of cols (multiple of 4)
  float* cols;                  // [3, ld]: kept coordinates, +inf elsewhere
  unsigned long long* count;    // kept pixels (zeroed before the fill)
  unsigned int* nonfinite;      // set when a kept coordinate is not finite (zeroed before the fill)
};

__global__ void __launch_bounds__(256) tsdf_fill_kernel(const TsdfBoundsParams p) {
  unsigned int kept = 0, bad = 0;
  for (long long i = blockIdx.x * 256LL + threadIdx.x; i < p.n; i += 256LL * gridDim.x) {
    const bool k = p.mask[i] != 0;
#pragma unroll
    for (int a = 0; a < 3; ++a) {
      const float v = p.points[3 * i + a];
      p.cols[a * p.ld + i] = k ? v : __int_as_float(0x7f800000);
      bad |= k && !isfinite(v);
    }
    kept += k;
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    kept += __shfl_xor_sync(0xffffffffu, kept, o);
    bad |= __shfl_xor_sync(0xffffffffu, bad, o);
  }
  if ((threadIdx.x & 31) == 0) {
    if (kept) atomicAdd(p.count, static_cast<unsigned long long>(kept));
    if (bad) atomicOr(p.nonfinite, 1u);
  }
}

// select_init_kernel with the ranks of numpy.percentile(kept, percent) computed from the kept count on the device; the
// interpolation weight goes to *frac.  The non-kept +inf entries sort after every kept value, so they never reach these ranks.
__global__ void tsdf_select_init_kernel(unsigned long long* state, unsigned int* hist, const unsigned long long* count,
                                        float percent, float* frac) {
  if (threadIdx.x == 0) {
    const unsigned long long n = *count;
    const double vi = n ? static_cast<double>(percent) / 100.0 * static_cast<double>(n - 1) : 0.0;
    const unsigned long long r0 = static_cast<unsigned long long>(vi);
    const unsigned long long r1 = r0 + 1 < n ? r0 + 1 : r0;
    state[0] = r0; state[1] = r1; state[2] = 0; state[3] = 0; state[4] = r0; state[5] = r1;
    *frac = static_cast<float>(vi - static_cast<double>(r0));
  }
  for (int i = threadIdx.x; i < 512; i += blockDim.x) hist[i] = 0;
}

// out fp64 [8] = kept count, lo x / y / z (1st percentiles), hi x / y / z (99th), non-finite flag.  sel: the [lo, hi] order
// statistics of each selection, frac their weights, in the order (axis, percentile).
__global__ void tsdf_bounds_kernel(const float* sel, const float* frac, const unsigned long long* count,
                                   const unsigned int* nonfinite, double* out) {
  if (threadIdx.x < 6) {
    const int a = threadIdx.x >> 1, q = threadIdx.x & 1;
    const float lo = sel[threadIdx.x * 3], hi = sel[threadIdx.x * 3 + 1];
    out[1 + q * 3 + a] = static_cast<double>(__fadd_rn(lo, __fmul_rn(__fsub_rn(hi, lo), frac[threadIdx.x])));
  }
  if (threadIdx.x == 0) {
    out[0] = static_cast<double>(*count);
    out[7] = *nonfinite ? 1.0 : 0.0;
  }
}

// ---------------------------------------------------------------------------------------------------------------- grid
struct TsdfGrid {
  int nx, ny, nz;               // voxels per axis; layout [nz, ny, nx]
  int bx, by, bz;               // bricks per axis (ceil(n / 8))
  float ox, oy, oz;             // voxel (0, 0, 0)
  float s, trunc;               // voxel size, truncation (4 s)
};

__device__ __forceinline__ float grid_coord(float o, int i, float s) { return __fadd_rn(o, __fmul_rn(static_cast<float>(i), s)); }

struct TsdfIntegrateParams {
  TsdfGrid g;
  const float* depth;           // [F, H, W]
  const unsigned char* mask;    // [F, H, W]
  const float* images;          // [F, 3, H, W]
  const float* ext;             // [F, 3, 4] world -> camera
  const float* intr;            // [F, 3, 3]
  int F, H, W;
  unsigned char* marked;        // [bricks]
  float* tsdf;                  // [nz, ny, nx]
  unsigned char* color;         // [nz, ny, nx, 4]
};

// Voxel range [lo, hi] along one axis of the box [g0, g1] (grid units) grown by one voxel, clamped to the grid; lo > hi when
// the box misses it.
__device__ __forceinline__ void band_range(float g0, float g1, int n, int& lo, int& hi) {
  const float a = fminf(g0, g1), b = fmaxf(g0, g1);
  lo = max(static_cast<int>(ceilf(fmaxf(a, -2.0f))) - 1, 0);
  hi = min(static_cast<int>(floorf(fminf(b, static_cast<float>(n + 1)))) + 1, n - 1);
}

// One thread per pixel: the points at depths d - trunc and d + trunc on its ray (pixel (x, y) -> ((x - cx) / fx, (y - cy) /
// fy), utils/geometry.py:236-264), taken to the world by the inverse of [R | t]; every brick their box touches is marked.
__global__ void __launch_bounds__(256) tsdf_mark_kernel(const TsdfIntegrateParams p) {
  const long long hw = static_cast<long long>(p.H) * p.W;
  const long long i = blockIdx.x * 256LL + threadIdx.x;
  if (i >= p.F * hw) return;
  const float d = p.depth[i];
  if (!p.mask[i] || !(d > 0.f)) return;
  const int f = static_cast<int>(i / hw);
  const int y = static_cast<int>((i - f * hw) / p.W), x = static_cast<int>(i - f * hw - static_cast<long long>(y) * p.W);
  const float* E = p.ext + f * 12;
  const float* K = p.intr + f * 9;
  const float rx = __fdiv_rn(__fsub_rn(static_cast<float>(x), K[2]), K[0]);
  const float ry = __fdiv_rn(__fsub_rn(static_cast<float>(y), K[5]), K[4]);
  float g[2][3];
  const float o[3] = {p.g.ox, p.g.oy, p.g.oz};
#pragma unroll
  for (int e = 0; e < 2; ++e) {
    const float z = e ? __fadd_rn(d, p.g.trunc) : __fsub_rn(d, p.g.trunc);
    const float q0 = __fsub_rn(__fmul_rn(rx, z), E[3]), q1 = __fsub_rn(__fmul_rn(ry, z), E[7]), q2 = __fsub_rn(z, E[11]);
#pragma unroll
    for (int a = 0; a < 3; ++a) {
      const float w = __fadd_rn(__fadd_rn(__fmul_rn(E[a], q0), __fmul_rn(E[4 + a], q1)), __fmul_rn(E[8 + a], q2));
      g[e][a] = __fdiv_rn(__fsub_rn(w, o[a]), p.g.s);
    }
  }
  int lo[3], hi[3];
  band_range(g[0][0], g[1][0], p.g.nx, lo[0], hi[0]);
  band_range(g[0][1], g[1][1], p.g.ny, lo[1], hi[1]);
  band_range(g[0][2], g[1][2], p.g.nz, lo[2], hi[2]);
  if (lo[0] > hi[0] || lo[1] > hi[1] || lo[2] > hi[2]) return;
  for (int bz = lo[2] / TSDF_BRICK; bz <= hi[2] / TSDF_BRICK; ++bz)
    for (int by = lo[1] / TSDF_BRICK; by <= hi[1] / TSDF_BRICK; ++by)
      for (int bx = lo[0] / TSDF_BRICK; bx <= hi[0] / TSDF_BRICK; ++bx)
        p.marked[(static_cast<long long>(bz) * p.g.by + by) * p.g.bx + bx] = 1;      // a constant: racing writers agree
}

__device__ __forceinline__ void brick_voxel(const TsdfGrid& g, long long b, int v, int& x, int& y, int& z) {
  const int bx = static_cast<int>(b % g.bx), by = static_cast<int>((b / g.bx) % g.by), bz = static_cast<int>(b / (g.bx * static_cast<long long>(g.by)));
  x = bx * TSDF_BRICK + (v & 7);
  y = by * TSDF_BRICK + ((v >> 3) & 7);
  z = bz * TSDF_BRICK + (v >> 6);
}

__device__ __forceinline__ long long voxel_index(const TsdfGrid& g, int x, int y, int z) {
  return (static_cast<long long>(z) * g.ny + y) * g.nx + x;
}

// One CTA of 512 threads per brick.  An unmarked brick writes "unobserved" (NaN, colour 0).
__global__ void __launch_bounds__(TSDF_BRICK_VOXELS) tsdf_integrate_kernel(const TsdfIntegrateParams p) {
  const long long b = blockIdx.x;
  int x, y, z;
  brick_voxel(p.g, b, threadIdx.x, x, y, z);
  if (x >= p.g.nx || y >= p.g.ny || z >= p.g.nz) return;
  const long long vi = voxel_index(p.g, x, y, z);
  float sum = 0.f;
  int n = 0;
  unsigned int c[3] = {0u, 0u, 0u};
  if (p.marked[b]) {
    const float px = grid_coord(p.g.ox, x, p.g.s), py = grid_coord(p.g.oy, y, p.g.s), pz = grid_coord(p.g.oz, z, p.g.s);
    const long long hw = static_cast<long long>(p.H) * p.W;
    for (int f = 0; f < p.F; ++f) {
      const float* E = p.ext + f * 12;
      const float Z = __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(E[8], px), __fmul_rn(E[9], py)), __fmul_rn(E[10], pz)), E[11]);
      if (!(Z > 0.f)) continue;
      const float X = __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(E[0], px), __fmul_rn(E[1], py)), __fmul_rn(E[2], pz)), E[3]);
      const float Y = __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(E[4], px), __fmul_rn(E[5], py)), __fmul_rn(E[6], pz)), E[7]);
      const float* K = p.intr + f * 9;
      const float u = __fadd_rn(__fmul_rn(__fdiv_rn(X, Z), K[0]), K[2]);
      const float v = __fadd_rn(__fmul_rn(__fdiv_rn(Y, Z), K[4]), K[5]);
      const float uf = floorf(__fadd_rn(u, 0.5f)), vf = floorf(__fadd_rn(v, 0.5f));
      if (!(uf >= 0.f && uf < static_cast<float>(p.W) && vf >= 0.f && vf < static_cast<float>(p.H))) continue;
      const long long pix = f * hw + static_cast<long long>(vf) * p.W + static_cast<long long>(uf);
      const float d = p.depth[pix];
      if (!p.mask[pix] || !(d > 0.f)) continue;
      const float sdf = __fsub_rn(d, Z);
      if (sdf < -p.g.trunc) continue;
      sum = __fadd_rn(sum, fminf(1.0f, __fdiv_rn(sdf, p.g.trunc)));
      ++n;
      const uchar3 rgb = pixel_rgb(p.images, hw, pix, f);
      c[0] += rgb.x; c[1] += rgb.y; c[2] += rgb.z;
    }
  }
  uchar4 col = make_uchar4(0, 0, 0, 0);
  if (n) {
    const unsigned int h = static_cast<unsigned int>(n) / 2;
    col = make_uchar4(static_cast<unsigned char>((c[0] + h) / n), static_cast<unsigned char>((c[1] + h) / n),
                      static_cast<unsigned char>((c[2] + h) / n), 255);
  }
  p.tsdf[vi] = n ? __fdiv_rn(sum, static_cast<float>(n)) : __int_as_float(0x7fc00000);   // numpy's NaN
  reinterpret_cast<uchar4*>(p.color)[vi] = col;
}

// ---------------------------------------------------------------------------------------------------------------- marching cubes
struct TsdfMeshParams {
  TsdfGrid g;
  const float* tsdf;                // [nz, ny, nx], NaN = unobserved
  const unsigned char* color;       // [nz, ny, nx, 4]
  long long bricks;
  unsigned int* tile_count;         // [2 * bricks]: vertices of each brick, then triangles
  unsigned long long* tile_offset;  // [2 * bricks + 1]: their exclusive scan, then the grand total
  int* edge_vertex;                 // [nz, ny, nx, 3]: the vertex of each owned edge, -1 for none
  float* positions;                 // [vertices, 3]
  unsigned char* colors;            // [vertices, 3]
  int* indices;                     // [triangles, 3]
  long long* totals;                // [2] vertices, triangles
};

__device__ __forceinline__ bool observed(float f) { return !isnan(f); }

// The case of the cube whose base voxel is (x, y, z), or -1 unless it lies in the grid with all 8 corners observed.
__device__ __forceinline__ int cube_case(const TsdfMeshParams& p, int x, int y, int z) {
  if (x < 0 || y < 0 || z < 0 || x + 1 >= p.g.nx || y + 1 >= p.g.ny || z + 1 >= p.g.nz) return -1;
  int c = 0;
#pragma unroll
  for (int k = 0; k < 8; ++k) {
    const float f = p.tsdf[voxel_index(p.g, x + ovg_mc_corner[k][0], y + ovg_mc_corner[k][1], z + ovg_mc_corner[k][2])];
    if (!observed(f)) return -1;
    c |= (f < 0.f) << k;
  }
  return c;
}

// Bit a set when voxel (x, y, z)'s +a edge has a vertex: both ends observed, signs differing, and a cube around it emitting
// (with the signs differing, any of the up-to-4 cubes with all corners observed does).
__device__ __forceinline__ int edge_bits(const TsdfMeshParams& p, int x, int y, int z) {
  const float f0 = p.tsdf[voxel_index(p.g, x, y, z)];
  if (!observed(f0)) return 0;
  int bits = 0;
#pragma unroll
  for (int a = 0; a < 3; ++a) {
    const int x1 = x + (a == 0), y1 = y + (a == 1), z1 = z + (a == 2);
    if (x1 >= p.g.nx || y1 >= p.g.ny || z1 >= p.g.nz) continue;
    const float f1 = p.tsdf[voxel_index(p.g, x1, y1, z1)];
    if (!observed(f1) || (f0 < 0.f) == (f1 < 0.f)) continue;
    bool emits = false;
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const int d1 = k & 1, d2 = k >> 1;    // offsets along the two other axes
      const int cx = x - (a == 0 ? 0 : d1), cy = y - (a == 1 ? 0 : (a == 0 ? d1 : d2)), cz = z - (a == 2 ? 0 : d2);
      emits = emits || cube_case(p, cx, cy, cz) >= 0;
    }
    bits |= emits << a;
  }
  return bits;
}

__device__ __forceinline__ int cube_tris(const TsdfMeshParams& p, int x, int y, int z) {
  const int c = cube_case(p, x, y, z);
  return c < 0 ? 0 : ovg_mc_tri_count[c];
}

// Whether voxel v of brick b lies in the grid and is observed; the whole CTA learns if any voxel of the brick is.
__device__ __forceinline__ bool brick_live(const TsdfMeshParams& p, long long b, int v, int& x, int& y, int& z) {
  brick_voxel(p.g, b, v, x, y, z);
  return x < p.g.nx && y < p.g.ny && z < p.g.nz && observed(p.tsdf[voxel_index(p.g, x, y, z)]);
}

// One CTA of COMPACT_THREADS per brick, its 512 voxels in two row-major chunks.  A brick without an observed voxel owns no
// vertex and no emitting cube (its base corner is unobserved).
__global__ void __launch_bounds__(COMPACT_THREADS) tsdf_count_kernel(const TsdfMeshParams p) {
  const long long b = blockIdx.x;
  unsigned int cnt[2] = {0u, 0u};
  int live = 0;
  for (int it = 0; it < 2; ++it) {
    int x, y, z;
    if (brick_live(p, b, it * COMPACT_THREADS + threadIdx.x, x, y, z)) {
      live = 1;
      cnt[0] += __popc(edge_bits(p, x, y, z));
      cnt[1] += cube_tris(p, x, y, z);
    }
  }
  if (!__syncthreads_or(live)) {
    if (threadIdx.x < 2) p.tile_count[threadIdx.x * p.bricks + b] = 0;
    return;
  }
  const unsigned int s = tile_sum<2>(cnt);
  if (threadIdx.x < 2) p.tile_count[threadIdx.x * p.bricks + b] = s;
}

__global__ void tsdf_totals_kernel(const TsdfMeshParams p) {
  if (threadIdx.x == 0) {
    p.totals[0] = static_cast<long long>(p.tile_offset[p.bricks]);
    p.totals[1] = static_cast<long long>(p.tile_offset[2 * p.bricks] - p.tile_offset[p.bricks]);
  }
}

// Vertices in brick-major order, each voxel's by axis x, y, z: t = f0 / (f0 - f1) along the edge, the colour of the endpoint
// with the smaller |tsdf| (endpoint 0 on ties).
__global__ void __launch_bounds__(COMPACT_THREADS) tsdf_vertices_kernel(const TsdfMeshParams p) {
  const long long b = blockIdx.x;
  unsigned long long out = p.tile_offset[b];
  for (int it = 0; it < 2; ++it) {
    int x, y, z;
    const bool live = brick_live(p, b, it * COMPACT_THREADS + threadIdx.x, x, y, z);
    if (!__syncthreads_or(live)) continue;
    const int bits = live ? edge_bits(p, x, y, z) : 0;
    const unsigned int val[1] = {static_cast<unsigned int>(__popc(bits))};
    unsigned int rank[1], sum[1];
    chunk_sums<1>(val, rank, sum);
    if (x < p.g.nx && y < p.g.ny && z < p.g.nz) {
      const long long vi = voxel_index(p.g, x, y, z);
      unsigned long long k = out + rank[0];
      const float f0 = p.tsdf[vi];
      const float c0[3] = {grid_coord(p.g.ox, x, p.g.s), grid_coord(p.g.oy, y, p.g.s), grid_coord(p.g.oz, z, p.g.s)};
#pragma unroll
      for (int a = 0; a < 3; ++a) {
        if (!((bits >> a) & 1)) {
          p.edge_vertex[vi * 3 + a] = -1;
          continue;
        }
        const long long v1 = voxel_index(p.g, x + (a == 0), y + (a == 1), z + (a == 2));
        const float f1 = p.tsdf[v1];
        const float t = __fdiv_rn(f0, __fsub_rn(f0, f1));
#pragma unroll
        for (int e = 0; e < 3; ++e) p.positions[3 * k + e] = e == a ? __fadd_rn(c0[e], __fmul_rn(t, p.g.s)) : c0[e];
        const unsigned char* c = p.color + 4 * (fabsf(f1) < fabsf(f0) ? v1 : vi);
        p.colors[3 * k] = c[0];
        p.colors[3 * k + 1] = c[1];
        p.colors[3 * k + 2] = c[2];
        p.edge_vertex[vi * 3 + a] = static_cast<int>(k);
        ++k;
      }
    }
    out += sum[0];
  }
}

// Triangles in brick-major cube order, each cube's in table order, from the owned edges' vertex indices.
__global__ void __launch_bounds__(COMPACT_THREADS) tsdf_triangles_kernel(const TsdfMeshParams p) {
  const long long b = blockIdx.x;
  unsigned long long out = p.tile_offset[p.bricks + b] - p.tile_offset[p.bricks];
  for (int it = 0; it < 2; ++it) {
    int x, y, z;
    const bool live = brick_live(p, b, it * COMPACT_THREADS + threadIdx.x, x, y, z);
    if (!__syncthreads_or(live)) continue;
    const int c = live ? cube_case(p, x, y, z) : -1;
    const unsigned int val[1] = {c < 0 ? 0u : static_cast<unsigned int>(ovg_mc_tri_count[c])};
    unsigned int rank[1], sum[1];
    chunk_sums<1>(val, rank, sum);
    const unsigned long long k0 = out + rank[0];
    for (int t = 0; t < static_cast<int>(val[0]); ++t)
#pragma unroll
      for (int j = 0; j < 3; ++j) {
        const int e = ovg_mc_tri_edges[c][3 * t + j];
        const signed char* o = ovg_mc_corner[ovg_mc_edge[e][0]];
        const int a = ovg_mc_corner[ovg_mc_edge[e][1]][0] != o[0] ? 0 : (ovg_mc_corner[ovg_mc_edge[e][1]][1] != o[1] ? 1 : 2);
        p.indices[3 * (k0 + t) + j] = p.edge_vertex[voxel_index(p.g, x + o[0], y + o[1], z + o[2]) * 3 + a];
      }
    out += sum[0];
  }
}

}  // namespace ovg
