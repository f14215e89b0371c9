// Multi-view tracks ("star tracks") over the reciprocal matches of ovg_match_query, in the matcher's kept-index space: node
// (v, k) is kept point k of view v, its pixel in pts[v, k].w.
//   track_count_kernel    step a: kept, unclaimed anchors of view a with 1 + partners >= min_views; tile counts of the two
//                         streams "new tracks" and "new observations"
//   tile_scan_kernel      one scan over both streams' tile counts, concatenated (compact.cuh)
//   track_write_kernel    step a: the new tracks in anchor order, their observations, the claims; the running totals
//   track_claimed_kernel  tile counts of the claimed nodes of every view
//   track_view_kernel     per view, the ordered compaction of the claimed nodes: track, pixel and rank of each
//   track_point_kernel    one thread per track: fp64 mean, colour, reprojection error, and the observations' outputs
// track_reproject is the per-observation reprojection, shared with the bundle adjuster (ba.cuh).
// A partner of anchor (a, k) is the reciprocal match jj of k in view j > a of pair (a, j), if (j, jj) is unclaimed.  Each pair's
// reciprocal matching is one-to-one, so a node of view j can only be the partner of one anchor of view a: inside a step no two
// threads read or write the same claim, and nothing is decided by an atomic.  Sums run in a fixed order: results are
// bit-identical from run to run.
#pragma once
#include "match.cuh"

namespace ovg {

constexpr int TRACK_POINT_THREADS = 128;

struct TrackParams {
  MatchParams m;                      // the matcher's workspace: pts, grid[v].n, nn, pairs, flag
  const int* pair_off;                // [V + 1]: the pairs (a, j) of anchor a are pairs[pair_off[a], pair_off[a + 1]), j ascending
  int min_views;
  int* claim;                         // [V, cap] track of node (v, k), -1 while unclaimed
  int* rank;                          // [V, cap] rank of a claimed node among its view's claimed nodes
  int* obs;                           // [V cap] node v cap + k of every observation: tracks in order, views ascending in a track
  int* track_start;                   // [V cap] first observation of each track
  unsigned int* tile_count;           // [max(2, V), tiles]
  unsigned long long* tile_offset;    // [max(2, V), tiles]
  unsigned long long* scan_total;
  unsigned long long* totals;         // [2][2] (tracks, observations) before step a in totals[2 (a & 1)]
};

// The reciprocal match of kept point k of view a in view vj, through pair pr = (a, vj); -1 when there is none.
__device__ __forceinline__ int track_partner(const MatchParams& m, int pr, int vj, long long k) {
  const int jj = m.nn[2LL * pr * m.cap + k];
  return (jj >= 0 && jj < m.grid[vj].n && m.nn[(2LL * pr + 1) * m.cap + jj] == k) ? jj : -1;
}

// Calls f(i, node) for the i-th unclaimed partner of anchor (a, k), node = view * cap + kept index, views ascending; returns
// their count.  Pairs that are not (a, j) with j > a and j above the previous pair's view are skipped, so a node is visited
// once.
template <typename F>
__device__ __forceinline__ unsigned int track_partners(const TrackParams& p, int a, long long k, F f) {
  unsigned int c = 0u;
  int last = a;
  for (int e = p.pair_off[a]; e < p.pair_off[a + 1]; ++e) {
    const int vj = p.m.pairs[2 * e + 1];
    if (p.m.pairs[2 * e] != a || vj <= last || vj >= p.m.V) continue;
    last = vj;
    const int jj = track_partner(p.m, e, vj, k);
    if (jj >= 0 && p.claim[vj * p.m.cap + jj] < 0) f(c++, vj * p.m.cap + jj);
  }
  return c;
}

// Observations of the track anchor (a, k) would start, 0 when it starts none (claimed, or fewer than min_views).
__device__ __forceinline__ unsigned int track_members(const TrackParams& p, int a, long long k) {
  if (k >= p.m.grid[a].n || p.claim[a * p.m.cap + k] >= 0) return 0u;
  const unsigned int c = 1u + track_partners(p, a, k, [](unsigned int, long long) {});
  return c >= static_cast<unsigned int>(p.min_views) ? c : 0u;
}

// grid tiles: tile counts of step a, tracks at [0, tiles), observations at [tiles, 2 tiles)
__global__ void __launch_bounds__(COMPACT_THREADS) track_count_kernel(const TrackParams p, int a) {
  const long long base = static_cast<long long>(blockIdx.x) * COMPACT_TILE;
  unsigned int c[2] = {0u, 0u};
  for (int it = 0; it < COMPACT_ITERS; ++it) {
    const unsigned int m = track_members(p, a, base + it * COMPACT_THREADS + threadIdx.x);
    c[0] += m ? 1u : 0u;
    c[1] += m;
  }
  const unsigned int s = tile_sum<2>(c);
  if (threadIdx.x < 2) p.tile_count[threadIdx.x * p.m.tiles + blockIdx.x] = s;
}

// grid tiles, after the scan of step a's tile counts.  The minimum of one block lifts the 32-register cap ptxas otherwise
// picks for this kernel, and with it 16 bytes of spills (40 registers, none spilled).
__global__ void __launch_bounds__(COMPACT_THREADS, 1) track_write_kernel(const TrackParams p, int a) {
  const int tiles = p.m.tiles;
  const long long base = static_cast<long long>(blockIdx.x) * COMPACT_TILE;
  const unsigned long long* before = p.totals + 2 * (a & 1);
  const unsigned long long step_tracks = p.tile_offset[tiles];
  unsigned long long t_out = before[0] + p.tile_offset[blockIdx.x];
  unsigned long long o_out = before[1] + (p.tile_offset[tiles + blockIdx.x] - step_tracks);
  if (blockIdx.x == 0 && threadIdx.x == 0) {        // the other slot: nothing reads it during this step
    unsigned long long* after = p.totals + 2 * ((a + 1) & 1);
    after[0] = before[0] + step_tracks;
    after[1] = before[1] + (*p.scan_total - step_tracks);
  }
  for (int it = 0; it < COMPACT_ITERS; ++it) {
    const long long k = base + it * COMPACT_THREADS + threadIdx.x;
    const unsigned int m = track_members(p, a, k);
    const unsigned int v[2] = {m ? 1u : 0u, m};
    unsigned int rank[2], sum[2];
    chunk_sums<2>(v, rank, sum);
    if (m) {
      const int t = static_cast<int>(t_out + rank[0]);
      const long long o = static_cast<long long>(o_out + rank[1]);
      p.track_start[t] = static_cast<int>(o);
      p.obs[o] = static_cast<int>(a * p.m.cap + k);
      p.claim[a * p.m.cap + k] = t;
      int* const obs = p.obs + o + 1;
      int* const claim = p.claim;
      track_partners(p, a, k, [=](unsigned int i, long long node) {
        obs[i] = static_cast<int>(node);
        claim[node] = t;
      });
    }
    t_out += sum[0];
    o_out += sum[1];
  }
}

// one thread, after the last step: tracks, observations, the non-finite flag of the index
__global__ void track_counts_kernel(const TrackParams p, long long* counts) {
  const unsigned long long* t = p.totals + 2 * (p.m.V & 1);
  counts[0] = static_cast<long long>(t[0]);
  counts[1] = static_cast<long long>(t[1]);
  counts[2] = static_cast<long long>(*p.m.flag & 1u);
}

__device__ __forceinline__ bool track_claimed(const TrackParams& p, int v, long long k) {
  return k < p.m.grid[v].n && p.claim[v * p.m.cap + k] >= 0;
}

// grid (tiles, V): claimed nodes per tile
__global__ void __launch_bounds__(COMPACT_THREADS) track_claimed_kernel(const TrackParams p) {
  const int v = blockIdx.y;
  const long long base = static_cast<long long>(blockIdx.x) * COMPACT_TILE;
  unsigned int c[1] = {0u};
  for (int it = 0; it < COMPACT_ITERS; ++it) c[0] += track_claimed(p, v, base + it * COMPACT_THREADS + threadIdx.x) ? 1u : 0u;
  const unsigned int s = tile_sum<1>(c);
  if (threadIdx.x == 0) p.tile_count[v * p.m.tiles + blockIdx.x] = s;
}

struct TrackOut {
  const float* images;                // [V, 3, H, W]
  const float* extrinsic;             // [V, 3, 4] world -> camera
  const float* intrinsic;             // [V, 3, 3]
  int W;
  long long n;                        // tracks
  long long m;                        // observations
  double* points;                     // [n, 3]
  unsigned char* colors;              // [n, 3]
  double* error;                      // [n]
  long long* offsets;                 // [n + 1]
  int* view;                          // [m]
  long long* xy;                      // [m, 2]
  int* point2d;                       // [m]
  long long* view_offsets;            // [V + 1]
  int* view_track;                    // [m]
  long long* view_xy;                 // [m, 2]
};

// grid (tiles, V), after the scan of the claimed counts: view v's claimed nodes in kept-index (= row-major pixel) order
__global__ void __launch_bounds__(COMPACT_THREADS) track_view_kernel(const TrackParams p, const TrackOut o) {
  const int v = blockIdx.y;
  const long long base = static_cast<long long>(blockIdx.x) * COMPACT_TILE;
  const unsigned long long first = p.tile_offset[static_cast<long long>(v) * p.m.tiles];
  unsigned long long out = p.tile_offset[static_cast<long long>(v) * p.m.tiles + blockIdx.x];
  if (blockIdx.x == 0 && threadIdx.x == 0) {
    o.view_offsets[v] = static_cast<long long>(first);
    if (v == p.m.V - 1) o.view_offsets[p.m.V] = static_cast<long long>(*p.scan_total);
  }
  for (int it = 0; it < COMPACT_ITERS; ++it) {
    const long long k = base + it * COMPACT_THREADS + threadIdx.x;
    const bool keep[1] = {track_claimed(p, v, k)};
    unsigned int rank[1], sum[1];
    chunk_ranks<1>(keep, rank, sum);
    if (keep[0]) {
      const unsigned long long q = out + rank[0];
      const long long node = v * p.m.cap + k;
      const long long pix = __float_as_int(p.m.pts[node].w);
      o.view_track[q] = p.claim[node];
      o.view_xy[2 * q] = pix % o.W;
      o.view_xy[2 * q + 1] = pix / o.W;
      p.rank[node] = static_cast<int>(q - first);
    }
    out += sum[0];
  }
}

// The reprojection of point c through camera (E world -> camera [R | t] row-major [3, 4], K [3, 3]) against the observation
// (ox, oy) in COLMAP's pixel frame, every fp64 operation rounded on its own:
//   (X, Y, Z) = R c + t, each row ((r0 c0 + r1 c1) + r2 c2) + t;  du = (fx (X / Z) + (cx + 0.5)) - ox;  dv likewise.
// Returns Z <= 0 (the camera sees the point behind it).  T is the cameras' element type: fp32 for tracks, fp64 for the bundle
// adjuster; an fp32 camera widened to fp64 gives the same bits either way.
template <typename T>
__device__ __forceinline__ bool track_reproject(const T* E, const T* K, const double c[3], double ox, double oy, double X[3],
                                                double& du, double& dv) {
#pragma unroll
  for (int r = 0; r < 3; ++r)
    X[r] = __dadd_rn(__dadd_rn(__dadd_rn(__dmul_rn(static_cast<double>(E[4 * r]), c[0]),
                                         __dmul_rn(static_cast<double>(E[4 * r + 1]), c[1])),
                               __dmul_rn(static_cast<double>(E[4 * r + 2]), c[2])),
                     static_cast<double>(E[4 * r + 3]));
  const double u = __dadd_rn(__dmul_rn(static_cast<double>(K[0]), __ddiv_rn(X[0], X[2])), __dadd_rn(static_cast<double>(K[2]), 0.5));
  const double w = __dadd_rn(__dmul_rn(static_cast<double>(K[4]), __ddiv_rn(X[1], X[2])), __dadd_rn(static_cast<double>(K[5]), 0.5));
  du = __dsub_rn(u, ox);
  dv = __dsub_rn(w, oy);
  return X[2] <= 0.0;
}

// grid ceil(n / TRACK_POINT_THREADS), after track_view_kernel.  Position: the fp64 sum of the observations' points in
// observation order, divided once by their count.  Error: the mean over the observations of the distance sqrt(du^2 + dv^2)
// of track_reproject against the pixel centre (x + 0.5, y + 0.5), summed in observation order and divided once; +inf when
// some Z <= 0.
__global__ void __launch_bounds__(TRACK_POINT_THREADS) track_point_kernel(const TrackParams p, const TrackOut o) {
  const long long t = static_cast<long long>(blockIdx.x) * TRACK_POINT_THREADS + threadIdx.x;
  if (t >= o.n) return;
  const long long cap = p.m.cap;
  const long long b = p.track_start[t], e = t + 1 < o.n ? p.track_start[t + 1] : o.m;
  o.offsets[t] = b;
  if (t == o.n - 1) o.offsets[o.n] = o.m;
  double s[3] = {0.0, 0.0, 0.0};
  for (long long q = b; q < e; ++q) {
    const int node = p.obs[q];
    const int v = static_cast<int>(node / cap);
    const float4 x = p.m.pts[node];
    s[0] = __dadd_rn(s[0], static_cast<double>(x.x));
    s[1] = __dadd_rn(s[1], static_cast<double>(x.y));
    s[2] = __dadd_rn(s[2], static_cast<double>(x.z));
    const long long pix = __float_as_int(x.w);
    o.view[q] = v;
    o.xy[2 * q] = pix % o.W;
    o.xy[2 * q + 1] = pix / o.W;
    o.point2d[q] = p.rank[node];
  }
  const double cnt = static_cast<double>(e - b);
  const double c[3] = {__ddiv_rn(s[0], cnt), __ddiv_rn(s[1], cnt), __ddiv_rn(s[2], cnt)};
  o.points[3 * t] = c[0];
  o.points[3 * t + 1] = c[1];
  o.points[3 * t + 2] = c[2];
  const int anchor = p.obs[b];
  const uchar3 rgb = pixel_rgb(o.images, cap, (anchor / cap) * cap + __float_as_int(p.m.pts[anchor].w),
                               static_cast<int>(anchor / cap));
  o.colors[3 * t] = rgb.x;
  o.colors[3 * t + 1] = rgb.y;
  o.colors[3 * t + 2] = rgb.z;
  double err = 0.0;
  bool behind = false;
  for (long long q = b; q < e; ++q) {
    const int node = p.obs[q];
    const int v = static_cast<int>(node / cap);
    const long long pix = __float_as_int(p.m.pts[node].w);
    double X[3], du, dv;
    behind |= track_reproject(o.extrinsic + 12 * v, o.intrinsic + 9 * v, c, static_cast<double>(pix % o.W) + 0.5,
                              static_cast<double>(pix / o.W) + 0.5, X, du, dv);
    err = __dadd_rn(err, __dsqrt_rn(__dadd_rn(__dmul_rn(du, du), __dmul_rn(dv, dv))));
  }
  o.error[t] = behind ? __longlong_as_double(0x7ff0000000000000LL) : __ddiv_rn(err, cnt);
}

}  // namespace ovg
