// Triangle mesh of the predicted point maps: the DUSt3R-family recipe of viz.py:40-77 (pts3d_to_trimesh) and :80-89
// (cat_meshes), all views in one pass.
//   mesh_keep_kernel      the per-pixel keep bit (pixel_keep of the point cloud, or a caller mask alone)
//   mesh_count_kernel     per tile of a view: kept TL / BR triangles of the pixel quads and vertices used by a kept one
//   tile_scan_kernel      one scan over the three streams' tile counts, concatenated (compact.cuh)
//   mesh_totals_kernel    reference faces, used vertices, forward faces
//   mesh_faces_kernel     the reference layout: every kept triangle and its reversed copy, int64 indices, face colours
//   mesh_vertices_kernel  the GLB layout: used vertices in index order and the remap of their indices
//   mesh_indices_kernel   the GLB layout: the forward triangles through the remap, int32
// The quad at (y, x) of a view, y < H - 1 and x < W - 1, has the corners tl (y, x), tr (y, x + 1), bl (y + 1, x) and
// br (y + 1, x + 1); its TL triangle (tl, tr, bl) is kept when all three corners are, its BR triangle (tr, bl, br) likewise.
// A view's faces are the kept TL triangles, the same reversed, the kept BR triangles, the same reversed, each class in
// row-major quad order.  Every stream is compacted per view by tiles of COMPACT_TILE pixels as compact.cuh describes.
#pragma once
#include "post.cuh"

namespace ovg {

constexpr int MESH_STREAMS = 3;   // TL triangles, BR triangles, used vertices

struct MeshParams {
  const unsigned char* conf_mask;   // [n]
  const float* images;              // [F, 3, H, W] in [0, 1], or nullptr (keep = conf_mask; colours from `colors`)
  int black_bg, white_bg;
  const float* points;              // [n, 3]
  const void* colors;               // [n, 3] elements of color_bytes: the face colours when images is nullptr
  int color_bytes;
  int H, W;
  long long hw, n;                  // H * W, F * H * W
  int tpv, T;                       // tiles per view, F * tpv
  unsigned char* keep;              // [n]
  int* remap;                       // [n] rank of a used vertex among the used vertices
  unsigned int* tile_count;         // [3][T] tile counts of the three streams
  unsigned long long* tile_offset;  // [3 T + 1] exclusive scan over the streams concatenated, then the grand total
  long long* totals;                // [3] reference faces, used vertices, forward faces
  long long* faces;                 // [reference faces, 3]
  void* face_colors;                // [reference faces, 3]: uint8 from images, else elements of color_bytes
  float* positions;                 // [used, 3]
  unsigned char* vertex_colors;     // [used, 3]
  int* indices;                     // [forward faces, 3]
};

// The TL / BR triangle of the quad at (y, x) of the pixel i = (f H + y) W + x; false outside the quads.
__device__ __forceinline__ bool mesh_tl(const MeshParams& p, long long i, int y, int x) {
  return y >= 0 && x >= 0 && y < p.H - 1 && x < p.W - 1 && p.keep[i] && p.keep[i + 1] && p.keep[i + p.W];
}
__device__ __forceinline__ bool mesh_br(const MeshParams& p, long long i, int y, int x) {
  return y >= 0 && x >= 0 && y < p.H - 1 && x < p.W - 1 && p.keep[i + 1] && p.keep[i + p.W] && p.keep[i + p.W + 1];
}
// Vertex (y, x) is a corner of TL(y, x) as tl, TL(y, x-1) as tr, TL(y-1, x) as bl, BR(y, x-1) as tr, BR(y-1, x) as bl and
// BR(y-1, x-1) as br.
__device__ __forceinline__ bool mesh_used(const MeshParams& p, long long i, int y, int x) {
  const long long up = i - p.W;
  return mesh_tl(p, i, y, x) || mesh_tl(p, i - 1, y, x - 1) || mesh_tl(p, up, y - 1, x) || mesh_br(p, i - 1, y, x - 1) ||
         mesh_br(p, up, y - 1, x) || mesh_br(p, up - 1, y - 1, x - 1);
}

__global__ void __launch_bounds__(256) mesh_keep_kernel(const MeshParams p) {
  const long long i = static_cast<long long>(blockIdx.x) * 256 + threadIdx.x;
  if (i >= p.n) return;
  bool k;
  if (p.images) {
    int f;
    uchar3 rgb;
    k = pixel_keep(p.conf_mask, p.images, p.hw, p.black_bg, p.white_bg, i, f, rgb);
  } else {
    k = p.conf_mask[i] != 0;
  }
  p.keep[i] = k ? 1 : 0;
}

// Block (t, f): pixels [t COMPACT_TILE, (t + 1) COMPACT_TILE) of view f.
__global__ void __launch_bounds__(COMPACT_THREADS) mesh_count_kernel(const MeshParams p) {
  const int f = blockIdx.y;
  unsigned int c[MESH_STREAMS] = {0u, 0u, 0u};
  for (int it = 0; it < COMPACT_ITERS; ++it) {
    const long long q = static_cast<long long>(blockIdx.x) * COMPACT_TILE + it * COMPACT_THREADS + threadIdx.x;
    if (q < p.hw) {
      const int y = static_cast<int>(q / p.W), x = static_cast<int>(q - static_cast<long long>(y) * p.W);
      const long long i = f * p.hw + q;
      c[0] += mesh_tl(p, i, y, x);
      c[1] += mesh_br(p, i, y, x);
      c[2] += mesh_used(p, i, y, x);
    }
  }
  const unsigned int sum = tile_sum<MESH_STREAMS>(c);
  if (threadIdx.x < MESH_STREAMS) p.tile_count[threadIdx.x * p.T + f * p.tpv + blockIdx.x] = sum;
}

__global__ void mesh_totals_kernel(const MeshParams p) {
  if (threadIdx.x == 0) {
    const unsigned long long* o = p.tile_offset;
    const long long tl = static_cast<long long>(o[p.T] - o[0]), br = static_cast<long long>(o[2 * p.T] - o[p.T]);
    p.totals[0] = 2 * (tl + br);
    p.totals[1] = static_cast<long long>(o[3 * p.T] - o[2 * p.T]);
    p.totals[2] = tl + br;
  }
}

// Colour of pixel j (frame f) into element k of the face colours.
__device__ __forceinline__ void mesh_face_color(const MeshParams& p, long long j, int f, unsigned long long k) {
  if (p.images) {
    const uchar3 rgb = pixel_rgb(p.images, p.hw, j, f);
    unsigned char* d = static_cast<unsigned char*>(p.face_colors) + 3 * k;
    d[0] = rgb.x; d[1] = rgb.y; d[2] = rgb.z;
    return;
  }
  switch (p.color_bytes) {                          // gathered without arithmetic: the caller's dtype is kept
    case 1: { const unsigned char* s = static_cast<const unsigned char*>(p.colors) + 3 * j;
              unsigned char* d = static_cast<unsigned char*>(p.face_colors) + 3 * k;
              d[0] = s[0]; d[1] = s[1]; d[2] = s[2]; break; }
    case 2: { const unsigned short* s = static_cast<const unsigned short*>(p.colors) + 3 * j;
              unsigned short* d = static_cast<unsigned short*>(p.face_colors) + 3 * k;
              d[0] = s[0]; d[1] = s[1]; d[2] = s[2]; break; }
    case 4: { const unsigned int* s = static_cast<const unsigned int*>(p.colors) + 3 * j;
              unsigned int* d = static_cast<unsigned int*>(p.face_colors) + 3 * k;
              d[0] = s[0]; d[1] = s[1]; d[2] = s[2]; break; }
    default: { const unsigned long long* s = static_cast<const unsigned long long*>(p.colors) + 3 * j;
               unsigned long long* d = static_cast<unsigned long long*>(p.face_colors) + 3 * k;
               d[0] = s[0]; d[1] = s[1]; d[2] = s[2]; break; }
  }
}

__device__ __forceinline__ void mesh_face(const MeshParams& p, unsigned long long k, long long a, long long b, long long c) {
  long long* d = p.faces + 3 * k;
  d[0] = a; d[1] = b; d[2] = c;
}

// Where view f's triangles go: the view's first TL / BR ranks over the whole scene and its TL / BR counts.
struct MeshView {
  unsigned long long tl0, br0, c1, c3;
};
__device__ __forceinline__ MeshView mesh_view(const MeshParams& p, int f) {
  const unsigned long long* o = p.tile_offset;
  MeshView v;
  v.tl0 = o[f * p.tpv] - o[0];
  v.br0 = o[p.T + f * p.tpv] - o[p.T];
  v.c1 = o[(f + 1) * p.tpv] - o[f * p.tpv];                // (f + 1) tpv = T for the last view: the next stream's start
  v.c3 = o[p.T + (f + 1) * p.tpv] - o[p.T + f * p.tpv];
  return v;
}

// Reference layout (viz.py:53-74 per view, :80-89 across views): view f's faces start at 2 (TL + BR kept before f).
__global__ void __launch_bounds__(COMPACT_THREADS) mesh_faces_kernel(const MeshParams p) {
  const int f = blockIdx.y;
  const MeshView v = mesh_view(p, f);
  const unsigned long long base = 2 * (v.tl0 + v.br0);
  unsigned long long r_tl = p.tile_offset[f * p.tpv + blockIdx.x] - p.tile_offset[f * p.tpv];
  unsigned long long r_br = p.tile_offset[p.T + f * p.tpv + blockIdx.x] - p.tile_offset[p.T + f * p.tpv];
  for (int it = 0; it < COMPACT_ITERS; ++it) {
    const long long q = static_cast<long long>(blockIdx.x) * COMPACT_TILE + it * COMPACT_THREADS + threadIdx.x;
    const int y = static_cast<int>(q / p.W), x = static_cast<int>(q - static_cast<long long>(y) * p.W);
    const long long i = f * p.hw + q;
    const bool in = q < p.hw;
    const bool flag[2] = {in && mesh_tl(p, i, y, x), in && mesh_br(p, i, y, x)};
    unsigned int rank[2], sum[2];
    chunk_ranks<2>(flag, rank, sum);
    const long long tr = i + 1, bl = i + p.W, br = i + p.W + 1;
    if (flag[0]) {
      const unsigned long long k = base + r_tl + rank[0];
      mesh_face(p, k, i, tr, bl);
      mesh_face(p, k + v.c1, bl, tr, i);
      mesh_face_color(p, i, f, k);
      mesh_face_color(p, i, f, k + v.c1);
    }
    if (flag[1]) {
      const unsigned long long k = base + 2 * v.c1 + r_br + rank[1];
      mesh_face(p, k, tr, bl, br);
      mesh_face(p, k + v.c3, br, bl, tr);
      mesh_face_color(p, br, f, k);
      mesh_face_color(p, br, f, k + v.c3);
    }
    r_tl += sum[0];
    r_br += sum[1];
  }
}

// GLB layout, part 1: the used vertices in index order with their own pixel's colour, and remap[i] = the rank of vertex i.
__global__ void __launch_bounds__(COMPACT_THREADS) mesh_vertices_kernel(const MeshParams p) {
  const int f = blockIdx.y;
  unsigned long long r = p.tile_offset[2 * p.T + f * p.tpv + blockIdx.x] - p.tile_offset[2 * p.T];
  for (int it = 0; it < COMPACT_ITERS; ++it) {
    const long long q = static_cast<long long>(blockIdx.x) * COMPACT_TILE + it * COMPACT_THREADS + threadIdx.x;
    const int y = static_cast<int>(q / p.W), x = static_cast<int>(q - static_cast<long long>(y) * p.W);
    const long long i = f * p.hw + q;
    const bool flag[1] = {q < p.hw && mesh_used(p, i, y, x)};
    unsigned int rank[1], sum[1];
    chunk_ranks<1>(flag, rank, sum);
    if (flag[0]) {
      const unsigned long long u = r + rank[0];
      p.remap[i] = static_cast<int>(u);
      p.positions[3 * u] = p.points[3 * i];
      p.positions[3 * u + 1] = p.points[3 * i + 1];
      p.positions[3 * u + 2] = p.points[3 * i + 2];
      const uchar3 rgb = pixel_rgb(p.images, p.hw, i, f);
      p.vertex_colors[3 * u] = rgb.x;
      p.vertex_colors[3 * u + 1] = rgb.y;
      p.vertex_colors[3 * u + 2] = rgb.z;
    }
    r += sum[0];
  }
}

// GLB layout, part 2: the forward triangles (classes 1 and 3 of the reference layout, same order) through the remap.
__global__ void __launch_bounds__(COMPACT_THREADS) mesh_indices_kernel(const MeshParams p) {
  const int f = blockIdx.y;
  const MeshView v = mesh_view(p, f);
  const unsigned long long base = v.tl0 + v.br0;
  unsigned long long r_tl = p.tile_offset[f * p.tpv + blockIdx.x] - p.tile_offset[f * p.tpv];
  unsigned long long r_br = p.tile_offset[p.T + f * p.tpv + blockIdx.x] - p.tile_offset[p.T + f * p.tpv];
  for (int it = 0; it < COMPACT_ITERS; ++it) {
    const long long q = static_cast<long long>(blockIdx.x) * COMPACT_TILE + it * COMPACT_THREADS + threadIdx.x;
    const int y = static_cast<int>(q / p.W), x = static_cast<int>(q - static_cast<long long>(y) * p.W);
    const long long i = f * p.hw + q;
    const bool in = q < p.hw;
    const bool flag[2] = {in && mesh_tl(p, i, y, x), in && mesh_br(p, i, y, x)};
    unsigned int rank[2], sum[2];
    chunk_ranks<2>(flag, rank, sum);
    if (flag[0] || flag[1]) {
      const int tr = p.remap[i + 1], bl = p.remap[i + p.W];
      if (flag[0]) {
        int* d = p.indices + 3 * (base + r_tl + rank[0]);
        d[0] = p.remap[i]; d[1] = tr; d[2] = bl;
      }
      if (flag[1]) {
        int* d = p.indices + 3 * (base + v.c1 + r_br + rank[1]);
        d[0] = tr; d[1] = bl; d[2] = p.remap[i + p.W + 1];
      }
    }
    r_tl += sum[0];
    r_br += sum[1];
  }
}

}  // namespace ovg
