// Model-free sky segmentation: the DUSt3R-family recipe of viz.py:357-393 (segment_sky), all views in one pass.
//   sky_open_kernel      per 32 x 32 tile: OpenCV's integer BGR2HSV and the colour test on the tile plus a 4-pixel halo, then
//                        the 5 x 5 binary opening (separable box min, then box max, outside the image = false) in shared
//                        memory; every opened pixel starts as its own label
//   sky_merge_kernel     8-connected union-find (Playne & Hawick, IEEE TPDS 2018): each pixel unites with the neighbours above
//                        and to its left that no other pixel unites it with; union by atomicMin, so a component's root is its
//                        smallest pixel index
//   sky_area_kernel      every label compressed to its root; the area of every root
//   sky_max_kernel       the largest area of every view
//   sky_select_kernel    sky = the pixels of the components with 2 area > the view's largest area, and conf * non-sky
// Labels are pixel indices i = (f H + y) W + x and never cross views.  The only atomics are integer atomicMin (the root a union
// settles on is the smallest index of the united set whatever the order) and atomicAdd / atomicMax of areas (a sum and a
// maximum of integers): every output is bit-identical from run to run.  The number of launches depends on nothing but the call.
#pragma once
#include <cuda_runtime.h>

namespace ovg {

constexpr int SKY_TILE = 32;                  // output pixels per tile side
constexpr int SKY_IN = SKY_TILE + 8;          // colour test of the tile and a 4-pixel halo: erosion and dilation take 2 each
constexpr int SKY_THREADS = 256;

struct SkyParams {
  const void* image;                // uint8 or fp32 elements: (f, y, x, c) at f view_stride + (y W + x) pixel_stride + c channel_stride
  int u8;
  long long view_stride, pixel_stride, channel_stride;
  int F, H, W, tiles_x;
  long long hw, n;                  // H W, F H W
  const float* conf;                // [n] or nullptr
  float* conf_out;                  // [n] conf * non-sky
  unsigned char* sky;               // [n]
  int* label;                       // [n] -1 = not in the opened mask, else a pixel of the same component (the root at the end)
  int* area;                        // [n] the area of a root
  int* view_max;                    // [F]
};

// Colour test of pixel (f, y, x): viz.py:362-375.  Channel 0 is read as B, as cv2.cvtColor(..., COLOR_BGR2HSV) does.
__device__ __forceinline__ unsigned char sky_color(const SkyParams& p, const int* sdiv, const int* hdiv, int f, int y, int x) {
  const long long e = f * p.view_stride + static_cast<long long>(y * p.W + x) * p.pixel_stride;
  int c[3];
  if (p.u8) {
    const unsigned char* s = static_cast<const unsigned char*>(p.image) + e;
#pragma unroll
    for (int k = 0; k < 3; ++k) c[k] = s[k * p.channel_stride];
  } else {                                          // np.uint8(255 * image.clip(0, 1)): an fp32 multiply, then truncation
    const float* s = static_cast<const float*>(p.image) + e;
#pragma unroll
    for (int k = 0; k < 3; ++k) c[k] = static_cast<int>(__fmul_rn(255.f, fminf(fmaxf(s[k * p.channel_stride], 0.f), 1.f)));
  }
  // OpenCV's 8-bit RGB2HSV with hsv_shift = 12, its division tables and round-half-up shifts; H in [0, 180)
  const int b = c[0], g = c[1], r = c[2];
  const int v = max(max(b, g), r), diff = v - min(min(b, g), r);
  const int s = (diff * sdiv[v] + (1 << 11)) >> 12;
  int h = v == r ? g - b : (v == g ? b - r + 2 * diff : r - g + 4 * diff);
  h = (h * hdiv[diff] + (1 << 11)) >> 12;
  if (h < 0) h += 180;
  return ((h <= 30 && v >= 100) || (s < 10 && v > 150) || (s < 30 && v > 180) || (s < 50 && v > 220)) ? 1 : 0;
}

// Block (tile, f).  scipy.ndimage.binary_opening(mask, ones((5, 5))): erosion then dilation, both with border_value 0.  A
// pixel outside the image is false in the colour test, so an eroded pixel outside the image (its own centre false) is too.
__global__ void __launch_bounds__(SKY_THREADS) sky_open_kernel(const SkyParams p) {
  __shared__ int sdiv[256], hdiv[256];
  __shared__ unsigned char m[SKY_IN][SKY_IN];             // colour test: row y0 - 4 + r, column x0 - 4 + c
  __shared__ unsigned char a[SKY_IN][SKY_IN - 4];         // 5-wide min of m: column x0 - 2 + c
  __shared__ unsigned char e[SKY_IN - 4][SKY_IN - 4];     // eroded: row y0 - 2 + r, column x0 - 2 + c
  __shared__ unsigned char d[SKY_IN - 4][SKY_TILE];       // 5-wide max of e: column x0 + c
  const int f = blockIdx.y;
  const int ty = blockIdx.x / p.tiles_x, tx = blockIdx.x - ty * p.tiles_x;
  const int y0 = ty * SKY_TILE, x0 = tx * SKY_TILE;
  {
    const int i = threadIdx.x;                              // saturate_cast<int>((255 << 12) / (1. i)), ((180 << 12) / (6. i))
    sdiv[i] = i ? __double2int_rn(static_cast<double>(255 << 12) / i) : 0;
    hdiv[i] = i ? __double2int_rn(static_cast<double>(180 << 12) / (6.0 * i)) : 0;
  }
  __syncthreads();
  for (int k = threadIdx.x; k < SKY_IN * SKY_IN; k += SKY_THREADS) {
    const int r = k / SKY_IN, c = k - r * SKY_IN, y = y0 - 4 + r, x = x0 - 4 + c;
    m[r][c] = (y >= 0 && y < p.H && x >= 0 && x < p.W) ? sky_color(p, sdiv, hdiv, f, y, x) : 0;
  }
  __syncthreads();
  for (int k = threadIdx.x; k < SKY_IN * (SKY_IN - 4); k += SKY_THREADS) {
    const int r = k / (SKY_IN - 4), c = k - r * (SKY_IN - 4);
    a[r][c] = m[r][c] & m[r][c + 1] & m[r][c + 2] & m[r][c + 3] & m[r][c + 4];
  }
  __syncthreads();
  for (int k = threadIdx.x; k < (SKY_IN - 4) * (SKY_IN - 4); k += SKY_THREADS) {
    const int r = k / (SKY_IN - 4), c = k - r * (SKY_IN - 4);
    e[r][c] = a[r][c] & a[r + 1][c] & a[r + 2][c] & a[r + 3][c] & a[r + 4][c];
  }
  __syncthreads();
  for (int k = threadIdx.x; k < (SKY_IN - 4) * SKY_TILE; k += SKY_THREADS) {
    const int r = k / SKY_TILE, c = k - r * SKY_TILE;
    d[r][c] = e[r][c] | e[r][c + 1] | e[r][c + 2] | e[r][c + 3] | e[r][c + 4];
  }
  __syncthreads();
  for (int k = threadIdx.x; k < SKY_TILE * SKY_TILE; k += SKY_THREADS) {
    const int r = k / SKY_TILE, c = k - r * SKY_TILE, y = y0 + r, x = x0 + c;
    if (y < p.H && x < p.W) {
      const long long i = f * p.hw + static_cast<long long>(y) * p.W + x;
      const bool on = d[r][c] | d[r + 1][c] | d[r + 2][c] | d[r + 3][c] | d[r + 4][c];
      p.label[i] = on ? static_cast<int>(i) : -1;
      p.area[i] = 0;
    }
  }
  if (blockIdx.x == 0 && threadIdx.x == 0) p.view_max[f] = 0;
}

// Labels are read through L2 (__ldcg): other SMs change them during the merge.  Every label points to a smaller (or the same)
// index of the same component; a root points to itself.
__device__ __forceinline__ int sky_find(int* L, int x) {
  int q = __ldcg(L + x);
  while (q != x) {
    const int g = __ldcg(L + q);
    if (g != q) atomicMin(L + x, g);                        // path splitting: x now points to its grandparent (or lower)
    x = q;
    q = g;
  }
  return x;
}

__device__ __forceinline__ void sky_union(int* L, int a, int b) {
  bool done;
  do {
    a = sky_find(L, a);
    b = sky_find(L, b);
    if (a < b) {
      const int old = atomicMin(L + b, a);
      done = old == b;                                      // b was still a root: it now hangs under a
      b = old;
    } else if (b < a) {
      const int old = atomicMin(L + a, b);
      done = old == a;
      a = old;
    } else {
      done = true;
    }
  } while (!done);
}

__device__ __forceinline__ bool sky_on(const int* L, long long j) { return __ldcg(L + j) >= 0; }   // the sign never changes

// 8-connectivity.  With N = (y-1, x) in the mask, N's own unions join it to NW (as its W), to NE (NE's W) and to W (W's NE):
// uniting with N alone suffices.  Without N, NW and NE are not neighbours of each other; W and NW are (W's N).
__global__ void __launch_bounds__(256) sky_merge_kernel(const SkyParams p) {
  const long long i = static_cast<long long>(blockIdx.x) * 256 + threadIdx.x;
  if (i >= p.n || !sky_on(p.label, i)) return;
  const long long q = i % p.hw;
  const int y = static_cast<int>(q / p.W), x = static_cast<int>(q - static_cast<long long>(y) * p.W);
  const int me = static_cast<int>(i);
  const long long w = i - 1;
  if (y > 0) {
    const long long n = i - p.W;
    if (sky_on(p.label, n)) {
      sky_union(p.label, me, static_cast<int>(n));
      return;
    }
    if (x + 1 < p.W && sky_on(p.label, n + 1)) sky_union(p.label, me, static_cast<int>(n + 1));
    if (x > 0 && sky_on(p.label, w)) sky_union(p.label, me, static_cast<int>(w));
    else if (x > 0 && sky_on(p.label, n - 1)) sky_union(p.label, me, static_cast<int>(n - 1));
  } else if (x > 0 && sky_on(p.label, w)) {
    sky_union(p.label, me, static_cast<int>(w));
  }
}

// Every label becomes its root; the lanes of a warp with the same root add their count at once.
__global__ void __launch_bounds__(256) sky_area_kernel(const SkyParams p) {
  const long long i = static_cast<long long>(blockIdx.x) * 256 + threadIdx.x;
  int root = -1;
  if (i < p.n) {
    root = __ldcg(p.label + i);
    if (root >= 0) {
      int up = __ldcg(p.label + root);
      while (up != root) {
        root = up;
        up = __ldcg(p.label + root);
      }
      p.label[i] = root;                                    // readers see the old label or the root: both lead to the root
    }
  }
  const unsigned same = __match_any_sync(0xffffffffu, root);
  if (root >= 0 && (threadIdx.x & 31) == __ffs(same) - 1) atomicAdd(p.area + root, __popc(same));
}

__global__ void __launch_bounds__(256) sky_max_kernel(const SkyParams p) {
  const long long i = static_cast<long long>(blockIdx.x) * 256 + threadIdx.x;
  if (i < p.n && p.label[i] == i) atomicMax(p.view_max + i / p.hw, p.area[i]);
}

// viz.py:381-390: the components taken in descending area while area > largest / 2, i.e. exactly those with 2 area > largest.
__global__ void __launch_bounds__(256) sky_select_kernel(const SkyParams p) {
  const long long i = static_cast<long long>(blockIdx.x) * 256 + threadIdx.x;
  if (i >= p.n) return;
  const int l = p.label[i];
  const bool sky = l >= 0 && 2LL * p.area[l] > p.view_max[i / p.hw];
  p.sky[i] = sky ? 1 : 0;
  if (p.conf) p.conf_out[i] = __fmul_rn(p.conf[i], sky ? 0.f : 1.f);
}

// conf * non-sky for a caller's mask (visual_util.py:186-188 with the mask file 255 = non-sky).
__global__ void __launch_bounds__(256) sky_mask_conf_kernel(const float* conf, const unsigned char* sky, long long n,
                                                            float* conf_out) {
  const long long i = static_cast<long long>(blockIdx.x) * 256 + threadIdx.x;
  if (i < n) conf_out[i] = __fmul_rn(conf[i], sky[i] ? 0.f : 1.f);
}

}  // namespace ovg
