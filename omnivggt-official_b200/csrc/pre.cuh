// GPU input pipeline (SURVEY.md section 8f rank 4): what reference visual_util.py:719-841 (load_images_and_cameras) does per
// view on the host with Pillow / OpenCV / numpy, as HBM-bound kernels on decoded pixels:
//   resize_h_u8 / resize_v_u8_f32   Image.resize(..., BICUBIC) -- Pillow's two-pass fixed-point convolution (Resample.c:
//                                   22-bit taps, rounding and clip to uint8 after EACH pass), bit-exact -- then the centre crop
//                                   and ToTensor (uint8 / 255, CHW fp32)                             visual_util.py:731-751
//                                   placed in a larger frame padded with a constant, for utils/load_fn.py's pad mode and
//                                   mixed-size lists (white padding)                                 load_fn.py:85-136
//   depth_nearest                   validity filter + cv2.resize(..., INTER_NEAREST) + crop + mask   visual_util.py:768-791
//   camera_prepare                  intrinsics rescale / crop shift, camera-to-world -> world-to-camera   :807-820
// The per-axis tap tables and nearest-neighbour index tables are a few KB, computed once per image size on the host
// (preprocess.py, same arithmetic as the libraries) and cached on the device.
#pragma once
#include "ptx.cuh"

namespace ovg {

constexpr int PRE_PRECISION_BITS = 22;

__device__ __forceinline__ int pre_clip8(int v) {
  v >>= PRE_PRECISION_BITS;
  return v < 0 ? 0 : (v > 255 ? 255 : v);
}

struct ResizeParams {
  const uint8_t* src;   // horizontal: [h, w, 3]; vertical: [h, nw, 3]
  uint8_t* dst_u8;      // horizontal: [h, nw, 3]
  float* dst_f32;       // vertical: [3, fh, nw]
  const int* kmin;      // [n_out] first source index
  const int* kcnt;      // [n_out] number of taps
  const int* kk;        // [n_out, ksize] fixed-point taps
  int ksize;
  int h, w, nw, crop, fh;
  int identity;         // this axis keeps its size: Pillow skips the pass
  int out_h, out_w;     // vertical: the output frame [3, out_h, out_w] ...
  int off_y, off_x;     // ... holds the [fh, nw] image at (off_y, off_x) ...
  float fill;           // ... and this value everywhere else (load_fn.py's white padding)
};

__global__ void __launch_bounds__(128) resize_h_u8_kernel(const ResizeParams p) {
  const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y;
  if (x >= p.nw) return;
  const uint8_t* row = p.src + static_cast<long long>(y) * p.w * 3;
  const int x0 = p.kmin[x], n = p.kcnt[x];
  const int* k = p.kk + static_cast<long long>(x) * p.ksize;
  int s0 = 1 << (PRE_PRECISION_BITS - 1), s1 = s0, s2 = s0;
  for (int t = 0; t < n; ++t) {
    const int kv = k[t];
    const uint8_t* px = row + (x0 + t) * 3;
    s0 += px[0] * kv;
    s1 += px[1] * kv;
    s2 += px[2] * kv;
  }
  uint8_t* o = p.dst_u8 + (static_cast<long long>(y) * p.nw + x) * 3;
  o[0] = static_cast<uint8_t>(pre_clip8(s0));
  o[1] = static_cast<uint8_t>(pre_clip8(s1));
  o[2] = static_cast<uint8_t>(pre_clip8(s2));
}

// vertical pass over the (already horizontally resized) rows, only for the rows that survive the centre crop; one thread per
// pixel of the output frame, so every output float is written exactly once (image pixels and padding alike)
__global__ void __launch_bounds__(128) resize_v_u8_f32_kernel(const ResizeParams p) {
  const int xo = blockIdx.x * blockDim.x + threadIdx.x, yo = blockIdx.y;
  if (xo >= p.out_w) return;
  const int x = xo - p.off_x, yi = yo - p.off_y;
  float f0 = p.fill, f1 = p.fill, f2 = p.fill;
  if (x >= 0 && x < p.nw && yi >= 0 && yi < p.fh) {
    const int y = yi + p.crop;
    int v0, v1, v2;
    if (p.identity) {
      const uint8_t* px = p.src + (static_cast<long long>(y) * p.nw + x) * 3;
      v0 = px[0]; v1 = px[1]; v2 = px[2];
    } else {
      const int y0 = p.kmin[y], n = p.kcnt[y];
      const int* k = p.kk + static_cast<long long>(y) * p.ksize;
      int s0 = 1 << (PRE_PRECISION_BITS - 1), s1 = s0, s2 = s0;
      for (int t = 0; t < n; ++t) {
        const int kv = k[t];
        const uint8_t* px = p.src + (static_cast<long long>(y0 + t) * p.nw + x) * 3;
        s0 += px[0] * kv;
        s1 += px[1] * kv;
        s2 += px[2] * kv;
      }
      v0 = pre_clip8(s0); v1 = pre_clip8(s1); v2 = pre_clip8(s2);
    }
    f0 = static_cast<float>(v0) / 255.0f;               // ToTensor: uint8 -> float32, div(255)
    f1 = static_cast<float>(v1) / 255.0f;
    f2 = static_cast<float>(v2) / 255.0f;
  }
  const long long plane = static_cast<long long>(p.out_h) * p.out_w;
  float* o = p.dst_f32 + static_cast<long long>(yo) * p.out_w + xo;
  o[0] = f0;
  o[plane] = f1;
  o[2 * plane] = f2;
}

struct DepthNearestParams {
  const float* src;              // element (r, c) at src[r * row_stride + c * col_stride] (a transposed view swaps the strides)
  long long row_stride, col_stride;
  const int* sy;                 // [nh] source row of every resized row
  const int* sx;                 // [nw] source column
  float* depth;                  // [fh, nw]
  float* mask;                   // [fh, nw]
  int crop, fh, nw;
  float max_depth;
};

__global__ void __launch_bounds__(256) depth_nearest_kernel(const DepthNearestParams p) {
  const int x = blockIdx.x * blockDim.x + threadIdx.x, yo = blockIdx.y;
  if (x >= p.nw) return;
  float d = p.src[p.sy[yo + p.crop] * p.row_stride + p.sx[x] * p.col_stride];
  if (!isfinite(d) || d > p.max_depth || d < 1e-5f) d = 0.f;      // visual_util.py:768,:776-777
  const long long o = static_cast<long long>(yo) * p.nw + x;
  p.depth[o] = d;
  p.mask[o] = d > 1e-5f ? 1.0f : 0.0f;
}

struct CameraPrepParams {
  const float* c2w;      // [K, 3, 4] camera-to-world
  const float* kin;      // [K, 3, 3]
  const float* geom;     // [K, 3] = scale_x, scale_y, crop_y (crop_y < 0: no crop shift)
  const int* has;        // [K] 1: camera given; 0: zero placeholders (visual_util.py:821-824)
  float* w2c;            // [K, 3, 4]
  float* kout;           // [K, 3, 3]
  int K;
};

__global__ void camera_prepare_kernel(const CameraPrepParams p) {
  const int k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= p.K) return;
  float* e = p.w2c + k * 12;
  float* m = p.kout + k * 9;
  if (!p.has[k]) {
    for (int i = 0; i < 12; ++i) e[i] = 0.f;
    for (int i = 0; i < 9; ++i) m[i] = 0.f;
    return;
  }
  const float* c = p.c2w + k * 12;
  for (int a = 0; a < 3; ++a) {        // [R | t]^-1 = [R^T | -R^T t]                       utils/geometry.py:269-318
    e[a * 4 + 0] = c[0 * 4 + a];
    e[a * 4 + 1] = c[1 * 4 + a];
    e[a * 4 + 2] = c[2 * 4 + a];
    e[a * 4 + 3] = -(c[0 * 4 + a] * c[3] + c[1 * 4 + a] * c[7] + c[2 * 4 + a] * c[11]);
  }
  const float sx = p.geom[k * 3 + 0], sy = p.geom[k * 3 + 1], crop = p.geom[k * 3 + 2];
  for (int i = 0; i < 9; ++i) m[i] = p.kin[k * 9 + i];
  m[0] *= sx; m[4] *= sy; m[2] *= sx; m[5] *= sy;
  if (crop >= 0.f) m[5] -= crop;
}

}  // namespace ovg
